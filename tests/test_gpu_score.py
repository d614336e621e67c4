"""Scoring (rwkv_b200_score, rwkv_b200_batch_score_ragged, rwkv_b200_score_logits): the log-probability of a caller-given target at
every position, computed on the device. The kernel is checked against float64; whole models bit for bit against the logits rwkv_eval
gives token by token wherever the head runs as the GEMV, and within the tensor-core bars where it runs on the tensor cores."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.special

from conftest import LONG_PROMPT, ROOT, VERSIONS, model_path

pytestmark = pytest.mark.gpu
P_F, P_U, P_U8 = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint8)
NO = 0xFFFFFFFF
SENTINEL = np.float32(-12345.5)
ERR_ARGS, ERR_CTX, ERR_UNSUPPORTED = 1 << 8, 6 << 8, 9   # include/rwkv.h


def u32(a):
    return np.ascontiguousarray(a, np.uint32)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8).tobytes()


def lp64(logits, targets):
    """float64 log_softmax of the float32 logits at the targets."""
    ls = scipy.special.log_softmax(logits.astype(np.float64), axis=1)
    return ls[np.arange(len(targets)), np.minimum(targets, logits.shape[1] - 1)]


def score_logits(lib, logits, targets):
    logits = np.ascontiguousarray(logits, np.float32)
    t = u32(targets)
    lp, g = np.full(len(t), SENTINEL, np.float32), np.full(len(t), 7, np.uint8)
    assert lib.library.rwkv_b200_score_logits(logits.ctypes.data_as(P_F), logits.shape[0], logits.shape[1], t.ctypes.data_as(P_U),
                                              lp.ctypes.data_as(P_F), g.ctypes.data_as(P_U8)), lib.rwkv_get_last_error(None)
    return lp, g


# ---- the kernel against float64 -----------------------------------------------------------------------------------------------

# |lp - lp64| <= 1e-6 (1 + |lp64|): expf is within 2 ulp (2.4e-7 relative), so the double sum of the exponentials and its log are off by
# at most ~2.4e-7 absolute; z_t - max is one float rounding (6e-8 |z_t - max|) and the result one more (6e-8 |lp|). Their sum stays
# below 1e-6 (1 + |lp|) with room for the log's own error.
def check_rows(lp, g, logits, targets):
    want = lp64(logits, targets)
    for r, t in enumerate(targets):
        if t == NO:
            assert lp[r] == SENTINEL and g[r] == 7, r
            continue
        row = logits[r]
        if np.isnan(row).any() or np.isposinf(row).any() or not np.isfinite(row).any():
            assert np.isnan(lp[r]) and g[r] == 0, r
            continue
        if np.isneginf(want[r]):
            assert np.isneginf(lp[r]), r
        else:
            assert abs(float(lp[r]) - want[r]) <= 1e-6 * (1 + abs(want[r])), (r, float(lp[r]), want[r])
        assert g[r] == int(np.argmax(row) == t), (r, g[r])


@pytest.mark.parametrize("V", [1, 7, 50277, 65536])
def test_score_kernel_against_float64(lib, V):
    rng = np.random.default_rng(V)
    rows = [rng.standard_normal(V) * 3, rng.standard_normal(V) * 30]
    with_inf = rng.standard_normal(V)
    with_inf[rng.integers(0, V, max(1, V // 3))] = -np.inf
    with_inf[0] = 1.0
    rows += [with_inf, np.full(V, 0.25)]
    tie = rng.standard_normal(V)
    tie[V // 2] = tie[V - 1] = 9.0
    rows += [tie, tie]
    rows += [rng.uniform(-1e4, 0, V)]                        # a spread of 1e4
    bad_nan, bad_inf, all_ninf = rng.standard_normal(V), rng.standard_normal(V), np.full(V, -np.inf)
    bad_nan[V // 3] = np.nan
    bad_inf[V - 1] = np.inf
    rows += [bad_nan, bad_inf, all_ninf, rng.standard_normal(V)]
    logits = np.stack(rows).astype(np.float32)
    targets = list(rng.integers(0, V, len(rows)))
    targets[3] = 0                                           # all equal: the first index is the greedy one
    targets[4], targets[5] = V - 1, V // 2                   # a tie: the later index is not greedy, the earlier is
    targets[6] = int(np.argmin(logits[6]))
    targets[-1] = NO
    if V > 1:
        targets[2] = int(np.flatnonzero(np.isneginf(logits[2]))[0])     # a -inf target
    lp, g = score_logits(lib, logits, targets)
    check_rows(lp, g, logits, targets)


def test_score_kernel_rows_without_target_keep_their_bytes(lib):
    logits = np.random.default_rng(1).standard_normal((5, 300)).astype(np.float32)
    lp, g = score_logits(lib, logits, [NO, 3, NO, NO, 299])
    assert (lp[[0, 2, 3]] == SENTINEL).all() and (g[[0, 2, 3]] == 7).all()
    check_rows(lp, g, logits, [NO, 3, NO, NO, 299])


# ---- whole models -----------------------------------------------------------------------------------------------------------

class Ctx:
    def __init__(self, lib, path, tensor_cores=True):
        self.lib, self.L = lib, lib.library
        self.c = lib.rwkv_init_from_file(path, 1, 0)
        self.ptr = self.c.ptr
        self.L.rwkv_b200_set_tensor_cores(self.ptr, tensor_cores)
        self.n_state, self.V = lib.rwkv_get_state_buffer_element_count(self.c), lib.rwkv_get_logits_buffer_element_count(self.c)

    def fresh(self):
        assert self.L.rwkv_b200_state_load(self.ptr, None)

    def score(self, tokens, targets, lp=None, g=None):
        n = len(tokens)
        lp = np.full(n, SENTINEL, np.float32) if lp is None else lp
        g = np.full(n, 7, np.uint8) if g is None else g
        ok = self.L.rwkv_b200_score(self.ptr, u32(tokens).ctypes.data_as(P_U), u32(targets).ctypes.data_as(P_U), n,
                                    lp.ctypes.data_as(P_F), g.ctypes.data_as(P_U8))
        assert ok, self.L.rwkv_get_last_error(self.ptr)
        return lp, g

    def eval_resident(self, tokens, want=True):
        assert self.L.rwkv_b200_eval_resident(self.ptr, u32(tokens).ctypes.data_as(P_U), len(tokens), want, None)

    def state(self):
        s = np.zeros(self.n_state, np.float32)
        assert self.L.rwkv_b200_state_store(self.ptr, s.ctypes.data_as(P_F))
        return s

    def logits(self):
        lg = np.zeros(self.V, np.float32)
        assert self.L.rwkv_b200_stage_logits(self.ptr, lg.ctypes.data_as(P_F), None)
        return lg

    def serial(self, tokens):
        """Logits after every token through rwkv_eval, one token at a time from a fresh state."""
        st, lg, out = np.zeros(self.n_state, np.float32), np.zeros(self.V, np.float32), []
        for i, t in enumerate(tokens):
            assert self.L.rwkv_eval(self.ptr, t, None if i == 0 else st.ctypes.data_as(P_F), st.ctypes.data_as(P_F), lg.ctypes.data_as(P_F))
            out.append(lg.copy())
        return np.stack(out), st

    def free(self):
        self.lib.rwkv_free(self.c)


def text_targets(tokens, V, drop=(4, 17)):
    t = list(tokens[1:]) + [NO]
    for i in drop:
        if i < len(t):
            t[i] = NO
    return [x % V if x != NO else NO for x in t]


def score_in_calls(ctx, tokens, targets, splits):
    lp, g = np.full(len(tokens), SENTINEL, np.float32), np.full(len(tokens), 7, np.uint8)
    ctx.fresh()
    off = 0
    for n in splits:
        a, b = ctx.score(tokens[off:off + n], targets[off:off + n])
        lp[off:off + n], g[off:off + n] = a, b
        off += n
    assert off == len(tokens)
    return lp, g


@pytest.mark.parametrize("ver", VERSIONS)
@pytest.mark.parametrize("fmt", ["FP32", "FP16", "Q5_1"])
def test_score_equals_serial_logits_bitwise(lib, ver, fmt):
    """The GEMV head gives each column the bits of rwkv_eval token by token, for any split of the tokens into calls: tensor cores
    off, or every pass below 32 tokens."""
    for tensor_cores, splits in [(False, [70]), (False, [5, 40, 25]), (True, [31, 1, 20, 18])]:
        ctx = Ctx(lib, model_path(ver, fmt), tensor_cores)
        try:
            toks = [t % ctx.V for t in LONG_PROMPT]
            targets = text_targets(toks, ctx.V)
            ref, _ = ctx.serial(toks)
            want_lp, want_g = score_logits(lib, ref, targets)
            lp, g = score_in_calls(ctx, toks, targets, splits)
            assert bits(lp) == bits(want_lp) and bits(g) == bits(want_g), (tensor_cores, splits)
            assert bits(ctx.logits()) == bits(ref[-1])
        finally:
            ctx.free()


@pytest.mark.parametrize("ver", VERSIONS)
@pytest.mark.parametrize("fmt", ["FP16", "Q5_1"])
def test_score_leaves_the_state_of_eval_resident(lib, ver, fmt):
    """With tensor cores on (passes of >= 32 tokens take the tensor-core head): the state is the bytes eval_resident leaves."""
    ctx = Ctx(lib, model_path(ver, fmt), True)
    try:
        toks = [t % ctx.V for t in LONG_PROMPT]
        ctx.fresh()
        ctx.eval_resident(toks[:7])
        start = ctx.state()
        ctx.eval_resident(toks[7:])
        want = ctx.state()
        assert ctx.L.rwkv_b200_state_load(ctx.ptr, start.ctypes.data_as(P_F))
        ctx.score(toks[7:], text_targets(toks[7:], ctx.V))
        assert bits(ctx.state()) == bits(want)
    finally:
        ctx.free()


def traced_names(ctx):
    N = 1024
    st, en = (ctypes.c_double * N)(), (ctypes.c_double * N)()
    names = ctypes.create_string_buffer(32 * N)
    n = ctx.L.rwkv_b200_trace_read(ctx.ptr, st, en, ctypes.cast(names, ctypes.c_void_p), N)
    return [names.raw[32 * i:32 * i + 32].split(b"\0")[0].decode() for i in range(n)]


def synthetic(tmp_path, preset, fmt):
    import synthetic_model as sm
    path = str(tmp_path / f"{preset}-{fmt}.bin")
    sm.write_direct(path, preset, fmt, seed=11)
    return path


@pytest.mark.parametrize("preset,fmt", [("rwkv6-small", "Q5_1"), ("rwkv7-small", "FP16"), ("rwkv5-small", "Q4_0"), ("rwkv4-169m", "Q5_1")])
def test_score_on_the_tensor_cores(lib, tmp_path, preset, fmt):
    """Passes of 32..256 tokens: the head runs as layer_norm_columns + gemm_tc + score (trace names), and every log-probability is
    within twice the tensor-core logits bar of float64 log_softmax over rwkv_eval's logits with tensor cores off (an error of the
    log-probability is at most that of z_t plus that of logsumexp)."""
    import synthetic_model as sm
    bar = 2 * (2e-2 if fmt == "FP16" else 1.5e-1)
    path = synthetic(tmp_path, preset, fmt)
    ref_ctx, ctx = Ctx(lib, path, False), Ctx(lib, path, True)
    try:
        n = 300 if preset != "rwkv4-169m" else 64
        toks = sm.synthetic_tokens(n, ctx.V)
        targets = text_targets(toks, ctx.V)
        ref, _ = ref_ctx.serial(toks)
        want = lp64(ref, np.array([t if t != NO else 0 for t in targets]))
        splits = [256, n - 256] if n > 256 else [32, n - 32]
        ctx.fresh()
        assert ctx.L.rwkv_b200_trace_enable(ctx.ptr)
        a, ga = ctx.score(toks[:splits[0]], targets[:splits[0]])
        names = traced_names(ctx)
        ctx.L.rwkv_b200_trace_disable(ctx.ptr)
        b, gb = ctx.score(toks[splits[0]:], targets[splits[0]:])
        lp, g = np.concatenate([a, b]), np.concatenate([ga, gb])
        assert names[-4:] == ["layer_norm_columns", "convert_f16", "gemm_tc", "score"], names[-6:]
        has = np.array([t != NO for t in targets])
        err = np.abs(lp[has].astype(np.float64) - want[has])
        assert np.isfinite(lp[has]).all() and err.max() <= bar, (preset, fmt, err.max())
        assert (lp[~has] == SENTINEL).all() and (g[~has] == 7).all()
    finally:
        ref_ctx.free()
        ctx.free()


# ---- against the reference ----------------------------------------------------------------------------------------------------

def reference_logits(path, tokens):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import ref_lib
    try:
        ref = ref_lib.load_reference_library()
    except (FileNotFoundError, OSError):
        pytest.skip("oracle/_ref is not built")
    ref.rwkv_set_print_errors(None, False)
    ctx = ref.rwkv_init_from_file(path.encode(), 2, 0)
    assert ctx
    n_state, V = ref.rwkv_get_state_len(ctx), ref.rwkv_get_logits_len(ctx)
    st, lg, out = np.zeros(n_state, np.float32), np.zeros(V, np.float32), []
    PF = ref_lib.P_FLOAT
    for i, t in enumerate(tokens):
        assert ref.rwkv_eval(ctx, t, None if i == 0 else st.ctypes.data_as(PF), st.ctypes.data_as(PF), lg.ctypes.data_as(PF))
        out.append(lg.copy())
    ref.rwkv_free(ctx)
    return np.stack(out)


@pytest.mark.parametrize("ver", VERSIONS)
@pytest.mark.parametrize("fmt", ["FP32", "Q5_1"])
def test_score_against_the_reference(lib, ver, fmt):
    """Per-position cross entropy of the 70-token prompt as measure_pexplexity.py computes it from the reference's logits: within twice
    the end-to-end logits bars of the long prompt (1e-3 FP32, 1.5e-1 quantised), and so is the perplexity tools/perplexity.py reports.
    Tensor cores off: the per-token path those bars were set for (the tensor-core head has its own bars against float64 above)."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import perplexity
    path = model_path(ver, fmt)
    toks = list(LONG_PROMPT)
    ref = reference_logits(path, toks[:-1]).astype(np.float64)
    want = -scipy.special.log_softmax(ref, axis=1)[np.arange(len(toks) - 1), toks[1:]]
    bar = 2 * (1e-3 if fmt == "FP32" else 1.5e-1)
    ctx = Ctx(lib, path, False)
    try:
        losses = perplexity.score_losses(lib, ctx.c, toks)
        assert np.abs(losses - want).max() <= bar, np.abs(losses - want).max()
        for ignore in (0, 10):
            loss, ppl = perplexity.average(losses, ignore)
            keep = [i for i in range(len(want)) if ignore == 0 or i + 1 >= ignore]
            assert abs(loss - want[keep].mean()) <= bar and abs(ppl / np.exp(want[keep].mean()) - 1) <= np.expm1(bar)
    finally:
        ctx.free()


def test_perplexity_tool_runs(lib, tmp_path):
    ids = tmp_path / "ids.txt"
    ids.write_text(" ".join(map(str, LONG_PROMPT * 5)))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "perplexity.py"), model_path("6v0-3m", "Q5_1"), str(ids), "3"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "perplexity" in r.stdout.splitlines()[-1] and "skipped 3 tokens" in r.stdout.splitlines()[-1], r.stdout[-500:]


# ---- ragged batch -------------------------------------------------------------------------------------------------------------

class Batch:
    def __init__(self, ctx, n_seq, tensor_cores):
        self.ctx, self.L, self.n = ctx, ctx.L, n_seq
        self.ptr = ctypes.c_void_p(self.L.rwkv_b200_batch_create(ctx.ptr, n_seq))
        assert self.ptr
        self.L.rwkv_b200_set_tensor_cores(self.ptr, tensor_cores)

    def set_state(self, b, st):
        assert self.L.rwkv_b200_batch_set_state(self.ptr, b, None if st is None else st.ctypes.data_as(P_F))

    def state(self, b):
        s = np.zeros(self.ctx.n_state, np.float32)
        assert self.L.rwkv_b200_batch_get_state(self.ptr, b, s.ctypes.data_as(P_F))
        return s

    def logits(self, b):
        lg = np.zeros(self.ctx.V, np.float32)
        assert self.L.rwkv_b200_batch_get_logits(self.ptr, b, lg.ctypes.data_as(P_F))
        return lg

    def score(self, tokens, counts, targets):
        n = len(tokens)
        lp, g = np.full(n, SENTINEL, np.float32), np.full(n, 7, np.uint8)
        ok = self.L.rwkv_b200_batch_score_ragged(self.ptr, u32(tokens).ctypes.data_as(P_U), u32(counts).ctypes.data_as(P_U),
                                                 u32(targets).ctypes.data_as(P_U), lp.ctypes.data_as(P_F), g.ctypes.data_as(P_U8))
        assert ok, self.L.rwkv_get_last_error(self.ptr)
        return lp, g

    def free(self):
        self.L.rwkv_free(self.ptr)


def ragged_case(lib, path, counts, tensor_cores, exact, bar=None):
    """k sequences from one prefix state score k continuations in one ragged pass; each equals rwkv_b200_score alone from that state.
    Idle sequences keep their state and logits column, and batch generation afterwards matches eval_ragged with logits."""
    ctx = Ctx(lib, path, tensor_cores)
    B = len(counts)
    bt = Batch(ctx, B, tensor_cores)
    twin = Batch(ctx, B, tensor_cores)
    try:
        prefix = [t % ctx.V for t in LONG_PROMPT[:9]]
        ctx.fresh()
        ctx.eval_resident(prefix)
        pre = ctx.state()
        for b in range(B):
            bt.set_state(b, pre)
            twin.set_state(b, pre)
        warm = [prefix[-1]] * B
        assert bt.L.rwkv_b200_batch_eval(bt.ptr, u32(warm).ctypes.data_as(P_U), True)
        assert twin.L.rwkv_b200_batch_eval(twin.ptr, u32(warm).ctypes.data_as(P_U), True)
        before = [(bt.state(b), bt.logits(b)) for b in range(B)]
        conts = [[(LONG_PROMPT[(i + 7 * b) % 70] + 3 * b) % ctx.V for i in range(counts[b])] for b in range(B)]
        toks = [t for c in conts for t in c]
        targets = [t for c in conts for t in text_targets(c, ctx.V, drop=(2,))]
        lp, g = bt.score(toks, counts, targets)
        assert bt.L.rwkv_b200_batch_eval_ragged(twin.ptr, u32(toks).ctypes.data_as(P_U), u32(counts).ctypes.data_as(P_U), True)
        off = 0
        for b in range(B):
            n = counts[b]
            if n == 0:
                assert bits(bt.state(b)) == bits(before[b][0]) and bits(bt.logits(b)) == bits(before[b][1]), b
                continue
            assert ctx.L.rwkv_b200_state_load(ctx.ptr, before[b][0].ctypes.data_as(P_F))
            a, ga = ctx.score(conts[b], targets[off:off + n])
            if exact:
                assert bits(a) == bits(lp[off:off + n]) and bits(ga) == bits(g[off:off + n]), b
                assert bits(bt.state(b)) == bits(ctx.state()) and bits(bt.logits(b)) == bits(ctx.logits()), b
            else:
                has = np.array([t != NO for t in targets[off:off + n]])
                assert np.abs(a[has] - lp[off:off + n][has]).max(initial=0.0) <= bar, b
                assert (lp[off:off + n][~has] == SENTINEL).all()
            off += n
        # generation follows as it follows a ragged pass with logits
        L = bt.L
        mt, temp, top = u32([4] * B), np.full(B, 0.8, np.float32), np.full(B, 0.9, np.float32)
        zeros = np.zeros(B, np.float32)
        u = np.random.default_rng(5).random((B, 4))
        outs = []
        for x in (bt, twin):
            tk, ng = np.zeros((B, 4), np.uint32), np.zeros(B, np.uint32)
            assert L.rwkv_b200_batch_generate(x.ptr, mt.ctypes.data_as(P_U), temp.ctypes.data_as(P_F), top.ctypes.data_as(P_F),
                                              zeros.ctypes.data_as(P_F), zeros.ctypes.data_as(P_F), None,
                                              u.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), None, 0, tk.ctypes.data_as(P_U), ng.ctypes.data_as(P_U))
            outs.append((tk, ng))
        if exact:
            assert bits(outs[0][0]) == bits(outs[1][0]) and bits(outs[0][1]) == bits(outs[1][1])
    finally:
        bt.free()
        twin.free()
        ctx.free()


@pytest.mark.parametrize("ver", VERSIONS)
def test_ragged_score_equals_single_bitwise(lib, ver):
    ragged_case(lib, model_path(ver, "Q5_1"), [3, 0, 5, 1, 0, 6], tensor_cores=True, exact=True)       # sum 15 < 16
    ragged_case(lib, model_path(ver, "FP32"), [30, 0, 40, 2], tensor_cores=False, exact=True)


def test_ragged_score_on_the_tensor_cores(lib, tmp_path):
    path = synthetic(tmp_path, "rwkv6-small", "Q5_1")
    ragged_case(lib, path, [40, 1, 0, 33, 20], tensor_cores=True, exact=False, bar=2 * 1.5e-1)


# ---- follow-on calls ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fmt", ["FP32", "Q5_1"])
def test_sample_and_generate_after_score(lib, fmt):
    """After score, sample and generate return what they return after eval_resident of the same tokens (tensor cores off)."""
    path = model_path("7v0-834K", fmt)
    a, b = Ctx(lib, path, False), Ctx(lib, path, False)
    try:
        toks = [t % a.V for t in LONG_PROMPT]
        a.fresh(); b.fresh()
        a.score(toks, text_targets(toks, a.V))
        b.eval_resident(toks)
        outs = []
        for c in (a, b):
            tok = ctypes.c_uint32()
            assert c.L.rwkv_b200_sample(c.ptr, 0.9, 0.8, 0.37, None, None, 0, ctypes.byref(tok))
            u = np.random.default_rng(2).random(8)
            gen, n = np.zeros(8, np.uint32), ctypes.c_size_t()
            assert c.L.rwkv_b200_generate(c.ptr, 8, 1.0, 0.9, 0.1, 0.1, False, u.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), None, 0,
                                          gen.ctypes.data_as(P_U), ctypes.byref(n))
            outs.append((tok.value, bits(gen), n.value, bits(c.state())))
        assert outs[0] == outs[1]
    finally:
        a.free(); b.free()


def test_seeded_interleaving_matches_serial_replay(lib):
    """A seeded mix of score / eval_resident / generate / clone on one context against the same steps replayed with serial
    rwkv_eval on a twin: states and scores bit for bit (tensor cores off)."""
    path = model_path("6v0-3m", "Q5_1")
    ctx, twin = Ctx(lib, path, False), Ctx(lib, path, False)
    rng = np.random.default_rng(1234)
    clones = []
    try:
        ctx.fresh(); twin.fresh()
        ctx.eval_resident([1]); twin.eval_resident([1])     # logits to draw from
        for step in range(24):
            kind = rng.choice(["score", "eval", "generate", "clone"])
            if kind == "clone":
                c = lib.rwkv_clone_context(ctx.c, 1)
                clones.append(c)
                continue
            if kind == "generate":
                u = rng.random(3)
                outs = []
                for x in (ctx, twin):
                    gen, n = np.zeros(3, np.uint32), ctypes.c_size_t()
                    assert x.L.rwkv_b200_generate(x.ptr, 3, 0.8, 0.9, 0.0, 0.0, False, u.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                                  None, 0, gen.ctypes.data_as(P_U), ctypes.byref(n))
                    outs.append(bits(gen))
                assert outs[0] == outs[1], step
                continue
            toks = [int(t) for t in rng.integers(0, ctx.V, int(rng.integers(1, 40)))]
            if kind == "eval":
                ctx.eval_resident(toks)
            else:
                targets = [int(t) for t in rng.integers(0, ctx.V, len(toks))]
                lp, g = ctx.score(toks, targets)
            # replay on the twin: serial rwkv_eval from its resident state, then the kernel on those logits
            st = twin.state()
            lg = np.zeros(twin.V, np.float32)
            ref = []
            for t in toks:
                assert twin.L.rwkv_eval(twin.ptr, t, st.ctypes.data_as(P_F), st.ctypes.data_as(P_F), lg.ctypes.data_as(P_F))
                ref.append(lg.copy())
            if kind == "score":
                want_lp, want_g = score_logits(lib, np.stack(ref), targets)
                assert bits(lp) == bits(want_lp) and bits(g) == bits(want_g), step
            assert bits(ctx.state()) == bits(twin.state()), (step, kind)
    finally:
        for c in clones:
            lib.rwkv_free(c)
        ctx.free(); twin.free()


# ---- refusals and memory ------------------------------------------------------------------------------------------------------

def test_refusals_change_nothing(lib):
    path = model_path("6v0-3m", "FP32")
    ctx = Ctx(lib, path, False)
    bt = Batch(ctx, 3, False)
    try:
        toks = [t % ctx.V for t in LONG_PROMPT[:12]]
        ctx.fresh()
        ctx.eval_resident(toks)
        st, lg = ctx.state(), ctx.logits()
        L, V = ctx.L, ctx.V
        good_t, good_tg = u32(toks), u32(text_targets(toks, V))
        lp = np.zeros(12, np.float32)

        def refused(args, flags, target=ctx.ptr):
            assert not L.rwkv_b200_score(target, *args)
            assert L.rwkv_get_last_error(target) == flags, args
        PU = lambda a: a.ctypes.data_as(P_U)       # noqa: E731
        refused((None, PU(good_tg), 12, lp.ctypes.data_as(P_F), None), ERR_ARGS)
        refused((PU(good_t), None, 12, lp.ctypes.data_as(P_F), None), ERR_ARGS)
        refused((PU(good_t), PU(good_tg), 12, None, None), ERR_ARGS)
        refused((PU(good_t), PU(good_tg), 0, lp.ctypes.data_as(P_F), None), ERR_ARGS)
        bad_t = good_t.copy(); bad_t[5] = V
        refused((PU(bad_t), PU(good_tg), 12, lp.ctypes.data_as(P_F), None), ERR_ARGS)
        bad_tg = good_tg.copy(); bad_tg[3] = V
        refused((PU(good_t), PU(bad_tg), 12, lp.ctypes.data_as(P_F), None), ERR_ARGS)
        refused((PU(good_t), PU(good_tg), 12, lp.ctypes.data_as(P_F), None), ERR_CTX | ERR_UNSUPPORTED, target=bt.ptr)
        # the batch call on an ordinary context, and its count rules
        c3 = u32([4, 0, 8])
        assert not L.rwkv_b200_batch_score_ragged(ctx.ptr, PU(good_t), PU(c3), PU(good_tg), lp.ctypes.data_as(P_F), None)
        assert L.rwkv_get_last_error(ctx.ptr) == ERR_CTX | ERR_UNSUPPORTED
        bst = [bt.state(b) for b in range(3)]
        for counts in ([0, 0, 0], [200, 50, 7]):
            big = u32([1] * 257)
            assert not L.rwkv_b200_batch_score_ragged(bt.ptr, PU(big), PU(u32(counts)), PU(u32([1] * 257)), np.zeros(257, np.float32).ctypes.data_as(P_F), None)
            assert L.rwkv_get_last_error(bt.ptr) == ERR_ARGS
        assert not L.rwkv_b200_batch_score_ragged(bt.ptr, PU(good_t), PU(c3), PU(bad_tg), lp.ctypes.data_as(P_F), None)
        assert L.rwkv_get_last_error(bt.ptr) == ERR_ARGS
        assert all(bits(bt.state(b)) == bits(bst[b]) for b in range(3))
        assert bits(ctx.state()) == bits(st) and bits(ctx.logits()) == bits(lg)
        tok = ctypes.c_uint32()
        assert L.rwkv_b200_sample(ctx.ptr, 0.0, 1.0, 0.5, None, None, 0, ctypes.byref(tok))      # the logits are still valid
    finally:
        bt.free()
        ctx.free()


def test_tiled_head_is_built_by_the_first_tensor_core_scoring_pass_and_freed_with_the_model(lib, tmp_path):
    import torch
    import synthetic_model as sm
    path = synthetic(tmp_path, "rwkv5-1b5", "Q5_1")      # FP16 head of 65536 x 2048: a 256 MiB tile-major copy
    p = sm.PRESETS["rwkv5-1b5"]
    tiled = ((p["V"] + 127) // 128) * (p["C"] // 64) * 128 * 64 * 2
    free = lambda: torch.cuda.mem_get_info(0)[0]          # noqa: E731
    torch.cuda.init()
    base = free()
    ctx = Ctx(lib, path, True)
    try:
        toks = sm.synthetic_tokens(64, ctx.V)
        ctx.fresh()
        ctx.eval_resident(toks)
        ctx.score(toks[:8], toks[1:9])                    # a GEMV-head scoring pass builds nothing
        f0 = free()
        ctx.score(toks[:40], toks[1:41])                  # the first tensor-core scoring pass builds the copy
        f1 = free()
        assert tiled <= f0 - f1 <= tiled + (8 << 20), (f0 - f1, tiled)
        clone = lib.rwkv_clone_context(ctx.c, 1)          # the model, and with it the copy, lives on in the clone
        ctx.free()
        ctx = None
        lib.rwkv_free(clone)
        assert free() >= base - (8 << 20), (base - free())
    finally:
        if ctx:
            ctx.free()
