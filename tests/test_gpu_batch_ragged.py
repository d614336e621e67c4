"""Ragged passes of a batch context (rwkv_b200_batch_eval_ragged and the ragged mode of the LayerNorm-mix and WKV kernels): in one
pass sequence b advances counts[b] tokens. Per kernel, a ragged launch equals the single-sequence launch on each sequence's columns
bit for bit; per model, each sequence equals a single context fed the same tokens one at a time, and an idle sequence is left exactly
as it was."""
import ctypes

import numpy as np
import pytest

import kernel_hooks as kh
from conftest import LONG_PROMPT, model_path
from test_gpu_kernels import F32, HEAD_SIZES, WKV6_MODES, WKV7_COLS, bits, guards, ln_mix_inputs, rng_for, run_wkv4, run_wkv6, run_wkv7, \
    slice_cols, wkv4_inputs, wkv6_inputs, wkv7_inputs

pytestmark = pytest.mark.gpu
P_F, P_U = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32)
COUNT_SETS = [[3, 0, 1, 8, 17, 0, 9], [0, 9, 16, 1, 0], [13]]       # chunk boundaries of WKV6_TB = 8, empty first / last, a lone sequence


def offsets(counts):
    return np.concatenate([[0], np.cumsum(counts)]).astype(int)


def call_ragged(lib, fn, args, counts):
    c = (ctypes.c_uint32 * len(counts))(*counts)
    if not getattr(lib.library, fn)(ctypes.byref(args), c, ctypes.c_size_t(len(counts))):
        raise kh.HookError(lib.rwkv_get_last_error(None))


def untouched(out, start, stop):
    return bool((out.buf[start:stop].view(np.uint8) == 0xFF).all())


# ---- per kernel ---------------------------------------------------------------------------------------------------------

def ln_mix_ragged(lib, x, w, b, states, coefs, formula, counts, stride):
    C, cols = x.shape
    i = kh.Inputs()
    a = kh.LnMixArgs(x=i(x, True), ln_w=i(w), ln_b=i(b), state_in=i(states), C=C, T=cols, formula=formula, n_out=len(coefs),
                     n_seq=len(counts), seq_stride=stride)
    o = {"state": kh.Out(states.size), "xx": kh.Out(C * cols), "sx": kh.Out(C * cols)}
    a.state_out, a.out_xx, a.out_sx = o["state"].ptr, o["xx"].ptr, o["sx"].ptr
    for j, m in enumerate(coefs):
        o["out%d" % j] = kh.Out(C * cols)
        a.coef[j], a.out[j] = i(m), o["out%d" % j].ptr
    call_ragged(lib, "rwkv_b200_test_ln_mix_ragged", a, counts)
    return o


@pytest.mark.parametrize("C", [64, 2048, 4096, 5120, 12288])          # 1, 2, 4, 8, 16 channels per thread
@pytest.mark.parametrize("n_out,formula", [(2, 0), (6, 1)])           # PRE_N 3 and 6
@pytest.mark.parametrize("counts", COUNT_SETS)
def test_ln_mix_ragged_equals_single_sequences(lib, C, n_out, formula, counts):
    T, off, stride = sum(counts), offsets(counts), C + 32
    x, w, b, _, coefs = ln_mix_inputs(C, T, n_out, rng_for("ln_mix-ragged", C, n_out, T))
    states = rng_for("ln_mix-ragged-state", C).standard_normal((len(counts) - 1) * stride + C).astype(F32)
    o = ln_mix_ragged(lib, x, w, b, states, coefs, formula, counts, stride)
    guards(o)
    for s, n in enumerate(counts):
        sl = slice(s * stride, s * stride + C)
        if n == 0:
            assert untouched(o["state"], sl.start, sl.stop), s
            continue
        one = kh.ln_mix(lib, x[:, off[s]:off[s + 1]], w, b, states[sl], coefs, formula)
        for key in [k for k in one if k != "state"]:
            assert bits(one[key].value) == bits(o[key].value[off[s] * C:off[s + 1] * C]), (s, key)
        assert bits(one["state"].value) == bits(o["state"].value[sl]), s
    for s in range(len(counts) - 1):
        assert untouched(o["state"], s * stride + C, (s + 1) * stride), s


def wkv6_ragged(lib, d, mode, counts, stride):
    C, cols = d["r"].shape
    i = kh.Inputs()
    a = kh.Wkv6Args(r=i(d["r"], True), k=i(d["k"], True), v=i(d["v"], True), td=i(d["td"], mode == "v6"), tf=i(d["tf"]),
                    td_per_token=int(mode == "v6"), per_head_scalars=int(mode == "v5.1"), state_in=i(d["state"]), lnx_w=i(d["lnx_w"]),
                    lnx_b=i(d["lnx_b"]), g=i(d["g"], True), eps=d["eps"], H=d["H"], S=d["S"], T=cols, n_seq=len(counts), seq_stride=stride)
    o = {"state": kh.Out(d["state"].size), "y": kh.Out(C * cols)}
    a.state_out, a.y = o["state"].ptr, o["y"].ptr
    call_ragged(lib, "rwkv_b200_test_wkv6_ragged", a, counts)
    return o


@pytest.mark.parametrize("S", HEAD_SIZES)
@pytest.mark.parametrize("mode", WKV6_MODES)
@pytest.mark.parametrize("counts", COUNT_SETS)
def test_wkv6_ragged_equals_single_sequences(lib, S, mode, counts):
    H, T, off = 2, sum(counts), offsets(counts)
    SS = H * S * S
    stride = SS + 24
    d = wkv6_inputs(mode, H, S, T, rng_for("wkv6-ragged", S, mode, T))
    states = rng_for("wkv6-ragged-state", S).standard_normal((len(counts) - 1) * stride + SS).astype(F32)
    o = wkv6_ragged(lib, dict(d, state=states), mode, counts, stride)
    guards(o)
    cols = ("r", "k", "v", "g") + (("td",) if mode == "v6" else ())
    for s, n in enumerate(counts):
        sl = slice(s * stride, s * stride + SS)
        if n == 0:
            assert untouched(o["state"], sl.start, sl.stop), s
            continue
        one = run_wkv6(lib, dict(slice_cols(d, off[s], off[s + 1], cols), state=states[sl]), mode)
        assert bits(one["y"].value) == bits(o["y"].value[off[s] * H * S:off[s + 1] * H * S]), s
        assert bits(one["state"].value) == bits(o["state"].value[sl]), s


def wkv7_ragged(lib, d, counts, stride):
    C, cols = d["r"].shape
    i = kh.Inputs()
    a = kh.Wkv7Args(r=i(d["r"], True), w=i(d["w"], True), k=i(d["k"], True), v=i(d["v"], True), a=i(d["aa"], True), g=i(d["g"], True),
                    vgate=i(d["vgate"], True), v_first=i(d["v_first"], True), k_k=i(d["k_k"]), k_a=i(d["k_a"]), r_k=i(d["r_k"]),
                    lnx_w=i(d["lnx_w"]), lnx_b=i(d["lnx_b"]), state_in=i(d["state"]), H=d["H"], S=d["S"], T=cols, n_seq=len(counts),
                    seq_stride=stride)
    o = {"state": kh.Out(d["state"].size), "y": kh.Out(C * cols), "v": kh.Out(C * cols)}
    a.state_out, a.y, a.v_out = o["state"].ptr, o["y"].ptr, o["v"].ptr
    call_ragged(lib, "rwkv_b200_test_wkv7_ragged", a, counts)
    return o


@pytest.mark.parametrize("S", HEAD_SIZES)
@pytest.mark.parametrize("counts", COUNT_SETS)
def test_wkv7_ragged_equals_single_sequences(lib, S, counts):
    H, T, off = 2, sum(counts), offsets(counts)
    SS = H * S * S
    stride = SS + 24
    d = wkv7_inputs(H, S, T, rng_for("wkv7-ragged", S, T), len(counts) != 5)
    states = (0.5 * rng_for("wkv7-ragged-state", S).standard_normal((len(counts) - 1) * stride + SS)).astype(F32)
    o = wkv7_ragged(lib, dict(d, state=states), counts, stride)
    guards(o)
    for s, n in enumerate(counts):
        sl = slice(s * stride, s * stride + SS)
        if n == 0:
            assert untouched(o["state"], sl.start, sl.stop), s
            continue
        one = run_wkv7(lib, dict(slice_cols(d, off[s], off[s + 1], WKV7_COLS), state=states[sl]))
        for key in ("y", "v"):
            assert bits(one[key].value) == bits(o[key].value[off[s] * H * S:off[s + 1] * H * S]), (s, key)
        assert bits(one["state"].value) == bits(o["state"].value[sl]), s


@pytest.mark.parametrize("C", [333, 1056])
@pytest.mark.parametrize("counts", COUNT_SETS)
def test_wkv4_ragged_equals_single_sequences(lib, C, counts):
    T, off, stride = sum(counts), offsets(counts), C + 8
    d = wkv4_inputs(C, T, rng_for("wkv4-ragged", C, T), False)
    rng = rng_for("wkv4-ragged-state", C)
    n = (len(counts) - 1) * stride + C
    st = dict(aa=rng.standard_normal(n).astype(F32), bb=rng.uniform(0.5, 3, n).astype(F32), pp=(5 * rng.standard_normal(n)).astype(F32))
    i = kh.Inputs()
    a = kh.Wkv4Args(k=i(d["k"], True), v=i(d["v"], True), r=i(d["r"], True), time_first=i(d["tf"]), time_decay=i(d["td"]), aa_in=i(st["aa"]),
                    bb_in=i(st["bb"]), pp_in=i(st["pp"]), C=C, T=T, n_seq=len(counts), seq_stride=stride)
    o = {"aa": kh.Out(n), "bb": kh.Out(n), "pp": kh.Out(n), "y": kh.Out(C * T)}
    a.aa_out, a.bb_out, a.pp_out, a.y = o["aa"].ptr, o["bb"].ptr, o["pp"].ptr, o["y"].ptr
    call_ragged(lib, "rwkv_b200_test_wkv4_ragged", a, counts)
    guards(o)
    for s, cnt in enumerate(counts):
        sl = slice(s * stride, s * stride + C)
        if cnt == 0:
            assert all(untouched(o[k], sl.start, sl.stop) for k in ("aa", "bb", "pp")), s
            continue
        one = run_wkv4(lib, dict(slice_cols(d, off[s], off[s + 1], ("k", "v", "r")), aa=st["aa"][sl], bb=st["bb"][sl], pp=st["pp"][sl]))
        assert bits(one["y"].value) == bits(o["y"].value[off[s] * C:off[s + 1] * C]), s
        for k in ("aa", "bb", "pp"):
            assert bits(one[k].value) == bits(o[k].value[sl]), (s, k)


# ---- whole model ---------------------------------------------------------------------------------------------------------

def token_streams(n_seq, n_tok, V):
    L = len(LONG_PROMPT)
    return [[(LONG_PROMPT[(i + 5 * b) % L] * (b + 1) + 7 * b + i // L) % V for i in range(n_tok)] for b in range(n_seq)]


def alone_all(lib, ctx, toks, n_state, n_logits):
    """Logits after every token and the final state of `toks` fed one at a time through rwkv_eval."""
    state = np.zeros(n_state, np.float32)
    logits = np.zeros(n_logits, np.float32)
    out = []
    for i, t in enumerate(toks):
        assert lib.library.rwkv_eval(ctx.ptr, t, None if i == 0 else state.ctypes.data_as(P_F), state.ctypes.data_as(P_F), logits.ctypes.data_as(P_F))
        out.append(logits.copy())
    return out, state


class Batch:
    def __init__(self, lib, ctx, n_seq, tensor_cores=True):
        self.lib, self.n_seq = lib, n_seq
        self.ptr = ctypes.c_void_p(lib.library.rwkv_b200_batch_create(ctx.ptr, n_seq))
        assert self.ptr
        lib.library.rwkv_b200_set_tensor_cores(self.ptr, tensor_cores)
        self.n_state, self.n_logits = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)

    def ragged(self, tokens, counts, want_logits=True):
        t = (ctypes.c_uint32 * max(1, len(tokens)))(*tokens)
        c = (ctypes.c_uint32 * self.n_seq)(*counts)
        return self.lib.library.rwkv_b200_batch_eval_ragged(self.ptr, t, c, want_logits)

    def state(self, b):
        st = np.zeros(self.n_state, np.float32)
        assert self.lib.library.rwkv_b200_batch_get_state(self.ptr, b, st.ctypes.data_as(P_F))
        return st

    def logits(self, b):
        lg = np.zeros(self.n_logits, np.float32)
        assert self.lib.library.rwkv_b200_batch_get_logits(self.ptr, b, lg.ctypes.data_as(P_F))
        return lg

    def free(self):
        self.lib.library.rwkv_free(self.ptr)


L_PROMPT = len(LONG_PROMPT)
# (counts, want_logits) for B = 5: prompts, single decode tokens and idle slots side by side, one pass of 256 tokens
SCHEDULE = [([L_PROMPT, 1, 0, 3, 1], True), ([0, 1, 1, 0, 8], True), ([100, 56, 50, 30, 20], True), ([1, 0, 17, 1, 0], False),
            ([1, 1, 1, 1, 1], True), ([0, 0, 0, 0, 9], True), ([2, 0, 0, 0, 0], False)]


def run_schedule(lib, path, schedule, tensor_cores, exact, bar=None):
    ctx = lib.rwkv_init_from_file(path, 1, 0)
    batch = None
    try:
        n_seq = len(schedule[0][0])
        totals = [sum(c[b] for c, _ in schedule) for b in range(n_seq)]
        batch = Batch(lib, ctx, n_seq, tensor_cores)
        streams = token_streams(n_seq, max(totals), batch.n_logits)
        want = [alone_all(lib, ctx, streams[b][:totals[b]], batch.n_state, batch.n_logits) if totals[b] else ([], None) for b in range(n_seq)]
        done = [0] * n_seq
        worst = 0.0
        for counts, want_logits in schedule:
            before = [(batch.state(b), batch.logits(b) if done != [0] * n_seq else None) for b in range(n_seq)]
            toks = [t for b in range(n_seq) for t in streams[b][done[b]:done[b] + counts[b]]]
            assert batch.ragged(toks, counts, want_logits), (counts, lib.library.rwkv_get_last_error(batch.ptr))
            for b in range(n_seq):
                done[b] += counts[b]
                if counts[b] == 0:
                    assert bits(batch.state(b)) == bits(before[b][0]), (counts, b)
                    if before[b][1] is not None:
                        assert bits(batch.logits(b)) == bits(before[b][1]), (counts, b)
                elif want_logits:
                    got, ref = batch.logits(b), want[b][0][done[b] - 1]
                    if exact:
                        assert bits(got) == bits(ref), (path, counts, b, np.abs(got - ref).max())
                    else:
                        assert np.isfinite(got).all()
                        worst = max(worst, float(np.abs(got - ref).max()))
        for b in range(n_seq):
            if exact and totals[b]:
                assert bits(batch.state(b)) == bits(want[b][1]), (path, b)
        if not exact:
            assert worst <= bar, (path, worst)
    finally:
        if batch:
            batch.free()
        lib.rwkv_free(ctx)


@pytest.mark.parametrize("ver", ["4v0-660K", "5v1-730K", "5v2-730K", "6v0-3m", "7v0-834K"])
@pytest.mark.parametrize("fmt", ["FP32", "Q5_1"])
def test_ragged_equals_alone_bitwise_fixtures(lib, ver, fmt):
    run_schedule(lib, model_path(ver, fmt), SCHEDULE, tensor_cores=False, exact=True)


def test_ragged_equals_alone_bitwise_fp16(lib):
    run_schedule(lib, model_path("6v0-3m", "FP16"), SCHEDULE, tensor_cores=False, exact=True)


def synthetic(tmp_path, preset, fmt):
    import synthetic_model as sm
    path = str(tmp_path / f"{preset}-{fmt}.bin")
    sm.write_direct(path, preset, fmt, seed=8)
    return path


@pytest.mark.parametrize("preset,fmt", [("rwkv6-small", "Q5_1"), ("rwkv7-small", "FP16"), ("rwkv5-small", "Q4_0")])
def test_ragged_on_the_tensor_cores(lib, tmp_path, preset, fmt):
    """Passes of >= 16 tokens send the layer matrices through the wgmma kernel: per sequence within the batch bar of the sequence
    alone; passes of fewer tokens stay on the GEMV and stay bit-exact."""
    path = synthetic(tmp_path, preset, fmt)
    big = [([20, 1, 0, 1, 1, 3], True), ([1, 1, 1, 1, 30, 0], True), ([0, 64, 1, 1, 1, 1], True), ([5, 5, 5, 5, 5, 5], True)]
    run_schedule(lib, path, big, tensor_cores=True, exact=False, bar=5e-3 if fmt == "FP16" else 5e-2)
    small = [([7, 1, 0, 1, 1, 3], True), ([1, 1, 1, 1, 9, 0], True), ([0, 0, 15, 0, 0, 0], True)]
    run_schedule(lib, path, small, tensor_cores=True, exact=True)


def twin_check(lib, path, n_seq, steps, tensor_cores):
    """counts = 1 everywhere against rwkv_b200_batch_eval on a twin batch context: the same bytes."""
    ctx = lib.rwkv_init_from_file(path, 1, 0)
    a = b = None
    try:
        a, b = Batch(lib, ctx, n_seq, tensor_cores), Batch(lib, ctx, n_seq, tensor_cores)
        streams = token_streams(n_seq, steps, a.n_logits)
        for step in range(steps):
            toks = [streams[s][step] for s in range(n_seq)]
            assert a.ragged(toks, [1] * n_seq)
            assert lib.library.rwkv_b200_batch_eval(b.ptr, (ctypes.c_uint32 * n_seq)(*toks), True)
            for s in range(n_seq):
                assert bits(a.logits(s)) == bits(b.logits(s)), (path, step, s)
        for s in range(n_seq):
            assert bits(a.state(s)) == bits(b.state(s)), (path, s)
    finally:
        for x in (a, b):
            if x:
                x.free()
        lib.rwkv_free(ctx)


@pytest.mark.parametrize("ver", ["5v2-730K", "6v0-3m", "7v0-834K"])
def test_all_ones_equals_batch_eval(lib, ver):
    twin_check(lib, model_path(ver, "Q5_1"), 5, 4, tensor_cores=True)


@pytest.mark.parametrize("preset,fmt,n_seq", [("rwkv6-small", "Q5_1", 16), ("rwkv7-small", "FP16", 16), ("rwkv5-small", "Q4_0", 40)])
def test_all_ones_equals_batch_eval_tensor_cores(lib, tmp_path, preset, fmt, n_seq):
    twin_check(lib, synthetic(tmp_path, preset, fmt), n_seq, 3, tensor_cores=True)


def test_sampling_after_a_ragged_pass(lib):
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    batch = None
    try:
        n_seq = 4
        batch = Batch(lib, ctx, n_seq, tensor_cores=False)
        fresh = Batch(lib, ctx, 2)
        assert fresh.ragged([5], [1, 0])
        assert not fresh.logits(1).any()                               # never computed: zeros from creation
        fresh.free()
        streams = token_streams(n_seq, 12, batch.n_logits)
        plan = [[3, 1, 2, 0], [0, 4, 1, 0]]
        done = [0] * n_seq
        for counts in plan:
            toks = [t for b in range(n_seq) for t in streams[b][done[b]:done[b] + counts[b]]]
            assert batch.ragged(toks, counts)
            done = [d + c for d, c in zip(done, counts)]
        temp = (ctypes.c_float * n_seq)(*[0.8, 1.0, 0.0, 1.2])
        top_p = (ctypes.c_float * n_seq)(*[0.9, 0.0, 1.0, 0.5])
        u = (ctypes.c_double * n_seq)(*[0.3, 0.71, 0.5, 0.05])
        out = (ctypes.c_uint32 * n_seq)()
        assert lib.library.rwkv_b200_batch_sample(batch.ptr, temp, top_p, u, None, None, None, out)
        for b in range(n_seq):
            tok = ctypes.c_uint32()
            if done[b]:
                alone_all(lib, ctx, streams[b][:done[b]], batch.n_state, batch.n_logits)     # leaves that sequence's logits in ctx
                assert lib.library.rwkv_b200_sample(ctx.ptr, temp[b], top_p[b], u[b], None, None, 0, ctypes.byref(tok))
            else:
                col = batch.logits(b)                                  # idle since creation: the zeros it holds
                assert not col.any()
                assert lib.library.rwkv_b200_sample_logits(col.ctypes.data_as(P_F), col.size, temp[b], top_p[b], u[b], None, None, 0,
                                                           ctypes.byref(tok), None)
            assert out[b] == tok.value, b
    finally:
        if batch:
            batch.free()
        lib.rwkv_free(ctx)


def test_ragged_rejections_leave_everything_untouched(lib):
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    batch = None
    try:
        batch = Batch(lib, ctx, 3, tensor_cores=False)
        V = batch.n_logits
        assert batch.ragged([1, 2, 3, 4], [2, 1, 1])
        states = [batch.state(b) for b in range(3)]
        logits = [batch.logits(b) for b in range(3)]
        CTX_UNSUPPORTED, ARGS = (6 << 8) | 9, 1 << 8
        c3 = (ctypes.c_uint32 * 3)(1, 1, 1)
        t3 = (ctypes.c_uint32 * 3)(1, 2, 3)
        assert not lib.library.rwkv_b200_batch_eval_ragged(ctx.ptr, t3, c3, True)
        assert lib.rwkv_get_last_error(ctx) == CTX_UNSUPPORTED
        cases = [(None, c3), (t3, None), (t3, (ctypes.c_uint32 * 3)(0, 0, 0)), ((ctypes.c_uint32 * 257)(*[1] * 257), (ctypes.c_uint32 * 3)(200, 57, 0)),
                 ((ctypes.c_uint32 * 3)(1, V, 3), c3)]
        for tokens, counts in cases:
            assert not lib.library.rwkv_b200_batch_eval_ragged(batch.ptr, tokens, counts, True)
            assert lib.library.rwkv_get_last_error(batch.ptr) == ARGS
        for b in range(3):
            assert bits(batch.state(b)) == bits(states[b]) and bits(batch.logits(b)) == bits(logits[b]), b
    finally:
        if batch:
            batch.free()
        lib.rwkv_free(ctx)
