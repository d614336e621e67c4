"""Generation with log-probabilities (rwkv_b200_generate_logprobs / rwkv_b200_batch_generate_logprobs, the logprob step kernels of
csrc/kernels/sampling.cu): generation itself must not change by a bit, every drawn token's log-probability and top alternatives must
be the bits rwkv_b200_score_logits gives for the logits it was drawn from, and its sampling probability the prob_out of
rwkv_b200_sample_logits with the step's bias list."""
import ctypes

import numpy as np
import pytest

import byte_dfa as bd
import generate_ref as gr
from conftest import LONG_PROMPT, model_path
from generate_ref import P_D, P_F, P_U
from test_gpu_generate import ERR_ARGS, P_U8, Batch, Pair, bias_arrays, f32, generate, logits, prime, ptr, state
from test_gpu_generate_constrained import NONE, Automaton, P16, batch_constrained, gen_constrained, mask_bias
from test_gpu_generate_stream import NULL_FN, Recorder

NO_TARGET = 0xFFFFFFFF
TOP_MAX = 20


# ---- float64 references ----------------------------------------------------------------------------------------------------------

def column_valid(z):
    z = np.asarray(z, np.float32)
    return not (np.isnan(z).any() or np.isposinf(z).any()) and np.isfinite(z).any()


def top_ref(z, n):
    """The top n ids of z: descending logit, the smaller id first among equal logits (-0 equals +0); NO_TARGET for an invalid column."""
    if not column_valid(z):
        return [NO_TARGET] * n
    z = np.asarray(z, np.float64)
    return [int(i) for i in np.lexsort((np.arange(len(z)), -z))[:n]]


def logprob_ref(z, t):
    z = np.asarray(z, np.float64)
    m = z.max()
    return (z[t] - m) - np.log(np.exp(z - m).sum())


# ---- library calls ---------------------------------------------------------------------------------------------------------------

class Out:
    """The output arrays of a logprob call, [rows][n] (top arrays [rows][n][top_n]), prefilled with a marker."""

    def __init__(self, rows, n, top_n, sample_probs=True):
        self.top_n = top_n
        self.logprobs = np.full((rows, n), 7.0, np.float32)
        self.sample_probs = np.full((rows, n), 7.0, np.float32) if sample_probs else None
        self.top_ids = np.full((rows, n, max(top_n, 1)), 7, np.uint32)
        self.top_logprobs = np.full((rows, n, max(top_n, 1)), 7.0, np.float32)

    def struct(self, **override):
        import rwkv_cpp_b200.shared_library as sl
        s = sl.Logprobs(top_n=self.top_n, logprobs=ptr(self.logprobs, P_F), top_ids=ptr(self.top_ids, P_U) if self.top_n else None,
                        top_logprobs=ptr(self.top_logprobs, P_F) if self.top_n else None, sample_probs=ptr(self.sample_probs, P_F))
        for k, v in override.items():
            setattr(s, k, v)
        return s

    def tops(self, b, i):
        return [int(x) for x in self.top_ids[b, i, :self.top_n]]


def gen_logprobs(lib, ctx_ptr, out, max_tokens, temperature, top_p, presence, frequency, us, stops=(), keep=False, rec=None, auto=None, st=0, lp=None):
    toks = np.zeros(max(max_tokens, 1), np.uint32)
    n = ctypes.c_size_t(0)
    s = np.array([st], np.uint32)
    sp = np.array(stops, np.uint32) if len(stops) else None
    lps = out.struct() if lp is None else lp
    ok = lib.library.rwkv_b200_generate_logprobs(ctx_ptr, auto.ptr if auto else None, ptr(s, P_U), max_tokens, temperature, top_p, presence, frequency, keep,
                                                 ptr(np.asarray(us, np.float64), P_D), ptr(sp, P_U), len(stops), rec.fn if rec else NULL_FN, None,
                                                 ptr(toks, P_U), ctypes.byref(n), ctypes.byref(lps) if lps is not False else None)
    return ok, [int(t) for t in toks[:n.value]], int(s[0])


def batch_logprobs(bt, out, max_tokens, temps, top_ps, pres, freq, us, stops=(), rec=None):
    n = max(max_tokens)
    toks = np.zeros(bt.n * max(n, 1), np.uint32)
    ng = np.zeros(bt.n, np.uint32)
    sp = np.array(stops, np.uint32) if len(stops) else None
    lps = out.struct()
    ok = bt.lib.library.rwkv_b200_batch_generate_logprobs(
        bt.ptr, None, None, ptr(np.asarray(max_tokens, np.uint32), P_U), ptr(f32(temps), P_F), ptr(f32(top_ps), P_F), ptr(f32(pres), P_F), ptr(f32(freq), P_F),
        None, ptr(np.ascontiguousarray(us, np.float64), P_D), ptr(sp, P_U), len(stops), rec.fn if rec else NULL_FN, None, ptr(toks, P_U), ptr(ng, P_U),
        ctypes.byref(lps))
    return ok, [[int(t) for t in toks[b * n:b * n + ng[b]]] for b in range(bt.n)]


def score_logits(lib, z, targets):
    """rwkv_b200_score_logits of column z at every target (one row per target)."""
    z = np.ascontiguousarray(z, np.float32)
    t = np.asarray(targets, np.uint32)
    rows = np.ascontiguousarray(np.broadcast_to(z, (len(t), len(z))))
    lp = np.zeros(len(t), np.float32)
    assert lib.library.rwkv_b200_score_logits(ptr(rows, P_F), len(t), len(z), ptr(t, P_U), ptr(lp, P_F), None)
    return lp


def check_entry(lib, z, tok, out, b, i):
    """Entry (b, i) of out against rwkv_b200_score_logits on z, the float64 top-N reference and score's float64 bar."""
    k = out.top_n
    want_ids = top_ref(z, k)
    assert out.tops(b, i) == want_ids, (b, i, out.tops(b, i), want_ids)
    ref = score_logits(lib, z, [tok] + [t for t in want_ids if t != NO_TARGET])
    assert out.logprobs[b, i].tobytes() == ref[0].tobytes(), (b, i, out.logprobs[b, i], ref[0])
    if not column_valid(z):
        assert np.isnan(out.logprobs[b, i]) and np.isnan(out.top_logprobs[b, i, :k]).all()
        return
    assert out.top_logprobs[b, i, :k].tobytes() == ref[1:].tobytes(), (b, i)
    for got, t in [(out.logprobs[b, i], tok)] + [(out.top_logprobs[b, i, j], want_ids[j]) for j in range(k)]:
        want = logprob_ref(z, t)
        if np.isinf(want):
            assert got == want
        else:
            assert abs(float(got) - want) <= 1e-6 * (1 + abs(want)), (b, i, t, got, want)


def check_tail(out, b, n_generated):
    assert np.isnan(out.logprobs[b, n_generated:]).all()
    if out.sample_probs is not None:
        assert np.isnan(out.sample_probs[b, n_generated:]).all()
    assert (out.top_ids[b, n_generated:, :out.top_n] == NO_TARGET).all() and np.isnan(out.top_logprobs[b, n_generated:, :out.top_n]).all()


# ---- 1. the step hook ------------------------------------------------------------------------------------------------------------

def hook_rows(rng, V, top_n):
    """Rows of every kind the contract names: normal and wide spreads, ties at the top and across the top_n boundary, -inf entries,
    fewer finite entries than top_n, NaN, +inf and all -inf."""
    rows = [rng.standard_normal(V) * 3.0, rng.standard_normal(V) * 40.0]
    t = rng.standard_normal(V) * 2.0
    t[rng.choice(V, size=min(3, V), replace=False)] = t.max() + 1.0      # three equal maxima
    rows.append(t)
    t = rng.standard_normal(V)
    order = np.argsort(-t)
    if V > top_n + 1 and top_n > 0:
        t[order[max(top_n - 2, 0):top_n + 2]] = t[order[max(top_n - 2, 0)]]  # equal values straddle the boundary
    rows.append(t)
    t = rng.standard_normal(V) * 2.0
    t[rng.rand(V) < 0.5] = -np.inf
    t[0] = 1.0
    rows.append(t)
    t = np.full(V, -np.inf)
    t[rng.choice(V, size=min(2, V), replace=False)] = [0.5, -0.0][:min(2, V)]
    rows.append(t)
    t = rng.standard_normal(V); t[V // 2] = np.nan; rows.append(t)
    t = rng.standard_normal(V); t[V - 1] = np.inf; rows.append(t)
    rows.append(np.full(V, -np.inf))
    t = np.zeros(V); t[::2] = -0.0; rows.append(t)                          # -0 and +0 tie by id
    return np.ascontiguousarray(np.array(rows), np.float32)


def step_args(logits, max_tokens, temps, top_ps, pres, freq, us, stops, step, frozen, counts, tokens):
    R, V = logits.shape
    keep = dict(step=np.array(step, np.uint32), frozen=np.array(frozen, np.uint8), counts=counts.copy(), tokens=tokens.copy(), nxt=np.zeros(R, np.int32),
                any_active=ctypes.c_uint32(7), st=np.array(stops, np.uint32) if len(stops) else None,
                arrs=(np.asarray(max_tokens, np.uint32), f32(temps), f32(top_ps), f32(pres), f32(freq), np.ascontiguousarray(us, np.float64)))
    mt, t, p, pr, fr, u = keep["arrs"]
    a = gr.StepArgs(logits=logits.ctypes.data, n_rows=R, n_vocab=V, max_tokens=mt.ctypes.data, temperature=t.ctypes.data, top_p=p.ctypes.data,
                    presence_penalty=pr.ctypes.data, frequency_penalty=fr.ctypes.data, u=u.ctypes.data,
                    stop_ids=None if keep["st"] is None else keep["st"].ctypes.data, n_stop=len(stops), step=keep["step"].ctypes.data,
                    frozen=keep["frozen"].ctypes.data, counts=keep["counts"].ctypes.data, tokens=keep["tokens"].ctypes.data,
                    next_tokens=keep["nxt"].ctypes.data, any_active=ctypes.addressof(keep["any_active"]))
    return a, keep


def result(keep, states):
    return (keep["step"].tobytes(), keep["frozen"].tobytes(), keep["counts"].tobytes(), keep["tokens"].tobytes(), keep["nxt"].tobytes(),
            keep["any_active"].value, None if states is None else states.tobytes())


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1, 7, 1000, 50277, 65536])
@pytest.mark.parametrize("top_n", [0, 1, 5, 20])
@pytest.mark.parametrize("table", [True, False], ids=["table", "no_table"])
def test_logprob_step_hook(lib, V, top_n, table):
    """One step at every instantiation, with a table (some rows constrained, some not) or with next = NULL (every row unconstrained
    through an all-NULL mask), against the step without log-probabilities and rwkv_b200_score_logits / sample_logits."""
    top_n = min(top_n, V)
    rng = np.random.RandomState(V * 31 + top_n)
    logits = hook_rows(rng, V, top_n)
    R = logits.shape[0]
    if table and V < 7:
        pytest.skip("the table rows need a few tokens")
    constrained = table
    table = None
    states = None
    if constrained:
        table = np.where(rng.rand(3, V) < 0.6, rng.randint(0, 3, size=(3, V)), bd.DEAD).astype(np.uint16)
        table[:, 0] = 0
        states = np.array([NONE if b % 3 == 0 else b % 3 for b in range(R)], np.uint32)
    max_tokens = [3] * R
    step = [b % 3 for b in range(R)]
    frozen = [0] * R
    temps = [[1.0, 0.0, 0.7, 1.3][b % 4] for b in range(R)]
    top_ps = [[1.0, 0.9, 0.5, 0.0][b % 4] for b in range(R)]
    pres, freq = [0.3 * (b % 2) for b in range(R)], [0.2 * (b % 3) for b in range(R)]
    n = 3
    us = rng.random_sample((R, n))
    counts = np.zeros((R, V), np.uint32)
    for b in range(R):
        ids = rng.choice(V, size=min(4, V), replace=False)
        counts[b, ids] = rng.randint(0, 3, size=len(ids))
    tokens = np.zeros((R, n), np.uint32)
    stops = [0] if V > 1 else []
    # the same step without log-probabilities
    a0, k0 = step_args(logits, max_tokens, temps, top_ps, pres, freq, us, stops, step, frozen, counts, tokens)
    s0 = None if states is None else states.copy()
    if constrained:
        assert lib.library.rwkv_b200_test_generate_step_constrained(ctypes.byref(a0), table.ctypes.data_as(P16), table.shape[0], s0.ctypes.data_as(P_U))
    else:
        assert lib.library.rwkv_b200_test_generate_step(ctypes.byref(a0))
    a1, k1 = step_args(logits, max_tokens, temps, top_ps, pres, freq, us, stops, step, frozen, counts, tokens)
    s1 = None if states is None else states.copy()
    out = Out(R, n, top_n)
    lps = out.struct()
    assert lib.library.rwkv_b200_test_generate_step_logprobs(ctypes.byref(a1), table.ctypes.data_as(P16) if constrained else None,
                                                             table.shape[0] if constrained else 0, ptr(s1, P_U), ctypes.byref(lps))
    assert result(k0, s0) == result(k1, s1)
    # sampling probabilities: rwkv_b200_sample_logits with the step's bias list
    for b in range(R):
        i = step[b]
        tok = int(k1["tokens"][b, i])
        cnt = {t: int(c) for t, c in enumerate(counts[b]) if c}
        bias = gr.penalty_bias(cnt, pres[b], freq[b]) if not constrained or states[b] == NONE else mask_bias(table[states[b]], cnt, pres[b], freq[b])
        ids, vals, nb = gr.bias_list(bias)
        t_ref, p_ref = ctypes.c_uint32(0), ctypes.c_float(0)
        assert lib.library.rwkv_b200_sample_logits(ptr(logits[b], P_F), V, temps[b], top_ps[b], float(us[b, i]), ids, vals, nb, ctypes.byref(t_ref),
                                                   ctypes.byref(p_ref))
        assert t_ref.value == tok, b
        assert out.sample_probs[b, i].tobytes() == np.float32(p_ref.value).tobytes(), (b, out.sample_probs[b, i], p_ref.value)
        check_entry(lib, logits[b], tok, out, b, i)
        others = [j for j in range(n) if j != i]                   # entries of other steps are not touched
        assert (out.logprobs[b, others] == 7.0).all() and (out.sample_probs[b, others] == 7.0).all()


# ---- 2. whole models -------------------------------------------------------------------------------------------------------------

FIXTURES = [(v, f) for v in ["4v0-660K", "5v1-730K", "5v2-730K", "6v0-3m", "7v0-834K"] for f in ["FP32", "Q5_1"]] + [("6v0-3m", "FP16")]
PROMPT = LONG_PROMPT[:24]


def host_logits_loop(lib, ctx_ptr, n_vocab, toks, presence, frequency):
    """The logits each token of `toks` was drawn from, by evaluating the tokens one at a time from the context's current state."""
    out = []
    for t in toks:
        out.append(logits(lib, ctx_ptr, n_vocab))
        gr.eval_token(lib, ctx_ptr, t)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("ver,fmt", FIXTURES)
def test_generate_logprobs_whole_model(lib, ver, fmt):
    ctx = lib.rwkv_init_from_file(model_path(ver, fmt), 1, 0)
    pair = Pair(lib, ctx)
    third = lib.rwkv_clone_context(ctx, 1)
    V = pair.n_vocab
    rng = np.random.RandomState(5)
    try:
        for (mt, temp, top_p, pres, freq), top_n in [((20, 1.0, 0.9, 0.3, 0.2), 5), ((12, 0.0, 1.0, 0.0, 0.0), 20), ((9, 0.8, 0.8, 0.0, 0.5), 0)]:
            us = rng.random_sample(mt)
            pair.prime(PROMPT)
            ok, want = generate(lib, pair.host.ptr, mt, temp, top_p, pres, freq, us)
            assert ok
            out = Out(1, mt, top_n)
            ok, got, _ = gen_logprobs(lib, pair.dev.ptr, out, mt, temp, top_p, pres, freq, us)
            assert ok and got == want
            pair.same((ver, fmt, "blocking"))
            # every entry against score_logits on the logits of a host loop over the same tokens
            prime(lib, third.ptr, PROMPT)
            for i, z in enumerate(host_logits_loop(lib, third.ptr, V, got, pres, freq)):
                check_entry(lib, z, got[i], out, 0, i)
            check_tail(out, 0, len(got))
            # rwkv_b200_score from the state before the prompt's last token runs the GEMV head below 32 tokens: the same bits
            prime(lib, third.ptr, PROMPT[:-1])
            toks = np.array([PROMPT[-1]] + got[:-1], np.uint32)
            lp = np.zeros(len(got), np.float32)
            assert lib.library.rwkv_b200_score(third.ptr, ptr(toks, P_U), ptr(np.array(got, np.uint32), P_U), len(got), ptr(lp, P_F), None)
            assert lp.tobytes() == out.logprobs[0, :len(got)].tobytes()
        # streaming: entry j is in the arrays when on_token(j) runs, and ending after token j gives max_tokens = j + 1
        mt, j = 14, 6
        us = rng.random_sample(mt)
        out = Out(1, mt, 5)
        seen = []
        rec = Recorder(stop_at={0: j}, inner=lambda s, i, t: seen.append((out.logprobs[0, i].tobytes(), out.tops(0, i), np.isnan(out.logprobs[0, i]))))
        pair.prime(PROMPT)
        ok, got, _ = gen_logprobs(lib, pair.dev.ptr, out, mt, 1.0, 1.0, 0.2, 0.2, us, rec=rec)
        assert ok and len(got) == j + 1 and rec.delivered(0) == got
        assert [s[0] for s in seen] == [out.logprobs[0, i].tobytes() for i in range(j + 1)] and [s[1] for s in seen] == [out.tops(0, i) for i in range(j + 1)]
        short = Out(1, j + 1, 5)
        ok, want, _ = gen_logprobs(lib, pair.host.ptr, short, j + 1, 1.0, 1.0, 0.2, 0.2, us[:j + 1])
        assert ok and want == got
        pair.same((ver, fmt, "stream"))
        assert out.logprobs[0, :j + 1].tobytes() == short.logprobs[0].tobytes() and out.sample_probs[0, :j + 1].tobytes() == short.sample_probs[0].tobytes()
        assert out.top_ids[0, :j + 1].tobytes() == short.top_ids[0].tobytes() and out.top_logprobs[0, :j + 1].tobytes() == short.top_logprobs[0].tobytes()
        check_tail(out, 0, j + 1)
        # constrained: the bytes of rwkv_b200_generate_constrained, automaton state included
        num = bd.ByteDFA(bd.NUMBER)
        auto = Automaton(lib, ctx.ptr, num.next)
        try:
            us = rng.random_sample(10)
            pair.prime(PROMPT)
            ok, want, st_want = gen_constrained(lib, pair.host.ptr, auto.ptr, 0, 10, 1.0, 1.0, 0.0, 0.0, us)
            assert ok
            out = Out(1, 10, 3)
            ok, got, st_got = gen_logprobs(lib, pair.dev.ptr, out, 10, 1.0, 1.0, 0.0, 0.0, us, auto=auto, st=0)
            assert ok and got == want and st_got == st_want
            pair.same((ver, fmt, "constrained"))
            prime(lib, third.ptr, PROMPT)
            for i, z in enumerate(host_logits_loop(lib, third.ptr, V, got, 0.0, 0.0)):
                check_entry(lib, z, got[i], out, 0, i)
            check_tail(out, 0, len(got))
        finally:
            auto.free()
    finally:
        lib.rwkv_free(third)
        pair.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_stop_id_entry_is_written(lib):
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "Q5_1"), 1, 0)
    try:
        us = np.full(10, 0.5)
        prime(lib, ctx.ptr, PROMPT)
        ok, greedy = generate(lib, ctx.ptr, 10, 0.0, 1.0, 0.0, 0.0, us)
        assert ok
        stop = greedy[3]
        k = greedy.index(stop)
        prime(lib, ctx.ptr, PROMPT)
        out = Out(1, 10, 4)
        ok, got, _ = gen_logprobs(lib, ctx.ptr, out, 10, 0.0, 1.0, 0.0, 0.0, us, stops=[stop])
        assert ok and got == greedy[:k + 1] and got[-1] == stop
        assert np.isfinite(out.logprobs[0, k]) and out.sample_probs[0, k] == 1.0 and out.tops(0, k)[0] == stop
        check_tail(out, 0, k + 1)
    finally:
        lib.rwkv_free(ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [4, 16])
def test_batch_generate_logprobs(lib, B):
    """Rows of a batch give the bytes of rwkv_b200_batch_generate; their logprobs are score_logits of each row's logits column, which
    a step-by-step rwkv_b200_batch_eval of the same tokens reproduces (16 rows: the tensor-core path of the layer matrices). With 4
    rows each row also equals the sequence alone."""
    path = model_path("6v0-3m", "Q5_1")
    ctx = lib.rwkv_init_from_file(path, 1, 0)
    a, b2, ref = Batch(lib, ctx, B), Batch(lib, ctx, B), Batch(lib, ctx, B)
    V = lib.rwkv_get_logits_buffer_element_count(ctx)
    rng = np.random.RandomState(B)
    try:
        prompts = [LONG_PROMPT[i:i + 6] for i in range(B)]
        n = 8
        temps, top_ps = [1.0] * B, [[1.0, 0.9][b % 2] for b in range(B)]
        pres, freq = [0.2] * B, [0.1] * B
        us = rng.random_sample((B, n))
        a.prime(prompts); b2.prime(prompts); ref.prime(prompts)
        ok, want = a.generate([n] * B, temps, top_ps, pres, freq, us, [])
        assert ok
        out = Out(B, n, 5)
        ok, got = batch_logprobs(b2, out, [n] * B, temps, top_ps, pres, freq, us)
        assert ok and got == want
        n_state = lib.rwkv_get_state_buffer_element_count(ctx)
        for b in range(B):
            assert a.state(b, n_state).tobytes() == b2.state(b, n_state).tobytes() and a.logits(b, V).tobytes() == b2.logits(b, V).tobytes()
        for i in range(n):
            for b in range(B):
                check_entry(lib, ref.logits(b, V), got[b][i], out, b, i)
            assert ref.eval([got[b][i] for b in range(B)])
        if B == 4:
            for b in range(B):
                single = lib.rwkv_clone_context(ctx, 1)
                prime(lib, single.ptr, prompts[b])
                alone = Out(1, n, 5)
                ok, toks, _ = gen_logprobs(lib, single.ptr, alone, n, temps[b], top_ps[b], pres[b], freq[b], us[b])
                lib.rwkv_free(single)
                assert ok and toks == got[b]
                for arr in ("logprobs", "sample_probs", "top_ids", "top_logprobs"):
                    assert getattr(alone, arr)[0].tobytes() == getattr(out, arr)[b].tobytes(), (b, arr)
    finally:
        a.free(); b2.free(); ref.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_logprob_refusals_change_nothing(lib):
    import rwkv_cpp_b200.shared_library as sl
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "Q5_1"), 1, 0)
    pair = Pair(lib, ctx)
    try:
        us = np.full(6, 0.3)
        pair.prime(PROMPT)
        # counts in both contexts, so that a refused call's effect on them would show in a keep_counts call below
        assert generate(lib, pair.host.ptr, 3, 1.0, 1.0, 0.5, 0.5, us)[0] and generate(lib, pair.dev.ptr, 3, 1.0, 1.0, 0.5, 0.5, us)[0]
        out = Out(1, 6, 5)
        bad = [False, out.struct(logprobs=None), out.struct(top_n=21), out.struct(top_ids=None), out.struct(top_logprobs=None)]
        for lp in bad:
            for rec in (None, Recorder()):
                ok, toks, _ = gen_logprobs(lib, pair.dev.ptr, out, 6, 1.0, 1.0, 0.5, 0.5, us, keep=True, rec=rec, lp=lp)
                assert not ok and toks == [] and lib.rwkv_get_last_error(pair.dev) == ERR_ARGS
                assert rec is None or rec.calls == []
        assert (out.logprobs == 7.0).all()
        pair.same("refused")
        ok1, t1 = generate(lib, pair.host.ptr, 6, 1.0, 1.0, 0.5, 0.5, us, keep=True)
        ok2, t2 = generate(lib, pair.dev.ptr, 6, 1.0, 1.0, 0.5, 0.5, us, keep=True)
        assert ok1 and ok2 and t1 == t2
        # top_n above n_vocab, through the step hook at V = 7
        logits_ = np.zeros((1, 7), np.float32)
        a, keep = step_args(logits_, [1], [1.0], [1.0], [0.0], [0.0], np.full((1, 1), 0.5), [], [0], [0], np.zeros((1, 7), np.uint32), np.zeros((1, 1), np.uint32))
        o = Out(1, 1, 8)
        assert not lib.library.rwkv_b200_test_generate_step_logprobs(ctypes.byref(a), None, 0, None, ctypes.byref(o.struct()))
        assert lib.rwkv_get_last_error(None) == ERR_ARGS and keep["step"][0] == 0
    finally:
        pair.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_batch_stream_entries_are_in_place_before_each_callback(lib):
    """Streaming in a batch of 4: when on_token(b, i) runs, entry [b][i] of every output array already holds its final value and no
    entry delivered before it has changed; ending row b after token j_b gives the outputs of max_tokens[b] = j_b + 1."""
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "Q5_1"), 1, 0)
    B, n = 4, 10
    live, ref = Batch(lib, ctx, B), Batch(lib, ctx, B)
    rng = np.random.RandomState(11)
    try:
        prompts = [LONG_PROMPT[i:i + 6] for i in range(B)]
        temps, top_ps, pres, freq = [1.0] * B, [1.0, 0.9, 1.0, 0.8], [0.2] * B, [0.1] * B
        us = rng.random_sample((B, n))
        end_at = {0: 3, 1: 0, 2: 9, 3: 6}           # row 2 runs to its budget
        out = Out(B, n, 5)
        snap = {}

        def entry(b, i):
            return (out.logprobs[b, i].tobytes(), out.sample_probs[b, i].tobytes(), out.top_ids[b, i].tobytes(), out.top_logprobs[b, i].tobytes())

        def inner(b, i, t):
            for key, val in snap.items():           # nothing delivered earlier was overwritten
                assert entry(*key) == val, ("changed", key, (b, i))
            snap[(int(b), int(i))] = entry(b, i)

        rec = Recorder(stop_at=end_at, inner=inner)
        live.prime(prompts)
        ok, got = batch_logprobs(live, out, [n] * B, temps, top_ps, pres, freq, us, rec=rec)
        assert ok and [len(g) for g in got] == [end_at[b] + 1 for b in range(B)]
        for b in range(B):
            assert rec.delivered(b) == got[b]
            for i in range(len(got[b])):
                assert snap[(b, i)] == entry(b, i), (b, i)
            check_tail(out, b, len(got[b]))
        short = Out(B, n, 5)
        ref.prime(prompts)
        budgets = [end_at[b] + 1 for b in range(B)]
        m = max(budgets)
        ok, want = batch_logprobs(ref, short, budgets, temps, top_ps, pres, freq, us[:, :m])
        assert ok and want == got
        for b in range(B):
            k = budgets[b]
            for arr in ("logprobs", "sample_probs", "top_ids", "top_logprobs"):
                assert getattr(out, arr)[b, :k].tobytes() == getattr(short, arr)[b, :k].tobytes(), (b, arr)
    finally:
        live.free(); ref.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_batch_logprobs_with_automata(lib):
    """A batch of 4 with automata [number, NULL, words, NULL]: tokens, states and logits are those of
    rwkv_b200_batch_generate_constrained, and every row's outputs are those of the sequence alone through rwkv_b200_generate_logprobs
    (its automaton, or none)."""
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "Q5_1"), 1, 0)
    B, n = 4, 10
    num, words = bd.ByteDFA(bd.NUMBER), bd.ByteDFA(bd.WORDS, eos=0)
    a_num, a_words = Automaton(lib, ctx.ptr, num.next), Automaton(lib, ctx.ptr, words.next)
    plain, lp_bt = Batch(lib, ctx, B), Batch(lib, ctx, B)
    V, n_state = lib.rwkv_get_logits_buffer_element_count(ctx), lib.rwkv_get_state_buffer_element_count(ctx)
    rng = np.random.RandomState(13)
    try:
        prompts = [LONG_PROMPT[i:i + 6] for i in range(B)]
        autos = [a_num, None, a_words, None]
        temps, top_ps, pres, freq = [1.0, 0.8, 1.0, 0.0], [1.0, 0.9, 0.9, 1.0], [0.0, 0.2, 0.1, 0.0], [0.0, 0.1, 0.3, 0.0]
        us = rng.random_sample((B, n))
        plain.prime(prompts)
        ok, want, st_want = batch_constrained(plain, autos, [0] * B, [n] * B, temps, top_ps, pres, freq, us)
        assert ok
        lp_bt.prime(prompts)
        out = Out(B, n, 5)
        toks = np.zeros(B * n, np.uint32)
        ng = np.zeros(B, np.uint32)
        st = np.zeros(B, np.uint32)
        arr = (ctypes.c_void_p * B)(*[a.ptr if a else None for a in autos])
        lps = out.struct()
        assert lib.library.rwkv_b200_batch_generate_logprobs(
            lp_bt.ptr, arr, ptr(st, P_U), ptr(np.full(B, n, np.uint32), P_U), ptr(f32(temps), P_F), ptr(f32(top_ps), P_F), ptr(f32(pres), P_F),
            ptr(f32(freq), P_F), None, ptr(np.ascontiguousarray(us, np.float64), P_D), None, 0, NULL_FN, None, ptr(toks, P_U), ptr(ng, P_U), ctypes.byref(lps))
        got = [[int(t) for t in toks[b * n:b * n + ng[b]]] for b in range(B)]
        assert got == want and [int(x) for x in st] == st_want
        for b in range(B):
            assert plain.state(b, n_state).tobytes() == lp_bt.state(b, n_state).tobytes() and plain.logits(b, V).tobytes() == lp_bt.logits(b, V).tobytes()
            check_tail(out, b, len(got[b]))
            single = lib.rwkv_clone_context(ctx, 1)
            prime(lib, single.ptr, prompts[b])
            alone = Out(1, n, 5)
            ok, t1, s1 = gen_logprobs(lib, single.ptr, alone, n, temps[b], top_ps[b], pres[b], freq[b], us[b], auto=autos[b], st=0)
            lib.rwkv_free(single)
            assert ok and t1 == got[b] and (autos[b] is None or s1 == st_want[b])
            for name in ("logprobs", "sample_probs", "top_ids", "top_logprobs"):
                assert getattr(alone, name)[0].tobytes() == getattr(out, name)[b].tobytes(), (b, name)
    finally:
        plain.free(); lp_bt.free()
        a_num.free(); a_words.free()
        lib.rwkv_free(ctx)
