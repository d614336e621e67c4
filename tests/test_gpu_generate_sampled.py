"""Generation with a per-sequence sampler (rwkv_b200_generate_sampled / rwkv_b200_batch_generate_sampled, the sampled step kernels of
csrc/kernels/sampling.cu): with top_k, min_p and the user bias off every call gives the bits of the existing generate call it
extends; with them on, one draw follows the float64 rules of tests/sampler_ref.py, and a whole call equals the host loop of the
step hook plus rwkv_b200_eval_resident (rwkv_b200_batch_eval for a batch)."""
import ctypes
from collections import Counter

import numpy as np
import pytest

import byte_dfa as bd
import generate_ref as gr
from conftest import LONG_PROMPT, model_path
from generate_ref import P_D, P_F, P_U
from sampler_ref import kept_mask, sampler_bias
from sampling_oracle import probs64
from test_gpu_generate import ERR_ARGS, P_U8, Batch, Pair, generate, logits, ptr, state
from test_gpu_generate_constrained import NONE, P16, Automaton, batch_constrained, gen_constrained
from test_gpu_generate_logprobs import Out, batch_logprobs, check_entry, gen_logprobs
from test_gpu_generate_stream import NULL_FN, Recorder, batch_generate_stream, generate_stream

PROMPT = LONG_PROMPT[:24]
VERSIONS = ["4v0-660K", "5v1-730K", "5v2-730K", "6v0-3m", "7v0-834K"]


class Smp:
    """One sequence's sampler; keeps its bias arrays alive."""

    def __init__(self, T=1.0, top_p=1.0, top_k=0, min_p=0.0, pres=0.0, freq=0.0, bias=None):
        self.T, self.top_p, self.top_k, self.min_p, self.pres, self.freq, self.bias = T, top_p, top_k, min_p, pres, freq, dict(bias or {})
        self.ids = np.array(list(self.bias.keys()), np.uint32)
        self.vals = np.array(list(self.bias.values()), np.float32)

    def struct(self):
        import rwkv_cpp_b200.shared_library as sl
        n = len(self.ids)
        return sl.Sampler(temperature=self.T, top_p=self.top_p, top_k=self.top_k, min_p=self.min_p, presence_penalty=self.pres,
                          frequency_penalty=self.freq, n_bias=n, bias_ids=ptr(self.ids, P_U) if n else None, bias_values=ptr(self.vals, P_F) if n else None)


def gen_sampled(lib, ctx_ptr, smp, max_tokens, us, stops=(), keep=False, rec=None, auto=None, st=0, out=None):
    toks = np.zeros(max(max_tokens, 1), np.uint32)
    n = ctypes.c_size_t(0)
    s = np.array([st], np.uint32)
    sp = np.array(stops, np.uint32) if len(stops) else None
    sm = smp.struct() if smp is not None else None
    lps = out.struct() if out is not None else None
    ok = lib.library.rwkv_b200_generate_sampled(ctx_ptr, ctypes.byref(sm) if sm is not None else None, auto.ptr if auto else None, ptr(s, P_U), max_tokens,
                                                keep, ptr(np.asarray(us, np.float64), P_D), ptr(sp, P_U), len(stops), rec.fn if rec else NULL_FN, None,
                                                ptr(toks, P_U), ctypes.byref(n), ctypes.byref(lps) if lps is not None else None)
    return ok, [int(t) for t in toks[:n.value]], int(s[0])


def batch_sampled(bt, smps, max_tokens, us, stops=(), rec=None, automata=None, states=None, out=None, keep=None):
    import rwkv_cpp_b200.shared_library as sl
    n = max(max_tokens)
    toks = np.zeros(bt.n * max(n, 1), np.uint32)
    ng = np.zeros(bt.n, np.uint32)
    st = np.array(states if states is not None else [0] * bt.n, np.uint32)
    arr = (sl.Sampler * bt.n)(*[s.struct() for s in smps])
    autos = (ctypes.c_void_p * bt.n)(*[a.ptr if a else None for a in automata]) if automata is not None else None
    sp = np.array(stops, np.uint32) if len(stops) else None
    lps = out.struct() if out is not None else None
    ok = bt.lib.library.rwkv_b200_batch_generate_sampled(
        bt.ptr, arr, autos, ptr(st, P_U), ptr(np.asarray(max_tokens, np.uint32), P_U), ptr(None if keep is None else np.asarray(keep, np.uint8), P_U8),
        ptr(np.ascontiguousarray(us, np.float64), P_D), ptr(sp, P_U), len(stops), rec.fn if rec else NULL_FN, None, ptr(toks, P_U), ptr(ng, P_U),
        ctypes.byref(lps) if lps is not None else None)
    return ok, [[int(t) for t in toks[b * n:b * n + ng[b]]] for b in range(bt.n)], [int(x) for x in st]


def hook(lib, logits_rows, smps, us, counts, table=None, states=None, out=None, step=0, n=1):
    """One step of the sampled kernel at `step` of n for every row; returns (tokens [R], counts after, states after)."""
    import rwkv_cpp_b200.shared_library as sl
    R, V = logits_rows.shape
    lg = np.ascontiguousarray(logits_rows, np.float32)
    keep = dict(mt=np.full(R, n, np.uint32), st=np.full(R, step, np.uint32), fr=np.zeros(R, np.uint8), cnt=np.ascontiguousarray(counts, np.uint32).copy(),
                tk=np.zeros((R, n), np.uint32), nx=np.zeros(R, np.int32), u=np.ascontiguousarray(us, np.float64).reshape(R, n), act=ctypes.c_uint32(0))
    a = gr.StepArgs(logits=lg.ctypes.data, n_rows=R, n_vocab=V, max_tokens=keep["mt"].ctypes.data, temperature=None, top_p=None, presence_penalty=None,
                    frequency_penalty=None, u=keep["u"].ctypes.data, stop_ids=None, n_stop=0, step=keep["st"].ctypes.data, frozen=keep["fr"].ctypes.data,
                    counts=keep["cnt"].ctypes.data, tokens=keep["tk"].ctypes.data, next_tokens=keep["nx"].ctypes.data, any_active=ctypes.addressof(keep["act"]))
    arr = (sl.Sampler * R)(*[s.struct() for s in smps])
    s = None if states is None else np.array(states, np.uint32)
    lps = out.struct() if out is not None else None
    assert lib.library.rwkv_b200_test_generate_step_sampled(ctypes.byref(a), arr, None if table is None else table.ctypes.data_as(P16),
                                                           0 if table is None else table.shape[0], ptr(s, P_U), ctypes.byref(lps) if lps is not None else None), \
        lib.rwkv_get_last_error(None)
    return [int(t) for t in keep["tk"][:, step]], keep["cnt"], s


def sample_logits(lib, z, T, top_p, u, bias):
    ids, vals, nb = gr.bias_list(bias)
    t, p = ctypes.c_uint32(0), ctypes.c_float(0)
    assert lib.library.rwkv_b200_sample_logits(ptr(np.ascontiguousarray(z, np.float32), P_F), len(z), T, top_p, float(u), ids, vals, nb, ctypes.byref(t),
                                               ctypes.byref(p))
    return int(t.value), np.float32(p.value)


# ---- 1. the step hook against the float64 rules ----------------------------------------------------------------------------------

def oracle_check(z, smp, bias, u, tok, prob):
    """tok / prob against rules 2-5 in float64. A token or threshold within rounding of a filter's edge (the float32 kernel may decide
    it either way) leaves only 'tok is kept by the looser reading'; otherwise tok must own u in the float64 CDF and prob must be the
    float64 probability."""
    p = probs64(z, 1.0, 1.0, bias)
    T, k, mp = smp.T, smp.top_k, smp.min_p
    keep = kept_mask(p, smp.top_p, k, mp)
    # tokens the float32 kernel may place on either side of a threshold: within 1e-5 of it without being equal to it (equal logits give
    # equal probabilities in both precisions), or on either side of a top-p cutoff moved by 1e-5
    amb = np.zeros(p.size, bool)
    for thr in ([np.sort(p)[::-1][k - 1]] if k else []) + ([mp * p.max()] if mp else []):
        amb |= (np.abs(p - thr) <= 1e-5 * thr) & (p != thr)
    if 0 < smp.top_p < 1:
        amb |= kept_mask(p, smp.top_p * (1 - 1e-5)) != kept_mask(p, smp.top_p * (1 + 1e-5))
    assert (keep | amb)[tok] and p[tok] > 0, (tok, p[tok])
    if amb.any():
        return "edge"
    strict = keep
    q = np.where(strict, p, 0.0)
    kept = q > 0
    lq = np.full(q.size, -np.inf)
    lq[kept] = np.log(q[kept])
    q = np.exp((lq - lq[kept].max()) / T)
    q /= q.sum()
    cdf = np.cumsum(q)
    cdf /= cdf[-1]
    left = cdf[tok - 1] if tok > 0 else 0.0
    eps = 1e-5 * max(1.0, 1.0 / T)
    assert left - eps <= u < cdf[tok] + eps, (tok, u, left, cdf[tok])
    assert abs(float(prob) - q[tok]) <= 1e-4 * max(1.0, 1.0 / T) * q[tok] + 1e-30, (tok, prob, q[tok])
    return "checked"


def hook_cases(rng, V):
    """(logits, sampler, counts, state) rows: every filter at temperatures 0.3, 1 and 4 with top-p 1 and 0.7, then the rows whose
    draw the filters must leave alone."""
    k_mid = min(40, V)
    rows = []
    for T in (0.3, 1.0, 4.0):
        for tp in (1.0, 0.7):
            z = rng.standard_normal(V) * 2.0
            rows.append((z, Smp(T, tp, top_k=1), {}))                                     # k = 1, unique maximum: greedy
            z = rng.standard_normal(V) * 2.0
            z[rng.choice(V, size=min(3, V), replace=False)] = z.max() + 1.0
            rows.append((z, Smp(T, tp, top_k=1), {}))                                     # k = 1, tied maxima
            rows.append((rng.standard_normal(V) * 2.0, Smp(T, tp, top_k=V), {}))          # k = n_vocab
            z = rng.standard_normal(V) * 2.0
            order = np.argsort(-z)
            z[order[max(k_mid - 3, 0):k_mid + 2]] = z[order[k_mid - 1]]                   # equal logits straddle the k-th value
            rows.append((z, Smp(T, tp, top_k=k_mid), {}))
            rows.append((rng.standard_normal(V) * 2.0, Smp(T, tp, min_p=1e-6), {}))
            z = rng.standard_normal(V) * 2.0
            z[rng.choice(V, size=min(2, V), replace=False)] = z.max() + 0.5
            rows.append((z, Smp(T, tp, min_p=1.0), {}))
            nb = min(300, V)
            ids = rng.choice(V, size=nb, replace=False)
            vals = np.where(rng.rand(nb) < 0.2, -np.inf, rng.standard_normal(nb) * 3.0).astype(np.float32)
            vals[0] = 5.0
            cnt = {int(i): int(rng.randint(1, 4)) for i in ids[:min(10, nb)]}
            cnt.update({int(i): 2 for i in rng.choice(V, size=min(5, V), replace=False)})
            rows.append((rng.standard_normal(V) * 2.0, Smp(T, tp, top_k=k_mid, min_p=0.05, pres=0.4, freq=0.3, bias=dict(zip(ids.tolist(), vals.tolist()))), cnt))
    return rows


def plain_cases(rng, V):
    """Rows that must draw exactly as rwkv_b200_sample_logits does with the rule-1 bias list: filters off with user bias, temperature 0,
    and columns with a NaN or +inf (filters on)."""
    nb = min(50, V)
    ids = rng.choice(V, size=nb, replace=False)
    bias = dict(zip(ids.tolist(), np.where(rng.rand(nb) < 0.3, -np.inf, rng.standard_normal(nb) * 2).astype(np.float32).tolist()))
    cnt = {int(i): 1 for i in ids[:min(5, nb)]}
    rows = [(rng.standard_normal(V) * 2.0, Smp(0.9, 0.8, pres=0.2, freq=0.5, bias=bias), cnt),
            (rng.standard_normal(V) * 2.0, Smp(1.0, 1.0, bias=bias), {}),
            (rng.standard_normal(V) * 2.0, Smp(0.0, 0.5, top_k=min(3, V), min_p=0.5, bias=bias), cnt)]
    z = rng.standard_normal(V); z[V // 2] = np.nan
    rows.append((z, Smp(1.0, 0.9, top_k=min(5, V), min_p=0.1), {}))
    z = rng.standard_normal(V); z[V - 1] = np.inf
    rows.append((z, Smp(0.7, 1.0, top_k=min(5, V), min_p=0.1), {}))
    return rows


@pytest.mark.gpu
@pytest.mark.parametrize("V", [1, 4, 1000, 50277, 65536])
def test_sampled_step_hook(lib, V):
    rng = np.random.RandomState(V)
    cases, plain = hook_cases(rng, V), plain_cases(rng, V)
    rows = cases + plain
    banned = V >= 4
    if banned:      # state 1 allows tokens 0 .. 2 and the user bias bans all three; every other row is unconstrained
        table = np.zeros((2, V), np.uint16)
        table[1, 3:] = bd.DEAD
        rows.append((rng.standard_normal(V), Smp(1.0, 1.0, top_k=2, min_p=0.1, bias={0: -np.inf, 1: -np.inf, 2: -np.inf}), {}))
    R = len(rows)
    z = np.array([r[0] for r in rows], np.float32)
    counts = np.zeros((R, V), np.uint32)
    for b, (_, _, cnt) in enumerate(rows):
        for t, c in cnt.items():
            counts[b, t] = c
    us = rng.random_sample(R)
    states = [NONE] * (R - 1) + [1] if banned else None
    out = Out(R, 1, min(3, V))
    toks, _, _ = hook(lib, z, [r[1] for r in rows], us, counts, table if banned else None, states, out)
    done = Counter()
    for b, (_, smp, cnt) in enumerate(rows):
        allowed = (table[1] != bd.DEAD) if banned and b == R - 1 else None
        bias = sampler_bias(cnt, smp.pres, smp.freq, smp.bias, allowed)
        if b < len(cases) and V > 1:
            done[oracle_check(z[b], smp, bias, us[b], toks[b], out.sample_probs[b, 0])] += 1
        else:       # rule 1's bias list through rwkv_b200_sample_logits, bit for bit
            t, p = sample_logits(lib, z[b], smp.T, smp.top_p, us[b], bias)
            assert toks[b] == t and out.sample_probs[b, 0].tobytes() == p.tobytes(), (b, toks[b], t)
        check_entry(lib, z[b], toks[b], out, b, 0)
    assert V == 1 or done["checked"] >= len(cases) // 3, done


# ---- 2. identity with the filters off --------------------------------------------------------------------------------------------

def off(T, tp, pres, freq):
    return Smp(T, tp, pres=pres, freq=freq)


@pytest.mark.gpu
@pytest.mark.parametrize("ver", VERSIONS)
def test_filters_off_is_every_existing_call(lib, ver):
    ctx = lib.rwkv_init_from_file(model_path(ver, "Q5_1"), 1, 0)
    pair = Pair(lib, ctx)
    rng = np.random.RandomState(3)
    try:
        for mt, T, tp, pres, freq in [(9, 1.0, 0.8, 0.2, 0.2), (8, 0.0, 1.0, 0.0, 0.0), (7, 0.6, 1.0, 0.3, 0.1)]:
            us = rng.random_sample(mt)
            pair.prime(PROMPT)
            ok, want = generate(lib, pair.host.ptr, mt, T, tp, pres, freq, us)
            ok2, got, _ = gen_sampled(lib, pair.dev.ptr, off(T, tp, pres, freq), mt, us)
            assert ok and ok2 and got == want
            pair.same((ver, "generate"))
            # keep_counts: a second call continues from the counts of the first on both sides
            ok, want = generate(lib, pair.host.ptr, mt, T, tp, pres, freq, us, keep=True)
            ok2, got, _ = gen_sampled(lib, pair.dev.ptr, off(T, tp, pres, freq), mt, us, keep=True)
            assert ok and ok2 and got == want
            pair.same((ver, "keep_counts"))
            pair.prime(PROMPT)
            r1, r2 = Recorder(stop_at={0: 4}), Recorder(stop_at={0: 4})
            ok, want = generate_stream(lib, pair.host.ptr, mt, T, tp, pres, freq, us, rec=r1)
            ok2, got, _ = gen_sampled(lib, pair.dev.ptr, off(T, tp, pres, freq), mt, us, rec=r2)
            assert ok and ok2 and got == want and r1.calls == r2.calls
            pair.same((ver, "stream"))
            pair.prime(PROMPT)
            o1, o2 = Out(1, mt, 5), Out(1, mt, 5)
            ok, want, _ = gen_logprobs(lib, pair.host.ptr, o1, mt, T, tp, pres, freq, us)
            ok2, got, _ = gen_sampled(lib, pair.dev.ptr, off(T, tp, pres, freq), mt, us, out=o2)
            assert ok and ok2 and got == want
            for f in ("logprobs", "sample_probs", "top_ids", "top_logprobs"):
                assert getattr(o1, f).tobytes() == getattr(o2, f).tobytes(), f
            pair.same((ver, "logprobs"))
        num = bd.ByteDFA(bd.NUMBER)
        auto = Automaton(lib, ctx.ptr, num.next)
        try:
            us = rng.random_sample(10)
            pair.prime(PROMPT)
            ok, want, st_want = gen_constrained(lib, pair.host.ptr, auto.ptr, 0, 10, 1.0, 1.0, 0.1, 0.1, us)
            ok2, got, st_got = gen_sampled(lib, pair.dev.ptr, off(1.0, 1.0, 0.1, 0.1), 10, us, auto=auto, st=0)
            assert ok and ok2 and got == want and st_got == st_want
            pair.same((ver, "constrained"))
        finally:
            auto.free()
    finally:
        pair.free()
        lib.rwkv_free(ctx)


def batch_same(b1, b2, n_state, n_vocab, what):
    for b in range(b1.n):
        assert b1.state(b, n_state).tobytes() == b2.state(b, n_state).tobytes(), (what, "state", b)
        assert b1.logits(b, n_vocab).tobytes() == b2.logits(b, n_vocab).tobytes(), (what, "logits", b)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 4, 16, 32])
def test_batch_filters_off_is_every_existing_call(lib, B):
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "Q5_1"), 1, 0)
    n_state, V = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
    b1, b2 = Batch(lib, ctx, B), Batch(lib, ctx, B)
    rng = np.random.RandomState(B)
    prompts = [[PROMPT[(i + b) % len(PROMPT)] for i in range(6)] for b in range(B)]
    try:
        mts = [int(x) for x in rng.randint(0, 9, size=B)]
        mts[0] = 8
        n = max(mts)
        temps, tps = [float(x) for x in rng.choice([0.0, 0.7, 1.0], size=B)], [float(x) for x in rng.choice([1.0, 0.8], size=B)]
        pres, freq = [0.2 * (b % 2) for b in range(B)], [0.1 * (b % 3) for b in range(B)]
        us = rng.random_sample((B, n))
        smps = [off(temps[b], tps[b], pres[b], freq[b]) for b in range(B)]
        b1.prime(prompts); b2.prime(prompts)
        ok, want = b1.generate(mts, temps, tps, pres, freq, us, [])
        ok2, got, _ = batch_sampled(b2, smps, mts, us)
        assert ok and ok2 and got == want
        batch_same(b1, b2, n_state, V, "generate")
        b1.prime(prompts); b2.prime(prompts)
        stop_at = {b: 2 for b in range(0, B, 3)}
        r1, r2 = Recorder(stop_at=stop_at), Recorder(stop_at=stop_at)
        ok, want = batch_generate_stream(b1, mts, temps, tps, pres, freq, us, [], r1)
        ok2, got, _ = batch_sampled(b2, smps, mts, us, rec=r2)
        assert ok and ok2 and got == want and sorted(r1.calls) == sorted(r2.calls)
        batch_same(b1, b2, n_state, V, "stream")
        b1.prime(prompts); b2.prime(prompts)
        o1, o2 = Out(B, n, 3), Out(B, n, 3)
        ok, want = batch_logprobs(b1, o1, mts, temps, tps, pres, freq, us)
        ok2, got, _ = batch_sampled(b2, smps, mts, us, out=o2)
        assert ok and ok2 and got == want
        for f in ("logprobs", "sample_probs", "top_ids", "top_logprobs"):
            assert getattr(o1, f).tobytes() == getattr(o2, f).tobytes(), f
        batch_same(b1, b2, n_state, V, "logprobs")
        num = bd.ByteDFA(bd.NUMBER)
        auto = Automaton(lib, ctx.ptr, num.next)
        try:
            automata = [auto if b % 2 == 0 else None for b in range(B)]
            b1.prime(prompts); b2.prime(prompts)
            ok, want, st1 = batch_constrained(b1, automata, [0] * B, mts, temps, tps, pres, freq, us)
            ok2, got, st2 = batch_sampled(b2, smps, mts, us, automata=automata, states=[0] * B)
            assert ok and ok2 and got == want and st1 == st2
            batch_same(b1, b2, n_state, V, "constrained")
        finally:
            auto.free()
    finally:
        b1.free(); b2.free()
        lib.rwkv_free(ctx)


# ---- 3. filters on against the host loop of the step hook ------------------------------------------------------------------------

ON = [Smp(1.0, 1.0, top_k=40, pres=0.3, freq=0.2), Smp(0.8, 0.9, min_p=0.05, pres=0.2, freq=0.2),
      Smp(1.2, 0.95, top_k=40, min_p=0.05, pres=0.4, freq=0.3, bias={32: 3.0, 101: -np.inf, 48: 1.5, 49: -2.0, 10: 2.5})]


@pytest.mark.gpu
@pytest.mark.parametrize("ver", VERSIONS)
def test_filters_on_equal_the_host_loop(lib, ver):
    ctx = lib.rwkv_init_from_file(model_path(ver, "Q5_1"), 1, 0)
    pair = Pair(lib, ctx)
    V = pair.n_vocab
    rng = np.random.RandomState(11)
    try:
        for smp in ON:
            mt = 12
            us = rng.random_sample(2 * mt)
            pair.prime(PROMPT)
            counts = np.zeros((1, V), np.uint32)
            want, zs = [], []
            hook_out = Out(1, 1, 0)
            probs = []
            for half in range(2):       # two calls, the second with keep_counts
                for i in range(mt):
                    z = logits(lib, pair.host.ptr, V)
                    zs.append(z)
                    (tok,), counts, _ = hook(lib, z[None, :], [smp], [us[half * mt + i]], counts, out=hook_out)
                    probs.append(hook_out.sample_probs[0, 0].copy())
                    want.append(tok)
                    gr.eval_token(lib, pair.host.ptr, tok)
            out = Out(1, mt, 4)
            ok, got1, _ = gen_sampled(lib, pair.dev.ptr, smp, mt, us[:mt], out=out)
            assert ok
            sp1 = out.sample_probs[0].copy()
            for i in range(mt):
                check_entry(lib, zs[i], got1[i], out, 0, i)
            ok, got2, _ = gen_sampled(lib, pair.dev.ptr, smp, mt, us[mt:], keep=True)
            assert ok and got1 + got2 == want
            assert np.array(probs[:mt], np.float32).tobytes() == sp1.tobytes()
            pair.same((ver, smp.top_k, smp.min_p))
        # streaming, ended after token j, equals max_tokens = j + 1
        smp, mt, j = ON[2], 14, 5
        us = rng.random_sample(mt)
        pair.prime(PROMPT)
        rec = Recorder(stop_at={0: j})
        ok, got, _ = gen_sampled(lib, pair.dev.ptr, smp, mt, us, rec=rec)
        assert ok and len(got) == j + 1 and rec.delivered(0) == got
        ok, want, _ = gen_sampled(lib, pair.host.ptr, smp, j + 1, us[:j + 1])
        assert ok and want == got
        pair.same((ver, "stream"))
    finally:
        pair.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_batch_filters_on_equal_the_host_loop(lib):
    ctx = lib.rwkv_init_from_file(model_path("7v0-834K", "Q5_1"), 1, 0)
    n_state, V = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
    B, mt = 4, 10
    host, dev = Batch(lib, ctx, B), Batch(lib, ctx, B)
    rng = np.random.RandomState(7)
    prompts = [[PROMPT[(i + 3 * b) % len(PROMPT)] for i in range(5)] for b in range(B)]
    smps = ON + [Smp(0.9, 1.0)]
    try:
        us = rng.random_sample((B, mt))
        host.prime(prompts); dev.prime(prompts)
        counts = np.zeros((B, V), np.uint32)
        want = [[] for _ in range(B)]
        for i in range(mt):
            z = np.array([host.logits(b, V) for b in range(B)])
            toks, counts, _ = hook(lib, z, smps, us[:, i], counts)
            for b in range(B):
                want[b].append(toks[b])
            assert host.eval(toks)
        ok, got, _ = batch_sampled(dev, smps, [mt] * B, us)
        assert ok and got == want
        batch_same(host, dev, n_state, V, "filters on")
    finally:
        host.free(); dev.free()
        lib.rwkv_free(ctx)


# ---- 4. refusals -----------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_sampled_refusals_change_nothing(lib):
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "Q5_1"), 1, 0)
    pair = Pair(lib, ctx)
    V = pair.n_vocab
    num = bd.ByteDFA(bd.NUMBER)
    auto = Automaton(lib, ctx.ptr, num.next)
    bt = Batch(lib, ctx, 2)
    try:
        us = np.full(6, 0.5)
        pair.prime(PROMPT)
        ok, _, _ = gen_sampled(lib, pair.dev.ptr, Smp(1.0, 1.0, pres=0.5, freq=0.5), 6, us)      # leaves counts behind
        assert ok
        ok, _, _ = gen_sampled(lib, pair.host.ptr, Smp(1.0, 1.0, pres=0.5, freq=0.5), 6, us)
        assert ok
        bad = [None, Smp(top_k=V + 1), Smp(min_p=float("nan")), Smp(min_p=1.5), Smp(bias={V: 1.0}), Smp(bias={1: float("nan")}),
               Smp(bias={1: float("inf")})]
        many, dup = Smp(), Smp(bias={1: 1.0, 2: 1.0})
        many.ids, many.vals = np.arange(1025, dtype=np.uint32) % V, np.zeros(1025, np.float32)     # one more entry than the maximum
        dup.ids = np.array([1, 1], np.uint32)
        bad += [many, dup]
        for s in bad:
            st = state(lib, pair.dev.ptr, pair.n_state).tobytes(), logits(lib, pair.dev.ptr, V).tobytes()
            ok, toks, a_st = gen_sampled(lib, pair.dev.ptr, s, 6, us, auto=auto, st=2, keep=True)
            assert not ok and toks == [] and a_st == 2 and lib.rwkv_get_last_error(pair.dev) == ERR_ARGS
            assert (state(lib, pair.dev.ptr, pair.n_state).tobytes(), logits(lib, pair.dev.ptr, V).tobytes()) == st
            if s is not None:
                ok, _, a_st = batch_sampled(bt, [Smp(), s], [3, 3], np.full((2, 3), 0.5), automata=[auto, auto], states=[1, 2])
                assert not ok and a_st == [1, 2] and lib.library.rwkv_get_last_error(bt.ptr) == ERR_ARGS
        # the counts were untouched too: the same keep_counts call on both contexts draws the same tokens
        ok, a, _ = gen_sampled(lib, pair.dev.ptr, Smp(1.0, 1.0, pres=0.5, freq=0.5), 6, us, keep=True)
        ok2, b, _ = gen_sampled(lib, pair.host.ptr, Smp(1.0, 1.0, pres=0.5, freq=0.5), 6, us, keep=True)
        assert ok and ok2 and a == b
        pair.same("after refusals")
    finally:
        bt.free()
        auto.free()
        pair.free()
        lib.rwkv_free(ctx)
