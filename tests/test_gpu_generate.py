"""Device-side generation (rwkv_b200_generate / rwkv_b200_batch_generate, the generation step of csrc/kernels/sampling.cu): the whole
sample-and-evaluate loop as one graph launch must give, byte for byte, the tokens, state and logits of the same loop driven from the
host one token at a time with rwkv_b200_sample (penalties as a bias list) and rwkv_b200_eval_resident / rwkv_b200_batch_eval."""
import ctypes
from collections import Counter

import numpy as np
import pytest

from conftest import LONG_PROMPT, model_path
import generate_ref as gr
from generate_ref import P_D, P_F, P_U

ERR_ARGS, ERR_CTX, ERR_UNSUPPORTED = 1 << 8, 6 << 8, 9
P_U8 = ctypes.POINTER(ctypes.c_uint8)


def ptr(a, typ):
    return None if a is None else a.ctypes.data_as(typ)


def f32(xs):
    return np.ascontiguousarray(xs, np.float32)


def generate(lib, ctx_ptr, max_tokens, temperature, top_p, presence, frequency, us, stops=(), keep=False, out_len=None):
    toks = np.zeros(max(out_len or max_tokens, 1), np.uint32)
    n = ctypes.c_size_t(0)
    st = np.array(stops, np.uint32) if len(stops) else None
    ok = lib.library.rwkv_b200_generate(ctx_ptr, max_tokens, temperature, top_p, presence, frequency, keep, ptr(np.asarray(us, np.float64), P_D),
                                        ptr(st, P_U), len(stops), ptr(toks, P_U), ctypes.byref(n))
    return ok, [int(t) for t in toks[:n.value]]


def state(lib, ctx_ptr, n_state):
    st = np.zeros(n_state, np.float32)
    assert lib.library.rwkv_b200_state_store(ctx_ptr, ptr(st, P_F))
    return st


def logits(lib, ctx_ptr, n_vocab):
    lg = np.zeros(n_vocab, np.float32)
    assert lib.library.rwkv_b200_stage_logits(ctx_ptr, ptr(lg, P_F), None)
    return lg


def prime(lib, ctx_ptr, prompt):
    assert lib.library.rwkv_b200_state_load(ctx_ptr, None)
    assert lib.library.rwkv_b200_eval_resident(ctx_ptr, ptr(np.asarray(prompt, np.uint32), P_U), len(prompt), True, None)


class Pair:
    """Two contexts of one model: `host` runs the host loop, `dev` rwkv_b200_generate."""

    def __init__(self, lib, ctx):
        self.lib, self.host, self.dev = lib, ctx, lib.rwkv_clone_context(ctx, 1)
        self.n_state, self.n_vocab = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)

    def prime(self, prompt):
        prime(self.lib, self.host.ptr, prompt)
        prime(self.lib, self.dev.ptr, prompt)

    def same(self, what):
        L = self.lib
        assert state(L, self.host.ptr, self.n_state).tobytes() == state(L, self.dev.ptr, self.n_state).tobytes(), ("state", what)
        assert logits(L, self.host.ptr, self.n_vocab).tobytes() == logits(L, self.dev.ptr, self.n_vocab).tobytes(), ("logits", what)

    def free(self):
        self.lib.rwkv_free(self.dev)


CASES = [  # max_tokens, temperature, top_p, presence, frequency (9 and 7 passes are odd, 8 even)
    (9, 0.0, 1.0, 0.0, 0.0),
    (9, 1.0, 0.8, 0.0, 0.0),
    (8, 0.5, 1.0, 0.2, 0.2),
    (7, 1.0, 0.8, 0.2, 0.2),
    (1, 1.0, 1.0, 0.0, 0.0),
]


def check_case(pair, prompt, case, us, stops=()):
    L = pair.lib
    pair.prime(prompt)
    mt, t, p, pres, freq = case
    want = gr.host_generate(L, pair.host.ptr, mt, t, p, pres, freq, us, stops)
    ok, got = generate(L, pair.dev.ptr, mt, t, p, pres, freq, us, stops)
    assert ok
    assert got == want, (case, stops)
    pair.same((case, stops))
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("ver", ["4v0-660K", "5v1-730K", "5v2-730K", "6v0-3m", "7v0-834K"])
@pytest.mark.parametrize("fmt", ["FP32", "Q5_1"])
def test_generate_equals_host_loop(lib, ver, fmt):
    ctx = lib.rwkv_init_from_file(model_path(ver, fmt), 1, 0)
    pair = Pair(lib, ctx)
    try:
        L = lib.library
        rng = np.random.RandomState(sum(map(ord, ver + fmt)))
        prompt = LONG_PROMPT[:5]
        for case in CASES:
            us = rng.random_sample(case[0])
            check_case(pair, prompt, case, us)
            # the state buffers and phase after an odd or even number of passes: later calls still follow the host loop
            tok_h, tok_d = ctypes.c_uint32(0), ctypes.c_uint32(0)
            u = float(rng.random_sample())
            assert L.rwkv_b200_eval_sample(pair.host.ptr, 17, 1.0, 0.9, u, ctypes.byref(tok_h))
            assert L.rwkv_b200_eval_sample(pair.dev.ptr, 17, 1.0, 0.9, u, ctypes.byref(tok_d))
            assert tok_h.value == tok_d.value, case
            for ctx_ptr in (pair.host.ptr, pair.dev.ptr):
                assert L.rwkv_b200_eval_resident(ctx_ptr, ptr(np.array(LONG_PROMPT[5:8], np.uint32), P_U), 3, True, None)
                gr.eval_token(lib, ctx_ptr, 40)
            pair.same(("after", case))
        # a stop token hit mid-way, taken from a run without stops; a second stop id that never comes
        case = (8, 1.0, 0.9, 0.1, 0.3)
        us = rng.random_sample(8)
        free_run = check_case(pair, prompt, case, us)
        stop = free_run[3]
        never = next(i for i in range(pair.n_vocab) if i not in free_run)
        got = check_case(pair, prompt, case, us, stops=(never, stop))
        assert got[-1] == stop and len(got) == free_run.index(stop) + 1
        # keep_counts: two calls equal one long one
        pres, freq = 0.3, 0.5
        us = rng.random_sample(10)
        pair.prime(prompt)
        want = gr.host_generate(lib, pair.host.ptr, 10, 1.0, 1.0, pres, freq, us)
        ok, first = generate(lib, pair.dev.ptr, 4, 1.0, 1.0, pres, freq, us[:4])
        assert ok
        ok, second = generate(lib, pair.dev.ptr, 6, 1.0, 1.0, pres, freq, us[4:], keep=True)
        assert ok and first + second == want
        pair.same("keep_counts")
    finally:
        pair.free()
        lib.rwkv_free(ctx)


def bias_arrays(biases):
    if not any(biases):
        return None, None, None
    offsets, ids, values = [0], [], []
    for b in biases:
        for k, v in (b or {}).items():
            ids.append(k)
            values.append(v)
        offsets.append(len(ids))
    return np.array(offsets, np.uint32), np.array(ids, np.uint32), np.array(values, np.float32)


class Batch:
    def __init__(self, lib, ctx, n):
        self.lib, self.n = lib, n
        self.ptr = ctypes.c_void_p(lib.library.rwkv_b200_batch_create(ctx.ptr, n))
        assert self.ptr

    def prime(self, prompts):
        for b in range(self.n):
            assert self.lib.library.rwkv_b200_batch_set_state(self.ptr, b, None)
        for i in range(len(prompts[0])):
            assert self.eval([p[i] for p in prompts])

    def eval(self, tokens):
        return self.lib.library.rwkv_b200_batch_eval(self.ptr, ptr(np.asarray(tokens, np.uint32), P_U), True)

    def sample(self, temps, top_ps, us, biases):
        off, ids, vals = bias_arrays(biases)
        out = np.zeros(self.n, np.uint32)
        assert self.lib.library.rwkv_b200_batch_sample(self.ptr, ptr(f32(temps), P_F), ptr(f32(top_ps), P_F), ptr(np.asarray(us, np.float64), P_D),
                                                       ptr(off, P_U), ptr(ids, P_U), ptr(vals, P_F), ptr(out, P_U))
        return [int(t) for t in out]

    def state(self, b, n_state):
        st = np.zeros(n_state, np.float32)
        assert self.lib.library.rwkv_b200_batch_get_state(self.ptr, b, ptr(st, P_F))
        return st

    def logits(self, b, n_vocab):
        lg = np.zeros(n_vocab, np.float32)
        assert self.lib.library.rwkv_b200_batch_get_logits(self.ptr, b, ptr(lg, P_F))
        return lg

    def generate(self, max_tokens, temps, top_ps, pres, freq, us, stops, keep=None):
        n = max(max_tokens)
        toks = np.zeros(self.n * max(n, 1), np.uint32)
        ng = np.zeros(self.n, np.uint32)
        st = np.array(stops, np.uint32) if len(stops) else None
        ok = self.lib.library.rwkv_b200_batch_generate(self.ptr, ptr(np.asarray(max_tokens, np.uint32), P_U), ptr(f32(temps), P_F), ptr(f32(top_ps), P_F),
                                                       ptr(f32(pres), P_F), ptr(f32(freq), P_F), ptr(None if keep is None else np.asarray(keep, np.uint8), P_U8),
                                                       ptr(np.ascontiguousarray(us, np.float64), P_D), ptr(st, P_U), len(stops), ptr(toks, P_U), ptr(ng, P_U))
        return ok, [[int(t) for t in toks[b * n:b * n + ng[b]]] for b in range(self.n)]

    def free(self):
        self.lib.library.rwkv_free(self.ptr)


def batch_host_loop(bt, n_state, n_vocab, max_tokens, temps, top_ps, pres, freq, us, stops):
    """rwkv_b200_batch_sample with the penalty biases + rwkv_b200_batch_eval, a stopped sequence put back with set_state after each
    pass. Returns (tokens per sequence, state and logits of every sequence at the moment it stopped)."""
    B = bt.n
    counts, step, frozen, out = [Counter() for _ in range(B)], [0] * B, [False] * B, [[] for _ in range(B)]
    saved = {}

    def freeze(b):
        frozen[b] = True
        saved[b] = (bt.state(b, n_state), bt.logits(b, n_vocab))

    while True:
        for b in range(B):
            if not frozen[b] and step[b] == max_tokens[b]:
                freeze(b)
        active = [b for b in range(B) if not frozen[b]]
        if not active:
            break
        toks = bt.sample(temps, top_ps, [us[b][step[b]] if not frozen[b] else 0.5 for b in range(B)],
                         [gr.penalty_bias(counts[b], pres[b], freq[b]) if not frozen[b] else None for b in range(B)])
        inputs = [0] * B
        for b in active:
            out[b].append(toks[b])
            step[b] += 1
            if toks[b] in stops:
                freeze(b)
            else:
                counts[b][toks[b]] += 1
                inputs[b] = toks[b]
        if all(frozen):
            break
        assert bt.eval(inputs)
        for b in range(B):
            if frozen[b]:
                assert bt.lib.library.rwkv_b200_batch_set_state(bt.ptr, b, ptr(saved[b][0], P_F))
    return out, saved


@pytest.mark.gpu
@pytest.mark.parametrize("model,B", [(("6v0-3m", "FP32"), 4), (("7v0-834K", "Q5_1"), 4), (("rwkv6-small", "Q5_1"), 20), (("rwkv7-small", "FP16"), 20)])
def test_batch_generate_equals_host_loop(lib, tmp_path, model, B):
    """B = 4 runs the multi-column GEMV, B = 20 the tensor-core path. Budgets include 0; penalties and parameters differ per
    sequence; the stop set is taken from a run without stops so that some sequences stop mid-way."""
    name, fmt = model
    if name.startswith("rwkv"):
        import synthetic_model as sm
        path = str(tmp_path / f"{name}-{fmt}.bin")
        sm.write_direct(path, name, fmt, seed=11)
    else:
        path = model_path(name, fmt)
    ctx = lib.rwkv_init_from_file(path, 1, 0)
    bh = bg = None
    try:
        n_state, n_vocab = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        bh, bg = Batch(lib, ctx, B), Batch(lib, ctx, B)
        rng = np.random.RandomState(B)
        max_tokens = [(6, 0, 9, 3, 7)[b % 5] for b in range(B)]
        temps = [(0.0, 0.7, 1.0, 1.3)[b % 4] for b in range(B)]
        top_ps = [(1.0, 0.6, 0.0, 0.9, 0.25)[b % 5] for b in range(B)]
        pres = [(0.0, 0.2, 0.5)[b % 3] for b in range(B)]
        freq = [(0.0, 0.2, 0.1, 0.4)[b % 4] for b in range(B)]
        n = max(max_tokens)
        us = rng.random_sample((B, n))
        prompts = [[(37 * b + 5 * i + 3) % n_vocab for i in range(2)] for b in range(B)]
        bh.prime(prompts)
        free_run, _ = batch_host_loop(bh, n_state, n_vocab, max_tokens, temps, top_ps, pres, freq, us, ())
        stops = sorted({free_run[2][4], free_run[3][1]})
        bh.prime(prompts)
        want, saved = batch_host_loop(bh, n_state, n_vocab, max_tokens, temps, top_ps, pres, freq, us, stops)
        assert any(0 < len(w) < m for w, m in zip(want, max_tokens)), "no sequence stopped mid-way"
        bg.prime(prompts)
        ok, got = bg.generate(max_tokens, temps, top_ps, pres, freq, us, stops)
        assert ok
        assert got == want
        for b in range(B):
            assert bg.state(b, n_state).tobytes() == saved[b][0].tobytes(), b
            assert bg.logits(b, n_vocab).tobytes() == saved[b][1].tobytes(), b
        if B < 16:      # below the tensor-core threshold every sequence is also what it gives alone
            for b in range(B):
                if not max_tokens[b]:
                    continue
                assert lib.library.rwkv_b200_state_load(ctx.ptr, None)
                for t in prompts[b]:
                    gr.eval_token(lib, ctx.ptr, t)
                ok, alone = generate(lib, ctx.ptr, max_tokens[b], temps[b], top_ps[b], pres[b], freq[b], us[b], stops)
                assert ok and alone == want[b], b
                assert state(lib, ctx.ptr, n_state).tobytes() == saved[b][0].tobytes(), b
    finally:
        for bt in (bh, bg):
            if bt:
                bt.free()
        lib.rwkv_free(ctx)


def hook_step(lib, logits, max_tokens, temps, top_ps, pres, freq, us, stops, step, frozen, counts, tokens):
    R, V = logits.shape
    step, frozen, counts, tokens = np.array(step, np.uint32), np.array(frozen, np.uint8), counts.copy(), tokens.copy()
    nxt, any_active = np.zeros(R, np.int32), ctypes.c_uint32(7)
    st = np.array(stops, np.uint32) if len(stops) else None
    mt, t, p, pr, fr, u = (np.asarray(max_tokens, np.uint32), f32(temps), f32(top_ps), f32(pres), f32(freq), np.ascontiguousarray(us, np.float64))
    a = gr.StepArgs(logits=logits.ctypes.data, n_rows=R, n_vocab=V, max_tokens=mt.ctypes.data, temperature=t.ctypes.data, top_p=p.ctypes.data,
                 presence_penalty=pr.ctypes.data, frequency_penalty=fr.ctypes.data, u=u.ctypes.data, stop_ids=None if st is None else st.ctypes.data,
                 n_stop=len(stops), step=step.ctypes.data, frozen=frozen.ctypes.data, counts=counts.ctypes.data, tokens=tokens.ctypes.data,
                 next_tokens=nxt.ctypes.data, any_active=ctypes.addressof(any_active))
    ok = lib.library.rwkv_b200_test_generate_step(ctypes.byref(a))
    return ok, step, frozen, counts, tokens, nxt, any_active.value


@pytest.mark.gpu
@pytest.mark.parametrize("V", [7, 1000, 16384, 50277, 65536])
def test_generate_step_hook(lib, V):
    """One step at every instantiation: each drawing row is, bit for bit, rwkv_b200_sample_logits_batch with the penalty biases as
    bias lists; steps, freezes, counts and next tokens match their restatement."""
    R = 7
    rng = np.random.RandomState(V)
    logits = (rng.standard_normal((R, V)) * 3.0).astype(np.float32)
    max_tokens = [3, 3, 0, 5, 2, 4, 1]
    step = [1, 3, 0, 2, 0, 1, 0]
    frozen = [0, 0, 0, 0, 0, 1, 0]
    temps, top_ps = [1.0, 0.8, 1.0, 0.0, 1.3, 1.0, 0.5], [0.9, 1.0, 1.0, 1.0, 0.3, 0.7, 0.0]
    pres, freq = [0.2, 0.0, 0.5, 1.0, 0.3, 0.0, 0.25], [0.2, 0.7, 0.0, 1.5, 0.1, 0.0, 3.0]
    n = max(max_tokens)
    us = rng.random_sample((R, n))
    counts = np.zeros((R, V), np.uint32)
    for b in range(R):
        ids = rng.choice(V, size=min(5, V), replace=False)
        counts[b, ids] = rng.randint(0, 4, size=len(ids))
    counts[3, int(np.argmax(logits[3]))] = 9           # the penalty moves row 3's argmax
    tokens = np.full((R, n), 5, np.uint32)
    drawing = [b for b in range(R) if not frozen[b] and step[b] < max_tokens[b]]
    biases = [gr.penalty_bias({i: int(c) for i, c in enumerate(counts[b]) if c}, pres[b], freq[b]) if b in drawing else None for b in range(R)]
    off, ids, vals = bias_arrays(biases)
    ref = np.zeros(R, np.uint32)
    assert lib.library.rwkv_b200_sample_logits_batch(ptr(logits, P_F), R, V, ptr(f32(temps), P_F), ptr(f32(top_ps), P_F),
                                                      ptr(np.array([us[b][min(step[b], n - 1)] for b in range(R)]), P_D), ptr(off, P_U), ptr(ids, P_U),
                                                      ptr(vals, P_F), ptr(ref, P_U), None)
    stops = [int(ref[0])] if V > 7 else []
    ok, s2, f2, c2, t2, nxt, any_active = hook_step(lib, logits, max_tokens, temps, top_ps, pres, freq, us, stops, step, frozen, counts, tokens)
    assert ok
    drawn = [int(ref[b]) if b in drawing else None for b in range(R)]
    want_step, want_frozen, want_active = gr.step_flags(max_tokens, step, frozen, drawn, stops)
    assert list(s2) == want_step and list(f2) == want_frozen and any_active == int(want_active)
    want_counts, want_tokens = counts.copy(), tokens.copy()
    for b in drawing:
        want_tokens[b, step[b]] = drawn[b]
        if drawn[b] not in stops:
            want_counts[b, drawn[b]] += 1
    assert np.array_equal(t2, want_tokens) and np.array_equal(c2, want_counts)
    assert list(nxt) == [drawn[b] if not want_frozen[b] else 0 for b in range(R)]
    if V > 7:
        assert int(np.argmax(logits[3])) != drawn[3]


@pytest.mark.gpu
def test_generate_rejections_change_nothing(lib):
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    pair = Pair(lib, ctx)
    bt = None
    try:
        L = lib.library
        V = pair.n_vocab
        err = lambda p: L.rwkv_get_last_error(p)
        pair.prime(LONG_PROMPT[:4])
        us = np.random.RandomState(3).random_sample(12)
        counts = Counter()
        want = gr.host_generate(lib, pair.host.ptr, 5, 1.0, 1.0, 0.4, 0.4, us[:5], counts=counts)
        ok, got = generate(lib, pair.dev.ptr, 5, 1.0, 1.0, 0.4, 0.4, us[:5])
        assert ok and got == want
        before = (state(lib, pair.dev.ptr, pair.n_state).tobytes(), logits(lib, pair.dev.ptr, V).tobytes())
        bad_u = us[5:].copy()
        bad_u[2] = 1.0
        cases = [  # keyword overrides of (max_tokens, temperature, top_p, presence, frequency, us, stops)
            dict(temperature=-1.0), dict(temperature=float("nan")), dict(top_p=1.5), dict(top_p=-0.1), dict(us=bad_u),
            dict(presence=float("nan")), dict(frequency=float("inf")), dict(stops=(V,)), dict(stops=tuple(range(17))), dict(max_tokens=0),
            dict(max_tokens=4097, out_len=4097, us=np.full(4097, 0.5)),
        ]
        base = dict(max_tokens=7, temperature=1.0, top_p=1.0, presence=0.4, frequency=0.4, us=us[5:], stops=())
        for kw in cases:
            a = dict(base, **kw)
            ok, _ = generate(lib, pair.dev.ptr, a["max_tokens"], a["temperature"], a["top_p"], a["presence"], a["frequency"], a["us"], a["stops"],
                             keep=True, out_len=kw.get("out_len"))
            assert not ok and err(pair.dev.ptr) == ERR_ARGS, kw
        n = ctypes.c_size_t(0)
        toks = np.zeros(7, np.uint32)
        assert not L.rwkv_b200_generate(pair.dev.ptr, 7, 1.0, 1.0, 0.0, 0.0, True, None, None, 0, ptr(toks, P_U), ctypes.byref(n))
        assert err(pair.dev.ptr) == ERR_ARGS
        assert not L.rwkv_b200_generate(pair.dev.ptr, 7, 1.0, 1.0, 0.0, 0.0, True, ptr(us, P_D), None, 0, None, ctypes.byref(n))
        assert err(pair.dev.ptr) == ERR_ARGS
        # a batch context is the wrong kind for the single call, and the other way round
        bt = Batch(lib, ctx, 2)
        assert not generate(lib, bt.ptr, 3, 1.0, 1.0, 0.0, 0.0, us[:3])[0] and err(bt.ptr) == ERR_CTX | ERR_UNSUPPORTED
        ng = np.zeros(1, np.uint32)
        assert not L.rwkv_b200_batch_generate(pair.dev.ptr, ptr(np.array([3], np.uint32), P_U), ptr(f32([1.0]), P_F), ptr(f32([1.0]), P_F),
                                              ptr(f32([0.0]), P_F), ptr(f32([0.0]), P_F), None, ptr(us, P_D), None, 0, ptr(toks, P_U), ptr(ng, P_U))
        assert err(pair.dev.ptr) == ERR_CTX | ERR_UNSUPPORTED
        # a stage of a pipeline (not every layer resident)
        stage = lib.rwkv_b200_init_from_file_ex(model_path("6v0-3m", "FP32"), 0, 0, 1)
        assert not generate(lib, stage.ptr, 3, 1.0, 1.0, 0.0, 0.0, us[:3])[0] and err(stage.ptr) == ERR_CTX | ERR_UNSUPPORTED
        lib.rwkv_free(stage)
        assert (state(lib, pair.dev.ptr, pair.n_state).tobytes(), logits(lib, pair.dev.ptr, V).tobytes()) == before
        # the counts are unchanged too: continuing equals the host loop continuing from its counts
        want = gr.host_generate(lib, pair.host.ptr, 7, 1.0, 1.0, 0.4, 0.4, us[5:], counts=counts)
        ok, got = generate(lib, pair.dev.ptr, 7, 1.0, 1.0, 0.4, 0.4, us[5:], keep=True)
        assert ok and got == want
        pair.same("after rejections")
        # no logits to draw from
        for p in (pair.dev.ptr,):
            assert L.rwkv_b200_eval_resident(p, ptr(np.array([3], np.uint32), P_U), 1, False, None)
            assert not generate(lib, p, 3, 1.0, 1.0, 0.0, 0.0, us[:3])[0] and err(p) == ERR_ARGS
    finally:
        if bt:
            bt.free()
        pair.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_generate_7b_shape(lib):
    """32 tokens of the synthetic RWKV-6 7B shape (Q5_1) with penalties equal the host loop."""
    import bench
    path, _ = bench.workload_file("rwkv6-7b:Q5_1")
    ctx = lib.rwkv_b200_init_from_file_ex(path, 0, 0, -1)
    pair = Pair(lib, ctx)
    try:
        us = np.random.RandomState(7).random_sample(32)
        pair.prime(LONG_PROMPT[:6])
        want = gr.host_generate(lib, pair.host.ptr, 32, 1.0, 0.8, 0.2, 0.2, us)
        ok, got = generate(lib, pair.dev.ptr, 32, 1.0, 0.8, 0.2, 0.2, us)
        assert ok and got == want
        pair.same("7b")
    finally:
        pair.free()
        lib.rwkv_free(ctx)
