"""Sampling the next token of every sequence of a batch context on the device (rwkv_b200_batch_sample / _batch_eval_sample, the
batched launch of csrc/kernels/sampling.cu). A row of the batched kernel runs the single-row kernel's arithmetic, so every row must
give the bits of rwkv_b200_sample_logits on that row alone, and a batch generation loop must give the tokens and states of each
sequence driven alone with rwkv_b200_eval_sample."""
import ctypes
import json
import os
from collections import defaultdict

import numpy as np
import pytest

from conftest import GOLDEN, LONG_PROMPT, model_path

import sampling_oracle as so

CASES = json.load(open(os.path.join(GOLDEN, "sampling_cases.json")))
P_F, P_U, P_D = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_double)
ERR_ARGS, ERR_CTX, ERR_UNSUPPORTED = 1 << 8, 6 << 8, 9
KNIFE_EDGE = 2e-6            # a draw this close to a CDF edge may land on the neighbouring token (test_sampling.py)


def f32(xs):
    return np.ascontiguousarray(xs, np.float32)


def ptr(a, typ):
    return None if a is None else a.ctypes.data_as(typ)


def bias_arrays(biases):
    """Per-row dicts (or None) -> (offsets[n + 1], ids, values); (None, None, None) when no row has a bias."""
    if not any(biases):
        return None, None, None
    offsets, ids, values = [0], [], []
    for b in biases:
        for k, v in (b or {}).items():
            ids.append(k)
            values.append(v)
        offsets.append(len(ids))
    return np.array(offsets, np.uint32), np.array(ids, np.uint32), np.array(values, np.float32)


def hook_batch(lib, logits, temps, top_ps, us, biases=None):
    """The batched kernel on [n_rows, n_vocab] logits: (ok, tokens, probs)."""
    n_rows, n_vocab = logits.shape
    off, ids, vals = bias_arrays(biases or [None] * n_rows)
    toks = np.zeros(n_rows, np.uint32)
    probs = np.zeros(n_rows, np.float32)
    logits = f32(logits)
    ok = lib.library.rwkv_b200_sample_logits_batch(ptr(logits, P_F), n_rows, n_vocab, ptr(f32(temps), P_F), ptr(f32(top_ps), P_F),
                                                   ptr(np.asarray(us, np.float64), P_D), ptr(off, P_U), ptr(ids, P_U), ptr(vals, P_F),
                                                   ptr(toks, P_U), ptr(probs, P_F))
    return ok, toks, probs


def hook_single(lib, logits, temperature, top_p, u, bias=None):
    tok, prob = ctypes.c_uint32(0), ctypes.c_float(0)
    ids = vals = None
    n = len(bias) if bias else 0
    if n:
        ids = (ctypes.c_uint32 * n)(*bias.keys())
        vals = (ctypes.c_float * n)(*bias.values())
    logits = f32(logits)
    assert lib.library.rwkv_b200_sample_logits(ptr(logits, P_F), logits.size, temperature, top_p, u, ids, vals, n, ctypes.byref(tok), ctypes.byref(prob))
    return int(tok.value), np.float32(prob.value)


def mixed_rows(rng, n_vocab, n_rows=16):
    """Every pairing of temperature {0, 0.5, 1, 1.3} with top_p {0, 0.3, 0.8, 1}; every third row has a bias, so the rows in
    between have empty bias ranges between two biased rows."""
    temps = [(0.0, 0.5, 1.0, 1.3)[i % 4] for i in range(n_rows)]
    top_ps = [(0.0, 0.3, 0.8, 1.0)[(i // 4) % 4] for i in range(n_rows)]
    us = rng.random_sample(n_rows)
    biases = []
    for i in range(n_rows):
        if i % 3:
            biases.append(None)
            continue
        ids = rng.choice(n_vocab, size=min(3, n_vocab), replace=False)
        biases.append({int(k): float(v) for k, v in zip(ids, (4.0, -30.0, 1.5))})
    return temps, top_ps, us, biases


@pytest.mark.gpu
@pytest.mark.parametrize("n_vocab", [7, 1000, 4000, 16384, 50277, 65536])
def test_batch_rows_equal_single_launches_bitwise(lib, n_vocab):
    """Every batched instantiation (PER 1, 4, 16, 50, 64): each row's token and probability carry the bits of the single-row
    launch on that row, with and without bias arrays in the call."""
    rng = np.random.RandomState(n_vocab)
    temps, top_ps, us, biases = mixed_rows(rng, n_vocab)
    logits = (rng.standard_normal((len(temps), n_vocab)) * 3.0).astype(np.float32)
    for row_biases in (biases, None):
        ok, toks, probs = hook_batch(lib, logits, temps, top_ps, us, row_biases)
        assert ok
        for b in range(len(temps)):
            bias = row_biases[b] if row_biases else None
            tok, prob = hook_single(lib, logits[b], temps[b], top_ps[b], float(us[b]), bias)
            assert (int(toks[b]), probs[b].tobytes()) == (tok, prob.tobytes()), (n_vocab, b, temps[b], top_ps[b], bias)


@pytest.mark.gpu
def test_batch_hook_matches_reference_cases(lib):
    """The golden draws of the reference module, each n_vocab group as one batched call."""
    groups = defaultdict(list)
    for c in CASES:
        groups[c["n_vocab"]].append(c)
    wrong = []
    for n_vocab, cases in groups.items():
        logits = np.stack([(np.random.RandomState(c["logits_seed"]).standard_normal(n_vocab) * c["scale"]).astype(np.float32) for c in cases])
        biases = [{int(k): v for k, v in c["bias"].items()} if c["bias"] else None for c in cases]
        ok, toks, _ = hook_batch(lib, logits, [c["temperature"] for c in cases], [c["top_p"] for c in cases], [c["u"] for c in cases], biases)
        assert ok
        for c, lg, bias, tok in zip(cases, logits, biases, toks):
            if int(tok) != c["token"] and so.boundary_distance(lg, c["temperature"], c["top_p"], c["u"], bias) > KNIFE_EDGE:
                wrong.append((c, int(tok)))
    assert not wrong, wrong[:3]


class Batch:
    def __init__(self, lib, ctx, n):
        self.lib, self.n = lib, n
        self.ptr = ctypes.c_void_p(lib.library.rwkv_b200_batch_create(ctx.ptr, n))
        assert self.ptr

    def eval_sample(self, tokens, temps, top_ps, us):
        out = np.zeros(self.n, np.uint32)
        ok = self.lib.library.rwkv_b200_batch_eval_sample(self.ptr, ptr(np.asarray(tokens, np.uint32), P_U), ptr(f32(temps), P_F),
                                                          ptr(f32(top_ps), P_F), ptr(np.asarray(us, np.float64), P_D), ptr(out, P_U))
        return ok, out

    def sample(self, temps, top_ps, us, biases=None, raw_bias=None):
        off, ids, vals = raw_bias if raw_bias else bias_arrays(biases or [None] * self.n)
        out = np.zeros(self.n, np.uint32)
        ok = self.lib.library.rwkv_b200_batch_sample(self.ptr, ptr(f32(temps), P_F), ptr(f32(top_ps), P_F), ptr(np.asarray(us, np.float64), P_D),
                                                     ptr(off, P_U), ptr(ids, P_U), ptr(vals, P_F), ptr(out, P_U))
        return ok, out

    def eval(self, tokens, want_logits=True):
        return self.lib.library.rwkv_b200_batch_eval(self.ptr, ptr(np.asarray(tokens, np.uint32), P_U), want_logits)

    def state(self, b, n_state):
        st = np.zeros(n_state, np.float32)
        assert self.lib.library.rwkv_b200_batch_get_state(self.ptr, b, ptr(st, P_F))
        return st

    def logits(self, b, n_vocab):
        lg = np.zeros(n_vocab, np.float32)
        assert self.lib.library.rwkv_b200_batch_get_logits(self.ptr, b, ptr(lg, P_F))
        return lg

    def free(self):
        self.lib.library.rwkv_free(self.ptr)


@pytest.mark.gpu
@pytest.mark.parametrize("ver", ["4v0-660K", "5v1-730K", "5v2-730K", "6v0-3m", "7v0-834K"])
@pytest.mark.parametrize("fmt", ["FP32", "Q5_1"])
def test_batch_generation_equals_sequences_alone(lib, ver, fmt):
    """5 sequences, 9 steps of rwkv_b200_batch_eval_sample feeding every sampled token back in, against each sequence driven alone
    through rwkv_b200_eval_sample with the same parameters and u: identical token streams and byte-identical final states."""
    B, steps = 5, 9
    ctx = lib.rwkv_init_from_file(model_path(ver, fmt), 1, 0)
    batch = None
    try:
        n_state = lib.rwkv_get_state_buffer_element_count(ctx)
        temps, top_ps = [0.0, 0.6, 1.0, 1.3, 0.9], [1.0, 0.5, 0.9, 0.0, 0.3]
        us = np.random.RandomState(sum(map(ord, ver + fmt))).random_sample((steps, B))
        first = [LONG_PROMPT[3 * b] for b in range(B)]
        batch = Batch(lib, ctx, B)
        cur, got = list(first), []
        for step in range(steps):
            ok, out = batch.eval_sample(cur, temps, top_ps, us[step])
            assert ok
            cur = [int(t) for t in out]
            got.append(cur)
        tok = ctypes.c_uint32(0)
        st = np.zeros(n_state, np.float32)
        for b in range(B):
            assert lib.library.rwkv_b200_state_load(ctx.ptr, None)
            c, alone = first[b], []
            for step in range(steps):
                assert lib.library.rwkv_b200_eval_sample(ctx.ptr, c, temps[b], top_ps[b], float(us[step, b]), ctypes.byref(tok))
                c = int(tok.value)
                alone.append(c)
            assert [g[b] for g in got] == alone, (ver, fmt, b)
            assert lib.library.rwkv_b200_state_store(ctx.ptr, ptr(st, P_F))
            assert batch.state(b, n_state).tobytes() == st.tobytes(), (ver, fmt, b)
    finally:
        if batch:
            batch.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_batch_bias_per_sequence(lib):
    """Different biases on different sequences of one batch_sample call, each against rwkv_b200_sample with the same bias on that
    sequence alone; one bias bans the argmax under temperature 0."""
    B = 5
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    batch = None
    try:
        n_state, n_vocab = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        batch = Batch(lib, ctx, B)
        prompt = [[LONG_PROMPT[(5 * b + i) % len(LONG_PROMPT)] for i in range(3)] for b in range(B)]
        for i in range(2):
            assert batch.eval([p[i] for p in prompt], want_logits=False)
        before = [batch.state(b, n_state) for b in range(B)]
        assert batch.eval([p[2] for p in prompt])
        argmax2 = int(np.argmax(batch.logits(2, n_vocab)))
        temps, top_ps, us = [1.0, 0.8, 0.0, 1.2, 0.7], [1.0, 0.9, 1.0, 0.5, 0.0], [0.3, 0.71, 0.5, 0.12, 0.94]
        biases = [{7: 50.0}, None, {argmax2: -1e9}, {1: 2.0, 40: -3.0, 200: 5.5, 9: 1.0}, None]
        ok, out = batch.sample(temps, top_ps, us, biases)
        assert ok
        assert out[0] == 7 and out[2] != argmax2
        tok = ctypes.c_uint32(0)
        for b in range(B):
            assert lib.library.rwkv_b200_state_load(ctx.ptr, ptr(before[b], P_F))
            assert lib.library.rwkv_b200_eval_resident(ctx.ptr, ptr(np.array([prompt[b][2]], np.uint32), P_U), 1, True, None)
            bias = biases[b] or {}
            n = len(bias)
            ids = (ctypes.c_uint32 * n)(*bias.keys()) if n else None
            vals = (ctypes.c_float * n)(*bias.values()) if n else None
            assert lib.library.rwkv_b200_sample(ctx.ptr, temps[b], top_ps[b], us[b], ids, vals, n, ctypes.byref(tok))
            assert int(out[b]) == tok.value, (b, bias)
        banned = batch.logits(2, n_vocab)
        banned[argmax2] = -np.inf
        assert out[2] == int(np.argmax(banned))
    finally:
        if batch:
            batch.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("preset,fmt,n_seq", [("rwkv6-small", "Q5_1", 16), ("rwkv6-small", "Q5_1", 40), ("rwkv7-small", "FP16", 16)])
def test_batch_sampling_on_tensor_core_batches(lib, tmp_path, preset, fmt, n_seq):
    """From 16 sequences on the layer matrices go through the wgmma kernel; every draw must still be the oracle's on that
    sequence's own logits (knife-edge draws aside), and temperature 0 exactly their argmax."""
    import synthetic_model as sm
    path = str(tmp_path / f"{preset}-{fmt}.bin")
    sm.write_direct(path, preset, fmt, seed=8)
    ctx = lib.rwkv_init_from_file(path, 1, 0)
    batch = None
    try:
        n_vocab = lib.rwkv_get_logits_buffer_element_count(ctx)
        batch = Batch(lib, ctx, n_seq)
        rng = np.random.RandomState(n_seq)
        temps = [(0.0, 0.7, 1.0, 1.4)[b % 4] for b in range(n_seq)]
        top_ps = [(1.0, 0.6, 0.0, 0.9, 0.25)[b % 5] for b in range(n_seq)]
        cur = [(131 * b + 5) % n_vocab for b in range(n_seq)]
        for step in range(3):
            us = rng.random_sample(n_seq)
            ok, out = batch.eval_sample(cur, temps, top_ps, us)
            assert ok
            for b in range(n_seq):
                lg = batch.logits(b, n_vocab)
                if temps[b] == 0.0:
                    assert int(out[b]) == int(np.argmax(lg)), (step, b)
                    continue
                want = so.sample_logits_u(lg, temps[b], top_ps[b], us[b])
                assert int(out[b]) == want or so.boundary_distance(lg, temps[b], top_ps[b], us[b]) <= KNIFE_EDGE, (step, b, int(out[b]), want)
            cur = [int(t) for t in out]
    finally:
        if batch:
            batch.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_batch_sampling_errors(lib):
    B = 3
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    batch = None
    try:
        n_state, n_vocab = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        batch = Batch(lib, ctx, B)
        last_error = lambda p: lib.library.rwkv_get_last_error(p)
        T, P, U = [1.0] * B, [0.8] * B, [0.5] * B

        def refused(ok_out, flags=ERR_ARGS, p=batch.ptr):
            assert not ok_out[0]
            assert last_error(p) == flags

        refused(batch.sample(T, P, U))                                    # nothing evaluated yet
        assert batch.eval([1, 2, 3], want_logits=False)
        refused(batch.sample(T, P, U))                                    # the last pass skipped the head
        assert batch.eval([4, 5, 6])
        assert batch.sample(T, P, U)[0]
        for field, bad in (("T", -1.0), ("T", float("nan")), ("P", -0.1), ("P", 1.5), ("U", 1.0), ("U", -0.25)):
            args = {"T": list(T), "P": list(P), "U": list(U)}
            args[field][1] = bad
            refused(batch.sample(args["T"], args["P"], args["U"]))
        one = (np.array([0, 1, 1, 1], np.uint32), np.array([3], np.uint32), np.array([1.0], np.float32))
        assert batch.sample(T, P, U, raw_bias=one)[0]
        refused(batch.sample(T, P, U, raw_bias=(np.array([1, 1, 1, 1], np.uint32),) + one[1:]))               # offsets not from 0
        refused(batch.sample(T, P, U, raw_bias=(np.array([0, 2, 1, 2], np.uint32), np.array([3, 4], np.uint32),
                                                np.array([1.0, 2.0], np.float32))))                            # offsets decrease
        refused(batch.sample(T, P, U, raw_bias=(one[0], np.array([n_vocab], np.uint32), one[2])))              # id out of range
        refused(batch.sample(T, P, U, raw_bias=(one[0], None, None)))                                          # NULL bias arrays
        out = np.zeros(B, np.uint32)
        assert not lib.library.rwkv_b200_batch_sample(batch.ptr, None, ptr(f32(P), P_F), ptr(np.array(U), P_D), None, None, None, ptr(out, P_U))
        assert last_error(batch.ptr) == ERR_ARGS
        assert not lib.library.rwkv_b200_batch_sample(batch.ptr, ptr(f32(T), P_F), ptr(f32(P), P_F), ptr(np.array(U), P_D), None, None, None, None)
        assert last_error(batch.ptr) == ERR_ARGS
        # an ordinary context is not a batch
        assert lib.library.rwkv_b200_eval_resident(ctx.ptr, ptr(np.array([1], np.uint32), P_U), 1, True, None)
        assert not lib.library.rwkv_b200_batch_sample(ctx.ptr, ptr(f32(T), P_F), ptr(f32(P), P_F), ptr(np.array(U), P_D), None, None, None, ptr(out, P_U))
        assert last_error(ctx.ptr) == ERR_ARGS
        assert not lib.library.rwkv_b200_batch_eval_sample(ctx.ptr, ptr(np.array([1], np.uint32), P_U), ptr(f32(T), P_F), ptr(f32(P), P_F),
                                                           ptr(np.array(U), P_D), ptr(out, P_U))
        assert last_error(ctx.ptr) == ERR_ARGS
        # a rejected eval_sample leaves every sequence's state as it was
        states = [batch.state(b, n_state).tobytes() for b in range(B)]
        refused(batch.eval_sample([7, 8, 9], [1.0, -0.5, 1.0], P, U))
        refused(batch.eval_sample([7, 8, 9], T, P, [0.1, 0.2, 1.5]))
        assert [batch.state(b, n_state).tobytes() for b in range(B)] == states
        ok, _ = batch.eval_sample([7, 8, 9], T, P, U)
        assert ok and [batch.state(b, n_state).tobytes() for b in range(B)] != states
        # single-sequence sampling still refuses a batch context
        tok = ctypes.c_uint32(0)
        assert not lib.library.rwkv_b200_sample(batch.ptr, 1.0, 0.8, 0.5, None, None, 0, ctypes.byref(tok))
        assert last_error(batch.ptr) == ERR_CTX | ERR_UNSUPPORTED
    finally:
        if batch:
            batch.free()
        lib.rwkv_free(ctx)


def test_batch_sampling_hook_rejects_invalid_arguments(lib):
    """The batched kernel's hook checks every argument before it touches a device (passes without one)."""
    n, V = 4, 16
    opt = lambda x, dtype: None if x is None else np.asarray(x, dtype)
    good = dict(logits=np.zeros((n, V), np.float32), n_rows=n, n_vocab=V, T=[1.0] * n, P=[0.8] * n, U=[0.5] * n, off=None, ids=None, vals=None,
                toks=np.zeros(n, np.uint32))

    def call(**kw):
        a = dict(good, **kw)
        return lib.library.rwkv_b200_sample_logits_batch(ptr(a["logits"], P_F), a["n_rows"], a["n_vocab"], ptr(opt(a["T"], np.float32), P_F),
                                                         ptr(opt(a["P"], np.float32), P_F), ptr(opt(a["U"], np.float64), P_D), ptr(a["off"], P_U),
                                                         ptr(a["ids"], P_U), ptr(a["vals"], P_F), ptr(a["toks"], P_U), None)

    def bad_row(field, value):
        arr = list(good[field])
        arr[2] = value
        return {field: arr}

    ids, vals = np.array([1, 2], np.uint32), np.array([1.0, -1.0], np.float32)
    cases = [
        dict(n_rows=0), dict(n_rows=257), dict(n_vocab=0), dict(n_vocab=65537),
        bad_row("T", -1.0), bad_row("T", float("nan")), bad_row("P", -0.5), bad_row("P", 1.01), bad_row("U", 1.0), bad_row("U", -1e-9),
        dict(off=np.array([1, 1, 2, 2, 2], np.uint32), ids=ids, vals=vals),          # does not start at 0
        dict(off=np.array([0, 2, 1, 2, 2], np.uint32), ids=ids, vals=vals),          # decreases
        dict(off=np.array([0, 1, 1, 2, 2], np.uint32), ids=np.array([1, V], np.uint32), vals=vals),   # id >= n_vocab
        dict(off=np.array([0, 1, 1, 2, 2], np.uint32), ids=None, vals=vals),
        dict(off=np.array([0, 1, 1, 2, 2], np.uint32), ids=ids, vals=None),
        dict(logits=None), dict(T=None), dict(P=None), dict(U=None), dict(toks=None),
    ]
    for i, kw in enumerate(cases):
        assert not call(**kw), (i, kw)
        assert lib.rwkv_get_last_error(None) == ERR_ARGS, (i, kw)
