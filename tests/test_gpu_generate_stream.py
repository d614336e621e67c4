"""Streaming generation (rwkv_b200_generate_stream / rwkv_b200_batch_generate_stream, the gated step kernel of
csrc/kernels/sampling.cu): every token reaches the callback once and in order, a nonzero return ends its sequence after that token
with the bytes of the blocking call whose budget ends there, and a callback that always returns 0 gives the bytes of the blocking
call. The blocking calls are the reference here; tests/test_gpu_generate.py ties them to the host loop."""
import ctypes
import time

import numpy as np
import pytest

from conftest import LONG_PROMPT, model_path
from generate_ref import P_D, P_F, P_U
from test_gpu_generate import CASES, ERR_ARGS, ERR_CTX, ERR_UNSUPPORTED, P_U8, Batch, Pair, f32, generate, logits, ptr, state

TOKEN_FN = ctypes.CFUNCTYPE(ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_size_t, ctypes.c_uint32)
NULL_FN = TOKEN_FN()     # a NULL on_token


class Recorder:
    """An on_token that records (sequence, index, token) and returns 1 for the index stop_at[sequence]; sleep {(sequence, index): s}
    delays the return, inner(sequence, index, token) runs inside the callback."""

    def __init__(self, stop_at=None, sleep=None, inner=None):
        self.calls, self.stop_at, self.sleep, self.inner = [], stop_at or {}, sleep or {}, inner
        self.fn = TOKEN_FN(self._call)

    def _call(self, user, seq, idx, tok):
        self.calls.append((int(seq), int(idx), int(tok)))
        if self.inner:
            self.inner(seq, idx, tok)
        if (seq, idx) in self.sleep:
            time.sleep(self.sleep[(seq, idx)])
        return 1 if self.stop_at.get(seq) == idx else 0

    def delivered(self, seq):
        """The tokens of `seq` in delivery order; asserts that their indices are 0, 1, 2, ..."""
        mine = [(i, t) for s, i, t in self.calls if s == seq]
        assert [i for i, _ in mine] == list(range(len(mine))), mine
        return [t for _, t in mine]


def generate_stream(lib, ctx_ptr, max_tokens, temperature, top_p, presence, frequency, us, stops=(), keep=False, rec=None, out_len=None):
    toks = np.zeros(max(out_len or max_tokens, 1), np.uint32)
    n = ctypes.c_size_t(0)
    st = np.array(stops, np.uint32) if len(stops) else None
    ok = lib.library.rwkv_b200_generate_stream(ctx_ptr, max_tokens, temperature, top_p, presence, frequency, keep, ptr(np.asarray(us, np.float64), P_D),
                                               ptr(st, P_U), len(stops), rec.fn if rec else NULL_FN, None, ptr(toks, P_U), ctypes.byref(n))
    return ok, [int(t) for t in toks[:n.value]]


def batch_generate_stream(bt, max_tokens, temps, top_ps, pres, freq, us, stops, rec, keep=None):
    n = max(max_tokens)
    toks = np.zeros(bt.n * max(n, 1), np.uint32)
    ng = np.zeros(bt.n, np.uint32)
    st = np.array(stops, np.uint32) if len(stops) else None
    ok = bt.lib.library.rwkv_b200_batch_generate_stream(bt.ptr, ptr(np.asarray(max_tokens, np.uint32), P_U), ptr(f32(temps), P_F), ptr(f32(top_ps), P_F),
                                                        ptr(f32(pres), P_F), ptr(f32(freq), P_F), ptr(None if keep is None else np.asarray(keep, np.uint8), P_U8),
                                                        ptr(np.ascontiguousarray(us, np.float64), P_D), ptr(st, P_U), len(stops), rec.fn if rec else NULL_FN, None,
                                                        ptr(toks, P_U), ptr(ng, P_U))
    return ok, [[int(t) for t in toks[b * n:b * n + ng[b]]] for b in range(bt.n)]


def check_stream_case(pair, prompt, case, us, stops=()):
    """`pair.host` runs the blocking call, `pair.dev` the streaming one with a callback that always returns 0."""
    lib = pair.lib
    pair.prime(prompt)
    mt, t, p, pres, freq = case
    ok, want = generate(lib, pair.host.ptr, mt, t, p, pres, freq, us, stops)
    assert ok
    rec = Recorder()
    ok, got = generate_stream(lib, pair.dev.ptr, mt, t, p, pres, freq, us, stops, rec=rec)
    assert ok and got == want, (case, stops)
    assert rec.calls == [(0, i, tok) for i, tok in enumerate(got)]
    pair.same((case, stops))
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("ver", ["4v0-660K", "5v1-730K", "5v2-730K", "6v0-3m", "7v0-834K"])
@pytest.mark.parametrize("fmt", ["FP32", "Q5_1"])
def test_generate_stream_equals_blocking(lib, ver, fmt):
    ctx = lib.rwkv_init_from_file(model_path(ver, fmt), 1, 0)
    pair = Pair(lib, ctx)
    try:
        L = lib.library
        rng = np.random.RandomState(sum(map(ord, ver + fmt)))
        prompt = LONG_PROMPT[:5]
        for case in CASES:
            check_stream_case(pair, prompt, case, rng.random_sample(case[0]))
            # the state-buffer parity after an odd or even number of passes
            tok_h, tok_d = ctypes.c_uint32(0), ctypes.c_uint32(0)
            u = float(rng.random_sample())
            assert L.rwkv_b200_eval_sample(pair.host.ptr, 17, 1.0, 0.9, u, ctypes.byref(tok_h))
            assert L.rwkv_b200_eval_sample(pair.dev.ptr, 17, 1.0, 0.9, u, ctypes.byref(tok_d))
            assert tok_h.value == tok_d.value, case
            pair.same(("after", case))
        # a stop token hit mid-way is delivered and ends the sequence
        case = (8, 1.0, 0.9, 0.1, 0.3)
        us = rng.random_sample(8)
        free_run = check_stream_case(pair, prompt, case, us)
        stop = free_run[3]
        never = next(i for i in range(pair.n_vocab) if i not in free_run)
        got = check_stream_case(pair, prompt, case, us, stops=(never, stop))
        assert got[-1] == stop and len(got) == free_run.index(stop) + 1
        # keep_counts over two calls
        us = rng.random_sample(10)
        pair.prime(prompt)
        ok, want1 = generate(lib, pair.host.ptr, 4, 1.0, 1.0, 0.3, 0.5, us[:4])
        ok2, want2 = generate(lib, pair.host.ptr, 6, 1.0, 1.0, 0.3, 0.5, us[4:], keep=True)
        assert ok and ok2
        ok, got1 = generate_stream(lib, pair.dev.ptr, 4, 1.0, 1.0, 0.3, 0.5, us[:4], rec=Recorder())
        ok2, got2 = generate_stream(lib, pair.dev.ptr, 6, 1.0, 1.0, 0.3, 0.5, us[4:], keep=True, rec=Recorder())
        assert ok and ok2 and (got1, got2) == (want1, want2)
        pair.same("keep_counts")
    finally:
        pair.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("ver,fmt", [("6v0-3m", "Q5_1"), ("7v0-834K", "FP32"), ("4v0-660K", "FP32")])
def test_generate_stream_ends_after_token_j(lib, ver, fmt):
    """A nonzero return for token j equals the blocking call with max_tokens = j + 1, follow-up keep_counts call included; so does
    a stop returned after sleeping far longer than a pass, which a loop without the gate would overshoot."""
    ctx = lib.rwkv_init_from_file(model_path(ver, fmt), 1, 0)
    pair = Pair(lib, ctx)
    try:
        rng = np.random.RandomState(5)
        prompt = LONG_PROMPT[:4]
        mt, pres, freq = 9, 0.2, 0.3
        for j, sleep in [(0, None), (1, None), (4, None), (mt - 1, None), (2, 0.05)]:
            us = rng.random_sample(mt)
            pair.prime(prompt)
            ok, want = generate(lib, pair.host.ptr, j + 1, 1.0, 0.9, pres, freq, us[:j + 1])
            assert ok and len(want) == j + 1
            rec = Recorder(stop_at={0: j}, sleep={(0, j): sleep} if sleep else None)
            ok, got = generate_stream(lib, pair.dev.ptr, mt, 1.0, 0.9, pres, freq, us, rec=rec)
            assert ok and got == want, j
            assert rec.delivered(0) == got
            pair.same(("stop", j))
            follow = rng.random_sample(5)
            ok, want = generate(lib, pair.host.ptr, 5, 1.0, 0.9, pres, freq, follow, keep=True)
            ok2, got = generate_stream(lib, pair.dev.ptr, 5, 1.0, 0.9, pres, freq, follow, keep=True, rec=Recorder())
            assert ok and ok2 and got == want, ("follow-up", j)
            pair.same(("follow-up", j))
    finally:
        pair.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
@pytest.mark.parametrize("model,B", [(("6v0-3m", "FP32"), 4), (("7v0-834K", "Q5_1"), 4), (("rwkv6-small", "Q5_1"), 20), (("rwkv7-small", "FP16"), 20)])
def test_batch_generate_stream_ends_each_sequence(lib, tmp_path, model, B):
    """Sequences end at different j (one has budget 0, some run out their budget): the results equal rwkv_b200_batch_generate with
    max_tokens[b] = j_b + 1, and a following keep_counts call agrees as well."""
    name, fmt = model
    if name.startswith("rwkv"):
        import synthetic_model as sm
        path = str(tmp_path / f"{name}-{fmt}.bin")
        sm.write_direct(path, name, fmt, seed=11)
    else:
        path = model_path(name, fmt)
    ctx = lib.rwkv_init_from_file(path, 1, 0)
    bh = bs = None
    try:
        n_state, n_vocab = lib.rwkv_get_state_buffer_element_count(ctx), lib.rwkv_get_logits_buffer_element_count(ctx)
        bh, bs = Batch(lib, ctx, B), Batch(lib, ctx, B)
        rng = np.random.RandomState(B + 1)
        max_tokens = [(6, 0, 9, 3, 7)[b % 5] for b in range(B)]
        ends = [(2, None, 0, None, 4, 5, None, 8, 1, None)[b % 10] for b in range(B)]
        ends = [e if e is not None and e < m else None for e, m in zip(ends, max_tokens)]
        assert len({e for e in ends if e is not None}) >= 2
        budgets = [m if e is None else e + 1 for e, m in zip(ends, max_tokens)]
        temps = [(0.0, 0.7, 1.0, 1.3)[b % 4] for b in range(B)]
        top_ps = [(1.0, 0.6, 0.0, 0.9, 0.25)[b % 5] for b in range(B)]
        pres = [(0.0, 0.2, 0.5)[b % 3] for b in range(B)]
        freq = [(0.0, 0.2, 0.1, 0.4)[b % 4] for b in range(B)]
        n = max(max_tokens)
        us = rng.random_sample((B, n))
        prompts = [[(37 * b + 5 * i + 3) % n_vocab for i in range(2)] for b in range(B)]
        bh.prime(prompts)
        bs.prime(prompts)
        ok, want = bh.generate(budgets, temps, top_ps, pres, freq, us[:, :max(budgets)], ())
        assert ok
        rec = Recorder(stop_at={b: e for b, e in enumerate(ends) if e is not None})
        ok, got = batch_generate_stream(bs, max_tokens, temps, top_ps, pres, freq, us, (), rec)
        assert ok and got == want
        for b in range(B):
            assert rec.delivered(b) == got[b], b
            assert bs.state(b, n_state).tobytes() == bh.state(b, n_state).tobytes(), b
            assert bs.logits(b, n_vocab).tobytes() == bh.logits(b, n_vocab).tobytes(), b
        # the penalty counts and the state-buffer parity: a following keep_counts call still agrees
        follow = [3] * B
        fus = rng.random_sample((B, 3))
        ok, want = bh.generate(follow, temps, top_ps, pres, freq, fus, (), keep=[1] * B)
        ok2, got = batch_generate_stream(bs, follow, temps, top_ps, pres, freq, fus, (), Recorder(), keep=[1] * B)
        assert ok and ok2 and got == want
        for b in range(B):
            assert bs.state(b, n_state).tobytes() == bh.state(b, n_state).tobytes(), ("follow-up", b)
            assert bs.logits(b, n_vocab).tobytes() == bh.logits(b, n_vocab).tobytes(), ("follow-up", b)
    finally:
        for bt in (bh, bs):
            if bt:
                bt.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_generate_stream_refuses_reentry(lib):
    """From inside the callback, calls on the generating context are refused with CTX | UNSUPPORTED and change nothing; a clone of
    the model stays usable. The generation still equals the blocking call."""
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    pair = Pair(lib, ctx)
    other = lib.rwkv_clone_context(ctx, 1)
    try:
        L = lib.library
        n_state, n_vocab = pair.n_state, pair.n_vocab
        prime_toks = np.array(LONG_PROMPT[:3], np.uint32)
        one = np.array([5], np.uint32)
        assert L.rwkv_b200_state_load(other.ptr, None)
        for _ in range(3):      # the clone's single-token pass is warm (graph captured) before the callback uses it
            assert L.rwkv_b200_eval_resident(other.ptr, ptr(one, P_U), 1, True, None)
        assert L.rwkv_b200_synchronize(other.ptr)
        st_buf, lg_buf = np.zeros(n_state, np.float32), np.zeros(n_vocab, np.float32)
        toks_buf, n_buf = np.zeros(4, np.uint32), ctypes.c_size_t(0)
        dev = pair.dev.ptr
        results = []

        def inner(seq, idx, tok):
            if idx != 1:
                return
            calls = {
                "rwkv_eval": lambda: L.rwkv_eval(dev, 3, ptr(st_buf, P_F), ptr(st_buf, P_F), ptr(lg_buf, P_F)),
                "eval_resident": lambda: L.rwkv_b200_eval_resident(dev, ptr(one, P_U), 1, True, None),
                "state_store": lambda: L.rwkv_b200_state_store(dev, ptr(st_buf, P_F)),
                "generate": lambda: L.rwkv_b200_generate(dev, 2, 1.0, 1.0, 0.0, 0.0, False, ptr(np.full(2, 0.5), P_D), None, 0, ptr(toks_buf, P_U),
                                                         ctypes.byref(n_buf)),
            }
            for name, call in calls.items():
                results.append((name, bool(call()), int(L.rwkv_get_last_error(dev))))
            results.append(("clone eval_resident", bool(L.rwkv_b200_eval_resident(other.ptr, ptr(one, P_U), 1, True, None)), 0))

        us = np.random.RandomState(9).random_sample(6)
        pair.prime(list(prime_toks))
        ok, want = generate(lib, pair.host.ptr, 6, 1.0, 0.9, 0.2, 0.2, us)
        assert ok
        rec = Recorder(inner=inner)
        ok, got = generate_stream(lib, dev, 6, 1.0, 0.9, 0.2, 0.2, us, rec=rec)
        assert ok and got == want
        assert rec.delivered(0) == got
        assert results[:4] == [(name, False, ERR_CTX | ERR_UNSUPPORTED) for name in ("rwkv_eval", "eval_resident", "state_store", "generate")], results
        assert results[4] == ("clone eval_resident", True, 0), results
        assert L.rwkv_b200_synchronize(other.ptr)
        pair.same("re-entry")
    finally:
        lib.rwkv_free(other)
        pair.free()
        lib.rwkv_free(ctx)


@pytest.mark.gpu
def test_generate_stream_rejections_change_nothing(lib):
    ctx = lib.rwkv_init_from_file(model_path("6v0-3m", "FP32"), 1, 0)
    pair = Pair(lib, ctx)
    bt = None
    try:
        L = lib.library
        V = pair.n_vocab
        err = lambda p: L.rwkv_get_last_error(p)
        pair.prime(LONG_PROMPT[:4])
        us = np.random.RandomState(3).random_sample(12)
        ok, want = generate(lib, pair.host.ptr, 5, 1.0, 1.0, 0.4, 0.4, us[:5])
        ok2, got = generate_stream(lib, pair.dev.ptr, 5, 1.0, 1.0, 0.4, 0.4, us[:5], rec=Recorder())
        assert ok and ok2 and got == want
        before = (state(lib, pair.dev.ptr, pair.n_state).tobytes(), logits(lib, pair.dev.ptr, V).tobytes())
        rec = Recorder()
        # NULL on_token
        ok, _ = generate_stream(lib, pair.dev.ptr, 7, 1.0, 1.0, 0.4, 0.4, us[5:], keep=True, rec=None)
        assert not ok and err(pair.dev.ptr) == ERR_ARGS
        bad_u = us[5:].copy()
        bad_u[2] = 1.0
        cases = [  # the argument errors of test_generate_rejections_change_nothing
            dict(temperature=-1.0), dict(temperature=float("nan")), dict(top_p=1.5), dict(top_p=-0.1), dict(us=bad_u),
            dict(presence=float("nan")), dict(frequency=float("inf")), dict(stops=(V,)), dict(stops=tuple(range(17))), dict(max_tokens=0),
            dict(max_tokens=4097, out_len=4097, us=np.full(4097, 0.5)),
        ]
        base = dict(max_tokens=7, temperature=1.0, top_p=1.0, presence=0.4, frequency=0.4, us=us[5:], stops=())
        for kw in cases:
            a = dict(base, **kw)
            ok, _ = generate_stream(lib, pair.dev.ptr, a["max_tokens"], a["temperature"], a["top_p"], a["presence"], a["frequency"], a["us"], a["stops"],
                                    keep=True, rec=rec, out_len=kw.get("out_len"))
            assert not ok and err(pair.dev.ptr) == ERR_ARGS, kw
        n = ctypes.c_size_t(0)
        toks = np.zeros(7, np.uint32)
        assert not L.rwkv_b200_generate_stream(pair.dev.ptr, 7, 1.0, 1.0, 0.0, 0.0, True, None, None, 0, rec.fn, None, ptr(toks, P_U), ctypes.byref(n))
        assert err(pair.dev.ptr) == ERR_ARGS
        assert not L.rwkv_b200_generate_stream(pair.dev.ptr, 7, 1.0, 1.0, 0.0, 0.0, True, ptr(us, P_D), None, 0, rec.fn, None, None, ctypes.byref(n))
        assert err(pair.dev.ptr) == ERR_ARGS
        # the wrong context kinds
        bt = Batch(lib, ctx, 2)
        assert not generate_stream(lib, bt.ptr, 3, 1.0, 1.0, 0.0, 0.0, us[:3], rec=rec)[0] and err(bt.ptr) == ERR_CTX | ERR_UNSUPPORTED
        ng = np.zeros(1, np.uint32)
        assert not L.rwkv_b200_batch_generate_stream(pair.dev.ptr, ptr(np.array([3], np.uint32), P_U), ptr(f32([1.0]), P_F), ptr(f32([1.0]), P_F),
                                                     ptr(f32([0.0]), P_F), ptr(f32([0.0]), P_F), None, ptr(us, P_D), None, 0, rec.fn, None, ptr(toks, P_U),
                                                     ptr(ng, P_U))
        assert err(pair.dev.ptr) == ERR_CTX | ERR_UNSUPPORTED
        ng2 = np.zeros(2, np.uint32)
        assert not L.rwkv_b200_batch_generate_stream(bt.ptr, ptr(np.array([3, 3], np.uint32), P_U), ptr(f32([1.0] * 2), P_F), ptr(f32([1.0] * 2), P_F),
                                                     ptr(f32([0.0] * 2), P_F), ptr(f32([0.0] * 2), P_F), None, ptr(np.full(6, 0.5), P_D), None, 0, NULL_FN, None,
                                                     ptr(np.zeros(6, np.uint32), P_U), ptr(ng2, P_U))
        assert err(bt.ptr) == ERR_ARGS
        stage = lib.rwkv_b200_init_from_file_ex(model_path("6v0-3m", "FP32"), 0, 0, 1)
        assert not generate_stream(lib, stage.ptr, 3, 1.0, 1.0, 0.0, 0.0, us[:3], rec=rec)[0] and err(stage.ptr) == ERR_CTX | ERR_UNSUPPORTED
        lib.rwkv_free(stage)
        assert rec.calls == []
        assert (state(lib, pair.dev.ptr, pair.n_state).tobytes(), logits(lib, pair.dev.ptr, V).tobytes()) == before
        # the counts are unchanged too: continuing equals the blocking call continuing
        ok, want = generate(lib, pair.host.ptr, 7, 1.0, 1.0, 0.4, 0.4, us[5:], keep=True)
        ok2, got = generate_stream(lib, pair.dev.ptr, 7, 1.0, 1.0, 0.4, 0.4, us[5:], keep=True, rec=Recorder())
        assert ok and ok2 and got == want
        pair.same("after rejections")
        # no logits to draw from
        assert L.rwkv_b200_eval_resident(pair.dev.ptr, ptr(np.array([3], np.uint32), P_U), 1, False, None)
        assert not generate_stream(lib, pair.dev.ptr, 3, 1.0, 1.0, 0.0, 0.0, us[:3], rec=rec)[0] and err(pair.dev.ptr) == ERR_ARGS
    finally:
        if bt:
            bt.free()
        pair.free()
        lib.rwkv_free(ctx)
