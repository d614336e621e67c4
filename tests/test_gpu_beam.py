"""Beam search on the device (rwkv_b200_beam_search, csrc/kernels/beam.cu) against the host search of beam_ref.py, bit for bit:
tokens, lengths, scores and finished flags of every result row, and the state and logits column of every slot the search leaves
live. Also: W = 1 is rwkv_b200_generate at temperature 0; generation continues from any live slot; the step kernel through
rwkv_b200_test_beam_step on planted columns; every refusal changes nothing; one graph launch per call."""
import ctypes

import numpy as np
import pytest

import beam_ref as br
import lora_ref as lr
from beam_ref import P_D, P_F, P_U
from conftest import LONG_PROMPT, VERSIONS, model_path
from test_gpu_generate import Batch, generate, logits, prime, state
from test_gpu_generate_stream import Recorder, batch_generate_stream
from test_gpu_lora_batch import kquant_file

pytestmark = pytest.mark.gpu
ERR_ARGS, ERR_CTX_UNSUPPORTED = 1 << 8, (6 << 8) | 9
P_U8 = ctypes.POINTER(ctypes.c_uint8)


def beam(lib, bt_ptr, W, max_tokens, length_penalty, stops, n_best, finished=True):
    """The raw call: (ok, tokens [n_best][max_tokens], lengths, scores, finished)."""
    toks = np.full((n_best, max_tokens), 7, np.uint32)
    lens, scores, fin = np.zeros(n_best, np.uint32), np.zeros(n_best, np.float64), np.full(n_best, 9, np.uint8)
    st = (ctypes.c_uint32 * max(1, len(stops)))(*stops)
    ok = lib.library.rwkv_b200_beam_search(bt_ptr, max_tokens, length_penalty, st, len(stops), n_best, toks.ctypes.data_as(P_U),
                                           lens.ctypes.data_as(P_U), scores.ctypes.data_as(P_D), fin.ctypes.data_as(P_U8) if finished else None)
    return ok, toks, lens, scores, fin


class Setup:
    """A single-sequence context (the reference's evaluator) and a batch of W sequences whose sequence 0 holds `prompt`."""

    def __init__(self, lib, path, W):
        self.lib, self.W = lib, W
        self.ctx = lib.rwkv_init_from_file(path, 1, 0)
        self.n_state = lib.rwkv_get_state_buffer_element_count(self.ctx)
        self.V = lib.rwkv_get_logits_buffer_element_count(self.ctx)
        self.bt = Batch(lib, self.ctx, W)
        self.ref = br.ModelBeams(lib, self.ctx.ptr, self.n_state, self.V)

    def prime(self, prompt):
        self.bt.prime([prompt] + [[(t * (s + 3) + s) % self.V for t in prompt] for s in range(1, self.W)])
        return self.root()

    def root(self):
        return self.bt.state(0, self.n_state), self.bt.logits(0, self.V)

    def check(self, root, max_tokens, length_penalty, stops, what):
        """Device search against the host one from root; returns the device results."""
        ok, toks, lens, scores, fin = beam(self.lib, self.bt.ptr, self.W, max_tokens, length_penalty, stops, self.W)
        assert ok, (what, self.lib.rwkv_get_last_error(None))
        want, last = self.ref.search(root, self.W, max_tokens, length_penalty, stops, self.W)
        for r in range(self.W):
            if r < len(want):
                wt, ws, wf = want[r]
                assert [int(t) for t in toks[r, :lens[r]]] == wt, (what, r)
                assert not toks[r, lens[r]:].any(), (what, r)
                assert scores[r] == ws and bool(fin[r]) == wf, (what, r, scores[r], ws)
            else:
                assert lens[r] == 0 and scores[r] == -np.inf and fin[r] == 0 and not toks[r].any(), (what, r)
        for k, (_, _, (st, lg)) in enumerate(last):
            assert self.bt.state(k, self.n_state).tobytes() == st.tobytes(), (what, "state of slot", k)
            assert self.bt.logits(k, self.V).tobytes() == lg.tobytes(), (what, "logits of slot", k)
        return toks, lens, scores, fin

    def free(self):
        self.bt.free()
        self.lib.rwkv_free(self.ctx)


def prompt_for(V, seed=0):
    return [(LONG_PROMPT[(i + seed) % len(LONG_PROMPT)] + 13 * seed) % V for i in range(6)]


def stop_sets(root_logits, W):
    """mid: two ids ranked just below the root's best, so some hypotheses end mid-search; fill: 16 ids among the root's top entries,
    so that the pool fills early."""
    top = [int(t) for t in br.top_order(root_logits, 40)]
    return {"none": (), "mid": (top[1], top[3]), "fill": tuple(top[1:33:2])}


CASES = [(1, 24, 0.0, "none"), (2, 24, 1.0, "mid"), (4, 24, -0.5, "mid"), (10, 24, 1.0, "fill"), (4, 1, 1.0, "none"), (10, 1, 0.0, "fill")]


@pytest.mark.parametrize("ver", VERSIONS)
@pytest.mark.parametrize("fmt", ["FP32", "Q5_1"])
def test_search_matches_the_host_search(lib, ver, fmt):
    for W, max_tokens, lp, kind in CASES:
        s = Setup(lib, model_path(ver, fmt), W)
        try:
            root = s.prime(prompt_for(s.V, W))
            s.check(root, max_tokens, lp, stop_sets(root[1], W)[kind], (ver, fmt, W, max_tokens, lp, kind))
        finally:
            s.free()


def test_search_on_k_quants(lib, tmp_path):
    path = kquant_file(lib, tmp_path)
    for W, kind in ((2, "mid"), (4, "fill")):
        s = Setup(lib, path, W)
        try:
            root = s.prime(prompt_for(s.V, 1))
            s.check(root, 16, 1.0, stop_sets(root[1], W)[kind], ("Q4_K", W, kind))
        finally:
            s.free()


def test_adapter_and_recapture(lib):
    """A context-wide adapter with non-zero B on the batch and the reference context; then a second search after the tensor-core switch
    and after detaching and re-attaching the adapter, each of which re-captures the loop."""
    path = model_path("6v0-3m", "Q5_1")
    s = Setup(lib, path, 4)
    ad = lib.rwkv_b200_adapter_create(s.ctx, lr.make_entries(path, 8, 3, b_scale=0.2), 1.5)
    try:
        root0 = s.prime(prompt_for(s.V, 2))
        lib.rwkv_b200_set_adapter(s.ctx, ad)
        assert lib.library.rwkv_b200_set_adapter(s.bt.ptr, ad)
        root = s.prime(prompt_for(s.V, 2))
        assert root[1].tobytes() != root0[1].tobytes(), "the adapter changed nothing"
        stops = stop_sets(root[1], 4)["mid"]
        s.check(root, 12, 1.0, stops, "adapter")
        root = s.prime(prompt_for(s.V, 3))
        lib.library.rwkv_b200_set_tensor_cores(s.bt.ptr, False)
        s.check(root, 12, 1.0, stops, "tensor cores off")
        lib.library.rwkv_b200_set_tensor_cores(s.bt.ptr, True)
        assert lib.library.rwkv_b200_set_adapter(s.bt.ptr, None)
        lib.rwkv_b200_set_adapter(s.ctx, None)
        root = s.prime(prompt_for(s.V, 4))
        s.check(root, 12, 0.0, stops, "detached")
        assert lib.library.rwkv_b200_set_adapter(s.bt.ptr, ad)
        lib.rwkv_b200_set_adapter(s.ctx, ad)
        root = s.prime(prompt_for(s.V, 5))
        s.check(root, 12, -0.5, stops, "re-attached")
        s.check(s.root(), 7, 1.0, (), "from slot 0 of the last search")
    finally:
        assert lib.library.rwkv_b200_set_adapter(s.bt.ptr, None)
        lib.rwkv_b200_set_adapter(s.ctx, None)
        s.free()
        lib.rwkv_b200_adapter_free(ad)


@pytest.mark.parametrize("ver", VERSIONS)
def test_width_one_is_greedy_generation(lib, ver):
    path = model_path(ver, "FP32")
    s = Setup(lib, path, 1)
    single = lib.rwkv_init_from_file(path, 1, 0)
    try:
        p = prompt_for(s.V, 7)
        prime(lib, single.ptr, p)
        s.prime(p)
        ok, greedy = generate(lib, single.ptr, 12, 0.0, 1.0, 0.0, 0.0, [0.5] * 12)
        assert ok
        for stops, n in (((), 12), ((greedy[3],), 12), ((), 5)):
            prime(lib, single.ptr, p)
            s.prime(p)
            ok, want = generate(lib, single.ptr, n, 0.0, 1.0, 0.0, 0.0, [0.5] * n, stops)
            assert ok
            ok, toks, lens, scores, fin = beam(lib, s.bt.ptr, 1, n, 1.0, stops, 1)
            assert ok and [int(t) for t in toks[0, :lens[0]]] == want, (ver, stops, n)
            assert bool(fin[0]) == (len(stops) > 0), (ver, stops)
            assert s.bt.state(0, s.n_state).tobytes() == state(lib, single.ptr, s.n_state).tobytes(), (ver, stops, n)
            assert s.bt.logits(0, s.V).tobytes() == logits(lib, single.ptr, s.V).tobytes(), (ver, stops, n)
    finally:
        lib.rwkv_free(single)
        s.free()


@pytest.mark.parametrize("ver", ["5v2-730K", "7v0-834K"])
def test_generation_continues_from_every_live_slot(lib, ver):
    path = model_path(ver, "Q5_1")
    W, n = 4, 5
    s = Setup(lib, path, W)
    single = lib.rwkv_init_from_file(path, 1, 0)
    try:
        p = prompt_for(s.V, 8)
        s.prime(p)
        ok, toks, lens, scores, fin = beam(lib, s.bt.ptr, W, 6, 1.0, (), W)
        assert ok and not fin.any() and (lens == 6).all()
        # without stops every result row is a live beam of the last step; find the row each slot holds by its state
        slots = []
        for k in range(W):
            for r in range(W):
                seq = p + [int(t) for t in toks[r, :lens[r]]]
                prime(lib, single.ptr, seq)
                if state(lib, single.ptr, s.n_state).tobytes() == s.bt.state(k, s.n_state).tobytes():
                    slots.append(seq)
                    break
            else:
                raise AssertionError(("no result row holds slot", k))
        temps, tops = [1.0, 0.7, 1.0, 0.0], [0.9, 1.0, 0.5, 1.0]
        us = np.random.default_rng(5).random((W, n))
        ok, got = s.bt.generate([n] * W, temps, tops, [0.0] * W, [0.0] * W, us, ())
        assert ok
        for k in range(W):
            prime(lib, single.ptr, slots[k])
            ok, want = generate(lib, single.ptr, n, temps[k], tops[k], 0.0, 0.0, us[k])
            assert ok and got[k] == want, (ver, k)
            assert s.bt.state(k, s.n_state).tobytes() == state(lib, single.ptr, s.n_state).tobytes(), (ver, k)
            assert s.bt.logits(k, s.V).tobytes() == logits(lib, single.ptr, s.V).tobytes(), (ver, k)
    finally:
        lib.rwkv_free(single)
        s.free()


# ---- the step kernel on planted columns ----------------------------------------------------------------------------------------

def hook_step(lib, z, scores, W, n_pool, stops):
    import rwkv_cpp_b200.shared_library as sl
    L, V = z.shape
    z = np.ascontiguousarray(z, np.float32)
    sc = np.ascontiguousarray(scores, np.float64)
    st = np.ascontiguousarray(stops, np.uint32) if len(stops) else None
    n_live, n_pool_out = np.zeros(1, np.uint32), np.zeros(1, np.uint32)
    par, tok, pp, pt = (np.full(W, 0xFFFF, np.uint32) for _ in range(4))
    so, ps = np.zeros(W, np.float64), np.zeros(W, np.float64)
    a = sl.BeamStepArgs(z.ctypes.data_as(P_F), W, V, L, sc.ctypes.data_as(P_D), n_pool, st.ctypes.data_as(P_U) if st is not None else None,
                        len(stops), n_live.ctypes.data_as(P_U), par.ctypes.data_as(P_U), tok.ctypes.data_as(P_U), so.ctypes.data_as(P_D),
                        n_pool_out.ctypes.data_as(P_U), pp.ctypes.data_as(P_U), pt.ctypes.data_as(P_U), ps.ctypes.data_as(P_D))
    assert lib.library.rwkv_b200_test_beam_step(ctypes.byref(a)), lib.rwkv_get_last_error(None)
    Lo, Po = int(n_live[0]), int(n_pool_out[0])
    taken = [(int(par[k]), int(tok[k]), float(so[k])) for k in range(Lo)]
    finished = [(int(pp[q]), int(pt[q]), float(ps[q])) for q in range(n_pool, Po)]
    return taken, finished


def python_step(lib, z, scores, W, n_pool, stops):
    return br.walk([br.model_candidates(lib, z[b], W) for b in range(z.shape[0])], list(scores), W, n_pool, set(stops))


def planted(V, W, rng):
    """(name, logits [L][V], scores, n_pool, stops) cases."""
    n = 2 * W
    base = lambda: (rng.standard_normal(V) * 2).astype(np.float32)
    out = []
    z = base()
    z[:] = np.minimum(z, 5.0)
    hi = [(i * 997 + 3) % V for i in range(n - 1)]
    for j, i in enumerate(hi):
        z[i] = 20.0 - j
    ties = [i for i in (1023, 1024, 2047, 2048, V - 1) if i < V and i not in hi] or [i for i in range(V) if i not in hi][:3]
    z[ties] = 10.0       # the 2W-th entry is a tie across a thread boundary of the top-N layout
    out.append(("tie at 2W", z[None], [0.0], 0, ()))
    z2 = base()
    out.append(("equal scores across beams", np.stack([z2, z2, base()][:min(3, W)]), [-1.25] * min(3, W), 0, ()))
    z3 = np.full(V, -np.inf, np.float32)
    z3[V // 2] = 1.0
    z4 = base()
    z4[V // 3] = np.nan
    out.append(("-inf but one, and a NaN column", np.stack([z3, z4]) if W >= 2 else z3[None], [-0.5, -0.25][:min(2, W)], 0, ()))
    z5 = base()
    z5[V - 1] = 30.0
    out.append(("stop id at V - 1", z5[None], [0.0], min(1, W - 1), (V - 1,)))
    z6 = np.full(V, -np.inf, np.float32)
    z6[[0, V - 1]] = [2.0, 1.0]
    z6[V // 2] = 3.0
    out.append(("fewer finite candidates than W", z6[None], [0.0], 0, (V // 2,)))
    z7 = np.stack([base() for _ in range(W)])
    top = [int(t) for t in br.top_order(z7[0], 4)]
    out.append(("a pool that fills", z7, list(-rng.random(W)), W - 1, tuple(top)))
    return out


@pytest.mark.parametrize("V", [16, 50277, 65536])
@pytest.mark.parametrize("W", [1, 4, 10])
def test_step_hook_matches_the_python_step(lib, V, W):
    rng = np.random.default_rng(V + W)
    for name, z, scores, n_pool, stops in planted(V, W, rng):
        z = z[:W]
        got = hook_step(lib, z, scores[:z.shape[0]], W, n_pool, stops)
        want = python_step(lib, z, scores[:z.shape[0]], W, n_pool, stops)
        assert got == want, (V, W, name, got, want)


# ---- refusals and launches -------------------------------------------------------------------------------------------------------

def test_refusals_change_nothing(lib):
    path = model_path("6v0-3m", "Q5_1")
    s = Setup(lib, path, 3)
    big = Batch(lib, s.ctx, 11)
    stage = lib.rwkv_b200_init_from_file_ex(path, 0, 0, 1)
    ad = lib.rwkv_b200_adapter_create(s.ctx, lr.make_entries(path, 4, 1, b_scale=0.2), 1.0)
    try:
        s.prime(prompt_for(s.V, 9))
        before = [(s.bt.state(k, s.n_state).tobytes(), s.bt.logits(k, s.V).tobytes()) for k in range(3)]

        def refused(err, what, ptr=None, **kw):
            args = dict(max_tokens=4, length_penalty=1.0, stops=(), n_best=2)
            args.update(kw)
            ptr = ptr or s.bt.ptr
            ok, *_ = beam(lib, ptr, 3, args["max_tokens"], args["length_penalty"], args["stops"], args["n_best"])
            assert not ok, what
            assert lib.library.rwkv_get_last_error(ptr) == err, what
            assert [(s.bt.state(k, s.n_state).tobytes(), s.bt.logits(k, s.V).tobytes()) for k in range(3)] == before, what

        refused(ERR_CTX_UNSUPPORTED, "ordinary context", s.ctx.ptr)
        refused(ERR_CTX_UNSUPPORTED, "stage", stage.ptr)
        refused(ERR_ARGS, "width 11", big.ptr)
        refused(ERR_ARGS, "n_best 0", n_best=0)
        refused(ERR_ARGS, "n_best above W", n_best=4)
        refused(ERR_ARGS, "max_tokens 0", max_tokens=0)
        refused(ERR_ARGS, "max_tokens above the limit", max_tokens=4097)
        refused(ERR_ARGS, "inf length penalty", length_penalty=float("inf"))
        refused(ERR_ARGS, "NaN length penalty", length_penalty=float("nan"))
        refused(ERR_ARGS, "17 stop ids", stops=tuple(range(17)))
        refused(ERR_ARGS, "stop id n_vocab", stops=(s.V,))
        for arr in range(3):
            toks, lens, scores = np.zeros((2, 4), np.uint32), np.zeros(2, np.uint32), np.zeros(2, np.float64)
            ptrs = [toks.ctypes.data_as(P_U), lens.ctypes.data_as(P_U), scores.ctypes.data_as(P_D)]
            ptrs[arr] = None
            assert not lib.library.rwkv_b200_beam_search(s.bt.ptr, 4, 1.0, None, 0, 2, *ptrs, None)
            assert lib.library.rwkv_get_last_error(s.bt.ptr) == ERR_ARGS, arr
        assert lib.library.rwkv_b200_batch_set_adapter(s.bt.ptr, 1, ad)
        refused(ERR_ARGS, "a sequence with its own adapter")
        assert lib.library.rwkv_b200_batch_set_adapter(s.bt.ptr, 1, None)
        inside = []
        rec = Recorder(inner=lambda seq, idx, tok: inside.append((beam(lib, s.bt.ptr, 3, 4, 1.0, (), 2)[0], lib.library.rwkv_get_last_error(s.bt.ptr))))
        s.prime(prompt_for(s.V, 9))
        ok, _ = batch_generate_stream(s.bt, [1, 0, 0], [1.0] * 3, [1.0] * 3, [0.0] * 3, [0.0] * 3, np.full((3, 1), 0.5), (), rec)
        assert ok and inside == [(False, ERR_CTX_UNSUPPORTED)], inside
        s.prime(prompt_for(s.V, 9))
        assert lib.library.rwkv_b200_batch_eval(s.bt.ptr, (ctypes.c_uint32 * 3)(1, 2, 3), False)
        states = [s.bt.state(k, s.n_state).tobytes() for k in range(3)]
        ok, *_ = beam(lib, s.bt.ptr, 3, 4, 1.0, (), 2)
        assert not ok and lib.library.rwkv_get_last_error(s.bt.ptr) == ERR_ARGS, "invalid logits"
        assert [s.bt.state(k, s.n_state).tobytes() for k in range(3)] == states
        lg = np.zeros(s.V, np.float32)
        assert not lib.library.rwkv_b200_batch_get_logits(s.bt.ptr, 0, lg.ctypes.data_as(P_F)), "the logits became valid"
    finally:
        big.free()
        lib.rwkv_free(stage)
        s.free()
        lib.rwkv_b200_adapter_free(ad)


def test_one_graph_launch_per_call(lib):
    """The first call runs one uncaptured pass and captures the gather and one batch pass of W sequences (the step is a graph node of
    its own); every call is one graph launch, and a replay enqueues no kernel from the host."""
    path = model_path("6v0-3m", "Q5_1")
    W = 4
    s = Setup(lib, path, W)
    try:
        s.prime(prompt_for(s.V, 10))
        L = lib.library
        k0 = L.rwkv_b200_kernel_launch_count()
        assert L.rwkv_b200_batch_eval(s.bt.ptr, (ctypes.c_uint32 * W)(1, 2, 3, 4), True)
        per_pass = L.rwkv_b200_kernel_launch_count() - k0
        for call in range(3):
            if call == 2:
                L.rwkv_b200_set_tensor_cores(s.bt.ptr, False)
            g0, k0 = L.rwkv_b200_graph_launch_count(), L.rwkv_b200_kernel_launch_count()
            ok, *_ = beam(lib, s.bt.ptr, W, 8, 1.0, (), 1)
            assert ok
            assert L.rwkv_b200_graph_launch_count() - g0 == 1, call
            assert L.rwkv_b200_kernel_launch_count() - k0 == (2 * per_pass + 1 if call != 1 else 0), call
    finally:
        s.free()
