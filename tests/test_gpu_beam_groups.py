"""Grouped beam search on the device (rwkv_b200_beam_search_groups) bit for bit: every group against beam_ref's search from its own
root below 16 sequences and with the tensor cores off, and against a host lockstep search over batch passes of the same batch with
them on; G = 1 against rwkv_b200_beam_search; groups under per-sequence adapters; generation continuing from the slots; the grouped
step kernel through rwkv_b200_test_beam_step_groups; refusals; one graph launch per call."""
import ctypes

import numpy as np
import pytest

import beam_groups_ref as bg
import beam_ref as br
import lora_ref as lr
from beam_ref import P_D, P_F, P_U
from conftest import VERSIONS, model_path
from test_gpu_beam import beam, hook_step, planted, prompt_for, stop_sets
from test_gpu_generate import Batch, generate, prime, state
from test_gpu_generate_stream import Recorder, batch_generate_stream
from test_gpu_lora_batch import kquant_file

pytestmark = pytest.mark.gpu
ERR_ARGS, ERR_CTX_UNSUPPORTED = 1 << 8, (6 << 8) | 9
P_U8 = ctypes.POINTER(ctypes.c_uint8)


def beam_groups(lib, ptr, G, max_tokens, penalties, stops, n_best):
    """The raw call: (ok, tokens [G][n_best][n], lengths, scores, finished)."""
    n = max(1, max(max_tokens))
    toks = np.full((G, n_best, n), 7, np.uint32)
    lens, scores, fin = np.zeros((G, n_best), np.uint32), np.zeros((G, n_best), np.float64), np.full((G, n_best), 9, np.uint8)
    st = (ctypes.c_uint32 * max(1, len(stops)))(*stops)
    ok = lib.library.rwkv_b200_beam_search_groups(ptr, G, np.ascontiguousarray(max_tokens, np.uint32).ctypes.data_as(P_U),
                                                  np.ascontiguousarray(penalties, np.float32).ctypes.data_as(P_F), st, len(stops), n_best,
                                                  toks.ctypes.data_as(P_U), lens.ctypes.data_as(P_U), scores.ctypes.data_as(P_D),
                                                  fin.ctypes.data_as(P_U8))
    return ok, toks, lens, scores, fin


class Groups:
    """A batch of G * W sequences whose sequence g * W holds group g's prompt, and a single-sequence context for the reference."""

    def __init__(self, lib, path, G, W, tensor_cores=True):
        self.lib, self.G, self.W, self.N = lib, G, W, G * W
        self.ctx = lib.rwkv_init_from_file(path, 1, 0)
        self.n_state = lib.rwkv_get_state_buffer_element_count(self.ctx)
        self.V = lib.rwkv_get_logits_buffer_element_count(self.ctx)
        self.bt = Batch(lib, self.ctx, self.N)
        if not tensor_cores:
            lib.library.rwkv_b200_set_tensor_cores(self.bt.ptr, False)
        self.ref = br.ModelBeams(lib, self.ctx.ptr, self.n_state, self.V)

    def prime(self, seed):
        self.prompts = [prompt_for(self.V, seed + s) for s in range(self.N)]
        self.bt.prime(self.prompts)
        return [self.slot(g * self.W) for g in range(self.G)]

    def slot(self, k):
        return self.bt.state(k, self.n_state), self.bt.logits(k, self.V)

    def slots(self):
        return [self.slot(k) for k in range(self.N)]

    def check(self, found, before, max_tokens, penalties, stops, what):
        """Device call against `found` (bg.search_groups' output): results of every group, the slots of its last step that took beams,
        and every slot of an idle group."""
        G, W = self.G, self.W
        ok, toks, lens, scores, fin = beam_groups(self.lib, self.bt.ptr, G, max_tokens, penalties, stops, W)
        assert ok, (what, self.lib.rwkv_get_last_error(None))
        want = bg.results_groups(found, penalties, W)
        for g in range(G):
            for r in range(W):
                if r < len(want[g]):
                    wt, ws, wf = want[g][r]
                    assert [int(t) for t in toks[g, r, :lens[g, r]]] == wt, (what, g, r)
                    assert not toks[g, r, lens[g, r]:].any(), (what, g, r)
                    assert scores[g, r] == ws and bool(fin[g, r]) == wf, (what, g, r, scores[g, r], ws)
                else:
                    assert lens[g, r] == 0 and scores[g, r] == -np.inf and fin[g, r] == 0 and not toks[g, r].any(), (what, g, r)
            kept = [h for _, _, h in found[g][2]] if max_tokens[g] else before[g * W:(g + 1) * W]
            for k, (st, lg) in enumerate(kept):
                assert self.bt.state(g * W + k, self.n_state).tobytes() == st.tobytes(), (what, g, "state of slot", k)
                assert self.bt.logits(g * W + k, self.V).tobytes() == lg.tobytes(), (what, g, "logits of slot", k)
        return toks, lens

    def free(self):
        self.bt.free()
        self.lib.rwkv_free(self.ctx)


def layout(G, W, roots, rng):
    """Mixed max_tokens (0 and 1 among them while G allows), per-group penalties, and stop ids from group 1's root that end some
    hypotheses mid-search and fill some pools early."""
    mt = [int(x) for x in rng.integers(2, 13, G)]
    if G >= 3:
        mt[0], mt[2] = 0, 1
    pen = [float(x) for x in rng.choice([-0.5, 0.0, 1.0, 1.5], G)]
    kind = "fill" if W <= 3 else "mid"
    return mt, pen, stop_sets(roots[min(1, G - 1)][1], W)[kind]


def run_host_reference(s, roots, mt, pen, stops):
    return bg.search_groups(roots, s.W, mt, set(stops), s.ref.candidates(s.W), bg.one_by_one(s.ref.advance))


@pytest.mark.parametrize("ver", VERSIONS)
@pytest.mark.parametrize("fmt", ["FP32", "Q5_1"])
def test_groups_match_the_search_from_each_root(lib, ver, fmt):
    rng = np.random.default_rng(hash((ver, fmt)) % 1000)
    for G, W in ((2, 2), (3, 4), (5, 3)):
        s = Groups(lib, model_path(ver, fmt), G, W)
        try:
            roots = s.prime(G * 7 + W)
            before = s.slots()
            mt, pen, stops = layout(G, W, roots, rng)
            s.check(run_host_reference(s, roots, mt, pen, stops), before, mt, pen, stops, (ver, fmt, G, W))
        finally:
            s.free()


def test_groups_on_k_quants_and_without_tensor_cores(lib, tmp_path):
    rng = np.random.default_rng(3)
    cases = [(kquant_file(lib, tmp_path), 3, 4, True), (model_path("6v0-3m", "Q5_1"), 8, 4, False), (model_path("5v2-730K", "FP32"), 64, 4, False)]
    for path, G, W, tc in cases:
        s = Groups(lib, path, G, W, tensor_cores=tc)
        try:
            roots = s.prime(G + W)
            before = s.slots()
            mt, pen, stops = layout(G, W, roots, rng)
            if G == 64:
                mt = [m % 6 for m in mt]        # several idle groups among 64, and short searches
                mt[1] = 5
            s.check(run_host_reference(s, roots, mt, pen, stops), before, mt, pen, stops, (path, G, W, tc))
        finally:
            s.free()


def batch_lockstep(s):
    """advance_all over the batch: each taken beam's parent state into its slot, one rwkv_b200_batch_eval of all N columns, then the
    state and logits of the taken slots as the new handles. The slots of other groups run the pass on whatever they hold."""
    def advance_all(moves):
        if not any(m for m in moves if m):
            return [None if m is None else [] for m in moves]
        tokens = [0] * s.N
        for g, m in enumerate(moves):
            for k, ((st, _), tok) in enumerate(m or []):
                assert s.lib.library.rwkv_b200_batch_set_state(s.bt.ptr, g * s.W + k, st.ctypes.data_as(P_F))
                tokens[g * s.W + k] = tok
        assert s.bt.eval(tokens)
        return [None if m is None else [s.slot(g * s.W + k) for k in range(len(m))] for g, m in enumerate(moves)]
    return advance_all


@pytest.mark.parametrize("G,W", [(4, 4), (8, 4), (25, 10)])
def test_tensor_cores_match_a_host_lockstep_search(lib, G, W):
    path = model_path("6v0-3m", "Q5_1")
    rng = np.random.default_rng(G * W)
    s = Groups(lib, path, G, W)
    try:
        roots = s.prime(G)
        before = s.slots()
        mt, pen, stops = layout(G, W, roots, rng)
        mt = [min(m, 8) for m in mt]
        found = bg.search_groups(roots, W, mt, set(stops), s.ref.candidates(W), batch_lockstep(s))
        s.bt.prime(s.prompts)       # every slot back as it was before the host search
        assert all(a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() for a, b in zip(s.slots(), before))
        s.check(found, before, mt, pen, stops, ("tensor cores", G, W))
    finally:
        s.free()


def test_one_group_is_beam_search(lib):
    """Results, the slots of the last step that took beams, and the launches of the capturing call and of replays."""
    path = model_path("7v0-834K", "Q5_1")
    W = 4
    a, b = Groups(lib, path, 1, W), Groups(lib, path, 1, W)
    L = lib.library
    try:
        for call, (n, pen, kind) in enumerate(((9, 1.0, "mid"), (6, -0.5, "fill"), (9, 0.0, "none"))):
            roots = a.prime(call)
            b.prime(call)
            stops = stop_sets(roots[0][1], W)[kind]
            _, last = a.ref.search(roots[0], W, n, pen, stops, W)
            g0, k0 = L.rwkv_b200_graph_launch_count(), L.rwkv_b200_kernel_launch_count()
            got = beam_groups(lib, a.bt.ptr, 1, [n], [pen], stops, W)
            counts_a = (L.rwkv_b200_graph_launch_count() - g0, L.rwkv_b200_kernel_launch_count() - k0)
            g0, k0 = L.rwkv_b200_graph_launch_count(), L.rwkv_b200_kernel_launch_count()
            want = beam(lib, b.bt.ptr, W, n, pen, stops, W)
            counts_b = (L.rwkv_b200_graph_launch_count() - g0, L.rwkv_b200_kernel_launch_count() - k0)
            assert got[0] and want[0]
            assert got[1][0].tobytes() == want[1].tobytes() and all(x[0].tobytes() == y.tobytes() for x, y in zip(got[2:], want[2:])), call
            assert counts_a == counts_b and counts_a[0] == 1, (call, counts_a, counts_b)
            for k in range(len(last)):
                assert a.slot(k)[0].tobytes() == b.slot(k)[0].tobytes() and a.slot(k)[1].tobytes() == b.slot(k)[1].tobytes(), (call, k)
    finally:
        a.free()
        b.free()


def test_groups_under_per_sequence_adapters(lib):
    """Groups of 2 carrying adapter X, adapter Y and the base; each equals rwkv_b200_beam_search on a 2-sequence batch with that adapter
    context-wide. A group whose two sequences hold different adapters is refused and changes nothing."""
    path = model_path("6v0-3m", "Q5_1")
    G, W = 3, 2
    s = Groups(lib, path, G, W)
    X = lib.rwkv_b200_adapter_create(s.ctx, lr.make_entries(path, 8, 11, b_scale=0.2), 1.5)
    Y = lib.rwkv_b200_adapter_create(s.ctx, lr.make_entries(path, 8, 12, b_scale=0.2), 1.0)
    single = Batch(lib, s.ctx, W)
    try:
        for k, ad in enumerate([X, X, Y, Y, None, None]):
            assert lib.library.rwkv_b200_batch_set_adapter(s.bt.ptr, k, ad)
        s.prime(40)
        mt, pen = [7, 5, 6], [1.0, 0.0, -0.5]
        ok, toks, lens, scores, fin = beam_groups(lib, s.bt.ptr, G, mt, pen, (), W)
        assert ok
        for g, ad in enumerate([X, Y, None]):
            assert lib.library.rwkv_b200_set_adapter(single.ptr, ad)
            single.prime(s.prompts[g * W:(g + 1) * W])
            ok1, t1, l1, s1, f1 = beam(lib, single.ptr, W, mt[g], pen[g], (), W)
            assert ok1 and (l1 == mt[g]).all()          # no stop ids: every row, and so every slot, is a live beam of the last step
            n = mt[g]
            assert (toks[g, :, :n] == t1).all() and (lens[g] == l1).all() and (scores[g] == s1).all() and (fin[g] == f1).all(), g
            assert not toks[g, :, n:].any()
            for k in range(W):
                assert s.bt.state(g * W + k, s.n_state).tobytes() == single.state(k, s.n_state).tobytes(), (g, k)
                assert s.bt.logits(g * W + k, s.V).tobytes() == single.logits(k, s.V).tobytes(), (g, k)
            assert lib.library.rwkv_b200_set_adapter(single.ptr, None)
        assert lib.library.rwkv_b200_batch_set_adapter(s.bt.ptr, 1, Y)
        s.prime(41)
        before = s.slots()
        ok, *_ = beam_groups(lib, s.bt.ptr, G, mt, pen, (), W)
        assert not ok and lib.library.rwkv_get_last_error(s.bt.ptr) == ERR_ARGS
        assert all(a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() for a, b in zip(s.slots(), before))
    finally:
        for k in range(s.N):
            lib.library.rwkv_b200_batch_set_adapter(s.bt.ptr, k, None)
        single.free()
        s.free()
        lib.rwkv_b200_adapter_free(X)
        lib.rwkv_b200_adapter_free(Y)


def test_generation_continues_from_every_defined_slot(lib):
    path = model_path("5v2-730K", "Q5_1")
    G, W, n = 3, 3, 4
    s = Groups(lib, path, G, W)
    single = lib.rwkv_init_from_file(path, 1, 0)
    try:
        roots = s.prime(50)
        mt, pen = [0, 5, 2], [1.0, 1.0, 0.0]
        found = run_host_reference(s, roots, mt, pen, ())
        s.prime(50)
        ok, *_ = beam_groups(lib, s.bt.ptr, G, mt, pen, (), W)
        assert ok
        seqs = {}
        for g in range(G):
            if mt[g] == 0:
                for k in range(W):
                    seqs[g * W + k] = s.prompts[g * W + k]
            else:
                for k, (_, toks, _) in enumerate(found[g][2]):
                    seqs[g * W + k] = s.prompts[g * W] + toks
        temps, tops = [0.8] * s.N, [0.9] * s.N
        us = np.random.default_rng(9).random((s.N, n))
        ok, got = s.bt.generate([n if k in seqs else 0 for k in range(s.N)], temps, tops, [0.0] * s.N, [0.0] * s.N, us, ())
        assert ok
        for k, seq in seqs.items():
            prime(lib, single.ptr, seq)
            ok, want = generate(lib, single.ptr, n, temps[k], tops[k], 0.0, 0.0, us[k])
            assert ok and got[k] == want, k
            assert s.bt.state(k, s.n_state).tobytes() == state(lib, single.ptr, s.n_state).tobytes(), k
    finally:
        lib.rwkv_free(single)
        s.free()


# ---- the grouped step kernel on planted columns --------------------------------------------------------------------------------

@pytest.mark.parametrize("V", [16, 50277, 65536])
def test_grouped_step_hook_matches_the_single_step_hook(lib, V):
    import rwkv_cpp_b200.shared_library as sl
    W = 4
    rng = np.random.default_rng(V)
    cases = [(z[:W], list(sc[:z[:W].shape[0]]), n_pool, stops) for _, z, sc, n_pool, stops in planted(V, W, rng)]
    cases += [(np.zeros((0, V), np.float32), [], 0, ()), (cases[0][0], cases[0][1], W, ())]     # an idle group, a full pool
    G = len(cases)
    keep, arr = [], (sl.BeamStepArgs * G)()
    outs = []
    for g, (z, sc, n_pool, stops) in enumerate(cases):
        z = np.ascontiguousarray(z, np.float32)
        scd = np.ascontiguousarray(sc if len(sc) else [0.0], np.float64)
        st = np.ascontiguousarray(stops if len(stops) else [0], np.uint32)
        o = dict(n_live=np.full(1, 77, np.uint32), n_pool=np.full(1, 77, np.uint32), par=np.full(W, 0xFFFF, np.uint32), tok=np.full(W, 0xFFFF, np.uint32),
                 so=np.zeros(W), pp=np.full(W, 0xFFFF, np.uint32), pt=np.full(W, 0xFFFF, np.uint32), ps=np.zeros(W))
        keep += [z, scd, st]
        outs.append(o)
        arr[g] = sl.BeamStepArgs(z.ctypes.data_as(P_F) if z.shape[0] else None, W, V, z.shape[0], scd.ctypes.data_as(P_D), n_pool,
                                 st.ctypes.data_as(P_U), len(stops), o["n_live"].ctypes.data_as(P_U), o["par"].ctypes.data_as(P_U),
                                 o["tok"].ctypes.data_as(P_U), o["so"].ctypes.data_as(P_D), o["n_pool"].ctypes.data_as(P_U),
                                 o["pp"].ctypes.data_as(P_U), o["pt"].ctypes.data_as(P_U), o["ps"].ctypes.data_as(P_D))
    assert lib.library.rwkv_b200_test_beam_step_groups(arr, G), lib.rwkv_get_last_error(None)
    for g, (z, sc, n_pool, stops) in enumerate(cases):
        o = outs[g]
        Lo, Po = int(o["n_live"][0]), int(o["n_pool"][0])
        if z.shape[0] == 0 or n_pool == W:
            assert (Lo, Po) == (z.shape[0], n_pool) and (o["par"] == 0xFFFF).all() and (o["pp"] == 0xFFFF).all(), g
            continue
        got = ([(int(o["par"][k]), int(o["tok"][k]), float(o["so"][k])) for k in range(Lo)],
               [(int(o["pp"][q]), int(o["pt"][q]), float(o["ps"][q])) for q in range(n_pool, Po)])
        assert got == hook_step(lib, z, sc, W, n_pool, stops), (V, g)


# ---- refusals and launches -------------------------------------------------------------------------------------------------------

def test_refusals_change_nothing(lib):
    """Every refusal leaves the states, the logits and their validity, and the per-sequence adapters as they were. Group 0 carries
    adapter X on all three of its sequences, which is allowed; the adapters are checked at the end by a pass against a second batch
    with the same attachments."""
    path = model_path("6v0-3m", "Q5_1")
    s = Groups(lib, path, 2, 3)
    big = Batch(lib, s.ctx, 22)
    stage = lib.rwkv_b200_init_from_file_ex(path, 0, 0, 1)
    pipe = ctypes.c_void_p(lib.library.rwkv_b200_init_pipeline(path.encode(), (ctypes.c_int * 2)(0, 0), 2))
    assert pipe.value
    X = lib.rwkv_b200_adapter_create(s.ctx, lr.make_entries(path, 4, 1, b_scale=0.2), 1.0)
    Y = lib.rwkv_b200_adapter_create(s.ctx, lr.make_entries(path, 4, 2, b_scale=0.2), 1.0)
    ref = Batch(lib, s.ctx, 6)
    try:
        for k in range(3):
            assert lib.library.rwkv_b200_batch_set_adapter(s.bt.ptr, k, X) and lib.library.rwkv_b200_batch_set_adapter(ref.ptr, k, X)
        s.prime(60)
        before = s.slots()

        def unchanged(what):
            lg = np.zeros(s.V, np.float32)
            assert lib.library.rwkv_b200_batch_get_logits(s.bt.ptr, 0, lg.ctypes.data_as(P_F)), (what, "the logits became invalid")
            assert all(a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes() for a, b in zip(s.slots(), before)), what

        def refused(err, what, ptr=None, G=2, mt=(4, 4), pen=(1.0, 1.0), stops=(), n_best=2):
            ptr = ptr or s.bt.ptr
            ok, *_ = beam_groups(lib, ptr, G, list(mt), list(pen), stops, n_best)
            assert not ok, what
            assert lib.library.rwkv_get_last_error(ptr) == err, what
            unchanged(what)

        refused(ERR_CTX_UNSUPPORTED, "ordinary context", s.ctx.ptr)
        refused(ERR_CTX_UNSUPPORTED, "stage", stage.ptr)
        refused(ERR_CTX_UNSUPPORTED, "pipeline", pipe)
        refused(ERR_ARGS, "G 0", G=0)
        refused(ERR_ARGS, "G does not divide", G=4, mt=(4,) * 4, pen=(1.0,) * 4)
        refused(ERR_ARGS, "W 11", big.ptr, G=2)
        refused(ERR_ARGS, "n_best 0", n_best=0)
        refused(ERR_ARGS, "n_best above W", n_best=4)
        refused(ERR_ARGS, "all max_tokens 0", mt=(0, 0))
        refused(ERR_ARGS, "max_tokens above the limit", mt=(4, 4097))
        refused(ERR_ARGS, "NaN length penalty", pen=(1.0, float("nan")))
        refused(ERR_ARGS, "inf length penalty", pen=(float("inf"), 1.0))
        refused(ERR_ARGS, "17 stop ids", stops=tuple(range(17)))
        refused(ERR_ARGS, "stop id n_vocab", stops=(s.V,))
        assert lib.library.rwkv_b200_batch_set_adapter(s.bt.ptr, 4, Y)
        refused(ERR_ARGS, "a group with mixed adapters")
        assert lib.library.rwkv_b200_batch_set_adapter(s.bt.ptr, 4, None)
        n = 4
        arrays = [np.full(2, 4, np.uint32), np.ones(2, np.float32), np.zeros((2, 2, n), np.uint32), np.zeros((2, 2), np.uint32), np.zeros((2, 2))]
        for i in range(5):
            ptrs = [arrays[0].ctypes.data_as(P_U), arrays[1].ctypes.data_as(P_F), arrays[2].ctypes.data_as(P_U), arrays[3].ctypes.data_as(P_U),
                    arrays[4].ctypes.data_as(P_D)]
            ptrs[i] = None
            assert not lib.library.rwkv_b200_beam_search_groups(s.bt.ptr, 2, ptrs[0], ptrs[1], None, 0, 2, *ptrs[2:], None), i
            assert lib.library.rwkv_get_last_error(s.bt.ptr) == ERR_ARGS, i
            unchanged(("NULL array", i))
        # from inside this context's streaming callback
        inside = []
        rec = Recorder(inner=lambda seq, idx, tok: inside.append((beam_groups(lib, s.bt.ptr, 2, [4, 4], [1.0, 1.0], (), 2)[0],
                                                                  lib.library.rwkv_get_last_error(s.bt.ptr))))
        ok, _ = batch_generate_stream(s.bt, [1, 0, 0, 0, 0, 0], [1.0] * 6, [1.0] * 6, [0.0] * 6, [0.0] * 6, np.full((6, 1), 0.5), (), rec)
        assert ok and inside == [(False, ERR_CTX_UNSUPPORTED)], inside
        # no valid logits
        s.prime(60)
        assert lib.library.rwkv_b200_batch_eval(s.bt.ptr, (ctypes.c_uint32 * 6)(1, 2, 3, 4, 5, 6), False)
        states = [s.bt.state(k, s.n_state).tobytes() for k in range(6)]
        ok, *_ = beam_groups(lib, s.bt.ptr, 2, [4, 4], [1.0, 1.0], (), 2)
        assert not ok and lib.library.rwkv_get_last_error(s.bt.ptr) == ERR_ARGS, "invalid logits"
        assert [s.bt.state(k, s.n_state).tobytes() for k in range(6)] == states
        lg = np.zeros(s.V, np.float32)
        assert not lib.library.rwkv_b200_batch_get_logits(s.bt.ptr, 0, lg.ctypes.data_as(P_F)), "the logits became valid"
        # the adapters: a pass of both batches from the same prompts gives the same bits
        s.prime(61)
        ref.prime(s.prompts)
        for k in range(6):
            assert s.bt.state(k, s.n_state).tobytes() == ref.state(k, s.n_state).tobytes(), ("adapters", k)
            assert s.bt.logits(k, s.V).tobytes() == ref.logits(k, s.V).tobytes(), ("adapters", k)
    finally:
        for k in range(6):
            lib.library.rwkv_b200_batch_set_adapter(s.bt.ptr, k, None)
            lib.library.rwkv_b200_batch_set_adapter(ref.ptr, k, None)
        ref.free()
        big.free()
        lib.rwkv_free(stage)
        lib.library.rwkv_free(pipe)
        s.free()
        lib.rwkv_b200_adapter_free(X)
        lib.rwkv_b200_adapter_free(Y)


def test_one_graph_launch_per_call_and_a_recapture_per_group_count(lib):
    path = model_path("6v0-3m", "Q5_1")
    s = Groups(lib, path, 4, 2)
    try:
        s.prime(70)
        L = lib.library
        for call, G in enumerate((4, 4, 2, 2, 4)):
            g0, k0 = L.rwkv_b200_graph_launch_count(), L.rwkv_b200_kernel_launch_count()
            ok, *_ = beam_groups(lib, s.bt.ptr, G, [3] * G, [1.0] * G, (), 1)
            assert ok, call
            assert L.rwkv_b200_graph_launch_count() - g0 == 1, call
            recaptured = L.rwkv_b200_kernel_launch_count() - k0
            assert (recaptured > 0) == (call in (0, 2, 4)), (call, recaptured)
    finally:
        s.free()
