"""LoRA adapters per sequence of a batch context (rwkv_b200_batch_set_adapter, the column groups of csrc/kernels/lora.cu) on the GPU:
- the grouped shrink and expand launches against float64 and against the one-adapter hook, column by column;
- a row of a mixed batch gives the bits of a single context (or, on the tensor-core route, of a batch) with that row's adapter attached
  to the whole context, over batch, ragged and scoring passes and device-side generation, streaming included;
- reassignments take effect on the next pass, one adapter everywhere is the context-wide adapter, NULL everywhere the base;
- distinct adapters cost no extra launch, and every refusal changes nothing."""
import ctypes

import numpy as np
import pytest

import lora_ref as lr
from conftest import VERSIONS, model_path
from test_gpu_generate import Batch, generate, logits, prime, ptr, state
from test_gpu_generate_sampled import Smp, batch_sampled, gen_sampled
from test_gpu_generate_stream import Recorder, batch_generate_stream
from test_gpu_lora import GUARD, HOOK_K, Ctx, batch_run, check_columns, fp, prompt, run_hook, same

pytestmark = pytest.mark.gpu
P_I = ctypes.POINTER(ctypes.c_int)
P_F = ctypes.POINTER(ctypes.c_float)
ERR_ARGS, ERR_CTX_UNSUPPORTED = 1 << 8, (6 << 8) | 9


# ---- 1. the grouped launches -----------------------------------------------------------------------------------------------------

def run_columns(lib, ads, col_adapter, x, z, gate, epi):
    """ads: [(a, b, scale)]; returns y [M, T], u [T, max rank] (NaN where not written) and both guards."""
    K, T = x.shape
    M = z.shape[0]
    R = max(a.shape[0] for a, _, _ in ads)
    u = np.zeros(T * R + GUARD, np.float32)
    y = np.zeros(T * M + GUARD, np.float32)
    keep = [np.ascontiguousarray(a) for a, _, _ in ads] + [np.ascontiguousarray(b) for _, b, _ in ads]
    A = (P_F * len(ads))(*[fp(k) for k in keep[:len(ads)]])
    B = (P_F * len(ads))(*[fp(k) for k in keep[len(ads):]])
    ranks = np.array([a.shape[0] for a, _, _ in ads], np.int32)
    scales = np.array([s for _, _, s in ads], np.float32)
    cols = np.array(col_adapter, np.int32)
    xc, zc = np.ascontiguousarray(x.T, np.float32), np.ascontiguousarray(z.T, np.float32)
    gc = np.ascontiguousarray(gate.T, np.float32) if gate is not None else None
    ok = lib.library.rwkv_b200_test_lora_columns(K, M, T, len(ads), ranks.ctypes.data_as(P_I), fp(scales), A, B, cols.ctypes.data_as(P_I), epi,
                                                 fp(xc), fp(zc), fp(gc) if gc is not None else None, fp(u), fp(y))
    assert ok, "rwkv_b200_test_lora_columns failed"
    return y[:T * M].reshape(T, M).T, u[:T * R].reshape(T, R), u[T * R:], y[T * M:]


EPIS = (lr.EPI_NONE, lr.EPI_SIGMOID, lr.EPI_SILU, lr.EPI_RELU_SQR, lr.EPI_ADD, lr.EPI_MUL_ADD)


def layouts(T, rng):
    """Mixed col_adapter layouts over 3 adapters: cyclic with gaps, runs, all one adapter, and a random one."""
    out = [[(t % 4) - 1 for t in range(T)], [min(t * 4 // T, 3) - 1 for t in range(T)], [1] * T, list(rng.integers(-1, 3, T))]
    return [list(map(int, l)) for l in out]


@pytest.mark.parametrize("T", [1, 5, 8, 9, 31, 256])
@pytest.mark.parametrize("epi", EPIS)
@pytest.mark.parametrize("K,M", [(64, 96), (4096, 1024)])
def test_grouped_columns_match_float64_and_the_one_adapter_hook(lib, T, epi, K, M):
    if K == 4096 and T not in (9, 256):
        pytest.skip("the large shape at two widths")
    rng = np.random.default_rng(K + 3 * M + 11 * T + epi)
    ads = []
    for rank in (1, 8, 64):
        a = (rng.standard_normal((rank, K)) * K ** -0.5).astype(np.float32)
        b = (rng.standard_normal((M, rank)) * 0.2).astype(np.float32)
        ads.append((a, b, float(0.5 + rank / 64)))
    x = rng.standard_normal((K, T)).astype(np.float32)
    z = rng.standard_normal((M, T)).astype(np.float32)
    linear = epi in (lr.EPI_NONE, lr.EPI_ADD, lr.EPI_MUL_ADD)
    if linear:
        z[::7, :] = -0.0
    gate = rng.random((M, T)).astype(np.float32) if epi == lr.EPI_MUL_ADD else None
    for layout in layouts(T, rng):
        y, u, gu, gy = run_columns(lib, ads, layout, x, z, gate, epi)
        assert np.isnan(gu).all() and np.isnan(gy).all(), "a guard was written"
        for t in sorted(set(range(0, T, max(1, T // 24))) | {T - 1}):
            k = layout[t]
            g1 = gate[:, t:t + 1] if gate is not None else None
            if k < 0:
                assert np.isnan(u[t]).all(), ("u of an unadapted column was written", t)
                if linear:
                    assert y[:, t].tobytes() == z[:, t].tobytes(), ("unadapted column", t)
                else:
                    a, _, s = ads[0]
                    _, y0, _, _ = run_hook(lib, a, np.zeros((M, a.shape[0]), np.float32), x[:, t:t + 1], z[:, t:t + 1], g1, s, epi)
                    assert y[:, t].tobytes() == y0[:, 0].tobytes(), ("unadapted column against the zero-B hook", t)
                continue
            a, b, s = ads[k]
            R = a.shape[0]
            assert np.isnan(u[t, R:]).all()
            u1, y1, _, _ = run_hook(lib, a, b, x[:, t:t + 1], z[:, t:t + 1], g1, s, epi)
            assert u[t, :R].tobytes() == u1[:, 0].tobytes() and y[:, t].tobytes() == y1[:, 0].tobytes(), ("column", t, "adapter", k)
            args = (a, b, x[:, t:t + 1], z[:, t:t + 1], g1, s, epi)
            u64, y64 = lr.lora_ref(*args, np.float64)
            u32, y32 = lr.lora_ref(*args, np.float32)
            mu, my = lr.lora_magnitude(*args)
            check_columns(u[t, :R, None], u64, u32, mu, HOOK_K, "u")
            check_columns(y[:, t:t + 1], y64, y32, my, HOOK_K, "y")


# ---- helpers on whole models -----------------------------------------------------------------------------------------------------

def adapters(lib, c, path, seed=0):
    """Three adapters of non-zero B that differ in rank and in the matrices they adapt: X (rank 8, every delta target), Y (rank 1,
    time mixing only), Z (rank 64, channel mixing and att.output)."""
    def pick(rank, s, keep):
        return [e for e in lr.make_entries(path, rank, s, b_scale=0.2) if keep(e[0])]
    X = c.adapter(pick(8, seed + 1, lambda n: True), 1.5)
    Y = c.adapter(pick(1, seed + 2, lambda n: ".att." in n and "output" not in n), 2.0)
    Z = c.adapter(pick(64, seed + 3, lambda n: ".ffn." in n or "att.output" in n), 0.5)
    return X, Y, Z


def free_adapters(lib, *ads):
    for a in ads:
        lib.rwkv_b200_adapter_free(a)


class MixedBatch(Batch):
    def __init__(self, lib, c, assign):
        super().__init__(lib, c.c, len(assign))
        self.n_state, self.n_vocab = c.n_state, c.n_logits
        self.assign(assign)

    def assign(self, assign):
        for s, a in enumerate(assign):
            assert self.lib.library.rwkv_b200_batch_set_adapter(self.ptr, s, a), s

    def rows(self):
        return [(self.logits(b, self.n_vocab), self.state(b, self.n_state)) for b in range(self.n)]


def single_serial(c, ad, toks, state0=None):
    c.attach(ad)
    out = c.serial(toks, state0)
    c.attach(None)
    return out


# ---- 2. / 3. mixed batches -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("ver", VERSIONS)
@pytest.mark.parametrize("fmt", ["FP32", "Q5_1"])
def test_mixed_batch_rows_equal_single_contexts(lib, ver, fmt):
    path = model_path(ver, fmt)
    c = Ctx(lib, path)
    X, Y, Z = adapters(lib, c, path)
    assign = [X, Y, None, X, Z, None]
    bt = MixedBatch(lib, c, assign)
    try:
        prompts = [prompt(5, c.n_logits, s) for s in range(len(assign))]
        for step in range(5):      # the single-token graph is captured on the second step
            assert bt.eval([p[step] for p in prompts])
        got = bt.rows()
        for b, ad in enumerate(assign):
            assert same(got[b], single_serial(c, ad, prompts[b])), (ver, fmt, b)
        assert not same(got[0], single_serial(c, None, prompts[0])) and not same(got[1], single_serial(c, None, prompts[1]))
    finally:
        bt.free()
        free_adapters(lib, X, Y, Z)
        c.free()


def kquant_file(lib, tmp_path):
    import kquant_ref as kr
    G = kr.golden()
    master, path = str(tmp_path / "master.bin"), str(tmp_path / "Q4_K.bin")
    kr.write_master(master, G["presets"]["rwkv6-small"], G["seed"])
    lib.rwkv_quantize_model_file(master, path, "Q4_K")
    return path


def test_mixed_batch_on_k_quants(lib, tmp_path):
    path = kquant_file(lib, tmp_path)
    c = Ctx(lib, path)
    X, Y, Z = adapters(lib, c, path, 5)
    assign = [Z, None, X, Y]
    bt = MixedBatch(lib, c, assign)
    try:
        prompts = [prompt(4, c.n_logits, s) for s in range(len(assign))]
        for step in range(4):
            assert bt.eval([p[step] for p in prompts])
        for b, (got, ad) in enumerate(zip(bt.rows(), assign)):
            assert same(got, single_serial(c, ad, prompts[b])), b
    finally:
        bt.free()
        free_adapters(lib, X, Y, Z)
        c.free()


@pytest.mark.parametrize("ver,fmt", [(v, "Q5_1") for v in VERSIONS] + [("6v0-3m", "FP32")])
def test_mixed_batch_on_tensor_cores_equals_context_wide_batches(lib, ver, fmt):
    """20 sequences take the tensor-core route: row b equals row b of a 20-sequence batch with adapter(b) attached to the whole batch."""
    path = model_path(ver, fmt)
    c = Ctx(lib, path)
    X, Y, Z = adapters(lib, c, path, 9)
    assign = [(X, Y, None, Z)[b % 4] for b in range(20)]
    assign[7] = X
    bt = MixedBatch(lib, c, assign)
    try:
        prompts = [prompt(4, c.n_logits, s) for s in range(20)]
        for step in range(4):
            assert bt.eval([p[step] for p in prompts])
        got = bt.rows()
        for ad in (X, Y, Z, None):
            want = batch_run(lib, c, ad, prompts, 4)
            for b in range(20):
                if assign[b] == ad:
                    assert same(got[b], want[b]), (ver, fmt, b)
    finally:
        bt.free()
        free_adapters(lib, X, Y, Z)
        c.free()


# ---- 4. ragged and scoring passes ------------------------------------------------------------------------------------------------

def ragged(bt, toks_per_seq, want_logits=True):
    counts = np.array([len(t) for t in toks_per_seq], np.uint32)
    flat = np.array([t for ts in toks_per_seq for t in ts], np.uint32)
    assert bt.lib.library.rwkv_b200_batch_eval_ragged(bt.ptr, ptr(flat, ctypes.POINTER(ctypes.c_uint32)), ptr(counts, ctypes.POINTER(ctypes.c_uint32)), want_logits)


@pytest.mark.parametrize("ver", VERSIONS)
def test_ragged_and_scoring_under_mixed_adapters(lib, ver):
    path = model_path(ver, "Q5_1")
    c = Ctx(lib, path)
    X, Y, Z = adapters(lib, c, path, 13)
    assign = [X, None, Y, Z, X, None]
    bt = MixedBatch(lib, c, assign)
    V = c.n_logits
    try:
        for passes, tc in (([[3, 1, 0, 4, 2, 1], [0, 2, 1, 1, 0, 3]], True), ([[8, 7, 0, 9, 5, 6], [1, 0, 12, 3, 9, 7]], False)):
            lib.library.rwkv_b200_set_tensor_cores(bt.ptr, tc)
            for b in range(bt.n):
                assert lib.library.rwkv_b200_batch_set_state(bt.ptr, b, None)
            fed = [[] for _ in range(bt.n)]
            for i, counts in enumerate(passes):
                chunk = [prompt(n, V, 3 * b + i) for b, n in enumerate(counts)]
                ragged(bt, chunk)
                for b in range(bt.n):
                    fed[b] += chunk[b]
            for b, ad in enumerate(assign):
                want = single_serial(c, ad, fed[b])
                assert bt.state(b, c.n_state).tobytes() == want[1].tobytes(), (ver, tc, b)
                assert bt.logits(b, V).tobytes() == want[0].tobytes(), (ver, tc, b)
        lib.library.rwkv_b200_set_tensor_cores(bt.ptr, True)
        # scoring: 2 + 0 + 3 + 4 + 1 + 2 columns, the head on the GEMV
        counts = [2, 0, 3, 4, 1, 2]
        toks = [prompt(n, V, 20 + b) for b, n in enumerate(counts)]
        targets = [prompt(n, V, 40 + b) for b, n in enumerate(counts)]
        for b in range(bt.n):
            assert lib.library.rwkv_b200_batch_set_state(bt.ptr, b, None)
        P_U = ctypes.POINTER(ctypes.c_uint32)
        flat_t, flat_g = np.array(sum(toks, []), np.uint32), np.array(sum(targets, []), np.uint32)
        lp = np.zeros(len(flat_t), np.float32)
        assert lib.library.rwkv_b200_batch_score_ragged(bt.ptr, ptr(flat_t, P_U), ptr(np.array(counts, np.uint32), P_U), ptr(flat_g, P_U), fp(lp), None)
        at = 0
        for b, ad in enumerate(assign):
            if not counts[b]:
                continue
            c.attach(ad)
            assert lib.library.rwkv_b200_state_load(c.c.ptr, None)
            one = np.zeros(counts[b], np.float32)
            assert lib.library.rwkv_b200_score(c.c.ptr, ptr(np.array(toks[b], np.uint32), P_U), ptr(np.array(targets[b], np.uint32), P_U), counts[b],
                                               fp(one), None)
            c.attach(None)
            assert lp[at:at + counts[b]].tobytes() == one.tobytes(), (ver, b)
            at += counts[b]
    finally:
        bt.free()
        free_adapters(lib, X, Y, Z)
        c.free()


# ---- 5. generation ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("ver", VERSIONS)
def test_generate_sampled_rows_equal_single_contexts(lib, ver):
    path = model_path(ver, "Q5_1")
    c = Ctx(lib, path)
    X, Y, Z = adapters(lib, c, path, 17)
    assign = [Y, X, None, Z, X]
    bt = MixedBatch(lib, c, assign)
    V = c.n_logits
    single = lib.rwkv_clone_context(c.c, 1)
    try:
        smps = [Smp(0.9, 0.95, 40, 0.02, 0.2, 0.1), Smp(1.0, 1.0, 0, 0.0, 0.5, 0.5), Smp(0.7, 0.8, 5, 0.0, 0.0, 0.3), Smp(1.2, 1.0, 0, 0.05, 0.1, 0.0),
                Smp(1.0, 0.9, 2, 0.0, 0.0, 0.0)]
        prompts = [prompt(4, V, 50 + b) for b in range(bt.n)]
        us = np.random.RandomState(3).random_sample((bt.n, 12))
        bt.prime(prompts)
        free = []
        for b, ad in enumerate(assign):          # each row alone, with its adapter, without stops
            lib.rwkv_b200_set_adapter(single, ad)
            prime(lib, single.ptr, prompts[b])
            ok, toks, _ = gen_sampled(lib, single.ptr, smps[b], 12, us[b])
            assert ok
            free.append(toks)
        stops = (free[0][4], free[3][2])
        ok, got, _ = batch_sampled(bt, smps, [12] * bt.n, us, stops)
        assert ok and any(len(g) < 12 for g in got)
        rows = bt.rows()
        # the penalty counts: a continuation that keeps them draws the same tokens
        ok, more, _ = batch_sampled(bt, smps, [4] * bt.n, us[:, :4], keep=[1] * bt.n)
        assert ok
        for b, ad in enumerate(assign):
            lib.rwkv_b200_set_adapter(single, ad)
            prime(lib, single.ptr, prompts[b])
            ok, want, _ = gen_sampled(lib, single.ptr, smps[b], 12, us[b], stops)
            assert ok and got[b] == want, (ver, b)
            assert rows[b][1].tobytes() == state(lib, single.ptr, c.n_state).tobytes(), (ver, b)
            assert rows[b][0].tobytes() == logits(lib, single.ptr, V).tobytes(), (ver, b)
            ok, want, _ = gen_sampled(lib, single.ptr, smps[b], 4, us[b][:4], keep=True)
            assert ok and more[b] == want, (ver, b)
        lib.rwkv_b200_set_adapter(single, None)
        # streaming: the callback ends sequence 1 after its third token; the blocking call with max_tokens 3 for it is the same
        bt.prime(prompts)
        rec = Recorder(stop_at={1: 2})
        temps, tps, pres, freq = [1.0] * bt.n, [0.9] * bt.n, [0.2] * bt.n, [0.1] * bt.n
        ok, streamed = batch_generate_stream(bt, [8] * bt.n, temps, tps, pres, freq, us[:, :8], (), rec)
        assert ok and len(streamed[1]) == 3
        st_stream = bt.rows()
        bt.prime(prompts)
        ok, blocking = bt.generate([8, 3, 8, 8, 8], temps, tps, pres, freq, us[:, :8], ())
        assert ok and blocking == streamed
        for a, b in zip(st_stream, bt.rows()):
            assert same(a, b)
    finally:
        lib.rwkv_free(single)
        bt.free()
        free_adapters(lib, X, Y, Z)
        c.free()


# ---- 6. reassignment -------------------------------------------------------------------------------------------------------------

def test_reassignment_takes_effect_on_the_next_pass(lib):
    path = model_path("6v0-3m", "Q5_1")
    c = Ctx(lib, path)
    X, Y, Z = adapters(lib, c, path, 21)
    assign = [X, None, Y, Z]
    bt = MixedBatch(lib, c, assign)
    V = c.n_logits
    single = lib.rwkv_clone_context(c.c, 1)
    try:
        prompts = [prompt(7, V, b) for b in range(bt.n)]
        for step in range(4):           # the single-token graph is in use from the second step
            assert bt.eval([p[step] for p in prompts])
        assert lib.library.rwkv_b200_batch_set_adapter(bt.ptr, 1, Y)
        assert lib.library.rwkv_b200_batch_set_adapter(bt.ptr, 3, None)
        for step in range(4, 7):
            assert bt.eval([p[step] for p in prompts])
        after = [X, Y, Y, None]
        rows = bt.rows()
        for b in range(bt.n):
            _, st = single_serial(c, assign[b], prompts[b][:4])
            want = single_serial(c, after[b], prompts[b][4:], st)
            assert same(rows[b], want), b
        # between two generate calls
        us = np.random.RandomState(5).random_sample((bt.n, 6))
        args = ([1.0] * bt.n, [0.9] * bt.n, [0.3] * bt.n, [0.2] * bt.n)
        bt.prime([p[:3] for p in prompts])
        ok, first = bt.generate([3] * bt.n, *args, us[:, :3], ())
        assert ok
        assert lib.library.rwkv_b200_batch_set_adapter(bt.ptr, 0, Z)
        ok, second = bt.generate([3] * bt.n, *args, us[:, 3:], (), keep=[1] * bt.n)
        assert ok
        final = [Z, Y, Y, None]
        for b in range(bt.n):
            lib.rwkv_b200_set_adapter(single, after[b])
            prime(lib, single.ptr, prompts[b][:3])
            ok, w1 = generate(lib, single.ptr, 3, 1.0, 0.9, 0.3, 0.2, us[b, :3])
            lib.rwkv_b200_set_adapter(single, final[b])
            ok2, w2 = generate(lib, single.ptr, 3, 1.0, 0.9, 0.3, 0.2, us[b, 3:], keep=True)
            assert ok and ok2 and first[b] == w1 and second[b] == w2, b
            assert bt.state(b, c.n_state).tobytes() == state(lib, single.ptr, c.n_state).tobytes(), b
            assert bt.logits(b, V).tobytes() == logits(lib, single.ptr, V).tobytes(), b
        lib.rwkv_b200_set_adapter(single, None)
    finally:
        lib.rwkv_free(single)
        bt.free()
        free_adapters(lib, X, Y, Z)
        c.free()


# ---- 7. equivalences -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n_seq", [6, 20])
def test_one_adapter_everywhere_is_the_context_wide_adapter(lib, n_seq):
    path = model_path("7v0-834K", "Q5_1")
    c = Ctx(lib, path)
    X, Y, Z = adapters(lib, c, path, 25)
    try:
        prompts = [prompt(4, c.n_logits, s) for s in range(n_seq)]
        want_x, want_base = batch_run(lib, c, X, prompts, 4), batch_run(lib, c, None, prompts, 4)
        bt = MixedBatch(lib, c, [X] * n_seq)
        try:
            for step in range(4):
                assert bt.eval([p[step] for p in prompts])
            for got, want in zip(bt.rows(), want_x):
                assert same(got, want)
            bt.assign([Y] * n_seq)
            bt.assign([None] * n_seq)
            for b in range(n_seq):
                assert lib.library.rwkv_b200_batch_set_state(bt.ptr, b, None)
            for step in range(4):
                assert bt.eval([p[step] for p in prompts])
            for got, want in zip(bt.rows(), want_base):
                assert same(got, want)
        finally:
            bt.free()
    finally:
        free_adapters(lib, X, Y, Z)
        c.free()


# ---- 8. launches -----------------------------------------------------------------------------------------------------------------

def test_distinct_adapters_cost_no_extra_launch(lib):
    path = model_path("6v0-3m", "Q5_1")
    c = Ctx(lib, path)
    ads = [c.adapter(lr.make_entries(path, r, 60 + r, b_scale=0.2), 1.0) for r in (1, 4, 8, 16)]
    L = lib.library
    bt = Batch(lib, c.c, 8)
    try:
        L.rwkv_b200_set_graphs(bt.ptr, False)
        toks = prompt(8, c.n_logits, 2)

        def step():
            before = L.rwkv_b200_kernel_launch_count()
            assert bt.eval(toks)
            return L.rwkv_b200_kernel_launch_count() - before
        base = step()
        assert L.rwkv_b200_set_adapter(bt.ptr, ads[0])
        wide = step()
        assert L.rwkv_b200_set_adapter(bt.ptr, None)
        for s in range(8):
            assert L.rwkv_b200_batch_set_adapter(bt.ptr, s, ads[s % 4])
        mixed = step()
        for s in range(8):
            assert L.rwkv_b200_batch_set_adapter(bt.ptr, s, None)
        none = step()
        assert wide > base and mixed == wide and none == base, (base, wide, mixed, none)
    finally:
        bt.free()
        free_adapters(lib, *ads)
        c.free()


# ---- 9. refusals -----------------------------------------------------------------------------------------------------------------

def test_refusals_change_nothing(lib):
    path = model_path("5v2-730K", "Q5_1")
    c = Ctx(lib, path)
    other = Ctx(lib, model_path("4v0-660K", "Q5_1"))
    X, Y, Z = adapters(lib, c, path, 33)
    R = c.adapter(lr.make_entries(path, 4, 34, vectors=True), 1.0)
    W = other.adapter(lr.make_entries(model_path("4v0-660K", "Q5_1"), 4, 35), 1.0)
    L = lib.library
    bt = MixedBatch(lib, c, [X, None, Y])
    V = c.n_logits
    try:
        prompts = [prompt(3, V, s) for s in range(3)]
        for step in range(3):
            assert bt.eval([p[step] for p in prompts])
        before = bt.rows()

        def refused(call, err, what, ctx=bt.ptr):
            assert not call(), what
            assert L.rwkv_get_last_error(ctx) == err, what
            for a, b in zip(before, bt.rows()):
                assert same(a, b), what

        refused(lambda: L.rwkv_b200_batch_set_adapter(bt.ptr, 1, R), ERR_ARGS, "replacements")
        refused(lambda: L.rwkv_b200_batch_set_adapter(bt.ptr, 1, W), ERR_ARGS, "another model")
        refused(lambda: L.rwkv_b200_batch_set_adapter(bt.ptr, 3, X), ERR_ARGS, "sequence out of range")
        refused(lambda: L.rwkv_b200_batch_set_adapter(bt.ptr, 3, None), ERR_ARGS, "sequence out of range, NULL")
        refused(lambda: L.rwkv_b200_batch_set_adapter(c.c.ptr, 0, X), ERR_CTX_UNSUPPORTED, "an ordinary context", c.c.ptr)
        refused(lambda: L.rwkv_b200_set_adapter(bt.ptr, X), ERR_ARGS, "context-wide while sequences carry adapters")
        refused(lambda: L.rwkv_b200_adapter_free(Y), ERR_ARGS, "free while a sequence holds it", None)
        # a call from the batch's own streaming callback
        seen = []
        rec = Recorder(inner=lambda s, i, t: seen.append(L.rwkv_b200_batch_set_adapter(bt.ptr, 0, None)) if not seen else None)
        ok, _ = batch_generate_stream(bt, [1, 1, 1], [1.0] * 3, [1.0] * 3, [0.0] * 3, [0.0] * 3, np.full((3, 1), 0.5), (), rec)
        assert ok and seen == [False]
        # the other direction of the exclusion
        bt.assign([None, None, None])
        assert L.rwkv_b200_set_adapter(bt.ptr, Z)
        keep = bt.rows()
        assert not L.rwkv_b200_batch_set_adapter(bt.ptr, 0, X) and L.rwkv_get_last_error(bt.ptr) == ERR_ARGS
        assert L.rwkv_b200_batch_set_adapter(bt.ptr, 0, None)        # detaching is always accepted
        for a, b in zip(keep, bt.rows()):
            assert same(a, b)
        assert L.rwkv_b200_set_adapter(bt.ptr, None)
        # lifetimes: batch freed before its adapters, and an adapter freed after the batch released it
        bt.assign([X, Y, X])
        bt.free()
        bt = None
        assert lib.library.rwkv_b200_adapter_free(X)
        X = None
        bt2 = MixedBatch(lib, c, [Y, Z, None])
        bt2.assign([None, None, None])
        assert lib.library.rwkv_b200_adapter_free(Z)
        Z = None
        assert lib.library.rwkv_b200_batch_set_adapter(bt2.ptr, 2, Y)
        bt2.free()
    finally:
        if bt is not None:
            bt.free()
        free_adapters(lib, *[a for a in (X, Y, Z, R) if a is not None])
        lib.rwkv_b200_adapter_free(W)
        other.free()
        c.free()


def test_a_32nd_distinct_adapter_is_refused(lib):
    path = model_path("4v0-660K", "Q5_1")
    c = Ctx(lib, path)
    ads = [c.adapter([e for e in lr.make_entries(path, 1, 70 + i) if "att.key" in e[0]], 1.0) for i in range(32)]
    bt = Batch(lib, c.c, 32)
    try:
        for s in range(31):
            assert lib.library.rwkv_b200_batch_set_adapter(bt.ptr, s, ads[s])
        assert not lib.library.rwkv_b200_batch_set_adapter(bt.ptr, 31, ads[31])
        assert lib.library.rwkv_get_last_error(bt.ptr) == ERR_ARGS
        assert lib.library.rwkv_b200_batch_set_adapter(bt.ptr, 31, ads[0])      # a 31st sequence on an adapter in use
        toks = prompt(32, c.n_logits, 4)
        assert bt.eval(toks)
        # the pass with 31 distinct adapters on all 32 sequences (tensor cores; att.key in 31 groups, none without a delta): row s equals
        # row s of the batch with its adapter attached to the whole context
        got = [(bt.logits(s, c.n_logits), bt.state(s, c.n_state)) for s in range(32)]
        for k in range(31):
            want = batch_run(lib, c, ads[k], [[t] for t in toks], 1)
            for s in (k, 31) if k == 0 else (k,):
                assert same(got[s], want[s]), (k, s)
        assert not same(got[1], batch_run(lib, c, None, [[t] for t in toks], 1)[1])
    finally:
        bt.free()
        free_adapters(lib, *ads)
        c.free()
