"""LoRA adapters (rwkv_b200_adapter_create / rwkv_b200_set_adapter, csrc/kernels/lora.cu) on the GPU:
- the shrink and expand launches against a float64 restatement, through the test hook;
- an adapter whose every B is zero gives exactly the unadapted bits, on every route; detaching gives them back;
- an adapted FP32 model matches a model file merged in float64; an adapted Q5_1 / Q4_K model matches the oracle on the same file with
  the delta added in float64;
- the invariants of the unadapted context hold bit for bit on an adapted one;
- refusals change nothing, and lora.py loads RWKV-PEFT-style checkpoints of every architecture."""
import ctypes
import threading

import numpy as np
import pytest

from conftest import LONG_PROMPT, VERSIONS, model_path
import lora_ref as lr
from lora_ref import read_model_file

pytestmark = pytest.mark.gpu
P_F, P_U = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_uint32)
GUARD = 64


def fp(a):
    return a.ctypes.data_as(P_F)


# ---- 1. the kernels against float64 ---------------------------------------------------------------------------------------------

def run_hook(lib, a, b, x, z, gate, scale, epi):
    """x [K, T], z / gate [M, T] column-major as numpy (dim, T) arrays; returns u [rank, T], y [M, T] and both guards."""
    rank, K = a.shape
    M, T = z.shape
    u = np.zeros(T * rank + GUARD, np.float32)
    y = np.zeros(T * M + GUARD, np.float32)
    xc, zc = np.ascontiguousarray(x.T, np.float32), np.ascontiguousarray(z.T, np.float32)
    gc = np.ascontiguousarray(gate.T, np.float32) if gate is not None else None
    ok = lib.library.rwkv_b200_test_lora(K, M, T, rank, ctypes.c_float(scale), epi, fp(np.ascontiguousarray(a)), fp(np.ascontiguousarray(b)),
                                         fp(xc), fp(zc), fp(gc) if gc is not None else None, fp(u), fp(y))
    assert ok, "rwkv_b200_test_lora failed"
    return u[:T * rank].reshape(T, rank).T, y[:T * M].reshape(T, M).T, u[T * rank:], y[T * M:]


def check_columns(got, ref64, ref32, mag, k, what):
    """Every column within k times the float32 restatement's distance from float64, or within k fp32 spacings of the magnitudes its
    arithmetic rounds (lora_ref.lora_magnitude), whichever is larger: a column of one or two entries can land on float64 by chance in
    the float32 restatement's order and not in the kernel's."""
    for t in range(got.shape[1]):
        bar = k * max(np.abs(ref32[:, t] - ref64[:, t]).max(), np.finfo(np.float32).eps * mag[:, t].max())
        err = np.abs(got[:, t].astype(np.float64) - ref64[:, t]).max()
        assert err <= bar, f"{what}: column {t}: |gpu - f64| = {err:.3e} above {bar:.3e}"


HOOK_K = 8
CASES = (
    [(64, 96, T, r, e) for T in (1, 2, 5, 31, 32, 256) for r, e in ((1, lr.EPI_NONE), (8, lr.EPI_SIGMOID), (16, lr.EPI_SILU), (64, lr.EPI_RELU_SQR),
                                                                       (256, lr.EPI_ADD), (8, lr.EPI_MUL_ADD))]
    + [(K, M, T, r, e) for (K, M) in ((4096, 4096), (4096, 14336), (14336, 4096)) for T, r, e in
       ((1, 16, lr.EPI_NONE), (2, 64, lr.EPI_RELU_SQR), (5, 8, lr.EPI_MUL_ADD), (31, 256, lr.EPI_SIGMOID), (32, 1, lr.EPI_ADD),
        (256, 16, lr.EPI_SILU))]
    + [(33, 7, T, r, e) for T in (1, 31) for r in (1, 8, 256) for e in (lr.EPI_NONE, lr.EPI_MUL_ADD)]
)


@pytest.mark.parametrize("K,M,T,rank,epi", CASES)
def test_shrink_expand_match_float64(lib, K, M, T, rank, epi):
    rng = np.random.default_rng(K * 7 + M * 3 + T * 11 + rank + epi)
    a = (rng.standard_normal((rank, K)) * K ** -0.5).astype(np.float32)
    b = (rng.standard_normal((M, rank)) * 0.2).astype(np.float32)
    x = rng.standard_normal((K, T)).astype(np.float32)
    z = rng.standard_normal((M, T)).astype(np.float32)
    gate = rng.random((M, T)).astype(np.float32) if epi == lr.EPI_MUL_ADD else None
    scale = 0.75
    u, y, gu, gy = run_hook(lib, a, b, x, z, gate, scale, epi)
    u64, y64 = lr.lora_ref(a, b, x, z, gate, scale, epi, np.float64)
    u32, y32 = lr.lora_ref(a, b, x, z, gate, scale, epi, np.float32)
    mu, my = lr.lora_magnitude(a, b, x, z, gate, scale, epi)
    assert np.isnan(gu).all() and np.isnan(gy).all(), "a guard was written"
    check_columns(u, u64, u32, mu, HOOK_K, "u")
    check_columns(y, y64, y32, my, HOOK_K, "y")


def test_hook_columns_do_not_depend_on_T(lib):
    """A column's bits are a function of (K, M, rank): the first column of a 256-column launch is the 1-column launch's."""
    rng = np.random.default_rng(5)
    K, M, rank = 4096, 1024, 16
    a = (rng.standard_normal((rank, K)) * K ** -0.5).astype(np.float32)
    b = (rng.standard_normal((M, rank)) * 0.2).astype(np.float32)
    x = rng.standard_normal((K, 256)).astype(np.float32)
    z = rng.standard_normal((M, 256)).astype(np.float32)
    _, y256, _, _ = run_hook(lib, a, b, x, z, None, 0.5, lr.EPI_SILU)
    for t in (0, 7, 8, 255):
        _, y1, _, _ = run_hook(lib, a, b, x[:, t:t + 1], z[:, t:t + 1], None, 0.5, lr.EPI_SILU)
        assert y1[:, 0].tobytes() == y256[:, t].tobytes(), t


# ---- helpers on whole models ----------------------------------------------------------------------------------------------------

class Ctx:
    def __init__(self, lib, path):
        self.lib, self.c = lib, lib.rwkv_init_from_file(path, 1, 0)
        self.n_state = lib.rwkv_get_state_buffer_element_count(self.c)
        self.n_logits = lib.rwkv_get_logits_buffer_element_count(self.c)

    def free(self):
        self.lib.rwkv_free(self.c)

    def serial(self, toks, state0=None):
        st = np.zeros(self.n_state, np.float32) if state0 is None else state0.copy()
        lg = np.zeros(self.n_logits, np.float32)
        for i, t in enumerate(toks):
            sin = None if (i == 0 and state0 is None) else fp(st)
            assert self.lib.library.rwkv_eval(self.c.ptr, t, sin, fp(st), fp(lg))
        return lg, st

    def sequence(self, toks):
        st = np.zeros(self.n_state, np.float32)
        lg = np.zeros(self.n_logits, np.float32)
        arr = (ctypes.c_uint32 * len(toks))(*toks)
        assert self.lib.library.rwkv_eval_sequence(self.c.ptr, arr, len(toks), None, fp(st), fp(lg))
        return lg, st

    def chunks(self, toks, chunk):
        st = np.zeros(self.n_state, np.float32)
        lg = np.zeros(self.n_logits, np.float32)
        arr = (ctypes.c_uint32 * len(toks))(*toks)
        assert self.lib.library.rwkv_eval_sequence_in_chunks(self.c.ptr, arr, len(toks), chunk, None, fp(st), fp(lg))
        return lg, st

    def adapter(self, entries, scale):
        return self.lib.rwkv_b200_adapter_create(self.c, entries, scale)

    def attach(self, adapter):
        self.lib.rwkv_b200_set_adapter(self.c, adapter)


def prompt(n, V, seed=0):
    return [(LONG_PROMPT[(i + seed) % len(LONG_PROMPT)] * (seed + 1) + i) % V for i in range(n)]


def same(a, b):
    return a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def batch_run(lib, ctx, adapter, prompts, n_steps):
    """Batch context of len(prompts) sequences from ctx with `adapter` attached: logits of the last step and the states."""
    n_seq = len(prompts)
    batch = ctypes.c_void_p(lib.library.rwkv_b200_batch_create(ctx.c.ptr, n_seq))
    assert batch.value
    try:
        if adapter is not None:
            assert lib.library.rwkv_b200_set_adapter(batch, adapter)
        for step in range(n_steps):
            assert lib.library.rwkv_b200_batch_eval(batch, (ctypes.c_uint32 * n_seq)(*[p[step] for p in prompts]), True)
        out = []
        for s in range(n_seq):
            lg, st = np.zeros(ctx.n_logits, np.float32), np.zeros(ctx.n_state, np.float32)
            assert lib.library.rwkv_b200_batch_get_logits(batch, s, fp(lg)) and lib.library.rwkv_b200_batch_get_state(batch, s, fp(st))
            out.append((lg, st))
        assert lib.library.rwkv_b200_set_adapter(batch, None)
        return out
    finally:
        lib.library.rwkv_free(batch)


# ---- 2. zero B is a no-op --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("ver", VERSIONS)
@pytest.mark.parametrize("fmt", ["FP32", "Q5_1"])
def test_zero_b_is_a_no_op(lib, ver, fmt):
    c = Ctx(lib, model_path(ver, fmt))
    try:
        toks = prompt(70, c.n_logits)
        base_serial = c.serial(toks[:6])                      # graphs are captured on the second use of a slot
        base_seq = c.sequence(toks)
        lib.library.rwkv_b200_set_tensor_cores(c.c.ptr, False)
        base_seq_simt = c.sequence(toks)
        lib.library.rwkv_b200_set_tensor_cores(c.c.ptr, True)
        prompts = [prompt(5, c.n_logits, s) for s in range(4)]
        base_batch = batch_run(lib, c, None, prompts, 5)
        ad = c.adapter(lr.make_entries(model_path(ver, fmt), 8, 1, zero_b=True), 2.0)
        c.attach(ad)
        assert same(c.serial(toks[:6]), base_serial)
        assert same(c.sequence(toks), base_seq)
        lib.library.rwkv_b200_set_tensor_cores(c.c.ptr, False)
        assert same(c.sequence(toks), base_seq_simt)
        lib.library.rwkv_b200_set_tensor_cores(c.c.ptr, True)
        for got, want in zip(batch_run(lib, c, ad, prompts, 5), base_batch):
            assert same(got, want)
        c.attach(None)
        lib.rwkv_b200_adapter_free(ad)
        assert same(c.serial(toks[:6]), base_serial) and same(c.sequence(toks), base_seq)
    finally:
        c.free()


def test_detach_gives_back_the_unadapted_bits(lib):
    path = model_path("6v0-3m", "Q5_1")
    c = Ctx(lib, path)
    try:
        toks = prompt(40, c.n_logits)
        base = (c.serial(toks[:4]), c.sequence(toks))
        ad = c.adapter(lr.make_entries(path, 16, 3, vectors=True), 1.0)
        c.attach(ad)
        adapted = c.sequence(toks)
        assert not same(adapted, base[1])
        c.attach(None)
        assert same(c.serial(toks[:4]), base[0]) and same(c.sequence(toks), base[1])
        lib.rwkv_b200_adapter_free(ad)
    finally:
        c.free()


# ---- 3. merged equivalence -------------------------------------------------------------------------------------------------------

def within(got, want, base, frac, floor, what):
    """|got - want| is at most `frac` of the adapter's own effect |want - base| (plus `floor`), and that effect is visible."""
    effect = np.abs(want.astype(np.float64) - base).max()
    err = np.abs(got.astype(np.float64) - want).max()
    assert effect > 1e-3, f"{what}: the adapter has no visible effect ({effect:.2e})"
    assert err <= frac * effect + floor, f"{what}: |adapted - reference| = {err:.3e}, effect {effect:.3e}"


def ragged(lib, ctx, adapter, counts, flat):
    """Logits of every sequence after one ragged pass of a fresh batch context."""
    n = len(counts)
    batch = ctypes.c_void_p(lib.library.rwkv_b200_batch_create(ctx.c.ptr, n))
    try:
        if adapter is not None:
            assert lib.library.rwkv_b200_set_adapter(batch, adapter)
        assert lib.library.rwkv_b200_batch_eval_ragged(batch, (ctypes.c_uint32 * len(flat))(*flat), (ctypes.c_uint32 * n)(*counts), True)
        out = np.zeros((n, ctx.n_logits), np.float32)
        for s in range(n):
            assert lib.library.rwkv_b200_batch_get_logits(batch, s, fp(out[s]))
        assert lib.library.rwkv_b200_set_adapter(batch, None)
        return out
    finally:
        lib.library.rwkv_free(batch)


def score(lib, ctx, toks):
    """rwkv_b200_score of toks from a fresh state, each position scored against the next token."""
    lp = np.zeros(len(toks), np.float32)
    targets = toks[1:] + [toks[0]]
    assert lib.library.rwkv_b200_state_load(ctx.c.ptr, None)
    assert lib.library.rwkv_b200_score(ctx.c.ptr, (ctypes.c_uint32 * len(toks))(*toks), (ctypes.c_uint32 * len(toks))(*targets), len(toks),
                                       fp(lp), None)
    return lp


def all_passes(lib, c, adapter, toks):
    """Logits / states of every kind of pass: serial, one 70-token sequence, chunks of 16, a batch of 4, a ragged pass and scoring."""
    out = {"serial": c.serial(toks[:12]), "sequence": c.sequence(toks), "chunks": c.chunks(toks, 16)}
    prompts = [prompt(6, c.n_logits, s) for s in range(4)]
    for s, r in enumerate(batch_run(lib, c, adapter, prompts, 6) if adapter is not None else batch_run(lib, c, None, prompts, 6)):
        out[f"batch{s}"] = r
    counts = [3, 0, 5, 1]
    flat = [t for s, n in enumerate(counts) for t in prompt(n, c.n_logits, s)]
    rg = ragged(lib, c, adapter, counts, flat)
    out["ragged"] = (rg[[0, 2, 3]].reshape(-1),)
    out["score"] = (score(lib, c, toks),)
    return out


@pytest.mark.parametrize("ver", VERSIONS)
def test_adapted_fp32_matches_the_merged_file(lib, tmp_path, ver):
    path = model_path(ver, "FP32")
    entries = lr.make_entries(path, 8, 11, vectors=True, matrices=True)
    scale = 0.5
    merged = str(tmp_path / "merged.bin")
    lr.merged_file(path, merged, entries, scale)
    a, m = Ctx(lib, path), Ctx(lib, merged)
    try:
        toks = prompt(70, a.n_logits, 2)
        base = all_passes(lib, a, None, toks)
        want = all_passes(lib, m, None, toks)
        ad = a.adapter(entries, scale)
        a.attach(ad)
        got = all_passes(lib, a, ad, toks)
        a.attach(None)
        lib.rwkv_b200_adapter_free(ad)
        for kind in want:
            for i, part in enumerate(want[kind]):
                # FP32 weights: the merged and the adapted model differ only in where the delta's products are rounded
                within(got[kind][i], part, base[kind][i], 0.01, 1e-5, f"{ver} {kind}[{i}]")
    finally:
        a.free()
        m.free()


def encode(lib, dtype, values, M, K):
    """The file bytes rwkv_b200_adapter_create encodes a replaced matrix to (rwkv_b200_test_encode_rows)."""
    blck, size = lr.KQUANT_BLOCK.get(dtype) or lr.ggml_file.BLOCK[dtype]
    out = np.zeros(M * K * size // blck, np.uint8)
    vals = np.ascontiguousarray(values, np.float32)
    assert lib.library.rwkv_b200_test_encode_rows(dtype, fp(vals), M, K, out.ctypes.data_as(ctypes.c_void_p))
    return out


class AdaptedOracle:
    """The numpy oracle on a model file, with every delta of `entries` added to its matrix product in float64 (A and B rounded to
    fp16 as the library keeps them) before the matrix's epilogue, and every replacement in place of the file's values: a replaced
    matrix as the library encodes it at the file's type."""

    def __init__(self, lib, path, entries, scale):
        import rwkv_oracle
        self.o = rwkv_oracle.OracleModel(path)
        for name, rank, a, b, values in entries:
            if rank:
                base = self.o.mat(name)
                a16, b16 = lr.f16(a), lr.f16(b)

                class Adapted:
                    K, M = base.K, base.M

                    def mul(self, x, base=base, a16=a16, b16=b16):
                        y = base.mul(x)
                        return (y.astype(np.float64) + scale * (b16 @ (a16 @ np.asarray(x, np.float64)))).astype(np.float32)
                self.o._cache[("m", name)] = Adapted()
            elif lr.is_replaced_matrix(name):
                t = self.o.file.tensors[name]
                M, K = lr.matrix_shape(t)
                self.o._cache[("m", name)] = rwkv_oracle.Mat(lr.Tensor(name, t.dtype, t.ne, encode(lib, t.dtype, values, M, K)))
            else:
                self.o._cache[("v", name)] = np.asarray(values, np.float32)


def check_against_oracle(got, want, base, ours_plain, what):
    """Without an adapter we sit `spread` from the oracle on the same quantized file (activation quantisation, summation order); the
    adapted pair may sit three times as far apart, plus 2 % of the adapter's effect."""
    spread = np.abs(ours_plain.astype(np.float64) - base).max()
    effect = np.abs(want.astype(np.float64) - base).max()
    err = np.abs(got.astype(np.float64) - want).max()
    assert effect > 1e-3, (what, effect)
    assert err <= 3 * spread + 0.02 * effect + 1e-4, (what, err, spread, effect)


@pytest.mark.parametrize("ver", VERSIONS)
def test_adapted_q5_1_matches_the_oracle(lib, ver):
    """Serial passes (single tokens: the v6 LoRA fold) and one 70-token sequence (the tensor cores), with deltas, replaced vectors and
    replaced LoRA-internal matrices."""
    import rwkv_oracle
    path = model_path(ver, "Q5_1")
    entries = lr.make_entries(path, 8, 13, vectors=True, matrices=True)
    scale = 0.5
    plain = rwkv_oracle.OracleModel(path)
    adapted = AdaptedOracle(lib, path, entries, scale).o
    c = Ctx(lib, path)
    try:
        for what, toks, run in (("serial", prompt(8, plain.n_vocab, 4), Ctx.serial), ("sequence", prompt(70, plain.n_vocab, 5), Ctx.sequence)):
            base = plain.eval_sequence(toks, None)
            want = adapted.eval_sequence(toks, None)
            ours_plain = run(c, toks)
            ad = c.adapter(entries, scale)
            c.attach(ad)
            got = run(c, toks)
            c.attach(None)
            lib.rwkv_b200_adapter_free(ad)
            for i in range(2):
                check_against_oracle(got[i], want[i], base[i], ours_plain[i], f"{ver} {what} {('logits', 'state')[i]}")
    finally:
        c.free()


def file_with(lib, src, dst, entries):
    """src with every replacement of `entries` written into the file: a matrix at its type, encoded as the adapter encodes it, a vector
    in FP32 (the loader widens every vector to fp32)."""
    from ggml_file import write_model_file
    mf = lr.read_model_file(src)
    by_name = {e[0]: e for e in entries}
    tensors = []
    for name, t in mf.tensors.items():
        dtype, raw = t.dtype, t.raw
        if name in by_name:
            values = by_name[name][4]
            M, K = lr.matrix_shape(t)
            if lr.is_replaced_matrix(name):
                raw = encode(lib, t.dtype, values, M, K)
            else:
                dtype, raw = lr.F32, np.asarray(values, np.float32)
        tensors.append((name, dtype, t.ne, raw))
    write_model_file(dst, mf.n_vocab, mf.n_embed, mf.n_layer, mf.data_type, tensors, mf.version)


@pytest.mark.parametrize("ver", ["6v0-3m", "7v0-834K"])
@pytest.mark.parametrize("fmt", ["FP32", "FP16", "Q5_1"])
def test_replacements_equal_a_file_holding_them(lib, tmp_path, ver, fmt):
    """A replaced matrix is uploaded as the loader uploads it (encoding, device layout, tile-major copy), so an adapter of
    replacements only gives, bit for bit, what a file holding those values gives: single tokens with graphs (the v6 LoRA fold reads
    the replaced time_maa_w1 / time_decay_w2), 70 tokens with tensor cores on and off, and a batch of 4."""
    path = model_path(ver, fmt)
    entries = lr.make_entries(path, 8, 19, vectors=True, matrices=True, deltas=False)
    assert any(lr.is_replaced_matrix(e[0]) for e in entries)
    other = str(tmp_path / "replaced.bin")
    file_with(lib, path, other, entries)
    a, f = Ctx(lib, path), Ctx(lib, other)
    try:
        if ver.startswith("6"):
            t = lr.read_model_file(path).tensors
            C, mix5 = lr.matrix_shape(t["blocks.0.att.time_maa_w1"])[1], lr.matrix_shape(t["blocks.0.att.time_maa_w1"])[0]
            decay = lr.matrix_shape(t["blocks.0.att.time_decay_w1"])[0]
            assert lib.library.rwkv_b200_v6_lora_fold_supported(C, 64, t["blocks.0.att.time_maa_w1"].dtype, mix5 // 5,
                                                                t["blocks.0.att.time_decay_w2"].dtype, decay)
        ad = a.adapter(entries, 1.0)
        a.attach(ad)
        toks = prompt(70, a.n_logits, 7)
        prompts = [prompt(5, a.n_logits, s) for s in range(4)]
        assert same(a.serial(toks[:6]), f.serial(toks[:6]))
        assert same(a.sequence(toks), f.sequence(toks))
        for c in (a, f):
            lib.library.rwkv_b200_set_tensor_cores(c.c.ptr, False)
        assert same(a.sequence(toks), f.sequence(toks))
        for c in (a, f):
            lib.library.rwkv_b200_set_tensor_cores(c.c.ptr, True)
        for g, w in zip(batch_run(lib, a, ad, prompts, 5), batch_run(lib, f, None, prompts, 5)):
            assert same(g, w)
        a.attach(None)
        lib.rwkv_b200_adapter_free(ad)
    finally:
        a.free()
        f.free()


@pytest.mark.parametrize("fmt", ["Q4_K", "Q5_K"])
def test_zero_b_is_a_no_op_on_k_quants(lib, tmp_path, fmt):
    """The K-quant GEMV route: adapted problems of nonlinear epilogue retargeted to EPI_NONE and their epilogue applied by the expand."""
    import kquant_ref as kr
    G = kr.golden()
    master, path = str(tmp_path / "master.bin"), str(tmp_path / (fmt + ".bin"))
    kr.write_master(master, G["presets"]["rwkv6-small"], G["seed"])
    lib.rwkv_quantize_model_file(master, path, fmt)
    assert any(t.dtype in lr.KQUANT_BLOCK for n, t in lr.read_model_file(path).tensors.items() if lr.is_delta_target(n))
    c = Ctx(lib, path)
    try:
        toks = prompt(40, c.n_logits, 3)
        prompts = [prompt(5, c.n_logits, s) for s in range(4)]
        base = (c.serial(toks[:6]), c.sequence(toks), batch_run(lib, c, None, prompts, 5))
        ad = c.adapter(lr.make_entries(path, 8, 2, zero_b=True), 1.5)
        c.attach(ad)
        assert same(c.serial(toks[:6]), base[0]) and same(c.sequence(toks), base[1])
        for g, w in zip(batch_run(lib, c, ad, prompts, 5), base[2]):
            assert same(g, w)
        c.attach(None)
        lib.rwkv_b200_adapter_free(ad)
    finally:
        c.free()


def test_adapter_outlives_its_contexts(lib):
    """The adapter holds a reference to its model's weights: freeing the contexts first leaves it usable by a surviving clone and
    freeable last."""
    path = model_path("5v2-730K", "Q5_1")
    c = Ctx(lib, path)
    clone = Ctx.__new__(Ctx)
    clone.lib, clone.c, clone.n_state, clone.n_logits = lib, lib.rwkv_clone_context(c.c, 1), c.n_state, c.n_logits
    ad = c.adapter(lr.make_entries(path, 4, 9, vectors=True), 1.0)
    toks = prompt(12, c.n_logits, 1)
    c.attach(ad)
    want = c.sequence(toks)
    c.attach(None)
    c.free()                                 # the first context goes before its adapter
    clone.attach(ad)
    assert same(clone.sequence(toks), want)
    clone.attach(None)
    clone.free()                             # the last context goes: the adapter still holds the weights
    lib.rwkv_b200_adapter_free(ad)           # ... and releases them


def dequantized_fp32_file(src, dst):
    """src with every matrix dequantized to FP32 (K-quant blocks by kquant_ref, the legacy formats by the oracle)."""
    import kquant_ref as kr
    import rwkv_oracle
    from ggml_file import write_model_file
    mf = lr.read_model_file(src)
    tensors = []
    for name, t in mf.tensors.items():
        M, K = lr.matrix_shape(t)
        if t.dtype in lr.KQUANT_BLOCK:
            d, dmin, sc, mn, q = kr.unpack(t.dtype, t.raw, M, K)
            w = d[:, :, None, None] * sc[..., None] * q - dmin[:, :, None, None] * mn[..., None]
            raw = w.reshape(M, K).astype(np.float32)
        else:
            raw = rwkv_oracle.dequantize(t.dtype, t.raw, int(np.prod(t.ne))).astype(np.float32)
        tensors.append((name, 0, t.ne, raw))
    write_model_file(dst, mf.n_vocab, mf.n_embed, mf.n_layer, 0, tensors, mf.version)


def test_adapted_q4_k_matches_its_dequantized_merge(lib, tmp_path):
    """Q4_K: the adapted model against the same file dequantized to FP32 with the delta merged in float64. Without an adapter the two
    sit `spread` apart (the K-quant GEMV's Q8_K activations); the adapted pair may sit three times as far apart, plus 2 % of the
    adapter's effect."""
    import kquant_ref as kr
    G = kr.golden()
    master, q4k, deq, merged = (str(tmp_path / n) for n in ("master.bin", "q4k.bin", "deq.bin", "merged.bin"))
    kr.write_master(master, G["presets"]["rwkv6-small"], G["seed"])
    lib.rwkv_quantize_model_file(master, q4k, "Q4_K")
    dequantized_fp32_file(q4k, deq)
    entries = lr.make_entries(q4k, 16, 17, vectors=True)
    scale = 0.5
    lr.merged_file(deq, merged, entries, scale)
    q, d, m = Ctx(lib, q4k), Ctx(lib, deq), Ctx(lib, merged)
    try:
        toks = prompt(40, q.n_logits, 1)
        for run in (lambda c: c.serial(toks[:8]), lambda c: c.sequence(toks)):
            plain_q, base = run(q), run(d)
            want = run(m)
            ad = q.adapter(entries, scale)
            q.attach(ad)
            got = run(q)
            q.attach(None)
            lib.rwkv_b200_adapter_free(ad)
            for i in range(2):
                check_against_oracle(got[i], want[i], base[i], plain_q[i], f"Q4_K {i}")
    finally:
        for c in (q, d, m):
            c.free()


# ---- 4. invariants on an adapted context, bit for bit ---------------------------------------------------------------------------

@pytest.mark.parametrize("ver", VERSIONS)
def test_adapted_invariants(lib, ver):
    path = model_path(ver, "Q5_1")
    c = Ctx(lib, path)
    try:
        ad = c.adapter(lr.make_entries(path, 16, 21, vectors=True), 0.7)
        c.attach(ad)
        toks = prompt(31, c.n_logits, 3)
        serial = c.serial(toks)
        assert same(c.sequence(toks), serial)                  # below 32 tokens a pass never takes the tensor cores
        for chunk in (1, 4, 7, 16):
            assert same(c.chunks(toks, chunk), serial), chunk
        prompts = [prompt(5, c.n_logits, s) for s in range(15)]
        for s, got in enumerate(batch_run(lib, c, ad, prompts, 5)):
            assert same(got, c.serial(prompts[s])), s
        c.attach(None)
        lib.rwkv_b200_adapter_free(ad)
    finally:
        c.free()


@pytest.mark.parametrize("ver", VERSIONS)
def test_adapted_generate_sampled_equals_the_host_loop(lib, ver):
    """rwkv_b200_generate_sampled (top_k, min_p and penalties on) on an adapted context against the host loop of the sampling step
    hook + one eval per token on an adapted clone, as tests/test_gpu_generate_sampled.py checks unadapted contexts."""
    import generate_ref as gr
    from test_gpu_generate import Pair, logits
    from test_gpu_generate_sampled import Smp, gen_sampled, hook
    path = model_path(ver, "Q5_1")
    ctx = lib.rwkv_init_from_file(path, 1, 0)
    pair = Pair(lib, ctx)
    V = pair.n_vocab
    ad = lib.rwkv_b200_adapter_create(ctx, lr.make_entries(path, 8, 23, vectors=True), 1.0)
    try:
        lib.rwkv_b200_set_adapter(pair.host, ad)
        lib.rwkv_b200_set_adapter(pair.dev, ad)
        smp, mt = Smp(T=0.9, top_p=0.95, top_k=40, min_p=0.02, pres=0.2, freq=0.1), 12
        us = np.random.RandomState(7).random_sample(mt)
        pair.prime(prompt(4, V, 8))
        counts = np.zeros((1, V), np.uint32)
        want = []
        for i in range(mt):
            (tok,), counts, _ = hook(lib, logits(lib, pair.host.ptr, V)[None, :], [smp], [us[i]], counts)
            want.append(tok)
            gr.eval_token(lib, pair.host.ptr, tok)
        ok, got, _ = gen_sampled(lib, pair.dev.ptr, smp, mt, us)
        assert ok and got == want
        pair.same((ver, "adapted"))
        lib.rwkv_b200_set_adapter(pair.host, None)
        lib.rwkv_b200_set_adapter(pair.dev, None)
    finally:
        pair.free()
        lib.rwkv_free(ctx)
        lib.rwkv_b200_adapter_free(ad)


def test_two_clones_with_different_adapters_on_two_threads(lib):
    path = model_path("6v0-3m", "Q5_1")
    base = Ctx(lib, path)
    clones = [Ctx.__new__(Ctx) for _ in range(2)]
    for cl in clones:
        cl.lib, cl.c, cl.n_state, cl.n_logits = lib, lib.rwkv_clone_context(base.c, 1), base.n_state, base.n_logits
    ads = [base.adapter(lr.make_entries(path, r, 30 + r, vectors=True), 1.0) for r in (8, 16)]
    try:
        toks = prompt(40, base.n_logits, 6)
        want = []
        for cl, ad in zip(clones, ads):
            cl.attach(ad)
            want.append((cl.serial(toks[:10]), cl.sequence(toks)))
        assert not same(want[0][1], want[1][1])
        got = [None, None]

        def work(i):
            got[i] = [(clones[i].serial(toks[:10]), clones[i].sequence(toks)) for _ in range(3)]
        threads = [threading.Thread(target=work, args=(i,)) for i in range(2)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        for i in range(2):
            for s, q in got[i]:
                assert same(s, want[i][0]) and same(q, want[i][1]), i
    finally:
        for cl in clones:
            cl.attach(None)
            cl.free()
        for ad in ads:
            lib.rwkv_b200_adapter_free(ad)
        base.free()


# ---- 5. refusals -----------------------------------------------------------------------------------------------------------------

ERR_ARGS, ERR_CTX_UNSUPPORTED = 1 << 8, (6 << 8) | 9


def create_raw(lib, ctx_ptr, entries, scale):
    """rwkv_b200_adapter_create without the binding's exception: the handle (0 on refusal) and the global error flags."""
    import rwkv_cpp_b200.shared_library as sl
    arr = (sl.AdapterTensor * max(1, len(entries)))()
    keep = []
    for i, (name, rank, a, b, values) in enumerate(entries):
        ptrs = []
        for x in (a, b, values):
            if x is not None:
                keep.append(np.ascontiguousarray(x, np.float32))
            ptrs.append(fp(keep[-1]) if x is not None else None)
        arr[i] = sl.AdapterTensor(name.encode() if name is not None else None, rank, *ptrs)
    h = lib.library.rwkv_b200_adapter_create(ctx_ptr, arr, len(entries), ctypes.c_float(scale))
    return h or 0, lib.rwkv_get_last_error(None)


def test_refusals_change_nothing(lib, pkg):
    path = model_path("5v2-730K", "Q5_1")
    c = Ctx(lib, path)
    other = Ctx(lib, model_path("4v0-660K", "Q5_1"))
    lib.rwkv_set_print_errors(None, False)
    lib.rwkv_set_print_errors(c.c, False)
    try:
        good = lr.make_entries(path, 4, 41)
        ad = c.adapter(good, 1.0)
        c.attach(ad)
        toks = prompt(20, c.n_logits, 9)
        c.serial(toks[:3])
        want = (c.serial(toks[:3]), c.sequence(toks))
        name, rank, a, b, _ = good[0]
        vec = next(n for n in read_model_file(path).tensors if n.endswith("ln1.weight"))
        C = c.lib.rwkv_get_n_embed(c.c)
        bad_cases = {
            "unknown name": [("blocks.0.att.nothing.weight", 0, None, None, np.zeros(4, np.float32))],
            "duplicate": [good[0], good[0]],
            "rank above 256": [(name, 257, np.zeros((257, a.shape[1]), np.float32), np.zeros((b.shape[0], 257), np.float32), None)],
            "NULL A": [(name, rank, None, b, None)],
            "NULL values": [(vec, 0, None, None, None)],
            "no name": [(None, 0, None, None, np.zeros(C, np.float32))],
            "delta on emb": [("emb.weight", rank, a, b, None)],
            "replacement of head": [("head.weight", 0, None, None, np.zeros(4, np.float32))],
            "delta on a vector": [(vec, rank, a, b, None)],
            "NaN value": [(vec, 0, None, None, np.full(C, np.nan, np.float32))],
            "inf in A": [(name, rank, np.full_like(a, np.inf), b, None)],
            "A beyond fp16": [(name, rank, np.full_like(a, 1e6), b, None)],
            "replaced Q5_1 matrix beyond fp16": [(name, 0, None, None, np.full(a.shape[1] * b.shape[0], 1e6, np.float32))],
        }
        for what, entries in bad_cases.items():
            h, err = create_raw(lib, c.c.ptr, entries, 1.0)
            assert h == 0 and err == ERR_ARGS, (what, err)
        for scale in (float("nan"), float("inf")):
            h, err = create_raw(lib, c.c.ptr, good, scale)
            assert h == 0 and err == ERR_ARGS, scale
        # v6 / v7 layer LoRA matrices take no delta
        p6 = model_path("6v0-3m", "Q5_1")
        c6 = Ctx(lib, p6)
        try:
            t = read_model_file(p6).tensors["blocks.0.att.time_maa_w1"]
            M, K = lr.matrix_shape(t)
            h, err = create_raw(lib, c6.c.ptr, [("blocks.0.att.time_maa_w1", 2, np.zeros((2, K), np.float32), np.zeros((M, 2), np.float32), None)], 1.0)
            assert h == 0 and err == ERR_ARGS
        finally:
            c6.free()
        # an adapter of another model; freeing an attached adapter
        assert not lib.library.rwkv_b200_set_adapter(other.c.ptr, ad)
        assert lib.rwkv_get_last_error(other.c) == ERR_ARGS
        assert not lib.library.rwkv_b200_adapter_free(ad)
        assert lib.rwkv_get_last_error(None) == ERR_ARGS
        # set_adapter from inside this context's streaming callback
        seen = []

        @pkg.shared_library.RWKV_TOKEN_FN
        def on_token(user, seq, index, token):
            seen.append((lib.library.rwkv_b200_set_adapter(c.c.ptr, None), lib.rwkv_get_last_error(c.c)))
            return 0
        assert lib.library.rwkv_b200_state_load(c.c.ptr, None)
        assert lib.library.rwkv_b200_eval_resident(c.c.ptr, (ctypes.c_uint32 * 1)(toks[0]), 1, True, None)
        out = np.zeros(2, np.uint32)
        n = ctypes.c_size_t(0)
        assert lib.library.rwkv_b200_generate_stream(c.c.ptr, 2, 0.0, 1.0, 0.0, 0.0, False, np.zeros(2).ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
                                                     None, 0, on_token, None, out.ctypes.data_as(P_U), ctypes.byref(n))
        assert seen and all(r == (False, ERR_CTX_UNSUPPORTED) for r in seen), seen
        # after every refusal: the same bits, from the graphs captured before
        assert same(c.serial(toks[:3]), want[0]) and same(c.sequence(toks), want[1])
        c.attach(None)
        lib.rwkv_b200_adapter_free(ad)
        # a pipeline stage and a pipeline
        stage = lib.library.rwkv_b200_init_from_file_ex(path.encode(), 0, 0, 1)
        assert stage
        try:
            h, err = create_raw(lib, stage, good, 1.0)
            assert h == 0 and err == ERR_CTX_UNSUPPORTED
        finally:
            lib.library.rwkv_free(stage)
        pipe = lib.library.rwkv_b200_init_pipeline(path.encode(), (ctypes.c_int * 2)(0, 0), 2)
        assert pipe
        try:
            h, err = create_raw(lib, pipe, good, 1.0)
            assert h == 0 and err == ERR_CTX_UNSUPPORTED
        finally:
            lib.library.rwkv_free(pipe)
    finally:
        lib.rwkv_set_print_errors(None, True)
        c.free()
        other.free()


# ---- 6. Python: lora.py on RWKV-PEFT-style checkpoints ---------------------------------------------------------------------------

def merged_state_dict(base, lora, alpha):
    """base with the checkpoint applied in float64: W + alpha / rank * B16 . A16, replacements in place."""
    import torch
    from rwkv_cpp_b200.lora import _lora_part
    out = dict(base)
    pairs = {}
    for k, t in lora.items():
        name, part = _lora_part(k)
        if name:
            pairs.setdefault(name, {})[part] = t
        else:
            out[k] = t
    for name, ab in pairs.items():
        a, b = lr.f16(ab["lora_A"].numpy()), lr.f16(ab["lora_B"].numpy())
        w = base[name].double().numpy() + alpha / a.shape[0] * (b @ a)
        out[name] = torch.from_numpy(w.astype(np.float32))
    return out


@pytest.mark.parametrize("kind", ["v4", "v5.2", "v6", "v7"])
def test_lora_py_matches_the_merged_file(lib, pkg, tmp_path, kind):
    import torch
    import synthetic_checkpoint as sc
    from rwkv_cpp_b200 import convert_pytorch_to_ggml as conv, lora
    base_sd = sc.make_state_dict(kind, seed=0)
    lora_sd = sc.make_lora_state_dict(kind, rank=8, seed=5)
    pth = str(tmp_path / "lora.pth")
    torch.save(lora_sd, pth)
    base_bin, merged_bin = str(tmp_path / "base.bin"), str(tmp_path / "merged.bin")
    conv.write_state_dict(base_sd, base_bin, "FP32")
    alpha = 16
    conv.write_state_dict(merged_state_dict(base_sd, lora_sd, alpha), merged_bin, "FP32")
    model = pkg.RWKVModel(lib, base_bin, thread_count=1)
    merged = pkg.RWKVModel(lib, merged_bin, thread_count=1)
    try:
        toks = [(7 * i + 3) % 50 for i in range(40)]
        base = model.eval_sequence(toks, None, use_numpy=True)
        adapter = lora.Adapter(model, pth, lora_alpha=alpha)
        assert adapter.scale == alpha / 8
        if kind in ("v6", "v7"):     # the LoRA-internal matrices RWKV-PEFT trains with the time_* parameters are replaced
            assert any(lr.is_replaced_matrix(n) for n in adapter.names)
        model.set_adapter(adapter)
        got = model.eval_sequence(toks, None, use_numpy=True)
        want = merged.eval_sequence(toks, None, use_numpy=True)
        for i in range(2):
            within(got[i], want[i], base[i], 0.01, 1e-5, f"{kind} {('logits', 'state')[i]}")

        def serial(m):               # single tokens: the v6 fold reads the replaced time_maa_w1 / time_decay_w2
            st = None
            for t in toks[:6]:
                lg, st = m.eval(t, st, use_numpy=True)
            return lg, st
        got_s, want_s = serial(model), serial(merged)
        model.set_adapter(None)
        base_s = serial(model)
        for i in range(2):
            within(got_s[i], want_s[i], base_s[i], 0.01, 1e-5, f"{kind} serial {('logits', 'state')[i]}")
        again = model.eval_sequence(toks, None, use_numpy=True)
        assert same(again, base)
        model.set_adapter(adapter)
    finally:
        model.free()                 # the model goes first, with the adapter attached ...
        merged.free()
    adapter.free()                   # ... and the adapter is freed after it
