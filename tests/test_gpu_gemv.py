"""Per-kernel parity: the fused dequantize-GEMV (csrc/kernels/gemv.cu) through the C-ABI test hook against the
oracle's restatement of ggml_mul_mat for every weight type, ragged shapes, multi-column batches and epilogues.
Single-op comparisons have no rounding-flip amplification, so the tolerances are tight."""
import ctypes

import numpy as np
import pytest

import ggml_file as gf
import rwkv_oracle as ro

pytestmark = pytest.mark.gpu
PF = ctypes.POINTER(ctypes.c_float)
TYPES = ["FP32", "FP16", "Q4_0", "Q4_1", "Q5_0", "Q5_1", "Q8_0"]


def make_weights(fmt, M, K, rng):
    w = (rng.standard_normal((M, K)) / np.sqrt(K)).astype(np.float32)
    tid = gf.TYPE_IDS[fmt]
    if fmt == "FP32":
        raw = w.view(np.uint8).reshape(-1)
    elif fmt == "FP16":
        raw = w.astype(np.float16).view(np.uint8).reshape(-1)
    else:
        raw = ro.quantize_row_ref(tid, w.reshape(-1))
    return tid, np.ascontiguousarray(raw)


def run(lib, tid, K, M, T, raw, x, epi=0):
    y = np.zeros((T, M), np.float32)
    xc = np.ascontiguousarray(x.T)   # [T, K]: column t contiguous
    ok = lib.library.rwkv_b200_matvec(tid, K, M, T, raw.ctypes.data, xc.ctypes.data_as(PF), y.ctypes.data_as(PF), epi)
    assert ok
    return y.T


@pytest.mark.parametrize("fmt", TYPES)
@pytest.mark.parametrize("shape", [(64, 64), (160, 128), (448, 128), (128, 448), (96, 32), (33, 96), (256, 4096), (64, 14336), (1000, 2048)])
def test_gemv_matches_oracle(lib, fmt, shape):
    M, K = shape
    rng = np.random.default_rng(M * 131 + K)
    tid, raw = make_weights(fmt, M, K, rng)
    x = rng.standard_normal((K, 1)).astype(np.float32) * 2.0
    got = run(lib, tid, K, M, 1, raw, x)
    t = gf.Tensor("w", tid, (K, M), raw)
    want = ro.Mat(t).mul(x)
    scale = np.abs(want).max() + 1e-6
    assert np.abs(got - want).max() / scale < 2e-5, (fmt, shape, np.abs(got - want).max())


@pytest.mark.parametrize("fmt", TYPES)
@pytest.mark.parametrize("T", [2, 3, 4, 7, 9])
@pytest.mark.parametrize("shape", [(192, 320), (200, 64), (72, 128), (40, 4096), (24, 14336)])
def test_gemv_columns_are_batch_invariant(lib, fmt, T, shape):
    """Each column of a multi-column call is bit-identical to the single-column call (serial == sequence), for long rows
    (32 lanes per row, 1 / 4 warps per row) and short LoRA rows (lane groups)."""
    M, K = shape
    rng = np.random.default_rng(T)
    tid, raw = make_weights(fmt, M, K, rng)
    x = rng.standard_normal((K, T)).astype(np.float32)
    full = run(lib, tid, K, M, T, raw, x)
    for t in range(T):
        one = run(lib, tid, K, M, 1, raw, x[:, t:t + 1])
        assert one.tobytes() == np.ascontiguousarray(full[:, t:t + 1]).tobytes()


@pytest.mark.parametrize("epi,fn", [(1, lambda v: 1 / (1 + np.exp(-v))), (2, lambda v: v / (1 + np.exp(-v))), (3, np.tanh), (4, lambda v: np.maximum(v, 0) ** 2)])
def test_gemv_epilogues(lib, epi, fn):
    M, K = 128, 256
    rng = np.random.default_rng(epi)
    tid, raw = make_weights("Q5_1", M, K, rng)
    x = rng.standard_normal((K, 1)).astype(np.float32)
    base = run(lib, tid, K, M, 1, raw, x)
    got = run(lib, tid, K, M, 1, raw, x, epi)
    assert np.abs(got - fn(base.astype(np.float64))).max() < 1e-5


def test_gemv_zero_and_extreme_activations(lib):
    """All-zero blocks (amax == 0 -> id = 0, ggml-cpu-quants.c:806) and large magnitudes."""
    M, K = 64, 128
    rng = np.random.default_rng(5)
    for fmt in ("Q4_0", "Q5_1", "Q8_0"):
        tid, raw = make_weights(fmt, M, K, rng)
        x = np.zeros((K, 1), np.float32)
        assert not run(lib, tid, K, M, 1, raw, x).any()
        x[40:44, 0] = [1e4, -3e4, 2.5e4, 1.0]
        got = run(lib, tid, K, M, 1, raw, x)
        want = ro.Mat(gf.Tensor("w", tid, (K, M), raw)).mul(x)
        assert np.abs(got - want).max() / np.abs(want).max() < 2e-5


def q8_block_values(x):
    """The operand values of the reference's Q8_0 / Q8_1 activation blocks (ggml-cpu-quants.c:781-846): per 32 elements of a column
    d = fp16(amax / 127), q = rint(x * 127 / amax), value d * q."""
    K, T = x.shape
    xb = x.T.reshape(T, K // 32, 32).astype(np.float32)
    amax = np.abs(xb).max(axis=2, keepdims=True)
    d = (amax / np.float32(127.0)).astype(np.float16).astype(np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = np.where(amax != 0, np.float32(127.0) / amax, np.float32(0)).astype(np.float32)
    q = np.rint(xb * inv).astype(np.float32)
    return (d * q).reshape(T, K).T


@pytest.mark.parametrize("fmt", ["FP16", "Q4_0", "Q4_1", "Q5_0", "Q5_1", "Q8_0"])
@pytest.mark.parametrize("shape,T", [((128, 64), 32), ((256, 128), 48), ((160, 4096), 128), ((4096, 256), 64), ((512, 14336), 128), ((130, 192), 33), ((128, 64), 256), ((300, 2688), 100), ((140, 320), 250),
                                     ((4096, 4096), 128), ((1024, 2048), 96)])
def test_tensor_core_gemm_matches_fp16_reference(lib, fmt, shape, T):
    """wgmma prefill kernel (csrc/kernels/gemm_tc.cu), used for passes of >= 32 tokens: weights exactly as stored (rounded once to
    fp16), the B operand = fp16(x) for F16 weights and fp16 of the reference's Q8 block values (d * q) for quantised weights, fp32
    accumulation -- compared with that computation done in float64. The shapes cover launches with enough row tiles to run without a
    K-split, K-splits over thread-block clusters of 2 / 4 / 8 CTAs (few tiles, long K) and ragged M / T."""
    M, K = shape
    rng = np.random.default_rng(M + K + T)
    tid, raw = make_weights(fmt, M, K, rng)
    x = rng.standard_normal((K, T)).astype(np.float32)
    got = run(lib, tid, K, M, T, raw, x)
    w = ro.Mat(gf.Tensor("w", tid, (K, M), raw)).dense().astype(np.float64)
    if fmt != "FP16":   # the kernel rounds dequantised weights to fp16 once
        w = w.astype(np.float16).astype(np.float64)
    xin = x if fmt == "FP16" else q8_block_values(x)
    want = w @ xin.astype(np.float16).astype(np.float64)
    scale = np.abs(want).max() + 1e-6
    # quantised weights are rounded to fp16 by one fused multiply-add in the kernel (numpy: fp32 product, fp32 add, then fp16):
    # rare 1-ulp(fp16) differences in single weights
    assert np.abs(got - want).max() / scale < (2e-5 if fmt == "FP16" else 2e-4), (fmt, shape, T, np.abs(got - want).max() / scale)


def test_tensor_core_gemm_is_deterministic_and_scales_large_columns(lib):
    """The K-splits of a tile are summed in cluster rank order through distributed shared memory: the same launch twice gives the same bits. A column
    whose values exceed the fp16 range carries a power-of-two scale through the GEMM and comes out finite and accurate."""
    M, K, T = 160, 4096, 64          # 2 row tiles, 64 K-steps: cut along K
    rng = np.random.default_rng(77)
    # Q5_0 weights: their activations are Q8_0 blocks, whose only fp16 field is d = fp16(amax / 127) -- finite up to a block maximum of
    # 65504 * 127 = 8.3e6 (ggml-cpu-quants.c:796-803). (Q8_1 blocks, which Q4_1 / Q5_1 weights multiply, also carry s = fp16(d * sum q)
    # and overflow in the reference -- and in the dp4a path that mirrors it -- from block maxima of a few 1e4 on: out of its range.)
    tid, raw = make_weights("Q5_0", M, K, rng)
    x = rng.standard_normal((K, T)).astype(np.float32)
    x[:, 3] *= 3.0e5
    x[:, 7] *= 1.0e6
    a = run(lib, tid, K, M, T, raw, x)
    b = run(lib, tid, K, M, T, raw, x)
    assert a.tobytes() == b.tobytes() and np.isfinite(a).all()
    cols = np.concatenate([run(lib, tid, K, M, 1, raw, x[:, t:t + 1]) for t in range(T)], axis=1)
    rel = np.abs(a - cols).max(axis=0) / (np.abs(cols).max(axis=0) + 1e-6)
    assert rel.max() < 2e-3, rel.max()


def test_tensor_core_gemm_epilogue_and_tracks_decode_path(lib):
    """Same matrix through the tensor-core path (T = 64) and the batch-invariant GEMV (T = 1 columns): both contract the reference's
    Q8 activation values, so they differ only by the fp16 rounding of the operands (2^-12 relative per element)."""
    M, K, T = 256, 512, 64
    rng = np.random.default_rng(9)
    tid, raw = make_weights("Q5_1", M, K, rng)
    x = rng.standard_normal((K, T)).astype(np.float32)
    tc = run(lib, tid, K, M, T, raw, x, epi=4)
    cols = np.concatenate([run(lib, tid, K, M, 1, raw, x[:, t:t + 1], epi=4) for t in range(T)], axis=1)
    assert np.abs(tc - cols).max() / (np.abs(cols).max() + 1e-6) < 2e-3
