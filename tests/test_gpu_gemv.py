"""Per-kernel parity of the matrix kernels: the streaming and generic GEMVs (csrc/kernels/gemv_tma.cu, gemv.cu) and the tensor-core
GEMM (gemm_tc.cu).

The first tests go through rwkv_b200_matvec (one problem, no epilogue beyond relu^2) against the oracle's ggml_mul_mat. The rest go
through rwkv_b200_test_gemv_batch, which launches a batch of up to eight problems the way the eval path does, and compare every
output column with the float64 restatements in kernel_ref.py (gemv, gemm_tc) under kernel_ref.bar. They cover every compiled
instantiation, asserted through the hook's launch record and cross-checked against the library's symbols; all ten epilogues on each
family, both in place where the engine runs them in place; batches shaped like the engine's at 7B and tiny-fixture dimensions; the
LayerNorm prologue of the head; staged inputs; and the bit-level contracts of the SIMT GEMV. No output may keep a NaN of the 0xFF fill
and no guard may change."""
import collections
import ctypes
import functools
import re
import subprocess
import zlib

import numpy as np
import pytest

import ggml_file as gf
import kernel_hooks as kh
import kernel_ref as kr
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
    if fmt != "FP16":   # exactly as the kernel's single fused multiply-add rounds them (kernel_ref.tc_weights)
        w = np.concatenate([kr.tc_weights(tid, W) for _, _, W in kr.row_chunks(tid, raw, M, K)]).astype(np.float64)
    xin = x if fmt == "FP16" else q8_block_values(x)
    want = w @ xin.astype(np.float16).astype(np.float64)
    scale = np.abs(want).max() + 1e-6
    assert np.abs(got - want).max() / scale < 2e-5, (fmt, shape, T, np.abs(got - want).max() / scale)


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


# ---- one batch at a time through rwkv_b200_test_gemv_batch, against float64 --------------------------------------------------

F64, F32 = np.float64, np.float32
FMT = {name: gf.TYPE_IDS[name] for name in TYPES}
TC_TYPES = ["FP16", "Q4_0", "Q4_1", "Q5_0", "Q5_1", "Q8_0"]
# wgmma accumulates in fp32, but not as a sequence of round-to-nearest additions: on an H100 80GB HBM3 (400 W) its outputs landed
# up to 43x as far from float64 as the float32 restatement (numpy's matmul) did -- the 14336 x 4096 ffn.key at T = 64 with relu^2 --
# and 4-18x for the other K = 1024 .. 14336 launches, growing with K as truncated accumulation does; at factor 4 every K <= 256
# launch stayed inside the bar. The tensor-core bar is this many times the float32 distance.
TC_BAR_FACTOR = 64
WORST = collections.defaultdict(float)
NEEDED = collections.defaultdict(float)   # error / |float32 - float64| where the error is above the 1e-6 floor: the factor a family needed
LAUNCHED = set()          # instantiations the tests below launched (launch_key)
CLUSTERS = set()          # cluster sizes of the tensor-core launches
CONVERT_INPUTS = set()    # distinct inputs of the fp16 conversion launches


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    for family in sorted(WORST):
        print("\n%-13s worst error / bar = %.3f (error / fp32 distance %.2f)" % (family, WORST[family], NEEDED[family]), end="")
    print()


def rng_for(*key):
    return np.random.default_rng(zlib.crc32(repr(key).encode()))


@functools.lru_cache(maxsize=64)
def random_raw(fmt, M, K, seed=0):
    """M rows of K weights in the file layout of fmt with entries of about 1/sqrt(K): random stored integers and scales (quantised),
    random values (F16 / F32). Built directly as bytes, so 7B-sized matrices cost no quantisation."""
    rng = rng_for("raw", fmt, M, K, seed)
    tid = FMT[fmt]
    if fmt in ("FP32", "FP16"):
        w = (rng.standard_normal((M, K)) / np.sqrt(K)).astype(np.float16 if fmt == "FP16" else np.float32)
        return tid, w.view(np.uint8).reshape(-1)
    nb = M * K // 32
    elems, nbytes = gf.BLOCK[tid]
    blk = rng.integers(0, 256, (nb, nbytes), dtype=np.uint8)
    spread = {"Q4_0": 4.6, "Q4_1": 4.6, "Q5_0": 9.2, "Q5_1": 9.2, "Q8_0": 73.0}[fmt]
    d = (rng.uniform(0.5, 1.5, nb) / (spread * np.sqrt(K))).astype(np.float16)
    blk[:, 0:2] = d.view(np.uint8).reshape(nb, 2)
    if fmt in ("Q4_1", "Q5_1"):
        m = (-d.astype(F64) * (7.5 if fmt == "Q4_1" else 15.5) * rng.uniform(0.8, 1.2, nb)).astype(np.float16)
        blk[:, 2:4] = m.view(np.uint8).reshape(nb, 2)
    return tid, blk.reshape(-1)


def problem(fmt, M, K, T, rng, input=0, epi=kr.EPI_NONE, tiled=None, alias=True, weights=None):
    """One problem of a batch: weights (random_raw's, or `weights` = (type, bytes) given), and the residual / gate / bias its epilogue
    reads. The bias puts a quarter of the rows deep into the saturation of the sigmoid / exp(-exp) epilogues, on both sides."""
    tid, raw = weights or random_raw(fmt, M, K)
    p = dict(type=tid, K=K, M=M, raw=raw, input=input, epi=epi, fmt=fmt,
             tiled=fmt != "FP32" and K % 64 == 0 if tiled is None else tiled)
    if epi in kr.RES_EPIS:
        p["res"], p["alias"] = rng.standard_normal((M, T)).astype(F32), alias
    if epi == kr.EPI_MUL_ADD:
        p["gate"] = rng.standard_normal((M, T)).astype(F32)
    if epi in kr.BIAS_EPIS:
        b = rng.standard_normal(M).astype(F32)
        far = rng.random(M) < 0.25
        b[far] = rng.choice([-30.0, -6.0, 6.0, 30.0], far.sum())
        p["bias"] = b
    return p


def with_layernorm(p, x, rng, **margins):
    """Give p the head's LayerNorm prologue, with ln_b chosen so that fp32 and float64 LayerNorms give the same operands (margins: of
    kernel_ref.ln_bias_away_from_roundings)."""
    K = p["K"]
    w = (1 + 0.2 * rng.standard_normal(K)).astype(F32)
    b = (0.2 * rng.standard_normal(K)).astype(F32)
    p.update(pro=1, ln_w=w, ln_b=kr.ln_bias_away_from_roundings(x, w, b, p["type"], rng, **margins))
    return p


def inputs(Ks, T, rng, scale=2.0):
    return [(rng.standard_normal((K, T)) * scale).astype(F32) for K in Ks]


def launch_key(l):
    fam, nc, only, has_ln, npad, cluster = l
    if fam == "streaming":
        return (fam, nc, only, has_ln)
    if fam == "generic":
        return (fam, nc)
    if fam == "tensor_cores":
        CLUSTERS.add(cluster)
        return (fam, npad)
    if fam == "convert":
        CONVERT_INPUTS.add(nc)
        return (fam,)
    return (fam, only)


def run_batch(lib, T, probs, xs, path="engine"):
    outs, launches = kh.gemv_batch(lib, T, probs, xs, path)
    for o in outs:
        assert o.guard_intact(), "write past the end of an output"
    LAUNCHED.update(launch_key(l) for l in launches)
    return [o.cols(p["M"]) for o, p in zip(outs, probs)], launches


def takes_tc(p, T, path):
    """Where the routing of the eval path (gemv_route) sends p."""
    if path == "tensor_cores":
        return True
    tc_min = {"engine": 32, "engine_batch_ctx": 16}.get(path)
    return tc_min is not None and T >= tc_min and p["tiled"] and not p.get("pro")


def reference(p, xs, dt, tc, bug=None):
    x = xs[p["input"]]
    kw = dict(epi=p["epi"], res=p.get("res"), gate=p.get("gate"), bias=p.get("bias"), bug=bug)
    if tc:
        return kr.gemm_tc(p["type"], p["raw"], p["M"], x, dt, **kw)
    return kr.gemv(p["type"], p["raw"], p["M"], x, dt, ln=(p["ln_w"], p["ln_b"]) if p.get("pro") else None, **kw)


def check(family, name, got, p, xs, tc):
    assert not np.isnan(got).any(), (family, name, "NaN left in the output")
    r64, r32 = reference(p, xs, F64, tc), reference(p, xs, F32, tc)
    ratio = kr.error_over_bar(got, r64, r32, TC_BAR_FACTOR if tc else 4)
    WORST[family] = max(WORST[family], ratio)
    err, d32 = np.abs(got - r64).max(axis=0), np.abs(r32 - r64).max(axis=0)
    NEEDED[family] = max(NEEDED[family], float((err / np.maximum(d32, 1e-30))[err > kr.bar(r64, r32, 0)].max(initial=0)))
    assert ratio <= 1, (family, name, ratio, np.abs(got - r64).max())


def check_all(name, T, probs, xs, path, outs, launches):
    """Every output against its float64 result, on the family the routing sent it to; the launches agree with that routing."""
    fams = [l[0] for l in launches if l[0] != "expand"]
    for p, got in zip(probs, outs):
        tc = takes_tc(p, T, path)
        family = "tensor_cores" if tc else ("generic" if "generic" in fams else "streaming")
        check(family, (name, p["fmt"], p["M"], p["K"], p["epi"]), got, p, xs, tc)
    n_tc = sum(takes_tc(p, T, path) for p in probs)
    assert ("tensor_cores" in fams) == (n_tc > 0) and ("convert" in fams) == (n_tc > 0), (name, launches)
    assert (("streaming" in fams) or ("generic" in fams)) == (n_tc < len(probs)), (name, launches)


def bits(a):
    return np.ascontiguousarray(a).tobytes()


def stream_nc(T, probs):
    """Columns per group of a streaming launch (gemv_tma_launch): 4 or 2 while the ring stages stay >= 28 KB next to that many
    staged columns of the batch's widest input, else 1."""
    def col_bytes(p):
        K = p["K"]
        if p["fmt"] in ("FP32", "FP16"):
            b = K * (4 if p["fmt"] == "FP32" else 2)
        else:
            nblk = K // 32
            b = (nblk if p["fmt"] in ("Q4_1", "Q5_1") else (nblk + 1) // 2 * 2) * 40
        return (b + 15) // 16 * 16
    mc = max(col_bytes(p) for p in probs)
    stage = lambda nc: (110 * 1024 - nc * mc - 2 * 64 * 8 * nc * 4) // 3 // 1024 * 1024
    return 4 if T >= 4 and stage(4) >= 28 * 1024 else 2 if T >= 2 and stage(2) >= 28 * 1024 else 1


# ---- every instantiation ---------------------------------------------------------------------------------------------

STREAM_SHAPES = [(300, 4096), (64, 14336), (4096, 64), (1000, 32)]      # (M, K): WK = 1 / G = 32, WK > 1, LoRA rows (G < 32), tiny


@pytest.mark.parametrize("fmt", TYPES)
@pytest.mark.parametrize("shape", STREAM_SHAPES)
@pytest.mark.parametrize("has_ln", [False, True])
def test_streaming_per_format_instantiation(lib, fmt, shape, has_ln):
    """gemv_tma_kernel<1, TYPE, HAS_LN> for all seven formats, with and without the LayerNorm prologue."""
    M, K = shape
    if fmt in ("FP32", "FP16") and K == 14336:
        K = 3584 if fmt == "FP32" else 7168       # 14 KB rows: 28 KB ones leave the ring no room next to the staged column
    rng = rng_for("stream", fmt, shape, has_ln)
    xs = inputs([K], 1, rng)
    p = problem(fmt, M, K, 1, rng, tiled=False)
    if has_ln:
        with_layernorm(p, xs[0], rng)
    (y,), launches = run_batch(lib, 1, [p], xs, "streaming")
    assert launches == [("streaming", 1, FMT[fmt], int(has_ln), 0, 0)], launches
    check("streaming", (fmt, shape, has_ln), y, p, xs, False)


EPI_CASES = [  # (family, fmt, M, K, T): streaming WK = 1 with G = 32 and G = 1 / 8 / 2 / 8 (LoRA rows), WK > 1; generic; tensor cores
    ("streaming", "Q5_1", 256, 4096, 1), ("streaming", "Q5_1", 4096, 32, 1), ("streaming", "FP16", 2048, 64, 1),
    ("streaming", "Q5_0", 4096, 96, 1), ("streaming", "Q5_1", 4096, 160, 1), ("streaming", "Q4_0", 128, 14336, 1),
    ("generic", "Q4_1", 300, 256, 5),
    ("tensor_cores", "FP16", 2048, 256, 40),      # 16 tiles of 4 K-steps: not cut, tc_epilogue_rows
    ("tensor_cores", "Q5_0", 256, 4096, 64),      # 2 tiles of 64 K-steps: cut over a cluster, tc_reduce_columns
]


@pytest.mark.parametrize("epi", range(10))
@pytest.mark.parametrize("case", EPI_CASES, ids=lambda c: "%s-%s-%dx%d-T%d" % c)
def test_epilogues(lib, epi, case):
    """All ten epilogues on every family; EPI_ADD and EPI_MUL_ADD in place (y is the residual), as att.output and ffn.value run."""
    family, fmt, M, K, T = case
    rng = rng_for("epi", epi, case)
    xs = inputs([K], T, rng)
    p = problem(fmt, M, K, T, rng, epi=epi, tiled=family == "tensor_cores")
    (y,), launches = run_batch(lib, T, [p], xs, family)
    assert launches[-1][0] == family, launches
    if family == "tensor_cores":
        assert (launches[-1][5] > 1) == (K == 4096), launches
    check(family, ("epi", epi, case), y, p, xs, family == "tensor_cores")


# T ragged inside every pad of 16 (NPAD 16 .. 256), shapes cycling through cluster sizes 8 / 4 / 2 / 1 and the six eligible formats
NPAD_T = [16, 17, 31, 33, 63, 79, 96, 112, 127, 144, 150, 161, 180, 200, 217, 239, 250]
TC_SHAPES = [(128, 2048), (2560, 1024), (5120, 512), (300, 128)]   # 1 tile (cluster 8), 20 tiles (4), 40 tiles (2), 3 tiles of 2 K-steps (1)


@pytest.mark.parametrize("i,T", list(enumerate(NPAD_T)))
def test_tensor_core_every_npad(lib, i, T):
    """gemm_tc_kernel<NPAD> for all sixteen pads, with the token count ragged inside the pad."""
    fmt, (M, K), epi = TC_TYPES[i % 6], TC_SHAPES[i % 4], (0, 4, 6, 8)[i % 4]
    rng = rng_for("npad", T)
    xs = inputs([K], T, rng)
    p = problem(fmt, M, K, T, rng, epi=epi, tiled=True)
    (y,), launches = run_batch(lib, T, [p], xs, "tensor_cores")
    assert launches[0] == ("expand", 0, FMT[fmt], 0, 0, 0) and launches[1][0] == "convert", launches
    assert launches[2][:5] == ("tensor_cores", 0, 0, 0, (T + 15) // 16 * 16), launches
    check("tensor_cores", ("npad", T, fmt), y, p, xs, True)


@pytest.mark.parametrize("n", range(1, 9))
def test_convert_distinct_inputs(lib, n):
    """convert_f16_kernel with 1 .. 8 distinct inputs, and operand sharing: problems reading one input share its fp16 copy only if
    their operand kinds agree (F16 weights multiply fp16(x), quantised ones the Q8 block values)."""
    T, K = 33, 256
    rng = rng_for("convert", n)
    xs = inputs([K] * n, T, rng)
    probs = [problem(TC_TYPES[j % 6], 128 + 32 * j, K, T, rng, input=j, epi=j % 10) for j in range(n)]
    outs, launches = run_batch(lib, T, probs, xs, "tensor_cores")
    assert [l for l in launches if l[0] == "convert"][0][1] == n, launches
    check_all("convert", T, probs, xs, "tensor_cores", outs, launches)
    # one input, F16 and quantised problems mixed: two converted copies
    probs = [problem(f, 200, K, T, rng, input=0, epi=e) for f, e in (("FP16", 0), ("Q5_1", 3), ("FP16", 8), ("Q4_0", 5))]
    outs, launches = run_batch(lib, T, probs, xs[:1], "tensor_cores")
    assert [l for l in launches if l[0] == "convert"][0][1] == 2, launches
    check_all("shared input", T, probs, xs[:1], "tensor_cores", outs, launches)


@pytest.mark.parametrize("T,nc", [(1, 1), (3, 2), (5, 4)])
def test_generic_instantiations(lib, T, nc):
    """gemv_kernel<1 | 2 | 4>, with a LayerNorm problem and epilogues in the batch; and the engine's fallback to it when one problem
    of a batch cannot stream (an F32 ffn.value at 7B: 57 KB rows)."""
    rng = rng_for("generic", T)
    xs = inputs([256, 320], T, rng)
    probs = [problem("Q5_1", 300, 256, T, rng, epi=kr.EPI_TANH), problem("FP16", 100, 320, T, rng, input=1, epi=kr.EPI_ADD),
             with_layernorm(problem("Q4_0", 129, 256, T, rng, tiled=False), xs[0], rng)]
    outs, launches = run_batch(lib, T, probs, xs, "generic")
    assert [l for l in launches if l[0] != "expand"] == [("generic", nc, -1, 0, 0, 0)], launches
    check_all("generic", T, probs, xs, "generic", outs, launches)
    xs = inputs([14336, 4096], T, rng)
    probs = [problem("FP32", 4096, 14336, T, rng, epi=kr.EPI_MUL_ADD), problem("Q5_1", 512, 4096, T, rng, input=1, epi=kr.EPI_SIGMOID)]
    outs, launches = run_batch(lib, T, probs, xs, "engine")
    # 57 KB columns: four of them do not fit the generic kernel's shared memory either
    assert [l for l in launches if l[0] != "expand"] == [("generic", min(nc, 2), -1, 0, 0, 0)], launches
    check_all("fallback", T, probs, xs, "engine", outs, launches)


# ---- batches shaped like the engine's (csrc/engine.cu) ----------------------------------------------------------------

DIMS = {"7B": dict(C=4096, F=14336, w=64, a=64, g=160, v=32, V=65536), "tiny": dict(C=32, F=128, w=32, a=32, g=32, v=32, V=1000)}


def engine_batch(name, d, fmt, lora, T, rng):
    """(problems, inputs) of one run_batch of engine.cu: att_v6 :335-341, att_v7 :367-375 / :378-383, ffn :220-230, att_output
    :236-241, the head :462-466. `lora`: the weight format of the v7 LoRA matrices (the quantiser keeps them F16 / F32)."""
    C, F = d["C"], d["F"]
    P = lambda f, M, K, i, epi=0: problem(f, M, K, T, rng, input=i, epi=epi)
    if name == "v6_att":        # r, k, v, g, decay LoRA: five distinct mixed inputs
        probs = [P(fmt, C, C, 0), P(fmt, C, C, 1), P(fmt, C, C, 2), P(fmt, C, C, 3, kr.EPI_SILU), P(fmt, d["w"], C, 4, kr.EPI_TANH)]
        Ks = [C] * 5
    elif name == "v7_first":    # r, k, v, w1, a1, g1, v1; v and v1 read the same input
        probs = [P(fmt, C, C, 0), P(fmt, C, C, 2), P(fmt, C, C, 3), P(lora, d["w"], C, 1, kr.EPI_TANH), P(lora, d["a"], C, 4),
                 P(lora, d["g"], C, 5, kr.EPI_SIGMOID), P(lora, d["v"], C, 3)]
        Ks = [C] * 6
    elif name == "v7_second":   # w2, a2, g2, v2: three bias epilogues on K = 32 .. 160 rows
        probs = [P(lora, C, d["w"], 0, kr.EPI_BIAS_W7), P(lora, C, d["a"], 1, kr.EPI_BIAS_SIGMOID), P(lora, C, d["g"], 2),
                 P(lora, C, d["v"], 3, kr.EPI_BIAS_SIGMOID)]
        Ks = [d["w"], d["a"], d["g"], d["v"]]
    elif name == "ffn_kr":
        probs, Ks = [P(fmt, F, C, 0, kr.EPI_RELU_SQR), P(fmt, C, C, 1, kr.EPI_SIGMOID)], [C, C]
    elif name == "ffn_value":   # in place: x += r * (Wv k) (v4-v6), x += Wv k (v7)
        probs, Ks = [P(fmt, C, F, 0, kr.EPI_MUL_ADD)], [F]
    elif name == "ffn_value_v7":
        probs, Ks = [P(fmt, C, F, 0, kr.EPI_ADD)], [F]
    elif name == "att_output":
        probs, Ks = [P(fmt, C, C, 0, kr.EPI_ADD)], [C]
    xs = inputs(Ks, T, rng)
    return probs, xs


ENGINE_CASES = ([("7B", b, "Q5_1", "FP16", T, path) for b in ("v6_att", "v7_first", "v7_second", "ffn_kr", "ffn_value", "ffn_value_v7", "att_output")
                 for T, path in ((1, "engine"), (64, "engine"))]
                + [("7B", b, "Q5_1", "FP32", T, path) for b in ("v7_first", "v7_second") for T, path in ((1, "engine"), (64, "engine"))]
                + [("7B", b, "Q5_1", "FP16", 20, "engine_batch_ctx") for b in ("v7_first", "v7_second", "att_output")]
                + [("tiny", b, f, "FP16", T, path) for f in ("Q4_0", "Q5_0", "Q8_0")
                   for b in ("v6_att", "v7_first", "v7_second", "ffn_kr", "ffn_value", "att_output")
                   for T, path in ((1, "engine"), (4, "engine_batch_ctx"), (20, "engine_batch_ctx"), (64, "engine"))])


@pytest.mark.parametrize("dims,batch,fmt,lora,T,path", ENGINE_CASES)
def test_engine_shaped_batches(lib, dims, batch, fmt, lora, T, path):
    rng = rng_for("engine", dims, batch, fmt, lora, T, path)
    probs, xs = engine_batch(batch, DIMS[dims], fmt, lora, T, rng)
    outs, launches = run_batch(lib, T, probs, xs, path)
    if T == 1:     # one format in the batch: its own instantiation without LayerNorm; else the mixed-format kernel
        only = probs[0]["type"] if len({p["type"] for p in probs}) == 1 else -1
        assert [l for l in launches if l[0] != "expand"] == [("streaming", 1, only, int(only < 0), 0, 0)], launches
    check_all((dims, batch), T, probs, xs, path, outs, launches)


HEAD_CASES = [("Q5_1", 65536, 4096, 1, "engine", 1.5), ("FP16", 50277, 2560, 1, "engine", 1.5), ("Q8_0", 4096, 1024, 1, "engine", 0.05),
              ("Q5_1", 1000, 4096, 4, "engine_batch_ctx", 1.5), ("FP16", 777, 2560, 2, "engine_batch_ctx", 0.05),
              ("Q5_0", 1000, 32, 20, "engine_batch_ctx", 1.5), ("FP32", 1000, 64, 3, "engine", 0.05)]


def head_case(fmt, V, C, T, scale):
    """(problem, inputs) of a head: the small-scale inputs give the LayerNorm a variance that eps 1e-5 visibly enters."""
    rng = rng_for("head", fmt, V, C, T, scale)
    xs = inputs([C], T, rng, scale=scale)
    return with_layernorm(problem(fmt, V, C, T, rng, tiled=False), xs[0], rng), xs


@pytest.mark.parametrize("fmt,V,C,T,path,scale", HEAD_CASES)
def test_head(lib, fmt, V, C, T, path, scale):
    """The head, LN(x; ln_out) . W (engine.cu:462-466): the single-token one (<1, TYPE, true>) at V = 65536 and at a ragged V, and a
    batch context's (one column per sequence: <2 | 4, -1, true>, and the LayerNorm problem staying off the tensor cores at T = 20)."""
    p, xs = head_case(fmt, V, C, T, scale)
    outs, launches = run_batch(lib, T, [p], xs, path)
    nc = stream_nc(T, [p])
    assert launches == [("streaming", nc, FMT[fmt] if nc == 1 else -1, 1, 0, 0)], launches
    check_all("head", T, [p], xs, path, outs, launches)


def test_mixed_format_kernel_with_layernorm(lib):
    """<1, -1, true> with a LayerNorm problem among quantised and F16 / F32 ones, and the multi-column kernel on the same batch."""
    for T in (1, 2, 7):
        rng = rng_for("mixed-ln", T)
        xs = inputs([4096, 64, 2560], T, rng)
        probs = [problem("Q5_1", 512, 4096, T, rng, epi=kr.EPI_SILU), problem("FP32", 256, 64, T, rng, input=1, epi=kr.EPI_TANH),
                 with_layernorm(problem("Q4_1", 300, 2560, T, rng, input=2, tiled=False), xs[2], rng),
                 problem("FP16", 160, 4096, T, rng, epi=kr.EPI_BIAS_W7)]
        outs, launches = run_batch(lib, T, probs, xs, "streaming")
        assert [l for l in launches if l[0] != "expand"] == [("streaming", stream_nc(T, probs), -1, 1, 0, 0)], launches
        check_all("mixed+ln", T, probs, xs, "streaming", outs, launches)


# ---- bit-level contracts of the SIMT GEMV (DESIGN.md section 3) -----------------------------------------------------------

@pytest.mark.parametrize("fmt", TYPES)
def test_problem_alone_equals_in_batch(lib, fmt):
    """A problem gives the same bits alone, inside a batch of its own format (per-format kernel) and inside a mixed batch."""
    rng = rng_for("alone", fmt)
    xs = inputs([4096, 1024], 1, rng)
    p = problem(fmt, 777, 4096, 1, rng, epi=kr.EPI_ADD)
    (alone,), l1 = run_batch(lib, 1, [p], xs[:1], "engine")
    same = [problem(fmt, 500, 1024, 1, rng, input=1, epi=kr.EPI_SIGMOID), p]
    outs, l2 = run_batch(lib, 1, same, xs, "engine")
    other = "Q5_1" if fmt != "Q5_1" else "FP16"
    mixed = [problem(other, 300, 1024, 1, rng, input=1), p, problem("FP32", 64, 1024, 1, rng, input=1)]
    outm, l3 = run_batch(lib, 1, mixed, xs, "engine")
    assert l1[-1][2] == l2[-1][2] == FMT[fmt] and l3[-1][2] == -1, (l1, l2, l3)
    assert bits(alone) == bits(outs[1]) == bits(outm[1])
    check("streaming", ("alone", fmt), alone, p, xs, False)


@pytest.mark.parametrize("T", [2, 3, 4, 7])
def test_multi_column_launches_equal_single_columns(lib, T):
    """Every column of an NC = 2 / 4 launch equals the T = 1 launch of that column, LayerNorm prologue and epilogues included. The
    NC = 2 batches carry a K = 7168 problem, whose rows are split over 4 warps (WK = 4)."""
    rng = rng_for("columns", T)
    xs = inputs([2048, 160, 1024, 7168], T, rng)
    probs = [with_layernorm(problem("Q5_1", 300, 2048, T, rng, tiled=False), xs[0], rng),
             problem("Q4_0", 2048, 160, T, rng, input=1, epi=kr.EPI_BIAS_EXPNEGEXP), problem("FP16", 96, 1024, T, rng, input=2, epi=kr.EPI_MUL_ADD)]
    if T < 4:
        probs.append(problem("Q8_0", 64, 7168, T, rng, input=3, epi=kr.EPI_TANH))
    full, launches = run_batch(lib, T, probs, xs, "streaming")
    assert launches[-1][:2] == ("streaming", stream_nc(T, probs)) and stream_nc(T, probs) == (4 if T >= 4 else 2), launches
    for t in range(T):
        col = lambda a: None if a is None else a[:, t:t + 1]
        one = [dict(p, res=col(p.get("res")), gate=col(p.get("gate"))) for p in probs]
        outs, _ = run_batch(lib, 1, one, [x[:, t:t + 1] for x in xs], "streaming")
        for a, b in zip(outs, full):
            assert bits(a) == bits(b[:, t:t + 1]), t
    for p, got in zip(probs, full):
        check("streaming", ("columns", T, p["fmt"]), got, p, xs, False)


@pytest.mark.parametrize("fmt", ["FP32", "FP16", "Q5_0", "Q5_1"])          # stage classes F32, F16, Q8_0, Q8_1
@pytest.mark.parametrize("mixed", [False, True])
def test_staged_input_is_what_the_kernel_reads(lib, fmt, mixed):
    """xq: the staged column of x gives the bits of staging from x, on the per-format and the mixed kernel; a column staged from a
    different vector gives that vector's result, so the consumer really reads xq."""
    rng = rng_for("xq", fmt, mixed)
    K = 4096
    xs, other = inputs([K, 512], 1, rng), inputs([K], 1, rng)[0]
    p = problem(fmt, 1000, K, 1, rng, epi=kr.EPI_ADD)
    extra = [problem("Q4_1" if fmt != "Q4_1" else "FP16", 200, 512, 1, rng, input=1)] if mixed else []
    base, l1 = run_batch(lib, 1, [p] + extra, xs, "streaming")
    staged, l2 = run_batch(lib, 1, [dict(p, xq=kr.staged_column(xs[0], FMT[fmt], guard=0))] + extra, xs, "streaming")
    assert l1 == l2 and l1[-1][2] == (-1 if mixed else FMT[fmt]), l1
    assert bits(base[0]) == bits(staged[0])
    moved, _ = run_batch(lib, 1, [dict(p, xq=kr.staged_column(other, FMT[fmt], guard=0))] + extra, xs, "streaming")
    want, _ = run_batch(lib, 1, [p] + extra, [other] + xs[1:], "streaming")
    assert bits(moved[0]) == bits(want[0]) and bits(moved[0]) != bits(base[0])


# ---- the tensor-core path: the LayerNorm prologue stays off it, large columns -----------------------------------------------

def test_tensor_cores_refuse_the_layernorm_prologue(lib):
    """convert_f16_kernel applies no LayerNorm, so a problem with the head's prologue never takes the tensor cores, even with a
    tile-major copy: TENSOR_CORES refuses the batch, and the engine's routing at T = 64 sends it to the streaming kernel."""
    T = 64
    rng = rng_for("tc-ln")
    xs = inputs([1024], T, rng)
    p = with_layernorm(problem("Q5_1", 500, 1024, T, rng, tiled=True), xs[0], rng)
    with pytest.raises(kh.HookError) as e:
        run_batch(lib, T, [p], xs, "tensor_cores")
    assert e.value.flags == (6 << 8) | 9          # RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED
    q = problem("Q5_1", 256, 1024, T, rng, epi=kr.EPI_TANH)
    outs, launches = run_batch(lib, T, [p, q], xs, "engine")
    assert [l[0] for l in launches if l[0] != "expand"] == ["convert", "tensor_cores", "streaming"], launches
    assert launches[-1] == ("streaming", 4, -1, 1, 0, 0), launches
    check_all("tc+ln", T, [p, q], xs, "engine", outs, launches)


def test_tensor_core_large_columns_with_epilogue_and_ksplit(lib):
    """Columns beyond the fp16 range through a K-split launch with an in-place epilogue: the column scale 2^e is taken out before
    the residual is added."""
    M, K, T = 256, 4096, 48
    rng = rng_for("tc-large")
    xs = inputs([K], T, rng)
    xs[0][:, 3] *= 3.0e5
    xs[0][:, 40] *= 5.0e5
    p = problem("Q5_0", M, K, T, rng, epi=kr.EPI_ADD)
    p["res"] *= 1e4
    outs, launches = run_batch(lib, T, [p], xs, "tensor_cores")
    assert launches[-1][5] > 1 and kr.tc_column_scale(xs[0])[[3, 40]].min() > 0, launches
    check_all("tc-large", T, [p], xs, "tensor_cores", outs, launches)


# ---- every compiled instantiation was launched above ------------------------------------------------------------------------

def library_instantiations(path):
    """launch_key of every matrix-kernel symbol in the library (cuobjdump)."""
    r = subprocess.run(["cuobjdump", "--dump-resource-usage", path], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    keys = set()
    for name in re.findall(r"Function ([^:\s]+):", r.stdout):
        if m := re.search(r"gemv_tma_kernelILi(\d+)ELi(n?\d+)ELb([01])EE", name):
            keys.add(("streaming", int(m[1]), int(m[2].replace("n", "-")), int(m[3])))
        elif m := re.search(r"gemv_kernelILi(\d+)EE", name):
            keys.add(("generic", int(m[1])))
        elif m := re.search(r"gemm_tc_kernelILi(\d+)EE", name):
            keys.add(("tensor_cores", int(m[1])))
        elif "convert_f16_kernel" in name:
            keys.add(("convert",))
        elif m := re.search(r"tc_expand_kernelILi(\d+)EE", name):
            keys.add(("expand", int(m[1])))
    return keys


def test_every_compiled_instantiation_was_launched(lib):
    """Runs after the tests above: each gemv_tma_kernel, gemv_kernel, gemm_tc_kernel, convert_f16_kernel and tc_expand_kernel in the
    library was launched by one of them (per the launch record), with cluster sizes 1 / 2 / 4 / 8 and 1 .. 8 converted inputs. A new
    instantiation fails here until a test reaches it."""
    compiled = library_instantiations(lib.path)
    assert len(compiled) >= 7 * 2 + 3 + 3 + 16 + 1 + 6, sorted(compiled)
    assert compiled <= LAUNCHED, sorted(compiled - LAUNCHED)
    assert CLUSTERS >= {1, 2, 4, 8} and CONVERT_INPUTS >= set(range(1, 9)), (CLUSTERS, CONVERT_INPUTS)
