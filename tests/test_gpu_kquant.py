"""Q4_K / Q5_K on the GPU: the K-quant streaming GEMV against its float64 restatement, and whole models against the compiled
reference's golden logits (tests/golden/make_kquant_ref.py) and the engine's own bit-for-bit invariants."""
import ctypes

import numpy as np
import pytest

import kernel_ref as kref
import kquant_ref as kr

pytestmark = pytest.mark.gpu
PF = ctypes.POINTER(ctypes.c_float)
G = kr.golden()
# shapes: multiples of 256 of the streaming tests' set, and the 7B projections (K = 14336 splits a row over 4 warps)
SHAPES = [(256, 64), (1024, 300), (2048, 1000), (4096, 4096), (4096, 14336), (14336, 4096),
          (20480, 256), (40960, 128)]      # RWKV-4 14B's ffn.value (one CTA per SM with the wide budget), and rows near 40k


def matvec(lib, tid, raw, M, K, x):
    T = x.shape[1]
    y = np.full((T, M), np.nan, np.float32)
    xc = np.ascontiguousarray(x.T, dtype=np.float32)
    assert lib.library.rwkv_b200_matvec(tid, K, M, T, raw.ctypes.data, xc.ctypes.data_as(PF), y.ctypes.data_as(PF), 0)
    return y.T


@pytest.mark.parametrize("fmt", ["Q4_K", "Q5_K"])
@pytest.mark.parametrize("K,M", SHAPES)
def test_gemv_against_float64(lib, fmt, K, M):
    tid = kr.TYPE_ID[fmt]
    rng = np.random.default_rng(K * 7 + M + tid)
    raw = kr.random_blocks(tid, M, K, rng)
    T = 5                                               # NC = 4 then 1 up to K = 2048, NC = 2 at K = 4096, NC = 1 from K = 14336
    x = rng.standard_normal((K, T)).astype(np.float32)
    x[:256, 1] = 0.0                                    # an all-zero super-block (d = 0)
    y = matvec(lib, tid, raw, M, K, x)
    assert np.isfinite(y).all()
    for t in range(T):
        want = kr.gemv64(tid, raw, M, K, x[:, t])
        scale = np.abs(want).max() + 1e-30
        assert np.abs(y[:, t] - want).max() <= 2e-5 * scale * np.sqrt(K / 256), (t, np.abs(y[:, t] - want).max(), scale)
    # the arithmetic of a column does not depend on T / NC: each column alone gives the same bits
    for t in (0, 4):
        assert np.array_equal(matvec(lib, tid, raw, M, K, x[:, t:t + 1])[:, 0], y[:, t])
    assert np.array_equal(matvec(lib, tid, raw, M, K, x[:, :2]), y[:, :2])


@pytest.fixture(scope="module")
def models(pkg, lib, tmp_path_factory):
    tmp = tmp_path_factory.mktemp("kq_models")
    cache = {}

    def get(key):
        if key not in cache:
            name, fmt = key.split(":")
            master = tmp / (name + ".bin")
            if not master.exists():
                kr.write_master(master, G["presets"][name], G["seed"])
            path = tmp / ("%s-%s.bin" % (name, fmt))
            lib.rwkv_quantize_model_file(str(master), str(path), fmt)
            cache[key] = pkg.RWKVModel(lib, str(path), thread_count=1)
        return cache[key]
    yield get
    for m in cache.values():
        m.free()


def tokens(name):
    V = G["presets"][name]["V"]
    return [(7919 * i + 11) % V for i in range(G["prompt_len"])]


def _other(key):
    name, fmt = key.split(":")
    return name + ":" + ("Q5_K" if fmt == "Q4_K" else "Q4_K")


@pytest.mark.parametrize("key", sorted(G["sha256"]))
def test_model_against_reference(models, key):
    m = models(key)
    toks = tokens(key.split(":")[0])
    ref = np.load(kr.GOLDEN + "/kquant_ref.npz")
    want, other = ref[key], ref[_other(key)]
    # The bar: a quarter of the distance between the reference's Q4_K and Q5_K logits of the same master, so that a model that ran
    # the other format's arithmetic (or a wrong Q8_K rounding / scale unpacking, which moves logits by as much) cannot pass.
    tol = 0.25 * np.abs(want - other).max()
    # 40 tokens in one pass: the tensor cores; serial and chunks of 32 and 7
    seq, seq_state = m.eval_sequence(toks, None, use_numpy=True)
    assert np.isfinite(seq).all() and np.isfinite(seq_state).all()
    st = None
    for t in toks:
        sl, st = m.eval(t, st, use_numpy=True)
    errs = {"sequence": np.abs(seq - want).max(), "serial": np.abs(sl - want).max()}
    st32 = None
    for c in range(0, len(toks), 32):
        c32, st32 = m.eval_sequence(toks[c:c + 32], st32, use_numpy=True)
    errs["chunks32"] = np.abs(c32 - want).max()
    assert max(errs.values()) < tol, (errs, tol)
    # below 32 tokens a pass never takes the tensor cores: serial == chunks, bit for bit
    st2 = None
    for c in range(0, len(toks), 7):
        cl, st2 = m.eval_sequence(toks[c:c + 7], st2, use_numpy=True)
    assert np.array_equal(cl, sl) and np.array_equal(st2, st)


def _xs(rng, K, T):
    return rng.standard_normal((K, T)).astype(np.float32)


@pytest.mark.parametrize("fmt", ["Q4_K", "Q5_K"])
def test_router_splits_mixed_batches_bit_exactly(lib, fmt):
    """A K-quant problem inside a batch with a legacy problem on the same input: one launch each (families 5 and 0), and each output
    is the bits of the problem run alone."""
    rng = np.random.default_rng(3)
    K, M, T = 1024, 512, 3
    tid = kr.TYPE_ID[fmt]
    kq = dict(type=tid, K=K, M=M, raw=kr.random_blocks(tid, M, K, rng), input=0)
    q51 = dict(type=8, K=K, M=256, raw=rng.integers(0, 256, 256 * (K // 32) * 24, dtype=np.uint8), input=0)
    q51["raw"].reshape(-1, 24)[:, 0:2] = np.array([0.01], np.float16).view(np.uint8)
    q51["raw"].reshape(-1, 24)[:, 2:4] = np.array([-0.1], np.float16).view(np.uint8)
    x = _xs(rng, K, T)
    both, launches = kr.gemv_batch(lib, T, [q51, kq], [x])
    assert sorted(f for f, *_ in launches) == [0, 5], launches
    alone, la = kr.gemv_batch(lib, T, [kq], [x])
    assert [(f, o) for f, _, o, *_ in la] == [(5, tid)]
    assert np.array_equal(both[1].value, alone[0].value)
    assert both[0].guard_intact() and both[1].guard_intact()
    assert np.array_equal(both[0].value, kr.gemv_batch(lib, T, [q51], [x])[0][0].value)


@pytest.mark.parametrize("fmt", ["Q4_K", "Q5_K"])
@pytest.mark.parametrize("epi", [kref.EPI_SIGMOID, kref.EPI_SILU, kref.EPI_TANH, kref.EPI_RELU_SQR, kref.EPI_ADD, kref.EPI_BIAS_SIGMOID,
                                 kref.EPI_BIAS_EXPNEGEXP, kref.EPI_BIAS_W7])
def test_epilogues(lib, fmt, epi):
    rng = np.random.default_rng(epi)
    K, M, T = 2048, 300, 2
    tid = kr.TYPE_ID[fmt]
    p = dict(type=tid, K=K, M=M, raw=kr.random_blocks(tid, M, K, rng), input=0, epi=epi)
    if epi == kref.EPI_ADD:
        p["res"] = rng.standard_normal((M, T)).astype(np.float32)
    if epi >= kref.EPI_BIAS_EXPNEGEXP:
        p["bias"] = (0.1 * rng.standard_normal(M)).astype(np.float32)
    x = _xs(rng, K, T)
    (out,), launches = kr.gemv_batch(lib, T, [p], [x], path="streaming")
    assert [f for f, *_ in launches] == [5] and out.guard_intact()
    got = out.cols(M)
    assert not np.isnan(got).any()
    v = np.stack([kr.gemv64(tid, p["raw"], M, K, x[:, t]) for t in range(T)], axis=1)
    want = kref.epilogue(v, epi, np.float64, p.get("res"), None, p.get("bias"))
    assert np.abs(got - want).max() <= 1e-5 * (np.abs(want).max() + 1)


@pytest.mark.parametrize("fmt", ["Q4_K", "Q5_K"])
@pytest.mark.parametrize("T", [16, 40, 64, 128])
def test_tensor_cores(lib, fmt, T):
    """The expansion (family 6) and the Q8_K operand (a convert launch with only = 16) against the float64 restatement, at the bar of
    the existing tensor-core tests; a legacy problem on the same input takes the fp16 conversion of its own kind."""
    rng = np.random.default_rng(T)
    tid = kr.TYPE_ID[fmt]
    K, M = 4096, 512                                     # 4 row tiles: the launch splits K over clusters
    p = dict(type=tid, K=K, M=M, raw=kr.random_blocks(tid, M, K, rng), input=0, tiled=1)
    f16 = dict(type=1, K=K, M=128, raw=(0.02 * rng.standard_normal((128, K))).astype(np.float16).view(np.uint8).reshape(-1), input=0, tiled=1)
    x = _xs(rng, K, T)
    outs, launches = kr.gemv_batch(lib, T, [p, f16], [x], path="tensor_cores")
    fams = [(f, o) for f, _, o, *_ in launches]
    assert (6, tid) in fams and (3, 16) in fams and (3, 0) in fams and (2, 0) in fams, launches
    assert any(f == 2 and c > 1 for f, _, _, _, _, c in launches), launches
    got = outs[0].cols(M)
    r64, r32 = kr.gemm_tc(tid, p["raw"], M, K, x, np.float64), kr.gemm_tc(tid, p["raw"], M, K, x, np.float32)
    assert kref.error_over_bar(got, r64, r32, 64) <= 1
    assert outs[0].guard_intact() and outs[1].guard_intact()
