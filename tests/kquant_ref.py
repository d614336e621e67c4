"""Float64 restatement of the Q4_K / Q5_K matrix-vector product (ggml_vec_dot_q{4,5}_K_q8_K) and the helpers the K-quant tests share.

The activations are quantised to Q8_K exactly as quantize_row_q8_K_ref does (ggml-quants.c:2479), so the integers match the kernel's;
only the float combination of the super-blocks is done in float64 here.
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, GOLDEN)

F32 = np.float32
TYPE_ID = {"Q4_K": 13, "Q5_K": 14}
BLOCK_BYTES = {13: 144, 14: 176}


def golden():
    with open(os.path.join(GOLDEN, "kquant_ref.json")) as f:
        return json.load(f)


def write_master(path, preset, seed):
    import synthetic_model as sm
    return sm.write_master(str(path), dict(preset, arch=tuple(preset["arch"])), "FP16", seed=seed)


def unpack(tid, raw, M, K):
    """-> d, dmin float64[M, nsb]; sc, mn int64[M, nsb, 8]; q int64[M, nsb, 8, 32] (levels 0..15 / 0..31)."""
    nsb = K // 256
    b = np.frombuffer(np.ascontiguousarray(raw).tobytes(), np.uint8).reshape(M, nsb, BLOCK_BYTES[tid])
    d = b[:, :, 0:2].copy().view(np.float16)[..., 0].astype(np.float64)
    dmin = b[:, :, 2:4].copy().view(np.float16)[..., 0].astype(np.float64)
    s = b[:, :, 4:16].astype(np.int64)
    sc, mn = np.zeros((M, nsb, 8), np.int64), np.zeros((M, nsb, 8), np.int64)
    for j in range(8):
        if j < 4:
            sc[..., j], mn[..., j] = s[..., j] & 63, s[..., j + 4] & 63
        else:
            sc[..., j] = (s[..., j + 4] & 0xF) | ((s[..., j - 4] >> 6) << 4)
            mn[..., j] = (s[..., j + 4] >> 4) | ((s[..., j] >> 6) << 4)
    qs = b[:, :, (48 if tid == 14 else 16):].astype(np.int64).reshape(M, nsb, 4, 32)
    q = np.zeros((M, nsb, 8, 32), np.int64)
    for j in range(8):
        q[:, :, j] = (qs[:, :, j // 2] >> (4 * (j & 1))) & 0xF
        if tid == 14:
            q[:, :, j] |= ((b[:, :, 16:48].astype(np.int64) >> j) & 1) << 4
    return d, dmin, sc, mn, q


def quantize_q8k(x):
    """x float32[K] -> (d float32[nsb], qs int64[nsb, 256], bsums int64[nsb, 16]), quantize_row_q8_K_ref."""
    xb = np.asarray(x, F32).reshape(-1, 256)
    nsb = xb.shape[0]
    idx = np.argmax(np.abs(xb), axis=1)                 # first maximum: `if (ax > amax)`
    mx = xb[np.arange(nsb), idx]
    d = np.zeros(nsb, F32)
    qs = np.zeros((nsb, 256), np.int64)
    live = mx != 0
    iscale = np.where(live, F32(-127.0) / np.where(live, mx, F32(1)), F32(0)).astype(F32)
    v = (iscale[:, None] * xb).astype(F32)
    qs[live] = np.minimum(127, np.rint(v[live]).astype(np.int64))
    d[live] = (F32(1.0) / iscale[live]).astype(F32)
    return d, qs, qs.reshape(nsb, 16, 16).sum(axis=2)


def gemv64(tid, raw, M, K, x):
    """float64[M]: sum over super-blocks of y.d*d*sum(sc*dot) - y.d*dmin*sum(mn*bsum pairs), integers exact."""
    d, dmin, sc, mn, q = unpack(tid, raw, M, K)
    yd, qs, bs = quantize_q8k(x)
    dots = np.einsum("msjl,sjl->msj", q, qs.reshape(-1, 8, 32))
    isum = (dots * sc).sum(axis=2)
    msum = (mn * (bs[:, 0::2] + bs[:, 1::2])[None]).sum(axis=2)
    yd = yd.astype(np.float64)[None]
    return (yd * d * isum - yd * dmin * msum).sum(axis=1)


def random_blocks(tid, M, K, rng):
    """Random super-blocks with fp16 scales of a typical magnitude (weights of std ~ 1/sqrt(K))."""
    nsb = K // 256
    b = rng.integers(0, 256, size=(M, nsb, BLOCK_BYTES[tid]), dtype=np.uint8)
    lev = 15 if tid == 13 else 31
    d = (F32(2.0 / np.sqrt(K)) / (lev * 32) * rng.uniform(0.5, 1.5, (M, nsb))).astype(np.float16)
    dmin = (F32(1.0 / np.sqrt(K)) / 32 * rng.uniform(0.5, 1.5, (M, nsb))).astype(np.float16)
    b[:, :, 0:2] = d.view(np.uint8).reshape(M, nsb, 2)
    b[:, :, 2:4] = dmin.view(np.uint8).reshape(M, nsb, 2)
    return b.reshape(-1)


def dequant_f16(tid, raw, M, K):
    """The tensor-core A operand: fp16(d*sc*q - dmin*m), one rounding (tc_expand_kq_kernel)."""
    d, dmin, sc, mn, q = unpack(tid, raw, M, K)
    w = (d[..., None] * sc)[..., None] * q - (dmin[..., None] * mn)[..., None]
    return w.reshape(M, K).astype(np.float16)


def tc_operand(x):
    """The tensor-core B operand of K-quant weights: fp16(q * d 2^-e) of the Q8_K blocks of every column, and e (convert_q8k_kernel)."""
    x = np.asarray(x, F32)
    K, T = x.shape
    cmax = np.abs(x).max(axis=0)
    e = np.where((cmax > 32768) & (cmax <= 3.0e38), np.frexp(cmax)[1] - 15, 0).astype(np.int32)
    B = np.empty((K, T), np.float16)
    for t in range(T):
        d, qs, _ = quantize_q8k(x[:, t])
        dd = (d * np.ldexp(F32(1), -int(e[t]))).astype(F32)
        B[:, t] = (qs.astype(F32) * dd[:, None]).reshape(-1).astype(np.float16)
    return B, e


def gemm_tc(tid, raw, M, K, x, dt):
    """A . B accumulated in dt, times 2^e per column."""
    B, e = tc_operand(x)
    y = dequant_f16(tid, raw, M, K).astype(dt) @ B.astype(dt)
    return y * np.ldexp(dt(1), e)[None, :].astype(dt)


def gemv_batch(lib, T, problems, xs, path="engine"):
    """rwkv_b200_test_gemv_batch as kernel_hooks.gemv_batch, with the launch families as numbers (5: K-quant GEMV, 6: K-quant
    expansion). Returns (one Out of M*T floats per problem, launches as (family, nc, only, has_ln, npad, cluster) tuples)."""
    import ctypes
    import kernel_hooks as kh
    i = kh.Inputs()
    a = kh.GemvBatchArgs(T=T, n=len(problems), path=kh.GEMV_PATHS[path])
    for j, x in enumerate(xs):
        a.x[j] = i(x, True)
    outs = []
    for j, p in enumerate(problems):
        raw = np.ascontiguousarray(p["raw"])
        i.keep.append(raw)
        q = a.p[j]
        q.type, q.K, q.M, q.weights = p["type"], p["K"], p["M"], raw.ctypes.data
        q.tiled, q.input, q.epi = int(p.get("tiled", 0)), p.get("input", 0), p.get("epi", 0)
        q.res, q.bias = i(p.get("res"), True), i(p.get("bias"))
        q.y_aliases_res = int(p.get("alias", 0))
        outs.append(kh.Out(p["M"] * T))
        q.y = outs[-1].ptr
    rec = (kh.GemvLaunch * 32)()
    n_rec = ctypes.c_int(0)
    a.launches, a.max_launches, a.n_launches = rec, 32, ctypes.pointer(n_rec)
    kh._call(lib, lib.library.rwkv_b200_test_gemv_batch, a)
    return outs, [(r.family, r.nc, r.only, r.has_ln, r.npad, r.cluster) for r in rec[:n_rec.value]]
