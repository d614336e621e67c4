"""Plain restatements of the eval path's element-wise and recurrent kernels (csrc/kernels/glue.cu, wkv.cu, batch.cu), one function
per operation, written from the reference's formulas and generic in the floating-point type: in float64 they give the truth, in
float32 they show how far a faithful fp32 implementation lands from it on the same input. tests/test_gpu_kernels.py compares the
kernels with both; tests/test_kernel_bars.py checks that plausible bugs move the results far beyond the bars derived from them.

Activations are column-major [dim, T] as in the engine. `bug` selects one deliberate mistake (see test_kernel_bars.py); None is the
correct operation."""
import numpy as np

import ggml_file as gf
import rwkv_oracle as ro


def bar(r64, r32):
    """How far a kernel output may land from the float64 result r64: four times the distance of the float32 restatement r32, but
    at least 1e-6 of the output's largest magnitude. For [dim, T] activations each token column has its own bar, so one
    ill-conditioned column (a constant one, say, whose variance fp32 cannot resolve) does not widen the bar of the others."""
    r64, r32 = np.asarray(r64, np.float64), np.asarray(r32, np.float64)
    return np.maximum(4 * np.abs(r32 - r64).max(axis=0), max(1e-6 * np.abs(r64).max(), 1e-30))


def error_over_bar(x, r64, r32):
    """The largest ratio of |x - r64| to the bar over the output's columns."""
    return float((np.abs(np.asarray(x, np.float64) - np.asarray(r64, np.float64)).max(axis=0) / bar(r64, r32)).max())


def norm(x, eps, dt):
    """ggml_norm over axis 0 (ggml_compute_forward_norm_f32, ggml-cpu.c:6880-6929): (x - mean) / sqrt(var + eps)."""
    x = x.astype(dt)
    n = dt(x.shape[0])
    mean = x.sum(axis=0, dtype=dt) / n
    v = x - mean
    var = (v * v).sum(axis=0, dtype=dt) / n
    return v / np.sqrt(var + dt(eps))


def layer_norm(x, w, b, dt, eps=1e-5):
    """rwkv_layer_norm (rwkv_operators.inc:93-97): ggml_norm(eps 1e-5) * w + b."""
    return norm(x, eps, dt) * w.astype(dt)[:, None] + b.astype(dt)[:, None]


def head_norm(y, H, eps, dt):
    """Per-head ggml_norm after the reshape to [S, H, T] (rwkv_graph.inc:281-284, 376-379)."""
    C, T = y.shape
    return norm(y.reshape(H, C // H, T).transpose(1, 0, 2), eps, dt).transpose(1, 0, 2).reshape(C, T)


def embed_ln0(emb, tokens, w, b, dt):
    """ggml_get_rows + ln0 (rwkv_graph.inc:655-658, 787-790). emb: [n_vocab, C] table values."""
    return layer_norm(np.asarray(emb)[np.asarray(tokens)].T, w, b, dt)


def ln_mix(x, w, b, state_in, coefs, formula, dt, bug=None):
    """LayerNorm + token shift (rwkv_carry_x, rwkv_graph.inc:56-82) + mixing. formula 0 (v4 / v5, :94-97): xx*m + (prev - prev*m);
    formula 1 (v6 / v7, :310-311, 406, 520-521, 538): (prev - xx)*m + xx. Returns (outs, xx, prev - xx, carry out)."""
    xx = layer_norm(x, w, b, dt)
    prev = np.concatenate([state_in.astype(dt)[:, None], xx[:, :-1]], axis=1)
    if bug == "shift":                  # token shift off by one: the previous token's LN(x) taken one column too late
        prev = np.concatenate([state_in.astype(dt)[:, None], prev[:, :-1]], axis=1) if x.shape[1] > 1 else xx
    outs = []
    for m in coefs:
        m = m.astype(dt)[:, None]
        outs.append(xx * m + (prev - prev * m) if formula == 0 else (prev - xx) * m + xx)
    return outs, xx, prev - xx, xx[:, -1].copy()


def v6_lerp(w2, z, xx, sx, maa, dt, bug=None):
    """v6 data-dependent lerp (rwkv_graph.inc:323-346): m_j = W2[j] . z_j, out_j = (m_j + maa_j) * sx + xx for j in w, k, v, r, g.
    w2: [5, C, mix]; z: [5*mix, T]; maa: [5, C]."""
    mix, T = w2.shape[2], z.shape[1]
    m = np.einsum("jcm,jmt->jct", w2.astype(dt), z.astype(dt).reshape(5, mix, T))
    outs = []
    for j in range(5):
        jm = (j + 1) % 5 if bug == "lerp_j" and j == 2 else j     # the v output built with the r coefficient
        outs.append((m[j] + maa[jm].astype(dt)[:, None]) * sx.astype(dt) + xx.astype(dt))
    return outs


def wkv4(k, v, r, tf, td, aa, bb, pp, dt, bug=None):
    """rwkv_att_wkv_v4 (rwkv_graph.inc:119-161) times r (:182, 195), with the aa / bb / pp carry. Returns (y, aa, bb, pp)."""
    k, v, r = (a.astype(dt) for a in (k, v, r))
    tf, td = tf.astype(dt), td.astype(dt)
    if bug == "tf_neighbour":
        tf = np.roll(tf, 1)
    aa, bb, pp = aa.astype(dt).copy(), bb.astype(dt).copy(), pp.astype(dt).copy()
    y = np.empty_like(k)
    with np.errstate(over="ignore", under="ignore"):
        for t in range(k.shape[1]):
            kt, vt = k[:, t], v[:, t]
            ww = tf + kt
            qq = np.maximum(pp, ww)
            e1, e2 = np.exp(pp - qq), np.exp(ww - qq)
            y[:, t] = r[:, t] * ((e1 * aa + e2 * vt) / (e1 * bb + e2))
            ww = pp + td
            qq = np.maximum(ww, kt)
            e1, e2 = np.exp(ww - qq), np.exp(kt - qq)
            aa, bb, pp = e1 * aa + e2 * vt, e1 * bb + e2, qq
    return y, aa, bb, pp


def wkv6(r, k, v, td, tf, state, lnx_w, lnx_b, g, eps, H, S, dt, bug=None):
    """WKV5 / 6 (ggml_compute_forward_rwkv_wkv6_f32, ggml-cpu.c:11803-11935) + head norm + ln_x + gate (rwkv_graph.inc:275-289,
    370-382). td: [C, T] per token (v6), [C] per channel (v5.2) or [H] per head (v5.1, ggml_repeat :262-267); tf: [C] or [H].
    state: [H, S(i, key), S(j, value)]. Per token: kv = k_i v_j, y_j = sum_i r_i (tf_i kv + S_ij), S_ij = S_ij td_i + kv.
    Returns (y, state_out)."""
    C, T = r.shape
    r, k, v = (a.astype(dt) for a in (r, k, v))
    td, tf = td.astype(dt), tf.astype(dt)
    if tf.shape[0] == H:
        tf = np.repeat(tf, S)
    if td.ndim == 1 and td.shape[0] == H:
        td = np.repeat(td, S)
    if bug == "eps":
        eps = 64e-5 if eps == 1e-5 else 1e-5
    if bug == "tf_neighbour":
        tf = np.roll(tf, 1)
    if bug == "per_head_decay":        # one decay per head (its first channel's) instead of one per channel
        td = np.repeat(td.reshape(H, S)[:, 0], S)
    n_run = T - T % 8 if bug == "drop_tail" and T % 8 else T
    st = state.astype(dt).reshape(H, S, S).copy()
    tfh = tf.reshape(H, S, 1)
    y = np.zeros((C, T), dt)
    for t in range(n_run):
        kh, vh, rh = k[:, t].reshape(H, S, 1), v[:, t].reshape(H, 1, S), r[:, t].reshape(H, S, 1)
        tdh = (td[:, t] if td.ndim == 2 else td).reshape(H, S, 1)
        kv = kh * vh
        y[:, t] = ((tfh * kv + st) * rh).sum(axis=1, dtype=dt).reshape(C)
        st = st * tdh + kv
    y = head_norm(y, H, eps, dt) * lnx_w.astype(dt)[:, None] + lnx_b.astype(dt)[:, None]
    if g is not None:
        y = y * g.astype(dt)
    return y, st.reshape(-1)


def wkv7(r, w, k, v, a, g, vgate, v_first, k_k, k_a, r_k, lnx_w, lnx_b, state, H, S, dt, bug=None):
    """v7 time mixing after the GEMVs (rwkv_att_v7, rwkv_graph.inc:432-479; rwkv_wkv_v7_impl, rwkv_operators_wkv_v7.inc:37-106):
    kk = l2norm_head(k * k_k) (rwkv_operators.inc:40-82, eps 1e-12); k += a*k*k_a - k*k_a; v += (v_first - v) * vgate (vgate given);
    S_ij = S_ij w_j + v_i k_j + (sum_l -kk_l S_il) kk_j a_j; y_i = sum_j S_ij r_j; head norm (eps 64e-5), ln_x;
    + v * sum_head(k r r_k); * g. state: [H, S(i, value), S(j, key)]. Returns (y, v used, state_out)."""
    C, T = r.shape
    r, w, k, v, a, g = (x.astype(dt) for x in (r, w, k, v, a, g))
    kk = (k * k_k.astype(dt)[:, None]).reshape(H, S, T)
    kk = (kk / np.maximum(np.sqrt((kk * kk).sum(axis=1, dtype=dt)), dt(1e-12))[:, None, :]).reshape(C, T)
    ka = k * k_a.astype(dt)[:, None]
    k = k + (a * ka - ka)
    if vgate is not None:
        v = v + (v_first.astype(dt) - v) * vgate.astype(dt)
    st = state.astype(dt).reshape(H, S, S).copy()
    y = np.zeros((C, T), dt)
    for t in range(T):
        rh, wh, kh, vh, kkh, ah = (x[:, t].reshape(H, S) for x in (r, w, k, v, kk, a))
        sa = (-kkh[:, None, :] * st).sum(axis=2, dtype=dt)
        st = st * wh[:, None, :] + vh[:, :, None] * kh[:, None, :] + sa[:, :, None] * (kkh * ah)[:, None, :]
        y[:, t] = (st * rh[:, None, :]).sum(axis=2, dtype=dt).reshape(C)
    y = head_norm(y, H, 64e-5, dt) * lnx_w.astype(dt)[:, None] + lnx_b.astype(dt)[:, None]
    rk = (k * r * r_k.astype(dt)[:, None]).reshape(H, S, T).sum(axis=1, dtype=dt)
    y = (y + (v.reshape(H, S, T) * rk[:, None, :]).reshape(C, T)) * g
    return y, v, st.reshape(-1)


# ---- staged activation columns (csrc/kernels/act_stage.cuh) ------------------------------------------------------------

TYPE_F32, TYPE_F16 = gf.TYPE_FP32, gf.TYPE_FP16
Q8_1_CONSUMERS = (gf.TYPE_Q4_1, gf.TYPE_Q5_1)


def staged_bytes(q_type, K):
    """act::bytes_per_column: fp32 / fp16 values, or Q8 blocks (pairs of them for the *_0 consumers) with an 8-byte scale each."""
    if q_type == TYPE_F32:
        n = 4 * K
    elif q_type == TYPE_F16:
        n = 2 * K
    else:
        nblk = K // 32
        n = (nblk if q_type in Q8_1_CONSUMERS else (nblk + 1) // 2 * 2) * 40
    return (n + 15) // 16 * 16


def staged_column(y, q_type, fill=0xFF, guard=0):
    """The bytes a producer kernel stages for consumers of weight type q_type from the fp32 vector y: what the reference's CPU path
    multiplies (ggml-cpu.c:253-311 vec_dot_type) -- fp32 for F32 weights, fp16 for F16, Q8_0 blocks for Q4_0 / Q5_0 / Q8_0, Q8_1
    blocks for Q4_1 / Q5_1 (quantize_activations: ggml-cpu-quants.c:781-846, 1085-1160) -- in the kernels' shared-memory layout:
    block b = u*UB + bi, half h at ((bi*2 + h)*nunits + u)*16, scale {d, s} at nunits*UB*32 + (bi*nunits + u)*8. Bytes no block
    owns (the pad block of an odd *_0 count, the 16-byte round-up) and `guard` bytes after the column keep `fill`."""
    y = np.asarray(y, np.float32).reshape(-1)
    K = y.size
    out = np.full(staged_bytes(q_type, K) + guard, fill, np.uint8)
    if q_type == TYPE_F32:
        out[:4 * K] = np.frombuffer(y.astype("<f4").tobytes(), np.uint8)
        return out
    if q_type == TYPE_F16:
        out[:2 * K] = np.frombuffer(y.astype("<f2").tobytes(), np.uint8)
        return out
    has_min = q_type in Q8_1_CONSUMERS
    q, d, s = ro.quantize_activations(y[:, None], with_sum=has_min)
    q, d = q[:, :, 0], d[:, 0]
    s = s[:, 0] if has_min else q.sum(axis=1).astype(np.float32)
    nblk = K // 32
    UB = 1 if has_min else 2
    nunits = (nblk + UB - 1) // UB
    for blk in range(nblk):
        u, bi = divmod(blk, UB)
        for h in range(2):
            o = ((bi * 2 + h) * nunits + u) * 16
            out[o:o + 16] = q[blk, 16 * h:16 * h + 16].astype(np.int8).view(np.uint8)
        o = nunits * UB * 32 + (bi * nunits + u) * 8
        out[o:o + 8] = np.frombuffer(np.array([d[blk], s[blk]], "<f4").tobytes(), np.uint8)
    return out
