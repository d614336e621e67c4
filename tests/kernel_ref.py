"""Plain restatements of the eval path's element-wise and recurrent kernels (csrc/kernels/glue.cu, wkv.cu), one function
per operation, written from the reference's formulas and generic in the floating-point type: in float64 they give the truth, in
float32 they show how far a faithful fp32 implementation lands from it on the same input. tests/test_gpu_kernels.py compares the
kernels with both; tests/test_kernel_bars.py checks that plausible bugs move the results far beyond the bars derived from them.

Activations are column-major [dim, T] as in the engine. `bug` selects one deliberate mistake (see test_kernel_bars.py); None is the
correct operation."""
import numpy as np

import ggml_file as gf
import rwkv_oracle as ro

F64 = np.float64


def bar(r64, r32, factor=4):
    """How far a kernel output may land from the float64 result r64: `factor` (four) times the distance of the float32 restatement
    r32, but at least 1e-6 of the output's largest magnitude. For [dim, T] activations each token column has its own bar, so one
    ill-conditioned column (a constant one, say, whose variance fp32 cannot resolve) does not widen the bar of the others."""
    r64, r32 = np.asarray(r64, np.float64), np.asarray(r32, np.float64)
    return np.maximum(factor * np.abs(r32 - r64).max(axis=0), max(1e-6 * np.abs(r64).max(), 1e-30))


def error_over_bar(x, r64, r32, factor=4):
    """The largest ratio of |x - r64| to the bar over the output's columns."""
    return float((np.abs(np.asarray(x, np.float64) - np.asarray(r64, np.float64)).max(axis=0) / bar(r64, r32, factor)).max())


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


def layer_norm_columns(x, w, b, dt, bug=None):
    """layer_norm_columns_kernel (csrc/kernels/score.cu): layer_norm of every column of x [C, T], the head's LayerNorm of a scoring
    pass on the tensor cores. bug: "eps" (1e-6 instead of 1e-5), "wb_neighbour" (w and b of the next channel), "no_bias", "no_mean"
    (the mean not subtracted), "var_c_minus_1" (the variance divided by C - 1)."""
    if bug is None:
        return layer_norm(x, w, b, dt)
    x, w, b = x.astype(dt), w.astype(dt), b.astype(dt)
    n = dt(x.shape[0])
    v = x if bug == "no_mean" else x - x.sum(axis=0, dtype=dt) / n
    var = (v * v).sum(axis=0, dtype=dt) / (n - 1 if bug == "var_c_minus_1" else n)
    if bug == "wb_neighbour":
        w, b = np.roll(w, -1), np.roll(b, -1)
    y = v / np.sqrt(var + dt(1e-6 if bug == "eps" else 1e-5)) * w[:, None]
    return y if bug == "no_bias" else y + b[:, None]


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


# ---- matrix kernels (csrc/kernels/gemv.cu, gemv_tma.cu, gemm_tc.cu) ----------------------------------------------------
# y[M, T] = epi(W[M, K] . pro(x[K, T])). The decode GEMV multiplies the reference's own operands (ggml-cpu.c:253-311 vec_dot_type);
# the tensor-core GEMM multiplies fp16 roundings of them. Both restatements take the exact operand values and accumulate in `dt`.

EPI_NONE, EPI_SIGMOID, EPI_SILU, EPI_TANH, EPI_RELU_SQR, EPI_ADD, EPI_MUL_ADD, EPI_BIAS_EXPNEGEXP, EPI_BIAS_SIGMOID, EPI_BIAS_W7 = range(10)
RES_EPIS, BIAS_EPIS = (EPI_ADD, EPI_MUL_ADD), (EPI_BIAS_EXPNEGEXP, EPI_BIAS_SIGMOID, EPI_BIAS_W7)
ROW_CHUNK = 4096          # rows restated at a time: bounds the memory of a 65536-row head


def weight_operands(w_type, raw, M, K):
    """The stored weights: dense [M, K] values for F32 / F16, else the blocks (q - offset [M, K/32, 32], d [M, K/32], m or None)
    of dequantize_row_q* (ggml-quants.c:255-363; ro.unpack_blocks)."""
    if w_type in (TYPE_F32, TYPE_F16):
        return ro.dequantize(w_type, raw, M * K).reshape(M, K)
    q, d, m, off = ro.unpack_blocks(w_type, raw, M * K)
    nb = K // 32
    return (q - off).reshape(M, nb, 32), d.reshape(M, nb), None if m is None else m.reshape(M, nb)


def act_operands(w_type, x, bug=None):
    """The activation operands the decode GEMV multiplies with weights of w_type, from the fp32 values x [K, T]: x for F32 (in the
    dtype given), fp16(x) for F16, else Q8 blocks (q [K/32, 32, T], d = fp16(amax / 127), s) as quantize_row_q8_0 / q8_1 make them
    (ggml-cpu-quants.c:781-846, 1085-1160; ro.quantize_activations). s is sum(q) for the *_0 formats (it folds their offset) and
    fp16(d32 * sum(q)) for Q4_1 / Q5_1: the block minimum multiplies the ROUNDED s."""
    if w_type == TYPE_F32:
        return x
    if w_type == TYPE_F16:
        return np.asarray(x, np.float32).astype(np.float16)
    has_min = w_type in Q8_1_CONSUMERS
    x32 = np.asarray(x, np.float32)
    q, d, s = ro.quantize_activations(x32, with_sum=has_min)
    if has_min and bug == "s_unrounded":
        amax = np.abs(x32.reshape(q.shape)).max(axis=1)
        s = (amax / np.float32(127)) * q.sum(axis=1).astype(np.float32)
    if not has_min:
        s = q.sum(axis=1).astype(np.float32)
    return q, d, s


def row_chunks(w_type, raw, M, K):
    """(r0, r1, weight_operands of rows r0..r1) over the matrix, ROW_CHUNK rows at a time."""
    elems, nbytes = gf.BLOCK[w_type]
    row = K // elems * nbytes
    raw = np.ascontiguousarray(raw).reshape(-1)
    for r0 in range(0, M, ROW_CHUNK):
        r1 = min(M, r0 + ROW_CHUNK)
        yield r0, r1, weight_operands(w_type, raw[r0 * row:r1 * row], r1 - r0, K)


def gemv_operands(w_type, raw, x, M, bug=None):
    """(weight operands, activation operands) of the decode GEMV."""
    return weight_operands(w_type, raw, M, x.shape[0]), act_operands(w_type, x, bug)


def epilogue(v, epi, dt, res=None, gate=None, bias=None, bug=None):
    """The fused epilogues of GemvEpilogue (csrc/kernels/gemv.h), per the reference's graph (rwkv_graph.inc:365-367, 417-430,
    445-450, 667-679). v, res, gate: [M, T]; bias: [M]."""
    if res is not None:
        res = res.astype(dt)
        if bug == "res_neighbour":
            res = np.roll(res, 1, axis=0)
    if gate is not None:
        gate = gate.astype(dt)
        if bug == "gate_prev_col":
            gate = np.roll(gate, 1, axis=1)
    if bias is not None:
        bias = bias.astype(dt)[:, None]
        if bug == "bias_next":
            bias = np.roll(bias, -1, axis=0)
    one = dt(1)
    sig = lambda z: one / (one + np.exp(-z))
    with np.errstate(over="ignore", under="ignore"):
        if epi == EPI_SIGMOID:
            return sig(v)
        if epi == EPI_SILU:
            return v / (one + np.exp(-v))
        if epi == EPI_TANH:
            return np.tanh(v)
        if epi == EPI_RELU_SQR:
            return np.maximum(v, dt(0)) ** 2
        if epi == EPI_ADD:
            return res + v
        if epi == EPI_MUL_ADD:
            return res + gate * v
        if epi == EPI_BIAS_EXPNEGEXP:
            return np.exp(-np.exp(v + bias))
        if epi == EPI_BIAS_SIGMOID:
            return sig(v + bias)
        if epi == EPI_BIAS_W7:
            return np.exp(sig(v + bias) * dt(-0.606531))
    return v


def prologue(x, ln, dt, bug=None):
    """The head's LayerNorm prologue (PRO_LAYERNORM: rwkv_layer_norm, rwkv_operators.inc:93-97) or x itself. ln: (w, b) or None."""
    if ln is None:
        return np.asarray(x, np.float32)
    w, b = ln
    if bug == "ln_no_b":
        b = np.zeros_like(b)
    return layer_norm(x, w, b, dt, eps=1e-6 if bug == "ln_eps" else 1e-5)


def gemv(w_type, raw, M, x, dt, epi=EPI_NONE, res=None, gate=None, bias=None, ln=None, bug=None):
    """The decode GEMV (gemv_tma_kernel, gemv_kernel): sum over blocks of d_w d_a sum(q_w q_a) + m_w s_a (ggml-cpu-quants.c:2302-2316,
    2594-2609, 2944-2963, 3318-3338, 3690-3698), fp16(x) . W for F16 (ggml-cpu.c:1463), plain for F32; then the epilogue. x: [K, T]
    fp32; with `ln` the LayerNorm output in dt is what gets quantised (the tests choose ln_b so that fp32 and float64 give the same
    operands). Accumulated in dt."""
    xin = prologue(x, ln, dt, bug)
    K, T = xin.shape
    A = act_operands(w_type, xin.astype(dt) if w_type == TYPE_F32 else xin, bug)
    y = np.empty((M, T), dt)
    for r0, r1, W in row_chunks(w_type, raw, M, K):
        if w_type in (TYPE_F32, TYPE_F16):
            y[r0:r1] = W.astype(dt) @ A.astype(dt)
            continue
        qw, dw, mw = W
        qa, da, sa = A
        nb = qw.shape[1]
        if bug == "drop_odd_block" and nb % 2:
            nb -= 1
        # exact integer block sums, [nb, rows, T]
        isum = np.matmul(qw[:, :nb].transpose(1, 0, 2).astype(F64), qa[:nb].astype(F64))
        part = (dw[:, :nb].T.astype(dt)[:, :, None] * da[:nb].astype(dt)[:, None, :]) * isum.astype(dt)
        if mw is not None and bug != "drop_min":
            part = part + mw[:, :nb].T.astype(dt)[:, :, None] * sa[:nb].astype(dt)[:, None, :]
        y[r0:r1] = np.moveaxis(part, 0, -1).sum(axis=-1, dtype=dt)
    return epilogue(y, epi, dt, res, gate, bias, bug)


def tc_column_scale(x):
    """e per token column (convert_f16_kernel): the column is multiplied by 2^-e before the fp16 rounding so that it stays inside the
    fp16 range, e = exponent(column maximum) - 15 above 32768, else 0."""
    cmax = np.abs(np.asarray(x, np.float32)).max(axis=0)
    e = np.where((cmax > 32768) & (cmax <= 3.0e38), np.frexp(cmax)[1] - 15, 0)
    return e.astype(np.int32)


def tc_weights(w_type, W):
    """A = fp16((q - offset) d + m) rounded ONCE (the kernel's __hfma2: the product and the sum are exact in float64, so float64 ->
    float16 is that single rounding), or the stored fp16 weights. W: weight_operands of some rows."""
    if w_type == TYPE_F16:
        return W.astype(np.float16)
    qw, dw, mw = W
    a = qw.astype(F64) * dw.astype(F64)[:, :, None]
    if mw is not None:
        a = a + mw.astype(F64)[:, :, None]
    return a.reshape(qw.shape[0], -1).astype(np.float16)


def tc_activations(w_type, x):
    """B = fp16(d q 2^-e) of the Q8 block values for quantised weights, fp16(x 2^-e) for F16 (convert_f16_kernel), and e [T]."""
    e = tc_column_scale(x)
    down = np.ldexp(np.float32(1), -e).astype(np.float32)
    if w_type == TYPE_F16:
        return (np.asarray(x, np.float32) * down).astype(np.float16), e
    q, d, _ = ro.quantize_activations(np.asarray(x, np.float32), with_sum=False)
    return (q.astype(np.float32) * (d * down)[:, None, :]).reshape(x.shape[0], -1).astype(np.float16), e


def gemm_tc(w_type, raw, M, x, dt, epi=EPI_NONE, res=None, gate=None, bias=None, bug=None, ksplit=1):
    """The tensor-core GEMM (gemm_tc_kernel): A . B accumulated in dt, times 2^e per column, then the epilogue. ksplit: the K-split
    count of the launch, only used by the "drop_last_ksplit" bug."""
    K = x.shape[0]
    B, e = tc_activations(w_type, x)
    k1 = K
    if bug == "drop_last_ksplit" and ksplit > 1:
        per = -(-(K // 64) // ksplit)
        k1 = (ksplit - 1) * per * 64
    y = np.empty((M, x.shape[1]), dt)
    for r0, r1, W in row_chunks(w_type, raw, M, K):
        y[r0:r1] = tc_weights(w_type, W)[:, :k1].astype(dt) @ B[:k1].astype(dt)
    if bug == "drop_last_tile":
        y[(M - 1) // 128 * 128:] = 0
    if bug != "no_colscale":
        y = y * np.ldexp(dt(1), e)[None, :].astype(dt)
    return epilogue(y, epi, dt, res, gate, bias, bug)


def _f16_tie_distance(v):
    """Distance of |v| from the nearest half-way point between two fp16 values, in units of the fp16 spacing there."""
    a = np.abs(np.asarray(v, F64))
    h = a.astype(np.float16)
    up = np.spacing(h).astype(F64)
    down = (h - np.nextafter(h, np.float16(0))).astype(F64)
    hd = h.astype(F64)
    dist = np.minimum(np.abs(a - (hd + up / 2)), np.abs(a - (hd - down / 2)))
    return dist / np.where(up > 0, up, 1.0)


def ln_columns_f32(x, w):
    """(x - mean) * rstd * w of layer_norm_columns_kernel (and of the GEMV's LayerNorm prologue) in float32, before the bias: the mean
    and the sum of squares in double, everything else one float32 rounding per operation in the kernel's order."""
    x = np.asarray(x, np.float32)
    C = x.shape[0]
    mean = (x.astype(F64).sum(axis=0) / C).astype(np.float32)
    v = x - mean
    s2 = (v * v).astype(F64).sum(axis=0)
    rstd = np.float32(1) / np.sqrt((s2 / C).astype(np.float32) + np.float32(1e-5))
    return (v * rstd) * np.asarray(w, np.float32)[:, None]


def ln_bias_away_from_roundings(x, ln_w, ln_b, w_type, rng, margin=1e-3, tie_margin=1e-2, kernel_error=False):
    """ln_b nudged element by element until the float64 LayerNorm output of x gives the same operands as any faithful fp32 LayerNorm:
    every Q8 value x 127 / amax at least `margin` (in units of q) away from a rint half-way point, and every block's amax / 127, every
    Q8_1 s and every fp16 operand at least `tie_margin` of an fp16 spacing away from an fp16 tie. ln_b enters after the normalisation,
    element by element, so moving ln_b[k] moves row k of the output and nothing else.

    With kernel_error, an fp16 operand is instead held four times its distance from the LayerNorm of the kernels (ln_columns_f32 + ln_b in
    float32 numpy) away from a tie: a margin that a single ln_b[k] can keep for all of a row's 256 columns at once, where tie_margin is
    out of reach for more than about 64. Operands below 2^-8 are left where they fall: their fp16 spacing is at most 2^-19, so another
    rounding of one moves a product with a head weight by less than the bar's floor of 1e-6 of the output."""
    b = np.asarray(ln_b, np.float32).copy()
    if w_type == TYPE_F32:
        return b
    n = norm(x, 1e-5, F64) * np.asarray(ln_w, F64)[:, None]
    K, T = n.shape
    if kernel_error:
        nw32 = ln_columns_f32(x, ln_w)
    for _ in range(200):
        y = n + b.astype(F64)[:, None]
        if w_type == TYPE_F16 and kernel_error:
            gap = _f16_tie_distance(y) * np.spacing(np.abs(y).astype(np.float16)).astype(F64)
            err = np.abs((nw32 + b[:, None]).astype(F64) - y) + 2.0 ** -24 * np.abs(y)
            bad = ((gap < 4 * err) & (np.abs(y) >= 2.0 ** -8)).any(axis=1)
            unit = np.abs(y).max(axis=1) * 2.0 ** -10 + 1e-8
        elif w_type == TYPE_F16:
            bad = (_f16_tie_distance(y) < tie_margin).any(axis=1)
            unit = np.abs(y).max(axis=1) * 2.0 ** -10 + 1e-8
        else:
            yb = y.reshape(K // 32, 32, T)
            amax = np.abs(yb).max(axis=1)                                             # [nb, T]
            qv = yb * 127 / np.where(amax > 0, amax, 1)[:, None, :]
            bad_el = np.abs(qv - np.floor(qv) - 0.5) < margin
            d32 = amax / 127
            bad_blk = _f16_tie_distance(d32) < tie_margin
            if w_type in Q8_1_CONSUMERS:
                bad_blk |= _f16_tie_distance(d32 * np.rint(qv).sum(axis=1)) < tie_margin
            # a bad block moves its largest element: that changes amax, d and s
            arg = np.abs(yb).argmax(axis=1)                                           # [nb, T]
            bad_el[np.nonzero(bad_blk)[0], arg[bad_blk], np.nonzero(bad_blk)[1]] = True
            bad = bad_el.reshape(K, T).any(axis=1)
            unit = np.repeat(amax.max(axis=1) / 127, 32)
        if not bad.any():
            return b
        b[bad] += (rng.uniform(0.05, 0.95, bad.sum()) * unit[bad]).astype(np.float32)
    raise AssertionError("could not move the LayerNorm output away from rounding boundaries")
