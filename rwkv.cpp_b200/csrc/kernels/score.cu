// Scoring passes (rwkv_b200_score, rwkv_b200_batch_score_ragged): the LayerNorm of the head's input columns for the tensor-core head,
// and the log-probability of a caller-given target in every column of the head's output.
#include "ops.h"

#include <cmath>

namespace rwkv {

namespace {

constexpr int SCORE_THREADS = 256;
constexpr int SCORE_WARPS = SCORE_THREADS / 32;

// y[:, t] = LN(x[:, t]; w, b, eps 1e-5) with the arithmetic of the GEMV's PRO_LAYERNORM prologue (stage_column): mean and variance
// summed in double, the normalised value as __fadd_rn(__fmul_rn(__fmul_rn(v - mean, rstd), w), b). One CTA per column.
__global__ void __launch_bounds__(SCORE_THREADS) layer_norm_columns_kernel(const float * x, const float * w, const float * b, int C, float * y,
                                                                          TraceRec * trace) {
    trace_begin(trace);
    pdl_prologue();
    __shared__ double red[SCORE_WARPS + 1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float * xc = x + (size_t) blockIdx.x * C;
    float * yc = y + (size_t) blockIdx.x * C;
    double s = 0;
    for (int k = tid; k < C; k += SCORE_THREADS) s += (double) xc[k];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    if (tid == 0) { double t = 0; for (int i = 0; i < SCORE_WARPS; i++) t += red[i]; red[SCORE_WARPS] = t; }
    __syncthreads();
    const float mean = (float) (red[SCORE_WARPS] / C);
    double s2 = 0;
    for (int k = tid; k < C; k += SCORE_THREADS) { const float v = xc[k] - mean; s2 += (double) (v * v); }
    for (int o = 16; o > 0; o >>= 1) s2 += __shfl_xor_sync(0xffffffffu, s2, o);
    __syncthreads();
    if (lane == 0) red[warp] = s2;
    __syncthreads();
    if (tid == 0) { double t = 0; for (int i = 0; i < SCORE_WARPS; i++) t += red[i]; red[SCORE_WARPS] = t; }
    __syncthreads();
    const float rstd = 1.0f / sqrtf((float) (red[SCORE_WARPS] / C) + 1e-5f);
    for (int k = tid; k < C; k += SCORE_THREADS) yc[k] = __fadd_rn(__fmul_rn(__fmul_rn(xc[k] - mean, rstd), w[k]), b[k]);
    trace_end(trace);
}

// Column t of logits (n_vocab floats, n_vocab apart): lp = log_softmax(z)[target], greedy = target is the first index of max(z).
// The maximum is taken in float; sum exp(z - max) is summed in double, thread-strided and then over a fixed tree, so the order depends on
// n_vocab alone and a column gives the same bits whatever T, its index or the batch. A column with a NaN or +inf, or without a finite
// logit, gives NaN and greedy 0.
__global__ void __launch_bounds__(SCORE_THREADS) score_kernel(const ScoreParams p) {
    trace_begin(p.trace);
    pdl_prologue();
    const int t = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t target = p.targets[t];
    if (target == SCORE_NO_TARGET) { trace_end(p.trace); return; }     // the whole CTA leaves: no barrier below is reached
    const int V = p.n_vocab;
    const float * z = p.logits + (size_t) t * V;
    __shared__ float s_max[SCORE_WARPS];
    __shared__ int s_arg[SCORE_WARPS], s_bad[SCORE_WARPS];
    __shared__ double s_sum[SCORE_WARPS];
    // max, its first index, and whether the column holds a NaN / +inf (bad) or any finite value (bit 1)
    float mx = -INFINITY;
    int arg = V, flags = 0;
    for (int i = tid; i < V; i += SCORE_THREADS) {
        const float v = z[i];
        if (isnan(v) || v == INFINITY) flags |= 1;
        else if (isfinite(v)) flags |= 2;
        if (v > mx) { mx = v; arg = i; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(0xffffffffu, mx, o);
        const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
        if (om > mx || (om == mx && oa < arg)) { mx = om; arg = oa; }
        flags |= __shfl_xor_sync(0xffffffffu, flags, o);
    }
    if (lane == 0) { s_max[warp] = mx; s_arg[warp] = arg; s_bad[warp] = flags; }
    __syncthreads();
    mx = s_max[0]; arg = s_arg[0]; flags = s_bad[0];
    for (int i = 1; i < SCORE_WARPS; i++) {
        if (s_max[i] > mx || (s_max[i] == mx && s_arg[i] < arg)) { mx = s_max[i]; arg = s_arg[i]; }
        flags |= s_bad[i];
    }
    const bool valid = flags == 2;
    double s = 0;
    if (valid)
        for (int i = tid; i < V; i += SCORE_THREADS) s += (double) expf(z[i] - mx);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) s_sum[warp] = s;
    __syncthreads();
    if (tid == 0) {
        double sum = 0;
        for (int i = 0; i < SCORE_WARPS; i++) sum += s_sum[i];
        const float lp = valid ? (float) ((double) (z[target] - mx) - log(sum)) : NAN;
        p.logprobs[t] = lp;
        if (p.greedy) p.greedy[t] = valid && arg == (int) target ? 1 : 0;
    }
    trace_end(p.trace);
}

}  // namespace

cudaError_t launch_layer_norm_columns(const float * x, const float * w, const float * b, int C, int T, float * y, cudaStream_t s) {
    return launch_pdl(layer_norm_columns_kernel, dim3((unsigned) T), dim3(SCORE_THREADS), 0, s, x, w, b, C, y, trace_slot("layer_norm_columns"));
}

cudaError_t launch_score(const ScoreParams & p, cudaStream_t s) {
    ScoreParams q = p;
    q.trace = trace_slot("score");
    return launch_pdl(score_kernel, dim3((unsigned) p.T), dim3(SCORE_THREADS), 0, s, q);
}

}  // namespace rwkv
