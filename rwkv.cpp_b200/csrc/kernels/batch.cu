// Batched multi-sequence decode (SURVEY.md 8f-2): one token of each of B independent sequences per pass, so every weight matrix
// is streamed ONCE for B tokens (the GEMVs run their multi-column path; per column they are bit-identical to a single-token pass).
// What differs from a B-token pass over ONE sequence is only where the recurrence reads and writes its state: the token shift takes
// the previous LN(x) of the column's own sequence instead of the neighbouring column, and every column has its own WKV state.
// The kernels here do exactly that: column t works on the state of sequence t (state base + t * seq_stride floats). They are
// built from the single-token steps of decode_steps.cuh, so a sequence evaluated inside a batch produces the same bits as the
// same sequence evaluated alone through rwkv_eval (tests/test_gpu_batch.py).
#include "ops.h"
#include "gemv.h"
#include "decode_steps.cuh"

namespace rwkv {
namespace {

using namespace steps;

constexpr int BATCH_THREADS = 256;      // decode_steps.cuh is written for 256-thread groups

// LayerNorm + token shift + mixing (rwkv_carry_x + lerps, rwkv_graph.inc:56-82, 94-97, 310-311), one CTA per sequence.
__global__ void __launch_bounds__(BATCH_THREADS) ln_mix_batch_kernel(const LnMixParams p, const long long seq_stride) {
    __shared__ double slots[2][32];
    trace_begin(p.trace);
    const int C = p.C, seq = blockIdx.x, t = threadIdx.x;
    const float * prev = p.state_in + (long long) seq * seq_stride;
    float * carry = p.state_out + (long long) seq * seq_stride;
    const size_t col = (size_t) seq * C;
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    // parameters and the carried LN(x) do not depend on the previous kernel
    float lw[LN_MAXCH], lb[LN_MAXCH], pv[LN_MAXCH];
#pragma unroll
    for (int m = 0; m < LN_MAXCH; m++) {
        const int c = t + 256 * m;
        const bool live = c < C;
        lw[m] = live ? p.ln_w[c] : 0.f;
        lb[m] = live ? p.ln_b[c] : 0.f;
        pv[m] = live ? prev[c] : 0.f;
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    float xa[LN_MAXCH], scale_a;
    ln_center_scale_256(p.x + col, C, xa, scale_a, slots);
#pragma unroll
    for (int m = 0; m < LN_MAXCH; m++) xa[m] = __fadd_rn(__fmul_rn(__fmul_rn(xa[m], scale_a), lw[m]), lb[m]);     // LN(x)
#pragma unroll 1
    for (int j = 0; j < p.n_out; j++) {
        const float * coef = p.coef[j];
        float * out = p.out[j] + col;
        float cf[LN_MAXCH];
#pragma unroll
        for (int m = 0; m < LN_MAXCH; m++) { const int c = t + 256 * m; cf[m] = c < C ? coef[c] : 0.f; }
#pragma unroll
        for (int m = 0; m < LN_MAXCH; m++) {
            const int c = t + 256 * m;
            if (c < C) out[c] = (p.formula == 0) ? __fadd_rn(__fmul_rn(xa[m], cf[m]), __fsub_rn(pv[m], __fmul_rn(pv[m], cf[m])))
                                                 : __fadd_rn(__fmul_rn(__fsub_rn(pv[m], xa[m]), cf[m]), xa[m]);
        }
    }
#pragma unroll
    for (int m = 0; m < LN_MAXCH; m++) {
        const int c = t + 256 * m;
        if (c >= C) continue;
        if (p.out_sx) p.out_sx[col + c] = __fsub_rn(pv[m], xa[m]);
        if (p.out_xx) p.out_xx[col + c] = xa[m];
        carry[c] = xa[m];
    }
    trace_end(p.trace);
}

// One WKV5/6 step per (head, sequence) + head norm + ln_x + gate.
template <int S>
__global__ void __launch_bounds__(BATCH_THREADS) wkv6_batch_kernel(WkvStep p, const int C, const long long seq_stride, TraceRec * trace) {
    __shared__ __align__(16) float ybuf[S];
    trace_begin(trace);
    pdl_prologue();
    const long long seq = blockIdx.y;
    p.r += seq * C; p.k += seq * C; p.v += seq * C; p.y += seq * C;
    if (p.g) p.g += seq * C;
    if (p.td_per_token) p.td += seq * C;
    p.state_in += seq * seq_stride; p.state_out += seq * seq_stride;
    wkv6_step<S>(p, (int) blockIdx.x, ybuf);
    trace_end(trace);
}

// v4 WKV for one token per sequence (wkv4_kernel, wkv.cu, T = 1): thread per channel, blockIdx.y = sequence.
__global__ void wkv4_batch_kernel(const Wkv4Params p, const long long seq_stride) {
    trace_begin(p.trace);
    pdl_prologue();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= p.C) return;
    const long long seq = blockIdx.y, so = seq * seq_stride;
    float aa = p.aa_in[so + c], bb = p.bb_in[so + c], pp = p.pp_in[so + c];
    const float tf = p.time_first[c], td = p.time_decay[c];
    const size_t o = (size_t) seq * p.C + c;
    const float k = p.k[o], v = p.v[o];
    float ww = __fadd_rn(tf, k);
    float qq = fmaxf(pp, ww);
    float e1 = expf(__fsub_rn(pp, qq)), e2 = expf(__fsub_rn(ww, qq));
    const float a = __fadd_rn(__fmul_rn(e1, aa), __fmul_rn(e2, v));
    const float b = __fadd_rn(__fmul_rn(e1, bb), e2);
    ww = __fadd_rn(pp, td);
    qq = fmaxf(ww, k);
    e1 = expf(__fsub_rn(ww, qq));
    e2 = expf(__fsub_rn(k, qq));
    aa = __fadd_rn(__fmul_rn(e1, aa), __fmul_rn(e2, v));
    bb = __fadd_rn(__fmul_rn(e1, bb), e2);
    pp = qq;
    p.y[o] = __fmul_rn(p.r[o], __fdiv_rn(a, b));
    p.aa_out[so + c] = aa; p.bb_out[so + c] = bb; p.pp_out[so + c] = pp;
    trace_end(p.trace);
}

}  // namespace

bool batch_shape_supported(int arch_major, int n_embed, int head_size) {
    if (arch_major == 4) return n_embed <= 256 * steps::LN_MAXCH;
    if (arch_major == 5 || arch_major == 6) return n_embed <= 256 * steps::LN_MAXCH && (head_size == 8 || head_size == 16 || head_size == 32 || head_size == 64);
    if (arch_major == 7) return n_embed <= 256 * steps::LN_MAXCH && (head_size == 8 || head_size == 16 || head_size == 32 || head_size == 64 || head_size == 128);
    return false;
}

cudaError_t launch_ln_mix_batch(const LnMixParams & p_in, long long seq_stride, cudaStream_t s) {
    LnMixParams p = p_in;
    if (p.C > 256 * steps::LN_MAXCH) return cudaErrorInvalidValue;
    p.trace = trace_slot("ln_mix_batch");
    return launch_pdl(ln_mix_batch_kernel, dim3(p.T), dim3(BATCH_THREADS), 0, s, p, seq_stride);
}

cudaError_t launch_wkv6_batch(const Wkv6Params & w, long long seq_stride, cudaStream_t s) {
    steps::WkvStep k;
    k.r = w.r; k.k = w.k; k.v = w.v; k.td = w.td; k.tf = w.tf; k.state_in = w.state_in; k.lnx_w = w.lnx_w; k.lnx_b = w.lnx_b; k.g = w.g;
    k.state_out = w.state_out; k.y = w.y; k.eps = w.eps; k.td_per_token = w.td_per_token; k.per_head_scalars = w.per_head_scalars; k.H = w.H; k.S = w.S;
    TraceRec * trace = trace_slot("wkv6_batch");
    const dim3 grid(w.H, w.T), block(BATCH_THREADS);
    const int C = w.H * w.S;
    switch (w.S) {
        case 8: return launch_pdl(wkv6_batch_kernel<8>, grid, block, 0, s, k, C, seq_stride, trace);
        case 16: return launch_pdl(wkv6_batch_kernel<16>, grid, block, 0, s, k, C, seq_stride, trace);
        case 32: return launch_pdl(wkv6_batch_kernel<32>, grid, block, 0, s, k, C, seq_stride, trace);
        case 64: return launch_pdl(wkv6_batch_kernel<64>, grid, block, 0, s, k, C, seq_stride, trace);
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_wkv4_batch(const Wkv4Params & p_in, long long seq_stride, cudaStream_t s) {
    Wkv4Params p = p_in;
    p.trace = trace_slot("wkv4_batch");
    const int threads = 128;
    return launch_pdl(wkv4_batch_kernel, dim3((p.C + threads - 1) / threads, p.T), dim3(threads), 0, s, p, seq_stride);
}

}  // namespace rwkv
