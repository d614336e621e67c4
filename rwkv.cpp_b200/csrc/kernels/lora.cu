// Shrink and expand launches of the low-rank deltas (lora.h).
#include "lora.h"
#include "gemv_tma_device.cuh"   // tma::prefetch_epilogue / tma::apply_epilogue / tma::warp_sum: the streaming GEMV's own arithmetic

#include <cuda_fp16.h>

namespace rwkv {

namespace {

constexpr int LORA_THREADS = 256;
constexpr int LORA_COLS = 8;                     // columns per CTA

__device__ __forceinline__ float h2f(uint16_t h) { return __half2float(__ushort_as_half(h)); }

__device__ __forceinline__ int find_problem(const LoraBatch & b, bool expand) {
    int pi = 0;
    for (int i = 1; i < b.n; i++) if ((int) blockIdx.x >= (expand ? b.p[i].first_expand : b.p[i].first_shrink)) pi = i;
    return pi;
}

// CTA: row r of A times columns [cg * 8, cg * 8 + 8) of x. Thread t sums the 8-element groups t, t + 256, t + 512, ... of the row,
// each group in element order (one 16-byte load of A and two of x per column where the addresses allow, else element by element: the
// same order either way); then a butterfly per warp and the 8 warps' partial sums in warp order. All of it a function of K alone.
__global__ void __launch_bounds__(LORA_THREADS) lora_shrink_kernel(const LoraBatch b, TraceRec * trace) {
    __shared__ float part[LORA_THREADS / 32][LORA_COLS];
    trace_begin(trace);
    pdl_prologue();
    const LoraProblem & P = b.p[find_problem(b, false)];
    const int local = (int) blockIdx.x - P.first_shrink;
    const int r = local % P.d.rank, c0 = (local / P.d.rank) * LORA_COLS;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nc = min(LORA_COLS, b.T - c0), K = P.K;
    const uint16_t * a = P.d.A + (size_t) r * K;
    const float * x = P.x + (long long) c0 * P.ldx;
    const bool vec = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(x)) & 15) == 0 && P.ldx % 4 == 0;
    float acc[LORA_COLS];
#pragma unroll
    for (int c = 0; c < LORA_COLS; c++) acc[c] = 0.f;
    for (int k0 = 8 * (int) threadIdx.x; k0 < K; k0 += 8 * LORA_THREADS) {
        float w[8];
        if (vec && k0 + 8 <= K) {
            const uint4 q = *reinterpret_cast<const uint4 *>(a + k0);
            const uint32_t h[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int e = 0; e < 4; e++) { w[2 * e] = h2f((uint16_t) (h[e] & 0xFFFFu)); w[2 * e + 1] = h2f((uint16_t) (h[e] >> 16)); }
#pragma unroll
            for (int c = 0; c < LORA_COLS; c++) {
                if (c >= nc) break;
                const float4 lo = *reinterpret_cast<const float4 *>(x + (long long) c * P.ldx + k0);
                const float4 hi = *reinterpret_cast<const float4 *>(x + (long long) c * P.ldx + k0 + 4);
                const float xv[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
                for (int e = 0; e < 8; e++) acc[c] = __fmaf_rn(w[e], xv[e], acc[c]);
            }
        } else {
            const int n = min(8, K - k0);
            for (int e = 0; e < n; e++) {
                const float we = h2f(a[k0 + e]);
#pragma unroll
                for (int c = 0; c < LORA_COLS; c++)
                    if (c < nc) acc[c] = __fmaf_rn(we, x[(long long) c * P.ldx + k0 + e], acc[c]);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < LORA_COLS; c++) {
        const float v = tma::warp_sum(acc[c]);
        if (lane == 0) part[warp][c] = v;
    }
    __syncthreads();
    if (threadIdx.x < (unsigned) nc) {
        float s = part[0][threadIdx.x];
#pragma unroll
        for (int w = 1; w < LORA_THREADS / 32; w++) s = __fadd_rn(s, part[w][threadIdx.x]);
        P.u[(size_t) (c0 + threadIdx.x) * P.d.rank + r] = s;
    }
    trace_end(trace);
}

// CTA: rows [rb * 256, rb * 256 + 256) of B (one per thread) times columns [cg * 8, cg * 8 + 8) of u.
__global__ void __launch_bounds__(LORA_THREADS) lora_expand_kernel(const LoraBatch b, TraceRec * trace) {
    __shared__ float us[LORA_MAX_RANK][LORA_COLS];
    trace_begin(trace);
    pdl_prologue();
    const LoraProblem & P = b.p[find_problem(b, true)];
    const int local = (int) blockIdx.x - P.first_expand;
    const int n_rb = (P.M + LORA_THREADS - 1) / LORA_THREADS;
    const int rb = local % n_rb, c0 = (local / n_rb) * LORA_COLS;
    const int nc = min(LORA_COLS, b.T - c0), R = P.d.rank;
    for (int i = threadIdx.x; i < R * LORA_COLS; i += LORA_THREADS) {
        const int r = i / LORA_COLS, c = i % LORA_COLS;
        us[r][c] = c < nc ? P.u[(size_t) (c0 + c) * R + r] : 0.f;
    }
    __syncthreads();
    const int row = rb * LORA_THREADS + (int) threadIdx.x;
    if (row >= P.M) { trace_end(trace); return; }
    float acc[LORA_COLS];
#pragma unroll
    for (int c = 0; c < LORA_COLS; c++) acc[c] = 0.f;
#pragma unroll 8
    for (int r = 0; r < R; r++) {
        const float w = h2f(P.d.Bt[(size_t) r * P.M + row]);
#pragma unroll
        for (int c = 0; c < LORA_COLS; c++) acc[c] = __fmaf_rn(w, us[r][c], acc[c]);
    }
#pragma unroll
    for (int c = 0; c < LORA_COLS; c++) {
        if (c >= nc) break;
        const int col = c0 + c;
        const tma::EpiOperands e = tma::prefetch_epilogue(P.P, row, col);
        const float delta = __fmul_rn(P.d.scale, acc[c]);
        const float v = P.z ? __fadd_rn(P.z[(long long) col * P.ldz + row], delta) : delta;
        P.P.y[(long long) col * P.P.ldy + row] = tma::apply_epilogue(P.P, v, e.a, e.b);
    }
    trace_end(trace);
}

}  // namespace

cudaError_t launch_lora_shrink(LoraBatch & b, cudaStream_t stream) {
    if (b.n <= 0) return cudaSuccess;
    const int ncg = (b.T + LORA_COLS - 1) / LORA_COLS;
    int next = 0;
    for (int i = 0; i < b.n; i++) {
        b.p[i].first_shrink = next;
        next += b.p[i].d.rank * ncg;
    }
    return launch_pdl(lora_shrink_kernel, dim3(next), dim3(LORA_THREADS), 0, stream, b, trace_slot("lora_shrink"));
}

cudaError_t launch_lora_expand(LoraBatch & b, cudaStream_t stream) {
    if (b.n <= 0) return cudaSuccess;
    const int ncg = (b.T + LORA_COLS - 1) / LORA_COLS;
    int next = 0;
    for (int i = 0; i < b.n; i++) {
        b.p[i].first_expand = next;
        next += (b.p[i].M + LORA_THREADS - 1) / LORA_THREADS * ncg;
    }
    return launch_pdl(lora_expand_kernel, dim3(next), dim3(LORA_THREADS), 0, stream, b, trace_slot("lora_expand"));
}

}  // namespace rwkv
