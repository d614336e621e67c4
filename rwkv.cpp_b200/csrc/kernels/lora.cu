// Shrink and expand launches of the low-rank deltas (lora.h).
#include "lora.h"
#include "gemv_tma_device.cuh"   // tma::prefetch_epilogue / tma::apply_epilogue / tma::warp_sum: the streaming GEMV's own arithmetic

#include <cuda_fp16.h>

namespace rwkv {

namespace {

constexpr int LORA_THREADS = 256;
constexpr int LORA_COLS = 8;                     // columns per CTA

__device__ __forceinline__ float h2f(uint16_t h) { return __half2float(__ushort_as_half(h)); }

// The group of CTA blockIdx.x: the last one whose first CTA is at or below it (a group without CTAs shares its first with the next).
__device__ __forceinline__ int find_group(const LoraBatch & b, bool expand) {
    int lo = 0, hi = b.n_groups - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if ((int) blockIdx.x >= (expand ? b.g[mid].first_expand : b.g[mid].first_shrink)) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// CTA: row r of a group's A times columns [cg * 8, cg * 8 + 8) of the group's list. Thread t sums the 8-element groups t, t + 256,
// t + 512, ... of the row, each group in element order (one 16-byte load of A and two of x per column where the addresses allow, else
// element by element: the same order either way); then a butterfly per warp and the 8 warps' partial sums in warp order. All of it a
// function of K alone.
__global__ void __launch_bounds__(LORA_THREADS) lora_shrink_kernel(const LoraBatch b, TraceRec * trace) {
    __shared__ float part[LORA_THREADS / 32][LORA_COLS];
    trace_begin(trace);
    pdl_prologue();
    const LoraGroup & G = b.g[find_group(b, false)];
    const LoraProblem & P = b.p[G.problem];
    const int local = (int) blockIdx.x - G.first_shrink;
    const int r = local % G.d.rank, c0 = (local / G.d.rank) * LORA_COLS;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int nc = min(LORA_COLS, G.n_cols - c0), K = P.K;
    const uint8_t * cols = b.col + G.col0 + c0;
    const uint16_t * a = G.d.A + (size_t) r * K;
    const float * x[LORA_COLS];
#pragma unroll
    for (int c = 0; c < LORA_COLS; c++) x[c] = P.x + (long long) cols[c < nc ? c : 0] * P.ldx;
    const bool vec = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(P.x)) & 15) == 0 && P.ldx % 4 == 0;
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
                const float4 lo = *reinterpret_cast<const float4 *>(x[c] + k0);
                const float4 hi = *reinterpret_cast<const float4 *>(x[c] + k0 + 4);
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
                    if (c < nc) acc[c] = __fmaf_rn(we, x[c][k0 + e], acc[c]);
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
        P.u[(size_t) cols[threadIdx.x] * P.ldu + r] = s;
    }
    trace_end(trace);
}

// CTA: rows [rb * 256, rb * 256 + 256) of a group's B (one per thread) times columns [cg * 8, cg * 8 + 8) of the group's list. A group of
// rank 0 writes epi(z) for its columns.
__global__ void __launch_bounds__(LORA_THREADS) lora_expand_kernel(const LoraBatch b, TraceRec * trace) {
    __shared__ float us[LORA_MAX_RANK][LORA_COLS];
    trace_begin(trace);
    pdl_prologue();
    const LoraGroup & G = b.g[find_group(b, true)];
    const LoraProblem & P = b.p[G.problem];
    const int local = (int) blockIdx.x - G.first_expand;
    const int n_rb = (P.M + LORA_THREADS - 1) / LORA_THREADS;
    const int rb = local % n_rb, c0 = (local / n_rb) * LORA_COLS;
    const int nc = min(LORA_COLS, G.n_cols - c0), R = G.d.rank;
    const uint8_t * cols = b.col + G.col0 + c0;
    for (int i = threadIdx.x; i < R * LORA_COLS; i += LORA_THREADS) {
        const int r = i / LORA_COLS, c = i % LORA_COLS;
        us[r][c] = c < nc ? P.u[(size_t) cols[c] * P.ldu + r] : 0.f;
    }
    __syncthreads();
    const int row = rb * LORA_THREADS + (int) threadIdx.x;
    if (row >= P.M) { trace_end(trace); return; }
    float acc[LORA_COLS];
#pragma unroll
    for (int c = 0; c < LORA_COLS; c++) acc[c] = 0.f;
#pragma unroll 8
    for (int r = 0; r < R; r++) {
        const float w = h2f(G.d.Bt[(size_t) r * P.M + row]);
#pragma unroll
        for (int c = 0; c < LORA_COLS; c++) acc[c] = __fmaf_rn(w, us[r][c], acc[c]);
    }
#pragma unroll
    for (int c = 0; c < LORA_COLS; c++) {
        if (c >= nc) break;
        const int col = cols[c];
        const tma::EpiOperands e = tma::prefetch_epilogue(P.P, row, col);
        float v;
        if (R == 0) {
            v = P.z[(long long) col * P.ldz + row];
        } else {
            const float delta = __fmul_rn(G.d.scale, acc[c]);
            v = P.z ? __fadd_rn(P.z[(long long) col * P.ldz + row], delta) : delta;
        }
        P.P.y[(long long) col * P.P.ldy + row] = tma::apply_epilogue(P.P, v, e.a, e.b);
    }
    trace_end(trace);
}

}  // namespace

cudaError_t launch_lora_shrink(LoraBatch & b, cudaStream_t stream) {
    if (b.n_groups <= 0) return cudaSuccess;
    int next = 0;
    for (int i = 0; i < b.n_groups; i++) {
        b.g[i].first_shrink = next;
        next += b.g[i].d.rank * ((b.g[i].n_cols + LORA_COLS - 1) / LORA_COLS);
    }
    if (next == 0) return cudaSuccess;
    return launch_pdl(lora_shrink_kernel, dim3(next), dim3(LORA_THREADS), 0, stream, b, trace_slot("lora_shrink"));
}

cudaError_t launch_lora_expand(LoraBatch & b, cudaStream_t stream) {
    if (b.n_groups <= 0) return cudaSuccess;
    int next = 0;
    for (int i = 0; i < b.n_groups; i++) {
        b.g[i].first_expand = next;
        next += (b.p[b.g[i].problem].M + LORA_THREADS - 1) / LORA_THREADS * ((b.g[i].n_cols + LORA_COLS - 1) / LORA_COLS);
    }
    return launch_pdl(lora_expand_kernel, dim3(next), dim3(LORA_THREADS), 0, stream, b, trace_slot("lora_expand"));
}

}  // namespace rwkv
