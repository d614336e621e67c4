// Top-N selection over one column of logits by a CTA of SAMPLE_THREADS threads, shared by the logprob step kernels (sampling.cu) and
// the beam search step (beam.cu), so that both list the same ids in the same order for the same column.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <type_traits>

#include "ops.h"    // GEN_TOP_MAX

namespace rwkv {

constexpr int SAMPLE_THREADS = 1024;
constexpr int SAMPLE_WARPS = SAMPLE_THREADS / 32;

// The column kernels of sampling.cu and beam.cu hold PER entries of a column per thread, PER in {1, 4, 16, 50, 64}
// (n_vocab <= SAMPLE_THREADS * 64). Returns f(std::integral_constant<int, PER>{}) for the smallest PER that covers n_vocab.
template <class F>
auto with_sample_per(int n_vocab, F && f) {
    const int per = (n_vocab + SAMPLE_THREADS - 1) / SAMPLE_THREADS;
    if (per <= 1) return f(std::integral_constant<int, 1>{});
    if (per <= 4) return f(std::integral_constant<int, 4>{});
    if (per <= 16) return f(std::integral_constant<int, 16>{});
    if (per <= 50) return f(std::integral_constant<int, 50>{});
    return f(std::integral_constant<int, 64>{});
}

// Top-N order over (logit, id): a larger logit first, the smaller id first among equal logits. The key holds the logit's bits mapped to
// an unsigned order in its upper half (-0 counted as +0, so that equal values differ by id alone) and ~id in its lower half, so every
// entry of a column has its own key and the largest keys are the top entries. No entry maps to key 0 (upper half 0xFFFFFFFF and id
// 0xFFFFFFFF together), so 0 stands for "none".
__device__ __forceinline__ unsigned long long top_key(float v, int i) {
    const uint32_t u = __float_as_uint(__fadd_rn(v, 0.0f));
    return ((unsigned long long) ((u & 0x80000000u) ? ~u : (u | 0x80000000u)) << 32) | (uint32_t) ~(uint32_t) i;
}
// The largest key below `limit` among this thread's entries tid + k * SAMPLE_THREADS of z, or 0.
template <int PER>
__device__ __forceinline__ unsigned long long top_below(const float * z, int V, int tid, unsigned long long limit) {
    unsigned long long best = 0;
#pragma unroll 4
    for (int k = 0; k < PER; k++) {
        const int i = tid + k * SAMPLE_THREADS;
        if (i < V) {
            const unsigned long long key = top_key(z[i], i);
            if (key < limit && key > best) best = key;
        }
    }
    return best;
}
__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w > v ? w : v;
    }
    return v;
}

// Every thread of the CTA: warp w's top_n largest keys, largest first, into s_top[w][0 .. top_n), by top_n rounds of a warp-wide key
// maximum (a round's winner rescans its own entries below the key it gave up). A warp out of entries writes 0. top_n <= GEN_TOP_MAX.
template <int PER>
__device__ __forceinline__ void warp_top_keys(const float * z, int V, int tid, int top_n, unsigned long long (*s_top)[GEN_TOP_MAX]) {
    if (top_n <= 0) return;
    const int lane = tid & 31, warp = tid >> 5;
    unsigned long long mine = top_below<PER>(z, V, tid, ~0ull);
    for (int k = 0; k < top_n; k++) {
        const unsigned long long w = warp_max_u64(mine);
        if (lane == 0) s_top[warp][k] = w;
        if (w != 0 && mine == w) mine = top_below<PER>(z, V, tid, w);
    }
}

// Warp 0, after a CTA barrier that follows warp_top_keys: merges the 32 sorted lists and calls emit(k, key) on every lane with the
// CTA's k-th largest key, k = 0 .. top_n - 1 in order (0 once the column has no more entries).
template <class Emit>
__device__ __forceinline__ void merge_top_keys(int lane, int top_n, const unsigned long long (*s_top)[GEN_TOP_MAX], Emit emit) {
    int head = 0;
    unsigned long long cur = top_n > 0 ? s_top[lane][0] : 0ull;
    for (int k = 0; k < top_n; k++) {
        const unsigned long long w = warp_max_u64(cur);
        emit(k, w);
        if (cur == w) { head++; cur = head < top_n ? s_top[lane][head] : 0ull; }
    }
}

}  // namespace rwkv
