// The log-softmax reduction of score_kernel (score.cu) for the generation step that reports the log-probability of every drawn token
// (sampling.cu): the same loads, comparisons and sums in the same order, so that both give the same bits for the same column.
// score_kernel keeps its own copy of these lines: routed through this function its SASS changes (register allocation only), and the
// scoring path is left exactly as it was. test_gpu_generate_logprobs.py holds the two to the same bits.
#pragma once
#include <cuda_runtime.h>
#include <cmath>

namespace rwkv {

constexpr int LP_SCORE_THREADS = 256;     // score.cu's SCORE_THREADS: the order of the sums depends on it
constexpr int LP_SCORE_WARPS = LP_SCORE_THREADS / 32;

// Run by threads tid = 0 .. LP_SCORE_THREADS - 1 of the CTA; `sync` is a barrier over exactly those threads, called twice. Thread 0 then
// calls finish(mx, arg, valid, sum): the maximum of z[0 .. V) (float), its first index, whether the column is valid (no NaN or +inf,
// some finite value) and sum exp(z - max) in double (0 when not valid). The order of every sum depends on V alone.
template <class Sync, class Finish>
__device__ __forceinline__ void score_column(int tid, const float * z, int V, float * s_max, int * s_arg, int * s_bad, double * s_sum, Sync sync,
                                             Finish finish) {
    const int lane = tid & 31, warp = tid >> 5;
    // max, its first index, and whether the column holds a NaN / +inf (bad) or any finite value (bit 1)
    float mx = -INFINITY;
    int arg = V, flags = 0;
    for (int i = tid; i < V; i += LP_SCORE_THREADS) {
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
    sync();
    mx = s_max[0]; arg = s_arg[0]; flags = s_bad[0];
    for (int i = 1; i < LP_SCORE_WARPS; i++) {
        if (s_max[i] > mx || (s_max[i] == mx && s_arg[i] < arg)) { mx = s_max[i]; arg = s_arg[i]; }
        flags |= s_bad[i];
    }
    const bool valid = flags == 2;
    double s = 0;
    if (valid)
        for (int i = tid; i < V; i += LP_SCORE_THREADS) s += (double) expf(z[i] - mx);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) s_sum[warp] = s;
    sync();
    if (tid == 0) {
        double sum = 0;
        for (int i = 0; i < LP_SCORE_WARPS; i++) sum += s_sum[i];
        finish(mx, arg, valid, sum);
    }
}

// log_softmax(z)[t] from z[t], the column's maximum and log(sum exp(z - max)): score_kernel's expression.
__device__ __forceinline__ float score_logprob(float zt, float mx, double log_sum) { return (float) ((double) (zt - mx) - log_sum); }

}  // namespace rwkv
