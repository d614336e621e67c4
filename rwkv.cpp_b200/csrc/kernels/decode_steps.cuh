// Single-token building blocks of the batched multi-sequence kernels (batch.cu): LayerNorm statistics and one WKV5/6 step,
// restated from glue.cu / wkv.cu for T = 1 with the same per-element operations and reduction trees, so their results are
// bit-identical to the per-launch kernels' (tests/test_gpu_kernels.py checks it). All of them are written for a group of exactly
// 256 threads that synchronises with tma::consumer_barrier() (named barrier 1).
#pragma once
#include "gemv_tma_device.cuh"

namespace rwkv {
namespace steps {

using tma::consumer_barrier;

constexpr int LN_MAXCH = 16;               // channels per thread in the LayerNorm stage: n_embed <= 4096

__device__ __forceinline__ double warp_tree_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// x -> (x - mean) per owned channel and 1 / sqrt(var + 1e-5), bit-identical to ln_mix_kernel<PER> (glue.cu): that kernel runs 1024
// threads, thread v summing channels v, v + 1024, ... in double, then a warp xor-tree, 32 slots and a second xor-tree over the
// slots. Thread t of the 256 plays the four virtual threads v = t + 256 q: virtual warp (t >> 5) + 8 q, same lane. Thread t ends
// up owning channels t + 256 m (m = q + 4 i: virtual thread q, its i-th channel); channels >= C hold 0.
__device__ __forceinline__ void ln_center_scale_256(const float * x, int C, float (&xa)[LN_MAXCH], float & scale_a, double (* slots)[32]) {
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    double sa[4] = {0, 0, 0, 0};
#pragma unroll
    for (int i = 0; i < 4; i++) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const int m = q + 4 * i, c = t + 256 * m;
            xa[m] = (c < C) ? __ldcg(x + c) : 0.f;       // L2, not L1: as a GEMV tail job x was written by OTHER SMs during this very kernel
            sa[q] += (double) xa[m];
        }
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const double r = warp_tree_d(sa[q]);
        if (lane == 0) slots[0][warp + 8 * q] = r;
    }
    consumer_barrier();
    const float mean_a = (float) (warp_tree_d(slots[0][lane]) / C);
    double va[4] = {0, 0, 0, 0};
#pragma unroll
    for (int i = 0; i < 4; i++) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const int m = q + 4 * i, c = t + 256 * m;
            xa[m] = (c < C) ? xa[m] - mean_a : 0.f;
            va[q] += (double) (xa[m] * xa[m]);
        }
    }
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const double r = warp_tree_d(va[q]);
        if (lane == 0) slots[1][warp + 8 * q] = r;
    }
    consumer_barrier();
    scale_a = 1.0f / sqrtf((float) (warp_tree_d(slots[1][lane]) / C) + 1e-5f);
}

struct WkvStep {             // Wkv6Params for one token of one sequence, without default member initialisers
    const float * r, * k, * v, * td, * tf, * state_in, * lnx_w, * lnx_b, * g;
    float * state_out, * y;
    float eps;
    int td_per_token, per_head_scalars, H, S;
};

// ---- one WKV5/6 step of head h + per-head norm + ln_x + gate (wkv6_kernel<S>, wkv.cu, for T = 1): thread (oct, jg) owns the
// 8 x 4 state patch, partial outputs meet over the octants by the same xor-shuffles, warp 0 normalises the head.
__device__ __forceinline__ void load8(const float * p, float (&o)[8]) {
    const float4 a = *reinterpret_cast<const float4 *>(p), b = *reinterpret_cast<const float4 *>(p + 4);
    o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
}
template <int S>
__device__ void wkv6_step(const WkvStep & p, int h, float * ybuf) {
    constexpr int NOCT = S / 8, NJG = S / 4, NT = NOCT * NJG, NW = (NT + 31) / 32, CPL = (S + 31) / 32;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t hb = (size_t) h * S;
    float lw[CPL], lb[CPL], gg[CPL];
    if (warp == 0) {      // parameters of the normalisation, requested before the recurrence
#pragma unroll
        for (int i = 0; i < CPL; i++) {
            const int col = lane + 32 * i;
            lw[i] = col < S ? p.lnx_w[hb + col] : 0.f;
            lb[i] = col < S ? p.lnx_b[hb + col] : 0.f;
            gg[i] = (col < S && p.g) ? p.g[hb + col] : 0.f;
        }
    }
    if (warp < NW) {
        const bool worker = tid < NT;
        const int oct = worker ? tid % NOCT : 0, jg = worker ? tid / NOCT : 0;
        const int i0 = oct * 8, j0 = jg * 4;
        float st[8][4], kk[8], rr[8], dv[8], tfr[8], vv[4];
#pragma unroll
        for (int ii = 0; ii < 8; ii++) {
            const float4 v = *reinterpret_cast<const float4 *>(p.state_in + (hb + i0 + ii) * S + j0);
            st[ii][0] = v.x; st[ii][1] = v.y; st[ii][2] = v.z; st[ii][3] = v.w;
        }
        load8(p.k + hb + i0, kk);
        load8(p.r + hb + i0, rr);
        if (p.per_head_scalars) {
            const float tf = p.tf[h], td = p.td[h];
#pragma unroll
            for (int ii = 0; ii < 8; ii++) { tfr[ii] = tf; dv[ii] = td; }
        } else {
            load8(p.tf + hb + i0, tfr);
            load8(p.td + hb + i0, dv);      // per token (v6) or per channel (v5.2): the same index for T = 1
        }
        {
            const float4 g4 = *reinterpret_cast<const float4 *>(p.v + hb + j0);
            vv[0] = g4.x; vv[1] = g4.y; vv[2] = g4.z; vv[3] = g4.w;
        }
        float y[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int ii = 0; ii < 8; ii++) {
#pragma unroll
            for (int jj = 0; jj < 4; jj++) {
                const float kv = __fmul_rn(vv[jj], kk[ii]);
                const float temp = __fmaf_rn(kv, tfr[ii], st[ii][jj]);
                y[jj] = __fmaf_rn(temp, rr[ii], y[jj]);
                st[ii][jj] = __fmaf_rn(st[ii][jj], dv[ii], kv);
            }
        }
#pragma unroll
        for (int o = 1; o < NOCT; o <<= 1) {
#pragma unroll
            for (int jj = 0; jj < 4; jj++) y[jj] += __shfl_xor_sync(0xffffffffu, y[jj], o);
        }
        if (worker && oct == 0) *reinterpret_cast<float4 *>(&ybuf[j0]) = make_float4(y[0], y[1], y[2], y[3]);
        if (worker) {
#pragma unroll
            for (int ii = 0; ii < 8; ii++)
                *reinterpret_cast<float4 *>(p.state_out + (hb + i0 + ii) * S + j0) = make_float4(st[ii][0], st[ii][1], st[ii][2], st[ii][3]);
        }
    }
    consumer_barrier();
    if (warp == 0) {
        float yv[CPL];
        double s1 = 0, s2 = 0;
#pragma unroll
        for (int i = 0; i < CPL; i++) {
            const int col = lane + 32 * i;
            yv[i] = col < S ? ybuf[col] : 0.f;
            s1 += (double) yv[i];
            s2 += (double) yv[i] * (double) yv[i];
        }
        s1 = warp_tree_d(s1);
        s2 = warp_tree_d(s2);
        const double mean_d = s1 / S;
        const float mean = (float) mean_d;
        const float var = (float) fmax(s2 / S - mean_d * mean_d, 0.0);
        const float rstd = 1.0f / sqrtf(var + p.eps);
#pragma unroll
        for (int i = 0; i < CPL; i++) {
            const int col = lane + 32 * i;
            if (col < S) {
                float n = (yv[i] - mean) * rstd;
                n = __fadd_rn(__fmul_rn(n, lw[i]), lb[i]);
                if (p.g) n = __fmul_rn(n, gg[i]);
                p.y[hb + col] = n;
            }
        }
    }
}

}  // namespace steps
}  // namespace rwkv
