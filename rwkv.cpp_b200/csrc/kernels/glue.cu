// Embedding gather + ln0, LayerNorm + token shift + mixing, and the v6 data-dependent lerp.
// These are the small fp32 element-wise stages between the GEMVs; each is one launch over [C, T].
#include "ops.h"
#include "gemv.h"          // launch_pdl
#include "../formats.h"
#include "act_stage.cuh"
#include "gemv_tma_device.cuh"   // stage_column / rows_dot of the v6 prologue

#include <cuda_fp16.h>

namespace rwkv {
namespace {

constexpr int GLUE_THREADS = 256;
constexpr int GLUE_WARPS = GLUE_THREADS / 32;

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ double block_sum_d(double v, double * scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum_d(v);
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0;
        for (int i = 0; i < GLUE_WARPS; i++) s += scratch[i];
        scratch[GLUE_WARPS] = s;
    }
    __syncthreads();
    return scratch[GLUE_WARPS];
}

// dst[c] = LN(src)[c] * w[c] + b[c]; statistics as ggml_compute_forward_norm_f32 (ggml-cpu.c:6906-6925),
// weight/bias as rwkv_layer_norm (rwkv_operators.inc:93-97). src may be shared or global.
__device__ void layer_norm_to(const float * src, const float * w, const float * b, int C, float * dst, double * scratch) {
    double s = 0;
    for (int c = threadIdx.x; c < C; c += GLUE_THREADS) s += (double) src[c];
    const float mean = (float) (block_sum_d(s, scratch) / C);
    double s2 = 0;
    for (int c = threadIdx.x; c < C; c += GLUE_THREADS) { float v = src[c] - mean; s2 += (double) (v * v); }
    const float var = (float) (block_sum_d(s2, scratch) / C);
    const float scale = 1.0f / sqrtf(var + 1e-5f);
    for (int c = threadIdx.x; c < C; c += GLUE_THREADS)
        dst[c] = __fadd_rn(__fmul_rn(__fmul_rn(src[c] - mean, scale), w[c]), b[c]);
    __syncthreads();
}

__global__ void __launch_bounds__(GLUE_THREADS) embed_ln0_kernel(const uint8_t * emb, int emb_type, long long pitch, const int * tokens, int C,
                                                                  const float * ln_w, const float * ln_b, float * x) {
    extern __shared__ float sh[];
    __shared__ double scratch[GLUE_WARPS + 1];
    pdl_prologue();
    const int t = blockIdx.x;
    const uint8_t * row = emb + (size_t) tokens[t] * (size_t) pitch;
    for (int c = threadIdx.x; c < C; c += GLUE_THREADS)
        sh[c] = (emb_type == DT_F16) ? __half2float(reinterpret_cast<const __half *>(row)[c]) : reinterpret_cast<const float *>(row)[c];
    __syncthreads();
    layer_norm_to(sh, ln_w, ln_b, C, x + (size_t) t * C, scratch);
}

constexpr int LN_THREADS = 1024;
constexpr int LN_WARPS = LN_THREADS / 32;

// CTA-wide sum, one barrier: warp shuffle, 32 warp partials in `slots`, then every warp reduces the 32 slots again.
__device__ __forceinline__ double block_sum_ln(double v, double * slots) {
    v = warp_sum_d(v);
    if ((threadIdx.x & 31) == 0) slots[threadIdx.x >> 5] = v;
    __syncthreads();
    return warp_sum_d(slots[threadIdx.x & 31]);
}

// Latency-optimised LayerNorm + token shift + mixing. This stage is ONE CTA per token sitting on the critical path
// between two weight-streaming kernels, so what matters is the length of its dependent instruction chain: 1024
// threads, PER = C/1024 channels per thread in registers, loads that do not depend on the previous kernel (LayerNorm
// weights, the carried state of the previous token) issued BEFORE the programmatic-dependency wait, the x loads
// right after it, two barrier-separated reductions, rolled output loop (small code: instruction fetch is the other
// cost of a run-once kernel). Statistics as ggml_compute_forward_norm_f32 (ggml-cpu.c:6906-6925, sums in double).
// PRE_N: how many of the mix-coefficient vectors are requested before the dependency wait (3 for blocks with up to three mixed
// vectors -- every v6 block --, 6 for v4 / v5.2 / v7 time mixing: a few spilled registers there against one HBM round trip per vector).
// MODE SEQ_BATCH: block t is the one token of sequence t. Its previous LN(x) is always that sequence's carry, never
// column t - 1, and it always writes the sequence's new carry.
// MODE SEQ_RAGGED: block t is a column of sequence s = col_seq[t]. Its previous LN(x) is the sequence's carry on the sequence's first
// column and LN(x[:, t-1]) on the others; the sequence's last column writes its new carry.
// The body is shared with v6_prologue_kernel: token t of the launch; out0, if not NULL, takes the place of p.out[0] (t == 0);
// write_carry = false skips out_sx, out_xx and state_out.
// MODE | SEQ_SNAP: a column with a checkpoint slot in *cp also writes its LN(x), the carry it would leave as the last column, into the slot.
template <int PER, int PRE_N, int MODE>
__device__ __forceinline__ void ln_mix_body(const LnMixParams & p, int t, float * out0, bool write_carry, double (&slots)[4][LN_WARPS],
                                            const CheckpointMap * cp = nullptr) {
    constexpr bool BATCH = (MODE & ~SEQ_SNAP) == SEQ_BATCH, RAGGED = (MODE & ~SEQ_SNAP) == SEQ_RAGGED;
    const int C = p.C, tid = threadIdx.x;
    // ragged: the sequence's first and last column and its state's offset. The column map is written by the host: safe before the
    // dependency wait. (The other modes keep their expressions below as they were: they are what their code was compiled from.)
    int r_first = 0, r_last = 0;
    long long r_so = 0;
    if constexpr (RAGGED) {
        const int s = p.col_seq[t];
        r_first = p.seq_off[s];
        r_last = p.seq_off[s + 1] - 1;
        r_so = s * p.seq_stride;
    }
    // LayerNorm weights and the carry are loaded before the wait where registers allow it (PER <= 8); at PER = 16 holding them
    // across the statistics spills past the stack budget, so they are read where they are used
    constexpr bool EARLY = PER <= 8;
    float lw[PER], lb[PER], pv[PER], xa[PER], xb[PER];
    auto load_ln = [&]() {
#pragma unroll
        for (int i = 0; i < PER; i++) {
            const int c = tid + i * LN_THREADS;
            const bool live = c < C;
            lw[i] = live ? p.ln_w[c] : 0.f;
            lb[i] = live ? p.ln_b[c] : 0.f;
            pv[i] = (live && (BATCH || (RAGGED ? t == r_first : t == 0))) ? p.state_in[BATCH ? t * p.seq_stride + c : RAGGED ? r_so + c : c] : 0.f;   // written by the previous token's pass: safe before the wait
        }
    };
    if constexpr (EARLY) load_ln();
    // the mix coefficients too (up to 6 vectors): last read one token ago, i.e. an HBM round trip each -- and the output loop below
    // used to take them one vector after the other, AFTER the statistics (a sizeable part of a kernel that runs 64 times per 7B token)
    // (1024 threads leave 64 registers each: PER <= 4 only)
    constexpr bool PRE = PER <= 4;
    float cf[PRE ? PRE_N : 1][PER];
    if constexpr (PRE) {
#pragma unroll
        for (int j = 0; j < PRE_N; j++) {
#pragma unroll
            for (int i = 0; i < PER; i++) {
                const int c = tid + i * LN_THREADS;
                cf[j][i] = (j < p.n_out && c < C) ? p.coef[j][c] : 0.f;
            }
        }
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    double sa = 0, sb = 0;
#pragma unroll
    for (int i = 0; i < PER; i++) {
        const int c = tid + i * LN_THREADS;
        const bool live = c < C;
        xa[i] = live ? p.x[(size_t) t * C + c] : 0.f;
        xb[i] = (live && !BATCH && (RAGGED ? t > r_first : t > 0)) ? p.x[(size_t) (t - 1) * C + c] : 0.f;
        sa += (double) xa[i];
        sb += (double) xb[i];
    }
    const float mean_a = (float) (block_sum_ln(sa, slots[0]) / C);
    const float mean_b = (!BATCH && (RAGGED ? t > r_first : t > 0)) ? (float) (block_sum_ln(sb, slots[1]) / C) : 0.f;
    double va = 0, vb = 0;
#pragma unroll
    for (int i = 0; i < PER; i++) {
        const bool live = tid + i * LN_THREADS < C;
        xa[i] = live ? xa[i] - mean_a : 0.f;
        xb[i] = live ? xb[i] - mean_b : 0.f;
        va += (double) (xa[i] * xa[i]);
        vb += (double) (xb[i] * xb[i]);
    }
    const float scale_a = 1.0f / sqrtf((float) (block_sum_ln(va, slots[2]) / C) + 1e-5f);
    const float scale_b = (!BATCH && (RAGGED ? t > r_first : t > 0)) ? 1.0f / sqrtf((float) (block_sum_ln(vb, slots[3]) / C) + 1e-5f) : 0.f;
    if constexpr (!EARLY) load_ln();
    // normalised current / previous token, in place
#pragma unroll
    for (int i = 0; i < PER; i++) {
        xa[i] = __fadd_rn(__fmul_rn(__fmul_rn(xa[i], scale_a), lw[i]), lb[i]);                            // LN(x[:, t])
        xb[i] = (!BATCH && (RAGGED ? t > r_first : t > 0)) ? __fadd_rn(__fmul_rn(__fmul_rn(xb[i], scale_b), lw[i]), lb[i]) : pv[i];   // LN(x[:, t-1]) or the carry
    }
    const size_t o0 = (size_t) t * C + tid;
    if constexpr (PRE) {
#pragma unroll
        for (int j = 0; j < PRE_N; j++) {
            if (j >= p.n_out) break;
            float * out = (out0 && j == 0) ? out0 : p.out[j];
#pragma unroll
            for (int i = 0; i < PER; i++) {
                const int c = tid + i * LN_THREADS;
                if (c < C) {
                    const float m = cf[j][i];
                    out[o0 + i * LN_THREADS] = (p.formula == 0) ? __fadd_rn(__fmul_rn(xa[i], m), __fsub_rn(xb[i], __fmul_rn(xb[i], m)))
                                                               : __fadd_rn(__fmul_rn(__fsub_rn(xb[i], xa[i]), m), xa[i]);
                }
            }
        }
    }
    {
#pragma unroll 1
        for (int j = PRE ? PRE_N : 0; j < p.n_out; j++) {     // rolled: kernel parameters are indexable in the constant bank
            const float * coef = p.coef[j];
            float * out = (out0 && j == 0) ? out0 : p.out[j];
#pragma unroll
            for (int i = 0; i < PER; i++) {
                const int c = tid + i * LN_THREADS;
                if (c < C) {
                    const float m = coef[c];
                    out[o0 + i * LN_THREADS] = (p.formula == 0) ? __fadd_rn(__fmul_rn(xa[i], m), __fsub_rn(xb[i], __fmul_rn(xb[i], m)))
                                                               : __fadd_rn(__fmul_rn(__fsub_rn(xb[i], xa[i]), m), xa[i]);
                }
            }
        }
    }
    if (!write_carry) return;
#pragma unroll
    for (int i = 0; i < PER; i++) {
        const int c = tid + i * LN_THREADS;
        if (c >= C) continue;
        if (p.out_sx) p.out_sx[o0 + i * LN_THREADS] = __fsub_rn(xb[i], xa[i]);
        if (p.out_xx) p.out_xx[o0 + i * LN_THREADS] = xa[i];
        if (BATCH || (RAGGED ? t == r_last : t == p.T - 1)) p.state_out[BATCH ? t * p.seq_stride + c : RAGGED ? r_so + c : c] = xa[i];
    }
    if constexpr ((MODE & SEQ_SNAP) != 0) {
        const int slot = cp->slot[t];
        if (slot < 0) return;
        float * dst = cp->dst[slot] + cp->at;
#pragma unroll
        for (int i = 0; i < PER; i++) {
            const int c = tid + i * LN_THREADS;
            if (c < C) dst[c] = xa[i];
        }
    }
}

template <int PER, int PRE_N, int MODE>
__global__ void __launch_bounds__(LN_THREADS) ln_mix_kernel(const LnMixParams p) {
    __shared__ double slots[4][LN_WARPS];
    trace_begin(p.trace);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    ln_mix_body<PER, PRE_N, MODE>(p, blockIdx.x, nullptr, true, slots);
    trace_end(p.trace);
}

// ln_mix_kernel with checkpoints (MODE SEQ_ONE or SEQ_RAGGED).
template <int PER, int PRE_N, int MODE>
__global__ void __launch_bounds__(LN_THREADS) ln_mix_snap_kernel(const LnMixParams p, const CheckpointMap cp) {
    __shared__ double slots[4][LN_WARPS];
    trace_begin(p.trace);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    ln_mix_body<PER, PRE_N, MODE | SEQ_SNAP>(p, blockIdx.x, nullptr, true, slots, &cp);
    trace_end(p.trace);
}

// ln_mix + the first v6 LoRA matrix of a single-token pass (launch_v6_prologue). CTA b computes rows [8b, 8b + 8) of W1 = w1.W, whose
// bytes it copies to shared memory before the dependency wait; after it, the LayerNorm and mix[0] of ln_mix_body (into shared
// memory), mix[0] staged as the streaming GEMV stages a column (TYPE = w1.type), and rows_dot.
template <int PER, int TYPE>
__global__ void __launch_bounds__(LN_THREADS) v6_prologue_kernel(const LnMixParams p, const GemvProblem w1) {
    extern __shared__ __align__(16) uint8_t v6p_smem[];       // [V6_PROLOGUE_ROWS rows of W1][mix[0]: C floats][staged mix[0]]
    __shared__ double slots[4][LN_WARPS];
    trace_begin(p.trace);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int row0 = blockIdx.x * V6_PROLOGUE_ROWS, rows = min(V6_PROLOGUE_ROWS, w1.M - row0);
    const int bytes = rows * (int) w1.pitch;
    const uint8_t * src = reinterpret_cast<const uint8_t *>(w1.W) + (size_t) row0 * w1.pitch;
    for (int i = threadIdx.x * 16; i < bytes; i += LN_THREADS * 16)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"((uint32_t) __cvta_generic_to_shared(v6p_smem + i)), "l"(src + i) : "memory");
    asm volatile("cp.async.commit_group;" ::: "memory");
    float * mix = reinterpret_cast<float *>(v6p_smem + (size_t) V6_PROLOGUE_ROWS * w1.pitch);
    uint8_t * act = reinterpret_cast<uint8_t *>(mix) + (((size_t) p.C * sizeof(float) + 15) & ~(size_t) 15);
    ln_mix_body<PER, 3, SEQ_ONE>(p, 0, mix, blockIdx.x == 0, slots);
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
    GemvProblem P = w1;
    P.x = mix;
    // the 8-lanes-per-block staging, not the GEMV's one-thread-per-block form: that one holds 16 float4 per thread, more than the 64
    // registers a 1024-thread CTA leaves (it spilled). Both write the same bytes (stage_column).
    if (threadIdx.x < tma::CONSUMER_THREADS) tma::stage_column<4, false, TYPE, false>(P, 0, act, nullptr);
    __syncthreads();
    tma::rows_dot<TYPE>(P, v6p_smem, rows, row0, act, w1.y + row0);
    trace_end(p.trace);
}

// Passes of fewer than LERP_MIN_TOKENS tokens (decode): 8 lanes per channel, 32 channels per CTA, one CTA row per token: each (j, channel) row of W2 is `mix` contiguous floats. The W2 rows
// (5.2 MB per layer at 7B, straight from HBM) are pulled into registers before the programmatic-dependency wait.
constexpr int LERP1_MAX_F4 = 4;   // float4 per lane per j held in registers: mix <= 128
__global__ void __launch_bounds__(GLUE_THREADS) v6_lerp_decode_kernel(const V6LerpParams p) {
    extern __shared__ float zs[];   // [5*mix]
    __shared__ float ob[5][32];     // the CTA's 32 channels of each output = one 32-element block of its staged column
    trace_begin(p.trace);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int t = blockIdx.y, mix = p.mix, C = p.C;
    const int grp = threadIdx.x >> 3, sub = threadIdx.x & 7;
    const int c = blockIdx.x * 32 + grp;
    const bool live = c < C;
    const bool vec = (mix & 3) == 0 && mix / 4 <= 8 * LERP1_MAX_F4;
    float4 wreg[5][LERP1_MAX_F4];
    float maa[5];
    if (vec) {
#pragma unroll
        for (int j = 0; j < 5; j++) {
            const float4 * wrow = reinterpret_cast<const float4 *>(p.w2 + ((size_t) j * C + (live ? c : 0)) * mix);
#pragma unroll
            for (int q = 0; q < LERP1_MAX_F4; q++) {
                const int i4 = sub + 8 * q;
                wreg[j][q] = (live && i4 < mix / 4) ? __ldg(wrow + i4) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            maa[j] = live ? p.maa[j][c] : 0.f;
        }
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    for (int i = threadIdx.x; i < 5 * mix; i += GLUE_THREADS) zs[i] = p.z[(size_t) t * 5 * mix + i];
    const size_t o = (size_t) t * C + (live ? c : 0);
    const float sx = live ? p.sx[o] : 0.f, xx = live ? p.xx[o] : 0.f;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 5; j++) {
        float acc = 0.f;
        const float * zj = zs + j * mix;
        if (vec) {
#pragma unroll
            for (int q = 0; q < LERP1_MAX_F4; q++) {
                const int i4 = sub + 8 * q;
                if (i4 < mix / 4) {
                    const float4 w = wreg[j][q], z = reinterpret_cast<const float4 *>(zj)[i4];
                    acc = __fmaf_rn(w.x, z.x, acc); acc = __fmaf_rn(w.y, z.y, acc);
                    acc = __fmaf_rn(w.z, z.z, acc); acc = __fmaf_rn(w.w, z.w, acc);
                }
            }
        } else if (live) {
            const float * wrow = p.w2 + ((size_t) j * C + c) * mix;
            if ((mix & 3) == 0) {
                for (int i4 = sub; i4 < mix / 4; i4 += 8) {
                    const float4 w = __ldg(reinterpret_cast<const float4 *>(wrow) + i4), z = reinterpret_cast<const float4 *>(zj)[i4];
                    acc = __fmaf_rn(w.x, z.x, acc); acc = __fmaf_rn(w.y, z.y, acc);
                    acc = __fmaf_rn(w.z, z.z, acc); acc = __fmaf_rn(w.w, z.w, acc);
                }
            } else {
                for (int i = sub; i < mix; i += 8) acc = __fmaf_rn(wrow[i], zj[i], acc);
            }
        }
        acc += __shfl_xor_sync(0xffffffffu, acc, 4);
        acc += __shfl_xor_sync(0xffffffffu, acc, 2);
        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        if (sub == 0) {
            const float val = live ? __fadd_rn(__fmul_rn(__fadd_rn(acc, vec ? maa[j] : p.maa[j][c]), sx), xx) : 0.f;
            if (live) p.out[j][o] = val;
            ob[j][grp] = val;
        }
    }
    if (p.q_out[0] != nullptr) {       // single-token passes with C % 32 == 0 (the caller checks): warp j emits block blockIdx.x of out_j
        __syncthreads();
        const int warp = threadIdx.x >> 5;
        if (warp < 5 && p.q_out[warp]) act::warp_emit_block(act::StagedOut{p.q_out[warp], p.q_type[warp], C}, blockIdx.x, ob[warp][threadIdx.x & 31]);
    }
    trace_end(p.trace);
}


// Passes of >= LERP_MIN_TOKENS tokens: one thread per channel, one CTA = 128 channels x a tile of TILE tokens x ONE of the five mixes
// (blockIdx.z). The thread holds its W2 row (`mix` contiguous floats) in registers and walks the tile's tokens; z[:, t] of the tile
// sits in shared memory and is read as broadcasts. TILE = 32 for chunks (each W2 row is fetched once per 32 tokens: 21 MB of L2
// traffic per 128-token layer pass at 7B instead of 84 MB with tiles of 8, and 5 x more CTAs than one CTA looping over the mixes),
// 8 for short passes. The W2 row is pulled before the programmatic-dependency wait.
constexpr int LERP_THREADS = 128;
constexpr int LERP_MIN_TOKENS = 8;
constexpr int LERP_MAX_F4 = 16;   // W2 row in registers: mix <= 64
// M4 > 0: mix == 4 * M4 known at compile time (32 and 64 in the released models): the dot product is M4 float4 steps with no
// predication and no other code path in the loop -- the generic body ran ~270 instructions per token where 60 do the work
// (the profiler showed a kernel moving 25 MB at under half its issue slots). M4 == 0: any mix.
template <int TILE, int M4>
__global__ void __launch_bounds__(LERP_THREADS) v6_lerp_kernel(const V6LerpParams p) {
    extern __shared__ __align__(16) float lerp_zs[];        // [tile][mix]: the z rows of mix j
    trace_begin(p.trace);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int mix = p.mix, C = p.C, tid = threadIdx.x, j = blockIdx.z;
    const int c = blockIdx.x * LERP_THREADS + tid;
    const bool live = c < C;
    const int cc = live ? c : 0;
    const int m4 = M4 > 0 ? M4 : mix / 4;
    const bool vec = M4 > 0 || ((mix & 3) == 0 && m4 <= LERP_MAX_F4);
    const int t0 = blockIdx.y * TILE, nt = min(TILE, p.T - t0);
    float4 w[LERP_MAX_F4];
    {
        const float4 * wrow = reinterpret_cast<const float4 *>(p.w2 + ((size_t) j * C + cc) * mix);
#pragma unroll
        for (int i = 0; i < LERP_MAX_F4; i++) w[i] = (vec && i < m4) ? __ldg(wrow + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const float maa = p.maa[j][cc];
    asm volatile("griddepcontrol.wait;" ::: "memory");
    for (int i = tid; i < nt * mix; i += LERP_THREADS) {
        const int tt = i / mix, k = i % mix;
        lerp_zs[i] = p.z[(size_t) (t0 + tt) * 5 * mix + j * mix + k];
    }
    __syncthreads();
    float * out = p.out[j];
#pragma unroll 8
    for (int tt = 0; tt < nt; tt++) {       // eight tokens' loads in flight: the loop is latency-bound (4-5 CTAs of 4 warps per SM)
        const size_t o = (size_t) (t0 + tt) * C + cc;
        const float sx = __ldg(p.sx + o), xx = __ldg(p.xx + o);
        const float * zj = lerp_zs + (size_t) tt * mix;
        // the same eight partial sums and the same combination tree as the decode kernel's 8 lanes + shuffles: a chunked
        // evaluation stays bit-identical to the serial one (tests/test_eval_sequence_in_chunks.c memcmp's them)
        float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if constexpr (M4 > 0) {
#pragma unroll
            for (int i = 0; i < M4; i++) {
                const float4 z = reinterpret_cast<const float4 *>(zj)[i];
                float & s8 = a[i & 7];
                s8 = __fmaf_rn(w[i].x, z.x, s8); s8 = __fmaf_rn(w[i].y, z.y, s8);
                s8 = __fmaf_rn(w[i].z, z.z, s8); s8 = __fmaf_rn(w[i].w, z.w, s8);
            }
        } else if (vec) {
#pragma unroll
            for (int i = 0; i < LERP_MAX_F4; i++) {
                if (i < m4) {
                    const float4 z = reinterpret_cast<const float4 *>(zj)[i];
                    float & s8 = a[i & 7];
                    s8 = __fmaf_rn(w[i].x, z.x, s8); s8 = __fmaf_rn(w[i].y, z.y, s8);
                    s8 = __fmaf_rn(w[i].z, z.z, s8); s8 = __fmaf_rn(w[i].w, z.w, s8);
                }
            }
        } else if ((mix & 3) == 0) {
            const float4 * wrow = reinterpret_cast<const float4 *>(p.w2 + ((size_t) j * C + cc) * mix);
            for (int i0 = 0; i0 < m4; i0 += 8) {
#pragma unroll
                for (int u = 0; u < 8; u++) {
                    if (i0 + u < m4) {
                        const float4 wv = __ldg(wrow + i0 + u), z = reinterpret_cast<const float4 *>(zj)[i0 + u];
                        a[u] = __fmaf_rn(wv.x, z.x, a[u]); a[u] = __fmaf_rn(wv.y, z.y, a[u]);
                        a[u] = __fmaf_rn(wv.z, z.z, a[u]); a[u] = __fmaf_rn(wv.w, z.w, a[u]);
                    }
                }
            }
        } else {
            const float * wrow = p.w2 + ((size_t) j * C + cc) * mix;
            for (int i0 = 0; i0 < mix; i0 += 8) {
#pragma unroll
                for (int u = 0; u < 8; u++)
                    if (i0 + u < mix) a[u] = __fmaf_rn(__ldg(wrow + i0 + u), zj[i0 + u], a[u]);
            }
        }
        const float acc = __fadd_rn(__fadd_rn(__fadd_rn(a[0], a[4]), __fadd_rn(a[2], a[6])), __fadd_rn(__fadd_rn(a[1], a[5]), __fadd_rn(a[3], a[7])));
        if (live) out[(size_t) (t0 + tt) * C + c] = __fadd_rn(__fmul_rn(__fadd_rn(acc, maa), sx), xx);
    }
    trace_end(p.trace);
}

}  // namespace

cudaError_t launch_embed_ln0(const void * emb, int emb_type, long long emb_pitch, const int * tokens, int T, int C,
                             const float * ln_w, const float * ln_b, float * x, cudaStream_t s) {
    return launch_pdl(embed_ln0_kernel, dim3(T), dim3(GLUE_THREADS), (size_t) C * sizeof(float), s, reinterpret_cast<const uint8_t *>(emb), emb_type, emb_pitch, tokens, C, ln_w, ln_b, x);
}

// Grid row t is token t, sequence t in batch mode, or column t in ragged mode. The single-sequence instantiation comes first: with
// the batch one first, nvcc emitted different code for the untouched v6_lerp_kernel<8, 16> of this file. The ragged one comes last.
// The checkpoint instantiations come after all of these.
template <int PER, int PRE_N>
cudaError_t launch_ln_mix_kernel(const LnMixParams & p, cudaStream_t s, const CheckpointMap & cp) {
    if (!cp.slot)
        return !p.seq_stride ? launch_pdl(ln_mix_kernel<PER, PRE_N, SEQ_ONE>, dim3(p.T), dim3(LN_THREADS), 0, s, p)
             : !p.seq_off    ? launch_pdl(ln_mix_kernel<PER, PRE_N, SEQ_BATCH>, dim3(p.T), dim3(LN_THREADS), 0, s, p)
                             : launch_pdl(ln_mix_kernel<PER, PRE_N, SEQ_RAGGED>, dim3(p.T), dim3(LN_THREADS), 0, s, p);
    if (p.seq_stride && !p.seq_off) return cudaErrorInvalidValue;
    return !p.seq_stride ? launch_pdl(ln_mix_snap_kernel<PER, PRE_N, SEQ_ONE>, dim3(p.T), dim3(LN_THREADS), 0, s, p, cp)
                         : launch_pdl(ln_mix_snap_kernel<PER, PRE_N, SEQ_RAGGED>, dim3(p.T), dim3(LN_THREADS), 0, s, p, cp);
}

cudaError_t launch_ln_mix(const LnMixParams & p_in, cudaStream_t s, const CheckpointMap & cp) {
    LnMixParams p = p_in;
    p.trace = trace_slot("ln_mix");
    const int per = (p.C + LN_THREADS - 1) / LN_THREADS;
#define RWKV_LN(PER_) return p.n_out > 3 ? launch_ln_mix_kernel<PER_, 6>(p, s, cp) : launch_ln_mix_kernel<PER_, 3>(p, s, cp);
    if (per <= 1) { RWKV_LN(1) }
    if (per <= 2) { RWKV_LN(2) }
    if (per <= 4) { RWKV_LN(4) }
    if (per <= 8) { RWKV_LN(8) }
    if (per <= 16) { RWKV_LN(16) }
#undef RWKV_LN
    return cudaErrorInvalidValue;   // n_embed > 16384
}

size_t v6_prologue_smem_bytes(const GemvProblem & w1, int C) {
    return (size_t) V6_PROLOGUE_ROWS * (size_t) w1.pitch + (((size_t) C * sizeof(float) + 15) & ~(size_t) 15) + tma::act_bytes_per_column(w1.type, w1.K);
}

template <int PER, int TYPE>
static cudaError_t launch_v6_prologue_kernel(const LnMixParams & p, const GemvProblem & w1, cudaStream_t s) {
    static PerDeviceOnce once;
    const cudaError_t e = once.run([&] { return cudaFuncSetAttribute(v6_prologue_kernel<PER, TYPE>, cudaFuncAttributeMaxDynamicSharedMemorySize, V6_PROLOGUE_MAX_SMEM); });
    if (e != cudaSuccess) return e;
    return launch_pdl(v6_prologue_kernel<PER, TYPE>, dim3((w1.M + V6_PROLOGUE_ROWS - 1) / V6_PROLOGUE_ROWS), dim3(LN_THREADS), v6_prologue_smem_bytes(w1, p.C), s, p, w1);
}

// Only the (PER, type) pairs a one-warp-per-row plan admits are compiled: F32 rows up to n_embed 896 (PER 1), F16 up to 1792 (PER <= 2).
template <int PER>
static cudaError_t launch_v6_prologue_per(const LnMixParams & p, const GemvProblem & w1, cudaStream_t s) {
    switch (w1.type) {
        case DT_Q4_0: return launch_v6_prologue_kernel<PER, DT_Q4_0>(p, w1, s);
        case DT_Q4_1: return launch_v6_prologue_kernel<PER, DT_Q4_1>(p, w1, s);
        case DT_Q5_0: return launch_v6_prologue_kernel<PER, DT_Q5_0>(p, w1, s);
        case DT_Q5_1: return launch_v6_prologue_kernel<PER, DT_Q5_1>(p, w1, s);
        case DT_Q8_0: return launch_v6_prologue_kernel<PER, DT_Q8_0>(p, w1, s);
        case DT_F16: if constexpr (PER <= 2) return launch_v6_prologue_kernel<PER, DT_F16>(p, w1, s); else return cudaErrorInvalidValue;
        case DT_F32: if constexpr (PER == 1) return launch_v6_prologue_kernel<PER, DT_F32>(p, w1, s); else return cudaErrorInvalidValue;
        default: return cudaErrorInvalidValue;
    }
}

// v6_lora_fold has checked the shape (C <= 4096, a WK == 1 plan, the shared memory); these checks only keep a wrong call from launching.
cudaError_t launch_v6_prologue(const LnMixParams & p_in, const GemvProblem & w1, cudaStream_t s) {
    LnMixParams p = p_in;
    p.trace = trace_slot("v6_prologue");
    if (p.T != 1 || p.seq_stride || p.n_out != 1 || p.formula != 1 || w1.K != p.C || w1.wk != 1 || v6_prologue_smem_bytes(w1, p.C) > V6_PROLOGUE_MAX_SMEM)
        return cudaErrorInvalidValue;
    const int per = (p.C + LN_THREADS - 1) / LN_THREADS;
    if (per <= 1) return launch_v6_prologue_per<1>(p, w1, s);
    if (per <= 2) return launch_v6_prologue_per<2>(p, w1, s);
    if (per <= 4) return launch_v6_prologue_per<4>(p, w1, s);
    return cudaErrorInvalidValue;
}

cudaError_t launch_v6_lerp(const V6LerpParams & p_in, cudaStream_t s) {
    V6LerpParams p = p_in;
    p.trace = trace_slot("v6_lerp");
    if (p.T < LERP_MIN_TOKENS) {
        dim3 grid((p.C + 31) / 32, p.T);
        return launch_pdl(v6_lerp_decode_kernel, grid, dim3(GLUE_THREADS), (size_t) 5 * p.mix * sizeof(float), s, p);
    }
    const int tile = (p.T >= 32 && (size_t) 32 * p.mix * sizeof(float) <= 48 * 1024) ? 32 : 8;      // which tile a token falls into does not touch its arithmetic
    const size_t smem = (size_t) tile * p.mix * sizeof(float);
    if (smem > 48 * 1024) return cudaErrorInvalidValue;
    dim3 grid((p.C + LERP_THREADS - 1) / LERP_THREADS, (p.T + tile - 1) / tile, 5);
    if (p.mix == 32) return tile == 32 ? launch_pdl(v6_lerp_kernel<32, 8>, grid, dim3(LERP_THREADS), smem, s, p) : launch_pdl(v6_lerp_kernel<8, 8>, grid, dim3(LERP_THREADS), smem, s, p);
    if (p.mix == 64) return tile == 32 ? launch_pdl(v6_lerp_kernel<32, 16>, grid, dim3(LERP_THREADS), smem, s, p) : launch_pdl(v6_lerp_kernel<8, 16>, grid, dim3(LERP_THREADS), smem, s, p);
    return tile == 32 ? launch_pdl(v6_lerp_kernel<32, 0>, grid, dim3(LERP_THREADS), smem, s, p) : launch_pdl(v6_lerp_kernel<8, 0>, grid, dim3(LERP_THREADS), smem, s, p);
}

}  // namespace rwkv
