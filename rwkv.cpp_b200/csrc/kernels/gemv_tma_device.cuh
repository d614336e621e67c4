// Device side of the TMA-streamed fused dequantize-GEMV (ring, activation staging, consumers), shared by the
// per-launch kernel (gemv_tma.cu) and the persistent single-token kernel (decode_persistent.cu). Everything here
// is arithmetic-defining: the per-row summation order is a function of (type, K) alone (see gemv_tma.cu).
#pragma once
#include "gemv.h"
#include "quant_decode.cuh"

#include <cuda_fp16.h>

namespace rwkv {
namespace tma {

constexpr int CONSUMER_WARPS = 8;
constexpr int CONSUMER_THREADS = CONSUMER_WARPS * 32;
constexpr int THREADS = CONSUMER_THREADS + 32;      // + one producer warp
constexpr int NSTAGES = 3;
constexpr int NOMINAL_STAGE_BYTES = 28 * 1024;      // WK is planned against this size, whatever the launch really gets (>= this)
// Dynamic shared memory per CTA so that TWO CTAs share an SM: 233 472 B per SM, 1 KB reserved per CTA, ~1.4 KB static (Shared).
// 110 KB gives the same tile heights as 111 KB for every shape of the BASELINE configurations (8 rows at K = 4096 Q5_1, 2 at
// K = 14336) and leaves 1 KB of slack: at 111 KB half a kilobyte more of static shared memory would silently halve the occupancy.
// (With 112 KB the K = 14336 launches came to 114 176 B and ran ONE CTA per SM.)
constexpr int CTA_SMEM_BUDGET = 110 * 1024;
constexpr int MAX_TILE_ROWS = 64;
constexpr int MAX_BLOCKS_PER_LANE = 4;              // activation blocks a lane keeps in registers

// ---- PTX wrappers --------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t * bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t * bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t * bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t * bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// Bounded wait for kernels that must never hang a device (the persistent decode kernel): polls try_wait and, should the
// phase not complete within ~4 s of SM clock, traps -- the launch then fails with an error instead of spinning forever.
constexpr long long GUARD_CYCLES = 8000000000ll;
__device__ __forceinline__ bool mbar_try_wait(uint64_t * bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
static __device__ __noinline__ void mbar_wait_slow(uint64_t * bar, uint32_t parity) {
    const long long t0 = clock64();
    unsigned spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0xFFFu) == 0 && clock64() - t0 > GUARD_CYCLES) __trap();
    }
}
template <bool GUARD> __device__ __forceinline__ void mbar_wait_t(uint64_t * bar, uint32_t parity) {
    if constexpr (GUARD) { if (!mbar_try_wait(bar, parity)) mbar_wait_slow(bar, parity); }
    else mbar_wait(bar, parity);
}
// global -> shared bulk copy completing on an mbarrier, with an L2 cache policy
__device__ __forceinline__ void bulk_copy_g2s(void * dst, const void * src, uint32_t bytes, uint64_t * bar, uint64_t policy) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
                 : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t policy_evict_normal() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void consumer_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(CONSUMER_THREADS) : "memory"); }
// programmatic dependent launch (PDL)
__device__ __forceinline__ void grid_dependency_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void grid_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum_double(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float round_to_half(float v) { return __half2float(__float2half_rn(v)); }
__device__ __forceinline__ float sigmoidf_(float v) { return 1.0f / (1.0f + expf(-v)); }

// Epilogue operands that live in global memory (residual, gate, per-row bias) are fetched at the START of a tile, so
// their latency hides behind the tile's dot products instead of sitting between the reduction and the store.
struct EpiOperands { float a, b; };
__device__ __forceinline__ EpiOperands prefetch_epilogue(const GemvProblem & P, int row, int col) {
    EpiOperands e; e.a = 0.f; e.b = 0.f;
    switch (P.epi) {
        case EPI_ADD: e.a = P.res[(long long) col * P.ldres + row]; break;
        case EPI_MUL_ADD: e.a = P.res[(long long) col * P.ldres + row]; e.b = P.gate[(long long) col * P.ldgate + row]; break;
        case EPI_BIAS_EXPNEGEXP: case EPI_BIAS_SIGMOID: case EPI_BIAS_W7: e.a = P.bias[row]; break;
        default: break;
    }
    return e;
}
__device__ __forceinline__ float apply_epilogue(const GemvProblem & P, float v, float ea, float eb) {
    switch (P.epi) {
        case EPI_SIGMOID: return sigmoidf_(v);
        case EPI_SILU: return v / (1.0f + expf(-v));
        case EPI_TANH: return tanhf(v);
        case EPI_RELU_SQR: { float r = fmaxf(v, 0.0f); return __fmul_rn(r, r); }
        case EPI_ADD: return __fadd_rn(ea, v);
        case EPI_MUL_ADD: return __fadd_rn(ea, __fmul_rn(eb, v));
        case EPI_BIAS_EXPNEGEXP: return expf(-expf(__fadd_rn(v, ea)));
        case EPI_BIAS_SIGMOID: return sigmoidf_(__fadd_rn(v, ea));
        case EPI_BIAS_W7: return expf(__fmul_rn(sigmoidf_(__fadd_rn(v, ea)), -0.606531f));
        default: return v;
    }
}

// ---- shared-memory layout:  [ ring: NSTAGES x stage_bytes ][ act: NC columns ][ red ] ----------------------------
// Blocks of a quantised activation column rounded up to whole units (pairs for the 2-byte-aligned formats).
__host__ __device__ inline int padded_blocks(int type, int K) {
    const int nblk = K / 32;
    return (type == DT_Q4_1 || type == DT_Q5_1) ? nblk : (nblk + 1) / 2 * 2;
}
__host__ __device__ inline size_t act_bytes_per_column(int type, int K) {
    size_t b;
    if (type == DT_F32) b = (size_t) K * 4;
    else if (type == DT_F16) b = (size_t) K * 2;
    else b = (size_t) padded_blocks(type, K) * (32 + sizeof(ActScale));
    return (b + 15) & ~(size_t) 15;
}

struct Shared {
    uint64_t full[NSTAGES];
    uint64_t empty[NSTAGES];
    double red_d[CONSUMER_WARPS + 1];
    TraceRec * trace;
    GemvProblem P;
};

// Quantised activation column in shared memory, laid out so that lanes working on consecutive units read
// consecutive 16-byte / 8-byte words: for block b = u*UB + bi, half h (elements 16h..16h+15):
//     q     at  ((bi*2 + h) * nunits + u) * 16
//     scale at  nunits*UB*32 + (bi * nunits + u) * 8
template <int UB> __device__ __forceinline__ const int4 * act_q_ptr(const uint8_t * col, int nunits, int u, int bi, int h) {
    return reinterpret_cast<const int4 *>(col + ((size_t) (bi * 2 + h) * nunits + u) * 16);
}
template <int UB> __device__ __forceinline__ const ActScale * act_s_ptr(const uint8_t * col, int nunits, int u, int bi) {
    return reinterpret_cast<const ActScale *>(col + (size_t) nunits * UB * 32 + ((size_t) bi * nunits + u) * 8);
}

// One unit of a staged row -> registers. Q5_1 units are 24 bytes on an 8-byte grid: three 64-bit loads whose
// lane stride (3 x 8 B) is conflict-free; the other formats have an odd number of 32-bit words per unit.
template <int TYPE> __device__ __forceinline__ void load_unit(const uint8_t * row, int u, uint32_t * w) {
    constexpr int UW = QTraits<TYPE>::UNIT_WORDS;
    if constexpr (TYPE == DT_Q5_1) {
        const uint2 * p = reinterpret_cast<const uint2 *>(row) + (size_t) u * 3;
#pragma unroll
        for (int i = 0; i < 3; i++) { const uint2 v = p[i]; w[2 * i] = v.x; w[2 * i + 1] = v.y; }
    } else {
        const uint32_t * p = reinterpret_cast<const uint32_t *>(row) + (size_t) u * UW;
#pragma unroll
        for (int i = 0; i < UW; i++) w[i] = p[i];
    }
}

// Cooperative staging of one activation column by the 256 consumer threads: the operand the reference's CPU path
// would multiply with (ggml-cpu.c:253-311 `vec_dot_type`): Q8_0 / Q8_1 blocks for quantised weights (x86 flavour of
// quantize_row_q8_0 / q8_1, ggml-cpu-quants.c:781-846, 1085-1160; one thread per 32-element block), fp16 for F16
// weights, fp32 for F32 weights. PRO_LAYERNORM applies rwkv_layer_norm (rwkv_operators.inc:93-97) on the fly.
// PER_BLOCK (single-column launches): one thread quantises a whole 32-element block instead of 8 lanes sharing it --
// the two IEEE divisions, the scale and the sums once per 32 elements instead of once per 4, no shuffles; ~4x fewer instructions for
// a stage that is instruction-bound. The staged bytes are identical: the maximum and the integer sum of a block do
// not depend on the order they are taken in.
// TYPE_HINT: the weight type when the whole launch has one (a compile-time constant: the other formats' code is not generated), else -1.
// HAS_LN = false: the launch has no PRO_LAYERNORM problem (every launch but the head): the LayerNorm code, ~1 500 of the 4 200
// instructions of a per-format instantiation, is not generated.
template <int UNR = 4, bool PER_BLOCK = false, int TYPE_HINT = -1, bool HAS_LN = true>     // UNR: float4 loads a thread keeps in flight per round of the quantising loop
static __device__ void stage_column(const GemvProblem & P, int col_index, uint8_t * col, double * red_d) {
    const int K = P.K, tid = threadIdx.x;
    const int ptype = TYPE_HINT >= 0 ? TYPE_HINT : P.type;
    const float * x = P.x + (long long) col_index * P.ldx;
    float mean = 0.f, rstd = 1.f;
    const bool ln = HAS_LN && P.pro == PRO_LAYERNORM;
    if (ln) {
        const int lane = tid & 31, warp = tid >> 5;
        double s = 0;
        for (int k = tid; k < K; k += CONSUMER_THREADS) s += (double) x[k];
        s = warp_sum_double(s);
        if (lane == 0) red_d[warp] = s;
        consumer_barrier();
        if (tid == 0) { double t = 0; for (int i = 0; i < CONSUMER_WARPS; i++) t += red_d[i]; red_d[CONSUMER_WARPS] = t; }
        consumer_barrier();
        mean = (float) (red_d[CONSUMER_WARPS] / K);
        double s2 = 0;
        for (int k = tid; k < K; k += CONSUMER_THREADS) { float v = x[k] - mean; s2 += (double) (v * v); }
        s2 = warp_sum_double(s2);
        consumer_barrier();
        if (lane == 0) red_d[warp] = s2;
        consumer_barrier();
        if (tid == 0) { double t = 0; for (int i = 0; i < CONSUMER_WARPS; i++) t += red_d[i]; red_d[CONSUMER_WARPS] = t; }
        consumer_barrier();
        rstd = 1.0f / sqrtf((float) (red_d[CONSUMER_WARPS] / K) + 1e-5f);
    }
    auto norm = [&](float v, int k) -> float {
        return ln ? __fadd_rn(__fmul_rn(__fmul_rn(v - mean, rstd), P.ln_w[k]), P.ln_b[k]) : v;
    };
    if (ptype == DT_F32) {
        float * d = reinterpret_cast<float *>(col);
        for (int k = tid; k < K; k += CONSUMER_THREADS) d[k] = norm(x[k], k);
    } else if (ptype == DT_F16) {
        __half * d = reinterpret_cast<__half *>(col);
        for (int k = tid; k < K; k += CONSUMER_THREADS) d[k] = __float2half_rn(norm(x[k], k));
    } else {
        const bool has_min = (ptype == DT_Q4_1 || ptype == DT_Q5_1);
        const int UB = has_min ? 1 : 2;
        const int nblk = K / 32, nunits = (nblk + UB - 1) / UB;
        if constexpr (PER_BLOCK) {
            // two blocks per thread and round (threads tid and tid + 256 blocks apart), all 16 float4 loads issued before the first use
            for (int blk0 = tid; blk0 < nblk; blk0 += 2 * CONSUMER_THREADS) {
                float4 v[2][8];
#pragma unroll
                for (int r = 0; r < 2; r++) {
                    const int blk = blk0 + r * CONSUMER_THREADS;
#pragma unroll
                    for (int j = 0; j < 8; j++)
                        v[r][j] = (blk < nblk) ? *reinterpret_cast<const float4 *>(x + (size_t) blk * 32 + j * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
#pragma unroll
                for (int r = 0; r < 2; r++) {
                    const int blk = blk0 + r * CONSUMER_THREADS;
                    if (blk >= nblk) break;
                    float amax = 0.f;
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        float4 & t = v[r][j];
                        if (ln) { const int k = blk * 32 + j * 4; t.x = norm(t.x, k); t.y = norm(t.y, k + 1); t.z = norm(t.z, k + 2); t.w = norm(t.w, k + 3); }
                        amax = fmaxf(amax, fmaxf(fmaxf(fabsf(t.x), fabsf(t.y)), fmaxf(fabsf(t.z), fabsf(t.w))));
                    }
                    const float d32 = amax / 127.0f;
                    const float id = (amax != 0.0f) ? 127.0f / amax : 0.0f;
                    int isum = 0, words[8];
#pragma unroll
                    for (int j = 0; j < 8; j++) {
                        const float4 t = v[r][j];
                        const int q0 = __float2int_rn(t.x * id), q1 = __float2int_rn(t.y * id), q2 = __float2int_rn(t.z * id), q3 = __float2int_rn(t.w * id);
                        isum += q0 + q1 + q2 + q3;
                        words[j] = (q0 & 0xFF) | ((q1 & 0xFF) << 8) | ((q2 & 0xFF) << 16) | ((q3 & 0xFF) << 24);
                    }
                    const int u = blk / UB, bi = blk % UB;
                    *reinterpret_cast<int4 *>(col + ((size_t) (bi * 2 + 0) * nunits + u) * 16) = make_int4(words[0], words[1], words[2], words[3]);
                    *reinterpret_cast<int4 *>(col + ((size_t) (bi * 2 + 1) * nunits + u) * 16) = make_int4(words[4], words[5], words[6], words[7]);
                    ActScale a;
                    a.d = round_to_half(d32);
                    a.s = has_min ? round_to_half(d32 * (float) isum) : (float) isum;
                    *reinterpret_cast<ActScale *>(col + (size_t) nunits * UB * 32 + ((size_t) bi * nunits + u) * 8) = a;
                }
            }
            return;
        }
        // 8 lanes per 32-element block, one float4 each: coalesced loads, amax / sum over the 8 lanes by shuffles
        const int sub = tid & 7;
        // loads of UNR iterations are issued together: the loop is L2-latency bound, not math bound
        const int kpad = (K + 127) & ~127;
        for (int base0 = tid * 4; base0 < kpad; base0 += CONSUMER_THREADS * 4 * UNR) {
            float4 tv[UNR];
#pragma unroll
            for (int q = 0; q < UNR; q++) {
                const int base = base0 + q * CONSUMER_THREADS * 4;
                tv[q] = (base < K) ? *reinterpret_cast<const float4 *>(x + base) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int q = 0; q < UNR; q++) {
                const int base = base0 + q * CONSUMER_THREADS * 4;
                if (base >= kpad) break;                     // warp-uniform
                const bool live = base < K;
                float4 t = tv[q];
                if (ln && live) { t.x = norm(t.x, base); t.y = norm(t.y, base + 1); t.z = norm(t.z, base + 2); t.w = norm(t.w, base + 3); }
                float amax = fmaxf(fmaxf(fabsf(t.x), fabsf(t.y)), fmaxf(fabsf(t.z), fabsf(t.w)));
                amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
                amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
                amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
                const float d32 = amax / 127.0f;
                const float id = (amax != 0.0f) ? 127.0f / amax : 0.0f;
                const int q0 = __float2int_rn(t.x * id), q1 = __float2int_rn(t.y * id), q2 = __float2int_rn(t.z * id), q3 = __float2int_rn(t.w * id);
                int isum = q0 + q1 + q2 + q3;
                isum += __shfl_xor_sync(0xffffffffu, isum, 1);
                isum += __shfl_xor_sync(0xffffffffu, isum, 2);
                isum += __shfl_xor_sync(0xffffffffu, isum, 4);
                if (live) {
                    const int blk = base >> 5, u = blk / UB, bi = blk % UB, h = sub >> 2, i = sub & 3;
                    const int word = (q0 & 0xFF) | ((q1 & 0xFF) << 8) | ((q2 & 0xFF) << 16) | ((q3 & 0xFF) << 24);
                    *reinterpret_cast<int *>(col + ((size_t) (bi * 2 + h) * nunits + u) * 16 + i * 4) = word;
                    if (sub == 0) {
                        ActScale a;
                        a.d = round_to_half(d32);
                        a.s = has_min ? round_to_half(d32 * (float) isum) : (float) isum;
                        *reinterpret_cast<ActScale *>(col + (size_t) nunits * UB * 32 + ((size_t) bi * nunits + u) * 8) = a;
                    }
                }
            }
        }
    }
}

// Row partials of a WK > 1 tile: summed in warp order, epilogue, store. Thread i owns (row i / nc, column i % nc) and
// fetched that element's epilogue operands at the start of the tile (rows * nc <= 256 = the consumer thread count).
template <int NC>
__device__ __forceinline__ void finish_split_rows(const GemvProblem & P, const float * red_t, int row0, int rows, int c0, int nc, EpiOperands pre) {
    const int WK = P.wk;
    const int i = threadIdx.x;
    if (i < rows * nc) {
        const int r = i / nc, c = i % nc;
        float v = 0.f;
        for (int w = 0; w < WK; w++) v += red_t[(r * CONSUMER_WARPS + w) * NC + c];
        P.y[(long long) (c0 + c) * P.ldy + row0 + r] = apply_epilogue(P, v, pre.a, pre.b);
    }
}

// Lane mapping shared by both consumers. A row's K-slice is cut into ITEMS (quant units / 8-half chunks / 4-float
// chunks). G = P.g lanes (a power of two) cooperate on one row, so a warp works on 32/G rows at once: G = 32 for long
// rows, smaller for the short rows of the LoRA matrices (K = 64..320), which would otherwise leave most lanes idle.
// Lane `sub` of a row group takes items sub, sub+G, ... of its slice; the G partial sums are combined by an
// xor-butterfly over offsets G/2 .. 1 -- the summation tree of a row is a function of (type, K) only.
struct LaneMap {
    int G, RPS, sub, rs;      // lanes per row, rows per warp step, my lane within the row group, my row slot
    int WK, WR, wk, wr;
};
__device__ __forceinline__ LaneMap lane_map(const GemvProblem & P) {
    LaneMap m;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    m.G = P.g; m.RPS = 32 / m.G; m.sub = lane & (m.G - 1); m.rs = lane / m.G;
    m.WK = P.wk; m.WR = CONSUMER_WARPS / m.WK; m.wk = warp % m.WK; m.wr = warp / m.WK;
    return m;
}
__device__ __forceinline__ float group_sum(float v, int G) {
    for (int o = G >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ---- Q4_K / Q5_K rows against Q8_K activation columns (gemv_kquant.cu) ------------------------------------------------------
// Staged column: qs[nsb][256] (int8), then d[nsb] (float), then bsums[nsb][16] (int16, sums of 16 consecutive qs).
__host__ __device__ inline size_t kq_act_bytes_per_column(int K) {
    const size_t nsb = (size_t) K / QK_K;
    return (nsb * (QK_K + 4 + 32) + 15) & ~(size_t) 15;
}
// Lane l of the warp (G = 32) takes sub-block l % 8 of super-blocks wk*per + l/8, + 4, ... The scale x sub-block dot and the
// min x bsums of a super-block are exact integers summed over its 8 lanes; the lane of sub-block 0 then adds
// y.d*fp16(d) * sum - y.d*fp16(dmin) * msum to its partial, as ggml_vec_dot_q{4,5}_K_q8_K combines a super-block.
template <int TYPE, int NC>
__device__ __forceinline__ void row_partial_kq(const uint8_t * wrow, const uint8_t * act, size_t colb, int nc, int K, const LaneMap & m, float (&acc)[NC]) {
    constexpr int BB = TYPE == DT_Q4_K ? 144 : 176, QS = TYPE == DT_Q4_K ? 16 : 48;
    const int nsb = K / QK_K, per = (nsb + m.WK - 1) / m.WK;
    const int sb0 = m.wk * per, sb1 = min(nsb, sb0 + per);
    const int j = m.sub & 7;
#pragma unroll
    for (int c = 0; c < NC; c++) acc[c] = 0.f;
    for (int s0 = sb0; s0 < sb1; s0 += 4) {                      // warp-uniform: every lane takes part in the shuffles
        const bool live = s0 + (m.sub >> 3) < sb1;
        const int s = live ? s0 + (m.sub >> 3) : s0;
        const uint8_t * blk = wrow + (size_t) s * BB;
        const uint32_t dm = *reinterpret_cast<const uint32_t *>(blk);
        int sc, mn;
        kquant_scale_min(blk + 4, j, sc, mn);
        const uint4 qa = *reinterpret_cast<const uint4 *>(blk + QS + 32 * (j >> 1)), qb = *reinterpret_cast<const uint4 *>(blk + QS + 32 * (j >> 1) + 16);
        uint32_t w[8] = {qa.x, qa.y, qa.z, qa.w, qb.x, qb.y, qb.z, qb.w};
        const int shift = 4 * (j & 1);
#pragma unroll
        for (int i = 0; i < 8; i++) w[i] = (w[i] >> shift) & 0x0F0F0F0Fu;
        if constexpr (TYPE == DT_Q5_K) {
            const uint4 ha = *reinterpret_cast<const uint4 *>(blk + 16), hb = *reinterpret_cast<const uint4 *>(blk + 32);
            const uint32_t h[8] = {ha.x, ha.y, ha.z, ha.w, hb.x, hb.y, hb.z, hb.w};
#pragma unroll
            for (int i = 0; i < 8; i++) w[i] |= ((h[i] >> j) & 0x01010101u) << 4;
        }
#pragma unroll
        for (int c = 0; c < NC; c++) if (c < nc) {
            const uint8_t * col = act + c * colb;
            const int4 xa = *reinterpret_cast<const int4 *>(col + (size_t) s * QK_K + 32 * j), xb = *reinterpret_cast<const int4 *>(col + (size_t) s * QK_K + 32 * j + 16);
            int dot = __dp4a((int) w[0], xa.x, 0);
            dot = __dp4a((int) w[1], xa.y, dot); dot = __dp4a((int) w[2], xa.z, dot); dot = __dp4a((int) w[3], xa.w, dot);
            dot = __dp4a((int) w[4], xb.x, dot); dot = __dp4a((int) w[5], xb.y, dot); dot = __dp4a((int) w[6], xb.z, dot); dot = __dp4a((int) w[7], xb.w, dot);
            const short2 bp = *reinterpret_cast<const short2 *>(col + (size_t) nsb * (QK_K + 4) + (size_t) s * 32 + 4 * j);
            int isum = dot * sc, msum = ((int) bp.x + (int) bp.y) * mn;
#pragma unroll
            for (int o = 1; o < 8; o <<= 1) { isum += __shfl_xor_sync(0xffffffffu, isum, o); msum += __shfl_xor_sync(0xffffffffu, msum, o); }
            if (live && j == 0) {
                const float yd = reinterpret_cast<const float *>(col + (size_t) nsb * QK_K)[s];
                const float d = __fmul_rn(yd, __half2float(__ushort_as_half((unsigned short) (dm & 0xFFFFu))));
                const float dmin = __fmul_rn(yd, __half2float(__ushort_as_half((unsigned short) (dm >> 16))));
                acc[c] = __fadd_rn(acc[c], __fsub_rn(__fmul_rn(d, (float) isum), __fmul_rn(dmin, (float) msum)));
            }
        }
    }
}

// One row's lane partials for NC activation columns in shared memory (colb bytes apart), the lane map's order: lane `sub` of
// warp slice `wk` takes items wk * per + sub, + G, ... (quantised types: units, each block in order). acc[] starts at 0 and is
// summed by group_sum, then across the WK warps of the row in warp order. The streaming GEMV and the fused v6 LoRA kernels
// (glue.cu, wkv.cu) all compute a row through this function, so their bits agree.
template <int TYPE, int NC>
__device__ __forceinline__ void row_partial(const uint8_t * wrow, const uint8_t * act, size_t colb, int nc, int K, const LaneMap & m, float (&acc)[NC]) {
#pragma unroll
    for (int c = 0; c < NC; c++) acc[c] = 0.f;
    if constexpr (TYPE == DT_F32) {
        const int n4 = K / 4, per = (n4 + m.WK - 1) / m.WK, end = min(n4, (m.wk + 1) * per);
        for (int i = m.wk * per + m.sub; i < end; i += m.G) {
            const float4 wv = reinterpret_cast<const float4 *>(wrow)[i];
#pragma unroll
            for (int c = 0; c < NC; c++) if (c < nc) {
                const float4 xv = reinterpret_cast<const float4 *>(act + c * colb)[i];
                acc[c] = __fmaf_rn(wv.x, xv.x, acc[c]); acc[c] = __fmaf_rn(wv.y, xv.y, acc[c]);
                acc[c] = __fmaf_rn(wv.z, xv.z, acc[c]); acc[c] = __fmaf_rn(wv.w, xv.w, acc[c]);
            }
        }
        if (m.wk == m.WK - 1) for (int k = n4 * 4 + m.sub; k < K; k += m.G) {
            const float wf = reinterpret_cast<const float *>(wrow)[k];
#pragma unroll
            for (int c = 0; c < NC; c++) if (c < nc) acc[c] = __fmaf_rn(wf, reinterpret_cast<const float *>(act + c * colb)[k], acc[c]);
        }
    } else if constexpr (TYPE == DT_F16) {
        const int n8 = K / 8, per = (n8 + m.WK - 1) / m.WK, end = min(n8, (m.wk + 1) * per);
        for (int i = m.wk * per + m.sub; i < end; i += m.G) {
            const uint4 wv = reinterpret_cast<const uint4 *>(wrow)[i];
            const __half2 * wh = reinterpret_cast<const __half2 *>(&wv);
#pragma unroll
            for (int c = 0; c < NC; c++) if (c < nc) {
                const uint4 xv = reinterpret_cast<const uint4 *>(act + c * colb)[i];
                const __half2 * xh = reinterpret_cast<const __half2 *>(&xv);
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const float2 wf = __half22float2(wh[q]), xf = __half22float2(xh[q]);
                    acc[c] = __fmaf_rn(wf.x, xf.x, acc[c]);
                    acc[c] = __fmaf_rn(wf.y, xf.y, acc[c]);
                }
            }
        }
        if (m.wk == m.WK - 1) for (int k = n8 * 8 + m.sub; k < K; k += m.G) {
            const float wf = __half2float(reinterpret_cast<const __half *>(wrow)[k]);
#pragma unroll
            for (int c = 0; c < NC; c++) if (c < nc) acc[c] = __fmaf_rn(wf, __half2float(reinterpret_cast<const __half *>(act + c * colb)[k]), acc[c]);
        }
    } else if constexpr (TYPE == DT_Q4_K || TYPE == DT_Q5_K) {
        row_partial_kq<TYPE, NC>(wrow, act, colb, nc, K, m, acc);
    } else {
        using TR = QTraits<TYPE>;
        constexpr int UB = TR::UNIT_BLOCKS, UW = TR::UNIT_WORDS;
        const int nblk = K / 32, nunits = (nblk + UB - 1) / UB;
        const int upw = (nunits + m.WK - 1) / m.WK, u_end = min(nunits, (m.wk + 1) * upw);
        // same block order per lane as consume_quant_regs: u = wk*upw + sub + G j, bi = 0..UB-1
        for (int u = m.wk * upw + m.sub; u < u_end; u += m.G) {
            uint32_t w[UW];
            load_unit<TYPE>(wrow, u, w);
#pragma unroll
            for (int bi = 0; bi < UB; bi++) {
                if (u * UB + bi < nblk) {
                    BlockQ bq;
                    decode_block<TYPE>(w, bi, bq);
#pragma unroll
                    for (int c = 0; c < NC; c++) if (c < nc) {
                        const uint8_t * col = act + c * colb;
                        const int4 lo = *act_q_ptr<UB>(col, nunits, u, bi, 0), hi = *act_q_ptr<UB>(col, nunits, u, bi, 1);
                        const int a8[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
                        acc[c] = block_dot<TYPE>(bq, a8, *act_s_ptr<UB>(col, nunits, u, bi), acc[c]);
                    }
                }
            }
        }
    }
}

// Rows [0, n_rows) of P starting at row0, held in shared memory (P.pitch bytes apart), against one activation column staged by
// stage_column, for a problem whose plan has WK == 1 (gemv_tma_plan): the CTA's warps take row groups of 32 / G rows in turn,
// and out[r] = epilogue(row row0 + r). Used by kernels that fold a small GEMV into themselves; blockDim.x is a multiple of 32.
template <int TYPE>
__device__ __forceinline__ void rows_dot(const GemvProblem & P, const uint8_t * rows, int n_rows, int row0, const uint8_t * act, float * out) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    LaneMap m;
    m.G = P.g; m.RPS = 32 / m.G; m.sub = lane & (m.G - 1); m.rs = lane / m.G;
    m.WK = 1; m.WR = nwarps; m.wk = 0; m.wr = warp;
    for (int rb = warp * m.RPS; rb < n_rows; rb += nwarps * m.RPS) {
        const int r = rb + m.rs;
        const bool store = r < n_rows && m.sub == 0;
        EpiOperands e; e.a = 0.f; e.b = 0.f;
        if (store) e = prefetch_epilogue(P, row0 + r, 0);
        float acc[1];
        row_partial<TYPE, 1>(rows + (size_t) min(r, n_rows - 1) * (size_t) P.pitch, act, 0, 1, P.K, m, acc);
        const float v = group_sum(acc[0], m.G);
        if (store) out[r] = apply_epilogue(P, v, e.a, e.b);
    }
}

// ---- consumer: quantised weights, one column, activations in registers (the decode hot path) ------------------
template <int TYPE, bool GUARD = false>
__device__ void consume_quant_regs(Shared & sh, uint8_t * ring, uint32_t stage_bytes, const uint8_t * act, int c0, float * red, int it0, int my_tiles,
                                   int first_tile, int tile_stride) {
    using TR = QTraits<TYPE>;
    constexpr int UB = TR::UNIT_BLOCKS, UW = TR::UNIT_WORDS;
    constexpr int MAXU = MAX_BLOCKS_PER_LANE / UB;
    const GemvProblem & P = sh.P;
    const LaneMap m = lane_map(P);
    const int lane = threadIdx.x & 31;
    const int nblk = P.K / 32, nunits = (nblk + UB - 1) / UB;
    const int upw = (nunits + m.WK - 1) / m.WK;                // units per warp slice
    const int u_end = min(nunits, (m.wk + 1) * upw);

    // my activation blocks -> registers, once. Slots past the slice (or past K) hold zeros and point at unit 0,
    // so the row loop below needs no branches: their contribution is exactly +0.
    int a8[MAXU][UB][8];
    ActScale as[MAXU][UB];
    int ucl[MAXU];
#pragma unroll
    for (int j = 0; j < MAXU; j++) {
        const int u = m.wk * upw + m.sub + m.G * j;
        const bool live_u = u < u_end;
        ucl[j] = live_u ? u : 0;
#pragma unroll
        for (int bi = 0; bi < UB; bi++) {
            const bool live = live_u && (u * UB + bi) < nblk;
            const int4 lo = live ? *act_q_ptr<UB>(act, nunits, u, bi, 0) : make_int4(0, 0, 0, 0);
            const int4 hi = live ? *act_q_ptr<UB>(act, nunits, u, bi, 1) : make_int4(0, 0, 0, 0);
            a8[j][bi][0] = lo.x; a8[j][bi][1] = lo.y; a8[j][bi][2] = lo.z; a8[j][bi][3] = lo.w;
            a8[j][bi][4] = hi.x; a8[j][bi][5] = hi.y; a8[j][bi][6] = hi.z; a8[j][bi][7] = hi.w;
            ActScale z; z.d = 0.f; z.s = 0.f;
            as[j][bi] = live ? *act_s_ptr<UB>(act, nunits, u, bi) : z;
        }
    }

    float * const ycol = P.y + (long long) c0 * P.ldy;
    for (int i0 = 0; i0 < my_tiles; i0++) {
        const int it = it0 + i0;                       // ring position continues across column groups
        const int tile = first_tile + i0 * tile_stride;
        const int row0 = tile * P.tile_rows;
        const int rows = min(P.tile_rows, P.M - row0);
        const int s = it % NSTAGES;
        // epilogue operands of this tile, requested before we block on the weights
        EpiOperands pre; pre.a = 0.f; pre.b = 0.f;
        if (m.WK == 1) {          // lane l <-> l-th output of this warp in this tile: step l / RPS, row slot l % RPS
            const int r = ((lane / m.RPS) * m.WR + m.wr) * m.RPS + (lane % m.RPS);
            if (r < rows) pre = prefetch_epilogue(P, row0 + r, c0);
        } else if ((int) threadIdx.x < rows) {
            pre = prefetch_epilogue(P, row0 + (int) threadIdx.x, c0);
        }
        mbar_wait_t<GUARD>(&sh.full[s], (uint32_t) ((it / NSTAGES) & 1));
        const uint8_t * stage = ring + (size_t) s * stage_bytes;
        float * red_t = red + (size_t) (it & 1) * MAX_TILE_ROWS * CONSUMER_WARPS;
        int step = 0;
        for (int rb = m.wr * m.RPS; rb < rows; rb += m.WR * m.RPS, step++) {
            const int r = rb + m.rs;
            const uint8_t * wrow = stage + (size_t) min(r, rows - 1) * (size_t) P.pitch;   // idle row slots recompute the last row
            float acc = 0.f;
#pragma unroll
            for (int j = 0; j < MAXU; j++) {
                uint32_t w[UW];
                load_unit<TYPE>(wrow, ucl[j], w);
#pragma unroll
                for (int bi = 0; bi < UB; bi++) {
                    BlockQ bq;
                    decode_block<TYPE>(w, bi, bq);
                    acc = block_dot<TYPE>(bq, a8[j][bi], as[j][bi], acc);
                }
            }
            acc = group_sum(acc, m.G);
            if (m.WK == 1) {
                const int src = (step * m.RPS + m.rs) & 31;
                const float ea = __shfl_sync(0xffffffffu, pre.a, src), eb = __shfl_sync(0xffffffffu, pre.b, src);
                if (m.sub == 0 && r < rows) ycol[row0 + r] = apply_epilogue(P, acc, ea, eb);
            } else if (lane == 0) {
                red_t[r * CONSUMER_WARPS + m.wk] = acc;
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sh.empty[s]);
        if (m.WK > 1) {
            consumer_barrier();
            finish_split_rows<1>(P, red_t, row0, rows, c0, 1, pre);
        }
        if (i0 == 0) trace_mark(sh.trace, 2);
        if (i0 == 2) trace_mark(sh.trace, 3);
    }
}

// ---- consumer: activations in shared memory (F16 / F32 weights, or several columns at once) -------------------
template <int TYPE, int NC, bool GUARD = false>
__device__ void consume_smem(Shared & sh, uint8_t * ring, uint32_t stage_bytes, const uint8_t * act, size_t colb, int c0, int nc, float * red, int it0,
                             int my_tiles, int first_tile, int tile_stride) {
    const GemvProblem & P = sh.P;
    const LaneMap m = lane_map(P);
    const int lane = threadIdx.x & 31;
    const int K = P.K;
    for (int i0 = 0; i0 < my_tiles; i0++) {
        const int it = it0 + i0;
        const int tile = first_tile + i0 * tile_stride;
        const int row0 = tile * P.tile_rows;
        const int rows = min(P.tile_rows, P.M - row0);
        const int s = it % NSTAGES;
        mbar_wait_t<GUARD>(&sh.full[s], (uint32_t) ((it / NSTAGES) & 1));
        const uint8_t * stage = ring + (size_t) s * stage_bytes;
        float * red_t = red + (size_t) (it & 1) * MAX_TILE_ROWS * CONSUMER_WARPS * NC;
        // WK > 1: thread i owns output (row i / nc, column i % nc) of the tile and fetches its epilogue operands now
        EpiOperands pre; pre.a = 0.f; pre.b = 0.f;
        if (m.WK > 1 && (int) threadIdx.x < rows * nc) pre = prefetch_epilogue(P, row0 + (int) threadIdx.x / nc, c0 + (int) threadIdx.x % nc);
        for (int rb = m.wr * m.RPS; rb < rows; rb += m.WR * m.RPS) {
            const int r = rb + m.rs;
            const bool live_row = r < rows;
            const uint8_t * wrow = stage + (size_t) min(r, rows - 1) * (size_t) P.pitch;
            // WK == 1: the lane that will store (sub == 0) fetches the epilogue operands of its row before the dot product
            EpiOperands e[NC];
#pragma unroll
            for (int c = 0; c < NC; c++) {
                e[c].a = 0.f; e[c].b = 0.f;
                if (m.WK == 1 && m.sub == 0 && live_row && c < nc) e[c] = prefetch_epilogue(P, row0 + r, c0 + c);
            }
            float acc[NC];
            row_partial<TYPE, NC>(wrow, act, colb, nc, K, m, acc);
#pragma unroll
            for (int c = 0; c < NC; c++) {
                const float v = group_sum(acc[c], m.G);
                if (m.WK == 1) {
                    if (m.sub == 0 && live_row && c < nc) P.y[(long long) (c0 + c) * P.ldy + row0 + r] = apply_epilogue(P, v, e[c].a, e[c].b);
                } else if (lane == 0 && c < nc) {
                    red_t[(r * CONSUMER_WARPS + m.wk) * NC + c] = v;
                }
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&sh.empty[s]);
        if (m.WK > 1) {
            consumer_barrier();
            finish_split_rows<NC>(P, red_t, row0, rows, c0, nc, pre);
        }
    }
}

}  // namespace tma
}  // namespace rwkv
