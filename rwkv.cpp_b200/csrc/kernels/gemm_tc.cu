// Chunked-prefill contraction on the Hopper tensor cores (wgmma):  Y[M, T] = epilogue(W[M, K] . X[K, T])  for T >= 32.
//
// This is the one place of the eval path where the chunk x embedding contraction is dense enough for tensor cores
// (SURVEY.md 8d).
//
//   * Weights for this path are expanded ONCE, at load time, to fp16 -- (q - offset) * d + m rounded once -- and stored
//     tile-major in the canonical no-swizzle K-major layout of the wgmma shared-memory descriptors: one [128 rows x 64 k]
//     operand block = 16 KB contiguous, core matrices (8 rows x 16 bytes) back to back. 2 bytes per weight: 17 GB at 7B next
//     to the 6 GB the decode path streams, which fits the 80 GB of an H100.
//   * Warp specialisation: ONE producer thread moves both operands with 1-D bulk copies (cp.async.bulk; no tensor map needed
//     because the global layout already is the shared-memory layout) into a ring of up to 8 stages; two consumer warpgroups
//     each own 64 rows of the 128-row tile and issue wgmma.mma_async m64nNk16 (A and B from shared memory, N = tokens padded to
//     16 in pieces of at most 64, fp32 accumulator in registers), then hand the stage back through an mbarrier once
//     wgmma.wait_group says the MMAs reading it are done. One mbarrier pair per stage, no __syncthreads in the K loop.
//     After the K loop the accumulator goes through the (by then idle) ring memory to a thread-per-row epilogue that applies
//     the GEMV's fused epilogues with column-major stores.
//   * At T = 128 the contraction is HBM-bound on the fp16 weights (128 FLOP per weight byte, below the H100's dense fp16
//     ridge of ~295): the target is the copy bandwidth, not the tensor peak.
//   * Launches whose tiles would leave most SMs idle (4096-row matrices: 32 tiles; LoRA matrices: 1-2) are cut along K over a
//     thread-block CLUSTER of 2 / 4 / 8 CTAs per tile: every CTA parks its fp32 accumulator in its own ring memory, and after a
//     cluster barrier CTA r adds up columns [r * npad / c, ...) of all c accumulators through distributed shared memory, in rank
//     order (deterministic), and runs the fused epilogue on them. (Partial tiles through global memory, the last-arriving CTA
//     adding all of them, cost 128 threads x up to 512 dependent L2 round trips per launch.)
//
// Numerics: weights exactly as the file stores them, rounded once to fp16 after dequantisation; activations are fp16 of the
// reference's own operand values (convert_f16_kernel below); fp32 accumulation in the tensor core. Not bit-identical to the
// dp4a decode path, so the engine uses it only for passes of >= 32 tokens and never for F32 weights, which keeps every
// serial == sequence memcmp test of the reference (tests/test_eval_sequence_in_chunks.c: chunks of 1, 2, 8, 10) exact.
#include "gemv.h"
#include "quant_decode.cuh"

#include <cuda_fp16.h>
#include <cstring>

namespace rwkv {
namespace tc {

constexpr int TILE_M = 128;
constexpr int KSTEP = 64;                 // K elements per ring stage = 4 MMAs of K = 16
constexpr int CONSUMERS = 256;            // warps 0-7: two consumer warpgroups (tile rows 0-63, 64-127), then the epilogue
constexpr int PRODUCER_WARP = 8;
constexpr int THREADS = CONSUMERS + 32;
constexpr int MAX_STAGES = 8;
constexpr int MAX_N = 256;
constexpr uint32_t A_BYTES = TILE_M * KSTEP * 2;      // one weight operand block: 16 KB
constexpr uint32_t A_LBO = (TILE_M / 8) * 128;        // bytes between core matrices adjacent along K (16 row groups x 128 B)
// Parked accumulator in the ring memory: column-major [npad][PARK_LD] fp32. The 4-float pad puts the four columns one store of the
// wgmma fragment writes (2 * (lane % 4)) into different banks.
constexpr int PARK_LD = TILE_M + 4;

__device__ __forceinline__ uint32_t smem_u32(const void * p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t * bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
// Bounded wait: a descriptor or barrier mistake shows up as a trapped kernel, never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t * bar, uint32_t parity) {
    uint32_t done = 0;
    for (uint32_t spins = 0; !done; spins++) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
        if (spins > 256) __nanosleep(32);          // a waiting role must not steal issue slots from a co-resident kernel
        if (spins > (1u << 24)) __trap();
    }
}

__device__ __forceinline__ void mbar_arrive(uint64_t * bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t * bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_load(void * dst, const void * src, uint32_t bytes, uint64_t * bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
                 "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ uint32_t lds32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint2 lds64(uint32_t a) { uint2 v; asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a)); return v; }
__device__ __forceinline__ uint4 lds128(uint32_t a) {
    uint4 v; asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a)); return v;
}
// ---- wgmma wrappers (PTX ISA 8.0+, sm_90a) -------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }
// D[64 x N] (+)= A[64 x 16] . B[16 x N], fp16 operands from shared memory (both K-major), fp32 accumulator in registers: thread t of the
// warpgroup holds d[4 j + i] = D[16 (t / 32) + (t % 32) / 4 + 8 (i / 2)][8 j + 2 (t % 4) + i % 2].
template <int N> __device__ __forceinline__ void wgmma_f16(float * d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <> __device__ __forceinline__ void wgmma_f16<16>(float * d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_f16<32>(float * d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
          "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_f16<48>(float * d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %26, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, "
        "%20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
          "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
          "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_f16<64>(float * d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, "
        "%20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
          "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
          "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
          "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// wgmma shared-memory matrix descriptor, K-major, no swizzle (PTX ISA "Matrix Descriptor Format"; canonical layout
// ((8,n),(8,2)):((16 B, SBO),(2 B, LBO))):
//   element (row, k) lives at  start + (row % 8) * 16 + (row / 8) * SBO + (k / 8) * LBO   bytes
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t) ((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t) ((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t) ((sbo_bytes >> 4) & 0x3FFFu) << 32;
    return d;                    // base_offset 0, layout_type 0 = no swizzle
}

// Dynamic shared memory: `stages` ring slots of [A: 128 rows x 64 k fp16 = 16 KB][B: NPAD tokens x 64 k fp16], both in the
// canonical K-major no-swizzle layout: element (row, k) at (k / 8) * LBO + (row / 8) * 128 + (row % 8) * 16 + (k % 8) * 2 bytes,
// LBO = (rows / 8) * 128. After the K loop the ring holds the parked accumulator (PARK_LD).
struct TcShared {
    uint64_t full[MAX_STAGES], empty[MAX_STAGES];
    GemvProblem P;
    float colscale[MAX_N];
};

__device__ __forceinline__ float sigmoidf_(float v) { return 1.0f / (1.0f + expf(-v)); }

// Epilogue of a tile that was not cut along K: parked accumulator -> fused epilogue -> y, column-major stores (a warp writes 32
// consecutive rows of a column: 128-byte runs). Consumer thread t takes tile row t % 128 and every other 8-column group, starting at
// group t / 128. The accumulator is walked in a ROLLED loop of 8-column groups: fully unrolled epilogues of all ten kinds are
// ~143 KB of straight-line code that every launch executes once, cold, at the instruction-fetch rate of L2; eight columns per trip
// keeps a kind's body at 0.5-4 KB, fetched once and run many times.
struct EpiRow { float * y; long long ldy; const float * res; long long ldres; const float * gate; long long ldgate; float bias; };
template <int EPI> __device__ __forceinline__ void store_cols8(const EpiRow & e, const float (&acc)[8], const float * cs, int c0, int T) {
    // the residual / gate inputs of the group are requested before the first store: the output may alias the residual (x += ...)
    float rv[8], gv[8];
    if constexpr (EPI == EPI_ADD || EPI == EPI_MUL_ADD) {
#pragma unroll
        for (int j = 0; j < 8; j++) rv[j] = c0 + j < T ? e.res[(long long) (c0 + j) * e.ldres] : 0.f;
    }
    if constexpr (EPI == EPI_MUL_ADD) {
#pragma unroll
        for (int j = 0; j < 8; j++) gv[j] = c0 + j < T ? e.gate[(long long) (c0 + j) * e.ldgate] : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 8; j++) {
        const int col = c0 + j;
        if (col >= T) break;
        float v = acc[j] * cs[col];
        if constexpr (EPI == EPI_SIGMOID) v = sigmoidf_(v);
        else if constexpr (EPI == EPI_SILU) v = v / (1.0f + expf(-v));
        else if constexpr (EPI == EPI_TANH) v = tanhf(v);
        else if constexpr (EPI == EPI_RELU_SQR) { const float r = fmaxf(v, 0.0f); v = r * r; }
        else if constexpr (EPI == EPI_ADD) v = rv[j] + v;
        else if constexpr (EPI == EPI_MUL_ADD) v = rv[j] + gv[j] * v;
        else if constexpr (EPI == EPI_BIAS_EXPNEGEXP) v = expf(-expf(v + e.bias));
        else if constexpr (EPI == EPI_BIAS_SIGMOID) v = sigmoidf_(v + e.bias);
        else if constexpr (EPI == EPI_BIAS_W7) v = expf(sigmoidf_(v + e.bias) * -0.606531f);
        e.y[(long long) col * e.ldy] = v;
    }
}
__device__ __noinline__ void tc_epilogue_rows(const GemvProblem & Psh, const float * cs, const float * park, int row0, int npad, int T) {
    const int r = threadIdx.x & (TILE_M - 1);
    const int row = row0 + r;
    if (row >= Psh.M) return;
    const int epi = Psh.epi;
    EpiRow e;
    e.y = Psh.y + row; e.ldy = Psh.ldy;
    e.res = Psh.res ? Psh.res + row : nullptr; e.ldres = Psh.ldres;
    e.gate = Psh.gate ? Psh.gate + row : nullptr; e.ldgate = Psh.ldgate;
    e.bias = Psh.bias ? Psh.bias[row] : 0.f;
#pragma unroll 1
    for (int c0 = 8 * (int) (threadIdx.x / TILE_M); c0 < npad && c0 < T; c0 += 16) {
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; j++) acc[j] = park[(c0 + j) * PARK_LD + r];
        switch (epi) {
            case EPI_SIGMOID: store_cols8<EPI_SIGMOID>(e, acc, cs, c0, T); break;
            case EPI_SILU: store_cols8<EPI_SILU>(e, acc, cs, c0, T); break;
            case EPI_TANH: store_cols8<EPI_TANH>(e, acc, cs, c0, T); break;
            case EPI_RELU_SQR: store_cols8<EPI_RELU_SQR>(e, acc, cs, c0, T); break;
            case EPI_ADD: store_cols8<EPI_ADD>(e, acc, cs, c0, T); break;
            case EPI_MUL_ADD: store_cols8<EPI_MUL_ADD>(e, acc, cs, c0, T); break;
            case EPI_BIAS_EXPNEGEXP: store_cols8<EPI_BIAS_EXPNEGEXP>(e, acc, cs, c0, T); break;
            case EPI_BIAS_SIGMOID: store_cols8<EPI_BIAS_SIGMOID>(e, acc, cs, c0, T); break;
            case EPI_BIAS_W7: store_cols8<EPI_BIAS_W7>(e, acc, cs, c0, T); break;
            default: store_cols8<EPI_NONE>(e, acc, cs, c0, T); break;
        }
    }
}

// ---- K-split over a thread-block cluster --------------------------------------------------------------------------------------
__device__ __forceinline__ void cluster_sync_all() {      // every thread of every CTA of the cluster
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t map_to_cta(uint32_t local_smem_addr, uint32_t rank) {
    uint32_t r; asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank)); return r;
}
__device__ __forceinline__ float ld_dsmem(uint32_t addr) { float v; asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(v) : "r"(addr)); return v; }

// The consumer warpgroups' register accumulators -> the CTA's own ring memory, column-major [NPAD][PARK_LD] fp32 (wgmma_f16's fragment
// layout; warpgroup g holds tile rows 64 g .. 64 g + 63).
template <int NPAD> __device__ __forceinline__ void tc_park_accumulator(const float (&acc)[NPAD / 2], float * park) {
    const int t = threadIdx.x, lane = t & 31;
    const int r = 64 * (t / 128) + 16 * ((t / 32) & 3) + lane / 4;
    const int c = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < NPAD / 8; j++) {
        float * p = park + (8 * j + c) * PARK_LD + r;
        p[0] = acc[4 * j]; p[PARK_LD] = acc[4 * j + 1];
        p[8] = acc[4 * j + 2]; p[PARK_LD + 8] = acc[4 * j + 3];
    }
}
__device__ __forceinline__ float tc_epilogue_value(int epi, float v, float res, float gate, float bias) {
    switch (epi) {
        case EPI_SIGMOID: return sigmoidf_(v);
        case EPI_SILU: return v / (1.0f + expf(-v));
        case EPI_TANH: return tanhf(v);
        case EPI_RELU_SQR: { const float r = fmaxf(v, 0.0f); return r * r; }
        case EPI_ADD: return res + v;
        case EPI_MUL_ADD: return res + gate * v;
        case EPI_BIAS_EXPNEGEXP: return expf(-expf(v + bias));
        case EPI_BIAS_SIGMOID: return sigmoidf_(v + bias);
        case EPI_BIAS_W7: return expf(sigmoidf_(v + bias) * -0.606531f);
        default: return v;
    }
}
// After the cluster barrier: columns [rank * cpr, (rank + 1) * cpr) of the tile = sum over the cluster's accumulators in rank order ->
// fused epilogue -> y. Consumer thread t takes tile row t % 128 (loads from a peer and the stores to y are 128-byte runs) and every
// other group of four columns, starting at group t / 128. A ROLLED, software-pipelined loop: the loads of the next group (residual /
// gate out of L2, the peers' partial sums out of distributed shared memory) are in flight while the current one is summed and stored.
// A fully unrolled loop is thousands of straight-line instructions executed once, fetched from L2 one cache line at a time.
struct ReduceGroup { float part[4][8], res[4], gate[4]; };
__device__ __forceinline__ void tc_load_group(const GemvProblem & Psh, const uint32_t (&peer)[8], int csize, int row, bool live, int c0, int c_hi, ReduceGroup & g) {
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int c = min(c0 + j, c_hi - 1);
        g.res[j] = (live && Psh.res) ? Psh.res[(long long) c * Psh.ldres + row] : 0.f;
        g.gate[j] = (live && Psh.gate) ? Psh.gate[(long long) c * Psh.ldgate + row] : 0.f;
#pragma unroll
        for (int p = 0; p < 8; p++) g.part[j][p] = p < csize ? ld_dsmem(peer[p] + (uint32_t) c * (PARK_LD * 4u)) : 0.f;
    }
}
__device__ __noinline__ void tc_reduce_columns(const GemvProblem & Psh, const float * cs, const float * park, int row0, int npad, int T, int csize) {
    const int r = (int) threadIdx.x & (TILE_M - 1);
    const int row = row0 + r;
    const bool live = row < Psh.M;
    const uint32_t rank = cluster_ctarank();
    const int cpr = (npad + csize - 1) / csize;
    const int c_lo = (int) rank * cpr + 4 * (int) (threadIdx.x / TILE_M), c_hi = min(min(npad, T), (int) rank * cpr + cpr);
    if (c_lo >= c_hi) return;
    const int epi = Psh.epi;
    const float bias = (live && Psh.bias) ? Psh.bias[row] : 0.f;
    const uint32_t park0 = smem_u32(park) + (uint32_t) r * 4u;
    uint32_t peer[8];
#pragma unroll
    for (int p = 0; p < 8; p++) peer[p] = map_to_cta(park0, (uint32_t) (p < csize ? p : 0));
    ReduceGroup cur, nxt;
    tc_load_group(Psh, peer, csize, row, live, c_lo, c_hi, cur);
#pragma unroll 1
    for (int c0 = c_lo; c0 < c_hi; c0 += 8) {
        if (c0 + 8 < c_hi) tc_load_group(Psh, peer, csize, row, live, c0 + 8, c_hi, nxt);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const int c = c0 + j;
            if (c >= c_hi || !live) continue;
            float v = 0.f;
#pragma unroll
            for (int p = 0; p < 8; p++) if (p < csize) v += cur.part[j][p];
            Psh.y[(long long) c * Psh.ldy + row] = tc_epilogue_value(epi, v * cs[c], cur.res[j], cur.gate[j], bias);
        }
        cur = nxt;
    }
}

// 32 weights of one ggml block (or 32 f16 values) -> 4 x 16 bytes of fp16, element order 0..31
template <int TYPE> struct BlockRegs { uint32_t w[TYPE == DT_F16 ? 16 : (TYPE == DT_Q8_0 ? 9 : 6)]; };

// block `blk` of a raw row in shared memory (32-bit shared address) -> registers
template <int TYPE> __device__ __forceinline__ void read_block(uint32_t row, int blk, BlockRegs<TYPE> & r) {
    if constexpr (TYPE == DT_F16) {
#pragma unroll
        for (int i = 0; i < 4; i++) { const uint4 v = lds128(row + blk * 64 + i * 16); r.w[4 * i] = v.x; r.w[4 * i + 1] = v.y; r.w[4 * i + 2] = v.z; r.w[4 * i + 3] = v.w; }
    } else if constexpr (TYPE == DT_Q5_1) {          // 24-byte blocks on an 8-byte grid
#pragma unroll
        for (int i = 0; i < 3; i++) { const uint2 v = lds64(row + blk * 24 + i * 8); r.w[2 * i] = v.x; r.w[2 * i + 1] = v.y; }
    } else if constexpr (TYPE == DT_Q4_1) {          // 20-byte blocks on a 4-byte grid
#pragma unroll
        for (int i = 0; i < 5; i++) r.w[i] = lds32(row + blk * 20 + i * 4);
    } else {
        // 18 / 22 / 34-byte blocks start on a 2-byte grid: read whole words from the aligned-down address and realign
        constexpr int BB = QTraits<TYPE>::BLOCK_BYTES;
        constexpr int NW = BB / 4 + 1;
        const uint32_t start = (uint32_t) blk * BB;
        const uint32_t base = row + (start & ~3u);
        uint32_t t[NW];
#pragma unroll
        for (int i = 0; i < NW; i++) t[i] = lds32(base + i * 4);
        if (start & 2) {
#pragma unroll
            for (int i = 0; i < NW - 1; i++) r.w[i] = funnel16(t[i], t[i + 1]);
        } else {
#pragma unroll
            for (int i = 0; i < NW - 1; i++) r.w[i] = t[i];
        }
        if (NW - 1 < (int) (sizeof(r.w) / 4)) r.w[NW - 1] = (start & 2) ? (t[NW - 1] >> 16) : t[NW - 1];
    }
}

// Dequantise one block to 32 fp16 values in element order with packed-half arithmetic: the stored integer goes into
// the mantissa of 1024.0h (0x6400 | q == 1024 + q exactly), one HSUB2 removes 1024 (+ the -8 / -16 offset of the
// symmetric formats, + 128 for the sign-flipped bytes of Q8_0), one HFMA2 applies w = q * d + m with a single rounding
// (dequantize_row_q*, ggml-quants.c:255-363, rounded to fp16). ~70 instructions per block instead of ~300 in fp32.
template <int TYPE> __device__ __forceinline__ void block_to_half(const BlockRegs<TYPE> & r, uint4 out[4]) {
    if constexpr (TYPE == DT_F16) {
#pragma unroll
        for (int i = 0; i < 4; i++) out[i] = make_uint4(r.w[4 * i], r.w[4 * i + 1], r.w[4 * i + 2], r.w[4 * i + 3]);
    } else {
        BlockQ bq;
        decode_block<TYPE>(r.w, 0, bq);          // q[0..3]: elements 0..15, q[4..7]: elements 16..31, 4 per word
        const __half2 d2 = __float2half2_rn(bq.d), m2 = __float2half2_rn(bq.m);
        const float bias = 1024.0f + (float) QTraits<TYPE>::OFFSET + (TYPE == DT_Q8_0 ? 128.0f : 0.0f);
        const __half2 bias2 = __float2half2_rn(bias);
        uint32_t * o = reinterpret_cast<uint32_t *>(out);
#pragma unroll
        for (int i = 0; i < 8; i++) {
            uint32_t q = (uint32_t) bq.q[i];
            if (TYPE == DT_Q8_0) q ^= 0x80808080u;                 // signed byte -> byte + 128
            const uint32_t p0 = __byte_perm(q, 0x64646464u, 0x5140);   // [b0, 0x64, b1, 0x64] = halves (1024 + b0, 1024 + b1)
            const uint32_t p1 = __byte_perm(q, 0x64646464u, 0x7362);   // [b2, 0x64, b3, 0x64]
            __half2 h0 = __hfma2(__hsub2(*reinterpret_cast<const __half2 *>(&p0), bias2), d2, m2);
            __half2 h1 = __hfma2(__hsub2(*reinterpret_cast<const __half2 *>(&p1), bias2), d2, m2);
            o[2 * i] = *reinterpret_cast<uint32_t *>(&h0);
            o[2 * i + 1] = *reinterpret_cast<uint32_t *>(&h1);
        }
    }
}

struct TcBatch {
    int n, T, npad;                  // problems, tokens, tokens padded to a multiple of 16
    int stages;                     // ring depth, 2 .. MAX_STAGES
    const __half * act16[GEMV_MAX_PROBLEMS];   // canonical-layout fp16 activations per problem (convert_f16_kernel)
    const float * colscale[GEMV_MAX_PROBLEMS]; // [npad] power-of-two factor per token that the epilogue multiplies back in
    GemvProblem p[GEMV_MAX_PROBLEMS];          // first_cta / n_cta: CTA range of the problem = splits x tiles
    // Work decomposition. The launch runs in clusters of `cluster` CTAs (1, 2, 4 or 8). A problem is either cut along K into exactly
    // `cluster` splits -- its CTA (tile, split) = (local / cluster, local % cluster): the cluster IS the tile, split = cluster rank --
    // or not cut at all (splits = 1, CTA local = tile; its CTA range is padded to a multiple of the cluster size, the padding exits).
    int cluster;
    int tiles[GEMV_MAX_PROBLEMS], splits[GEMV_MAX_PROBLEMS], steps_per_split[GEMV_MAX_PROBLEMS];
    TraceRec * trace;
};

// One CTA = one 128-row tile (or one K-split of it), NPAD = batch.npad tokens.
template <int NPAD>
__global__ void __launch_bounds__(THREADS, 1) gemm_tc_kernel(const TcBatch batch) {
    extern __shared__ __align__(1024) uint8_t smem[];
    __shared__ TcShared sh;
    trace_begin(batch.trace);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    int pi = 0;
    for (int i = 1; i < batch.n; i++) if ((int) blockIdx.x >= batch.p[i].first_cta) pi = i;
    // padding CTAs of an un-split problem (its CTA range is rounded up to whole clusters): nothing to do, and nobody in their
    // cluster talks to them (cluster barriers and distributed shared memory are used by K-split tiles only)
    if (batch.splits[pi] == 1 && (int) blockIdx.x - batch.p[pi].first_cta >= batch.tiles[pi]) return;
    const int nst = batch.stages;
    if (tid == 0) {
        sh.P = batch.p[pi];
        // empty[s]: one arrival per consumer warp once its wgmma reading stage s have completed
        for (int s = 0; s < MAX_STAGES; s++) { mbar_init(&sh.full[s], 1); mbar_init(&sh.empty[s], CONSUMERS / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const GemvProblem & P = sh.P;
    constexpr int NG = NPAD / 8;
    const uint32_t b_bytes = (uint32_t) NPAD * KSTEP * 2, stage_bytes = A_BYTES + b_bytes;
    const int nsteps_total = P.K / KSTEP;
    const int local = (int) blockIdx.x - P.first_cta, ntiles = batch.tiles[pi];
    const int nsplit = batch.splits[pi];
    const int split = nsplit > 1 ? local % nsplit : 0, tile = nsplit > 1 ? local / nsplit : local;
    (void) ntiles;
    const int ks0 = split * batch.steps_per_split[pi], ks1 = min(nsteps_total, ks0 + batch.steps_per_split[pi]);
    const int n = ks1 - ks0;                   // K-steps of this CTA (>= 1 by construction)
    const int row0 = tile * TILE_M;

    if (warp == PRODUCER_WARP) {
        if (lane == 0) {
            // ===== producer: weights do not depend on the previous kernel -- the first ring-full of A blocks is on its way before
            // the programmatic-dependency wait; the activations (B) follow once the kernels that produced them are done
            const uint8_t * a_src = reinterpret_cast<const uint8_t *>(P.Wt) + ((size_t) tile * nsteps_total + ks0) * A_BYTES;
            const uint8_t * b_src = reinterpret_cast<const uint8_t *>(batch.act16[pi]) + (size_t) ks0 * b_bytes;
            // Every CTA of a problem multiplies the SAME activation block at K-step ks. Marching through K in lockstep, ~130 CTAs would
            // pull the same 16-32 KB out of the same few L2 slices at the same moment (microseconds per K-step however the weights
            // arrive). So CTA (tile, split) starts at K-step `rot` of its range and wraps around: at any moment the CTAs read different
            // blocks. The accumulation order of a tile is then a function of its tile index: fixed from run to run.
            const int rot = (int) (((unsigned) tile * 29u + (unsigned) split * 11u) % (unsigned) n);
            auto kstep = [&](int it) { const int k = it + rot; return k >= n ? k - n : k; };
            const int pre = n < nst ? n : nst;
            for (int i = 0; i < pre; i++) {
                mbar_expect_tx(&sh.full[i], stage_bytes);
                bulk_load(smem + (size_t) i * stage_bytes, a_src + (size_t) kstep(i) * A_BYTES, A_BYTES, &sh.full[i]);
            }
            asm volatile("griddepcontrol.wait;" ::: "memory");
            for (int i = 0; i < pre; i++) bulk_load(smem + (size_t) i * stage_bytes + A_BYTES, b_src + (size_t) kstep(i) * b_bytes, b_bytes, &sh.full[i]);
            for (int it = pre; it < n; it++) {
                const int s = it % nst;
                mbar_wait(&sh.empty[s], (uint32_t) (((it / nst) - 1) & 1));
                mbar_expect_tx(&sh.full[s], stage_bytes);
                bulk_load(smem + (size_t) s * stage_bytes, a_src + (size_t) kstep(it) * A_BYTES, A_BYTES, &sh.full[s]);
                bulk_load(smem + (size_t) s * stage_bytes + A_BYTES, b_src + (size_t) kstep(it) * b_bytes, b_bytes, &sh.full[s]);
            }
        }
        if (nsplit > 1) {      // the producer warp takes part in both cluster barriers
            __syncwarp();
            cluster_sync_all();
            __syncwarp();
            cluster_sync_all();
        }
    } else {
        // ===== consumers (warps 0-7): residual / gate inputs and the token scales belong to the previous kernels until the
        // programmatic-dependency wait
        asm volatile("griddepcontrol.wait;" ::: "memory");
        for (int i = tid; i < NPAD; i += CONSUMERS) sh.colscale[i] = batch.colscale[pi][i];
        // per K-step one wait, 4 x (NPAD / 64 rounded up) wgmma (K = 16 each: two core-matrix columns of A and of B), one commit;
        // the stage of the PREVIOUS K-step is handed back once wait_group(1) says its wgmma are done
        float acc[NPAD / 2];
        const uint64_t a_fixed = make_desc(0, A_LBO, 128), b_fixed = make_desc(0, (uint32_t) NG * 128, 128);
        const uint32_t smem0 = smem_u32(smem), rows16 = (uint32_t) (tid / 128) * 8 * 128;     // warpgroup g: row groups 8 g .. 8 g + 7
        // trace marks of CTA 0 (%globaltimer): [0] first stage complete = first MMA issued, [1] last MMA issued, [2] accumulator final
        const bool acct = batch.trace != nullptr && blockIdx.x == 0 && tid == 0;
        for (int it = 0; it < n; it++) {
            const int s = it % nst;
            const uint32_t a0 = smem0 + (uint32_t) s * stage_bytes + rows16, b0 = smem0 + (uint32_t) s * stage_bytes + A_BYTES;
            mbar_wait(&sh.full[s], (uint32_t) ((it / nst) & 1));
            if (acct && it == 0) { unsigned long long g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g)); batch.trace->mark[0] = g; }
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < KSTEP / 16; k++) {
                const uint64_t ad = a_fixed | (uint64_t) (((a0 + (uint32_t) k * 2 * A_LBO) & 0x3FFFFu) >> 4);
                const uint32_t bk = b0 + (uint32_t) k * 2 * NG * 128;
                const uint32_t acc_in = (it > 0 || k > 0) ? 1u : 0u;
#pragma unroll
                for (int c = 0; c < NPAD / 64; c++)
                    wgmma_f16<64>(acc + 32 * c, ad, b_fixed | (uint64_t) (((bk + (uint32_t) c * 8 * 128) & 0x3FFFFu) >> 4), acc_in);
                if constexpr (NPAD % 64 != 0)
                    wgmma_f16<NPAD % 64>(acc + 32 * (NPAD / 64), ad, b_fixed | (uint64_t) (((bk + (uint32_t) (NPAD / 64) * 8 * 128) & 0x3FFFFu) >> 4), acc_in);
            }
            wgmma_commit();
            wgmma_wait<1>();
            if (it > 0 && lane == 0) mbar_arrive(&sh.empty[(it - 1) % nst]);
        }
        wgmma_wait<0>();
        if (acct) { unsigned long long g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g)); batch.trace->mark[1] = g; batch.trace->mark[2] = g; }
        // both warpgroups are done reading the ring -> park the accumulator there -> [barrier] -> thread-per-row epilogue
        float * park = reinterpret_cast<float *>(smem);
        asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
        tc_park_accumulator<NPAD>(acc, park);
        if (nsplit == 1) {
            asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
            tc_epilogue_rows(P, sh.colscale, park, row0, NPAD, batch.T);
        } else {
            // every thread of the cluster: accumulators parked -> [barrier] -> each CTA reduces its column slice out of all of them ->
            // [barrier] so that no CTA retires (and frees its shared memory) while a peer still reads it
            __syncwarp();
            cluster_sync_all();
            tc_reduce_columns(P, sh.colscale, park, row0, NPAD, batch.T, nsplit);
            __syncwarp();
            cluster_sync_all();
        }
        if (acct) { unsigned long long g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g)); batch.trace->mark[3] = g; }
    }
    trace_end(batch.trace);
}

// x fp32 [K, T] column-major (column t contiguous) -> the fp16 B operand in the canonical wgmma layout, one contiguous B stage per
// K-step:  [K / 64][kc = 8][g = npad / 8][8 tokens][8 k]  (tokens >= T zero-filled). One CTA = one token column of one distinct
// input of the GEMM batch (blockIdx.y = input; up to 8: x_r, x_k, x_v, x_g, x_w of the time mix).
//
// What the halves hold. For QUANTISED weights the reference multiplies Q8_0 / Q8_1 activation blocks (ggml-cpu.c:7439-7458,
// quantize_row_q8_0 / q8_1 ggml-cpu-quants.c:781-846, 1085-1160): per 32 elements d = fp16(amax / 127), q = rint(x * 127 / amax),
// and the dot product sees d * q. So does this path: the half written is d * q (exact in fp32: 11 x 7 bits) rounded once to fp16,
// i.e. the tensor cores contract the reference's own operand values instead of a "more accurate" fp16 rounding of x, and the
// >= 32-token path tracks the dp4a path to fp16 rounding of the products (2^-12 relative per element) instead of to the Q8
// quantisation noise (~4e-3 of the block maximum). For F16 weights the reference rounds activations to fp16
// (ggml-cpu.c:259-264): the half is fp16(x).
// Range. fp16 ends at 65504 where the reference's operands do not (d is fp16 but q * d goes up to amax): every token column
// carries a power-of-two scale 2^-e, e = max(0, exponent(column maximum) - 15), applied before the rounding (exact) and taken
// out by the GEMM epilogue through colscale[t] = 2^e, so activations up to 3e38 / 127 stay finite and equally precise.
struct ConvertBatch {
    int n, T, npad;
    const float * x[GEMV_MAX_PROBLEMS];
    long long ldx[GEMV_MAX_PROBLEMS];
    int K[GEMV_MAX_PROBLEMS];
    int quant[GEMV_MAX_PROBLEMS];      // 1: Q8 block values (quantised weights), 0: plain fp16 rounding (F16 weights)
    __half * out[GEMV_MAX_PROBLEMS];
    float * colscale[GEMV_MAX_PROBLEMS];   // [npad] per input
    TraceRec * trace;
};
constexpr int CVT_THREADS = 256;
__global__ void __launch_bounds__(CVT_THREADS) convert_f16_kernel(const ConvertBatch cb) {
    __shared__ float red[CVT_THREADS / 32];
    trace_begin(cb.trace);
    pdl_prologue();
    const int q = blockIdx.y, t = blockIdx.x, T = cb.T, npad = cb.npad, K = cb.K[q];
    const int tid = threadIdx.x;
    uint4 * out = reinterpret_cast<uint4 *>(cb.out[q]);
    const int NG = npad / 8, g = t >> 3, t8 = t & 7;
    const int nblk = K / 32;
    // 16-byte chunk (ks, kc) of this token sits at ((ks * 8 + kc) * NG + g) * 8 + t8
    if (t >= T) {
        for (int c = tid; c < K / 8; c += CVT_THREADS) out[((size_t) c * NG + g) * 8 + t8] = make_uint4(0, 0, 0, 0);
        if (tid == 0) cb.colscale[q][t] = 1.0f;
        return;
    }
    const float4 * x4 = reinterpret_cast<const float4 *>(cb.x[q] + (long long) t * cb.ldx[q]);
    float cmax = 0.f;
    for (int i = tid; i < K / 4; i += CVT_THREADS) {
        const float4 v = x4[i];
        cmax = fmaxf(cmax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cmax = fmaxf(cmax, __shfl_xor_sync(0xffffffffu, cmax, o));
    if ((tid & 31) == 0) red[tid >> 5] = cmax;
    __syncthreads();
    cmax = red[0];
#pragma unroll
    for (int i = 1; i < CVT_THREADS / 32; i++) cmax = fmaxf(cmax, red[i]);
    int ex = 0;
    if (cmax > 32768.0f && cmax <= 3.0e38f) { (void) frexpf(cmax, &ex); ex -= 15; }      // cmax <= 2^ex_raw  ->  cmax * 2^-ex <= 2^15
    const float down = ex > 0 ? exp2f((float) -ex) : 1.0f;
    if (tid == 0) cb.colscale[q][t] = ex > 0 ? exp2f((float) ex) : 1.0f;
    const bool quant = cb.quant[q] != 0;
    for (int blk = tid; blk < nblk; blk += CVT_THREADS) {
        float4 v[8];
#pragma unroll
        for (int j = 0; j < 8; j++) v[j] = x4[blk * 8 + j];      // second touch of the column: L1 / L2
        if (quant) {
            float amax = 0.f;
#pragma unroll
            for (int j = 0; j < 8; j++) amax = fmaxf(amax, fmaxf(fmaxf(fabsf(v[j].x), fabsf(v[j].y)), fmaxf(fabsf(v[j].z), fabsf(v[j].w))));
            const float d = __half2float(__float2half_rn(amax / 127.0f)) * down;
            const float id = (amax != 0.0f) ? 127.0f / amax : 0.0f;
#pragma unroll
            for (int j = 0; j < 8; j++) {
                v[j].x = (float) __float2int_rn(v[j].x * id) * d; v[j].y = (float) __float2int_rn(v[j].y * id) * d;
                v[j].z = (float) __float2int_rn(v[j].z * id) * d; v[j].w = (float) __float2int_rn(v[j].w * id) * d;
            }
        } else if (ex > 0) {
#pragma unroll
            for (int j = 0; j < 8; j++) { v[j].x *= down; v[j].y *= down; v[j].z *= down; v[j].w *= down; }
        }
        const int c0 = blk * 4;            // first of the block's four 8-element chunks
#pragma unroll
        for (int cc = 0; cc < 4; cc++) {
            __half2 a = __floats2half2_rn(v[2 * cc].x, v[2 * cc].y), b = __floats2half2_rn(v[2 * cc].z, v[2 * cc].w);
            __half2 c = __floats2half2_rn(v[2 * cc + 1].x, v[2 * cc + 1].y), d2 = __floats2half2_rn(v[2 * cc + 1].z, v[2 * cc + 1].w);
            out[((size_t) (c0 + cc) * NG + g) * 8 + t8] =
                make_uint4(*reinterpret_cast<uint32_t *>(&a), *reinterpret_cast<uint32_t *>(&b), *reinterpret_cast<uint32_t *>(&c), *reinterpret_cast<uint32_t *>(&d2));
        }
    }
    trace_end(cb.trace);
}

// Load-time expansion: row-major matrix (rows of `pitch` bytes, quantised or f16) -> the fp16 operand blocks gemm_tc_kernel streams.
// One CTA = one (row tile, K-step): the 128 rows' two blocks of the K-step are staged in shared memory, thread r dequantises row r
// (block_to_half: packed-half (q - offset) * d + m, rounded once) and writes its eight 16-byte k-groups into the canonical layout
// (warp-contiguous 512-byte runs). Rows >= M are zero.
template <int TYPE>
__global__ void __launch_bounds__(TILE_M) tc_expand_kernel(const uint8_t * src, long long pitch, int M, int nsteps, uint4 * dst) {
    constexpr int BB = TYPE == DT_F16 ? 64 : QTraits<TYPE == DT_F16 ? DT_Q4_0 : TYPE>::BLOCK_BYTES;
    constexpr int ROW_WORDS = 2 * BB / 4;                       // the two blocks of a K-step start on a 4-byte boundary of the row
    constexpr int ROW_STRIDE = (2 * BB + 15) / 16 * 16;         // shared-memory row pitch: keeps 64- / 128-bit reads aligned
    __shared__ __align__(16) uint8_t rows[TILE_M * ROW_STRIDE];
    const int ks = blockIdx.x, tile = blockIdx.y, r = threadIdx.x;
    for (int i = threadIdx.x; i < TILE_M * ROW_WORDS; i += TILE_M) {
        const int rr = i / ROW_WORDS, w = i % ROW_WORDS;
        const int row = tile * TILE_M + rr;
        uint32_t v = 0;
        if (row < M) v = *reinterpret_cast<const uint32_t *>(src + (long long) row * pitch + (long long) ks * 2 * BB + w * 4);
        *reinterpret_cast<uint32_t *>(rows + rr * ROW_STRIDE + w * 4) = v;
    }
    __syncthreads();
    uint4 h[8];
    if (tile * TILE_M + r < M) {
        const uint32_t row_addr = smem_u32(rows) + (uint32_t) r * ROW_STRIDE;
        BlockRegs<TYPE> r0, r1;
        read_block<TYPE>(row_addr, 0, r0);
        read_block<TYPE>(row_addr, 1, r1);
        block_to_half<TYPE>(r0, h);
        block_to_half<TYPE>(r1, h + 4);
    } else {
#pragma unroll
        for (int i = 0; i < 8; i++) h[i] = make_uint4(0, 0, 0, 0);
    }
    uint4 * blk = dst + ((size_t) tile * nsteps + ks) * (A_BYTES / 16);
#pragma unroll
    for (int kc = 0; kc < 8; kc++) blk[(kc * (TILE_M / 8) + (r >> 3)) * 8 + (r & 7)] = h[kc];
}

// Q4_K / Q5_K rows -> the same fp16 operand blocks. A K-step (64 weights) is sub-blocks 2j and 2j + 1 of super-block ks / 4,
// j = ks % 4: the low and the high nibbles of qs[32j .. 32j + 32). Thread r expands row r: w = d*sc*q - dmin*m, where d*sc, dmin*m
// and d*sc*q are exact in fp32, so the fp16 conversion of the difference is the one rounding.
template <int TYPE>
__global__ void __launch_bounds__(TILE_M) tc_expand_kq_kernel(const uint8_t * src, long long pitch, int M, int nsteps, uint4 * dst) {
    constexpr int BB = TYPE == DT_Q4_K ? 144 : 176, QS = TYPE == DT_Q4_K ? 16 : 48;
    const int ks = blockIdx.x, tile = blockIdx.y, r = threadIdx.x, row = tile * TILE_M + r, j = ks & 3;
    uint4 h[8];
    if (row < M) {
        const uint8_t * blk = src + (long long) row * pitch + (long long) (ks >> 2) * BB;
        const float d = __half2float(__ushort_as_half(*reinterpret_cast<const unsigned short *>(blk)));
        const float dmin = __half2float(__ushort_as_half(*reinterpret_cast<const unsigned short *>(blk + 2)));
        float a[2], b[2];
        for (int hi = 0; hi < 2; hi++) {
            int sc, mn;
            kquant_scale_min(blk + 4, 2 * j + hi, sc, mn);
            a[hi] = d * (float) sc;
            b[hi] = dmin * (float) mn;
        }
        const uint8_t * qs = blk + QS + 32 * j;
#pragma unroll
        for (int kc = 0; kc < 8; kc++) {
            const int hi = kc >> 2;
            __half v[8];
#pragma unroll
            for (int e = 0; e < 8; e++) {
                const int l = (kc & 3) * 8 + e;
                int q = (qs[l] >> (4 * hi)) & 0xF;
                if (TYPE == DT_Q5_K) q |= ((blk[16 + l] >> (2 * j + hi)) & 1) << 4;
                v[e] = __float2half_rn(__fsub_rn(__fmul_rn(a[hi], (float) q), b[hi]));
            }
            h[kc] = *reinterpret_cast<const uint4 *>(v);
        }
    } else {
#pragma unroll
        for (int i = 0; i < 8; i++) h[i] = make_uint4(0, 0, 0, 0);
    }
    uint4 * out = dst + ((size_t) tile * nsteps + ks) * (A_BYTES / 16);
#pragma unroll
    for (int kc = 0; kc < 8; kc++) out[(kc * (TILE_M / 8) + (r >> 3)) * 8 + (r & 7)] = h[kc];
}

// The B operand of K-quant weights: the Q8_K block values q * d the reference multiplies them with (quantize_row_q8_K_ref: d =
// 1 / (-127 / max) in float32, max the first element of largest magnitude, q = min(127, rint(-127 / max * x))), with the same
// power-of-two column scale as convert_f16_kernel. A separate kernel, so that convert_f16_kernel's code stays as it is. One CTA =
// one token column of one input; one warp per super-block, 8 elements per lane (one 16-byte chunk of the canonical layout).
__global__ void __launch_bounds__(CVT_THREADS) convert_q8k_kernel(const ConvertBatch cb) {
    __shared__ float red[CVT_THREADS / 32];
    trace_begin(cb.trace);
    pdl_prologue();
    const int q = blockIdx.y, t = blockIdx.x, T = cb.T, npad = cb.npad, K = cb.K[q];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint4 * out = reinterpret_cast<uint4 *>(cb.out[q]);
    const int NG = npad / 8, g = t >> 3, t8 = t & 7;
    if (t >= T) {
        for (int c = tid; c < K / 8; c += CVT_THREADS) out[((size_t) c * NG + g) * 8 + t8] = make_uint4(0, 0, 0, 0);
        if (tid == 0) cb.colscale[q][t] = 1.0f;
        return;
    }
    const float * x = cb.x[q] + (long long) t * cb.ldx[q];
    const float4 * x4 = reinterpret_cast<const float4 *>(x);
    float cmax = 0.f;
    for (int i = tid; i < K / 4; i += CVT_THREADS) {
        const float4 v = x4[i];
        cmax = fmaxf(cmax, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cmax = fmaxf(cmax, __shfl_xor_sync(0xffffffffu, cmax, o));
    if (lane == 0) red[warp] = cmax;
    __syncthreads();
    cmax = red[0];
#pragma unroll
    for (int i = 1; i < CVT_THREADS / 32; i++) cmax = fmaxf(cmax, red[i]);
    int ex = 0;
    if (cmax > 32768.0f && cmax <= 3.0e38f) { (void) frexpf(cmax, &ex); ex -= 15; }
    const float down = ex > 0 ? exp2f((float) -ex) : 1.0f;
    if (tid == 0) cb.colscale[q][t] = ex > 0 ? exp2f((float) ex) : 1.0f;
    for (int s = warp; s < K / QK_K; s += CVT_THREADS / 32) {
        const float4 a = x4[s * 64 + lane * 2], b = x4[s * 64 + lane * 2 + 1];
        const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        float amax = 0.f, mx = 0.f;
        int idx = QK_K;
#pragma unroll
        for (int e = 0; e < 8; e++) if (fabsf(v[e]) > amax) { amax = fabsf(v[e]); mx = v[e]; idx = lane * 8 + e; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float oa = __shfl_xor_sync(0xffffffffu, amax, o), om = __shfl_xor_sync(0xffffffffu, mx, o);
            const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
            if (oa > amax || (oa == amax && oi < idx)) { amax = oa; mx = om; idx = oi; }
        }
        __half hv[8];
        if (amax != 0.f) {
            const float iscale = __fdiv_rn(-127.f, mx), d = __fmul_rn(__fdiv_rn(1.f, iscale), down);
#pragma unroll
            for (int e = 0; e < 8; e++) hv[e] = __float2half_rn(__fmul_rn((float) min(127, __float2int_rn(__fmul_rn(iscale, v[e]))), d));
        } else {
#pragma unroll
            for (int e = 0; e < 8; e++) hv[e] = __float2half_rn(0.f);
        }
        out[((size_t) (s * 32 + lane) * NG + g) * 8 + t8] = *reinterpret_cast<const uint4 *>(hv);
    }
    trace_end(cb.trace);
}

}  // namespace tc

// K-quant matrices need whole super-blocks (the loader guarantees them); a K-step never straddles one.
bool gemm_tc_eligible(int type, int K) {
    return type != DT_F32 && K % tc::KSTEP == 0 && K >= tc::KSTEP && (!dtype_kquant(type) || K % QK_K == 0);
}

size_t gemm_tc_tiled_bytes(int type, int M, int K) {
    if (!gemm_tc_eligible(type, K)) return 0;
    const size_t nsteps = (size_t) K / tc::KSTEP, ntiles = ((size_t) M + tc::TILE_M - 1) / tc::TILE_M;
    return ntiles * nsteps * tc::A_BYTES;
}

cudaError_t gemm_tc_repack(const void * W, long long pitch, int type, int M, int K, void * dst, cudaStream_t stream) {
    if (!gemm_tc_eligible(type, K)) return cudaErrorInvalidValue;
    const int nsteps = K / tc::KSTEP, ntiles = (M + tc::TILE_M - 1) / tc::TILE_M;
    const dim3 grid((unsigned) nsteps, (unsigned) ntiles);
    const uint8_t * src = reinterpret_cast<const uint8_t *>(W);
    uint4 * out = reinterpret_cast<uint4 *>(dst);
    if (dtype_kquant(type)) {
        log_launch(LF_KQ_EXPAND, 0, type, 0, 0, 0);
        if (type == DT_Q4_K) tc::tc_expand_kq_kernel<DT_Q4_K><<<grid, tc::TILE_M, 0, stream>>>(src, pitch, M, nsteps, out);
        else tc::tc_expand_kq_kernel<DT_Q5_K><<<grid, tc::TILE_M, 0, stream>>>(src, pitch, M, nsteps, out);
        return cudaGetLastError();
    }
    log_launch(LF_EXPAND, 0, type, 0, 0, 0);
    switch (type) {
        case DT_Q4_0: tc::tc_expand_kernel<DT_Q4_0><<<grid, tc::TILE_M, 0, stream>>>(src, pitch, M, nsteps, out); break;
        case DT_Q4_1: tc::tc_expand_kernel<DT_Q4_1><<<grid, tc::TILE_M, 0, stream>>>(src, pitch, M, nsteps, out); break;
        case DT_Q5_0: tc::tc_expand_kernel<DT_Q5_0><<<grid, tc::TILE_M, 0, stream>>>(src, pitch, M, nsteps, out); break;
        case DT_Q5_1: tc::tc_expand_kernel<DT_Q5_1><<<grid, tc::TILE_M, 0, stream>>>(src, pitch, M, nsteps, out); break;
        case DT_Q8_0: tc::tc_expand_kernel<DT_Q8_0><<<grid, tc::TILE_M, 0, stream>>>(src, pitch, M, nsteps, out); break;
        case DT_F16: tc::tc_expand_kernel<DT_F16><<<grid, tc::TILE_M, 0, stream>>>(src, pitch, M, nsteps, out); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// convert_f16_kernel applies no LayerNorm: a problem with a prologue takes the GEMV.
bool gemm_tc_supported(const GemvProblem & p, int T) {
    return T >= 16 && T <= tc::MAX_N && p.Wt != nullptr && p.pro == PRO_NONE && gemm_tc_eligible(p.type, p.K) && (p.ldx % 4) == 0 &&
           (reinterpret_cast<uintptr_t>(p.x) & 15) == 0 && (reinterpret_cast<uintptr_t>(p.Wt) & 15) == 0;
}

// Workspace layout (gemm_tc_workspace_bytes): the fp16 operands + per-token scales of the batch's distinct inputs, each part starting
// on a 256-byte boundary.
size_t gemm_tc_workspace_bytes(int T, size_t operand_halves) {
    const size_t npad = (size_t) (T + 15) / 16 * 16;
    return operand_halves * 2 + (size_t) GEMV_MAX_PROBLEMS * (npad * 4 + 512);
}

cudaError_t gemm_tc_launch(GemvBatch & batch, const DeviceInfo & dev, cudaStream_t stream, void * workspace, size_t workspace_bytes) {
    tc::TcBatch tb;
    memset(&tb, 0, sizeof(tb));
    tb.n = batch.n; tb.T = batch.T;
    tb.npad = (batch.T + 15) / 16 * 16;

    uint8_t * scratch = reinterpret_cast<uint8_t *>(workspace);
    size_t used = 0;
    // operand kinds: fp16(x) for F16 weights, Q8_0 / Q8_1 block values for the legacy formats (both convert_f16_kernel), Q8_K block
    // values for K-quant weights (convert_q8k_kernel)
    tc::ConvertBatch cvt, cvk;
    memset(&cvt, 0, sizeof(cvt));
    memset(&cvk, 0, sizeof(cvk));
    cvt.T = cvk.T = batch.T; cvt.npad = cvk.npad = tb.npad;
    auto kind = [](int type) { return type == DT_F16 ? 0 : (dtype_kquant(type) ? 2 : 1); };
    int share_of[GEMV_MAX_PROBLEMS];
    for (int i = 0; i < batch.n; i++) {
        GemvProblem & p = batch.p[i];
        const int k = kind(p.type);
        tc::ConvertBatch & cb = k == 2 ? cvk : cvt;
        const size_t need = (((size_t) tb.npad * p.K * sizeof(__half) + 255) & ~(size_t) 255) + (((size_t) tb.npad * sizeof(float) + 255) & ~(size_t) 255);
        // problems that share an input (and its operand kind) share the converted copy
        int shared = -1;
        for (int j = 0; j < i; j++)
            if (batch.p[j].x == p.x && batch.p[j].K == p.K && batch.p[j].ldx == p.ldx && kind(batch.p[j].type) == k) shared = share_of[j];
        if (shared < 0) {
            if (used + need > workspace_bytes) return cudaErrorMemoryAllocation;
            shared = cb.n;
            cb.x[cb.n] = p.x; cb.ldx[cb.n] = p.ldx; cb.K[cb.n] = p.K; cb.quant[cb.n] = k != 0;
            cb.out[cb.n] = reinterpret_cast<__half *>(scratch + used);
            cb.colscale[cb.n] = reinterpret_cast<float *>(scratch + used + (((size_t) tb.npad * p.K * sizeof(__half) + 255) & ~(size_t) 255));
            cb.n++;
            used += need;
        }
        share_of[i] = shared;
        tb.act16[i] = cb.out[shared];
        tb.colscale[i] = cb.colscale[shared];
    }
    // ---- work decomposition: one CTA per (row tile, K-split). Every CTA streams its share of the weights from HBM, so what matters
    // is that close to all SMs have a CTA: launches with few tiles (4096-row matrices: 32; LoRA: 1-2) are cut along K over clusters
    // of c = 2 / 4 / 8 CTAs (a problem is cut c ways or not at all: the cluster size is one per launch).
    int total = 0;
    for (int i = 0; i < batch.n; i++) { tb.tiles[i] = (batch.p[i].M + tc::TILE_M - 1) / tc::TILE_M; total += tb.tiles[i]; }
    const int sms = dev.num_sms > 0 ? dev.num_sms : 132;
    const int want = total * 4 < sms * 3 ? sms / total : 1;      // below 75 % of the SMs: split, but never into a second wave
    int cluster = 1;
    while (cluster * 2 <= want && cluster < 8) cluster *= 2;
    bool any_split = false;
    for (int i = 0; i < batch.n; i++) {
        const int nsteps = batch.p[i].K / tc::KSTEP;
        const int per = (nsteps + cluster - 1) / cluster;
        // at least four K-steps per split, and the last split must not come out empty
        const bool cut = cluster > 1 && nsteps >= 4 * cluster && (cluster - 1) * per < nsteps;
        tb.splits[i] = cut ? cluster : 1;
        tb.steps_per_split[i] = cut ? per : nsteps;
        any_split = any_split || cut;
    }
    if (!any_split) cluster = 1;
    tb.cluster = cluster;
    int next = 0;
    for (int i = 0; i < batch.n; i++) {
        GemvProblem & p = batch.p[i];
        p.first_cta = next;                                               // a multiple of the cluster size
        p.n_cta = tb.splits[i] > 1 ? tb.tiles[i] * cluster : (tb.tiles[i] + cluster - 1) / cluster * cluster;
        next += p.n_cta;
        tb.p[i] = p;
    }
    if (cvt.n) {   // every distinct input of the batch -> fp16 canonical layout, one launch: one CTA per (token column, input)
        cvt.trace = trace_slot("convert_f16");
        log_launch(LF_CONVERT, cvt.n, 0, 0, tb.npad, 0);
        cudaError_t e = launch_pdl(tc::convert_f16_kernel, dim3(tb.npad, cvt.n), dim3(tc::CVT_THREADS), 0, stream, cvt);
        if (e != cudaSuccess) return e;
    }
    if (cvk.n) {
        cvk.trace = trace_slot("convert_q8k");
        log_launch(LF_CONVERT, cvk.n, DT_Q8_K, 0, tb.npad, 0);
        cudaError_t e = launch_pdl(tc::convert_q8k_kernel, dim3(tb.npad, cvk.n), dim3(tc::CVT_THREADS), 0, stream, cvk);
        if (e != cudaSuccess) return e;
    }
    // shared memory: as many [A | B] ring stages as fit, at most 8
    constexpr size_t smem_budget = 227 * 1024 - 2048;
    const size_t stage_bytes = (size_t) tc::A_BYTES + (size_t) tb.npad * tc::KSTEP * 2;
    int nst = (int) (smem_budget / stage_bytes);
    if (nst > tc::MAX_STAGES) nst = tc::MAX_STAGES;
    if (nst < 2) return cudaErrorInvalidValue;
    tb.stages = nst;
    const size_t smem = (size_t) nst * stage_bytes;
    if (smem < (size_t) tb.npad * tc::PARK_LD * sizeof(float)) return cudaErrorInvalidValue;     // the parked accumulator
    // one instantiation per padded token count (the wgmma N and the accumulator registers are compile-time)
    using Kernel = void (*)(const tc::TcBatch);
    static const Kernel kernels[tc::MAX_N / 16] = {
        tc::gemm_tc_kernel<16>, tc::gemm_tc_kernel<32>, tc::gemm_tc_kernel<48>, tc::gemm_tc_kernel<64>,
        tc::gemm_tc_kernel<80>, tc::gemm_tc_kernel<96>, tc::gemm_tc_kernel<112>, tc::gemm_tc_kernel<128>,
        tc::gemm_tc_kernel<144>, tc::gemm_tc_kernel<160>, tc::gemm_tc_kernel<176>, tc::gemm_tc_kernel<192>,
        tc::gemm_tc_kernel<208>, tc::gemm_tc_kernel<224>, tc::gemm_tc_kernel<240>, tc::gemm_tc_kernel<256>};
    const int ki = tb.npad / 16 - 1;
    if (ki < 0 || ki >= tc::MAX_N / 16) return cudaErrorInvalidValue;
    const Kernel kernel = kernels[ki];
    static PerDeviceOnce once[tc::MAX_N / 16];   // the opt-in is per (device, instantiation)
    const cudaError_t ae = once[ki].run([&] { return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem_budget); });
    if (ae != cudaSuccess) return ae;
    tb.trace = trace_slot("gemm_tc");
    log_launch(LF_TENSOR_CORES, 0, 0, 0, tb.npad, cluster);
    return launch_pdl((unsigned) cluster, kernel, dim3((unsigned) next), dim3(tc::THREADS), smem, stream, tb);
}

}  // namespace rwkv
