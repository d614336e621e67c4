// Fused dequantize-and-GEMV, sm_90a streaming version.
//
// Weights travel HBM -> shared memory as large 1-D TMA bulk copies (cp.async.bulk, SASS UBLKCP) through a
// 3-stage mbarrier ring driven by ONE producer thread per CTA, so the bytes in flight per SM (2 CTAs x 3
// stages x ~30 KB) are set by the ring depth, not by how many loads the math warps keep outstanding. Eight
// consumer warps per CTA pull 4/8-byte-aligned block units out of the staged rows (native ggml layout), decode
// to int8x4 and accumulate with dp4a against activation blocks that every lane keeps in registers for the whole
// kernel; the unit loop is branch-free so four independent block chains are in flight per lane.
//
//   grid     2 CTAs per SM (persistent for the launch), CTAs split over the problems of the batch by weight bytes
//   tile     R consecutive rows x full K = one contiguous bulk copy (rows are 16-byte pitched)
//   warps    WK warps share a row along K (WK = 1 up to K = 4096 for quantised rows: a warp owns whole rows),
//            WR = 8 / WK rows of a tile in flight; partial sums of a row meet in shared memory in a fixed order
//   PDL      launched with programmatic stream serialisation: the producer starts prefetching weights (which no
//            kernel ever writes) while the previous kernel is still running; consumers wait on the grid
//            dependency before they touch activations.
//
// Arithmetic per output element depends only on (type, K): which lane adds which block in which order is fixed by
// WK, itself a function of (type, K, pitch) alone -- never of T, the batch composition or the tile size. A token
// evaluated alone and inside a chunk therefore produces identical bits (tests/test_eval_sequence_in_chunks.c:54).
#include "gemv_tma_device.cuh"
#include "act_stage.cuh"

namespace rwkv {
namespace tma {

// ONLY: the weight type of EVERY problem of the launch (a single-token launch of a model whose matrices share one format: all of a
// v4 / v5 / v6 layer), or -1 for launches that mix formats. The one-kernel-for-everything instantiation is 15 500 instructions
// (248 KB) of which a launch runs ~1 500 scattered ones; ncu attributes 34 % of the warp stall cycles of a 12 MB launch, and 50-64 %
// of the LoRA launches', to instruction fetch. A per-format instantiation is ~2 000
// instructions, contiguous.
template <int NC, int ONLY = -1, bool HAS_LN = true>
__global__ void __launch_bounds__(THREADS, 2) gemv_tma_kernel(const GemvBatch batch) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ Shared sh;
    trace_begin(batch.trace);

    {
        int pi = 0;
        for (int i = 1; i < batch.n; i++) if ((int) blockIdx.x >= batch.p[i].first_cta) pi = i;
        if (threadIdx.x == 0) {
            sh.P = batch.p[pi];
            sh.trace = batch.trace;
            for (int s = 0; s < NSTAGES; s++) { mbar_init(&sh.full[s], 1); mbar_init(&sh.empty[s], CONSUMER_WARPS); }
            fence_barrier_init();
        }
        __syncthreads();
    }
    grid_launch_dependents();   // let the next kernel's CTAs start (and prefetch their weights) as soon as SM space frees up
    const GemvProblem & P = sh.P;
    const int local_cta = (int) blockIdx.x - P.first_cta;
    const int n_tiles = (P.M + P.tile_rows - 1) / P.tile_rows;
    const int my_tiles = (n_tiles - local_cta + P.n_cta - 1) / P.n_cta;   // tiles local_cta, local_cta + n_cta, ...
    const int n_groups = (batch.T + NC - 1) / NC;
    const uint32_t stage_bytes = (uint32_t) batch.stage_bytes;

    uint8_t * ring = smem;
    const int ptype = ONLY >= 0 ? ONLY : P.type;
    const size_t colb = act_bytes_per_column(ptype, P.K);
    uint8_t * act = smem + (size_t) NSTAGES * stage_bytes;
    float * red = reinterpret_cast<float *>(act + (size_t) NC * batch.max_col_bytes);

    if (threadIdx.x >= CONSUMER_THREADS) {
        // ===== producer: one thread streams every tile of every column group through the ring. Weights are
        // immutable, so it does not wait for the previous kernel. =====
        if (threadIdx.x == CONSUMER_THREADS) {
            const uint64_t policy = (n_groups == 1) ? policy_evict_first() : policy_evict_normal();
            const uint8_t * Wb = reinterpret_cast<const uint8_t *>(P.W);
            int it = 0;
            for (int g = 0; g < n_groups; g++) {
                for (int i = 0; i < my_tiles; i++, it++) {
                    const int tile = local_cta + i * P.n_cta;
                    const int row0 = tile * P.tile_rows;
                    const int rows = min(P.tile_rows, P.M - row0);
                    const int s = it % NSTAGES;
                    if (it >= NSTAGES) mbar_wait(&sh.empty[s], (uint32_t) (((it / NSTAGES) - 1) & 1));
                    const uint32_t bytes = (uint32_t) ((size_t) rows * (size_t) P.pitch);
                    mbar_expect_tx(&sh.full[s], bytes);
                    bulk_copy_g2s(ring + (size_t) s * stage_bytes, Wb + (size_t) row0 * (size_t) P.pitch, bytes, &sh.full[s], policy);
                }
            }
        }
        return;
    }

    // ===== consumers =====
    grid_dependency_wait();          // activations / residuals come from the previous kernel
    trace_mark(batch.trace, 0);
    const bool quant = ptype != DT_F16 && ptype != DT_F32;
    for (int g = 0; g < n_groups; g++) {
        const int c0 = g * NC, nc = min(NC, batch.T - c0);
        if (g > 0) consumer_barrier();   // everyone finished reading the previous group's activations
        if (NC == 1 && P.xq && batch.T == 1) {
            // the producer of x left the staged column in global memory (act_stage.cuh): one 16-byte-per-thread copy out of L2
            const int4 * src = reinterpret_cast<const int4 *>(P.xq);
            int4 * dst = reinterpret_cast<int4 *>(act);
            for (int i = threadIdx.x; i < (int) (colb / 16); i += CONSUMER_THREADS) dst[i] = __ldcg(src + i);
        } else {
            for (int c = 0; c < nc; c++) stage_column<4, NC == 1, ONLY, HAS_LN>(P, c0 + c, act + c * colb, sh.red_d);
        }
        consumer_barrier();
        trace_mark(batch.trace, 1);
        const int it0 = g * my_tiles;
#define RWKV_CONSUME_REGS(T_) consume_quant_regs<T_>(sh, ring, stage_bytes, act, c0, red, it0, my_tiles, local_cta, P.n_cta)
#define RWKV_CONSUME_SMEM(T_) consume_smem<T_, NC>(sh, ring, stage_bytes, act, colb, c0, nc, red, it0, my_tiles, local_cta, P.n_cta)
        if constexpr (ONLY >= 0) {
            if constexpr (NC == 1 && ONLY != DT_F16 && ONLY != DT_F32) RWKV_CONSUME_REGS(ONLY);
            else RWKV_CONSUME_SMEM(ONLY);
        } else if (NC == 1 && quant) {
            switch (ptype) {
                case DT_Q4_0: RWKV_CONSUME_REGS(DT_Q4_0); break;
                case DT_Q4_1: RWKV_CONSUME_REGS(DT_Q4_1); break;
                case DT_Q5_0: RWKV_CONSUME_REGS(DT_Q5_0); break;
                case DT_Q5_1: RWKV_CONSUME_REGS(DT_Q5_1); break;
                default: RWKV_CONSUME_REGS(DT_Q8_0); break;
            }
        } else if constexpr (NC == 1) {      // quantised columns of a single-column launch never come here
            if (ptype == DT_F16) RWKV_CONSUME_SMEM(DT_F16); else RWKV_CONSUME_SMEM(DT_F32);
        } else {
            switch (ptype) {
                case DT_Q4_0: RWKV_CONSUME_SMEM(DT_Q4_0); break;
                case DT_Q4_1: RWKV_CONSUME_SMEM(DT_Q4_1); break;
                case DT_Q5_0: RWKV_CONSUME_SMEM(DT_Q5_0); break;
                case DT_Q5_1: RWKV_CONSUME_SMEM(DT_Q5_1); break;
                case DT_Q8_0: RWKV_CONSUME_SMEM(DT_Q8_0); break;
                case DT_F16: RWKV_CONSUME_SMEM(DT_F16); break;
                default: RWKV_CONSUME_SMEM(DT_F32); break;
            }
        }
#undef RWKV_CONSUME_REGS
#undef RWKV_CONSUME_SMEM
    }
    trace_end(batch.trace);
}

}  // namespace tma

// ---- host side: shape planning + launch ----------------------------------------------------------------
namespace {

// WK (warps sharing a row along K) from (type, K, pitch) alone; false if the shape needs the generic kernel.
bool plan_wk(GemvProblem & p) {
    using namespace tma;
    if (p.pitch % 16 != 0 || (reinterpret_cast<uintptr_t>(p.W) & 15)) return false;
    const bool quant = p.type != DT_F16 && p.type != DT_F32;
    for (int wk = 1; wk <= CONSUMER_WARPS; wk *= 2) {
        const int wr = CONSUMER_WARPS / wk;
        if ((long long) wr * p.pitch > NOMINAL_STAGE_BYTES) continue;
        if (quant && p.K / 32 > MAX_BLOCKS_PER_LANE * 32 * wk) continue;   // activation blocks must fit a lane's registers
        p.wk = wk;
        // lanes per row: 32, or fewer (a power of two) when a whole row has fewer than 32 items (LoRA matrices)
        p.g = 32;
        if (wk == 1) {
            const int ub = (p.type == DT_Q4_1 || p.type == DT_Q5_1) ? 1 : 2;
            const int items = quant ? (p.K / 32 + ub - 1) / ub : (p.type == DT_F16 ? (p.K + 7) / 8 : (p.K + 3) / 4);
            int g = 1;
            while (g < items && g < 32) g *= 2;
            p.g = g;
        }
        return true;
    }
    return false;
}

}  // namespace

bool gemv_tma_plan(GemvProblem & p) { return plan_wk(p); }

namespace {

template <int NC, int ONLY = -1, bool HAS_LN = true>
cudaError_t launch_tma_nc(const GemvBatch & batch, int grid, size_t smem, cudaStream_t stream) {
    static PerDeviceOnce once;                // the shared-memory opt-in is per device
    const cudaError_t ae = once.run([&] { return cudaFuncSetAttribute(tma::gemv_tma_kernel<NC, ONLY, HAS_LN>, cudaFuncAttributeMaxDynamicSharedMemorySize, tma::CTA_SMEM_BUDGET); });
    if (ae != cudaSuccess) return ae;
    log_launch(LF_STREAMING, NC, ONLY, HAS_LN, 0, 0);
    return launch_pdl(tma::gemv_tma_kernel<NC, ONLY, HAS_LN>, dim3((unsigned) grid), dim3(tma::THREADS), smem, stream, batch);
}

// Single-column launches run the instantiation of their weight format when every problem of the launch has the same one.
cudaError_t launch_tma_single(const GemvBatch & batch, int grid, size_t smem, cudaStream_t stream) {
    int only = batch.p[0].type;
    for (int i = 1; i < batch.n; i++) if (batch.p[i].type != only) only = -1;
    bool has_ln = false;
    for (int i = 0; i < batch.n; i++) has_ln = has_ln || batch.p[i].pro == PRO_LAYERNORM;
#define RWKV_PER_TYPE(T_) case T_: return has_ln ? launch_tma_nc<1, T_, true>(batch, grid, smem, stream) : launch_tma_nc<1, T_, false>(batch, grid, smem, stream);
    switch (only) {
        RWKV_PER_TYPE(DT_Q4_0) RWKV_PER_TYPE(DT_Q4_1) RWKV_PER_TYPE(DT_Q5_0) RWKV_PER_TYPE(DT_Q5_1) RWKV_PER_TYPE(DT_Q8_0) RWKV_PER_TYPE(DT_F16) RWKV_PER_TYPE(DT_F32)
        default: return launch_tma_nc<1>(batch, grid, smem, stream);
    }
#undef RWKV_PER_TYPE
}

}  // namespace

// Tile height and CTA share of every problem for ring stages of `stage_bytes`: CTAs are split over the problems by weight
// bytes (largest remainders get the leftovers). Returns the number of CTAs used (<= total_ctas).
int assign_tiles_and_ctas(GemvBatch & batch, int total_ctas, long long stage_bytes) {
    using namespace tma;
    double total_bytes = 0;
    for (int i = 0; i < batch.n; i++) total_bytes += (double) batch.p[i].M * (double) batch.p[i].pitch;
    for (int i = 0; i < batch.n; i++) {
        GemvProblem & p = batch.p[i];
        // a multiple of the warp row-groups: every warp gets the same number of rows per tile. (Filling the whole ring stage -- 12 rows
        // instead of 8 at K = 4096 Q5_1, warps' row slots rotating from tile to tile -- raised the steady-state rate per CTA by 39 % but
        // cost more in the first tile and the tail: 3 % slower per 7B token. Not kept.)
        const int wr = CONSUMER_WARPS / p.wk;
        int rows = (int) (stage_bytes / p.pitch);
        rows -= rows % wr;
        if (rows > MAX_TILE_ROWS) rows = MAX_TILE_ROWS;
        p.tile_rows = rows;
    }
    int assigned = 0, cap[GEMV_MAX_PROBLEMS];
    double frac[GEMV_MAX_PROBLEMS];
    for (int i = 0; i < batch.n; i++) {
        GemvProblem & p = batch.p[i];
        const double share = (double) total_ctas * ((double) p.M * (double) p.pitch) / total_bytes;
        cap[i] = (p.M + p.tile_rows - 1) / p.tile_rows;
        int base = (int) share;
        if (base < 1) base = 1;
        if (base > cap[i]) base = cap[i];
        p.n_cta = base;
        frac[i] = share - (double) base;
        assigned += base;
    }
    while (assigned < total_ctas) {
        int best = -1;
        for (int i = 0; i < batch.n; i++) if (batch.p[i].n_cta < cap[i] && (best < 0 || frac[i] > frac[best])) best = i;
        if (best < 0) break;
        batch.p[best].n_cta++; frac[best] -= 1.0; assigned++;
    }
    int next = 0;
    for (int i = 0; i < batch.n; i++) { batch.p[i].first_cta = next; next += batch.p[i].n_cta; }
    return next;
}

// Returns cudaErrorNotSupported when some problem of the batch does not fit the streaming kernel
// (the caller then uses the generic kernel for the whole batch).
cudaError_t gemv_tma_launch(GemvBatch & batch, const DeviceInfo & dev, cudaStream_t stream) {
    using namespace tma;
    size_t max_col = 0;
    for (int i = 0; i < batch.n; i++) {
        GemvProblem & p = batch.p[i];
        if (dtype_kquant(p.type) || !plan_wk(p)) return cudaErrorNotSupported;
        const size_t cb = act_bytes_per_column(p.type, p.K);
        if (cb > max_col) max_col = cb;
    }
    // columns staged together, and the ring stage size that leaves
    auto stage_for = [&](int nc) -> long long {
        const long long rest = (long long) nc * (long long) max_col + (long long) 2 * MAX_TILE_ROWS * CONSUMER_WARPS * nc * (long long) sizeof(float);
        return ((long long) CTA_SMEM_BUDGET - rest) / NSTAGES / 1024 * 1024;
    };
    int nc = 1;
    if (batch.T >= 4 && stage_for(4) >= NOMINAL_STAGE_BYTES) nc = 4;
    else if (batch.T >= 2 && stage_for(2) >= NOMINAL_STAGE_BYTES) nc = 2;
    const long long stage_bytes = stage_for(nc);
    if (stage_bytes < NOMINAL_STAGE_BYTES) return cudaErrorNotSupported;
    // two CTAs per SM
    const int next = assign_tiles_and_ctas(batch, 2 * dev.num_sms, stage_bytes);
    batch.max_col_bytes = (long long) max_col;
    batch.stage_bytes = stage_bytes;
    batch.trace = trace_slot(batch.n > 1 ? "gemv_tma(batch)" : "gemv_tma");
    const size_t smem = (size_t) NSTAGES * (size_t) stage_bytes + (size_t) nc * max_col + (size_t) 2 * MAX_TILE_ROWS * CONSUMER_WARPS * nc * sizeof(float);
    switch (nc) {
        case 4: return launch_tma_nc<4>(batch, next, smem, stream);
        case 2: return launch_tma_nc<2>(batch, next, smem, stream);
        default: return launch_tma_single(batch, next, smem, stream);
    }
}

}  // namespace rwkv
