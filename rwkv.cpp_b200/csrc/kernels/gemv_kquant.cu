// Fused dequantize-and-GEMV for Q4_K / Q5_K matrices (ggml's K-quants: 256-weight super-blocks of eight 32-weight sub-blocks, each
// with a 6-bit scale and min), sm_90a.
//
// The weights stream exactly as in the legacy kernel (gemv_tma.cu): one producer thread per CTA feeds a 3-stage mbarrier ring of TMA
// bulk copies (evict_first for single-column launches), tiles and CTAs are planned by assign_tiles_and_ctas, consumers wait on the
// grid dependency before they touch activations. What differs is the operand the weights meet:
//   staging   each column becomes Q8_K blocks, the activation the reference's CPU path multiplies a K-quant weight with
//             (quantize_row_q8_K_ref): max = the element of largest magnitude (the first of a tie), qs = min(127, rint(-127/max * x)),
//             d = 1 / (-127/max) in float32, and the sum of every 16 qs. One warp per super-block, 8 elements per lane.
//   dot       row_partial_kq (gemv_tma_device.cuh): 8 lanes per super-block, one per sub-block; nibbles (and the fifth bit of Q5_K)
//             widen to int8x4 for dp4a; the integer sums stay exact up to one float combination per super-block.
// No staged-column hand-off (GemvProblem::xq) and no LayerNorm prologue: the producers of x never stage Q8_K, and the loader refuses a
// K-quant head. Arithmetic per output depends only on (type, K) -- WK comes from the row pitch -- never on T, NC or the batch.
#include "gemv_tma_device.cuh"

namespace rwkv {
namespace tma {

__device__ void stage_q8k(const GemvProblem & P, int col_index, uint8_t * col) {
    const int nsb = P.K / QK_K, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float * x = P.x + (long long) col_index * P.ldx;
    float * dcol = reinterpret_cast<float *>(col + (size_t) nsb * QK_K);
    short * bsums = reinterpret_cast<short *>(col + (size_t) nsb * (QK_K + 4));
    for (int s = warp; s < nsb; s += CONSUMER_WARPS) {
        const float4 a = *reinterpret_cast<const float4 *>(x + (size_t) s * QK_K + lane * 8);
        const float4 b = *reinterpret_cast<const float4 *>(x + (size_t) s * QK_K + lane * 8 + 4);
        const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        float amax = 0.f, mx = 0.f;
        int idx = QK_K;
#pragma unroll
        for (int j = 0; j < 8; j++) if (fabsf(v[j]) > amax) { amax = fabsf(v[j]); mx = v[j]; idx = lane * 8 + j; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float oa = __shfl_xor_sync(0xffffffffu, amax, o), om = __shfl_xor_sync(0xffffffffu, mx, o);
            const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
            if (oa > amax || (oa == amax && oi < idx)) { amax = oa; mx = om; idx = oi; }
        }
        int q[8], sum = 0;
        float d = 0.f;
        if (amax != 0.f) {
            const float iscale = __fdiv_rn(-127.f, mx);
#pragma unroll
            for (int j = 0; j < 8; j++) { q[j] = min(127, __float2int_rn(__fmul_rn(iscale, v[j]))); sum += q[j]; }
            d = __fdiv_rn(1.f, iscale);
        } else {
#pragma unroll
            for (int j = 0; j < 8; j++) q[j] = 0;
        }
        const uint32_t w0 = (q[0] & 0xFF) | ((q[1] & 0xFF) << 8) | ((q[2] & 0xFF) << 16) | ((uint32_t) (q[3] & 0xFF) << 24);
        const uint32_t w1 = (q[4] & 0xFF) | ((q[5] & 0xFF) << 8) | ((q[6] & 0xFF) << 16) | ((uint32_t) (q[7] & 0xFF) << 24);
        *reinterpret_cast<uint2 *>(col + (size_t) s * QK_K + lane * 8) = make_uint2(w0, w1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        if ((lane & 1) == 0) bsums[s * 16 + lane / 2] = (short) sum;
        if (lane == 0) dcol[s] = d;
    }
}

template <int NC, int TYPE>
__global__ void __launch_bounds__(THREADS, 2) gemv_kq_kernel(const GemvBatch batch) {
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
    grid_launch_dependents();
    const GemvProblem & P = sh.P;
    const int local_cta = (int) blockIdx.x - P.first_cta;
    const int n_tiles = (P.M + P.tile_rows - 1) / P.tile_rows;
    const int my_tiles = (n_tiles - local_cta + P.n_cta - 1) / P.n_cta;
    const int n_groups = (batch.T + NC - 1) / NC;
    const uint32_t stage_bytes = (uint32_t) batch.stage_bytes;
    uint8_t * ring = smem;
    const size_t colb = kq_act_bytes_per_column(P.K);
    uint8_t * act = smem + (size_t) NSTAGES * stage_bytes;
    float * red = reinterpret_cast<float *>(act + (size_t) NC * batch.max_col_bytes);

    if (threadIdx.x >= CONSUMER_THREADS) {
        if (threadIdx.x == CONSUMER_THREADS) {      // producer: weights are immutable, no dependency wait
            const uint64_t policy = (n_groups == 1) ? policy_evict_first() : policy_evict_normal();
            const uint8_t * Wb = reinterpret_cast<const uint8_t *>(P.W);
            int it = 0;
            for (int g = 0; g < n_groups; g++) {
                for (int i = 0; i < my_tiles; i++, it++) {
                    const int row0 = (local_cta + i * P.n_cta) * P.tile_rows;
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

    grid_dependency_wait();
    trace_mark(batch.trace, 0);
    for (int g = 0; g < n_groups; g++) {
        const int c0 = g * NC, nc = min(NC, batch.T - c0);
        if (g > 0) consumer_barrier();
        for (int c = 0; c < nc; c++) stage_q8k(P, c0 + c, act + c * colb);
        consumer_barrier();
        trace_mark(batch.trace, 1);
        consume_smem<TYPE, NC>(sh, ring, stage_bytes, act, colb, c0, nc, red, g * my_tiles, my_tiles, local_cta, P.n_cta);
    }
    trace_end(batch.trace);
}

}  // namespace tma

namespace {

using namespace tma;

// WK (warps sharing a row along K) from the row pitch alone, as plan_wk does for the legacy formats: the fewest warps per row whose
// rows of one tile fit NOMINAL_STAGE_BYTES, or one row per warp (WK = 8) when even that does not. G = 32 always (a warp holds four
// super-blocks per step). Activations live in shared memory, so there is no register limit on K.
bool plan_kq(GemvProblem & p) {
    if (!dtype_kquant(p.type) || p.K < QK_K || p.K % QK_K || p.pitch % 16 != 0 || (reinterpret_cast<uintptr_t>(p.W) & 15)) return false;
    p.wk = CONSUMER_WARPS;
    for (int wk = 1; wk <= CONSUMER_WARPS; wk *= 2) {
        if ((long long) (CONSUMER_WARPS / wk) * p.pitch <= NOMINAL_STAGE_BYTES) { p.wk = wk; break; }
    }
    p.g = 32;
    return true;
}
// bytes of one tile of the plan: a ring stage must hold at least this
long long kq_tile_need(const GemvProblem & p) { return (long long) (CONSUMER_WARPS / p.wk) * p.pitch; }

// Shared memory per CTA. Two CTAs per SM (CTA_SMEM_BUDGET each) whenever the launch's tiles fit; rows beyond ~20k weights stage a
// column too large for that (RWKV-4 14B's ffn.value, K = 20480 in Q5_K), and those launches run one CTA per SM with twice the budget.
constexpr int KQ_WIDE_BUDGET = 2 * CTA_SMEM_BUDGET;
long long kq_stage_bytes(int budget, int nc, size_t max_col) {
    const long long rest = (long long) nc * (long long) max_col + (long long) 2 * MAX_TILE_ROWS * CONSUMER_WARPS * nc * (long long) sizeof(float);
    return ((long long) budget - rest) / NSTAGES / 1024 * 1024;
}

template <int NC, int TYPE>
cudaError_t launch_kq(const GemvBatch & batch, int grid, size_t smem, cudaStream_t stream) {
    static PerDeviceOnce once;
    const cudaError_t ae = once.run([&] { return cudaFuncSetAttribute(gemv_kq_kernel<NC, TYPE>, cudaFuncAttributeMaxDynamicSharedMemorySize, KQ_WIDE_BUDGET); });
    if (ae != cudaSuccess) return ae;
    log_launch(LF_KQ_STREAMING, NC, TYPE, 0, 0, 0);
    return launch_pdl(gemv_kq_kernel<NC, TYPE>, dim3((unsigned) grid), dim3(THREADS), smem, stream, batch);
}

}  // namespace

bool gemv_kq_fits(int type, int K) {
    if (!dtype_kquant(type) || K < QK_K || K % QK_K) return false;
    GemvProblem p{};
    p.type = type; p.K = K;
    p.pitch = (long long) ((size_t) dtype_block_bytes(type) * (size_t) (K / QK_K));
    return plan_kq(p) && kq_stage_bytes(KQ_WIDE_BUDGET, 1, kq_act_bytes_per_column(K)) >= kq_tile_need(p);
}

cudaError_t gemv_kq_launch(GemvBatch & batch, const DeviceInfo & dev, cudaStream_t stream) {
    if (batch.n <= 0 || batch.T <= 0) return cudaSuccess;
    const int type = batch.p[0].type;
    size_t max_col = 0;
    long long need = 0;
    for (int i = 0; i < batch.n; i++) {
        GemvProblem & p = batch.p[i];
        if (p.type != type || p.pro != PRO_NONE || !plan_kq(p)) return cudaErrorNotSupported;
        max_col = std::max(max_col, kq_act_bytes_per_column(p.K));
        need = std::max(need, kq_tile_need(p));
    }
    const bool wide = kq_stage_bytes(CTA_SMEM_BUDGET, 1, max_col) < need;
    const int budget = wide ? KQ_WIDE_BUDGET : CTA_SMEM_BUDGET;
    int nc = 1;
    if (batch.T >= 4 && kq_stage_bytes(budget, 4, max_col) >= std::max(need, (long long) NOMINAL_STAGE_BYTES)) nc = 4;
    else if (batch.T >= 2 && kq_stage_bytes(budget, 2, max_col) >= std::max(need, (long long) NOMINAL_STAGE_BYTES)) nc = 2;
    const long long stage_bytes = kq_stage_bytes(budget, nc, max_col);
    if (stage_bytes < need) return cudaErrorNotSupported;
    const int grid = assign_tiles_and_ctas(batch, (wide ? 1 : 2) * dev.num_sms, stage_bytes);
    batch.max_col_bytes = (long long) max_col;
    batch.stage_bytes = stage_bytes;
    batch.trace = trace_slot(batch.n > 1 ? "gemv_kq(batch)" : "gemv_kq");
    const size_t smem = (size_t) NSTAGES * (size_t) stage_bytes + (size_t) nc * max_col + (size_t) 2 * MAX_TILE_ROWS * CONSUMER_WARPS * nc * sizeof(float);
    if (type == DT_Q4_K) {
        switch (nc) {
            case 4: return launch_kq<4, DT_Q4_K>(batch, grid, smem, stream);
            case 2: return launch_kq<2, DT_Q4_K>(batch, grid, smem, stream);
            default: return launch_kq<1, DT_Q4_K>(batch, grid, smem, stream);
        }
    }
    switch (nc) {
        case 4: return launch_kq<4, DT_Q5_K>(batch, grid, smem, stream);
        case 2: return launch_kq<2, DT_Q5_K>(batch, grid, smem, stream);
        default: return launch_kq<1, DT_Q5_K>(batch, grid, smem, stream);
    }
}

}  // namespace rwkv
