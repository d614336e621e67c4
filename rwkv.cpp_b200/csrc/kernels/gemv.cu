// Fused dequantize-and-GEMV for single-token decode and short chunks (SIMT, batch-invariant).
//
// Shape of the kernel
//   * persistent grid: num_SMs x CTAS_PER_SM CTAs, partitioned over the problems of the batch in
//     proportion to their weight bytes; a CTA serves exactly one problem, so it stages exactly one
//     activation vector;
//   * prologue: the CTA converts the fp32 input column(s) into the operand the reference's CPU path
//     would multiply with -- Q8_0 / Q8_1 blocks for quantised weights, fp16 for F16 weights, fp32 for
//     F32 weights (ggml-cpu.c:253-311 `vec_dot_type`) -- and keeps it in shared memory;
//   * main loop: one warp per output row, lanes stride over 4-byte-aligned block units of the row in
//     the native ggml layout, int8 dot products with dp4a, fp32 accumulate, xor-shuffle reduction;
//   * epilogue: activation / bias / residual fused, single writer per output.
// The per-column arithmetic does not depend on how many columns are processed together, so a token
// evaluated alone (rwkv_eval) and inside a chunk (rwkv_eval_sequence) produces identical bits -- the
// reference's tests memcmp those states (tests/test_eval_sequence_in_chunks.c:54).
#include "gemv.h"
#include "quant_decode.cuh"

#include <cuda_fp16.h>
#include <cstring>
#include <mutex>
#include <set>
#include <utility>

namespace rwkv {

std::atomic<unsigned long long> g_kernel_launches{0};
thread_local TraceRec * g_trace_base = nullptr;
thread_local int g_trace_next = 0;
thread_local const char * g_trace_names[1024];
thread_local LaunchLog * g_launch_log = nullptr;

namespace {

constexpr int GEMV_WARPS = 8;
constexpr int GEMV_THREADS = GEMV_WARPS * 32;
constexpr int CTAS_PER_SM = 2;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ int warp_sum_int(int v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_sum_double(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Sum over the whole CTA in double (LayerNorm statistics, as ggml-cpu.c:6906-6923 sums in double).
__device__ double block_sum_double(double v, double * scratch /* GEMV_WARPS + 1 */) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    v = warp_sum_double(v);
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0;
        for (int i = 0; i < GEMV_WARPS; i++) s += scratch[i];
        scratch[GEMV_WARPS] = s;
    }
    __syncthreads();
    return scratch[GEMV_WARPS];
}

__device__ __forceinline__ float round_to_half(float v) { return __half2float(__float2half_rn(v)); }

// Bytes of shared memory one staged activation column takes.
__host__ __device__ inline size_t stage_bytes_per_column(int type, int K) {
    size_t b;
    if (type == DT_F32) b = (size_t) K * 4;
    else if (type == DT_F16) b = (size_t) K * 2;
    else b = (size_t) K + (size_t) (K / 32) * sizeof(ActScale);
    return (b + 15) & ~(size_t) 15;
}

struct LnStats { float mean, rstd; };

// ---- prologue: stage `nc` activation columns ----------------------------------------------------
__device__ void stage_columns(const GemvProblem & P, int c0, int nc, uint8_t * smem, double * red) {
    const int K = P.K, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t colb = stage_bytes_per_column(P.type, K);
    for (int c = 0; c < nc; c++) {
        const float * x = P.x + (long long) (c0 + c) * P.ldx;
        float mean = 0.f, rstd = 1.f;
        if (P.pro == PRO_LAYERNORM) {   // rwkv_layer_norm (rwkv_operators.inc:93-97) fused into the load
            double s = 0;
            for (int k = threadIdx.x; k < K; k += GEMV_THREADS) s += (double) x[k];
            mean = (float) (block_sum_double(s, red) / K);
            double s2 = 0;
            for (int k = threadIdx.x; k < K; k += GEMV_THREADS) { float v = x[k] - mean; s2 += (double) (v * v); }
            float var = (float) (block_sum_double(s2, red) / K);
            rstd = 1.0f / sqrtf(var + 1e-5f);
        }
        auto load = [&](int k) -> float {
            float v = x[k];
            if (P.pro == PRO_LAYERNORM) v = __fadd_rn(__fmul_rn(__fmul_rn(v - mean, rstd), P.ln_w[k]), P.ln_b[k]);
            return v;
        };
        uint8_t * col = smem + c * colb;
        if (P.type == DT_F32) {
            float * d = reinterpret_cast<float *>(col);
            for (int k = threadIdx.x; k < K; k += GEMV_THREADS) d[k] = load(k);
        } else if (P.type == DT_F16) {
            __half * d = reinterpret_cast<__half *>(col);
            for (int k = threadIdx.x; k < K; k += GEMV_THREADS) d[k] = __float2half_rn(load(k));
        } else {
            // quantize_row_q8_0 / quantize_row_q8_1, x86 flavour (ggml-cpu-quants.c:781-846, 1085-1160)
            const bool has_min = (P.type == DT_Q4_1 || P.type == DT_Q5_1);
            int8_t * q = reinterpret_cast<int8_t *>(col);
            ActScale * sc = reinterpret_cast<ActScale *>(col + K);
            const int nblk = K / 32;
            for (int b = warp; b < nblk; b += GEMV_WARPS) {
                float v = load(b * 32 + lane);
                float amax = warp_max(fabsf(v));
                float d32 = amax / 127.0f;
                float id = (amax != 0.0f) ? 127.0f / amax : 0.0f;
                int qi = __float2int_rn(v * id);
                int isum = warp_sum_int(qi);
                q[b * 32 + lane] = (int8_t) qi;
                if (lane == 0) {
                    ActScale a;
                    a.d = round_to_half(d32);
                    a.s = has_min ? round_to_half(d32 * (float) isum) : (float) isum;
                    sc[b] = a;
                }
            }
        }
    }
}

// ---- row dot products ----------------------------------------------------------------------------
template <int TYPE, int NC>
__device__ __forceinline__ void row_dot_quant(const uint8_t * wrow, int K, const uint8_t * smem, size_t colb, int nc, float acc[NC]) {
    using TR = QTraits<TYPE>;
    const int lane = threadIdx.x & 31;
    const int nblk = K / 32;
    const int nunits = (nblk + TR::UNIT_BLOCKS - 1) / TR::UNIT_BLOCKS;
    for (int u = lane; u < nunits; u += 32) {
        const uint32_t * wp = reinterpret_cast<const uint32_t *>(wrow) + (size_t) u * TR::UNIT_WORDS;
        uint32_t w[TR::UNIT_WORDS];
#pragma unroll
        for (int i = 0; i < TR::UNIT_WORDS; i++) w[i] = __ldg(wp + i);
#pragma unroll
        for (int b = 0; b < TR::UNIT_BLOCKS; b++) {
            const int blk = u * TR::UNIT_BLOCKS + b;
            if (blk < nblk) {
                BlockQ bq;
                decode_block<TYPE>(w, b, bq);
#pragma unroll
                for (int c = 0; c < NC; c++) {
                    if (c < nc) {
                        const uint8_t * col = smem + c * colb;
                        const int4 * ap = reinterpret_cast<const int4 *>(col + blk * 32);
                        int4 a0 = ap[0], a1 = ap[1];
                        int a8[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                        ActScale as = reinterpret_cast<const ActScale *>(col + K)[blk];
                        acc[c] = block_dot<TYPE>(bq, a8, as, acc[c]);
                    }
                }
            }
        }
    }
}

template <int NC>
__device__ __forceinline__ void row_dot_f16(const uint8_t * wrow, int K, const uint8_t * smem, size_t colb, int nc, float acc[NC]) {
    const int lane = threadIdx.x & 31;
    const int K8 = K & ~7;
    for (int k = lane * 8; k < K8; k += 256) {
        uint4 wv = __ldg(reinterpret_cast<const uint4 *>(wrow + (size_t) k * 2));
        const __half2 * wh = reinterpret_cast<const __half2 *>(&wv);
#pragma unroll
        for (int c = 0; c < NC; c++) {
            if (c < nc) {
                uint4 xv = *reinterpret_cast<const uint4 *>(smem + c * colb + (size_t) k * 2);
                const __half2 * xh = reinterpret_cast<const __half2 *>(&xv);
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    float2 wf = __half22float2(wh[i]), xf = __half22float2(xh[i]);
                    acc[c] = __fmaf_rn(wf.x, xf.x, acc[c]);
                    acc[c] = __fmaf_rn(wf.y, xf.y, acc[c]);
                }
            }
        }
    }
    for (int k = K8 + lane; k < K; k += 32) {   // ragged tail (never hit by real models)
        float wf = __half2float(reinterpret_cast<const __half *>(wrow)[k]);
#pragma unroll
        for (int c = 0; c < NC; c++)
            if (c < nc) acc[c] = __fmaf_rn(wf, __half2float(reinterpret_cast<const __half *>(smem + c * colb)[k]), acc[c]);
    }
}

template <int NC>
__device__ __forceinline__ void row_dot_f32(const uint8_t * wrow, int K, const uint8_t * smem, size_t colb, int nc, float acc[NC]) {
    const int lane = threadIdx.x & 31;
    const int K4 = K & ~3;
    for (int k = lane * 4; k < K4; k += 128) {
        float4 wv = __ldg(reinterpret_cast<const float4 *>(wrow + (size_t) k * 4));
#pragma unroll
        for (int c = 0; c < NC; c++) {
            if (c < nc) {
                float4 xv = *reinterpret_cast<const float4 *>(smem + c * colb + (size_t) k * 4);
                acc[c] = __fmaf_rn(wv.x, xv.x, acc[c]);
                acc[c] = __fmaf_rn(wv.y, xv.y, acc[c]);
                acc[c] = __fmaf_rn(wv.z, xv.z, acc[c]);
                acc[c] = __fmaf_rn(wv.w, xv.w, acc[c]);
            }
        }
    }
    for (int k = K4 + lane; k < K; k += 32) {
        float wf = reinterpret_cast<const float *>(wrow)[k];
#pragma unroll
        for (int c = 0; c < NC; c++)
            if (c < nc) acc[c] = __fmaf_rn(wf, reinterpret_cast<const float *>(smem + c * colb)[k], acc[c]);
    }
}

__device__ __forceinline__ float sigmoidf_(float v) { return 1.0f / (1.0f + expf(-v)); }

__device__ __forceinline__ float apply_epilogue(const GemvProblem & P, int row, int col, float v) {
    switch (P.epi) {
        case EPI_SIGMOID: return sigmoidf_(v);
        case EPI_SILU: return v / (1.0f + expf(-v));
        case EPI_TANH: return tanhf(v);
        case EPI_RELU_SQR: { float r = fmaxf(v, 0.0f); return __fmul_rn(r, r); }
        case EPI_ADD: return __fadd_rn(P.res[(long long) col * P.ldres + row], v);
        case EPI_MUL_ADD: return __fadd_rn(P.res[(long long) col * P.ldres + row], __fmul_rn(P.gate[(long long) col * P.ldgate + row], v));
        case EPI_BIAS_EXPNEGEXP: return expf(-expf(__fadd_rn(v, P.bias[row])));
        case EPI_BIAS_SIGMOID: return sigmoidf_(__fadd_rn(v, P.bias[row]));
        case EPI_BIAS_W7: return expf(__fmul_rn(sigmoidf_(__fadd_rn(v, P.bias[row])), -0.606531f));
        default: return v;
    }
}

template <int NC>
__global__ void __launch_bounds__(GEMV_THREADS) gemv_kernel(const GemvBatch batch) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ double red[GEMV_WARPS + 1];
    __shared__ GemvProblem P;
    trace_begin(batch.trace);
    pdl_prologue();

    {   // which problem does this CTA serve?
        int pi = 0;
        for (int i = 1; i < batch.n; i++) if ((int) blockIdx.x >= batch.p[i].first_cta) pi = i;
        if (threadIdx.x == 0) P = batch.p[pi];
        __syncthreads();
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int local_cta = (int) blockIdx.x - P.first_cta;
    const size_t colb = stage_bytes_per_column(P.type, P.K);
    const uint8_t * Wb = reinterpret_cast<const uint8_t *>(P.W);

    for (int c0 = 0; c0 < batch.T; c0 += NC) {
        const int nc = min(NC, batch.T - c0);
        if (c0 > 0) __syncthreads();
        stage_columns(P, c0, nc, smem, red);
        __syncthreads();
        for (int row = local_cta * GEMV_WARPS + warp; row < P.M; row += P.n_cta * GEMV_WARPS) {
            const uint8_t * wrow = Wb + (size_t) row * (size_t) P.pitch;
            float acc[NC];
#pragma unroll
            for (int c = 0; c < NC; c++) acc[c] = 0.0f;
            switch (P.type) {
                case DT_Q4_0: row_dot_quant<DT_Q4_0, NC>(wrow, P.K, smem, colb, nc, acc); break;
                case DT_Q4_1: row_dot_quant<DT_Q4_1, NC>(wrow, P.K, smem, colb, nc, acc); break;
                case DT_Q5_0: row_dot_quant<DT_Q5_0, NC>(wrow, P.K, smem, colb, nc, acc); break;
                case DT_Q5_1: row_dot_quant<DT_Q5_1, NC>(wrow, P.K, smem, colb, nc, acc); break;
                case DT_Q8_0: row_dot_quant<DT_Q8_0, NC>(wrow, P.K, smem, colb, nc, acc); break;
                case DT_F16: row_dot_f16<NC>(wrow, P.K, smem, colb, nc, acc); break;
                default: row_dot_f32<NC>(wrow, P.K, smem, colb, nc, acc); break;
            }
#pragma unroll
            for (int c = 0; c < NC; c++) {
                float v = warp_sum(acc[c]);
                if (c < nc && lane == 0) P.y[(long long) (c0 + c) * P.ldy + row] = apply_epilogue(P, row, c0 + c, v);
            }
        }
    }
    trace_end(batch.trace);
}

template <int NC>
cudaError_t launch_nc(const GemvBatch & batch, int grid, size_t smem, int max_optin, cudaStream_t stream) {
    static PerDeviceOnce once;                // the shared-memory opt-in is per device
    const cudaError_t ae = once.run([&] { return cudaFuncSetAttribute(gemv_kernel<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_optin - 1024); });
    if (ae != cudaSuccess) return ae;
    log_launch(LF_GENERIC, NC, -1, 0, 0, 0);
    return launch_pdl(gemv_kernel<NC>, dim3(grid), dim3(GEMV_THREADS), smem, stream, batch);
}

}  // namespace

namespace {
// one thread per quant block: the block's qh word (2 bytes into a Q5_0 block, 4 bytes into a Q5_1 block; 2-byte aligned) -> device order
__global__ void qh5_to_device_kernel(uint8_t * W, long long pitch, int M, int nblk, int block_bytes, int qh_offset) {
    const long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long) M * nblk) return;
    const int row = (int) (i / nblk), blk = (int) (i % nblk);
    unsigned short * p = reinterpret_cast<unsigned short *>(W + (long long) row * pitch + (long long) blk * block_bytes + qh_offset);
    const uint32_t qh = qh5_to_device((uint32_t) p[0] | ((uint32_t) p[1] << 16));
    p[0] = (unsigned short) (qh & 0xFFFFu);
    p[1] = (unsigned short) (qh >> 16);
}
}  // namespace

void prefer_max_shared_carveout(const void * kernel) {
    static std::mutex mu;
    static std::set<std::pair<int, const void *>> done;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lock(mu);
    if (!done.insert({dev, kernel}).second) return;
    cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, (int) cudaSharedmemCarveoutMaxShared);      // a preference: failure is harmless
    cudaGetLastError();
}

cudaError_t weights_to_device_layout(void * W, long long pitch, int type, int M, int K, cudaStream_t stream) {
    if (type != DT_Q5_0 && type != DT_Q5_1) return cudaSuccess;
    const int nblk = K / 32;
    const long long n = (long long) M * nblk;
    if (n <= 0) return cudaSuccess;
    qh5_to_device_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, stream>>>(reinterpret_cast<uint8_t *>(W), pitch, M, nblk, dtype_block_bytes(type), type == DT_Q5_0 ? 2 : 4);
    return cudaGetLastError();
}

cudaError_t gemv_launch(GemvBatch & batch, const DeviceInfo & dev, cudaStream_t stream) {
    if (batch.n <= 0 || batch.T <= 0) return cudaSuccess;
    bool any_kq = false;
    for (int i = 0; i < batch.n; i++) any_kq = any_kq || dtype_kquant(batch.p[i].type);
    if (any_kq) {
        // one launch per K-quant type present and one for the rest: a v7 layer keeps its LoRA matrices in FP16, a v6 layer's decay
        // LoRA falls back to a legacy format, so mixed batches are the common case
        GemvBatch part[3];
        for (GemvBatch & b : part) { memset(&b, 0, sizeof(b)); b.T = batch.T; }
        for (int i = 0; i < batch.n; i++) {
            const int t = batch.p[i].type;
            GemvBatch & b = part[t == DT_Q4_K ? 0 : (t == DT_Q5_K ? 1 : 2)];
            b.p[b.n++] = batch.p[i];
        }
        for (int k = 0; k < 2; k++) if (part[k].n) {
            const cudaError_t e = gemv_kq_launch(part[k], dev, stream);
            if (e != cudaSuccess) return e;
        }
        return gemv_launch(part[2], dev, stream);
    }
    const cudaError_t e = gemv_tma_launch(batch, dev, stream);
    if (e != cudaErrorNotSupported) return e;
    return gemv_generic_launch(batch, dev, stream);
}

cudaError_t gemv_route(GemvBatch & batch, const DeviceInfo & dev, cudaStream_t stream, void * workspace, size_t workspace_bytes, int tc_min_T) {
    if (!workspace || batch.T < tc_min_T) return gemv_launch(batch, dev, stream);
    GemvBatch tcb, rest;
    memset(&tcb, 0, sizeof(tcb)); memset(&rest, 0, sizeof(rest));
    tcb.T = rest.T = batch.T;
    for (int i = 0; i < batch.n; i++) {
        if (gemm_tc_supported(batch.p[i], batch.T)) tcb.p[tcb.n++] = batch.p[i];
        else rest.p[rest.n++] = batch.p[i];
    }
    if (tcb.n) {
        const cudaError_t e = gemm_tc_launch(tcb, dev, stream, workspace, workspace_bytes);
        if (e != cudaSuccess) return e;
    }
    return rest.n ? gemv_launch(rest, dev, stream) : cudaSuccess;
}

cudaError_t gemv_generic_launch(GemvBatch & batch, const DeviceInfo & dev, cudaStream_t stream) {
    for (int i = 0; i < batch.n; i++) if (dtype_kquant(batch.p[i].type)) return cudaErrorNotSupported;   // gemv_kq_launch only
    batch.trace = trace_slot("gemv_generic");
    // CTA budget split over the problems in proportion to their weight bytes.
    const int total_ctas = dev.num_sms * CTAS_PER_SM;
    double total_bytes = 0;
    size_t max_col = 0;
    for (int i = 0; i < batch.n; i++) {
        total_bytes += (double) batch.p[i].M * (double) batch.p[i].pitch;
        size_t cb = stage_bytes_per_column(batch.p[i].type, batch.p[i].K);
        if (cb > max_col) max_col = cb;
    }
    int next = 0;
    for (int i = 0; i < batch.n; i++) {
        GemvProblem & p = batch.p[i];
        int want = (int) ((double) total_ctas * ((double) p.M * (double) p.pitch) / total_bytes + 0.5);
        int cap = (p.M + GEMV_WARPS - 1) / GEMV_WARPS;
        if (want > cap) want = cap;
        if (want < 1) want = 1;
        p.first_cta = next;
        p.n_cta = want;
        next += want;
    }
    // columns staged together: as many as fit (weights are re-read from L2 once per column group)
    const size_t budget = (size_t) dev.max_smem_optin - 4096;
    int nc = 1;
    if (batch.T >= 4 && 4 * max_col <= budget) nc = 4;
    else if (batch.T >= 2 && 2 * max_col <= budget) nc = 2;
    if (max_col > budget) return cudaErrorInvalidValue;
    switch (nc) {
        case 4: return launch_nc<4>(batch, next, 4 * max_col, dev.max_smem_optin, stream);
        case 2: return launch_nc<2>(batch, next, 2 * max_col, dev.max_smem_optin, stream);
        default: return launch_nc<1>(batch, next, max_col, dev.max_smem_optin, stream);
    }
}

}  // namespace rwkv
