// Fused dequantize-and-GEMV: y[M, T] = epilogue(W[M, K] . prologue(x[K, T])) for a batch of
// independent problems in one launch (e.g. r/k/v/g + decay-LoRA of one RWKV layer).
// Replaces ggml_mul_mat on the eval path (reference rwkv_graph.inc:112-116, 244-252, 349-363, 384,
// 504-510, 708; CPU ggml-cpu.c:7377 + quant vec_dot kernels; CUDA ggml-cuda/mmvq.cu:55, mmv.cu:5).
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include <cstdint>
#include <utility>

namespace rwkv {

enum GemvEpilogue : int {
    EPI_NONE = 0,
    EPI_SIGMOID,          // 1/(1+exp(-v))
    EPI_SILU,             // v/(1+exp(-v))
    EPI_TANH,
    EPI_RELU_SQR,         // max(v,0)^2
    EPI_ADD,              // res + v                       (residual add after att.output)
    EPI_MUL_ADD,          // res + gate*v                  (x + r*(Wv k) of the channel mix)
    EPI_BIAS_EXPNEGEXP,   // exp(-exp(v + bias[row]))      (v6 decay, rwkv_graph.inc:365-367)
    EPI_BIAS_SIGMOID,     // sigmoid(v + bias[row])        (v7 a / v-gate, rwkv_graph.inc:417-423, 445-450)
    EPI_BIAS_W7,          // exp(-0.606531*sigmoid(v+bias[row]))  (v7 decay, rwkv_graph.inc:425-430)
};
// PRO_LAYERNORM: LN(x; ln_w, ln_b, eps 1e-5) applied while staging x (the head).
enum GemvPrologue : int { PRO_NONE = 0, PRO_LAYERNORM = 1 };

struct GemvProblem {
    const void * W;          // device, rows of quant blocks / f16 / f32, `pitch` bytes apart (16-B multiple)
    const void * Wt;         // device, tile-major prefill copy of W (gemm_tc_repack) or NULL: no tensor-core path
    long long pitch;
    int type, K, M;
    const float * x;  long long ldx;      // input  column t at x + t*ldx
    // Single-token launches of the streaming kernel: x[:, 0] already in the staged layout of this problem's (type, K) (act_stage.cuh),
    // emitted by the kernel that produced x. The consumers copy it instead of quantising x; NULL = stage from x. Ignored by the
    // generic kernel and the tensor-core path.
    const unsigned char * xq;
    float * y;        long long ldy;      // output column t at y + t*ldy
    const float * res;  long long ldres;
    const float * gate; long long ldgate;
    const float * bias;                   // [M]
    const float * ln_w; const float * ln_b;  // [K]
    int epi, pro;
    int first_cta, n_cta;                 // filled by gemv_launch
    int wk, g, tile_rows;                 // streaming kernel only: warps sharing a row along K, lanes per row, rows per TMA tile
};

// In-kernel timeline (our stand-in for nsys, which this image lacks): when a trace slot is attached, thread 0 of every
// CTA folds %globaltimer into [min start, max end] of the slot. Works inside CUDA-graph replays.
struct TraceRec { unsigned long long start, end, mark[4]; };   // mark[]: optional intra-kernel points of CTA 0
// The cursor belongs to the host thread that is enqueuing a pass (contexts are evaluated one thread each, rwkv.h:94-96): thread_local,
// so two clones traced from two threads never share slots; enqueue_pass copies the names into its Context when the pass is complete.
extern thread_local TraceRec * g_trace_base;        // device buffer, or nullptr when tracing is off
extern thread_local int g_trace_next;               // next free slot of the current pass
extern thread_local const char * g_trace_names[1024];
inline TraceRec * trace_slot(const char * name) {
    if (!g_trace_base || g_trace_next >= 1024) return nullptr;
    g_trace_names[g_trace_next] = name;
    return g_trace_base + g_trace_next++;
}

constexpr int GEMV_MAX_PROBLEMS = 8;
struct GemvBatch {
    int n, T;
    TraceRec * trace;
    long long max_col_bytes, stage_bytes; // streaming kernel only: shared-memory carve-up
    GemvProblem p[GEMV_MAX_PROBLEMS];
};

struct DeviceInfo { int device; int num_sms; int max_smem_optin; };

// Enqueues one kernel on `stream` covering all problems. Returns cudaSuccess or the launch error.
// Uses the TMA streaming kernel (gemv_tma.cu) whenever every problem's shape fits it, else the generic
// direct-load kernel (gemv.cu); the choice depends on the problem shapes only, never on T.
cudaError_t gemv_launch(GemvBatch & batch, const DeviceInfo & dev, cudaStream_t stream);
// The eval path's routing of a batch: with a tensor-core workspace and T >= tc_min_T, the problems gemm_tc_supported accepts go to one
// gemm_tc_launch and the rest to gemv_launch; otherwise the whole batch goes to gemv_launch. workspace may be NULL (no tensor cores).
cudaError_t gemv_route(GemvBatch & batch, const DeviceInfo & dev, cudaStream_t stream, void * workspace, size_t workspace_bytes, int tc_min_T);
cudaError_t gemv_tma_launch(GemvBatch & batch, const DeviceInfo & dev, cudaStream_t stream);      // cudaErrorNotSupported if a shape does not fit
// The streaming kernel's row plan of p (p.wk, p.g), a function of (type, K, pitch) alone; false if the shape needs the generic kernel.
bool gemv_tma_plan(GemvProblem & p);
cudaError_t gemv_generic_launch(GemvBatch & batch, const DeviceInfo & dev, cudaStream_t stream);
// Q4_K / Q5_K matrices (gemv_kquant.cu): the only kernel that takes them; every problem of `batch` has the same K-quant type and no
// prologue. gemv_kq_fits: whether rows of K weights fit its streaming plan (the loader refuses a matrix that does not).
bool gemv_kq_fits(int type, int K);
cudaError_t gemv_kq_launch(GemvBatch & batch, const DeviceInfo & dev, cudaStream_t stream);
// Tile height and CTA share of every problem of a streaming launch (gemv_tma.cu), shared by both streaming kernels.
int assign_tiles_and_ctas(GemvBatch & batch, int total_ctas, long long stage_bytes);

// Brings a freshly uploaded matrix (file bytes, rows `pitch` bytes apart) into the device layout of quant_decode.cuh, in place: the
// fifth-bit word of every Q5_0 / Q5_1 block is bit-transposed (qh5_to_device); every other type is left as it is. Must run before any
// kernel reads the matrix (including gemm_tc_repack).
cudaError_t weights_to_device_layout(void * W, long long pitch, int type, int M, int K, cudaStream_t stream);

// Tensor-core (wgmma) path for chunks of >= 32 tokens (gemm_tc.cu). act16_scratch: device scratch for the fp16 copies of the
// input matrices (sum over distinct inputs of round16(T) * K halves).
bool gemm_tc_supported(const GemvProblem & p, int T);
// The tile-major prefill copy of a matrix the tensor-core path streams (0 bytes = the matrix cannot take that path).
bool gemm_tc_eligible(int type, int K);
size_t gemm_tc_tiled_bytes(int type, int M, int K);
cudaError_t gemm_tc_repack(const void * W, long long pitch, int type, int M, int K, void * dst, cudaStream_t stream);
// workspace: gemm_tc_workspace_bytes(T, sum over the batch's distinct inputs of round16(T) * K) bytes of device memory, 256-byte aligned
// (what cudaMalloc returns).
size_t gemm_tc_workspace_bytes(int T, size_t operand_halves);
// Enough for any batch of T tokens whose inputs have at most k_max rows (GEMV_MAX_PROBLEMS distinct inputs).
inline size_t gemm_tc_batch_workspace_bytes(int T, size_t k_max) {
    return gemm_tc_workspace_bytes(T, (size_t) GEMV_MAX_PROBLEMS * (k_max * (size_t) ((T + 15) / 16 * 16) + 128));
}
cudaError_t gemm_tc_launch(GemvBatch & batch, const DeviceInfo & dev, cudaStream_t stream, void * workspace, size_t workspace_bytes);

// Every kernel of the eval path asks for the SAME L1 / shared-memory split (all shared): an SM can only change its carve-out when it is
// idle, so a stream that alternates between 113-225 KB weight-streaming kernels and small glue kernels with the default (L1-heavy)
// preference makes every kernel boundary wait for the SMs to drain instead of overlapping through programmatic dependent launch.
// Once per (device, kernel).
void prefer_max_shared_carveout(const void * kernel);

// Per-launch count of kernels this module has enqueued (bench.py reports it as gpu_launches).
extern std::atomic<unsigned long long> g_kernel_launches;

// Which instantiation of the matrix kernels a launch ran, recorded while a log is attached to the calling thread (the GEMV test hook
// attaches one, so its tests can assert the kernel they reached instead of assuming it). Fields that do not apply to a family are 0,
// except `only`, -1 where a kernel serves every format.
enum LaunchFamily : int { LF_STREAMING = 0, LF_GENERIC = 1, LF_TENSOR_CORES = 2, LF_CONVERT = 3, LF_EXPAND = 4, LF_KQ_STREAMING = 5, LF_KQ_EXPAND = 6 };
struct LaunchRec {
    int family;
    int nc;        // streaming / generic / K-quant streaming: columns per group (NC); convert: distinct inputs
    int only;      // streaming: ONLY (-1 = mixed formats); expand, K-quant streaming / expand: the weight type; convert: 16 (Q8_K) or 0
    int has_ln;    // streaming: HAS_LN
    int npad;      // tensor cores / convert: tokens padded to 16
    int cluster;   // tensor cores: CTAs per cluster
};
struct LaunchLog { static constexpr int CAP = 32; LaunchRec rec[CAP]; int n; };
extern thread_local LaunchLog * g_launch_log;
inline void log_launch(int family, int nc, int only, int has_ln, int npad, int cluster) {
    LaunchLog * l = g_launch_log;
    if (l && l->n < LaunchLog::CAP) l->rec[l->n++] = LaunchRec{family, nc, only, has_ln, npad, cluster};
}

// Launches every kernel of the eval path, and counts it: with the PDL attribute (the kernel may start while its predecessor in the
// stream is still running; it must execute griddepcontrol.wait before touching anything the predecessor writes), the carve-out
// preference above and, when cluster > 1, thread-block clusters of that many CTAs along x.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(unsigned cluster, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args &&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[2];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.numAttrs = 1;
    if (cluster > 1) {
        attr[1].id = cudaLaunchAttributeClusterDimension;
        attr[1].val.clusterDim.x = cluster; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = 1;
        cfg.numAttrs = 2;
    }
    cfg.attrs = attr;
    prefer_max_shared_carveout(reinterpret_cast<const void *>(kernel));
    g_kernel_launches++;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args &&... args) {
    return launch_pdl(1u, kernel, grid, block, smem, stream, std::forward<Args>(args)...);
}
#if defined(__CUDACC__)
// First statement of every non-GEMV kernel: let the successor start (it will prefetch its weights), then wait for the
// predecessor's results.
__device__ __forceinline__ void trace_begin(TraceRec * t) {
    if (t && threadIdx.x == 0) { unsigned long long g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g)); atomicMin(&t->start, g); }
}
__device__ __forceinline__ void trace_end(TraceRec * t) {
    if (t && threadIdx.x == 0) { unsigned long long g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g)); atomicMax(&t->end, g); }
}
__device__ __forceinline__ void trace_mark(TraceRec * t, int i) {
    if (t && threadIdx.x == 0 && blockIdx.x == 0) { unsigned long long g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g)); t->mark[i] = g; }
}
__device__ __forceinline__ void pdl_prologue() {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
}
#endif

// One-time per-device function attribute (dynamic shared-memory opt-in): several host threads may launch concurrently.
struct PerDeviceOnce {
    std::atomic<bool> done[64] = {};
    template <typename F> cudaError_t run(F && set) {
        int dev = 0;
        cudaGetDevice(&dev);
        if (dev < 0 || dev >= 64) return set();
        if (done[dev].load(std::memory_order_acquire)) return cudaSuccess;
        const cudaError_t e = set();               // idempotent: a second thread repeating it is harmless
        if (e == cudaSuccess) done[dev].store(true, std::memory_order_release);
        return e;
    }
};

}  // namespace rwkv
