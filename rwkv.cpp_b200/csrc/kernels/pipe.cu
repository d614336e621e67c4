// Stage hand-off of the layer pipeline (SURVEY.md 8e) over peer memory: NVLink stores + flags instead of NCCL calls from the host.
//
// Every stage owns a MAILBOX in its own HBM that the previous stage writes (P2P stores through NVLink / NVSwitch, mapped with CUDA
// IPC between processes or peer access inside one) and a CREDIT word that the next stage writes back:
//
//   sender  (pipe_send_kernel, last kernel of a stage's pass)     receiver (pipe_recv_kernel, first kernel of a stage's pass)
//     wait   credit  > item - SLOTS      (slot is free)              wait   full[slot] == item + 1       (ld.acquire.sys)
//     store  x (+ v_first) -> peer mailbox slot                      copy   slot -> the pass's activation buffer
//     fence.sys, last CTA: st.release.sys full[slot] = item + 1      last CTA: st.release.sys credit = item + 1 (into the sender)
//
// Item numbers come from device-side ticket counters, so nothing in a launch depends on the host: the kernels are stream-ordered
// with the stage's GEMVs (and replay inside CUDA graphs), the host of a stage never synchronises with its neighbours, and the
// only data that crosses a stage boundary is x f32[C x T] (+ v_first for v7): 16 KB per token at 7B. The recurrent state never
// leaves the GPU that owns the layer. Waits are bounded (a lost neighbour traps the kernel instead of hanging the GPU).
#include "ops.h"
#include "gemv.h"

namespace rwkv {
namespace {

constexpr int PIPE_THREADS = 256;
constexpr long long PIPE_GUARD_CYCLES = 40000000000ll;      // ~20 s of SM clock

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long * p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long * p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// counters: [0] recv tickets, [1] recv CTAs done, [2] send tickets, [3] send CTAs done (monotonic; every launch has PIPE_CTAS CTAs)
template <bool SEND>
__global__ void __launch_bounds__(PIPE_THREADS) pipe_kernel(PipeBox * mine, PipeBox * peer, unsigned long long * counters, size_t slot_floats,
                                                            float * a0, size_t n0, float * a1, size_t n1, TraceRec * trace) {
    __shared__ unsigned long long item_sh;
    trace_begin(trace);
    asm volatile("griddepcontrol.wait;" ::: "memory");          // SEND reads what the stage's last kernel wrote
    const int tid = threadIdx.x;
    unsigned long long * tickets = counters + (SEND ? 2 : 0), * done = counters + (SEND ? 3 : 1);
    if (tid == 0) item_sh = atomicAdd(tickets, 1ull) / gridDim.x;
    __syncthreads();
    const unsigned long long item = item_sh;
    const int slot = (int) (item % PIPE_SLOTS);
    if (tid == 0) {
        const long long t0 = clock64();
        unsigned spins = 0;
        if (SEND) {      // the receiver has drained what this slot held before
            while (ld_acquire_sys(&mine->credit) + PIPE_SLOTS <= item) { __nanosleep(64); if ((++spins & 0x3FFu) == 0 && clock64() - t0 > PIPE_GUARD_CYCLES) __trap(); }
        } else {         // the sender has filled the slot
            while (ld_acquire_sys(&mine->full[slot]) != item + 1) { __nanosleep(64); if ((++spins & 0x3FFu) == 0 && clock64() - t0 > PIPE_GUARD_CYCLES) __trap(); }
        }
    }
    __syncthreads();
    PipeBox * box = SEND ? peer : mine;
    float * data = reinterpret_cast<float *>(box + 1) + (size_t) slot * slot_floats;
    const size_t n4 = (n0 + n1) / 4, per = (n4 + gridDim.x - 1) / gridDim.x;
    const size_t lo = blockIdx.x * per, hi = lo + per < n4 ? lo + per : n4;
    for (size_t i = lo + tid; i < hi; i += PIPE_THREADS) {
        const size_t e = i * 4;
        float * act = e < n0 ? a0 + e : a1 + (e - n0);          // n0 is a multiple of 4
        if (SEND) reinterpret_cast<float4 *>(data)[i] = *reinterpret_cast<const float4 *>(act);
        else *reinterpret_cast<float4 *>(act) = __ldcv(reinterpret_cast<const float4 *>(data) + i);      // written by the peer: never from a stale cache line
    }
    if (SEND) __threadfence_system(); else __threadfence();
    __syncthreads();
    if (tid == 0 && (atomicAdd(done, 1ull) + 1) % gridDim.x == 0) {      // last CTA of this launch: everybody's copies are fenced
        __threadfence_system();
        if (SEND) st_release_sys(&peer->full[slot], item + 1);
        else if (peer) st_release_sys(&peer->credit, item + 1);
    }
    trace_end(trace);
}

}  // namespace

cudaError_t launch_pipe_recv(PipeBox * mine, PipeBox * prev, unsigned long long * counters, size_t slot_floats, float * x, size_t nx, float * v, size_t nv, cudaStream_t s) {
    g_kernel_launches++;
    pipe_kernel<false><<<PIPE_CTAS, PIPE_THREADS, 0, s>>>(mine, prev, counters, slot_floats, x, nx, v, nv, trace_slot("pipe_recv"));
    return cudaGetLastError();
}

cudaError_t launch_pipe_send(PipeBox * mine, PipeBox * next, unsigned long long * counters, size_t slot_floats, float * x, size_t nx, float * v, size_t nv, cudaStream_t s) {
    return launch_pdl(pipe_kernel<true>, dim3(PIPE_CTAS), dim3(PIPE_THREADS), 0, s, mine, next, counters, slot_floats, x, nx, v, nv, trace_slot("pipe_send"));
}

}  // namespace rwkv
