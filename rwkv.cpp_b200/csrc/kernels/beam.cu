// Beam search on the device (rwkv_b200_beam_search, rwkv_b200_beam_search_groups): the step that ranks the candidates of every live
// beam of every group and walks them into the next live beams and the pool of finished hypotheses, the gather that gives every live
// slot the state of its parent before the pass that evaluates it, and the copies that keep the slots of groups that stopped. Each
// candidate's log-probability is score_kernel's (score_row.cuh) and its top-N order that of the logprob step kernels (top_n.cuh), so a
// host search built from rwkv_b200_score_logits gives the same ranking bit for bit.
#include "ops.h"
#include "gemv.h"
#include "score_row.cuh"
#include "top_n.cuh"

namespace rwkv {
namespace {

constexpr int BEAM_RANKED = BEAM_MAX * BEAM_CANDS;

// The last CTA of group g's step (every thread): rank its ≤ n_live * 2W candidates, then thread 0 walks them (ops.h: BeamState) and
// takes the step's second ticket; the last walker sets the loop's conditionals.
__device__ __forceinline__ void beam_walk(const BeamStepParams & p, int g) {
    __shared__ double s_score[BEAM_RANKED];
    __shared__ uint32_t s_id[BEAM_RANKED];
    __shared__ int s_order[BEAM_RANKED];
    __shared__ int s_count;
    BeamState * st = p.st + g;
    const int tid = threadIdx.x, W = p.width, n = 2 * W, nc = (int) st->n_live * n;
    if (tid == 0) s_count = 0;
    double sc = 0.0;
    bool ok = false;
    if (tid < nc) {     // candidate tid = (beam b, position j); other CTAs wrote it: read past L1
        const int b = tid / n, j = tid % n;
        const float lp = __ldcg(&st->cand_lp[b][j]);
        ok = isfinite(lp);
        sc = __ldcg(&st->score[b]) + (double) lp;
        s_id[tid] = __ldcg(&st->cand_id[b][j]);
        s_score[tid] = ok ? sc : (double) NAN;
    }
    __syncthreads();
    if (ok) {           // rank = candidates that come first: a larger score, or the same score at a lower index (NaN: none)
        int r = 0;
        for (int j = 0; j < nc; j++) {
            const double o = s_score[j];
            r += (o > sc || (o == sc && j < tid)) ? 1 : 0;
        }
        s_order[r] = tid;
        atomicAdd(&s_count, 1);
    }
    __syncthreads();
    if (tid != 0) return;
    const uint32_t step = st->step;
    const size_t slots = (size_t) p.groups * W, first = (size_t) g * W;
    uint32_t L = 0, pool = st->n_pool;
    for (int r = 0; r < s_count && L < (uint32_t) W && pool < (uint32_t) W; r++) {
        const int c = s_order[r];
        const uint32_t b = (uint32_t) (c / n), tok = s_id[c];
        bool stop = false;
        for (uint32_t q = 0; q < st->n_stop; q++) stop = stop || st->stop[q] == tok;
        if (stop) {     // reported, never evaluated
            st->pool[pool++] = BeamHyp{s_score[c], step, b, tok, 0};
        } else {
            uint32_t * bp = p.back + ((size_t) step * slots + first + L) * 2;
            bp[0] = b; bp[1] = tok;
            st->parent[L] = b;
            st->score[L] = s_score[c];
            p.next_tokens[first + L] = (int) tok;
            L++;
        }
    }
    for (int k = (int) L; k < W; k++) p.next_tokens[first + k] = 0;
    const bool runs_on = L > 0 && pool < (uint32_t) W && step + 1 < st->max_tokens;
    if (!runs_on) {     // its last slots: those this step takes, or (L = 0) those of the step before, from the pass after them
        st->n_keep = L > 0 ? L : st->n_live;
        st->park_at = step + (L > 0 ? 2 : 1);
    }
    st->n_live = L; st->n_pool = pool; st->step = step + 1; st->ticket = 0;
    BeamLoop * lp = p.loop;
    // n_active was written by the previous launch; the last walker of this step rewrites it once it holds the final ticket, so it is
    // read before the ticket is taken (the fence orders the load before the atomic)
    const uint32_t n_active = *reinterpret_cast<volatile const uint32_t *>(&lp->n_active);
    if (L > 0) atomicAdd(&lp->any_live, 1u);
    if (runs_on) atomicAdd(&lp->n_next, 1u);
    __threadfence();
    if (atomicAdd(&lp->ticket, 1u) != n_active - 1) return;
    __threadfence();
    const uint32_t any_live = atomicAdd(&lp->any_live, 0u), n_next = atomicAdd(&lp->n_next, 0u);
    lp->n_active = n_next; lp->n_next = 0; lp->any_live = 0; lp->ticket = 0; lp->steps++;
    if (p.set_handles) {
        cudaGraphSetConditional(p.run_pass, any_live > 0 ? 1u : 0u);
        cudaGraphSetConditional(p.keep_going, n_next > 0 ? 1u : 0u);
    }
}

// CTA (k, g) of a group that runs, k < n_live: live beam k's top 2W entries and their log-probabilities into cand_*[k] of its group,
// in the order and arithmetic of Logprobs::record (sampling.cu); an invalid column or a missing entry (2W > n_vocab) gives NaN. The
// last CTA of the group to arrive walks it.
template <int PER>
__global__ void __launch_bounds__(SAMPLE_THREADS) beam_step_kernel(const BeamStepParams p) {
    pdl_prologue();
    __shared__ float s_max[LP_SCORE_WARPS];
    __shared__ int s_arg[LP_SCORE_WARPS], s_bad[LP_SCORE_WARPS];
    __shared__ double s_sum[LP_SCORE_WARPS];
    __shared__ unsigned long long s_top[SAMPLE_WARPS][GEN_TOP_MAX];
    __shared__ bool s_last;
    const int k = blockIdx.x, g = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, V = p.n_vocab, n = 2 * p.width;
    BeamState * st = p.st + g;
    const uint32_t n_live = st->n_live;
    if (n_live == 0 || st->n_pool >= (uint32_t) p.width || st->step >= st->max_tokens) return;     // stopped, or never ran
    if (k < (int) n_live) {
        const float * z = p.logits + ((size_t) g * p.width + k) * V;
        float mx = 0.f;
        bool valid = false;
        double log_sum = 0.0;
        if (tid < LP_SCORE_THREADS)
            score_column(tid, z, V, s_max, s_arg, s_bad, s_sum, [] { asm volatile("bar.sync 1, %0;" :: "n"(LP_SCORE_THREADS) : "memory"); },
                         [&](float m, int, bool v, double sum) { mx = m; valid = v; if (v) log_sum = log(sum); });
        warp_top_keys<PER>(z, V, tid, n, s_top);
        __syncthreads();
        if (warp == 0)
            merge_top_keys(lane, n, s_top, [&](int j, unsigned long long w) {
                if (lane != 0) return;
                const uint32_t id = ~(uint32_t) w;
                st->cand_id[k][j] = id;
                st->cand_lp[k][j] = (valid && w != 0) ? score_logprob(z[id], mx, log_sum) : NAN;
            });
    }
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        s_last = atomicAdd(&st->ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    beam_walk(p, g);
}

constexpr int GATHER_THREADS = 256, GATHER_BLOCKS_PER_SLOT = 128;

// n floats from -> to by the CTAs of blockIdx.x, as float4 when both start 16-byte aligned (aligned: every slice does).
__device__ __forceinline__ void copy_slice(const float * from, float * to, size_t n, bool aligned) {
    const size_t i0 = (size_t) blockIdx.x * GATHER_THREADS + threadIdx.x, stride = (size_t) gridDim.x * GATHER_THREADS;
    size_t done = 0;
    if (aligned) {
        const size_t n4 = n / 4;
        for (size_t i = i0; i < n4; i += stride) reinterpret_cast<float4 *>(to)[i] = reinterpret_cast<const float4 *>(from)[i];
        done = n4 * 4;
    }
    for (size_t i = done + i0; i < n; i += stride) to[i] = from[i];
}

// Grid (blocks, W, G): slot k of group g (ops.h: launch_beam_gather).
__global__ void __launch_bounds__(GATHER_THREADS) beam_gather_kernel(const BeamCopyParams p) {
    pdl_prologue();
    const int k = blockIdx.y, g = blockIdx.z;
    BeamState & st = p.st[g];
    const uint32_t steps = p.loop->steps;
    const size_t slot = (size_t) g * p.width + k, S = (size_t) p.seq_stride;
    const bool aligned = p.seq_stride % 4 == 0;
    if (st.step == steps && k < (int) st.n_live) {       // took live beams at the last step
        copy_slice(p.y + ((size_t) g * p.width + st.parent[k]) * S, p.x + slot * S, p.state_len, aligned);
    } else if (st.park_at == steps && k < (int) st.n_keep) {
        copy_slice(p.y + slot * S, p.x + slot * S, p.state_len, aligned);
        copy_slice(p.logits + slot * p.n_vocab, p.park + slot * p.n_vocab, (size_t) p.n_vocab, p.n_vocab % 4 == 0);
        if (k == 0 && blockIdx.x == 0 && threadIdx.x == 0) st.parked = 1;     // read only by the restore
    }
}

__global__ void __launch_bounds__(GATHER_THREADS) beam_restore_kernel(const BeamCopyParams p) {
    const int k = blockIdx.y, g = blockIdx.z;
    const BeamState & st = p.st[g];
    if (!st.parked || k >= (int) st.n_keep) return;
    const size_t slot = (size_t) g * p.width + k, S = (size_t) p.seq_stride;
    copy_slice(p.x + slot * S, p.y + slot * S, p.state_len, p.seq_stride % 4 == 0);
    copy_slice(p.park + slot * p.n_vocab, p.logits + slot * p.n_vocab, (size_t) p.n_vocab, p.n_vocab % 4 == 0);
}

void * beam_step_for(int n_vocab) {
    return with_sample_per(n_vocab, [](auto per) { return reinterpret_cast<void *>(beam_step_kernel<decltype(per)::value>); });
}

bool beam_args_ok(const BeamStepParams & p) {
    return p.n_vocab > 0 && p.n_vocab <= SAMPLE_THREADS * 64 && p.width >= 1 && p.width <= BEAM_MAX && p.groups >= 1 && p.groups <= 65535;
}

}  // namespace

cudaError_t launch_beam_step(const BeamStepParams & p, cudaStream_t s) {
    if (!beam_args_ok(p)) return cudaErrorInvalidValue;
    BeamStepParams copy = p;
    void * args[] = {&copy};
    return cudaLaunchKernel(beam_step_for(p.n_vocab), dim3(p.width, p.groups), dim3(SAMPLE_THREADS), args, 0, s);
}

cudaError_t add_beam_step_node(cudaGraph_t g, const cudaGraphNode_t * deps, size_t n_deps, const BeamStepParams & p, cudaGraphNode_t * node) {
    if (!beam_args_ok(p)) return cudaErrorInvalidValue;
    BeamStepParams copy = p;
    void * args[] = {&copy};
    cudaKernelNodeParams kp = {};
    kp.func = beam_step_for(p.n_vocab);
    kp.gridDim = dim3(p.width, p.groups); kp.blockDim = dim3(SAMPLE_THREADS); kp.sharedMemBytes = 0;
    kp.kernelParams = args; kp.extra = nullptr;
    return cudaGraphAddKernelNode(node, g, deps, n_deps, &kp);
}

cudaError_t launch_beam_gather(const BeamCopyParams & p, cudaStream_t s) {
    return launch_pdl(beam_gather_kernel, dim3(GATHER_BLOCKS_PER_SLOT, p.width, p.groups), dim3(GATHER_THREADS), 0, s, p);
}

cudaError_t add_beam_restore_node(cudaGraph_t g, const cudaGraphNode_t * deps, size_t n_deps, const BeamCopyParams & p, cudaGraphNode_t * node) {
    BeamCopyParams copy = p;
    void * args[] = {&copy};
    cudaKernelNodeParams kp = {};
    kp.func = reinterpret_cast<void *>(beam_restore_kernel);
    kp.gridDim = dim3(GATHER_BLOCKS_PER_SLOT, p.width, p.groups); kp.blockDim = dim3(GATHER_THREADS); kp.sharedMemBytes = 0;
    kp.kernelParams = args; kp.extra = nullptr;
    return cudaGraphAddKernelNode(node, g, deps, n_deps, &kp);
}

}  // namespace rwkv
