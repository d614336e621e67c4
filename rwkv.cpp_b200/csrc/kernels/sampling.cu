// On-device sampling of the next token from the logits the head just produced, so that only a token id crosses PCIe
// (SURVEY.md 8f-4). Follows the reference's python/sampling.py:10-52 step for step: softmax -> (logit bias) -> temperature 0 =
// argmax -> top-p cutoff -> power by 1/temperature -> renormalise -> inverse-CDF draw, where the draw uses a uniform number `u`
// supplied by the caller exactly as numpy's RandomState.choice uses its one random_sample(): cdf = cumsum(p); cdf /= cdf[-1];
// index = searchsorted(cdf, u, side="right").
//
// One CTA of 1024 threads, thread t owns the PER consecutive vocabulary entries [t*PER, (t+1)*PER) in registers (n_vocab <= 65536).
// The top-p cutoff -- the value of the sorted probabilities at the first index whose running sum exceeds top_p (:42-45) -- is found
// without sorting: it is the largest value v for which sum(p[p >= v]) > top_p, located by bisection on the float bit pattern
// (31 masked block sums over registers).
//
// The batched launch runs one such CTA per row of a [n_rows, n_vocab] logits block (a batch context's head output), each row with
// its own parameters and bias; both kernels call the same sample_row body.
#include "ops.h"
#include "gemv.h"
#include "score_row.cuh"
#include "top_n.cuh"

namespace rwkv {
namespace {

__device__ __forceinline__ double warp_sum_dd(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ double block_sum_dd(double v, double * slots) {      // every thread gets the total
    v = warp_sum_dd(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) slots[threadIdx.x >> 5] = v;
    __syncthreads();
    return warp_sum_dd(slots[threadIdx.x & 31]);
}
__device__ float block_max_f(float v, float * slots) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) slots[threadIdx.x >> 5] = v;
    __syncthreads();
    float r = slots[threadIdx.x & 31];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r = fmaxf(r, __shfl_xor_sync(0xffffffffu, r, o));
    return r;
}

__device__ int block_count(int v, int * slots) {                 // every thread gets the total
    v = __reduce_add_sync(0xffffffffu, v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) slots[threadIdx.x >> 5] = v;
    __syncthreads();
    return __reduce_add_sync(0xffffffffu, slots[threadIdx.x & 31]);
}

// sample_row's filter of the kept set beside top-p: none.
struct NoFilter {
    static constexpr bool active = false;
};

// Keeps token n iff p[n] >= the top_k-th largest probability, counted with multiplicity (top_k = 0: off), and p[n] >= min_p * p_max.
// Both come from the softmax v that also gives the top-p cutoff, so the kept set is the intersection of the three, whatever the order.
struct KeepFilter {
    static constexpr bool active = true;
    uint32_t top_k;
    float min_p;
    // The smallest probability this filter keeps. The top_k-th largest value of v is the largest bit pattern t (non-negative floats
    // order as their bits) with at least top_k entries >= t: a bisection over [0, bits(p_max)] with integer block counts. The pad
    // entries past n_vocab are 0 <= every probability, so they never move it while top_k <= n_vocab. NaN probabilities (a column
    // with a NaN or +inf) compare false everywhere, so whatever comes out keeps them as sample_row without a filter does.
    template <int PER>
    __device__ __forceinline__ float threshold(const float (&v)[PER], float p_max, int V) const {
        __shared__ int islots[SAMPLE_WARPS];
        float kth = 0.f;
        if (top_k > 0 && top_k < (uint32_t) V) {
            uint32_t lo = 0u, hi = __float_as_uint(p_max) + 1u;       // count(>= lo) >= top_k > count(>= hi)
            while (hi - lo > 1u) {
                const uint32_t mid = lo + (hi - lo) / 2u;
                const float t = __uint_as_float(mid);
                int c = 0;
#pragma unroll
                for (int j = 0; j < PER; j++) c += (v[j] >= t) ? 1 : 0;
                if (block_count(c, islots) >= (int) top_k) lo = mid; else hi = mid;
            }
            kth = __uint_as_float(lo);
        }
        return fmaxf(kth, __fmul_rn(min_p, p_max));
    }
};

// The whole draw for one row of logits, shared by the single-row and the batched kernel so that a row of a batch gives the bits of
// a single launch. `p` is that row's view: its logits, parameters, bias, scratch and result words; `filter` narrows the kept set.
template <int PER, class Filter = NoFilter>
__device__ __forceinline__ void sample_row(const SampleParams & p, const Filter filter = Filter{}) {
    __shared__ double dslots[SAMPLE_WARPS];
    __shared__ float fslots[SAMPLE_WARPS];
    __shared__ int first_flagged, last_massive;
    const int tid = threadIdx.x, V = p.n_vocab, base = tid * PER;
    const float * src = p.logits;
    if (p.n_bias > 0) {     // logits + bias through the scratch copy (a dict has no duplicate ids, :30-33; the callers reject them)
        for (int i = tid; i < V; i += SAMPLE_THREADS) p.scratch[i] = p.logits[i];
        __syncthreads();
        for (int i = tid; i < p.n_bias; i += SAMPLE_THREADS) if (p.bias_ids[i] < (uint32_t) V) p.scratch[p.bias_ids[i]] += p.bias_values[i];
        __syncthreads();
        src = p.scratch;
    }
    float v[PER];
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < PER; j++) {
        v[j] = (base + j < V) ? src[base + j] : -INFINITY;
        mx = fmaxf(mx, v[j]);
    }
    mx = block_max_f(mx, fslots);
    if (p.temperature == 0.0f) {    // :39-40 argmax, first index among equals
        int best = V;
#pragma unroll
        for (int j = 0; j < PER; j++) if (base + j < V && v[j] == mx && base + j < best) best = base + j;
        if (tid == 0) first_flagged = V;
        __syncthreads();
        if (best < V) atomicMin(&first_flagged, best);
        __syncthreads();
        if (tid == 0) { *p.token_out = (uint32_t) first_flagged; if (p.prob_out) *p.prob_out = 1.0f; }
        return;
    }
    // softmax (:5-8)
    double s = 0;
#pragma unroll
    for (int j = 0; j < PER; j++) { v[j] = (base + j < V) ? expf(v[j] - mx) : 0.f; s += (double) v[j]; }
    const float total = (float) block_sum_dd(s, dslots);
#pragma unroll
    for (int j = 0; j < PER; j++) v[j] = __fdiv_rn(v[j], total);
    // the filter's threshold, from the same probabilities as the top-p cutoff below (p_max = 1 / total, as for the tempering)
    float keep = 0.f;
    if constexpr (Filter::active) keep = filter.template threshold<PER>(v, __fdiv_rn(1.0f, total), V);
    // top-p (:42-45)
    const float top_p = (p.top_p == 0.0f) ? 1.0f : p.top_p;
    if constexpr (Filter::active) {
        if (!(top_p < 1.0f) && keep > 0.f) {
#pragma unroll
            for (int j = 0; j < PER; j++) if (v[j] < keep) v[j] = 0.f;
        }
    }
    if (top_p < 1.0f) {
        auto mass_at_least = [&](float thr) {
            double m = 0;
#pragma unroll
            for (int j = 0; j < PER; j++) m += (v[j] >= thr) ? (double) v[j] : 0.0;
            return block_sum_dd(m, dslots);
        };
        float cutoff;
        if (!(mass_at_least(0.0f) > (double) top_p)) {
            float m2 = 0.f;
#pragma unroll
            for (int j = 0; j < PER; j++) m2 = fmaxf(m2, v[j]);
            cutoff = block_max_f(m2, fslots);       // np.argmax of an all-False mask is 0: the largest probability
        } else {
            uint32_t lo = 0u, hi = 0x7F800000u;     // f(lo) > top_p >= f(hi)
            while (hi - lo > 1u) {
                const uint32_t mid = lo + (hi - lo) / 2u;
                if (mass_at_least(__uint_as_float(mid)) > (double) top_p) lo = mid; else hi = mid;
            }
            cutoff = __uint_as_float(lo);
        }
        if constexpr (Filter::active) cutoff = fmaxf(cutoff, keep);
#pragma unroll
        for (int j = 0; j < PER; j++) if (v[j] < cutoff) v[j] = 0.f;
    }
    if (p.temperature != 1.0f) {    // :47-48, relative to the largest probability so that no T > 0 underflows every kept token
        // expf(0) = 1 is the largest softmax numerator and top-p always keeps it, so 1 / total is the largest kept probability.
        // The largest tempered mass is then exactly 1, and a kept token is lost only if its share is below 2^-149.
        const float inv_t = 1.0f / p.temperature, p_max = __fdiv_rn(1.0f, total);
#pragma unroll
        for (int j = 0; j < PER; j++) v[j] = (v[j] > 0.f) ? powf(__fdiv_rn(v[j], p_max), inv_t) : 0.f;
    }
    double s2 = 0;
#pragma unroll
    for (int j = 0; j < PER; j++) s2 += (double) v[j];
    const float total2 = (float) block_sum_dd(s2, dslots);
    // :50-52  p / sum(p), then RandomState.choice's inverse CDF in double
    double mine = 0;
#pragma unroll
    for (int j = 0; j < PER; j++) { v[j] = __fdiv_rn(v[j], total2); mine += (double) v[j]; }
    // exclusive prefix of the per-thread masses: warp scan, then a scan of the 32 warp totals
    double incl = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double up = __shfl_up_sync(0xffffffffu, incl, o);
        if ((tid & 31) >= o) incl += up;
    }
    __syncthreads();
    if ((tid & 31) == 31) dslots[tid >> 5] = incl;
    if (tid == 0) { first_flagged = SAMPLE_THREADS; last_massive = -1; }
    __syncthreads();
    double warp_base = 0, grand = 0;
    for (int w = 0; w < SAMPLE_WARPS; w++) { const double t = dslots[w]; if (w < (tid >> 5)) warp_base += t; grand += t; }
    const double before = warp_base + incl - mine;
    // The warp scan, the sum of the warp totals and the owner's element sum round differently, so near u = 1 a thread without mass
    // can see its end above u while the last thread with mass does not: only a thread with mass may own the draw.
    if (mine > 0.0 && (before + mine) / grand > p.u) atomicMin(&first_flagged, tid);
    __syncthreads();
    const int owner = first_flagged;
    if (owner == SAMPLE_THREADS) {      // no end above u (u within rounding of 1): the last token with mass, or V - 1 if none has any
        int last = -1;
        float last_p = 0.f;
#pragma unroll
        for (int j = 0; j < PER; j++) if (v[j] > 0.f) { last = base + j; last_p = v[j]; }
        if (last >= 0) atomicMax(&last_massive, last);
        __syncthreads();
        const int pick = last_massive;
        if (pick < 0 ? tid == 0 : pick == last) {
            *p.token_out = (uint32_t) (pick < 0 ? V - 1 : pick);
            if (p.prob_out) *p.prob_out = last_p;
        }
        return;
    }
    if (tid == owner) {
        double c = before;
        int pick = base;
        float pp = 0.f;
#pragma unroll
        for (int j = 0; j < PER; j++) {
            if (!(v[j] > 0.f)) continue;
            c += (double) v[j];
            pick = base + j; pp = v[j];         // the owner has mass: if its own sum falls short of u, its last token with mass
            if (c / grand > p.u) break;
        }
        *p.token_out = (uint32_t) pick;
        if (p.prob_out) *p.prob_out = pp;
    }
}

template <int PER>
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_kernel(const SampleParams p) {
    pdl_prologue();
    sample_row<PER>(p);
}

// CTA b draws row b: logits + b * n_vocab with rows[b]'s parameters and bias entries [bias_begin, bias_end), scratch slice b.
template <int PER>
__global__ void __launch_bounds__(SAMPLE_THREADS) batch_sample_kernel(const SampleBatchParams bp) {
    pdl_prologue();
    const int b = blockIdx.x;
    const SampleRow r = bp.rows[b];
    const size_t off = (size_t) b * bp.n_vocab;
    SampleParams p;
    p.logits = bp.logits + off; p.n_vocab = bp.n_vocab;
    p.temperature = r.temperature; p.top_p = r.top_p; p.u = r.u;
    p.bias_ids = bp.bias_ids + r.bias_begin; p.bias_values = bp.bias_values + r.bias_begin; p.n_bias = r.bias_end - r.bias_begin;
    p.scratch = bp.scratch ? bp.scratch + off : nullptr; p.token_out = bp.token_out + b; p.prob_out = bp.prob_out ? bp.prob_out + b : nullptr;
    sample_row<PER>(p);
}

// The blocking loop's gate: a row never waits, nothing is published.
struct NoGate {
    __device__ __forceinline__ bool stop_before(int, uint32_t) const { return false; }
    __device__ __forceinline__ void publish(int, uint32_t, uint32_t) const {}
};

__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// The streaming loop's gate over the mapped words of GenStepParams (ops.h).
struct StreamGate {
    uint32_t * tokens, * published;
    const uint32_t * acked;
    uint32_t * timed_out;
    // Thread 0, before row b draws token step (> 0): waits for the host's acknowledgement of token step - 1. True: the host asked
    // the row to stop, or the wait ran out.
    __device__ __forceinline__ bool stop_before(int b, uint32_t step) const {
        const unsigned long long deadline = global_ns() + (unsigned long long) STREAM_TIMEOUT_MS * 1000000ull;
        for (unsigned int ns = 32;; ns = min(2 * ns, 1024u)) {
            uint32_t a;
            asm volatile("ld.acquire.sys.u32 %0, [%1];" : "=r"(a) : "l"(acked + b) : "memory");
            if ((a >> 1) >= step) return a & 1u;
            if (global_ns() > deadline) {
                *(volatile uint32_t *) timed_out = 1;
                return true;
            }
            __nanosleep(ns);
        }
    }
    // Thread 0, after row b drew token step: the token first, then the count that makes it visible to the host.
    __device__ __forceinline__ void publish(int b, uint32_t step, uint32_t tok) const {
        *(volatile uint32_t *) (tokens + (size_t) b * GENERATE_MAX + step) = tok;
        asm volatile("st.release.sys.u32 [%0], %1;" :: "l"(published + b), "r"(step + 1) : "memory");
    }
};

// The unconstrained loop's mask: every token is allowed, no state is kept.
struct NoMask {
    __device__ __forceinline__ bool dead_end(int) const { return false; }
    __device__ __forceinline__ const uint16_t * table_row(int, int) const { return nullptr; }
    __device__ __forceinline__ void advance(int, int, uint32_t) const {}
    __device__ __forceinline__ void report(int) const {}
};

// The constrained loop's mask over the per-row automata of GenStepParams::mask (ops.h); a row with a NULL table is unconstrained.
struct TableMask {
    GenMaskRow * rows;
    uint32_t * states_out;
    // Thread 0, before the row draws: its state allows no token.
    __device__ __forceinline__ bool dead_end(int b) const { const GenMaskRow m = rows[b]; return m.next && !m.live[m.state]; }
    // Every thread: the row's transitions out of its current state, or NULL.
    __device__ __forceinline__ const uint16_t * table_row(int b, int V) const {
        const GenMaskRow m = rows[b];
        return m.next ? m.next + (size_t) m.state * V : nullptr;
    }
    // Thread 0, after the row evaluated tok. A draw never picks a token of zero mass while any token has mass, so only a row whose
    // allowed tokens all have logit -inf or NaN can draw a token its state does not allow; that keeps the state.
    __device__ __forceinline__ void advance(int b, int V, uint32_t tok) const {
        GenMaskRow & m = rows[b];
        if (!m.next) return;
        const uint16_t s = m.next[(size_t) m.state * V + tok];
        if (s != GEN_MASK_DEAD) m.state = s;
    }
    __device__ __forceinline__ void report(int b) const { states_out[b] = rows[b].state; }
};

// The loops without log-probabilities: sample_row gets no prob_out, nothing is recorded.
struct NoLogprobs {
    __device__ __forceinline__ float * prob_slot(size_t) const { return nullptr; }
    __device__ __forceinline__ void record(int, size_t, uint32_t, const float *, int, uint32_t) const {}
};

// The log-probability policy of the logprob kernels (GenLogprobRequest, ops.h). After the draw of token tok from row b's raw logits z:
// warps 0-7 run score_kernel's reduction (score_row.cuh) under named barrier 1 while every warp selects its top_n entries
// (warp_top_keys, top_n.cuh). Warp 0 then merges the 32 sorted lists in shared memory (merge_top_keys), and its lane 0 writes the
// outputs at `at` (and, streaming, the ring record).
template <int PER>
struct Logprobs {
    const GenLogprobRequest * req;
    bool ring;
    __device__ __forceinline__ float * prob_slot(size_t at) const { return req->sample_probs + at; }
    __device__ __forceinline__ void record(int b, size_t at, uint32_t step, const float * z, int V, uint32_t tok) const {
        __shared__ float s_max[LP_SCORE_WARPS];
        __shared__ int s_arg[LP_SCORE_WARPS], s_bad[LP_SCORE_WARPS];
        __shared__ double s_sum[LP_SCORE_WARPS];
        __shared__ unsigned long long s_top[SAMPLE_WARPS][GEN_TOP_MAX];
        const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, top_n = (int) req->top_n;
        float mx = 0.f;
        bool valid = false;
        double log_sum = 0.0;
        if (tid < LP_SCORE_THREADS)
            score_column(tid, z, V, s_max, s_arg, s_bad, s_sum, [] { asm volatile("bar.sync 1, %0;" :: "n"(LP_SCORE_THREADS) : "memory"); },
                         [&](float m, int, bool v, double sum) { mx = m; valid = v; if (v) log_sum = log(sum); });
        warp_top_keys<PER>(z, V, tid, top_n, s_top);
        __syncthreads();
        if (warp != 0) return;
        uint32_t * rec = ring ? req->ring + ((size_t) b * 2 + (step & 1u)) * GEN_LP_RECORD : nullptr;
        merge_top_keys(lane, top_n, s_top, [&](int k, unsigned long long w) {
            if (lane != 0) return;
            const uint32_t id = ~(uint32_t) w;
            const uint32_t out_id = valid ? id : SCORE_NO_TARGET;
            const float out_lp = valid ? score_logprob(z[id], mx, log_sum) : NAN;
            req->top_ids[at * top_n + k] = out_id;
            req->top_logprobs[at * top_n + k] = out_lp;
            if (rec) { ((volatile uint32_t *) rec)[2 + k] = out_id; ((volatile float *) rec)[2 + GEN_TOP_MAX + k] = out_lp; }
        });
        if (lane == 0) {
            const float lp = valid ? score_logprob(z[tok], mx, log_sum) : NAN;
            const float prob = req->sample_probs[at];
            req->logprobs[at] = lp;
            if (rec) { ((volatile float *) rec)[0] = lp; ((volatile float *) rec)[1] = prob; }
        }
    }
};

// The sampled loops' log-probabilities: the Logprobs policy when the call asked for them (req not NULL), nothing otherwise.
template <int PER>
struct RequestedLogprobs {
    const GenLogprobRequest * req;
    bool ring;
    __device__ __forceinline__ float * prob_slot(size_t at) const { return req ? req->sample_probs + at : nullptr; }
    __device__ __forceinline__ void record(int b, size_t at, uint32_t step, const float * z, int V, uint32_t tok) const {
        if (req) Logprobs<PER>{req, ring}.record(b, at, step, z, V, tok);
    }
};

// The loops without a sampler: no user bias, no filter.
struct NoSampler {
    __device__ __forceinline__ void add_bias(int, int, const float *, const uint16_t *, float, float, uint32_t *, float *) const {}
    __device__ __forceinline__ NoFilter filter(int) const { return NoFilter{}; }
};

// The per-row samplers of GenStepParams::samplers (ops.h).
struct RowSampler {
    const GenSamplerRow * rows;
    const GenBiasEntry * bias;
    // Every thread, once row b's penalty / mask list (ids, values, one entry per token) is written: the row's user entries over their
    // ids. A token the state does not allow keeps its -inf; a counted one (count c != 0) gets value - (presence + c * frequency),
    // rounded as the penalty alone is and then once more; any other gets value.
    __device__ __forceinline__ void add_bias(int b, int V, const float * counts, const uint16_t * allowed, float presence, float frequency,
                                             uint32_t * ids, float * values) const {
        const GenSamplerRow r = rows[b];
        for (uint32_t k = r.bias_begin + threadIdx.x; k < r.bias_end; k += SAMPLE_THREADS) {
            const GenBiasEntry e = bias[k];
            if (e.id >= (uint32_t) V || (allowed && allowed[e.id] == GEN_MASK_DEAD)) continue;
            const float c = counts[e.id];
            ids[e.id] = e.id;
            values[e.id] = c != 0.f ? __fsub_rn(e.value, __fadd_rn(presence, __fmul_rn(c, frequency))) : e.value;
        }
        __syncthreads();
    }
    __device__ __forceinline__ KeepFilter filter(int b) const { return KeepFilter{rows[b].top_k, rows[b].min_p}; }
};

// One step of the generation loop for row blockIdx.x (ops.h: GenStepParams), gated by `gate`, its draws restricted by `mask`, every
// draw reported by `lp`, its bias list and kept set extended by `smp`.
template <int PER, class Gate, class Mask, class Lp = NoLogprobs, class Smp = NoSampler>
__device__ __forceinline__ void generate_step(const GenStepParams gp, const Gate gate, const Mask mask, const Lp lp = Lp{}, const Smp smp = Smp{}) {
    __shared__ int draw, park;
    const int b = blockIdx.x, tid = threadIdx.x, V = gp.n_vocab;
    const size_t off = (size_t) b * V;
    GenRow * r = gp.rows + b;
    GenShared * sh = gp.shared;
    if (tid == 0) {
        // a state that allows no token freezes the row exactly as an exhausted budget does
        bool freeze = !r->frozen && (r->step == r->max_tokens || mask.dead_end(b));
        // a stop request (or a wait that ran out) freezes the row exactly as an exhausted budget does
        if (!r->frozen && !freeze && r->step > 0 && gate.stop_before(b, r->step)) freeze = true;
        if (freeze) r->frozen = 1;
        draw = !r->frozen;
        park = freeze;
    }
    __syncthreads();
    uint32_t tok = 0;
    if (draw) {
        const uint32_t step = r->step;
        const float presence = r->presence, frequency = r->frequency, decay = r->decay;
        const uint16_t * allowed = mask.table_row(b, V);
        for (int i = tid; i < V; i += SAMPLE_THREADS) {      // chat_with_bot.py:244-247, as a bias list over every token
            const float c = gp.counts[off + i];
            const bool dead = allowed && allowed[i] == GEN_MASK_DEAD;     // a token the state does not allow: -inf, whatever its count
            gp.bias_ids[off + i] = (c != 0.f || dead) ? (uint32_t) i : (uint32_t) V;
            gp.bias_values[off + i] = dead ? -INFINITY : -__fadd_rn(presence, __fmul_rn(c, frequency));
        }
        __syncthreads();
        smp.add_bias(b, V, gp.counts + off, allowed, presence, frequency, gp.bias_ids + off, gp.bias_values + off);
        SampleParams p;
        p.logits = gp.logits + off; p.n_vocab = V;
        p.temperature = r->temperature; p.top_p = r->top_p; p.u = gp.u[(size_t) b * sh->stride + step];
        p.bias_ids = gp.bias_ids + off; p.bias_values = gp.bias_values + off; p.n_bias = V;
        p.scratch = gp.scratch + off; p.token_out = gp.tokens + (size_t) b * sh->stride + step;
        p.prob_out = lp.prob_slot((size_t) b * sh->stride + step);
        sample_row<PER>(p, smp.filter(b));
        __syncthreads();
        if (tid == 0) {
            tok = *(volatile uint32_t *) p.token_out;
            r->step = step + 1;
            bool stop = false;
            for (uint32_t k = 0; k < sh->n_stop; k++) stop = stop || sh->stop[k] == tok;
            if (stop) { r->frozen = 1; park = 1; }      // reported, not evaluated, not counted (chat_with_bot.py:249-252)
            else {
                if (decay == 1.0f) gp.counts[off + tok] = __fadd_rn(gp.counts[off + tok], sh->weights ? sh->weights[tok] : 1.0f);
                mask.advance(b, V, tok);
            }
        }
        __syncthreads();
        // The decay of an evaluated token: every count becomes c * decay, then the drawn token's own count adds its weight, both in
        // the thread that owns it, so that no barrier orders them. It cannot share the bias loop above: that runs before the draw,
        // and a drawn stop id leaves the counts as they were. The row was read by that loop, so this pass reads it from L2.
        if (decay != 1.0f && !park) {
            const uint32_t t = *(volatile uint32_t *) p.token_out;
            const float w = sh->weights ? sh->weights[t] : 1.0f;
            for (int i = tid; i < V; i += SAMPLE_THREADS) {
                const float c = gp.counts[off + i];
                if (c == 0.f && i != (int) t) continue;         // 0 * decay is 0: most of a row is never written
                const float d = __fmul_rn(c, decay);
                gp.counts[off + i] = i == (int) t ? __fadd_rn(d, w) : d;
            }
        }
        lp.record(b, (size_t) b * sh->stride + step, step, gp.logits + off, V, tok);
    }
    if (park && gp.park)
        for (int i = tid; i < V; i += SAMPLE_THREADS) gp.park[off + i] = gp.logits[off + i];
    if (tid == 0) {
        if (draw) gate.publish(b, r->step - 1, tok);
        const bool active = !r->frozen;
        gp.n_generated[b] = r->step;
        mask.report(b);
        gp.next_tokens[b] = active ? (int) tok : 0;
        if (active) atomicAdd(&sh->active, 1u);
        __threadfence();
        if (atomicAdd(&sh->ticket, 1u) == (uint32_t) gridDim.x - 1) {       // the last CTA of the step
            const uint32_t any = atomicAdd(&sh->active, 0u);
            sh->active = 0; sh->ticket = 0;
            if (any) *gp.passes += 1;
            if (gp.set_handles) {
                cudaGraphSetConditional(gp.run_pass, any ? 1u : 0u);
                cudaGraphSetConditional(gp.keep_going, any ? 1u : 0u);
            }
        }
    }
}

// generate_step's parameters in the kernels with a gate or a mask: a copy with one field stored, which the compiler loads into
// registers at entry. Passed gp itself, as generate_sample_kernel passes it, these kernels would read each field from the parameter
// space where it is used: another schedule, with other register and spill counts than those DESIGN.md 6.4.5 lists. The store keeps
// the compiler from folding the copy back into the parameter.
__device__ __forceinline__ GenStepParams local_copy(const GenStepParams & gp) {
    GenStepParams p = gp;
    p.set_handles = gp.set_handles;
    return p;
}

template <int PER>
__global__ void __launch_bounds__(SAMPLE_THREADS) generate_sample_kernel(const GenStepParams gp) {
    pdl_prologue();
    generate_step<PER>(gp, NoGate{}, NoMask{});
}

// At one CTA per SM ptxas may give every thread 64 registers: with the default bound it holds PER <= 4 to 32, and the gate's wait
// loop then spills more than generate_sample_kernel does. Only a step of more than one row per SM pays for it, with a second wave.
template <int PER>
__global__ void __launch_bounds__(SAMPLE_THREADS, 1) generate_stream_sample_kernel(const GenStepParams gp) {
    pdl_prologue();
    generate_step<PER>(local_copy(gp), StreamGate{gp.stream_tokens, gp.published, gp.acked, gp.timed_out}, NoMask{});
}

// The constrained twins of the two step kernels (rwkv_b200_generate_constrained). Both are bounded at one CTA per SM: with the default
// bound the mask's table read makes PER = 4 spill more than generate_sample_kernel<4>.
template <int PER>
__global__ void __launch_bounds__(SAMPLE_THREADS, 1) generate_constrained_sample_kernel(const GenStepParams gp) {
    pdl_prologue();
    generate_step<PER>(local_copy(gp), NoGate{}, TableMask{gp.mask, gp.states_out});
}

template <int PER>
__global__ void __launch_bounds__(SAMPLE_THREADS, 1) generate_stream_constrained_sample_kernel(const GenStepParams gp) {
    pdl_prologue();
    generate_step<PER>(local_copy(gp), StreamGate{gp.stream_tokens, gp.published, gp.acked, gp.timed_out}, TableMask{gp.mask, gp.states_out});
}

// The constrained steps that also report log-probabilities; a row with a NULL table is unconstrained, so these two serve the logprob
// calls with and without automata.
template <int PER>
__global__ void __launch_bounds__(SAMPLE_THREADS, 1) generate_logprob_sample_kernel(const GenStepParams gp) {
    pdl_prologue();
    generate_step<PER>(local_copy(gp), NoGate{}, TableMask{gp.mask, gp.states_out}, Logprobs<PER>{gp.lp, false});
}

template <int PER>
__global__ void __launch_bounds__(SAMPLE_THREADS, 1) generate_stream_logprob_sample_kernel(const GenStepParams gp) {
    pdl_prologue();
    generate_step<PER>(local_copy(gp), StreamGate{gp.stream_tokens, gp.published, gp.acked, gp.timed_out}, TableMask{gp.mask, gp.states_out},
                       Logprobs<PER>{gp.lp, true});
}

// The constrained steps with a per-row sampler and, when the call's request word is set, log-probabilities; a row with a NULL table
// is unconstrained, so these two serve every sampled call.
template <int PER>
__global__ void __launch_bounds__(SAMPLE_THREADS, 1) generate_sampled_sample_kernel(const GenStepParams gp) {
    pdl_prologue();
    generate_step<PER>(local_copy(gp), NoGate{}, TableMask{gp.mask, gp.states_out}, RequestedLogprobs<PER>{*gp.lp_word, false},
                       RowSampler{gp.samplers, gp.user_bias});
}

template <int PER>
__global__ void __launch_bounds__(SAMPLE_THREADS, 1) generate_stream_sampled_sample_kernel(const GenStepParams gp) {
    pdl_prologue();
    generate_step<PER>(local_copy(gp), StreamGate{gp.stream_tokens, gp.published, gp.acked, gp.timed_out}, TableMask{gp.mask, gp.states_out},
                       RequestedLogprobs<PER>{*gp.lp_word, true}, RowSampler{gp.samplers, gp.user_bias});
}

constexpr int RESTORE_THREADS = 256, RESTORE_BLOCKS_PER_ROW = 64;

__global__ void __launch_bounds__(RESTORE_THREADS) restore_frozen_kernel(const GenRow * rows, const float * src, float * dst, long long seq_stride, size_t n) {
    pdl_prologue();
    const int b = blockIdx.y;
    if (!rows[b].frozen) return;
    const size_t base = (size_t) b * (size_t) seq_stride;
    for (size_t i = (size_t) blockIdx.x * RESTORE_THREADS + threadIdx.x; i < n; i += (size_t) gridDim.x * RESTORE_THREADS) dst[base + i] = src[base + i];
}

using StepKernel = void (*)(const GenStepParams);

// The step kernels of one PER by family and streaming.
template <int PER>
const StepKernel step_kernels[4][2] = {
    {generate_sample_kernel<PER>, generate_stream_sample_kernel<PER>},
    {generate_constrained_sample_kernel<PER>, generate_stream_constrained_sample_kernel<PER>},
    {generate_logprob_sample_kernel<PER>, generate_stream_logprob_sample_kernel<PER>},
    {generate_sampled_sample_kernel<PER>, generate_stream_sampled_sample_kernel<PER>},
};

// The kernel of a step, or NULL when its vocabulary or its rows are out of range.
StepKernel step_kernel(const GenStepParams & p, GenFamily family, bool stream) {
    if (p.n_vocab <= 0 || p.n_vocab > SAMPLE_THREADS * 64 || p.n_rows <= 0 || p.n_rows > SAMPLE_MAX_ROWS) return nullptr;
    return with_sample_per(p.n_vocab, [&](auto per) { return step_kernels<decltype(per)::value>[family][stream]; });
}

}  // namespace

cudaError_t launch_generate_step(const GenStepParams & p, GenFamily family, cudaStream_t s) {
    const StepKernel k = step_kernel(p, family, false);
    if (!k) return cudaErrorInvalidValue;
    return launch_pdl(k, dim3(p.n_rows), dim3(SAMPLE_THREADS), 0, s, p);
}

cudaError_t add_generate_step_node(cudaGraph_t g, const cudaGraphNode_t * deps, size_t n_deps, const GenStepParams & p, GenFamily family, bool stream,
                                   cudaGraphNode_t * node) {
    const StepKernel k = step_kernel(p, family, stream);
    if (!k) return cudaErrorInvalidValue;
    GenStepParams copy = p;
    void * args[] = {&copy};
    cudaKernelNodeParams kp = {};
    kp.func = reinterpret_cast<void *>(k);
    kp.gridDim = dim3(p.n_rows); kp.blockDim = dim3(SAMPLE_THREADS); kp.sharedMemBytes = 0;
    kp.kernelParams = args; kp.extra = nullptr;
    return cudaGraphAddKernelNode(node, g, deps, n_deps, &kp);
}

cudaError_t launch_restore_frozen(const GenRow * rows, int n_rows, const float * src, float * dst, long long seq_stride, size_t state_len, cudaStream_t s) {
    return launch_pdl(restore_frozen_kernel, dim3(RESTORE_BLOCKS_PER_ROW, n_rows), dim3(RESTORE_THREADS), 0, s, rows, src, dst, seq_stride, state_len);
}

cudaError_t launch_sample(const SampleParams & p, cudaStream_t s) {
    if (p.n_vocab <= 0 || p.n_vocab > SAMPLE_THREADS * 64) return cudaErrorInvalidValue;
    return with_sample_per(p.n_vocab, [&](auto per) { return launch_pdl(sample_kernel<decltype(per)::value>, dim3(1), dim3(SAMPLE_THREADS), 0, s, p); });
}

cudaError_t launch_sample_batch(const SampleBatchParams & p, cudaStream_t s) {
    if (p.n_vocab <= 0 || p.n_vocab > SAMPLE_THREADS * 64 || p.n_rows <= 0 || p.n_rows > SAMPLE_MAX_ROWS) return cudaErrorInvalidValue;
    return with_sample_per(p.n_vocab, [&](auto per) {
        return launch_pdl(batch_sample_kernel<decltype(per)::value>, dim3(p.n_rows), dim3(SAMPLE_THREADS), 0, s, p);
    });
}

}  // namespace rwkv
