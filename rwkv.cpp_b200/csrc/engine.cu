// Forward pass over a resident model: the per-architecture launch sequences.
// Math follows rwkv_graph.inc (serial graph :611-720, sequence graph :744-866); every stage below
// names the graph lines it covers. All launches of a pass go to its stream (Pass::stream); nothing here blocks the host
// except the token upload.
#include "engine.h"

#include <algorithm>
#include <cinttypes>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <new>
#include <thread>
#include <vector>

#include "kernels/act_stage.cuh"
#include "kernels/gemv.h"
#include "kernels/ops.h"

namespace rwkv {

namespace {

// rwkv_eval with host state buffers: pipeline the state copies against layer groups? (RWKV_B200_OVERLAP=0/1, rwkv_b200_set_overlap)
constexpr bool OVERLAP_DEFAULT = true;

struct Scratch {      // carve-up of ctx->act.scratch for T tokens
    float * x, * xx, * sx;
    float * mix[6];
    float * r, * k, * v, * g, * w, * a, * vgate, * v_first, * y;
    float * ffn_k, * ffn_r;
    float * lora[4];
};

constexpr int BATCH_TC_MIN = 16;

struct Dims { size_t C, F, R; };

Dims model_dims(const Model & m) {
    Dims d{(size_t) m.n_embed, 0, 0};
    for (int i = m.layer_begin; i < m.layer_end; i++) {
        const Layer & L = m.layers[i];
        if ((size_t) L.ffn_key.M > d.F) d.F = L.ffn_key.M;
        const int ranks[] = {L.att_maa_w1.M, L.att_decay_w1.M, L.att_w1.M, L.att_a1.M, L.att_g1.M, L.att_v1.M};
        for (int r : ranks) if ((size_t) r > d.R) d.R = r;
    }
    if (d.R == 0) d.R = 1;
    return d;
}

// Layers [l0, l1) of segment `seg` (0 = every resident layer).
void segment_range(const Context * ctx, int seg, int & l0, int & l1) {
    const Model & m = *ctx->model;
    l0 = m.layer_begin; l1 = m.layer_end;
    if (seg <= 0) return;
    const int n = m.layer_end - m.layer_begin, G = ctx->n_segments;
    // Graded groups: 1, 2, 3, 5, 10, 6, 3, 2 thirty-seconds of the layers. The upload of the first group's state slice and the download
    // of the last group's are the two copies nothing can overlap, so those groups are small; a group may grow by about the ratio of
    // compute time to copy time per layer (about 1.7 at 7B) over its predecessor without starving the kernels, and shrink the same
    // way towards the end without queueing the downloads; a pipeline model with those two rates puts a 7B token closer to the
    // kernels-alone time than eight even groups do.
    static const int cum32[9] = {0, 1, 3, 6, 11, 21, 27, 30, 32};
    if (G != 8 || n < 16) {
        l0 = m.layer_begin + (int) ((long long) n * (seg - 1) / G);
        l1 = m.layer_begin + (int) ((long long) n * seg / G);
        return;
    }
    auto cut = [&](int s) -> int { return (int) (((long long) cum32[s] * n + 16) / 32); };      // strictly increasing for n >= 16
    l0 = m.layer_begin + cut(seg - 1);
    l1 = m.layer_begin + cut(seg);
}

size_t scratch_floats_for(const Model & m, int T) {
    Dims d = model_dims(m);
    return ((size_t) 19 * d.C + d.F + 4 * d.R) * (size_t) T + 64;
}

Scratch carve(const Model & m, float * base, int T) {
    Dims d = model_dims(m);
    Scratch s;
    float * p = base;
    auto take = [&](size_t n) { float * q = p; p += n * (size_t) T; return q; };
    s.x = take(d.C); s.xx = take(d.C); s.sx = take(d.C);
    for (int i = 0; i < 6; i++) s.mix[i] = take(d.C);
    s.r = take(d.C); s.k = take(d.C); s.v = take(d.C); s.g = take(d.C); s.w = take(d.C); s.a = take(d.C);
    s.vgate = take(d.C); s.v_first = take(d.C); s.y = take(d.C);
    s.ffn_r = take(d.C);
    s.ffn_k = take(d.F);
    for (int i = 0; i < 4; i++) s.lora[i] = take(d.R);
    return s;
}

// Everything one pass reads that is not the context's standing state: make_pass fills in the defaults, an entry point changes what
// its pass needs. Nothing of a pass is left on the context for the next one to find.
struct Pass {
    int T = 0;
    bool want_logits = false;
    int phase = 0;                        // ctx->phase: the pinned token slot, and the graph slot of a single-token pass
    cudaStream_t stream = nullptr;        // ctx->stream, or the stream of a pipeline stage's caller
    float * state_in = nullptr, * state_out = nullptr;   // ctx->state_a -> ctx->state_b
    float * logits = nullptr;             // where the head writes: ctx->logits
    Scratch s{};                          // ctx->act.scratch carved for T tokens
    bool tokens_in_place = false;         // ctx->act.tokens already holds the tokens (the generation loop's step writes them): no upload
    // Pipeline-stage hand-off (SURVEY.md 8e): device pointers of the caller, or NULL.
    // Layout: x f32[C x T], then (v7 only) v_first f32[C x T].
    const float * hidden_in = nullptr;
    float * hidden_out = nullptr;
    // a ragged pass: its device map (Context::ragged_map), and how many sequences advance (the head's columns)
    const int * seq_off = nullptr, * col_seq = nullptr, * head_col = nullptr, * head_seq = nullptr;
    const int * col_seq_host = nullptr;   // ... and the host copy of col_seq (the pinned slot it is uploaded from); NULL: column t is sequence t
    int n_active = 0;
    // a scoring pass: the targets of its columns and where their results go (greedy may be NULL)
    const uint32_t * targets = nullptr;
    float * lp = nullptr;
    uint8_t * greedy = nullptr;
    // a pass with checkpoints inside it (Context::cps): the device map of its columns' slots and of the slots' destinations
    const int * cp_slot = nullptr;
    float * const * cp_dst = nullptr;
};

// The checkpoint map of a launch whose state slice starts at `slice` of the pass's output (kernels/ops.h: CheckpointMap), or none.
CheckpointMap checkpoints_at(const Pass & p, const float * slice) {
    CheckpointMap cp;
    if (p.cp_slot) { cp.slot = p.cp_slot; cp.dst = p.cp_dst; cp.at = slice - p.state_out; }
    return cp;
}

// ---- GEMV batch builder -------------------------------------------------------------------------
struct Batch {
    GemvBatch b;
    const LoraDelta * lora[GEMV_MAX_PROBLEMS] = {};   // the delta of each problem's matrix under the attached adapter, or NULL
    const DevMatrix * mat[GEMV_MAX_PROBLEMS] = {};    // each problem's matrix, in the table the pass reads
    explicit Batch(int T) { memset(&b, 0, sizeof(b)); b.T = T; }
    GemvProblem & add(const DevMatrix & W, const float * x, float * y, int epi = EPI_NONE) {
        lora[b.n] = W.lora;
        mat[b.n] = &W;
        GemvProblem & p = b.p[b.n++];
        p.W = W.data; p.Wt = W.tiled; p.pitch = W.pitch; p.type = W.type; p.K = W.K; p.M = W.M;
        p.x = x; p.ldx = W.K;
        p.y = y; p.ldy = W.M;
        p.epi = epi; p.pro = PRO_NONE;
        return p;
    }
};

// ---- staged activation columns (act_stage.cuh) --------------------------------------------------------------------------------------
// Single-token passes: the kernel that produces a GEMV's input vector (the v6 lerp, a WKV kernel) also writes it in the layout
// the streaming GEMV keeps in shared memory, so the consumer copies ~5 KB instead of quantising 16 KB of fp32 on its critical
// path. One slot per (producer, output); a slot serves every consumer whose weight type multiplies the same staged format.
constexpr int XQ_SLOTS = 6;
enum XqSlot { XQ_LERP = 0 /* .. 4 */, XQ_WKV = 5 };

// The slot to fill for a consumer matrix W of this pass, or NULL when the pass / shape cannot use the hand-off.
unsigned char * xq_slot(const Context * ctx, int T, int slot, const DevMatrix & W) {
    if (T != 1 || ctx->batch_stride || !ctx->xq || !W.data || W.K % 32 != 0 || W.type == DT_F32 || act::stage_class(W.type) == act::SC_NONE) return nullptr;
    if (act::bytes_per_column(W.type, W.K) > ctx->xq_slot_bytes) return nullptr;
    return ctx->xq + (size_t) slot * ctx->xq_slot_bytes;
}
// Point problem p at a staged copy of its input that was written for weight type q_type.
void xq_bind(GemvProblem & p, const unsigned char * q, int q_type) {
    if (q && act::stage_class(p.type) == act::stage_class(q_type)) p.xq = q;
}
#define CUDA_OK(ctx, call)                                                                               \
    do { cudaError_t _e = (call);                                                                        \
         RWKV_CHECK((ctx)->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, _e == cudaSuccess,       \
                    "CUDA error: %s", cudaGetErrorString(_e)); } while (0)

// Passes of >= 32 tokens send every problem the tensor-core kernel can take (any weight type but F32, K % 64 == 0) to
// gemm_tc.cu; the rest (and all shorter passes) use the batch-invariant GEMV, so serial == sequence stays bit-exact
// wherever the reference's tests compare states. Every eligible problem goes, however small: a tensor-core launch has a fixed cost
// of tens of microseconds even for the 160 x 4096 LoRA matrix of a v6 layer, but the multi-column GEMV is worse for such a matrix
// at T = 128 (32 column groups), and a 7B chunk measured slower with a 2^20-weight threshold than with none.
bool launch_batch(Context * ctx, GemvBatch & b, cudaStream_t stream) {
    // tensor cores: chunks of >= 32 tokens; batch contexts (one token of each of B sequences: nothing to stay bit-identical with
    // across pass sizes) from 16 sequences on, where the multi-column SIMT consumer is instruction-bound
    void * ws = ctx->use_tensor_cores ? ctx->act.act16.get() : nullptr;
    CUDA_OK(ctx, gemv_route(b, ctx->model->dev, stream, ws, ctx->act.act16_bytes, ctx->batch_n > 0 ? BATCH_TC_MIN : 32));
    return true;
}

bool run_base(Context * ctx, const Pass & p, Batch & batch) {
    if (!ctx->profiling) return launch_batch(ctx, batch.b, p.stream);
    Context::ProfRecord rec;
    CUDA_OK(ctx, rec.start.create());
    CUDA_OK(ctx, rec.stop.create());
    for (int i = 0; i < batch.b.n; i++)
        rec.bytes += (double) tensor_nbytes(batch.b.p[i].type, (uint64_t) batch.b.p[i].K, (uint64_t) batch.b.p[i].M, 1);
    CUDA_OK(ctx, cudaEventRecord(rec.start, p.stream));
    if (!launch_batch(ctx, batch.b, p.stream)) return false;
    CUDA_OK(ctx, cudaEventRecord(rec.stop, p.stream));
    ctx->prof.push_back(std::move(rec));
    return true;
}

// The delta of matrix W of the model's layer table in adapter a's table (the same slot of a copy of that table), or NULL. Matrices outside
// the layers (the head) take none.
const LoraDelta * delta_in(const Model & m, const Adapter & a, const DevMatrix & W) {
    const uintptr_t base = reinterpret_cast<uintptr_t>(m.layers.data()), w = reinterpret_cast<uintptr_t>(&W);
    if (w < base || w - base >= m.layers.size() * sizeof(Layer)) return nullptr;
    return reinterpret_cast<const DevMatrix *>(reinterpret_cast<const unsigned char *>(a.layers.data()) + (w - base))->lora;
}

// A batch with low-rank deltas (kernels/lora.h): build_lora_batch's shrink of every adapted problem, the batch through its unchanged
// route with the adapted problems of nonlinear epilogue retargeted to EPI_NONE into lora_z, then the expand. Problems without a delta
// stay as they were. The columns of a problem are grouped by delta: all of them under the context's adapter (one slot holding every
// column); under per-sequence adapters (a batch context) a slot per distinct adapter, a column in the slot of its sequence's adapter.
bool run_batch(Context * ctx, const Pass & p, Batch & batch) {
    const int T = batch.b.T, n_ad = (int) ctx->seq_adapters.size(), n_slots = n_ad ? n_ad : 1;
    const LoraDelta * delta[GEMV_MAX_PROBLEMS][LORA_MAX_ADAPTERS];
    bool any = false;
    for (int i = 0; i < batch.b.n; i++)
        for (int k = 0; k < n_slots; k++)
            any = (delta[i][k] = n_ad ? delta_in(*ctx->model, *ctx->seq_adapters[k], *batch.mat[i]) : batch.lora[i]) || any;
    if (!any) return run_base(ctx, p, batch);
    int col_slot[LORA_MAX_T];
    if (n_ad) {
        // only layer matrices carry deltas, and their batches have the pass's columns
        RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, T == p.T, "A batch of %d columns in a pass of %d carries deltas", T, p.T);
        for (int t = 0; t < T; t++) col_slot[t] = ctx->seq_slot[p.col_seq_host ? p.col_seq_host[t] : t];
    } else {
        for (int t = 0; t < T; t++) col_slot[t] = 0;
    }
    LoraBatch lb;
    size_t u_used, z_used;
    if (!build_lora_batch(ctx->sink(), batch.b, n_slots, delta, col_slot, ctx->lora.u, ctx->lora.z, lb, u_used, z_used)) return false;
    if (lb.n) CUDA_OK(ctx, launch_lora_shrink(lb, p.stream));
    if (!run_base(ctx, p, batch)) return false;
    if (lb.n) CUDA_OK(ctx, launch_lora_expand(lb, p.stream));
    return true;
}

// The stages that touch the recurrent state pass seq_stride = batch_stride: in a batch context (one token of each of batch_n
// sequences) their kernels work on sequence t's state for column t; everything else is identical for both kinds of context.
// LayerNorm + token shift + mix in front of a batch of GEMVs is a launch of its own (ln_mix_kernel). Four variations were built,
// measured at 7B Q5_1 and removed:
// (a) fused into the CONSUMING GEMV, every CTA recomputing the LayerNorm in its prologue: a third slower per token;
// (b) as the tail job of the PRODUCING GEMV (att.output / ffn.value), run by the CTA that draws the last ticket: a quarter slower
//     -- every CTA pays a device-wide fence + ticket before it may retire, and the one CTA left behind does
//     the LayerNorm of 4096 channels with 256 threads where this kernel uses 1024 and has its parameter loads in flight before the
//     dependency wait;
// (c) ln_mix_kernel emitting the staged columns of its consumers (act_stage.cuh, as the lerp and WKV kernels do): it adds more to
//     every launch of the single-CTA, latency-bound kernel than it takes out of the consumer: 3 % slower per token;
// (d) for passes of >= 32 tokens, ln_mix_kernel writing the fp16 GEMM operands of its consumers itself, so that two of the six
//     convert_f16 launches of a v6 layer disappear: 1 % per 7B chunk, and the tail of the state went NaN in the shift-state-3e5
//     robustness test of the 64-channel fixture (not understood). 1 % was not worth an unexplained failure.

// LayerNorm + mix parameters of the channel-mixing block (rwkv_ffn_v4_v5 :484-511, rwkv_ffn_v6 :513-531, rwkv_ffn_v7 :533-543).
LnMixParams ffn_ln(const Context * ctx, const Layer & L, const Pass & p, const float * st_in, float * st_out) {
    const Model & m = *ctx->model;
    LnMixParams lp{};
    lp.x = p.s.x; lp.ln_w = L.ln2_w.data; lp.ln_b = L.ln2_b.data;
    lp.state_in = st_in; lp.state_out = st_out; lp.C = m.n_embed; lp.T = p.T; lp.seq_stride = ctx->batch_stride;
    lp.seq_off = p.seq_off; lp.col_seq = p.col_seq;
    if (m.arch_major == 7) {
        lp.formula = 1; lp.n_out = 1; lp.coef[0] = L.ffn_x_k.data; lp.out[0] = p.s.mix[0];
    } else if (m.arch_major == 6) {
        lp.formula = 1; lp.n_out = 2;
        lp.coef[0] = L.ffn_maa_k.data; lp.out[0] = p.s.mix[0];
        lp.coef[1] = L.ffn_maa_r.data; lp.out[1] = p.s.mix[1];
    } else {
        lp.formula = 0; lp.n_out = 2;
        lp.coef[0] = L.ffn_time_mix_k.data; lp.out[0] = p.s.mix[0];
        lp.coef[1] = L.ffn_time_mix_r.data; lp.out[1] = p.s.mix[1];
    }
    return lp;
}

// Channel mixing, all versions.
bool ffn(Context * ctx, const Layer & L, const Pass & p, const LnMixParams & lp) {
    const Model & m = *ctx->model;
    const int C = m.n_embed;
    CUDA_OK(ctx, launch_ln_mix(lp, p.stream, checkpoints_at(p, lp.state_out)));
    {
        Batch b(p.T);
        b.add(L.ffn_key, p.s.mix[0], p.s.ffn_k, EPI_RELU_SQR);
        if (m.arch_major != 7) b.add(L.ffn_receptance, p.s.mix[1], p.s.ffn_r, EPI_SIGMOID);
        if (!run_batch(ctx, p, b)) return false;
    }
    {
        Batch b(p.T);
        GemvProblem & q = b.add(L.ffn_value, p.s.ffn_k, p.s.x, m.arch_major == 7 ? EPI_ADD : EPI_MUL_ADD);
        q.res = p.s.x; q.ldres = C;
        q.gate = p.s.ffn_r; q.ldgate = C;
        if (!run_batch(ctx, p, b)) return false;
    }
    return true;
}

// yq: y as a staged column (written by the WKV kernel) or NULL
bool att_output(Context * ctx, const Layer & L, const Pass & p, const unsigned char * yq) {
    Batch b(p.T);
    GemvProblem & q = b.add(L.att_output, p.s.y, p.s.x, EPI_ADD);   // x + Wo.y  (:182/:291/:384/:481 + residual :667-679)
    q.res = p.s.x; q.ldres = ctx->model->n_embed;
    xq_bind(q, yq, L.att_output.type);
    return run_batch(ctx, p, b);
}

// LayerNorm + mix parameters of the time-mixing block, per architecture (:94-97, :306-311, :400-413).
LnMixParams att_ln(const Context * ctx, const Layer & L, const Pass & p, const float * st_in, float * st_out) {
    const Model & m = *ctx->model;
    const int C = m.n_embed;
    LnMixParams lp{};
    lp.x = p.s.x; lp.ln_w = L.ln1_w.data; lp.ln_b = L.ln1_b.data;
    lp.state_in = st_in + C; lp.state_out = st_out + C; lp.C = C; lp.T = p.T; lp.seq_stride = ctx->batch_stride;
    lp.seq_off = p.seq_off; lp.col_seq = p.col_seq;
    if (m.arch_major == 7) {
        lp.formula = 1; lp.n_out = 6;
        for (int j = 0; j < 6; j++) { lp.coef[j] = L.att_x_rwkvag.data + (size_t) j * C; lp.out[j] = p.s.mix[j]; }   // r w k v a g
    } else if (m.arch_major == 6) {
        lp.formula = 1; lp.n_out = 1; lp.coef[0] = L.att_maa_x.data; lp.out[0] = p.s.mix[0];
        lp.out_xx = p.s.xx; lp.out_sx = p.s.sx;
    } else {
        const bool v52 = m.arch_major == 5 && m.arch_minor >= 2;
        lp.formula = 0; lp.n_out = v52 ? 4 : 3;
        lp.coef[0] = L.att_time_mix_k.data; lp.out[0] = p.s.mix[0];
        lp.coef[1] = L.att_time_mix_v.data; lp.out[1] = p.s.mix[1];
        lp.coef[2] = L.att_time_mix_r.data; lp.out[2] = p.s.mix[2];
        if (v52) { lp.coef[3] = L.att_time_mix_g.data; lp.out[3] = p.s.mix[3]; }
    }
    return lp;
}

bool att_v4(Context * ctx, const Layer & L, const Pass & p, const float * st_in, float * st_out, const LnMixParams & lp) {
    const int C = ctx->model->n_embed;
    CUDA_OK(ctx, launch_ln_mix(lp, p.stream, checkpoints_at(p, lp.state_out)));
    Batch b(p.T);
    b.add(L.att_receptance, p.s.mix[2], p.s.r, EPI_SIGMOID);
    b.add(L.att_key, p.s.mix[0], p.s.k);
    b.add(L.att_value, p.s.mix[1], p.s.v);
    if (!run_batch(ctx, p, b)) return false;
    Wkv4Params wp{};
    wp.k = p.s.k; wp.v = p.s.v; wp.r = p.s.r;
    wp.time_first = L.att_time_first.data; wp.time_decay = L.att_time_decay.data;
    wp.aa_in = st_in + 2 * C; wp.bb_in = st_in + 3 * C; wp.pp_in = st_in + 4 * C;
    wp.aa_out = st_out + 2 * C; wp.bb_out = st_out + 3 * C; wp.pp_out = st_out + 4 * C;
    wp.y = p.s.y; wp.C = C; wp.T = p.T; wp.seq_stride = ctx->batch_stride; wp.seq_off = p.seq_off; wp.n_seq = ctx->batch_n;
    wp.q_out = (C % 32 == 0) ? xq_slot(ctx, p.T, XQ_WKV, L.att_output) : nullptr; wp.q_type = L.att_output.type;
    wp.cp = checkpoints_at(p, wp.aa_out);
    CUDA_OK(ctx, launch_wkv4(wp, p.stream));
    return att_output(ctx, L, p, wp.q_out);
}

bool att_v5(Context * ctx, const Layer & L, const Pass & p, const float * st_in, float * st_out, const LnMixParams & lp) {
    const Model & m = *ctx->model;
    const int C = m.n_embed;
    const bool v52 = m.arch_minor >= 2;
    CUDA_OK(ctx, launch_ln_mix(lp, p.stream, checkpoints_at(p, lp.state_out)));
    Batch b(p.T);
    b.add(L.att_receptance, p.s.mix[2], p.s.r);
    b.add(L.att_key, p.s.mix[0], p.s.k);
    b.add(L.att_value, p.s.mix[1], p.s.v);
    if (v52) b.add(L.att_gate, p.s.mix[3], p.s.g, EPI_SILU);
    if (!run_batch(ctx, p, b)) return false;
    Wkv6Params wp{};
    wp.r = p.s.r; wp.k = p.s.k; wp.v = p.s.v;
    wp.td = L.att_time_decay.data; wp.td_per_token = 0;
    wp.tf = v52 ? L.att_time_faaaa.data : L.att_time_first.data;
    wp.per_head_scalars = v52 ? 0 : 1;
    wp.state_in = st_in + 2 * C; wp.state_out = st_out + 2 * C;
    wp.lnx_w = L.att_ln_x_w.data; wp.lnx_b = L.att_ln_x_b.data;
    wp.g = v52 ? p.s.g : nullptr;
    wp.y = p.s.y; wp.eps = 1e-5f; wp.H = m.head_count; wp.S = m.head_size; wp.T = p.T; wp.seq_stride = ctx->batch_stride; wp.seq_off = p.seq_off; wp.n_seq = ctx->batch_n;
    wp.q_out = (m.head_size % 32 == 0) ? xq_slot(ctx, p.T, XQ_WKV, L.att_output) : nullptr; wp.q_type = L.att_output.type;
    wp.cp = checkpoints_at(p, wp.state_out);
    CUDA_OK(ctx, launch_wkv6(wp, p.stream));
    return att_output(ctx, L, p, wp.q_out);
}

}  // namespace

LoraScratchSize lora_scratch_floats(size_t C, size_t F) {
    const size_t T = MAX_TOKENS_PER_PASS;
    return LoraScratchSize{(size_t) GEMV_MAX_PROBLEMS * LORA_MAX_RANK * T, std::max(4 * C, F + C) * T};
}

bool build_lora_batch(ErrorSink sink, GemvBatch & b, int n_slots, const LoraDelta * const delta[][LORA_MAX_ADAPTERS], const int * col_slot,
                      float * u, float * z, LoraBatch & lb, size_t & u_used, size_t & z_used) {
    const int T = b.T;
    lb.n = 0; lb.T = T; lb.n_groups = 0;
    float * const u0 = u, * const z0 = z;
    int n_col = 0;
    for (int i = 0; i < b.n; i++) {
        GemvProblem & q = b.p[i];
        const bool residual = q.epi == EPI_ADD || q.epi == EPI_MUL_ADD;
        const LoraDelta * d[LORA_MAX_ADAPTERS + 1];     // the delta of each slot; slot n_slots: the columns without one
        int slot_cols[LORA_MAX_ADAPTERS + 1] = {};
        int slot[LORA_MAX_T];
        for (int k = 0; k < n_slots; k++) d[k] = delta[i][k];
        d[n_slots] = nullptr;
        bool adapted = false;
        for (int t = 0; t < T; t++) {
            const int k = col_slot[t];
            slot[t] = k >= 0 && d[k] ? k : n_slots;
            slot_cols[slot[t]]++;
            adapted = adapted || slot[t] < n_slots;
        }
        if (!adapted) continue;
        int ldu = 0, groups = 0;
        for (int k = 0; k <= n_slots; k++)
            if (slot_cols[k] && (d[k] || !residual)) { groups++; if (d[k]) ldu = std::max(ldu, d[k]->rank); }
        RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, lb.n_groups + groups <= LORA_MAX_GROUPS, "Too many delta groups in one launch");
        const int pi = lb.n++;
        LoraProblem & l = lb.p[pi];
        for (int k = 0; k <= n_slots; k++) {
            if (!slot_cols[k] || (!d[k] && residual)) continue;
            LoraGroup & g = lb.g[lb.n_groups++];
            g.d = d[k] ? *d[k] : LoraDelta{};
            g.problem = pi;
            g.col0 = n_col; g.n_cols = 0;
            for (int t = 0; t < T; t++) if (slot[t] == k) lb.col[n_col + g.n_cols++] = (uint8_t) t;
            n_col += g.n_cols;
        }
        l.K = q.K; l.M = q.M;
        l.x = q.x; l.ldx = q.ldx;
        l.u = u; l.ldu = ldu; u += (size_t) ldu * T;
        l.P = q;
        if (residual) {      // residual epilogues: the base writes y, the expand adds to it
            l.z = nullptr; l.ldz = 0;
            l.P.res = q.y; l.P.ldres = q.ldy;
        } else {
            l.z = z; l.ldz = q.M;
            q.y = z; q.ldy = q.M; q.epi = EPI_NONE; q.res = q.gate = q.bias = nullptr;
            z += (size_t) q.M * T;
        }
    }
    u_used = (size_t) (u - u0); z_used = (size_t) (z - z0);
    return true;
}

bool v6_prologue_fits(int C, GemvProblem & w1) {
    if (C < 1 || C > 4096 || w1.K != C || w1.M < 1 || !dtype_supported(w1.type) || w1.K % dtype_block_elems(w1.type)) return false;
    return gemv_tma_plan(w1) && w1.wk == 1 && v6_prologue_smem_bytes(w1, C) <= V6_PROLOGUE_MAX_SMEM;
}

bool wkv6_decay_fits(int C, int S, GemvProblem & dw2) {
    // dw2.K <= 128: lora1 is staged by stage_column, whose F16 / F32 loops give element k to thread k with a stride of 256, run by the
    // 192 threads of the WKV block -- elements 192..255 of a stride would be skipped, so K must stay below 192
    if (S != 64 || C < S || C % S || dw2.M != C || dw2.K < 32 || dw2.K > 128 || !dtype_supported(dw2.type) || dw2.K % dtype_block_elems(dw2.type)) return false;
    return gemv_tma_plan(dw2) && dw2.wk == 1 && wkv6_decay_smem_bytes(dw2) <= WKV6_DECAY_MAX_SMEM;
}

bool v6_lora_fold_shapes(int C, int S, GemvProblem & w1, GemvProblem & dw2) {
    return v6_prologue_fits(C, w1) && wkv6_decay_fits(C, S, dw2);
}

bool v6_lora_fold(const Layer & L, int C, int S, GemvProblem & w1, GemvProblem & dw2) {
    if (!L.att_maa_w1.data || !L.att_decay_w2.data) return false;
    auto problem = [](const DevMatrix & W, int epi) {
        GemvProblem p{};
        p.W = W.data; p.Wt = W.tiled; p.pitch = W.pitch; p.type = W.type; p.K = W.K; p.M = W.M;
        p.ldx = W.K; p.ldy = W.M; p.epi = epi; p.pro = PRO_NONE;
        return p;
    };
    w1 = problem(L.att_maa_w1, EPI_TANH);
    dw2 = problem(L.att_decay_w2, EPI_BIAS_EXPNEGEXP);
    return v6_lora_fold_shapes(C, S, w1, dw2);
}

size_t v6_folded_gemv_bytes(const Model & m) {
    if (m.arch_major != 6) return 0;
    size_t n = 0;
    for (int i = m.layer_begin; i < m.layer_end; i++) {
        const Layer & L = m.layers[i];
        GemvProblem w1, dw2;
        if (v6_lora_fold(L, m.n_embed, m.head_size, w1, dw2))
            n += tensor_nbytes(w1.type, (uint64_t) w1.K, (uint64_t) w1.M, 1) + tensor_nbytes(dw2.type, (uint64_t) dw2.K, (uint64_t) dw2.M, 1);
    }
    return n;
}

namespace {

bool att_v6(Context * ctx, const Layer & L, const Pass & p, const float * st_in, float * st_out, const LnMixParams & lp) {
    const Model & m = *ctx->model;
    const int C = m.n_embed;
    // single-token passes of one sequence: maa_w1 folded into the LayerNorm-mix launch and decay_w2 into the WKV launch
    GemvProblem w1{}, dw2{};
    const bool fold = p.T == 1 && !ctx->batch_stride && v6_lora_fold(L, m.n_embed, m.head_size, w1, dw2);
    if (fold) {
        w1.x = p.s.mix[0]; w1.y = p.s.lora[0];
        dw2.x = p.s.lora[1]; dw2.bias = L.att_time_decay.data;     // dw2's output is the WKV kernel's decay row in shared memory
        CUDA_OK(ctx, launch_v6_prologue(lp, w1, p.stream));
    } else {
        CUDA_OK(ctx, launch_ln_mix(lp, p.stream, checkpoints_at(p, lp.state_out)));
        Batch b(p.T);   // :313-321  tanh(W1 . xxx)
        b.add(L.att_maa_w1, p.s.mix[0], p.s.lora[0], EPI_TANH);
        if (!run_batch(ctx, p, b)) return false;
    }
    V6LerpParams vp{};   // :323-346
    vp.w2 = L.att_maa_w2.data; vp.z = p.s.lora[0]; vp.xx = p.s.xx; vp.sx = p.s.sx;
    vp.maa[0] = L.att_maa_w.data; vp.maa[1] = L.att_maa_k.data; vp.maa[2] = L.att_maa_v.data;
    vp.maa[3] = L.att_maa_r.data; vp.maa[4] = L.att_maa_g.data;
    for (int j = 0; j < 5; j++) vp.out[j] = p.s.mix[1 + j];   // w, k, v, r, g
    vp.C = C; vp.T = p.T; vp.mix = L.maa_mix;
    {   // staged columns for the five consumers (w, k, v, r, g order of the lerp outputs): all or none
        const DevMatrix * cons[5] = {&L.att_decay_w1, &L.att_key, &L.att_value, &L.att_receptance, &L.att_gate};
        bool all = C % 32 == 0;
        for (int j = 0; j < 5; j++) { vp.q_out[j] = xq_slot(ctx, p.T, XQ_LERP + j, *cons[j]); vp.q_type[j] = cons[j]->type; all = all && vp.q_out[j]; }
        if (!all) for (int j = 0; j < 5; j++) vp.q_out[j] = nullptr;
    }
    CUDA_OK(ctx, launch_v6_lerp(vp, p.stream));
    {   // :349-363
        Batch b(p.T);
        xq_bind(b.add(L.att_receptance, p.s.mix[4], p.s.r), vp.q_out[3], vp.q_type[3]);
        xq_bind(b.add(L.att_key, p.s.mix[2], p.s.k), vp.q_out[1], vp.q_type[1]);
        xq_bind(b.add(L.att_value, p.s.mix[3], p.s.v), vp.q_out[2], vp.q_type[2]);
        xq_bind(b.add(L.att_gate, p.s.mix[5], p.s.g, EPI_SILU), vp.q_out[4], vp.q_type[4]);
        xq_bind(b.add(L.att_decay_w1, p.s.mix[1], p.s.lora[1], EPI_TANH), vp.q_out[0], vp.q_type[0]);
        if (!run_batch(ctx, p, b)) return false;
    }
    if (!fold) {   // :357-367  w = exp(-exp(Wd2 . tanh(..) + time_decay))
        Batch b(p.T);
        GemvProblem & q = b.add(L.att_decay_w2, p.s.lora[1], p.s.w, EPI_BIAS_EXPNEGEXP);
        q.bias = L.att_time_decay.data;
        if (!run_batch(ctx, p, b)) return false;
    }
    Wkv6Params wp{};   // :370-382
    wp.r = p.s.r; wp.k = p.s.k; wp.v = p.s.v;
    wp.td = fold ? nullptr : p.s.w; wp.td_per_token = fold ? 0 : 1; wp.tf = L.att_time_faaaa.data; wp.per_head_scalars = 0;
    if (fold) wp.dw2 = dw2;
    wp.state_in = st_in + 2 * C; wp.state_out = st_out + 2 * C;
    wp.lnx_w = L.att_ln_x_w.data; wp.lnx_b = L.att_ln_x_b.data;
    wp.g = p.s.g; wp.y = p.s.y; wp.eps = 64e-5f; wp.H = m.head_count; wp.S = m.head_size; wp.T = p.T; wp.seq_stride = ctx->batch_stride; wp.seq_off = p.seq_off; wp.n_seq = ctx->batch_n;
    wp.q_out = (m.head_size % 32 == 0) ? xq_slot(ctx, p.T, XQ_WKV, L.att_output) : nullptr; wp.q_type = L.att_output.type;
    wp.cp = checkpoints_at(p, wp.state_out);
    CUDA_OK(ctx, launch_wkv6(wp, p.stream));
    return att_output(ctx, L, p, wp.q_out);
}

bool att_v7(Context * ctx, const Layer & L, int layer, const Pass & p, const float * st_in, float * st_out, const LnMixParams & lp) {
    const Model & m = *ctx->model;
    const int C = m.n_embed;
    const bool first = layer == 0;
    float * v_dst = first ? p.s.v_first : p.s.v;
    CUDA_OK(ctx, launch_ln_mix(lp, p.stream, checkpoints_at(p, lp.state_out)));
    {   // :415-432, 439, 447 -- first halves of the LoRA pairs
        Batch b(p.T);
        b.add(L.att_receptance, p.s.mix[0], p.s.r);
        b.add(L.att_key, p.s.mix[2], p.s.k);
        b.add(L.att_value, p.s.mix[3], v_dst);
        b.add(L.att_w1, p.s.mix[1], p.s.lora[0], EPI_TANH);
        b.add(L.att_a1, p.s.mix[4], p.s.lora[1]);
        b.add(L.att_g1, p.s.mix[5], p.s.lora[2], EPI_SIGMOID);
        if (!first) b.add(L.att_v1, p.s.mix[3], p.s.lora[3]);
        if (!run_batch(ctx, p, b)) return false;
    }
    {   // second halves
        Batch b(p.T);
        GemvProblem & pw = b.add(L.att_w2, p.s.lora[0], p.s.w, EPI_BIAS_W7);      pw.bias = L.att_w0.data;
        GemvProblem & pa = b.add(L.att_a2, p.s.lora[1], p.s.a, EPI_BIAS_SIGMOID); pa.bias = L.att_a0.data;
        b.add(L.att_g2, p.s.lora[2], p.s.g);
        if (!first) { GemvProblem & pv = b.add(L.att_v2, p.s.lora[3], p.s.vgate, EPI_BIAS_SIGMOID); pv.bias = L.att_v0.data; }
        if (!run_batch(ctx, p, b)) return false;
    }
    Wkv7Params wp{};   // :433-479
    wp.r = p.s.r; wp.w = p.s.w; wp.k = p.s.k; wp.v = v_dst; wp.a = p.s.a; wp.g = p.s.g;
    wp.vgate = first ? nullptr : p.s.vgate; wp.v_first = p.s.v_first; wp.v_out = nullptr;
    wp.k_k = L.att_k_k.data; wp.k_a = L.att_k_a.data; wp.r_k = L.att_r_k.data;
    wp.lnx_w = L.att_ln_x_w.data; wp.lnx_b = L.att_ln_x_b.data;
    wp.state_in = st_in + 2 * C; wp.state_out = st_out + 2 * C;
    wp.y = p.s.y; wp.H = m.head_count; wp.S = m.head_size; wp.T = p.T; wp.seq_stride = ctx->batch_stride; wp.seq_off = p.seq_off; wp.n_seq = ctx->batch_n;
    wp.q_out = (m.head_size % 32 == 0) ? xq_slot(ctx, p.T, XQ_WKV, L.att_output) : nullptr; wp.q_type = L.att_output.type;
    wp.cp = checkpoints_at(p, wp.state_out);
    CUDA_OK(ctx, launch_wkv7(wp, p.stream));
    return att_output(ctx, L, p, wp.q_out);
}

bool ensure_capacity(Context * ctx, int T, cudaStream_t stream) {
    if (T <= ctx->act.capacity_T) return true;
    const Model & m = *ctx->model;
    int cap = ctx->act.capacity_T ? ctx->act.capacity_T : 1;
    while (cap < T) cap *= 2;
    if (cap > MAX_TOKENS_PER_PASS) cap = MAX_TOKENS_PER_PASS;
    CUDA_OK(ctx, cudaStreamSynchronize(stream));
    ctx->act = {};
    drop_all_graphs(ctx);
    Context::Activations a;
    const size_t n = scratch_floats_for(m, cap);
    cudaError_t e = a.scratch.alloc(n * sizeof(float));
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, false, e == cudaSuccess, "Failed to allocate %zu bytes of activation memory: %s", n * sizeof(float), cudaGetErrorString(e));
    e = a.tokens.alloc((size_t) cap * sizeof(int));
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, false, e == cudaSuccess, "Failed to allocate the token buffer: %s", cudaGetErrorString(e));
    for (int i = 0; i < 2; i++) {
        e = a.tokens_host[i].alloc((size_t) cap * sizeof(int));
        RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, false, e == cudaSuccess, "Failed to allocate pinned token staging: %s", cudaGetErrorString(e));
    }
    if (cap >= BATCH_TC_MIN) {   // fp16 staging for the tensor-core path: up to 8 distinct inputs of max(C, F) x round16(cap)
        Dims d = model_dims(m);
        const size_t kmax = d.F > d.C ? d.F : d.C;
        a.act16_bytes = gemm_tc_batch_workspace_bytes(cap, kmax);
        e = a.act16.alloc(a.act16_bytes);
        RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, false, e == cudaSuccess, "Failed to allocate fp16 staging: %s", cudaGetErrorString(e));
    }
    a.capacity_T = cap;
    ctx->act = std::move(a);
    return true;
}

// A pass of T tokens with the defaults of Pass on `stream` (NULL: the context's), once the context has room for T tokens.
bool make_pass(Context * ctx, int T, bool want_logits, cudaStream_t stream, Pass & p) {
    p = Pass{};
    p.stream = stream ? stream : ctx->stream;
    if (!ensure_capacity(ctx, T, p.stream)) return false;
    p.T = T; p.want_logits = want_logits; p.phase = ctx->phase;
    p.state_in = ctx->state_a; p.state_out = ctx->state_b; p.logits = ctx->logits;
    p.s = carve(*ctx->model, ctx->act.scratch, T);
    return true;
}

// The head's LayerNorm parameters: the attached adapter's replacements, or the model's.
const float * ln_out_w(const Context * ctx) { return (ctx->adapter ? ctx->adapter->ln_out_w : ctx->model->ln_out_w).data; }
const float * ln_out_b(const Context * ctx) { return (ctx->adapter ? ctx->adapter->ln_out_b : ctx->model->ln_out_b).data; }

// The head of a scoring pass of T columns runs on the tensor cores when the layers of such a pass would (T >= 32 in a single-sequence
// context, >= BATCH_TC_MIN in a batch context, tensor cores on) and the head's type and width have a tile-major form.
bool score_on_tensor_cores(const Context * ctx, int T) {
    const Model & m = *ctx->model;
    return T >= (ctx->batch_n > 0 ? BATCH_TC_MIN : 32) && ctx->use_tensor_cores && getenv("RWKV_B200_NO_TC") == nullptr &&
           gemm_tc_eligible(m.head.type, m.head.K);
}

// Head of a scoring pass: logits of every column into score_logits [T, n_vocab], the scoring kernel over them, and the last column of
// every advancing sequence (of the pass, for a single sequence) into its logits column.
bool score_head(Context * ctx, const Pass & p) {
    const Model & m = *ctx->model;
    const int C = m.n_embed, V = m.n_vocab, T = p.T;
    Batch b(T);
    if (score_on_tensor_cores(ctx, T)) {
        RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, m.head_tiled && ctx->act.act16, "The head has no tile-major copy");
        // the columns' LayerNorm goes to mix[0], which the layers no longer need
        CUDA_OK(ctx, launch_layer_norm_columns(p.s.x, ln_out_w(ctx), ln_out_b(ctx), C, T, p.s.mix[0], p.stream));
        GemvProblem & q = b.add(m.head, p.s.mix[0], ctx->score_logits);
        q.Wt = m.head_tiled;
        CUDA_OK(ctx, gemm_tc_launch(b.b, m.dev, p.stream, ctx->act.act16, ctx->act.act16_bytes));
    } else {
        GemvProblem & q = b.add(m.head, p.s.x, ctx->score_logits);
        q.pro = PRO_LAYERNORM; q.ln_w = ln_out_w(ctx); q.ln_b = ln_out_b(ctx);
        if (!run_batch(ctx, p, b)) return false;
    }
    ScoreParams sp{};
    sp.logits = ctx->score_logits; sp.n_vocab = V; sp.T = T;
    sp.targets = p.targets; sp.logprobs = p.lp; sp.greedy = p.greedy;
    CUDA_OK(ctx, launch_score(sp, p.stream));
    if (p.seq_off) CUDA_OK(ctx, launch_copy_columns(ctx->score_logits, p.head_col, p.logits, p.head_seq, V, p.n_active, p.stream));
    else CUDA_OK(ctx, launch_copy_columns(ctx->score_logits + (size_t) (T - 1) * V, nullptr, p.logits, nullptr, V, 1, p.stream));
    return true;
}

// Enqueues segment `seg` of pass p (token upload + every kernel) on its stream; pure stream work, so it can be captured.
bool enqueue_pass(Context * ctx, const Pass & p, int seg) {
    const Model & m = *ctx->model;
    int l0, l1;
    segment_range(ctx, seg, l0, l1);
    g_trace_base = ctx->trace_buf;
    g_trace_next = 0;
    const int C = m.n_embed, T = p.T;
    if (l0 == 0) {
        if (!p.tokens_in_place) CUDA_OK(ctx, cudaMemcpyAsync(ctx->act.tokens, ctx->act.tokens_host[p.phase], (size_t) T * sizeof(int), cudaMemcpyHostToDevice, p.stream));
        const DevVec & ln0_w = ctx->adapter ? ctx->adapter->ln0_w : m.ln0_w, & ln0_b = ctx->adapter ? ctx->adapter->ln0_b : m.ln0_b;
        CUDA_OK(ctx, launch_embed_ln0(m.emb.data, m.emb.type, m.emb.pitch, ctx->act.tokens, T, C, ln0_w.data, ln0_b.data, p.s.x, p.stream));
    }   // a later pipeline stage / layer group finds x (and v_first) already in place
    const size_t per_layer = m.state_floats_per_layer();
    for (int i = l0; i < l1; i++) {
        const Layer & L = ctx->adapter ? ctx->adapter->layers[i] : m.layers[i];
        const float * st_in = p.state_in + (size_t) i * per_layer;
        float * st_out = p.state_out + (size_t) i * per_layer;
        const LnMixParams alp = att_ln(ctx, L, p, st_in, st_out), flp = ffn_ln(ctx, L, p, st_in, st_out);
        bool ok;
        switch (m.arch_major) {
            case 7: ok = att_v7(ctx, L, i, p, st_in, st_out, alp); break;
            case 6: ok = att_v6(ctx, L, p, st_in, st_out, alp); break;
            case 5: ok = att_v5(ctx, L, p, st_in, st_out, alp); break;
            default: ok = att_v4(ctx, L, p, st_in, st_out, alp); break;
        }
        if (!ok || !ffn(ctx, L, p, flp)) return false;
    }
    if (p.targets && l1 == m.n_layer) {
        if (!score_head(ctx, p)) return false;
    } else if (p.want_logits && l1 == m.n_layer && p.seq_off) {
        // ragged: the head on the last column of every advancing sequence, gathered; its columns go to those sequences' logits
        const int n = p.n_active;
        CUDA_OK(ctx, launch_copy_columns(p.s.x, p.head_col, ctx->ragged.head_x, nullptr, C, n, p.stream));
        Batch b(n);
        GemvProblem & q = b.add(m.head, ctx->ragged.head_x, ctx->ragged.head_y);
        q.pro = PRO_LAYERNORM; q.ln_w = ln_out_w(ctx); q.ln_b = ln_out_b(ctx);
        if (!run_batch(ctx, p, b)) return false;
        CUDA_OK(ctx, launch_copy_columns(ctx->ragged.head_y, nullptr, p.logits, p.head_seq, m.n_vocab, n, p.stream));
    } else if (p.want_logits && l1 == m.n_layer) {   // :705-708 / :851-854  head . LN(x_last; ln_out); a batch context wants every column
        Batch b(ctx->batch_n ? T : 1);
        GemvProblem & q = b.add(m.head, ctx->batch_n ? p.s.x : p.s.x + (size_t) (T - 1) * C, p.logits);
        q.pro = PRO_LAYERNORM; q.ln_w = ln_out_w(ctx); q.ln_b = ln_out_b(ctx);
        if (!run_batch(ctx, p, b)) return false;
    }
    if (ctx->trace_buf) {
        ctx->trace_count = g_trace_next;
        for (int i = 0; i < g_trace_next; i++) ctx->trace_names[i] = g_trace_names[i];
    }
    g_trace_base = nullptr;
    return true;
}

// One pass of at most MAX_TOKENS_PER_PASS tokens (state_a -> state_b, then swap) in three steps, so that the overlapped path can
// put copies between the layer groups: begin_pass (token staging, hand-off in), run_layers per segment, end_pass.
bool begin_pass(Context * ctx, const uint32_t * tokens, const Pass & p) {
    const int phase = p.phase, T = p.T;
    if (ctx->act.slot_used[phase]) CUDA_OK(ctx, cudaEventSynchronize(ctx->slot_free[phase]));   // pass n-2 has consumed this slot
    const Model & m = *ctx->model;
    if (m.layer_begin == 0) for (int t = 0; t < T; t++) ctx->act.tokens_host[phase][t] = (int) tokens[t];
    const size_t ct = (size_t) m.n_embed * (size_t) T * sizeof(float);
    CUDA_OK(ctx, cudaEventRecord(ctx->ev_start, p.stream));
    if (p.hidden_in) {    // outside the captured graph: the caller's pointers may change from call to call
        CUDA_OK(ctx, cudaMemcpyAsync(p.s.x, p.hidden_in, ct, cudaMemcpyDeviceToDevice, p.stream));
        if (m.arch_major == 7) CUDA_OK(ctx, cudaMemcpyAsync(p.s.v_first, p.hidden_in + (size_t) m.n_embed * T, ct, cudaMemcpyDeviceToDevice, p.stream));
    }
    return true;
}

// The kernels of segment `seg` (0 = all resident layers) for the pass begun by begin_pass.
bool run_layers(Context * ctx, const Pass & p, int seg) {
    const Model & m = *ctx->model;
    int l0, l1;
    segment_range(ctx, seg, l0, l1);
    // only the group that ends the model can run the head
    const int slot = Context::slot_index(p.want_logits && l1 == m.n_layer, p.phase, seg);
    Context::GraphSlot * g = (p.T == 1 && ctx->use_graphs && !ctx->profiling) ? &ctx->graphs[slot] : nullptr;
    if (g && g->exec) {
        CUDA_OK(ctx, cudaGraphLaunch(g->exec, p.stream));
        g_kernel_launches += g->launches;
        g_graph_launches++;
    } else if (g && g->uses >= 1) {
        // second use of this slot: capture the launch sequence once, replay from now on
        const unsigned long long before = g_kernel_launches;
        CUDA_OK(ctx, cudaStreamBeginCapture(p.stream, cudaStreamCaptureModeThreadLocal));
        const bool ok = enqueue_pass(ctx, p, seg);
        Graph graph;
        cudaError_t e = graph.end_capture(p.stream);
        RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, ok && e == cudaSuccess && graph, "CUDA graph capture failed: %s", cudaGetErrorString(e));
        g->launches = g_kernel_launches - before;
        e = g->exec.instantiate(graph);
        RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, e == cudaSuccess, "cudaGraphInstantiate failed: %s", cudaGetErrorString(e));
        CUDA_OK(ctx, cudaGraphLaunch(g->exec, p.stream));
        g_graph_launches++;
    } else {
        if (g) g->uses++;
        if (!enqueue_pass(ctx, p, seg)) return false;
    }
    return true;
}

bool end_pass(Context * ctx, const Pass & p) {
    const Model & m = *ctx->model;
    if (p.hidden_out) {
        const size_t ct = (size_t) m.n_embed * (size_t) p.T * sizeof(float);
        CUDA_OK(ctx, cudaMemcpyAsync(p.hidden_out, p.s.x, ct, cudaMemcpyDeviceToDevice, p.stream));
        if (m.arch_major == 7) CUDA_OK(ctx, cudaMemcpyAsync(p.hidden_out + (size_t) m.n_embed * p.T, p.s.v_first, ct, cudaMemcpyDeviceToDevice, p.stream));
    }
    CUDA_OK(ctx, cudaEventRecord(ctx->ev_stop, p.stream));
    CUDA_OK(ctx, cudaEventRecord(ctx->slot_free[p.phase], p.stream));
    ctx->act.slot_used[p.phase] = true;
    std::swap(ctx->state_a, ctx->state_b);
    ctx->phase ^= 1;
    ctx->logits_valid = p.want_logits && m.layer_end == m.n_layer;
    return true;
}

bool forward_pass(Context * ctx, const uint32_t * tokens, const Pass & p) {
    return begin_pass(ctx, tokens, p) && run_layers(ctx, p, 0) && end_pass(ctx, p);
}

bool ensure_copy_streams(Context * ctx) {
    if (ctx->copies.in) return true;
    Context::CopyStreams c;
    CUDA_OK(ctx, c.in.create());
    CUDA_OK(ctx, c.out.create());
    CUDA_OK(ctx, c.pass_begin.create(cudaEventDisableTiming));
    for (int i = 0; i < Context::MAX_SEGMENTS; i++) {
        CUDA_OK(ctx, c.seg_in[i].create(cudaEventDisableTiming));
        CUDA_OK(ctx, c.seg_out[i].create(cudaEventDisableTiming));
    }
    ctx->copies = std::move(c);
    return true;
}

}  // namespace

void fill_init_state(const Model & m, float * state) {
    const size_t n = m.state_len();
    memset(state, 0, n * sizeof(float));
    if (m.arch_major >= 5) return;
    const size_t C = m.n_embed;
    for (int l = 0; l < m.n_layer; l++)
        for (size_t c = 0; c < C; c++) state[(size_t) l * 5 * C + 4 * C + c] = -1e30f;
}

Context * create_context(Model * model, ErrorSink sink, int batch_n) {
    Context * ctx = new (std::nothrow) Context();
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, nullptr, ctx, "Failed to allocate rwkv_context");
    ctx->model = model;
    model->refcount.fetch_add(1);
    ctx->print_errors = *sink.print;
    { const char * e = getenv("RWKV_B200_OVERLAP"); ctx->overlap_copies = e ? atoi(e) != 0 : OVERLAP_DEFAULT; }
    {   // layer groups of the overlapped host-state path: at least 4 layers each, at most MAX_SEGMENTS groups
        const int n = model->layer_end - model->layer_begin;
        ctx->n_segments = std::clamp(n / 4, 1, Context::MAX_SEGMENTS);
    }
    const size_t n = model->state_len();
    const size_t seqs = batch_n > 0 ? (size_t) batch_n : 1;
    if (batch_n > 0) { ctx->batch_n = batch_n; ctx->batch_stride = (long long) n; ctx->overlap_copies = false; }
    ctx->penalty_decay.assign(seqs, 1.0f);
    bool ok = cudaSetDevice(model->dev.device) == cudaSuccess
        && ctx->stream.create() == cudaSuccess
        && ctx->ev_start.create() == cudaSuccess && ctx->ev_stop.create() == cudaSuccess
        && ctx->slot_free[0].create(cudaEventDisableTiming) == cudaSuccess
        && ctx->slot_free[1].create(cudaEventDisableTiming) == cudaSuccess
        && ctx->state_a.alloc(seqs * n * sizeof(float)) == cudaSuccess
        && ctx->state_b.alloc(seqs * n * sizeof(float)) == cudaSuccess
        && ctx->state_init.alloc(n * sizeof(float)) == cudaSuccess
        && ctx->logits.alloc(seqs * (size_t) model->n_vocab * sizeof(float)) == cudaSuccess;
    if (ok && batch_n == 0) {      // staged-column hand-off slots (every handed-off vector has n_embed elements, at most 2 bytes each) 
        ctx->xq_slot_bytes = ((size_t) 2 * model->n_embed + 64 + 255) / 256 * 256;
        ok = ctx->xq.alloc((size_t) XQ_SLOTS * ctx->xq_slot_bytes) == cudaSuccess;
    }
    // a batch context's logits start as zeros: after ragged passes a column that was never computed is a uniform draw, not garbage
    if (ok && batch_n > 0) ok = cudaMemset(ctx->logits, 0, seqs * (size_t) model->n_vocab * sizeof(float)) == cudaSuccess;
    if (ok) {
        std::vector<float> init(n);
        fill_init_state(*model, init.data());
        ok = cudaMemcpy(ctx->state_init, init.data(), n * sizeof(float), cudaMemcpyHostToDevice) == cudaSuccess;
        for (size_t q = 0; ok && batch_n > 0 && q < seqs; q++)
            ok = cudaMemcpy(ctx->state_a + q * n, ctx->state_init, n * sizeof(float), cudaMemcpyDeviceToDevice) == cudaSuccess;
    }
    if (!ok) {
        cudaError_t e = cudaGetLastError();
        destroy_context(ctx);
        RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, nullptr, false, "Failed to set up the context on the device: %s", cudaGetErrorString(e));
    }
    return ctx;
}

void destroy_context(Context * ctx) {
    if (!ctx) return;
    for (Context * s : ctx->stages) destroy_context(s);
    ctx->stages.clear();
    if (PipeGroup * g = ctx->group) {
        ctx->group = nullptr;
        if (g->refs.fetch_sub(1) == 1) {
            for (size_t r = 0; r < g->streams.size(); r++) { cudaSetDevice(g->devices[r]); cudaStreamSynchronize(g->streams[r]); cudaStreamDestroy(g->streams[r]); }
            delete g;
        }
    }
    Model * model = ctx->model;
    if (model) cudaSetDevice(model->dev.device);
    for (cudaStream_t s : {ctx->stream.get(), ctx->copies.in.get(), ctx->copies.out.get()}) if (s) cudaStreamSynchronize(s);
    if (ctx->adapter) ctx->adapter->attached.fetch_sub(1);
    for (const Adapter * a : ctx->seq_adapter) if (a) a->attached.fetch_sub(1);
    delete ctx;      // the members' owners release every buffer, event, stream and graph, on the model's device
    if (model && model->refcount.fetch_sub(1) == 1) delete model;
}

bool upload_state(Context * ctx, const float * state_in) {
    const size_t bytes = ctx->model->state_len() * sizeof(float);
    // cudaMemcpyDefault: state_in / state_out / logits_out may be host memory (the rwkv.h contract) or device memory of this process
    // (a CUDA tensor handed over by the Python wrapper): unified addressing tells them apart
    if (state_in) CUDA_OK(ctx, cudaMemcpyAsync(ctx->state_a, state_in, bytes, cudaMemcpyDefault, ctx->stream));
    else CUDA_OK(ctx, cudaMemcpyAsync(ctx->state_a, ctx->state_init, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
    return true;
}

bool download_outputs(Context * ctx, float * state_out, float * logits_out) {
    if (state_out) CUDA_OK(ctx, cudaMemcpyAsync(state_out, ctx->state_a, ctx->model->state_len() * sizeof(float), cudaMemcpyDefault, ctx->stream));
    if (logits_out) CUDA_OK(ctx, cudaMemcpyAsync(logits_out, ctx->logits, (size_t) ctx->model->n_vocab * sizeof(float), cudaMemcpyDefault, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return true;
}

// ---- pageable caller buffers ----------------------------------------------------------------------------------------------------
// The reference's bindings hand over ordinary (pageable) memory (python/rwkv_cpp/rwkv_cpp_model.py:330-351: fresh torch / numpy buffers per
// call). A cudaMemcpyAsync from pageable memory is staged by the driver on the calling thread, synchronously and at a few GB/s: the
// eight slice copies of a 7B state took milliseconds before the first kernel was even enqueued. Registering the caller's pages (cudaHostRegister) would be as fast as pinned memory, but a registration
// outlives a free(): the next buffer malloc() places at the same address would be DMA'd from the OLD pages. So the state travels
// through pinned bounce buffers owned by the context, copied by two helper threads (one per direction) slice by slice, in step with
// the layer groups: memcpy of slice g+1 || H2D of slice g || kernels of group g-1 ... and the mirror image on the way out.
static bool is_pageable_host(const void * p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}
static bool bounce_enabled() {
    static const bool on = getenv("RWKV_B200_NO_BOUNCE") == nullptr;
    return on;
}
// states below this size go the plain way (two helper threads cost ~0.1 ms); rwkv_b200_set_bounce_min_bytes moves the bar (tests)
std::atomic<size_t> g_bounce_min_bytes{(size_t) 4 << 20};
std::atomic<unsigned long long> g_graph_launches{0};

// The helper threads of the bounce path: COPY_LANES per direction, created with the bounce buffers and parked on a condition variable
// between passes (spawning eight threads per token would cost more than the copies). One job = one pass: lane k of a direction copies
// the k-th part of every slice, so slices complete in order at the combined memcpy rate of the lanes (one thread alone needs
// milliseconds for the 34.6 MB state of a 7B model).
struct CopyPool {
    static constexpr int LANES = 4, N = 2 * LANES;
    std::thread th[N];
    std::mutex m;
    std::condition_variable cv;
    unsigned long long generation = 0;
    bool quit = false;
    std::function<void(int)> job;
    std::atomic<int> running{0};
    CopyPool() {
        for (int k = 0; k < N; k++) th[k] = std::thread([this, k] {
            unsigned long long seen = 0;
            for (;;) {
                std::function<void(int)> f;
                {
                    std::unique_lock<std::mutex> lk(m);
                    cv.wait(lk, [&] { return quit || generation != seen; });
                    if (quit) return;
                    seen = generation;
                    f = job;
                }
                f(k);
                running.fetch_sub(1, std::memory_order_release);
            }
        });
    }
    void start(std::function<void(int)> f) {
        { std::lock_guard<std::mutex> lk(m); job = std::move(f); running.store(N); generation++; }
        cv.notify_all();
    }
    void wait() { while (running.load(std::memory_order_acquire) > 0) std::this_thread::yield(); }
    ~CopyPool() {
        wait();
        { std::lock_guard<std::mutex> lk(m); quit = true; }
        cv.notify_all();
        for (auto & t : th) if (t.joinable()) t.join();
    }
};
void CopyPoolDelete::operator()(CopyPool * p) const { delete p; }

static bool ensure_bounce(Context * ctx) {
    if (ctx->bounce.in) return true;
    const size_t bytes = ctx->model->state_len() * sizeof(float);
    Context::Bounce b;
    bool ok = b.in.alloc(bytes) == cudaSuccess && b.out.alloc(bytes) == cudaSuccess &&
              b.logits.alloc((size_t) ctx->model->n_vocab * sizeof(float)) == cudaSuccess;
    for (int i = 0; ok && i < Context::MAX_SEGMENTS; i++) ok = b.seg_d2h[i].create(cudaEventDisableTiming) == cudaSuccess;
    if (ok) b.pool.reset(new (std::nothrow) CopyPool());
    if (!ok || !b.pool) {
        cudaGetLastError();
        return false;                      // not an error: the caller falls back to plain copies
    }
    ctx->bounce = std::move(b);
    return true;
}

namespace {
// Progress of one pass's copies; waits for the lanes whatever way the pass ends.
struct BouncePass {
    CopyPool * pool = nullptr;
    std::atomic<int> in_parts[Context::MAX_SEGMENTS];     // lanes that have copied their part of slice g into bounce_in
    std::atomic<int> out_posted{0};                        // slices whose D2H copy + event have been enqueued
    std::atomic<int> out_arrived{0};                       // slices that have landed in bounce_out
    std::atomic<bool> abort{false};
    BouncePass() { for (auto & a : in_parts) a.store(0); }
    ~BouncePass() { if (pool) { abort.store(true); pool->wait(); } }
};
}  // namespace

// One pass with the caller's host state pipelined against the layer groups: H2D of group g+1 and D2H of group g-1 run on their
// own streams while group g computes (the state layout is layer-major, rwkv_graph.inc:545-606, so a group is one contiguous
// slice). state_in == NULL starts from the init image (a device copy); state_out / logits_out may be NULL.
static bool eval_host_overlapped(Context * ctx, const uint32_t * tokens, int T, const float * state_in, bool resident_in, float * state_out, float * logits_out) {
    const Model & m = *ctx->model;
    const int G = ctx->n_segments;
    if (!ensure_copy_streams(ctx)) return false;
    const size_t per_layer = m.state_floats_per_layer();
    const size_t state_bytes = m.state_len() * sizeof(float);
    // pageable caller memory takes the bounce path (worth waking eight threads from a few MB on)
    const bool big = state_bytes >= g_bounce_min_bytes.load() && bounce_enabled();
    bool b_in = big && state_in && is_pageable_host(state_in);
    bool b_out = big && state_out && is_pageable_host(state_out);
    if ((b_in || b_out) && !ensure_bounce(ctx)) b_in = b_out = false;
    const bool b_log = b_out && logits_out && is_pageable_host(logits_out);
    const int dev = m.dev.device;
    auto slice = [&](int g, size_t & off, size_t & cnt) { int l0, l1; segment_range(ctx, g, l0, l1); off = (size_t) l0 * per_layer; cnt = (size_t) (l1 - l0) * per_layer; };
    constexpr int LANES = CopyPool::LANES;
    auto part = [&](int g, int lane, size_t & off, size_t & cnt) {      // lane's share of slice g, in whole 64-byte lines
        size_t o, c; slice(g, o, c);
        const size_t per = ((c + LANES - 1) / LANES + 15) & ~(size_t) 15;
        const size_t b = std::min(c, per * (size_t) lane), e = std::min(c, per * (size_t) (lane + 1));
        off = o + b; cnt = e - b;
    };
    BouncePass bp;
    if (b_in || b_out) {
        bp.pool = ctx->bounce.pool.get();
        bp.pool->start([&, G, dev, b_in, b_out](int k) {
            const bool inward = k < LANES;
            const int lane = inward ? k : k - LANES;
            if (inward) {
                if (!b_in) return;
                for (int g = 1; g <= G && !bp.abort.load(); g++) {
                    size_t off, cnt; part(g, lane, off, cnt);
                    if (cnt) memcpy(ctx->bounce.in + off, state_in + off, cnt * sizeof(float));
                    bp.in_parts[g - 1].fetch_add(1, std::memory_order_release);
                }
            } else {
                if (!b_out) return;
                if (lane == 0) cudaSetDevice(dev);
                for (int g = 1; g <= G; g++) {
                    if (lane == 0) {      // one lane waits for the DMA, the others for that lane
                        while (bp.out_posted.load(std::memory_order_acquire) < g) { if (bp.abort.load()) return; std::this_thread::yield(); }
                        if (cudaEventSynchronize(ctx->bounce.seg_d2h[g - 1]) != cudaSuccess) { bp.abort.store(true); return; }
                        bp.out_arrived.store(g, std::memory_order_release);
                    } else {
                        while (bp.out_arrived.load(std::memory_order_acquire) < g) { if (bp.abort.load()) return; std::this_thread::yield(); }
                    }
                    size_t off, cnt; part(g, lane, off, cnt);
                    if (cnt) memcpy(state_out + off, ctx->bounce.out + off, cnt * sizeof(float));
                }
            }
        });
    }
    // nothing of this pass may start before everything enqueued earlier on the context's stream has finished with the state
    CUDA_OK(ctx, cudaEventRecord(ctx->copies.pass_begin, ctx->stream));
    CUDA_OK(ctx, cudaStreamWaitEvent(ctx->copies.in, ctx->copies.pass_begin, 0));
    if (state_in && !b_in) {
        for (int g = 1; g <= G; g++) {
            size_t off, cnt; slice(g, off, cnt);
            CUDA_OK(ctx, cudaMemcpyAsync(ctx->state_a + off, state_in + off, cnt * sizeof(float), cudaMemcpyDefault, ctx->copies.in));
            CUDA_OK(ctx, cudaEventRecord(ctx->copies.seg_in[g - 1], ctx->copies.in));
        }
    } else if (!state_in && !resident_in) {
        CUDA_OK(ctx, cudaMemcpyAsync(ctx->state_a, ctx->state_init, m.state_len() * sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
    }
    Pass p;
    if (!make_pass(ctx, T, logits_out != nullptr, nullptr, p) || !begin_pass(ctx, tokens, p)) return false;
    for (int g = 1; g <= G; g++) {
        if (b_in) {      // the slice is in pinned memory once every lane has delivered its part
            while (bp.in_parts[g - 1].load(std::memory_order_acquire) < LANES) std::this_thread::yield();
            size_t off, cnt; slice(g, off, cnt);
            CUDA_OK(ctx, cudaMemcpyAsync(ctx->state_a + off, ctx->bounce.in + off, cnt * sizeof(float), cudaMemcpyHostToDevice, ctx->copies.in));
            CUDA_OK(ctx, cudaEventRecord(ctx->copies.seg_in[g - 1], ctx->copies.in));
        }
        if (state_in) CUDA_OK(ctx, cudaStreamWaitEvent(ctx->stream, ctx->copies.seg_in[g - 1], 0));
        if (!run_layers(ctx, p, g)) return false;
        CUDA_OK(ctx, cudaEventRecord(ctx->copies.seg_out[g - 1], ctx->stream));
        if (b_out && g > 1) {      // one group behind: the copy-out stream never waits for something that has not been enqueued
            size_t off, cnt; slice(g - 1, off, cnt);
            // the new state of group g-1 is in state_b until end_pass swaps the buffers
            CUDA_OK(ctx, cudaStreamWaitEvent(ctx->copies.out, ctx->copies.seg_out[g - 2], 0));
            CUDA_OK(ctx, cudaMemcpyAsync(ctx->bounce.out + off, ctx->state_b + off, cnt * sizeof(float), cudaMemcpyDeviceToHost, ctx->copies.out));
            CUDA_OK(ctx, cudaEventRecord(ctx->bounce.seg_d2h[g - 2], ctx->copies.out));
            bp.out_posted.store(g - 1, std::memory_order_release);
        }
    }
    if (!end_pass(ctx, p)) return false;      // the new state is ctx->state_a from here on
    if (logits_out) CUDA_OK(ctx, cudaMemcpyAsync(b_log ? ctx->bounce.logits : logits_out, ctx->logits, (size_t) m.n_vocab * sizeof(float), cudaMemcpyDefault, ctx->stream));
    if (state_out && b_out) {
        size_t off, cnt; slice(G, off, cnt);
        CUDA_OK(ctx, cudaStreamWaitEvent(ctx->copies.out, ctx->copies.seg_out[G - 1], 0));
        CUDA_OK(ctx, cudaMemcpyAsync(ctx->bounce.out + off, ctx->state_a + off, cnt * sizeof(float), cudaMemcpyDeviceToHost, ctx->copies.out));
        CUDA_OK(ctx, cudaEventRecord(ctx->bounce.seg_d2h[G - 1], ctx->copies.out));
        bp.out_posted.store(G, std::memory_order_release);
    } else if (state_out) {
        for (int g = 1; g <= G; g++) {
            size_t off, cnt; slice(g, off, cnt);
            CUDA_OK(ctx, cudaStreamWaitEvent(ctx->copies.out, ctx->copies.seg_out[g - 1], 0));
            CUDA_OK(ctx, cudaMemcpyAsync(state_out + off, ctx->state_a + off, cnt * sizeof(float), cudaMemcpyDefault, ctx->copies.out));
        }
    }
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    if (b_log) memcpy(logits_out, ctx->bounce.logits, (size_t) m.n_vocab * sizeof(float));
    if (state_out) CUDA_OK(ctx, cudaStreamSynchronize(ctx->copies.out));
    if (bp.pool) { bp.pool->wait(); bp.pool = nullptr; }      // the last slices have been copied to the caller
    return !bp.abort.load();
}

static bool can_overlap(const Context * ctx) {
    const Model & m = *ctx->model;
    return ctx->overlap_copies && ctx->n_segments > 1 && m.layer_begin == 0 && m.layer_end == m.n_layer && !ctx->profiling;
}

bool eval_host(Context * ctx, const uint32_t * tokens, size_t T, const float * state_in, float * state_out, float * logits_out) {
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    if (can_overlap(ctx) && T <= (size_t) MAX_TOKENS_PER_PASS && (state_in || state_out))
        return eval_host_overlapped(ctx, tokens, (int) T, state_in, false, state_out, logits_out);
    return upload_state(ctx, state_in) && forward(ctx, tokens, T, logits_out != nullptr) && download_outputs(ctx, state_out, logits_out);
}

bool eval_host_chunks(Context * ctx, const uint32_t * tokens, size_t T, size_t chunk, const float * state_in, float * state_out, float * logits_out) {
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    const bool overlap = can_overlap(ctx) && chunk <= (size_t) MAX_TOKENS_PER_PASS && (state_in || state_out);
    if (!overlap && !upload_state(ctx, state_in)) return false;
    // Same chunk boundaries as the reference loop (rwkv_eval.inc:179-218); the state never leaves HBM between chunks, logits are
    // computed for the final chunk only. With overlap the first chunk takes the caller's state group by group while it computes and
    // the last one hands the new state back the same way.
    size_t off = 0;
    while (off < T) {
        const size_t n = T - off < chunk ? T - off : chunk;
        const bool first = off == 0, last = off + n == T;
        if (overlap && (first || last)) {
            if (!eval_host_overlapped(ctx, tokens + off, (int) n, first ? state_in : nullptr, !first, last ? state_out : nullptr, last ? logits_out : nullptr)) return false;
        } else if (!forward(ctx, tokens + off, n, last && logits_out != nullptr)) {
            return false;
        }
        off += n;
    }
    return overlap ? true : download_outputs(ctx, state_out, logits_out);
}

bool forward(Context * ctx, const uint32_t * tokens, size_t T, bool want_logits) {
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    size_t done = 0;
    while (done < T) {
        const size_t n = (T - done < (size_t) MAX_TOKENS_PER_PASS) ? T - done : (size_t) MAX_TOKENS_PER_PASS;
        const bool last = done + n == T;
        Pass p;
        if (!make_pass(ctx, (int) n, want_logits && last, nullptr, p) || !forward_pass(ctx, tokens + done, p)) return false;
        done += n;
    }
    return true;
}

bool batch_set_state(Context * ctx, int seq, const float * state_in) {
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, ctx->batch_n > 0 && seq >= 0 && seq < ctx->batch_n, "Not a batch context or sequence index out of range");
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    const size_t n = ctx->model->state_len();
    float * dst = ctx->state_a + (size_t) seq * n;
    if (state_in) CUDA_OK(ctx, cudaMemcpyAsync(dst, state_in, n * sizeof(float), cudaMemcpyDefault, ctx->stream));
    else CUDA_OK(ctx, cudaMemcpyAsync(dst, ctx->state_init, n * sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
    return true;
}

bool batch_get_state(Context * ctx, int seq, float * state_out) {
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, ctx->batch_n > 0 && seq >= 0 && seq < ctx->batch_n && state_out, "Not a batch context, sequence index out of range or NULL buffer");
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    const size_t n = ctx->model->state_len();
    CUDA_OK(ctx, cudaMemcpyAsync(state_out, ctx->state_a + (size_t) seq * n, n * sizeof(float), cudaMemcpyDefault, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return true;
}

bool batch_eval(Context * ctx, const uint32_t * tokens, bool want_logits) {
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, ctx->batch_n > 0 && tokens, "Not a batch context or NULL tokens");
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    Pass p;
    return make_pass(ctx, ctx->batch_n, want_logits, nullptr, p) && forward_pass(ctx, tokens, p);
}

// ---- checkpoints ---------------------------------------------------------------------------------------------------------------
// The checkpoints of one pass: those at a column inside it, which the kernels write, and those at the last column of their sequence,
// copies of that sequence's state after the pass.
struct PassCheckpoints {
    struct Inner { int col; float * dst; };
    struct AtEnd { int seq; float * dst; };
    std::vector<Inner> inner;
    std::vector<AtEnd> at_end;
};

static bool on_device(const void * p, int * device = nullptr) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    if (device) *device = a.device;
    return a.type == cudaMemoryTypeDevice;
}

// The kernels write a checkpoint straight into device memory that is 16-byte aligned (wkv6_kernel stores float4s); every other
// destination (host memory, or a device pointer at another offset) is written to Context::cp_staging and copied after the pass.
static bool written_in_place(const float * p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0 && on_device(p); }

bool check_checkpoints(ErrorSink sink, size_t n_seq, const uint32_t * counts, size_t state_len, int device, const CheckpointReq * cp, size_t n_cp) {
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, cp || n_cp == 0, "NULL checkpoints");
    std::vector<uintptr_t> at(n_cp);
    for (size_t i = 0; i < n_cp; i++) {
        const CheckpointReq & c = cp[i];
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, c.state_out, "Checkpoint %zu has a NULL state_out", i);
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, c.sequence < n_seq && c.position < counts[c.sequence],
                   "Checkpoint %zu (sequence %u, position %u) is out of range", i, c.sequence, c.position);
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, i == 0 || c.sequence > cp[i - 1].sequence || (c.sequence == cp[i - 1].sequence && c.position > cp[i - 1].position),
                   "Checkpoint %zu is not after checkpoint %zu", i, i - 1);
        int dev = -1;
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, device < 0 || !on_device(c.state_out, &dev) || dev == device,
                   "Checkpoint %zu's state_out is memory of device %d, not of the context's device %d", i, dev, device);
        at[i] = reinterpret_cast<uintptr_t>(c.state_out);
    }
    std::sort(at.begin(), at.end());
    for (size_t i = 1; i < n_cp; i++)
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, at[i] - at[i - 1] >= state_len * sizeof(float), "Two checkpoints' state_out ranges overlap");
    return true;
}

// The maps and the staging for the passes of a call (plan), built before the call enqueues anything; a grown staging replaces the old
// one after a synchronise, as the other sets grow.
static bool ensure_checkpoint_buffers(Context * ctx, const std::vector<PassCheckpoints> & plan) {
    size_t inner = 0, host = 0;
    for (const PassCheckpoints & pc : plan) {
        inner += pc.inner.size();
        size_t h = 0;
        for (const PassCheckpoints::Inner & c : pc.inner) h += !written_in_place(c.dst);
        host = std::max(host, h);
    }
    if (inner && !ctx->cps.map) {
        Context::CheckpointMaps m;
        const size_t bytes = (size_t) MAX_TOKENS_PER_PASS * (sizeof(int) + sizeof(float *));
        cudaError_t e = m.map.alloc(bytes);
        for (int i = 0; i < 2 && e == cudaSuccess; i++) e = m.host[i].alloc(bytes);
        RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, false, e == cudaSuccess, "Failed to allocate the checkpoint maps: %s", cudaGetErrorString(e));
        ctx->cps = std::move(m);
    }
    if (host > ctx->cp_staging.count) {
        CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
        ctx->cp_staging = {};
        Context::CheckpointStaging st;
        const size_t bytes = host * ctx->model->state_len() * sizeof(float);
        const cudaError_t e = st.states.alloc(bytes);
        RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, false, e == cudaSuccess, "Failed to allocate %zu bytes of checkpoint staging: %s", bytes, cudaGetErrorString(e));
        st.count = host;
        ctx->cp_staging = std::move(st);
    }
    return true;
}

// After begin_pass (which waited for the pass that last read this phase's slot): the map of the pass's inner checkpoints, uploaded, and
// the copies of staged states that follow the pass.
struct StagedCopy { float * dst; const float * src; };
static bool stage_checkpoints(Context * ctx, Pass & p, const PassCheckpoints & pc, std::vector<StagedCopy> & staged) {
    staged.clear();
    if (pc.inner.empty()) return true;
    unsigned char * host = ctx->cps.host[p.phase];
    int * slot = reinterpret_cast<int *>(host);
    float ** dst = reinterpret_cast<float **>(host + MAX_TOKENS_PER_PASS * sizeof(int));
    for (int t = 0; t < p.T; t++) slot[t] = -1;
    const size_t n = ctx->model->state_len();
    for (size_t k = 0; k < pc.inner.size(); k++) {
        slot[pc.inner[k].col] = (int) k;
        dst[k] = pc.inner[k].dst;
        if (!written_in_place(dst[k])) {
            dst[k] = ctx->cp_staging.states + staged.size() * n;
            staged.push_back({pc.inner[k].dst, dst[k]});
        }
    }
    const size_t bytes = (size_t) MAX_TOKENS_PER_PASS * (sizeof(int) + sizeof(float *));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->cps.map, host, bytes, cudaMemcpyHostToDevice, p.stream));
    p.cp_slot = reinterpret_cast<const int *>(ctx->cps.map.get());
    p.cp_dst = reinterpret_cast<float * const *>(ctx->cps.map.get() + MAX_TOKENS_PER_PASS * sizeof(int));
    return true;
}

// After end_pass: the staged states to their host destinations, and the checkpoints at the pass's end from the new state (state_a).
static bool finish_checkpoints(Context * ctx, const Pass & p, const PassCheckpoints & pc, const std::vector<StagedCopy> & staged) {
    const size_t n = ctx->model->state_len();
    for (const StagedCopy & c : staged) CUDA_OK(ctx, cudaMemcpyAsync(c.dst, c.src, n * sizeof(float), cudaMemcpyDefault, p.stream));
    for (const PassCheckpoints::AtEnd & c : pc.at_end)
        CUDA_OK(ctx, cudaMemcpyAsync(c.dst, ctx->state_a + (size_t) c.seq * n, n * sizeof(float), cudaMemcpyDefault, p.stream));
    return true;
}

bool forward_checkpoints(Context * ctx, const uint32_t * tokens, size_t T, bool want_logits, const CheckpointReq * cp, size_t n_cp) {
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    const size_t P = MAX_TOKENS_PER_PASS;
    std::vector<PassCheckpoints> plan((T + P - 1) / P);
    for (size_t i = 0; i < n_cp; i++) {
        const size_t pass = cp[i].position / P, col = cp[i].position % P, n = std::min(P, T - pass * P);
        if (col + 1 == n) plan[pass].at_end.push_back({0, cp[i].state_out});
        else plan[pass].inner.push_back({(int) col, cp[i].state_out});
    }
    if (!ensure_checkpoint_buffers(ctx, plan)) return false;
    std::vector<StagedCopy> staged;
    for (size_t k = 0, done = 0; done < T; k++) {
        const size_t n = std::min(P, T - done);
        Pass p;
        if (!make_pass(ctx, (int) n, want_logits && done + n == T, nullptr, p) || !begin_pass(ctx, tokens + done, p) ||
            !stage_checkpoints(ctx, p, plan[k], staged) || !run_layers(ctx, p, 0) || !end_pass(ctx, p) || !finish_checkpoints(ctx, p, plan[k], staged))
            return false;
        done += n;
    }
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return true;
}

// Ints of one ragged map (Context::ragged_host): offsets [B + 1], column sequences [MAX_TOKENS_PER_PASS], head columns and sequences [B each].
static size_t ragged_map_ints(int B) { return (size_t) 3 * B + 1 + MAX_TOKENS_PER_PASS; }

bool check_ragged(Context * ctx, const uint32_t * tokens, const uint32_t * counts, size_t & total) {
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, ctx->batch_n > 0, "Not a batch context");
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, tokens && counts, "NULL tokens or counts");
    const Model & m = *ctx->model;
    total = 0;
    for (int b = 0; b < ctx->batch_n; b++) total += counts[b];
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, total >= 1 && total <= (size_t) MAX_TOKENS_PER_PASS, "A ragged pass takes 1 .. %d tokens in all, not %zu", MAX_TOKENS_PER_PASS, total);
    for (size_t i = 0; i < total; i++)
        RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, tokens[i] < (uint32_t) m.n_vocab, "Token at index %zu (%" PRIu32 ") is out of range (0 .. %d)", i, tokens[i], m.n_vocab - 1);
    return true;
}

// batch_eval_ragged on arguments that passed check_ragged (T tokens in all); with targets, a scoring pass whose results go to lp and
// greedy (greedy may be NULL).
static bool ragged_pass(Context * ctx, const uint32_t * tokens, const uint32_t * counts, int T, bool want_logits, const uint32_t * targets,
                        float * lp, uint8_t * greedy, const PassCheckpoints * pc = nullptr) {
    const Model & m = *ctx->model;
    const int B = ctx->batch_n;
    CUDA_OK(ctx, cudaSetDevice(m.dev.device));
    const size_t map_bytes = ragged_map_ints(B) * sizeof(int);
    if (!ctx->ragged.map) {
        Context::Ragged r;
        for (int i = 0; i < 2; i++) CUDA_OK(ctx, r.host[i].alloc(map_bytes));
        CUDA_OK(ctx, r.head_x.alloc((size_t) B * m.n_embed * sizeof(float)));
        CUDA_OK(ctx, r.head_y.alloc((size_t) B * m.n_vocab * sizeof(float)));
        CUDA_OK(ctx, r.map.alloc(map_bytes));
        ctx->ragged = std::move(r);
    }
    Pass p;
    if (!make_pass(ctx, T, want_logits, nullptr, p) || !begin_pass(ctx, tokens, p)) return false;   // waits until the pass that last used this phase's slots has read them
    int * off = ctx->ragged.host[p.phase], * col_seq = off + B + 1, * head_col = col_seq + MAX_TOKENS_PER_PASS, * head_seq = head_col + B;
    off[0] = 0;
    for (int b = 0; b < B; b++) {
        off[b + 1] = off[b] + (int) counts[b];
        for (int t = off[b]; t < off[b + 1]; t++) col_seq[t] = b;
        if (counts[b]) { head_col[p.n_active] = off[b + 1] - 1; head_seq[p.n_active] = b; p.n_active++; }
    }
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->ragged.map, off, map_bytes, cudaMemcpyHostToDevice, p.stream));
    // the state of every idle sequence (runs of them are contiguous) goes to state_b as it is: end_pass swaps the whole buffers
    const size_t n = m.state_len();
    for (int b = 0; b < B;) {
        if (counts[b]) { b++; continue; }
        int e = b;
        while (e < B && !counts[e]) e++;
        CUDA_OK(ctx, cudaMemcpyAsync(p.state_out + (size_t) b * n, p.state_in + (size_t) b * n, (size_t) (e - b) * n * sizeof(float), cudaMemcpyDeviceToDevice, p.stream));
        b = e;
    }
    p.seq_off = ctx->ragged.map;
    p.col_seq = p.seq_off + B + 1;
    p.col_seq_host = col_seq;
    p.head_col = p.col_seq + MAX_TOKENS_PER_PASS;
    p.head_seq = p.head_col + B;
    p.targets = targets; p.lp = lp; p.greedy = greedy;
    std::vector<StagedCopy> staged;
    if (pc && !stage_checkpoints(ctx, p, *pc, staged)) return false;
    if (!enqueue_pass(ctx, p, 0)) return false;     // never a graph: the map changes from call to call
    const bool had_logits = ctx->logits_valid;
    if (!end_pass(ctx, p)) return false;
    ctx->logits_valid = had_logits || want_logits;     // idle columns keep what they held
    return !pc || finish_checkpoints(ctx, p, *pc, staged);
}

bool batch_eval_ragged(Context * ctx, const uint32_t * tokens, const uint32_t * counts, bool want_logits) {
    size_t total = 0;
    return check_ragged(ctx, tokens, counts, total) && ragged_pass(ctx, tokens, counts, (int) total, want_logits, nullptr, nullptr, nullptr);
}

bool batch_eval_ragged_checkpoints(Context * ctx, const uint32_t * tokens, const uint32_t * counts, size_t total, bool want_logits, const CheckpointReq * cp,
                                   size_t n_cp) {
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    std::vector<PassCheckpoints> plan(1);
    std::vector<uint32_t> off(ctx->batch_n + 1, 0);
    for (int b = 0; b < ctx->batch_n; b++) off[b + 1] = off[b] + counts[b];
    for (size_t i = 0; i < n_cp; i++) {
        const uint32_t s = cp[i].sequence, pos = cp[i].position;
        if (pos + 1 == counts[s]) plan[0].at_end.push_back({(int) s, cp[i].state_out});
        else plan[0].inner.push_back({(int) (off[s] + pos), cp[i].state_out});
    }
    if (!ensure_checkpoint_buffers(ctx, plan) || !ragged_pass(ctx, tokens, counts, (int) total, want_logits, nullptr, nullptr, nullptr, &plan[0])) return false;
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return true;
}

bool batch_get_logits(Context * ctx, int seq, float * logits_out) {
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, ctx->batch_n > 0 && seq >= 0 && seq < ctx->batch_n && logits_out, "Not a batch context, sequence index out of range or NULL buffer");
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, ctx->logits_valid, "The last batch evaluation skipped the head");
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    const size_t V = (size_t) ctx->model->n_vocab;
    CUDA_OK(ctx, cudaMemcpyAsync(logits_out, ctx->logits + (size_t) seq * V, V * sizeof(float), cudaMemcpyDefault, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return true;
}

namespace {

// The head's tile-major copy (Model::head_tiled), built once per model by the first scoring pass that routes its head to the tensor
// cores: 2 bytes per weight, so a model that is never scored that way does not pay for it.
bool ensure_head_tiled(Context * ctx) {
    Model & m = *ctx->model;
    std::lock_guard<std::mutex> lk(m.head_tiled_lock);
    if (m.head_tiled) return true;
    const size_t bytes = gemm_tc_tiled_bytes(m.head.type, m.head.M, m.head.K);
    DeviceBuffer<uint8_t> p;
    cudaError_t e = p.alloc(bytes);
    if (e != cudaSuccess) cudaGetLastError();
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, false, e == cudaSuccess, "Failed to allocate %zu bytes for the head's tile-major copy: %s", bytes, cudaGetErrorString(e));
    e = gemm_tc_repack(m.head.data, m.head.pitch, m.head.type, m.head.M, m.head.K, p, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);      // other contexts' streams use it from now on
    CUDA_OK(ctx, e);
    m.head_tiled = std::move(p);
    return true;
}

// The scoring buffers for a call of n tokens (the targets and results grow to the largest call so far), and the head's tile-major copy
// if any pass of the call routes its head to the tensor cores. Allocates, enqueues nothing.
bool prepare_score(Context * ctx, size_t n, bool any_tc) {
    const Model & m = *ctx->model;
    CUDA_OK(ctx, cudaSetDevice(m.dev.device));
    auto alloc = [&](auto & buf, size_t bytes) {
        const cudaError_t e = buf.alloc(bytes);
        if (e != cudaSuccess) cudaGetLastError();
        RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, false, e == cudaSuccess, "Failed to allocate %zu bytes of scoring buffers: %s", bytes, cudaGetErrorString(e));
        return true;
    };
    if (!ctx->score_logits && !alloc(ctx->score_logits, (size_t) MAX_TOKENS_PER_PASS * m.n_vocab * sizeof(float))) return false;
    if (n > ctx->score.capacity) {
        CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
        ctx->score = {};
        Context::ScoreIo io;
        io.capacity = 256;
        while (io.capacity < n) io.capacity *= 2;
        if (!alloc(io.targets, io.capacity * sizeof(uint32_t)) || !alloc(io.lp, io.capacity * sizeof(float)) || !alloc(io.greedy, io.capacity)) return false;
        ctx->score = std::move(io);
    }
    return !any_tc || ensure_head_tiled(ctx);
}

// Targets in, and the caller's outputs too, so that positions without a target come back as they were.
bool score_copy_in(Context * ctx, const uint32_t * targets, size_t n, const float * logprobs_out, const uint8_t * greedy_out) {
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->score.targets, targets, n * sizeof(uint32_t), cudaMemcpyDefault, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->score.lp, logprobs_out, n * sizeof(float), cudaMemcpyDefault, ctx->stream));
    if (greedy_out) CUDA_OK(ctx, cudaMemcpyAsync(ctx->score.greedy, greedy_out, n, cudaMemcpyDefault, ctx->stream));
    return true;
}

bool score_copy_out(Context * ctx, size_t n, float * logprobs_out, uint8_t * greedy_out) {
    CUDA_OK(ctx, cudaMemcpyAsync(logprobs_out, ctx->score.lp, n * sizeof(float), cudaMemcpyDefault, ctx->stream));
    if (greedy_out) CUDA_OK(ctx, cudaMemcpyAsync(greedy_out, ctx->score.greedy, n, cudaMemcpyDefault, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return true;
}

}  // namespace

bool score(Context * ctx, const uint32_t * tokens, const uint32_t * targets, size_t n, float * logprobs_out, uint8_t * greedy_out) {
    // the passes of forward(): MAX_TOKENS_PER_PASS tokens each, then the rest; only the first can be the longest
    const int first = (int) std::min(n, (size_t) MAX_TOKENS_PER_PASS);
    if (!prepare_score(ctx, n, score_on_tensor_cores(ctx, first))) return false;
    if (!score_copy_in(ctx, targets, n, logprobs_out, greedy_out)) return false;
    for (size_t done = 0; done < n;) {
        const int T = (int) std::min(n - done, (size_t) MAX_TOKENS_PER_PASS);
        Pass p;
        if (!make_pass(ctx, T, true, nullptr, p)) return false;
        p.targets = ctx->score.targets + done;
        p.lp = ctx->score.lp + done;
        p.greedy = greedy_out ? ctx->score.greedy + done : nullptr;
        // enqueue_pass directly: a scoring pass is never captured into a graph or replayed from one
        if (!begin_pass(ctx, tokens + done, p) || !enqueue_pass(ctx, p, 0) || !end_pass(ctx, p)) return false;
        done += (size_t) T;
    }
    return score_copy_out(ctx, n, logprobs_out, greedy_out);
}

bool batch_score_ragged(Context * ctx, const uint32_t * tokens, const uint32_t * counts, const uint32_t * targets, float * logprobs_out, uint8_t * greedy_out) {
    size_t total = 0;
    if (!check_ragged(ctx, tokens, counts, total)) return false;
    if (!prepare_score(ctx, total, score_on_tensor_cores(ctx, (int) total))) return false;
    if (!score_copy_in(ctx, targets, total, logprobs_out, greedy_out)) return false;
    return ragged_pass(ctx, tokens, counts, (int) total, true, ctx->score.targets, ctx->score.lp, greedy_out ? ctx->score.greedy.get() : nullptr) &&
           score_copy_out(ctx, total, logprobs_out, greedy_out);
}

namespace {

// Device copy of a logit bias list (the buffers grow as needed) and the scratch of scratch_floats floats the biased logits go to.
bool upload_bias(Context * ctx, const uint32_t * bias_ids, const float * bias_values, size_t n_bias, size_t scratch_floats) {
    if (!ctx->sample_scratch) CUDA_OK(ctx, ctx->sample_scratch.alloc(scratch_floats * sizeof(float)));
    if (n_bias > ctx->bias.capacity) {
        CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
        ctx->bias = {};
        Context::Bias b;
        CUDA_OK(ctx, b.ids.alloc(n_bias * sizeof(uint32_t)));
        CUDA_OK(ctx, b.values.alloc(n_bias * sizeof(float)));
        b.capacity = n_bias;
        ctx->bias = std::move(b);
    }
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->bias.ids, bias_ids, n_bias * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->bias.values, bias_values, n_bias * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    return true;
}

}  // namespace

bool sample_token(Context * ctx, float temperature, float top_p, double u, const uint32_t * bias_ids, const float * bias_values, size_t n_bias, uint32_t * token_out) {
    const Model & m = *ctx->model;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, token_out != nullptr, "token_out is NULL");
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, ctx->batch_n == 0, "Sampling on a batch context is not supported");
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, temperature >= 0.0f, "temperature must be >= 0");            // sampling.py:20-21
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, top_p >= 0.0f && top_p <= 1.0f, "top_p must be in [0, 1]");    // sampling.py:22-23
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, u >= 0.0 && u < 1.0, "u must be in [0, 1)");
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, n_bias == 0 || (bias_ids && bias_values), "logit bias arrays are NULL");
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, ctx->logits_valid, "No logits to sample from: the last evaluation skipped the head");
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, m.n_vocab <= 65536, "On-device sampling supports n_vocab <= 65536");
    CUDA_OK(ctx, cudaSetDevice(m.dev.device));
    if (!ctx->sample_out.token) {
        Context::SampleOut o;
        CUDA_OK(ctx, o.token.alloc(2 * sizeof(uint32_t)));
        CUDA_OK(ctx, o.token_host.alloc(2 * sizeof(uint32_t)));
        ctx->sample_out = std::move(o);
    }
    std::vector<uint64_t> seen;
    if (!check_bias_ids(ctx->sink(), bias_ids, n_bias, (size_t) m.n_vocab, seen)) return false;
    if (n_bias > 0 && !upload_bias(ctx, bias_ids, bias_values, n_bias, (size_t) m.n_vocab)) return false;
    SampleParams sp{};
    sp.logits = ctx->logits; sp.n_vocab = m.n_vocab; sp.temperature = temperature; sp.top_p = top_p; sp.u = u;
    sp.bias_ids = ctx->bias.ids; sp.bias_values = ctx->bias.values; sp.n_bias = (int) n_bias;
    sp.scratch = ctx->sample_scratch; sp.token_out = ctx->sample_out.token; sp.prob_out = nullptr;
    CUDA_OK(ctx, launch_sample(sp, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->sample_out.token_host, ctx->sample_out.token, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    *token_out = ctx->sample_out.token_host[0];
    return true;
}

static_assert(SAMPLE_MAX_ROWS == MAX_TOKENS_PER_PASS, "the batched sampling launch takes a row per sequence of the largest batch");

bool check_bias_ids(ErrorSink sink, const uint32_t * bias_ids, size_t n_bias, size_t n_vocab, std::vector<uint64_t> & seen) {
    if (seen.size() < (n_vocab + 63) / 64) seen.assign((n_vocab + 63) / 64, 0);
    bool ok = true;
    size_t i = 0;
    for (; i < n_bias && ok; i++) {
        const uint32_t id = bias_ids[i];
        ok = id < n_vocab && !(seen[id >> 6] >> (id & 63) & 1);
        if (ok) seen[id >> 6] |= 1ull << (id & 63);
    }
    for (size_t k = 0; k < i; k++) if (bias_ids[k] < n_vocab) seen[bias_ids[k] >> 6] = 0;
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, ok, "logit bias id %u is %s", bias_ids[i - 1], bias_ids[i - 1] < n_vocab ? "given twice" : "out of range");
    return true;
}

bool check_sample_rows(ErrorSink sink, size_t n_rows, size_t n_vocab, const float * temperature, const float * top_p, const double * u,
                       const uint32_t * bias_offsets, const uint32_t * bias_ids, const float * bias_values, const uint32_t * tokens_out) {
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, temperature && top_p && u && tokens_out, "NULL temperature, top_p, u or tokens_out");
    for (size_t b = 0; b < n_rows; b++) {     // sampling.py:20-23, as sample_token checks its one row
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, temperature[b] >= 0.0f, "temperature of row %zu must be >= 0", b);
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, top_p[b] >= 0.0f && top_p[b] <= 1.0f, "top_p of row %zu must be in [0, 1]", b);
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, u[b] >= 0.0 && u[b] < 1.0, "u of row %zu must be in [0, 1)", b);
    }
    if (!bias_offsets) return true;
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, bias_offsets[0] == 0, "bias_offsets must start at 0");
    for (size_t b = 0; b < n_rows; b++)
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, bias_offsets[b + 1] >= bias_offsets[b], "bias_offsets decrease after row %zu", b);
    const size_t n_bias = bias_offsets[n_rows];
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, n_bias <= (size_t) INT32_MAX, "More than 2^31 - 1 logit bias entries");
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, n_bias == 0 || (bias_ids && bias_values), "logit bias arrays are NULL");
    std::vector<uint64_t> seen;
    for (size_t b = 0; b < n_rows; b++)
        if (!check_bias_ids(sink, bias_ids + bias_offsets[b], bias_offsets[b + 1] - bias_offsets[b], n_vocab, seen)) return false;
    return true;
}

void fill_sample_rows(SampleRow * rows, size_t n_rows, const float * temperature, const float * top_p, const double * u, const uint32_t * bias_offsets) {
    for (size_t b = 0; b < n_rows; b++)
        rows[b] = SampleRow{temperature[b], top_p[b], u[b], bias_offsets ? (int) bias_offsets[b] : 0, bias_offsets ? (int) bias_offsets[b + 1] : 0};
}

bool batch_sample(Context * ctx, const float * temperature, const float * top_p, const double * u, const uint32_t * bias_offsets,
                  const uint32_t * bias_ids, const float * bias_values, uint32_t * tokens_out) {
    const Model & m = *ctx->model;
    const int B = ctx->batch_n;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, B > 0, "Not a batch context");
    if (!check_sample_rows(ctx->sink(), B, m.n_vocab, temperature, top_p, u, bias_offsets, bias_ids, bias_values, tokens_out)) return false;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, ctx->logits_valid, "No logits to sample from: the last batch evaluation skipped the head");
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, m.n_vocab <= 65536, "On-device sampling supports n_vocab <= 65536");
    const size_t n_bias = bias_offsets ? bias_offsets[B] : 0;
    CUDA_OK(ctx, cudaSetDevice(m.dev.device));
    if (!ctx->sample_rows.rows) {
        Context::SampleRows r;
        CUDA_OK(ctx, r.rows.alloc((size_t) B * sizeof(SampleRow)));
        CUDA_OK(ctx, r.rows_host.alloc((size_t) B * sizeof(SampleRow)));
        CUDA_OK(ctx, r.tokens.alloc((size_t) B * sizeof(uint32_t)));
        CUDA_OK(ctx, r.tokens_host.alloc((size_t) B * sizeof(uint32_t)));
        ctx->sample_rows = std::move(r);
    }
    if (n_bias > 0 && !upload_bias(ctx, bias_ids, bias_values, n_bias, (size_t) B * m.n_vocab)) return false;
    // every call ends with a stream synchronisation, so the previous copy out of the pinned rows has completed
    fill_sample_rows(ctx->sample_rows.rows_host, B, temperature, top_p, u, bias_offsets);
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->sample_rows.rows, ctx->sample_rows.rows_host, (size_t) B * sizeof(SampleRow), cudaMemcpyHostToDevice, ctx->stream));
    SampleBatchParams bp{};
    bp.logits = ctx->logits; bp.n_vocab = m.n_vocab; bp.n_rows = B; bp.rows = ctx->sample_rows.rows;
    bp.bias_ids = n_bias ? ctx->bias.ids.get() : nullptr; bp.bias_values = n_bias ? ctx->bias.values.get() : nullptr;
    bp.scratch = n_bias ? ctx->sample_scratch.get() : nullptr; bp.token_out = ctx->sample_rows.tokens; bp.prob_out = nullptr;
    CUDA_OK(ctx, launch_sample_batch(bp, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->sample_rows.tokens_host, ctx->sample_rows.tokens, (size_t) B * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    memcpy(tokens_out, ctx->sample_rows.tokens_host, (size_t) B * sizeof(uint32_t));
    return true;
}

bool batch_eval_sample(Context * ctx, const uint32_t * tokens, const float * temperature, const float * top_p, const double * u, uint32_t * tokens_out) {
    const Model & m = *ctx->model;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, ctx->batch_n > 0, "Not a batch context");
    if (!check_sample_rows(ctx->sink(), ctx->batch_n, m.n_vocab, temperature, top_p, u, nullptr, nullptr, nullptr, tokens_out)) return false;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, m.n_vocab <= 65536, "On-device sampling supports n_vocab <= 65536");
    return batch_eval(ctx, tokens, true) && batch_sample(ctx, temperature, top_p, u, nullptr, nullptr, nullptr, tokens_out);
}

// ---- device-side generation -----------------------------------------------------------------------------------------------------
// The loop of a generate call is one graph launch: WHILE { step -> IF { pass X -> Y } -> step -> IF { pass Y -> X } }. Each step
// (generate_sample_kernel) draws every active row's next token and writes it into ctx->act.tokens, then sets both conditions to "a row is
// still active". A body holds two passes because the passes double-buffer the state. In a batch context every pass computes all
// columns, so its shape and graph stay fixed; a frozen row's state is copied back over its output after each pass and its logits,
// parked by the step that froze it, come back after the loop.
// A streaming loop runs generate_stream_sample_kernel instead: after each draw it publishes the token to mapped host memory, and
// before the next draw of that row it waits for the calling thread to acknowledge it (stream_tokens), so that the pass evaluating
// token j overlaps the callback of token j, and a callback can end its row before token j + 1 is drawn.
// A loop that reports log-probabilities runs the logprob step kernels instead, in graphs of their own (gen_graphs[..][GEN_LOGPROBS]);
// they read the call's GenLogprobRequest from ctx->lp_req.dev, and the streaming one writes each token's record into the mapped ring
// before it publishes the token, so that stream_tokens can hand the record to the caller before on_token.
// A loop with per-row samplers runs the sampled step kernels, in graphs of their own too (gen_graphs[..][GEN_SAMPLED]); they read the
// rows, the bias pool and the request word (ctx->lp_req.dev, or NULL without log-probabilities) from ctx->smp.dev.
namespace {

size_t gen_mask_offset(int rows) { return (sizeof(GenShared) + (size_t) rows * sizeof(GenRow) + 7) / 8 * 8; }
size_t gen_u_offset(int rows) { return gen_mask_offset(rows) + (size_t) rows * sizeof(GenMaskRow); }
size_t gen_tokens_word(int rows) { return 2 * (size_t) rows + 1; }
size_t gen_out_words(int rows, size_t n) { return gen_tokens_word(rows) + (size_t) rows * n; }

size_t stream_token_offset(int rows) { return 2 * (size_t) rows + 1; }
size_t smp_rows_offset() { return sizeof(const GenLogprobRequest *); }
size_t smp_bias_offset(int rows) { return smp_rows_offset() + (size_t) rows * sizeof(GenSamplerRow); }

// The step kernel's parameters over the context's buffers, with the fields that `family` and `streaming` read.
GenStepParams generate_step_params(Context * ctx, GenFamily family, bool streaming) {
    const int rows = ctx->batch_n ? ctx->batch_n : 1;
    GenStepParams gp{};
    gp.logits = ctx->logits; gp.n_vocab = ctx->model->n_vocab; gp.n_rows = rows;
    gp.shared = reinterpret_cast<GenShared *>(ctx->gen.in.get());
    gp.rows = reinterpret_cast<GenRow *>(ctx->gen.in + sizeof(GenShared));
    gp.u = reinterpret_cast<const double *>(ctx->gen.in + gen_u_offset(rows));
    gp.counts = ctx->gen.counts; gp.bias_ids = ctx->gen.bias_ids; gp.bias_values = ctx->gen.bias_values; gp.scratch = ctx->gen.scratch;
    gp.n_generated = ctx->gen.out; gp.passes = ctx->gen.out + rows; gp.tokens = ctx->gen.out + gen_tokens_word(rows);
    gp.next_tokens = ctx->act.tokens; gp.park = ctx->batch_n ? ctx->gen.park.get() : nullptr;
    if (streaming) {
        uint32_t * words = ctx->streamed.words.device();
        gp.published = words; gp.acked = words + rows; gp.timed_out = words + 2 * rows; gp.stream_tokens = words + stream_token_offset(rows);
    }
    if (family != GEN_PLAIN) {
        gp.mask = reinterpret_cast<GenMaskRow *>(ctx->gen.in + gen_mask_offset(rows));
        gp.states_out = ctx->gen.out + rows + 1;
    }
    if (family == GEN_LOGPROBS) gp.lp = ctx->lp_req.dev;
    if (family == GEN_SAMPLED) {
        gp.lp_word = reinterpret_cast<const GenLogprobRequest * const *>(ctx->smp.dev.get());
        gp.samplers = reinterpret_cast<const GenSamplerRow *>(ctx->smp.dev + smp_rows_offset());
        gp.user_bias = reinterpret_cast<const GenBiasEntry *>(ctx->smp.dev + smp_bias_offset(rows));
    }
    return gp;
}

// Pass p of the loop (input tokens already in ctx->act.tokens) captured into `body`; in a batch context the frozen rows of `rows`
// keep their state.
bool capture_generate_pass(Context * ctx, cudaGraph_t body, const Pass & p, const GenRow * rows) {
    CUDA_OK(ctx, cudaStreamBeginCaptureToGraph(p.stream, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
    bool ok = enqueue_pass(ctx, p, 0);
    cudaError_t e = cudaSuccess;
    if (ok && ctx->batch_n)
        e = launch_restore_frozen(rows, p.T, p.state_in, p.state_out, ctx->batch_stride, ctx->model->state_len(), p.stream);
    cudaGraph_t out = nullptr;
    const cudaError_t ec = cudaStreamEndCapture(p.stream, &out);
    if (e == cudaSuccess) e = ec;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, ok && e == cudaSuccess, "Capturing the generation pass failed: %s", cudaGetErrorString(e));
    return true;
}

bool build_generate_graph(Context * ctx, GenFamily family, bool streaming) {
    const int rows = ctx->batch_n ? ctx->batch_n : 1;
    Pass p;
    if (!make_pass(ctx, rows, true, nullptr, p)) return false;
    p.tokens_in_place = true;
    {   // one uncaptured pass of the loop's shape first, as run_layers does before it captures; its logits go to the step's scratch
        // and its state to state_b, which holds nothing between passes
        CUDA_OK(ctx, cudaMemsetAsync(ctx->act.tokens, 0, (size_t) rows * sizeof(int), p.stream));
        Pass warm = p;
        warm.logits = ctx->gen.scratch;
        if (!enqueue_pass(ctx, warm, 0)) return false;
    }
    Graph top;
    CUDA_OK(ctx, top.create());
    cudaGraphConditionalHandle keep_going;
    CUDA_OK(ctx, cudaGraphConditionalHandleCreate(&keep_going, top, 1, cudaGraphCondAssignDefault));
    cudaGraphNodeParams wp = {};
    wp.type = cudaGraphNodeTypeConditional;
    wp.conditional.handle = keep_going; wp.conditional.type = cudaGraphCondTypeWhile; wp.conditional.size = 1;
    cudaGraphNode_t loop = nullptr;
    CUDA_OK(ctx, cudaGraphAddNode(&loop, top, nullptr, 0, &wp));
    cudaGraph_t body = wp.conditional.phGraph_out[0];
    cudaGraphNode_t prev = nullptr;
    for (int half = 0; half < 2; half++) {
        cudaGraphConditionalHandle run_pass;
        CUDA_OK(ctx, cudaGraphConditionalHandleCreate(&run_pass, body, 0, cudaGraphCondAssignDefault));
        GenStepParams gp = generate_step_params(ctx, family, streaming);
        gp.set_handles = true; gp.run_pass = run_pass; gp.keep_going = keep_going;
        cudaGraphNode_t step = nullptr, cond = nullptr;
        CUDA_OK(ctx, add_generate_step_node(body, prev ? &prev : nullptr, prev ? 1 : 0, gp, family, streaming, &step));
        cudaGraphNodeParams ip = {};
        ip.type = cudaGraphNodeTypeConditional;
        ip.conditional.handle = run_pass; ip.conditional.type = cudaGraphCondTypeIf; ip.conditional.size = 1;
        CUDA_OK(ctx, cudaGraphAddNode(&cond, body, &step, 1, &ip));
        if (!capture_generate_pass(ctx, ip.conditional.phGraph_out[0], p, gp.rows)) return false;
        std::swap(p.state_in, p.state_out);      // the second pass reads what the first one wrote
        prev = cond;
    }
    CUDA_OK(ctx, ctx->gen_graphs[ctx->phase][family][streaming].instantiate(top));
    return true;
}

bool ensure_generate_buffers(Context * ctx) {
    if (ctx->gen.in) return true;
    const int rows = ctx->batch_n ? ctx->batch_n : 1;
    const size_t V = (size_t) ctx->model->n_vocab, in_bytes = gen_u_offset(rows) + (size_t) rows * GENERATE_MAX * sizeof(double);
    const size_t out_bytes = gen_out_words(rows, GENERATE_MAX) * sizeof(uint32_t), table = (size_t) rows * V;
    Context::Generate g;
    CUDA_OK(ctx, g.in_host.alloc(in_bytes));
    CUDA_OK(ctx, g.out_host.alloc(out_bytes));
    CUDA_OK(ctx, g.out.alloc(out_bytes));
    CUDA_OK(ctx, g.counts.alloc(table * sizeof(float)));
    CUDA_OK(ctx, cudaMemsetAsync(g.counts, 0, table * sizeof(float), ctx->stream));
    CUDA_OK(ctx, g.bias_ids.alloc(table * sizeof(uint32_t)));
    CUDA_OK(ctx, g.bias_values.alloc(table * sizeof(float)));
    CUDA_OK(ctx, g.scratch.alloc(table * sizeof(float)));
    if (ctx->batch_n) CUDA_OK(ctx, g.park.alloc(table * sizeof(float)));
    CUDA_OK(ctx, g.in.alloc(in_bytes));
    ctx->gen = std::move(g);
    return true;
}

bool ensure_stream_buffers(Context * ctx) {
    if (ctx->streamed.words) return true;
    const int rows = ctx->batch_n ? ctx->batch_n : 1;
    Context::Streaming st;
    CUDA_OK(ctx, st.done.create(cudaEventDisableTiming));
    CUDA_OK(ctx, st.words.alloc_mapped((stream_token_offset(rows) + (size_t) rows * GENERATE_MAX) * sizeof(uint32_t)));
    ctx->streamed = std::move(st);
    return true;
}

// The request and output buffers of a logprob call whose outputs take `words` 32-bit words, and for a streaming one the ring.
bool ensure_logprob_buffers(Context * ctx, size_t words, bool streaming) {
    const int rows = ctx->batch_n ? ctx->batch_n : 1;
    if (!ctx->lp_req.dev) {
        Context::LogprobRequest r;
        CUDA_OK(ctx, r.host.alloc(sizeof(GenLogprobRequest)));
        CUDA_OK(ctx, r.dev.alloc(sizeof(GenLogprobRequest)));
        ctx->lp_req = std::move(r);
    }
    if (words > ctx->lp_out.words) {      // no graph holds these addresses: they travel in the request
        ctx->lp_out = {};
        Context::LogprobOut o;
        CUDA_OK(ctx, o.dev.alloc(words * sizeof(uint32_t)));
        CUDA_OK(ctx, o.host.alloc(words * sizeof(uint32_t)));
        o.words = words;
        ctx->lp_out = std::move(o);
    }
    if (streaming && !ctx->lp_ring) CUDA_OK(ctx, ctx->lp_ring.alloc_mapped((size_t) rows * 2 * GEN_LP_RECORD * sizeof(uint32_t)));
    return true;
}

// The sampler upload at its largest (GEN_BIAS_MAX entries per row), on the device and pinned.
bool ensure_sampler_buffers(Context * ctx) {
    if (ctx->smp.dev) return true;
    const size_t bytes = smp_bias_offset(ctx->batch_n ? ctx->batch_n : 1) + (size_t) (ctx->batch_n ? ctx->batch_n : 1) * GEN_BIAS_MAX * sizeof(GenBiasEntry);
    Context::Samplers smp;
    CUDA_OK(ctx, smp.host.alloc(bytes));
    CUDA_OK(ctx, smp.dev.alloc(bytes));
    ctx->smp = std::move(smp);
    return true;
}

// Entry at = b * n + j of the caller's logprob arrays <- words[w] of a record laid out as the ring's (GenLogprobRequest, ops.h).
void put_logprob_entry(const LogprobsOut & lp, size_t at, float logprob, float sample_prob, const uint32_t * ids, const float * top_lps) {
    lp.logprobs[at] = logprob;
    if (lp.sample_probs) lp.sample_probs[at] = sample_prob;
    for (size_t k = 0; k < lp.top_n; k++) { lp.top_ids[at * lp.top_n + k] = ids[k]; lp.top_logprobs[at * lp.top_n + k] = top_lps[k]; }
}

// The calling thread's side of a streaming loop that has been enqueued up to ctx->streamed.done: calls on_token for every token the
// step kernel publishes, in order per row, and acknowledges each one (the stop bit set when on_token returned nonzero), until the
// stream has passed the event and every published token is delivered. Busy-polls, yielding between empty sweeps. Returns false when
// a wait of the device for an acknowledgement ran out. With lp, token j's ring record goes to entry j of lp's arrays (`stride` entries per row) first.
bool stream_tokens(Context * ctx, TokenFn on_token, void * user, const LogprobsOut * lp, size_t stride) {
    const int rows = ctx->batch_n ? ctx->batch_n : 1;
    uint32_t * published = ctx->streamed.words, * acked = published + rows, * tokens = published + stream_token_offset(rows);
    std::vector<uint32_t> delivered((size_t) rows, 0);
    ctx->in_stream = true;
    for (bool done = false; !done;) {
        done = cudaEventQuery(ctx->streamed.done) != cudaErrorNotReady;      // before the sweep, so that the last sweep sees every token
        bool any = false;
        for (int b = 0; b < rows; b++) {
            const uint32_t n = __atomic_load_n(published + b, __ATOMIC_ACQUIRE);
            for (uint32_t j = delivered[b]; j < n; j++) {
                const uint32_t tok = __atomic_load_n(tokens + (size_t) b * GENERATE_MAX + j, __ATOMIC_RELAXED);
                if (lp) {
                    uint32_t rec[GEN_LP_RECORD];
                    const uint32_t * src = ctx->lp_ring + ((size_t) b * 2 + (j & 1u)) * GEN_LP_RECORD;
                    for (int w = 0; w < GEN_LP_RECORD; w++) rec[w] = __atomic_load_n(src + w, __ATOMIC_RELAXED);
                    float f[2 + GEN_TOP_MAX];
                    memcpy(f, rec, 2 * sizeof(float));
                    memcpy(f + 2, rec + 2 + GEN_TOP_MAX, GEN_TOP_MAX * sizeof(float));
                    put_logprob_entry(*lp, (size_t) b * stride + j, f[0], f[1], rec + 2, f + 2);
                }
                const uint32_t stop = on_token(user, (size_t) b, j, tok) != 0 ? 1u : 0u;
                __atomic_store_n(acked + b, 2 * (j + 1) + stop, __ATOMIC_RELEASE);
                any = true;
            }
            delivered[b] = std::max(delivered[b], n);
        }
        if (!any && !done) std::this_thread::yield();
    }
    ctx->in_stream = false;
    return __atomic_load_n(published + 2 * rows, __ATOMIC_ACQUIRE) == 0;
}

}  // namespace

void drop_generate_graphs(Context * ctx) {
    for (auto & by_phase : ctx->gen_graphs)
        for (auto & by_family : by_phase)
            for (auto & e : by_family) e.reset();
    for (auto & e : ctx->beam_graphs) e.reset();
}

// The captured passes hold the adapters, the trace buffer and the activation buffers of the time they were captured.
void drop_all_graphs(Context * ctx) {
    for (auto & g : ctx->graphs) g = Context::GraphSlot();
    drop_generate_graphs(ctx);
}

namespace {

// The scratch of the deltas (Context::lora), allocated once for passes of up to MAX_TOKENS_PER_PASS columns.
bool ensure_lora_scratch(Context * ctx) {
    if (ctx->lora.u) return true;
    const Dims d = model_dims(*ctx->model);
    const LoraScratchSize s = lora_scratch_floats(d.C, d.F);
    Context::LoraScratch l;
    cudaError_t e = l.u.alloc(s.u * sizeof(float));
    if (e == cudaSuccess) e = l.z.alloc(s.z * sizeof(float));
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, false, e == cudaSuccess, "Failed to allocate the adapter's scratch: %s", cudaGetErrorString(e));
    ctx->lora = std::move(l);
    return true;
}

}  // namespace

bool set_adapter(Context * ctx, const Adapter * a) {
    if (a == ctx->adapter) return true;
    const Model & m = *ctx->model;
    CUDA_OK(ctx, cudaSetDevice(m.dev.device));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    if (a && !ensure_lora_scratch(ctx)) return false;
    drop_all_graphs(ctx);
    if (a) a->attached.fetch_add(1);
    if (ctx->adapter) ctx->adapter->attached.fetch_sub(1);
    ctx->adapter = a;
    return true;
}

bool batch_set_adapter(Context * ctx, int seq, const Adapter * a) {
    const Adapter * old = ctx->seq_adapter.empty() ? nullptr : ctx->seq_adapter[seq];
    if (a == old) return true;
    std::vector<const Adapter *> next = ctx->seq_adapter.empty() ? std::vector<const Adapter *>(ctx->batch_n, nullptr) : ctx->seq_adapter;
    next[seq] = a;
    std::vector<const Adapter *> distinct;
    std::vector<int> slot(ctx->batch_n, -1);
    for (int b = 0; b < ctx->batch_n; b++) {
        if (!next[b]) continue;
        const auto it = std::find(distinct.begin(), distinct.end(), next[b]);
        slot[b] = (int) (it - distinct.begin());
        if (it == distinct.end()) distinct.push_back(next[b]);
    }
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, distinct.size() <= (size_t) LORA_MAX_ADAPTERS,
               "A batch context carries at most %d distinct adapters on its sequences", LORA_MAX_ADAPTERS);
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    if (a && !ensure_lora_scratch(ctx)) return false;
    drop_all_graphs(ctx);
    if (a) a->attached.fetch_add(1);
    if (old) old->attached.fetch_sub(1);
    ctx->seq_adapter = std::move(next);
    ctx->seq_adapters = std::move(distinct);
    ctx->seq_slot = std::move(slot);
    return true;
}

bool check_logprobs(ErrorSink sink, size_t n_vocab, const LogprobsOut * lp) {
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, lp && lp->logprobs, "NULL logprob request or logprobs array");
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, lp->top_n <= (size_t) GEN_TOP_MAX && lp->top_n <= n_vocab, "top_n (%zu) must be at most %d and n_vocab",
               lp->top_n, GEN_TOP_MAX);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, lp->top_n == 0 || (lp->top_ids && lp->top_logprobs), "NULL top_ids or top_logprobs with top_n > 0");
    return true;
}

bool check_samplers(ErrorSink sink, size_t n_rows, size_t n_vocab, const SamplerIn * samplers) {
    std::vector<uint32_t> seen;       // seen[id] = 1 + the last row that listed id
    for (size_t b = 0; b < n_rows; b++) {
        const SamplerIn & s = samplers[b];
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, s.top_k <= n_vocab, "top_k of row %zu (%u) is above n_vocab", b, s.top_k);
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, s.min_p >= 0.0f && s.min_p <= 1.0f, "min_p of row %zu must be in [0, 1]", b);
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, s.n_bias <= (size_t) GEN_BIAS_MAX && (s.n_bias == 0 || (s.bias_ids && s.bias_values)),
                   "Row %zu: at most %d bias entries, with ids and values not NULL", b, GEN_BIAS_MAX);
        if (s.n_bias && seen.empty()) seen.assign(n_vocab, 0);
        for (size_t k = 0; k < s.n_bias; k++) {
            const uint32_t id = s.bias_ids[k];
            const float v = s.bias_values[k];
            RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, id < n_vocab, "Bias id %u of row %zu is out of range", id, b);
            RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, seen[id] != b + 1, "Bias id %u of row %zu is listed twice", id, b);
            RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, !std::isnan(v) && v != INFINITY, "Bias value of id %u of row %zu must be finite or -inf", id, b);
            seen[id] = (uint32_t) b + 1;
        }
    }
    return true;
}

bool check_automaton_table(ErrorSink sink, const uint16_t * next, size_t n_states, size_t n_vocab) {
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, next && n_states >= 1 && n_states <= 65535, "An automaton needs a table and 1 .. 65535 states");
    for (size_t i = 0, n = n_states * n_vocab; i < n; i++)
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, next[i] < n_states || next[i] == GEN_MASK_DEAD, "Transition %zu of state %zu (%u) is neither a state nor dead",
                   i % n_vocab, i / n_vocab, (unsigned) next[i]);
    return true;
}

void automaton_live(const uint16_t * next, size_t n_states, size_t n_vocab, uint8_t * live) {
    for (size_t s = 0; s < n_states; s++) {
        const uint16_t * row = next + s * n_vocab;
        live[s] = std::any_of(row, row + n_vocab, [](uint16_t t) { return t != GEN_MASK_DEAD; }) ? 1 : 0;
    }
}

Automaton * create_automaton(const Model * model, const uint16_t * next, size_t n_states, ErrorSink sink) {
    const size_t V = (size_t) model->n_vocab;
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, next && n_states >= 1 && n_states <= 65535, "An automaton needs a table and 1 .. 65535 states");
    // a device table is checked from a host copy; nothing is allocated before the checks pass
    std::vector<uint16_t> staged;
    const uint16_t * host = next;
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, next) == cudaSuccess && (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged)) {
        staged.resize(n_states * V);
        RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, nullptr, cudaMemcpy(staged.data(), next, staged.size() * sizeof(uint16_t), cudaMemcpyDefault) == cudaSuccess,
                   "Reading the automaton's device table failed");
        host = staged.data();
    }
    cudaGetLastError();     // a host pointer unknown to CUDA is not an error
    if (!check_automaton_table(sink, host, n_states, V)) return nullptr;
    std::vector<uint8_t> live(n_states);
    automaton_live(host, n_states, V, live.data());
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, nullptr, cudaSetDevice(model->dev.device) == cudaSuccess, "Cannot select the model's device");
    Automaton * a = new Automaton;
    a->model = model; a->device = model->dev.device; a->n_vocab = V; a->n_states = (uint32_t) n_states;
    const bool ok = a->next.alloc(n_states * V * sizeof(uint16_t)) == cudaSuccess && a->live.alloc(n_states) == cudaSuccess &&
                    cudaMemcpy(a->next, next, n_states * V * sizeof(uint16_t), cudaMemcpyDefault) == cudaSuccess &&
                    cudaMemcpy(a->live, live.data(), n_states, cudaMemcpyHostToDevice) == cudaSuccess;
    if (!ok) {
        const cudaError_t e = cudaGetLastError();
        destroy_automaton(a);
        RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, nullptr, false, "Uploading the automaton failed: %s", cudaGetErrorString(e));
    }
    return a;
}

void destroy_automaton(Automaton * a) {
    if (!a) return;
    cudaSetDevice(a->device);
    delete a;
}

bool check_generate_rows(ErrorSink sink, size_t n_rows, size_t n_vocab, const uint32_t * max_tokens, const float * temperature, const float * top_p,
                         const float * presence, const float * frequency, const double * u, const uint32_t * stop_ids, size_t n_stop,
                         const void * tokens_out, const void * n_generated) {
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, max_tokens && temperature && top_p && presence && frequency && u && tokens_out && n_generated,
               "NULL max_tokens, temperature, top_p, penalty, u, tokens_out or n_generated");
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, n_stop <= (size_t) GENERATE_MAX_STOP && (n_stop == 0 || stop_ids), "At most %d stop ids, not NULL", GENERATE_MAX_STOP);
    for (size_t k = 0; k < n_stop; k++)
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, stop_ids[k] < n_vocab, "Stop id %u is out of range", stop_ids[k]);
    size_t n = 0;
    for (size_t b = 0; b < n_rows; b++) {
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, max_tokens[b] <= (uint32_t) GENERATE_MAX, "max_tokens of row %zu is above %d", b, GENERATE_MAX);
        n = std::max(n, (size_t) max_tokens[b]);
    }
    for (size_t b = 0; b < n_rows; b++) {     // sampling.py:20-23, as check_sample_rows checks a row
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, temperature[b] >= 0.0f, "temperature of row %zu must be >= 0", b);
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, top_p[b] >= 0.0f && top_p[b] <= 1.0f, "top_p of row %zu must be in [0, 1]", b);
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, std::isfinite(presence[b]) && std::isfinite(frequency[b]), "penalties of row %zu must be finite", b);
        for (size_t i = 0; i < max_tokens[b]; i++)
            RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, u[b * n + i] >= 0.0 && u[b * n + i] < 1.0, "u[%zu][%zu] must be in [0, 1)", b, i);
    }
    return true;
}

bool generate(Context * ctx, const uint32_t * max_tokens, const float * temperature, const float * top_p, const float * presence,
              const float * frequency, const uint8_t * keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop,
              uint32_t * tokens_out, uint32_t * n_generated, TokenFn on_token, void * user, const Automaton * const * automata,
              uint32_t * automaton_states, const LogprobsOut * lp, const SamplerIn * samplers) {
    const Model & m = *ctx->model;
    const int rows = ctx->batch_n ? ctx->batch_n : 1;
    const size_t V = (size_t) m.n_vocab;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, !ctx->group && m.layer_begin == 0 && m.layer_end == m.n_layer,
               "Generation runs on a whole-model context or batch context, not on a pipeline or one of its stages");
    if (!check_generate_rows(ctx->sink(), rows, V, max_tokens, temperature, top_p, presence, frequency, u, stop_ids, n_stop, tokens_out, n_generated)) return false;
    const bool constrained = automata != nullptr;
    if (constrained) {
        RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, automaton_states, "NULL automaton states");
        for (int b = 0; b < rows; b++) {
            if (!automata[b]) continue;
            RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, automata[b]->model == ctx->model && automata[b]->n_vocab == V,
                       "The automaton of sequence %d was created for another model", b);
            RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, automaton_states[b] < automata[b]->n_states, "Automaton state %u of sequence %d is not below %u",
                       automaton_states[b], b, automata[b]->n_states);
        }
    }
    if (lp && !check_logprobs(ctx->sink(), V, lp)) return false;
    if (samplers && !check_samplers(ctx->sink(), rows, V, samplers)) return false;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, V <= 65536, "On-device sampling supports n_vocab <= 65536");
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, ctx->logits_valid, "No logits to sample from: the last evaluation skipped the head");
    int driver = 0;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, cudaDriverGetVersion(&driver) == cudaSuccess && driver >= 12040,
               "Device-side generation needs conditional graph nodes: a CUDA driver of 12.4 or newer (found %d)", driver);
    size_t n = 0;
    for (int b = 0; b < rows; b++) n = std::max(n, (size_t) max_tokens[b]);
    CUDA_OK(ctx, cudaSetDevice(m.dev.device));
    const bool streaming = on_token != nullptr;
    if (!ensure_generate_buffers(ctx) || (streaming && !ensure_stream_buffers(ctx)) || !ensure_capacity(ctx, rows, ctx->stream)) return false;
    const size_t lp_cells = (size_t) rows * n, lp_words = lp ? lp_cells * (2 + 2 * lp->top_n) : 0;
    if (lp && !ensure_logprob_buffers(ctx, lp_words, streaming)) return false;
    if (samplers && !ensure_sampler_buffers(ctx)) return false;
    // the call's parameters, loop state and u in one upload (every call ends with a synchronisation, so the pinned buffer is free)
    GenShared * sh = reinterpret_cast<GenShared *>(ctx->gen.in_host.get());
    memset(sh, 0, sizeof(GenShared));
    for (size_t k = 0; k < n_stop; k++) sh->stop[k] = stop_ids[k];
    sh->n_stop = (uint32_t) n_stop; sh->stride = (uint32_t) n;
    sh->weights = ctx->pen_weights.set ? ctx->pen_weights.table.get() : nullptr;
    GenRow * gr = reinterpret_cast<GenRow *>(ctx->gen.in_host + sizeof(GenShared));
    for (int b = 0; b < rows; b++) gr[b] = GenRow{temperature[b], top_p[b], presence[b], frequency[b], max_tokens[b], 0, 0, ctx->penalty_decay[b]};
    GenMaskRow * mr = reinterpret_cast<GenMaskRow *>(ctx->gen.in_host + gen_mask_offset(rows));
    for (int b = 0; b < rows; b++)
        mr[b] = constrained && automata[b] ? GenMaskRow{automata[b]->next, automata[b]->live, automaton_states[b], 0} : GenMaskRow{nullptr, nullptr, 0, 0};
    const size_t u_off = gen_u_offset(rows);
    memcpy(ctx->gen.in_host + u_off, u, (size_t) rows * n * sizeof(double));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->gen.in, ctx->gen.in_host, u_off + (size_t) rows * n * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    for (int b = 0; b < rows;) {      // counts of the rows that start from zero (runs of them are contiguous)
        if (keep_counts && keep_counts[b]) { b++; continue; }
        int e = b;
        while (e < rows && !(keep_counts && keep_counts[e])) e++;
        CUDA_OK(ctx, cudaMemsetAsync(ctx->gen.counts + (size_t) b * V, 0, (size_t) (e - b) * V * sizeof(float), ctx->stream));
        b = e;
    }
    const size_t out_words = gen_out_words(rows, n);
    CUDA_OK(ctx, cudaMemsetAsync(ctx->gen.out, 0, out_words * sizeof(uint32_t), ctx->stream));
    if (streaming) memset(ctx->streamed.words, 0, stream_token_offset(rows) * sizeof(uint32_t));     // published, acked, timed_out
    if (lp) {
        float * f = reinterpret_cast<float *>(ctx->lp_out.dev.get());
        *ctx->lp_req.host = GenLogprobRequest{(uint32_t) lp->top_n, 0, f, f + lp_cells, ctx->lp_out.dev + 2 * lp_cells, f + 2 * lp_cells + lp_cells * lp->top_n,
                                              streaming ? ctx->lp_ring.device() : nullptr};
        CUDA_OK(ctx, cudaMemcpyAsync(ctx->lp_req.dev, ctx->lp_req.host, sizeof(GenLogprobRequest), cudaMemcpyHostToDevice, ctx->stream));
    }
    if (samplers) {     // the request word, the rows and the bias pool in one upload
        *reinterpret_cast<const GenLogprobRequest **>(ctx->smp.host.get()) = lp ? ctx->lp_req.dev.get() : nullptr;
        GenSamplerRow * sr = reinterpret_cast<GenSamplerRow *>(ctx->smp.host + smp_rows_offset());
        GenBiasEntry * pool = reinterpret_cast<GenBiasEntry *>(ctx->smp.host + smp_bias_offset(rows));
        uint32_t used = 0;
        for (int b = 0; b < rows; b++) {
            const SamplerIn & s = samplers[b];
            sr[b] = GenSamplerRow{s.top_k, s.min_p, used, used + (uint32_t) s.n_bias};
            for (size_t k = 0; k < s.n_bias; k++) pool[used++] = GenBiasEntry{s.bias_ids[k], s.bias_values[k]};
        }
        CUDA_OK(ctx, cudaMemcpyAsync(ctx->smp.dev, ctx->smp.host, smp_bias_offset(rows) + used * sizeof(GenBiasEntry), cudaMemcpyHostToDevice, ctx->stream));
    }
    const GenFamily family = samplers ? GEN_SAMPLED : lp ? GEN_LOGPROBS : constrained ? GEN_CONSTRAINED : GEN_PLAIN;
    GraphExec & graph = ctx->gen_graphs[ctx->phase][family][streaming];
    if (!graph && !build_generate_graph(ctx, family, streaming)) return false;
    CUDA_OK(ctx, cudaGraphLaunch(graph, ctx->stream));
    g_graph_launches++;
    if (ctx->batch_n) CUDA_OK(ctx, cudaMemcpyAsync(ctx->logits, ctx->gen.park, (size_t) rows * V * sizeof(float), cudaMemcpyDeviceToDevice, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->gen.out_host, ctx->gen.out, out_words * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    if (lp_words) CUDA_OK(ctx, cudaMemcpyAsync(ctx->lp_out.host, ctx->lp_out.dev, lp_words * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    bool in_time = true;
    if (streaming) {
        CUDA_OK(ctx, cudaEventRecord(ctx->streamed.done, ctx->stream));
        in_time = stream_tokens(ctx, on_token, user, lp, n);
    }
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    const uint32_t * res = ctx->gen.out_host;
    memcpy(n_generated, res, (size_t) rows * sizeof(uint32_t));
    memcpy(tokens_out, res + gen_tokens_word(rows), (size_t) rows * n * sizeof(uint32_t));
    for (int b = 0; constrained && b < rows; b++)
        if (automata[b]) automaton_states[b] = res[rows + 1 + b];
    if (lp) {       // drawn entries from the device, the rest NaN / SCORE_NO_TARGET
        const float * f = reinterpret_cast<const float *>(ctx->lp_out.host.get());
        const std::vector<uint32_t> none(lp->top_n, SCORE_NO_TARGET);
        const std::vector<float> nans(lp->top_n, NAN);
        for (int b = 0; b < rows; b++)
            for (size_t i = 0; i < n; i++) {
                const size_t at = (size_t) b * n + i, k = lp->top_n;
                if (i < res[b]) put_logprob_entry(*lp, at, f[at], f[lp_cells + at], ctx->lp_out.host + 2 * lp_cells + at * k, f + 2 * lp_cells + lp_cells * k + at * k);
                else put_logprob_entry(*lp, at, NAN, NAN, none.data(), nans.data());
            }
    }
    if (res[rows] & 1u) {      // an odd number of passes leaves the state in state_b
        std::swap(ctx->state_a, ctx->state_b);
        ctx->phase ^= 1;
    }
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX, false, in_time, "A token callback kept the device waiting for more than %d ms; its sequence was ended there",
               STREAM_TIMEOUT_MS);
    return true;
}

bool read_penalty_table(ErrorSink sink, const float * p, size_t n, int device, std::vector<float> & host, const char * what) {
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, p, "NULL %s", what);
    int dev = -1;
    const bool in_hbm = on_device(p, &dev);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, !in_hbm || dev == device, "The %s are in the memory of device %d, not of the context's device %d", what, dev, device);
    host.resize(n);
    if (in_hbm) RWKV_CHECK(sink, RWKV_ERROR_CTX, false, cudaMemcpy(host.data(), p, n * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess,
                           "Reading the %s failed", what);
    else memcpy(host.data(), p, n * sizeof(float));
    for (size_t i = 0; i < n; i++)
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, std::isfinite(host[i]) && host[i] >= 0.0f, "The %s must be finite and >= 0 (entry %zu is %g)", what, i, host[i]);
    return true;
}

bool set_penalty_weights(Context * ctx, const float * weights) {
    if (!weights) { ctx->pen_weights.set = false; return true; }
    const size_t V = (size_t) ctx->model->n_vocab;
    std::vector<float> host;
    if (!read_penalty_table(ctx->sink(), weights, V, ctx->model->dev.device, host, "penalty weights")) return false;
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    if (!ctx->pen_weights.table) CUDA_OK(ctx, ctx->pen_weights.table.alloc(V * sizeof(float)));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->pen_weights.table, host.data(), V * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->pen_weights.set = true;
    return true;
}

bool get_penalty_counts(Context * ctx, int seq, float * counts_out) {
    const size_t V = (size_t) ctx->model->n_vocab;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, counts_out, "NULL counts_out");
    int dev = -1;
    const bool in_hbm = on_device(counts_out, &dev);
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, !in_hbm || dev == ctx->model->dev.device, "counts_out is in the memory of device %d, not of the context's device %d",
               dev, ctx->model->dev.device);
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    if (ctx->gen.counts) CUDA_OK(ctx, cudaMemcpyAsync(counts_out, ctx->gen.counts + (size_t) seq * V, V * sizeof(float), cudaMemcpyDefault, ctx->stream));
    else if (in_hbm) CUDA_OK(ctx, cudaMemsetAsync(counts_out, 0, V * sizeof(float), ctx->stream));      // never generated: zeros, nothing allocated
    else memset(counts_out, 0, V * sizeof(float));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return true;
}

bool set_penalty_counts(Context * ctx, int seq, const float * counts_in) {
    const size_t V = (size_t) ctx->model->n_vocab;
    std::vector<float> host;
    if (!read_penalty_table(ctx->sink(), counts_in, V, ctx->model->dev.device, host, "penalty counts")) return false;
    CUDA_OK(ctx, cudaSetDevice(ctx->model->dev.device));
    if (!ensure_generate_buffers(ctx)) return false;
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->gen.counts + (size_t) seq * V, host.data(), V * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return true;
}

// Beam search: WHILE keep_going { beam step -> IF run_pass { gather ; pass } }, one pass per body, then (several groups) the restore
// of the slots that groups which stopped keep. Y = state_a holds the current slots: the gather copies each live slot's parent from Y
// into X = state_b and the pass evaluates X into Y, so the current state stays in state_a and the phase does not change. The graph is
// keyed by the phase at entry, which decides which buffer is state_a, and by the number of groups.
namespace {

bool ensure_beam_buffers(Context * ctx, size_t groups, size_t max_tokens) {
    const size_t N = (size_t) ctx->batch_n;
    if (!ctx->beam_park) CUDA_OK(ctx, ctx->beam_park.alloc(N * (size_t) ctx->model->n_vocab * sizeof(float)));
    if (groups <= ctx->beam.groups && max_tokens <= ctx->beam.capacity) return true;
    groups = std::max(groups, ctx->beam.groups);
    max_tokens = std::max(max_tokens, ctx->beam.capacity);
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    for (auto & e : ctx->beam_graphs) e.reset();
    ctx->beam = {};
    const size_t state_bytes = sizeof(BeamLoop) + groups * sizeof(BeamState), back_bytes = max_tokens * N * 2 * sizeof(uint32_t);
    Context::Beam b;
    CUDA_OK(ctx, b.loop.alloc(state_bytes));
    CUDA_OK(ctx, b.back.alloc(back_bytes));
    CUDA_OK(ctx, b.host.alloc(state_bytes + back_bytes));
    b.groups = groups; b.capacity = max_tokens;
    ctx->beam = std::move(b);
    return true;
}

bool build_beam_graph(Context * ctx, int groups) {
    const int N = ctx->batch_n, W = N / groups;
    Pass p;
    if (!make_pass(ctx, N, true, nullptr, p)) return false;
    p.tokens_in_place = true;
    {   // one uncaptured pass of the loop's shape first, as build_generate_graph runs one: Y -> X with its logits set aside
        CUDA_OK(ctx, cudaMemsetAsync(ctx->act.tokens, 0, (size_t) N * sizeof(int), p.stream));
        Pass warm = p;
        warm.logits = ctx->beam_park;
        if (!enqueue_pass(ctx, warm, 0)) return false;
    }
    p.state_in = ctx->state_b; p.state_out = ctx->state_a;
    Graph top;
    CUDA_OK(ctx, top.create());
    cudaGraphConditionalHandle keep_going, run_pass;
    CUDA_OK(ctx, cudaGraphConditionalHandleCreate(&keep_going, top, 1, cudaGraphCondAssignDefault));
    cudaGraphNodeParams wp = {};
    wp.type = cudaGraphNodeTypeConditional;
    wp.conditional.handle = keep_going; wp.conditional.type = cudaGraphCondTypeWhile; wp.conditional.size = 1;
    cudaGraphNode_t loop = nullptr, step = nullptr, cond = nullptr, restore = nullptr;
    CUDA_OK(ctx, cudaGraphAddNode(&loop, top, nullptr, 0, &wp));
    cudaGraph_t body = wp.conditional.phGraph_out[0];
    CUDA_OK(ctx, cudaGraphConditionalHandleCreate(&run_pass, body, 0, cudaGraphCondAssignDefault));
    const BeamStepParams bp{ctx->logits, ctx->model->n_vocab, W, groups, ctx->beam.loop, ctx->beam.states(), ctx->beam.back, ctx->act.tokens, true,
                            run_pass, keep_going};
    CUDA_OK(ctx, add_beam_step_node(body, nullptr, 0, bp, &step));
    const BeamCopyParams cp{ctx->beam.loop, ctx->beam.states(), W, groups, ctx->model->n_vocab, p.state_out, p.state_in, ctx->batch_stride,
                            ctx->model->state_len(), ctx->logits, ctx->beam_park};
    if (groups > 1) CUDA_OK(ctx, add_beam_restore_node(top, &loop, 1, cp, &restore));     // one group stops only when the loop does
    cudaGraphNodeParams ip = {};
    ip.type = cudaGraphNodeTypeConditional;
    ip.conditional.handle = run_pass; ip.conditional.type = cudaGraphCondTypeIf; ip.conditional.size = 1;
    CUDA_OK(ctx, cudaGraphAddNode(&cond, body, &step, 1, &ip));
    CUDA_OK(ctx, cudaStreamBeginCaptureToGraph(p.stream, ip.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
    cudaError_t e = launch_beam_gather(cp, p.stream);
    const bool ok = e == cudaSuccess && enqueue_pass(ctx, p, 0);
    cudaGraph_t out = nullptr;
    const cudaError_t ec = cudaStreamEndCapture(p.stream, &out);
    if (e == cudaSuccess) e = ec;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, ok && e == cudaSuccess, "Capturing the beam search pass failed: %s", cudaGetErrorString(e));
    CUDA_OK(ctx, ctx->beam_graphs[ctx->phase].instantiate(top));
    ctx->beam_graph_groups[ctx->phase] = groups;
    return true;
}

struct BeamResult {
    double score, norm;
    bool finished;
    std::vector<uint32_t> tokens;
};

}  // namespace

bool beam_search(Context * ctx, int n_groups, const uint32_t * max_tokens, const float * length_penalty, const uint32_t * stop_ids, size_t n_stop,
                 size_t n_best, uint32_t * tokens_out, uint32_t * lengths_out, double * scores_out, uint8_t * finished_out) {
    const Model & m = *ctx->model;
    const int N = ctx->batch_n, W = N / n_groups;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, m.n_vocab <= 65536, "Beam search supports n_vocab <= 65536");
    int driver = 0;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, cudaDriverGetVersion(&driver) == cudaSuccess && driver >= 12040,
               "Beam search needs conditional graph nodes: a CUDA driver of 12.4 or newer (found %d)", driver);
    size_t n = 0;
    for (int g = 0; g < n_groups; g++) n = std::max(n, (size_t) max_tokens[g]);
    CUDA_OK(ctx, cudaSetDevice(m.dev.device));
    if (!ensure_beam_buffers(ctx, (size_t) n_groups, n) || !ensure_capacity(ctx, N, ctx->stream)) return false;
    BeamLoop * hl = reinterpret_cast<BeamLoop *>(ctx->beam.host.get());
    BeamState * hs = reinterpret_cast<BeamState *>(hl + 1);
    memset(hl, 0, sizeof(BeamLoop) + (size_t) n_groups * sizeof(BeamState));
    for (int g = 0; g < n_groups; g++) {
        BeamState & st = hs[g];
        for (size_t k = 0; k < n_stop; k++) st.stop[k] = stop_ids[k];
        st.n_stop = (uint32_t) n_stop; st.width = (uint32_t) W; st.max_tokens = max_tokens[g];
        if (max_tokens[g] > 0) {
            st.n_live = 1;      // the root: sequence g*W, score 0
            hl->n_active++;
        } else {
            st.n_keep = (uint32_t) W; st.park_at = 1;     // never runs: every slot is kept from the first pass on
        }
    }
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->beam.loop, hl, sizeof(BeamLoop) + (size_t) n_groups * sizeof(BeamState), cudaMemcpyHostToDevice, ctx->stream));
    // a group that never runs takes no token; its slots still run in the passes, on token 0
    if (n_groups > 1) CUDA_OK(ctx, cudaMemsetAsync(ctx->act.tokens, 0, (size_t) N * sizeof(int), ctx->stream));
    GraphExec & graph = ctx->beam_graphs[ctx->phase];
    if (ctx->beam_graph_groups[ctx->phase] != n_groups) graph.reset();
    if (!graph && !build_beam_graph(ctx, n_groups)) return false;
    CUDA_OK(ctx, cudaGraphLaunch(graph, ctx->stream));
    g_graph_launches++;
    uint32_t * back = reinterpret_cast<uint32_t *>(hs + n_groups);
    CUDA_OK(ctx, cudaMemcpyAsync(hl, ctx->beam.loop, sizeof(BeamLoop) + (size_t) n_groups * sizeof(BeamState), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(back, ctx->beam.back, n * N * 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    memset(tokens_out, 0, (size_t) n_groups * n_best * n * sizeof(uint32_t));
    for (int g = 0; g < n_groups; g++) {
        const BeamState & st = hs[g];
        // the tokens of the beam in slot k of group g after step i, from the back-pointers
        auto history = [&](int64_t i, uint32_t k) {
            std::vector<uint32_t> t((size_t) (i + 1));
            for (; i >= 0; i--) {
                const uint32_t * e = back + ((size_t) i * N + (size_t) g * W + k) * 2;
                t[(size_t) i] = e[1];
                k = e[0];
            }
            return t;
        };
        std::vector<BeamResult> res;
        for (uint32_t q = 0; q < st.n_pool; q++) {
            const BeamHyp & h = st.pool[q];
            BeamResult r{h.score, 0.0, true, history((int64_t) h.step - 1, h.parent)};
            r.tokens.push_back(h.token);
            res.push_back(std::move(r));
        }
        for (uint32_t k = 0; k < st.n_live; k++) res.push_back(BeamResult{st.score[k], 0.0, false, history((int64_t) st.step - 1, k)});
        for (BeamResult & r : res) r.norm = r.score / std::pow((double) r.tokens.size(), (double) length_penalty[g]);
        std::stable_sort(res.begin(), res.end(), [](const BeamResult & a, const BeamResult & b) { return a.norm > b.norm; });
        for (size_t r = 0; r < n_best; r++) {
            const size_t row = (size_t) g * n_best + r;
            const bool have = r < res.size();
            if (have) std::copy(res[r].tokens.begin(), res[r].tokens.end(), tokens_out + row * n);
            lengths_out[row] = have ? (uint32_t) res[r].tokens.size() : 0;
            scores_out[row] = have ? res[r].score : -INFINITY;
            if (finished_out) finished_out[row] = have && res[r].finished ? 1 : 0;
        }
    }
    return true;
}

bool pipe_ensure_box(Context * ctx) {
    Model & m = *ctx->model;
    if (m.link.box) return true;      // a link without a box has no neighbours yet: the connect calls make the box first
    CUDA_OK(ctx, cudaSetDevice(m.dev.device));
    PipeLink link;
    link.slot_floats = stage_hidden_len(m, (size_t) MAX_TOKENS_PER_PASS);
    link.bytes = sizeof(PipeBox) + (size_t) PIPE_SLOTS * link.slot_floats * sizeof(float);
    CUDA_OK(ctx, link.box.alloc(link.bytes));
    CUDA_OK(ctx, cudaMemset(link.box, 0, sizeof(PipeBox)));
    CUDA_OK(ctx, link.counters.alloc(8 * sizeof(unsigned long long)));
    CUDA_OK(ctx, cudaMemset(link.counters, 0, 8 * sizeof(unsigned long long)));
    CUDA_OK(ctx, cudaDeviceSynchronize());
    m.link = std::move(link);
    return true;
}

bool pipe_forward(Context * ctx, const uint32_t * tokens, size_t T, bool want_logits, cudaStream_t stream) {
    Model & m = *ctx->model;
    const bool first = m.layer_begin == 0, last = m.layer_end == m.n_layer;
    RWKV_CHECK(ctx->sink(), RWKV_ERROR_ARGS, false, m.link.box && (first || m.link.prev) && (last || m.link.next), "The stage is not connected to its neighbours");
    CUDA_OK(ctx, cudaSetDevice(m.dev.device));
    Pass p;
    if (!make_pass(ctx, (int) T, want_logits && last, stream, p) || !begin_pass(ctx, tokens, p)) return false;
    const size_t n = (size_t) m.n_embed * T, nv = m.arch_major == 7 ? n : 0;
    cudaError_t e = cudaSuccess;
    if (!first) e = launch_pipe_recv(m.link.box, m.link.prev, m.link.counters, m.link.slot_floats, p.s.x, n, p.s.v_first, nv, p.stream);
    bool ok = e == cudaSuccess && run_layers(ctx, p, 0);
    if (ok && !last) e = launch_pipe_send(m.link.box, m.link.next, m.link.counters, m.link.slot_floats, p.s.x, n, p.s.v_first, nv, p.stream);
    ok = ok && e == cudaSuccess && end_pass(ctx, p);
    if (e != cudaSuccess) { ctx->last_error |= RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED; if (ctx->print_errors) fprintf(stderr, "pipeline hand-off launch failed: %s\n", cudaGetErrorString(e)); }
    return ok;
}

// ---- in-process pipeline behind rwkv.h ---------------------------------------------------------------------------
namespace {

// contiguous min-max partition of n_layer layers over `world` stages, the last one carrying `head_layers` extra (pipeline.py:
// stage_layers_balanced is the same recurrence)
std::vector<int> balanced_cuts(int n_layer, int world, double head_layers) {
    const double INF = 1e300;
    std::vector<std::vector<double>> best((size_t) world, std::vector<double>((size_t) n_layer + 1, INF));
    std::vector<std::vector<int>> cut((size_t) world, std::vector<int>((size_t) n_layer + 1, 0));
    auto cost = [&](int st, int a, int b) { return (double) (b - a) + (st == world - 1 ? head_layers : 0.0); };
    for (int e = 1; e <= n_layer; e++) best[0][(size_t) e] = cost(0, 0, e);
    for (int st = 1; st < world; st++)
        for (int e = st + 1; e <= n_layer; e++)
            for (int a = st; a < e; a++) {
                const double v = std::max(best[(size_t) st - 1][(size_t) a], cost(st, a, e));
                if (v < best[(size_t) st][(size_t) e] - 1e-12) { best[(size_t) st][(size_t) e] = v; cut[(size_t) st][(size_t) e] = a; }
            }
    std::vector<int> bounds((size_t) world + 1, 0);
    bounds[(size_t) world] = n_layer;
    for (int st = world - 1, e = n_layer; st >= 1; st--) { e = cut[(size_t) st][(size_t) e]; bounds[(size_t) st] = e; }
    return bounds;
}

Context * stage_of(Context * head, size_t r) { return r == 0 ? head : head->stages[r - 1]; }

bool connect_stages(Context * head, ErrorSink sink) {
    const size_t n = head->stages.size() + 1;
    for (size_t r = 0; r < n; r++) if (!pipe_ensure_box(stage_of(head, r))) return false;
    for (size_t r = 0; r < n; r++) {
        Model & m = *stage_of(head, r)->model;
        for (int dir = 0; dir < 2; dir++) {
            if ((dir == 0 && r == 0) || (dir == 1 && r + 1 == n)) continue;
            Model & o = *stage_of(head, dir == 0 ? r - 1 : r + 1)->model;
            if (o.dev.device != m.dev.device) {
                int can = 0;
                cudaDeviceCanAccessPeer(&can, m.dev.device, o.dev.device);
                RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, can, "Device %d cannot access device %d's memory", m.dev.device, o.dev.device);
                cudaSetDevice(m.dev.device);
                const cudaError_t e = cudaDeviceEnablePeerAccess(o.dev.device, 0);
                if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
                else RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, e == cudaSuccess, "cudaDeviceEnablePeerAccess failed: %s", cudaGetErrorString(e));
            }
            (dir == 0 ? m.link.prev : m.link.next) = o.link.box;
        }
    }
    return true;
}

}  // namespace

Context * create_pipeline(const char * path, const std::vector<int> & devices, ErrorSink sink) {
    ModelFile mf;
    if (!scan_model_file(path, mf, sink)) return nullptr;
    const int n_layer = (int) mf.header.n_layer, world = (int) devices.size();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, world >= 2 && world <= n_layer, "A pipeline needs 2 .. n_layer (%d) stages, got %d", n_layer, world);
    double layer_bytes = 0, head_bytes = 0;
    for (const TensorInfo & t : mf.tensors) {
        if (t.name == "head.weight") head_bytes += (double) t.nbytes;
        else if (t.name.compare(0, 7, "blocks.") == 0) layer_bytes += (double) t.nbytes;
    }
    layer_bytes /= n_layer;
    const std::vector<int> bounds = balanced_cuts(n_layer, world, layer_bytes > 0 ? head_bytes / layer_bytes : 0.0);
    Context * head = nullptr;
    PipeGroup * group = new (std::nothrow) PipeGroup();
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, nullptr, group, "Failed to allocate the pipeline group");
    group->devices = devices;
    bool ok = true;
    for (int r = 0; r < world && ok; r++) {
        Model * m = load_model(path, devices[(size_t) r], bounds[(size_t) r], bounds[(size_t) r + 1], sink);
        Context * c = m ? create_context(m, sink) : nullptr;
        if (!c) { ok = false; break; }
        c->overlap_copies = false;
        if (r == 0) { head = c; head->group = group; group->refs.fetch_add(1); } else head->stages.push_back(c);
        cudaStream_t s = nullptr;
        ok = cudaSetDevice(devices[(size_t) r]) == cudaSuccess && cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess;
        group->streams.push_back(s);
    }
    ok = ok && connect_stages(head, sink);
    if (!ok) {
        if (head) destroy_context(head); else delete group;
        return nullptr;
    }
    return head;
}

Context * clone_pipeline(Context * src, ErrorSink sink) {
    Context * head = create_context(src->model, sink);
    if (!head) return nullptr;
    head->overlap_copies = false;
    head->group = src->group;
    src->group->refs.fetch_add(1);
    for (Context * s : src->stages) {
        Context * c = create_context(s->model, sink);
        if (!c) { destroy_context(head); return nullptr; }
        c->overlap_copies = false;
        head->stages.push_back(c);
    }
    return head;
}

bool pipeline_eval_host(Context * head, const uint32_t * tokens, size_t T, size_t chunk, const float * state_in, float * state_out, float * logits_out) {
    PipeGroup & g = *head->group;
    const size_t n = head->stages.size() + 1;
    const size_t per_layer = head->model->state_floats_per_layer();
    {
        std::lock_guard<std::mutex> lock(g.order);      // the passes of one evaluation enter every link back to back
        for (size_t r = 0; r < n; r++) {                // every stage takes ITS slice of the caller's state (layer-major ABI layout)
            Context * c = stage_of(head, r);
            const Model & m = *c->model;
            CUDA_OK(head, cudaSetDevice(m.dev.device));
            const size_t off = (size_t) m.layer_begin * per_layer, cnt = (size_t) (m.layer_end - m.layer_begin) * per_layer;
            CUDA_OK(head, cudaMemcpyAsync(c->state_a + off, state_in ? state_in + off : c->state_init + off, cnt * sizeof(float), cudaMemcpyDefault, g.streams[r]));
        }
        // chunk boundaries as the reference loop (rwkv_eval.inc:179-218), each cut further into passes the kernels take
        size_t off = 0;
        while (off < T) {
            size_t nchunk = T - off;
            if (chunk && nchunk > chunk) nchunk = chunk;
            size_t done = 0;
            while (done < nchunk) {
                const size_t np = nchunk - done < (size_t) MAX_TOKENS_PER_PASS ? nchunk - done : (size_t) MAX_TOKENS_PER_PASS;
                const bool final_pass = off + done + np == T;
                for (size_t r = 0; r < n; r++) {
                    Context * c = stage_of(head, r);
                    if (!pipe_forward(c, tokens + off + done, np, final_pass && logits_out != nullptr, g.streams[r])) { head->last_error |= c->last_error; return false; }
                }
                done += np;
            }
            off += nchunk;
        }
        for (size_t r = 0; r < n; r++) {
            Context * c = stage_of(head, r);
            const Model & m = *c->model;
            CUDA_OK(head, cudaSetDevice(m.dev.device));
            const size_t so = (size_t) m.layer_begin * per_layer, cnt = (size_t) (m.layer_end - m.layer_begin) * per_layer;
            if (state_out) CUDA_OK(head, cudaMemcpyAsync(state_out + so, c->state_a + so, cnt * sizeof(float), cudaMemcpyDefault, g.streams[r]));
            if (logits_out && r + 1 == n) CUDA_OK(head, cudaMemcpyAsync(logits_out, c->logits, (size_t) m.n_vocab * sizeof(float), cudaMemcpyDefault, g.streams[r]));
            // completion marker of THIS evaluation on stage r. Waiting on the stream itself (cudaStreamSynchronize) outside the lock
            // would be illegal whenever another host thread is capturing its stage graph on the same stream at that moment (found by
            // compute-sanitizer's slower timing: cudaErrorStreamCaptureInvalidated); an event recorded before that capture began is fine.
            if (!c->pipe_done) CUDA_OK(head, c->pipe_done.create(cudaEventDisableTiming));
            CUDA_OK(head, cudaEventRecord(c->pipe_done, g.streams[r]));
        }
    }
    for (size_t r = 0; r < n; r++) {
        CUDA_OK(head, cudaSetDevice(g.devices[r]));
        CUDA_OK(head, cudaEventSynchronize(stage_of(head, r)->pipe_done));
    }
    return true;
}

size_t stage_hidden_len(const Model & m, size_t T) { return (size_t) (m.arch_major == 7 ? 2 : 1) * (size_t) m.n_embed * T; }

bool stage_forward(Context * ctx, const uint32_t * tokens, size_t T, const float * hidden_in, float * hidden_out, bool want_logits, cudaStream_t stream) {
    const Model & m = *ctx->model;
    CUDA_OK(ctx, cudaSetDevice(m.dev.device));
    Pass p;
    if (!make_pass(ctx, (int) T, want_logits, stream, p)) return false;
    p.hidden_in = m.layer_begin == 0 ? nullptr : hidden_in;
    p.hidden_out = m.layer_end == m.n_layer ? nullptr : hidden_out;
    return forward_pass(ctx, tokens, p);
}

}  // namespace rwkv
