// Launchers for the non-GEMV kernels of the RWKV eval path: embedding gather + ln0, LayerNorm +
// token shift + mixing, the v6 data-dependent lerp, and the WKV4/5/6/7 recurrences with their
// per-head normalisation and gating fused in. All activations are fp32, column-major [dim, T].
//
// The four stages that carry recurrent state (LayerNorm + mix, WKV4, WKV5/6, WKV7) also serve batch contexts, which evaluate one
// token of each of several sequences per pass. Their seq_stride selects the mode: 0 means T tokens of one sequence; > 0 means T
// sequences of one token each, column t working on the state of sequence t, which lives t * seq_stride floats after the state
// pointers (sequence 0's). Both modes run the same arithmetic, so a sequence gives the same bits in a batch as alone.
// A third, ragged mode (seq_off set, seq_stride > 0) lies between them: sequence s advances seq_off[s + 1] - seq_off[s] tokens, its
// columns [seq_off[s], seq_off[s + 1]) back to back in the pass, on the state s * seq_stride floats on; T is the sum of the counts.
// A sequence without columns is not touched. seq_off (and LnMixParams::col_seq) are written by the host before the pass.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "gemv.h"   // TraceRec

namespace rwkv {

// The MODE template argument of the state-carrying kernels: T tokens of one sequence, one token of each of T sequences, ragged.
constexpr int SEQ_ONE = 0, SEQ_BATCH = 1, SEQ_RAGGED = 2;
// Checkpoints (rwkv_b200_eval_checkpoints): the SEQ_SNAP | SEQ_ONE and SEQ_SNAP | SEQ_RAGGED instantiations run exactly the arithmetic
// of the plain mode and also write the state after every column t with slot[t] >= 0 into the state that starts at dst[slot[t]], in the
// ABI layout: the launch's slice sits `at` floats into it. A launch takes them whenever slot is set. (A batch pass needs none: each
// sequence advances one token, so its checkpoint is the state after the pass.)
constexpr int SEQ_SNAP = 4;
struct CheckpointMap {
    const int * slot = nullptr;       // [T] the checkpoint slot of each column, -1: none
    float * const * dst = nullptr;    // device array: the state each slot writes
    long long at = 0;
};

// x[:, t] = LN(emb[tokens[t]]; ln0)     (rwkv_graph.inc:655-658, 787-790)
cudaError_t launch_embed_ln0(const void * emb, int emb_type, long long emb_pitch, const int * tokens, int T, int C,
                             const float * ln_w, const float * ln_b, float * x, cudaStream_t s);

// LayerNorm + token shift (rwkv_carry_x, rwkv_graph.inc:56-82) + per-arch mixing.
struct LnMixParams {
    TraceRec * trace = nullptr;
    const float * x;          // [C, T] residual stream
    const float * ln_w, * ln_b;
    const float * state_in;   // [C] previous token's LN(x) (att_xx / ffn_xx slot of the input state)
    float * state_out;        // [C] <- LN(x[:, T-1])
    int C, T;
    // formula 0 (v4/v5, rwkv_graph.inc:94-97):  out_j = xx*m_j + (prev - prev*m_j)
    // formula 1 (v6/v7, rwkv_graph.inc:310-311, 406, 520-521, 538):  out_j = (prev - xx)*m_j + xx
    int formula;
    int n_out;
    const float * coef[6];    // [C] each
    float * out[6];           // [C, T] each
    float * out_xx;           // optional [C, T]: LN(x)
    float * out_sx;           // optional [C, T]: prev - xx
    long long seq_stride = 0;
    const int * seq_off = nullptr;   // ragged mode: [n_seq + 1] column offsets of the sequences
    const int * col_seq = nullptr;   // ragged mode: [T] the sequence of each column
};
// cp.slot set: the checkpoint kernel (a kernel argument of its own: v6_prologue_kernel takes LnMixParams by value before another struct)
cudaError_t launch_ln_mix(const LnMixParams & p, cudaStream_t s, const CheckpointMap & cp = {});

// v6 time-mixing prologue of a single-token pass, ln_mix (one token, n_out == 1) and the first LoRA matrix in one launch:
// w1.y = tanh(W1 . mix[0]) with w1 = {maa_w1, EPI_TANH} planned by gemv_tma_plan. Every CTA runs the LayerNorm of ln_mix_kernel on
// all channels, CTA 0 alone writes out_xx / out_sx / state_out, and each CTA computes V6_PROLOGUE_ROWS rows of W1 from a staged
// copy of mix[0]. p.out[0] is not written. The bits equal launch_ln_mix followed by the GEMV.
constexpr int V6_PROLOGUE_ROWS = 8;
constexpr size_t V6_PROLOGUE_MAX_SMEM = 96 * 1024;
size_t v6_prologue_smem_bytes(const GemvProblem & w1, int C);
cudaError_t launch_v6_prologue(const LnMixParams & p, const GemvProblem & w1, cudaStream_t s);

// v6 data-dependent lerp (rwkv_graph.inc:323-346): for j in {w,k,v,r,g}
//   m_j[c,t] = sum_i W2[j][c][i] * z[j*mix + i, t];   out_j = (m_j + maa_j[c]) * sx + xx
struct V6LerpParams {
    TraceRec * trace = nullptr;
    const float * w2;         // [5][C][mix] fp32 (ggml ne = [mix, C, 5])
    const float * z;          // [5*mix, T] = tanh(W1 . xxx)
    const float * xx, * sx;   // [C, T]
    const float * maa[5];     // [C]
    float * out[5];           // [C, T]
    int C, T, mix;
    unsigned char * q_out[5]; // T == 1, C % 32 == 0 only: staged columns (act_stage.cuh) for consumers of weight type q_type[j]; all or none
    int q_type[5];
};
cudaError_t launch_v6_lerp(const V6LerpParams & p, cudaStream_t s);

// v4 WKV (rwkv_att_wkv_v4, rwkv_graph.inc:119-161) fused with the r* multiply (:182,195).
struct Wkv4Params {
    TraceRec * trace = nullptr;
    const float * k, * v, * r;        // [C, T]; r already sigmoid-ed
    const float * time_first, * time_decay;   // [C]
    const float * aa_in, * bb_in, * pp_in;    // [C]
    float * aa_out, * bb_out, * pp_out;
    float * y;                        // [C, T] = r * wkv
    int C, T;
    unsigned char * q_out; int q_type;  // T == 1, C % 32 == 0 only: y as a staged column (act_stage.cuh)
    long long seq_stride = 0;
    const int * seq_off = nullptr; int n_seq = 0;   // ragged mode: [n_seq + 1] column offsets of the sequences
    CheckpointMap cp;                 // appended last: the other members keep their offsets
};
cudaError_t launch_wkv4(const Wkv4Params & p, cudaStream_t s);

// v5/v6 WKV (ggml_compute_forward_rwkv_wkv6_f32, ggml-cpu.c:11803) + per-head norm + ln_x + gate
// (rwkv_graph.inc:275-289, 370-382).
struct Wkv6Params {
    TraceRec * trace = nullptr;
    const float * r, * k, * v;        // [C, T]
    const float * td;                 // decay: [C, T] if td_per_token else per-channel [C] (v5.2) / per-head [H] (v5.1)
    const float * tf;                 // time_first / time_faaaa: [C] or per-head [H]
    int td_per_token, per_head_scalars;
    const float * state_in;           // [H][S][S]  (i_key major, j_val minor)
    float * state_out;
    const float * lnx_w, * lnx_b;     // [C]
    const float * g;                  // optional [C, T] gate (already silu-ed)
    float * y;                        // [C, T]
    float eps;                        // 1e-5 (v5) or 64e-5 (v6)
    int H, S, T;
    unsigned char * q_out; int q_type;  // T == 1, S % 32 == 0 only: y as a staged column (act_stage.cuh)
    long long seq_stride = 0;         // a multiple of 4: the state moves in float4s
    // v6 single-token passes with dw2.W set (v6_lora_fold): the decay is computed here, w = exp(-exp(Wd2 . lora1 + time_decay)) with
    // dw2 = {decay_w2, x = lora1, bias = time_decay, EPI_BIAS_EXPNEGEXP} planned by gemv_tma_plan, instead of read from td.
    GemvProblem dw2 = {};
    const int * seq_off = nullptr; int n_seq = 0;   // ragged mode: [n_seq + 1] column offsets of the sequences
    CheckpointMap cp;                 // appended last: the other members keep their offsets
};
cudaError_t launch_wkv6(const Wkv6Params & p, cudaStream_t s);
// Dynamic shared memory of a wkv6 launch that computes the decay (head size 64): the head's rows of dw2 and the staged lora1.
constexpr size_t WKV6_DECAY_MAX_SMEM = 96 * 1024;
size_t wkv6_decay_smem_bytes(const GemvProblem & dw2);

// v7 (rwkv_att_v7, rwkv_graph.inc:432-479 + rwkv_wkv_v7_impl, rwkv_operators_wkv_v7.inc:37-106):
// kk/l2norm, k and v corrections, the recurrence, per-head norm, ln_x, the r*k*r_k bonus and the gate.
struct Wkv7Params {
    TraceRec * trace = nullptr;
    const float * r, * w, * k, * v, * a;   // [C, T]: r raw, w decay, k raw, v raw, a = sigmoid(..)
    const float * g;                  // [C, T] gate
    const float * vgate;              // [C, T] sigmoid(v0 + ...) or NULL for layer 0
    const float * v_first;            // [C, T] layer-0 value (ignored when vgate == NULL)
    float * v_out;                    // optional [C, T]: corrected v (layer 0 stores v_first through it)
    const float * k_k, * k_a, * r_k;  // [C]
    const float * lnx_w, * lnx_b;     // [C]
    const float * state_in;           // [H][S][S]  (i_val major, j_key minor)
    float * state_out;
    float * y;                        // [C, T]
    int H, S, T;
    unsigned char * q_out; int q_type;  // T == 1, S % 32 == 0 only: y as a staged column (act_stage.cuh)
    long long seq_stride = 0;
    const int * seq_off = nullptr; int n_seq = 0;   // ragged mode: [n_seq + 1] column offsets of the sequences
    CheckpointMap cp;                 // appended last: the other members keep their offsets
};
cudaError_t launch_wkv7(const Wkv7Params & p, cudaStream_t s);

// dst[:, dst_col[j]] = src[:, src_col[j]] for j < n, columns of `rows` floats (columns.cu); a NULL map stands for column j. The
// ragged pass of a batch context gathers the last column of every advancing sequence for the head and scatters the head's output.
cudaError_t launch_copy_columns(const float * src, const int * src_col, float * dst, const int * dst_col, int rows, int n, cudaStream_t s);

// Scoring passes (score.cu). y[:, t] = LN(x[:, t]; w, b) for t < T, columns of C floats, with the arithmetic of the head GEMV's
// PRO_LAYERNORM prologue: the tensor-core head of a scoring pass contracts these columns.
cudaError_t launch_layer_norm_columns(const float * x, const float * w, const float * b, int C, int T, float * y, cudaStream_t s);
// One CTA per column t < T of logits ([T, n_vocab], column t at logits + t * n_vocab): unless targets[t] is SCORE_NO_TARGET,
// logprobs[t] = log_softmax(column)[targets[t]] and, if greedy, greedy[t] = 1 when targets[t] is the first index of the column's
// maximum, else 0. A column with a NaN or +inf, or with no finite value, gives NaN and 0. Columns without a target are not written.
constexpr uint32_t SCORE_NO_TARGET = 0xFFFFFFFFu;
struct ScoreParams {
    TraceRec * trace = nullptr;
    const float * logits;
    int n_vocab, T;
    const uint32_t * targets;         // [T]
    float * logprobs;                 // [T]
    uint8_t * greedy;                 // [T] or NULL
};
cudaError_t launch_score(const ScoreParams & p, cudaStream_t s);

// Layer-pipeline hand-off over peer memory (pipe.cu). A PipeBox sits at the start of every stage's mailbox allocation, followed by
// PIPE_SLOTS data areas of slot_floats floats each.
constexpr int PIPE_SLOTS = 2;
constexpr int PIPE_CTAS = 8;               // every hand-off launch has this many CTAs (the device-side item counters rely on it)
struct PipeBox {
    unsigned long long credit;             // written by the NEXT stage: items of mine it has drained
    unsigned long long pad0[15];
    unsigned long long full[PIPE_SLOTS];   // written by the PREVIOUS stage: item + 1 that the slot holds
    unsigned long long pad1[16 - PIPE_SLOTS];
};
cudaError_t launch_pipe_recv(PipeBox * mine, PipeBox * prev, unsigned long long * counters, size_t slot_floats, float * x, size_t nx, float * v, size_t nv, cudaStream_t s);
cudaError_t launch_pipe_send(PipeBox * mine, PipeBox * next, unsigned long long * counters, size_t slot_floats, float * x, size_t nx, float * v, size_t nv, cudaStream_t s);

// On-device sampling from the logits of the last evaluated token (reference python/sampling.py:10-52); see sampling.cu.
struct SampleParams {
    const float * logits;             // [n_vocab] device
    int n_vocab;
    float temperature, top_p;
    double u;                         // uniform number in [0, 1) drawn by the caller
    const uint32_t * bias_ids;        // device, n_bias entries (logit_bias of the reference), or NULL
    const float * bias_values;
    int n_bias;
    float * scratch;                  // [n_vocab] device, used only when n_bias > 0
    uint32_t * token_out;             // device
    float * prob_out;                 // optional device: probability the chosen token had
};
cudaError_t launch_sample(const SampleParams & p, cudaStream_t s);

// The same draw for each row of a [n_rows, n_vocab] block of logits (a batch context's head output), one CTA per row. Row b uses
// logits + b * n_vocab, rows[b] and bias entries [rows[b].bias_begin, rows[b].bias_end) of bias_ids / bias_values, and, when it has a
// bias, scratch + b * n_vocab; it writes token_out[b] and, if prob_out, prob_out[b]. Each row gives the bits of launch_sample on it.
struct SampleRow {
    float temperature, top_p;
    double u;
    int bias_begin, bias_end;
};
constexpr int SAMPLE_MAX_ROWS = 256;  // MAX_TOKENS_PER_PASS: the sequences of the largest batch context
struct SampleBatchParams {
    const float * logits;             // [n_rows, n_vocab] device
    int n_vocab, n_rows;
    const SampleRow * rows;           // [n_rows] device
    const uint32_t * bias_ids;        // device, concatenated bias lists of all rows, or NULL when no row has one
    const float * bias_values;
    float * scratch;                  // [n_rows, n_vocab] device, or NULL when no row has a bias
    uint32_t * token_out;             // [n_rows] device
    float * prob_out;                 // optional [n_rows] device
};
cudaError_t launch_sample_batch(const SampleBatchParams & p, cudaStream_t s);

// Device-side generation (rwkv_b200_generate / rwkv_b200_batch_generate): one step of the sample-and-evaluate loop per launch, CTA b
// for row b. A row that is not frozen freezes when it has drawn max_tokens tokens; otherwise it draws with u[b * stride + step] from
// its logits with the bias -(presence + c[n] * frequency) on every token n with penalty count c[n] != 0 (sample_row's bias path),
// writes the token to tokens[b * stride + step], and freezes on a stop token; any other token is evaluated: every count of the row
// becomes c[n] * decay, then c[tok] += weights[tok] (1 without a table), and tok is the row's next input token. The last CTA of the
// step sets both conditional handles to "some row is still active" and, if so, counts one more pass.
struct GenRow {                       // written by the host per call; step and frozen are then the loop's state
    float temperature, top_p, presence, frequency;
    uint32_t max_tokens, step, frozen;
    float decay;                      // penalty decay, 0 < decay <= 1 (1: the counts only grow)
};
constexpr int GENERATE_MAX_STOP = 16;
struct GenShared {                    // written by the host per call (ticket = active = 0)
    uint32_t stop[GENERATE_MAX_STOP];
    uint32_t n_stop, stride;
    uint32_t ticket, active;          // CTAs done with this step / rows active after it; reset by the step's last CTA
    const float * weights;            // [n_vocab] penalty weights, or NULL for all 1; in the upload so that no graph holds it
};
// Streaming generation (rwkv_b200_generate_stream / rwkv_b200_batch_generate_stream): the same step with a gate and a publisher over
// words in mapped pinned host memory. Gate: before a row that is not frozen draws token step (0 < step < max_tokens), thread 0 waits
// until acked[b] >> 1 == step, i.e. the host has acknowledged token step - 1; acked bit 0 asks the row to stop, which freezes it as an
// exhausted budget does. A wait longer than STREAM_TIMEOUT_MS freezes the row the same way and sets *timed_out. Publisher: after a
// draw, stream_tokens[b * GENERATE_MAX + step] = token, then (release, system scope) published[b] = step + 1.
constexpr int GENERATE_MAX = 4096;
constexpr int STREAM_TIMEOUT_MS = 10000;
// Constrained generation (rwkv_b200_generate_constrained / rwkv_b200_batch_generate_constrained): the same steps, blocking or streaming,
// with row b restricted by a token automaton, next[s * n_vocab + t] the state after token t in state s or GEN_MASK_DEAD. A row in a
// state s with !live[s] freezes before it draws, as an exhausted budget freezes it; otherwise every token t with next[s][t] dead
// gets the bias -inf in place of its penalty, and a drawn token that is evaluated (not a stop id) moves the row to next[s][tok].
// After every step states_out[b] = the row's state. A row with next == NULL is unconstrained. The rows live in the per-call upload,
// so that the graph holds only their address and serves every automaton.
constexpr uint16_t GEN_MASK_DEAD = 0xFFFF;
struct GenMaskRow {                   // written by the host per call; state is then the loop's
    const uint16_t * next;            // [n_states, n_vocab] device, or NULL
    const uint8_t * live;             // [n_states]: the state allows some token
    uint32_t state, pad;
};
// Generation with log-probabilities (rwkv_b200_generate_logprobs / rwkv_b200_batch_generate_logprobs): the constrained steps (a row
// with a NULL table is unconstrained) that also report, for every token they draw at [b][step] of the request's [n_rows][stride]
// arrays: logprobs = log_softmax(z)[tok] of the raw logits z the token was drawn from, in the arithmetic and order of score_kernel;
// the top_n largest logits of z (descending, the smaller id first among equals) with their log-probabilities; and sample_probs = the
// probability the token had after bias, mask, top-p and temperature (sample_row's prob_out). A column with a NaN or +inf, or without a
// finite logit, gives NaN log-probabilities and SCORE_NO_TARGET ids. The streaming kernel also writes the token's record into the
// mapped ring (row b, slot step % 2: logprob, sample prob, top_n ids, top_n log-probabilities) before it publishes the token.
// The request lives in the per-call upload, so that one graph serves every top_n and output buffer.
constexpr int GEN_TOP_MAX = 20;
constexpr int GEN_LP_RECORD = 2 + 2 * GEN_TOP_MAX;     // words of a ring record
struct GenLogprobRequest {            // written by the host per call
    uint32_t top_n, pad;
    float * logprobs;                 // [n_rows][stride] device
    float * sample_probs;             // [n_rows][stride] device
    uint32_t * top_ids;               // [n_rows][stride][top_n] device
    float * top_logprobs;             // [n_rows][stride][top_n] device
    uint32_t * ring;                  // mapped [n_rows][2][GEN_LP_RECORD], streaming only
};
// Generation with a per-row sampler (rwkv_b200_generate_sampled / rwkv_b200_batch_generate_sampled): the constrained steps (a row with
// a NULL table is unconstrained), with log-probabilities when *lp_word is not NULL, where row b also has
// - user bias entries user_bias[bias_begin, bias_end) (distinct ids): after the penalty / mask list is written, an id its state allows
//   gets the entry value - (presence + c * frequency) if its penalty count c is not 0, else value;
// - top_k (0 = off) and min_p (0 = off): a token is kept iff its probability is at least the top-p cutoff, the top_k-th largest
//   probability (with multiplicity) and min_p * the largest probability (sample_row's KeepFilter).
// The rows, the pool and the request word live in the per-call upload, so that one graph serves every sampler.
constexpr int GEN_BIAS_MAX = 1024;    // user bias entries per row
struct GenSamplerRow {                // written by the host per call
    uint32_t top_k;
    float min_p;
    uint32_t bias_begin, bias_end;
};
struct GenBiasEntry {
    uint32_t id;
    float value;
};
// The step kernels come in four families, each blocking or streaming: plain, constrained, logprobs and sampled as described above.
enum GenFamily { GEN_PLAIN, GEN_CONSTRAINED, GEN_LOGPROBS, GEN_SAMPLED };
// The parameters of every step kernel. A family reads the step fields, the mapped words when it streams and the fields marked with its
// name; it leaves the others NULL.
struct GenStepParams {
    const float * logits;             // [n_rows, n_vocab]
    int n_vocab, n_rows;
    GenRow * rows;                    // [n_rows]
    GenShared * shared;
    const double * u;                 // [n_rows][stride]
    float * counts;                   // [n_rows, n_vocab] penalty counts
    uint32_t * bias_ids;              // [n_rows, n_vocab] scratch: the bias list of a row, one entry per token (id n_vocab = none)
    float * bias_values;
    float * scratch;                  // [n_rows, n_vocab]: the biased logits
    uint32_t * tokens;                // [n_rows][stride]
    uint32_t * n_generated;           // [n_rows]: the row's step after this launch
    uint32_t * passes;                // +1 for every step after which a row is active
    int * next_tokens;                // [n_rows]: input tokens of the next pass (0 for a frozen row)
    float * park;                     // [n_rows, n_vocab] or NULL: a row's logits are copied here when it freezes (batch contexts)
    bool set_handles;                 // inside a conditional graph: set run_pass and keep_going
    cudaGraphConditionalHandle run_pass, keep_going;
    // streaming
    uint32_t * stream_tokens;         // mapped [n_rows][GENERATE_MAX]
    uint32_t * published;             // mapped [n_rows]: tokens published this call
    const uint32_t * acked;           // mapped [n_rows]: 2 * tokens acknowledged + stop request
    uint32_t * timed_out;             // mapped: set when a wait ran out
    // constrained, logprobs and sampled
    GenMaskRow * mask;                // [n_rows]
    uint32_t * states_out;            // [n_rows]
    // The logprobs kernels read the request itself; the sampled kernels read it through a device word that the call sets to the
    // request or to NULL, so that one sampled graph serves calls with and without log-probabilities.
    const GenLogprobRequest * lp;                 // logprobs: device
    const GenLogprobRequest * const * lp_word;    // sampled: device word, the call's request or NULL for none
    const GenSamplerRow * samplers;               // sampled: [n_rows] device
    const GenBiasEntry * user_bias;               // sampled: device, the rows' entries
};
// The blocking step kernel of `family`. The streaming kernels run only as graph nodes.
cudaError_t launch_generate_step(const GenStepParams & p, GenFamily family, cudaStream_t s);
// The step kernel of `family`, streaming or not, as a kernel node of graph g after deps (the body of the generation loop).
cudaError_t add_generate_step_node(cudaGraph_t g, const cudaGraphNode_t * deps, size_t n_deps, const GenStepParams & p, GenFamily family, bool stream,
                                   cudaGraphNode_t * node);
// After a pass of a batch context inside the generation loop: dst slice b <- src slice b (state_len floats, seq_stride apart) for
// every frozen row, so that its state stays what it was.
cudaError_t launch_restore_frozen(const GenRow * rows, int n_rows, const float * src, float * dst, long long seq_stride, size_t state_len, cudaStream_t s);

// Beam search (rwkv_b200_beam_search, beam.cu) over the width W sequences of a batch context, W <= BEAM_MAX. One step: CTA k < n_live
// lists live beam k's top 2W tokens in the logprob kernels' top-N order (top_n.cuh) with their log-probabilities (score_row.cuh); the
// last CTA ranks every candidate with a finite log-probability by score = beam score + lp (double; ties: lower beam, then earlier
// position), walks the ranking until W live beams are taken, the pool holds W hypotheses or the list ends (a stop id goes to the pool,
// any other token becomes live slot L in the order taken), records slot L's parent and token at back[step][L], writes the next input
// tokens (0 past L) and, inside the loop's graph, sets run_pass = L > 0 and keep_going = L > 0 && pool < W && step + 1 < max_tokens.
// Grouped (rwkv_b200_beam_search_groups): G independent searches of width W over the G * W slots, group g in slots g*W .. g*W + W - 1
// with its own BeamState. The step's grid is (W, G); a group runs while n_live > 0, n_pool < W and step < max_tokens, and the CTAs of a
// group that does not run return at once. The last CTA of each running group walks it as above; the last walker of the step sets
// run_pass = some group took L > 0 and keep_going = some group runs on. A group that stops, or never ran (max_tokens 0), keeps its
// slots k < n_keep: the gather of pass park_at (BeamLoop::steps at that pass) copies them (state Y -> X, logits -> park) and the
// restore after the loop copies them back, as every pass in between evaluates all columns.
constexpr int BEAM_MAX = 10;
constexpr int BEAM_CANDS = 2 * BEAM_MAX;
struct BeamHyp {                      // a finished hypothesis: stop id `token` drawn at `step` from live beam `parent` of the step before
    double score;
    uint32_t step, parent, token, pad;
};
struct BeamState {                    // written by the host per call (n_live = 1, score[0] = 0: the root); then the loop's
    uint32_t stop[GENERATE_MAX_STOP];
    uint32_t n_stop, width, max_tokens;
    uint32_t step;                    // steps run
    uint32_t n_live, n_pool;          // live beams and pool entries after the last step
    uint32_t ticket;
    uint32_t n_keep, park_at, parked;  // slots kept once the group stops; the pass that parks them (0: none); set by that pass
    double score[BEAM_MAX];           // of the live beams
    uint32_t parent[BEAM_MAX];        // of the live beams: the gather map of the pass that evaluates them
    BeamHyp pool[BEAM_MAX];
    uint32_t cand_id[BEAM_MAX][BEAM_CANDS];
    float cand_lp[BEAM_MAX][BEAM_CANDS];    // NaN: no candidate
};
struct BeamLoop {                     // shared by the groups of one call; written by the host per call (n_active: groups that run)
    uint32_t n_active, ticket, n_next, any_live;    // this step's walkers, their ticket, groups that run on, groups that took L > 0
    uint32_t steps, pad[3];                         // steps run
};
struct BeamStepParams {
    const float * logits;             // [groups * width, n_vocab]: column g*W + k that of live beam k of group g
    int n_vocab, width, groups;
    BeamLoop * loop;
    BeamState * st;                   // [groups]
    uint32_t * back;                  // [max_tokens][groups * width][2]: parent slot (in its group) and token of every live slot of every step
    int * next_tokens;                // [groups * width]
    bool set_handles;                 // inside a conditional graph: set run_pass and keep_going
    cudaGraphConditionalHandle run_pass, keep_going;
};
cudaError_t launch_beam_step(const BeamStepParams & p, cudaStream_t s);
cudaError_t add_beam_step_node(cudaGraph_t g, const cudaGraphNode_t * deps, size_t n_deps, const BeamStepParams & p, cudaGraphNode_t * node);
struct BeamCopyParams {
    const BeamLoop * loop;
    BeamState * st;                   // [groups]; the gather sets `parked` of the groups it parks
    int width, groups, n_vocab;
    float * y, * x;                   // the current slots and the pass's input (state_len floats, seq_stride apart)
    long long seq_stride;
    size_t state_len;
    float * logits, * park;           // [groups * width, n_vocab]
};
// Before a pass, for every group g: x slice g*W + k <- y slice g*W + parent[k] for k < n_live if it took live beams at the last step,
// or x <- y and park <- logits for its slots k < n_keep if this pass is its park_at.
cudaError_t launch_beam_gather(const BeamCopyParams & p, cudaStream_t s);
// After the loop: y <- x and logits <- park for the kept slots of every parked group.
cudaError_t add_beam_restore_node(cudaGraph_t g, const cudaGraphNode_t * deps, size_t n_deps, const BeamCopyParams & p, cudaGraphNode_t * node);

}  // namespace rwkv
