// Per-context execution state and the forward pass (serial + sequence mode) over a resident Model.
// Replaces rwkv_computation_graph + ggml_backend_sched (reference rwkv_graph.inc:16-54, 611-882;
// rwkv_eval.inc:25-35): there is no graph IR -- the launch sequence is written out per architecture.
#pragma once
#include <cuda_runtime.h>
#include <atomic>
#include <cstdint>
#include <memory>
#include <mutex>
#include <vector>

#include "model.h"

namespace rwkv {

// One process, several GPUs, behind the plain rwkv.h API (RWKV_B200_PIPELINE_DEVICES=0,1,...): the layers are cut into stages, one
// per listed device, connected by the peer-memory hand-off (kernels/pipe.cu). The handle the caller holds is the stage-0 context;
// it owns one context per further stage. All contexts of a stage (the original and its clones) enqueue on the stage's ONE stream,
// and one pass over all stages is enqueued under `order`, so items travel through every link in the same order.
struct PipeGroup {
    std::vector<cudaStream_t> streams;     // one per stage, on that stage's device
    std::vector<int> devices;
    std::mutex order;
    std::atomic<int> refs{0};
};

struct CopyPool;                        // helper threads of the pageable-buffer bounce path (engine.cu)
struct CopyPoolDelete { void operator()(CopyPool * p) const; };

// A LoRA adapter of rwkv_b200_adapter_create (include/rwkv_b200.h), in the HBM of its model's device: copies of the model's layers and
// top-level vectors in which every replaced tensor points at its replacement and every adapted matrix carries its LoraDelta. A
// context with the adapter attached reads these instead of the model's. It serves every context of that model.
struct Adapter {
    Model * model = nullptr;             // holds a reference (Model::refcount), released by destroy_adapter
    std::vector<Layer> layers;           // indexed by absolute layer id, as Model::layers
    DevVec ln0_w, ln0_b, ln_out_w, ln_out_b;
    std::vector<LoraDelta> deltas;       // DevMatrix::lora points into it
    DeviceBuffer<uint8_t> arena;         // A, B and the replacements
    bool replaces = false;               // some entry is a replacement (rank 0): it cannot be attached to one sequence of a batch
    mutable std::atomic<int> attached{0};   // contexts, and sequences of batch contexts, that have it attached
};
// M rows of K values in the file layout of `type`, as a replaced matrix is encoded before its upload: F32 copied, F16 rounded, the
// other types by quantize_row. `out` has M * tensor_nbytes(type, K, 1, 1) bytes.
void encode_rows(int type, const float * values, size_t M, size_t K, uint8_t * out);
// One entry of rwkv_b200_adapter_create (the layout of struct rwkv_b200_adapter_tensor).
struct AdapterTensor {
    const char * name;
    uint32_t rank;
    const float * a, * b, * values;
};
// Checks every entry before it allocates anything (RWKV_ERROR_ARGS), then uploads. NULL on failure, with the flags set.
Adapter * create_adapter(Model * model, const AdapterTensor * t, size_t n, float scale, ErrorSink sink);
// false with RWKV_ERROR_ARGS while a context has it attached. Deletes the model when the adapter held its last reference.
bool destroy_adapter(Adapter * a, ErrorSink sink);

// Every CUDA resource of a context is a member owner (cuda_handles.h), released when the context is deleted, in the reverse order of
// declaration. A lazily allocated set is a member struct built by one ensure function in engine.cu: complete or empty, never partial.
struct Context {
    Stream stream;                         // declared first, so destroyed last: the other members' work is enqueued on it
    Model * model = nullptr;
    PipeGroup * group = nullptr;           // set on the stage-0 context of an in-process pipeline
    std::vector<Context *> stages;         // ... which owns the contexts of stages 1 .. N-1
    Event ev_start, ev_stop;

    // device buffers
    DeviceBuffer<float> state_a;           // current input state
    DeviceBuffer<float> state_b;           // output state of the running evaluation
    DeviceBuffer<float> state_init;        // rwkv_init_state image, copied when state_in == NULL
    DeviceBuffer<float> logits;            // [n_vocab]
    DeviceBuffer<unsigned char> xq;        // staged activation columns handed from producer kernels to single-token GEMVs (act_stage.cuh)
    size_t xq_slot_bytes = 0;
    Event pipe_done;                 // in-process pipeline: end of this context's latest evaluation on its stage's stream
    bool use_tensor_cores = true;
    // The buffers of passes of up to capacity_T tokens (ensure_capacity): the tokens, the activation arena, fp16 copies of GEMM inputs
    // for the tensor-core path, and two pinned token slots, used alternately (`phase`): the host may prepare pass n+1 while pass n runs.
    struct Activations {
        DeviceBuffer<int> tokens;          // [capacity_T]
        DeviceBuffer<float> scratch;
        DeviceBuffer<void> act16; size_t act16_bytes = 0;
        PinnedBuffer<int> tokens_host[2];
        bool slot_used[2] = {false, false};   // slot_free has been recorded since the slot was allocated
        int capacity_T = 0;
    } act;
    Event slot_free[2];                    // recorded after the pass that last read the slot
    int phase = 0;                   // flips every pass together with the state_a/state_b swap

    // A single-token pass runs either over all resident layers at once (segment 0) or, when the caller's host state is copied in
    // and out around it, as n_segments consecutive layer groups (segments 1..n_segments) so that the H2D copy of group g+1 and the
    // D2H copy of group g-1 overlap the kernels of group g. Slots below are keyed by slot_index(want_logits, phase, segment).
    static constexpr int MAX_SEGMENTS = 8;
    static constexpr int N_SLOTS = 2 * 2 * (1 + MAX_SEGMENTS);
    static int slot_index(bool want_logits, int phase, int segment) { return ((want_logits ? 1 : 0) * 2 + phase) * (1 + MAX_SEGMENTS) + segment; }
    int n_segments = 1;              // layer groups of the overlapped path (1 = no overlap)
    bool overlap_copies = false;     // rwkv_eval with host state: pipeline the state copies against the layer groups
    struct CopyStreams { Stream in, out; Event pass_begin, seg_in[MAX_SEGMENTS], seg_out[MAX_SEGMENTS]; } copies;
    // pinned bounce buffers for pageable caller memory (engine.cu: eval_host_overlapped), allocated on first need
    struct Bounce {
        PinnedBuffer<float> in, out, logits;
        Event seg_d2h[MAX_SEGMENTS];       // slice g has arrived in `out`
        std::unique_ptr<CopyPool, CopyPoolDelete> pool;   // declared after the buffers, so its threads are joined before they are freed
    } bounce;

    // CUDA graphs for single-token passes; captured on the second use of a slot.
    struct GraphSlot { GraphExec exec; int uses = 0; unsigned long long launches = 0; };
    GraphSlot graphs[N_SLOTS];
    bool use_graphs = true;

    // Profiling mode (bench.py roofline leg): CUDA events around every GEMV launch, graphs off.
    bool profiling = false;
    struct ProfRecord { Event start, stop; double bytes = 0; };
    std::vector<ProfRecord> prof;

    DeviceBuffer<TraceRec> trace_buf;  // in-kernel timeline records (rwkv_b200_trace_*), 1024 slots
    int trace_count = 0;             // slots used by the last enqueued / captured pass
    const char * trace_names[1024] = {};   // kernel name per slot (string literals)

    // Batched multi-sequence decode (rwkv_b200_batch_*): batch_n > 0 makes this a batch context whose state
    // buffers hold batch_n states back to back (batch_stride = state_len floats apart) and whose logits buffer holds batch_n columns;
    // every pass evaluates exactly one token of each sequence.
    int batch_n = 0;
    long long batch_stride = 0;
    // Ragged passes of a batch context (batch_eval_ragged), allocated on the first one. The host writes each pass's map into a pinned
    // slot that follows the tokens_host / slot_free rule: column offsets [batch_n + 1], the sequence of every column
    // [MAX_TOKENS_PER_PASS], then the last column and the index of every advancing sequence [batch_n each]; map is its device
    // copy. The head runs on the gathered last columns (head_x [C, batch_n]) into head_y [n_vocab, batch_n].
    struct Ragged { PinnedBuffer<int> host[2]; DeviceBuffer<int> map; DeviceBuffer<float> head_x, head_y; } ragged;
    // Scoring passes (score, batch_score_ragged): the head's output for every column of a pass ([MAX_TOKENS_PER_PASS, n_vocab]),
    // allocated on the first, and the targets and results of a call's tokens (capacity entries each), grown to the largest call.
    DeviceBuffer<float> score_logits;
    // Checkpoints inside passes (eval_checkpoints), allocated on the first pass that has one: a pinned map per phase, which follows the
    // tokens_host / slot_free rule, and its device copy: the slot of every column [MAX_TOKENS_PER_PASS] (-1: none), then the state each
    // slot writes [MAX_TOKENS_PER_PASS]. Host destinations, and device ones that are not 16-byte aligned, are written to `staging`
    // (count states) and copied out after the pass; it grows to the most such checkpoints inside one pass of a call.
    struct CheckpointMaps { PinnedBuffer<unsigned char> host[2]; DeviceBuffer<unsigned char> map; } cps;
    struct CheckpointStaging { DeviceBuffer<float> states; size_t count = 0; } cp_staging;
    struct ScoreIo { DeviceBuffer<uint32_t> targets; DeviceBuffer<float> lp; DeviceBuffer<uint8_t> greedy; size_t capacity = 0; } score;

    // On-device sampling (kernels/sampling.cu): result word, scratch for biased logits, device copy of the caller's logit bias.
    bool logits_valid = false;       // ctx->logits holds the head output of the most recent pass
    struct SampleOut { DeviceBuffer<uint32_t> token; PinnedBuffer<uint32_t> token_host; } sample_out;
    DeviceBuffer<float> sample_scratch;    // [n_vocab] ([batch_n, n_vocab] in a batch context)
    struct Bias { DeviceBuffer<uint32_t> ids; DeviceBuffer<float> values; size_t capacity = 0; } bias;   // a batch: all rows' lists back to back
    // ... and in a batch context the per-sequence parameters and results, [batch_n] each, allocated on the first batch_sample
    struct SampleRows {
        DeviceBuffer<SampleRow> rows; PinnedBuffer<SampleRow> rows_host;
        DeviceBuffer<uint32_t> tokens; PinnedBuffer<uint32_t> tokens_host;
    } sample_rows;

    // Device-side generation (generate), allocated on the first call at GENERATE_MAX tokens per row so that the pointers captured in
    // the loop's graph never change. in: GenShared, GenRow [rows], GenMaskRow [rows], u [rows][GENERATE_MAX]; out: n_generated
    // [rows], the number of passes that ran, automaton states [rows], tokens [rows][GENERATE_MAX]. Both are packed with the call's
    // row stride, so each crosses PCIe once.
    struct Generate {
        DeviceBuffer<unsigned char> in; PinnedBuffer<unsigned char> in_host;
        DeviceBuffer<uint32_t> out; PinnedBuffer<uint32_t> out_host;
        DeviceBuffer<float> counts;        // [rows, n_vocab] penalty counts
        DeviceBuffer<uint32_t> bias_ids;   // [rows, n_vocab]
        DeviceBuffer<float> bias_values, scratch;   // [rows, n_vocab] each
        DeviceBuffer<float> park;          // batch contexts: [rows, n_vocab] logits of frozen rows
    } gen;
    // The penalty decay of every row (set_penalty_decay), 1 until set; it travels in the call's GenRow. The penalty weights
    // (set_penalty_weights): n_vocab floats, allocated by the first call that sets a table and kept at that address; `set` false
    // means all 1. The call's GenShared carries the table's address, so no graph holds it.
    std::vector<float> penalty_decay;
    struct PenaltyWeights { DeviceBuffer<float> table; bool set = false; } pen_weights;
    // the loop's graphs, keyed by phase (which state buffer holds the current state), as the single-token slots are, by the family
    // of its step kernel (GenFamily) and by whether the loop streams its tokens to a callback
    GraphExec gen_graphs[2][4][2];
    // Streaming generation, allocated on the first streaming call: mapped pinned words shared by the step kernel and the calling
    // thread (GenStepParams), at device addresses the streaming graphs capture. Layout: published [rows], acked [rows], timed_out,
    // then tokens [rows][GENERATE_MAX].
    struct Streaming { PinnedBuffer<uint32_t> words; Event done; } streamed;   // done: recorded after the streaming loop's copies
    bool in_stream = false;          // the calling thread is inside a streaming call's callbacks: this context's stream is busy
    // Log-probabilities of generated tokens (generate with a LogprobsOut), allocated only by calls that ask for them. lp_req: the
    // call's GenLogprobRequest, at a device address the logprob graphs capture, and its pinned copy. lp_out: the call's outputs
    // [rows][n] logprobs, sample probs, then [rows][n][top_n] ids and log-probabilities, `words` 32-bit words each, grown to the
    // largest rows * n * (2 + 2 * top_n) asked for. lp_ring: mapped [rows][2][GEN_LP_RECORD] records of the streaming loop.
    struct LogprobRequest { DeviceBuffer<GenLogprobRequest> dev; PinnedBuffer<GenLogprobRequest> host; } lp_req;
    struct LogprobOut { DeviceBuffer<uint32_t> dev; PinnedBuffer<uint32_t> host; size_t words = 0; } lp_out;
    PinnedBuffer<uint32_t> lp_ring;
    // Per-row samplers (generate with SamplerIn rows), allocated only by calls that use them: the call's upload at a device address
    // the sampled graphs capture, and its pinned copy: the log-probability request word (lp_req or NULL), GenSamplerRow[rows], then
    // room for rows * GEN_BIAS_MAX GenBiasEntry.
    struct Samplers { DeviceBuffer<unsigned char> dev; PinnedBuffer<unsigned char> host; } smp;
    // Beam search (beam_search): the park [batch_n, n_vocab] (the logits of the pass that runs before the loop is captured, then the
    // logits of the slots that groups which stopped keep), allocated on the first call; the loop state and a search state per group
    // (kernels/ops.h: BeamLoop, BeamState[groups], one allocation) and the back-pointers [capacity][batch_n][2], grown to the most
    // groups and the largest max_tokens asked for, which drops beam_graphs, as they hold their addresses. host: pinned BeamLoop, the
    // BeamStates and the back-pointers.
    DeviceBuffer<float> beam_park;
    struct Beam {
        DeviceBuffer<BeamLoop> loop; DeviceBuffer<uint32_t> back; PinnedBuffer<unsigned char> host;
        size_t capacity = 0, groups = 0;
        BeamState * states() const { return reinterpret_cast<BeamState *>(loop.get() + 1); }
    } beam;
    GraphExec beam_graphs[2];              // the search loop's graphs, keyed by phase and by the groups they were built for
    int beam_graph_groups[2] = {};

    // The attached adapter (set_adapter) or NULL, and the scratch of its deltas, allocated on the first attach for passes of up to
    // MAX_TOKENS_PER_PASS columns so that captured graphs never see it move: u [GEMV_MAX_PROBLEMS][LORA_MAX_RANK][T] and the base
    // outputs z of a batch's adapted problems with a nonlinear epilogue, max(4 C, F + C) rows of T.
    const Adapter * adapter = nullptr;
    struct LoraScratch { DeviceBuffer<float> u, z; } lora;
    // A batch context's adapters per sequence (batch_set_adapter): seq_adapter [batch_n] (NULL: the base weights), empty until the first
    // attach; the distinct adapters among them (at most LORA_MAX_ADAPTERS), and each sequence's index into that list or -1.
    std::vector<const Adapter *> seq_adapter, seq_adapters;
    std::vector<int> seq_slot;

    float last_device_ms = 0.f;      // CUDA-event time of the last forward (kernels only)
    int last_error = 0;              // rwkv_error_flags
    bool print_errors = true;
    uint32_t n_threads = 1;

    ErrorSink sink() { return ErrorSink{&last_error, &print_errors}; }
};

// Largest number of tokens pushed through the kernels in one go; longer sequences are cut into
// pieces of this size with the state staying on the device.
constexpr int MAX_TOKENS_PER_PASS = 256;
extern std::atomic<unsigned long long> g_graph_launches;   // CUDA graphs launched by this process: single-token replays and generation loops
extern std::atomic<size_t> g_bounce_min_bytes;   // pageable caller states of at least this many bytes travel through pinned bounce buffers

Context * create_context(Model * model, ErrorSink sink, int batch_n = 0);   // batch_n > 0: a batch context for that many sequences
void destroy_context(Context * ctx);

// In-process pipeline over `devices` (one stage per entry, layer blocks balanced by bytes with the head on the last stage).
Context * create_pipeline(const char * path, const std::vector<int> & devices, ErrorSink sink);
Context * clone_pipeline(Context * head, ErrorSink sink);
// rwkv_eval / rwkv_eval_sequence / rwkv_eval_sequence_in_chunks for a pipeline handle: every stage takes its slice of the caller's
// host state, passes of <= MAX_TOKENS_PER_PASS tokens run through all stages (the state stays resident in between), every stage
// hands its slice back, the last one the logits. chunk == 0: plain sequence evaluation.
bool pipeline_eval_host(Context * head, const uint32_t * tokens, size_t T, size_t chunk, const float * state_in, float * state_out, float * logits_out);

// Host image of a fresh state (rwkv_init_state, rwkv_eval.inc:224-241).
void fill_init_state(const Model & m, float * state);

// state_a <- host state (or the init image when NULL). Asynchronous on ctx->stream.
bool upload_state(Context * ctx, const float * state_in);
// host <- state_a / logits; synchronises the stream.
bool download_outputs(Context * ctx, float * state_out, float * logits_out);

// rwkv_eval / rwkv_eval_sequence with caller-owned host buffers: state_in (NULL = fresh state) -> T tokens -> state_out / logits_out
// (either may be NULL). With ctx->overlap_copies and a pass that fits one launch sequence the state travels per layer group,
// overlapped with the kernels; otherwise upload_state + forward + download_outputs. Synchronises before returning.
bool eval_host(Context * ctx, const uint32_t * tokens, size_t T, const float * state_in, float * state_out, float * logits_out);

// rwkv_eval_sequence_in_chunks: the reference's chunk loop (rwkv_eval.inc:158-222) with the state resident between chunks.
bool eval_host_chunks(Context * ctx, const uint32_t * tokens, size_t T, size_t chunk, const float * state_in, float * state_out, float * logits_out);

// Runs T tokens (host pointer) through all resident layers: reads state_a, leaves the new state in
// state_a (buffers are swapped internally), and, if want_logits, ln_out + head of the last token
// into ctx->logits. Asynchronous except for the token upload.
bool forward(Context * ctx, const uint32_t * tokens, size_t T, bool want_logits);

// Batch contexts: state of sequence `seq` <- host state (NULL = fresh) / -> host; one token of every sequence; logits of `seq`.
bool batch_set_state(Context * ctx, int seq, const float * state_in);
bool batch_get_state(Context * ctx, int seq, float * state_out);
bool batch_eval(Context * ctx, const uint32_t * tokens, bool want_logits);
bool batch_get_logits(Context * ctx, int seq, float * logits_out);
// Ragged pass arguments (batch_eval_ragged, batch_score_ragged): a batch context, non-NULL arrays, 1 <= sum of counts <= MAX_TOKENS_PER_PASS
// (returned in total), every token below n_vocab.
bool check_ragged(Context * ctx, const uint32_t * tokens, const uint32_t * counts, size_t & total);

// Scoring (rwkv_b200_score / rwkv_b200_batch_score_ragged, include/rwkv_b200.h): the passes of forward(tokens, n, want_logits) or of
// batch_eval_ragged(tokens, counts, want_logits), with the head over every column of a pass and the scoring kernel over its output:
// logprobs_out[i] / greedy_out[i] (host or device pointers; greedy_out may be NULL) for every i whose target is not SCORE_NO_TARGET, the
// others left as they were. The logits of the last column (of every advancing sequence) go to ctx->logits. The head runs on the tensor
// cores (score_on_tensor_cores) or as the GEMV with the LayerNorm prologue. The arguments are checked by the caller, except the ragged
// counts, which batch_score_ragged checks before it enqueues anything. Never a CUDA graph. Synchronises.
bool score(Context * ctx, const uint32_t * tokens, const uint32_t * targets, size_t n, float * logprobs_out, uint8_t * greedy_out);
bool batch_score_ragged(Context * ctx, const uint32_t * tokens, const uint32_t * counts, const uint32_t * targets, float * logprobs_out, uint8_t * greedy_out);
// Ragged pass: sequence b advances counts[b] tokens (tokens back to back in sequence order; 0 leaves it exactly as it was), all in one
// pass over the weights. Checks every argument before it enqueues anything. want_logits: the logits column of every sequence with
// counts[b] > 0 receives the logits of its last token, the other columns keep what they held. Never replays a CUDA graph.
bool batch_eval_ragged(Context * ctx, const uint32_t * tokens, const uint32_t * counts, bool want_logits);

// Checkpoints (rwkv_b200_eval_checkpoints / rwkv_b200_batch_eval_ragged_checkpoints, include/rwkv_b200.h): the state after token
// `position` of sequence `sequence`'s tokens of the call, into state_out (host or device memory). The layout of struct rwkv_b200_checkpoint.
struct CheckpointReq {
    uint32_t sequence, position;
    float * state_out;
};
// The entries' own rules (RWKV_ERROR_ARGS): cp not NULL when n_cp > 0, strictly increasing (sequence, position), sequence < n_seq,
// position < counts[sequence], no NULL destination, no two destinations of state_len floats that overlap and, when device >= 0, no
// device pointer of another device than `device`.
bool check_checkpoints(ErrorSink sink, size_t n_seq, const uint32_t * counts, size_t state_len, int device, const CheckpointReq * cp, size_t n_cp);
// forward(tokens, T, want_logits) / batch_eval_ragged(tokens, counts, want_logits) with the same passes and launches, which also write
// the checkpoints: one at the last column of its sequence in a pass is a copy of that state after the pass; the kernels write the others
// (16-byte aligned device destinations directly, the others through Context::cp_staging). The arguments have been checked (check_checkpoints, and
// check_ragged, which gave `total`, for the ragged call); nothing is enqueued before the staging is allocated. Synchronises.
bool forward_checkpoints(Context * ctx, const uint32_t * tokens, size_t T, bool want_logits, const CheckpointReq * cp, size_t n_cp);
bool batch_eval_ragged_checkpoints(Context * ctx, const uint32_t * tokens, const uint32_t * counts, size_t total, bool want_logits, const CheckpointReq * cp,
                                   size_t n_cp);

// Samples the next token from ctx->logits on the device (reference python/sampling.py:10-52 with the caller's uniform number u in
// [0, 1) in place of numpy's RandomState draw); only the token id is copied back. Requires a preceding pass that computed logits.
bool sample_token(Context * ctx, float temperature, float top_p, double u, const uint32_t * bias_ids, const float * bias_values, size_t n_bias, uint32_t * token_out);

// One row's logit bias ids: each below n_vocab and none twice (the kernel adds the entries without atomics, and the reference takes
// a dict). `seen` is a bitmap of n_vocab bits, all clear on entry and on return.
bool check_bias_ids(ErrorSink sink, const uint32_t * bias_ids, size_t n_bias, size_t n_vocab, std::vector<uint64_t> & seen);

// The arguments of a draw for each of n_rows rows (batch_sample, the batched kernel's test hook): non-NULL arrays, every row's
// temperature, top_p and u in range, and, with bias_offsets, offsets from 0 that never decrease and bias ids below n_vocab, none
// twice within a row.
bool check_sample_rows(ErrorSink sink, size_t n_rows, size_t n_vocab, const float * temperature, const float * top_p, const double * u,
                       const uint32_t * bias_offsets, const uint32_t * bias_ids, const float * bias_values, const uint32_t * tokens_out);
// rows[b] <- row b's parameters and its bias range (empty without bias_offsets); the arguments passed check_sample_rows.
void fill_sample_rows(SampleRow * rows, size_t n_rows, const float * temperature, const float * top_p, const double * u, const uint32_t * bias_offsets);

// Batch contexts: one draw per sequence from its column of ctx->logits, row b exactly what sample_token draws from the same logits
// with temperature[b], top_p[b], u[b] and bias entries [bias_offsets[b], bias_offsets[b + 1]) of bias_ids / bias_values
// (bias_offsets NULL = no bias; else batch_n + 1 entries from 0, non-decreasing). Checks every argument before it enqueues anything,
// then one launch; only the batch_n token ids are copied back. Synchronises.
bool batch_sample(Context * ctx, const float * temperature, const float * top_p, const double * u, const uint32_t * bias_offsets,
                  const uint32_t * bias_ids, const float * bias_values, uint32_t * tokens_out);
// batch_eval(tokens, want_logits = true) + batch_sample without bias. The sampling arguments are checked before the pass, so a
// rejected call leaves every sequence's state as it was.
bool batch_eval_sample(Context * ctx, const uint32_t * tokens, const float * temperature, const float * top_p, const double * u, uint32_t * tokens_out);

// Device-side generation over n_rows rows (1 for a single-sequence context, batch_n for a batch context), the loop of
// rwkv_b200_generate / rwkv_b200_batch_generate (include/rwkv_b200.h). Host arrays of n_rows entries; u and tokens_out are
// [n_rows][n] with n the largest max_tokens; keep_counts may be NULL. check_generate_rows checks every argument (also for the test
// hook); generate checks the context too and runs the whole loop as one graph launch, then copies tokens and counts back. Synchronises.
// With on_token, the loop streams: the calling thread busy-polls the published tokens, calls on_token(user, row, index, token) for
// each, in order per row, and acknowledges it; a nonzero return ends the row after that token (rwkv_b200_generate_stream).
using TokenFn = int (*)(void * user, size_t sequence, size_t index, uint32_t token);
bool check_generate_rows(ErrorSink sink, size_t n_rows, size_t n_vocab, const uint32_t * max_tokens, const float * temperature, const float * top_p,
                         const float * presence, const float * frequency, const double * u, const uint32_t * stop_ids, size_t n_stop,
                         const void * tokens_out, const void * n_generated);
// With automata (rwkv_b200_generate_constrained), row b is restricted by automata[b] from state automaton_states[b] (a NULL entry:
// unconstrained), and automaton_states[b] receives the row's final state.
// With lp (rwkv_b200_generate_logprobs), every drawn token's log-probability, top alternatives and sampling probability go to lp's
// host arrays, [n_rows][n] (top arrays [n_rows][n][top_n]), entries past n_generated[b] NaN / SCORE_NO_TARGET; the loop runs the logprob
// kernels, which take automata == NULL as "no row constrained". check_logprobs checks lp (also for the test hook).
struct Automaton;
struct LogprobsOut {
    size_t top_n;
    float * logprobs;
    uint32_t * top_ids;
    float * top_logprobs;
    float * sample_probs;             // may be NULL
};
bool check_logprobs(ErrorSink sink, size_t n_vocab, const LogprobsOut * lp);
// With samplers (rwkv_b200_generate_sampled), samplers[b] adds row b's top_k, min_p and user bias entries to its draws, and lp may be
// NULL; the loop runs the sampled kernels, which also take automata == NULL as "no row constrained". check_samplers checks the rows
// (also for the test hook).
struct SamplerIn {
    uint32_t top_k;                   // 0 = off
    float min_p;                      // 0 = off
    size_t n_bias;
    const uint32_t * bias_ids;
    const float * bias_values;
};
bool check_samplers(ErrorSink sink, size_t n_rows, size_t n_vocab, const SamplerIn * samplers);
bool generate(Context * ctx, const uint32_t * max_tokens, const float * temperature, const float * top_p, const float * presence,
              const float * frequency, const uint8_t * keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop,
              uint32_t * tokens_out, uint32_t * n_generated, TokenFn on_token = nullptr, void * user = nullptr,
              const Automaton * const * automata = nullptr, uint32_t * automaton_states = nullptr, const LogprobsOut * lp = nullptr,
              const SamplerIn * samplers = nullptr);
// The penalty tables of generation (rwkv_b200_set_penalty_weights, rwkv_b200_get_penalty_counts / rwkv_b200_set_penalty_counts,
// include/rwkv_b200.h). read_penalty_table copies n floats from host memory or device memory of `device` into `host` and checks that
// each is finite and >= 0 (RWKV_ERROR_ARGS, also for a device pointer of another device). The others have their context and sequence
// checked by the caller, check their table, allocate what they need all or nothing, and synchronise. weights NULL: all 1.
bool read_penalty_table(ErrorSink sink, const float * p, size_t n, int device, std::vector<float> & host, const char * what);
bool set_penalty_weights(Context * ctx, const float * weights);
bool get_penalty_counts(Context * ctx, int seq, float * counts_out);
bool set_penalty_counts(Context * ctx, int seq, const float * counts_in);

// Beam search over the sequences of a batch context (rwkv_b200_beam_search_groups, include/rwkv_b200.h): n_groups searches of width
// W = batch_n / n_groups, group g from sequence g*W's state and logits, as one graph launch; rwkv_b200_beam_search is n_groups = 1. The
// context, its logits and the arguments have been checked by the caller, except n_vocab and the driver, which this checks. Outputs as
// the C call's, [n_groups][n_best][n] with n the largest max_tokens. Synchronises.
bool beam_search(Context * ctx, int n_groups, const uint32_t * max_tokens, const float * length_penalty, const uint32_t * stop_ids, size_t n_stop,
                 size_t n_best, uint32_t * tokens_out, uint32_t * lengths_out, double * scores_out, uint8_t * finished_out);

// A token automaton of rwkv_b200_automaton_create: the transition table next[s * n_vocab + t] (GEN_MASK_DEAD: t not allowed in s)
// and live[s] (s allows some token) in the HBM of the model's device. It serves every context of that model.
struct Automaton {
    const Model * model = nullptr;
    int device = 0;
    size_t n_vocab = 0;
    uint32_t n_states = 0;
    DeviceBuffer<uint16_t> next;
    DeviceBuffer<uint8_t> live;
};
// Host checks of a table (1 <= n_states <= 65535, every entry below n_states or dead) and its live flags, [n_states].
bool check_automaton_table(ErrorSink sink, const uint16_t * next, size_t n_states, size_t n_vocab);
void automaton_live(const uint16_t * next, size_t n_states, size_t n_vocab, uint8_t * live);
// The automaton's table on the model's device; `next` may be a host or a device pointer. NULL on failure, with the flags set.
Automaton * create_automaton(const Model * model, const uint16_t * next, size_t n_states, ErrorSink sink);
void destroy_automaton(Automaton * a);
// Drops the loop's graphs (they hold the activation buffers and the GEMM routing of the time they were captured).
void drop_generate_graphs(Context * ctx);
// Drops the single-token graphs as well: every graph the context holds.
void drop_all_graphs(Context * ctx);
// Attaches `a` (NULL: detaches), dropping the single-token and generation graphs; the state is untouched. The caller has checked the
// context and that `a` belongs to its model.
bool set_adapter(Context * ctx, const Adapter * a);
// Gives sequence `seq` of a batch context adapter `a` (NULL: the base weights), with the same waits and dropped graphs as set_adapter.
// The caller has checked the context, the sequence, that `a` belongs to its model, replaces nothing and that the context has no
// adapter of its own; this checks the number of distinct adapters.
bool batch_set_adapter(Context * ctx, int seq, const Adapter * a);

// Floats of a context's delta scratch (Context::lora_u / lora_z) for a model of n_embed C and largest n_ffn F.
struct LoraScratchSize { size_t u, z; };
LoraScratchSize lora_scratch_floats(size_t C, size_t F);
// The LoraBatch of GEMV batch b, whose columns carry deltas through n_slots adapters (1 .. LORA_MAX_ADAPTERS): delta[i][k] is the delta
// of problem i under adapter k or NULL, col_slot[t] the adapter of column t or -1. A problem gets one group per adapter that adapts it
// and has columns, plus, with a nonlinear epilogue, one group of rank 0 with its other columns; a problem none of whose columns is
// under a delta is not adapted at all. An adapted problem of nonlinear epilogue is retargeted in b to EPI_NONE into z, the next
// M * T floats of z; u gives each adapted problem its largest rank times T floats. u_used / z_used: the floats taken. False (CTX |
// UNSUPPORTED) past LORA_MAX_GROUPS groups. Host only: b's pointers are not read.
bool build_lora_batch(ErrorSink sink, GemvBatch & b, int n_slots, const LoraDelta * const delta[][LORA_MAX_ADAPTERS], const int * col_slot,
                      float * u, float * z, LoraBatch & lb, size_t & u_used, size_t & z_used);

size_t stage_hidden_len(const Model & m, size_t T);

// Single-token passes of a single-sequence v6 context fold the two LoRA matrices that stream almost nothing into their neighbours:
// maa_w1 into the LayerNorm-mix launch (launch_v6_prologue), decay_w2 into the WKV launch (Wkv6Params::dw2). This is the one
// predicate that decides it, from shapes alone: head size 64, n_embed <= 4096, both matrices planned by the streaming GEMV with one
// warp per row (WK == 1) and their rows fitting the shared memory of the two kernels. On true, w1 and dw2 hold the matrices' problems
// (weights, plan, epilogue) without activation pointers.
bool v6_lora_fold_shapes(int C, int S, GemvProblem & w1, GemvProblem & dw2);
// Its two halves, also the argument checks of the fused kernels' test hooks: maa_w1 (w1) for launch_v6_prologue, decay_w2 (dw2) for
// launch_wkv6 with Wkv6Params::dw2 set. Both fill the plan (wk, g) of the problem they are given.
bool v6_prologue_fits(int C, GemvProblem & w1);
bool wkv6_decay_fits(int C, int S, GemvProblem & dw2);
bool v6_lora_fold(const Layer & L, int C, int S, GemvProblem & w1, GemvProblem & dw2);
// GEMV-streamed weight bytes of one token that the fold takes out of the GEMV launches (maa_w1 + decay_w2 of the folded layers).
size_t v6_folded_gemv_bytes(const Model & m);

// One pipeline stage: the resident layers [layer_begin, layer_end) for T <= MAX_TOKENS_PER_PASS tokens. The first stage
// embeds `tokens`, the others start from `hidden_in`; every stage but the last leaves its result in `hidden_out`
// (device pointers, stage_hidden_len(T) floats); the last one computes the logits when asked. `stream` (may be NULL = the
// context's own) is the CUDA stream everything is enqueued on.
bool stage_forward(Context * ctx, const uint32_t * tokens, size_t T, const float * hidden_in, float * hidden_out, bool want_logits, cudaStream_t stream);
// The same with the hand-off done by peer-memory kernels on the stream (kernels/pipe.cu): receive from the previous stage's
// stores (unless this stage embeds tokens), run the resident layers, store into the next stage's mailbox (unless this is the last).
bool pipe_forward(Context * ctx, const uint32_t * tokens, size_t T, bool want_logits, cudaStream_t stream);
// Allocates (once) the stage's mailbox for passes of up to MAX_TOKENS_PER_PASS tokens.
bool pipe_ensure_box(Context * ctx);

}  // namespace rwkv
