/* rwkv_b200.h -- additive entry points of the H100 engine that the reference ABI has no slot for.
 * Nothing here is needed by a drop-in consumer; bench.py, the multi-GPU layer pipeline and the
 * tests use them. All follow the conventions of rwkv.h (bool / NULL returns, flags readable with
 * rwkv_get_last_error).
 */
#ifndef RWKV_B200_H
#define RWKV_B200_H

#include "rwkv.h"

#if defined(__cplusplus)
extern "C" {
#endif

/* Host-only summary of a model file (no GPU needed): what rwkv_init_from_file would load.
 * Architecture detection as reference rwkv_model_loading.inc:319-340, head geometry :403-409. */
struct rwkv_b200_file_info {
    uint32_t version, n_vocab, n_embed, n_layer, data_type;
    uint32_t arch_major, arch_minor, head_count, head_size;
    uint64_t n_tensors, file_size;
    uint64_t state_len;          /* floats, rwkv.cpp:171-179 */
    uint64_t bytes_per_token;    /* SURVEY.md 8(d) byte model: all layer tensors + head + 1 emb row + 2x state */
};
RWKV_API bool rwkv_b200_inspect_file(const char * model_file_path, struct rwkv_b200_file_info * out);

/* rwkv_init_from_file on an explicit CUDA device, keeping only layers [layer_begin, layer_end)
 * resident (layer_end < 0 = n_layer). A context that lacks layer 0 takes its input activations
 * from the previous pipeline stage, one that lacks the last layer cannot produce logits. */
RWKV_API struct rwkv_context * rwkv_b200_init_from_file_ex(const char * model_file_path, int device, int layer_begin, int layer_end);

/* Device-resident evaluation: the recurrent state stays in HBM between calls.
 *   rwkv_b200_state_load : state_in (host, may be NULL = fresh) -> device
 *   rwkv_b200_eval_resident: run n tokens from the resident state; logits stay on the device unless logits_out != NULL
 *   rwkv_b200_state_store: device -> state_out (host) */
/* The resident state is the state after the context's most recent evaluation of any kind: rwkv_eval, rwkv_eval_sequence and
 * rwkv_eval_sequence_in_chunks leave the state they computed resident too (whether or not state_out was given; state_in NULL starts
 * them from a fresh state), so rwkv_b200_state_store after one of them returns the bytes of its state_out. rwkv_b200_profile_pass and
 * rwkv_b200_time_resident are resident passes and advance it. rwkv_clone_context gives a new context that shares the weights and
 * nothing else: its resident state is unspecified until rwkv_b200_state_load or a rwkv_eval* call sets it, it has no logits (a draw
 * is refused until a pass computes them) and its penalty counts start from zero.
 * The logits are those of the most recent pass that ran the head; a pass that skips it (want_logits false and logits_out NULL,
 * rwkv_eval* with logits_out NULL) makes rwkv_b200_sample and rwkv_b200_generate* refuse with RWKV_ERROR_ARGS until the next one. */
RWKV_API bool rwkv_b200_state_load(struct rwkv_context * ctx, const float * state_in);
RWKV_API bool rwkv_b200_eval_resident(struct rwkv_context * ctx, const uint32_t * tokens, size_t n_tokens, bool want_logits, float * logits_out);
RWKV_API bool rwkv_b200_state_store(struct rwkv_context * ctx, float * state_out);
/* Blocks until everything enqueued on the context's stream has finished. */
RWKV_API bool rwkv_b200_synchronize(struct rwkv_context * ctx);

/* Batched multi-sequence decode (SURVEY.md 8f-2; the reference has no equivalent -- it evaluates one context per call): a batch
 * context holds the recurrent states of n_sequences independent sequences in HBM and evaluates ONE token of EACH per call, so every
 * weight matrix is streamed once for n_sequences tokens (the fused dequantize-GEMV runs its multi-column path). Per sequence the
 * result is bit-identical to evaluating that sequence alone with rwkv_eval (below 32 sequences; from 32 on the tensor-core path
 * takes the layer matrices, with its own rounding of the activations). RWKV v4 / v5 / v6 / v7, n_embed <= 4096, head size <= 64
 * (v7: 128).
 *   rwkv_b200_batch_create    : from any context of the model (shares its weights); free with rwkv_free; NULL on failure
 *   rwkv_b200_batch_set_state : state of one sequence <- state_in (host or device pointer, NULL = fresh state)
 *   rwkv_b200_batch_eval      : tokens[n_sequences], one per sequence; want_logits = run the head for every sequence
 *   rwkv_b200_batch_eval_ragged : continuous batching -- sequence b advances counts[b] tokens (a prompt, one decode token, or none)
 *                                 in the same single pass over the weights
 *   rwkv_b200_batch_get_logits / rwkv_b200_batch_get_state : copy one sequence's logits / state out (host or device pointer)
 * The next token of every sequence is drawn on the device by rwkv_b200_batch_sample / rwkv_b200_batch_eval_sample (below).
 * A batch context's logits start as zeros. rwkv_eval*, rwkv_b200_sample and the resident / stage entry points refuse a batch context. */
RWKV_API struct rwkv_context * rwkv_b200_batch_create(struct rwkv_context * ctx, size_t n_sequences);
RWKV_API bool rwkv_b200_batch_set_state(struct rwkv_context * batch, size_t sequence, const float * state_in);
RWKV_API bool rwkv_b200_batch_get_state(struct rwkv_context * batch, size_t sequence, float * state_out);
RWKV_API bool rwkv_b200_batch_eval(struct rwkv_context * batch, const uint32_t * tokens, bool want_logits);
/* Ragged pass of a batch context: sequence b advances counts[b] tokens (0 = the sequence is left exactly as it is), all in one pass
 * over the weights. tokens holds the sequences' tokens back to back in sequence order (sum of counts entries);
 * 1 <= sum of counts <= 256. want_logits: the logits column of every sequence with counts[b] > 0 receives the logits of its last
 * token; the other columns keep what they held. Longer prompts are fed over several calls; the states stay resident in between.
 * Every argument is checked before anything is enqueued, so a rejected call changes no state and no logits column: a context that is
 * not a batch context gives RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED; NULL arrays, a sum of 0 or above 256 and a token >= n_vocab give
 * RWKV_ERROR_ARGS. Per sequence the result is bit-identical to feeding its tokens to a single-sequence context one at a time while the
 * sum stays below 16, and with rwkv_b200_set_tensor_cores(batch, false) at any sum. rwkv_b200_batch_sample / get_logits / get_state
 * work after it unchanged; an idle sequence's row draws from the column it still holds. Validity is per context, the bytes per column:
 * after a pass that skipped the head (rwkv_b200_batch_eval with want_logits false, or a ragged pass without logits on a context whose
 * logits were not valid), a ragged pass with want_logits makes the logits valid again, and an idle sequence's column then holds the logits
 * of the last pass that ran the head for it (zeros if none ever did), not those of its latest token. */
RWKV_API bool rwkv_b200_batch_eval_ragged(struct rwkv_context * batch, const uint32_t * tokens, const uint32_t * counts, bool want_logits);
RWKV_API bool rwkv_b200_batch_get_logits(struct rwkv_context * batch, size_t sequence, float * logits_out);
RWKV_API size_t rwkv_b200_batch_size(const struct rwkv_context * ctx);   /* 0 for an ordinary context */

/* Scoring a known text (perplexity, likelihood-based evaluation, "echo + logprobs"): the log-probability the model gives each of
 * caller-given targets, computed on the device; no per-position logits cross PCIe.
 *   rwkv_b200_score: advances the resident state of a single-sequence context over tokens[0 .. n_tokens) exactly as
 *     rwkv_b200_eval_resident(ctx, tokens, n_tokens, true, NULL) does (same passes, same layer kernels). With z_i the logits after
 *     tokens[0 .. i], for every i whose targets[i] is not RWKV_B200_SCORE_NO_TARGET: logprobs_out[i] = log_softmax(z_i)[targets[i]] and
 *     greedy_out[i] = 1 if targets[i] is the first index of max(z_i), else 0 (greedy_out may be NULL). Other positions are not written.
 *     For perplexity, targets[i] = tokens[i + 1] and the last target is the first token of the next window, or NO_TARGET.
 *     Afterwards the resident state is what rwkv_b200_eval_resident leaves, the logits are z_{n-1} as the scoring head computed them
 *     (rwkv_b200_sample / rwkv_b200_generate* can follow), and the penalty counts are untouched.
 *   rwkv_b200_batch_score_ragged: the same over a ragged pass of a batch context, with the rules of rwkv_b200_batch_eval_ragged (with
 *     want_logits); targets, logprobs_out and greedy_out are indexed like tokens. Multiple-choice scoring: set k sequences to one prefix
 *     state and score k continuations in one pass over the weights.
 * The output pointers may be host or device memory; both calls synchronise before they return. A log-probability is computed from the
 * head's float logits in double (sum of expf(z - max), then log); -inf logits contribute nothing, a -inf target gives -inf, and a
 * position whose logits hold a NaN or +inf, or nothing finite, gives NaN with greedy 0. Passes of >= 32 tokens (batch contexts: >= 16)
 * with tensor cores on run the head on the tensor cores, from a tile-major copy of the head (2 bytes per weight) that the first such
 * pass builds and the model keeps until its last context is freed; their logits carry the rounding of that path. Every other pass
 * runs the head's GEMV on every column, which gives each position the bits rwkv_eval gives it token by token.
 * Refusals change no state, logits or validity: RWKV_ERROR_ARGS for NULL tokens, targets or logprobs_out, no tokens, a token >= n_vocab,
 * a target >= n_vocab other than NO_TARGET, n_vocab > 65536 and the ragged count rules; RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED for the
 * wrong kind of context, a pipeline handle or stage, and a call from inside a streaming callback of the context. A failed allocation of
 * the head's copy gives RWKV_ERROR_CTX | RWKV_ERROR_ALLOC before anything is enqueued. */
#define RWKV_B200_SCORE_NO_TARGET 0xFFFFFFFFu
RWKV_API bool rwkv_b200_score(struct rwkv_context * ctx, const uint32_t * tokens, const uint32_t * targets, size_t n_tokens,
                              float * logprobs_out, uint8_t * greedy_out);
RWKV_API bool rwkv_b200_batch_score_ragged(struct rwkv_context * batch, const uint32_t * tokens, const uint32_t * counts,
                                           const uint32_t * targets, float * logprobs_out, uint8_t * greedy_out);
/* Test hook: the scoring kernel on n_rows x n_vocab host logits (row-major), no model needed. Rows whose target is NO_TARGET keep what
 * logprobs_out / greedy_out held. */
RWKV_API bool rwkv_b200_score_logits(const float * logits, size_t n_rows, size_t n_vocab, const uint32_t * targets,
                                     float * logprobs_out, uint8_t * greedy_out);

/* On-device sampling (SURVEY.md 8f-4): the next token is drawn on the GPU from the logits of the most recent evaluation that
 * computed them, following the reference's python/sampling.py:10-52 (softmax, optional logit bias, temperature 0 = argmax, top-p
 * cutoff, power by 1/temperature, renormalise, inverse-CDF draw); only the 4-byte token id crosses PCIe instead of n_vocab floats.
 * `u` is a uniform number in [0, 1) from the caller's generator -- with u = numpy's RandomState.random_sample() the result is the
 * token numpy.random.choice would return in the reference. temperature >= 0, 0 <= top_p <= 1 (0 means 1), n_vocab <= 65536.
 * Every draw (these calls, the batch calls and every generate step) follows three rules:
 * - the drawn token has positive probability after bias, top-p and temperature, unless every biased logit is -inf or NaN;
 * - tempering is relative to the largest kept probability, (p / p_max)^(1 / temperature), so no temperature > 0 underflows: a kept
 *   token is lost only if its share is below 2^-149;
 * - a bias list that names a token twice, or a token >= n_vocab, is refused with RWKV_ERROR_ARGS.
 * rwkv_b200_eval_sample = rwkv_b200_eval_resident(token, with logits) + rwkv_b200_sample without bias. */
RWKV_API bool rwkv_b200_sample(struct rwkv_context * ctx, float temperature, float top_p, double u, const uint32_t * bias_ids, const float * bias_values,
                               size_t n_bias, uint32_t * token_out);
RWKV_API bool rwkv_b200_eval_sample(struct rwkv_context * ctx, uint32_t token, float temperature, float top_p, double u, uint32_t * next_token_out);

/* Test hook: the same sampling kernel on caller-provided host logits (any n_vocab <= 65536), no model needed.
 * prob_out (optional) receives the probability the chosen token had after top-p / temperature. */
RWKV_API bool rwkv_b200_sample_logits(const float * logits, size_t n_vocab, float temperature, float top_p, double u, const uint32_t * bias_ids,
                                      const float * bias_values, size_t n_bias, uint32_t * token_out, float * prob_out);

/* On-device sampling for a batch context: one kernel launch draws every sequence's next token and only n_sequences token ids cross
 * PCIe. One draw per sequence from that sequence's logits of the most recent rwkv_b200_batch_eval that computed them; row b
 * is exactly what rwkv_b200_sample draws from the same logits with temperature[b], top_p[b], u[b] and that row's bias.
 * Arrays of n_sequences host values; bias_offsets (NULL = no bias) has n_sequences + 1 entries, starting at 0 and
 * non-decreasing, and sequence b's bias is bias_ids / bias_values [bias_offsets[b], bias_offsets[b + 1]). */
RWKV_API bool rwkv_b200_batch_sample(struct rwkv_context * batch, const float * temperature, const float * top_p, const double * u,
                                     const uint32_t * bias_offsets, const uint32_t * bias_ids, const float * bias_values,
                                     uint32_t * tokens_out);
/* rwkv_b200_batch_eval(tokens, true) + rwkv_b200_batch_sample without bias; arguments are checked before the pass. */
RWKV_API bool rwkv_b200_batch_eval_sample(struct rwkv_context * batch, const uint32_t * tokens, const float * temperature,
                                          const float * top_p, const double * u, uint32_t * tokens_out);
/* Test hook: the batched kernel on n_rows x n_vocab host logits (row-major), no model needed; probs_out optional.
 * 1 <= n_rows <= 256, n_vocab <= 65536. */
RWKV_API bool rwkv_b200_sample_logits_batch(const float * logits, size_t n_rows, size_t n_vocab, const float * temperature,
                                            const float * top_p, const double * u, const uint32_t * bias_offsets,
                                            const uint32_t * bias_ids, const float * bias_values, uint32_t * tokens_out,
                                            float * probs_out);

/* Device-side generation: up to max_tokens sample-and-evaluate steps in one call, without the host in any step. For a sequence with
 * valid logits, step i = 0, 1, ...: (1) if i == max_tokens, stop; (2) draw tok from the current logits with temperature, top_p and
 * u[i] and the logit bias -(presence_penalty + count[n] * frequency_penalty) on every token n with count[n] > 0 (computed in float32,
 * the multiply and the add rounded separately) -- bit for bit what rwkv_b200_sample returns with that bias list; (3) tokens_out[i] =
 * tok; (4) if tok is one of the stop ids, stop: it is reported but neither evaluated nor counted; (5) otherwise count[tok] += 1,
 * evaluate tok (a single-token resident pass with logits) and continue. This is the loop of the reference's
 * python/chat_with_bot.py:244-260 and python/generate_completions.py:60-67. Afterwards the state has consumed every evaluated token,
 * the logits are those of the last evaluated token (the row the last token was drawn from), and n_generated counts the tokens written,
 * a stop token included.
 * The penalty counts are a per-sequence table in HBM, allocated on first use. keep_counts false starts the sequence from zero counts;
 * true continues from its previous generate call, so that a server can generate in short windows (between ragged admissions in a
 * batch) without losing its penalties. keep_counts applies to every sequence of an accepted call, also one that generates nothing
 * (max_tokens[b] = 0, or a constrained sequence that starts in a state that allows no token): its state and logits are left as they
 * are, its counts are cleared unless keep_counts[b] is set. At most RWKV_B200_GENERATE_MAX_STOP stop ids, shared by all sequences, each below n_vocab.
 * The whole loop is one CUDA-graph launch (a conditional WHILE node; a CUDA driver of 12.4 or newer); only the tokens come back.
 * Every argument is checked before anything is enqueued, and a rejected call changes no state, logits or count: a context of the
 * wrong kind (a batch context here, an ordinary one for the batch call, a pipeline or a stage of one) or an older driver gives
 * RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED; NULL arrays, max_tokens out of range, temperature, top_p or u out of the ranges of
 * rwkv_b200_sample, non-finite penalties, ids >= n_vocab, more than 16 stop ids, and a context whose last pass skipped the head give
 * RWKV_ERROR_ARGS. n_vocab <= 65536.
 * rwkv_b200_generate: a single-sequence context; 1 <= max_tokens <= RWKV_B200_GENERATE_MAX; u holds max_tokens numbers in [0, 1). */
#define RWKV_B200_GENERATE_MAX 4096
#define RWKV_B200_GENERATE_MAX_STOP 16
RWKV_API bool rwkv_b200_generate(struct rwkv_context * ctx, size_t max_tokens, float temperature, float top_p, float presence_penalty,
                                 float frequency_penalty, bool keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop,
                                 uint32_t * tokens_out, size_t * n_generated);
/* rwkv_b200_batch_generate: a batch context; per-sequence arrays of n_sequences entries: max_tokens (0 .. RWKV_B200_GENERATE_MAX; 0
 * leaves the sequence exactly as it is), temperature, top_p, penalties, keep_counts (NULL = none kept). With n the largest max_tokens,
 * u and tokens_out are [n_sequences][n]: sequence b's entries at b * n + i (tokens_out entries past n_generated[b] are 0). Every
 * sequence gives the tokens, state and logits rwkv_b200_generate gives it alone on the same logits and state (below 16 sequences;
 * from 16 on the layer matrices take the tensor-core path of rwkv_b200_batch_eval). The pass computes every sequence until the last
 * one stops; a stopped sequence's state and logits are put back after each pass and after the loop. */
RWKV_API bool rwkv_b200_batch_generate(struct rwkv_context * batch, const uint32_t * max_tokens, const float * temperature, const float * top_p,
                                       const float * presence_penalty, const float * frequency_penalty, const uint8_t * keep_counts,
                                       const double * u, const uint32_t * stop_ids, size_t n_stop, uint32_t * tokens_out, uint32_t * n_generated);

/* Streaming generation: the loops of rwkv_b200_generate / rwkv_b200_batch_generate, with every token handed to on_token while the loop
 * runs, so that an interactive caller can print it and end a sequence on a condition of its own (a decoded text, say) exactly after
 * any token. The arguments and their checks are those of the blocking calls, the same context kinds are refused, and on_token must
 * not be NULL (RWKV_ERROR_ARGS); a rejected call changes nothing.
 * 1. Delivery: on_token(user, sequence, index, token) runs on the calling thread exactly once for every token written to tokens_out
 *    (index: the token's position in this call), in index order per sequence; calls for different sequences interleave in the order
 *    their tokens arrive. Every call happens before the API call returns. A stop id is delivered too and ends its sequence whatever
 *    on_token returns.
 * 2. Gate: token j + 1 of a sequence is not drawn until on_token has returned for token j. The pass that evaluates token j runs while
 *    on_token runs, so the device waits only when a callback takes longer than a pass (in a batch, the step waits for every sequence).
 * 3. Ending a sequence: a nonzero return for token j ends that sequence after token j, which has been evaluated and counted, as
 *    python/chat_with_bot.py does. Its tokens, n_generated, state, logits and penalty counts are then bit-identical to the blocking
 *    call with max_tokens = j + 1 for that sequence and the same u; in a batch the other sequences are unaffected.
 * 4. Otherwise nothing changes: when on_token always returns 0, the results are bit-identical to the blocking call, and so are the
 *    results of later calls.
 * 5. Re-entrancy: from inside on_token, every call that would enqueue work on the generating context's stream or wait on it
 *    (rwkv_eval*, rwkv_b200_eval_resident, rwkv_b200_eval_sample, rwkv_b200_state_load / _store, rwkv_b200_synchronize,
 *    rwkv_b200_sample, rwkv_b200_generate*, rwkv_b200_batch_*, rwkv_b200_stage_eval / _logits on that context) returns false with
 *    RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED and enqueues nothing. Other contexts, clones of the same model included, stay usable; a
 *    call that has to allocate or free device memory (a first pass of a new size, creating or freeing a context) may wait for the
 *    whole device and belongs outside the callback. rwkv_free of the generating context from on_token is not allowed.
 * 6. Bounded wait: the device waits at most RWKV_B200_STREAM_TIMEOUT_MS for a callback. When the bound runs out it ends that sequence as
 *    if on_token had asked it to; once the callback has returned, the call returns false with RWKV_ERROR_CTX, and tokens_out,
 *    n_generated, state and logits keep what was delivered up to then. This is a safety net against a kernel spinning on a stuck host.
 * The calling thread busy-polls (yielding between polls) for the length of the call. While the device waits on the gate, each
 * waiting sequence holds one CTA of 1024 threads on an SM. */
#define RWKV_B200_STREAM_TIMEOUT_MS 10000
/* Return 0 to go on, nonzero to end `sequence` after `token` (its index-th token of this call). */
typedef int (*rwkv_b200_token_fn)(void * user, size_t sequence, size_t index, uint32_t token);
RWKV_API bool rwkv_b200_generate_stream(struct rwkv_context * ctx, size_t max_tokens, float temperature, float top_p, float presence_penalty,
                                        float frequency_penalty, bool keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop,
                                        rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out, size_t * n_generated);
RWKV_API bool rwkv_b200_batch_generate_stream(struct rwkv_context * batch, const uint32_t * max_tokens, const float * temperature,
                                              const float * top_p, const float * presence_penalty, const float * frequency_penalty,
                                              const uint8_t * keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop,
                                              rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out, uint32_t * n_generated);
/* Constrained generation: the loops above with every sequence's tokens restricted by a token automaton, so that structured output
 * (a number, a choice from a list, a fixed schema, tool-call syntax) stays on the device instead of a host loop of rwkv_b200_sample
 * calls with an n_vocab-entry -inf bias list.
 * An automaton is a dense transition table next[s * n_vocab + t] over the vocabulary of ctx's model, 1 <= n_states <= 65535: the state
 * after token t in state s, or RWKV_B200_AUTOMATON_DEAD when t is not allowed in s. next may be a host or a device pointer.
 * rwkv_b200_automaton_create checks every entry (< n_states or dead) and the context (a whole-model or a batch context) before it
 * allocates anything, then uploads the table once to the HBM of the model's device (n_states * n_vocab * 2 bytes, 128 KB per state at
 * n_vocab 65536) with a flag per state that says whether it allows any token. It returns NULL with RWKV_ERROR_ARGS for a NULL context
 * or a bad table, and RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED for a pipeline or one of its stages (flags read with
 * rwkv_get_last_error(NULL)). The automaton serves every context of that model (clones, batch contexts created from it); a context
 * of another model refuses it with RWKV_ERROR_ARGS. Free it with rwkv_b200_automaton_free once no call uses it, never from a token
 * callback.
 * The generate calls take the arguments of rwkv_b200_generate / rwkv_b200_batch_generate with the same checks, plus the automaton
 * and the caller's automaton state (in / out); on_token NULL is the blocking loop, otherwise the loop streams with every rule of
 * rwkv_b200_generate_stream. A rejected call changes no state, logits, counts or automaton state: a NULL automaton or state
 * pointer, a state >= n_states and an automaton of another model give RWKV_ERROR_ARGS. A constrained sequence in state s, at each step:
 * 1. if s allows no token, the sequence stops before it draws, exactly as at an exhausted budget (one that starts there generates 0
 *    tokens and is left as it is);
 * 2. it draws with the bias -inf on every token s does not allow, in place of any penalty, and the penalty on every other counted
 *    token: bit for bit what rwkv_b200_sample returns from the same logits, u and that bias list;
 * 3. a stop id can be drawn only where s allows it; it is reported, neither evaluated nor counted, and s stays;
 * 4. any other token is counted and evaluated, and s becomes next[s][token].
 * automaton_state receives the state after the last evaluated token. A callback that ends a sequence after token j gives the results
 * of max_tokens = j + 1, automaton state included. A one-state automaton that allows every token gives the bytes of the unconstrained
 * call. In a batch, automata[b] == NULL leaves sequence b unconstrained and automaton_states[b] untouched; such a row gives what
 * rwkv_b200_batch_generate gives it. */
#define RWKV_B200_AUTOMATON_DEAD 0xFFFF
struct rwkv_b200_automaton;
RWKV_API struct rwkv_b200_automaton * rwkv_b200_automaton_create(struct rwkv_context * ctx, const uint16_t * next, size_t n_states);
RWKV_API void rwkv_b200_automaton_free(struct rwkv_b200_automaton * automaton);
RWKV_API bool rwkv_b200_generate_constrained(struct rwkv_context * ctx, const struct rwkv_b200_automaton * automaton, uint32_t * automaton_state,
                                             size_t max_tokens, float temperature, float top_p, float presence_penalty, float frequency_penalty,
                                             bool keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop,
                                             rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out, size_t * n_generated);
RWKV_API bool rwkv_b200_batch_generate_constrained(struct rwkv_context * batch, const struct rwkv_b200_automaton * const * automata,
                                                   uint32_t * automaton_states, const uint32_t * max_tokens, const float * temperature,
                                                   const float * top_p, const float * presence_penalty, const float * frequency_penalty,
                                                   const uint8_t * keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop,
                                                   rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out, uint32_t * n_generated);

/* LoRA adapters: a fine-tune of the model (RWKV-LM-LoRA / RWKV-PEFT checkpoints, python lora.py) applied on the GPU beside the base
 * weights, which stay as loaded, at whatever type the file has (quantized included). An adapter lives in the HBM of the model's device
 * and serves every context of that model; attached to a context, it changes what every entry point of that context computes:
 * rwkv_eval*, the resident and ragged passes, rwkv_b200_score, sampling and every rwkv_b200_generate* family.
 *
 * Each entry of `t` names one tensor as the model file does ("blocks.3.att.key.weight", "blocks.0.ln0.weight", ...):
 * - rank > 0: a low-rank delta of a layer matrix W [M][K]: a is A, [rank][K], b is B, [M][rank], both row-major host arrays. Every pass
 *   computes y = epi(W.x + scale * B.(A.x)), where epi is that matrix's own epilogue (sigmoid, silu, relu^2, the residual add, the
 *   gated residual add), applied once to the sum. A and B are stored as fp16 and accumulated in fp32. 1 <= rank <= 256. The matrices
 *   that take a delta are att key / value / receptance / gate / output and ffn key / value / receptance (whichever the architecture
 *   has); emb, head and the small LoRA matrices inside a v6 / v7 layer (time_maa_w1, time_decay_w1 / w2, w1 .. v2) are refused.
 *   The caller's scale is lora_alpha / rank times any user scale; one scale serves every delta of the adapter.
 * - rank == 0: a full replacement of that tensor, `values` in the file's element order and shape (the element count of the tensor).
 *   Any tensor but emb.weight and head.weight. A replaced vector is kept in fp32; a replaced matrix is uploaded as the loader uploads
 *   the base: at the base file's type (quantized by the library's own quantizer when the base is quantized), in the device layout, with
 *   the tile-major copy when the base has one. A context with the adapter reads the replacement wherever it would read the base tensor.
 *
 * rwkv_b200_adapter_create checks every entry before it allocates anything and returns NULL with RWKV_ERROR_ARGS (read with
 * rwkv_get_last_error(NULL)) for: an unknown name, a name listed twice, a delta on a matrix that takes none, rank above 256, NULL arrays,
 * a non-finite scale or value. A and B, and the values of a replaced matrix whose base is not F32 (stored in fp16 or quantized with
 * fp16 scales), must also be finite in fp16: |v| < 65520. The values are copied: the caller's arrays may be freed when it
 * returns. A pipeline or one of its stages gives RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED.
 * rwkv_b200_adapter_free returns false with RWKV_ERROR_ARGS, changing nothing, while any context has the adapter attached; NULL is
 * accepted and returns true. Lifetime: the adapter holds a reference to its model's weights, as a context does, so the adapter and
 * the contexts of that model may be freed in any order; the weights are released with the last of them.
 * rwkv_b200_set_adapter attaches one adapter to ctx (a single-sequence or a batch context; in a batch, every sequence uses it), or
 * detaches with adapter == NULL. It waits for the context's queued work and drops its single-token and generation graphs, which are
 * captured again on later calls; the state, resident state and logits are untouched. A clone or a batch context made from an adapted
 * context starts with no adapter. Refused, changing
 * nothing: an adapter of another model (RWKV_ERROR_ARGS), a pipeline or a stage, and a call from inside that context's streaming
 * callback (RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED).
 * The invariants of the unadapted context hold for an adapted one: a sequence gives the bits of serial evaluation under any chunking
 * of passes below 32 tokens, a batch row those of a single context below 16 sequences, device-side generation those of the host loop.
 * An adapter whose every B is zero and that replaces nothing gives exactly the unadapted logits and states. */
struct rwkv_b200_adapter;
struct rwkv_b200_adapter_tensor {
    const char * name;        /* tensor name as in the model file */
    uint32_t rank;            /* > 0: low-rank delta of that matrix; 0: full replacement of that tensor */
    const float * a;          /* rank > 0: A, [rank][K] row-major */
    const float * b;          /* rank > 0: B, [M][rank] row-major */
    const float * values;     /* rank == 0: the replacement, in the file's element order and shape */
};
RWKV_API struct rwkv_b200_adapter * rwkv_b200_adapter_create(struct rwkv_context * ctx, const struct rwkv_b200_adapter_tensor * t, size_t n, float scale);
RWKV_API bool rwkv_b200_adapter_free(struct rwkv_b200_adapter * adapter);
RWKV_API bool rwkv_b200_set_adapter(struct rwkv_context * ctx, const struct rwkv_b200_adapter * adapter);

/* Generation with log-probabilities: the loops above that also report, for every token they draw, how likely it was, as completion
 * servers (logprobs / top_logprobs), evaluation and RL callers need, without per-token logits crossing PCIe.
 * The arguments, checks, context kinds and refusals are those of rwkv_b200_generate_constrained / rwkv_b200_batch_generate_constrained,
 * except that automaton may be NULL (no constraint; automaton_state is then not used) and automata may be NULL (no sequence
 * constrained); on_token NULL is the blocking loop. The outputs are host arrays indexed like tokens_out ([rows][n], n the largest
 * max_tokens, rows 1 or n_sequences); the top arrays are [rows][n][top_n]. With z the logits token i of a sequence was drawn from:
 * 1. Generation itself does not change: tokens, n_generated, state, logits, penalty counts and automaton states are bit-identical to
 *    the call without log-probabilities (rwkv_b200_generate* or its _constrained twin) with the same arguments.
 * 2. logprobs[i] = log_softmax(z)[token i] of the raw logits, before penalties, mask, top-p and temperature: bit for bit what
 *    rwkv_b200_score_logits returns for z and that target (a -inf logit gives -inf; a column with a NaN or +inf, or without a finite
 *    value, gives NaN). So rwkv_b200_score over the same text from the same state returns the same bits wherever it runs the GEMV head.
 * 3. top_ids[i][0 .. top_n) are the top_n largest entries of z in descending order, the smaller id first among equal logits, and
 *    top_logprobs their log-probabilities, each bit for bit rwkv_b200_score_logits with that id as target. -inf entries appear only when
 *    fewer than top_n are finite. For a column with a NaN or +inf, or without a finite value, every id is RWKV_B200_SCORE_NO_TARGET and
 *    every log-probability NaN.
 * 4. sample_probs[i] (optional) is the probability the token had under the distribution it was drawn from, after penalty bias,
 *    automaton mask, top-p and temperature: bit for bit rwkv_b200_sample_logits' prob_out for z, u and that bias list (1 at
 *    temperature 0).
 * 5. A stop id's entries are written too. Entries at or past n_generated[b] are NaN (floats) and RWKV_B200_SCORE_NO_TARGET (ids).
 * 6. Streaming: entry i of every output array is written before on_token(..., i, ...) is called; ending a sequence after token i gives
 *    the outputs of max_tokens = i + 1.
 * 7. RWKV_ERROR_ARGS, changing nothing, for a NULL lp or lp->logprobs, top_n > RWKV_B200_TOP_LOGPROBS_MAX or > n_vocab, and NULL top
 *    arrays with top_n > 0.
 * The first call that asks for log-probabilities allocates their buffers (rows * n * (2 + 2 * top_n) words on the device and pinned on
 * the host, grown to the largest call, and for streaming a small mapped ring); contexts that never ask allocate nothing. */
#define RWKV_B200_TOP_LOGPROBS_MAX 20
struct rwkv_b200_logprobs {
    size_t top_n;                              /* 0 .. RWKV_B200_TOP_LOGPROBS_MAX, and <= n_vocab */
    float * logprobs;                          /* [rows][n], required */
    uint32_t * top_ids;                        /* [rows][n][top_n], NULL iff top_n == 0 */
    float * top_logprobs;                      /* [rows][n][top_n], NULL iff top_n == 0 */
    float * sample_probs;                      /* [rows][n], optional */
};
RWKV_API bool rwkv_b200_generate_logprobs(struct rwkv_context * ctx, const struct rwkv_b200_automaton * automaton, uint32_t * automaton_state,
                                          size_t max_tokens, float temperature, float top_p, float presence_penalty, float frequency_penalty,
                                          bool keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop,
                                          rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out, size_t * n_generated,
                                          const struct rwkv_b200_logprobs * lp);
RWKV_API bool rwkv_b200_batch_generate_logprobs(struct rwkv_context * batch, const struct rwkv_b200_automaton * const * automata,
                                                uint32_t * automaton_states, const uint32_t * max_tokens, const float * temperature,
                                                const float * top_p, const float * presence_penalty, const float * frequency_penalty,
                                                const uint8_t * keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop,
                                                rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out, uint32_t * n_generated,
                                                const struct rwkv_b200_logprobs * lp);

/* Generation with a sampler per sequence: the knobs completion servers send on ordinary requests (top_k, min_p, logit_bias) inside the
 * device-side loop, so that such a request does not take every token's logits to the host. The arguments, checks, context kinds,
 * streaming, automata (NULL: unconstrained) and outputs are those of rwkv_b200_generate_logprobs / rwkv_b200_batch_generate_logprobs,
 * except that temperature, top_p and the penalties come from the sampler (samplers[b] for sequence b) and lp may be NULL (no
 * log-probabilities; nothing is allocated for them). One draw of a sequence in automaton state s with penalty counts c, logits z and
 * user bias ub (ub[n] for the ids bias_ids lists):
 * 1. Bias entry of token n: -inf if s does not allow n, whatever c[n] or ub[n]. Otherwise, with pen = presence + c[n] * frequency
 *    (float32, multiply and add rounded separately): c[n] > 0 with a user entry: ub[n] - pen (one more rounding); c[n] > 0 without one:
 *    -pen; c[n] = 0 with one: ub[n]; otherwise no entry. The biased logits are y = z + entry, as rwkv_b200_sample's bias list adds them.
 * 2. Temperature 0: the first index of max(y); top_k and min_p have no effect.
 * 3. p = softmax(y), the float32 values rwkv_b200_sample computes, and p_max = 1 / total its largest entry.
 * 4. Token n is kept iff p[n] >= the top-p cutoff of rwkv_b200_sample, p[n] >= the top_k-th largest entry of p counted with
 *    multiplicity (every tie at the k-th value is kept; top_k = 0 is off), and p[n] >= fl(min_p * p_max) (min_p = 0 is off). All three
 *    come from the same p, so the kept set is their intersection, in any order; the largest probability is always kept.
 * 5. Tempering relative to p_max, normalisation and the inverse-CDF draw with u are those of rwkv_b200_sample. lp->sample_probs is the
 *    chosen token's probability after all of this; lp->logprobs and the top entries are those of the raw z.
 * A column with a NaN or +inf draws as rwkv_b200_sample draws it. With top_k = 0, min_p = 0 and n_bias = 0 on every sequence, a call
 * returns the bits of the matching rwkv_b200_generate / _stream / _constrained / _logprobs call (tokens, n_generated, state, logits,
 * counts, automaton states, lp outputs). RWKV_ERROR_ARGS, changing nothing, for NULL sampler(s), top_k > n_vocab, min_p NaN or outside
 * [0, 1], n_bias > RWKV_B200_LOGIT_BIAS_MAX or n_bias > 0 with NULL arrays, a duplicate id or an id >= n_vocab in one sampler, and a
 * bias value that is NaN or +inf. The first call allocates the sampler upload (rows * RWKV_B200_LOGIT_BIAS_MAX * 8 bytes plus the rows,
 * on the device and pinned); contexts that never call these allocate nothing for it. */
#define RWKV_B200_LOGIT_BIAS_MAX 1024
struct rwkv_b200_sampler {
    float temperature, top_p;                  /* as rwkv_b200_sample */
    uint32_t top_k;                            /* 0 = off; <= n_vocab */
    float min_p;                               /* 0 = off; 0 .. 1 */
    float presence_penalty, frequency_penalty; /* as rwkv_b200_generate */
    size_t n_bias;                             /* 0 .. RWKV_B200_LOGIT_BIAS_MAX */
    const uint32_t * bias_ids;                 /* host, n_bias distinct ids < n_vocab */
    const float * bias_values;                 /* host, finite or -inf (a ban) */
};
RWKV_API bool rwkv_b200_generate_sampled(struct rwkv_context * ctx, const struct rwkv_b200_sampler * sampler, const struct rwkv_b200_automaton * automaton,
                                         uint32_t * automaton_state, size_t max_tokens, bool keep_counts, const double * u, const uint32_t * stop_ids,
                                         size_t n_stop, rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out, size_t * n_generated,
                                         const struct rwkv_b200_logprobs * lp /* NULL = none */);
RWKV_API bool rwkv_b200_batch_generate_sampled(struct rwkv_context * batch, const struct rwkv_b200_sampler * samplers /* [n_sequences] */,
                                               const struct rwkv_b200_automaton * const * automata, uint32_t * automaton_states,
                                               const uint32_t * max_tokens, const uint8_t * keep_counts, const double * u, const uint32_t * stop_ids,
                                               size_t n_stop, rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out, uint32_t * n_generated,
                                               const struct rwkv_b200_logprobs * lp /* NULL = none */);

/* Test hook: one step of the generation loop's kernel on n_rows x n_vocab host logits, no model needed. n is the largest max_tokens
 * (>= 1); u and tokens are [n_rows][n]. A row that is not frozen freezes once step == max_tokens, otherwise draws with u[b * n + step],
 * writes tokens[b * n + step], increments step, and freezes on a stop id or else increments counts[b][tok]. next_tokens receives each
 * row's next input token (0 when frozen), any_active 1 when a row is still active. Arguments are checked before a device is touched. */
struct rwkv_b200_generate_step_args {
    const float * logits;
    size_t n_rows, n_vocab;                    /* 1 .. 256, 1 .. 65536 */
    const uint32_t * max_tokens;
    const float * temperature, * top_p, * presence_penalty, * frequency_penalty;
    const double * u;
    const uint32_t * stop_ids;
    size_t n_stop;
    uint32_t * step;                           /* in / out, <= max_tokens */
    uint8_t * frozen;                          /* in / out */
    uint32_t * counts;                         /* [n_rows, n_vocab] in / out */
    uint32_t * tokens;                         /* [n_rows][n] in / out */
    int32_t * next_tokens;                     /* out */
    uint32_t * any_active;                     /* out */
};
RWKV_API bool rwkv_b200_test_generate_step(const struct rwkv_b200_generate_step_args * a);
/* The same step of the constrained kernel: row b follows the table next (n_states x n_vocab, as for rwkv_b200_automaton_create) from
 * states[b], which receives its new state; states[b] == UINT32_MAX marks an unconstrained row. */
RWKV_API bool rwkv_b200_test_generate_step_constrained(const struct rwkv_b200_generate_step_args * a, const uint16_t * next, size_t n_states,
                                                       uint32_t * states);
/* The same step of the logprob kernel: next NULL leaves every row unconstrained (states not used), otherwise as above. The outputs of
 * lp ([n_rows][n], top arrays [n_rows][n][top_n]) are written at [b][step] for every row that draws; other entries keep what they held. */
RWKV_API bool rwkv_b200_test_generate_step_logprobs(const struct rwkv_b200_generate_step_args * a, const uint16_t * next, size_t n_states,
                                                    uint32_t * states, const struct rwkv_b200_logprobs * lp);
/* The same step of the sampled kernel. a->temperature, top_p, presence_penalty and frequency_penalty must be NULL; samplers[n_rows]
 * supplies them. next may be NULL (unconstrained) and lp may be NULL, otherwise as for rwkv_b200_test_generate_step_logprobs. */
RWKV_API bool rwkv_b200_test_generate_step_sampled(const struct rwkv_b200_generate_step_args * a, const struct rwkv_b200_sampler * samplers,
                                                   const uint16_t * next, size_t n_states, uint32_t * states, const struct rwkv_b200_logprobs * lp);
/* The same step of a streaming kernel, the one the *_stream calls and the streaming generate calls run: `family` picks the twin of
 * rwkv_b200_test_generate_step (PLAIN: samplers, next and lp NULL), _constrained (CONSTRAINED: next needed, lp NULL), _logprobs
 * (LOGPROBS: lp needed) or _sampled (SAMPLED: samplers needed, a's temperature / top_p / penalty arrays NULL), with the arguments and
 * outputs of that hook. It runs as the one node of a graph over pinned mapped copies of the streaming words, which are freed on return:
 *   acked[n_rows]             in: 2 * tokens acknowledged + stop request, as the streaming loop's host thread writes it;
 *   published[n_rows]         in / out: step + 1 for every row that drew;
 *   stream_tokens             in / out, [n_rows][RWKV_B200_GENERATE_MAX]: the token a row drew at [b][step];
 *   ring                      in / out, [n_rows][2][2 + 2 * RWKV_B200_TOP_LOGPROBS_MAX] words, needed with lp, else NULL: slot step % 2
 *                             of a row that drew holds its log-probability, sample probability, top ids and their log-probabilities;
 *   timed_out                 out: 1 if a wait ran out.
 * A row that would draw token step > 0 with acked[b] >> 1 < step would wait for the host; the call refuses it (RWKV_ERROR_ARGS) before
 * a device is touched, so the hook never waits. A row whose acked word has the stop bit freezes without drawing. */
#define RWKV_B200_STEP_PLAIN 0
#define RWKV_B200_STEP_CONSTRAINED 1
#define RWKV_B200_STEP_LOGPROBS 2
#define RWKV_B200_STEP_SAMPLED 3
RWKV_API bool rwkv_b200_test_generate_step_streaming(const struct rwkv_b200_generate_step_args * a, int family, const struct rwkv_b200_sampler * samplers,
                                                     const uint16_t * next, size_t n_states, uint32_t * states, const struct rwkv_b200_logprobs * lp,
                                                     const uint32_t * acked, uint32_t * published, uint32_t * stream_tokens, uint32_t * ring,
                                                     uint32_t * timed_out);

/* Layer pipeline across GPUs (SURVEY.md 8e; the reference has no equivalent: ggml offloads layers of ONE context,
 * rwkv.cpp:97-116). A context created with rwkv_b200_init_from_file_ex(path, device, begin, end) is one stage; its slice
 * of the recurrent state stays resident on that device. Per pass of n_tokens (<= 256):
 *   first stage : embeds `tokens`, writes its output activations to hidden_out
 *   inner stage : reads hidden_in, writes hidden_out
 *   last stage  : reads hidden_in, computes the logits when want_logits (fetch them with rwkv_b200_stage_logits)
 * hidden_in / hidden_out are DEVICE pointers to rwkv_b200_stage_hidden_len(ctx, n_tokens) floats: x f32[n_embed x n_tokens]
 * followed, for RWKV v7, by v_first f32[n_embed x n_tokens]; the caller moves them between GPUs (NCCL send/recv or a peer
 * copy). cuda_stream (a cudaStream_t, NULL = the context's own stream) is where the pass is enqueued, so it can be ordered
 * against the transfers without host synchronisation (note that the legacy default stream's handle IS NULL: create a stream).
 * A single-stage context (all layers) accepts the call too. */
RWKV_API size_t rwkv_b200_stage_hidden_len(const struct rwkv_context * ctx, size_t n_tokens);
RWKV_API bool rwkv_b200_stage_eval(struct rwkv_context * ctx, const uint32_t * tokens, size_t n_tokens, const float * hidden_in, float * hidden_out,
                                   bool want_logits, void * cuda_stream);
RWKV_API bool rwkv_b200_stage_logits(struct rwkv_context * ctx, float * logits_out, void * cuda_stream);

/* The same pipeline with the hand-off INSIDE the library: every stage owns a mailbox in its HBM that the previous stage fills with
 * NVLink peer stores from the last kernel of its pass, and a credit word the next stage writes back (csrc/kernels/pipe.cu) -- no
 * NCCL call, no host synchronisation and no data-dependent launch parameter per token, so single-token passes keep replaying
 * their CUDA graph. Set-up (once): every stage exports a handle, the handles travel between the ranks by any means (an
 * all_gather of rwkv_b200_pipe_handle_size() bytes; NCCL / gloo are needed for nothing else), every stage connects to its
 * neighbours. One process driving several GPUs uses rwkv_b200_pipe_connect_local instead (peer access, no IPC).
 *   rwkv_b200_pipe_eval: receive (unless first stage) -> resident layers -> send (unless last stage), all enqueued on cuda_stream
 *   (NULL = the context's own). Every context of a stage shares the stage's link: enqueue a link's passes in item order on ONE
 *   stream. The last stage computes logits when asked (rwkv_b200_stage_logits fetches them). A neighbour that never shows up
 *   makes the waiting kernel trap after ~20 s instead of hanging the GPU. */
/* The whole pipeline inside ONE process, behind the plain rwkv.h entry points: rwkv_b200_init_pipeline loads one stage per listed CUDA
 * device (layer blocks balanced by bytes, the head on the last one), connects them with peer access, and returns a handle that
 * rwkv_eval / rwkv_eval_sequence / rwkv_eval_sequence_in_chunks / rwkv_clone_context / rwkv_free accept like any other: every stage
 * takes and returns its own slice of the caller's state buffer, the token ids enter stage 0, the logits leave the last stage.
 * rwkv_init_from_file does the same when the environment holds RWKV_B200_PIPELINE_DEVICES="0,1,2,3" -- an unchanged consumer of the
 * reference binding reaches several GPUs that way (capacity; clones evaluated from several threads fill the stages concurrently). */
RWKV_API struct rwkv_context * rwkv_b200_init_pipeline(const char * model_file_path, const int * devices, size_t n_devices);
RWKV_API size_t rwkv_b200_pipeline_stages(const struct rwkv_context * ctx);   /* 0 for an ordinary context */
RWKV_API void * rwkv_b200_stream(struct rwkv_context * ctx);            /* the context's own cudaStream_t */
RWKV_API size_t rwkv_b200_pipe_handle_size(void);
RWKV_API bool rwkv_b200_pipe_export(struct rwkv_context * ctx, void * handle_out);
RWKV_API bool rwkv_b200_pipe_connect(struct rwkv_context * ctx, const void * prev_handle, const void * next_handle);
RWKV_API bool rwkv_b200_pipe_connect_local(struct rwkv_context * ctx, struct rwkv_context * prev, struct rwkv_context * next);
RWKV_API bool rwkv_b200_pipe_eval(struct rwkv_context * ctx, const uint32_t * tokens, size_t n_tokens, bool want_logits, void * cuda_stream);

/* Measurement hooks. */
RWKV_API float rwkv_b200_last_device_ms(const struct rwkv_context * ctx);     /* CUDA-event time of the last pass */
RWKV_API uint64_t rwkv_b200_kernel_launch_count(void);                         /* kernels enqueued by this process */
RWKV_API uint64_t rwkv_b200_graph_launch_count(void);   /* CUDA graphs launched by this process: single-token replays, generation loops */
RWKV_API uint64_t rwkv_b200_bytes_per_token(const struct rwkv_context * ctx, bool with_logits);
/* The part of that byte model the GEMV launches of the context's decode pass stream: every layer matrix (+ the head), at file
 * precision -- except, in a single-sequence context, the v6 LoRA matrices maa_w1 / decay_w2 of the layers whose single-token pass folds
 * them into the LayerNorm-mix and WKV launches (rwkv_b200_v6_lora_fold_supported). */
RWKV_API uint64_t rwkv_b200_gemv_bytes_per_token(const struct rwkv_context * ctx, bool with_logits);
/* Times `n_steps` back-to-back resident passes of `tokens_per_step` tokens each (after `warmup_steps` untimed ones)
 * with CUDA events on the context's own stream. `tokens` holds (warmup_steps + n_steps) * tokens_per_step ids.
 * Returns the milliseconds of the timed steps, or a negative value on error. Single-token passes replay a CUDA graph. */
RWKV_API float rwkv_b200_time_resident(struct rwkv_context * ctx, const uint32_t * tokens, size_t tokens_per_step, int n_steps, int warmup_steps, bool want_logits);

/* Roofline leg: runs ONE resident pass of n_tokens with CUDA events around every fused dequantize-GEMV launch (graphs off)
 * and reports their summed duration, the algorithmic weight bytes they streamed (rwkv_tensor_nbytes of each matrix, reference
 * rwkv_utilities.inc:1-3), their count, and the duration of the whole pass. */
struct rwkv_b200_profile {
    double gemv_ms, gemv_bytes, pass_ms;
    double top_ms, top_bytes;      /* the single slowest GEMV launch of the pass */
    uint32_t gemv_launches, total_launches;
};
RWKV_API bool rwkv_b200_profile_pass(struct rwkv_context * ctx, const uint32_t * tokens, size_t n_tokens, bool want_logits, struct rwkv_b200_profile * out);

/* In-kernel timeline (stand-in for nsys): after rwkv_b200_trace_enable every kernel of a pass folds %globaltimer of its first
 * and last CTA into one record, also inside CUDA-graph replays. rwkv_b200_trace_read returns the records of the most recent
 * pass (microseconds relative to the first kernel's start, names up to 31 chars) and re-arms the buffer. */
RWKV_API bool rwkv_b200_trace_enable(struct rwkv_context * ctx);
RWKV_API void rwkv_b200_trace_disable(struct rwkv_context * ctx);      /* frees the buffer; graphs are re-captured without trace slots */
RWKV_API void rwkv_b200_trace_set_marks_buffer(double * marks_us);   /* optional [max_records][4]: intra-kernel marks of CTA 0 */
RWKV_API int rwkv_b200_trace_read(struct rwkv_context * ctx, double * start_us, double * end_us, char (*names)[32], int max_records);

/* Enables / disables CUDA-graph replay of single-token passes (on by default). */
RWKV_API void rwkv_b200_set_graphs(struct rwkv_context * ctx, bool enabled);
/* Enables / disables the wgmma tensor-core kernel for passes of >= 32 tokens (on by default; off = batch-invariant SIMT path). */
RWKV_API void rwkv_b200_set_tensor_cores(struct rwkv_context * ctx, bool enabled);

/* rwkv_eval / rwkv_eval_sequence with caller-owned HOST state: copy the state per layer group (n_layer / 4 groups, at most 8) on
 * dedicated copy streams so that the host-to-device copy of group g+1 and the device-to-host copy of group g-1 overlap the kernels
 * of group g (the ABI state layout is layer-major, so a group is one contiguous slice). Results are bit-identical to the plain
 * upload - evaluate - download order. On by default; RWKV_B200_OVERLAP=0/1 sets the default of new contexts. rwkv_eval_sequence_in_chunks
 * pipelines the upload against its first chunk and the download against its last one. */
RWKV_API void rwkv_b200_set_overlap(struct rwkv_context * ctx, bool enabled);
/* Pageable caller buffers (what the reference's bindings pass: python/rwkv_cpp/rwkv_cpp_model.py:330-351): with overlap on, a host
 * state of at least `bytes` bytes (default 4 MiB; process-wide) that is neither pinned nor device memory is copied slice by slice
 * through pinned bounce buffers of the context by two helper threads, in step with the layer groups, instead of by the driver's
 * synchronous pageable staging. Same bytes either way. RWKV_B200_NO_BOUNCE=1 turns the bounce path off. */
RWKV_API void rwkv_b200_set_bounce_min_bytes(size_t bytes);
/* Number of layer groups the overlapped path uses for this context (0 = overlap off or a single group). */
RWKV_API int rwkv_b200_overlap_groups(const struct rwkv_context * ctx);

/* Test hook: one fused dequantize-GEMV on host buffers, y[M,T] = W[M,K] . x[K,T] (column-major activations),
 * through exactly the kernel the eval path uses (csrc/kernels/gemv.cu). `weights` holds M rows in the file
 * layout of `data_type` (rwkv_file_format.inc:5-24 ids; ggml quant blocks / f16 / f32, unpadded).
 * epilogue: 0 none, 1 sigmoid, 2 silu, 3 tanh, 4 relu^2. */
RWKV_API bool rwkv_b200_matvec(int data_type, int K, int M, int T, const void * weights, const float * x, float * y, int epilogue);

/* Test hooks for the element-wise and recurrent kernels between the GEMVs (csrc/kernels/glue.cu, wkv.cu). Each runs
 * exactly the launcher the eval path calls, on host buffers: copy in, launch, synchronise, copy out. Activations are column-major
 * [dim, T] (column t = token t, contiguous). n_seq = 0 runs the kernel on T tokens of one sequence; n_seq > 0 runs it in batch mode,
 * one token of each of n_seq sequences (T must be 1, the activations have n_seq columns) on per-sequence states seq_stride floats apart.
 * Every output (outputs, states, staged columns) must have room for RWKV_B200_GUARD floats (4 * RWKV_B200_GUARD bytes) after its
 * end: the device copy is filled with 0xFF bytes (NaN) before the launch, including that guard region, and returned whole, so a
 * value the kernel never wrote and a write past the end are both visible. Optional pointers may be NULL. Staged columns (q_out,
 * written for consumers of weight type q_type; layout in csrc/kernels/act_stage.cuh) are accepted for T = 1 and n_seq = 0 only,
 * and only where the kernel emits whole 32-element blocks from whole warps: n_embed a multiple of 32 for the v4 WKV and the lerp,
 * the head size a multiple of 32 for the v5/6/7 WKV. The v5/6 WKV needs seq_stride a multiple of 4, embed_ln0 an
 * emb_pitch that is a multiple of the element size. False with RWKV_ERROR_ARGS for invalid arguments, RWKV_ERROR_CTX | UNSUPPORTED
 * when the launcher refuses the shape or the device fails. */
#define RWKV_B200_GUARD 64

/* Test hook, no device needed: M rows of K values encoded in the file layout of data_type exactly as rwkv_b200_adapter_create encodes a
 * replaced matrix before its upload (F32 copied, F16 rounded to nearest even, the quantized types by the library's quantizer, the one
 * rwkv_quantize_model_file uses). out: M * (bytes of a row of K elements). K must be a multiple of the type's block. */
RWKV_API bool rwkv_b200_test_encode_rows(int data_type, const float * values, size_t M, size_t K, void * out);

/* The shrink and expand launches of an adapter's low-rank delta (csrc/kernels/lora.cu) on host buffers, column-major [dim, T]:
 * u[:, t] = A . x[:, t] with A (rank x K, row-major) rounded to fp16, then y[:, t] = epi(z[:, t] + scale * B . u[:, t]) with B (M x rank,
 * row-major) rounded to fp16. epilogue: 0 none, 1 sigmoid, 2 silu, 4 relu^2 (z is the base product W.x), 5 add and 6 gated add (z is
 * the base's output y = res + W.x, resp. res + gate * W.x, and y = z + scale * B.u, resp. z + gate * (scale * B.u)); gate [M, T] is
 * read by 6 only. u and y are guarded outputs. 1 <= T <= 256, 1 <= rank <= 256. */
RWKV_API bool rwkv_b200_test_lora(int K, int M, int T, int rank, float scale, int epilogue, const float * a, const float * b, const float * x,
                                  const float * z, const float * gate, float * u, float * y);

/* x[:, t] = LN(emb[tokens[t]]; ln0). emb: n_vocab rows of emb_pitch bytes, F32 or F16 (emb_type 0 / 1). */
RWKV_API bool rwkv_b200_test_embed_ln0(const void * emb, int emb_type, size_t emb_pitch, int n_vocab, const int * tokens, int T, int C,
                                       const float * ln_w, const float * ln_b, float * x);

/* y[:, t] = LN(x[:, t]; w, b) for t < T (launch_layer_norm_columns: the LayerNorm of the tensor-core head of scoring passes).
 * x, y: [C, T]; T at most 256, the columns of one pass. */
RWKV_API bool rwkv_b200_test_layer_norm_columns(const float * x, const float * w, const float * b, int C, int T, float * y);

/* LayerNorm + token shift + mix (launch_ln_mix). formula 0: out_j = xx*m_j + (prev - prev*m_j);
 * formula 1: out_j = (prev - xx)*m_j + xx. state_in / state_out: the carried LN(x) of the previous token, [C] per sequence. */
struct rwkv_b200_ln_mix_args {
    const float * x, * ln_w, * ln_b, * state_in;
    float * state_out;
    int C, T, formula, n_out;
    const float * coef[6];
    float * out[6];
    float * out_xx, * out_sx;        /* optional: LN(x), prev - LN(x) */
    int n_seq;
    long long seq_stride;
};
RWKV_API bool rwkv_b200_test_ln_mix(const struct rwkv_b200_ln_mix_args * a);

/* v6 data-dependent lerp (launch_v6_lerp): out_j = (W2[j] . z[j*mix .. +mix, t] + maa_j) * sx + xx for j in w, k, v, r, g.
 * w2: [5][C][mix]; z: [5*mix, T]. q_out: all five or none. */
struct rwkv_b200_v6_lerp_args {
    const float * w2, * z, * xx, * sx;
    const float * maa[5];
    float * out[5];
    int C, T, mix;
    unsigned char * q_out[5];
    int q_type[5];
};
RWKV_API bool rwkv_b200_test_v6_lerp(const struct rwkv_b200_v6_lerp_args * a);

/* v4 WKV with the r* multiply (launch_wkv4). aa / bb / pp: [C] per sequence. */
struct rwkv_b200_wkv4_args {
    const float * k, * v, * r, * time_first, * time_decay;
    const float * aa_in, * bb_in, * pp_in;
    float * aa_out, * bb_out, * pp_out, * y;
    int C, T;
    unsigned char * q_out;
    int q_type;
    int n_seq;
    long long seq_stride;
};
RWKV_API bool rwkv_b200_test_wkv4(const struct rwkv_b200_wkv4_args * a);

/* v5 / v6 WKV + head norm + ln_x + gate (launch_wkv6). td: [C, T] when td_per_token, else [H] when
 * per_head_scalars, else [C]; tf: [H] when per_head_scalars, else [C]. State [H][S][S] per sequence. g optional. */
struct rwkv_b200_wkv6_args {
    const float * r, * k, * v, * td, * tf;
    int td_per_token, per_head_scalars;
    const float * state_in;
    float * state_out;
    const float * lnx_w, * lnx_b, * g;
    float * y;
    float eps;
    int H, S, T;
    unsigned char * q_out;
    int q_type;
    int n_seq;
    long long seq_stride;
};
RWKV_API bool rwkv_b200_test_wkv6(const struct rwkv_b200_wkv6_args * a);

/* v7 WKV with kk / k / v corrections, head norm, ln_x, bonus and gate (launch_wkv7). vgate NULL = layer 0
 * (v_first ignored); v_out optional. State [H][S][S] per sequence. */
struct rwkv_b200_wkv7_args {
    const float * r, * w, * k, * v, * a, * g, * vgate, * v_first;
    float * v_out;
    const float * k_k, * k_a, * r_k, * lnx_w, * lnx_b, * state_in;
    float * state_out, * y;
    int H, S, T;
    unsigned char * q_out;
    int q_type;
    int n_seq;
    long long seq_stride;
};
RWKV_API bool rwkv_b200_test_wkv7(const struct rwkv_b200_wkv7_args * a);

/* The same four kernels in ragged mode (the mode of rwkv_b200_batch_eval_ragged): sequence s advances counts[s] tokens, its columns
 * back to back in sequence order, on its state seq_stride floats after sequence s - 1's. The struct's T is the sum of the counts (the
 * activations' columns), its n_seq equals n_seq (1 .. 256), its seq_stride is at least one sequence's state; no staged columns.
 * A sequence with no tokens is not touched: its state_out slice keeps the 0xFF fill. */
RWKV_API bool rwkv_b200_test_ln_mix_ragged(const struct rwkv_b200_ln_mix_args * a, const uint32_t * counts, size_t n_seq);
RWKV_API bool rwkv_b200_test_wkv4_ragged(const struct rwkv_b200_wkv4_args * a, const uint32_t * counts, size_t n_seq);
RWKV_API bool rwkv_b200_test_wkv6_ragged(const struct rwkv_b200_wkv6_args * a, const uint32_t * counts, size_t n_seq);
RWKV_API bool rwkv_b200_test_wkv7_ragged(const struct rwkv_b200_wkv7_args * a, const uint32_t * counts, size_t n_seq);

/* A batch of up to 8 matrix problems y_i[M_i, T] = epi_i(W_i . pro_i(x[input_i])) launched the way the eval path launches them
 * (csrc/kernels/gemv.h). Weights go up through the model loader's code (row pitch, zeroed row padding, device layout, and the
 * tile-major tensor-core copy when `tiled` is set). Problems whose `input` index is the same share one device input, as the
 * mixed inputs of a layer do. epi: 0 none, 1 sigmoid, 2 silu, 3 tanh, 4 relu^2, 5 res + v, 6 res + gate * v, 7 exp(-exp(v + bias)),
 * 8 sigmoid(v + bias), 9 exp(-0.606531 * sigmoid(v + bias)); res / gate [M, T], bias [M]. pro 1: LayerNorm of the input (ln_w,
 * ln_b [K], eps 1e-5). y_aliases_res: the device y starts as a copy of res and is also the residual the kernel reads (x += ...).
 * xq: the input's column already staged for this problem's weight type (csrc/kernels/act_stage.cuh layout), T = 1 only.
 * Outputs need RWKV_B200_GUARD floats of room after their end, as for the hooks above.
 * path: */
#define RWKV_B200_GEMV_ENGINE 0            /* single-sequence context: tensor cores for T >= 32, the rest through the GEMV */
#define RWKV_B200_GEMV_ENGINE_BATCH_CTX 1  /* batch context: tensor cores from T >= 16 */
#define RWKV_B200_GEMV_STREAMING 2         /* the TMA streaming GEMV only (CTX | UNSUPPORTED if a shape does not fit it) */
#define RWKV_B200_GEMV_GENERIC 3           /* the generic GEMV only */
#define RWKV_B200_GEMV_TENSOR_CORES 4      /* the tensor-core GEMM only (CTX | UNSUPPORTED unless every problem can take it) */
struct rwkv_b200_gemv_problem {
    int type, K, M;
    const void * weights;                  /* M rows in the file layout of `type`, unpadded */
    int tiled;
    int input;                             /* 0 .. 7: which x[] */
    int epi, pro;
    const float * res, * gate, * bias, * ln_w, * ln_b;
    const unsigned char * xq;
    int y_aliases_res;
    float * y;
};
/* One kernel launch: family 0 streaming GEMV, 1 generic GEMV, 2 tensor-core GEMM, 3 fp16 operand conversion, 4 tensor-core weight
 * expansion (of the upload), 5 Q4_K / Q5_K streaming GEMV, 6 Q4_K / Q5_K tensor-core weight expansion; a conversion of
 * Q8_K operands (K-quant weights) reports only = 16. nc: columns per group (streaming, generic, K-quant) or distinct inputs
 * (conversion); only: the streaming kernel's single weight type (-1: mixed), the expanded type or the K-quant type; has_ln: the streaming kernel's LayerNorm code; npad: tokens padded
 * to 16; cluster: CTAs per cluster of the GEMM. */
struct rwkv_b200_gemv_launch { int family, nc, only, has_ln, npad, cluster; };
struct rwkv_b200_gemv_batch_args {
    int T, n, path;
    const float * x[8];                    /* [K, T] column-major, K of the problems that read it */
    struct rwkv_b200_gemv_problem p[8];
    struct rwkv_b200_gemv_launch * launches;   /* optional record, max_launches entries; *n_launches = entries written */
    int max_launches;
    int * n_launches;
};
RWKV_API bool rwkv_b200_test_gemv_batch(const struct rwkv_b200_gemv_batch_args * a);

/* The v6 fold of single-token passes of single-sequence contexts: does a layer of this shape run maa_w1 (5 * mix rows of n_embed, type
 * w1_type) inside the LayerNorm-mix launch and decay_w2 (n_embed rows of `decay`, type w2_type) inside the WKV launch? Shapes only, no
 * device. Otherwise the layer runs the two GEMV launches. */
RWKV_API bool rwkv_b200_v6_lora_fold_supported(int n_embed, int head_size, int w1_type, int mix, int w2_type, int decay);

/* The two folded kernels on host buffers. Arguments outside what rwkv_b200_v6_lora_fold_supported admits are rejected (ARGS) before any
 * device is touched. Weights are in the file layout of their type, unpadded.
 * v6 prologue (launch_v6_prologue): ln_mix of one token, formula 1, one mix vector `coef` (state_out, out_xx, out_sx [C]), then
 * y1[M1] = tanh(W1 . mix), W1 [M1, C]; equal to rwkv_b200_test_ln_mix followed by rwkv_b200_test_gemv_batch (epi 3) on its out0. */
struct rwkv_b200_v6_prologue_args {
    const float * x, * ln_w, * ln_b, * state_in, * coef;
    float * state_out, * out_xx, * out_sx;
    const void * w1;
    int w1_type, M1;
    float * y1;
    int C;
};
RWKV_API bool rwkv_b200_test_v6_prologue(const struct rwkv_b200_v6_prologue_args * a);
/* wkv6 of one token of one sequence with head size 64 whose decay is exp(-exp(W2 . lora1 + td_bias)), W2 [C, K2]: equal to
 * rwkv_b200_test_gemv_batch (epi 7) followed by rwkv_b200_test_wkv6 with td_per_token. Other fields as in rwkv_b200_wkv6_args. */
struct rwkv_b200_wkv6_decay_args {
    const float * r, * k, * v, * tf, * state_in;
    float * state_out;
    const float * lnx_w, * lnx_b, * g;
    float * y;
    float eps;
    int H;
    const void * w2;
    int w2_type, K2;
    const float * lora1, * td_bias;
    unsigned char * q_out;
    int q_type;
};
RWKV_API bool rwkv_b200_test_wkv6_decay(const struct rwkv_b200_wkv6_decay_args * a);

#if defined(__cplusplus)
}
#endif
#endif /* RWKV_B200_H */
