/* rwkv.h -- C ABI of the H100-native RWKV engine (librwkv.so).
 *
 * Drop-in for the evaluation path of RWKV/rwkv.cpp: every symbol, signature, enum value and
 * ownership rule below is the one the reference exports (reference rwkv.h:23-221 plus the two
 * legacy getters defined in rwkv.cpp:145,151), so its C tests, its ctypes binding
 * (python/rwkv_cpp/rwkv_cpp_shared_library.py:49-107) and third-party Go/Node bindings load this
 * library unchanged. The implementation behind it is new: C++ host code + sm_90a CUDA kernels,
 * no ggml graph, no CPU fallback.
 *
 * Differences a caller can observe (all within what the reference header leaves unspecified):
 *   - n_threads is accepted and ignored (must still be > 0 to mirror the documented contract);
 *   - n_gpu_layers is accepted and ignored: all layers always run on the GPU;
 *   - a missing / unusable CUDA device makes rwkv_init_from_file return NULL with
 *     RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED -- there is no host execution path;
 *   - rwkv_get_system_info_string describes the CUDA device instead of CPU features;
 *   - tensor data types: FP32, FP16, Q4_0, Q4_1, Q4_K, Q5_0, Q5_1, Q5_K, Q8_0 -- the formats the reference's Python binding
 *     offers. The reference's type table (rwkv_file_format.inc:28-47) also lets ggml's Q8_1, Q2_K, Q3_K, Q6_K and Q8_K ids
 *     (10, 11, 12, 15, 16) through; a file that contains such a tensor is refused by rwkv_init_from_file with
 *     RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_UNSUPPORTED, and rwkv_quantize_model_file refuses those format names with
 *     RWKV_ERROR_ARGS | RWKV_ERROR_DATA_TYPE. The same load error covers a Q4_K / Q5_K emb.weight or head.weight and a Q4_K /
 *     Q5_K tensor whose rows are not multiples of 256 weights.
 */
#ifndef RWKV_H
#define RWKV_H

#include <stddef.h>
#include <stdint.h>
#include <stdbool.h>

#if defined(RWKV_SHARED)
#  if defined(_WIN32) && !defined(__MINGW32__)
#    if defined(RWKV_BUILD)
#      define RWKV_API __declspec(dllexport)
#    else
#      define RWKV_API __declspec(dllimport)
#    endif
#  else
#    define RWKV_API __attribute__((visibility("default")))
#  endif
#else
#  define RWKV_API
#endif

/* File container constants (reference rwkv.h:23-31, docs/FILE_FORMAT.md). 'ggmf'. */
#define RWKV_FILE_MAGIC 0x67676d66
#define RWKV_FILE_VERSION_0 100
#define RWKV_FILE_VERSION_1 101
#define RWKV_FILE_VERSION_MIN RWKV_FILE_VERSION_0
#define RWKV_FILE_VERSION_MAX RWKV_FILE_VERSION_1
#define RWKV_FILE_VERSION RWKV_FILE_VERSION_MAX

#if defined(__cplusplus)
extern "C" {
#endif

/* Error word = OR of one category (bits 8+) and one code (low byte); reference rwkv.h:38-62. */
enum rwkv_error_flags {
    RWKV_ERROR_NONE = 0,

    RWKV_ERROR_ARGS = 1 << 8,
    RWKV_ERROR_FILE = 2 << 8,
    RWKV_ERROR_MODEL = 3 << 8,
    RWKV_ERROR_MODEL_PARAMS = 4 << 8,
    RWKV_ERROR_GRAPH = 5 << 8,
    RWKV_ERROR_CTX = 6 << 8,

    RWKV_ERROR_ALLOC = 1,
    RWKV_ERROR_FILE_OPEN = 2,
    RWKV_ERROR_FILE_STAT = 3,
    RWKV_ERROR_FILE_READ = 4,
    RWKV_ERROR_FILE_WRITE = 5,
    RWKV_ERROR_FILE_MAGIC = 6,
    RWKV_ERROR_FILE_VERSION = 7,
    RWKV_ERROR_DATA_TYPE = 8,
    RWKV_ERROR_UNSUPPORTED = 9,
    RWKV_ERROR_SHAPE = 10,
    RWKV_ERROR_DIMENSION = 11,
    RWKV_ERROR_KEY = 12,
    RWKV_ERROR_DATA = 13,
    RWKV_ERROR_PARAM_MISSING = 14
};

/* Opaque inference context: one CUDA stream + activation arena + device state, sharing read-only
 * weights with its clones. A context may move between host threads between calls; one eval at a
 * time per context (reference rwkv.h:64-68, 94-96). */
struct rwkv_context;

/* replaces rwkv.h:76 -- ctx==NULL addresses the calling thread's global flag (load/quantize errors
 * and the default inherited by new contexts). */
RWKV_API void rwkv_set_print_errors(struct rwkv_context * ctx, const bool print_errors);
/* replaces rwkv.h:80 */
RWKV_API bool rwkv_get_print_errors(const struct rwkv_context * ctx);
/* replaces rwkv.h:84 -- returns the accumulated flags and clears them. */
RWKV_API enum rwkv_error_flags rwkv_get_last_error(struct rwkv_context * ctx);

/* replaces rwkv.h:91 (rwkv.cpp:71). Reads a ggml-format RWKV file (v4/v5.1/v5.2/v6/v7; FP32, FP16,
 * Q4_0, Q4_1, Q4_K, Q5_0, Q5_1, Q5_K, Q8_0 per tensor), uploads every tensor to HBM. NULL on error. */
RWKV_API struct rwkv_context * rwkv_init_from_file(const char * model_file_path, const uint32_t n_threads, const uint32_t n_gpu_layers);

/* replaces rwkv.h:99 (rwkv.cpp:123). New stream/arena/state over the same weights (atomic refcount). */
RWKV_API struct rwkv_context * rwkv_clone_context(struct rwkv_context * ctx, const uint32_t n_threads);

/* replaces rwkv.h:109 (rwkv_eval.inc:38). Buffers are caller-owned host fp32:
 *   state_in   rwkv_get_state_len() floats, or NULL for a fresh state;
 *   state_out  same length, written if non-NULL; may alias state_in;
 *   logits_out rwkv_get_logits_len() floats; NULL skips ln_out + head entirely.
 * false + RWKV_ERROR_ARGS if token >= n_vocab. */
RWKV_API bool rwkv_eval(struct rwkv_context * ctx, const uint32_t token, const float * state_in, float * state_out, float * logits_out);

/* replaces rwkv.h:140 (rwkv_eval.inc:79). State after all tokens, logits of the last one.
 * tokens==NULL is a warm-up that executes nothing. Any sequence_len > 0 is accepted (there is no
 * graph-node limit here); results equal token-by-token rwkv_eval. */
RWKV_API bool rwkv_eval_sequence(struct rwkv_context * ctx, const uint32_t * tokens, const size_t sequence_len, const float * state_in, float * state_out, float * logits_out);

/* replaces rwkv.h:165 (rwkv_eval.inc:158). The state stays in HBM between chunks. */
RWKV_API bool rwkv_eval_sequence_in_chunks(struct rwkv_context * ctx, const uint32_t * tokens, const size_t sequence_len, const size_t chunk_size, const float * state_in, float * state_out, float * logits_out);

/* replace rwkv.h:177,181,187,191,195 (rwkv.cpp:156-184). */
RWKV_API size_t rwkv_get_n_vocab(const struct rwkv_context * ctx);
RWKV_API size_t rwkv_get_n_embed(const struct rwkv_context * ctx);
RWKV_API size_t rwkv_get_n_layer(const struct rwkv_context * ctx);
RWKV_API size_t rwkv_get_state_len(const struct rwkv_context * ctx);
RWKV_API size_t rwkv_get_logits_len(const struct rwkv_context * ctx);

/* Legacy names still used by the reference's Python binding (rwkv.cpp:145,151;
 * rwkv_cpp_shared_library.py:91-95). Not declared in the reference header either. */
RWKV_API uint32_t rwkv_get_state_buffer_element_count(const struct rwkv_context * ctx);
RWKV_API uint32_t rwkv_get_logits_buffer_element_count(const struct rwkv_context * ctx);

/* replaces rwkv.h:201 (rwkv_eval.inc:224). Zeros; v4 `pp` slots = -1e30. Equivalent to state_in==NULL. */
RWKV_API void rwkv_init_state(const struct rwkv_context * ctx, float * state);

/* replaces rwkv.h:205 (rwkv.cpp:187). NULL-safe; the last context of a model releases the weights. */
RWKV_API void rwkv_free(struct rwkv_context * ctx);

/* replaces rwkv.h:218 (rwkv_quantize.inc:16). Host-side, bit-identical to ggml's quantize_row_*_ref
 * (ggml-quants.c:31-217, 1208-1480). format_name in {Q4_0, Q4_1, Q4_K, Q5_0, Q5_1, Q5_K, Q8_0}. A Q4_K / Q5_K tensor whose rows
 * are not multiples of 256 weights is written as Q5_0 / Q5_1 (the reference writes super-blocks that straddle rows there). */
RWKV_API bool rwkv_quantize_model_file(const char * model_file_path_in, const char * model_file_path_out, const char * format_name);

/* replaces rwkv.h:221 (rwkv.cpp:239). Static storage. */
RWKV_API const char * rwkv_get_system_info_string(void);

#if defined(__cplusplus)
}
#endif

#endif /* RWKV_H */
