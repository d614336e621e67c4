// The rwkv.h C ABI over the H100 engine, plus the additive rwkv_b200_* entry points.
// Argument checks, error categories and NULL conventions follow the reference entry points
// (rwkv.cpp:71-258, rwkv_eval.inc:38-241) so its C tests run unchanged against this library.
#include <algorithm>
#include <cinttypes>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/rwkv.h"
#include "../../include/rwkv_b200.h"
#include "engine.h"
#include "kernels/act_stage.cuh"
#include "kernels/ops.h"
#include "quantizer.h"

using namespace rwkv;

// The opaque handle of the C API is the engine's Context.
struct rwkv_context : public rwkv::Context {};

static inline Context * C(struct rwkv_context * c) { return static_cast<Context *>(c); }
static inline const Context * C(const struct rwkv_context * c) { return static_cast<const Context *>(c); }

static int default_device() {
    const char * e = getenv("RWKV_B200_DEVICE");
    return e ? atoi(e) : 0;
}

namespace {

// Device copies of a kernel test hook's host buffers. Inputs are copied in; outputs get a guard region of RWKV_B200_GUARD floats
// after their end, are filled with 0xFF bytes (NaN) before the launch and copied back whole, guard included. NULL host pointers stay
// NULL on the device.
struct HookBuffers {
    struct Out { void * dev; void * host; size_t bytes; };
    std::vector<void *> allocs;
    std::vector<Out> outs;
    bool ok = true;

    void * alloc(size_t bytes) {
        void * d = nullptr;
        if (ok) ok = cudaMalloc(&d, bytes) == cudaSuccess;
        if (ok) allocs.push_back(d);
        return ok ? d : nullptr;
    }
    template <class T> const T * in(const T * host, size_t n) {
        if (!host) return nullptr;
        void * d = alloc(n * sizeof(T));
        if (ok) ok = cudaMemcpy(d, host, n * sizeof(T), cudaMemcpyHostToDevice) == cudaSuccess;
        return static_cast<const T *>(d);
    }
    template <class T> T * out(T * host, size_t n) {
        if (!host) return nullptr;
        const size_t bytes = n * sizeof(T) + RWKV_B200_GUARD * sizeof(float);
        void * d = alloc(bytes);
        if (ok) ok = cudaMemset(d, 0xFF, bytes) == cudaSuccess;
        if (ok) outs.push_back(Out{d, host, bytes});
        return static_cast<T *>(d);
    }
    // An output that starts as a copy of `init` (a buffer the kernel updates in place); guard and return as for out().
    template <class T> T * inout(const T * init, T * host, size_t n) {
        T * d = out(host, n);
        if (ok && d) ok = cudaMemcpy(d, init, n * sizeof(T), cudaMemcpyHostToDevice) == cudaSuccess;
        return d;
    }
    // After the launch: wait for it and return every output to the host. The launch error, if any, is what gets reported.
    bool finish(cudaError_t launch) {
        ok = ok && launch == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess;
        for (const Out & o : outs)
            if (ok) ok = cudaMemcpy(o.host, o.dev, o.bytes, cudaMemcpyDeviceToHost) == cudaSuccess;
        return ok;
    }
    ~HookBuffers() { for (void * d : allocs) cudaFree(d); }
};

// The device every test hook runs on; false (and the flags set) without one.
bool hook_device(ErrorSink sink) {
    int dev = default_device(), n_dev = 0;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, cudaGetDeviceCount(&n_dev) == cudaSuccess && dev < n_dev && cudaSetDevice(dev) == cudaSuccess,
               "No usable CUDA device; this engine has no CPU execution path");
    return true;
}

// Shape of a state or activation set: n_seq = 0 -> one, else n_seq sequences seq_stride floats apart, each per_seq floats long.
bool seq_layout_ok(int n_seq, long long seq_stride, int T, size_t per_seq) {
    return n_seq == 0 || (n_seq > 0 && T == 1 && seq_stride >= (long long) per_seq);
}
size_t seq_floats(int n_seq, long long seq_stride, size_t per_seq) {
    return n_seq > 0 ? (size_t) (n_seq - 1) * (size_t) seq_stride + per_seq : per_seq;
}

// A staged column may be requested only where the kernels emit one: single-token, single-sequence passes in which every emitting
// warp is whole and owns whole 32-blocks of the vector. `unit` is what one warp-aligned group of threads covers: the whole vector
// for the v4 WKV and the lerp (one thread per channel), one head (S) for the v5/6/7 WKV (act::warp_emit_block uses full-warp
// reductions, and with S % 32 != 0 a block would straddle two heads' CTAs).
bool staged_ok(const unsigned char * q_out, int q_type, int T, int n_seq, int unit) {
    return !q_out || (T == 1 && n_seq == 0 && unit % 32 == 0 && act::stage_class(q_type) != act::SC_NONE);
}

// Ragged hooks: counts[n_seq] with 1 <= n_seq <= MAX_TOKENS_PER_PASS, the struct's n_seq equal to n_seq, its T the sum of the counts
// (the activations' columns), its seq_stride at least one sequence's state.
bool ragged_ok(const uint32_t * counts, size_t n_seq, int a_n_seq, int T, long long seq_stride, size_t per_seq) {
    if (!counts || n_seq < 1 || n_seq > (size_t) MAX_TOKENS_PER_PASS || a_n_seq != (int) n_seq || T < 1 || seq_stride < (long long) per_seq) return false;
    size_t sum = 0;
    for (size_t s = 0; s < n_seq; s++) sum += counts[s];
    return sum == (size_t) T;
}
// The device map of a ragged launch: column offsets [n_seq + 1] and the sequence of every column.
struct RaggedMap {
    std::vector<int> off, col_seq;
    RaggedMap(const uint32_t * counts, size_t n_seq) : off(n_seq + 1, 0) {
        for (size_t s = 0; s < n_seq; s++) {
            off[s + 1] = off[s] + (int) counts[s];
            col_seq.insert(col_seq.end(), counts[s], (int) s);
        }
    }
};

}  // namespace

// Entry points that enqueue work on a context's stream, or wait on it, refuse while a streaming generation of that context calls
// its callback: the device waits for that callback to return, so the work would deadlock against it. Nothing is enqueued.
#define RWKV_NOT_STREAMING(c) RWKV_CHECK((c)->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, !(c)->in_stream, \
                                         "This context is inside a streaming generation; use another context from its callback")

extern "C" {

struct rwkv_context * rwkv_b200_init_from_file_ex(const char * file_path, int device, int layer_begin, int layer_end) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, file_path != nullptr, "Model file path is NULL");
    Model * model = load_model(file_path, device, layer_begin, layer_end, sink);
    RWKV_PROPAGATE(sink, nullptr, model != nullptr);
    Context * ctx = create_context(model, sink);   // deletes the model itself on failure
    RWKV_PROPAGATE(sink, nullptr, ctx != nullptr);
    return static_cast<struct rwkv_context *>(ctx);
}

// RWKV_B200_PIPELINE_DEVICES="0,1,2,3": one stage per listed CUDA device (a device may repeat), all inside this process
static std::vector<int> pipeline_devices() {
    std::vector<int> d;
    const char * e = getenv("RWKV_B200_PIPELINE_DEVICES");
    if (!e) return d;
    for (const char * p = e; *p;) {
        char * end = nullptr;
        const long v = strtol(p, &end, 10);
        if (end == p) break;
        d.push_back((int) v);
        p = *end == ',' ? end + 1 : end;
    }
    return d;
}

struct rwkv_context * rwkv_b200_init_pipeline(const char * file_path, const int * devices, size_t n_devices) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, file_path && devices && n_devices >= 2, "A pipeline needs a model file and at least two devices");
    Context * head = create_pipeline(file_path, std::vector<int>(devices, devices + n_devices), sink);
    RWKV_PROPAGATE(sink, nullptr, head != nullptr);
    return static_cast<struct rwkv_context *>(head);
}

size_t rwkv_b200_pipeline_stages(const struct rwkv_context * ctx) { return ctx && C(ctx)->group ? C(ctx)->stages.size() + 1 : 0; }

static bool whole_model(const Context * c) {
    return (c->group || (c->model->layer_begin == 0 && c->model->layer_end == c->model->n_layer)) && c->batch_n == 0;
}

struct rwkv_context * rwkv_init_from_file(const char * file_path, const uint32_t n_threads, const uint32_t n_gpu_layers) {
    (void) n_gpu_layers;   // every layer always lives on the GPU
    const std::vector<int> devs = pipeline_devices();
    struct rwkv_context * ctx = devs.size() >= 2 ? rwkv_b200_init_pipeline(file_path, devs.data(), devs.size())
                                                 : rwkv_b200_init_from_file_ex(file_path, default_device(), 0, -1);
    if (ctx) C(ctx)->n_threads = n_threads;
    return ctx;
}

struct rwkv_context * rwkv_clone_context(struct rwkv_context * ctx, const uint32_t n_threads) {
    if (!ctx) return nullptr;
    bool print = C(ctx)->print_errors;
    int flags = 0;
    ErrorSink sink{&flags, &print};
    Context * clone = C(ctx)->group ? clone_pipeline(C(ctx), sink) : create_context(C(ctx)->model, sink);
    if (!clone) { g_last_error |= flags; return nullptr; }
    clone->n_threads = n_threads;
    clone->print_errors = C(ctx)->print_errors;
    return static_cast<struct rwkv_context *>(clone);
}

bool rwkv_eval(struct rwkv_context * ctx, const uint32_t token, const float * state_in, float * state_out, float * logits_out) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    const size_t n_vocab = (size_t) c->model->n_vocab;
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, token < n_vocab, "Token (%" PRIu32 ") is out of range (0 .. %zu)", token, n_vocab - 1);
    RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, whole_model(c),
               "This context holds only a pipeline stage or is a batch context; use the rwkv_b200 stage / batch API");
    if (c->group) return pipeline_eval_host(c, &token, 1, 0, state_in, state_out, logits_out);
    return eval_host(c, &token, 1, state_in, state_out, logits_out);
}

bool rwkv_eval_sequence(struct rwkv_context * ctx, const uint32_t * sequence, const size_t sequence_len, const float * state_in, float * state_out, float * logits_out) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, sequence_len > 0, "Sequence length is 0");
    if (!sequence) return true;   // "build the graph only" in the reference (rwkv_eval.inc:122); nothing to build here
    const size_t n_vocab = (size_t) c->model->n_vocab;
    for (size_t i = 0; i < sequence_len; i++)
        RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, sequence[i] < n_vocab, "Token at index %zu (%" PRIu32 ") is out of range (0 .. %zu)", i, sequence[i], n_vocab - 1);
    RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, whole_model(c),
               "This context holds only a pipeline stage or is a batch context; use the rwkv_b200 stage / batch API");
    if (c->group) return pipeline_eval_host(c, sequence, sequence_len, 0, state_in, state_out, logits_out);
    return eval_host(c, sequence, sequence_len, state_in, state_out, logits_out);
}

bool rwkv_eval_sequence_in_chunks(struct rwkv_context * ctx, const uint32_t * tokens, const size_t sequence_len, const size_t chunk_size,
                                  const float * state_in, float * state_out, float * logits_out) {
    Context * c = C(ctx);
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, sequence_len > 0, "Sequence length is 0");
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, chunk_size > 0, "Chunk size is 0");
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    if (!tokens) return true;
    const size_t n_vocab = (size_t) c->model->n_vocab;
    for (size_t i = 0; i < sequence_len; i++)
        RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, tokens[i] < n_vocab, "Token at index %zu (%" PRIu32 ") is out of range (0 .. %zu)", i, tokens[i], n_vocab - 1);
    RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, whole_model(c),
               "This context holds only a pipeline stage or is a batch context; use the rwkv_b200 stage / batch API");
    if (c->group) return pipeline_eval_host(c, tokens, sequence_len, chunk_size, state_in, state_out, logits_out);
    return eval_host_chunks(c, tokens, sequence_len, chunk_size, state_in, state_out, logits_out);
}

size_t rwkv_get_n_vocab(const struct rwkv_context * ctx) { return (size_t) C(ctx)->model->n_vocab; }
size_t rwkv_get_n_embed(const struct rwkv_context * ctx) { return (size_t) C(ctx)->model->n_embed; }
size_t rwkv_get_n_layer(const struct rwkv_context * ctx) { return (size_t) C(ctx)->model->n_layer; }
size_t rwkv_get_state_len(const struct rwkv_context * ctx) { return C(ctx)->model->state_len(); }
size_t rwkv_get_logits_len(const struct rwkv_context * ctx) { return (size_t) C(ctx)->model->n_vocab; }
uint32_t rwkv_get_state_buffer_element_count(const struct rwkv_context * ctx) { return (uint32_t) rwkv_get_state_len(ctx); }
uint32_t rwkv_get_logits_buffer_element_count(const struct rwkv_context * ctx) { return (uint32_t) rwkv_get_logits_len(ctx); }

void rwkv_init_state(const struct rwkv_context * ctx, float * state) { fill_init_state(*C(ctx)->model, state); }

void rwkv_free(struct rwkv_context * ctx) {
    if (!ctx) return;
    destroy_context(C(ctx));
}

void rwkv_set_print_errors(struct rwkv_context * ctx, const bool print_errors) {
    if (ctx) C(ctx)->print_errors = print_errors; else g_print_errors = print_errors;
}
bool rwkv_get_print_errors(const struct rwkv_context * ctx) { return ctx ? C(ctx)->print_errors : g_print_errors; }
enum rwkv_error_flags rwkv_get_last_error(struct rwkv_context * ctx) {
    int * p = ctx ? &C(ctx)->last_error : &g_last_error;
    int v = *p;
    *p = RWKV_ERROR_NONE;
    return (enum rwkv_error_flags) v;
}

bool rwkv_quantize_model_file(const char * in_path, const char * out_path, const char * format_name) {
    g_last_error = RWKV_ERROR_NONE;
    return quantize_model_file(in_path, out_path, format_name, global_sink());
}

const char * rwkv_get_system_info_string(void) {
    static std::string s;
    if (s.empty()) {
        s = "RWKV_B200=1 ARCH=sm_90a";
        int n = 0;
        if (cudaGetDeviceCount(&n) == cudaSuccess && n > 0) {
            cudaDeviceProp p;
            int drv = 0, rt = 0;
            cudaDriverGetVersion(&drv); cudaRuntimeGetVersion(&rt);
            if (cudaGetDeviceProperties(&p, default_device() < n ? default_device() : 0) == cudaSuccess) {
                s += " CUDA_DEVICES=" + std::to_string(n) + " DEVICE=\"" + p.name + "\" SM=" + std::to_string(p.major) + std::to_string(p.minor) +
                     " SMS=" + std::to_string(p.multiProcessorCount) + " HBM_GB=" + std::to_string((unsigned long long) (p.totalGlobalMem >> 30)) +
                     " DRIVER=" + std::to_string(drv) + " RUNTIME=" + std::to_string(rt);
            }
        } else {
            s += " CUDA_DEVICES=0";
        }
    }
    return s.c_str();
}

// ---- additive entry points (include/rwkv_b200.h) ----------------------------------------------------

bool rwkv_b200_inspect_file(const char * path, struct rwkv_b200_file_info * out) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, path && out, "NULL argument");
    ModelFile mf;
    RWKV_PROPAGATE(sink, false, scan_model_file(path, mf, sink));
    memset(out, 0, sizeof(*out));
    out->version = mf.header.version; out->n_vocab = mf.header.n_vocab; out->n_embed = mf.header.n_embed;
    out->n_layer = mf.header.n_layer; out->data_type = mf.header.data_type;
    out->n_tensors = mf.tensors.size(); out->file_size = mf.file_size;
    out->arch_major = 4; out->arch_minor = 0;
    if (mf.find("blocks.0.att.ln_x.weight")) { out->arch_major = 5; out->arch_minor = mf.find("blocks.0.att.gate.weight") ? 2 : 1; }
    if (mf.find("blocks.0.att.time_maa_x")) { out->arch_major = 6; out->arch_minor = 0; }
    if (mf.find("blocks.0.att.r_k")) { out->arch_major = 7; out->arch_minor = 0; }
    if (out->arch_major == 7) out->head_count = (uint32_t) mf.find("blocks.0.att.r_k")->ne[1];
    else if (out->arch_major >= 5) {
        const TensorInfo * td = mf.find("blocks.0.att.time_decay");
        RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_PARAM_MISSING, false, td, "Model parameter blocks.0.att.time_decay not found");
        out->head_count = (uint32_t) td->ne[2];
    }
    if (out->head_count) out->head_size = out->n_embed / out->head_count;
    out->state_len = (uint64_t) out->n_embed * (out->arch_major >= 5 ? 2 + out->head_size : 5) * out->n_layer;
    uint64_t bytes = 0;
    for (const TensorInfo & t : mf.tensors) bytes += (t.name == "emb.weight") ? t.nbytes / t.ne[1] : t.nbytes;
    out->bytes_per_token = bytes + 2 * 4 * out->state_len;
    return true;
}

bool rwkv_b200_state_load(struct rwkv_context * ctx, const float * state_in) {
    C(ctx)->last_error = 0;
    RWKV_NOT_STREAMING(C(ctx));
    return C(ctx)->batch_n == 0 && upload_state(C(ctx), state_in);
}
bool rwkv_b200_state_store(struct rwkv_context * ctx, float * state_out) {
    RWKV_NOT_STREAMING(C(ctx));
    return C(ctx)->batch_n == 0 && download_outputs(C(ctx), state_out, nullptr);
}
bool rwkv_b200_synchronize(struct rwkv_context * ctx) {
    RWKV_NOT_STREAMING(C(ctx));
    return download_outputs(C(ctx), nullptr, nullptr);
}

bool rwkv_b200_eval_resident(struct rwkv_context * ctx, const uint32_t * tokens, size_t n_tokens, bool want_logits, float * logits_out) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, tokens && n_tokens > 0, "No tokens");
    RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, c->batch_n == 0, "This is a batch context; use rwkv_b200_batch_eval");
    const size_t n_vocab = (size_t) c->model->n_vocab;
    for (size_t i = 0; i < n_tokens; i++)
        RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, tokens[i] < n_vocab, "Token at index %zu (%" PRIu32 ") is out of range (0 .. %zu)", i, tokens[i], n_vocab - 1);
    if (!forward(c, tokens, n_tokens, want_logits || logits_out)) return false;
    if (logits_out) return download_outputs(c, nullptr, logits_out);
    return true;
}

// Batch contexts accept the shapes tests/test_gpu_batch.py checks whole, sequence in a batch against sequence alone: n_embed up to
// 4096, head sizes up to 64 (v7: 128). This is not a bound of the kernels, which take what a single-sequence context takes;
// a wider range wants whole-context tests of its own.
static bool batch_shape_supported(int arch_major, int n_embed, int head_size) {
    if (n_embed > 4096) return false;
    const bool head_upto_64 = head_size == 8 || head_size == 16 || head_size == 32 || head_size == 64;
    if (arch_major == 4) return true;
    if (arch_major == 5 || arch_major == 6) return head_upto_64;
    if (arch_major == 7) return head_upto_64 || head_size == 128;
    return false;
}

struct rwkv_context * rwkv_b200_batch_create(struct rwkv_context * ctx, size_t n_sequences) {
    if (!ctx) return nullptr;
    Context * c = C(ctx);
    bool print = c->print_errors;
    int flags = 0;
    ErrorSink sink{&flags, &print};
    const Model & m = *c->model;
    Context * b = nullptr;
    if (n_sequences == 0 || n_sequences > (size_t) MAX_TOKENS_PER_PASS) {
        flags |= RWKV_ERROR_ARGS;
        if (print) fprintf(stderr, "A batch holds 1 .. %d sequences\n", MAX_TOKENS_PER_PASS);
    } else if (m.layer_begin != 0 || m.layer_end != m.n_layer || !batch_shape_supported(m.arch_major, m.n_embed, m.head_size)) {
        flags |= RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED;
        if (print) fprintf(stderr, "Batched decode supports whole RWKV v4 / v5 / v6 / v7 models with n_embed <= 4096 and head size <= 64 (v7: 128)\n");
    } else {
        b = create_context(c->model, sink, (int) n_sequences);
    }
    if (!b) { g_last_error |= flags; return nullptr; }
    b->print_errors = c->print_errors;
    return static_cast<struct rwkv_context *>(b);
}
bool rwkv_b200_batch_set_state(struct rwkv_context * batch, size_t sequence, const float * state_in) {
    C(batch)->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(C(batch));
    return batch_set_state(C(batch), (int) sequence, state_in);
}
bool rwkv_b200_batch_get_state(struct rwkv_context * batch, size_t sequence, float * state_out) {
    C(batch)->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(C(batch));
    return batch_get_state(C(batch), (int) sequence, state_out);
}
bool rwkv_b200_batch_eval(struct rwkv_context * batch, const uint32_t * tokens, bool want_logits) {
    Context * c = C(batch);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, c->batch_n > 0 && tokens, "Not a batch context or NULL tokens");
    for (int i = 0; i < c->batch_n; i++)
        RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, tokens[i] < (uint32_t) c->model->n_vocab, "Token of sequence %d (%" PRIu32 ") is out of range (0 .. %d)", i, tokens[i], c->model->n_vocab - 1);
    return batch_eval(c, tokens, want_logits);
}
bool rwkv_b200_batch_eval_ragged(struct rwkv_context * batch, const uint32_t * tokens, const uint32_t * counts, bool want_logits) {
    Context * c = C(batch);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    return batch_eval_ragged(c, tokens, counts, want_logits);
}
bool rwkv_b200_batch_get_logits(struct rwkv_context * batch, size_t sequence, float * logits_out) {
    C(batch)->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(C(batch));
    return batch_get_logits(C(batch), (int) sequence, logits_out);
}
size_t rwkv_b200_batch_size(const struct rwkv_context * ctx) { return (size_t) C(ctx)->batch_n; }

static_assert(RWKV_B200_SCORE_NO_TARGET == SCORE_NO_TARGET, "no-target marker of the header and the kernel");

// The arguments every scoring entry point checks: non-NULL arrays, n > 0, n_vocab <= 65536 and every target below n_vocab or
// SCORE_NO_TARGET (tokens: tokens_checked, or here).
static bool score_args_ok(ErrorSink sink, size_t n_vocab, const uint32_t * tokens, bool tokens_checked, const uint32_t * targets, size_t n,
                          const float * logprobs_out) {
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, tokens && targets && logprobs_out, "NULL tokens, targets or logprobs_out");
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, n > 0, "No tokens");
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, n_vocab > 0 && n_vocab <= 65536, "Scoring supports n_vocab <= 65536, not %zu", n_vocab);
    for (size_t i = 0; !tokens_checked && i < n; i++)
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, tokens[i] < n_vocab, "Token at index %zu (%" PRIu32 ") is out of range (0 .. %zu)", i, tokens[i], n_vocab - 1);
    for (size_t i = 0; i < n; i++)
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, targets[i] < n_vocab || targets[i] == SCORE_NO_TARGET,
                   "Target at index %zu (%" PRIu32 ") is out of range (0 .. %zu, or RWKV_B200_SCORE_NO_TARGET)", i, targets[i], n_vocab - 1);
    return true;
}

bool rwkv_b200_score(struct rwkv_context * ctx, const uint32_t * tokens, const uint32_t * targets, size_t n_tokens, float * logprobs_out, uint8_t * greedy_out) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, c->batch_n == 0 && !c->group && whole_model(c),
               "Scoring takes a single-sequence context of the whole model: use rwkv_b200_batch_score_ragged on a batch context; pipelines are not supported");
    if (!score_args_ok(c->sink(), (size_t) c->model->n_vocab, tokens, false, targets, n_tokens, logprobs_out)) return false;
    return score(c, tokens, targets, n_tokens, logprobs_out, greedy_out);
}

bool rwkv_b200_batch_score_ragged(struct rwkv_context * batch, const uint32_t * tokens, const uint32_t * counts, const uint32_t * targets,
                                  float * logprobs_out, uint8_t * greedy_out) {
    Context * c = C(batch);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    size_t total = 0;
    if (!check_ragged(c, tokens, counts, total)) return false;
    if (!score_args_ok(c->sink(), (size_t) c->model->n_vocab, tokens, true, targets, total, logprobs_out)) return false;
    return batch_score_ragged(c, tokens, counts, targets, logprobs_out, greedy_out);
}

bool rwkv_b200_score_logits(const float * logits, size_t n_rows, size_t n_vocab, const uint32_t * targets, float * logprobs_out, uint8_t * greedy_out) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, logits && n_rows <= (size_t) 1 << 24, "NULL logits or more than 2^24 rows");
    if (!score_args_ok(sink, n_vocab, targets, true, targets, n_rows, logprobs_out)) return false;
    if (!hook_device(sink)) return false;
    HookBuffers hb;     // the results start as the caller's buffers (rows without a target are not written) and return at their exact size
    ScoreParams sp{};
    sp.logits = hb.in(logits, n_rows * n_vocab); sp.n_vocab = (int) n_vocab; sp.T = (int) n_rows;
    sp.targets = hb.in(targets, n_rows);
    sp.logprobs = const_cast<float *>(hb.in(logprobs_out, n_rows));
    sp.greedy = greedy_out ? const_cast<uint8_t *>(hb.in(greedy_out, n_rows)) : nullptr;
    const cudaError_t e = hb.ok ? launch_score(sp, 0) : cudaSuccess;
    bool ok = hb.finish(e) && cudaMemcpy(logprobs_out, sp.logprobs, n_rows * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess;
    if (ok && greedy_out) ok = cudaMemcpy(greedy_out, sp.greedy, n_rows, cudaMemcpyDeviceToHost) == cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, ok, "scoring failed on the device: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_sample(struct rwkv_context * ctx, float temperature, float top_p, double u, const uint32_t * bias_ids, const float * bias_values, size_t n_bias,
                      uint32_t * token_out) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    return sample_token(c, temperature, top_p, u, bias_ids, bias_values, n_bias, token_out);
}

bool rwkv_b200_sample_logits(const float * logits, size_t n_vocab, float temperature, float top_p, double u, const uint32_t * bias_ids, const float * bias_values,
                             size_t n_bias, uint32_t * token_out, float * prob_out) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, logits && token_out && n_vocab > 0 && n_vocab <= 65536 && temperature >= 0.0f && top_p >= 0.0f && top_p <= 1.0f &&
               u >= 0.0 && u < 1.0 && (n_bias == 0 || (bias_ids && bias_values)), "Invalid sampling arguments");
    std::vector<uint64_t> seen;
    if (!check_bias_ids(sink, bias_ids, n_bias, n_vocab, seen)) return false;
    int dev = default_device(), n_dev = 0;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, cudaGetDeviceCount(&n_dev) == cudaSuccess && dev < n_dev && cudaSetDevice(dev) == cudaSuccess,
               "No usable CUDA device; this engine has no CPU execution path");
    float * d_logits = nullptr, * d_scratch = nullptr, * d_bv = nullptr, * d_prob = nullptr;
    uint32_t * d_bi = nullptr, * d_tok = nullptr;
    bool ok = cudaMalloc((void **) &d_logits, n_vocab * 4) == cudaSuccess && cudaMalloc((void **) &d_scratch, n_vocab * 4) == cudaSuccess &&
              cudaMalloc((void **) &d_tok, 4) == cudaSuccess && cudaMalloc((void **) &d_prob, 4) == cudaSuccess &&
              cudaMemcpy(d_logits, logits, n_vocab * 4, cudaMemcpyHostToDevice) == cudaSuccess;
    if (ok && n_bias) ok = cudaMalloc((void **) &d_bi, n_bias * 4) == cudaSuccess && cudaMalloc((void **) &d_bv, n_bias * 4) == cudaSuccess &&
                           cudaMemcpy(d_bi, bias_ids, n_bias * 4, cudaMemcpyHostToDevice) == cudaSuccess && cudaMemcpy(d_bv, bias_values, n_bias * 4, cudaMemcpyHostToDevice) == cudaSuccess;
    if (ok) {
        SampleParams sp{};
        sp.logits = d_logits; sp.n_vocab = (int) n_vocab; sp.temperature = temperature; sp.top_p = top_p; sp.u = u;
        sp.bias_ids = d_bi; sp.bias_values = d_bv; sp.n_bias = (int) n_bias; sp.scratch = d_scratch; sp.token_out = d_tok; sp.prob_out = d_prob;
        ok = launch_sample(sp, 0) == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess && cudaMemcpy(token_out, d_tok, 4, cudaMemcpyDeviceToHost) == cudaSuccess;
        if (ok && prob_out) ok = cudaMemcpy(prob_out, d_prob, 4, cudaMemcpyDeviceToHost) == cudaSuccess;
    }
    cudaError_t e = cudaGetLastError();
    cudaFree(d_logits); cudaFree(d_scratch); cudaFree(d_tok); cudaFree(d_prob); cudaFree(d_bi); cudaFree(d_bv);
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, ok, "sampling failed on the device: %s", cudaGetErrorString(e));
    return true;
}

bool rwkv_b200_eval_sample(struct rwkv_context * ctx, uint32_t token, float temperature, float top_p, double u, uint32_t * next_token_out) {
    if (!rwkv_b200_eval_resident(ctx, &token, 1, true, nullptr)) return false;
    return sample_token(C(ctx), temperature, top_p, u, nullptr, nullptr, 0, next_token_out);
}

bool rwkv_b200_batch_sample(struct rwkv_context * batch, const float * temperature, const float * top_p, const double * u, const uint32_t * bias_offsets,
                            const uint32_t * bias_ids, const float * bias_values, uint32_t * tokens_out) {
    C(batch)->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(C(batch));
    return batch_sample(C(batch), temperature, top_p, u, bias_offsets, bias_ids, bias_values, tokens_out);
}

bool rwkv_b200_batch_eval_sample(struct rwkv_context * batch, const uint32_t * tokens, const float * temperature, const float * top_p, const double * u,
                                 uint32_t * tokens_out) {
    Context * c = C(batch);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, c->batch_n > 0 && tokens, "Not a batch context or NULL tokens");
    for (int i = 0; i < c->batch_n; i++)
        RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, tokens[i] < (uint32_t) c->model->n_vocab, "Token of sequence %d (%" PRIu32 ") is out of range (0 .. %d)", i, tokens[i], c->model->n_vocab - 1);
    return batch_eval_sample(c, tokens, temperature, top_p, u, tokens_out);
}

bool rwkv_b200_sample_logits_batch(const float * logits, size_t n_rows, size_t n_vocab, const float * temperature, const float * top_p, const double * u,
                                   const uint32_t * bias_offsets, const uint32_t * bias_ids, const float * bias_values, uint32_t * tokens_out, float * probs_out) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, logits && n_rows > 0 && n_rows <= (size_t) SAMPLE_MAX_ROWS && n_vocab > 0 && n_vocab <= 65536,
               "Invalid batch sampling arguments");
    if (!check_sample_rows(sink, n_rows, n_vocab, temperature, top_p, u, bias_offsets, bias_ids, bias_values, tokens_out)) return false;
    if (!hook_device(sink)) return false;
    const size_t n_bias = bias_offsets ? bias_offsets[n_rows] : 0;
    std::vector<SampleRow> rows(n_rows);
    fill_sample_rows(rows.data(), n_rows, temperature, top_p, u, bias_offsets);
    HookBuffers hb;     // the results are copied back at their exact size, without the guard region of HookBuffers::out
    SampleBatchParams bp{};
    bp.logits = hb.in(logits, n_rows * n_vocab); bp.n_vocab = (int) n_vocab; bp.n_rows = (int) n_rows;
    bp.rows = hb.in(rows.data(), n_rows);
    bp.bias_ids = n_bias ? hb.in(bias_ids, n_bias) : nullptr; bp.bias_values = n_bias ? hb.in(bias_values, n_bias) : nullptr;
    bp.scratch = n_bias ? static_cast<float *>(hb.alloc(n_rows * n_vocab * sizeof(float))) : nullptr;
    bp.token_out = static_cast<uint32_t *>(hb.alloc(n_rows * sizeof(uint32_t)));
    bp.prob_out = probs_out ? static_cast<float *>(hb.alloc(n_rows * sizeof(float))) : nullptr;
    const cudaError_t e = hb.ok ? launch_sample_batch(bp, 0) : cudaSuccess;
    bool ok = hb.finish(e) && cudaMemcpy(tokens_out, bp.token_out, n_rows * sizeof(uint32_t), cudaMemcpyDeviceToHost) == cudaSuccess;
    if (ok && probs_out) ok = cudaMemcpy(probs_out, bp.prob_out, n_rows * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, ok, "batch sampling failed on the device: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

static_assert(RWKV_B200_GENERATE_MAX == GENERATE_MAX && RWKV_B200_GENERATE_MAX_STOP == GENERATE_MAX_STOP, "generation limits of the header and the engine");

static_assert(RWKV_B200_STREAM_TIMEOUT_MS == STREAM_TIMEOUT_MS, "streaming wait bound of the header and the kernel");

// The public logprob request as the engine's; NULL is refused.
static bool logprobs_arg(ErrorSink sink, const struct rwkv_b200_logprobs * lp, LogprobsOut & out) {
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, lp, "NULL logprob request");
    out = LogprobsOut{lp->top_n, lp->logprobs, lp->top_ids, lp->top_logprobs, lp->sample_probs};
    return true;
}

// The engine's part of a public sampler (temperature, top_p and the penalties travel in GenRow).
static SamplerIn sampler_in(const struct rwkv_b200_sampler & s) { return SamplerIn{s.top_k, s.min_p, s.n_bias, s.bias_ids, s.bias_values}; }

// The single-sequence generate calls; on_token NULL is the blocking loop. `constrained`: the row follows *automaton from
// *automaton_state (both checked here, the rest by generate). `sampled`: *sampler (checked here) replaces temperature, top_p and the
// penalties, and lp may be NULL.
static bool generate_single(struct rwkv_context * ctx, size_t max_tokens, float temperature, float top_p, float presence_penalty, float frequency_penalty,
                            bool keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop, uint32_t * tokens_out, size_t * n_generated,
                            bool streaming, TokenFn on_token, void * user, bool constrained = false, const Automaton * automaton = nullptr,
                            uint32_t * automaton_state = nullptr, bool logprobs = false, const struct rwkv_b200_logprobs * lp = nullptr,
                            bool sampled = false, const struct rwkv_b200_sampler * sampler = nullptr) {
    if (!ctx) { ErrorSink sink = global_sink(); g_last_error = RWKV_ERROR_NONE; RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, false, "NULL context"); }
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    const char * suffix = sampled ? "_sampled" : logprobs ? "_logprobs" : constrained ? "_constrained" : streaming ? "_stream" : "";
    RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, c->batch_n == 0, "This is a batch context; use rwkv_b200_batch_generate%s", suffix);
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, max_tokens >= 1 && max_tokens <= (size_t) RWKV_B200_GENERATE_MAX && n_generated,
               "max_tokens must be in 1 .. %d and n_generated not NULL", RWKV_B200_GENERATE_MAX);
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, !streaming || on_token, "NULL on_token");
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, !constrained || (automaton && automaton_state), "NULL automaton or automaton_state");
    LogprobsOut out{};
    if (logprobs && !logprobs_arg(c->sink(), lp, out)) return false;
    SamplerIn smp{};
    if (sampled) {
        RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, sampler, "NULL sampler");
        temperature = sampler->temperature; top_p = sampler->top_p;
        presence_penalty = sampler->presence_penalty; frequency_penalty = sampler->frequency_penalty;
        smp = sampler_in(*sampler);
    }
    const uint32_t budget = (uint32_t) max_tokens;
    const uint8_t keep = keep_counts ? 1 : 0;
    uint32_t n = 0;
    const bool ok = generate(c, &budget, &temperature, &top_p, &presence_penalty, &frequency_penalty, &keep, u, stop_ids, n_stop, tokens_out, &n, on_token, user,
                             constrained ? &automaton : nullptr, automaton_state, logprobs ? &out : nullptr, sampled ? &smp : nullptr);
    if (ok || n) *n_generated = n;      // a callback that kept the device waiting too long still gets what was delivered
    return ok;
}

// The batch generate calls; on_token NULL is the blocking loop. `sampled`: samplers[n_sequences] (checked here) replace the
// temperature, top_p and penalty arrays.
static bool generate_batch(struct rwkv_context * batch, const uint32_t * max_tokens, const float * temperature, const float * top_p,
                           const float * presence_penalty, const float * frequency_penalty, const uint8_t * keep_counts, const double * u,
                           const uint32_t * stop_ids, size_t n_stop, uint32_t * tokens_out, uint32_t * n_generated, bool streaming, TokenFn on_token, void * user,
                           bool constrained = false, const Automaton * const * automata = nullptr, uint32_t * automaton_states = nullptr,
                           bool logprobs = false, const struct rwkv_b200_logprobs * lp = nullptr, bool sampled = false,
                           const struct rwkv_b200_sampler * samplers = nullptr) {
    if (!batch) { ErrorSink sink = global_sink(); g_last_error = RWKV_ERROR_NONE; RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, false, "NULL context"); }
    Context * c = C(batch);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, c->batch_n > 0, "Not a batch context; use rwkv_b200_generate%s",
               sampled ? "_sampled" : logprobs ? "_logprobs" : constrained ? "_constrained" : streaming ? "_stream" : "");
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, !streaming || on_token, "NULL on_token");
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, !constrained || (automata && automaton_states), "NULL automata or automaton_states");
    LogprobsOut out{};
    if (logprobs && !logprobs_arg(c->sink(), lp, out)) return false;
    if (!sampled)
        return generate(c, max_tokens, temperature, top_p, presence_penalty, frequency_penalty, keep_counts, u, stop_ids, n_stop, tokens_out, n_generated,
                        on_token, user, automata, automaton_states, logprobs ? &out : nullptr);
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, samplers, "NULL samplers");
    const size_t rows = (size_t) c->batch_n;
    std::vector<float> t(rows), p(rows), pres(rows), freq(rows);
    std::vector<SamplerIn> smp(rows);
    for (size_t b = 0; b < rows; b++) {
        t[b] = samplers[b].temperature; p[b] = samplers[b].top_p;
        pres[b] = samplers[b].presence_penalty; freq[b] = samplers[b].frequency_penalty;
        smp[b] = sampler_in(samplers[b]);
    }
    return generate(c, max_tokens, t.data(), p.data(), pres.data(), freq.data(), keep_counts, u, stop_ids, n_stop, tokens_out, n_generated, on_token, user,
                    automata, automaton_states, logprobs ? &out : nullptr, smp.data());
}

bool rwkv_b200_generate(struct rwkv_context * ctx, size_t max_tokens, float temperature, float top_p, float presence_penalty, float frequency_penalty,
                        bool keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop, uint32_t * tokens_out, size_t * n_generated) {
    return generate_single(ctx, max_tokens, temperature, top_p, presence_penalty, frequency_penalty, keep_counts, u, stop_ids, n_stop, tokens_out, n_generated,
                           false, nullptr, nullptr);
}

bool rwkv_b200_batch_generate(struct rwkv_context * batch, const uint32_t * max_tokens, const float * temperature, const float * top_p,
                              const float * presence_penalty, const float * frequency_penalty, const uint8_t * keep_counts, const double * u,
                              const uint32_t * stop_ids, size_t n_stop, uint32_t * tokens_out, uint32_t * n_generated) {
    return generate_batch(batch, max_tokens, temperature, top_p, presence_penalty, frequency_penalty, keep_counts, u, stop_ids, n_stop, tokens_out, n_generated,
                          false, nullptr, nullptr);
}

bool rwkv_b200_generate_stream(struct rwkv_context * ctx, size_t max_tokens, float temperature, float top_p, float presence_penalty,
                               float frequency_penalty, bool keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop,
                               rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out, size_t * n_generated) {
    return generate_single(ctx, max_tokens, temperature, top_p, presence_penalty, frequency_penalty, keep_counts, u, stop_ids, n_stop, tokens_out, n_generated,
                           true, on_token, user);
}

bool rwkv_b200_batch_generate_stream(struct rwkv_context * batch, const uint32_t * max_tokens, const float * temperature, const float * top_p,
                                     const float * presence_penalty, const float * frequency_penalty, const uint8_t * keep_counts, const double * u,
                                     const uint32_t * stop_ids, size_t n_stop, rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out,
                                     uint32_t * n_generated) {
    return generate_batch(batch, max_tokens, temperature, top_p, presence_penalty, frequency_penalty, keep_counts, u, stop_ids, n_stop, tokens_out, n_generated,
                          true, on_token, user);
}

}  // extern "C"

// The opaque handle of the automaton API is the engine's Automaton.
struct rwkv_b200_automaton : public rwkv::Automaton {};
// ... and that of the adapter API the engine's Adapter.
struct rwkv_b200_adapter : public rwkv::Adapter {};

extern "C" {

struct rwkv_b200_automaton * rwkv_b200_automaton_create(struct rwkv_context * ctx, const uint16_t * next, size_t n_states) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, ctx, "NULL context");
    const Model & m = *C(ctx)->model;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, nullptr, !C(ctx)->group && m.layer_begin == 0 && m.layer_end == m.n_layer,
               "Automata serve whole-model and batch contexts, not a pipeline or one of its stages");
    return static_cast<struct rwkv_b200_automaton *>(create_automaton(&m, next, n_states, sink));
}

void rwkv_b200_automaton_free(struct rwkv_b200_automaton * a) { destroy_automaton(a); }

struct rwkv_b200_adapter * rwkv_b200_adapter_create(struct rwkv_context * ctx, const struct rwkv_b200_adapter_tensor * t, size_t n, float scale) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, ctx, "NULL context");
    Model & m = *C(ctx)->model;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, nullptr, !C(ctx)->group && m.layer_begin == 0 && m.layer_end == m.n_layer,
               "Adapters serve whole-model and batch contexts, not a pipeline or one of its stages");
    static_assert(sizeof(rwkv_b200_adapter_tensor) == sizeof(AdapterTensor), "rwkv_b200_adapter_tensor and AdapterTensor differ");
    return static_cast<struct rwkv_b200_adapter *>(create_adapter(&m, reinterpret_cast<const AdapterTensor *>(t), n, scale, sink));
}

bool rwkv_b200_adapter_free(struct rwkv_b200_adapter * adapter) {
    g_last_error = RWKV_ERROR_NONE;
    return destroy_adapter(adapter, global_sink());
}

bool rwkv_b200_set_adapter(struct rwkv_context * ctx, const struct rwkv_b200_adapter * adapter) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, !c->group && c->model->layer_begin == 0 && c->model->layer_end == c->model->n_layer,
               "Adapters serve whole-model and batch contexts, not a pipeline or one of its stages");
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, !adapter || adapter->model == c->model, "The adapter belongs to another model");
    return set_adapter(c, adapter);
}

bool rwkv_b200_generate_constrained(struct rwkv_context * ctx, const struct rwkv_b200_automaton * automaton, uint32_t * automaton_state, size_t max_tokens,
                                    float temperature, float top_p, float presence_penalty, float frequency_penalty, bool keep_counts, const double * u,
                                    const uint32_t * stop_ids, size_t n_stop, rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out,
                                    size_t * n_generated) {
    return generate_single(ctx, max_tokens, temperature, top_p, presence_penalty, frequency_penalty, keep_counts, u, stop_ids, n_stop, tokens_out, n_generated,
                           false, on_token, user, true, automaton, automaton_state);
}

bool rwkv_b200_batch_generate_constrained(struct rwkv_context * batch, const struct rwkv_b200_automaton * const * automata, uint32_t * automaton_states,
                                          const uint32_t * max_tokens, const float * temperature, const float * top_p, const float * presence_penalty,
                                          const float * frequency_penalty, const uint8_t * keep_counts, const double * u, const uint32_t * stop_ids,
                                          size_t n_stop, rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out, uint32_t * n_generated) {
    static_assert(sizeof(struct rwkv_b200_automaton) == sizeof(Automaton), "the handle is the engine's automaton");
    return generate_batch(batch, max_tokens, temperature, top_p, presence_penalty, frequency_penalty, keep_counts, u, stop_ids, n_stop, tokens_out, n_generated,
                          false, on_token, user, true, reinterpret_cast<const Automaton * const *>(automata), automaton_states);
}

bool rwkv_b200_generate_logprobs(struct rwkv_context * ctx, const struct rwkv_b200_automaton * automaton, uint32_t * automaton_state, size_t max_tokens,
                                 float temperature, float top_p, float presence_penalty, float frequency_penalty, bool keep_counts, const double * u,
                                 const uint32_t * stop_ids, size_t n_stop, rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out,
                                 size_t * n_generated, const struct rwkv_b200_logprobs * lp) {
    return generate_single(ctx, max_tokens, temperature, top_p, presence_penalty, frequency_penalty, keep_counts, u, stop_ids, n_stop, tokens_out, n_generated,
                           on_token != nullptr, on_token, user, automaton != nullptr, automaton, automaton_state, true, lp);
}

bool rwkv_b200_batch_generate_logprobs(struct rwkv_context * batch, const struct rwkv_b200_automaton * const * automata, uint32_t * automaton_states,
                                       const uint32_t * max_tokens, const float * temperature, const float * top_p, const float * presence_penalty,
                                       const float * frequency_penalty, const uint8_t * keep_counts, const double * u, const uint32_t * stop_ids,
                                       size_t n_stop, rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out, uint32_t * n_generated,
                                       const struct rwkv_b200_logprobs * lp) {
    return generate_batch(batch, max_tokens, temperature, top_p, presence_penalty, frequency_penalty, keep_counts, u, stop_ids, n_stop, tokens_out, n_generated,
                          on_token != nullptr, on_token, user, automata != nullptr, reinterpret_cast<const Automaton * const *>(automata), automaton_states,
                          true, lp);
}

bool rwkv_b200_generate_sampled(struct rwkv_context * ctx, const struct rwkv_b200_sampler * sampler, const struct rwkv_b200_automaton * automaton,
                                uint32_t * automaton_state, size_t max_tokens, bool keep_counts, const double * u, const uint32_t * stop_ids, size_t n_stop,
                                rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out, size_t * n_generated, const struct rwkv_b200_logprobs * lp) {
    return generate_single(ctx, max_tokens, 0.0f, 0.0f, 0.0f, 0.0f, keep_counts, u, stop_ids, n_stop, tokens_out, n_generated, on_token != nullptr, on_token, user,
                           automaton != nullptr, automaton, automaton_state, lp != nullptr, lp, true, sampler);
}

bool rwkv_b200_batch_generate_sampled(struct rwkv_context * batch, const struct rwkv_b200_sampler * samplers, const struct rwkv_b200_automaton * const * automata,
                                      uint32_t * automaton_states, const uint32_t * max_tokens, const uint8_t * keep_counts, const double * u,
                                      const uint32_t * stop_ids, size_t n_stop, rwkv_b200_token_fn on_token, void * user, uint32_t * tokens_out,
                                      uint32_t * n_generated, const struct rwkv_b200_logprobs * lp) {
    return generate_batch(batch, max_tokens, nullptr, nullptr, nullptr, nullptr, keep_counts, u, stop_ids, n_stop, tokens_out, n_generated, on_token != nullptr,
                          on_token, user, automata != nullptr, reinterpret_cast<const Automaton * const *>(automata), automaton_states, lp != nullptr, lp,
                          true, samplers);
}

static_assert(RWKV_B200_AUTOMATON_DEAD == GEN_MASK_DEAD, "dead transition of the header and the kernel");
static_assert(RWKV_B200_TOP_LOGPROBS_MAX == GEN_TOP_MAX, "top log-probabilities of the header and the kernel");
static_assert(2 + 2 * RWKV_B200_TOP_LOGPROBS_MAX == GEN_LP_RECORD, "ring record of the header and the kernel");
static_assert(RWKV_B200_LOGIT_BIAS_MAX == GEN_BIAS_MAX, "user bias entries of the header and the kernel");

// The mapped words of the streaming step hook: acked is read, the others are written back ([n_rows], [n_rows][GENERATE_MAX],
// [n_rows][2][GEN_LP_RECORD] or NULL without log-probabilities, one word).
struct StreamHook {
    const uint32_t * acked;
    uint32_t * published, * tokens, * ring, * timed_out;
};

// One step of the generation kernel on host logits: the unconstrained kernel, or with `next` the constrained one, row b following
// the table from states[b] (UINT32_MAX: unconstrained); with lp the logprob kernel (next may then be NULL: no row constrained); with
// samplers the sampled kernel (next and lp may then be NULL). With `stream` the streaming twin of that kernel runs, as the one node
// of a graph, over pinned mapped copies of the caller's words.
static bool generate_step_hook(const struct rwkv_b200_generate_step_args * a, const uint16_t * next, size_t n_states, uint32_t * states,
                               const LogprobsOut * lp = nullptr, const SamplerIn * samplers = nullptr, const StreamHook * stream = nullptr) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, a && a->logits && a->n_rows >= 1 && a->n_rows <= (size_t) SAMPLE_MAX_ROWS && a->n_vocab >= 1 && a->n_vocab <= 65536 &&
               a->step && a->frozen && a->counts && a->next_tokens && a->any_active, "Invalid generate-step arguments");
    const size_t R = a->n_rows, V = a->n_vocab;
    if (!check_generate_rows(sink, R, V, a->max_tokens, a->temperature, a->top_p, a->presence_penalty, a->frequency_penalty, a->u, a->stop_ids, a->n_stop,
                             a->tokens, a->step)) return false;
    uint32_t n = 0;
    for (size_t b = 0; b < R; b++) {
        n = std::max(n, a->max_tokens[b]);
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, a->step[b] <= a->max_tokens[b], "step of row %zu is above its max_tokens", b);
    }
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, n >= 1, "Every row has max_tokens 0");
    if (lp && !check_logprobs(sink, V, lp)) return false;
    if (samplers && !check_samplers(sink, R, V, samplers)) return false;
    const bool constrained = next != nullptr;
    std::vector<uint8_t> live;
    if (constrained) {
        if (!check_automaton_table(sink, next, n_states, V)) return false;
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, states, "NULL states");
        for (size_t b = 0; b < R; b++)
            RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, states[b] < n_states || states[b] == UINT32_MAX, "state of row %zu is out of range", b);
        live.resize(n_states);
        automaton_live(next, n_states, V, live.data());
    }
    if (stream) {
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, stream->acked && stream->published && stream->tokens && stream->timed_out && (!lp || stream->ring),
                   "NULL mapped word");
        for (size_t b = 0; b < R; b++) {     // the gate of a row that draws token step > 0 waits until token step - 1 is acknowledged
            const bool dead = constrained && states[b] != UINT32_MAX && !live[states[b]];
            const bool draws = !a->frozen[b] && a->step[b] < a->max_tokens[b] && !dead;
            RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, !draws || a->step[b] == 0 || (stream->acked[b] >> 1) >= a->step[b],
                       "row %zu would wait for the acknowledgement of its token %u", b, a->step[b] - 1);
        }
    }
    if (!hook_device(sink)) return false;
    GenShared sh{};
    for (size_t k = 0; k < a->n_stop; k++) sh.stop[k] = a->stop_ids[k];
    sh.n_stop = (uint32_t) a->n_stop; sh.stride = n;
    std::vector<GenRow> rows(R);
    for (size_t b = 0; b < R; b++)
        rows[b] = GenRow{a->temperature[b], a->top_p[b], a->presence_penalty[b], a->frequency_penalty[b], a->max_tokens[b], a->step[b], a->frozen[b] ? 1u : 0u, 0};
    const uint32_t zero = 0;
    HookBuffers hb;
    GenStepParams gp{};
    gp.logits = hb.in(a->logits, R * V); gp.n_vocab = (int) V; gp.n_rows = (int) R;
    gp.rows = const_cast<GenRow *>(hb.in(rows.data(), R));
    gp.shared = const_cast<GenShared *>(hb.in(&sh, 1));
    gp.u = hb.in(a->u, R * n);
    gp.counts = const_cast<uint32_t *>(hb.in(a->counts, R * V));
    gp.bias_ids = static_cast<uint32_t *>(hb.alloc(R * V * sizeof(uint32_t)));
    gp.bias_values = static_cast<float *>(hb.alloc(R * V * sizeof(float)));
    gp.scratch = static_cast<float *>(hb.alloc(R * V * sizeof(float)));
    gp.tokens = const_cast<uint32_t *>(hb.in(a->tokens, R * n));
    gp.n_generated = static_cast<uint32_t *>(hb.alloc(R * sizeof(uint32_t)));
    gp.passes = const_cast<uint32_t *>(hb.in(&zero, 1));
    gp.next_tokens = static_cast<int *>(hb.alloc(R * sizeof(int)));
    GenConstrainedParams cp{};
    cp.stream.step = gp;
    // the streaming kernel's words in pinned mapped memory, as the engine keeps them: acked [R], published [R], timed_out, tokens
    // [R][GENERATE_MAX], ring [R][2][GEN_LP_RECORD]
    struct Pinned {
        uint32_t * host = nullptr;
        ~Pinned() { if (host) cudaFreeHost(host); }
    } pinned;
    const size_t ring_words = lp ? R * 2 * GEN_LP_RECORD : 0, tok_at = 2 * R + 1, ring_at = tok_at + R * GENERATE_MAX;
    uint32_t * mapped = nullptr;
    if (stream && hb.ok) {
        hb.ok = cudaHostAlloc(reinterpret_cast<void **>(&pinned.host), (ring_at + ring_words) * sizeof(uint32_t), cudaHostAllocMapped) == cudaSuccess &&
                cudaHostGetDevicePointer(reinterpret_cast<void **>(&mapped), pinned.host, 0) == cudaSuccess;
        if (hb.ok) {
            std::copy(stream->acked, stream->acked + R, pinned.host);
            std::copy(stream->published, stream->published + R, pinned.host + R);
            pinned.host[2 * R] = 0;
            std::copy(stream->tokens, stream->tokens + R * GENERATE_MAX, pinned.host + tok_at);
            if (lp) std::copy(stream->ring, stream->ring + ring_words, pinned.host + ring_at);
            cp.stream.acked = mapped; cp.stream.published = mapped + R; cp.stream.timed_out = mapped + 2 * R; cp.stream.tokens = mapped + tok_at;
        }
    }
    std::vector<uint32_t> states_out(R);
    if (constrained) {
        const uint16_t * d_next = hb.in(next, n_states * V);
        const uint8_t * d_live = hb.in(live.data(), n_states);
        std::vector<GenMaskRow> mask(R);
        for (size_t b = 0; b < R; b++)
            mask[b] = states[b] == UINT32_MAX ? GenMaskRow{nullptr, nullptr, 0, 0} : GenMaskRow{d_next, d_live, states[b], 0};
        cp.mask = const_cast<GenMaskRow *>(hb.in(mask.data(), R));
        cp.states_out = static_cast<uint32_t *>(hb.alloc(R * sizeof(uint32_t)));
    }
    GenLogprobParams lpp{};
    GenLogprobRequest req{};
    const size_t cells = R * n, k = lp ? lp->top_n : 0;
    if (!constrained && (lp || samplers)) {     // every row unconstrained without a table
        const std::vector<GenMaskRow> none(R, GenMaskRow{nullptr, nullptr, 0, 0});
        cp.mask = const_cast<GenMaskRow *>(hb.in(none.data(), R));
        cp.states_out = static_cast<uint32_t *>(hb.alloc(R * sizeof(uint32_t)));
    }
    if (lp) {       // the outputs start as the caller's arrays
        req.top_n = (uint32_t) k;
        req.logprobs = const_cast<float *>(hb.in(lp->logprobs, cells));
        req.sample_probs = lp->sample_probs ? const_cast<float *>(hb.in(lp->sample_probs, cells)) : static_cast<float *>(hb.alloc(cells * sizeof(float)));
        req.top_ids = k ? const_cast<uint32_t *>(hb.in(lp->top_ids, cells * k)) : nullptr;
        req.top_logprobs = k ? const_cast<float *>(hb.in(lp->top_logprobs, cells * k)) : nullptr;
        req.ring = mapped ? mapped + ring_at : nullptr;
        lpp.gen = cp;
        lpp.req = hb.in(&req, 1);
    }
    GenSamplerParams smp{};
    if (samplers) {
        std::vector<GenSamplerRow> srows(R);
        std::vector<GenBiasEntry> pool;
        for (size_t b = 0; b < R; b++) {
            const SamplerIn & s = samplers[b];
            srows[b] = GenSamplerRow{s.top_k, s.min_p, (uint32_t) pool.size(), (uint32_t) (pool.size() + s.n_bias)};
            for (size_t k = 0; k < s.n_bias; k++) pool.push_back(GenBiasEntry{s.bias_ids[k], s.bias_values[k]});
        }
        const GenLogprobRequest * word = lp ? lpp.req : nullptr;
        smp.gen = cp;
        smp.req = hb.in(&word, 1);
        smp.rows = hb.in(srows.data(), R);
        smp.bias = pool.empty() ? nullptr : hb.in(pool.data(), pool.size());
    }
    cudaError_t e = cudaSuccess;
    if (hb.ok && stream) {      // the streaming kernels exist only as graph nodes
        cudaGraph_t g = nullptr;
        cudaGraphExec_t x = nullptr;
        cudaGraphNode_t node = nullptr;
        e = cudaGraphCreate(&g, 0);
        if (e == cudaSuccess)
            e = samplers ? add_generate_sampled_step_node(g, nullptr, 0, smp, true, &node) : lp ? add_generate_logprob_step_node(g, nullptr, 0, lpp, true, &node)
              : constrained ? add_generate_constrained_step_node(g, nullptr, 0, cp, true, &node) : add_generate_stream_step_node(g, nullptr, 0, cp.stream, &node);
        if (e == cudaSuccess) e = cudaGraphInstantiate(&x, g, 0);
        if (e == cudaSuccess) e = cudaGraphLaunch(x, 0);
        if (e == cudaSuccess) e = cudaStreamSynchronize(0);
        if (x) cudaGraphExecDestroy(x);
        if (g) cudaGraphDestroy(g);
    } else if (hb.ok) {
        e = samplers ? launch_generate_sampled_step(smp, 0) : lp ? launch_generate_logprob_step(lpp, 0)
          : constrained ? launch_generate_constrained_step(cp, 0) : launch_generate_step(gp, 0);
    }
    bool ok = hb.finish(e) && cudaMemcpy(rows.data(), gp.rows, R * sizeof(GenRow), cudaMemcpyDeviceToHost) == cudaSuccess &&
              cudaMemcpy(a->counts, gp.counts, R * V * sizeof(uint32_t), cudaMemcpyDeviceToHost) == cudaSuccess &&
              cudaMemcpy(a->tokens, gp.tokens, R * n * sizeof(uint32_t), cudaMemcpyDeviceToHost) == cudaSuccess &&
              cudaMemcpy(a->next_tokens, gp.next_tokens, R * sizeof(int), cudaMemcpyDeviceToHost) == cudaSuccess &&
              cudaMemcpy(a->any_active, gp.passes, sizeof(uint32_t), cudaMemcpyDeviceToHost) == cudaSuccess &&
              (!constrained || cudaMemcpy(states_out.data(), cp.states_out, R * sizeof(uint32_t), cudaMemcpyDeviceToHost) == cudaSuccess) &&
              (!lp || cudaMemcpy(lp->logprobs, req.logprobs, cells * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess) &&
              (!lp || !lp->sample_probs || cudaMemcpy(lp->sample_probs, req.sample_probs, cells * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess) &&
              (!k || (cudaMemcpy(lp->top_ids, req.top_ids, cells * k * sizeof(uint32_t), cudaMemcpyDeviceToHost) == cudaSuccess &&
                      cudaMemcpy(lp->top_logprobs, req.top_logprobs, cells * k * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess));
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, ok, "generate step failed on the device: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    for (size_t b = 0; b < R; b++) { a->step[b] = rows[b].step; a->frozen[b] = rows[b].frozen ? 1 : 0; }
    for (size_t b = 0; constrained && b < R; b++)
        if (states[b] != UINT32_MAX) states[b] = states_out[b];
    if (stream) {
        std::copy(pinned.host + R, pinned.host + 2 * R, stream->published);
        *stream->timed_out = pinned.host[2 * R];
        std::copy(pinned.host + tok_at, pinned.host + tok_at + R * GENERATE_MAX, stream->tokens);
        if (lp) std::copy(pinned.host + ring_at, pinned.host + ring_at + ring_words, stream->ring);
    }
    return true;
}

bool rwkv_b200_test_generate_step(const struct rwkv_b200_generate_step_args * a) { return generate_step_hook(a, nullptr, 0, nullptr); }

bool rwkv_b200_test_generate_step_constrained(const struct rwkv_b200_generate_step_args * a, const uint16_t * next, size_t n_states, uint32_t * states) {
    if (!next) { g_last_error = RWKV_ERROR_NONE; ErrorSink sink = global_sink(); RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, false, "NULL table"); }
    return generate_step_hook(a, next, n_states, states);
}

bool rwkv_b200_test_generate_step_logprobs(const struct rwkv_b200_generate_step_args * a, const uint16_t * next, size_t n_states, uint32_t * states,
                                           const struct rwkv_b200_logprobs * lp) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    LogprobsOut out{};
    if (!logprobs_arg(sink, lp, out)) return false;
    return generate_step_hook(a, next, n_states, states, &out);
}

// The sampled kernel's step: samplers[n_rows] in place of a's temperature, top_p and penalty arrays.
static bool sampled_step_hook(const struct rwkv_b200_generate_step_args * a, const struct rwkv_b200_sampler * samplers, const uint16_t * next,
                              size_t n_states, uint32_t * states, const struct rwkv_b200_logprobs * lp, const StreamHook * stream = nullptr) {
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, a && a->n_rows >= 1 && a->n_rows <= (size_t) SAMPLE_MAX_ROWS, "Invalid generate-step arguments");
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, samplers, "NULL samplers");
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, !a->temperature && !a->top_p && !a->presence_penalty && !a->frequency_penalty,
               "temperature, top_p and the penalties come from the samplers: pass NULL");
    LogprobsOut out{};
    if (lp && !logprobs_arg(sink, lp, out)) return false;
    const size_t R = a->n_rows;
    std::vector<float> t(R), p(R), pres(R), freq(R);
    std::vector<SamplerIn> smp(R);
    for (size_t b = 0; b < R; b++) {
        t[b] = samplers[b].temperature; p[b] = samplers[b].top_p;
        pres[b] = samplers[b].presence_penalty; freq[b] = samplers[b].frequency_penalty;
        smp[b] = sampler_in(samplers[b]);
    }
    struct rwkv_b200_generate_step_args args = *a;
    args.temperature = t.data(); args.top_p = p.data(); args.presence_penalty = pres.data(); args.frequency_penalty = freq.data();
    return generate_step_hook(&args, next, n_states, states, lp ? &out : nullptr, smp.data(), stream);
}

bool rwkv_b200_test_generate_step_sampled(const struct rwkv_b200_generate_step_args * a, const struct rwkv_b200_sampler * samplers, const uint16_t * next,
                                          size_t n_states, uint32_t * states, const struct rwkv_b200_logprobs * lp) {
    g_last_error = RWKV_ERROR_NONE;
    return sampled_step_hook(a, samplers, next, n_states, states, lp);
}

bool rwkv_b200_test_generate_step_streaming(const struct rwkv_b200_generate_step_args * a, int family, const struct rwkv_b200_sampler * samplers,
                                            const uint16_t * next, size_t n_states, uint32_t * states, const struct rwkv_b200_logprobs * lp,
                                            const uint32_t * acked, uint32_t * published, uint32_t * stream_tokens, uint32_t * ring, uint32_t * timed_out) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, family >= RWKV_B200_STEP_PLAIN && family <= RWKV_B200_STEP_SAMPLED, "Unknown step family %d", family);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, (family == RWKV_B200_STEP_SAMPLED) == (samplers != nullptr), "samplers go with the sampled family alone");
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, family == RWKV_B200_STEP_CONSTRAINED ? next != nullptr : family != RWKV_B200_STEP_PLAIN || !next,
               "The constrained family needs a table, the plain one takes none");
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, family == RWKV_B200_STEP_LOGPROBS ? lp != nullptr : family == RWKV_B200_STEP_SAMPLED || !lp,
               "The logprobs family needs lp, the plain and constrained ones take none");
    const StreamHook stream{acked, published, stream_tokens, ring, timed_out};
    if (family == RWKV_B200_STEP_SAMPLED) return sampled_step_hook(a, samplers, next, n_states, states, lp, &stream);
    LogprobsOut out{};
    if (lp && !logprobs_arg(sink, lp, out)) return false;
    return generate_step_hook(a, next, n_states, states, lp ? &out : nullptr, nullptr, &stream);
}

size_t rwkv_b200_stage_hidden_len(const struct rwkv_context * ctx, size_t n_tokens) { return stage_hidden_len(*C(ctx)->model, n_tokens); }

bool rwkv_b200_stage_eval(struct rwkv_context * ctx, const uint32_t * tokens, size_t n_tokens, const float * hidden_in, float * hidden_out, bool want_logits,
                          void * cuda_stream) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    const Model & m = *c->model;
    const bool first = m.layer_begin == 0, last = m.layer_end == m.n_layer;
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, n_tokens > 0 && n_tokens <= (size_t) MAX_TOKENS_PER_PASS, "A stage pass takes 1 .. %d tokens", MAX_TOKENS_PER_PASS);
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, first ? tokens != nullptr : hidden_in != nullptr, "Stage [%d, %d) needs %s", m.layer_begin, m.layer_end,
               first ? "tokens" : "the previous stage's activations");
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, last || hidden_out != nullptr, "Stage [%d, %d) needs an output buffer for its activations", m.layer_begin, m.layer_end);
    if (first)
        for (size_t i = 0; i < n_tokens; i++)
            RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, tokens[i] < (uint32_t) m.n_vocab, "Token at index %zu (%" PRIu32 ") is out of range (0 .. %d)", i, tokens[i], m.n_vocab - 1);
    return stage_forward(c, tokens, n_tokens, hidden_in, hidden_out, want_logits && last, reinterpret_cast<cudaStream_t>(cuda_stream));
}

// ---- layer pipeline over peer memory (kernels/pipe.cu) ----
void * rwkv_b200_stream(struct rwkv_context * ctx) { return ctx ? reinterpret_cast<void *>(C(ctx)->stream) : nullptr; }
size_t rwkv_b200_pipe_handle_size(void) { return sizeof(cudaIpcMemHandle_t); }

bool rwkv_b200_pipe_export(struct rwkv_context * ctx, void * handle_out) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, handle_out != nullptr, "handle_out is NULL");
    if (!pipe_ensure_box(c)) return false;
    cudaIpcMemHandle_t h;
    const cudaError_t e = cudaIpcGetMemHandle(&h, c->model->link.box);
    RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, e == cudaSuccess, "cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
    memcpy(handle_out, &h, sizeof(h));
    return true;
}

static bool pipe_open(Context * c, const void * handle, PipeBox ** out) {
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof(h));
    void * p = nullptr;
    const cudaError_t e = cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess);
    RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, e == cudaSuccess, "cudaIpcOpenMemHandle failed: %s", cudaGetErrorString(e));
    *out = reinterpret_cast<PipeBox *>(p);
    return true;
}

bool rwkv_b200_pipe_connect(struct rwkv_context * ctx, const void * prev_handle, const void * next_handle) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    Model & m = *c->model;
    if (!pipe_ensure_box(c)) return false;
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, (m.layer_begin == 0) == (prev_handle == nullptr) && (m.layer_end == m.n_layer) == (next_handle == nullptr),
               "Stage [%d, %d): a first stage has no previous neighbour, a last stage no next one, every other stage both", m.layer_begin, m.layer_end);
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, !m.link.prev && !m.link.next, "The stage is already connected");
    if (cudaSetDevice(m.dev.device) != cudaSuccess) return false;
    if (prev_handle) { if (!pipe_open(c, prev_handle, &m.link.prev)) return false; m.link.prev_ipc = true; }
    if (next_handle) { if (!pipe_open(c, next_handle, &m.link.next)) return false; m.link.next_ipc = true; }
    return true;
}

bool rwkv_b200_pipe_connect_local(struct rwkv_context * ctx, struct rwkv_context * prev, struct rwkv_context * next) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    Model & m = *c->model;
    if (!pipe_ensure_box(c)) return false;
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, (m.layer_begin == 0) == (prev == nullptr) && (m.layer_end == m.n_layer) == (next == nullptr),
               "Stage [%d, %d): a first stage has no previous neighbour, a last stage no next one, every other stage both", m.layer_begin, m.layer_end);
    for (struct rwkv_context * other : {prev, next}) {
        if (!other) continue;
        Context * o = C(other);
        if (!pipe_ensure_box(o)) return false;
        if (o->model->dev.device != m.dev.device) {      // one process, two GPUs: peer access in both directions
            for (int pass = 0; pass < 2; pass++) {
                const int from = pass ? o->model->dev.device : m.dev.device, to = pass ? m.dev.device : o->model->dev.device;
                int can = 0;
                cudaDeviceCanAccessPeer(&can, from, to);
                RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, can, "Device %d cannot access device %d's memory", from, to);
                cudaSetDevice(from);
                const cudaError_t e = cudaDeviceEnablePeerAccess(to, 0);
                if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
                else RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, e == cudaSuccess, "cudaDeviceEnablePeerAccess failed: %s", cudaGetErrorString(e));
            }
        }
        (other == prev ? m.link.prev : m.link.next) = o->model->link.box;
    }
    return true;
}

bool rwkv_b200_pipe_eval(struct rwkv_context * ctx, const uint32_t * tokens, size_t n_tokens, bool want_logits, void * cuda_stream) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    const Model & m = *c->model;
    const bool first = m.layer_begin == 0;
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, n_tokens > 0 && n_tokens <= (size_t) MAX_TOKENS_PER_PASS, "A stage pass takes 1 .. %d tokens", MAX_TOKENS_PER_PASS);
    RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, c->batch_n == 0, "Batch contexts cannot be pipeline stages");
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, !first || tokens != nullptr, "The first stage needs tokens");
    if (first)
        for (size_t i = 0; i < n_tokens; i++)
            RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, tokens[i] < (uint32_t) m.n_vocab, "Token at index %zu (%" PRIu32 ") is out of range (0 .. %d)", i, tokens[i], m.n_vocab - 1);
    return pipe_forward(c, tokens, n_tokens, want_logits, reinterpret_cast<cudaStream_t>(cuda_stream));
}

bool rwkv_b200_stage_logits(struct rwkv_context * ctx, float * logits_out, void * cuda_stream) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_NOT_STREAMING(c);
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, logits_out && c->model->layer_end == c->model->n_layer, "Only the last stage holds logits");
    cudaStream_t s = cuda_stream ? reinterpret_cast<cudaStream_t>(cuda_stream) : c->stream;
    cudaError_t e = cudaMemcpyAsync(logits_out, c->logits, (size_t) c->model->n_vocab * sizeof(float), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    RWKV_CHECK(c->sink(), RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, e == cudaSuccess, "Reading the logits failed: %s", cudaGetErrorString(e));
    return true;
}

float rwkv_b200_last_device_ms(const struct rwkv_context * ctx) {
    float ms = -1.f;
    const Context * c = C(ctx);
    if (cudaEventSynchronize(c->ev_stop) != cudaSuccess) return -1.f;
    if (cudaEventElapsedTime(&ms, c->ev_start, c->ev_stop) != cudaSuccess) return -1.f;
    return ms;
}

uint64_t rwkv_b200_kernel_launch_count(void) { return g_kernel_launches; }
uint64_t rwkv_b200_graph_launch_count(void) { return g_graph_launches; }

uint64_t rwkv_b200_gemv_bytes_per_token(const struct rwkv_context * ctx, bool with_logits) {
    const Model & m = *C(ctx)->model;
    // the decode pass of a single-sequence context folds v6 LoRA matrices into other kernels; a batch context streams them all
    const size_t folded = C(ctx)->batch_n ? 0 : v6_folded_gemv_bytes(m);
    return (uint64_t) (m.gemv_bytes_per_token - (with_logits ? 0 : m.head_matrix_bytes) - folded);
}

uint64_t rwkv_b200_bytes_per_token(const struct rwkv_context * ctx, bool with_logits) {
    const Model & m = *C(ctx)->model;
    return (uint64_t) (m.weight_bytes_per_token - (with_logits ? 0 : m.head_bytes) + 2 * 4 * m.state_len());
}

float rwkv_b200_time_resident(struct rwkv_context * ctx, const uint32_t * tokens, size_t tokens_per_step, int n_steps, int warmup_steps, bool want_logits) {
    Context * c = C(ctx);
    cudaEvent_t e0, e1;
    if (!tokens || tokens_per_step == 0 || n_steps <= 0 || cudaSetDevice(c->model->dev.device) != cudaSuccess) return -1.f;
    const uint32_t * t = tokens;
    for (int i = 0; i < warmup_steps; i++, t += tokens_per_step) if (!rwkv_b200_eval_resident(ctx, t, tokens_per_step, want_logits, nullptr)) return -1.f;
    if (cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess) return -1.f;
    cudaStreamSynchronize(c->stream);
    cudaEventRecord(e0, c->stream);
    bool ok = true;
    for (int i = 0; i < n_steps && ok; i++, t += tokens_per_step) ok = rwkv_b200_eval_resident(ctx, t, tokens_per_step, want_logits, nullptr);
    cudaEventRecord(e1, c->stream);
    float ms = -1.f;
    if (ok && cudaEventSynchronize(e1) == cudaSuccess) cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return ok ? ms : -1.f;
}

bool rwkv_b200_profile_pass(struct rwkv_context * ctx, const uint32_t * tokens, size_t n_tokens, bool want_logits, struct rwkv_b200_profile * out) {
    Context * c = C(ctx);
    c->last_error = RWKV_ERROR_NONE;
    RWKV_CHECK(c->sink(), RWKV_ERROR_ARGS, false, tokens && out && n_tokens > 0 && n_tokens <= (size_t) MAX_TOKENS_PER_PASS, "Invalid profile arguments");
    memset(out, 0, sizeof(*out));
    c->profiling = true;
    const unsigned long long before = g_kernel_launches;
    bool ok = rwkv_b200_eval_resident(ctx, tokens, n_tokens, want_logits, nullptr) && cudaStreamSynchronize(c->stream) == cudaSuccess;
    c->profiling = false;
    out->total_launches = (uint32_t) (g_kernel_launches - before);
    if (ok) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, c->ev_start, c->ev_stop);
        out->pass_ms = ms;
        for (auto & r : c->prof) {
            cudaEventElapsedTime(&ms, r.start, r.stop);
            out->gemv_ms += ms; out->gemv_bytes += r.bytes; out->gemv_launches++;
            if (ms > out->top_ms) { out->top_ms = ms; out->top_bytes = r.bytes; }
        }
    }
    for (auto & r : c->prof) { cudaEventDestroy(r.start); cudaEventDestroy(r.stop); }
    c->prof.clear();
    return ok;
}

void rwkv_b200_set_graphs(struct rwkv_context * ctx, bool enabled) { C(ctx)->use_graphs = enabled; }
void rwkv_b200_set_tensor_cores(struct rwkv_context * ctx, bool enabled) {
    if (C(ctx)->use_tensor_cores != enabled) drop_generate_graphs(C(ctx));     // a batch's generation graph holds its GEMM routing
    C(ctx)->use_tensor_cores = enabled;
}
void rwkv_b200_set_overlap(struct rwkv_context * ctx, bool enabled) { C(ctx)->overlap_copies = enabled; }
void rwkv_b200_set_bounce_min_bytes(size_t bytes) { g_bounce_min_bytes.store(bytes); }
int rwkv_b200_overlap_groups(const struct rwkv_context * ctx) { return C(ctx)->overlap_copies && C(ctx)->n_segments > 1 ? C(ctx)->n_segments : 0; }
static bool trace_rearm(Context * c) {
    std::vector<TraceRec> init(1024);
    for (auto & r : init) { r.start = ~0ull; r.end = 0; for (auto & m : r.mark) m = 0; }
    return cudaMemcpy(c->trace_buf, init.data(), init.size() * sizeof(TraceRec), cudaMemcpyHostToDevice) == cudaSuccess;
}

bool rwkv_b200_trace_enable(struct rwkv_context * ctx) {
    Context * c = C(ctx);
    if (cudaSetDevice(c->model->dev.device) != cudaSuccess || cudaStreamSynchronize(c->stream) != cudaSuccess) return false;
    if (!c->trace_buf && cudaMalloc((void **) &c->trace_buf, 1024 * sizeof(TraceRec)) != cudaSuccess) return false;
    // graphs captured so far carry no trace slots: drop them so they are re-captured
    for (auto & g : c->graphs) { if (g.exec) cudaGraphExecDestroy(g.exec); g = Context::GraphSlot(); }
    drop_generate_graphs(c);
    return trace_rearm(c);
}

void rwkv_b200_trace_disable(struct rwkv_context * ctx) {
    Context * c = C(ctx);
    if (!c->trace_buf || cudaSetDevice(c->model->dev.device) != cudaSuccess) return;
    cudaStreamSynchronize(c->stream);
    for (auto & g : c->graphs) { if (g.exec) cudaGraphExecDestroy(g.exec); g = Context::GraphSlot(); }
    drop_generate_graphs(c);
    cudaFree(c->trace_buf);
    c->trace_buf = nullptr; c->trace_count = 0;
}

// marks_us: optional [max_records][4] intra-kernel marks of CTA 0 (-1 when absent)
static double * g_trace_marks_out = nullptr;
void rwkv_b200_trace_set_marks_buffer(double * marks_us) { g_trace_marks_out = marks_us; }

int rwkv_b200_trace_read(struct rwkv_context * ctx, double * start_us, double * end_us, char (*names)[32], int max_records) {
    Context * c = C(ctx);
    if (!c->trace_buf || cudaStreamSynchronize(c->stream) != cudaSuccess) return -1;
    std::vector<TraceRec> recs(1024);
    if (cudaMemcpy(recs.data(), c->trace_buf, recs.size() * sizeof(TraceRec), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    const int n = c->trace_count < max_records ? c->trace_count : max_records;
    unsigned long long t0 = ~0ull;
    for (int i = 0; i < n; i++) if (recs[i].start < t0) t0 = recs[i].start;
    for (int i = 0; i < n; i++) {
        start_us[i] = recs[i].start == ~0ull ? -1.0 : (double) (recs[i].start - t0) * 1e-3;
        end_us[i] = recs[i].end == 0 ? -1.0 : (double) (recs[i].end - t0) * 1e-3;
        if (g_trace_marks_out) for (int k = 0; k < 4; k++) g_trace_marks_out[i * 4 + k] = recs[i].mark[k] ? (double) (recs[i].mark[k] - t0) * 1e-3 : -1.0;
        const char * nm = c->trace_names[i] ? c->trace_names[i] : "?";
        strncpy(names[i], nm, 31); names[i][31] = 0;
    }
    trace_rearm(c);
    return n;
}

bool rwkv_b200_matvec(int data_type, int K, int M, int T, const void * weights, const float * x, float * y, int epilogue) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, weights && x && y && K > 0 && M > 0 && T > 0 && dtype_loadable(data_type) && K % dtype_block_elems(data_type) == 0 && epilogue >= 0 && epilogue <= EPI_RELU_SQR,
               "Invalid matvec arguments");
    int dev = default_device(), n_dev = 0;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, cudaGetDeviceCount(&n_dev) == cudaSuccess && dev < n_dev && cudaSetDevice(dev) == cudaSuccess,
               "No usable CUDA device; this engine has no CPU execution path");
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, dev);
    DeviceInfo di{dev, prop.multiProcessorCount, (int) prop.sharedMemPerBlockOptin};
    // passes of >= 32 tokens go through the tensor-core kernel, which streams the tile-major copy of the matrix
    const bool tiled = T >= 32 && gemm_tc_eligible(data_type, K) && !getenv("RWKV_B200_NO_TC");
    const size_t ws_bytes = gemm_tc_batch_workspace_bytes(T, (size_t) K);
    uint8_t * dW = nullptr, * dWt = nullptr; float * dx = nullptr, * dy = nullptr; void * ws = nullptr;
    bool ok = cudaMalloc((void **) &dW, (size_t) matrix_pitch(data_type, (uint64_t) K) * M + 256) == cudaSuccess && cudaMalloc((void **) &dx, sizeof(float) * K * T) == cudaSuccess &&
              cudaMalloc((void **) &dy, sizeof(float) * M * T) == cudaSuccess && cudaMemcpy(dx, x, sizeof(float) * K * T, cudaMemcpyHostToDevice) == cudaSuccess &&
              (!tiled || (cudaMalloc((void **) &dWt, gemm_tc_tiled_bytes(data_type, M, K)) == cudaSuccess && cudaMalloc(&ws, ws_bytes) == cudaSuccess)) &&
              upload_matrix(weights, data_type, M, K, dW, dWt) == cudaSuccess;
    if (ok) {
        GemvBatch b;
        memset(&b, 0, sizeof(b));
        b.n = 1; b.T = T;
        GemvProblem & p = b.p[0];
        p.W = dW; p.Wt = dWt; p.pitch = matrix_pitch(data_type, (uint64_t) K); p.type = data_type; p.K = K; p.M = M;
        p.x = dx; p.ldx = K; p.y = dy; p.ldy = M; p.epi = epilogue; p.pro = PRO_NONE;
        ok = gemv_route(b, di, 0, ws, ws_bytes, 32) == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess &&
             cudaMemcpy(y, dy, sizeof(float) * M * T, cudaMemcpyDeviceToHost) == cudaSuccess;
    }
    cudaError_t e = cudaGetLastError();
    cudaFree(dW); cudaFree(dWt); cudaFree(dx); cudaFree(dy); cudaFree(ws);
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, ok, "matvec failed on the device: %s", cudaGetErrorString(e));
    return true;
}

// ---- kernel test hooks (include/rwkv_b200.h): one launcher each, on host buffers ----

bool rwkv_b200_test_embed_ln0(const void * emb, int emb_type, size_t emb_pitch, int n_vocab, const int * tokens, int T, int C,
                              const float * ln_w, const float * ln_b, float * x) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    bool args = emb && tokens && ln_w && ln_b && x && T > 0 && C > 0 && n_vocab > 0 && (emb_type == DT_F32 || emb_type == DT_F16) &&
                emb_pitch >= (size_t) C * (emb_type == DT_F32 ? 4 : 2) && emb_pitch % (emb_type == DT_F32 ? 4 : 2) == 0;   // rows are read as elements
    for (int t = 0; args && t < T; t++) args = tokens[t] >= 0 && tokens[t] < n_vocab;
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args, "Invalid embed_ln0 arguments");
    if (!hook_device(sink)) return false;
    HookBuffers b;
    const void * d_emb = b.in(static_cast<const uint8_t *>(emb), (size_t) n_vocab * emb_pitch);
    const int * d_tok = b.in(tokens, T);
    const float * d_w = b.in(ln_w, C), * d_b = b.in(ln_b, C);
    float * d_x = b.out(x, (size_t) C * T);
    const cudaError_t e = b.ok ? launch_embed_ln0(d_emb, emb_type, (long long) emb_pitch, d_tok, T, C, d_w, d_b, d_x, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "embed_ln0 failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_encode_rows(int data_type, const float * values, size_t M, size_t K, void * out) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, values && out && M > 0 && K > 0 && (data_type == DT_F32 || dtype_loadable(data_type)) &&
               K % (size_t) dtype_block_elems(data_type) == 0, "Invalid encode_rows arguments");
    encode_rows(data_type, values, M, K, static_cast<uint8_t *>(out));
    return true;
}

bool rwkv_b200_test_lora(int K, int M, int T, int rank, float scale, int epilogue, const float * a, const float * b, const float * x,
                         const float * z, const float * gate, float * u, float * y) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    const bool epi_ok = epilogue == EPI_NONE || epilogue == EPI_SIGMOID || epilogue == EPI_SILU || epilogue == EPI_RELU_SQR || epilogue == EPI_ADD ||
                        epilogue == EPI_MUL_ADD;
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, a && b && x && z && u && y && K > 0 && M > 0 && T >= 1 && T <= MAX_TOKENS_PER_PASS && rank >= 1 &&
               rank <= LORA_MAX_RANK && epi_ok && (epilogue != EPI_MUL_ADD || gate), "Invalid lora arguments");
    if (!hook_device(sink)) return false;
    const size_t R = (size_t) rank;
    std::vector<uint16_t> ha(R * (size_t) K), hbt(R * (size_t) M);
    for (size_t i = 0; i < ha.size(); i++) ha[i] = fp32_to_fp16(a[i]);
    for (size_t r = 0; r < R; r++) for (size_t i = 0; i < (size_t) M; i++) hbt[r * M + i] = fp32_to_fp16(b[i * R + r]);
    HookBuffers hb;
    LoraBatch lb{};
    lb.n = 1; lb.T = T;
    LoraProblem & l = lb.p[0];
    l.d.A = hb.in(ha.data(), ha.size()); l.d.Bt = hb.in(hbt.data(), hbt.size()); l.d.rank = rank; l.d.scale = scale;
    l.K = K; l.M = M;
    l.x = hb.in(x, (size_t) K * T); l.ldx = K;
    l.u = hb.out(u, R * T);
    l.P.epi = epilogue; l.P.ldy = M;
    const bool residual = epilogue == EPI_ADD || epilogue == EPI_MUL_ADD;
    if (residual) {
        l.P.y = hb.inout(z, y, (size_t) M * T);
        l.P.res = l.P.y; l.P.ldres = M;
        if (epilogue == EPI_MUL_ADD) { l.P.gate = hb.in(gate, (size_t) M * T); l.P.ldgate = M; }
    } else {
        l.z = hb.in(z, (size_t) M * T); l.ldz = M;
        l.P.y = hb.out(y, (size_t) M * T);
    }
    cudaError_t e = cudaSuccess;
    if (hb.ok) e = launch_lora_shrink(lb, 0);
    if (hb.ok && e == cudaSuccess) e = launch_lora_expand(lb, 0);
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, hb.finish(e), "lora failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_layer_norm_columns(const float * x, const float * w, const float * b, int C, int T, float * y) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, x && w && b && y && C > 0 && T > 0 && T <= 256, "Invalid layer_norm_columns arguments");
    if (!hook_device(sink)) return false;
    HookBuffers hb;
    const float * d_x = hb.in(x, (size_t) C * T), * d_w = hb.in(w, C), * d_b = hb.in(b, C);
    float * d_y = hb.out(y, (size_t) C * T);
    const cudaError_t e = hb.ok ? launch_layer_norm_columns(d_x, d_w, d_b, C, T, d_y, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, hb.finish(e), "layer_norm_columns failed: %s",
               cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_ln_mix(const struct rwkv_b200_ln_mix_args * a) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    bool args = a && a->x && a->ln_w && a->ln_b && a->state_in && a->state_out && a->C > 0 && a->T > 0 && (a->formula == 0 || a->formula == 1) &&
                a->n_out >= 1 && a->n_out <= 6 && seq_layout_ok(a->n_seq, a->seq_stride, a->T, (size_t) a->C);
    for (int j = 0; args && j < a->n_out; j++) args = a->coef[j] && a->out[j];
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args, "Invalid ln_mix arguments");
    if (!hook_device(sink)) return false;
    const size_t C = (size_t) a->C, cols = a->n_seq > 0 ? (size_t) a->n_seq : (size_t) a->T, st = seq_floats(a->n_seq, a->seq_stride, C);
    HookBuffers b;
    LnMixParams p{};
    p.x = b.in(a->x, C * cols); p.ln_w = b.in(a->ln_w, C); p.ln_b = b.in(a->ln_b, C);
    p.state_in = b.in(a->state_in, st); p.state_out = b.out(a->state_out, st);
    p.C = a->C; p.T = (int) cols; p.formula = a->formula; p.n_out = a->n_out; p.seq_stride = a->n_seq > 0 ? a->seq_stride : 0;
    for (int j = 0; j < a->n_out; j++) { p.coef[j] = b.in(a->coef[j], C); p.out[j] = b.out(a->out[j], C * cols); }
    p.out_xx = b.out(a->out_xx, C * cols); p.out_sx = b.out(a->out_sx, C * cols);
    const cudaError_t e = b.ok ? launch_ln_mix(p, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "ln_mix failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_v6_lerp(const struct rwkv_b200_v6_lerp_args * a) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    bool args = a && a->w2 && a->z && a->xx && a->sx && a->C > 0 && a->T > 0 && a->mix > 0;
    int n_q = 0;
    for (int j = 0; args && j < 5; j++) {
        args = a->maa[j] && a->out[j] && staged_ok(a->q_out[j], a->q_type[j], a->T, 0, a->C);
        n_q += a->q_out[j] != nullptr;
    }
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args && (n_q == 0 || n_q == 5), "Invalid v6_lerp arguments (staged columns: all five or none)");
    if (!hook_device(sink)) return false;
    const size_t C = (size_t) a->C, T = (size_t) a->T, mix = (size_t) a->mix;
    HookBuffers b;
    V6LerpParams p{};
    p.w2 = b.in(a->w2, 5 * C * mix); p.z = b.in(a->z, 5 * mix * T); p.xx = b.in(a->xx, C * T); p.sx = b.in(a->sx, C * T);
    for (int j = 0; j < 5; j++) {
        p.maa[j] = b.in(a->maa[j], C); p.out[j] = b.out(a->out[j], C * T);
        p.q_out[j] = a->q_out[j] ? b.out(a->q_out[j], act::bytes_per_column(a->q_type[j], a->C)) : nullptr;
        p.q_type[j] = a->q_type[j];
    }
    p.C = a->C; p.T = a->T; p.mix = a->mix;
    const cudaError_t e = b.ok ? launch_v6_lerp(p, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "v6_lerp failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_wkv4(const struct rwkv_b200_wkv4_args * a) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    const bool args = a && a->k && a->v && a->r && a->time_first && a->time_decay && a->aa_in && a->bb_in && a->pp_in && a->aa_out && a->bb_out && a->pp_out && a->y &&
                      a->C > 0 && a->T > 0 && seq_layout_ok(a->n_seq, a->seq_stride, a->T, (size_t) a->C) && staged_ok(a->q_out, a->q_type, a->T, a->n_seq, a->C);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args, "Invalid wkv4 arguments");
    if (!hook_device(sink)) return false;
    const size_t C = (size_t) a->C, cols = a->n_seq > 0 ? (size_t) a->n_seq : (size_t) a->T, st = seq_floats(a->n_seq, a->seq_stride, C);
    HookBuffers b;
    Wkv4Params p{};
    p.k = b.in(a->k, C * cols); p.v = b.in(a->v, C * cols); p.r = b.in(a->r, C * cols);
    p.time_first = b.in(a->time_first, C); p.time_decay = b.in(a->time_decay, C);
    p.aa_in = b.in(a->aa_in, st); p.bb_in = b.in(a->bb_in, st); p.pp_in = b.in(a->pp_in, st);
    p.aa_out = b.out(a->aa_out, st); p.bb_out = b.out(a->bb_out, st); p.pp_out = b.out(a->pp_out, st);
    p.y = b.out(a->y, C * cols);
    p.C = a->C; p.T = (int) cols; p.seq_stride = a->n_seq > 0 ? a->seq_stride : 0;
    p.q_out = a->q_out ? b.out(a->q_out, act::bytes_per_column(a->q_type, a->C)) : nullptr; p.q_type = a->q_type;
    const cudaError_t e = b.ok ? launch_wkv4(p, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "wkv4 failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_wkv6(const struct rwkv_b200_wkv6_args * a) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    const size_t C = a ? (size_t) a->H * (size_t) a->S : 0, SS = a ? C * (size_t) a->S : 0;
    const bool args = a && a->r && a->k && a->v && a->td && a->tf && a->state_in && a->state_out && a->lnx_w && a->lnx_b && a->y && a->H > 0 && a->S > 0 && a->T > 0 &&
                      !(a->td_per_token && a->per_head_scalars) && seq_layout_ok(a->n_seq, a->seq_stride, a->T, SS) &&
                      a->seq_stride % 4 == 0 &&          // wkv6_kernel moves the state in float4s from state + seq * seq_stride
                      staged_ok(a->q_out, a->q_type, a->T, a->n_seq, a->S);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args, "Invalid wkv6 arguments");
    if (!hook_device(sink)) return false;
    const size_t cols = a->n_seq > 0 ? (size_t) a->n_seq : (size_t) a->T, st = seq_floats(a->n_seq, a->seq_stride, SS);
    HookBuffers b;
    Wkv6Params p{};
    p.r = b.in(a->r, C * cols); p.k = b.in(a->k, C * cols); p.v = b.in(a->v, C * cols);
    p.td = b.in(a->td, a->td_per_token ? C * cols : a->per_head_scalars ? (size_t) a->H : C);
    p.tf = b.in(a->tf, a->per_head_scalars ? (size_t) a->H : C);
    p.td_per_token = a->td_per_token; p.per_head_scalars = a->per_head_scalars;
    p.state_in = b.in(a->state_in, st); p.state_out = b.out(a->state_out, st);
    p.lnx_w = b.in(a->lnx_w, C); p.lnx_b = b.in(a->lnx_b, C); p.g = b.in(a->g, C * cols);
    p.y = b.out(a->y, C * cols);
    p.eps = a->eps; p.H = a->H; p.S = a->S; p.T = (int) cols; p.seq_stride = a->n_seq > 0 ? a->seq_stride : 0;
    p.q_out = a->q_out ? b.out(a->q_out, act::bytes_per_column(a->q_type, (int) C)) : nullptr; p.q_type = a->q_type;
    const cudaError_t e = b.ok ? launch_wkv6(p, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "wkv6 failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_wkv7(const struct rwkv_b200_wkv7_args * a) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    const size_t C = a ? (size_t) a->H * (size_t) a->S : 0, SS = a ? C * (size_t) a->S : 0;
    const bool args = a && a->r && a->w && a->k && a->v && a->a && a->g && (!a->vgate || a->v_first) && a->k_k && a->k_a && a->r_k && a->lnx_w && a->lnx_b &&
                      a->state_in && a->state_out && a->y && a->H > 0 && a->S > 0 && a->T > 0 && seq_layout_ok(a->n_seq, a->seq_stride, a->T, SS) &&
                      staged_ok(a->q_out, a->q_type, a->T, a->n_seq, a->S);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args, "Invalid wkv7 arguments");
    if (!hook_device(sink)) return false;
    const size_t cols = a->n_seq > 0 ? (size_t) a->n_seq : (size_t) a->T, st = seq_floats(a->n_seq, a->seq_stride, SS), n = C * cols;
    HookBuffers b;
    Wkv7Params p{};
    p.r = b.in(a->r, n); p.w = b.in(a->w, n); p.k = b.in(a->k, n); p.v = b.in(a->v, n); p.a = b.in(a->a, n); p.g = b.in(a->g, n);
    p.vgate = b.in(a->vgate, n); p.v_first = a->vgate ? b.in(a->v_first, n) : nullptr; p.v_out = b.out(a->v_out, n);
    p.k_k = b.in(a->k_k, C); p.k_a = b.in(a->k_a, C); p.r_k = b.in(a->r_k, C); p.lnx_w = b.in(a->lnx_w, C); p.lnx_b = b.in(a->lnx_b, C);
    p.state_in = b.in(a->state_in, st); p.state_out = b.out(a->state_out, st);
    p.y = b.out(a->y, n);
    p.H = a->H; p.S = a->S; p.T = (int) cols; p.seq_stride = a->n_seq > 0 ? a->seq_stride : 0;
    p.q_out = a->q_out ? b.out(a->q_out, act::bytes_per_column(a->q_type, (int) C)) : nullptr; p.q_type = a->q_type;
    const cudaError_t e = b.ok ? launch_wkv7(p, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "wkv7 failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_ln_mix_ragged(const struct rwkv_b200_ln_mix_args * a, const uint32_t * counts, size_t n_seq) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    bool args = a && a->x && a->ln_w && a->ln_b && a->state_in && a->state_out && a->C > 0 && (a->formula == 0 || a->formula == 1) &&
                a->n_out >= 1 && a->n_out <= 6 && ragged_ok(counts, n_seq, a->n_seq, a->T, a->seq_stride, (size_t) a->C);
    for (int j = 0; args && j < a->n_out; j++) args = a->coef[j] && a->out[j];
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args, "Invalid ragged ln_mix arguments");
    if (!hook_device(sink)) return false;
    const size_t C = (size_t) a->C, cols = (size_t) a->T, st = seq_floats((int) n_seq, a->seq_stride, C);
    const RaggedMap map(counts, n_seq);
    HookBuffers b;
    LnMixParams p{};
    p.x = b.in(a->x, C * cols); p.ln_w = b.in(a->ln_w, C); p.ln_b = b.in(a->ln_b, C);
    p.state_in = b.in(a->state_in, st); p.state_out = b.out(a->state_out, st);
    p.C = a->C; p.T = a->T; p.formula = a->formula; p.n_out = a->n_out; p.seq_stride = a->seq_stride;
    p.seq_off = b.in(map.off.data(), map.off.size()); p.col_seq = b.in(map.col_seq.data(), map.col_seq.size());
    for (int j = 0; j < a->n_out; j++) { p.coef[j] = b.in(a->coef[j], C); p.out[j] = b.out(a->out[j], C * cols); }
    p.out_xx = b.out(a->out_xx, C * cols); p.out_sx = b.out(a->out_sx, C * cols);
    const cudaError_t e = b.ok ? launch_ln_mix(p, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "ragged ln_mix failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_wkv4_ragged(const struct rwkv_b200_wkv4_args * a, const uint32_t * counts, size_t n_seq) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    const bool args = a && a->k && a->v && a->r && a->time_first && a->time_decay && a->aa_in && a->bb_in && a->pp_in && a->aa_out && a->bb_out && a->pp_out && a->y &&
                      a->C > 0 && !a->q_out && ragged_ok(counts, n_seq, a->n_seq, a->T, a->seq_stride, (size_t) a->C);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args, "Invalid ragged wkv4 arguments");
    if (!hook_device(sink)) return false;
    const size_t C = (size_t) a->C, cols = (size_t) a->T, st = seq_floats((int) n_seq, a->seq_stride, C);
    const RaggedMap map(counts, n_seq);
    HookBuffers b;
    Wkv4Params p{};
    p.k = b.in(a->k, C * cols); p.v = b.in(a->v, C * cols); p.r = b.in(a->r, C * cols);
    p.time_first = b.in(a->time_first, C); p.time_decay = b.in(a->time_decay, C);
    p.aa_in = b.in(a->aa_in, st); p.bb_in = b.in(a->bb_in, st); p.pp_in = b.in(a->pp_in, st);
    p.aa_out = b.out(a->aa_out, st); p.bb_out = b.out(a->bb_out, st); p.pp_out = b.out(a->pp_out, st);
    p.y = b.out(a->y, C * cols);
    p.C = a->C; p.T = a->T; p.seq_stride = a->seq_stride; p.q_out = nullptr; p.q_type = 0;
    p.seq_off = b.in(map.off.data(), map.off.size()); p.n_seq = (int) n_seq;
    const cudaError_t e = b.ok ? launch_wkv4(p, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "ragged wkv4 failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_wkv6_ragged(const struct rwkv_b200_wkv6_args * a, const uint32_t * counts, size_t n_seq) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    const size_t C = a ? (size_t) a->H * (size_t) a->S : 0, SS = a ? C * (size_t) a->S : 0;
    const bool args = a && a->r && a->k && a->v && a->td && a->tf && a->state_in && a->state_out && a->lnx_w && a->lnx_b && a->y && a->H > 0 && a->S > 0 &&
                      !(a->td_per_token && a->per_head_scalars) && !a->q_out && a->seq_stride % 4 == 0 &&
                      ragged_ok(counts, n_seq, a->n_seq, a->T, a->seq_stride, SS);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args, "Invalid ragged wkv6 arguments");
    if (!hook_device(sink)) return false;
    const size_t cols = (size_t) a->T, st = seq_floats((int) n_seq, a->seq_stride, SS);
    const RaggedMap map(counts, n_seq);
    HookBuffers b;
    Wkv6Params p{};
    p.r = b.in(a->r, C * cols); p.k = b.in(a->k, C * cols); p.v = b.in(a->v, C * cols);
    p.td = b.in(a->td, a->td_per_token ? C * cols : a->per_head_scalars ? (size_t) a->H : C);
    p.tf = b.in(a->tf, a->per_head_scalars ? (size_t) a->H : C);
    p.td_per_token = a->td_per_token; p.per_head_scalars = a->per_head_scalars;
    p.state_in = b.in(a->state_in, st); p.state_out = b.out(a->state_out, st);
    p.lnx_w = b.in(a->lnx_w, C); p.lnx_b = b.in(a->lnx_b, C); p.g = b.in(a->g, C * cols);
    p.y = b.out(a->y, C * cols);
    p.eps = a->eps; p.H = a->H; p.S = a->S; p.T = a->T; p.seq_stride = a->seq_stride; p.q_out = nullptr; p.q_type = 0;
    p.seq_off = b.in(map.off.data(), map.off.size()); p.n_seq = (int) n_seq;
    const cudaError_t e = b.ok ? launch_wkv6(p, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "ragged wkv6 failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_wkv7_ragged(const struct rwkv_b200_wkv7_args * a, const uint32_t * counts, size_t n_seq) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    const size_t C = a ? (size_t) a->H * (size_t) a->S : 0, SS = a ? C * (size_t) a->S : 0;
    const bool args = a && a->r && a->w && a->k && a->v && a->a && a->g && (!a->vgate || a->v_first) && a->k_k && a->k_a && a->r_k && a->lnx_w && a->lnx_b &&
                      a->state_in && a->state_out && a->y && a->H > 0 && a->S > 0 && !a->q_out && ragged_ok(counts, n_seq, a->n_seq, a->T, a->seq_stride, SS);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args, "Invalid ragged wkv7 arguments");
    if (!hook_device(sink)) return false;
    const size_t cols = (size_t) a->T, st = seq_floats((int) n_seq, a->seq_stride, SS), n = C * cols;
    const RaggedMap map(counts, n_seq);
    HookBuffers b;
    Wkv7Params p{};
    p.r = b.in(a->r, n); p.w = b.in(a->w, n); p.k = b.in(a->k, n); p.v = b.in(a->v, n); p.a = b.in(a->a, n); p.g = b.in(a->g, n);
    p.vgate = b.in(a->vgate, n); p.v_first = a->vgate ? b.in(a->v_first, n) : nullptr; p.v_out = b.out(a->v_out, n);
    p.k_k = b.in(a->k_k, C); p.k_a = b.in(a->k_a, C); p.r_k = b.in(a->r_k, C); p.lnx_w = b.in(a->lnx_w, C); p.lnx_b = b.in(a->lnx_b, C);
    p.state_in = b.in(a->state_in, st); p.state_out = b.out(a->state_out, st);
    p.y = b.out(a->y, n);
    p.H = a->H; p.S = a->S; p.T = a->T; p.seq_stride = a->seq_stride; p.q_out = nullptr; p.q_type = 0;
    p.seq_off = b.in(map.off.data(), map.off.size()); p.n_seq = (int) n_seq;
    const cudaError_t e = b.ok ? launch_wkv7(p, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "ragged wkv7 failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

static GemvProblem fold_problem(int type, int K, int M, int epi) {
    GemvProblem p{};
    p.type = type; p.K = K; p.M = M; p.epi = epi; p.ldx = K; p.ldy = M;
    p.pitch = dtype_loadable(type) && K > 0 && K % dtype_block_elems(type) == 0 ? matrix_pitch(type, (uint64_t) K) : 0;
    return p;
}

bool rwkv_b200_v6_lora_fold_supported(int n_embed, int head_size, int w1_type, int mix, int w2_type, int decay) {
    if (mix < 1 || decay < 1) return false;
    GemvProblem w1 = fold_problem(w1_type, n_embed, 5 * mix, EPI_TANH), dw2 = fold_problem(w2_type, decay, n_embed, EPI_BIAS_EXPNEGEXP);
    return v6_lora_fold_shapes(n_embed, head_size, w1, dw2);
}

bool rwkv_b200_test_v6_prologue(const struct rwkv_b200_v6_prologue_args * a) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    GemvProblem w1 = fold_problem(a ? a->w1_type : -1, a ? a->C : 0, a ? a->M1 : 0, EPI_TANH);
    const bool args = a && a->x && a->ln_w && a->ln_b && a->state_in && a->coef && a->state_out && a->out_xx && a->out_sx && a->w1 && a->y1 &&
                      a->M1 > 0 && v6_prologue_fits(a->C, w1);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args, "Invalid v6_prologue arguments");
    if (!hook_device(sink)) return false;
    const size_t C = (size_t) a->C;
    HookBuffers b;
    LnMixParams p{};
    p.x = b.in(a->x, C); p.ln_w = b.in(a->ln_w, C); p.ln_b = b.in(a->ln_b, C);
    p.state_in = b.in(a->state_in, C); p.state_out = b.out(a->state_out, C);
    p.C = a->C; p.T = 1; p.formula = 1; p.n_out = 1; p.coef[0] = b.in(a->coef, C);
    p.out_xx = b.out(a->out_xx, C); p.out_sx = b.out(a->out_sx, C);
    uint8_t * W = static_cast<uint8_t *>(b.alloc((size_t) a->M1 * (size_t) w1.pitch + 256));
    if (b.ok) b.ok = upload_matrix(a->w1, a->w1_type, a->M1, a->C, W, nullptr) == cudaSuccess;
    w1.W = W; w1.y = b.out(a->y1, (size_t) a->M1);
    const cudaError_t e = b.ok ? launch_v6_prologue(p, w1, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "v6_prologue failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_wkv6_decay(const struct rwkv_b200_wkv6_decay_args * a) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    const int C = a ? a->H * 64 : 0;
    GemvProblem dw2 = fold_problem(a ? a->w2_type : -1, a ? a->K2 : 0, C, EPI_BIAS_EXPNEGEXP);
    const bool args = a && a->r && a->k && a->v && a->tf && a->state_in && a->state_out && a->lnx_w && a->lnx_b && a->y && a->w2 && a->lora1 &&
                      a->td_bias && a->H > 0 && a->H <= 4096 / 64 && wkv6_decay_fits(C, 64, dw2) && staged_ok(a->q_out, a->q_type, 1, 0, 64);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args, "Invalid wkv6_decay arguments");
    if (!hook_device(sink)) return false;
    const size_t Cs = (size_t) C;
    HookBuffers b;
    Wkv6Params p{};
    p.r = b.in(a->r, Cs); p.k = b.in(a->k, Cs); p.v = b.in(a->v, Cs); p.tf = b.in(a->tf, Cs);
    p.td = nullptr; p.td_per_token = 0; p.per_head_scalars = 0;
    p.state_in = b.in(a->state_in, Cs * 64); p.state_out = b.out(a->state_out, Cs * 64);
    p.lnx_w = b.in(a->lnx_w, Cs); p.lnx_b = b.in(a->lnx_b, Cs); p.g = b.in(a->g, Cs);
    p.y = b.out(a->y, Cs);
    p.eps = a->eps; p.H = a->H; p.S = 64; p.T = 1;
    p.q_out = a->q_out ? b.out(a->q_out, act::bytes_per_column(a->q_type, C)) : nullptr; p.q_type = a->q_type;
    uint8_t * W = static_cast<uint8_t *>(b.alloc(Cs * (size_t) dw2.pitch + 256));
    if (b.ok) b.ok = upload_matrix(a->w2, a->w2_type, C, a->K2, W, nullptr) == cudaSuccess;
    dw2.W = W; dw2.x = b.in(a->lora1, (size_t) a->K2); dw2.bias = b.in(a->td_bias, Cs);
    p.dw2 = dw2;
    const cudaError_t e = b.ok ? launch_wkv6(p, 0) : cudaSuccess;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "wkv6_decay failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

bool rwkv_b200_test_gemv_batch(const struct rwkv_b200_gemv_batch_args * a) {
    g_last_error = RWKV_ERROR_NONE;
    ErrorSink sink = global_sink();
    bool args = a && a->T >= 1 && a->T <= 256 && a->n >= 1 && a->n <= GEMV_MAX_PROBLEMS && a->path >= RWKV_B200_GEMV_ENGINE &&
                a->path <= RWKV_B200_GEMV_TENSOR_CORES && (!a->launches || (a->n_launches && a->max_launches >= 0));
    int input_K[GEMV_MAX_PROBLEMS] = {};
    for (int i = 0; args && i < a->n; i++) {
        const rwkv_b200_gemv_problem & q = a->p[i];
        const bool ln = q.pro == PRO_LAYERNORM, res_epi = q.epi == EPI_ADD || q.epi == EPI_MUL_ADD, bias_epi = q.epi >= EPI_BIAS_EXPNEGEXP;
        args = q.weights && q.y && dtype_loadable(q.type) && q.K > 0 && q.M > 0 && q.K % dtype_block_elems(q.type) == 0 &&
               q.input >= 0 && q.input < GEMV_MAX_PROBLEMS && a->x[q.input] && (input_K[q.input] == 0 || input_K[q.input] == q.K) &&
               q.epi >= EPI_NONE && q.epi <= EPI_BIAS_W7 && (q.pro == PRO_NONE || ln) &&
               !q.res == !res_epi && !q.gate == (q.epi != EPI_MUL_ADD) && !q.bias == !bias_epi && (!q.y_aliases_res || q.res) &&
               !q.ln_w == !ln && !q.ln_b == !ln &&
               (!q.xq || (a->T == 1 && act::stage_class(q.type) != act::SC_NONE)) &&   // the streaming kernel reads xq of single-token launches only
               (!q.tiled || gemm_tc_eligible(q.type, q.K));
        if (args) input_K[q.input] = q.K;
        // the streaming path runs one kernel: all problems K-quant of one type (gemv_kq_launch) or none (gemv_tma_launch)
        if (args && a->path == RWKV_B200_GEMV_STREAMING) args = dtype_kquant(q.type) ? q.type == a->p[0].type : !dtype_kquant(a->p[0].type);
    }
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, args, "Invalid gemv_batch arguments");
    if (!hook_device(sink)) return false;
    cudaDeviceProp prop;
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, cudaGetDeviceProperties(&prop, default_device()) == cudaSuccess, "cudaGetDeviceProperties failed");
    const DeviceInfo di{default_device(), prop.multiProcessorCount, (int) prop.sharedMemPerBlockOptin};
    LaunchLog log{};
    struct LogScope {
        explicit LogScope(LaunchLog * l) { g_launch_log = l; }
        ~LogScope() { g_launch_log = nullptr; }
    } scope(a->launches ? &log : nullptr);      // from the upload on: the tensor-core weight expansion is recorded too
    HookBuffers b;
    const size_t T = (size_t) a->T;
    const float * dx[GEMV_MAX_PROBLEMS] = {};
    size_t k_max = 0;
    for (int j = 0; j < GEMV_MAX_PROBLEMS; j++) {
        if (input_K[j]) dx[j] = b.in(a->x[j], (size_t) input_K[j] * T);
        if ((size_t) input_K[j] > k_max) k_max = (size_t) input_K[j];
    }
    GemvBatch batch;
    memset(&batch, 0, sizeof(batch));
    batch.n = a->n; batch.T = a->T;
    bool tc_ok = true;
    for (int i = 0; i < a->n; i++) {
        const rwkv_b200_gemv_problem & q = a->p[i];
        GemvProblem & p = batch.p[i];
        const size_t MT = (size_t) q.M * T;
        p.type = q.type; p.K = q.K; p.M = q.M;
        p.pitch = matrix_pitch(q.type, (uint64_t) q.K);
        uint8_t * W = static_cast<uint8_t *>(b.alloc((size_t) q.M * (size_t) p.pitch + 256));
        uint8_t * Wt = q.tiled ? static_cast<uint8_t *>(b.alloc(gemm_tc_tiled_bytes(q.type, q.M, q.K))) : nullptr;
        if (b.ok) b.ok = upload_matrix(q.weights, q.type, q.M, q.K, W, Wt) == cudaSuccess;
        p.W = W; p.Wt = Wt;
        p.x = dx[q.input]; p.ldx = q.K;
        p.y = q.y_aliases_res ? b.inout(q.res, q.y, MT) : b.out(q.y, MT); p.ldy = q.M;
        p.res = q.y_aliases_res ? p.y : b.in(q.res, MT); p.ldres = q.M;
        p.gate = b.in(q.gate, MT); p.ldgate = q.M;
        p.bias = b.in(q.bias, (size_t) q.M);
        p.ln_w = b.in(q.ln_w, (size_t) q.K); p.ln_b = b.in(q.ln_b, (size_t) q.K);
        p.xq = q.xq ? b.in(q.xq, act::bytes_per_column(q.type, q.K)) : nullptr;
        p.epi = q.epi; p.pro = q.pro;
        tc_ok = tc_ok && gemm_tc_supported(p, a->T);
    }
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, a->path != RWKV_B200_GEMV_TENSOR_CORES || !b.ok || tc_ok,
               "A problem of the batch cannot take the tensor-core path");
    void * ws = nullptr;
    size_t ws_bytes = 0;
    if (a->path == RWKV_B200_GEMV_ENGINE || a->path == RWKV_B200_GEMV_ENGINE_BATCH_CTX || a->path == RWKV_B200_GEMV_TENSOR_CORES) {
        ws_bytes = gemm_tc_batch_workspace_bytes(a->T, k_max);      // as the engine sizes its workspace (ensure_capacity)
        ws = b.alloc(ws_bytes);
    }
    cudaError_t e = cudaSuccess;
    if (b.ok) {
        switch (a->path) {
            case RWKV_B200_GEMV_STREAMING: e = dtype_kquant(batch.p[0].type) ? gemv_kq_launch(batch, di, 0) : gemv_tma_launch(batch, di, 0); break;
            case RWKV_B200_GEMV_GENERIC: e = gemv_generic_launch(batch, di, 0); break;
            case RWKV_B200_GEMV_TENSOR_CORES: e = gemm_tc_launch(batch, di, 0, ws, ws_bytes); break;
            default: e = gemv_route(batch, di, 0, ws, ws_bytes, a->path == RWKV_B200_GEMV_ENGINE ? 32 : 16); break;
        }
    }
    if (a->launches) {
        const int n = log.n < a->max_launches ? log.n : a->max_launches;
        for (int i = 0; i < n; i++) {
            const LaunchRec & r = log.rec[i];
            a->launches[i] = rwkv_b200_gemv_launch{r.family, r.nc, r.only, r.has_ln, r.npad, r.cluster};
        }
        *a->n_launches = n;
    }
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, false, b.finish(e), "gemv_batch failed: %s", cudaGetErrorString(e != cudaSuccess ? e : cudaGetLastError()));
    return true;
}

}  // extern "C"
