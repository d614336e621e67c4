// Device-resident RWKV model: per-arch tensor table + loader.
// Mirrors the reference's rwkv_model / rwkv_layer (rwkv_model_loading.inc:1-112) but every tensor
// lives in one HBM arena: matrices keep their file format (ggml quant blocks / f16 / f32, rows
// padded to a 16-byte pitch), everything that is consumed element-wise is widened to fp32 once.
#pragma once
#include <atomic>
#include <cstdint>
#include <mutex>
#include <string>
#include <vector>

#include "cuda_handles.h"
#include "errors.h"
#include "ggml_file.h"
#include "kernels/gemv.h"
#include "kernels/lora.h"
#include "kernels/ops.h"

namespace rwkv {

struct DevMatrix {          // y = W x : K = ne0 (input), M = ne1*ne2 (output rows)
    const uint8_t * data = nullptr;
    const uint8_t * tiled = nullptr;   // tile-major prefill copy (gemm_tc_repack) or NULL
    int type = 0, K = 0, M = 0;
    long long pitch = 0;
    const LoraDelta * lora = nullptr;  // the low-rank delta of an attached adapter (Adapter::layers only), or NULL
    explicit operator bool() const { return data != nullptr; }
};
struct DevVec {
    const float * data = nullptr;
    size_t n = 0;
    explicit operator bool() const { return data != nullptr; }
};

struct Layer {
    DevVec ln1_w, ln1_b, ln2_w, ln2_b;
    // time mixing, v4 / v5 (rwkv_model_loading.inc:210-250)
    DevVec att_time_mix_k, att_time_mix_v, att_time_mix_r, att_time_mix_g;
    DevVec att_time_first, att_time_decay, att_time_faaaa;
    DevMatrix att_key, att_value, att_receptance, att_output, att_gate;
    DevVec att_ln_x_w, att_ln_x_b;
    // v6 (rwkv_model_loading.inc:186-209)
    DevVec att_maa_x, att_maa_w, att_maa_k, att_maa_v, att_maa_r, att_maa_g;
    DevMatrix att_maa_w1, att_decay_w1, att_decay_w2;
    DevVec att_maa_w2;      // fp32 [5][C][mix]
    int maa_mix = 0;
    // v7 (rwkv_model_loading.inc:152-185)
    DevVec att_x_rwkvag;    // [6][C]: r, w, k, v, a, g
    DevVec att_w0, att_a0, att_v0, att_k_k, att_k_a, att_r_k;
    DevMatrix att_w1, att_w2, att_a1, att_a2, att_g1, att_g2, att_v1, att_v2;
    // channel mixing
    DevVec ffn_time_mix_k, ffn_time_mix_r, ffn_maa_k, ffn_maa_r, ffn_x_k;
    DevMatrix ffn_key, ffn_value, ffn_receptance;
};

// Peer-memory hand-off of a pipeline stage (kernels/pipe.cu): the stage's own mailbox + credit word (`box`, exported through CUDA
// IPC or shared inside the process) and the mappings of its neighbours'. One per model: every context (in-flight sequence) of a
// stage sends and receives through the same link, in item order, on one stream.
struct PipeLink {
    DeviceBuffer<PipeBox> box;             // my mailbox allocation: PipeBox + PIPE_SLOTS x slot_floats floats
    size_t slot_floats = 0, bytes = 0;
    PipeBox * prev = nullptr, * next = nullptr;
    bool prev_ipc = false, next_ipc = false;
    DeviceBuffer<unsigned long long> counters;   // device: tickets / completions of the hand-off kernels
};

struct Model {
    FileHeader header{};
    int arch_major = 4, arch_minor = 0;
    int head_count = 0, head_size = 0;
    int n_embed = 0, n_vocab = 0, n_layer = 0;
    // layers [layer_begin, layer_end) are resident on this device; emb iff layer_begin == 0,
    // ln_out + head iff layer_end == n_layer (pipeline stages, SURVEY.md section 8e).
    int layer_begin = 0, layer_end = 0;
    DevMatrix emb, head;
    DevVec ln0_w, ln0_b, ln_out_w, ln_out_b;
    std::vector<Layer> layers;      // indexed by absolute layer id; non-resident entries are empty

    DeviceInfo dev{};
    DeviceBuffer<uint8_t> arena;
    size_t arena_bytes = 0;
    size_t tiled_bytes = 0;              // of which: tile-major prefill copies of the layer matrices
    size_t weight_bytes_per_token = 0;   // byte model of SURVEY.md 8(d), resident layers, with head
    size_t head_bytes = 0;
    size_t gemv_bytes_per_token = 0;     // of which: matrices streamed by the fused dequantize-GEMV (layer matrices + head)
    size_t head_matrix_bytes = 0;
    // The head's tile-major copy for the tensor-core head of scoring passes (engine.cu: ensure_head_tiled), built by the first one
    // that needs it, under head_tiled_lock, and freed with the model. Every other pass streams the head with the GEMV.
    DeviceBuffer<uint8_t> head_tiled;
    std::mutex head_tiled_lock;
    std::atomic<int> refcount{0};
    PipeLink link;
    std::string device_name;

    size_t state_floats_per_layer() const {
        return (size_t) n_embed * (arch_major >= 5 ? (size_t) (2 + head_size) : (size_t) 5);
    }
    size_t state_len() const { return state_floats_per_layer() * (size_t) n_layer; }
    ~Model();
};

// One entry of a model's parameter table (rwkv_set_params, rwkv_model_loading.inc:128-285): the tensor's name in the file, the
// matrix or vector it is loaded into (exactly one is set) and its expected shape (0 = unchecked).
struct ParamSlot {
    std::string name;
    DevMatrix * mat = nullptr;
    DevVec * vec = nullptr;
    uint64_t expect_k = 0, expect_m = 0;
    uint64_t expect_n = 0;
};
struct TopTensors { DevMatrix * emb, * head; DevVec * ln0_w, * ln0_b, * ln_out_w, * ln_out_b; };
// The table of m's architecture, resident layers and head geometry, in the loader's key order, with the slots pointing into
// `layers` (indexed by absolute layer id) and `top`. The loader passes m's own tensors; an adapter passes its copies of them.
std::vector<ParamSlot> param_table(const Model & m, Layer * layers, const TopTensors & top);

// Loads `path` onto CUDA device `device`. layer_end < 0 means n_layer. Returns nullptr after
// recording the failure in `sink` (same categories/codes as rwkv_model_loading.inc:288-419).
Model * load_model(const char * path, int device, int layer_begin, int layer_end, ErrorSink sink);

// Device row pitch of a matrix: whole 4-byte-aligned units (pairs of blocks for the 2-byte-aligned formats), then 16-byte rows.
long long matrix_pitch(int type, uint64_t K);
// Uploads M rows of K elements in the file layout of `type` to dst (M * matrix_pitch bytes; the padding of every row is zeroed) and
// brings them into the device layout (weights_to_device_layout). When tiled is not NULL (gemm_tc_tiled_bytes of room) it also writes
// the tile-major copy the tensor-core path streams. The host buffer may be reused when it returns.
cudaError_t upload_matrix(const void * host, int type, int M, int K, uint8_t * dst, uint8_t * tiled);

}  // namespace rwkv
