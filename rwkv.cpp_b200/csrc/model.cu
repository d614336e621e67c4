// Model loader: ggml file -> one HBM arena. Follows the two-pass structure of
// rwkv_load_model_from_file (reference rwkv_model_loading.inc:288-419): scan all tensor records,
// detect the architecture from key names, resolve the per-arch parameter table, then stream the
// payloads to the device.
#define _FILE_OFFSET_BITS 64
#include "model.h"
#include "kernels/gemv.h"   // gemm_tc_tiled_bytes / gemm_tc_repack

#include <cinttypes>
#include <cstdlib>
#include <memory>

#include <cuda_runtime.h>

namespace rwkv {

Model::~Model() {
    if (arena || link.box || head_tiled) cudaSetDevice(dev.device);
    cudaFree(head_tiled);
    if (link.prev && link.prev_ipc) cudaIpcCloseMemHandle(link.prev);
    if (link.next && link.next_ipc) cudaIpcCloseMemHandle(link.next);
    cudaFree(link.box);
    cudaFree(link.counters);
    if (arena) cudaFree(arena);
}

namespace {

struct Request : ParamSlot {
    const TensorInfo * info = nullptr;
    size_t arena_offset = 0;
    size_t tiled_offset = 0, tiled_bytes = 0;   // matrices that get a tile-major prefill copy
};

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Host dequantisation of a whole tensor to fp32 (only for element-wise parameters that someone
// stored in a narrower type; dequantize_row_q*, ggml-quants.c:255-363).
void widen_to_f32(int type, const uint8_t * src, size_t n, float * dst) {
    if (type == DT_F32) { memcpy(dst, src, n * 4); return; }
    if (type == DT_F16) {
        const uint16_t * h = reinterpret_cast<const uint16_t *>(src);
        for (size_t i = 0; i < n; i++) dst[i] = fp16_to_fp32(h[i]);
        return;
    }
    const int bb = dtype_block_bytes(type);
    if (dtype_kquant(type)) {   // dequantize_row_q4_K / dequantize_row_q5_K (ggml-quants.c:1280, 1482)
        for (size_t b = 0; b < n / QK_K; b++) {
            const uint8_t * p = src + b * bb;
            uint16_t dh, mh; memcpy(&dh, p, 2); memcpy(&mh, p + 2, 2);
            const float d = fp16_to_fp32(dh), dmin = fp16_to_fp32(mh);
            const uint8_t * sc = p + 4, * qh = p + 16, * qs = p + (type == DT_Q5_K ? 48 : 16);
            for (int j = 0; j < 8; j++) {
                int s, m;
                kquant_scale_min(sc, j, s, m);
                const float dj = d * (float) s, mj = dmin * (float) m;
                for (int l = 0; l < 32; l++) {
                    int q = (qs[32 * (j / 2) + l] >> (4 * (j & 1))) & 0xF;
                    if (type == DT_Q5_K) q |= ((qh[l] >> j) & 1) << 4;
                    dst[b * QK_K + 32 * j + l] = dj * (float) q - mj;
                }
            }
        }
        return;
    }
    for (size_t b = 0; b < n / 32; b++) {
        const uint8_t * p = src + b * bb;
        uint16_t dh; memcpy(&dh, p, 2);
        const float d = fp16_to_fp32(dh);
        float m = 0.f;
        const uint8_t * qs; uint32_t qh = 0; int off = 0;
        switch (type) {
            case DT_Q4_0: qs = p + 2; off = 8; break;
            case DT_Q4_1: { uint16_t mh; memcpy(&mh, p + 2, 2); m = fp16_to_fp32(mh); qs = p + 4; } break;
            case DT_Q5_0: memcpy(&qh, p + 2, 4); qs = p + 6; off = 16; break;
            case DT_Q5_1: { uint16_t mh; memcpy(&mh, p + 2, 2); m = fp16_to_fp32(mh); memcpy(&qh, p + 4, 4); qs = p + 8; } break;
            default: qs = p + 2; break;  // Q8_0
        }
        float * o = dst + b * 32;
        if (type == DT_Q8_0) {
            for (int j = 0; j < 32; j++) o[j] = (float) (int8_t) qs[j] * d;
        } else {
            const bool five = (type == DT_Q5_0 || type == DT_Q5_1);
            for (int j = 0; j < 16; j++) {
                int q0 = qs[j] & 0x0F, q1 = qs[j] >> 4;
                if (five) { q0 |= ((qh >> j) & 1) << 4; q1 |= ((qh >> (j + 16)) & 1) << 4; }
                o[j] = (float) (q0 - off) * d + m;
                o[j + 16] = (float) (q1 - off) * d + m;
            }
        }
    }
}

}  // namespace

long long matrix_pitch(int type, uint64_t K) {
    size_t bytes = tensor_nbytes(type, K, 1, 1);
    if (type == DT_Q4_0 || type == DT_Q5_0 || type == DT_Q8_0) {
        uint64_t nblk = K / 32;
        bytes = (size_t) ((nblk + 1) / 2 * 2) * dtype_block_bytes(type);
    }
    return (long long) align_up(bytes, 16);
}

cudaError_t upload_matrix(const void * host, int type, int M, int K, uint8_t * dst, uint8_t * tiled) {
    const long long pitch = matrix_pitch(type, (uint64_t) K);
    const size_t row_bytes = tensor_nbytes(type, (uint64_t) K, 1, 1);
    cudaError_t ce;
    if ((size_t) pitch == row_bytes) {
        ce = cudaMemcpy(dst, host, row_bytes * (size_t) M, cudaMemcpyHostToDevice);
    } else {
        ce = cudaMemset(dst, 0, (size_t) M * (size_t) pitch);
        if (ce == cudaSuccess) ce = cudaMemcpy2D(dst, (size_t) pitch, host, row_bytes, row_bytes, (size_t) M, cudaMemcpyHostToDevice);
    }
    if (ce == cudaSuccess) ce = weights_to_device_layout(dst, pitch, type, M, K, 0);      // Q5 fifth-bit words -> device order
    if (ce == cudaSuccess && tiled) {
        ce = gemm_tc_repack(dst, pitch, type, M, K, tiled, 0);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(0);     // the caller may reuse the host buffer
    }
    return ce;
}

std::vector<ParamSlot> param_table(const Model & m, Layer * layers, const TopTensors & top) {
    std::vector<ParamSlot> reqs;
    auto want_vec = [&](const std::string & name, DevVec & dst, uint64_t n) { ParamSlot r; r.name = name; r.vec = &dst; r.expect_n = n; reqs.push_back(r); };
    auto want_mat = [&](const std::string & name, DevMatrix & dst, uint64_t k, uint64_t mm) { ParamSlot r; r.name = name; r.mat = &dst; r.expect_k = k; r.expect_m = mm; reqs.push_back(r); };
    const uint64_t C = (uint64_t) m.n_embed, V = (uint64_t) m.n_vocab, H = (uint64_t) m.head_count;
    const int layer_begin = m.layer_begin, layer_end = m.layer_end;

    if (layer_begin == 0) {
        want_mat("emb.weight", *top.emb, C, V);
        want_vec("blocks.0.ln0.weight", *top.ln0_w, C);
        want_vec("blocks.0.ln0.bias", *top.ln0_b, C);
    }
    for (int i = layer_begin; i < layer_end; i++) {
        Layer & L = layers[i];
        const std::string p = "blocks." + std::to_string(i) + ".";
        want_vec(p + "ln1.weight", L.ln1_w, C);
        want_vec(p + "ln1.bias", L.ln1_b, C);
        switch (m.arch_major) {
            case 7:
                want_vec(p + "att.x_rwkvag", L.att_x_rwkvag, 6 * C);
                want_vec(p + "att.w0", L.att_w0, C);
                want_mat(p + "att.w1", L.att_w1, C, 0);
                want_mat(p + "att.w2", L.att_w2, 0, C);
                want_vec(p + "att.a0", L.att_a0, C);
                want_mat(p + "att.a1", L.att_a1, C, 0);
                want_mat(p + "att.a2", L.att_a2, 0, C);
                want_mat(p + "att.g1", L.att_g1, C, 0);
                want_mat(p + "att.g2", L.att_g2, 0, C);
                if (i != 0) {
                    want_vec(p + "att.v0", L.att_v0, C);
                    want_mat(p + "att.v1", L.att_v1, C, 0);
                    want_mat(p + "att.v2", L.att_v2, 0, C);
                }
                want_vec(p + "att.r_k", L.att_r_k, C);
                want_vec(p + "att.k_k", L.att_k_k, C);
                want_vec(p + "att.k_a", L.att_k_a, C);
                want_mat(p + "att.key.weight", L.att_key, C, C);
                want_mat(p + "att.value.weight", L.att_value, C, C);
                want_mat(p + "att.receptance.weight", L.att_receptance, C, C);
                want_mat(p + "att.output.weight", L.att_output, C, C);
                want_vec(p + "att.ln_x.weight", L.att_ln_x_w, C);
                want_vec(p + "att.ln_x.bias", L.att_ln_x_b, C);
                break;
            case 6:
                want_vec(p + "att.time_maa_x", L.att_maa_x, C);
                want_vec(p + "att.time_maa_w", L.att_maa_w, C);
                want_vec(p + "att.time_maa_k", L.att_maa_k, C);
                want_vec(p + "att.time_maa_v", L.att_maa_v, C);
                want_vec(p + "att.time_maa_r", L.att_maa_r, C);
                want_vec(p + "att.time_maa_g", L.att_maa_g, C);
                want_mat(p + "att.time_maa_w1", L.att_maa_w1, C, 0);
                want_vec(p + "att.time_maa_w2", L.att_maa_w2, 0);
                want_vec(p + "att.time_faaaa", L.att_time_faaaa, C);
                want_vec(p + "att.time_decay", L.att_time_decay, C);
                want_mat(p + "att.time_decay_w1", L.att_decay_w1, C, 0);
                want_mat(p + "att.time_decay_w2", L.att_decay_w2, 0, C);
                want_mat(p + "att.key.weight", L.att_key, C, C);
                want_mat(p + "att.value.weight", L.att_value, C, C);
                want_mat(p + "att.receptance.weight", L.att_receptance, C, C);
                want_mat(p + "att.gate.weight", L.att_gate, C, C);
                want_mat(p + "att.output.weight", L.att_output, C, C);
                want_vec(p + "att.ln_x.weight", L.att_ln_x_w, C);
                want_vec(p + "att.ln_x.bias", L.att_ln_x_b, C);
                break;
            case 5:
                want_vec(p + "att.time_mix_k", L.att_time_mix_k, C);
                want_vec(p + "att.time_mix_v", L.att_time_mix_v, C);
                want_vec(p + "att.time_mix_r", L.att_time_mix_r, C);
                if (m.arch_minor >= 2) want_vec(p + "att.time_faaaa", L.att_time_faaaa, C);
                else want_vec(p + "att.time_first", L.att_time_first, H);
                want_vec(p + "att.time_decay", L.att_time_decay, m.arch_minor >= 2 ? C : H);
                want_mat(p + "att.key.weight", L.att_key, C, C);
                want_mat(p + "att.value.weight", L.att_value, C, C);
                want_mat(p + "att.receptance.weight", L.att_receptance, C, C);
                want_mat(p + "att.output.weight", L.att_output, C, C);
                want_vec(p + "att.ln_x.weight", L.att_ln_x_w, C);
                want_vec(p + "att.ln_x.bias", L.att_ln_x_b, C);
                if (m.arch_minor >= 2) {
                    want_vec(p + "att.time_mix_g", L.att_time_mix_g, C);
                    want_mat(p + "att.gate.weight", L.att_gate, C, C);
                }
                break;
            default:
                want_vec(p + "att.time_mix_k", L.att_time_mix_k, C);
                want_vec(p + "att.time_mix_v", L.att_time_mix_v, C);
                want_vec(p + "att.time_mix_r", L.att_time_mix_r, C);
                want_vec(p + "att.time_first", L.att_time_first, C);
                want_vec(p + "att.time_decay", L.att_time_decay, C);
                want_mat(p + "att.key.weight", L.att_key, C, C);
                want_mat(p + "att.value.weight", L.att_value, C, C);
                want_mat(p + "att.receptance.weight", L.att_receptance, C, C);
                want_mat(p + "att.output.weight", L.att_output, C, C);
                break;
        }
        want_vec(p + "ln2.weight", L.ln2_w, C);
        want_vec(p + "ln2.bias", L.ln2_b, C);
        if (m.arch_major == 7) want_vec(p + "ffn.x_k", L.ffn_x_k, C);
        else if (m.arch_major == 6) { want_vec(p + "ffn.time_maa_k", L.ffn_maa_k, C); want_vec(p + "ffn.time_maa_r", L.ffn_maa_r, C); }
        else { want_vec(p + "ffn.time_mix_k", L.ffn_time_mix_k, C); want_vec(p + "ffn.time_mix_r", L.ffn_time_mix_r, C); }
        want_mat(p + "ffn.key.weight", L.ffn_key, C, 0);
        want_mat(p + "ffn.value.weight", L.ffn_value, 0, C);
        if (m.arch_major != 7) want_mat(p + "ffn.receptance.weight", L.ffn_receptance, C, C);
    }
    if (layer_end == m.n_layer) {
        want_vec("ln_out.weight", *top.ln_out_w, C);
        want_vec("ln_out.bias", *top.ln_out_b, C);
        want_mat("head.weight", *top.head, C, V);
    }
    return reqs;
}

Model * load_model(const char * path, int device, int layer_begin, int layer_end, ErrorSink sink) {
    ModelFile mf;
    RWKV_PROPAGATE(sink, nullptr, scan_model_file(path, mf, sink));

    std::unique_ptr<Model> model(new (std::nothrow) Model());
    RWKV_CHECK(sink, RWKV_ERROR_MODEL | RWKV_ERROR_ALLOC, nullptr, model, "Failed to allocate the model");
    Model & m = *model;
    m.header = mf.header;
    m.n_embed = (int) mf.header.n_embed;
    m.n_vocab = (int) mf.header.n_vocab;
    m.n_layer = (int) mf.header.n_layer;
    if (layer_end < 0 || layer_end > m.n_layer) layer_end = m.n_layer;
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, layer_begin >= 0 && layer_begin < layer_end, "Invalid layer range [%d, %d)", layer_begin, layer_end);
    m.layer_begin = layer_begin;
    m.layer_end = layer_end;

    // Architecture detection by key presence (rwkv_model_loading.inc:319-340).
    m.arch_major = 4; m.arch_minor = 0;
    if (mf.find("blocks.0.att.ln_x.weight")) { m.arch_major = 5; m.arch_minor = mf.find("blocks.0.att.gate.weight") ? 2 : 1; }
    if (mf.find("blocks.0.att.time_maa_x")) { m.arch_major = 6; m.arch_minor = 0; }
    if (mf.find("blocks.0.att.r_k")) { m.arch_major = 7; m.arch_minor = 0; }

    const uint64_t C = mf.header.n_embed, V = mf.header.n_vocab;
    // head geometry (rwkv_model_loading.inc:403-409)
    uint64_t H = 0, S = 0;
    if (m.arch_major == 7) {
        const TensorInfo * rk = mf.find("blocks.0.att.r_k");
        H = rk->ne[1];
    } else if (m.arch_major >= 5) {
        const TensorInfo * td = mf.find("blocks.0.att.time_decay");
        RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_PARAM_MISSING, nullptr, td, "Model parameter %s not found", "blocks.0.att.time_decay");
        H = td->ne[2];
    }
    if (m.arch_major >= 5) {
        RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_SHAPE, nullptr, H > 0 && C % H == 0, "Head count %" PRIu64 " does not divide n_embed %" PRIu64, H, C);
        S = C / H;
        RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_UNSUPPORTED, nullptr, S == 8 || S == 16 || S == 32 || S == 64 || S == 128,
                   "Unsupported head size %" PRIu64, S);
    }
    m.head_count = (int) H;
    m.head_size = (int) S;

    // ---- parameter table (rwkv_set_params, rwkv_model_loading.inc:128-285), same key order ----
    m.layers.resize(m.n_layer);
    std::vector<Request> reqs;
    for (const ParamSlot & ps : param_table(m, m.layers.data(), TopTensors{&m.emb, &m.head, &m.ln0_w, &m.ln0_b, &m.ln_out_w, &m.ln_out_b})) {
        Request r;
        static_cast<ParamSlot &>(r) = ps;
        reqs.push_back(r);
    }

    // ---- resolve + validate + lay out the arena ----
    const bool tc_copies = getenv("RWKV_B200_NO_TC") == nullptr;
    size_t arena_bytes = 0, staging_bytes = 0;
    for (Request & r : reqs) {
        r.info = mf.find(r.name);
        RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_PARAM_MISSING, nullptr, r.info, "Model parameter %s not found", r.name.c_str());
        const TensorInfo & t = *r.info;
        const uint64_t n = t.ne[0] * t.ne[1] * t.ne[2];
        if (r.mat) {
            const uint64_t K = t.ne[0], M = t.ne[1] * t.ne[2];
            if (r.name == "emb.weight") {   // rwkv_model_loading.inc:411-416
                RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_SHAPE, nullptr, t.dim_count == 2 && t.ne[2] == 1, "Unexpected dimension count of embedding matrix %" PRIu32, t.dim_count);
                RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_DIMENSION, nullptr, K == C, "Unexpected dimension of embedding matrix %" PRIu64, K);
                RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_DIMENSION, nullptr, M == V, "Unexpected dimension of embedding matrix %" PRIu64, M);
                RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_UNSUPPORTED, nullptr, t.data_type == DT_F32 || t.data_type == DT_F16,
                           "Embedding matrix must be FP32 or FP16, got %s", dtype_name((int) t.data_type));
            }
            RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_SHAPE, nullptr, (r.expect_k == 0 || K == r.expect_k) && (r.expect_m == 0 || M == r.expect_m) && K > 0 && M > 0,
                       "Unexpected shape [%" PRIu64 ", %" PRIu64 "] of parameter %s", K, M, r.name.c_str());
            // no other kernel takes a K-quant matrix, so one whose rows do not fit the K-quant GEMV's streaming plan cannot run
            RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_UNSUPPORTED, nullptr, !dtype_kquant((int) t.data_type) || gemv_kq_fits((int) t.data_type, (int) K),
                       "Rows of %" PRIu64 " weights of %s are too long for the %s kernel; requantize the model in another format", K, r.name.c_str(), dtype_name((int) t.data_type));
            const long long pitch = matrix_pitch((int) t.data_type, K);
            r.arena_offset = arena_bytes;
            arena_bytes += align_up((size_t) M * (size_t) pitch + 256, 256);
            // every per-layer matrix also gets the tile-major copy the tensor-core prefill kernel streams (gemm_tc.cu); the
            // embedding is a gather, and every pass but a scoring pass runs the head on one column per sequence (a scoring pass builds
            // the head's copy when it first needs it, Model::head_tiled)
            if (tc_copies && r.name != "emb.weight" && r.name != "head.weight") {
                r.tiled_bytes = gemm_tc_tiled_bytes((int) t.data_type, (int) M, (int) K);
                r.tiled_offset = arena_bytes;
                arena_bytes += align_up(r.tiled_bytes, 256);
            }
        } else {
            RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_SHAPE, nullptr, (r.expect_n == 0 || n == r.expect_n) && n > 0,
                       "Unexpected element count %" PRIu64 " of parameter %s", n, r.name.c_str());
            r.arena_offset = arena_bytes;
            arena_bytes += align_up((size_t) n * 4, 256);
        }
        if (t.nbytes > staging_bytes) staging_bytes = t.nbytes;
    }

    // ---- device ----
    int n_dev = 0;
    cudaError_t ce = cudaGetDeviceCount(&n_dev);
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, nullptr, ce == cudaSuccess && n_dev > 0,
               "No usable CUDA device (%s); this engine has no CPU execution path", ce == cudaSuccess ? "device count is 0" : cudaGetErrorString(ce));
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, device >= 0 && device < n_dev, "CUDA device %d out of range (0 .. %d)", device, n_dev - 1);
    ce = cudaSetDevice(device);
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, nullptr, ce == cudaSuccess, "cudaSetDevice(%d) failed: %s", device, cudaGetErrorString(ce));
    cudaDeviceProp prop;
    ce = cudaGetDeviceProperties(&prop, device);
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, nullptr, ce == cudaSuccess, "cudaGetDeviceProperties failed: %s", cudaGetErrorString(ce));
    // arch-specific sm_90a code (wgmma) loads on compute capability 9.0 and nothing else
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, nullptr, prop.major == 9 && prop.minor == 0,
               "Device %s is sm_%d%d; this library is built for sm_90a (H100) only", prop.name, prop.major, prop.minor);
    m.dev.device = device;
    m.dev.num_sms = prop.multiProcessorCount;
    m.dev.max_smem_optin = (int) prop.sharedMemPerBlockOptin;
    m.device_name = prop.name;

    ce = cudaMalloc(reinterpret_cast<void **>(&m.arena), arena_bytes);
    RWKV_CHECK(sink, RWKV_ERROR_MODEL | RWKV_ERROR_ALLOC, nullptr, ce == cudaSuccess, "Failed to allocate %zu bytes of device memory: %s", arena_bytes, cudaGetErrorString(ce));
    m.arena_bytes = arena_bytes;

    // ---- pass 2: stream payloads (rwkv_model_loading.inc:395-401) ----
    File file(fopen(path, "rb"));
    RWKV_CHECK(sink, RWKV_ERROR_FILE | RWKV_ERROR_FILE_OPEN, nullptr, file.f, "Failed to open file %s", path);
    std::unique_ptr<uint8_t[]> staging(new (std::nothrow) uint8_t[staging_bytes + 64]);
    RWKV_CHECK(sink, RWKV_ERROR_MODEL | RWKV_ERROR_ALLOC, nullptr, staging, "Failed to allocate %zu bytes of staging memory", staging_bytes);
    std::vector<float> widened;
    for (Request & r : reqs) {
        const TensorInfo & t = *r.info;
        RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_FILE_READ, nullptr,
                   fseeko(file.f, (off_t) t.file_offset, SEEK_SET) == 0 && fread(staging.get(), 1, t.nbytes, file.f) == t.nbytes,
                   "Failed to read data of parameter %s", r.name.c_str());
        uint8_t * dst = m.arena + r.arena_offset;
        if (r.mat) {
            DevMatrix & d = *r.mat;
            d.type = (int) t.data_type;
            d.K = (int) t.ne[0];
            d.M = (int) (t.ne[1] * t.ne[2]);
            d.pitch = matrix_pitch(d.type, t.ne[0]);
            d.data = dst;
            const size_t row_bytes = tensor_nbytes(d.type, t.ne[0], 1, 1);
            uint8_t * td = r.tiled_bytes ? m.arena + r.tiled_offset : nullptr;
            ce = upload_matrix(staging.get(), d.type, d.M, d.K, dst, td);
            if (td) {
                d.tiled = td;
                m.tiled_bytes += r.tiled_bytes;
            }
            const size_t bytes = t.nbytes;
            if (r.name == "emb.weight") m.weight_bytes_per_token += row_bytes;
            else if (r.name == "head.weight") { m.weight_bytes_per_token += bytes; m.head_bytes += bytes; m.gemv_bytes_per_token += bytes; m.head_matrix_bytes += bytes; }
            else { m.weight_bytes_per_token += bytes; m.gemv_bytes_per_token += bytes; }
        } else {
            DevVec & d = *r.vec;
            d.n = (size_t) (t.ne[0] * t.ne[1] * t.ne[2]);
            d.data = reinterpret_cast<const float *>(dst);
            const void * src = staging.get();
            if (t.data_type != DT_F32) {
                widened.resize(d.n);
                widen_to_f32((int) t.data_type, staging.get(), d.n, widened.data());
                src = widened.data();
            }
            ce = cudaMemcpy(dst, src, d.n * 4, cudaMemcpyHostToDevice);
            m.weight_bytes_per_token += t.nbytes;
            if (r.name == "ln_out.weight" || r.name == "ln_out.bias") m.head_bytes += t.nbytes;
        }
        RWKV_CHECK(sink, RWKV_ERROR_MODEL | RWKV_ERROR_ALLOC, nullptr, ce == cudaSuccess, "Failed to upload parameter %s: %s", r.name.c_str(), cudaGetErrorString(ce));
    }
    if (m.arch_major == 6) {
        for (int i = layer_begin; i < layer_end; i++) {
            const TensorInfo * w2 = mf.find("blocks." + std::to_string(i) + ".att.time_maa_w2");
            Layer & L = m.layers[i];
            L.maa_mix = (int) w2->ne[0];
            RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_SHAPE, nullptr,
                       w2->ne[1] == C && w2->ne[2] == 5 && L.att_maa_w1.M == 5 * L.maa_mix,
                       "Unexpected shape of blocks.%d.att.time_maa_w1/w2", i);
            RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_SHAPE, nullptr, L.att_decay_w1.M == L.att_decay_w2.K, "Mismatched decay LoRA rank in layer %d", i);
        }
    }
    for (int i = layer_begin; i < layer_end; i++) {
        Layer & L = m.layers[i];
        RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_SHAPE, nullptr, L.ffn_key.M == L.ffn_value.K, "Mismatched FFN width in layer %d", i);
        if (m.arch_major == 7) {
            RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_SHAPE, nullptr,
                       L.att_w1.M == L.att_w2.K && L.att_a1.M == L.att_a2.K && L.att_g1.M == L.att_g2.K && (i == 0 || L.att_v1.M == L.att_v2.K),
                       "Mismatched LoRA ranks in layer %d", i);
        }
    }
    ce = cudaDeviceSynchronize();
    RWKV_CHECK(sink, RWKV_ERROR_MODEL | RWKV_ERROR_ALLOC, nullptr, ce == cudaSuccess, "Device error after upload: %s", cudaGetErrorString(ce));
    return model.release();
}

}  // namespace rwkv
