// LoRA adapters (rwkv_b200_adapter_create, include/rwkv_b200.h): argument checks, then the upload of the deltas and replacements into
// one device allocation, and the adapter's copies of the model's layers that point at them.
#include "engine.h"
#include "quantizer.h"

#include <cinttypes>
#include <cmath>
#include <cstring>
#include <memory>
#include <new>
#include <string>
#include <unordered_map>
#include <vector>

namespace rwkv {

namespace {

inline size_t align256(size_t v) { return (v + 255) / 256 * 256; }

bool all_finite(const float * v, size_t n) {
    for (size_t i = 0; i < n; i++) if (!std::isfinite(v[i])) return false;
    return true;
}
// Finite after rounding to fp16, the type A and B are kept in on the device.
bool all_finite_f16(const float * v, size_t n) {
    for (size_t i = 0; i < n; i++) if (!std::isfinite(v[i]) || std::fabs(v[i]) >= 65520.0f) return false;
    return true;
}

// The layer matrices that take a low-rank delta: att key / value / receptance / gate / output and ffn key / value / receptance of every
// architecture. The LoRA matrices inside a v6 / v7 layer, emb and head do not.
bool delta_target(const Layer & L, const DevMatrix * w) {
    return w == &L.att_key || w == &L.att_value || w == &L.att_receptance || w == &L.att_gate || w == &L.att_output ||
           w == &L.ffn_key || w == &L.ffn_value || w == &L.ffn_receptance;
}

}  // namespace

void encode_rows(int type, const float * values, size_t M, size_t K, uint8_t * out) {
    const size_t row_bytes = tensor_nbytes(type, K, 1, 1);
    for (size_t r = 0; r < M; r++) {
        const float * x = values + r * K;
        uint8_t * o = out + r * row_bytes;
        if (type == DT_F32) memcpy(o, x, K * sizeof(float));
        else if (type == DT_F16) for (size_t k = 0; k < K; k++) { const uint16_t h = fp32_to_fp16(x[k]); memcpy(o + 2 * k, &h, 2); }
        else quantize_row(type, x, o, K);
    }
}

namespace {

// A replacement matrix in the device form the loader gives the base: the base's type (encode_rows), the device layout, and the
// tile-major copy when the base has one.
cudaError_t upload_replacement(const DevMatrix & base, const float * values, uint8_t * dst, uint8_t * tiled) {
    std::vector<uint8_t> host(tensor_nbytes(base.type, (uint64_t) base.K, 1, 1) * (size_t) base.M);
    encode_rows(base.type, values, (size_t) base.M, (size_t) base.K, host.data());
    return upload_matrix(host.data(), base.type, base.M, base.K, dst, tiled);
}

}  // namespace

Adapter * create_adapter(Model * model, const AdapterTensor * t, size_t n, float scale, ErrorSink sink) {
    Model & m = *model;    // param_table hands out mutable slots; nothing of the model is written
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, n == 0 || t, "NULL tensor array with n = %zu", n);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, std::isfinite(scale), "The scale is not finite");

    // the adapter's copies, and the model's table and the adapter's side by side (same order)
    std::unique_ptr<Adapter> a(new (std::nothrow) Adapter());
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, nullptr, a, "Failed to allocate the adapter");
    a->model = model;
    a->layers = m.layers;
    a->ln0_w = m.ln0_w; a->ln0_b = m.ln0_b; a->ln_out_w = m.ln_out_w; a->ln_out_b = m.ln_out_b;
    DevMatrix emb_copy = m.emb, head_copy = m.head;
    const std::vector<ParamSlot> base = param_table(m, m.layers.data(), TopTensors{&m.emb, &m.head, &m.ln0_w, &m.ln0_b, &m.ln_out_w, &m.ln_out_b});
    const std::vector<ParamSlot> mine = param_table(m, a->layers.data(), TopTensors{&emb_copy, &head_copy, &a->ln0_w, &a->ln0_b, &a->ln_out_w, &a->ln_out_b});
    std::unordered_map<std::string, size_t> index;
    for (size_t i = 0; i < base.size(); i++) index[base[i].name] = i;

    // ---- checks: nothing is allocated before every entry passed ----
    std::vector<size_t> slot(n);
    std::vector<bool> used(base.size(), false);
    size_t bytes = 0, n_delta = 0;
    for (size_t e = 0; e < n; e++) {
        const AdapterTensor & x = t[e];
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, x.name, "Entry %zu has no name", e);
        const auto it = index.find(x.name);
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, it != index.end(), "Entry %zu: the model has no tensor %s", e, x.name);
        const size_t i = it->second;
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, !used[i], "Entry %zu: %s is listed twice", e, x.name);
        used[i] = true;
        slot[e] = i;
        const ParamSlot & s = base[i];
        RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, s.mat != &m.emb && s.mat != &m.head, "Entry %zu: %s cannot be adapted", e, x.name);
        if (x.rank > 0) {
            int layer = -1;
            for (int l = m.layer_begin; l < m.layer_end && layer < 0; l++) if (delta_target(m.layers[l], s.mat)) layer = l;
            RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, layer >= 0, "Entry %zu: %s takes no low-rank delta (only the att / ffn layer matrices do)", e, x.name);
            RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, x.rank <= (uint32_t) LORA_MAX_RANK, "Entry %zu: rank %" PRIu32 " is above %d", e, x.rank, LORA_MAX_RANK);
            RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, x.a && x.b, "Entry %zu: NULL A or B", e);
            const size_t K = (size_t) s.mat->K, M = (size_t) s.mat->M, R = x.rank;
            RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, all_finite_f16(x.a, R * K) && all_finite_f16(x.b, M * R),
                       "Entry %zu: A or B of %s has a value that is not finite in fp16", e, x.name);
            bytes += align256(R * K * 2) + align256(M * R * 2);
            n_delta++;
        } else {
            RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, x.values, "Entry %zu: NULL values", e);
            a->replaces = true;
            const size_t count = s.mat ? (size_t) s.mat->K * (size_t) s.mat->M : s.vec->n;
            // a matrix stored in fp16, or quantized with fp16 block scales, must be finite in fp16 (|v| < 65520)
            const bool f16_values = s.mat && s.mat->type != DT_F32;
            RWKV_CHECK(sink, RWKV_ERROR_ARGS, nullptr, f16_values ? all_finite_f16(x.values, count) : all_finite(x.values, count),
                       "Entry %zu: a value of %s is not finite%s", e, x.name, f16_values ? " in fp16" : "");
            if (s.mat) {
                bytes += align256((size_t) s.mat->M * (size_t) matrix_pitch(s.mat->type, (uint64_t) s.mat->K) + 256);
                if (s.mat->tiled) bytes += align256(gemm_tc_tiled_bytes(s.mat->type, s.mat->M, s.mat->K));
            } else {
                bytes += align256(count * sizeof(float));
            }
        }
    }

    // ---- upload ----
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_UNSUPPORTED, nullptr, cudaSetDevice(m.dev.device) == cudaSuccess, "cudaSetDevice failed");
    if (bytes) {
        const cudaError_t e = a->arena.alloc(bytes);
        RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, nullptr, e == cudaSuccess, "Failed to allocate %zu bytes for the adapter: %s", bytes, cudaGetErrorString(e));
    }
    a->deltas.reserve(n_delta);                 // DevMatrix::lora points into it
    size_t off = 0;
    std::vector<uint16_t> h;
    cudaError_t ce = cudaSuccess;
    for (size_t e = 0; e < n && ce == cudaSuccess; e++) {
        const AdapterTensor & x = t[e];
        const ParamSlot & s = base[slot[e]], & d = mine[slot[e]];
        if (x.rank > 0) {
            const size_t K = (size_t) s.mat->K, M = (size_t) s.mat->M, R = x.rank;
            LoraDelta delta;
            delta.rank = (int) R; delta.scale = scale;
            h.resize(R * K);
            for (size_t i = 0; i < R * K; i++) h[i] = fp32_to_fp16(x.a[i]);
            uint16_t * A = reinterpret_cast<uint16_t *>(a->arena + off);
            ce = cudaMemcpy(A, h.data(), R * K * 2, cudaMemcpyHostToDevice);
            off += align256(R * K * 2);
            h.resize(M * R);
            for (size_t r = 0; r < R; r++) for (size_t i = 0; i < M; i++) h[r * M + i] = fp32_to_fp16(x.b[i * R + r]);     // B^T
            uint16_t * Bt = reinterpret_cast<uint16_t *>(a->arena + off);
            if (ce == cudaSuccess) ce = cudaMemcpy(Bt, h.data(), M * R * 2, cudaMemcpyHostToDevice);
            off += align256(M * R * 2);
            delta.A = A; delta.Bt = Bt;
            a->deltas.push_back(delta);
            d.mat->lora = &a->deltas.back();
        } else if (s.mat) {
            uint8_t * dst = a->arena + off;
            off += align256((size_t) s.mat->M * (size_t) matrix_pitch(s.mat->type, (uint64_t) s.mat->K) + 256);
            uint8_t * tiled = nullptr;
            if (s.mat->tiled) { tiled = a->arena + off; off += align256(gemm_tc_tiled_bytes(s.mat->type, s.mat->M, s.mat->K)); }
            ce = upload_replacement(*s.mat, x.values, dst, tiled);
            d.mat->data = dst; d.mat->tiled = tiled;
        } else {
            float * dst = reinterpret_cast<float *>(a->arena + off);
            ce = cudaMemcpy(dst, x.values, s.vec->n * sizeof(float), cudaMemcpyHostToDevice);
            off += align256(s.vec->n * sizeof(float));
            d.vec->data = dst;
        }
    }
    if (ce == cudaSuccess) ce = cudaDeviceSynchronize();
    RWKV_CHECK(sink, RWKV_ERROR_CTX | RWKV_ERROR_ALLOC, nullptr, ce == cudaSuccess, "Failed to upload the adapter: %s", cudaGetErrorString(ce));
    m.refcount.fetch_add(1);      // the adapter's tables point into the model's arena: it keeps the model alive
    return a.release();
}

bool destroy_adapter(Adapter * a, ErrorSink sink) {
    if (!a) return true;
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, a->attached.load() == 0, "The adapter is attached to %d context(s); detach it first", a->attached.load());
    Model * model = a->model;
    cudaSetDevice(model->dev.device);
    delete a;
    if (model->refcount.fetch_sub(1) == 1) delete model;      // the last holder of the model
    return true;
}

}  // namespace rwkv
