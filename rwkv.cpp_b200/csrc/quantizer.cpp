#define _FILE_OFFSET_BITS 64
#include "quantizer.h"

#include <cfloat>
#include <cinttypes>
#include <cmath>
#include <cstring>
#include <memory>
#include <string>
#include <sys/stat.h>
#include <vector>

#include "formats.h"
#include "ggml_file.h"

// The encoders below must round exactly like the reference's scalar code: one rounding per
// operation, no fused multiply-add.
#if defined(__GNUC__)
#pragma GCC optimize("fp-contract=off")
#endif

namespace rwkv {

namespace {

inline void put_half(uint8_t * p, float v) { uint16_t h = fp32_to_fp16(v); memcpy(p, &h, 2); }
inline int min_int(int a, int b) { return a < b ? a : b; }

// quantize_row_q4_0_ref / quantize_row_q5_0_ref (ggml-quants.c:31-66, 107-150): symmetric, the element
// of largest magnitude maps to -8 / -16.
void encode_sym(const float * x, uint8_t * out, int levels /* 8 or 16 */) {
    float amax = 0.0f, max = 0.0f;
    for (int j = 0; j < 32; j++) {
        const float v = x[j];
        if (amax < fabsf(v)) { amax = fabsf(v); max = v; }
    }
    const float d = max / (float) -levels;
    const float id = d ? 1.0f / d : 0.0f;
    put_half(out, d);
    uint8_t * qs = out + (levels == 8 ? 2 : 6);
    uint32_t qh = 0;
    for (int j = 0; j < 16; j++) {
        const float x0 = x[j] * id, x1 = x[16 + j] * id;
        const uint8_t xi0 = (uint8_t) min_int(2 * levels - 1, (int8_t) (x0 + ((float) levels + 0.5f)));
        const uint8_t xi1 = (uint8_t) min_int(2 * levels - 1, (int8_t) (x1 + ((float) levels + 0.5f)));
        qs[j] = (uint8_t) ((xi0 & 0x0F) | ((xi1 & 0x0F) << 4));
        qh |= ((xi0 & 0x10u) >> 4) << (j + 0);
        qh |= ((xi1 & 0x10u) >> 4) << (j + 16);
    }
    if (levels == 16) memcpy(out + 2, &qh, 4);
}

// quantize_row_q4_1_ref / quantize_row_q5_1_ref (ggml-quants.c:68-105, 152-192): min/max affine.
void encode_affine(const float * x, uint8_t * out, int nlev /* 15 or 31 */) {
    float min = FLT_MAX, max = -FLT_MAX;
    for (int j = 0; j < 32; j++) {
        const float v = x[j];
        if (v < min) min = v;
        if (v > max) max = v;
    }
    const float d = (max - min) / (float) nlev;
    const float id = d ? 1.0f / d : 0.0f;
    put_half(out, d);
    put_half(out + 2, min);
    uint8_t * qs = out + (nlev == 15 ? 4 : 8);
    uint32_t qh = 0;
    for (int j = 0; j < 16; j++) {
        const float x0 = (x[j] - min) * id, x1 = (x[16 + j] - min) * id;
        uint8_t xi0, xi1;
        if (nlev == 15) {
            xi0 = (uint8_t) min_int(15, (int8_t) (x0 + 0.5f));
            xi1 = (uint8_t) min_int(15, (int8_t) (x1 + 0.5f));
        } else {
            xi0 = (uint8_t) (x0 + 0.5f);
            xi1 = (uint8_t) (x1 + 0.5f);
        }
        qs[j] = (uint8_t) ((xi0 & 0x0F) | ((xi1 & 0x0F) << 4));
        qh |= ((xi0 & 0x10u) >> 4) << (j + 0);
        qh |= ((xi1 & 0x10u) >> 4) << (j + 16);
    }
    if (nlev == 31) memcpy(out + 4, &qh, 4);
}

// quantize_row_q8_0_ref (ggml-quants.c:194-217)
void encode_q8_0(const float * x, uint8_t * out) {
    float amax = 0.0f;
    for (int j = 0; j < 32; j++) { const float v = fabsf(x[j]); if (v > amax) amax = v; }
    const float d = amax / 127.0f;
    const float id = d ? 1.0f / d : 0.0f;
    put_half(out, d);
    for (int j = 0; j < 32; j++) out[2 + j] = (uint8_t) (int8_t) roundf(x[j] * id);
}

// ---- K-quants: quantize_row_q4_K_ref / quantize_row_q5_K_ref (ggml-quants.c:1208-1278, 1395-1480) ----

// round to nearest, ties to even, through the float adder (ggml's nearest_int): valid for |v| < 2^22
inline int nearest_int(float v) {
    const float t = v + 12582912.f;
    int i; memcpy(&i, &t, 4);
    return (i & 0x007fffff) - 0x00400000;
}

// make_qkx2_quants (ggml-quants.c:550-629) with use_mad = false: levels L[0..n) in [0, nmax] and the scale of an affine fit
// x ~ scale*L - the_min, refined over nstep+1 trial scales by weighted least squares.
float fit_affine_levels(int n, int nmax, const float * x, const float * w, uint8_t * L, float * the_min, uint8_t * Laux,
                        float rmin, float rdelta, int nstep) {
    float min = x[0], max = x[0], sum_w = w[0], sum_x = sum_w * x[0];
    for (int i = 1; i < n; i++) {
        if (x[i] < min) min = x[i];
        if (x[i] > max) max = x[i];
        sum_w += w[i];
        sum_x += w[i] * x[i];
    }
    if (min > 0) min = 0;
    if (max == min) {
        for (int i = 0; i < n; i++) L[i] = 0;
        *the_min = -min;
        return 0.f;
    }
    float iscale = nmax / (max - min), scale = 1 / iscale, best = 0;
    for (int i = 0; i < n; i++) {
        const int l = nearest_int(iscale * (x[i] - min));
        L[i] = (uint8_t) (l < 0 ? 0 : (l > nmax ? nmax : l));
        const float diff = scale * L[i] + min - x[i];
        best += w[i] * (diff * diff);
    }
    for (int is = 0; is <= nstep; is++) {
        iscale = (rmin + rdelta * is + nmax) / (max - min);
        float sum_l = 0, sum_l2 = 0, sum_xl = 0;
        for (int i = 0; i < n; i++) {
            int l = nearest_int(iscale * (x[i] - min));
            l = l < 0 ? 0 : (l > nmax ? nmax : l);
            Laux[i] = (uint8_t) l;
            sum_l += w[i] * l;
            sum_l2 += w[i] * l * l;
            sum_xl += w[i] * l * x[i];
        }
        const float D = sum_w * sum_l2 - sum_l * sum_l;
        if (D > 0) {
            float this_scale = (sum_w * sum_xl - sum_x * sum_l) / D;
            float this_min = (sum_l2 * sum_x - sum_l * sum_xl) / D;
            if (this_min > 0) {
                this_min = 0;
                this_scale = sum_xl / sum_l2;
            }
            float mad = 0;
            for (int i = 0; i < n; i++) {
                const float diff = this_scale * Laux[i] + this_min - x[i];
                mad += w[i] * (diff * diff);
            }
            if (mad < best) {
                memcpy(L, Laux, (size_t) n);
                best = mad;
                scale = this_scale;
                min = this_min;
            }
        }
    }
    *the_min = -min;
    return scale;
}

// One 256-weight super-block. Q4_K: nmax 15, 21 trial scales from -1.0; Q5_K: nmax 31, 16 trial scales from -0.5.
void encode_kquant(const float * x, uint8_t * out, bool five) {
    const int nmax = five ? 31 : 15;
    uint8_t L[QK_K], Laux[32];
    float w[32], mins[8], scales[8], max_scale = 0, max_min = 0;
    for (int j = 0; j < 8; j++) {
        const float * xj = x + 32 * j;
        float sum_x2 = 0;
        for (int l = 0; l < 32; l++) sum_x2 += xj[l] * xj[l];
        const float av_x = sqrtf(sum_x2 / 32);
        for (int l = 0; l < 32; l++) w[l] = av_x + fabsf(xj[l]);
        scales[j] = fit_affine_levels(32, nmax, xj, w, L + 32 * j, &mins[j], Laux, five ? -0.5f : -1.f, 0.1f, five ? 15 : 20);
        if (scales[j] > max_scale) max_scale = scales[j];
        if (mins[j] > max_min) max_min = mins[j];
    }
    // 6-bit scales and mins, packed as get_scale_min_k4 unpacks them
    uint8_t * sc = out + 4;
    const float inv_scale = max_scale > 0 ? 63.f / max_scale : 0.f, inv_min = max_min > 0 ? 63.f / max_min : 0.f;
    for (int j = 0; j < 8; j++) {
        uint8_t ls = (uint8_t) nearest_int(inv_scale * scales[j]), lm = (uint8_t) nearest_int(inv_min * mins[j]);
        ls = ls < 63 ? ls : 63;
        lm = lm < 63 ? lm : 63;
        if (j < 4) {
            sc[j] = ls;
            sc[j + 4] = lm;
        } else {
            sc[j + 4] = (uint8_t) ((ls & 0xF) | ((lm & 0xF) << 4));
            sc[j - 4] |= (uint8_t) ((ls >> 4) << 6);
            sc[j] |= (uint8_t) ((lm >> 4) << 6);
        }
    }
    put_half(out, max_scale / 63.f);
    put_half(out + 2, max_min / 63.f);
    // levels again against the rounded scales
    uint16_t dh, mh; memcpy(&dh, out, 2); memcpy(&mh, out + 2, 2);
    for (int j = 0; j < 8; j++) {
        int s, m;
        kquant_scale_min(sc, j, s, m);
        const float d = fp16_to_fp32(dh) * s;
        if (!d) continue;
        const float dm = fp16_to_fp32(mh) * m;
        for (int i = 0; i < 32; i++) {
            const int l = nearest_int((x[32 * j + i] + dm) / d);
            L[32 * j + i] = (uint8_t) (l < 0 ? 0 : (l > nmax ? nmax : l));
        }
    }
    // sub-blocks 2k and 2k+1 share qs[32k .. 32k+32) as low and high nibbles; Q5_K keeps bit 4 of sub-block j in bit j of qh[l]
    uint8_t * qh = out + 16, * qs = out + (five ? 48 : 16);
    if (five) memset(qh, 0, 32);
    for (int k = 0; k < 4; k++) {
        for (int l = 0; l < 32; l++) {
            int lo = L[64 * k + l], hi = L[64 * k + 32 + l];
            if (five) {
                if (lo > 15) { lo -= 16; qh[l] |= (uint8_t) (1u << (2 * k)); }
                if (hi > 15) { hi -= 16; qh[l] |= (uint8_t) (2u << (2 * k)); }
            }
            qs[32 * k + l] = (uint8_t) (lo | (hi << 4));
        }
    }
}

// Tensors the reference never quantizes (rwkv_quantize.inc:1-13).
bool tensor_needs_quant(const std::string & name) {
    static const char * skip[] = {"att.v1", "att.v2", "att.g1", "att.g2", "att.a1", "att.a2", "att.w1", "att.w2", "att.r_k"};
    if (name == "emb.weight" || name == "head.weight") return false;
    for (const char * s : skip) if (name.find(s) != std::string::npos) return false;
    return true;
}

}  // namespace

size_t quantize_row(int type, const float * x, void * dst, size_t n) {
    uint8_t * out = static_cast<uint8_t *>(dst);
    const int bb = dtype_block_bytes(type);
    if (dtype_kquant(type)) {
        for (size_t b = 0; b < n / QK_K; b++) encode_kquant(x + b * QK_K, out + b * bb, type == DT_Q5_K);
        return n / QK_K * (size_t) bb;
    }
    for (size_t b = 0; b < n / 32; b++) {
        const float * xb = x + b * 32;
        uint8_t * ob = out + b * bb;
        switch (type) {
            case DT_Q4_0: encode_sym(xb, ob, 8); break;
            case DT_Q5_0: encode_sym(xb, ob, 16); break;
            case DT_Q4_1: encode_affine(xb, ob, 15); break;
            case DT_Q5_1: encode_affine(xb, ob, 31); break;
            default: encode_q8_0(xb, ob); break;
        }
    }
    return n / 32 * (size_t) bb;
}

#define MSG(...) do { if (*sink.print) fprintf(stderr, __VA_ARGS__); } while (0)

bool quantize_model_file(const char * in_path, const char * out_path, const char * format_name, ErrorSink sink) {
    RWKV_CHECK(sink, RWKV_ERROR_ARGS, false, in_path && out_path && format_name, "NULL argument");
    const int out_type = dtype_from_name(format_name);
    RWKV_CHECK(sink, RWKV_ERROR_ARGS | RWKV_ERROR_DATA_TYPE, false,
               out_type == DT_Q4_0 || out_type == DT_Q4_1 || out_type == DT_Q5_0 || out_type == DT_Q5_1 || out_type == DT_Q8_0 ||
               dtype_kquant(out_type),
               "Unsupported output data type (%s)", format_name);
    MSG("Loading model from '%s'\n", in_path);

    File in(fopen(in_path, "rb"));
    RWKV_CHECK(sink, RWKV_ERROR_FILE | RWKV_ERROR_FILE_OPEN, false, in.f, "Failed to open %s for reading", in_path);
    struct stat st;
    RWKV_CHECK(sink, RWKV_ERROR_FILE | RWKV_ERROR_FILE_STAT, false, fstat(fileno(in.f), &st) == 0, "failed to stat file %s", in_path);
    File out(fopen(out_path, "wb"));
    RWKV_CHECK(sink, RWKV_ERROR_FILE | RWKV_ERROR_FILE_OPEN, false, out.f, "Failed to open %s for writing", out_path);

    FileHeader header;
    {
        bool ok = read_file_header(in.f, header, sink);
        RWKV_CHECK(sink, RWKV_ERROR_FILE, false, ok, "Invalid file header");
    }
    RWKV_CHECK(sink, RWKV_ERROR_FILE, false, header.data_type == DT_F32 || header.data_type == DT_F16,
               "Unsupported input data type (%s); needs to be FP32 or FP16", dtype_name((int) header.data_type));
    FileHeader out_header = header;
    out_header.version = RWKV_FILE_VERSION;
    out_header.data_type = (uint32_t) out_type;
    RWKV_CHECK(sink, RWKV_ERROR_FILE | RWKV_ERROR_FILE_WRITE, false, fwrite(&out_header, sizeof(out_header), 1, out.f) == 1, "Failed to write file header");

    size_t orig_total = 0, new_total = 0;
    std::vector<uint8_t> raw, packed;
    std::vector<float> f32;
    while ((uint64_t) ftello(in.f) < (uint64_t) st.st_size) {
        TensorInfo t;
        {
            bool ok = read_tensor_info(in.f, t, sink);
            RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS, false, ok, "Failed to read tensor header");
        }
        MSG("%48s - [%5" PRIu64 ", %5" PRIu64 ", %5" PRIu64 "], type = %6s ", t.name.c_str(), t.ne[0], t.ne[1], t.ne[2], dtype_name((int) t.data_type));
        raw.resize(t.nbytes);
        RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_FILE_READ, false, t.nbytes == 0 || fread(raw.data(), t.nbytes, 1, in.f) == 1,
                   "\nFailed to read tensor data of %s", t.name.c_str());
        const uint8_t * payload = raw.data();
        size_t payload_bytes = t.nbytes;
        uint32_t out_dtype = t.data_type;
        // 2-D FP32/FP16 tensors except embedding/head and the v7 LoRA / r_k tensors (rwkv_quantize.inc:133-140)
        if ((t.data_type == DT_F32 || t.data_type == DT_F16) && t.dim_count == 2 && tensor_needs_quant(t.name)) {
            const size_t n = (size_t) (t.ne[0] * t.ne[1] * t.ne[2]);
            RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_SHAPE, false, t.ne[0] % 32 == 0, "\nRow length of %s is not a multiple of 32", t.name.c_str());
            const float * src;
            if (t.data_type == DT_F16) {
                f32.resize(n);
                const uint16_t * h = reinterpret_cast<const uint16_t *>(raw.data());
                for (size_t i = 0; i < n; i++) f32[i] = fp16_to_fp32(h[i]);
                src = f32.data();
            } else {
                src = reinterpret_cast<const float *>(raw.data());
            }
            // The reference quantises a K-quant tensor as one flat array, so when rows are not whole super-blocks its blocks straddle
            // rows and no engine can evaluate the result. Such tensors (v6 decay LoRA, n_embed or ffn widths that are not multiples of
            // 256) go to the legacy format of the same or more bytes per weight instead, as llama.cpp's quantizer does.
            int type = out_type;
            if (dtype_kquant(type) && t.ne[0] % QK_K != 0) type = (type == DT_Q4_K) ? DT_Q5_0 : DT_Q5_1;
            packed.resize(tensor_nbytes(type, t.ne[0], t.ne[1], t.ne[2]));
            payload_bytes = quantize_row(type, src, packed.data(), n);
            payload = packed.data();
            out_dtype = (uint32_t) type;
            MSG("-> %6s size = %8.2f MB -> %8.2f MB\n", dtype_name(type), t.nbytes / 1024.0 / 1024.0, payload_bytes / 1024.0 / 1024.0);
        } else {
            MSG("size = %8.3f MB\n", t.nbytes / 1024.0 / 1024.0);
        }
        // tensor record (rwkv_fwrite_tensor, rwkv_file_format.inc:199-236)
        uint32_t head[6] = {t.dim_count, (uint32_t) t.name.size(), out_dtype, (uint32_t) t.ne[0], (uint32_t) t.ne[1], (uint32_t) t.ne[2]};
        bool ok = fwrite(head, sizeof(uint32_t), 3 + t.dim_count, out.f) == 3 + t.dim_count
               && (t.name.empty() || fwrite(t.name.data(), t.name.size(), 1, out.f) == 1)
               && (payload_bytes == 0 || fwrite(payload, payload_bytes, 1, out.f) == 1);
        RWKV_CHECK(sink, RWKV_ERROR_FILE_WRITE, false, ok, "Failed to write tensor %s", t.name.c_str());
        orig_total += t.nbytes;
        new_total += payload_bytes;
    }
    MSG("original size     = %8.2f MB\n", orig_total / 1024.0 / 1024.0);
    MSG("quantized size    = %8.2f MB\n", new_total / 1024.0 / 1024.0);
    MSG("compression ratio = %8.2f\n", orig_total / (double) new_total);
    return true;
}

}  // namespace rwkv
