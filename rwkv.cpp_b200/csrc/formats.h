// Tensor data types and quant-block geometry of the rwkv.cpp ggml file format.
// Type ids are the on-disk ids (reference rwkv_file_format.inc:5-24); block layouts are
// ggml's (ggml/src/ggml-common.h:161-221): 32 weights per block along the input dimension,
// 256 per super-block for the K-quants Q4_K / Q5_K (ggml-common.h:296-322).
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>

namespace rwkv {

enum DType : int32_t {
    DT_F32 = 0, DT_F16 = 1, DT_Q4_0 = 2, DT_Q4_1 = 3,
    DT_Q4_1_O = 4, DT_Q4_2 = 5, DT_Q4_3 = 6,       // removed formats: rejected at load (rwkv_file_format.inc:123-130)
    DT_Q5_0 = 7, DT_Q5_1 = 8, DT_Q8_0 = 9,
    DT_Q8_1 = 10, DT_Q2_K = 11, DT_Q3_K = 12, DT_Q4_K = 13, DT_Q5_K = 14, DT_Q6_K = 15, DT_Q8_K = 16,
    DT_COUNT = 17
};

inline bool dtype_supported(int t) {
    return t == DT_F32 || t == DT_F16 || t == DT_Q4_0 || t == DT_Q4_1 || t == DT_Q5_0 || t == DT_Q5_1 || t == DT_Q8_0;
}
// Q4_K / Q5_K: matrices only, streamed by their own GEMV (kernels/gemv_kquant.cu). dtype_supported() stays the set of types every
// legacy-block kernel handles.
inline bool dtype_kquant(int t) { return t == DT_Q4_K || t == DT_Q5_K; }
inline bool dtype_loadable(int t) { return dtype_supported(t) || dtype_kquant(t); }
inline bool dtype_quantized(int t) { return t >= DT_Q4_0 && t != DT_COUNT; }
constexpr int QK_K = 256;
inline int dtype_block_elems(int t) { return (t == DT_F32 || t == DT_F16) ? 1 : (dtype_kquant(t) ? QK_K : 32); }
inline int dtype_block_bytes(int t) {
    switch (t) {
        case DT_F32: return 4;  case DT_F16: return 2;
        case DT_Q4_0: return 18; case DT_Q4_1: return 20; case DT_Q5_0: return 22; case DT_Q5_1: return 24; case DT_Q8_0: return 34;
        case DT_Q4_K: return 144;   // d, dmin (fp16), scales[12] (6-bit scale and min of 8 sub-blocks), qs[128]
        case DT_Q5_K: return 176;   // d, dmin, scales[12], qh[32] (fifth bits), qs[128]
        default: return 0;
    }
}
#if defined(__CUDACC__)
#define RWKV_FORMATS_HD __host__ __device__
#else
#define RWKV_FORMATS_HD
#endif
// 6-bit scale and min of sub-block j (32 weights) of a Q4_K / Q5_K super-block, from its packed scales[12] (ggml's get_scale_min_k4).
// Shared by the host widening, the quantizer and the kernels.
RWKV_FORMATS_HD inline void kquant_scale_min(const uint8_t * q, int j, int & sc, int & m) {
    if (j < 4) { sc = q[j] & 63; m = q[j + 4] & 63; }
    else { sc = (q[j + 4] & 0xF) | ((q[j - 4] >> 6) << 4); m = (q[j + 4] >> 4) | ((q[j] >> 6) << 4); }
}
inline const char * dtype_name(int t) {
    static const char * names[DT_COUNT + 1] = {"FP32", "FP16", "Q4_0", "Q4_1", "Q4_1_O", "Q4_2", "Q4_3", "Q5_0", "Q5_1", "Q8_0",
                                                "Q8_1", "Q2_K", "Q3_K", "Q4_K", "Q5_K", "Q6_K", "Q8_K", "unknown"};
    return (t >= 0 && t < DT_COUNT) ? names[t] : names[DT_COUNT];
}
inline int dtype_from_name(const char * s) {
    for (int t = 0; t < DT_COUNT; t++) if (!strcmp(s, dtype_name(t))) return t;
    return DT_COUNT;
}
// Bytes of a tensor: type_size * ne0*ne1*ne2 / block (reference rwkv_utilities.inc:1-3).
inline size_t tensor_nbytes(int t, uint64_t ne0, uint64_t ne1, uint64_t ne2) {
    return (size_t) dtype_block_bytes(t) * ne0 * ne1 * ne2 / (size_t) dtype_block_elems(t);
}

// ---- IEEE fp16 <-> fp32 on the host (round-to-nearest-even, like F16C / GGML_FP32_TO_FP16) ----
inline float fp16_to_fp32(uint16_t h) {
    uint32_t sign = (uint32_t) (h & 0x8000u) << 16;
    uint32_t exp = (h >> 10) & 0x1Fu, man = h & 0x3FFu, bits;
    if (exp == 0) {
        if (man == 0) bits = sign;
        else {  // subnormal
            int e = -1;
            do { e++; man <<= 1; } while (!(man & 0x400u));
            bits = sign | (uint32_t) (127 - 15 - e) << 23 | (man & 0x3FFu) << 13;
        }
    } else if (exp == 31) bits = sign | 0x7F800000u | man << 13;
    else bits = sign | (exp + 112) << 23 | man << 13;
    float f; memcpy(&f, &bits, 4); return f;
}
inline uint16_t fp32_to_fp16(float f) {
    uint32_t x; memcpy(&x, &f, 4);
    uint32_t sign = (x >> 16) & 0x8000u;
    x &= 0x7FFFFFFFu;
    if (x >= 0x7F800000u) return (uint16_t) (sign | 0x7C00u | (x > 0x7F800000u ? 0x200u | ((x >> 13) & 0x3FFu) : 0));
    if (x >= 0x477FF000u) return (uint16_t) (sign | 0x7C00u);   // rounds to inf (>= 65520)
    if (x < 0x33000001u) return (uint16_t) sign;                 // rounds to zero (<= 2^-25)
    int32_t e = (int32_t) (x >> 23) - 127;
    uint32_t m = (x & 0x7FFFFFu) | 0x800000u;
    uint32_t shift = (e < -14) ? (uint32_t) (13 + (-14 - e)) : 13u;
    uint32_t half_m = m >> shift;
    uint32_t rem = m & ((1u << shift) - 1), halfway = 1u << (shift - 1);
    if (rem > halfway || (rem == halfway && (half_m & 1))) half_m++;
    uint32_t out = (e < -14) ? half_m : (((uint32_t) (e + 15) << 10) + (half_m - 0x400u));
    return (uint16_t) (sign | out);
}

}  // namespace rwkv
