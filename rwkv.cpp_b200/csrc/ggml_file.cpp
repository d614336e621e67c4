#define _FILE_OFFSET_BITS 64
#include "ggml_file.h"
#include <cinttypes>
#include <sys/stat.h>

namespace rwkv {

thread_local int g_last_error = RWKV_ERROR_NONE;
thread_local bool g_print_errors = true;

static_assert(sizeof(off_t) >= 8, "file offsets must be 64-bit: model files exceed 2 GB");

bool read_file_header(FILE * f, FileHeader & h, ErrorSink sink) {
    RWKV_CHECK(sink, RWKV_ERROR_FILE_READ, false, fread(&h, sizeof(FileHeader), 1, f) == 1, "Failed to read the file header");
    RWKV_CHECK(sink, RWKV_ERROR_FILE_MAGIC, false, h.magic == RWKV_FILE_MAGIC, "Wrong file magic 0x%08" PRIx32, h.magic);
    RWKV_CHECK(sink, RWKV_ERROR_FILE_VERSION, false, h.version >= RWKV_FILE_VERSION_MIN && h.version <= RWKV_FILE_VERSION_MAX,
               "Unsupported file version %" PRIu32, h.version);
    RWKV_CHECK(sink, RWKV_ERROR_DATA_TYPE, false, h.data_type < DT_COUNT, "Model data type out of range (%" PRIu32 " > %d)", h.data_type, DT_COUNT - 1);
    RWKV_CHECK(sink, RWKV_ERROR_DATA_TYPE, false, h.data_type != DT_Q4_1_O && h.data_type != DT_Q4_2 && h.data_type != DT_Q4_3,
               "Models in %s format cannot be loaded anymore because the format was removed.\n"
               "You need to quantize the model into another format.", dtype_name((int) h.data_type));
    RWKV_CHECK(sink, RWKV_ERROR_DATA_TYPE, false, !dtype_quantized((int) h.data_type) || h.version == RWKV_FILE_VERSION_1,
               "The quantized model file in %s format was created with an old version of rwkv.cpp and can not be loaded anymore.\n"
               "You need to requantize the model.", dtype_name((int) h.data_type));
    return true;
}

bool read_tensor_info(FILE * f, TensorInfo & t, ErrorSink sink) {
    uint32_t head[3];
    RWKV_CHECK(sink, RWKV_ERROR_FILE_READ, false, fread(head, sizeof(uint32_t), 3, f) == 3, "Failed to read a tensor header");
    t.dim_count = head[0];
    const uint32_t key_length = head[1];
    t.data_type = head[2];
    RWKV_CHECK(sink, RWKV_ERROR_SHAPE, false, t.dim_count >= 1 && t.dim_count <= 3, "Tensor has an invalid shape (%" PRIu32 " dimensions)", t.dim_count);
    RWKV_CHECK(sink, RWKV_ERROR_DATA_TYPE, false, t.data_type < DT_COUNT, "Tensor data type out of range (%" PRIu32 " > %d)", t.data_type, DT_COUNT - 1);
    RWKV_CHECK(sink, RWKV_ERROR_DATA_TYPE, false, t.data_type != DT_Q4_1_O && t.data_type != DT_Q4_2 && t.data_type != DT_Q4_3,
               "Tensor data type (%s) is no longer supported", dtype_name((int) t.data_type));
    uint32_t ne[3] = {1, 1, 1};
    RWKV_CHECK(sink, RWKV_ERROR_FILE_READ, false, fread(ne, sizeof(uint32_t), t.dim_count, f) == t.dim_count, "Failed to read tensor dimensions");
    for (int i = 0; i < 3; i++) t.ne[i] = ne[i];
    RWKV_CHECK(sink, RWKV_ERROR_FILE_READ, false, key_length < (1u << 20), "Implausible tensor name length %" PRIu32, key_length);
    t.name.resize(key_length);
    RWKV_CHECK(sink, RWKV_ERROR_FILE_READ, false, key_length == 0 || fread(&t.name[0], key_length, 1, f) == 1, "Failed to read tensor name");
    // The reference accepts every K-quant / Q8_1 id in its table (rwkv_file_format.inc:28-47); its Python binding offers Q4_K and
    // Q5_K next to the five legacy formats, and this engine has kernels for exactly those plus FP16 / FP32.
    RWKV_CHECK(sink, RWKV_ERROR_UNSUPPORTED, false, dtype_loadable((int) t.data_type), "Unsupported data type %s in parameter %s",
               dtype_name((int) t.data_type), t.name.c_str());
    if (dtype_kquant((int) t.data_type)) {
        // ggml's K-quant rows are whole 256-weight super-blocks; a shorter row has no defined meaning
        RWKV_CHECK(sink, RWKV_ERROR_UNSUPPORTED, false, t.ne[0] % QK_K == 0,
                   "Row length %" PRIu64 " of %s is not a multiple of %d, which %s needs; requantize the model with this library's quantizer",
                   t.ne[0], t.name.c_str(), QK_K, dtype_name((int) t.data_type));
        RWKV_CHECK(sink, RWKV_ERROR_UNSUPPORTED, false, t.name != "emb.weight" && t.name != "head.weight",
                   "%s in %s is not supported (the quantizer keeps it in FP16); requantize the model", t.name.c_str(), dtype_name((int) t.data_type));
    }
    RWKV_CHECK(sink, RWKV_ERROR_SHAPE, false, t.ne[0] % dtype_block_elems((int) t.data_type) == 0,
               "Row length %" PRIu64 " of %s is not a multiple of the %s block size", t.ne[0], t.name.c_str(), dtype_name((int) t.data_type));
    t.nbytes = tensor_nbytes((int) t.data_type, t.ne[0], t.ne[1], t.ne[2]);
    t.file_offset = (uint64_t) ftello(f);
    return true;
}

bool scan_model_file(const char * path, ModelFile & out, ErrorSink sink) {
    File file(fopen(path, "rb"));
    RWKV_CHECK(sink, RWKV_ERROR_FILE | RWKV_ERROR_FILE_OPEN, false, file.f, "Failed to open file %s", path);
    struct stat st;
    RWKV_CHECK(sink, RWKV_ERROR_FILE | RWKV_ERROR_FILE_STAT, false, fstat(fileno(file.f), &st) == 0, "Failed to stat file %s", path);
    out.file_size = (uint64_t) st.st_size;
    {   // header failures carry the FILE category in the reference (rwkv_model_loading.inc:298)
        ErrorSink s = sink;
        bool ok = read_file_header(file.f, out.header, s);
        RWKV_CHECK(sink, RWKV_ERROR_FILE, false, ok, "Invalid file header");
    }
    while ((uint64_t) ftello(file.f) < out.file_size) {
        TensorInfo t;
        bool ok = read_tensor_info(file.f, t, sink);
        RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS, false, ok, "Failed to read a model parameter");
        RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_FILE_READ, false, t.file_offset + t.nbytes <= out.file_size,
                   "Parameter %s runs past the end of the file", t.name.c_str());
        RWKV_CHECK(sink, RWKV_ERROR_MODEL_PARAMS | RWKV_ERROR_FILE_READ, false, fseeko(file.f, (off_t) t.nbytes, SEEK_CUR) == 0,
                   "Failed to seek to next tensor after parameter %s", t.name.c_str());
        out.index[t.name] = out.tensors.size();
        out.tensors.push_back(std::move(t));
    }
    return true;
}

}  // namespace rwkv
