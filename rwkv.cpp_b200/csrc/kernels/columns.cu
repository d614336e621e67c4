// Column gather / scatter between [rows, n] fp32 blocks: the head of a ragged batch pass runs on the last column of every advancing
// sequence only, gathered into a compact block, and its output columns go back to those sequences' logits columns.
#include "ops.h"
#include "gemv.h"   // launch_pdl

namespace rwkv {
namespace {

constexpr int COPY_THREADS = 256;

// grid (row blocks, n): CTA (b, j) copies rows [b * COPY_THREADS * 4, ...) of column j, a float4 per thread where the columns allow it
__global__ void __launch_bounds__(COPY_THREADS) copy_columns_kernel(const float * src, const int * src_col, float * dst, const int * dst_col, int rows) {
    pdl_prologue();
    const int j = blockIdx.y;
    const float * s = src + (size_t) (src_col ? src_col[j] : j) * rows;
    float * d = dst + (size_t) (dst_col ? dst_col[j] : j) * rows;
    const int r0 = (blockIdx.x * COPY_THREADS + threadIdx.x) * 4;
    if ((rows & 3) == 0 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0) {
        if (r0 < rows) *reinterpret_cast<float4 *>(d + r0) = *reinterpret_cast<const float4 *>(s + r0);
    } else {
        for (int r = r0; r < r0 + 4 && r < rows; r++) d[r] = s[r];
    }
}

}  // namespace

cudaError_t launch_copy_columns(const float * src, const int * src_col, float * dst, const int * dst_col, int rows, int n, cudaStream_t s) {
    if (rows < 1 || n < 1) return cudaErrorInvalidValue;
    const dim3 grid((rows + COPY_THREADS * 4 - 1) / (COPY_THREADS * 4), n);
    return launch_pdl(copy_columns_kernel, grid, dim3(COPY_THREADS), 0, s, src, src_col, dst, dst_col, rows);
}

}  // namespace rwkv
