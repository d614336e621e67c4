// Low-rank deltas of the layer matrices (rwkv_b200_adapter_*, include/rwkv_b200.h): y = epi(W.x + scale * B.(A.x)) for the adapted
// problems of one GEMV batch, as two launches around the batch's unchanged base route:
//   shrink  u[:, t] = A . x[:, t]                       ([rank, T] fp32 per problem, from the fp32 input x)
//   expand  y[:, t] = epi(z[:, t] + scale * B . u[:, t])
// A problem whose epilogue is nonlinear (none, sigmoid, silu, relu^2) runs its base with EPI_NONE into z. A residual epilogue (the add
// after att.output, the gated add after ffn.value) is linear in W.x, so its base keeps the epilogue and writes y in place; the expand
// then adds the delta as the same epilogue with y as the residual: y + scale * B.u, or y + gate * (scale * B.u). Either way the expand
// calls the streaming GEMV's epilogue functions (gemv_tma_device.cuh), and B = 0 leaves every output equal (==) to what the base
// route wrote.
// Each output column's arithmetic is a function of (K, M, rank) only: a row of A is summed by one CTA, each thread over fixed 8-element
// groups of K, then a butterfly per warp and the warps in order; a row of B by one thread in rank order. So it never depends on T or
// on the column's position in the pass.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "gemv.h"

namespace rwkv {

constexpr int LORA_MAX_RANK = 256;

// A delta on the device: A [rank][K] and B transposed, [rank][M], both fp16 (uint16_t bit patterns).
struct LoraDelta {
    const uint16_t * A = nullptr;
    const uint16_t * Bt = nullptr;
    int rank = 0;
    float scale = 0.f;
};

struct LoraProblem {
    LoraDelta d;
    int K, M;
    const float * x; long long ldx;    // the base problem's fp32 input
    float * u;                         // [T][rank]: column t at u + t * rank
    const float * z; long long ldz;    // base output without epilogue, or NULL: y already holds the residual epilogue's result
    GemvProblem P;                     // epi, y / ldy and the epilogue operands; a residual epilogue reads res = y
    int first_shrink, first_expand;    // filled by the launchers
};
struct LoraBatch {
    int n, T;
    LoraProblem p[GEMV_MAX_PROBLEMS];
};

// One launch each for every problem of the batch. Checked by the caller: 1 <= T <= 256, 1 <= rank <= LORA_MAX_RANK.
cudaError_t launch_lora_shrink(LoraBatch & b, cudaStream_t stream);
cudaError_t launch_lora_expand(LoraBatch & b, cudaStream_t stream);

}  // namespace rwkv
