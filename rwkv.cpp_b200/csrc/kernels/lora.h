// Low-rank deltas of the layer matrices (rwkv_b200_adapter_*, include/rwkv_b200.h): y = epi(W.x + scale * B.(A.x)) for the adapted
// problems of one GEMV batch, as two launches around the batch's unchanged base route:
//   shrink  u[:, t] = A . x[:, t]                       ([rank, T] fp32 per problem, from the fp32 input x)
//   expand  y[:, t] = epi(z[:, t] + scale * B . u[:, t])
// A problem whose epilogue is nonlinear (none, sigmoid, silu, relu^2) runs its base with EPI_NONE into z. A residual epilogue (the add
// after att.output, the gated add after ffn.value) is linear in W.x, so its base keeps the epilogue and writes y in place; the expand
// then adds the delta as the same epilogue with y as the residual: y + scale * B.u, or y + gate * (scale * B.u). Either way the expand
// calls the streaming GEMV's epilogue functions (gemv_tma_device.cuh), and B = 0 leaves every output equal (==) to what the base
// route wrote.
// The columns of a problem come in groups, each with its own delta and its own list of columns of the pass (an adapter per sequence of
// a batch context, rwkv_b200_batch_set_adapter); an adapter of the whole context is the one group of every column. A CTA works on the
// columns of one group only. A group of rank 0 holds the columns without a delta of a problem whose base was retargeted to z: the expand
// writes epi(z) for them, nothing added (z + 0 would turn a -0 into +0). Columns without a delta of a residual problem are in no group:
// the base has already written them.
// Each output column's arithmetic is a function of (K, M, rank) only: a row of A is summed by one CTA, each thread over fixed 8-element
// groups of K, then a butterfly per warp and the warps in order; a row of B by one thread in rank order. So it never depends on T, on
// the column's position in the pass or on the other columns of the launch.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "gemv.h"

namespace rwkv {

constexpr int LORA_MAX_RANK = 256;
// Groups of one launch, all problems together. The engine's GEMV batches hold at most 4 adapted problems, so a batch context with up
// to LORA_MAX_ADAPTERS distinct adapters on its sequences needs at most 4 * (LORA_MAX_ADAPTERS + 1) (the unadapted columns) groups.
constexpr int LORA_MAX_ADAPTERS = 31;
constexpr int LORA_MAX_GROUPS = 4 * (LORA_MAX_ADAPTERS + 1);
constexpr int LORA_MAX_T = 256;       // columns of a pass (MAX_TOKENS_PER_PASS)

// A delta on the device: A [rank][K] and B transposed, [rank][M], both fp16 (uint16_t bit patterns).
struct LoraDelta {
    const uint16_t * A = nullptr;
    const uint16_t * Bt = nullptr;
    int rank = 0;
    float scale = 0.f;
};

struct LoraGroup {
    LoraDelta d;                       // rank 0: columns without a delta (expand only)
    int problem;                       // index into LoraBatch::p
    int col0, n_cols;                  // its columns: LoraBatch::col[col0 .. col0 + n_cols), indices into the pass
    int first_shrink, first_expand;    // filled by the launchers
};
struct LoraProblem {
    int K, M;
    const float * x; long long ldx;    // the base problem's fp32 input
    float * u; int ldu;                // [T][ldu]: column t at u + t * ldu, ldu at least every group's rank
    const float * z; long long ldz;    // base output without epilogue, or NULL: y already holds the residual epilogue's result
    GemvProblem P;                     // epi, y / ldy and the epilogue operands; a residual epilogue reads res = y
};
struct LoraBatch {
    int n, T, n_groups;
    LoraProblem p[GEMV_MAX_PROBLEMS];
    LoraGroup g[LORA_MAX_GROUPS];      // in problem order
    uint8_t col[GEMV_MAX_PROBLEMS * LORA_MAX_T];
};

// One launch each for every group of the batch (none when there is none). Checked by the caller: 1 <= T <= LORA_MAX_T,
// 0 <= rank <= LORA_MAX_RANK, every group's columns below T.
cudaError_t launch_lora_shrink(LoraBatch & b, cudaStream_t stream);
cudaError_t launch_lora_expand(LoraBatch & b, cudaStream_t stream);

}  // namespace rwkv
