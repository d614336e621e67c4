// WKV time-mixing recurrences for RWKV v4 / v5 / v6 / v7, each fused with the normalisation and
// gating that follows it in the reference graph. The recurrent state stays in registers for the
// whole chunk; one CTA per head (v5+), one thread per state column (v5/v6) or row (v7).
#include "ops.h"
#include "gemv.h"   // launch_pdl
#include "act_stage.cuh"
#include "gemv_tma_device.cuh"   // row_partial / rows_dot, stage_column: the decay LoRA folded into wkv6_kernel
#include "../formats.h"

#include <cuda_fp16.h>

namespace rwkv {
namespace {

// ---------------------------------------------------------------------------------------------
// v4: rwkv_att_wkv_v4 (rwkv_graph.inc:119-161). One thread per channel, sequential over tokens.
// Every ggml node is its own rounding, so no FMA contraction here.
// MODE SEQ_BATCH: one token, column blockIdx.y, on the state of sequence blockIdx.y.
// MODE SEQ_RAGGED: the columns [seq_off[y], seq_off[y + 1]) of sequence y = blockIdx.y on its state.
// MODE | SEQ_SNAP: aa, bb, pp after every column with a checkpoint slot also go to the slot (aa at cp.at, bb and pp C and 2 C after it).
// ---------------------------------------------------------------------------------------------
template <int MODE>
__global__ void wkv4_kernel(const Wkv4Params p) {
    constexpr int M = MODE & ~SEQ_SNAP;
    constexpr bool BATCH = M == SEQ_BATCH;
    trace_begin(p.trace);
    pdl_prologue();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= p.C) return;
    const long long so = M != SEQ_ONE ? blockIdx.y * p.seq_stride : 0;
    int t_begin = BATCH ? blockIdx.y : 0, t_end = BATCH ? blockIdx.y + 1 : p.T;
    if constexpr (M == SEQ_RAGGED) {
        t_begin = p.seq_off[blockIdx.y]; t_end = p.seq_off[blockIdx.y + 1];
        if (t_begin == t_end) return;
    }
    float aa = p.aa_in[so + c], bb = p.bb_in[so + c], pp = p.pp_in[so + c];
    const float tf = p.time_first[c], td = p.time_decay[c];
    for (int t = t_begin; t < t_end; t++) {
        const size_t o = (size_t) t * p.C + c;
        const float k = p.k[o], v = p.v[o];
        float ww = __fadd_rn(tf, k);
        float qq = fmaxf(pp, ww);
        float e1 = expf(__fsub_rn(pp, qq)), e2 = expf(__fsub_rn(ww, qq));
        const float a = __fadd_rn(__fmul_rn(e1, aa), __fmul_rn(e2, v));
        const float b = __fadd_rn(__fmul_rn(e1, bb), e2);
        ww = __fadd_rn(pp, td);
        qq = fmaxf(ww, k);
        e1 = expf(__fsub_rn(ww, qq));
        e2 = expf(__fsub_rn(k, qq));
        aa = __fadd_rn(__fmul_rn(e1, aa), __fmul_rn(e2, v));
        bb = __fadd_rn(__fmul_rn(e1, bb), e2);
        pp = qq;
        if constexpr ((MODE & SEQ_SNAP) != 0) {
            const int slot = p.cp.slot[t];
            if (slot >= 0) {
                float * dst = p.cp.dst[slot] + p.cp.at + c;
                dst[0] = aa; dst[p.C] = bb; dst[2 * p.C] = pp;
            }
        }
        const float yv = __fmul_rn(p.r[o], __fdiv_rn(a, b));
        p.y[o] = yv;
        if (p.q_out) act::warp_emit_block(act::StagedOut{p.q_out, p.q_type, p.C}, c >> 5, yv);      // T == 1, C % 32 == 0: whole warps only
    }
    p.aa_out[so + c] = aa; p.bb_out[so + c] = bb; p.pp_out[so + c] = pp;
    trace_end(p.trace);
}

// Per-head normalisation of S values held one per thread: ggml_norm over a head
// (ggml-cpu.c:6906-6925: mean and variance summed sequentially in double).
template <int S>
__device__ __forceinline__ float head_norm(float y, float eps, float * red) {
    const int j = threadIdx.x;
    __syncthreads();
    red[j] = y;
    __syncthreads();
    double s = 0;
#pragma unroll 8
    for (int i = 0; i < S; i++) s += (double) red[i];
    const float mean = (float) (s / S);
    const float v = y - mean;
    __syncthreads();
    red[j] = v * v;
    __syncthreads();
    double s2 = 0;
#pragma unroll 8
    for (int i = 0; i < S; i++) s2 += (double) red[i];
    const float var = (float) (s2 / S);
    return v * (1.0f / sqrtf(var + eps));
}

// ---------------------------------------------------------------------------------------------
// v5 / v6: ggml_compute_forward_rwkv_wkv6_f32 (ggml-cpu.c:11870-11905). Four threads share state column S[.][j]
// (thread 4j+q owns key rows i in [q*S/4, (q+1)*S/4)), so the per-token loop is S/4 long and the head's S outputs are
// combined with two shuffles;  kv = v_j*k_i;  y_j += (kv*tf_i + S_ij) * r_i;  S_ij = S_ij*td_i + kv  with the same FMA
// grouping as the reference's vector path. Per-head norm statistics (ggml_norm, double sums) by warp shuffles.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double wkv_warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ void wkv_cp16(void * smem_dst, const void * gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"((uint32_t) __cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void wkv_cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wkv_cp_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

constexpr int WKV6_TB = 8;   // tokens per staged chunk
template <int S> struct __align__(16) Wkv6Chunk { float k[WKV6_TB][S], r[WKV6_TB][S], d[WKV6_TB][S], v[WKV6_TB][S]; };

// Thread layout: NOCT = S/8 "octants" of 8 key rows x S/4 groups of 4 value columns; a WORKER thread owns the 8 x 4 state
// patch S[oct*8 .. +8][jg*4 .. +4] in registers. Per token it reads its 8 k / r / decay / first values and 4 v values
// from shared memory (8 lanes = one 128-byte wavefront) and does 32 x 4 FMA-class operations.
// One or two further warps (NORM) do nothing but the per-head normalisation of finished chunks, concurrently with the
// recurrence of the next chunk (round 2: with all warps alternating between the two phases a 128-token pass of a 7B layer spent
// 109k cycles in the recurrence and 57k in the normalisation, one after the other).
template <int S> struct Wkv6Layout {
    static constexpr int NOCT = S / 8, NJG = S / 4, NT = NOCT * NJG, WORK = NT < 32 ? 32 : NT;
    static constexpr int NORM_WARPS = S >= 64 ? 2 : 1, NORM = NORM_WARPS * 32, BLOCK = WORK + NORM;
};
__device__ __forceinline__ void wkv_bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void wkv_bar_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(count) : "memory"); }

// MODE SEQ_BATCH: the block walks ONE token, column blockIdx.y, on the state of sequence blockIdx.y.
// MODE SEQ_RAGGED: the block walks the columns [seq_off[y], seq_off[y + 1]) of sequence y = blockIdx.y, as a single sequence's
// block walks its T tokens, on the state of sequence y; a sequence without columns leaves at once.
// DW2 >= 0 (v6, one token of one sequence): the decay of the head's S channels is the last LoRA GEMV, p.dw2 with weights of type DW2,
// computed here: its S rows are copied to shared memory before the dependency wait, lora1 is staged after it as the streaming GEMV
// stages a column, and rows_dot writes exp(-exp(..)) straight into the decay row the recurrence reads.
// DW2 == WKV6_RAGGED (with BATCH_OR_RAGGED = true): the ragged mode. (A value of the third argument rather than a MODE argument of its own, so
// that the names of the other instantiations stay what they were.)
// DW2 == WKV6_SNAP (BATCH_OR_RAGGED = false) / WKV6_RAGGED_SNAP (true): the single-sequence / ragged mode with checkpoints: after every
// column with a checkpoint slot, each worker also writes its 8 x 4 state patch into the slot.
constexpr int WKV6_RAGGED = -2, WKV6_SNAP = -3, WKV6_RAGGED_SNAP = -4;
template <int S, bool BATCH_OR_RAGGED, int DW2 = -1>
__global__ void __launch_bounds__(Wkv6Layout<S>::BLOCK) wkv6_kernel(const Wkv6Params p) {
    using LY = Wkv6Layout<S>;
    constexpr bool SNAP = DW2 == WKV6_SNAP || DW2 == WKV6_RAGGED_SNAP;
    constexpr int MODE = (DW2 == WKV6_RAGGED || DW2 == WKV6_RAGGED_SNAP) ? SEQ_RAGGED : BATCH_OR_RAGGED ? SEQ_BATCH : SEQ_ONE;
    constexpr bool BATCH = MODE == SEQ_BATCH;
    constexpr int TB = WKV6_TB, NOCT = LY::NOCT, NT = LY::NT, WORK = LY::WORK, BLOCK = LY::BLOCK, NNW = LY::NORM_WARPS, CPL = (S + 31) / 32;
    constexpr int BAR_FULL = 1, BAR_EMPTY = 3, BAR_WORK = 5;        // named barriers: FULL / EMPTY + (chunk & 1), the workers' own
    __shared__ Wkv6Chunk<S> buf[2];
    __shared__ __align__(16) float sf[S], sdc[S];
    __shared__ __align__(16) float ybuf[2][TB][S];
    trace_begin(p.trace);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int h = blockIdx.x, tid = threadIdx.x, C = p.H * S;
    constexpr bool RAGGED = MODE == SEQ_RAGGED;
    int col0 = BATCH ? blockIdx.y : 0;            // column of the block's first token
    int r_T = 0;                                  // ragged: the sequence's tokens (the other modes: p.T / 1 as written below)
    if constexpr (RAGGED) {
        col0 = p.seq_off[blockIdx.y]; r_T = p.seq_off[blockIdx.y + 1] - col0;
        if (r_T == 0) return;
    }
    const long long so = MODE != SEQ_ONE ? blockIdx.y * p.seq_stride : 0;
    const bool is_norm = tid >= WORK;
    const bool worker = tid < NT;
    const int oct = worker ? tid % NOCT : 0, jg = worker ? tid / NOCT : 0;
    const int i0 = oct * 8, j0 = jg * 4;
    const int lane = tid & 31;
    const int nchunks = BATCH ? 1 : ((RAGGED ? r_T : p.T) + TB - 1) / TB;
    // the recurrent state (written by the previous token's pass) and the parameters do not depend on the previous
    // kernel: pull them in before the programmatic-dependency wait
    float st[8][4];
    if (!is_norm) {
#pragma unroll
        for (int ii = 0; ii < 8; ii++) {
            const float4 v = *reinterpret_cast<const float4 *>(p.state_in + so + ((size_t) h * S + i0 + ii) * S + j0);
            st[ii][0] = v.x; st[ii][1] = v.y; st[ii][2] = v.z; st[ii][3] = v.w;
        }
    }
    extern __shared__ __align__(16) uint8_t wkv_dw2_smem[];      // DW2 >= 0: [S rows of dw2][staged lora1]
    if constexpr (DW2 >= 0) {
        const int bytes = S * (int) p.dw2.pitch;
        const uint8_t * src = reinterpret_cast<const uint8_t *>(p.dw2.W) + (size_t) h * bytes;
        for (int i = tid * 16; i < bytes; i += BLOCK * 16) wkv_cp16(wkv_dw2_smem + i, src + i);
        wkv_cp_commit();
    }
    for (int i = tid; i < S; i += BLOCK) {
        sf[i] = p.per_head_scalars ? p.tf[h] : p.tf[h * S + i];
        if constexpr (DW2 < 0) sdc[i] = p.td_per_token ? 0.f : (p.per_head_scalars ? p.td[h] : p.td[h * S + i]);
    }
    float lw[CPL], lb[CPL];
#pragma unroll
    for (int i = 0; i < CPL; i++) {
        const int col = lane + 32 * i;
        lw[i] = (is_norm && col < S) ? p.lnx_w[h * S + col] : 0.f;
        lb[i] = (is_norm && col < S) ? p.lnx_b[h * S + col] : 0.f;
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if constexpr (DW2 >= 0) {
        // the token's k / r / v rows (chunk 0, which the workers' stage(0) copies on the other paths) are requested first: their L2
        // round trip overlaps the one of lora1 and the decay rows instead of following it
        for (int f = tid * 4; f < S && tid < WORK; f += WORK * 4) {
            const size_t o = (size_t) h * S + f;
            wkv_cp16(&buf[0].k[0][f], p.k + o);
            wkv_cp16(&buf[0].r[0][f], p.r + o);
            wkv_cp16(&buf[0].v[0][f], p.v + o);
        }
        wkv_cp_commit();
        uint8_t * act = wkv_dw2_smem + (size_t) S * p.dw2.pitch;
        // stage_column's F16 / F32 loops take element k on thread k (stride 256): with 192 threads that needs dw2.K <= 192
        // (v6_lora_fold_shapes: K <= 128); quantised columns use one thread per 32-element block
        if (tid < tma::CONSUMER_THREADS) tma::stage_column<4, true, DW2, false>(p.dw2, 0, act, nullptr);
        wkv_cp_wait<0>();
        __syncthreads();
        tma::rows_dot<DW2>(p.dw2, wkv_dw2_smem, S, h * S, act, sdc);
    }
    __syncthreads();                                   // sf / sdc

    if (!is_norm) {
        // ===== workers. Chunks of TB tokens of the head's (k, r, decay, v) rows travel to shared memory by cp.async, one chunk ahead;
        // the recurrence walks a chunk's tokens serially with the state in registers and no barrier inside the chunk.
        auto stage = [&](int c) {
            Wkv6Chunk<S> & B = buf[c & 1];
            const int t0 = c * TB, nt = BATCH ? 1 : min(TB, (RAGGED ? r_T : p.T) - t0);
            constexpr int PER_ROW = S / 4;
            for (int idx = tid; idx < nt * PER_ROW; idx += WORK) {
                const int tt = idx / PER_ROW, f = (idx % PER_ROW) * 4;
                const size_t o = (size_t) (col0 + t0 + tt) * C + h * S + f;
                wkv_cp16(&B.k[tt][f], p.k + o);
                wkv_cp16(&B.r[tt][f], p.r + o);
                wkv_cp16(&B.v[tt][f], p.v + o);
                if (p.td_per_token) wkv_cp16(&B.d[tt][f], p.td + o);
            }
        };
        // trace marks of CTA 0 (cycles, stored as start + cycles): [0] waiting for the staged chunk, [1] the recurrence,
        // [2] waiting for the normalising warps to hand an output buffer back
        const bool acct = p.trace != nullptr && blockIdx.x == 0 && (MODE == SEQ_ONE || blockIdx.y == 0) && tid == 0;
        long long a0 = 0, a1 = 0, a2 = 0, tq = acct ? clock64() : 0;
        auto tick = [&](long long & a) { if (acct) { const long long now = clock64(); a += now - tq; tq = now; } };
        float tfr[8];     // time_first of my key rows
#pragma unroll
        for (int ii = 0; ii < 8; ii++) tfr[ii] = sf[i0 + ii];
        if constexpr (DW2 < 0) stage(0);               // DW2 >= 0: already on its way
        wkv_cp_commit();
        for (int c = 0; c < nchunks; c++) {
            wkv_cp_wait<0>();
            wkv_bar_sync(BAR_WORK, WORK);              // chunk c is staged for everybody, and everybody is done reading chunk c - 1
            if (c + 1 < nchunks) stage(c + 1);         // into the buffer chunk c - 1 occupied; lands while chunk c is being walked
            wkv_cp_commit();
            tick(a0);
            if (c >= 2) wkv_bar_sync(BAR_EMPTY + (c & 1), BLOCK);      // ybuf[c & 1] has been normalised (chunk c - 2)
            tick(a2);
            const Wkv6Chunk<S> & B = buf[c & 1];
            float (* yb)[S] = ybuf[c & 1];
            const int t0 = c * TB, nt = BATCH ? 1 : min(TB, (RAGGED ? r_T : p.T) - t0);
            unsigned snap = 0;     // SNAP: bit tt = token tt of the chunk has a checkpoint slot
            if constexpr (SNAP) {
                for (int tt = 0; tt < nt; tt++) snap |= (p.cp.slot[col0 + t0 + tt] >= 0 ? 1u : 0u) << tt;
            }
            // recurrence (kv = v_j*k_i;  y_j += (kv*tf_i + S_ij) * r_i;  S_ij = S_ij*td_i + kv), 8 + 8 + 8 + 4 operands per token from
            // shared memory
            float kk[8], rr[8], dv[8], vv[4];
            auto fetch = [&](int tt, float (&k_)[8], float (&r_)[8], float (&d_)[8], float (&v_)[4]) {
                const float * dd = p.td_per_token ? B.d[tt] : sdc;
                const float4 a = *reinterpret_cast<const float4 *>(&B.k[tt][i0]), b = *reinterpret_cast<const float4 *>(&B.k[tt][i0 + 4]);
                k_[0] = a.x; k_[1] = a.y; k_[2] = a.z; k_[3] = a.w; k_[4] = b.x; k_[5] = b.y; k_[6] = b.z; k_[7] = b.w;
                const float4 c4 = *reinterpret_cast<const float4 *>(&B.r[tt][i0]), d4 = *reinterpret_cast<const float4 *>(&B.r[tt][i0 + 4]);
                r_[0] = c4.x; r_[1] = c4.y; r_[2] = c4.z; r_[3] = c4.w; r_[4] = d4.x; r_[5] = d4.y; r_[6] = d4.z; r_[7] = d4.w;
                const float4 e = *reinterpret_cast<const float4 *>(&dd[i0]), f = *reinterpret_cast<const float4 *>(&dd[i0 + 4]);
                d_[0] = e.x; d_[1] = e.y; d_[2] = e.z; d_[3] = e.w; d_[4] = f.x; d_[5] = f.y; d_[6] = f.z; d_[7] = f.w;
                const float4 g = *reinterpret_cast<const float4 *>(&B.v[tt][j0]);
                v_[0] = g.x; v_[1] = g.y; v_[2] = g.z; v_[3] = g.w;
            };
            // two tokens per trip where the register file allows it: the shuffles and the shared-memory loads of one token then
            // overlap the multiply-adds of its neighbour (a warp is alone on its scheduler: nothing else hides their latency).
            // (A full chunk written out as ONE basic block with two explicit operand sets, loads of token t + 1 ahead of the arithmetic
            // of token t, was slower: 93k vs 83k cycles per 128 tokens.)
#pragma unroll(S <= 64 ? 2 : 1)
            for (int tt = 0; tt < nt; tt++) {
                fetch(tt, kk, rr, dv, vv);
                float y[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int ii = 0; ii < 8; ii++) {
#pragma unroll
                    for (int jj = 0; jj < 4; jj++) {
                        const float kv = __fmul_rn(vv[jj], kk[ii]);
                        const float temp = __fmaf_rn(kv, tfr[ii], st[ii][jj]);
                        y[jj] = __fmaf_rn(temp, rr[ii], y[jj]);
                        st[ii][jj] = __fmaf_rn(st[ii][jj], dv[ii], kv);
                    }
                }
#pragma unroll
                for (int o = 1; o < NOCT; o <<= 1) {
#pragma unroll
                    for (int jj = 0; jj < 4; jj++) y[jj] += __shfl_xor_sync(0xffffffffu, y[jj], o);
                }
                if (worker && oct == 0) *reinterpret_cast<float4 *>(&yb[tt][j0]) = make_float4(y[0], y[1], y[2], y[3]);
                if constexpr (SNAP) {
                    if (worker && ((snap >> tt) & 1u)) {
                        float * dst = p.cp.dst[p.cp.slot[col0 + t0 + tt]] + p.cp.at + ((size_t) h * S + i0) * S + j0;
#pragma unroll
                        for (int ii = 0; ii < 8; ii++)
                            *reinterpret_cast<float4 *>(dst + (size_t) ii * S) = make_float4(st[ii][0], st[ii][1], st[ii][2], st[ii][3]);
                    }
                }
            }
            tick(a1);
            wkv_bar_arrive(BAR_FULL + (c & 1), BLOCK);     // the chunk's output rows are complete: over to the normalising warps
        }
        if (worker) {
#pragma unroll
            for (int ii = 0; ii < 8; ii++)
                *reinterpret_cast<float4 *>(p.state_out + so + ((size_t) h * S + i0 + ii) * S + j0) = make_float4(st[ii][0], st[ii][1], st[ii][2], st[ii][3]);
        }
        if (acct) {
            p.trace->mark[0] = p.trace->start + (unsigned long long) a0;
            p.trace->mark[1] = p.trace->start + (unsigned long long) a1;
            p.trace->mark[2] = p.trace->start + (unsigned long long) a2;
            p.trace->mark[3] = p.trace->start;
        }
    } else {
        // ===== normalising warps: per-head norm (ggml_norm over the head, ggml-cpu.c:6906-6925; sum and sum of squares in double),
        // ln_x and the gate for a finished chunk's tokens, one warp per token, while the workers walk the next chunk
        const int nwarp = (tid - WORK) >> 5;
        constexpr int PER = (TB + NNW - 1) / NNW;        // tokens of a chunk per normalising warp
        for (int c = 0; c < nchunks; c++) {
            const int t0 = c * TB, nt = BATCH ? 1 : min(TB, (RAGGED ? r_T : p.T) - t0);
            // the gate values of my tokens: requested before the wait for the chunk, so their latency hides behind the recurrence
            float gg[PER][CPL];
#pragma unroll
            for (int u = 0; u < PER; u++) {
                const int tt = nwarp + u * NNW;
#pragma unroll
                for (int i = 0; i < CPL; i++) {
                    const int col = lane + 32 * i;
                    gg[u][i] = (p.g && tt < nt && col < S) ? p.g[(size_t) (col0 + t0 + tt) * C + h * S + col] : 0.f;
                }
            }
            wkv_bar_sync(BAR_FULL + (c & 1), BLOCK);
            const float (* yb)[S] = ybuf[c & 1];
#pragma unroll
            for (int u = 0; u < PER; u++) {
                const int tt = nwarp + u * NNW;
                if (tt >= nt) break;
                float yv[CPL];
                double s1 = 0, s2 = 0;
#pragma unroll
                for (int i = 0; i < CPL; i++) {
                    const int col = lane + 32 * i;
                    yv[i] = col < S ? yb[tt][col] : 0.f;
                    s1 += (double) yv[i];
                    s2 += (double) yv[i] * (double) yv[i];
                }
                s1 = wkv_warp_sum_d(s1);
                s2 = wkv_warp_sum_d(s2);
                constexpr double INV_S = 1.0 / S;                          // S is a power of two: x * INV_S == x / S bit for bit, without the
                const double mean_d = s1 * INV_S;                          // two double-precision divisions per token
                const float mean = (float) mean_d;
                const float var = (float) fmax(s2 * INV_S - mean_d * mean_d, 0.0);
                const float rstd = 1.0f / sqrtf(var + p.eps);
                const size_t o = (size_t) (col0 + t0 + tt) * C + h * S;
#pragma unroll
                for (int i = 0; i < CPL; i++) {
                    const int col = lane + 32 * i;
                    if (col < S) {
                        float n = (yv[i] - mean) * rstd;
                        n = __fadd_rn(__fmul_rn(n, lw[i]), lb[i]);
                        if (p.g) n = __fmul_rn(n, gg[u][i]);
                        p.y[o + col] = n;
                        if (p.q_out) act::warp_emit_block(act::StagedOut{p.q_out, p.q_type, C}, (h * S) / 32 + i, n);   // T == 1, S % 32 == 0: col < S for all lanes
                    }
                }
            }
            if (c + 2 < nchunks) wkv_bar_arrive(BAR_EMPTY + (c & 1), BLOCK);     // ybuf[c & 1] may take chunk c + 2
        }
    }
    trace_end(p.trace);
}

// ---------------------------------------------------------------------------------------------
// v7: rwkv_att_v7 (rwkv_graph.inc:432-479) around rwkv_wkv_v7_impl (rwkv_operators_wkv_v7.inc:63-101).
// Thread i owns state row S[i][.] (value index i, key index j).
// ---------------------------------------------------------------------------------------------
// MODE SEQ_BATCH: the block handles ONE token, column blockIdx.y, on the state of sequence blockIdx.y.
// MODE SEQ_RAGGED: the columns [seq_off[y], seq_off[y + 1]) of sequence y = blockIdx.y on its state; none: the block leaves at once.
// MODE | SEQ_SNAP: after every column with a checkpoint slot, thread i also writes its state row into the slot.
template <int S, int MODE>
__global__ void __launch_bounds__(S) wkv7_kernel(const Wkv7Params p) {
    constexpr int M = MODE & ~SEQ_SNAP;
    constexpr bool BATCH = M == SEQ_BATCH;
    __shared__ float sr[S], sw[S], sk[S], sa[S], sb[S], red[S];
    trace_begin(p.trace);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int h = blockIdx.x, i = threadIdx.x, C = p.H * S, c = h * S + i;
    const long long so = M != SEQ_ONE ? blockIdx.y * p.seq_stride : 0;
    int t_begin = BATCH ? blockIdx.y : 0, t_end = BATCH ? blockIdx.y + 1 : p.T;
    if constexpr (M == SEQ_RAGGED) {
        t_begin = p.seq_off[blockIdx.y]; t_end = p.seq_off[blockIdx.y + 1];
        if (t_begin == t_end) return;
    }
    float st[S];
#pragma unroll
    for (int j = 0; j < S; j++) st[j] = p.state_in[so + ((size_t) h * S + i) * S + j];
    const float kk_w = p.k_k[c], ka_w = p.k_a[c], rk_w = p.r_k[c];
    const float lw = p.lnx_w[c], lb = p.lnx_b[c];
    asm volatile("griddepcontrol.wait;" ::: "memory");
    for (int t = t_begin; t < t_end; t++) {
        const size_t o = (size_t) t * C + c;
        const float r = p.r[o], w = p.w[o], k0 = p.k[o], a = p.a[o];
        float v = p.v[o];
        // kk = l2norm_head(k * k_k)  (rwkv_graph.inc:433-434, rwkv_operators.inc:61-76: float sum, eps 1e-12)
        const float kk0 = __fmul_rn(k0, kk_w);
        __syncthreads();
        red[i] = kk0;
        __syncthreads();
        float ss = 0.f;
#pragma unroll 8
        for (int j = 0; j < S; j++) ss = __fmaf_rn(red[j], red[j], ss);
        const float kk = __fmul_rn(kk0, 1.0f / fmaxf(sqrtf(ss), 1e-12f));
        // k = k + (a*ka - ka), ka = k*k_a   (rwkv_graph.inc:436-437)
        const float ka = __fmul_rn(k0, ka_w);
        const float k = __fadd_rn(k0, __fsub_rn(__fmul_rn(a, ka), ka));
        // v = v + (v_first - v) * gate   (rwkv_graph.inc:440-453)
        if (p.vgate) v = __fadd_rn(v, __fmul_rn(__fsub_rn(p.v_first[o], v), p.vgate[o]));
        if (p.v_out) p.v_out[o] = v;
        __syncthreads();
        sr[i] = r; sw[i] = w; sk[i] = k; sa[i] = -kk; sb[i] = __fmul_rn(kk, a);
        __syncthreads();
        float dot_a = 0.f;
#pragma unroll
        for (int j = 0; j < S; j++) dot_a = __fmaf_rn(sa[j], st[j], dot_a);
        float y = 0.f;
#pragma unroll
        for (int j = 0; j < S; j++) {
            const float kv = __fmul_rn(v, sk[j]);
            st[j] = __fmaf_rn(dot_a, sb[j], __fmaf_rn(st[j], sw[j], kv));
            y = __fmaf_rn(st[j], sr[j], y);
        }
        if constexpr ((MODE & SEQ_SNAP) != 0) {
            const int slot = p.cp.slot[t];
            if (slot >= 0) {
                float * dst = p.cp.dst[slot] + p.cp.at + ((size_t) h * S + i) * S;
#pragma unroll
                for (int j = 0; j < S; j++) dst[j] = st[j];
            }
        }
        float n = head_norm<S>(y, 64e-5f, red);
        n = __fadd_rn(__fmul_rn(n, lw), lb);
        // + v * sum_head(k*r*r_k)   (rwkv_graph.inc:472-477; ggml_sum_rows accumulates in double)
        __syncthreads();
        red[i] = __fmul_rn(__fmul_rn(k, r), rk_w);
        __syncthreads();
        double rk = 0;
#pragma unroll 8
        for (int j = 0; j < S; j++) rk += (double) red[j];
        n = __fadd_rn(n, __fmul_rn(v, (float) rk));
        const float yv = __fmul_rn(n, p.g[o]);
        p.y[o] = yv;
        if (p.q_out) act::warp_emit_block(act::StagedOut{p.q_out, p.q_type, C}, c >> 5, yv);       // T == 1, S % 32 == 0: whole warps only
    }
#pragma unroll
    for (int j = 0; j < S; j++) p.state_out[so + ((size_t) h * S + i) * S + j] = st[j];
    trace_end(p.trace);
}

}  // namespace

// Grid row y is sequence y in batch mode (seq_stride > 0) and in ragged mode (seq_off set: n_seq rows); one sequence has a single
// row. The ragged instantiations come after the two others.
// The checkpoint instantiations (cp.slot set: single-sequence or ragged passes) come last.
cudaError_t launch_wkv4(const Wkv4Params & p_in, cudaStream_t s) {
    Wkv4Params p = p_in;
    p.trace = trace_slot("wkv4");
    const int threads = 128;
    if (!p.cp.slot)
        return !p.seq_stride ? launch_pdl(wkv4_kernel<SEQ_ONE>, dim3((p.C + threads - 1) / threads), dim3(threads), 0, s, p)
             : !p.seq_off    ? launch_pdl(wkv4_kernel<SEQ_BATCH>, dim3((p.C + threads - 1) / threads, p.T), dim3(threads), 0, s, p)
                             : launch_pdl(wkv4_kernel<SEQ_RAGGED>, dim3((p.C + threads - 1) / threads, p.n_seq), dim3(threads), 0, s, p);
    if (p.seq_stride && !p.seq_off) return cudaErrorInvalidValue;
    return !p.seq_stride ? launch_pdl(wkv4_kernel<SEQ_SNAP | SEQ_ONE>, dim3((p.C + threads - 1) / threads), dim3(threads), 0, s, p)
                         : launch_pdl(wkv4_kernel<SEQ_SNAP | SEQ_RAGGED>, dim3((p.C + threads - 1) / threads, p.n_seq), dim3(threads), 0, s, p);
}

template <int S>
cudaError_t launch_wkv6_kernel(const Wkv6Params & p, cudaStream_t s) {
    if (!p.cp.slot)
        return !p.seq_stride ? launch_pdl(wkv6_kernel<S, false>, dim3(p.H), dim3(Wkv6Layout<S>::BLOCK), 0, s, p)
             : !p.seq_off    ? launch_pdl(wkv6_kernel<S, true>, dim3(p.H, p.T), dim3(Wkv6Layout<S>::BLOCK), 0, s, p)
                             : launch_pdl(wkv6_kernel<S, true, WKV6_RAGGED>, dim3(p.H, p.n_seq), dim3(Wkv6Layout<S>::BLOCK), 0, s, p);
    if (p.seq_stride && !p.seq_off) return cudaErrorInvalidValue;
    return !p.seq_stride ? launch_pdl(wkv6_kernel<S, false, WKV6_SNAP>, dim3(p.H), dim3(Wkv6Layout<S>::BLOCK), 0, s, p)
                         : launch_pdl(wkv6_kernel<S, true, WKV6_RAGGED_SNAP>, dim3(p.H, p.n_seq), dim3(Wkv6Layout<S>::BLOCK), 0, s, p);
}

template <int DW2>
cudaError_t launch_wkv6_decay(const Wkv6Params & p, cudaStream_t s) {
    static PerDeviceOnce once;
    const size_t smem = wkv6_decay_smem_bytes(p.dw2);
    const cudaError_t e = once.run([&] { return cudaFuncSetAttribute(wkv6_kernel<64, false, DW2>, cudaFuncAttributeMaxDynamicSharedMemorySize, WKV6_DECAY_MAX_SMEM); });
    if (e != cudaSuccess) return e;
    return launch_pdl(wkv6_kernel<64, false, DW2>, dim3(p.H), dim3(Wkv6Layout<64>::BLOCK), smem, s, p);
}

size_t wkv6_decay_smem_bytes(const GemvProblem & dw2) {
    return (size_t) 64 * (size_t) dw2.pitch + tma::act_bytes_per_column(dw2.type, dw2.K);
}

cudaError_t launch_wkv6(const Wkv6Params & p_in, cudaStream_t s) {
    Wkv6Params p = p_in;
    p.trace = trace_slot("wkv6");
    if (p.dw2.W) {      // v6_lora_fold has checked the shape: S == 64, one token of one sequence, a WK == 1 plan
        if (p.S != 64 || p.T != 1 || p.seq_stride || p.cp.slot || wkv6_decay_smem_bytes(p.dw2) > WKV6_DECAY_MAX_SMEM) return cudaErrorInvalidValue;
        switch (p.dw2.type) {
            case DT_Q4_0: return launch_wkv6_decay<DT_Q4_0>(p, s);
            case DT_Q4_1: return launch_wkv6_decay<DT_Q4_1>(p, s);
            case DT_Q5_0: return launch_wkv6_decay<DT_Q5_0>(p, s);
            case DT_Q5_1: return launch_wkv6_decay<DT_Q5_1>(p, s);
            case DT_Q8_0: return launch_wkv6_decay<DT_Q8_0>(p, s);
            case DT_F16: return launch_wkv6_decay<DT_F16>(p, s);
            case DT_F32: return launch_wkv6_decay<DT_F32>(p, s);
            default: return cudaErrorInvalidValue;
        }
    }
    switch (p.S) {
        case 8: return launch_wkv6_kernel<8>(p, s);
        case 16: return launch_wkv6_kernel<16>(p, s);
        case 32: return launch_wkv6_kernel<32>(p, s);
        case 64: return launch_wkv6_kernel<64>(p, s);
        case 128: return launch_wkv6_kernel<128>(p, s);
        default: return cudaErrorInvalidValue;
    }
}

template <int S>
cudaError_t launch_wkv7_kernel(const Wkv7Params & p, cudaStream_t s) {
    if (!p.cp.slot)
        return !p.seq_stride ? launch_pdl(wkv7_kernel<S, SEQ_ONE>, dim3(p.H), dim3(S), 0, s, p)
             : !p.seq_off    ? launch_pdl(wkv7_kernel<S, SEQ_BATCH>, dim3(p.H, p.T), dim3(S), 0, s, p)
                             : launch_pdl(wkv7_kernel<S, SEQ_RAGGED>, dim3(p.H, p.n_seq), dim3(S), 0, s, p);
    if (p.seq_stride && !p.seq_off) return cudaErrorInvalidValue;
    return !p.seq_stride ? launch_pdl(wkv7_kernel<S, SEQ_SNAP | SEQ_ONE>, dim3(p.H), dim3(S), 0, s, p)
                         : launch_pdl(wkv7_kernel<S, SEQ_SNAP | SEQ_RAGGED>, dim3(p.H, p.n_seq), dim3(S), 0, s, p);
}

cudaError_t launch_wkv7(const Wkv7Params & p_in, cudaStream_t s) {
    Wkv7Params p = p_in;
    p.trace = trace_slot("wkv7");
    switch (p.S) {
        case 8: return launch_wkv7_kernel<8>(p, s);
        case 16: return launch_wkv7_kernel<16>(p, s);
        case 32: return launch_wkv7_kernel<32>(p, s);
        case 64: return launch_wkv7_kernel<64>(p, s);
        case 128: return launch_wkv7_kernel<128>(p, s);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace rwkv
