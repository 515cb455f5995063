// Streaming integer GEMV kernels for quantised-MoE decode (sm_90a).
//
// Both kernels are HBM-bound byte streamers (3.1 FLOP/B at bs=1): every weight byte is read exactly
// once with 16-byte read-only loads that bypass L1, many loads are put in flight per lane before any
// is consumed, and the arithmetic is int8 dp4a against activations staged in shared memory.
// No tensor cores: at M = 1..8 rows per expert the MMA tile would be >87% padding and the kernel
// would still be bound by the same bytes.
//
//   rows_kernel  ("phase 1" of MOE::forward_one, moe.cpp:171-210; Linear::forward_many, linear.cpp:37-63)
//       out[slot][r] = epilogue( W0[e_slot][r,:] . xq_t , W1[e_slot][r,:] . xq_t )
//       one activation row per token shared by all of the token's slots.
//   reduce_kernel ("phase 2", moe.cpp:216-245; MLP down, mlp.cpp:99-117)
//       out[t][h] = sum_j w[t][j] * ( W[e_tj][h,:] . aq_tj )   — aq quantised in the prologue
//
// grid = (gx, T): blockIdx.y is the token, blockIdx.x splits that token's work into contiguous,
// equally sized ranges (gx is chosen so gx*T ~ kGemvCtasPerSm CTAs per SM).
//
// A warp walks a row in "steps" (32 lanes = Fmt::kBlocksPerStep super-blocks).  Steps are consumed in
// batches of NB: all global loads of a batch (RW rows x NM matrices x NB steps) are issued before the
// first dot product, which is what keeps ~16 x 16 B per lane in flight.
#pragma once
#include "act_quant.cuh"
#include "formats.cuh"

namespace ktb {

constexpr int kGemvThreads = 256;
constexpr int kGemvCtasPerSm = 2;   // rows_kernel / reduce_kernel: launch bounds and grid size

struct RowsParams {
    const void* w0;         // [E][rows][ncols] blocks
    const void* w1;         // second matrix (PAIR) or null
    int type0, type1;       // ggml types (FmtGenK reads them at run time)
    int n_experts;          // E behind w0/w1 (1 for a dense linear)
    int rows, ncols;        // per-expert matrix shape (out features, in features)
    int slots;              // slots per token (k for MoE, 1 for dense)
    const int64_t* ids;     // [T][slots] expert ids or null (dense: expert 0)
    int id_offset;          // expert-parallel shard offset
    const void* x;          // [T][ncols] hidden_type
    int hidden_type;
    int use_silu;
    float* out_f32;         // PAIR: [T*nslots][rows] fp32 act(g)*u ; else optional fp32 out
    void* out_hidden;       // !PAIR: [T][rows] hidden_type (slots must be 1) or null
    const float* bias;      // !PAIR optional [rows]
    const int* bsz;         // optional device batch size
    int ntokens;            // T (used by the token-looping kernels; the (gx, T)-grid kernels read blockIdx.y)
    // optional extra slot (index == slots) served from separate tensors: the shared expert fused into
    // the routed launch (KDeepseekV3MoE: y = experts(x) + shared_experts(x), experts.py:984-1011)
    const void* x0;
    const void* x1;
    int shared_token;       // -1: the extra slot applies to every token; t >= 0: to token t only (expert-parallel shards
                            // compute the shared expert for their own token)
};

// one batch of N steps starting at step s0 for RW rows x NM matrices; all rows share ONE activation row
template <class Fmt, int RW, int NM, int N>
__device__ __forceinline__ void gemv_batch(const typename Fmt::Row (&rp)[RW][NM], const bool (&valid)[RW], const ActQ8K& act,
                                           int s0, int nblk, const typename Fmt::Lane& L, float (&acc)[RW][NM]) {
    typename Fmt::Regs regs[RW][NM][N];
#pragma unroll
    for (int rw = 0; rw < RW; rw++)
#pragma unroll
        for (int n = 0; n < N; n++) {
            const int blk = (s0 + n) * Fmt::kBlocksPerStep + L.blk;
            if (valid[rw] && blk < nblk) {
#pragma unroll
                for (int m = 0; m < NM; m++) Fmt::load(rp[rw][m], blk, L, regs[rw][m][n]);
            }
        }
#pragma unroll
    for (int n = 0; n < N; n++) {
        const int blk = (s0 + n) * Fmt::kBlocksPerStep + L.blk;
        if (blk < nblk) {
            typename Fmt::Act A;
            Fmt::load_act(act, blk, L, A);
#pragma unroll
            for (int rw = 0; rw < RW; rw++)
                if (valid[rw]) {
#pragma unroll
                    for (int m = 0; m < NM; m++) acc[rw][m] += Fmt::dot(regs[rw][m][n], A, L);
                }
        }
    }
}

template <class Fmt, int RW, int NM, int NB>
__device__ __forceinline__ void gemv_rows(const typename Fmt::Row (&rp)[RW][NM], const bool (&valid)[RW], const ActQ8K& act,
                                          int nblk, const typename Fmt::Lane& L, float (&acc)[RW][NM]) {
    const int nsteps = (nblk + Fmt::kBlocksPerStep - 1) / Fmt::kBlocksPerStep;
    int s0 = 0;
    for (; s0 + NB <= nsteps; s0 += NB) gemv_batch<Fmt, RW, NM, NB>(rp, valid, act, s0, nblk, L, acc);
    const int tail = nsteps - s0;
    if (NB > 1 && tail == 1) gemv_batch<Fmt, RW, NM, 1>(rp, valid, act, s0, nblk, L, acc);
    if (NB > 2 && tail == 2) gemv_batch<Fmt, RW, NM, 2>(rp, valid, act, s0, nblk, L, acc);
    if (NB > 3 && tail == 3) gemv_batch<Fmt, RW, NM, 3>(rp, valid, act, s0, nblk, L, acc);
}

// Reduce 4 per-lane partial sums over the warp with 6 shuffles; the total of value i ends up in every
// lane whose bits (4,3) equal i, i.e. lanes 0, 8, 16, 24 hold totals 0, 1, 2, 3.
__device__ __forceinline__ float warp_reduce4(float v0, float v1, float v2, float v3, int lane) {
    const bool hi16 = lane & 16, hi8 = lane & 8;
    float a0 = hi16 ? v2 : v0, a1 = hi16 ? v3 : v1;
    const float b0 = hi16 ? v0 : v2, b1 = hi16 ? v1 : v3;
    a0 += __shfl_xor_sync(0xffffffffu, b0, 16);
    a1 += __shfl_xor_sync(0xffffffffu, b1, 16);
    float c = hi8 ? a1 : a0;
    const float d = hi8 ? a0 : a1;
    c += __shfl_xor_sync(0xffffffffu, d, 8);
    c += __shfl_xor_sync(0xffffffffu, c, 4);
    c += __shfl_xor_sync(0xffffffffu, c, 2);
    c += __shfl_xor_sync(0xffffffffu, c, 1);
    return c;
}

template <class Fmt, bool PAIR, int RW, int NB>
__global__ void __launch_bounds__(kGemvThreads, kGemvCtasPerSm) rows_kernel(const RowsParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int t = blockIdx.y;
    if (p.bsz && t >= *p.bsz) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = kGemvThreads / 32;
    const int nblk = p.ncols / QK_K;
    uint8_t* q8 = smem;                                                        // ncols
    float* dx = reinterpret_cast<float*>(smem + p.ncols);                      // nblk
    int16_t* bsums = reinterpret_cast<int16_t*>(smem + p.ncols + nblk * 4);    // ncols/16
    const ActQ8K act{q8, dx, bsums};
    const typename Fmt::Lane L = Fmt::lane(lane);

    const int nslots = p.slots + (p.x0 ? 1 : 0);
    const int total = nslots * p.rows;   // < 2^31 (launcher checks): keep the per-unit index math 32-bit
    const int u0 = (int)((long)total * blockIdx.x / gridDim.x), u1 = (int)((long)total * (blockIdx.x + 1) / gridDim.x);
    constexpr int NM = PAIR ? 2 : 1;

    // rows of unit u (one per matrix); returns false for skipped experts / out-of-range units
    auto unit_rows = [&](int u, typename Fmt::Row (&r)[NM]) -> bool {
        if (u >= u1) return false;
        const int s = u / p.rows, rr = u - s * p.rows;
        if (s == p.slots) {  // the fused extra slot
            r[0] = Fmt::row(p.x0, rr, p.ncols, p.type0);
            if (PAIR) r[NM - 1] = Fmt::row(p.x1, rr, p.ncols, p.type1);
            return true;
        }
        const long e = p.ids ? (long)p.ids[(long)t * p.slots + s] - p.id_offset : 0;
        if (e < 0 || e >= p.n_experts) return false;
        r[0] = Fmt::row(p.w0, e * p.rows + rr, p.ncols, p.type0);
        if (PAIR) r[NM - 1] = Fmt::row(p.w1, e * p.rows + rr, p.ncols, p.type1);
        return true;
    };
    // L2 prefetch of the rows a warp will stream NEXT: one lane, one instruction per row, no registers held.
    auto prefetch_units = [&](int ub) {
        if (lane < RW) {
            typename Fmt::Row r[NM];
            if (unit_rows(ub + lane, r)) {
#pragma unroll
                for (int m = 0; m < NM; m++) Fmt::prefetch(r[m], nblk);
            }
        }
    };

    prefetch_units(u0 + warp * RW);   // first units go to L2 while the activation row is quantised
    cta_quantize_q8k_rows<4>(p.x, (long)t * p.ncols, 0, p.hidden_type, 1, p.ncols, 0u, q8, dx, bsums);
    __syncthreads();

    for (int ub = u0 + warp * RW; ub < u1; ub += nwarps * RW) {
        prefetch_units(ub + nwarps * RW);
        typename Fmt::Row rp[RW][NM];
        bool valid[RW];
        float acc[RW][NM];
#pragma unroll
        for (int rw = 0; rw < RW; rw++) {
#pragma unroll
            for (int m = 0; m < NM; m++) acc[rw][m] = 0.f;
            valid[rw] = unit_rows(ub + rw, rp[rw]);
        }
        gemv_rows<Fmt, RW, NM, NB>(rp, valid, act, nblk, L, acc);
#pragma unroll
        for (int rw = 0; rw < RW; rw++) {
            const int u = ub + rw;
            if (u >= u1) continue;
            float g = warp_sum(acc[rw][0]);
            float uu = PAIR ? warp_sum(acc[rw][NM - 1]) : 0.f;
            if (lane == 0) {
                if (PAIR) {
                    const float a = valid[rw] ? (p.use_silu ? act_silu(g) : act_relu(g)) * uu : 0.f;
                    p.out_f32[(long)t * total + u] = a;
                } else {
                    if (!valid[rw]) g = 0.f;
                    if (p.bias) g += p.bias[u % p.rows];
                    if (p.out_f32) p.out_f32[(long)t * total + u] = g;
                    if (p.out_hidden) store_hidden(p.out_hidden, (long)t * total + u, p.hidden_type, g);
                }
            }
        }
    }
}

struct ReduceParams {
    const void* w;          // [E][rows][ncols]
    int type;
    int n_experts;
    int rows, ncols;        // rows = output features (H), ncols = reduction length (I)
    int slots;              // k
    const int64_t* ids;     // [T][slots] or null (dense)
    int id_offset;
    const float* weights;   // [T][slots] or null (all 1)
    const float* a;         // [T*ns][ncols] fp32 activations (phase-1 output), ns = slots + (xw != null)
    void* out;              // [T][rows] hidden_type
    int hidden_type;
    int accumulate;         // out = round(out + round(result)) in hidden_type (torch `y += y_` semantics)
    const int* bsz;
    int ntokens;            // T
    const void* xw;         // optional extra slot (shared expert down_proj); its result is rounded to
                            // hidden_type separately and added like `y += y_` (experts.py:1011)
    int shared_token;       // see RowsParams
    void* xw_out;           // null: add the shared term to `out` as above; else store it, rounded to xw_out_type, to
    int xw_out_type;        // xw_out[t][rows] and leave `out` = the routed sum only
};

// Slots of a token whose expert lies outside the shard contribute nothing (common.hpp:255-258): the down kernels neither read
// their weights nor quantise their activations.  The mask holds slots 0..31 (the quantiser's row mask); a slot from 32 on
// (k <= 200) is tested against its id where it is used.
__device__ __forceinline__ bool slot_outside(const ReduceParams& p, int t, int j) {
    const long e = p.ids ? (long)p.ids[(long)t * p.slots + j] - p.id_offset : 0;
    return e < 0 || e >= p.n_experts;
}
__device__ __forceinline__ unsigned skip_mask32(const ReduceParams& p, int t) {
    unsigned skip = 0;
    for (int j = 0; j < p.slots && j < 32; j++)
        if (slot_outside(p, t, j)) skip |= 1u << j;
    return skip;
}
__device__ __forceinline__ bool slot_skipped(const ReduceParams& p, int t, unsigned skip, int j) {
    return j < 32 ? (skip >> j) & 1u : slot_outside(p, t, j);
}

// Work item of a warp = (slot j, 4 consecutive output rows): the 4 rows share slot j's int8 activations,
// one ids lookup and one 6-shuffle reduction.
template <class Fmt, int NB>
__global__ void __launch_bounds__(kGemvThreads, kGemvCtasPerSm) reduce_kernel(const ReduceParams p) {
    constexpr int RW = 4;
    extern __shared__ __align__(16) uint8_t smem[];
    const int t = blockIdx.y;
    if (p.bsz && t >= *p.bsz) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = kGemvThreads / 32;
    const int nblk = p.ncols / QK_K;
    const int k = p.slots;
    const int ns = k + (p.xw ? 1 : 0);  // slots staged
    // per-slot staging: q8 [ns][ncols] | dx [ns][nblk] | bsums [ns][ncols/16] | partial [rows_local][ns]
    uint8_t* q8 = smem;
    float* dx = reinterpret_cast<float*>(smem + (size_t)ns * p.ncols);
    int16_t* bsums = reinterpret_cast<int16_t*>(smem + (size_t)ns * p.ncols + (size_t)ns * nblk * 4);
    float* partial = reinterpret_cast<float*>(smem + (size_t)ns * p.ncols + (size_t)ns * nblk * 4 + (size_t)ns * (p.ncols / 16) * 2);

    const int r0 = (int)((long)p.rows * blockIdx.x / gridDim.x), r1 = (int)((long)p.rows * (blockIdx.x + 1) / gridDim.x);
    const int nrows = r1 - r0;

    const unsigned skip = skip_mask32(p, t);
    const typename Fmt::Lane L = Fmt::lane(lane);
    const int ngroups = (nrows + RW - 1) / RW;
    const int total = ngroups * ns;
    auto item_base = [&](int item, const void*& wbase, long& row0, int& j, int& hl0) -> bool {
        if (item >= total) return false;
        j = item / ngroups;
        hl0 = (item - j * ngroups) * RW;
        wbase = p.w;
        row0 = r0 + hl0;
        if (j == k) { wbase = p.xw; return true; }
        if (slot_skipped(p, t, skip, j)) return false;
        const long e = p.ids ? (long)p.ids[(long)t * k + j] - p.id_offset : 0;
        row0 += e * p.rows;
        return true;
    };
    auto prefetch_item = [&](int item) {
        const void* wb; long row0; int j, hl0;
        if (lane < RW && item_base(item, wb, row0, j, hl0) && hl0 + lane < nrows)
            Fmt::prefetch(Fmt::row(wb, row0 + lane, p.ncols, p.type), nblk);
    };
    prefetch_item(warp);   // weights do not depend on phase 1: pull the first rows into L2 during the prologue
    cta_quantize_q8k_rows<4>(p.a, (long)t * ns * p.ncols, p.ncols, KTB200_TYPE_F32, ns, p.ncols, skip, q8, dx, bsums);
    __syncthreads();
    for (int item = warp; item < total; item += nwarps) {
        prefetch_item(item + nwarps);
        const int j = item / ngroups, hl0 = (item - j * ngroups) * RW;
        float res = 0.f;
        if (j == k || !slot_skipped(p, t, skip, j)) {   // warp-uniform
            const void* wbase = p.w;
            long row0 = r0 + hl0;
            if (j == k) {
                wbase = p.xw;
            } else {
                const long e = p.ids ? (long)p.ids[(long)t * k + j] - p.id_offset : 0;
                row0 += e * p.rows;
            }
            typename Fmt::Row rp[RW][1];
            bool valid[RW];
            float acc[RW][1];
#pragma unroll
            for (int rw = 0; rw < RW; rw++) {
                valid[rw] = hl0 + rw < nrows;
                acc[rw][0] = 0.f;
                if (valid[rw]) rp[rw][0] = Fmt::row(wbase, row0 + rw, p.ncols, p.type);
            }
            const ActQ8K act{q8 + (size_t)j * p.ncols, dx + j * nblk, bsums + j * (p.ncols / 16)};
            gemv_rows<Fmt, RW, 1, NB>(rp, valid, act, nblk, L, acc);
            res = warp_reduce4(acc[0][0], acc[1][0], acc[2][0], acc[3][0], lane);
        }
        const int rw = lane >> 3;
        if ((lane & 7) == 0 && hl0 + rw < nrows) partial[(hl0 + rw) * ns + j] = res;
    }
    __syncthreads();
    // weighted accumulation over the k experts IN expert_ids ORDER (moe.cpp:222-236); the reference's
    // `out += d * w` is one fused multiply-add in every FMA-capable build.
    for (int hl = threadIdx.x; hl < nrows; hl += kGemvThreads) {
        float acc = 0.f;
        for (int j = 0; j < k; j++) {
            if (slot_skipped(p, t, skip, j)) continue;
            const float d = partial[hl * ns + j];
            acc = p.weights ? __fmaf_rn(d, p.weights[(long)t * k + j], acc) : acc + d;
        }
        const long o = (long)t * p.rows + r0 + hl;
        if (p.xw) acc = round_hidden(acc, p.hidden_type) + round_hidden(partial[hl * ns + k], p.hidden_type);
        if (p.accumulate) {
            // `y += y_` on hidden-type tensors (experts.py:1011): both operands are already rounded
            // to hidden_type, the sum is rounded once more.
            acc = load_hidden(p.out, o, p.hidden_type) + round_hidden(acc, p.hidden_type);
        }
        store_hidden(p.out, o, p.hidden_type, acc);
    }
}

}  // namespace ktb
