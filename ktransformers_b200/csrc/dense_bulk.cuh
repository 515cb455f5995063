// Dense Q4_K linear (y = x . W^T, decode batches of <= 8 rows) on the bulk-copy ring: q_a / kv_a / q_b / o_proj of the MLA
// block and every other KLinearB200 with Q4_K weights (archive/ktransformers/operators/linear.py:57-155 KLinearBase.forward;
// CPU twin operators/llamafile/linear.cpp:37-70).  The expert kernel (rows_bulk_q4k_kernel) wants rows of >= 16 super-
// blocks — one lane per block — which leaves q_b (6 blocks per row) on the slower register-staged kernel and gives
// o_proj (64 blocks per row) 9 KB slots.  Here a ring slot is a SEGMENT of <= 32 consecutive blocks of the row-major weight
// stream, one lane per block:
//     short rows (nblk <= 16): a segment is R = 32 / nblk whole rows (one contiguous copy), reduced per group of nblk lanes
//     long rows  (nblk  > 32): a row is G segments of nblk / G blocks; the lanes keep their partial sums across the G slots
// Arithmetic: as everywhere (Q8_K activations quantised in the prologue, integer block dots, fp32 once per block).
#pragma once
#include "gemv_bulk.cuh"

namespace ktb {

constexpr int kDenseMaxTokens = 8;
constexpr int kDenseWarps = 16;

struct DenseParams {
    const uint8_t* w;      // [rows][nblk] Q4_K blocks
    const void* x;         // [T][ncols] hidden_type
    void* out;             // [T][rows] hidden_type
    const float* bias;     // optional [rows]
    const int* bsz;
    int rows, ncols, T, hidden_type;
    int R, G, segb;        // rows per segment | segments per row | blocks per segment
    int act_tok;           // bytes of one staged activation row
};

template <int SLOTS>
__global__ void __launch_bounds__(kDenseWarps * 32, 1) dense_q4k_kernel(const DenseParams p) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    griddep_launch_dependents();
    int T = p.T;
    if (p.bsz) { griddep_wait(); T = min(T, *p.bsz); }
    const int nblk = p.ncols / QK_K;
    const int seg_bytes = p.segb * SZ_Q4_K;
    BulkRing<SLOTS> ring(smem, (size_t)p.T * p.act_tok, seg_bytes, lane, warp, W);
    // units: groups of R rows; this CTA's contiguous range, dealt round-robin to its warps
    const int nunits = (p.rows + p.R - 1) / p.R;
    const int u0 = (int)((long)nunits * blockIdx.x / gridDim.x), u1 = (int)((long)nunits * (blockIdx.x + 1) / gridDim.x);
    const int nseg = warp_units(u0, u1, warp, W) * p.G;   // slots this warp consumes
    int iu = u0 + warp, ig = 0, iss = 0;                  // issue cursor: unit, segment of the unit, slots requested
    auto issue_one = [&]() {
        if (iss < nseg) {
            const int row0 = iu * p.R;
            const int nrows = min(p.R, p.rows - row0);
            const uint32_t bytes = (uint32_t)((p.G > 1 ? p.segb : nrows * nblk) * SZ_Q4_K);
            ring.issue(lane, 1, bytes, [&](int) { return p.w + ((long)row0 * nblk + (long)ig * p.segb) * SZ_Q4_K; });
            iss++;
            if (++ig == p.G) { ig = 0; iu += W; }
        }
    };
#pragma unroll
    for (int s = 0; s < SLOTS; s++) issue_one();   // weights do not depend on the previous kernel: requested before the wait
    griddep_wait();

    stage_q8k_rows<8>(p.x, p.hidden_type, 0, T, p.ncols, smem, p.act_tok, lane, warp, W);   // as in rows_bulk_q4k_kernel
    __syncthreads();

    float acc[kDenseMaxTokens];
#pragma unroll
    for (int t = 0; t < kDenseMaxTokens; t++) acc[t] = 0.f;
    int cu = u0 + warp, cg = 0;
    for (int n = 0; n < nseg; n++) {
        const uint8_t* sl = ring.wait();
        const int row0 = cu * p.R;
        const int nrows = min(p.R, p.rows - row0);
        const int nact = p.G > 1 ? p.segb : nrows * nblk;            // blocks in this slot
        if (lane < nact) {
            const int blk = p.G > 1 ? cg * p.segb + lane : lane % nblk;   // block of the row = activation block
#pragma unroll
            for (int t = 0; t < kDenseMaxTokens; t++) {
                if (t < T) {
                    const uint8_t* at = smem + (size_t)t * p.act_tok;
                    acc[t] += q4k_block_dot(sl + lane * SZ_Q4_K, at + (size_t)blk * kActBlkStride,
                                            *reinterpret_cast<const uint4*>(at + (size_t)nblk * kActBlkStride + blk * 16),
                                            reinterpret_cast<const float*>(at + (size_t)nblk * (kActBlkStride + 16))[blk]);
                }
            }
        }
        ring.release();
        issue_one();
        if (++cg < p.G) continue;
        cg = 0;
        // the unit is complete: reduce and store
        if (p.R == 1) {
#pragma unroll
            for (int t = 0; t < kDenseMaxTokens; t++) {
                if (t < T) {
                    float v = warp_sum(acc[t]);
                    if (lane == 0) {
                        if (p.bias) v += p.bias[row0];
                        store_hidden(p.out, (long)t * p.rows + row0, p.hidden_type, v);
                    }
                }
                acc[t] = 0.f;
            }
        } else {
            const int r = lane / nblk, j0 = r * nblk;
#pragma unroll
            for (int t = 0; t < kDenseMaxTokens; t++) {
                if (t < T) {
                    float v = 0.f;
                    for (int j = 0; j < nblk; j++) v += __shfl_sync(0xffffffffu, acc[t], (j0 + j) & 31);   // ascending block order
                    if (lane == j0 && r < nrows) {
                        if (p.bias) v += p.bias[row0 + r];
                        store_hidden(p.out, (long)t * p.rows + row0 + r, p.hidden_type, v);
                    }
                }
                acc[t] = 0.f;
            }
        }
        cu += W;
    }
}

}  // namespace ktb
