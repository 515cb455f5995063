// Fourth generation of the expert GEMV kernels: bulk-copy (TMA engine) staging + one lane per super-block.
//
// Why not the cp.async generation: of the ~700 warp instructions a warp spent per 8 KB unit almost
// 230 were the copy itself (16 LDGSTS per lane, each with its own 64-bit address arithmetic) plus index
// divisions — LSU/MIO time shared with the LDS of the dot product.  Here:
//
//   * every ring slot is filled by ONE `cp.async.bulk.shared.global` issued by one lane and tracked by an
//     mbarrier (expect_tx / complete_tx): no per-lane copy instructions, no LSU time for the copy;
//   * slots are one weight row (Q4_K gate/up: nblk x 144 B) or one 4-row item (down) and a warp keeps SLOTS-1
//     of them in flight while it computes on one: smaller slots -> up to 18 warps per SM (was 12);
//   * unit -> (slot, row) bookkeeping is incremental (one division per token instead of one per unit);
//   * Q6_K down tensors are re-tiled once at load time into 4-row "chunk-major" items (`repack_q6k4t`, moe.cu):
//       item = rows 4q..4q+3 of one expert, f = rw*nb + blk (nrb = 4*nb (row, block) pairs)
//       [ql: c=0..7][f][16 B] | [qh: c=0..3][f][16 B] | [scales: f][16 B] | [d: f][2 B]       (= nrb * 210 B)
//     so an item is ONE contiguous bulk copy and lane f's 16-byte loads of chunk c sit next to lane f+1's:
//     bank-conflict free without padding.  Q4_K rows need no re-tiling (144-byte blocks, 36-word stride).
//
// Arithmetic is unchanged from the earlier generations (bit-exact Q8_K activations, integer dot products, fp32
// once per super-block): see DESIGN.md §2.
//
// Kernels on this ring: rows_bulk_q4k_kernel and reduce_bulk_kernel (here; the down item formats BulkQ4K, BulkQ6K4T,
// BulkQ2K and BulkQ3K here, BulkIQ1S / BulkIQ1M / BulkIQ2XXS in iq.cuh, BulkI4 in rawint4.cuh), rows_bulk_iq_kernel (iq.cuh),
// rows_bulk_i4_kernel (rawint4.cuh) and dense_q4k_kernel (dense_bulk.cuh).  The ring, work split, work lists and Q8_K
// staging they share are in bulk_ring.cuh.
#pragma once
#include "bulk_ring.cuh"

namespace ktb {

constexpr int kBulkMaxWarps = 18;        // gate/up kernel (<= 96 registers per thread)
constexpr int kBulkMaxWarpsDown = 16;    // down kernel: 128 registers per thread, and shared memory caps it at 15 anyway

// ---------------------------------------------------------------------------------------------------------------
// One Q4_K super-block (144 B at `wb`, shared memory, 16-byte aligned) against one padded int8 activation block.
// bsv = the block's eight 32-value activation sums (int16), dxb = the activation block scale.
// `act4(i)` returns the i-th 16-byte word of the block's 256 int8 activations (from shared memory or from registers).
template <class ActFn>
__device__ __forceinline__ float q4k_block_dot_t(const uint8_t* wb, ActFn&& act4, const uint4 bsv, const float dxb) {
    const uint4 hdr = *reinterpret_cast<const uint4*>(wb);
    const float2 dm = __half22float2(*reinterpret_cast<const __half2*>(&hdr.x));
    const uint32_t scl = hdr.y & 0x3f3f3f3fu;                                          // scales 0..3
    const uint32_t mnl = hdr.z & 0x3f3f3f3fu;                                          // mins   0..3
    const uint32_t sch = (hdr.w & 0x0f0f0f0fu) | ((hdr.y >> 2) & 0x30303030u);         // scales 4..7
    const uint32_t mnh = ((hdr.w >> 4) & 0x0f0f0f0fu) | ((hdr.z >> 2) & 0x30303030u);  // mins   4..7
    int isum = 0;
#pragma unroll
    for (int g = 0; g < 4; g++) {
        const uint4 a0 = act4(4 * g), a1 = act4(4 * g + 1), a2 = act4(4 * g + 2), a3 = act4(4 * g + 3);
        const uint4 q0 = *reinterpret_cast<const uint4*>(wb + 16 + 32 * g);
        const uint4 q1 = *reinterpret_cast<const uint4*>(wb + 32 + 32 * g);
        int slo = 0, shi = 0, slo2 = 0, shi2 = 0;
        slo = dp4a_s8s8(q0.x & 0x0f0f0f0fu, a0.x, slo); slo2 = dp4a_s8s8(q0.y & 0x0f0f0f0fu, a0.y, slo2);
        slo = dp4a_s8s8(q0.z & 0x0f0f0f0fu, a0.z, slo); slo2 = dp4a_s8s8(q0.w & 0x0f0f0f0fu, a0.w, slo2);
        slo = dp4a_s8s8(q1.x & 0x0f0f0f0fu, a1.x, slo); slo2 = dp4a_s8s8(q1.y & 0x0f0f0f0fu, a1.y, slo2);
        slo = dp4a_s8s8(q1.z & 0x0f0f0f0fu, a1.z, slo); slo2 = dp4a_s8s8(q1.w & 0x0f0f0f0fu, a1.w, slo2);
        // high nibbles stay in place (x16): the sums are exact multiples of 16
        shi = dp4a_u8s8(q0.x & 0xf0f0f0f0u, a2.x, shi); shi2 = dp4a_u8s8(q0.y & 0xf0f0f0f0u, a2.y, shi2);
        shi = dp4a_u8s8(q0.z & 0xf0f0f0f0u, a2.z, shi); shi2 = dp4a_u8s8(q0.w & 0xf0f0f0f0u, a2.w, shi2);
        shi = dp4a_u8s8(q1.x & 0xf0f0f0f0u, a3.x, shi); shi2 = dp4a_u8s8(q1.y & 0xf0f0f0f0u, a3.y, shi2);
        shi = dp4a_u8s8(q1.z & 0xf0f0f0f0u, a3.z, shi); shi2 = dp4a_u8s8(q1.w & 0xf0f0f0f0u, a3.w, shi2);
        const uint32_t scw = (g < 2) ? scl : sch;
        const int sc0 = (int)((scw >> (16 * (g & 1))) & 0xff), sc1 = (int)((scw >> (16 * (g & 1) + 8)) & 0xff);
        isum += sc0 * (slo + slo2) + sc1 * ((shi + shi2) >> 4);
    }
    int msum = __dp2a_lo((int)bsv.x, (int)mnl, 0);
    msum = __dp2a_hi((int)bsv.y, (int)mnl, msum);
    msum = __dp2a_lo((int)bsv.z, (int)mnh, msum);
    msum = __dp2a_hi((int)bsv.w, (int)mnh, msum);
    return (dm.x * dxb) * (float)isum - (dm.y * dxb) * (float)msum;
}
__device__ __forceinline__ float q4k_block_dot(const uint8_t* wb, const uint8_t* aq, const uint4 bsv, const float dxb) {
    return q4k_block_dot_t(wb, [&](int i) { return *reinterpret_cast<const uint4*>(aq + 16 * i); }, bsv, dxb);
}

// ---------------------------------------------------------------------------------------------------------------
// Gate/up (PAIR) or dense (PAIR = false) rows of Q4_K tensors.  Per warp: a private ring of SLOTS row slots; the
// warp's stream of sub-units is g(u0), u(u0), g(u0+W), u(u0+W), ... (PAIR) and at any time SLOTS-1 rows are in
// flight behind the one being consumed.
//
// Tokens are processed in chunks of `tc` (launcher: as many as fit next to >= 12 rings).  Within a chunk ALL
// (token, slot) pairs this launch owns form ONE work list — expert-parallel shards and decode batches keep the ring
// streaming across tokens instead of draining it once per token — and all the chunk's activation rows are staged as
// Q8_K side by side (`act_tok` bytes each).
template <bool PAIR, int SLOTS>
__global__ void __launch_bounds__(kBulkMaxWarps * 32, 1) rows_bulk_q4k_kernel(const RowsParams p, int act_tok, int tc) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ int s_np;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    int Teff = p.ntokens;
    if (p.bsz) Teff = min(Teff, *p.bsz);
    const int nblk = p.ncols / QK_K;
    const int row_bytes = nblk * SZ_Q4_K;
    constexpr int NM = PAIR ? 2 : 1;
    const int nslots = p.slots + (p.x0 ? 1 : 0);
    const int total_out = nslots * p.rows;
    // [tc activation rows: q8 [nblk][272] | bs32 [nblk][8] int16 | dx [nblk]] [pair list: tc*nslots ints] [ring]
    int* pairs = reinterpret_cast<int*>(smem + (size_t)tc * act_tok);                 // (token in chunk) << 8 | slot
    BulkRing<SLOTS> ring(smem, (size_t)tc * act_tok + (size_t)tc * nslots * 4, row_bytes, lane, warp, W);

  for (int t0 = 0; t0 < Teff; t0 += tc) {
    const int nt = min(tc, Teff - t0);
    __syncthreads();   // previous chunk: everyone is done with the staging and the pair list (and the barriers are initialised)
    if (threadIdx.x == 0) s_np = gateup_pairs(p, t0, nt, p.x0 != nullptr, pairs);
    __syncthreads();
    const int total = s_np * p.rows;
    const int u0 = (int)((long)total * blockIdx.x / gridDim.x), u1 = (int)((long)total * (blockIdx.x + 1) / gridDim.x);
    const int nsub = warp_units(u0, u1, warp, W) * NM;
    UnitCursor ic;                                          // (pair, row) of the next unit to request
    if (nsub > 0) ic.start(u0 + warp, p.rows);
    UnitCursor cc = ic;                                     // and of the unit being consumed
    int isub = 0;                                           // rows requested

    auto issue_one = [&]() {
        if (isub < nsub) {
            const bool second = PAIR && (isub & 1);
            ring.issue(lane, 1, (uint32_t)row_bytes, [&](int) -> const uint8_t* {
                const int pr = pairs[ic.pi], s = pr & 0xff;
                if (s == p.slots) return reinterpret_cast<const uint8_t*>(second ? p.x1 : p.x0) + (long)ic.r * row_bytes;
                const long e = pair_expert(p, t0 + (pr >> 8), s);
                return reinterpret_cast<const uint8_t*>(second ? p.w1 : p.w0) + (e * p.rows + ic.r) * row_bytes;
            });
            isub++;
            if (!PAIR || !(isub & 1)) ic.step(W, p.rows);
        }
    };
#pragma unroll
    for (int s = 0; s < SLOTS; s++) issue_one();

    stage_q8k_rows<8>(p.x, p.hidden_type, t0, nt, p.ncols, smem, act_tok, lane, warp, W);
    __syncthreads();

    float acc_first = 0.f;
    for (int n = 0; n < nsub; n++) {
        const uint8_t* row0 = ring.wait();
        const int pr = pairs[cc.pi];
        const uint8_t* at = smem + (size_t)(pr >> 8) * act_tok;
        const int16_t* bs32 = reinterpret_cast<const int16_t*>(at + (size_t)nblk * kActBlkStride);
        const float* dx = reinterpret_cast<const float*>(at + (size_t)nblk * (kActBlkStride + 16));
        float acc = 0.f;
        for (int blk = lane; blk < nblk; blk += 32)
            acc += q4k_block_dot(row0 + blk * SZ_Q4_K, at + (size_t)blk * kActBlkStride,
                                 *reinterpret_cast<const uint4*>(bs32 + blk * 8), dx[blk]);
        ring.release();
        issue_one();
        if (PAIR && !(n & 1)) { acc_first = acc; continue; }
        float g = PAIR ? acc_first : acc, uu = acc;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            g += __shfl_xor_sync(0xffffffffu, g, o);
            if (PAIR) uu += __shfl_xor_sync(0xffffffffu, uu, o);
        }
        if (lane == 0) {
            const int oidx = (pr & 0xff) * p.rows + cc.r;
            const long o = (long)(t0 + (pr >> 8)) * total_out + oidx;
            if (PAIR) {
                p.out_f32[o] = (p.use_silu ? act_silu(g) : act_relu(g)) * uu;
            } else {
                if (p.bias) g += p.bias[cc.r];
                if (p.out_f32) p.out_f32[o] = g;
                if (p.out_hidden) store_hidden(p.out_hidden, o, p.hidden_type, g);
            }
        }
        cc.step(W, p.rows);
    }
  }  // token chunks
}

// ---------------------------------------------------------------------------------------------------------------
// Item formats of the down-projection kernel.  An item is 4 consecutive rows x nb super-blocks, f = rw*nb + blk.
// BulkFmt holds the defaults of these formats and of the gate/up units of rows_bulk_iq_kernel (iq.cuh).
struct BulkFmt {
    static constexpr bool kFp32Act = false;   // true: the format stages fp32 activations itself (stage_act), not Q8_K
    static constexpr bool kSharedSlot = true; // a shared expert of the format can ride in the routed launch as slot `slots`
    static constexpr int kMinWarps = 2;       // reduce_bulk_kernel: fewer warps per CTA do not launch
    static constexpr int kTableBytes = 0;     // static shared memory of the format's tables (iq.cuh)
    __device__ static __forceinline__ void stage_tables() {}
};
// staged bytes per activation block of a down item format: padded int8 block, kBs int16 sums and scale; or the fp32 block
template <class Fmt>
constexpr int act_block_bytes() {
    if constexpr (Fmt::kFp32Act) return Fmt::kActBytes;
    else return kActBlkStride + 2 * Fmt::kBs + 4;
}

struct BulkQ4K : BulkFmt {   // raw Q4_K rows: block f of the item at f*144
    static constexpr int kBlockBytes = SZ_Q4_K;
    static constexpr int kBs = 8;   // int16 activation sums per block (32-value groups)
    __device__ static __forceinline__ float dot(const uint8_t* sl, int f, int /*nrb*/, const uint8_t* aq, const int16_t* bs, float dxb) {
        return q4k_block_dot(sl + f * SZ_Q4_K, aq, *reinterpret_cast<const uint4*>(bs), dxb);
    }
};

struct BulkQ6K4T : BulkFmt {   // chunk-major 4-row tiles (see the header comment)
    static constexpr int kBlockBytes = SZ_Q6_K;
    static constexpr int kBs = 16;  // int16 activation sums per block (16-value groups)
    __device__ static __forceinline__ float dot(const uint8_t* sl, int f, int nrb, const uint8_t* aq, const int16_t* bs, float dxb) {
        const uint8_t* ql = sl + f * 16;                  // chunk c at ql + c*nrb*16
        const uint8_t* qh = sl + nrb * 128 + f * 16;      // chunk c at qh + c*nrb*16
        const uint4 scv = *reinterpret_cast<const uint4*>(sl + nrb * 192 + f * 16);
        const float d = fp16_bits_to_f32(*reinterpret_cast<const uint16_t*>(sl + nrb * 208 + f * 2));
        const uint4 bs0 = *reinterpret_cast<const uint4*>(bs);
        const uint4 bs1 = *reinterpret_cast<const uint4*>(bs + 8);
        const uint32_t scw[4] = {scv.x, scv.y, scv.z, scv.w};
        const int cs = nrb * 16;
        int isum = 0;
#pragma unroll
        for (int hh = 0; hh < 2; hh++) {
            uint32_t a[8], b[8], h[8];
            *reinterpret_cast<uint4*>(a) = *reinterpret_cast<const uint4*>(ql + (4 * hh + 0) * cs);
            *reinterpret_cast<uint4*>(a + 4) = *reinterpret_cast<const uint4*>(ql + (4 * hh + 1) * cs);
            *reinterpret_cast<uint4*>(b) = *reinterpret_cast<const uint4*>(ql + (4 * hh + 2) * cs);
            *reinterpret_cast<uint4*>(b + 4) = *reinterpret_cast<const uint4*>(ql + (4 * hh + 3) * cs);
            *reinterpret_cast<uint4*>(h) = *reinterpret_cast<const uint4*>(qh + (2 * hh + 0) * cs);
            *reinterpret_cast<uint4*>(h + 4) = *reinterpret_cast<const uint4*>(qh + (2 * hh + 1) * cs);
            int s[4][2] = {{0, 0}, {0, 0}, {0, 0}, {0, 0}};   // [quarter i][l >= 16]
#pragma unroll
            for (int i = 0; i < 4; i++) {   // the four 32-value quarters of this 128-half
                uint32_t x[8];
                *reinterpret_cast<uint4*>(x) = *reinterpret_cast<const uint4*>(aq + 128 * hh + 32 * i);
                *reinterpret_cast<uint4*>(x + 4) = *reinterpret_cast<const uint4*>(aq + 128 * hh + 32 * i + 16);
#pragma unroll
                for (int w = 0; w < 8; w++) {
                    // 6-bit value = 4 low bits from ql | 2 high bits from qh; 0..63 (the -32 is folded below)
                    uint32_t v;
                    if (i == 0) v = (a[w] & 0x0f0f0f0fu) | ((h[w] << 4) & 0x30303030u);
                    else if (i == 1) v = (b[w] & 0x0f0f0f0fu) | ((h[w] << 2) & 0x30303030u);
                    else if (i == 2) v = ((a[w] >> 4) & 0x0f0f0f0fu) | (h[w] & 0x30303030u);
                    else v = ((b[w] >> 4) & 0x0f0f0f0fu) | ((h[w] >> 2) & 0x30303030u);
                    s[i][w >> 2] = dp4a_s8s8(v, x[w], s[i][w >> 2]);
                }
            }
            // 16-value group g = 8*hh + 2*i + (l >= 16) carries scale byte g
            const uint32_t lo = scw[2 * hh], hi = scw[2 * hh + 1];
            isum += sext8(lo) * s[0][0] + sext8(lo >> 8) * s[0][1] + sext8(lo >> 16) * s[1][0] + sext8(lo >> 24) * s[1][1];
            isum += sext8(hi) * s[2][0] + sext8(hi >> 8) * s[2][1] + sext8(hi >> 16) * s[3][0] + sext8(hi >> 24) * s[3][1];
        }
        // sum (q-32) x = sum q x - 32 * sum_g sc_g * bsum_g   (dp2a: int16 bsums x int8 scales)
        int corr = __dp2a_lo((int)bs0.x, (int)scw[0], 0);
        corr = __dp2a_hi((int)bs0.y, (int)scw[0], corr);
        corr = __dp2a_lo((int)bs0.z, (int)scw[1], corr);
        corr = __dp2a_hi((int)bs0.w, (int)scw[1], corr);
        corr = __dp2a_lo((int)bs1.x, (int)scw[2], corr);
        corr = __dp2a_hi((int)bs1.y, (int)scw[2], corr);
        corr = __dp2a_lo((int)bs1.z, (int)scw[3], corr);
        corr = __dp2a_hi((int)bs1.w, (int)scw[3], corr);
        return (d * dxb) * (float)(isum - 32 * corr);
    }
};

// Raw Q2_K and Q3_K super-blocks, one per lane: the down items of reduce_bulk_kernel (4 rows x nb blocks, block f at
// f * kBlockBytes) and the gate/up formats of rows_bulk_iq_kernel (iq.cuh).  No load-time re-layout: the grouped GEMM reads the
// same tensors.  Value 128 n + 32 j + l (n < 2, j < 4, l < 32) is bits 2j..2j+1 of qs[32 n + l] and lies in 16-value group
// g = 8 n + 2 j + (l >= 16).  Integer sums per super-block are exact; the fp32 finish is the grouped GEMM's (common.cuh).
struct BulkQ2K : BulkFmt {   // {scales[16] (scale | min << 4), qs[64], d, dmin} = 84 B: 4-byte aligned
    static constexpr int kType = KTB200_TYPE_Q2_K;
    static constexpr int kBlockBytes = SZ_Q2_K;
    static constexpr int kBs = 16;          // the mins need the 16-value activation sums
    static constexpr int kNblkMultiple = 4;
    // isum = sum_g sc_g * sum q * q8 (q 0..3), msum = sum_g m_g * bsum16_g
    __device__ static __forceinline__ float block_dot(const uint8_t* wb, const uint8_t* aq, const int16_t* bs16, float dxb) {
        const uint32_t* w = reinterpret_cast<const uint32_t*>(wb);
        const uint32_t sm[4] = {w[0], w[1], w[2], w[3]};   // byte g of the 16: group g
        int isum = 0;
#pragma unroll
        for (int n = 0; n < 2; n++) {
            uint32_t q[8];
#pragma unroll
            for (int i = 0; i < 8; i++) q[i] = w[4 + 8 * n + i];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint4 a0 = *reinterpret_cast<const uint4*>(aq + 128 * n + 32 * j);
                const uint4 a1 = *reinterpret_cast<const uint4*>(aq + 128 * n + 32 * j + 16);
                int s0 = dp4a_s8s8((q[0] >> (2 * j)) & 0x03030303u, a0.x, 0);
                s0 = dp4a_s8s8((q[1] >> (2 * j)) & 0x03030303u, a0.y, s0);
                s0 = dp4a_s8s8((q[2] >> (2 * j)) & 0x03030303u, a0.z, s0);
                s0 = dp4a_s8s8((q[3] >> (2 * j)) & 0x03030303u, a0.w, s0);
                int s1 = dp4a_s8s8((q[4] >> (2 * j)) & 0x03030303u, a1.x, 0);
                s1 = dp4a_s8s8((q[5] >> (2 * j)) & 0x03030303u, a1.y, s1);
                s1 = dp4a_s8s8((q[6] >> (2 * j)) & 0x03030303u, a1.z, s1);
                s1 = dp4a_s8s8((q[7] >> (2 * j)) & 0x03030303u, a1.w, s1);
                const uint32_t scw = sm[2 * n + (j >> 1)] >> (16 * (j & 1));   // groups 8n + 2j, 8n + 2j + 1 in bytes 0, 1
                isum += (int)(scw & 0xf) * s0 + (int)((scw >> 8) & 0xf) * s1;
            }
        }
        const uint4 b0 = *reinterpret_cast<const uint4*>(bs16), b1 = *reinterpret_cast<const uint4*>(bs16 + 8);
        const uint32_t m0 = (sm[0] >> 4) & 0x0f0f0f0fu, m1 = (sm[1] >> 4) & 0x0f0f0f0fu;
        const uint32_t m2 = (sm[2] >> 4) & 0x0f0f0f0fu, m3 = (sm[3] >> 4) & 0x0f0f0f0fu;
        int msum = __dp2a_lo((int)b0.x, (int)m0, 0);
        msum = __dp2a_hi((int)b0.y, (int)m0, msum);
        msum = __dp2a_lo((int)b0.z, (int)m1, msum);
        msum = __dp2a_hi((int)b0.w, (int)m1, msum);
        msum = __dp2a_lo((int)b1.x, (int)m2, msum);
        msum = __dp2a_hi((int)b1.y, (int)m2, msum);
        msum = __dp2a_lo((int)b1.z, (int)m3, msum);
        msum = __dp2a_hi((int)b1.w, (int)m3, msum);
        const float2 dm = __half22float2(*reinterpret_cast<const __half2*>(w + 20));
        return kq_min_term(dm.x, dm.y, dxb, isum, (float)msum);
    }
    __device__ static __forceinline__ float dot(const uint8_t* sl, int f, int /*nrb*/, const uint8_t* aq, const int16_t* bs, float dxb) {
        return block_dot(sl + f * SZ_Q2_K, aq, bs, dxb);
    }
};

struct BulkQ3K : BulkFmt {   // {hmask[32], qs[64], scales[12], d} = 110 B: 2-byte aligned, 4-byte aligned on even f
    static constexpr int kType = KTB200_TYPE_Q3_K;
    static constexpr int kBlockBytes = SZ_Q3_K;
    static constexpr int kBs = 8;           // staged, not read
    static constexpr int kNblkMultiple = 4;
    // isum = sum_g (sc_g - 32) * sum (q - 4 [hmask bit clear]) * q8, the hmask term as a second dp4a on the clear bits.
    // Words are read as the grouped producer reads them: the aligned words covering the block, funnel-shifted by 16 bits when
    // the block starts mid-word.  The last word read (27) ends inside this block or the next one, which always exists: units
    // and items hold an even number of blocks.
    __device__ static __forceinline__ float block_dot(const uint8_t* wb, const uint8_t* aq, const int16_t* /*bs*/, float dxb) {
        const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(wb) & 2u) * 8u;
        const uint32_t* w = reinterpret_cast<const uint32_t*>(wb - (sh >> 3));
        auto word = [&](int i) { return __funnelshift_r(w[i], w[i + 1], sh); };
        const uint32_t s0 = word(24), s1 = word(25), s2 = word(26);
        const float d = fp16_bits_to_f32((uint16_t)(w[27] >> sh));
        // 6-bit scales of groups 4c..4c+3 in word c: low nibbles from s0 / s1, high bit pairs from s2
        const uint32_t sc[4] = {(s0 & 0x0f0f0f0fu) | ((s2 << 4) & 0x30303030u), (s1 & 0x0f0f0f0fu) | ((s2 << 2) & 0x30303030u),
                                ((s0 >> 4) & 0x0f0f0f0fu) | (s2 & 0x30303030u), ((s1 >> 4) & 0x0f0f0f0fu) | ((s2 >> 2) & 0x30303030u)};
        int isum = 0;
#pragma unroll
        for (int h = 0; h < 2; h++) {   // l < 16, l >= 16: a quarter of the words live at a time
            uint32_t nh[4];   // hmask complemented: bit 4n + j of byte l set where value 128 n + 32 j + l takes the - 4
#pragma unroll
            for (int i = 0; i < 4; i++) nh[i] = ~word(4 * h + i);
#pragma unroll
            for (int n = 0; n < 2; n++) {
                uint32_t q[4];
#pragma unroll
                for (int i = 0; i < 4; i++) q[i] = word(8 + 8 * n + 4 * h + i);
#pragma unroll
                for (int j = 0; j < 4; j++) {
                    const uint4 a = *reinterpret_cast<const uint4*>(aq + 128 * n + 32 * j + 16 * h);
                    const uint32_t ax[4] = {a.x, a.y, a.z, a.w};
                    int s = 0, t = 0;
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        s = dp4a_s8s8((q[i] >> (2 * j)) & 0x03030303u, ax[i], s);
                        t = dp4a_s8s8((nh[i] >> (4 * n + j)) & 0x01010101u, ax[i], t);
                    }
                    // group 8n + 2j + h: byte 2 (j & 1) + h of scale word 2n + (j >> 1)
                    const int sg = (int)((sc[2 * n + (j >> 1)] >> (16 * (j & 1) + 8 * h)) & 0xff) - 32;
                    isum += sg * (s - 4 * t);
                }
            }
        }
        return iq_term(d, dxb, isum);
    }
    __device__ static __forceinline__ float dot(const uint8_t* sl, int f, int /*nrb*/, const uint8_t* aq, const int16_t* bs, float dxb) {
        return block_dot(sl + f * SZ_Q3_K, aq, bs, dxb);
    }
};

// Down projection + weighted combine.  Work item of a warp = (pair, 4 consecutive output rows) = one bulk copy; every
// CTA owns a contiguous range of row quads for ALL pairs so the combine over experts stays in the CTA.
//
// Tokens are processed in chunks: as many consecutive tokens as have, together, at most `pcap` (token, slot) pairs
// owned by this launch (launcher: pcap >= slots + 1, so a chunk always holds at least one token).  Within a chunk all
// pairs form ONE work list (expert-parallel shards and decode batches do not drain the ring per token) and all their
// activation rows are staged side by side: as Q8_K, or as the format's fp32 blocks (Fmt::kFp32Act, RAWINT4).
// Fmt::kSharedSlot = false compiles the shared-expert slot out.
template <class Fmt, int SLOTS>
__global__ void __launch_bounds__(kBulkMaxWarpsDown * 32, 1) reduce_bulk_kernel(const ReduceParams p, int nrows_max, int pcap) {
    constexpr int RW = 4;
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ int s_np, s_nt;
    __shared__ int s_first[kBulkMaxChunkTokens + 1];   // first pair of every token of the chunk (+ end)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    Fmt::stage_tables();   // codebooks of the IQ formats; read only after the token loop's first __syncthreads
    int Teff = p.ntokens;
    if (p.bsz) Teff = min(Teff, *p.bsz);
    const int nb = p.ncols / QK_K;
    const int k = p.slots;
    const int ns = k + (Fmt::kSharedSlot && p.xw ? 1 : 0);
    const int nrb = RW * nb;                                  // (row, block) pairs per item
    const int item_bytes = nrb * Fmt::kBlockBytes;
    // staging: activations [pcap][nb] | partial [nrows_max][pcap] | pair list [pcap] | ring.  Q8_K activations are
    // q8 [pcap][nb][272] | bs [pcap][nb][kBs] int16 | dx [pcap][nb]; fp32 ones [pcap][nb][Fmt::kActBytes].
    const size_t nab = (size_t)pcap * nb;
    uint8_t* q8 = smem;
    int16_t* bs = reinterpret_cast<int16_t*>(smem + nab * kActBlkStride);
    float* dx = reinterpret_cast<float*>(smem + nab * (kActBlkStride + 2 * Fmt::kBs));
    float* partial = reinterpret_cast<float*>(smem + nab * act_block_bytes<Fmt>());
    int* pairs = reinterpret_cast<int*>(partial + (size_t)nrows_max * pcap);   // (token in chunk) << 8 | slot
    BulkRing<SLOTS> ring(smem, nab * act_block_bytes<Fmt>() + (size_t)nrows_max * pcap * 4 + (size_t)pcap * 4, item_bytes,
                         lane, warp, W);
    const int quads = p.rows / RW;
    const int q0 = (int)((long)quads * blockIdx.x / gridDim.x), q1 = (int)((long)quads * (blockIdx.x + 1) / gridDim.x);
    const int r0 = q0 * RW, nquads = q1 - q0, nrows = nquads * RW;

  for (int t0 = 0; t0 < Teff;) {
    __syncthreads();
    if (threadIdx.x == 0) {
        int np;
        s_nt = down_pairs(p, t0, Teff, pcap, Fmt::kSharedSlot && p.xw, pairs, s_first, np);
        s_np = np;
    }
    __syncthreads();
    const int np = s_np, nt = s_nt;
    const int ni = warp_units(0, nquads * np, warp, W);   // item = pair * nquads + quad
    UnitCursor ic;
    if (ni > 0) ic.start(warp, nquads);
    UnitCursor cc = ic;
    int iss = 0;

    auto issue_one = [&]() {
        if (iss < ni) {
            ring.issue(lane, 1, (uint32_t)item_bytes, [&](int) {
                const int pr = pairs[ic.pi], j = pr & 0xff;
                long row = r0 + ic.r * RW;
                const uint8_t* wbase = reinterpret_cast<const uint8_t*>(p.w);
                if (Fmt::kSharedSlot && j == k) wbase = reinterpret_cast<const uint8_t*>(p.xw);
                else row += pair_expert(p, t0 + (pr >> 8), j) * p.rows;
                return wbase + (row >> 2) * item_bytes;
            });
            iss++;
            ic.step(W, nquads);
        }
    };
#pragma unroll
    for (int s = 0; s < SLOTS; s++) issue_one();

    // the pairs' activation rows (fp32 phase-1 output)
    auto src_row = [&](int pi) {
        const int pr = pairs[pi];
        return ((long)(t0 + (pr >> 8)) * ns + (pr & 0xff)) * p.ncols;
    };
    if constexpr (Fmt::kFp32Act) {
        Fmt::stage_act(smem, p.a, np, p.ncols, src_row);
    } else {   // block g = (pair, block)
        stage_q8k<Fmt::kBs>(
            p.a, KTB200_TYPE_F32, np * nb, lane, warp, W,
            [&](int g) {
                const int pi = g / nb, b = g - pi * nb;
                return src_row(pi) + (long)b * QK_K;
            },
            [&](int g) { return StagedBlock{q8 + (size_t)g * kActBlkStride, bs + g * Fmt::kBs, dx + g}; });
    }
    __syncthreads();

    for (int n = 0; n < ni; n++) {
        const uint8_t* sl = ring.wait();
        float res;
        {
            float acc[RW] = {0.f, 0.f, 0.f, 0.f};
            for (int f = lane; f < nrb; f += 32) {   // (row, block) pairs of the tile; 4 x 8 = one per lane for I = 2048
                const int rw = f / nb, blk = f - rw * nb;
                const int ab = cc.pi * nb + blk;
                float val;
                if constexpr (Fmt::kFp32Act)
                    val = Fmt::dot(sl, f, reinterpret_cast<const float*>(smem) + (size_t)ab * (Fmt::kActBytes / 4));
                else
                    val = Fmt::dot(sl, f, nrb, q8 + (size_t)ab * kActBlkStride, bs + ab * Fmt::kBs, dx[ab]);
                acc[0] += rw == 0 ? val : 0.f; acc[1] += rw == 1 ? val : 0.f; acc[2] += rw == 2 ? val : 0.f; acc[3] += rw == 3 ? val : 0.f;
            }
            res = warp_reduce4(acc[0], acc[1], acc[2], acc[3], lane);
        }
        ring.release();
        issue_one();
        if ((lane & 7) == 0) partial[(cc.r * RW + (lane >> 3)) * pcap + cc.pi] = res;
        cc.step(W, nquads);
    }
    __syncthreads();
    // weighted accumulation over a token's experts IN expert_ids ORDER (moe.cpp:222-236), one FMA per expert
    for (int idx = threadIdx.x; idx < nrows * nt; idx += W * 32) {
        const int tl = idx / nrows, hl = idx - tl * nrows;
        const long t = t0 + tl;
        float acc = 0.f, shared = 0.f;
        for (int pi = s_first[tl]; pi < s_first[tl + 1]; pi++) {
            const int j = pairs[pi] & 0xff;
            const float dv = partial[hl * pcap + pi];
            if (Fmt::kSharedSlot && j == k) shared = dv;
            else acc = p.weights ? __fmaf_rn(dv, p.weights[t * k + j], acc) : acc + dv;
        }
        const long o = t * p.rows + r0 + hl;
        if constexpr (Fmt::kSharedSlot) {
            bool has_sh = false;
            for (int pi = s_first[tl]; pi < s_first[tl + 1]; pi++) has_sh |= (pairs[pi] & 0xff) == k;
            if (p.xw_out) { if (has_sh) store_hidden(p.xw_out, o, p.xw_out_type, shared); }
            else if (p.xw) acc = round_hidden(acc, p.hidden_type) + round_hidden(shared, p.hidden_type);
        }
        if (p.accumulate) acc = load_hidden(p.out, o, p.hidden_type) + round_hidden(acc, p.hidden_type);
        store_hidden(p.out, o, p.hidden_type, acc);
    }
    t0 += nt;
  }  // token chunks
}

}  // namespace ktb
