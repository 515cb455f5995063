// RAWINT4_G32 routed experts: symmetric INT4 weights in groups of 32 with bf16 scales (compressed-tensors
// "pack-quantized", the format Kimi-K2 ships its experts in), W4A16 arithmetic on the bulk-copy ring of gemv_bulk.cuh.
//
// Device block (KTB200_TYPE_RAWINT4_G32, 144 B per 256 values of a row, 16-byte aligned like Q4_K):
//   bytes 0..15         the eight bf16 group scales s_0..s_7
//   bytes 16+16j..31+16j group j: four little-endian 32-bit words, word w holds columns 8w..8w+7 of the group,
//                        column 8w+i in bits 4i..4i+3, stored as u = q + 8 (u in 0..15)
// The group words are compressed-tensors' `weight_packed` words unchanged, so the pack is a copy with the scales
// interleaved.  Value = (u - 8) * s.
//
// Arithmetic (DESIGN.md §2): activations stay in fp32 (bf16 / fp16 inputs convert exactly), each group sums (u - 8) * x
// in fp32, the group sum is multiplied by s and added into the fp32 row sum.  No activation quantisation.
//
// Nibble -> float without I2F (the kernels have ~5.6 lane-instructions per weight value before they become issue-bound
// rather than HBM-bound): OR-ing a nibble that sits at bits 4p..4p+3 into the mantissa of 2^23 gives the float
// 2^23 + u * 16^p exactly, and one FADD of -(2^23 + 8 * 16^p) gives (u - 8) * 16^p exactly.  Bits 0..19 of a word hold
// nibbles 0..4 (p = 0..4); one shift by 12 brings nibbles 5..7 to p = 2..4.  Every p has its own accumulator, and the
// accumulators are combined with exact power-of-two factors 16^-p once per group.  Per word: 1 SHF + 8 LOP3 + 8 FADD +
// 8 FFMA = 25 instructions for 8 values (the mask-and-OR is one LOP3 only with the magic in a register: i4_magic).
#pragma once
#include "gemv_bulk.cuh"

namespace ktb {

constexpr int kI4ActStride = QK_K * 4 + 16;   // fp32 activation block padded to 1040 B: lanes on different blocks hit distinct banks
constexpr int kI4MaxChunkTokens = 8;

// 0x4b000000 (the bits of 2^23) in a register: with the mask as the one immediate, (w & mask) | magic is ONE LOP3 (the
// compiler splits it into two when both constants are immediates)
__device__ __forceinline__ uint32_t i4_magic() {
    uint32_t r;
    asm volatile("mov.b32 %0, 0x4b000000;" : "=r"(r));
    return r;
}
// (u - 8) * 16^P for the nibble at bits 4P..4P+3 of w (P <= 4)
template <int P>
__device__ __forceinline__ float i4_nib(uint32_t w, uint32_t magic) {
    constexpr float kBias = 8388608.0f + 8.0f * (float)(1u << (4 * P));
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(r) : "r"(w), "n"(0xfu << (4 * P)), "r"(magic));   // (w & mask) | magic
    return __uint_as_float(r) - kBias;
}

// One 32-value group of NM weight rows that share the activations: q[m] = the group's four words of row m, x = its 32
// fp32 activations (shared memory, 16-byte aligned).  Returns sum_i (u_i - 8) * x_i per row.
template <int NM>
__device__ __forceinline__ void i4_group_dot(const uint4 (&q)[NM], const float* x, uint32_t magic, float (&out)[NM]) {
    float a[NM][5];
#pragma unroll
    for (int m = 0; m < NM; m++)
#pragma unroll
        for (int p = 0; p < 5; p++) a[m][p] = 0.f;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const float4 xa = *reinterpret_cast<const float4*>(x + 8 * k);
        const float4 xb = *reinterpret_cast<const float4*>(x + 8 * k + 4);
#pragma unroll
        for (int m = 0; m < NM; m++) {
            const uint32_t w = k == 0 ? q[m].x : k == 1 ? q[m].y : k == 2 ? q[m].z : q[m].w;
            const uint32_t h = w >> 12;
            a[m][0] = __fmaf_rn(i4_nib<0>(w, magic), xa.x, a[m][0]);
            a[m][1] = __fmaf_rn(i4_nib<1>(w, magic), xa.y, a[m][1]);
            a[m][2] = __fmaf_rn(i4_nib<2>(w, magic), xa.z, a[m][2]);
            a[m][3] = __fmaf_rn(i4_nib<3>(w, magic), xa.w, a[m][3]);
            a[m][4] = __fmaf_rn(i4_nib<4>(w, magic), xb.x, a[m][4]);
            a[m][2] = __fmaf_rn(i4_nib<2>(h, magic), xb.y, a[m][2]);
            a[m][3] = __fmaf_rn(i4_nib<3>(h, magic), xb.z, a[m][3]);
            a[m][4] = __fmaf_rn(i4_nib<4>(h, magic), xb.w, a[m][4]);
        }
    }
#pragma unroll
    for (int m = 0; m < NM; m++) {   // the factors 16^-p are exact: each FMA rounds once, like an add
        float s = __fmaf_rn(a[m][4], 1.0f / 65536.0f, a[m][3] * (1.0f / 4096.0f));
        s = __fmaf_rn(a[m][2], 1.0f / 256.0f, s);
        s = __fmaf_rn(a[m][1], 1.0f / 16.0f, s);
        out[m] = s + a[m][0];
    }
}

__device__ __forceinline__ float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }

// NM super-blocks (144 B each, shared memory) against the same 256 fp32 activations: acc[m] += row m's dot
template <int NM>
__device__ __forceinline__ void i4_block_dot(const uint8_t* const (&wb)[NM], const float* xb, float (&acc)[NM]) {
    const uint32_t magic = i4_magic();
    uint4 hdr[NM];
#pragma unroll
    for (int m = 0; m < NM; m++) hdr[m] = *reinterpret_cast<const uint4*>(wb[m]);
#pragma unroll
    for (int j = 0; j < 8; j++) {
        uint4 q[NM];
#pragma unroll
        for (int m = 0; m < NM; m++) q[m] = *reinterpret_cast<const uint4*>(wb[m] + 16 + 16 * j);
        float g[NM];
        i4_group_dot<NM>(q, xb + 32 * j, magic, g);
#pragma unroll
        for (int m = 0; m < NM; m++) {
            const uint32_t sw = (j >> 1) == 0 ? hdr[m].x : (j >> 1) == 1 ? hdr[m].y : (j >> 1) == 2 ? hdr[m].z : hdr[m].w;
            acc[m] = __fmaf_rn(g[m], (j & 1) ? bf16_hi(sw) : bf16_lo(sw), acc[m]);
        }
    }
}

// Stage rows of fp32-convertible activations into the padded layout: row r, block b at r * nblk * kI4ActStride + b *
// kI4ActStride.  src(r) = element offset of row r in `x`.
template <class SrcFn>
__device__ __forceinline__ void i4_stage(float* dst, const void* x, int hidden_type, int nrows, int ncols, SrcFn&& src) {
    const int nblk = ncols / QK_K;
    for (int r = 0; r < nrows; r++) {
        const long s0 = src(r);
        float* d = dst + (size_t)r * nblk * (kI4ActStride / 4);
        for (int c = threadIdx.x; c < ncols; c += blockDim.x)
            d[(c >> 8) * (kI4ActStride / 4) + (c & 255)] = load_hidden(x, s0 + c, hidden_type);
    }
}

// Down item format of reduce_bulk_kernel: 4 rows x nb raw super-blocks, block f at f * 144.  The fp32 intermediate rows `a`
// of a chunk's pairs are staged unchanged (not requantised), and a RAWINT4 down projection never carries the shared expert.
struct BulkI4 : BulkFmt {
    static constexpr int kBlockBytes = SZ_RAWINT4;
    static constexpr int kBs = 0;
    static constexpr bool kFp32Act = true;
    static constexpr int kActBytes = kI4ActStride;
    static constexpr bool kSharedSlot = false;
    static constexpr int kMinWarps = 1;
    // rows 0 .. n-1 of `a` (fp32), src(r) = element offset of row r, as [n][nb] padded blocks
    template <class SrcFn>
    __device__ static __forceinline__ void stage_act(uint8_t* dst, const void* a, int n, int ncols, SrcFn&& src) {
        i4_stage(reinterpret_cast<float*>(dst), a, KTB200_TYPE_F32, n, ncols, src);
    }
    __device__ static __forceinline__ float dot(const uint8_t* sl, int f, const float* xb) {
        const uint8_t* const wb[1] = {sl + f * SZ_RAWINT4};
        float v[1] = {0.f};
        i4_block_dot<1>(wb, xb, v);
        return v[0];
    }
};

// ---------------------------------------------------------------------------------------------------------------
// Gate/up rows + silu(g) * u.  One ring slot = the gate row AND the up row of one (pair, row) unit (two bulk copies on
// one mbarrier), so a lane reads its 256 activations once for both matrices.  Otherwise the work split of
// rows_bulk_q4k_kernel: ALL (token, slot) pairs of a chunk of `tc` tokens form one work list, CTA = contiguous range of
// units, warp = every W-th unit of it.
template <int SLOTS>
__global__ void __launch_bounds__(kBulkMaxWarps * 32, 1) rows_bulk_i4_kernel(const RowsParams p, int tc) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ int s_np;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    int Teff = p.ntokens;
    if (p.bsz) Teff = min(Teff, *p.bsz);
    const int nblk = p.ncols / QK_K;
    const int row_bytes = nblk * SZ_RAWINT4;
    const int act_tok = nblk * kI4ActStride;
    const int total_out = p.slots * p.rows;
    // [tc activation rows, fp32 padded] [pair list: tc*slots ints] [ring: slot = gate row | up row]
    int* pairs = reinterpret_cast<int*>(smem + (size_t)tc * act_tok);   // (token in chunk) << 8 | slot
    BulkRing<SLOTS> ring(smem, (size_t)tc * act_tok + (size_t)tc * p.slots * 4, 2 * row_bytes, lane, warp, W);

  for (int t0 = 0; t0 < Teff; t0 += tc) {
    const int nt = min(tc, Teff - t0);
    __syncthreads();
    if (threadIdx.x == 0) s_np = gateup_pairs(p, t0, nt, false, pairs);
    __syncthreads();
    const int total = s_np * p.rows;
    const int u0 = (int)((long)total * blockIdx.x / gridDim.x), u1 = (int)((long)total * (blockIdx.x + 1) / gridDim.x);
    const int nu = warp_units(u0, u1, warp, W);
    UnitCursor ic;
    if (nu > 0) ic.start(u0 + warp, p.rows);
    UnitCursor cc = ic;
    int iu = 0;

    auto issue_one = [&]() {
        if (iu < nu) {
            ring.issue(lane, 2, (uint32_t)row_bytes, [&](int c) {
                const int pr = pairs[ic.pi];
                const long e = pair_expert(p, t0 + (pr >> 8), pr & 0xff);
                return reinterpret_cast<const uint8_t*>(c ? p.w1 : p.w0) + (e * p.rows + ic.r) * row_bytes;
            });
            iu++;
            ic.step(W, p.rows);
        }
    };
#pragma unroll
    for (int s = 0; s < SLOTS; s++) issue_one();

    i4_stage(reinterpret_cast<float*>(smem), p.x, p.hidden_type, nt, p.ncols, [&](int r) { return (long)(t0 + r) * p.ncols; });
    __syncthreads();

    for (int n = 0; n < nu; n++) {
        const uint8_t* row0 = ring.wait();
        const int pr = pairs[cc.pi];
        const float* xt = reinterpret_cast<const float*>(smem + (size_t)(pr >> 8) * act_tok);
        float acc[2] = {0.f, 0.f};
        for (int blk = lane; blk < nblk; blk += 32) {
            const uint8_t* const wb[2] = {row0 + blk * SZ_RAWINT4, row0 + row_bytes + blk * SZ_RAWINT4};
            i4_block_dot<2>(wb, xt + blk * (kI4ActStride / 4), acc);
        }
        ring.release();
        issue_one();
        float g = acc[0], uu = acc[1];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            g += __shfl_xor_sync(0xffffffffu, g, o);
            uu += __shfl_xor_sync(0xffffffffu, uu, o);
        }
        if (lane == 0) {
            const long o = (long)(t0 + (pr >> 8)) * total_out + (pr & 0xff) * p.rows + cc.r;
            p.out_f32[o] = (p.use_silu ? act_silu(g) : act_relu(g)) * uu;
        }
        cc.step(W, p.rows);
    }
  }  // token chunks
}

// ---------------------------------------------------------------------------------------------------------------
// Load-time conversion: compressed-tensors weight_packed int32 [rows][cols/8] + weight_scale bf16 [rows][cols/32] ->
// device blocks.  Thread = one 16-byte chunk of the output (9 per super-block: scales, then groups 0..7).
__global__ void __launch_bounds__(256) rawint4_pack_kernel(const uint32_t* packed, const uint16_t* scale, long n_sb, int nb,
                                                           uint4* out) {
    for (long t = (long)blockIdx.x * blockDim.x + threadIdx.x; t < n_sb * 9; t += (long)gridDim.x * blockDim.x) {
        const long sb = t / 9;
        const int c = (int)(t - sb * 9);
        const long r = sb / nb, b = sb - r * nb;
        uint4 v;
        if (c == 0) {
            const uint16_t* s = scale + r * nb * 8 + b * 8;
            v.x = s[0] | ((uint32_t)s[1] << 16); v.y = s[2] | ((uint32_t)s[3] << 16);
            v.z = s[4] | ((uint32_t)s[5] << 16); v.w = s[6] | ((uint32_t)s[7] << 16);
        } else {
            const uint32_t* q = packed + r * nb * 32 + b * 32 + (c - 1) * 4;
            v.x = q[0]; v.y = q[1]; v.z = q[2]; v.w = q[3];
        }
        out[t] = v;
    }
}

}  // namespace ktb
