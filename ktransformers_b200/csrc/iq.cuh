// IQ1_S, IQ1_M, IQ2_XXS, IQ2_XS, IQ2_S, IQ3_XXS and IQ3_S routed experts on the bulk-copy ring (gemv_bulk.cuh): one lane per
// super-block, codebooks in shared memory.  IQ1_M (56-byte blocks, 8-byte aligned) takes every block count: its unit is
// 112 * nblk B and its item 224 * nb B, so its launches skip the nblk % 4 (kNblkMultiple) condition of the 50 / 66 / 74 / 82 /
// 98 / 110-byte formats.  IQ3_S blocks are Q3_K's size (110 B), so its units and items are Q3_K's; IQ3_XXS's 98-byte blocks
// give 196 * nblk B units (16-byte sized when nblk % 4 == 0) and 392 * nb B items (when nb is even); IQ2_XS / IQ2_S likewise
// 148 / 164 * nblk B units and 296 / 328 * nb B items.
//
//   * down: item formats BulkIQ1S / BulkIQ2XXS of reduce_bulk_kernel — 4 rows x nb raw ggml blocks, one bulk copy
//     (4 * nb * 50 B / 4 * nb * 66 B, a multiple of 16 when nb is even; 1600 B / 2112 B at I = 2048 = one block per lane);
//   * gate/up: rows_bulk_iq_kernel.  A row is nblk * 50 B (IQ1_S) or nblk * 66 B (IQ2_XXS): 1400 B / 1848 B at H = 7168,
//     not a multiple of 16, so a single row cannot be one bulk copy.  The unit is two consecutive rows (2800 B / 3696 B,
//     16-byte aligned when nblk % 4 == 0): one ring slot holds the gate rows 2r, 2r+1 and the up rows 2r, 2r+1 (two copies
//     on one mbarrier), so one read of x serves both matrices and the raw GGUF bytes are used as they are.  The same kernel
//     takes Q2_K and Q3_K gate/up (formats BulkQ2K / BulkQ3K, gemv_bulk.cuh): 168 B / 220 B per block pair of a unit.
//
// Codebooks: IQ1_S's (and IQ1_M's) 2048 x 8 int8 grid as 16 KB of uint2 (one LDS.64 per 8 values, no unpacking); IQ2_XXS's 256 x 8
// grid (2 KB) and its 128 sign patterns expanded to byte masks (1 KB: value = (g ^ m) - m per byte); IQ2_XS's 512 x 8 grid
// (4 KB) with IQ2_XXS's sign masks; IQ2_S's 1024 x 8 grid (8 KB) with IQ3_S's sign-byte masks; IQ3_XXS's 256 x 4 grid (1 KB)
// with IQ2_XXS's sign masks; IQ3_S's 512 x 4 grid (2 KB) and its 256 sign bytes as byte masks (2 KB).  All are copied from the
// device tables of iq_tables.h / iq2_tables.h / iq3_tables.h once per CTA.
//
// Arithmetic (DESIGN.md §2): IQ1_S  S = sum_ib ls * (8 * sum grid * q8 + delta * bsum32) and term = ((d/8) * dx) * S;
// IQ2_XXS  term = ((d/8) * dx) * sum_ib ls * sum (+-grid) * q8; IQ2_XS / IQ2_S the same with ls per 16 values; IQ3_XXS the
// same as IQ2_XXS with d/4, IQ3_S with d.  All equal the reference's per-super-block fp32 terms.
#pragma once
#include "gemv_bulk.cuh"

namespace ktb {

__device__ __forceinline__ uint2* iq1s_grid_smem() { __shared__ uint2 t[2048]; return t; }
__device__ __forceinline__ uint2* iq2xxs_grid_smem() { __shared__ uint2 t[256]; return t; }
__device__ __forceinline__ uint2* iq2xxs_signs_smem() { __shared__ uint2 t[128]; return t; }
__device__ __forceinline__ uint32_t* iq3xxs_grid_smem() { __shared__ uint32_t t[256]; return t; }
__device__ __forceinline__ uint32_t* iq3s_grid_smem() { __shared__ uint32_t t[512]; return t; }
__device__ __forceinline__ uint2* iq3s_signs_smem() { __shared__ uint2 t[256]; return t; }
__device__ __forceinline__ uint2* iq2xs_grid_smem() { __shared__ uint2 t[512]; return t; }
__device__ __forceinline__ uint2* iq2s_grid_smem() { __shared__ uint2 t[1024]; return t; }

// 32 bits from a 2-byte aligned shared-memory address
__device__ __forceinline__ uint32_t lds_u32_a2(const uint8_t* p) {
    const uint16_t* h = reinterpret_cast<const uint16_t*>(p);
    return (uint32_t)h[0] | ((uint32_t)h[1] << 16);
}

struct BulkIQ1S : BulkFmt {
    static constexpr int kType = KTB200_TYPE_IQ1_S;
    static constexpr int kBlockBytes = SZ_IQ1_S;
    static constexpr int kBs = 8;            // int16 activation sums per block (32-value groups)
    static constexpr int kTableBytes = 2048 * 8;
    static constexpr bool kSharedSlot = false;   // shared experts are never i-quants (MLPs take K-quants only)
    static constexpr int kNblkMultiple = 4;      // rows_bulk_iq_kernel: blocks per row for a 2-row unit of 16-byte size
    __device__ static __forceinline__ void stage_tables() {
        uint2* g = iq1s_grid_smem();
        for (int i = threadIdx.x; i < 2048; i += blockDim.x) g[i] = *reinterpret_cast<const uint2*>(ktb_iq1s_grid[i]);
    }
    // one super-block at `wb` (shared memory, 2-byte aligned) against one padded int8 activation block
    __device__ static __forceinline__ float block_dot(const uint8_t* wb, const uint8_t* aq, const int16_t* bs32, float dxb) {
        const uint2* grid = iq1s_grid_smem();
        const float d = iq_d8(*reinterpret_cast<const uint16_t*>(wb));
        int isum = 0;
#pragma unroll
        for (int ib = 0; ib < 8; ib++) {
            const uint32_t qh = *reinterpret_cast<const uint16_t*>(wb + 34 + 2 * ib);
            const uint32_t qs = lds_u32_a2(wb + 2 + 4 * ib);
            const uint4 a0 = *reinterpret_cast<const uint4*>(aq + 32 * ib);
            const uint4 a1 = *reinterpret_cast<const uint4*>(aq + 32 * ib + 16);
            const uint2 g0 = grid[(qs & 0xff) | ((qh << 8) & 0x700)];
            const uint2 g1 = grid[((qs >> 8) & 0xff) | ((qh << 5) & 0x700)];
            const uint2 g2 = grid[((qs >> 16) & 0xff) | ((qh << 2) & 0x700)];
            const uint2 g3 = grid[(qs >> 24) | ((qh >> 1) & 0x700)];
            int s = dp4a_s8s8(g0.x, a0.x, 0);
            s = dp4a_s8s8(g0.y, a0.y, s);
            s = dp4a_s8s8(g1.x, a0.z, s);
            s = dp4a_s8s8(g1.y, a0.w, s);
            s = dp4a_s8s8(g2.x, a1.x, s);
            s = dp4a_s8s8(g2.y, a1.y, s);
            s = dp4a_s8s8(g3.x, a1.z, s);
            s = dp4a_s8s8(g3.y, a1.w, s);
            const int b = bs32[ib];
            const int ls = 2 * (int)((qh >> 12) & 7) + 1;
            isum += ls * (8 * s + ((qh & 0x8000u) ? -b : b));
        }
        return iq_term(d, dxb, isum);
    }
    __device__ static __forceinline__ float dot(const uint8_t* sl, int f, int /*nrb*/, const uint8_t* aq, const int16_t* bs, float dxb) {
        return block_dot(sl + f * SZ_IQ1_S, aq, bs, dxb);
    }
};

// IQ1_S's codebook with the scale per 16 values and the delta per 8.  The Q8_K sums cover 16 or 32 values, so the delta term is
// summed per 8-value group: dp4a of the group's activations against 0x01010101 (+1) or 0xffffffff (-1).  56-byte blocks are
// 8-byte aligned: words and the 8-byte scale field load whole.
struct BulkIQ1M : BulkFmt {
    static constexpr int kType = KTB200_TYPE_IQ1_M;
    static constexpr int kBlockBytes = SZ_IQ1_M;
    static constexpr int kBs = 8;            // staged, not read
    static constexpr int kTableBytes = 2048 * 8;
    static constexpr bool kSharedSlot = false;
    static constexpr int kNblkMultiple = 1;  // a 2-row unit is 112 * nblk B
    __device__ static __forceinline__ void stage_tables() { BulkIQ1S::stage_tables(); }
    // S = sum_h ls_h * sum_(8-groups l of h) (8 * sum grid * q8 + delta_l * sum q8); term = ((d/8) * dx) * S
    __device__ static __forceinline__ float block_dot(const uint8_t* wb, const uint8_t* aq, const int16_t* /*bs*/, float dxb) {
        const uint2* grid = iq1s_grid_smem();
        const uint2 sc = *reinterpret_cast<const uint2*>(wb + 48);
        const float d = iq_d8(iq1m_d_bits(sc.x, sc.y));
        int isum = 0;
#pragma unroll
        for (int ib = 0; ib < 8; ib++) {
            const uint32_t qs = *reinterpret_cast<const uint32_t*>(wb + 4 * ib);
            const uint32_t qh = *reinterpret_cast<const uint16_t*>(wb + 32 + 2 * ib);   // nibble l (group 4 ib + l) at bits 4 l
            const uint32_t sw = (ib < 4 ? sc.x : sc.y) >> (16 * ((ib >> 1) & 1) + 6 * (ib & 1));   // ls of the halves: bits 0-2, 3-5
            const uint4 a0 = *reinterpret_cast<const uint4*>(aq + 32 * ib);
            const uint4 a1 = *reinterpret_cast<const uint4*>(aq + 32 * ib + 16);
            const uint32_t ax[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            int v[2] = {0, 0};
#pragma unroll
            for (int l = 0; l < 4; l++) {
                const uint2 g = grid[((qs >> (8 * l)) & 0xff) | (((qh >> (4 * l)) & 7) << 8)];
                const uint32_t m = ((qh >> (4 * l + 3)) & 1) ? 0xffffffffu : 0x01010101u;
                int s = dp4a_s8s8(g.x, ax[2 * l], 0);
                s = dp4a_s8s8(g.y, ax[2 * l + 1], s);
                int t = dp4a_s8s8(m, ax[2 * l], 0);
                t = dp4a_s8s8(m, ax[2 * l + 1], t);
                v[l >> 1] += 8 * s + t;
            }
            isum += (2 * (int)(sw & 7) + 1) * v[0] + (2 * (int)((sw >> 3) & 7) + 1) * v[1];
        }
        return iq_term(d, dxb, isum);
    }
    __device__ static __forceinline__ float dot(const uint8_t* sl, int f, int /*nrb*/, const uint8_t* aq, const int16_t* bs, float dxb) {
        return block_dot(sl + f * SZ_IQ1_M, aq, bs, dxb);
    }
};

struct BulkIQ2XXS : BulkFmt {
    static constexpr int kType = KTB200_TYPE_IQ2_XXS;
    static constexpr int kBlockBytes = SZ_IQ2_XXS;
    static constexpr int kBs = 8;
    static constexpr int kTableBytes = 256 * 8 + 128 * 8;
    static constexpr bool kSharedSlot = false;
    static constexpr int kNblkMultiple = 4;
    __device__ static __forceinline__ void stage_tables() {
        uint2* g = iq2xxs_grid_smem();
        uint2* m = iq2xxs_signs_smem();
        for (int i = threadIdx.x; i < 256; i += blockDim.x) g[i] = *reinterpret_cast<const uint2*>(ktb_iq2xxs_grid[i]);
        for (int i = threadIdx.x; i < 128; i += blockDim.x) m[i] = iq2_sign_masks(ktb_ksigns_iq2xs[i]);
    }
    __device__ static __forceinline__ float block_dot(const uint8_t* wb, const uint8_t* aq, const int16_t* /*bs32*/, float dxb) {
        const uint2* grid = iq2xxs_grid_smem();
        const uint2* sgn = iq2xxs_signs_smem();
        const float d = iq_d8(*reinterpret_cast<const uint16_t*>(wb));
        int isum = 0;
#pragma unroll
        for (int ib = 0; ib < 8; ib++) {
            const uint32_t aux0 = lds_u32_a2(wb + 2 + 8 * ib), aux1 = lds_u32_a2(wb + 6 + 8 * ib);
            const uint4 a0 = *reinterpret_cast<const uint4*>(aq + 32 * ib);
            const uint4 a1 = *reinterpret_cast<const uint4*>(aq + 32 * ib + 16);
            const uint32_t ax[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            int s = 0;
#pragma unroll
            for (int l = 0; l < 4; l++) {
                const uint2 g = grid[(aux0 >> (8 * l)) & 0xff];
                const uint2 m = sgn[(aux1 >> (7 * l)) & 127];
                s = dp4a_s8s8(__vsub4(g.x ^ m.x, m.x), ax[2 * l], s);
                s = dp4a_s8s8(__vsub4(g.y ^ m.y, m.y), ax[2 * l + 1], s);
            }
            isum += (2 * (int)(aux1 >> 28) + 1) * s;
        }
        return iq_term(d, dxb, isum);
    }
    __device__ static __forceinline__ float dot(const uint8_t* sl, int f, int /*nrb*/, const uint8_t* aq, const int16_t* bs, float dxb) {
        return block_dot(sl + f * SZ_IQ2_XXS, aq, bs, dxb);
    }
};

// IQ2_XXS's sub-block form with 4-value groups: eight 8-bit indices into the 256 x 4 grid (values 4..62) and one word of four
// 7-bit sign indices and the 4-bit scale.  The sign masks are IQ2_XXS's shared-memory table; term = ((d/4) * dx) * S.
struct BulkIQ3XXS : BulkFmt {
    static constexpr int kType = KTB200_TYPE_IQ3_XXS;
    static constexpr int kBlockBytes = SZ_IQ3_XXS;
    static constexpr int kBs = 8;            // staged, not read
    static constexpr int kTableBytes = 256 * 4 + 128 * 8;
    static constexpr bool kSharedSlot = false;
    static constexpr int kNblkMultiple = 4;  // a 2-row unit is 196 * nblk B
    __device__ static __forceinline__ void stage_tables() {
        uint32_t* g = iq3xxs_grid_smem();
        uint2* m = iq2xxs_signs_smem();
        for (int i = threadIdx.x; i < 256; i += blockDim.x) g[i] = *reinterpret_cast<const uint32_t*>(ktb_iq3xxs_grid[i]);
        for (int i = threadIdx.x; i < 128; i += blockDim.x) m[i] = iq2_sign_masks(ktb_ksigns_iq2xs[i]);
    }
    __device__ static __forceinline__ float block_dot(const uint8_t* wb, const uint8_t* aq, const int16_t* /*bs*/, float dxb) {
        const uint32_t* grid = iq3xxs_grid_smem();
        const uint2* sgn = iq2xxs_signs_smem();
        const float d = iq_d4(*reinterpret_cast<const uint16_t*>(wb));
        int isum = 0;
#pragma unroll
        for (int ib = 0; ib < 8; ib++) {
            const uint32_t q[2] = {lds_u32_a2(wb + 2 + 8 * ib), lds_u32_a2(wb + 6 + 8 * ib)};
            const uint32_t aux = lds_u32_a2(wb + 66 + 4 * ib);
            const uint4 a0 = *reinterpret_cast<const uint4*>(aq + 32 * ib);
            const uint4 a1 = *reinterpret_cast<const uint4*>(aq + 32 * ib + 16);
            const uint32_t ax[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            int s = 0;
#pragma unroll
            for (int l = 0; l < 4; l++) {   // 8 values: 4-value groups 2l, 2l + 1 (bytes 2l, 2l + 1 of the sub-block's qs)
                const uint32_t g0 = grid[(q[l >> 1] >> (16 * (l & 1))) & 0xff], g1 = grid[(q[l >> 1] >> (16 * (l & 1) + 8)) & 0xff];
                const uint2 m = sgn[(aux >> (7 * l)) & 127];
                s = dp4a_s8s8(__vsub4(g0 ^ m.x, m.x), ax[2 * l], s);
                s = dp4a_s8s8(__vsub4(g1 ^ m.y, m.y), ax[2 * l + 1], s);
            }
            isum += (2 * (int)(aux >> 28) + 1) * s;
        }
        return iq_term(d, dxb, isum);
    }
    __device__ static __forceinline__ float dot(const uint8_t* sl, int f, int /*nrb*/, const uint8_t* aq, const int16_t* bs, float dxb) {
        return block_dot(sl + f * SZ_IQ3_XXS, aq, bs, dxb);
    }
};

// 9-bit indices into the 512 x 4 grid (values 1..15: qs byte | qh bit), one sign bit per value, a 4-bit scale per 32 values.
// The sign bytes become byte masks through a 256 x 8 B shared-memory table (one LDS.64 per 8 values, as IQ2_XXS); term =
// (d * dx) * S.  110-byte blocks: Q3_K's size, so its units, items and alignment conditions.
struct BulkIQ3S : BulkFmt {
    static constexpr int kType = KTB200_TYPE_IQ3_S;
    static constexpr int kBlockBytes = SZ_IQ3_S;
    static constexpr int kBs = 8;            // staged, not read
    static constexpr int kTableBytes = 512 * 4 + 256 * 8;
    static constexpr bool kSharedSlot = false;
    static constexpr int kNblkMultiple = 4;  // a 2-row unit is 220 * nblk B
    __device__ static __forceinline__ void stage_tables() {
        uint32_t* g = iq3s_grid_smem();
        uint2* m = iq3s_signs_smem();
        for (int i = threadIdx.x; i < 512; i += blockDim.x) g[i] = *reinterpret_cast<const uint32_t*>(ktb_iq3s_grid[i]);
        for (int i = threadIdx.x; i < 256; i += blockDim.x) m[i] = iq2_sign_masks(i);
    }
    __device__ static __forceinline__ float block_dot(const uint8_t* wb, const uint8_t* aq, const int16_t* /*bs*/, float dxb) {
        const uint32_t* grid = iq3s_grid_smem();
        const uint2* sgn = iq3s_signs_smem();
        const float d = fp16_bits_to_f32(*reinterpret_cast<const uint16_t*>(wb));
        const uint32_t sc = lds_u32_a2(wb + 106);   // scale of sub-block ib: bits 4 ib .. 4 ib + 3
        int isum = 0;
#pragma unroll
        for (int ib = 0; ib < 8; ib++) {
            const uint32_t q[2] = {lds_u32_a2(wb + 2 + 8 * ib), lds_u32_a2(wb + 6 + 8 * ib)};
            const uint32_t qh = wb[66 + ib];
            const uint32_t sg = lds_u32_a2(wb + 74 + 4 * ib);   // byte l: the signs of values 8l..8l+7
            const uint4 a0 = *reinterpret_cast<const uint4*>(aq + 32 * ib);
            const uint4 a1 = *reinterpret_cast<const uint4*>(aq + 32 * ib + 16);
            const uint32_t ax[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            int s = 0;
#pragma unroll
            for (int l = 0; l < 4; l++) {
                const uint32_t w = q[l >> 1] >> (16 * (l & 1));
                const uint32_t g0 = grid[(w & 0xff) | ((qh << (8 - 2 * l)) & 0x100)];
                const uint32_t g1 = grid[((w >> 8) & 0xff) | ((qh << (7 - 2 * l)) & 0x100)];
                const uint2 m = sgn[(sg >> (8 * l)) & 0xff];
                s = dp4a_s8s8(__vsub4(g0 ^ m.x, m.x), ax[2 * l], s);
                s = dp4a_s8s8(__vsub4(g1 ^ m.y, m.y), ax[2 * l + 1], s);
            }
            isum += (2 * (int)((sc >> (4 * ib)) & 15) + 1) * s;
        }
        return iq_term(d, dxb, isum);
    }
    __device__ static __forceinline__ float dot(const uint8_t* sl, int f, int /*nrb*/, const uint8_t* aq, const int16_t* bs, float dxb) {
        return block_dot(sl + f * SZ_IQ3_S, aq, bs, dxb);
    }
};

// IQ2_XXS's values with a 9-bit grid index per 8 values (one uint16: index | 7-bit sign index << 9) into the 512 x 8 grid and
// one scale per 16 values (two nibbles per sub-block byte, low first).  The two 16-value halves of a sub-block are summed
// apart and scaled by their own ls, as IQ1_M; term = ((d/8) * dx) * S.
struct BulkIQ2XS : BulkFmt {
    static constexpr int kType = KTB200_TYPE_IQ2_XS;
    static constexpr int kBlockBytes = SZ_IQ2_XS;
    static constexpr int kBs = 8;            // staged, not read
    static constexpr int kTableBytes = 512 * 8 + 128 * 8;
    static constexpr bool kSharedSlot = false;
    static constexpr int kNblkMultiple = 4;  // a 2-row unit is 148 * nblk B
    __device__ static __forceinline__ void stage_tables() {
        uint2* g = iq2xs_grid_smem();
        uint2* m = iq2xxs_signs_smem();
        for (int i = threadIdx.x; i < 512; i += blockDim.x) g[i] = *reinterpret_cast<const uint2*>(ktb_iq2xs_grid[i]);
        for (int i = threadIdx.x; i < 128; i += blockDim.x) m[i] = iq2_sign_masks(ktb_ksigns_iq2xs[i]);
    }
    __device__ static __forceinline__ float block_dot(const uint8_t* wb, const uint8_t* aq, const int16_t* /*bs*/, float dxb) {
        const uint2* grid = iq2xs_grid_smem();
        const uint2* sgn = iq2xxs_signs_smem();
        const float d = iq_d8(*reinterpret_cast<const uint16_t*>(wb));
        const uint32_t sc[2] = {lds_u32_a2(wb + 66), lds_u32_a2(wb + 70)};   // byte ib: the nibbles of sub-block ib's halves
        int isum = 0;
#pragma unroll
        for (int ib = 0; ib < 8; ib++) {
            const uint32_t q[2] = {lds_u32_a2(wb + 2 + 8 * ib), lds_u32_a2(wb + 6 + 8 * ib)};
            const uint32_t s = sc[ib >> 2] >> (8 * (ib & 3));
            const uint4 a0 = *reinterpret_cast<const uint4*>(aq + 32 * ib);
            const uint4 a1 = *reinterpret_cast<const uint4*>(aq + 32 * ib + 16);
            const uint32_t ax[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            int v[2] = {0, 0};
#pragma unroll
            for (int l = 0; l < 4; l++) {   // 8-value group l: uint16 l of the sub-block
                const uint32_t u = q[l >> 1] >> (16 * (l & 1));
                const uint2 g = grid[u & 511];
                const uint2 m = sgn[(u >> 9) & 127];
                v[l >> 1] = dp4a_s8s8(__vsub4(g.x ^ m.x, m.x), ax[2 * l], v[l >> 1]);
                v[l >> 1] = dp4a_s8s8(__vsub4(g.y ^ m.y, m.y), ax[2 * l + 1], v[l >> 1]);
            }
            isum += (2 * (int)(s & 15) + 1) * v[0] + (2 * (int)((s >> 4) & 15) + 1) * v[1];
        }
        return iq_term(d, dxb, isum);
    }
    __device__ static __forceinline__ float dot(const uint8_t* sl, int f, int /*nrb*/, const uint8_t* aq, const int16_t* bs, float dxb) {
        return block_dot(sl + f * SZ_IQ2_XS, aq, bs, dxb);
    }
};

// 10-bit indices into the 1024 x 8 grid (qs byte | two bits of qh), one sign byte per 8 values (IQ3_S's byte-mask table) and
// IQ2_XS's scale per 16 values; term = ((d/8) * dx) * S.
struct BulkIQ2S : BulkFmt {
    static constexpr int kType = KTB200_TYPE_IQ2_S;
    static constexpr int kBlockBytes = SZ_IQ2_S;
    static constexpr int kBs = 8;            // staged, not read
    static constexpr int kTableBytes = 1024 * 8 + 256 * 8;
    static constexpr bool kSharedSlot = false;
    static constexpr int kNblkMultiple = 4;  // a 2-row unit is 164 * nblk B
    __device__ static __forceinline__ void stage_tables() {
        uint2* g = iq2s_grid_smem();
        uint2* m = iq3s_signs_smem();
        for (int i = threadIdx.x; i < 1024; i += blockDim.x) g[i] = *reinterpret_cast<const uint2*>(ktb_iq2s_grid[i]);
        for (int i = threadIdx.x; i < 256; i += blockDim.x) m[i] = iq2_sign_masks(i);
    }
    __device__ static __forceinline__ float block_dot(const uint8_t* wb, const uint8_t* aq, const int16_t* /*bs*/, float dxb) {
        const uint2* grid = iq2s_grid_smem();
        const uint2* sgn = iq3s_signs_smem();
        const float d = iq_d8(*reinterpret_cast<const uint16_t*>(wb));
        const uint32_t qhw[2] = {lds_u32_a2(wb + 66), lds_u32_a2(wb + 70)};   // byte ib: 2 high index bits per 8-value group
        const uint32_t sc[2] = {lds_u32_a2(wb + 74), lds_u32_a2(wb + 78)};
        int isum = 0;
#pragma unroll
        for (int ib = 0; ib < 8; ib++) {
            const uint32_t qs = lds_u32_a2(wb + 2 + 4 * ib);
            const uint32_t sg = lds_u32_a2(wb + 34 + 4 * ib);   // byte l: the signs of values 8l..8l+7
            const uint32_t qh = qhw[ib >> 2] >> (8 * (ib & 3)), s = sc[ib >> 2] >> (8 * (ib & 3));
            const uint4 a0 = *reinterpret_cast<const uint4*>(aq + 32 * ib);
            const uint4 a1 = *reinterpret_cast<const uint4*>(aq + 32 * ib + 16);
            const uint32_t ax[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            int v[2] = {0, 0};
#pragma unroll
            for (int l = 0; l < 4; l++) {
                const uint2 g = grid[((qs >> (8 * l)) & 0xff) | ((qh << (8 - 2 * l)) & 0x300)];
                const uint2 m = sgn[(sg >> (8 * l)) & 0xff];
                v[l >> 1] = dp4a_s8s8(__vsub4(g.x ^ m.x, m.x), ax[2 * l], v[l >> 1]);
                v[l >> 1] = dp4a_s8s8(__vsub4(g.y ^ m.y, m.y), ax[2 * l + 1], v[l >> 1]);
            }
            isum += (2 * (int)(s & 15) + 1) * v[0] + (2 * (int)((s >> 4) & 15) + 1) * v[1];
        }
        return iq_term(d, dxb, isum);
    }
    __device__ static __forceinline__ float dot(const uint8_t* sl, int f, int /*nrb*/, const uint8_t* aq, const int16_t* bs, float dxb) {
        return block_dot(sl + f * SZ_IQ2_S, aq, bs, dxb);
    }
};

// ---------------------------------------------------------------------------------------------------------------
// Gate/up pairs of IQ1_S, IQ1_M, IQ2_XXS, IQ2_XS, IQ2_S, IQ3_XXS, IQ3_S, Q2_K or Q3_K experts (gate and up of the same type).
// Structure of rows_bulk_q4k_kernel
// (token chunks, one (token, slot) work list per chunk, Q8_K activations staged side by side), with a 2-row unit per ring slot.
// Fmt::kSharedSlot: a shared expert (p.x0 / p.x1, launcher: every token of the chunk) is slot p.slots of every token.
constexpr int kIqMaxWarps = 16;
template <class Fmt, int SLOTS>
__global__ void __launch_bounds__(kIqMaxWarps * 32, 1) rows_bulk_iq_kernel(const RowsParams p, int act_tok, int tc) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ int s_np;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    Fmt::stage_tables();     // read only after the first __syncthreads below
    int Teff = p.ntokens;
    if (p.bsz) Teff = min(Teff, *p.bsz);
    const int nblk = p.ncols / QK_K;
    const int row_bytes = nblk * Fmt::kBlockBytes;
    const int unit_bytes = 2 * row_bytes;             // rows 2r, 2r+1 of one matrix
    const int nru = p.rows / 2;                       // row pairs per matrix
    const int nslots = p.slots + (Fmt::kSharedSlot && p.x0 ? 1 : 0);
    const int total_out = nslots * p.rows;
    // [tc activation rows: q8 [nblk][272] | bs [nblk][kBs] int16 | dx [nblk]] [pair list] [ring: slot = gate unit | up unit]
    int* pairs = reinterpret_cast<int*>(smem + (size_t)tc * act_tok);
    BulkRing<SLOTS> ring(smem, (size_t)tc * act_tok + (size_t)tc * nslots * 4, 2 * unit_bytes, lane, warp, W);

  for (int t0 = 0; t0 < Teff; t0 += tc) {
    const int nt = min(tc, Teff - t0);
    __syncthreads();
    if (threadIdx.x == 0) s_np = gateup_pairs(p, t0, nt, Fmt::kSharedSlot && p.x0, pairs);
    __syncthreads();
    const int total = s_np * nru;
    const int u0 = (int)((long)total * blockIdx.x / gridDim.x), u1 = (int)((long)total * (blockIdx.x + 1) / gridDim.x);
    const int nu = warp_units(u0, u1, warp, W);
    UnitCursor ic;
    if (nu > 0) ic.start(u0 + warp, nru);
    UnitCursor cc = ic;
    int iss = 0;

    auto issue_one = [&]() {
        if (iss < nu) {
            ring.issue(lane, 2, (uint32_t)unit_bytes, [&](int c) {
                const int pr = pairs[ic.pi];
                const bool sh = Fmt::kSharedSlot && (pr & 0xff) == p.slots;
                const long e = sh ? 0L : pair_expert(p, t0 + (pr >> 8), pr & 0xff);
                const void* w = sh ? (c ? p.x1 : p.x0) : (c ? p.w1 : p.w0);
                return reinterpret_cast<const uint8_t*>(w) + (e * p.rows + 2L * ic.r) * row_bytes;
            });
            iss++;
            ic.step(W, nru);
        }
    };
#pragma unroll
    for (int s = 0; s < SLOTS; s++) issue_one();

    stage_q8k_rows<Fmt::kBs>(p.x, p.hidden_type, t0, nt, p.ncols, smem, act_tok, lane, warp, W);
    __syncthreads();

    for (int n = 0; n < nu; n++) {
        const uint8_t* sl = ring.wait();
        const int pr = pairs[cc.pi];
        const uint8_t* at = smem + (size_t)(pr >> 8) * act_tok;
        const int16_t* bs = reinterpret_cast<const int16_t*>(at + (size_t)nblk * kActBlkStride);
        const float* dx = reinterpret_cast<const float*>(at + (size_t)nblk * (kActBlkStride + 2 * Fmt::kBs));
        float g0 = 0.f, g1 = 0.f, v0 = 0.f, v1 = 0.f;
        for (int f = lane; f < 2 * nblk; f += 32) {   // (row, block) of the unit: f = rw * nblk + blk
            const int rw = f >= nblk, blk = f - rw * nblk;
            const uint8_t* aq = at + (size_t)blk * kActBlkStride;
            const float g = Fmt::block_dot(sl + f * Fmt::kBlockBytes, aq, bs + blk * Fmt::kBs, dx[blk]);
            const float u = Fmt::block_dot(sl + unit_bytes + f * Fmt::kBlockBytes, aq, bs + blk * Fmt::kBs, dx[blk]);
            if (rw) { g1 += g; v1 += u; } else { g0 += g; v0 += u; }
        }
        const float r = warp_reduce4(g0, g1, v0, v1, lane);   // lane 0: g0, 8: g1, 16: u0, 24: u1
        ring.release();
        issue_one();
        const float gs = __shfl_sync(0xffffffffu, r, 8 * (lane & 1)), us = __shfl_sync(0xffffffffu, r, 16 + 8 * (lane & 1));
        if (lane < 2) {
            const long o = (long)(t0 + (pr >> 8)) * total_out + (long)(pr & 0xff) * p.rows + 2L * cc.r + lane;
            p.out_f32[o] = (p.use_silu ? act_silu(gs) : act_relu(gs)) * us;
        }
        cc.step(W, nru);
    }
  }  // token chunks
}

}  // namespace ktb
