// Weight-format policies for the streaming integer GEMV kernels (gemv.cuh).
//
// A policy describes how one warp lane pulls a "unit" (a fixed-size slice of one 256-element
// super-block of a weight row) out of HBM with aligned vector loads and reduces it against the int8
// activations staged in shared memory.  The arithmetic is the reference's integer dot product
// (ggml_vec_dot_*_q8_K, third_party/llama.cpp/ggml-quants.c:6962/8167/...): int8 x intN -> int32
// exactly, then fp32 (d_w * d_x) * isum - (dmin_w * d_x) * msum.
//
// In one "step" the 32 lanes of a warp cover kBlocksPerStep consecutive super-blocks of a row; which
// slice of which block a lane owns is a per-lane constant (struct Lane), computed once per thread so
// that shifts, byte offsets and the scale-decode variant are loop invariant.
//
//   FmtQ4K    raw GGUF block_q4_K (144 B, already 16-byte aligned)   unit = 16 B of qs = 32 weights, 4 blocks/step
//   FmtQ5K    raw GGUF block_q5_K (176 B, 16-byte aligned)           unit = 16 B qs + qh   = 32 weights, 4 blocks/step
//   FmtQ6K8   block_q6_K re-laid as "8-row SoA" (moe.cu repack)      unit = 48 B           = 64 weights, 8 blocks/step
//   FmtGenK   any raw K-quant / IQ4_XS / IQ2_XXS / IQ1_S / IQ1_M / IQ3_XXS / IQ3_S / IQ2_XS / IQ2_S through byte loads (fallback)
//                                                                    unit = 16 weights,              2 blocks/step
#pragma once
#include "common.cuh"

// The IQ codebooks (device globals) only exist in the translation units that dispatch those types
// (moe.cu, dequant.cu define KTB_IQ_CODEBOOKS); elsewhere unpack_group16 has no IQ cases and no table is emitted.
#ifdef KTB_IQ_CODEBOOKS
#define KTB_IQ_TABLE static __device__ const
#include "iq_tables.h"
#include "iq3_tables.h"
#include "iq2_tables.h"
#endif

namespace ktb {

// int8 activations of ONE row staged in shared memory.
struct ActQ8K {
    const uint8_t* q8;     // [n] int8
    const float* dx;       // [n/256]
    const int16_t* bsums;  // [n/16]
};

__device__ __forceinline__ int sext8(uint32_t v) { return (int)(int8_t)(v & 0xff); }

// 6-bit (scale, min) pair of sub-blocks (2j, 2j+1) from the 12 packed bytes (get_scale_min_k4,
// ggml-quants.c:1891-1899), branch-free; `sh` = 16*(j&1), `big` = (j >= 2) are lane constants.
// Returns sc = sc0 | sc1<<8 and mn = m0 | m1<<8.
__device__ __forceinline__ void k4_pair(uint32_t w0, uint32_t w1, uint32_t w2, int sh, bool big, uint32_t& sc, uint32_t& mn) {
    const uint32_t a0 = w0 >> sh, a1 = w1 >> sh, a2 = w2 >> sh;
    const uint32_t sc_lo = a0 & 0x3f3fu, mn_lo = a1 & 0x3f3fu;
    const uint32_t sc_hi = (a2 & 0x0f0fu) | ((a0 >> 2) & 0x3030u);
    const uint32_t mn_hi = ((a2 >> 4) & 0x0f0fu) | ((a1 >> 2) & 0x3030u);
    sc = big ? sc_hi : sc_lo;
    mn = big ? mn_hi : mn_lo;
}

// ---------------------------------------------------------------------------------------------
struct FmtQ4K {
    static constexpr int kType = KTB200_TYPE_Q4_K;
    static constexpr int kBlocksPerStep = 4;
    static constexpr int kBlockBytes = SZ_Q4_K;
    struct Lane { int blk, qs_off, act_off, bs_off, sh; bool big, half; };
    struct Row { const uint8_t* p; };
    struct Regs { uint4 hdr, qs; };
    struct Act { uint4 lo, hi; float dx; int bsum; };

    __device__ static __forceinline__ Lane lane(int l) {
        const int cc = l & 7, j = cc >> 1, half = cc & 1;
        return Lane{l >> 3, 16 + cc * 16, 64 * j + 16 * half, 4 * j + 2 * half, 16 * (j & 1), j >= 2, half != 0};
    }
    __device__ static __forceinline__ Row row(const void* base, long row_idx, int ncols, int /*type*/) {
        return Row{reinterpret_cast<const uint8_t*>(base) + row_idx * (long)(ncols / QK_K) * SZ_Q4_K};
    }
    __device__ static __forceinline__ void prefetch(const Row& r, int nblk) { prefetch_l2_bulk(r.p, nblk * SZ_Q4_K); }
    __device__ static __forceinline__ void load(const Row& r, int blk, const Lane& L, Regs& R) {
        const uint8_t* b = r.p + blk * SZ_Q4_K;
        R.hdr = ldg_stream16(b);
        R.qs = ldg_stream16(b + L.qs_off);
    }
    // the same slice from a row staged in shared memory (gemv_pipe.cuh)
    __device__ static __forceinline__ void load_smem(const uint8_t* row, int blk, const Lane& L, Regs& R) {
        const uint8_t* b = row + blk * SZ_Q4_K;
        R.hdr = *reinterpret_cast<const uint4*>(b);
        R.qs = *reinterpret_cast<const uint4*>(b + L.qs_off);
    }
    __device__ static __forceinline__ void load_act(const ActQ8K& a, int blk, const Lane& L, Act& A) {
        const uint8_t* q = a.q8 + blk * QK_K + L.act_off;
        A.lo = *reinterpret_cast<const uint4*>(q);
        A.hi = *reinterpret_cast<const uint4*>(q + 32);
        A.dx = a.dx[blk];
        // sum of the 32 activations of this lane's sub-block = bsums[2s] + bsums[2s+1]
        const uint32_t w = *reinterpret_cast<const uint32_t*>(a.bsums + blk * 16 + L.bs_off);
        A.bsum = (int)(int16_t)(w & 0xffff) + (int)(int16_t)(w >> 16);
    }
    __device__ static __forceinline__ float dot(const Regs& R, const Act& A, const Lane& L) {
        uint32_t sc, mn;
        k4_pair(R.hdr.y, R.hdr.z, R.hdr.w, L.sh, L.big, sc, mn);
        int slo = 0, shi = 0;
        slo = dp4a_s8s8(R.qs.x & 0x0f0f0f0fu, A.lo.x, slo);
        slo = dp4a_s8s8(R.qs.y & 0x0f0f0f0fu, A.lo.y, slo);
        slo = dp4a_s8s8(R.qs.z & 0x0f0f0f0fu, A.lo.z, slo);
        slo = dp4a_s8s8(R.qs.w & 0x0f0f0f0fu, A.lo.w, slo);
        // high nibbles stay in place (value*16, unsigned byte): the sum is an exact multiple of 16
        shi = dp4a_u8s8(R.qs.x & 0xf0f0f0f0u, A.hi.x, shi);
        shi = dp4a_u8s8(R.qs.y & 0xf0f0f0f0u, A.hi.y, shi);
        shi = dp4a_u8s8(R.qs.z & 0xf0f0f0f0u, A.hi.z, shi);
        shi = dp4a_u8s8(R.qs.w & 0xf0f0f0f0u, A.hi.w, shi);
        const int isum = (int)(sc & 0xff) * slo + (int)(sc >> 8) * (shi >> 4);
        const int m = L.half ? (int)(mn >> 8) : (int)(mn & 0xff);
        const float2 dm = __half22float2(*reinterpret_cast<const __half2*>(&R.hdr.x));
        return (dm.x * A.dx) * (float)isum - (dm.y * A.dx) * (float)(m * A.bsum);
    }
};

// ---------------------------------------------------------------------------------------------
// Q4_K with 32-byte units (one whole 64-value group per lane: both nibble planes, both sub-blocks), used when
// the row is staged in shared memory (gemv_pipe.cuh).  4 lanes per block, 8 blocks per step: the 6-bit scale
// decode, the fp16 conversions and the fp32 scale application are paid once per 64 weights instead of once
// per 32, which is what the issue-bound gate/up kernel needs (ncu: ~1200 warp instructions per row pair).
struct FmtQ4K32 {
    static constexpr int kType = KTB200_TYPE_Q4_K;
    static constexpr int kBlocksPerStep = 8;
    static constexpr int kBlockBytes = SZ_Q4_K;
    struct Lane { int blk, qs_off, act_off, bs_off, sh; bool big; };
    struct Regs { uint4 hdr, q0, q1; };
    struct Act { uint4 l0, l1, h0, h1; float dx; int bs_lo, bs_hi; };

    __device__ static __forceinline__ Lane lane(int l) {
        const int j = l & 3;
        return Lane{l >> 2, 16 + 32 * j, 64 * j, 4 * j, 16 * (j & 1), j >= 2};
    }
    __device__ static __forceinline__ void load_smem(const uint8_t* row, int blk, const Lane& L, Regs& R) {
        const uint8_t* b = row + blk * SZ_Q4_K;
        R.hdr = *reinterpret_cast<const uint4*>(b);
        R.q0 = *reinterpret_cast<const uint4*>(b + L.qs_off);
        R.q1 = *reinterpret_cast<const uint4*>(b + L.qs_off + 16);
    }
    __device__ static __forceinline__ void load_act(const ActQ8K& a, int blk, const Lane& L, Act& A) {
        const uint8_t* q = a.q8 + blk * QK_K + L.act_off;
        A.l0 = *reinterpret_cast<const uint4*>(q);
        A.l1 = *reinterpret_cast<const uint4*>(q + 16);
        A.h0 = *reinterpret_cast<const uint4*>(q + 32);
        A.h1 = *reinterpret_cast<const uint4*>(q + 48);
        A.dx = a.dx[blk];
        const uint2 w = *reinterpret_cast<const uint2*>(a.bsums + blk * 16 + L.bs_off);   // 4 x int16
        A.bs_lo = (int)(int16_t)(w.x & 0xffff) + (int)(int16_t)(w.x >> 16);
        A.bs_hi = (int)(int16_t)(w.y & 0xffff) + (int)(int16_t)(w.y >> 16);
    }
    __device__ static __forceinline__ float dot(const Regs& R, const Act& A, const Lane& L) {
        uint32_t sc, mn;
        k4_pair(R.hdr.y, R.hdr.z, R.hdr.w, L.sh, L.big, sc, mn);
        int slo = 0, shi = 0;
        slo = dp4a_s8s8(R.q0.x & 0x0f0f0f0fu, A.l0.x, slo);
        slo = dp4a_s8s8(R.q0.y & 0x0f0f0f0fu, A.l0.y, slo);
        slo = dp4a_s8s8(R.q0.z & 0x0f0f0f0fu, A.l0.z, slo);
        slo = dp4a_s8s8(R.q0.w & 0x0f0f0f0fu, A.l0.w, slo);
        slo = dp4a_s8s8(R.q1.x & 0x0f0f0f0fu, A.l1.x, slo);
        slo = dp4a_s8s8(R.q1.y & 0x0f0f0f0fu, A.l1.y, slo);
        slo = dp4a_s8s8(R.q1.z & 0x0f0f0f0fu, A.l1.z, slo);
        slo = dp4a_s8s8(R.q1.w & 0x0f0f0f0fu, A.l1.w, slo);
        shi = dp4a_u8s8(R.q0.x & 0xf0f0f0f0u, A.h0.x, shi);
        shi = dp4a_u8s8(R.q0.y & 0xf0f0f0f0u, A.h0.y, shi);
        shi = dp4a_u8s8(R.q0.z & 0xf0f0f0f0u, A.h0.z, shi);
        shi = dp4a_u8s8(R.q0.w & 0xf0f0f0f0u, A.h0.w, shi);
        shi = dp4a_u8s8(R.q1.x & 0xf0f0f0f0u, A.h1.x, shi);
        shi = dp4a_u8s8(R.q1.y & 0xf0f0f0f0u, A.h1.y, shi);
        shi = dp4a_u8s8(R.q1.z & 0xf0f0f0f0u, A.h1.z, shi);
        shi = dp4a_u8s8(R.q1.w & 0xf0f0f0f0u, A.h1.w, shi);
        const int isum = (int)(sc & 0xff) * slo + (int)(sc >> 8) * (shi >> 4);
        const int msum = (int)(mn & 0xff) * A.bs_lo + (int)(mn >> 8) * A.bs_hi;
        const float2 dm = __half22float2(*reinterpret_cast<const __half2*>(&R.hdr.x));
        return (dm.x * A.dx) * (float)isum - (dm.y * A.dx) * (float)msum;
    }
};

// ---------------------------------------------------------------------------------------------
// Q6_K in the 8-row SoA layout produced by repack_q6k (moe.cu).  For a group of 8 consecutive rows,
// each of nb = ncols/256 blocks:  [ql: 8 x nb x 128][qh: 8 x nb x 64][scales: 8 x nb x 16][d: 8 x nb x 2]
// (= 8 * nb * 210 bytes, same as raw).  Every ql/qh/scales slice a lane touches is 16-byte aligned.
struct FmtQ6K8 {
    static constexpr int kType = KTB200_TYPE_Q6_K;
    static constexpr int kBlocksPerStep = 8;
    struct Lane { int blk, ql_off, qh_off, act_off, bs_off, sc_sh; bool hh; };
    struct Row { const uint8_t *ql, *qh, *sc, *d; };
    struct Regs { uint4 a, b, h, s; uint32_t d; };
    struct Act { uint4 x0, x1, x2, x3; float dx; int bs0, bs1, bs2, bs3; };

    __device__ static __forceinline__ Lane lane(int l) {
        const int hh = (l >> 1) & 1, odd = l & 1;
        return Lane{l >> 2, 64 * hh + 16 * odd, 32 * hh + 16 * odd, 128 * hh + 16 * odd, 8 * hh + odd, 8 * odd, hh != 0};
    }
    __device__ static __forceinline__ Row row(const void* base, long row_idx, int ncols, int /*type*/) {
        const long nb = ncols / QK_K;
        const long G = row_idx >> 3, r8 = row_idx & 7;
        const uint8_t* g = reinterpret_cast<const uint8_t*>(base) + G * (8 * SZ_Q6_K) * nb;
        return Row{g + r8 * 128 * nb, g + 1024 * nb + r8 * 64 * nb, g + 1536 * nb + r8 * 16 * nb,
                   g + 1664 * nb + r8 * 2 * nb};
    }
    __device__ static __forceinline__ void prefetch(const Row& r, int nblk) {
        prefetch_l2_bulk(r.ql, nblk * 128);
        prefetch_l2_bulk(r.qh, nblk * 64);
        prefetch_l2_bulk(r.sc, nblk * 16);
    }
    __device__ static __forceinline__ void load(const Row& r, int blk, const Lane& L, Regs& R) {
        R.a = ldg_stream16(r.ql + blk * 128 + L.ql_off);
        R.b = ldg_stream16(r.ql + blk * 128 + L.ql_off + 32);
        R.h = ldg_stream16(r.qh + blk * 64 + L.qh_off);
        R.s = ldg_stream16(r.sc + blk * 16);
        R.d = ldg_u16(r.d + blk * 2);
    }
    // the same slices from an item staged in shared memory (gemv_pipe.cuh): Row pointers point into smem
    __device__ static __forceinline__ void load_smem(const Row& r, int blk, const Lane& L, Regs& R) {
        R.a = *reinterpret_cast<const uint4*>(r.ql + blk * 128 + L.ql_off);
        R.b = *reinterpret_cast<const uint4*>(r.ql + blk * 128 + L.ql_off + 32);
        R.h = *reinterpret_cast<const uint4*>(r.qh + blk * 64 + L.qh_off);
        R.s = *reinterpret_cast<const uint4*>(r.sc + blk * 16);
        R.d = *reinterpret_cast<const uint16_t*>(r.d + blk * 2);
    }
    __device__ static __forceinline__ void load_act(const ActQ8K& a, int blk, const Lane& L, Act& A) {
        const uint8_t* q = a.q8 + blk * QK_K + L.act_off;
        A.x0 = *reinterpret_cast<const uint4*>(q);
        A.x1 = *reinterpret_cast<const uint4*>(q + 32);
        A.x2 = *reinterpret_cast<const uint4*>(q + 64);
        A.x3 = *reinterpret_cast<const uint4*>(q + 96);
        A.dx = a.dx[blk];
        const int16_t* bs = a.bsums + blk * 16 + L.bs_off;
        A.bs0 = bs[0]; A.bs1 = bs[2]; A.bs2 = bs[4]; A.bs3 = bs[6];
    }
    __device__ static __forceinline__ void dot_word(uint32_t a, uint32_t b, uint32_t h, uint32_t x0, uint32_t x1,
                                                    uint32_t x2, uint32_t x3, int& s0, int& s1, int& s2, int& s3) {
        // 6-bit value = 4 low bits from ql | 2 high bits from qh; values 0..63 (the -32 is folded into bsums).
        // v2/v3 keep the ql high nibble in place (x16) and add the qh bits at x16 too: sums are multiples of 16.
        const uint32_t v0 = (a & 0x0f0f0f0fu) | ((h << 4) & 0x30303030u);
        const uint32_t v1 = (b & 0x0f0f0f0fu) | ((h << 2) & 0x30303030u);
        const uint32_t v2 = ((a >> 4) & 0x0f0f0f0fu) | (h & 0x30303030u);
        const uint32_t v3 = ((b >> 4) & 0x0f0f0f0fu) | ((h >> 2) & 0x30303030u);
        s0 = dp4a_s8s8(v0, x0, s0);
        s1 = dp4a_s8s8(v1, x1, s1);
        s2 = dp4a_s8s8(v2, x2, s2);
        s3 = dp4a_s8s8(v3, x3, s3);
    }
    __device__ static __forceinline__ float dot(const Regs& R, const Act& A, const Lane& L) {
        int s0 = 0, s1 = 0, s2 = 0, s3 = 0;
        dot_word(R.a.x, R.b.x, R.h.x, A.x0.x, A.x1.x, A.x2.x, A.x3.x, s0, s1, s2, s3);
        dot_word(R.a.y, R.b.y, R.h.y, A.x0.y, A.x1.y, A.x2.y, A.x3.y, s0, s1, s2, s3);
        dot_word(R.a.z, R.b.z, R.h.z, A.x0.z, A.x1.z, A.x2.z, A.x3.z, s0, s1, s2, s3);
        dot_word(R.a.w, R.b.w, R.h.w, A.x0.w, A.x1.w, A.x2.w, A.x3.w, s0, s1, s2, s3);
        // 16 int8 scales of the block; this unit uses groups 8*hh + 2*i + odd, i = 0..3
        const uint32_t lo = L.hh ? R.s.z : R.s.x, hi = L.hh ? R.s.w : R.s.y;  // bytes 8hh..8hh+3 / +4..+7
        const int c0 = sext8(lo >> L.sc_sh), c1 = sext8(lo >> (16 + L.sc_sh)), c2 = sext8(hi >> L.sc_sh), c3 = sext8(hi >> (16 + L.sc_sh));
        // q stored with +32 offset: sum (q-32) x = sum q x - 32 * bsum
        const int isum = c0 * (s0 - 32 * A.bs0) + c1 * (s1 - 32 * A.bs1) + c2 * (s2 - 32 * A.bs2) + c3 * (s3 - 32 * A.bs3);
        return (fp16_bits_to_f32((uint16_t)R.d) * A.dx) * (float)isum;
    }
};

// ---------------------------------------------------------------------------------------------
// Raw Q5_K: {half d, dmin; u8 scales[12]; u8 qh[32]; u8 qs[128]} = 176 B (16-byte aligned).
struct FmtQ5K {
    static constexpr int kType = KTB200_TYPE_Q5_K;
    static constexpr int kBlocksPerStep = 4;
    static constexpr int kBlockBytes = SZ_Q5_K;
    struct Lane { int blk, qs_off, qh_off, act_off, bs_off, sh, hsh; bool big, half; };
    struct Row { const uint8_t* p; };
    struct Regs { uint4 hdr, qh, qs; };
    using Act = FmtQ4K::Act;

    __device__ static __forceinline__ Lane lane(int l) {
        const int cc = l & 7, j = cc >> 1, half = cc & 1;
        return Lane{l >> 3, 48 + cc * 16, 16 + half * 16, 64 * j + 16 * half, 4 * j + 2 * half, 16 * (j & 1), 2 * j, j >= 2, half != 0};
    }
    __device__ static __forceinline__ Row row(const void* base, long row_idx, int ncols, int) {
        return Row{reinterpret_cast<const uint8_t*>(base) + row_idx * (long)(ncols / QK_K) * SZ_Q5_K};
    }
    __device__ static __forceinline__ void prefetch(const Row& r, int nblk) { prefetch_l2_bulk(r.p, nblk * SZ_Q5_K); }
    __device__ static __forceinline__ void load_smem(const uint8_t* row, int blk, const Lane& L, Regs& R) {
        const uint8_t* b = row + blk * SZ_Q5_K;
        R.hdr = *reinterpret_cast<const uint4*>(b);
        R.qh = *reinterpret_cast<const uint4*>(b + L.qh_off);
        R.qs = *reinterpret_cast<const uint4*>(b + L.qs_off);
    }
    __device__ static __forceinline__ void load(const Row& r, int blk, const Lane& L, Regs& R) {
        const uint8_t* b = r.p + blk * SZ_Q5_K;
        R.hdr = ldg_stream16(b);
        R.qh = ldg_stream16(b + L.qh_off);
        R.qs = ldg_stream16(b + L.qs_off);
    }
    __device__ static __forceinline__ void load_act(const ActQ8K& a, int blk, const Lane& L, Act& A) {
        const uint8_t* q = a.q8 + blk * QK_K + L.act_off;
        A.lo = *reinterpret_cast<const uint4*>(q);
        A.hi = *reinterpret_cast<const uint4*>(q + 32);
        A.dx = a.dx[blk];
        const uint32_t w = *reinterpret_cast<const uint32_t*>(a.bsums + blk * 16 + L.bs_off);
        A.bsum = (int)(int16_t)(w & 0xffff) + (int)(int16_t)(w >> 16);
    }
    __device__ static __forceinline__ float dot(const Regs& R, const Act& A, const Lane& L) {
        uint32_t sc, mn;
        k4_pair(R.hdr.y, R.hdr.z, R.hdr.w, L.sh, L.big, sc, mn);
        const uint32_t qs[4] = {R.qs.x, R.qs.y, R.qs.z, R.qs.w};
        const uint32_t qh[4] = {R.qh.x, R.qh.y, R.qh.z, R.qh.w};
        const uint32_t lo[4] = {A.lo.x, A.lo.y, A.lo.z, A.lo.w};
        const uint32_t hi[4] = {A.hi.x, A.hi.y, A.hi.z, A.hi.w};
        int slo = 0, shi = 0;
#pragma unroll
        for (int w = 0; w < 4; w++) {
            // bit 2j of the qh byte -> +16 on the low-nibble value, bit 2j+1 -> +16 on the high-nibble value
            const uint32_t hb = qh[w] >> L.hsh;
            const uint32_t vlo = (qs[w] & 0x0f0f0f0fu) | ((hb << 4) & 0x10101010u);
            const uint32_t vhi = ((qs[w] >> 4) & 0x0f0f0f0fu) | ((hb << 3) & 0x10101010u);
            slo = dp4a_s8s8(vlo, lo[w], slo);
            shi = dp4a_s8s8(vhi, hi[w], shi);
        }
        const int isum = (int)(sc & 0xff) * slo + (int)(sc >> 8) * shi;
        const int m = L.half ? (int)(mn >> 8) : (int)(mn & 0xff);
        const float2 dm = __half22float2(*reinterpret_cast<const __half2*>(&R.hdr.x));
        return (dm.x * A.dx) * (float)isum - (dm.y * A.dx) * (float)(m * A.bsum);
    }
};

// ---------------------------------------------------------------------------------------------
// Generic raw K-quant fallback: unit = one 16-element group, decoded with byte loads.
// value[i] = d * isc[g] * q[i] - dmin * imn[g]   (oracle/ktoracle.c unpack_block is the same map)
static __device__ __constant__ int8_t c_kvalues_iq4nl[16] = {-127, -104, -83, -65, -49, -35, -22, -10, 1, 13, 25, 38, 53, 69, 89, 113};

struct GroupK {
    uint32_t q[4];  // 16 signed int8
    int isc, imn;
    float d, dmin;
};

__device__ __forceinline__ void k4_scale_min(const uint8_t* sc12, int s, int& sc, int& mn) {
    if (s < 4) {
        sc = ldg_u8(sc12 + s) & 63;
        mn = ldg_u8(sc12 + s + 4) & 63;
    } else {
        sc = (ldg_u8(sc12 + s + 4) & 0xF) | ((ldg_u8(sc12 + s - 4) >> 6) << 4);
        mn = (ldg_u8(sc12 + s + 4) >> 4) | ((ldg_u8(sc12 + s) >> 6) << 4);
    }
}

__device__ inline void unpack_group16(int type, const uint8_t* b, int g, GroupK& o) {
    int8_t v[16];
    o.imn = 0;
    o.dmin = 0.f;
    switch (type) {
        case KTB200_TYPE_Q4_K: {
            o.d = fp16_bits_to_f32(ldg_u16(b));
            o.dmin = fp16_bits_to_f32(ldg_u16(b + 2));
            const int j = g >> 2, sub = g & 3;
            k4_scale_min(b + 4, 2 * j + (sub >> 1), o.isc, o.imn);
            const uint8_t* qs = b + 16 + 32 * j + 16 * (sub & 1);
            for (int l = 0; l < 16; l++) v[l] = (sub >> 1) ? (ldg_u8(qs + l) >> 4) : (ldg_u8(qs + l) & 0xF);
            break;
        }
        case KTB200_TYPE_Q5_K: {
            o.d = fp16_bits_to_f32(ldg_u16(b));
            o.dmin = fp16_bits_to_f32(ldg_u16(b + 2));
            const int j = g >> 2, sub = g & 3;
            k4_scale_min(b + 4, 2 * j + (sub >> 1), o.isc, o.imn);
            const uint8_t* qh = b + 16 + 16 * (sub & 1);
            const uint8_t* qs = b + 48 + 32 * j + 16 * (sub & 1);
            for (int l = 0; l < 16; l++) {
                const int hb = (ldg_u8(qh + l) >> (2 * j + (sub >> 1))) & 1;
                v[l] = ((sub >> 1) ? (ldg_u8(qs + l) >> 4) : (ldg_u8(qs + l) & 0xF)) + 16 * hb;
            }
            break;
        }
        case KTB200_TYPE_Q6_K: {
            o.d = fp16_bits_to_f32(ldg_u16(b + 208));
            o.isc = (int8_t)ldg_u8(b + 192 + g);
            const int e0 = 16 * g, n = e0 >> 7, within = e0 & 127, quarter = within >> 5, l0 = within & 31;
            const uint8_t* ql = b + 64 * n + (quarter & 1) * 32 + l0;
            const uint8_t* qh = b + 128 + 32 * n + l0;
            for (int l = 0; l < 16; l++) {
                const int lo4 = (quarter >> 1) ? (ldg_u8(ql + l) >> 4) : (ldg_u8(ql + l) & 0xF);
                v[l] = (lo4 | (((ldg_u8(qh + l) >> (2 * quarter)) & 3) << 4)) - 32;
            }
            break;
        }
        case KTB200_TYPE_Q2_K: {
            o.d = fp16_bits_to_f32(ldg_u16(b + 80));
            o.dmin = fp16_bits_to_f32(ldg_u16(b + 82));
            const uint8_t s = ldg_u8(b + g);
            o.isc = s & 0xF;
            o.imn = s >> 4;
            const int e0 = 16 * g, n = e0 >> 7, within = e0 & 127, j = within >> 5, l0 = within & 31;
            const uint8_t* qs = b + 16 + 32 * n + l0;
            for (int l = 0; l < 16; l++) v[l] = (ldg_u8(qs + l) >> (2 * j)) & 3;
            break;
        }
        case KTB200_TYPE_Q3_K: {
            o.d = fp16_bits_to_f32(ldg_u16(b + 108));
            // 6-bit scales: low 4 bits in bytes 0..7 (nibbles), high 2 bits in bytes 8..11
            const uint8_t* s12 = b + 96;
            const int lo4 = (g < 8) ? (ldg_u8(s12 + g) & 0xF) : (ldg_u8(s12 + g - 8) >> 4);
            const int hi2 = (ldg_u8(s12 + 8 + (g & 3)) >> (2 * (g >> 2))) & 3;
            o.isc = (lo4 | (hi2 << 4)) - 32;
            const int e0 = 16 * g, n = e0 >> 7, within = e0 & 127, j = within >> 5, l0 = within & 31;
            const uint8_t* qs = b + 32 + 32 * n + l0;
            const uint8_t* hm = b + l0;
            for (int l = 0; l < 16; l++) {
                const int bit = (ldg_u8(hm + l) >> (4 * n + j)) & 1;
                v[l] = ((ldg_u8(qs + l) >> (2 * j)) & 3) - (bit ? 0 : 4);
            }
            break;
        }
        case KTB200_TYPE_IQ4_XS: {
            o.d = fp16_bits_to_f32(ldg_u16(b));
            const uint32_t sh = ldg_u16(b + 2);
            const int ib = g >> 1, half = g & 1;
            const int ls = ((ldg_u8(b + 4 + (ib >> 1)) >> (4 * (ib & 1))) & 0xf) | (((sh >> (2 * ib)) & 3) << 4);
            o.isc = ls - 32;
            const uint8_t* qs = b + 8 + 16 * ib;
            for (int l = 0; l < 16; l++) v[l] = c_kvalues_iq4nl[half ? (ldg_u8(qs + l) >> 4) : (ldg_u8(qs + l) & 0xf)];
            break;
        }
#ifdef KTB_IQ_CODEBOOKS
        case KTB200_TYPE_IQ1_S: {
            // values held as 8*grid + delta (-9..9) with d/8: the dot's fp32 term is the reference's (d*dx)*(S/8) exactly
            o.d = fp16_bits_to_f32(ldg_u16(b)) * 0.125f;
            const int ib = g >> 1, l0 = 2 * (g & 1);
            const uint32_t qh = ldg_u16(b + 34 + 2 * ib);
            o.isc = 2 * (int)((qh >> 12) & 7) + 1;
            const int delta = (qh & 0x8000u) ? -1 : 1;
            for (int l = 0; l < 2; l++) {
                const int idx = ldg_u8(b + 2 + 4 * ib + l0 + l) | (int)(((qh >> (3 * (l0 + l))) & 7) << 8);
                for (int j = 0; j < 8; j++) v[8 * l + j] = (int8_t)(8 * (int)(int8_t)ldg_u8(&ktb_iq1s_grid[idx][j]) + delta);
            }
            break;
        }
        case KTB200_TYPE_IQ1_M: {
            // IQ1_S's form with the scale per 16 values and the delta per 8: 8*grid + delta (-9..9) with d/8
            const uint32_t s01 = (uint32_t)ldg_u16(b + 48) | ((uint32_t)ldg_u16(b + 50) << 16);
            const uint32_t s23 = (uint32_t)ldg_u16(b + 52) | ((uint32_t)ldg_u16(b + 54) << 16);
            o.d = fp16_bits_to_f32(iq1m_d_bits(s01, s23)) * 0.125f;
            o.isc = 2 * (int)((ldg_u16(b + 48 + 2 * (g >> 2)) >> (3 * (g & 3))) & 7) + 1;
            const uint32_t qh = ldg_u8(b + 32 + g);   // low nibble: 8-value group 2g, high nibble: 2g + 1
            for (int l = 0; l < 2; l++) {
                const uint32_t nib = (qh >> (4 * l)) & 15;
                const int idx = ldg_u8(b + 2 * g + l) | (int)((nib & 7) << 8);
                const int delta = (nib & 8) ? -1 : 1;
                for (int j = 0; j < 8; j++) v[8 * l + j] = (int8_t)(8 * (int)(int8_t)ldg_u8(&ktb_iq1s_grid[idx][j]) + delta);
            }
            break;
        }
        case KTB200_TYPE_IQ2_XXS: {
            // d/8 and ls = 2s+1: the reference's final 0.125 folded into the scale (exact, a power of two)
            o.d = fp16_bits_to_f32(ldg_u16(b)) * 0.125f;
            const int ib = g >> 1, l0 = 2 * (g & 1);
            const uint8_t* q = b + 2 + 8 * ib;
            const uint32_t aux1 = (uint32_t)ldg_u16(q + 4) | ((uint32_t)ldg_u16(q + 6) << 16);
            o.isc = 2 * (int)(aux1 >> 28) + 1;
            for (int l = 0; l < 2; l++) {
                const int idx = ldg_u8(q + l0 + l);
                const uint32_t signs = ldg_u8(&ktb_ksigns_iq2xs[(aux1 >> (7 * (l0 + l))) & 127]);
                for (int j = 0; j < 8; j++) {
                    const int gv = ldg_u8(&ktb_iq2xxs_grid[idx][j]);
                    v[8 * l + j] = (int8_t)(((signs >> j) & 1) ? -gv : gv);
                }
            }
            break;
        }
        case KTB200_TYPE_IQ3_XXS: {
            // d/4 and ls = 2s+1: the reference's final 0.25 folded into the scale; values +-grid (4..62)
            o.d = fp16_bits_to_f32(ldg_u16(b)) * 0.25f;
            const int ib = g >> 1, l0 = 2 * (g & 1);
            const uint8_t* q = b + 2 + 8 * ib;
            const uint32_t aux = (uint32_t)ldg_u16(b + 66 + 4 * ib) | ((uint32_t)ldg_u16(b + 68 + 4 * ib) << 16);
            o.isc = 2 * (int)(aux >> 28) + 1;
            for (int l = 0; l < 2; l++) {
                const uint32_t signs = ldg_u8(&ktb_ksigns_iq2xs[(aux >> (7 * (l0 + l))) & 127]);
                for (int j = 0; j < 8; j++) {
                    const int gv = ldg_u8(&ktb_iq3xxs_grid[ldg_u8(q + 2 * (l0 + l) + (j >> 2))][j & 3]);
                    v[8 * l + j] = (int8_t)(((signs >> j) & 1) ? -gv : gv);
                }
            }
            break;
        }
        case KTB200_TYPE_IQ3_S: {
            // d and ls = 2s+1; values +-grid (1..15).  16-value group g: 4-value groups 4g..4g+3, sign bytes 2g, 2g+1
            o.d = fp16_bits_to_f32(ldg_u16(b));
            const int ib = g >> 1;
            o.isc = 2 * (int)((ldg_u8(b + 106 + (ib >> 1)) >> (4 * (ib & 1))) & 15) + 1;
            const uint32_t qh = ldg_u8(b + 66 + ib);
            const uint32_t signs = (uint32_t)ldg_u8(b + 74 + 2 * g) | ((uint32_t)ldg_u8(b + 75 + 2 * g) << 8);
            for (int k = 0; k < 4; k++) {
                const int j = 4 * g + k;   // 4-value group of the block; j % 8 = 4 (g & 1) + k
                const int idx = ldg_u8(b + 2 + j) | (int)(((qh >> (j & 7)) & 1) << 8);
                for (int i = 0; i < 4; i++) {
                    const int gv = ldg_u8(&ktb_iq3s_grid[idx][i]);
                    v[4 * k + i] = (int8_t)(((signs >> (4 * k + i)) & 1) ? -gv : gv);
                }
            }
            break;
        }
        case KTB200_TYPE_IQ2_XS: {
            // d/8 and ls = 2s+1 per 16 values (nibble g % 2 of scales[g / 2]); 8-value group 2g + l: qs[2g + l] & 511 indexes
            // iq2xs_grid, qs[2g + l] >> 9 ksigns_iq2xs
            o.d = fp16_bits_to_f32(ldg_u16(b)) * 0.125f;
            o.isc = 2 * (int)((ldg_u8(b + 66 + (g >> 1)) >> (4 * (g & 1))) & 15) + 1;
            for (int l = 0; l < 2; l++) {
                const uint32_t q = ldg_u16(b + 2 + 2 * (2 * g + l));
                const uint32_t signs = ldg_u8(&ktb_ksigns_iq2xs[q >> 9]);
                for (int j = 0; j < 8; j++) {
                    const int gv = ldg_u8(&ktb_iq2xs_grid[q & 511][j]);
                    v[8 * l + j] = (int8_t)(((signs >> j) & 1) ? -gv : gv);
                }
            }
            break;
        }
        case KTB200_TYPE_IQ2_S: {
            // d/8 and ls = 2s+1 per 16 values as IQ2_XS; 8-value group 2g + l: iq2s_grid[qs | 2 bits of qh << 8], sign byte
            o.d = fp16_bits_to_f32(ldg_u16(b)) * 0.125f;
            o.isc = 2 * (int)((ldg_u8(b + 74 + (g >> 1)) >> (4 * (g & 1))) & 15) + 1;
            const uint32_t qh = ldg_u8(b + 66 + (g >> 1));
            for (int l = 0; l < 2; l++) {
                const int k = 2 * g + l;   // 8-value group of the block; k % 4 = 2 (g & 1) + l
                const int idx = ldg_u8(b + 2 + k) | (int)(((qh >> (2 * (k & 3))) & 3) << 8);
                const uint32_t signs = ldg_u8(b + 34 + k);
                for (int j = 0; j < 8; j++) {
                    const int gv = ldg_u8(&ktb_iq2s_grid[idx][j]);
                    v[8 * l + j] = (int8_t)(((signs >> j) & 1) ? -gv : gv);
                }
            }
            break;
        }
#endif
        default:
            o.d = 0.f; o.isc = 0;
            for (int l = 0; l < 16; l++) v[l] = 0;
    }
#pragma unroll
    for (int w = 0; w < 4; w++)
        o.q[w] = (uint32_t)(uint8_t)v[4 * w] | ((uint32_t)(uint8_t)v[4 * w + 1] << 8) |
                 ((uint32_t)(uint8_t)v[4 * w + 2] << 16) | ((uint32_t)(uint8_t)v[4 * w + 3] << 24);
}

struct FmtGenK {
    static constexpr int kType = -1;  // runtime
    static constexpr int kBlocksPerStep = 2;
    struct Lane { int blk, g; };
    struct Row { const uint8_t* p; int type; int bsz; };
    using Regs = GroupK;
    struct Act { uint4 x; float dx; int bsum; };

    __device__ static __forceinline__ Lane lane(int l) { return Lane{l >> 4, l & 15}; }
    __device__ static __forceinline__ Row row(const void* base, long row_idx, int ncols, int type) {
        const int bsz = (int)weight_block_bytes(type);
        return Row{reinterpret_cast<const uint8_t*>(base) + row_idx * (long)(ncols / QK_K) * bsz, type, bsz};
    }
    __device__ static __forceinline__ void prefetch(const Row&, int) {}
    __device__ static __forceinline__ void load(const Row& r, int blk, const Lane& L, Regs& R) {
        unpack_group16(r.type, r.p + (long)blk * r.bsz, L.g, R);
    }
    __device__ static __forceinline__ void load_act(const ActQ8K& a, int blk, const Lane& L, Act& A) {
        A.x = *reinterpret_cast<const uint4*>(a.q8 + blk * QK_K + L.g * 16);
        A.dx = a.dx[blk];
        A.bsum = a.bsums[blk * 16 + L.g];
    }
    __device__ static __forceinline__ float dot(const Regs& R, const Act& A, const Lane&) {
        int s = 0;
        s = dp4a_s8s8(R.q[0], A.x.x, s);
        s = dp4a_s8s8(R.q[1], A.x.y, s);
        s = dp4a_s8s8(R.q[2], A.x.z, s);
        s = dp4a_s8s8(R.q[3], A.x.w, s);
        return (R.d * A.dx) * (float)(R.isc * s) - (R.dmin * A.dx) * (float)(R.imn * A.bsum);
    }
};

}  // namespace ktb
