// GGUF Q4_K / Q6_K dense linears at prompt sizes (ktb200_linear_forward_prompt, DESIGN.md §4.17): the decode GEMVs stream the
// whole weight once per token chunk of at most 8 (one token at in_features 16384 / 18432); here a prompt chunk of at most
// 2048 tokens is quantised once (grp_quant_x_kernel, the grouped path's Q8_K quantiser) and gguf_gemm_kernel reads every
// weight once per chunk.  The arithmetic is the decode kernels' (DESIGN §2): per super-block an exact integer
//     Q4_K  isum = sum_j sc_j * (q_j . x8_j)        (8 sub-blocks of 32, u8 nibbles . s8)
//           msum = sum_j m_j * (sum of x8_j)         (the mins against the activation sums)
//           term = kq_min_term(d, dmin, dx, isum, msum) = (d * dx) * isum - (dmin * dx) * msum
//     Q6_K  isum = sum_s sc_s * ((q_s - 32) . x8_s)  (16 sub-blocks of 16, s8 . s8, signed 8-bit scales)
//           term = (d * dx) * isum
// summed in fp32 over the super-blocks in kb order, plus the fp32 bias, rounded once by store_hidden.  Only that fp32 order
// differs from the GEMV route.
// Integer wgmma with A in registers: each MMA thread unpacks its two weight rows of a K = 32 step (a u8 or s8 fragment, four
// registers) straight from the weight box; B is the activation box, K-major with the 128-byte swizzle.  Every sub-block's dot
// gets its own accumulator (the scale multiplies it in int32 before isum takes it).  Q4_K's msum is one more accumulator that
// runs over the whole super-block: A = each sub-block's min repeated over its 32 K positions, so the MMA sums m_j * x8 over
// the block, the same integer as the mins times the 16-value sums.  Q6_K's 16-value sub-blocks: the even one is the MMA with
// registers 2, 3 of A zeroed (K 0-15), the odd one with registers 0, 1 zeroed.
//     CTA = 128 weight rows x 64 tokens: the sub-block accumulator, isum, msum and acc are 4 x 32 registers per thread at 64
//     tokens, 256 at 128 (over the 232 an MMA thread may hold).  grid = row tiles x token tiles (banded raster, as fp8_gemm_kernel), one
//     CTA per SM; 384 threads: warps 0-7 two MMA warpgroups of 64 weight rows (setmaxnreg 232), warp 8 the TMA producer
//     (4-stage ring of one super-block each: two activation boxes [64 tokens x 128 B] and the weight boxes), warps 9-11 idle
//     (setmaxnreg 40).
// Weight boxes, no second copy of any weight:
//     Q4_K  raw blocks, a 2-D box [128 rows x 144 B] (rows of 144 B: the nibble words of 8 rows fall in 8 distinct bank quads)
//     Q6_K  the 8-row SoA layout of ktb200_linear_load_weights (repack_q6k): ql / qh / scales as 4-D boxes [16 groups][8 rows]
//           [1 block][128 / 64 / 16 B] (ql with the 128-byte swizzle, qh with the 64-byte one: conflict-free word loads);
//           the 2-byte d per (row, block) is read from global memory
#include <cuda.h>

#include "common.cuh"
#include "formats.cuh"
#include "handles.cuh"
#include "wgmma.cuh"

namespace ktb {
using namespace wg;

constexpr int kGgT = 64;                      // tokens per CTA (the MMA's N)
constexpr int kGgStages = 4;
constexpr int kGgB = kGgT * 128;              // one activation box: 64 token rows x 128 bytes of K
constexpr int kGgChunk = 2048;                // tokens per GEMM launch at most: bounds the arena
constexpr int kGgBand = 16;                   // row tiles per raster band: a wave shares weight and activation boxes in L2
constexpr int kGgConsumerWarps = 8, kGgThreads = (kGgConsumerWarps + 4) * 32;
// stage plans: [activation box 0][activation box 1][weights]
constexpr int kGgW = 2 * kGgB;
constexpr int kGgW4 = 128 * SZ_Q4_K;                                     // Q4_K: 128 rows x 144 B
constexpr int kGgQh = kGgW + 128 * 128, kGgSc = kGgQh + 128 * 64;        // Q6_K: ql 128 x 128 B, qh 128 x 64 B, scales 128 x 16 B
constexpr int kGgStage4 = kGgW + kGgW4, kGgStage6 = kGgSc + 128 * 16;
static_assert(kGgStage4 % 1024 == 0 && kGgStage6 % 1024 == 0 && kGgQh % 512 == 0, "swizzled boxes need aligned stages");
struct GgufMisc {
    unsigned long long full[kGgStages], free_[kGgStages];
};
template <int FMT>
constexpr int gg_stage() { return FMT == 0 ? kGgStage4 : kGgStage6; }
template <int FMT>
constexpr int gg_smem() { return kGgStages * gg_stage<FMT>() + (int)sizeof(GgufMisc) + 1024; }
static_assert(gg_smem<1>() <= 227 * 1024, "shared memory budget");

struct GgufGemmParams {
    void* y;                  // [T][N], already offset to the chunk
    const float* bias;        // [N] or null
    const int* bsz;
    const float* xd;          // [T][nblk] Q8_K token scales of the chunk
    const uint8_t* w;         // Q6_K: the weights (d is read from them)
    int hidden_type, T, N, nblk, row_tiles, token_tiles, t0;
};

// FMT 0: Q4_K raw, 1: Q6_K in the 8-row SoA layout.  Maps: w = the weight box (Q6_K: ql), h = Q6_K qh, s = Q6_K scales,
// x = the quantised chunk [T][K] int8.
template <int FMT>
__global__ void __launch_bounds__(kGgThreads, 1) gguf_gemm_kernel(const __grid_constant__ CUtensorMap wmap, const __grid_constant__ CUtensorMap hmap,
                                                                  const __grid_constant__ CUtensorMap smap, const __grid_constant__ CUtensorMap xmap,
                                                                  const GgufGemmParams p) {
    constexpr int kStage = gg_stage<FMT>();
    const int band_ctas = kGgBand * p.token_tiles, band = blockIdx.x / band_ctas, in_band = blockIdx.x - band * band_ctas;
    const int band_rows = min(kGgBand, p.row_tiles - band * kGgBand);
    const int rt = band * kGgBand + in_band % band_rows, tt = in_band / band_rows;
    const int live = p.bsz ? max(0, min(p.T, *p.bsz - p.t0)) : p.T;   // bsz was written before the quantiser (a full dependency)
    if (tt * kGgT >= live) return;                                    // a token tile wholly beyond the live batch: no MMA, no store
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base - raw);
    GgufMisc& misc = *reinterpret_cast<GgufMisc*>(smem + kGgStages * kStage);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        for (int s = 0; s < kGgStages; s++) { bar_init(smem_u32(&misc.full[s]), 1); bar_init(smem_u32(&misc.free_[s]), kGgConsumerWarps); }
        bar_fence_init();
        tma_prefetch_desc(&wmap); tma_prefetch_desc(&xmap);
        if (FMT == 1) { tma_prefetch_desc(&hmap); tma_prefetch_desc(&smap); }
    }
    __syncthreads();

    if (warp >= kGgConsumerWarps) {
        regs_dec<40>();
        if (warp == kGgConsumerWarps && lane == 0) {
            for (int b = 0; b < p.nblk; b++) {
                const int s = b % kGgStages;
                const uint32_t full = smem_u32(&misc.full[s]), st = base + s * kStage;
                bar_wait(smem_u32(&misc.free_[s]), ((b / kGgStages) & 1) ^ 1);
                bar_expect_tx(full, kStage);
                tma_load_2d(st, &xmap, full, b * QK_K, tt * kGgT);
                tma_load_2d(st + kGgB, &xmap, full, b * QK_K + 128, tt * kGgT);
                if (FMT == 0) {
                    tma_load_2d(st + kGgW, &wmap, full, b * SZ_Q4_K, rt * 128);
                } else {
                    tma_load_4d(st + kGgW, &wmap, full, 0, b, 0, rt * 16);
                    tma_load_4d(st + kGgQh, &hmap, full, 0, b, 0, rt * 16);
                    tma_load_4d(st + kGgSc, &smap, full, 0, b, 0, rt * 16);
                }
            }
        }
        return;
    }
    regs_inc<232>();   // 128 x 40 + 256 x 232 <= 64 K registers
    // warpgroup g owns weight rows 64 g .. 64 g + 63 of the tile; accumulator register i: row r0 + 8 ((i >> 1) & 1),
    // token 8 (i >> 2) + 2 c + (i & 1) of the tile
    const int g = warp >> 2, r0 = 64 * g + 16 * (warp & 3) + (lane >> 2), c = lane & 3;
    const int n0 = rt * 128 + r0;
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; i++) acc[i] = 0.f;
    for (int b = 0; b < p.nblk; b++) {
        const int s = b % kGgStages;
        float d6[2] = {0.f, 0.f};
        if (FMT == 1) {
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int n = n0 + 8 * h;
                if (n < p.N) d6[h] = fp16_bits_to_f32(ldg_u16(p.w + (long)(n >> 3) * 8 * SZ_Q6_K * p.nblk + 1664L * p.nblk + (long)(n & 7) * 2 * p.nblk + 2 * b));
            }
        }
        bar_wait(smem_u32(&misc.full[s]), (b / kGgStages) & 1);
        const uint8_t* st = smem + s * kStage;
        const uint32_t bx = base + s * kStage;   // activation boxes: K 0-127, 128-255 of the block
        int isum[32];
#pragma unroll
        for (int i = 0; i < 32; i++) isum[i] = 0;
        if (FMT == 0) {
            const uint8_t* w0 = st + kGgW + r0 * SZ_Q4_K;
            const uint8_t* w1 = w0 + 8 * SZ_Q4_K;
            const uint4 h0 = *reinterpret_cast<const uint4*>(w0), h1 = *reinterpret_cast<const uint4*>(w1);
            uint32_t ms[32];
#pragma unroll
            for (int q = 0; q < 4; q++) {   // qs[32 q .. 32 q + 31]: low nibbles sub-block 2 q, high nibbles 2 q + 1
                const uint32_t a00 = *reinterpret_cast<const uint32_t*>(w0 + 16 + 32 * q + 4 * c), a01 = *reinterpret_cast<const uint32_t*>(w0 + 32 + 32 * q + 4 * c);
                const uint32_t a10 = *reinterpret_cast<const uint32_t*>(w1 + 16 + 32 * q + 4 * c), a11 = *reinterpret_cast<const uint32_t*>(w1 + 32 + 32 * q + 4 * c);
                const uint32_t lo[4] = {a00 & 0x0F0F0F0Fu, a10 & 0x0F0F0F0Fu, a01 & 0x0F0F0F0Fu, a11 & 0x0F0F0F0Fu};
                const uint32_t hi[4] = {(a00 >> 4) & 0x0F0F0F0Fu, (a10 >> 4) & 0x0F0F0F0Fu, (a01 >> 4) & 0x0F0F0F0Fu, (a11 >> 4) & 0x0F0F0F0Fu};
                uint32_t sc0, mn0, sc1, mn1;   // (sub-block 2 q) | (2 q + 1) << 8 of rows r0, r0 + 8
                k4_pair(h0.y, h0.z, h0.w, 16 * (q & 1), q >= 2, sc0, mn0);
                k4_pair(h1.y, h1.z, h1.w, 16 * (q & 1), q >= 2, sc1, mn1);
                const uint32_t ml[4] = {(mn0 & 0xffu) * 0x01010101u, (mn1 & 0xffu) * 0x01010101u, (mn0 & 0xffu) * 0x01010101u, (mn1 & 0xffu) * 0x01010101u};
                const uint32_t mh[4] = {(mn0 >> 8) * 0x01010101u, (mn1 >> 8) * 0x01010101u, (mn0 >> 8) * 0x01010101u, (mn1 >> 8) * 0x01010101u};
                const uint64_t dlo = smem_desc(bx + (q >> 1) * kGgB + 64 * (q & 1), 16, 1024, kLayoutSw128);
                const uint64_t dhi = smem_desc(bx + (q >> 1) * kGgB + 64 * (q & 1) + 32, 16, 1024, kLayoutSw128);
                uint32_t v[32];   // one sub-block accumulator: the high nibbles' MMA runs after the low nibbles' scale-and-add
                fence();
                mma_u8s8_rs_m64n64(v, lo, dlo, 0);
                mma_u8s8_rs_m64n64(ms, ml, dlo, q > 0);
                mma_u8s8_rs_m64n64(ms, mh, dhi, 1);
                commit();
                wait<0>();
                fence_regs(v);
#pragma unroll
                for (int i = 0; i < 32; i++) isum[i] += (int)(((i & 2) ? sc1 : sc0) & 0xffu) * (int)v[i];
                fence();
                mma_u8s8_rs_m64n64(v, hi, dhi, 0);
                commit();
                wait<0>();
                fence_regs(v);
#pragma unroll
                for (int i = 0; i < 32; i++) isum[i] += (int)(((i & 2) ? sc1 : sc0) >> 8) * (int)v[i];
            }
            float dx[16];   // token scales of block b (rows beyond the chunk: zero, their outputs are never stored)
#pragma unroll
            for (int q = 0; q < 16; q++) {
                const int t = tt * kGgT + 8 * (q >> 1) + 2 * c + (q & 1);
                dx[q] = t < p.T ? __ldg(p.xd + (long)t * p.nblk + b) : 0.f;
            }
            fence_regs(ms);
            __syncwarp();
            if (lane == 0) bar_arrive(smem_u32(&misc.free_[s]));   // every read of the stage has completed
            const float2 dm0 = __half22float2(*reinterpret_cast<const __half2*>(&h0.x)), dm1 = __half22float2(*reinterpret_cast<const __half2*>(&h1.x));
#pragma unroll
            for (int i = 0; i < 32; i++) {
                const float2 dm = (i & 2) ? dm1 : dm0;
                acc[i] += kq_min_term(dm.x, dm.y, dx[2 * (i >> 2) + (i & 1)], isum[i], (float)(int)ms[i]);
            }
        } else {
            const int ra = r0, rb = r0 + 8;
            const uint8_t *ql = st + kGgW, *qh = st + kGgQh;
            const uint4 s0 = *reinterpret_cast<const uint4*>(st + kGgSc + ra * 16), s1 = *reinterpret_cast<const uint4*>(st + kGgSc + rb * 16);
            const uint32_t sw0[4] = {s0.x, s0.y, s0.z, s0.w}, sw1[4] = {s1.x, s1.y, s1.z, s1.w};
            // byte o of a row's ql (128-byte swizzle) / qh (64-byte swizzle) slice
            auto lq = [&](int r, int o) { return *reinterpret_cast<const uint32_t*>(ql + r * 128 + ((((o >> 4) ^ (r & 7))) << 4) + (o & 15)); };
            auto lh = [&](int r, int o) { return *reinterpret_cast<const uint32_t*>(qh + r * 64 + ((((o >> 4) ^ ((r >> 1) & 3))) << 4) + (o & 15)); };
#pragma unroll
            for (int hh = 0; hh < 2; hh++) {
                // values l (K 4 c .. 4 c + 3 and 16 + 4 c ..) of the half's four 32-value groups: ql[64 hh + l], ql[64 hh + 32 + l],
                // qh[32 hh + l] (ggml dequantize_row_q6_K)
                uint32_t L[2][4], Hq[2][2];
#pragma unroll
                for (int rr = 0; rr < 2; rr++) {
                    const int r = rr ? rb : ra;
#pragma unroll
                    for (int u = 0; u < 4; u++) L[rr][u] = lq(r, 64 * hh + 16 * u + 4 * c);
                    Hq[rr][0] = lh(r, 32 * hh + 4 * c);
                    Hq[rr][1] = lh(r, 32 * hh + 16 + 4 * c);
                }
#pragma unroll
                for (int gq = 0; gq < 4; gq++) {
                    const int m = 4 * hh + gq;   // K = 32 m .. 32 m + 31 of the block: sub-blocks 2 m (K 0-15), 2 m + 1
                    uint32_t q6[2][2];           // [row][first / second 16 values]
#pragma unroll
                    for (int rr = 0; rr < 2; rr++)
#pragma unroll
                        for (int f = 0; f < 2; f++) {
                            const uint32_t qlw = L[rr][2 * (gq & 1) + f], qhw = Hq[rr][f];
                            const uint32_t lo4 = (gq < 2) ? (qlw & 0x0F0F0F0Fu) : ((qlw >> 4) & 0x0F0F0F0Fu);
                            const uint32_t t6 = lo4 | (((qhw >> (2 * gq)) << 4) & 0x30303030u);
                            const uint32_t tt6 = t6 ^ 0x20202020u;   // q - 32 per byte: flip bit 5, copy it into bits 6 and 7
                            q6[rr][f] = tt6 + (tt6 & 0x20202020u) * 6u;
                        }
                    const uint32_t ae[4] = {q6[0][0], q6[1][0], 0u, 0u}, ao[4] = {0u, 0u, q6[0][1], q6[1][1]};
                    const uint64_t db = smem_desc(bx + hh * kGgB + 32 * gq, 16, 1024, kLayoutSw128);
                    const int sce0 = (int)(int8_t)(sw0[m >> 1] >> (16 * (m & 1))), sco0 = (int)(int8_t)(sw0[m >> 1] >> (16 * (m & 1) + 8));
                    const int sce1 = (int)(int8_t)(sw1[m >> 1] >> (16 * (m & 1))), sco1 = (int)(int8_t)(sw1[m >> 1] >> (16 * (m & 1) + 8));
                    uint32_t v[32];   // one sub-block accumulator, as Q4_K
                    fence();
                    mma_s8s8_rs_m64n64(v, ae, db, 0);
                    commit();
                    wait<0>();
                    fence_regs(v);
#pragma unroll
                    for (int i = 0; i < 32; i++) isum[i] += ((i & 2) ? sce1 : sce0) * (int)v[i];
                    fence();
                    mma_s8s8_rs_m64n64(v, ao, db, 0);
                    commit();
                    wait<0>();
                    fence_regs(v);
#pragma unroll
                    for (int i = 0; i < 32; i++) isum[i] += ((i & 2) ? sco1 : sco0) * (int)v[i];
                }
            }
            float dx[16];   // token scales of block b (rows beyond the chunk: zero, their outputs are never stored)
#pragma unroll
            for (int q = 0; q < 16; q++) {
                const int t = tt * kGgT + 8 * (q >> 1) + 2 * c + (q & 1);
                dx[q] = t < p.T ? __ldg(p.xd + (long)t * p.nblk + b) : 0.f;
            }
            __syncwarp();
            if (lane == 0) bar_arrive(smem_u32(&misc.free_[s]));
#pragma unroll
            for (int i = 0; i < 32; i++) acc[i] += iq_term(d6[(i >> 1) & 1], dx[2 * (i >> 2) + (i & 1)], isum[i]);
        }
    }
    const int live_end = p.bsz ? max(0, min(p.T, *p.bsz - p.t0)) : p.T;   // re-read: one register less across the K loop
#pragma unroll
    for (int i = 0; i < 32; i++) {
        const int t = tt * kGgT + 8 * (i >> 2) + 2 * c + (i & 1), n = n0 + 8 * ((i >> 1) & 1);
        if (t < live_end && n < p.N) store_hidden(p.y, (long)t * p.N + n, p.hidden_type, p.bias ? acc[i] + __ldg(p.bias + n) : acc[i]);
    }
}

typedef CUresult (*EncodeTiledFnG)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFnG encode_tiled_g() {
    static EncodeTiledFnG fn = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) f = nullptr;
        return (EncodeTiledFnG)f;
    }();
    return fn;
}

// -1: the GEMM does not take this weight (type, layout)
static int gg_fmt(int type, int layout) {
    if (type == KTB200_TYPE_Q4_K) return 0;
    if (type == KTB200_TYPE_Q6_K && layout == LAYOUT_SOA8) return 1;
    return -1;
}

// The qlen from which the GEMM is the faster route; 0: never.  Up to 64 tokens the GEMM costs one token tile whatever the
// count, so the crossover is where the GEMV's passes overtake it.  Measured at DeepSeek-V3's module shapes with
// tools/gguf_prefill_probe.py (DESIGN.md §4.17):
//   N <= 1024   (kv_a: 5 row tiles, few CTAs per token tile)   from 24 tokens (16 is faster on the GEMV)
//   otherwise                                                  from 16 tokens, the floor: 8-token calls keep the GEMV, which
//                                                              the GEMM beats at 8 only where the GEMV takes one token per
//                                                              pass (o_proj) or tokens in grid.y (Q6_K, q_b's FmtQ4K rows)
int gguf_prompt_min(int type, int layout, int K, int N) {
    (void)K;
    return gg_fmt(type, layout) < 0 ? 0 : N <= 1024 ? 24 : 16;
}

int gguf_forward_prompt(const void* w, int type, int layout, int K, int N, int hidden_type, int dev, int qlen, const void* x, void* y,
                        const float* bias, const int* bsz, cudaStream_t s) {
    const int fmt = gg_fmt(type, layout);
    if (fmt < 0) {
        if (type == KTB200_TYPE_Q6_K)
            set_error("linear prompt route: this Q6_K handle keeps the raw block layout (out_features %% 8 != 0 or rows too long for the "
                      "8-row SoA re-layout); it takes ktb200_linear_forward only");
        else
            set_error("linear prompt route: %s weights take ktb200_linear_forward only (the tiled GEMM takes Q4_K and Q6_K)",
                      type == KTB200_TYPE_Q2_K ? "Q2_K" : type == KTB200_TYPE_Q3_K ? "Q3_K" : type == KTB200_TYPE_Q5_K ? "Q5_K"
                      : type == KTB200_TYPE_IQ4_XS ? "IQ4_XS" : "these");
        return KTB200_EINVAL;
    }
    EncodeTiledFnG enc = encode_tiled_g();
    if (!enc) { set_error("linear prompt route: cuTensorMapEncodeTiled is not available from this driver"); return KTB200_ECUDA; }
    // qlen tokens in balanced chunks of whole token tiles (at most kGgChunk): per chunk one quantiser and one GEMM launch
    const int nch = (qlen + kGgChunk - 1) / kGgChunk;
    const int Tc = ((qlen + nch - 1) / nch + kGgT - 1) / kGgT * kGgT;
    GrpX xb;
    // grow to a whole chunk at this K, so that one warm-up call of any prompt length covers every later length
    int rc = grp_prompt_x(dev, (size_t)Tc * K, (size_t)kGgChunk * K, s, &xb);
    if (rc == KTB200_ESTATE) {
        set_error("linear prompt route: this call needs %zu bytes of Q8_K prompt scratch on device %d, more than the arena holds; the arena "
                  "cannot grow while the stream is capturing: run one eager ktb200_linear_forward_prompt call at in_features >= %d on this "
                  "device before capture", (size_t)Tc * K, dev, K);
        return rc;
    }
    if (rc) return rc;
    static bool attr[64] = {};
    if (!attr[dev & 63]) {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(gguf_gemm_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, gg_smem<0>()));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(gguf_gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, gg_smem<1>()));
        attr[dev & 63] = true;
    }
    const int nblk = K / QK_K, row_tiles = (N + 127) / 128;
    const cuuint32_t e1[2] = {1, 1}, e4[4] = {1, 1, 1, 1};
    CUtensorMap wmap, hmap, smap;
    CUresult cr;
    void* wp = const_cast<void*>(w);
    if (fmt == 0) {   // rows beyond N are filled with zeros by TMA; no output of theirs is stored
        const cuuint64_t dim[2] = {(cuuint64_t)nblk * SZ_Q4_K, (cuuint64_t)N}, str[1] = {(cuuint64_t)nblk * SZ_Q4_K};
        const cuuint32_t box[2] = {SZ_Q4_K, 128};
        cr = enc(&wmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, wp, dim, str, box, e1, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        hmap = wmap; smap = wmap;
    } else {          // [N / 8 groups][8 rows][nblk blocks][bytes] inside each SoA section (ql at 0, qh at 1024 nblk, scales at 1536 nblk)
        const cuuint64_t gs = (cuuint64_t)8 * SZ_Q6_K * nblk;
        const int bytes[3] = {128, 64, 16};
        const size_t off[3] = {0, (size_t)1024 * nblk, (size_t)1536 * nblk};
        const CUtensorMapSwizzle swz[3] = {CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_SWIZZLE_NONE};
        CUtensorMap* maps[3] = {&wmap, &hmap, &smap};
        cr = CUDA_SUCCESS;
        for (int i = 0; i < 3 && cr == CUDA_SUCCESS; i++) {
            const cuuint64_t dim[4] = {(cuuint64_t)bytes[i], (cuuint64_t)nblk, 8, (cuuint64_t)N / 8};
            const cuuint64_t str[3] = {(cuuint64_t)bytes[i], (cuuint64_t)bytes[i] * nblk, gs};
            const cuuint32_t box[4] = {(cuuint32_t)bytes[i], 1, 8, 16};
            cr = enc(maps[i], CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, reinterpret_cast<uint8_t*>(wp) + off[i], dim, str, box, e4, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swz[i], CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        }
    }
    if (cr != CUDA_SUCCESS) { set_error("linear prompt route: cuTensorMapEncodeTiled failed for the weights (%d)", (int)cr); return KTB200_ECUDA; }
    const size_t hb = type_size(hidden_type);
    for (int t0 = 0; t0 < qlen; t0 += Tc) {
        const int T = qlen - t0 < Tc ? qlen - t0 : Tc;
        CUtensorMap xmap;   // rows T .. of a token tile are filled with zeros by TMA; no output of theirs is stored
        const cuuint64_t xdim[2] = {(cuuint64_t)K, (cuuint64_t)T}, xstr[1] = {(cuuint64_t)K};
        const cuuint32_t xbox[2] = {128, kGgT};
        cr = enc(&xmap, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, xb.q, xdim, xstr, xbox, e1, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (cr != CUDA_SUCCESS) { set_error("linear prompt route: cuTensorMapEncodeTiled failed for the prompt scratch (%d)", (int)cr); return KTB200_ECUDA; }
        rc = grp_prompt_quant(reinterpret_cast<const uint8_t*>(x) + (size_t)t0 * K * hb, hidden_type, T, K, xb, s);
        if (rc) return rc;
        GgufGemmParams p{};
        p.y = reinterpret_cast<uint8_t*>(y) + (size_t)t0 * N * hb;
        p.bias = bias; p.bsz = bsz; p.xd = xb.d; p.w = reinterpret_cast<const uint8_t*>(w); p.t0 = t0;
        p.hidden_type = hidden_type; p.T = T; p.N = N; p.nblk = nblk; p.row_tiles = row_tiles; p.token_tiles = (T + kGgT - 1) / kGgT;
        if (fmt == 0) gguf_gemm_kernel<0><<<p.row_tiles * p.token_tiles, kGgThreads, gg_smem<0>(), s>>>(wmap, hmap, smap, xmap, p);
        else gguf_gemm_kernel<1><<<p.row_tiles * p.token_tiles, kGgThreads, gg_smem<1>(), s>>>(wmap, hmap, smap, xmap, p);
        KTB_LAUNCH_CHECK();
    }
    return KTB200_OK;
}
}  // namespace ktb
