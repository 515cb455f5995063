// Grouped expert GEMM for prefill-sized batches on the Hopper tensor path — MOE::forward_many
// (archive/csrc/ktransformers_ext/operators/llamafile/moe.cpp:248-365 ≡ kt-kernel/operators/llamafile/moe.hpp:461-746):
//     count tokens per expert -> per-token Q8_K quantisation + scatter into per-expert contiguous order ->
//     per-expert GEMM (gate, up) -> silu * mul -> requantise -> per-expert GEMM (down) -> per-token weighted gather.
// The decode kernels stream every (token, expert) pair's weights; here an expert's weights are read ONCE per 32-token tile.
//
// Arithmetic: the reference's dot is an exact integer per super-block — sum_j sc_j * (sum over sub-block j of q * x8) — scaled in
// fp32.  The integer tensor path (wgmma u8/s8 . s8 -> s32) computes the INNER sums exactly: one MMA of K = 32 per Q4_K sub-block
// (A = the raw 4-bit quants as u8, B = the Q8_K activation bytes), its own accumulator per sub-block; Q6_K sub-blocks are 16
// long, so one K = 32 MMA covers two of them against a B operand of 64 rows — the 32 tokens with the odd sub-block zeroed, then
// the 32 tokens with the even one zeroed.  The MMA warpgroups multiply every accumulator by its 6/8-bit sub-block scale in
// int32, convert ONCE per super-block and apply (d_w * d_x) * isum - (dmin_w * d_x) * msum in fp32, the decode kernels'
// formula; msum (Q4_K mins x activation block sums) is one K = 16 fp16 MMA of exact small integers.
// Nothing is rounded that the reference does not round.
//
// grouped_gemm_kernel: persistent CTAs, tile = (expert, 128 weight rows, 32 tokens), stage = half a super-block (128 of K):
//     warps 0-7    producers (half a weight row per thread): weights (global, 16-byte loads, next stage prefetched in registers) -> int8 A tile in the K-major
//                  128-byte-swizzle layout (Q4_K: nibble split; Q6_K: 4 + 2 bit merge, -32); activation rows gathered through the
//                  sorted pair list -> B tile; row headers (scales, d, dmin) and token scales for the scale-and-add
//     warps 8-15   two MMA warpgroups, 64 weight rows each: the integer MMAs of a stage (+ the mins MMA on the second half),
//                  int32 scale-and-add in registers, fp32 finish per super-block, stores at the end of the tile; 3 shared-memory
//                  stages between the two roles
//
// IQ1_S (FMT 2) and IQ2_XXS (FMT 3), DeepSeek-R1's codebook experts: 32-value sub-blocks with one odd integer scale ls each and
// no mins, so the Q4_K shape minus its mins MMA.  The producers expand the codebooks (staged in shared memory from iq_tables.h)
// into the s8 A tile — IQ1_S 8 * grid + delta (-9..9), IQ2_XXS +-grid — the operands the decode kernels (iq.cuh) feed to dp4a;
// one s8.s8 K = 32 MMA per sub-block, isum += ls * that, and per super-block the decode kernels' iq_term((d/8), dx, isum).
// The raw blocks (50 / 66 B) are only 2-byte aligned: a producer fetches the aligned 4-byte words that cover its bytes with
// cp.async and funnel-shifts them by 16 bits when the block starts on an odd half-word (the block parity, tracked per row).
// That keeps the Q4_K producers' asynchronous 6-stage prefetch; 16-bit loads staged in registers would hold those stages in
// the producers' 96 registers and take two to four times the load instructions.  Their own shared-memory plan: no mins tiles,
// 32-row B, 48-byte raw slots and the 16 KB codebook in place of the Q4_K / Q6_K plan's 80-byte slots.
//
// Q5_K (FMT 5), Q3_K (FMT 6) and Q2_K (FMT 7), the other K-quants of llama.cpp's expert mixes, reuse those two shapes:
//   Q5_K  the Q4_K path with the fifth bit: bit 2c / 2c + 1 of qh[l] ORed in as bit 4 of the u8 operand (0..31); same header,
//         mins MMA and finish.  Seven 16-byte raw units per thread (qh adds two), so a 112-byte pitch (odd multiple of 16)
//         and a 4-deep raw ring in the region of the 6-deep 80-byte one.
//   Q3_K  the Q6_K path: s8 operands q - 4 (hmask bit clear) in -4..3, the 6-bit scales - 32 as the header's 8 signed bytes,
//         finish (d * dx) * isum.  110-byte blocks are 2-byte aligned: covering 4-byte words + 16-bit funnel shift (as IQ).
//   Q2_K  the Q6_K sub-block MMAs on operands 0..3, the 4-bit scales in the int32 scale-and-add, the 16 4-bit mins through
//         the Q4_K mins MMA (K = 16, one min per 16-value sum) and Q4_K's finish.  84-byte blocks: 4-byte cp.async words.
// Q3_K / Q2_K split a row's stage between its two producer threads by byte position l (as Q6_K), so a thread converts 16 qs
// (and 16 hmask) bytes and the 80-byte plan holds its share.
// IQ1_M (FMT 8), the experts of DeepSeek-R1's 1.73-bit files: IQ1_S's codebook with an odd scale ls per 16 values and the delta
// per 8, so FMT 2's producers (sub-blocks 4 hh + 2 part + {0, 1}, 8 * grid + delta from the staged codebook) feeding the Q6_K
// MMAs (one K = 32 MMA per sub-block against the 64-row B, the two halves' ls as the header's signed bytes) and Q3_K's finish
// with d / 8.  56-byte blocks are 8-byte aligned: a thread's 8 B of qs, 4 B of qh and the 8-byte scale field (which holds d) are
// plain cp.async words in FMT 2's 48-byte raw slots; own plan constants (kGSmemM) for the 64-row B.
// IQ3_XXS (FMT 9) and IQ3_S (FMT 10), the experts of llama.cpp's 3-bit i-quant files: FMT 3 with 4-value codebook groups.  The
// producers expand +-grid (IQ3_XXS 256 x 4, values 4..62, signs through IQ2_XXS's masks; IQ3_S 512 x 4, values 1..15, its sign
// bytes through a 256-entry mask table) into the s8 A tile; the consumers are FMT 3's (32-row B, one K = 32 MMA per sub-block,
// ls = 2s + 1 from the header) and the finish is iq_term with d / 4 (IQ3_XXS) or d (IQ3_S).  A thread's share of a stage
// (two sub-blocks) does not fit the 20 payload bytes of FMT 2's raw slots: the covering 4-byte words of the 98 / 110-byte
// blocks (2-byte aligned, funnel-shifted as FMT 2) are at most 36 B (qs 20, sign / scale words 12, d 4) and 44 B (qs 20, qh 4,
// signs 12, scales 4, d 4).  Own plan (kGSmem3): the IQ plan with Q4_K's 80-byte raw slots and a 4 KB codebook region.
// IQ2_XS (FMT 11) and IQ2_S (FMT 12), the experts of llama.cpp's IQ2_XS / IQ2_S / IQ2_M files: IQ2_XXS's +-grid values with an
// odd scale ls per 16 values, so IQ1_M's consumers (the Q6_K MMAs against the 64-row B, the two halves' ls as the header's
// signed bytes, the d / 8 finish).  The producers expand +-grid (IQ2_XS 512 x 8 with 9-bit indices, signs through IQ2_XXS's
// masks; IQ2_S 1024 x 8 with 10-bit indices, its sign bytes through IQ3_S's mask table) into the s8 A tile.  The covering
// words of a thread's two sub-blocks in the 74 / 82-byte blocks (2-byte aligned, funnel-shifted as FMT 2) are at most 28 B (qs
// 20, scales 4, d 4) and 36 B (qs 12, signs 12, qh 4, scales 4, d 4): IQ3's 80-byte raw slots.  Own plan (kGSmemI2): the IQ1_M
// plan with those slots and a 10 KB codebook region.
#include <cuda_fp16.h>

#include "act_quant.cuh"
#include "common.cuh"
#include "handles.cuh"
#include "wgmma.cuh"
#define KTB_IQ_TABLE static __device__ const
#include "iq_tables.h"
#include "iq3_tables.h"
#include "iq2_tables.h"

namespace ktb {

using namespace wg;

constexpr int kGM = 128, kGN = 32, kGStages = 3, kGRaw = 6, kGHdr = 6;
constexpr int kGProdWarps = 8, kGMmaWarps = 8, kGThreads = (kGProdWarps + kGMmaWarps) * 32;   // 16 warps: producers 96 registers, MMA warpgroups 160
constexpr int kGA = kGM * 128;            // 16,384: 128 rows x 128 int8 of K, one swizzle atom column
constexpr int kGB = 2 * kGN * 128;        //  8,192: 32 rows (Q4_K) or 64 rows (Q6_K even / odd variants)
constexpr int kGA2 = kGM * 32, kGB2 = kGN * 32;
constexpr int kRawPitch = 80, kRawSlot = 2 * kGM * kRawPitch;   // 5 x 16 bytes per producer thread and stage (odd pitch: conflict-free LDS.128)
constexpr int kOffB = kGStages * kGA, kOffA2 = kOffB + kGStages * kGB, kOffB2 = kOffA2 + kGStages * kGA2, kOffRaw = kOffB2 + kGStages * kGB2,
              kOffMiscG = kOffRaw + kGRaw * kRawSlot;

struct GrpMisc {
    unsigned long long ab_full[kGStages], smem_free[kGStages], hdr_free[kGHdr];
    // what only the scale-and-add reads rides in its own, deeper ring
    float dxs[kGHdr][kGN];
    uint4 hdr[kGHdr][kGM];      // Q4_K: the block header (d, dmin, 12 scale bytes); Q6_K: 8 scales of the half, d as f32
};
constexpr int kGSmem = kOffMiscG + (int)sizeof(GrpMisc) + 1024;
static_assert(kGSmem <= 227 * 1024, "shared memory budget");
// Q5_K: the kGSmem plan with seven-unit raw slots (7 x 16 = 112 bytes, an odd multiple of 16) 4 deep in the raw region
constexpr int kGRaw5 = 4, kRawPitch5 = 112, kRawSlot5 = 2 * kGM * kRawPitch5;
static_assert(kGRaw5 * kRawSlot5 <= kGRaw * kRawSlot, "Q5_K raw ring");
// IQ1_S / IQ2_XXS plan: A stages as above, B of 32 token rows, raw slots of three 16-byte units per thread (0-1 the covering
// weight words and the word of d, 24 the token scale, 2 the activation piece), the codebook (IQ1_S 2048 x 8 B; IQ2_XXS 256 x 8 B
// grid + 128 x 8 B sign masks), the same misc block
constexpr int kGBI = kGN * 128, kRawPitchI = 48, kRawSlotI = 2 * kGM * kRawPitchI, kTabI = 2048 * 8;
constexpr int kOffBI = kGStages * kGA, kOffRawI = kOffBI + kGStages * kGBI, kOffTabI = kOffRawI + kGRaw * kRawSlotI, kOffMiscI = kOffTabI + kTabI;
constexpr int kGSmemI = kOffMiscI + (int)sizeof(GrpMisc) + 1024;
static_assert(kGSmemI <= 227 * 1024 && kOffBI % 1024 == 0 && kGBI % 1024 == 0, "IQ shared-memory plan");
// IQ1_M plan: the IQ plan with the 64-row B of the 16-value sub-block formats (even / odd halves zeroed)
constexpr int kOffBM = kGStages * kGA, kOffRawM = kOffBM + kGStages * kGB, kOffTabM = kOffRawM + kGRaw * kRawSlotI, kOffMiscM = kOffTabM + kTabI;
constexpr int kGSmemM = kOffMiscM + (int)sizeof(GrpMisc) + 1024;
static_assert(kGSmemM <= 227 * 1024 && kOffBM % 1024 == 0 && kGB % 1024 == 0, "IQ1_M shared-memory plan");
// IQ3_XXS / IQ3_S plan: the IQ plan with the 80-byte raw slots of the Q4_K plan and the IQ3 codebooks (IQ3_XXS 256 x 4 B grid +
// 128 x 8 B sign masks; IQ3_S 512 x 4 B grid + 256 x 8 B sign masks)
constexpr int kTab3 = 512 * 4 + 256 * 8;
constexpr int kOffB3 = kGStages * kGA, kOffRaw3 = kOffB3 + kGStages * kGBI, kOffTab3 = kOffRaw3 + kGRaw * kRawSlot, kOffMisc3 = kOffTab3 + kTab3;
constexpr int kGSmem3 = kOffMisc3 + (int)sizeof(GrpMisc) + 1024;
static_assert(kGSmem3 <= 227 * 1024 && kOffB3 % 1024 == 0 && kGBI % 1024 == 0 && kOffRaw3 % 16 == 0, "IQ3 shared-memory plan");
// IQ2_XS / IQ2_S plan: the IQ1_M plan (64-row B) with the 80-byte raw slots and the IQ2 codebooks (IQ2_XS 512 x 8 B grid +
// 128 x 8 B sign masks; IQ2_S 1024 x 8 B grid + 256 x 8 B sign masks)
constexpr int kTabI2 = 1024 * 8 + 256 * 8;
constexpr int kOffBI2 = kGStages * kGA, kOffRawI2 = kOffBI2 + kGStages * kGB, kOffTabI2 = kOffRawI2 + kGRaw * kRawSlot, kOffMiscI2 = kOffTabI2 + kTabI2;
constexpr int kGSmemI2 = kOffMiscI2 + (int)sizeof(GrpMisc) + 1024;
static_assert(kGSmemI2 <= 227 * 1024 && kOffBI2 % 1024 == 0 && kGB % 1024 == 0 && kOffRawI2 % 16 == 0, "IQ2_XS / IQ2_S shared-memory plan");

struct GrpGemmParams {
    const uint8_t* w;          // expert weights
    long expert_bytes;         // bytes per expert
    int R, Kc;                 // rows per expert, reduction length
    const int8_t* xq;          // activations: int8 [rows][Kc]
    const float* xd;           // [rows][Kc / 256]
    const int16_t* xbs;        // [rows][Kc / 16]
    const int* rowmap;         // sorted position -> activation row (null: identity)
    const int4* tinfo;         // [tiles] {expert, first weight row, first sorted position, valid tokens}
    const int* nt_prefix;      // [E + 1] 32-token tiles before every expert
    int E;
    float* out;                // [P][R] fp32
    long long* trace;          // optional (ktb200_debug_grouped): clock64 stamps of CTA 0, [role 3][stage 96][4] (role 2 unused)
};

// byte b of a register array (b is a compile-time constant after unrolling: no local-memory byte addressing)
__device__ __forceinline__ int ub(const uint32_t* a, int b) { return (int)((a[b >> 2] >> ((b & 3) * 8)) & 0xffu); }
__device__ __forceinline__ int sb8(const uint32_t* a, int b) { return (int)(int8_t)((a[b >> 2] >> ((b & 3) * 8)) & 0xffu); }
__device__ __forceinline__ uint32_t h2(int a, int b) {
    const __half2 v = __halves2half2(__int2half_rn(a), __int2half_rn(b));
    return *reinterpret_cast<const uint32_t*>(&v);
}
// the 6-bit (scale, min) pair j of a Q4_K header held as 4 words (get_scale_min_k4, ggml-quants.c)
__device__ __forceinline__ void q4k_scale_min(const uint32_t* hw, int j, int& sc, int& mn) {
    if (j < 4) { sc = ub(hw, 4 + j) & 63; mn = ub(hw, 8 + j) & 63; }
    else { sc = (ub(hw, 8 + j) & 0xF) | ((ub(hw, j) >> 6) << 4); mn = (ub(hw, 8 + j) >> 4) | ((ub(hw, 4 + j) >> 6) << 4); }
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async8(uint32_t dst, const void* src) { asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src) { asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// tile table: tile -> (expert, row tile, token tile), token tile fastest so that CTAs running side by side share the weight tile
// through L2.  One thread per tile; tiles beyond the data-dependent total are left alone.
__global__ void grp_tiles_kernel(const int* nt_prefix, const int* offsets, int E, int MT, int4* tinfo) {
    const int tile = blockIdx.x * blockDim.x + threadIdx.x;
    if (tile >= nt_prefix[E] * MT) return;
    int lo = 0, hi = E;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (nt_prefix[mid] * MT <= tile) lo = mid; else hi = mid;
    }
    const int local = tile - nt_prefix[lo] * MT, ntile_e = nt_prefix[lo + 1] - nt_prefix[lo];
    const int mt = local / ntile_e, nt = local - mt * ntile_e;
    const int p0 = offsets[lo] + nt * kGN;
    tinfo[tile] = make_int4(lo, mt * kGM, p0, min(kGN, offsets[lo + 1] - p0));
}

// A producer thread's share of one stage, as it sits in its raw-ring slot (five 16-byte units, thread = (weight row, half `part`)):
//   Q4_K: 0-1 the 32 bytes of qs of chunk 2 hh + part, 2 block header, 3 activation piece, 4 activation 16-sums (threads 0-63) or
//         token scale (threads 64-95)
//   Q6_K: 0-1 ql (16 bytes at l and at 32 + l), 2 qh, 3 activation piece, 4 = 8 scales | d (2 of 4 bytes) | token scale (threads 64-95)
//   IQ (three units, sub-blocks 4 hh + 2 part + {0, 1}): IQ1_S bytes 0-11 the words covering qs[8 (2 hh + part) .. + 8],
//         12-19 those covering qh[2 (2 hh + part) .. + 2]; IQ2_XXS 0-19 those covering the 16 bytes of the two sub-blocks;
//         20 the word holding d, 24 token scale (threads 64-95), 2 activation piece
//   Q5_K: Q4_K's five units, 5-6 the 32 bytes of qh
//   Q3_K (l = 16 part + 0..15 of the half): bytes 0-15 the words covering scales[12] and d, 16-35 those covering hmask[l],
//         36-55 those covering qs[32 hh + l], 56 token scale (threads 64-95), 4 activation piece
//   Q2_K: 0 scales[16], 1 qs[32 hh + l], 2 d | dmin (bytes 32-35), 3 activation piece, 4 as Q4_K
//   IQ1_M (the IQ slots, sub-blocks q = 2 hh + part times 2 + {0, 1}): bytes 0-7 qs[8 q .. + 8], 8-11 qh[4 q .. + 4], 16-23 the
//         scale words (d and word q's ls), 24 token scale (threads 64-95), 2 activation piece
//   IQ3 (five units, sub-blocks 2 q, 2 q + 1, q = 2 hh + part; "covering" = the aligned words over the field, a last one only when
//         the block starts on a word): bytes 0-19 those covering qs[16 q .. + 16]; IQ3_XXS 20-31 those covering its two sign /
//         scale words, 32 the word holding d; IQ3_S 20 the word holding qh[2 q .. + 2], 24-35 those covering signs[8 q .. + 8],
//         36 the word holding scales[q], 40 the word holding d; 44 token scale (threads 64-95), 3 activation piece
//   IQ2 (IQ3's five units and sub-blocks): IQ2_XS bytes 0-19 those covering qs[16 q .. + 16] (eight uint16), 20 the word holding
//         scales[2 q .. + 2], 24 the word holding d; IQ2_S 0-11 those covering qs[8 q .. + 8], 12-23 those covering
//         signs[8 q .. + 8], 24 the word holding qh[2 q .. + 2], 28 the word holding scales[2 q .. + 2], 32 the word holding d;
//         44 token scale (threads 64-95), 3 activation piece
template <int FMT>
__global__ void __launch_bounds__(kGThreads, 1) grouped_gemm_kernel(const GrpGemmParams p) {
    constexpr bool IQ = FMT == 2 || FMT == 3;
    constexpr bool K4 = FMT == 0 || FMT == 5;                 // 32-value sub-blocks with mins, u8 operands (Q4_K, Q5_K)
    constexpr bool MINS = K4 || FMT == 7;                     // the mins MMA and Q4_K's finish (Q4_K, Q5_K, Q2_K)
    // 16-value sub-blocks on the 64-row B (Q6_K, Q3_K, Q2_K, IQ1_M, IQ2_XS, IQ2_S)
    constexpr bool SUB16 = FMT == 1 || FMT == 6 || FMT == 7 || FMT == 8 || FMT == 11 || FMT == 12;
    constexpr bool IQM = FMT == 8;                            // IQ1_M: the IQ raw slots and codebook, the Q6_K MMAs
    constexpr bool IQS = IQ || IQM;                           // the IQ raw-slot layout
    constexpr bool IQ3 = FMT == 9 || FMT == 10;               // IQ3_XXS, IQ3_S: FMT 3's consumers, own raw slots and codebooks
    constexpr bool IQ2 = FMT == 11 || FMT == 12;              // IQ2_XS, IQ2_S: IQ1_M's consumers, IQ3's raw slots, own codebooks
    constexpr int nRaw = FMT == 5 ? kGRaw5 : kGRaw;
    constexpr int offB = IQ ? kOffBI : IQM ? kOffBM : IQ3 ? kOffB3 : IQ2 ? kOffBI2 : kOffB, strideB = (IQ || IQ3) ? kGBI : kGB,
                  offRaw = IQ ? kOffRawI : IQM ? kOffRawM : IQ3 ? kOffRaw3 : IQ2 ? kOffRawI2 : kOffRaw,
                  rawPitch = IQS ? kRawPitchI : FMT == 5 ? kRawPitch5 : kRawPitch, rawSlot = IQS ? kRawSlotI : FMT == 5 ? kRawSlot5 : kRawSlot,
                  BS = FMT == 2 ? SZ_IQ1_S : FMT == 3 ? SZ_IQ2_XXS : FMT == 6 ? SZ_Q3_K : FMT == 8 ? SZ_IQ1_M : FMT == 9 ? SZ_IQ3_XXS
                     : FMT == 10 ? SZ_IQ3_S : FMT == 11 ? SZ_IQ2_XS : FMT == 12 ? SZ_IQ2_S : SZ_Q2_K;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base - raw);
    GrpMisc& misc = *reinterpret_cast<GrpMisc*>(smem + (IQ ? kOffMiscI : IQM ? kOffMiscM : IQ3 ? kOffMisc3 : IQ2 ? kOffMiscI2 : kOffMiscG));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nblk = p.Kc / QK_K, nst = 2 * nblk, MT = p.R / kGM;
    uint2* tab = reinterpret_cast<uint2*>(smem + (IQM ? kOffTabM : IQ3 ? kOffTab3 : IQ2 ? kOffTabI2 : kOffTabI));   // IQ codebooks (read after the __syncthreads below)
    uint32_t* tab4 = reinterpret_cast<uint32_t*>(tab);   // IQ3 grids (4 bytes per entry); their sign masks follow them
    if (FMT == 2 || IQM) {
        for (int i = tid; i < 2048; i += kGThreads) tab[i] = *reinterpret_cast<const uint2*>(ktb_iq1s_grid[i]);
    } else if (FMT == 3) {
        for (int i = tid; i < 256; i += kGThreads) tab[i] = *reinterpret_cast<const uint2*>(ktb_iq2xxs_grid[i]);
        if (tid < 128) tab[256 + tid] = iq2_sign_masks(ktb_ksigns_iq2xs[tid]);
    } else if (FMT == 9) {
        for (int i = tid; i < 256; i += kGThreads) tab4[i] = *reinterpret_cast<const uint32_t*>(ktb_iq3xxs_grid[i]);
        if (tid < 128) tab[128 + tid] = iq2_sign_masks(ktb_ksigns_iq2xs[tid]);
    } else if (FMT == 10) {
        for (int i = tid; i < 512; i += kGThreads) tab4[i] = *reinterpret_cast<const uint32_t*>(ktb_iq3s_grid[i]);
        if (tid < 256) tab[256 + tid] = iq2_sign_masks(tid);
    } else if (FMT == 11) {
        for (int i = tid; i < 512; i += kGThreads) tab[i] = *reinterpret_cast<const uint2*>(ktb_iq2xs_grid[i]);
        if (tid < 128) tab[512 + tid] = iq2_sign_masks(ktb_ksigns_iq2xs[tid]);
    } else if (FMT == 12) {
        for (int i = tid; i < 1024; i += kGThreads) tab[i] = *reinterpret_cast<const uint2*>(ktb_iq2s_grid[i]);
        if (tid < 256) tab[1024 + tid] = iq2_sign_masks(tid);
    }
    if (tid == 0) {
        for (int s = 0; s < kGStages; s++) { bar_init(smem_u32(&misc.ab_full[s]), kGProdWarps); bar_init(smem_u32(&misc.smem_free[s]), kGMmaWarps); }
        for (int s = 0; s < kGHdr; s++) bar_init(smem_u32(&misc.hdr_free[s]), kGMmaWarps);
        bar_fence_init();
    }
    __syncthreads();
    const int total_tiles = p.nt_prefix[p.E] * MT;
    int stage = 0, sphase = 0;   // shared-memory stage of the current iteration and how often it has wrapped (parity)
    int hs = 0, hphase = 0;      // the same for the header ring

    if (warp < kGProdWarps) {
        // ========================================================================== producers: thread = (weight row r, half `part`)
        // `part` is warp-uniform (warps 0-3: first half of the row's share, warps 4-7: second) so that no branch below diverges
        regs_dec<96>();
        const int pt = tid, r = pt & (kGM - 1), part = pt >> 7, sw = r & 7, bn = pt >> 3, pc = pt & 7;
        const uint32_t raw_dst = base + offRaw + pt * rawPitch;
        const uint8_t* raw_src = smem + offRaw + pt * rawPitch;
        const int c16 = 4 * nblk * 16;   // Q6_K tiles: bytes between two 16-byte chunk planes of an item
        // fetch cursor: runs kGRaw stages ahead of the conversion, across tile boundaries; plain running pointers
        int ftile = blockIdx.x, fst = 0, ffi = 0;
        const uint8_t *fw = nullptr, *fitem = nullptr;
        const int8_t* fxq = nullptr;
        const int16_t* fbs = nullptr;
        const float* fdx = nullptr;
        auto enter_tile = [&]() {
            if (ftile >= total_tiles) return;
            const int4 ti = __ldg(p.tinfo + ftile);
            fxq = nullptr; fbs = nullptr; fdx = nullptr;
            if (bn < ti.w) fxq = p.xq + (long)(p.rowmap ? __ldg(p.rowmap + ti.z + bn) : ti.z + bn) * p.Kc + pc * 16;
            if (MINS && pt < 64 && (pt >> 1) < ti.w) fbs = p.xbs + (long)(p.rowmap ? __ldg(p.rowmap + ti.z + (pt >> 1)) : ti.z + (pt >> 1)) * (p.Kc / 16) + (pt & 1) * 8;
            if (pt >= 64 && pt < 96 && pt - 64 < ti.w) fdx = p.xd + (long)(p.rowmap ? __ldg(p.rowmap + ti.z + pt - 64) : ti.z + pt - 64) * nblk;
            const int row = ti.y + r;
            if (FMT == 0) fw = p.w + (long)ti.x * p.expert_bytes + (long)row * nblk * SZ_Q4_K + 16 + part * 32;   // this thread's qs of block 0, first half
            else if (FMT == 5) fw = p.w + (long)ti.x * p.expert_bytes + (long)row * nblk * SZ_Q5_K + 48 + part * 32;
            else if (IQ || FMT >= 6) fw = p.w + (long)ti.x * p.expert_bytes + (long)row * nblk * BS;              // block 0 of the row
            else {
                fitem = p.w + (long)ti.x * p.expert_bytes + (long)(row >> 2) * 4 * nblk * SZ_Q6_K;
                ffi = (row & 3) * nblk;
                fw = fitem + (long)ffi * 16 + part * c16;
            }
        };
        auto issue = [&](uint32_t dst) {
            if (ftile < total_tiles) {
                const int hh = fst & 1;
                if (K4) {
                    const uint8_t* q = fw + hh * 64;
                    cp_async16(dst, q);
                    cp_async16(dst + 16, q + 16);
                    if (part == 0 || hh == 1) cp_async16(dst + 32, fw - (FMT == 5 ? 48 : 16) - part * 32);
                    if (FMT == 5) {   // qh[0..31]
                        cp_async16(dst + 80, fw - 32 - part * 32);
                        cp_async16(dst + 96, fw - 16 - part * 32);
                    }
                } else if (FMT == 6) {
                    // the words covering hmask[l] and qs[32 hh + l] (l = 16 part + 0..15): a fifth one only when the block starts
                    // mid-word; part 0 the four covering scales[12] and d (bytes 96-109)
                    const bool odd = (reinterpret_cast<uintptr_t>(fw) & 2) != 0;
                    const uint8_t* hm = reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(fw + 16 * part) & ~(uintptr_t)3);
                    const uint8_t* qs = reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(fw + 32 + 32 * hh + 16 * part) & ~(uintptr_t)3);
#pragma unroll
                    for (int i = 0; i < 4; i++) { cp_async4(dst + 16 + 4 * i, hm + 4 * i); cp_async4(dst + 36 + 4 * i, qs + 4 * i); }
                    if (odd) { cp_async4(dst + 32, hm + 16); cp_async4(dst + 52, qs + 16); }
                    if (part == 0) {
                        const uint8_t* sc = reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(fw + 96) & ~(uintptr_t)3);
#pragma unroll
                        for (int i = 0; i < 4; i++) cp_async4(dst + 4 * i, sc + 4 * i);
                    }
                } else if (FMT == 7) {
                    // qs[32 hh + l] (l = 16 part + 0..15); scales[16] where this thread needs them (part 1: its mins); d | dmin
                    const uint8_t* q = fw + 16 + 32 * hh + 16 * part;
#pragma unroll
                    for (int i = 0; i < 4; i++) cp_async4(dst + 16 + 4 * i, q + 4 * i);
                    if (part == 0 || hh == 1) {
#pragma unroll
                        for (int i = 0; i < 4; i++) cp_async4(dst + 4 * i, fw + 4 * i);
                    }
                    if (part == 0) cp_async4(dst + 32, fw + 80);
                } else if (IQM) {
                    // sub-blocks 2 q, 2 q + 1: 8 bytes of qs, 4 of qh, the 8-byte scale field (d and their ls); 8-byte aligned blocks
                    const int q = 2 * hh + part;
                    cp_async8(dst, fw + 8 * q);
                    cp_async4(dst + 8, fw + 32 + 4 * q);
                    cp_async8(dst + 16, fw + 48);
                } else if (IQ3) {
                    // as FMT 2: every word fetched holds at least one byte this thread needs; the last word of a multi-word field
                    // only when the block starts on a word (its fields then start mid-word)
                    const int q = 2 * hh + part;
                    const bool mid = (reinterpret_cast<uintptr_t>(fw) & 2) == 0;
                    auto cover = [&](int off) { return reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(fw + off) & ~(uintptr_t)3); };
                    const uint8_t* qs = cover(2 + 16 * q);
#pragma unroll
                    for (int i = 0; i < 4; i++) cp_async4(dst + 4 * i, qs + 4 * i);
                    if (mid) cp_async4(dst + 16, qs + 16);
                    const uint8_t* sg = cover(FMT == 9 ? 66 + 8 * q : 74 + 8 * q);
                    const int o = FMT == 9 ? 20 : 24;
                    cp_async4(dst + o, sg);
                    cp_async4(dst + o + 4, sg + 4);
                    if (mid) cp_async4(dst + o + 8, sg + 8);
                    if (FMT == 10) {
                        cp_async4(dst + 20, cover(66 + 2 * q));
                        cp_async4(dst + 36, cover(106 + q));
                    }
                    cp_async4(dst + (FMT == 9 ? 32 : 40), cover(0));
                } else if (IQ2) {
                    // as IQ3: the covering words of each multi-word field (a last one only when the block starts on a word), the
                    // words holding the 2-byte fields
                    const int q = 2 * hh + part;
                    const bool mid = (reinterpret_cast<uintptr_t>(fw) & 2) == 0;
                    auto cover = [&](int off) { return reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(fw + off) & ~(uintptr_t)3); };
                    if (FMT == 11) {
                        const uint8_t* qs = cover(2 + 16 * q);
#pragma unroll
                        for (int i = 0; i < 4; i++) cp_async4(dst + 4 * i, qs + 4 * i);
                        if (mid) cp_async4(dst + 16, qs + 16);
                        cp_async4(dst + 20, cover(66 + 2 * q));
                        cp_async4(dst + 24, cover(0));
                    } else {
                        const uint8_t *qs = cover(2 + 8 * q), *sg = cover(34 + 8 * q);
                        cp_async4(dst, qs);
                        cp_async4(dst + 4, qs + 4);
                        if (mid) cp_async4(dst + 8, qs + 8);
                        cp_async4(dst + 12, sg);
                        cp_async4(dst + 16, sg + 4);
                        if (mid) cp_async4(dst + 20, sg + 8);
                        cp_async4(dst + 24, cover(66 + 2 * q));
                        cp_async4(dst + 28, cover(74 + 2 * q));
                        cp_async4(dst + 32, cover(0));
                    }
                } else if (IQ) {
                    // every word fetched holds at least one byte this thread needs (so it lies inside the tensor's pages);
                    // the last word of a field is only needed when the block starts on a word (the fields then start mid-word)
                    const int q = 2 * hh + part;
                    const bool mid = (reinterpret_cast<uintptr_t>(fw) & 2) == 0;
                    const uint8_t* qs = reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(fw + 2 + (FMT == 2 ? 8 : 16) * q) & ~(uintptr_t)3);
                    cp_async4(dst, qs);
                    cp_async4(dst + 4, qs + 4);
                    if (FMT == 2) {
                        if (mid) cp_async4(dst + 8, qs + 8);
                        const uint8_t* qh = reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(fw + 34 + 4 * q) & ~(uintptr_t)3);
                        cp_async4(dst + 12, qh);
                        if (mid) cp_async4(dst + 16, qh + 4);
                    } else {
                        cp_async4(dst + 8, qs + 8);
                        cp_async4(dst + 12, qs + 12);
                        if (mid) cp_async4(dst + 16, qs + 16);
                    }
                    cp_async4(dst + 20, reinterpret_cast<const uint8_t*>(reinterpret_cast<uintptr_t>(fw) & ~(uintptr_t)3));
                } else {
                    const uint8_t* q = fw + (long)(4 * hh) * c16;
                    cp_async16(dst, q);
                    cp_async16(dst + 16, q + 2 * c16);
                    cp_async16(dst + 32, fw + (long)(8 + 2 * hh) * c16);
                    if (part == 0) {
                        cp_async8(dst + 64, fw + (long)12 * c16 + hh * 8);
                        cp_async4(dst + 72, fitem + (long)13 * c16 + (ffi >> 1) * 4);
                    }
                }
                if (fxq) { cp_async16(dst + (IQS ? 32 : FMT == 6 ? 64 : 48), fxq); fxq += 128; }   // IQ3, IQ2: 48
                if (hh == 1) {
                    if (MINS && fbs) { cp_async16(dst + 64, fbs); fbs += 16; }
                    if (fdx) { cp_async4(dst + (MINS ? 64 : IQS ? 24 : FMT == 6 ? 56 : (IQ3 || IQ2) ? 44 : 76), fdx); fdx += 1; }
                    fw += FMT == 0 ? SZ_Q4_K : FMT == 5 ? SZ_Q5_K : (IQ || FMT >= 6) ? BS : 16;
                    ffi++;
                }
                if (++fst == nst) { fst = 0; ftile += gridDim.x; enter_tile(); }
            }
            cp_async_commit();
        };
        enter_tile();
        for (int i = 0; i < nRaw; i++) issue(raw_dst + i * rawSlot);
        int slot = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int4 ti = __ldg(p.tinfo + tile);
            const int n_valid = ti.w;
            int dsel = ((ti.y + r) & 3) * nblk;   // Q6_K: which half of the fetched word holds this block's d
            // IQ: 16 when the current block starts on a word (its fields then start mid-word), else 0; Q3_K (fields at word
            // offsets of the block): 16 when it starts mid-word.  50, 66, 74, 82, 98 and 110 are 2 mod 4, so it alternates block
            // by block
            uint32_t ish = (IQ || IQ3 || IQ2) ? ((reinterpret_cast<uintptr_t>(p.w + (long)ti.x * p.expert_bytes + (long)(ti.y + r) * nblk * BS) & 2) ? 0u : 16u)
                         : FMT == 6 ? ((reinterpret_cast<uintptr_t>(p.w + (long)ti.x * p.expert_bytes + (long)(ti.y + r) * nblk * BS) & 2) ? 16u : 0u) : 0u;
            for (int st = 0; st < nst; st++) {
                const int hh = st & 1;
                const bool tr = p.trace && blockIdx.x == 0 && tid == 0 && tile == 0 && st < 96;
                if (tr) p.trace[(0 * 96 + st) * 4 + 0] = clock64();
                cp_async_wait<nRaw - 1>();
                if (tr) p.trace[(0 * 96 + st) * 4 + 1] = clock64();
                const uint4* rs = reinterpret_cast<const uint4*>(raw_src + slot * rawSlot);
                const uint4 f0 = rs[0], f1 = rs[1], f2 = rs[2], f3 = rs[IQS ? 2 : FMT == 6 ? 4 : 3], f4 = rs[IQS ? 1 : FMT == 6 ? 3 : (IQ3 || IQ2) ? 2 : 4];
                const uint4 f5 = rs[FMT == 5 ? 5 : 0], f6 = rs[FMT == 5 ? 6 : 0];   // Q5_K: qh
                issue(raw_dst + slot * rawSlot);   // refill the slot just read (thread-private bytes: no barrier involved)
                slot = slot == nRaw - 1 ? 0 : slot + 1;
                bar_wait(smem_u32(&misc.smem_free[stage]), sphase ^ 1);
                bar_wait(smem_u32(&misc.hdr_free[hs]), hphase ^ 1);
                if (tr) p.trace[(0 * 96 + st) * 4 + 2] = clock64();
                uint8_t* arow = smem + stage * kGA + r * 128;
                const uint4 z = make_uint4(0, 0, 0, 0);
                if (K4) {
                    // chunk c = 2 hh + part (32 bytes of qs): low nibbles = sub-block 2c (elements 64c .. 64c+31), high nibbles = sub-block 2c+1
                    const int pi = 4 * part;
                    if (FMT == 0) {
                        *reinterpret_cast<uint4*>(arow + (((pi + 0) ^ sw) << 4)) = make_uint4(f0.x & 0x0F0F0F0Fu, f0.y & 0x0F0F0F0Fu, f0.z & 0x0F0F0F0Fu, f0.w & 0x0F0F0F0Fu);
                        *reinterpret_cast<uint4*>(arow + (((pi + 1) ^ sw) << 4)) = make_uint4(f1.x & 0x0F0F0F0Fu, f1.y & 0x0F0F0F0Fu, f1.z & 0x0F0F0F0Fu, f1.w & 0x0F0F0F0Fu);
                        *reinterpret_cast<uint4*>(arow + (((pi + 2) ^ sw) << 4)) =
                            make_uint4((f0.x >> 4) & 0x0F0F0F0Fu, (f0.y >> 4) & 0x0F0F0F0Fu, (f0.z >> 4) & 0x0F0F0F0Fu, (f0.w >> 4) & 0x0F0F0F0Fu);
                        *reinterpret_cast<uint4*>(arow + (((pi + 3) ^ sw) << 4)) =
                            make_uint4((f1.x >> 4) & 0x0F0F0F0Fu, (f1.y >> 4) & 0x0F0F0F0Fu, (f1.z >> 4) & 0x0F0F0F0Fu, (f1.w >> 4) & 0x0F0F0F0Fu);
                    } else {   // Q5_K: bit 2c (low nibbles) or 2c + 1 (high nibbles) of qh[l] as bit 4
                        const int hb = 2 * (2 * hh + part);
                        const uint32_t q[8] = {f0.x, f0.y, f0.z, f0.w, f1.x, f1.y, f1.z, f1.w}, h[8] = {f5.x, f5.y, f5.z, f5.w, f6.x, f6.y, f6.z, f6.w};
                        uint32_t lo[8], hi[8];
#pragma unroll
                        for (int i = 0; i < 8; i++) {
                            lo[i] = (q[i] & 0x0F0F0F0Fu) | (((h[i] >> hb) << 4) & 0x10101010u);
                            hi[i] = ((q[i] >> 4) & 0x0F0F0F0Fu) | (((h[i] >> hb) << 3) & 0x10101010u);
                        }
                        *reinterpret_cast<uint4*>(arow + (((pi + 0) ^ sw) << 4)) = make_uint4(lo[0], lo[1], lo[2], lo[3]);
                        *reinterpret_cast<uint4*>(arow + (((pi + 1) ^ sw) << 4)) = make_uint4(lo[4], lo[5], lo[6], lo[7]);
                        *reinterpret_cast<uint4*>(arow + (((pi + 2) ^ sw) << 4)) = make_uint4(hi[0], hi[1], hi[2], hi[3]);
                        *reinterpret_cast<uint4*>(arow + (((pi + 3) ^ sw) << 4)) = make_uint4(hi[4], hi[5], hi[6], hi[7]);
                    }
                    if (part == 0) misc.hdr[hs][r] = f2;
                    if (hh == 1) {   // A2 row: [m_0 m_0 m_1 m_1 ... m_7 m_7] against the sixteen 16-value activation sums; 4 mins per part
                        const uint32_t hw[4] = {f2.x, f2.y, f2.z, f2.w};
                        int sc, mn[4];
                        if (part == 0) {
#pragma unroll
                            for (int j = 0; j < 4; j++) q4k_scale_min(hw, j, sc, mn[j]);
                        } else {
#pragma unroll
                            for (int j = 0; j < 4; j++) q4k_scale_min(hw, 4 + j, sc, mn[j]);
                        }
                        uint8_t* a2 = smem + kOffA2 + stage * kGA2 + (r >> 3) * 256 + (r & 7) * 16 + part * 128;
                        *reinterpret_cast<uint4*>(a2) = make_uint4(h2(mn[0], mn[0]), h2(mn[1], mn[1]), h2(mn[2], mn[2]), h2(mn[3], mn[3]));
                    }
                } else if (IQM) {
                    // sub-block 4 hh + 2 part + j -> A chunks 4 part + 2 j, + 1 as FMT 2 with the delta per 8 values; header: the
                    // stage's eight ls as bytes 0-7 (the Q6_K layout, byte 4 part + 2 j + half), word 2 = d / 8 as f32
                    const uint32_t qs[2] = {f0.x, f0.y}, qh = f0.z;   // nibble 4 j + l of qh: group l of sub-block j, at bits 16 j + 4 l
                    const uint32_t scw = (hh ? f1.y : f1.x) >> (16 * part);   // scale word 2 hh + part: ls of sub-block j at bits 6 j, 6 j + 3
#pragma unroll
                    for (int j = 0; j < 2; j++) {
                        uint32_t v[8];
#pragma unroll
                        for (int l = 0; l < 4; l++) {
                            const uint32_t nib = qh >> (16 * j + 4 * l);
                            const uint2 g = tab[((qs[j] >> (8 * l)) & 0xffu) | ((nib & 7u) << 8)];
                            const uint32_t dl = (nib & 8u) ? 0xffffffffu : 0x01010101u;
                            v[2 * l] = __vadd4((g.x << 3) & 0xf8f8f8f8u, dl);
                            v[2 * l + 1] = __vadd4((g.y << 3) & 0xf8f8f8f8u, dl);
                        }
                        const int c0 = 4 * part + 2 * j;
                        *reinterpret_cast<uint4*>(arow + (((c0 + 0) ^ sw) << 4)) = make_uint4(v[0], v[1], v[2], v[3]);
                        *reinterpret_cast<uint4*>(arow + (((c0 + 1) ^ sw) << 4)) = make_uint4(v[4], v[5], v[6], v[7]);
                    }
                    uint32_t ls = 0;
#pragma unroll
                    for (int i = 0; i < 4; i++) ls |= (2 * ((scw >> (3 * i)) & 7u) + 1) << (8 * i);
                    uint32_t* hrow = reinterpret_cast<uint32_t*>(&misc.hdr[hs][r]);
                    hrow[part] = ls;
                    if (part == 0) hrow[2] = __float_as_uint(iq_d8(iq1m_d_bits(f1.x, f1.y)));
                } else if (IQ3) {
                    // sub-block 4 hh + 2 part + j -> A chunks 4 part + 2 j, + 1 as FMT 3 (value word g of 8 = 4-value group g, +-grid
                    // through the sign masks); header word `part` = the two ls (16 bits each), word 2 = d / 4 (IQ3_XXS) or d as f32
                    const int q = 2 * hh + part;
                    const uint32_t w[5] = {f0.x, f0.y, f0.z, f0.w, f1.x};
                    const uint32_t sgw[3] = {FMT == 9 ? f1.y : f1.z, FMT == 9 ? f1.z : f1.w, FMT == 9 ? f1.w : f2.x};
                    const uint32_t dw = FMT == 9 ? f2.x : f2.z, dbits = ish ? (dw & 0xffffu) : (dw >> 16);
                    // IQ3_S: qh[2 q], qh[2 q + 1] and scales[q] from the words holding them (2-byte / byte positions from ish)
                    const uint32_t qh16 = f1.y >> ((q & 1) ? (ish ^ 16u) : ish), scb = f2.y >> (8 * ((q + (ish ? 2 : 0)) & 3));
                    const uint2* sgn = tab + (FMT == 9 ? 128 : 256);
                    uint32_t ls[2];
#pragma unroll
                    for (int j = 0; j < 2; j++) {
                        const uint32_t sg = __funnelshift_r(sgw[j], sgw[j + 1], ish);   // IQ3_XXS: 4 x 7-bit sign index | s; IQ3_S: 4 sign bytes
                        uint32_t v[8];
#pragma unroll
                        for (int l = 0; l < 4; l++) {   // 8 values: 4-value groups 2 l, 2 l + 1 = bytes 2 (l & 1), + 1 of qs word 2 j + l / 2
                            const uint32_t qw = __funnelshift_r(w[2 * j + (l >> 1)], w[2 * j + (l >> 1) + 1], ish) >> (16 * (l & 1));
                            uint32_t i0 = qw & 0xffu, i1 = (qw >> 8) & 0xffu;
                            if (FMT == 10) {
                                const uint32_t qh = qh16 >> (8 * j);
                                i0 |= ((qh >> (2 * l)) & 1u) << 8;
                                i1 |= ((qh >> (2 * l + 1)) & 1u) << 8;
                            }
                            const uint2 m = sgn[FMT == 9 ? (sg >> (7 * l)) & 127u : (sg >> (8 * l)) & 0xffu];
                            v[2 * l] = __vsub4(tab4[i0] ^ m.x, m.x);
                            v[2 * l + 1] = __vsub4(tab4[i1] ^ m.y, m.y);
                        }
                        ls[j] = FMT == 9 ? 2 * (sg >> 28) + 1 : 2 * ((scb >> (4 * j)) & 15u) + 1;
                        const int c0 = 4 * part + 2 * j;
                        *reinterpret_cast<uint4*>(arow + (((c0 + 0) ^ sw) << 4)) = make_uint4(v[0], v[1], v[2], v[3]);
                        *reinterpret_cast<uint4*>(arow + (((c0 + 1) ^ sw) << 4)) = make_uint4(v[4], v[5], v[6], v[7]);
                    }
                    uint32_t* hrow = reinterpret_cast<uint32_t*>(&misc.hdr[hs][r]);
                    hrow[part] = ls[0] | (ls[1] << 16);
                    if (part == 0) hrow[2] = __float_as_uint(FMT == 9 ? iq_d4((uint16_t)dbits) : fp16_bits_to_f32((uint16_t)dbits));
                    if (hh == 1) ish ^= 16u;
                } else if (IQ2) {
                    // sub-block 4 hh + 2 part + j -> A chunks 4 part + 2 j (values 0-15), + 1 (16-31), value word 2 l + {0, 1} = 8-value
                    // group l as +-grid through the sign masks; header as IQ1_M: the stage's eight ls as bytes 0-7 (byte 4 part + 2 j +
                    // half), word 2 = d / 8 as f32.  The 2-byte fields of sub-blocks 2 q, 2 q + 1 sit at 16-bit position ish for even q
                    const uint32_t fsh = part ? (ish ^ 16u) : ish;   // q = 2 hh + part
                    const uint32_t sc16 = (FMT == 11 ? f1.y : f1.w) >> fsh, qh16 = f1.z >> fsh;
                    const uint32_t dw = FMT == 11 ? f1.z : f2.x, dbits = ish ? (dw & 0xffffu) : (dw >> 16);
                    const uint2* sgn = tab + (FMT == 11 ? 512 : 1024);
#pragma unroll
                    for (int j = 0; j < 2; j++) {
                        uint32_t v[8];
                        if (FMT == 11) {   // uint16 l: 9-bit grid index | 7-bit sign index << 9
                            const uint32_t w[5] = {f0.x, f0.y, f0.z, f0.w, f1.x};
                            const uint32_t u[2] = {__funnelshift_r(w[2 * j], w[2 * j + 1], ish), __funnelshift_r(w[2 * j + 1], w[2 * j + 2], ish)};
#pragma unroll
                            for (int l = 0; l < 4; l++) {
                                const uint32_t ul = u[l >> 1] >> (16 * (l & 1));
                                const uint2 g = tab[ul & 511u], m = sgn[(ul >> 9) & 127u];
                                v[2 * l] = __vsub4(g.x ^ m.x, m.x);
                                v[2 * l + 1] = __vsub4(g.y ^ m.y, m.y);
                            }
                        } else {           // qs byte l | bits 2 l, 2 l + 1 of qh << 8; sign byte l
                            const uint32_t qw[3] = {f0.x, f0.y, f0.z}, sgw[3] = {f0.w, f1.x, f1.y};
                            const uint32_t qs = __funnelshift_r(qw[j], qw[j + 1], ish), sg = __funnelshift_r(sgw[j], sgw[j + 1], ish);
                            const uint32_t qh = qh16 >> (8 * j);
#pragma unroll
                            for (int l = 0; l < 4; l++) {
                                const uint2 g = tab[((qs >> (8 * l)) & 0xffu) | ((qh << (8 - 2 * l)) & 0x300u)], m = sgn[(sg >> (8 * l)) & 0xffu];
                                v[2 * l] = __vsub4(g.x ^ m.x, m.x);
                                v[2 * l + 1] = __vsub4(g.y ^ m.y, m.y);
                            }
                        }
                        const int c0 = 4 * part + 2 * j;
                        *reinterpret_cast<uint4*>(arow + (((c0 + 0) ^ sw) << 4)) = make_uint4(v[0], v[1], v[2], v[3]);
                        *reinterpret_cast<uint4*>(arow + (((c0 + 1) ^ sw) << 4)) = make_uint4(v[4], v[5], v[6], v[7]);
                    }
                    uint32_t ls = 0;   // nibble i of scales[2 q], scales[2 q + 1]: half i % 2 of sub-block 2 q + i / 2
#pragma unroll
                    for (int i = 0; i < 4; i++) ls |= (2 * ((sc16 >> (4 * i)) & 15u) + 1) << (8 * i);
                    uint32_t* hrow = reinterpret_cast<uint32_t*>(&misc.hdr[hs][r]);
                    hrow[part] = ls;
                    if (part == 0) hrow[2] = __float_as_uint(iq_d8((uint16_t)dbits));
                    if (hh == 1) ish ^= 16u;
                } else if (IQ) {
                    // sub-block 4 hh + 2 part + j -> A chunks 4 part + 2 j and 4 part + 2 j + 1; header word `part` = its two ls
                    // (16 bits each), word 2 = d / 8 as f32
                    const uint32_t w[5] = {f0.x, f0.y, f0.z, f0.w, f1.x};
                    const uint32_t dbits = ish ? (f1.y & 0xffffu) : (f1.y >> 16);
                    uint32_t ls[2];
#pragma unroll
                    for (int j = 0; j < 2; j++) {
                        uint32_t v[8];
                        if (FMT == 2) {   // 8 * grid + delta, delta = qh bit 15 ? -1 : +1 per byte
                            const uint32_t qs = __funnelshift_r(w[j], w[j + 1], ish), qh = __funnelshift_r(w[3], w[4], ish) >> (16 * j);
                            const uint32_t dl = (qh & 0x8000u) ? 0xffffffffu : 0x01010101u;
#pragma unroll
                            for (int l = 0; l < 4; l++) {
                                const uint2 g = tab[((qs >> (8 * l)) & 0xffu) | (((qh >> (3 * l)) & 7u) << 8)];
                                v[2 * l] = __vadd4((g.x << 3) & 0xf8f8f8f8u, dl);
                                v[2 * l + 1] = __vadd4((g.y << 3) & 0xf8f8f8f8u, dl);
                            }
                            ls[j] = 2 * ((qh >> 12) & 7u) + 1;
                        } else {          // +-grid through the sign masks
                            const uint32_t aux0 = __funnelshift_r(w[2 * j], w[2 * j + 1], ish), aux1 = __funnelshift_r(w[2 * j + 1], w[2 * j + 2], ish);
#pragma unroll
                            for (int l = 0; l < 4; l++) {
                                const uint2 g = tab[(aux0 >> (8 * l)) & 0xffu], m = tab[256 + ((aux1 >> (7 * l)) & 127u)];
                                v[2 * l] = __vsub4(g.x ^ m.x, m.x);
                                v[2 * l + 1] = __vsub4(g.y ^ m.y, m.y);
                            }
                            ls[j] = 2 * (aux1 >> 28) + 1;
                        }
                        const int c0 = 4 * part + 2 * j;
                        *reinterpret_cast<uint4*>(arow + (((c0 + 0) ^ sw) << 4)) = make_uint4(v[0], v[1], v[2], v[3]);
                        *reinterpret_cast<uint4*>(arow + (((c0 + 1) ^ sw) << 4)) = make_uint4(v[4], v[5], v[6], v[7]);
                    }
                    uint32_t* hrow = reinterpret_cast<uint32_t*>(&misc.hdr[hs][r]);
                    hrow[part] = ls[0] | (ls[1] << 16);
                    if (part == 0) hrow[2] = __float_as_uint(iq_d8((uint16_t)dbits));
                    if (hh == 1) ish ^= 16u;
                } else if (FMT == 6) {
                    // element 32 j + l of the half (l = 16 part + 0..15): (qs[32 hh + l] >> 2j & 3) - 4 unless bit 4 hh + j of
                    // hmask[l] is set, built as (q | h << 2) - 4 per byte (flip bit 2, copy it into bits 3-7: no carries)
                    const uint32_t hw5[5] = {f1.x, f1.y, f1.z, f1.w, f2.x}, qw5[5] = {f2.y, f2.z, f2.w, f4.x, f4.y};
                    uint32_t m[4], q[4];
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        m[i] = __funnelshift_r(hw5[i], hw5[i + 1], ish) >> (4 * hh);
                        q[i] = __funnelshift_r(qw5[i], qw5[i + 1], ish);
                    }
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        uint32_t v[4];
#pragma unroll
                        for (int i = 0; i < 4; i++) {
                            const uint32_t tt = (((q[i] >> (2 * j)) & 0x03030303u) | (((m[i] >> j) & 0x01010101u) << 2)) ^ 0x04040404u;
                            v[i] = tt + (tt & 0x04040404u) * 62u;
                        }
                        *reinterpret_cast<uint4*>(arow + (((2 * j + part) ^ sw) << 4)) = make_uint4(v[0], v[1], v[2], v[3]);
                    }
                    if (part == 0) {   // the header of Q6_K: the half's 8 scales (6-bit, - 32) as int8, d as f32
                        const uint32_t s0 = __funnelshift_r(f0.x, f0.y, ish), s1 = __funnelshift_r(f0.y, f0.z, ish), s2 = __funnelshift_r(f0.z, f0.w, ish);
                        const uint32_t dbits = ish ? (f0.w >> 16) : (f0.w & 0xffffu);
                        uint32_t c[2] = {((s0 >> (4 * hh)) & 0x0F0F0F0Fu) | (((s2 >> (4 * hh)) & 0x03030303u) << 4),
                                         ((s1 >> (4 * hh)) & 0x0F0F0F0Fu) | (((s2 >> (4 * hh + 2)) & 0x03030303u) << 4)};
#pragma unroll
                        for (int i = 0; i < 2; i++) {   // - 32 as for Q6_K's quants
                            const uint32_t tt = c[i] ^ 0x20202020u;
                            c[i] = tt + (tt & 0x20202020u) * 6u;
                        }
                        misc.hdr[hs][r] = make_uint4(c[0], c[1], __float_as_uint(fp16_bits_to_f32((uint16_t)dbits)), 0);
                    }
                    if (hh == 1) ish ^= 16u;
                } else if (FMT == 7) {
                    // element 32 j + l of the half (l = 16 part + 0..15): qs[32 hh + l] >> 2j & 3
#pragma unroll
                    for (int j = 0; j < 4; j++)
                        *reinterpret_cast<uint4*>(arow + (((2 * j + part) ^ sw) << 4)) =
                            make_uint4((f1.x >> (2 * j)) & 0x03030303u, (f1.y >> (2 * j)) & 0x03030303u, (f1.z >> (2 * j)) & 0x03030303u, (f1.w >> (2 * j)) & 0x03030303u);
                    // header: the half's 8 scales (low nibbles), d | dmin; A2 row (second half): the 16 mins (high nibbles), 8 per part
                    if (part == 0) misc.hdr[hs][r] = make_uint4((hh ? f0.z : f0.x) & 0x0F0F0F0Fu, (hh ? f0.w : f0.y) & 0x0F0F0F0Fu, f2.x, 0);
                    if (hh == 1) {
                        const uint32_t m0 = part ? f0.z : f0.x, m1 = part ? f0.w : f0.y;
                        uint8_t* a2 = smem + kOffA2 + stage * kGA2 + (r >> 3) * 256 + (r & 7) * 16 + part * 128;
                        *reinterpret_cast<uint4*>(a2) = make_uint4(h2((m0 >> 4) & 15, (m0 >> 12) & 15), h2((m0 >> 20) & 15, m0 >> 28),
                                                                   h2((m1 >> 4) & 15, (m1 >> 12) & 15), h2((m1 >> 20) & 15, m1 >> 28));
                    }
                } else {
                    // element 32 g + l of the half (l = 16 part + 0..15): g = 0 ql[l] & 15 | (qh & 3) << 4, g = 1 ql[32 + l] & 15 | (qh >> 2 & 3) << 4,
                    // g = 2 ql[l] >> 4 | (qh >> 4 & 3) << 4, g = 3 ql[32 + l] >> 4 | (qh >> 6 & 3) << 4; stored as q - 32 in int8
                    const uint32_t a[4] = {f0.x, f0.y, f0.z, f0.w}, b[4] = {f1.x, f1.y, f1.z, f1.w}, h[4] = {f2.x, f2.y, f2.z, f2.w};
                    uint32_t v[4][4];
#pragma unroll
                    for (int i = 0; i < 4; i++) {
                        v[0][i] = (a[i] & 0x0F0F0F0Fu) | ((h[i] << 4) & 0x30303030u);
                        v[1][i] = (b[i] & 0x0F0F0F0Fu) | ((h[i] << 2) & 0x30303030u);
                        v[2][i] = ((a[i] >> 4) & 0x0F0F0F0Fu) | (h[i] & 0x30303030u);
                        v[3][i] = ((b[i] >> 4) & 0x0F0F0F0Fu) | ((h[i] >> 2) & 0x30303030u);
                    }
#pragma unroll
                    for (int g = 0; g < 4; g++) {
#pragma unroll
                        for (int i = 0; i < 4; i++) {   // q - 32 per byte: flip bit 5, then copy it into bits 6 and 7 (no carries between bytes)
                            const uint32_t tt = v[g][i] ^ 0x20202020u;
                            v[g][i] = tt + (tt & 0x20202020u) * 6u;
                        }
                        *reinterpret_cast<uint4*>(arow + (((2 * g + part) ^ sw) << 4)) = make_uint4(v[g][0], v[g][1], v[g][2], v[g][3]);
                    }
                    if (part == 0) {
                        const uint32_t dbits = (dsel & 1) ? (f4.z >> 16) : (f4.z & 0xffffu);
                        misc.hdr[hs][r] = make_uint4(f4.x, f4.y, __float_as_uint(fp16_bits_to_f32((uint16_t)dbits)), 0);
                    }
                    dsel += hh;
                }
                // activations: piece (bn, pc)
                uint8_t* Bs = smem + offB + stage * strideB;
                const uint4 bv = bn < n_valid ? f3 : z;
                if (!SUB16) {
                    *reinterpret_cast<uint4*>(Bs + bn * 128 + ((pc ^ (bn & 7)) << 4)) = bv;
                } else {   // a 16-byte piece is one 16-value sub-block: rows 0-31 keep the even pieces, rows 32-63 the odd ones
                    *reinterpret_cast<uint4*>(Bs + bn * 128 + ((pc ^ (bn & 7)) << 4)) = (pc & 1) ? z : bv;
                    *reinterpret_cast<uint4*>(Bs + (kGN + bn) * 128 + ((pc ^ (bn & 7)) << 4)) = (pc & 1) ? bv : z;
                }
                if (hh == 1 && pt < 96) {   // token scales, and (formats with mins) the sixteen 16-value sums of the super-block as fp16
                    if (pt >= 64) misc.dxs[hs][pt - 64] = pt - 64 < n_valid ? __uint_as_float(MINS ? f4.x : (IQS || FMT == 6) ? f4.z : f4.w) : 0.f;   // IQ3: f2.w
                    else if (MINS) {
                        const int n2 = pt >> 1, kg = pt & 1;
                        uint4 vv = z;
                        if (n2 < n_valid) {
                            const uint32_t bw[4] = {f4.x, f4.y, f4.z, f4.w};
#define KTB_S16(w, hi) ((int)(short)((hi) ? ((w) >> 16) : ((w) & 0xffffu)))
                            vv = make_uint4(h2(KTB_S16(bw[0], 0), KTB_S16(bw[0], 1)), h2(KTB_S16(bw[1], 0), KTB_S16(bw[1], 1)), h2(KTB_S16(bw[2], 0), KTB_S16(bw[2], 1)),
                                            h2(KTB_S16(bw[3], 0), KTB_S16(bw[3], 1)));
#undef KTB_S16
                        }
                        *reinterpret_cast<uint4*>(smem + kOffB2 + stage * kGB2 + (n2 >> 3) * 256 + kg * 128 + (n2 & 7) * 16) = vv;
                    }
                }
                fence_async_smem();
                __syncwarp();
                if (lane == 0) bar_arrive(smem_u32(&misc.ab_full[stage]));
                if (tr) p.trace[(0 * 96 + st) * 4 + 3] = clock64();
                if (++stage == kGStages) { stage = 0; sphase ^= 1; }
                if (++hs == kGHdr) { hs = 0; hphase ^= 1; }
            }
        }
        cp_async_wait<0>();
    } else {
        // ========================================================================== MMA warpgroups: g owns weight rows 64 g .. 64 g + 63
        // thread = rows ra = 64 g + 16 (warp % 4) + lane / 4 and ra + 8; accumulator register 4 jb + 2 h + e holds row ra + 8 h,
        // column 8 jb + 2 (lane % 4) + e; isum / acc use the same index for (row, token) with the token columns of jb < 4
        regs_inc<160>();   // 256 x 96 + 256 x 160 = 64 K registers
        const int mw = warp - kGProdWarps, g = mw >> 2, ra = 64 * g + 16 * (mw & 3) + (lane >> 2), cq = 2 * (lane & 3);
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int4 ti = __ldg(p.tinfo + tile);
            float acc[16];
            int isum[16];
#pragma unroll
            for (int i = 0; i < 16; i++) { acc[i] = 0.f; isum[i] = 0; }
            for (int st = 0; st < nst; st++) {
                const int hh = st & 1;
                const bool tr = p.trace && blockIdx.x == 0 && mw == 0 && lane == 0 && tile == 0 && st < 96;
                if (tr) p.trace[(1 * 96 + st) * 4 + 0] = clock64();
                bar_wait(smem_u32(&misc.ab_full[stage]), sphase);
                if (tr) p.trace[(1 * 96 + st) * 4 + 1] = clock64();
                const uint32_t a = base + stage * kGA + g * (kGA / 2), b = base + offB + stage * strideB;
                uint32_t hw[2][4];
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const uint4 hd = misc.hdr[hs][ra + 8 * h];
                    hw[h][0] = hd.x; hw[h][1] = hd.y; hw[h][2] = hd.z; hw[h][3] = hd.w;
                }
                if (K4) {
                    int sc[2][4], mn;
#pragma unroll
                    for (int h = 0; h < 2; h++) {   // (compile-time byte indices: no local-memory copy of the header)
                        if (hh == 0) {
#pragma unroll
                            for (int c = 0; c < 4; c++) q4k_scale_min(hw[h], c, sc[h][c], mn);
                        } else {
#pragma unroll
                            for (int c = 0; c < 4; c++) q4k_scale_min(hw[h], 4 + c, sc[h][c], mn);
                        }
                    }
#pragma unroll
                    for (int c = 0; c < 4; c += 2) {
                        uint32_t v0[16], v1[16];
                        fence();
                        mma_u8s8_m64n32(v0, smem_desc(a + c * 32, 16, 1024, kLayoutSw128), smem_desc(b + c * 32, 16, 1024, kLayoutSw128), 0);
                        mma_u8s8_m64n32(v1, smem_desc(a + c * 32 + 32, 16, 1024, kLayoutSw128), smem_desc(b + c * 32 + 32, 16, 1024, kLayoutSw128), 0);
                        commit();
                        wait<0>();
                        fence_regs(v0);
                        fence_regs(v1);
#pragma unroll
                        for (int i = 0; i < 16; i++) isum[i] += sc[(i >> 1) & 1][c] * (int)v0[i] + sc[(i >> 1) & 1][c + 1] * (int)v1[i];
                    }
                } else if (IQ || IQ3) {
                    // sub-block c of the stage: one MMA into its own accumulator, times its ls (header word c / 2, half c % 2)
#pragma unroll
                    for (int c = 0; c < 4; c += 2) {
                        uint32_t v0[16], v1[16];
                        fence();
                        mma_s8s8_m64n32(v0, smem_desc(a + c * 32, 16, 1024, kLayoutSw128), smem_desc(b + c * 32, 16, 1024, kLayoutSw128), 0);
                        mma_s8s8_m64n32(v1, smem_desc(a + c * 32 + 32, 16, 1024, kLayoutSw128), smem_desc(b + c * 32 + 32, 16, 1024, kLayoutSw128), 0);
                        commit();
                        wait<0>();
                        fence_regs(v0);
                        fence_regs(v1);
#pragma unroll
                        for (int i = 0; i < 16; i++) {
                            const uint32_t lw = hw[(i >> 1) & 1][c >> 1];
                            isum[i] += (int)(lw & 0xffffu) * (int)v0[i] + (int)(lw >> 16) * (int)v1[i];
                        }
                    }
                    if (hh == 1) {
#pragma unroll
                        for (int i = 0; i < 16; i++) {
                            acc[i] += iq_term(__uint_as_float(hw[(i >> 1) & 1][2]), misc.dxs[hs][8 * (i >> 2) + cq + (i & 1)], isum[i]);
                            isum[i] = 0;
                        }
                    }
                } else {
#pragma unroll
                    for (int c = 0; c < 4; c++) {
                        uint32_t v[32];
                        fence();
                        mma_s8s8_m64n64(v, smem_desc(a + c * 32, 16, 1024, kLayoutSw128), smem_desc(b + c * 32, 16, 1024, kLayoutSw128), 0);
                        commit();
                        wait<0>();
                        fence_regs(v);
                        // columns 0-31: the tokens against the even sub-block 2 c, columns 32-63: against the odd one
#pragma unroll
                        for (int i = 0; i < 32; i++) isum[i & 15] += sb8(hw[(i >> 1) & 1], 2 * c + (i >> 4)) * (int)v[i];
                    }
                    if (!MINS && hh == 1) {
#pragma unroll
                        for (int i = 0; i < 16; i++) {
                            acc[i] += iq_term(__uint_as_float(hw[(i >> 1) & 1][2]), misc.dxs[hs][8 * (i >> 2) + cq + (i & 1)], isum[i]);
                            isum[i] = 0;
                        }
                    }
                }
                if (MINS && hh == 1) {   // the mins MMA and the finish; d | dmin in header word 0 (Q4_K, Q5_K) or 2 (Q2_K)
                    float ms[16];
                    fence();
                    mma_f16_m64n32(ms, smem_desc(base + kOffA2 + stage * kGA2 + g * (kGA2 / 2), 128, 256, kLayoutNone),
                                   smem_desc(base + kOffB2 + stage * kGB2, 128, 256, kLayoutNone), 0);
                    commit();
                    wait<0>();
                    fence_regs(ms);
#pragma unroll
                    for (int i = 0; i < 16; i++) {
                        const __half2 dm = *reinterpret_cast<const __half2*>(&hw[(i >> 1) & 1][FMT == 7 ? 2 : 0]);
                        const float dw = __low2float(dm), dmin = __high2float(dm);
                        const float dx = misc.dxs[hs][8 * (i >> 2) + cq + (i & 1)];
                        acc[i] += kq_min_term(dw, dmin, dx, isum[i], ms[i]);
                        isum[i] = 0;
                    }
                }
                if (tr) p.trace[(1 * 96 + st) * 4 + 2] = clock64();
                __syncwarp();
                if (lane == 0) { bar_arrive(smem_u32(&misc.smem_free[stage])); bar_arrive(smem_u32(&misc.hdr_free[hs])); }
                if (tr) p.trace[(1 * 96 + st) * 4 + 3] = clock64();
                if (++stage == kGStages) { stage = 0; sphase ^= 1; }
                if (++hs == kGHdr) { hs = 0; hphase ^= 1; }
            }
#pragma unroll
            for (int i = 0; i < 16; i++) {
                const int n = 8 * (i >> 2) + cq + (i & 1);
                if (n < ti.w) p.out[(long)(ti.z + n) * p.R + ti.y + ra + 8 * ((i >> 1) & 1)] = acc[i];
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// RAWINT4_G32 (Kimi-K2's compressed-tensors experts) on the bf16 tensor path: W4A16, nothing quantised (DESIGN.md §2).
// A = u - 8 (-8..7, exact in bf16); B = the activations split into NP exact bf16 planes x = hi + mid + lo (grp_split_*):
// every product (u - 8) * plane is exact in fp32 (4 x 8 significant bits), and all 2 NP MMAs of a 32-value group sum into one
// group accumulator, so the tensor core sums exact products in fp32 — the per-pair kernels' group sum in another order.  Then
// one FFMA per group, acc = fma(gsum, s, acc) with the row's bf16 scale, as i4_block_dot.  NP = 1 for BF16 gate/up (hi = x),
// NP = 3 for F16 / F32 gate/up and for the down projection (a = act(g) * u in fp32).  The planes are a function of the fp32
// value only, so a narrow input and the same value widened to F32 give bit-identical sums: the extra planes add exact zeros.
// grouped_i4_kernel: the tile table, persistent tile loop, roles, rings and stores of grouped_gemm_kernel; stage = 64 of K =
// two groups.  Producer thread (row, part) converts group `part` of its row: (w >> 4j) & 0x000F000F | 0x43004300 is the bf16
// pair (128 + u of column 8i + j, 128 + u of column 8i + j + 4) of word i, minus 136 that is u - 8; so within every 8 columns
// K position 2j holds column j and 2j + 1 column j + 4, and the split kernels write B in that order (i4_split8).
// Shared-memory plan (I4Plan): A stages as kGA, NP B planes of 32 token rows per stage, raw slots of 2 + NP 16-byte units per
// thread (0 the group's four words, 1 the stage's scale word, 2.. the activation pieces), the misc block with hdr[.][row].x =
// the scale word (low half group 2q, high half group 2q + 1 of the block's quarter q).
template <int NP>
struct I4Plan {
    static constexpr int kB = NP * kGN * 128, kPitch = 16 * (2 + NP), kSlot = 2 * kGM * kPitch;
    static constexpr int kOffB = kGStages * kGA, kOffRaw = kOffB + kGStages * kB, kOffMisc = kOffRaw + kGRaw * kSlot;
    static constexpr int kSmem = kOffMisc + (int)sizeof(GrpMisc) + 1024;
};
static_assert(I4Plan<1>::kSmem <= 227 * 1024 && I4Plan<3>::kSmem <= 227 * 1024 && I4Plan<1>::kOffB % 1024 == 0 && kGN * 128 % 1024 == 0,
              "RAWINT4 shared-memory plan");

struct GrpI4Params {
    const uint8_t* w;          // expert weights, RAWINT4_G32 blocks
    long expert_bytes;
    int R, Kc;
    const uint16_t* x;         // bf16 planes [rows][NP][Kc] in the K order of the A tile (i4_split8)
    const int* rowmap;         // sorted position -> activation row (null: identity)
    const int4* tinfo;
    const int* nt_prefix;
    int E;
    float* out;                // [P][R] fp32
    long long* trace;          // as GrpGemmParams::trace
};

// the bf16 pair (u - 8 of column j, u - 8 of column j + 4) of the 8 columns in word w
__device__ __forceinline__ uint32_t i4_bf16x2(uint32_t w, int j) {
    const uint32_t v = ((w >> (4 * j)) & 0x000F000Fu) | 0x43004300u;
    uint32_t r;
    asm("sub.rn.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(v), "r"(0x43084308u));   // (128 + u) - 136, exact
    return r;
}
// 8 consecutive values -> NP bf16 planes (hi = bf16_rn(x), mid = bf16_rn(x - hi), lo = bf16_rn(x - hi - mid); every difference
// is exact) in the K order of i4_bf16x2; plane p at dst + p * Kc
template <int NP>
__device__ __forceinline__ void i4_split8(const float (&x)[8], uint16_t* dst, int Kc) {
    uint32_t v[NP][4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
        float r0 = x[j], r1 = x[j + 4];
#pragma unroll
        for (int p = 0; p < NP; p++) {
            const __nv_bfloat16 b0 = __float2bfloat16_rn(r0), b1 = __float2bfloat16_rn(r1);
            v[p][j] = (uint32_t)__bfloat16_as_ushort(b0) | ((uint32_t)__bfloat16_as_ushort(b1) << 16);
            r0 -= __bfloat162float(b0);
            r1 -= __bfloat162float(b1);
        }
    }
#pragma unroll
    for (int p = 0; p < NP; p++) *reinterpret_cast<uint4*>(dst + (long)p * Kc) = make_uint4(v[p][0], v[p][1], v[p][2], v[p][3]);
}

template <int NP>
__global__ void __launch_bounds__(kGThreads, 1) grouped_i4_kernel(const GrpI4Params p) {
    using L = I4Plan<NP>;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base - raw);
    GrpMisc& misc = *reinterpret_cast<GrpMisc*>(smem + L::kOffMisc);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nst = p.Kc / 64, MT = p.R / kGM;
    if (tid == 0) {
        for (int s = 0; s < kGStages; s++) { bar_init(smem_u32(&misc.ab_full[s]), kGProdWarps); bar_init(smem_u32(&misc.smem_free[s]), kGMmaWarps); }
        for (int s = 0; s < kGHdr; s++) bar_init(smem_u32(&misc.hdr_free[s]), kGMmaWarps);
        bar_fence_init();
    }
    __syncthreads();
    const int total_tiles = p.nt_prefix[p.E] * MT;
    int stage = 0, sphase = 0, hs = 0, hphase = 0;

    if (warp < kGProdWarps) {
        // ========================================================================== producers: thread = (weight row r, group `part`)
        regs_dec<96>();
        const int pt = tid, r = pt & (kGM - 1), part = pt >> 7, sw = r & 7, bn = pt >> 3, pc = pt & 7;
        const uint32_t raw_dst = base + L::kOffRaw + pt * L::kPitch;
        const uint8_t* raw_src = smem + L::kOffRaw + pt * L::kPitch;
        int ftile = blockIdx.x, fst = 0;
        const uint8_t* fw = nullptr;    // block 0 of this thread's weight row
        const uint16_t* fx = nullptr;   // this thread's activation piece of stage 0, plane 0 (null: no token row)
        auto enter_tile = [&]() {
            if (ftile >= total_tiles) return;
            const int4 ti = __ldg(p.tinfo + ftile);
            fx = bn < ti.w ? p.x + (long)(p.rowmap ? __ldg(p.rowmap + ti.z + bn) : ti.z + bn) * NP * p.Kc + pc * 8 : nullptr;
            fw = p.w + (long)ti.x * p.expert_bytes + (long)(ti.y + r) * (p.Kc / QK_K) * SZ_RAWINT4;
        };
        auto issue = [&](uint32_t dst) {
            if (ftile < total_tiles) {
                const uint8_t* blk = fw + (fst >> 2) * SZ_RAWINT4;
                const int q = fst & 3;
                cp_async16(dst, blk + 16 + 16 * (2 * q + part));
                if (part == 0) cp_async4(dst + 16, blk + 4 * q);
                if (fx) {
#pragma unroll
                    for (int pl = 0; pl < NP; pl++) cp_async16(dst + 32 + 16 * pl, fx + (long)pl * p.Kc + fst * 64);
                }
                if (++fst == nst) { fst = 0; ftile += gridDim.x; enter_tile(); }
            }
            cp_async_commit();
        };
        enter_tile();
        for (int i = 0; i < kGRaw; i++) issue(raw_dst + i * L::kSlot);
        int slot = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int n_valid = __ldg(p.tinfo + tile).w;
            for (int st = 0; st < nst; st++) {
                const bool tr = p.trace && blockIdx.x == 0 && tid == 0 && tile == 0 && st < 96;
                if (tr) p.trace[(0 * 96 + st) * 4 + 0] = clock64();
                cp_async_wait<kGRaw - 1>();
                if (tr) p.trace[(0 * 96 + st) * 4 + 1] = clock64();
                const uint4* rs = reinterpret_cast<const uint4*>(raw_src + slot * L::kSlot);
                const uint4 f0 = rs[0];
                const uint32_t scw = rs[1].x;
                uint4 fb[NP];
#pragma unroll
                for (int pl = 0; pl < NP; pl++) fb[pl] = rs[2 + pl];
                issue(raw_dst + slot * L::kSlot);   // refill the slot just read (thread-private bytes)
                slot = slot == kGRaw - 1 ? 0 : slot + 1;
                bar_wait(smem_u32(&misc.smem_free[stage]), sphase ^ 1);
                bar_wait(smem_u32(&misc.hdr_free[hs]), hphase ^ 1);
                if (tr) p.trace[(0 * 96 + st) * 4 + 2] = clock64();
                uint8_t* arow = smem + stage * kGA + r * 128;
                const uint32_t wd[4] = {f0.x, f0.y, f0.z, f0.w};
#pragma unroll
                for (int i = 0; i < 4; i++)   // word i of group `part` -> 16-byte chunk 4 part + i of the row
                    *reinterpret_cast<uint4*>(arow + (((4 * part + i) ^ sw) << 4)) =
                        make_uint4(i4_bf16x2(wd[i], 0), i4_bf16x2(wd[i], 1), i4_bf16x2(wd[i], 2), i4_bf16x2(wd[i], 3));
                if (part == 0) misc.hdr[hs][r].x = scw;
                uint8_t* Bs = smem + L::kOffB + stage * L::kB + bn * 128 + ((pc ^ (bn & 7)) << 4);
                const uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll
                for (int pl = 0; pl < NP; pl++) *reinterpret_cast<uint4*>(Bs + pl * (kGN * 128)) = bn < n_valid ? fb[pl] : z;
                fence_async_smem();
                __syncwarp();
                if (lane == 0) bar_arrive(smem_u32(&misc.ab_full[stage]));
                if (tr) p.trace[(0 * 96 + st) * 4 + 3] = clock64();
                if (++stage == kGStages) { stage = 0; sphase ^= 1; }
                if (++hs == kGHdr) { hs = 0; hphase ^= 1; }
            }
        }
        cp_async_wait<0>();
    } else {
        // ========================================================================== MMA warpgroups: g owns weight rows 64 g .. 64 g + 63
        // register i of an accumulator: row ra + 8 ((i >> 1) & 1), token column 8 (i >> 2) + cq + (i & 1)
        regs_inc<160>();
        const int mw = warp - kGProdWarps, g = mw >> 2, ra = 64 * g + 16 * (mw & 3) + (lane >> 2), cq = 2 * (lane & 3);
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int4 ti = __ldg(p.tinfo + tile);
            float acc[16];
#pragma unroll
            for (int i = 0; i < 16; i++) acc[i] = 0.f;
            for (int st = 0; st < nst; st++) {
                const bool tr = p.trace && blockIdx.x == 0 && mw == 0 && lane == 0 && tile == 0 && st < 96;
                if (tr) p.trace[(1 * 96 + st) * 4 + 0] = clock64();
                bar_wait(smem_u32(&misc.ab_full[stage]), sphase);
                if (tr) p.trace[(1 * 96 + st) * 4 + 1] = clock64();
                const uint32_t a = base + stage * kGA + g * (kGA / 2), b = base + L::kOffB + stage * L::kB;
                // group accumulators of the stage's two groups: every plane's two K = 16 MMAs into the same one
                float g0[16], g1[16];
#pragma unroll
                for (int i = 0; i < 16; i++) { g0[i] = 0.f; g1[i] = 0.f; }
                fence();
#pragma unroll
                for (int pl = 0; pl < NP; pl++)
#pragma unroll
                    for (int ks = 0; ks < 2; ks++) {
                        mma_bf16_m64n32(g0, smem_desc(a + 32 * ks, 16, 1024, kLayoutSw128), smem_desc(b + pl * (kGN * 128) + 32 * ks, 16, 1024, kLayoutSw128), 1);
                        mma_bf16_m64n32(g1, smem_desc(a + 64 + 32 * ks, 16, 1024, kLayoutSw128), smem_desc(b + pl * (kGN * 128) + 64 + 32 * ks, 16, 1024, kLayoutSw128), 1);
                    }
                commit();
                wait<0>();
                fence_regs(g0);
                fence_regs(g1);
                const uint32_t s0 = misc.hdr[hs][ra].x, s1 = misc.hdr[hs][ra + 8].x;
#pragma unroll
                for (int i = 0; i < 16; i++) {
                    const uint32_t sc = (i & 2) ? s1 : s0;
                    acc[i] = __fmaf_rn(g0[i], __uint_as_float(sc << 16), acc[i]);
                    acc[i] = __fmaf_rn(g1[i], __uint_as_float(sc & 0xffff0000u), acc[i]);
                }
                if (tr) p.trace[(1 * 96 + st) * 4 + 2] = clock64();
                __syncwarp();
                if (lane == 0) { bar_arrive(smem_u32(&misc.smem_free[stage])); bar_arrive(smem_u32(&misc.hdr_free[hs])); }
                if (tr) p.trace[(1 * 96 + st) * 4 + 3] = clock64();
                if (++stage == kGStages) { stage = 0; sphase ^= 1; }
                if (++hs == kGHdr) { hs = 0; hphase ^= 1; }
            }
#pragma unroll
            for (int i = 0; i < 16; i++) {
                const int n = 8 * (i >> 2) + cq + (i & 1);
                if (n < ti.w) p.out[(long)(ti.z + n) * p.R + ti.y + ra + 8 * ((i >> 1) & 1)] = acc[i];
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// bookkeeping kernels (moe.cpp:250-290: m_local_num_, m_local_pos_, prefix offsets)
__global__ void grp_count_kernel(const int64_t* ids, int npairs, int k, int id_offset, int n_local, const int* bsz, int t0, int* counts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npairs) return;
    if (bsz && t0 + i / k >= *bsz) return;
    const long e = (long)ids[i] - id_offset;
    if (e >= 0 && e < n_local) atomicAdd(counts + e, 1);
}
__global__ void grp_scan_kernel(const int* counts, int E, int* offsets, int* nt_prefix, int* cursor) {
    if (threadIdx.x == 0) {
        int o = 0, t = 0;
        for (int e = 0; e < E; e++) {
            offsets[e] = o; nt_prefix[e] = t; cursor[e] = o;
            o += counts[e];
            t += (counts[e] + kGN - 1) / kGN;
        }
        offsets[E] = o; nt_prefix[E] = t;
    }
}
__global__ void grp_scatter_kernel(const int64_t* ids, int npairs, int k, int id_offset, int n_local, const int* bsz, int t0, int* cursor, int* tokmap, int* pos) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= npairs) return;
    const long e = (long)ids[i] - id_offset;
    if ((bsz && t0 + i / k >= *bsz) || e < 0 || e >= n_local) { pos[i] = -1; return; }
    const int s = atomicAdd(cursor + e, 1);   // order inside an expert is irrelevant: every pair's result is independent
    tokmap[s] = i / k;
    pos[i] = s;
}
// rows of `src` (hidden type, [n][ncols]) -> int8 SoA + block scales + 16-value sums; one warp per 256-block
__global__ void __launch_bounds__(256) grp_quant_x_kernel(const void* src, int hidden_type, int nrows, int ncols, int8_t* q, float* d, int16_t* bs) {
    const int lane = threadIdx.x & 31, gw = blockIdx.x * 8 + (threadIdx.x >> 5), nblk = ncols / QK_K;
    if (gw >= nrows * nblk) return;
    const int r = gw / nblk, b = gw - r * nblk;
    float x[8];
    load_block8(src, (long)r * ncols + (long)b * QK_K + lane * 8, hidden_type, x);
    warp_quantize_q8k_block(x, lane, reinterpret_cast<uint32_t*>(q + (long)r * ncols + (long)b * QK_K), d + (long)r * nblk + b, bs + (long)r * (ncols / 16) + b * 16);
}
// a = act(g) * u (fp32, sorted pair rows) -> Q8_K SoA      (moe.cpp:300-318: silu * mul, then from_float to vec_dot_type)
__global__ void __launch_bounds__(256) grp_act_quant_kernel(const float* g, const float* u, const int* offsets, int E, int ncols, int use_silu, int8_t* q, float* d, int16_t* bs) {
    const int lane = threadIdx.x & 31, gw = blockIdx.x * 8 + (threadIdx.x >> 5), nblk = ncols / QK_K;
    if (gw >= offsets[E] * nblk) return;
    const int r = gw / nblk, b = gw - r * nblk;
    const long o = (long)r * ncols + (long)b * QK_K + lane * 8;
    float x[8];
    const float4 g0 = *reinterpret_cast<const float4*>(g + o), g1 = *reinterpret_cast<const float4*>(g + o + 4);
    const float4 u0 = *reinterpret_cast<const float4*>(u + o), u1 = *reinterpret_cast<const float4*>(u + o + 4);
    const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w}, uv[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
#pragma unroll
    for (int i = 0; i < 8; i++) x[i] = (use_silu ? act_silu(gv[i]) : act_relu(gv[i])) * uv[i];
    warp_quantize_q8k_block(x, lane, reinterpret_cast<uint32_t*>(q + (long)r * ncols + (long)b * QK_K), d + (long)r * nblk + b, bs + (long)r * (ncols / 16) + b * 16);
}
// RAWINT4 counterparts of the two kernels above: rows of `src` (hidden type) -> NP bf16 planes [nrows][NP][ncols], and
// a = act(g) * u (fp32, sorted pair rows, the per-pair kernels' formula) -> 3 planes; one thread per 8 values
template <int NP>
__global__ void __launch_bounds__(256) grp_split_x_kernel(const void* src, int hidden_type, int nrows, int ncols, uint16_t* out) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x, n8 = ncols / 8;
    if (i >= (long)nrows * n8) return;
    const long r = i / n8, c = (i - r * n8) * 8;
    float x[8];
    load_block8(src, r * ncols + c, hidden_type, x);
    i4_split8<NP>(x, out + r * NP * ncols + c, ncols);
}
__global__ void __launch_bounds__(256) grp_split_act_kernel(const float* g, const float* u, const int* offsets, int E, int ncols, int use_silu, uint16_t* out) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x, n8 = ncols / 8;
    if (i >= (long)offsets[E] * n8) return;
    const long r = i / n8, c = (i - r * n8) * 8, o = r * ncols + c;
    const float4 g0 = *reinterpret_cast<const float4*>(g + o), g1 = *reinterpret_cast<const float4*>(g + o + 4);
    const float4 u0 = *reinterpret_cast<const float4*>(u + o), u1 = *reinterpret_cast<const float4*>(u + o + 4);
    const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w}, uv[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
    float x[8];
#pragma unroll
    for (int j = 0; j < 8; j++) x[j] = (use_silu ? act_silu(gv[j]) : act_relu(gv[j])) * uv[j];
    i4_split8<3>(x, out + r * 3 * ncols + c, ncols);
}
// out[t] = sum_j w[t][j] * down[pos[t][j]] in expert_ids order, one FMA per expert (moe.cpp:340-358), rounded like from_float
__global__ void __launch_bounds__(256) grp_combine_kernel(const float* dd, const int* pos, const float* weights, int T, int k, int H, const int* bsz, int t0, void* out,
                                                          int hidden_type) {
    const int t = blockIdx.y;
    if (bsz && t0 + t >= *bsz) return;
    const int h = blockIdx.x * blockDim.x + threadIdx.x;
    if (h >= H) return;
    float acc = 0.f;
    for (int j = 0; j < k; j++) {
        const int s = pos[t * k + j];
        if (s >= 0) acc = __fmaf_rn(dd[(long)s * H + h], weights[t * k + j], acc);
    }
    store_hidden(out, (long)t * H + h, hidden_type, acc);
}

struct GrpScratch {
    size_t cap_pairs = 0, cap_x = 0, cap_a = 0, cap_d = 0;   // pairs, tokens * H, pairs * I, pairs * H
    int *counts = nullptr, *offsets = nullptr, *nt_prefix = nullptr, *cursor = nullptr, *tokmap = nullptr, *pos = nullptr;
    int4 *tinfo_gu = nullptr, *tinfo_d = nullptr;
    size_t cap_tiles_gu = 0, cap_tiles_d = 0;
    int8_t *xq = nullptr, *aq = nullptr;
    float *xd = nullptr, *ad = nullptr, *g = nullptr, *u = nullptr, *dd = nullptr;
    int16_t *xbs = nullptr, *abs16 = nullptr;
    size_t cap_xp = 0, cap_ap = 0;           // RAWINT4 bf16 planes (elements): tokens * 3 H, pairs * 3 I
    uint16_t *xp = nullptr, *ap = nullptr;
};
static long long* g_grp_trace = nullptr;
void grouped_set_trace(long long* t) { g_grp_trace = t; }
static GrpScratch g_grp[64];   // one arena per device, shared by every handle (calls on one device are stream-ordered by the caller)

// planes: the handle is RAWINT4 and needs the bf16 plane buffers (other handles leave them as they are)
static int grp_ensure(int dev, int tokens, int k, int E, int H, int I, bool planes) {
    GrpScratch& s = g_grp[dev & 63];
    size_t P = (size_t)tokens * k, nx = (size_t)tokens * H, na = P * I, nd = P * H;
    size_t tg = (P / kGN + E) * (size_t)(I / kGM), td = (P / kGN + E) * (size_t)(H / kGM);   // upper bounds of the tile counts
    size_t nxp = planes ? 3 * nx : 0, nap = planes ? 3 * na : 0;
    if (s.cap_pairs >= P && s.cap_x >= nx && s.cap_a >= na && s.cap_d >= nd && s.cap_tiles_gu >= tg && s.cap_tiles_d >= td && s.cap_xp >= nxp &&
        s.cap_ap >= nap)
        return KTB200_OK;
    tg = tg > s.cap_tiles_gu ? tg : s.cap_tiles_gu; td = td > s.cap_tiles_d ? td : s.cap_tiles_d;
    P = P > s.cap_pairs ? P : s.cap_pairs; nx = nx > s.cap_x ? nx : s.cap_x; na = na > s.cap_a ? na : s.cap_a; nd = nd > s.cap_d ? nd : s.cap_d;   // grow only
    nxp = nxp > s.cap_xp ? nxp : s.cap_xp; nap = nap > s.cap_ap ? nap : s.cap_ap;
    KTB_CUDA_CHECK(cudaDeviceSynchronize());   // earlier calls may still be using the arena
    cudaFree(s.counts); cudaFree(s.tokmap); cudaFree(s.pos); cudaFree(s.xq); cudaFree(s.xd); cudaFree(s.xbs); cudaFree(s.aq); cudaFree(s.ad); cudaFree(s.abs16);
    cudaFree(s.g); cudaFree(s.u); cudaFree(s.dd); cudaFree(s.tinfo_gu); cudaFree(s.tinfo_d); cudaFree(s.xp); cudaFree(s.ap);
    s = GrpScratch();
    if (nxp) KTB_CUDA_CHECK(cudaMalloc(&s.xp, nxp * sizeof(uint16_t)));
    if (nap) KTB_CUDA_CHECK(cudaMalloc(&s.ap, nap * sizeof(uint16_t)));
    s.cap_xp = nxp; s.cap_ap = nap;
    const size_t cp = P;
    KTB_CUDA_CHECK(cudaMalloc(&s.counts, (size_t)(4 * 1024 + 8) * sizeof(int)));
    s.offsets = s.counts + 1024; s.nt_prefix = s.counts + 2048 + 1; s.cursor = s.counts + 3072 + 2;
    KTB_CUDA_CHECK(cudaMalloc(&s.tokmap, cp * sizeof(int)));
    KTB_CUDA_CHECK(cudaMalloc(&s.pos, cp * sizeof(int)));
    KTB_CUDA_CHECK(cudaMalloc(&s.xq, nx));
    KTB_CUDA_CHECK(cudaMalloc(&s.xd, nx / 256 * sizeof(float)));
    KTB_CUDA_CHECK(cudaMalloc(&s.xbs, nx / 16 * sizeof(int16_t)));
    KTB_CUDA_CHECK(cudaMalloc(&s.aq, na));
    KTB_CUDA_CHECK(cudaMalloc(&s.ad, na / 256 * sizeof(float)));
    KTB_CUDA_CHECK(cudaMalloc(&s.abs16, na / 16 * sizeof(int16_t)));
    KTB_CUDA_CHECK(cudaMalloc(&s.g, na * sizeof(float)));
    KTB_CUDA_CHECK(cudaMalloc(&s.u, na * sizeof(float)));
    KTB_CUDA_CHECK(cudaMalloc(&s.dd, nd * sizeof(float)));
    KTB_CUDA_CHECK(cudaMalloc(&s.tinfo_gu, tg * sizeof(int4)));
    KTB_CUDA_CHECK(cudaMalloc(&s.tinfo_d, td * sizeof(int4)));
    s.cap_pairs = cp; s.cap_x = nx; s.cap_a = na; s.cap_d = nd; s.cap_tiles_gu = tg; s.cap_tiles_d = td;
    return KTB200_OK;
}

// the grouped_gemm_kernel format of one weight tensor (gate, up and down are separate launches), -1: none.  Q6_K only in the
// 4-row tile layout, which ktb200_moe_load_weights gives down tensors of eligible shapes.
static int grouped_fmt(int type, int layout) {
    if (type == KTB200_TYPE_Q4_K) return 0;
    if (type == KTB200_TYPE_Q6_K && layout == LAYOUT_T4) return 1;
    if (type == KTB200_TYPE_IQ1_S) return 2;
    if (type == KTB200_TYPE_IQ2_XXS) return 3;
    if (type == KTB200_TYPE_RAWINT4_G32) return 4;   // grouped_i4_kernel (NP picked per launch), never mixed with the others
    if (type == KTB200_TYPE_Q5_K) return 5;
    if (type == KTB200_TYPE_Q3_K) return 6;
    if (type == KTB200_TYPE_Q2_K) return 7;
    if (type == KTB200_TYPE_IQ1_M) return 8;
    if (type == KTB200_TYPE_IQ3_XXS) return 9;
    if (type == KTB200_TYPE_IQ3_S) return 10;
    if (type == KTB200_TYPE_IQ2_XS) return 11;
    if (type == KTB200_TYPE_IQ2_S) return 12;
    return -1;
}
static void grouped_i4(int np, const GrpI4Params& p, int grid, cudaStream_t s) {
    if (np == 1) grouped_i4_kernel<1><<<grid, kGThreads, I4Plan<1>::kSmem, s>>>(p);
    else grouped_i4_kernel<3><<<grid, kGThreads, I4Plan<3>::kSmem, s>>>(p);
}
static void grouped_gemm(int fmt, const GrpGemmParams& p, int grid, cudaStream_t s) {
    switch (fmt) {
        case 0: grouped_gemm_kernel<0><<<grid, kGThreads, kGSmem, s>>>(p); break;
        case 1: grouped_gemm_kernel<1><<<grid, kGThreads, kGSmem, s>>>(p); break;
        case 2: grouped_gemm_kernel<2><<<grid, kGThreads, kGSmemI, s>>>(p); break;
        case 3: grouped_gemm_kernel<3><<<grid, kGThreads, kGSmemI, s>>>(p); break;
        case 5: grouped_gemm_kernel<5><<<grid, kGThreads, kGSmem, s>>>(p); break;
        case 6: grouped_gemm_kernel<6><<<grid, kGThreads, kGSmem, s>>>(p); break;
        case 7: grouped_gemm_kernel<7><<<grid, kGThreads, kGSmem, s>>>(p); break;
        case 8: grouped_gemm_kernel<8><<<grid, kGThreads, kGSmemM, s>>>(p); break;
        case 9: grouped_gemm_kernel<9><<<grid, kGThreads, kGSmem3, s>>>(p); break;
        case 10: grouped_gemm_kernel<10><<<grid, kGThreads, kGSmem3, s>>>(p); break;
        case 11: grouped_gemm_kernel<11><<<grid, kGThreads, kGSmemI2, s>>>(p); break;
        default: grouped_gemm_kernel<12><<<grid, kGThreads, kGSmemI2, s>>>(p); break;
    }
}

// true when ktb200_moe_forward may take the grouped tensor-core path for this handle: gate and up Q4_K, Q5_K, Q3_K, Q2_K, IQ1_S,
// IQ1_M, IQ2_XXS, IQ2_XS, IQ2_S, IQ3_XXS or IQ3_S (each on its own), down any of those or Q6_K in the tile layout; or all three
// RAWINT4_G32
bool grouped_ok(const ktb200_moe* m, int k) {
    const ktb200_moe_config& c = m->cfg;
    const int fg = grouped_fmt(c.gate_type, LAYOUT_RAW), fu = grouped_fmt(c.up_type, LAYOUT_RAW), fd = grouped_fmt(c.down_type, m->down_layout);
    return fg >= 0 && fg != 1 && fu >= 0 && fu != 1 && fd >= 0 && (fg == 4) == (fu == 4) && (fu == 4) == (fd == 4) && c.hidden_size % 256 == 0 &&
           c.intermediate_size % 256 == 0 && c.hidden_size % kGM == 0 && c.intermediate_size % kGM == 0 && c.expert_num <= 1023 && k <= 32;
}

int moe_forward_grouped(ktb200_moe* m, int qlen, int k, const int64_t* ids, const float* weights, const void* input, void* output, const int* bsz, cudaStream_t s,
                        int out_type) {
    const ktb200_moe_config& c = m->cfg;
    const int E = c.expert_num, H = c.hidden_size, I = c.intermediate_size, dev = m->device;
    static const int chunk_cap = [] { const char* e = getenv("KTB200_GROUPED_CHUNK"); return e ? atoi(e) : 1024; }();
    const int Tc = qlen < chunk_cap ? qlen : chunk_cap;
    const int fg = grouped_fmt(c.gate_type, LAYOUT_RAW), fu = grouped_fmt(c.up_type, LAYOUT_RAW), fd = grouped_fmt(c.down_type, m->down_layout);
    const bool i4 = fg == 4;
    const int np = c.hidden_type == KTB200_TYPE_BF16 ? 1 : 3;   // RAWINT4 gate/up planes: one holds bf16, three any fp32
    int rc = grp_ensure(dev, Tc, k, E, H, I, i4);   // grow-only scratch: not capturable on first use (like ktb200_moe_gate_forward)
    if (rc) return rc;
    GrpScratch& g = g_grp[dev & 63];
    static bool attr[64] = {};
    if (!attr[dev & 63]) {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmem));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmem));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmemI));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmemI));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmem));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmem));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<7>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmem));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmemM));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<9>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmem3));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<10>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmem3));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<11>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmemI2));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<12>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmemI2));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_i4_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, I4Plan<1>::kSmem));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_i4_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, I4Plan<3>::kSmem));
        attr[dev & 63] = true;
    }
    const size_t hb = type_size(c.hidden_type), ob = type_size(out_type);
    const int grid = num_sms(dev);
    for (int t0 = 0; t0 < qlen; t0 += Tc) {
        const int T = qlen - t0 < Tc ? qlen - t0 : Tc, P = T * k;
        const int64_t* ids_c = ids + (size_t)t0 * k;
        const float* w_c = weights + (size_t)t0 * k;
        const uint8_t* x_c = reinterpret_cast<const uint8_t*>(input) + (size_t)t0 * H * hb;
        uint8_t* o_c = reinterpret_cast<uint8_t*>(output) + (size_t)t0 * H * ob;
        KTB_CUDA_CHECK(cudaMemsetAsync(g.counts, 0, (size_t)E * sizeof(int), s));
        grp_count_kernel<<<(P + 255) / 256, 256, 0, s>>>(ids_c, P, k, c.expert_id_offset, E, bsz, t0, g.counts);
        grp_scan_kernel<<<1, 32, 0, s>>>(g.counts, E, g.offsets, g.nt_prefix, g.cursor);
        grp_scatter_kernel<<<(P + 255) / 256, 256, 0, s>>>(ids_c, P, k, c.expert_id_offset, E, bsz, t0, g.cursor, g.tokmap, g.pos);
        const int ub_gu = (P / kGN + E) * (I / kGM), ub_d = (P / kGN + E) * (H / kGM);
        grp_tiles_kernel<<<(ub_gu + 255) / 256, 256, 0, s>>>(g.nt_prefix, g.offsets, E, I / kGM, g.tinfo_gu);
        grp_tiles_kernel<<<(ub_d + 255) / 256, 256, 0, s>>>(g.nt_prefix, g.offsets, E, H / kGM, g.tinfo_d);
        if (i4) {   // the same ten launches with the plane splits in place of the Q8_K quantisers
            if (np == 1) grp_split_x_kernel<1><<<(T * (H / 8) + 255) / 256, 256, 0, s>>>(x_c, c.hidden_type, T, H, g.xp);
            else grp_split_x_kernel<3><<<(T * (H / 8) + 255) / 256, 256, 0, s>>>(x_c, c.hidden_type, T, H, g.xp);
            GrpI4Params ip{};
            ip.R = I; ip.Kc = H; ip.x = g.xp; ip.rowmap = g.tokmap; ip.tinfo = g.tinfo_gu; ip.nt_prefix = g.nt_prefix; ip.E = E;
            ip.expert_bytes = (long)I * (H / 256) * SZ_RAWINT4;
            ip.w = reinterpret_cast<const uint8_t*>(c.gate_proj); ip.out = g.g; ip.trace = g_grp_trace;
            grouped_i4(np, ip, grid, s);
            ip.w = reinterpret_cast<const uint8_t*>(c.up_proj); ip.out = g.u; ip.trace = nullptr;
            grouped_i4(np, ip, grid, s);
            grp_split_act_kernel<<<(P * (I / 8) + 255) / 256, 256, 0, s>>>(g.g, g.u, g.offsets, E, I, c.use_silu, g.ap);
            GrpI4Params id{};
            id.R = H; id.Kc = I; id.x = g.ap; id.rowmap = nullptr; id.tinfo = g.tinfo_d; id.nt_prefix = g.nt_prefix; id.E = E;
            id.expert_bytes = (long)H * (I / 256) * SZ_RAWINT4;
            id.w = reinterpret_cast<const uint8_t*>(c.down_proj); id.out = g.dd; id.trace = g_grp_trace ? g_grp_trace + 3 * 96 * 4 : nullptr;
            grouped_i4(3, id, grid, s);
        } else {
            grp_quant_x_kernel<<<(T * (H / 256) + 7) / 8, 256, 0, s>>>(x_c, c.hidden_type, T, H, g.xq, g.xd, g.xbs);
            GrpGemmParams gp{};
            gp.R = I; gp.Kc = H; gp.xq = g.xq; gp.xd = g.xd; gp.xbs = g.xbs; gp.rowmap = g.tokmap; gp.tinfo = g.tinfo_gu; gp.nt_prefix = g.nt_prefix; gp.E = E;
            gp.expert_bytes = (long)I * (H / 256) * weight_block_bytes(c.gate_type);
            gp.w = reinterpret_cast<const uint8_t*>(c.gate_proj); gp.out = g.g; gp.trace = g_grp_trace;
            grouped_gemm(fg, gp, grid, s);
            gp.expert_bytes = (long)I * (H / 256) * weight_block_bytes(c.up_type);
            gp.w = reinterpret_cast<const uint8_t*>(c.up_proj); gp.out = g.u; gp.trace = nullptr;
            grouped_gemm(fu, gp, grid, s);
            grp_act_quant_kernel<<<(P * (I / 256) + 7) / 8, 256, 0, s>>>(g.g, g.u, g.offsets, E, I, c.use_silu, g.aq, g.ad, g.abs16);
            GrpGemmParams gd{};
            gd.R = H; gd.Kc = I; gd.xq = g.aq; gd.xd = g.ad; gd.xbs = g.abs16; gd.rowmap = nullptr; gd.tinfo = g.tinfo_d; gd.nt_prefix = g.nt_prefix;
            gd.E = E; gd.expert_bytes = (long)H * (I / 256) * weight_block_bytes(c.down_type);
            gd.w = reinterpret_cast<const uint8_t*>(c.down_proj); gd.out = g.dd; gd.trace = g_grp_trace ? g_grp_trace + 3 * 96 * 4 : nullptr;
            grouped_gemm(fd, gd, grid, s);
        }
        grp_combine_kernel<<<dim3((H + 255) / 256, T), 256, 0, s>>>(g.dd, g.pos, w_c, T, k, H, bsz, t0, o_c, out_type);
        KTB_LAUNCH_CHECK();
        count_launch(9);   // + the one KTB_LAUNCH_CHECK counts = 10 launches per chunk
    }
    return KTB200_OK;
}

// The arena's Q8_K activation buffers (xq, xd, xbs) for the tiled linear GEMM (gguf_gemm.cu): at least `need` values (tokens x
// in_features), grown to `grow` when they hold fewer.  Growing is synchronous and cannot be captured: on a capturing stream
// it returns KTB200_ESTATE before any device work, and the caller names the warm-up.
int grp_prompt_x(int dev, size_t need, size_t grow, cudaStream_t s, GrpX* out) {
    GrpScratch& g = g_grp[dev & 63];
    if (g.cap_x < need) {
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        KTB_CUDA_CHECK(cudaStreamIsCapturing(s, &cs));
        if (cs != cudaStreamCaptureStatusNone) return KTB200_ESTATE;
        const size_t nx = grow > need ? grow : need;
        KTB_CUDA_CHECK(cudaDeviceSynchronize());   // earlier calls may still be using the arena
        cudaFree(g.xq); cudaFree(g.xd); cudaFree(g.xbs);
        g.xq = nullptr; g.xd = nullptr; g.xbs = nullptr; g.cap_x = 0;
        KTB_CUDA_CHECK(cudaMalloc(&g.xq, nx));
        KTB_CUDA_CHECK(cudaMalloc(&g.xd, nx / 256 * sizeof(float)));
        KTB_CUDA_CHECK(cudaMalloc(&g.xbs, nx / 16 * sizeof(int16_t)));
        g.cap_x = nx;
    }
    *out = GrpX{g.xq, g.xd, g.xbs};
    return KTB200_OK;
}
// T rows of x (hidden type, [T][K]) -> Q8_K in those buffers: the grouped path's quantiser, one launch
int grp_prompt_quant(const void* x, int hidden_type, int T, int K, const GrpX& b, cudaStream_t s) {
    grp_quant_x_kernel<<<(T * (K / QK_K) + 7) / 8, 256, 0, s>>>(x, hidden_type, T, K, b.q, b.d, b.bs);
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

}  // namespace ktb
