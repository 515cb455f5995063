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
#include <cuda_fp16.h>

#include "act_quant.cuh"
#include "common.cuh"
#include "handles.cuh"
#include "wgmma.cuh"

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
template <int FMT>
__global__ void __launch_bounds__(kGThreads, 1) grouped_gemm_kernel(const GrpGemmParams p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base - raw);
    GrpMisc& misc = *reinterpret_cast<GrpMisc*>(smem + kOffMiscG);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nblk = p.Kc / QK_K, nst = 2 * nblk, MT = p.R / kGM;
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
        const uint32_t raw_dst = base + kOffRaw + pt * kRawPitch;
        const uint8_t* raw_src = smem + kOffRaw + pt * kRawPitch;
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
            if (FMT == 0 && pt < 64 && (pt >> 1) < ti.w) fbs = p.xbs + (long)(p.rowmap ? __ldg(p.rowmap + ti.z + (pt >> 1)) : ti.z + (pt >> 1)) * (p.Kc / 16) + (pt & 1) * 8;
            if (pt >= 64 && pt < 96 && pt - 64 < ti.w) fdx = p.xd + (long)(p.rowmap ? __ldg(p.rowmap + ti.z + pt - 64) : ti.z + pt - 64) * nblk;
            const int row = ti.y + r;
            if (FMT == 0) fw = p.w + (long)ti.x * p.expert_bytes + (long)row * nblk * SZ_Q4_K + 16 + part * 32;   // this thread's qs of block 0, first half
            else {
                fitem = p.w + (long)ti.x * p.expert_bytes + (long)(row >> 2) * 4 * nblk * SZ_Q6_K;
                ffi = (row & 3) * nblk;
                fw = fitem + (long)ffi * 16 + part * c16;
            }
        };
        auto issue = [&](uint32_t dst) {
            if (ftile < total_tiles) {
                const int hh = fst & 1;
                if (FMT == 0) {
                    const uint8_t* q = fw + hh * 64;
                    cp_async16(dst, q);
                    cp_async16(dst + 16, q + 16);
                    if (part == 0 || hh == 1) cp_async16(dst + 32, fw - 16 - part * 32);
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
                if (fxq) { cp_async16(dst + 48, fxq); fxq += 128; }
                if (hh == 1) {
                    if (FMT == 0 && fbs) { cp_async16(dst + 64, fbs); fbs += 16; }
                    if (fdx) { cp_async4(dst + (FMT == 0 ? 64 : 76), fdx); fdx += 1; }
                    fw += FMT == 0 ? SZ_Q4_K : 16;
                    ffi++;
                }
                if (++fst == nst) { fst = 0; ftile += gridDim.x; enter_tile(); }
            }
            cp_async_commit();
        };
        enter_tile();
        for (int i = 0; i < kGRaw; i++) issue(raw_dst + i * kRawSlot);
        int slot = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int4 ti = __ldg(p.tinfo + tile);
            const int n_valid = ti.w;
            int dsel = ((ti.y + r) & 3) * nblk;   // Q6_K: which half of the fetched word holds this block's d
            for (int st = 0; st < nst; st++) {
                const int hh = st & 1;
                const bool tr = p.trace && blockIdx.x == 0 && tid == 0 && tile == 0 && st < 96;
                if (tr) p.trace[(0 * 96 + st) * 4 + 0] = clock64();
                cp_async_wait<kGRaw - 1>();
                if (tr) p.trace[(0 * 96 + st) * 4 + 1] = clock64();
                const uint4* rs = reinterpret_cast<const uint4*>(raw_src + slot * kRawSlot);
                const uint4 f0 = rs[0], f1 = rs[1], f2 = rs[2], f3 = rs[3], f4 = rs[4];
                issue(raw_dst + slot * kRawSlot);   // refill the slot just read (thread-private bytes: no barrier involved)
                slot = slot == kGRaw - 1 ? 0 : slot + 1;
                bar_wait(smem_u32(&misc.smem_free[stage]), sphase ^ 1);
                bar_wait(smem_u32(&misc.hdr_free[hs]), hphase ^ 1);
                if (tr) p.trace[(0 * 96 + st) * 4 + 2] = clock64();
                uint8_t* arow = smem + stage * kGA + r * 128;
                const uint4 z = make_uint4(0, 0, 0, 0);
                if (FMT == 0) {
                    // chunk c = 2 hh + part (32 bytes of qs): low nibbles = sub-block 2c (elements 64c .. 64c+31), high nibbles = sub-block 2c+1
                    const int pi = 4 * part;
                    *reinterpret_cast<uint4*>(arow + (((pi + 0) ^ sw) << 4)) = make_uint4(f0.x & 0x0F0F0F0Fu, f0.y & 0x0F0F0F0Fu, f0.z & 0x0F0F0F0Fu, f0.w & 0x0F0F0F0Fu);
                    *reinterpret_cast<uint4*>(arow + (((pi + 1) ^ sw) << 4)) = make_uint4(f1.x & 0x0F0F0F0Fu, f1.y & 0x0F0F0F0Fu, f1.z & 0x0F0F0F0Fu, f1.w & 0x0F0F0F0Fu);
                    *reinterpret_cast<uint4*>(arow + (((pi + 2) ^ sw) << 4)) =
                        make_uint4((f0.x >> 4) & 0x0F0F0F0Fu, (f0.y >> 4) & 0x0F0F0F0Fu, (f0.z >> 4) & 0x0F0F0F0Fu, (f0.w >> 4) & 0x0F0F0F0Fu);
                    *reinterpret_cast<uint4*>(arow + (((pi + 3) ^ sw) << 4)) =
                        make_uint4((f1.x >> 4) & 0x0F0F0F0Fu, (f1.y >> 4) & 0x0F0F0F0Fu, (f1.z >> 4) & 0x0F0F0F0Fu, (f1.w >> 4) & 0x0F0F0F0Fu);
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
                uint8_t* Bs = smem + kOffB + stage * kGB;
                const uint4 bv = bn < n_valid ? f3 : z;
                if (FMT == 0) {
                    *reinterpret_cast<uint4*>(Bs + bn * 128 + ((pc ^ (bn & 7)) << 4)) = bv;
                } else {   // a 16-byte piece is one Q6_K sub-block: rows 0-31 keep the even pieces, rows 32-63 the odd ones
                    *reinterpret_cast<uint4*>(Bs + bn * 128 + ((pc ^ (bn & 7)) << 4)) = (pc & 1) ? z : bv;
                    *reinterpret_cast<uint4*>(Bs + (kGN + bn) * 128 + ((pc ^ (bn & 7)) << 4)) = (pc & 1) ? bv : z;
                }
                if (hh == 1 && pt < 96) {   // token scales, and (Q4_K) the sixteen 16-value sums of the super-block as fp16
                    if (pt >= 64) misc.dxs[hs][pt - 64] = pt - 64 < n_valid ? __uint_as_float(FMT == 0 ? f4.x : f4.w) : 0.f;
                    else if (FMT == 0) {
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
                const uint32_t a = base + stage * kGA + g * (kGA / 2), b = base + kOffB + stage * kGB;
                uint32_t hw[2][4];
#pragma unroll
                for (int h = 0; h < 2; h++) {
                    const uint4 hd = misc.hdr[hs][ra + 8 * h];
                    hw[h][0] = hd.x; hw[h][1] = hd.y; hw[h][2] = hd.z; hw[h][3] = hd.w;
                }
                if (FMT == 0) {
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
                    if (hh == 1) {
                        float ms[16];
                        fence();
                        mma_f16_m64n32(ms, smem_desc(base + kOffA2 + stage * kGA2 + g * (kGA2 / 2), 128, 256, kLayoutNone),
                                       smem_desc(base + kOffB2 + stage * kGB2, 128, 256, kLayoutNone), 0);
                        commit();
                        wait<0>();
                        fence_regs(ms);
#pragma unroll
                        for (int i = 0; i < 16; i++) {
                            const __half2 dm = *reinterpret_cast<const __half2*>(&hw[(i >> 1) & 1][0]);
                            const float dw = __low2float(dm), dmin = __high2float(dm);
                            const float dx = misc.dxs[hs][8 * (i >> 2) + cq + (i & 1)];
                            acc[i] += (dw * dx) * (float)isum[i] - (dmin * dx) * ms[i];
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
                    if (hh == 1) {
#pragma unroll
                        for (int i = 0; i < 16; i++) {
                            acc[i] += (__uint_as_float(hw[(i >> 1) & 1][2]) * misc.dxs[hs][8 * (i >> 2) + cq + (i & 1)]) * (float)isum[i];
                            isum[i] = 0;
                        }
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
};
static long long* g_grp_trace = nullptr;
void grouped_set_trace(long long* t) { g_grp_trace = t; }
static GrpScratch g_grp[64];   // one arena per device, shared by every handle (calls on one device are stream-ordered by the caller)

static int grp_ensure(int dev, int tokens, int k, int E, int H, int I) {
    GrpScratch& s = g_grp[dev & 63];
    size_t P = (size_t)tokens * k, nx = (size_t)tokens * H, na = P * I, nd = P * H;
    size_t tg = (P / kGN + E) * (size_t)(I / kGM), td = (P / kGN + E) * (size_t)(H / kGM);   // upper bounds of the tile counts
    if (s.cap_pairs >= P && s.cap_x >= nx && s.cap_a >= na && s.cap_d >= nd && s.cap_tiles_gu >= tg && s.cap_tiles_d >= td) return KTB200_OK;
    tg = tg > s.cap_tiles_gu ? tg : s.cap_tiles_gu; td = td > s.cap_tiles_d ? td : s.cap_tiles_d;
    P = P > s.cap_pairs ? P : s.cap_pairs; nx = nx > s.cap_x ? nx : s.cap_x; na = na > s.cap_a ? na : s.cap_a; nd = nd > s.cap_d ? nd : s.cap_d;   // grow only
    KTB_CUDA_CHECK(cudaDeviceSynchronize());   // earlier calls may still be using the arena
    cudaFree(s.counts); cudaFree(s.tokmap); cudaFree(s.pos); cudaFree(s.xq); cudaFree(s.xd); cudaFree(s.xbs); cudaFree(s.aq); cudaFree(s.ad); cudaFree(s.abs16);
    cudaFree(s.g); cudaFree(s.u); cudaFree(s.dd); cudaFree(s.tinfo_gu); cudaFree(s.tinfo_d);
    s = GrpScratch();
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

// true when ktb200_moe_forward may take the grouped tensor-core path for this handle
bool grouped_ok(const ktb200_moe* m, int k) {
    const ktb200_moe_config& c = m->cfg;
    const FmtId fd = pick_fmt(c.down_type, m->down_layout);
    return c.gate_type == KTB200_TYPE_Q4_K && c.up_type == KTB200_TYPE_Q4_K && (fd == FMT_Q6K4T || fd == FMT_Q4K) && c.hidden_size % 256 == 0 &&
           c.intermediate_size % 256 == 0 && c.hidden_size % kGM == 0 && c.intermediate_size % kGM == 0 && c.expert_num <= 1023 && k <= 32;
}

int moe_forward_grouped(ktb200_moe* m, int qlen, int k, const int64_t* ids, const float* weights, const void* input, void* output, const int* bsz, cudaStream_t s,
                        int out_type) {
    const ktb200_moe_config& c = m->cfg;
    const int E = c.expert_num, H = c.hidden_size, I = c.intermediate_size, dev = m->device;
    static const int chunk_cap = [] { const char* e = getenv("KTB200_GROUPED_CHUNK"); return e ? atoi(e) : 1024; }();
    const int Tc = qlen < chunk_cap ? qlen : chunk_cap;
    int rc = grp_ensure(dev, Tc, k, E, H, I);   // grow-only scratch: not capturable on first use (like ktb200_moe_gate_forward)
    if (rc) return rc;
    GrpScratch& g = g_grp[dev & 63];
    static bool attr[64] = {};
    if (!attr[dev & 63]) {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmem));
        KTB_CUDA_CHECK(cudaFuncSetAttribute(grouped_gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGSmem));
        attr[dev & 63] = true;
    }
    const FmtId fd = pick_fmt(c.down_type, m->down_layout);
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
        grp_quant_x_kernel<<<(T * (H / 256) + 7) / 8, 256, 0, s>>>(x_c, c.hidden_type, T, H, g.xq, g.xd, g.xbs);
        GrpGemmParams gp{};
        gp.R = I; gp.Kc = H; gp.xq = g.xq; gp.xd = g.xd; gp.xbs = g.xbs; gp.rowmap = g.tokmap; gp.tinfo = g.tinfo_gu; gp.nt_prefix = g.nt_prefix; gp.E = E;
        gp.expert_bytes = (long)I * (H / 256) * SZ_Q4_K;
        gp.w = reinterpret_cast<const uint8_t*>(c.gate_proj); gp.out = g.g; gp.trace = g_grp_trace;
        grouped_gemm_kernel<0><<<grid, kGThreads, kGSmem, s>>>(gp);
        gp.w = reinterpret_cast<const uint8_t*>(c.up_proj); gp.out = g.u; gp.trace = nullptr;
        grouped_gemm_kernel<0><<<grid, kGThreads, kGSmem, s>>>(gp);
        grp_act_quant_kernel<<<(P * (I / 256) + 7) / 8, 256, 0, s>>>(g.g, g.u, g.offsets, E, I, c.use_silu, g.aq, g.ad, g.abs16);
        GrpGemmParams gd{};
        gd.R = H; gd.Kc = I; gd.xq = g.aq; gd.xd = g.ad; gd.xbs = g.abs16; gd.rowmap = nullptr; gd.tinfo = g.tinfo_d; gd.nt_prefix = g.nt_prefix;
        gd.E = E; gd.expert_bytes = (long)H * (I / 256) * (fd == FMT_Q6K4T ? SZ_Q6_K : SZ_Q4_K);
        gd.w = reinterpret_cast<const uint8_t*>(c.down_proj); gd.out = g.dd; gd.trace = g_grp_trace ? g_grp_trace + 3 * 96 * 4 : nullptr;
        if (fd == FMT_Q6K4T) grouped_gemm_kernel<1><<<grid, kGThreads, kGSmem, s>>>(gd);
        else grouped_gemm_kernel<0><<<grid, kGThreads, kGSmem, s>>>(gd);
        grp_combine_kernel<<<dim3((H + 255) / 256, T), 256, 0, s>>>(g.dd, g.pos, w_c, T, k, H, bsz, t0, o_c, out_type);
        KTB_LAUNCH_CHECK();
        count_launch(9);   // + the one KTB_LAUNCH_CHECK counts = 10 launches per chunk
    }
    return KTB200_OK;
}

}  // namespace ktb
