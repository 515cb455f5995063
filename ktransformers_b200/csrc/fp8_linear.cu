// FP8 (e4m3, 128 x 128 block scales) linear for decode batches — KLinearFP8 (archive/ktransformers/operators/linear.py:388-435)
// = act_quant (fp8gemm.py:10-47) -> fp8_gemm (fp8gemm.py:104-192), DeepSeek-V3's native checkpoint format:
//     s[t][kb] = max|x[t][128 kb .. +128]| / 448,   xq = e4m3(x / s)                         (per token and 128 of K)
//     acc[t][n] += dot_e4m3(xq[t][kb], W[n][kb]) * s[t][kb] * scale_inv[n / 128][kb]          fp32, kb ascending
//     y = cast(acc)
// One byte per weight: a pure HBM stream.  TMA drops [128 rows x 128 bytes] boxes of W into shared memory (128-byte swizzle);
// each MMA warpgroup widens its 64 rows to fp16 in registers (exact: e4m3 is a subset of fp16) and feeds them as the A operand
// of an fp16 wgmma whose B operand is the quantised activations (16 token rows, padded), also held as fp16.  The products of two
// e4m3 values are exact and sum in fp32; the e4m3 form of the MMA would sum them with fewer bits on this architecture.  Every
// 128 of K (8 MMAs of K = 16) the partial dot is taken out of the accumulator and the two scales are applied in the
// reference's order.
// K order inside each 64-value half of a 128 block: the thread that supplies weight row r for the MMA reads 16 contiguous
// bytes, physical k = 16 c + 4 s + e (c = lane % 4, s = the K = 16 step of the half, e = 0..3), and hands them to the fragment
// slots that the MMA treats as logical k = 16 s + 2 c + e (e < 2) and 16 s + 8 + 2 c + (e - 2); the B tile stores x in that
// same logical order (a permutation of K inside a dot product changes nothing).
//     grid = (ceil(N / 128) row tiles, K splits), two CTAs per SM; 288 threads: warps 0-7 = two warpgroups of 64 weight rows
//     each (quantise x for the CTA's K range while the first weight boxes are in flight, then MMA and scale), warp 8 the TMA
//     producer (4-stage ring).
// K splits add their fp32 partial sums with atomics into a zeroed workspace; the last CTA of a row tile converts and re-zeroes.
//
// Prompt-sized batches (qlen >= fp8_prompt_min) take a second route that reads each weight once per token chunk instead of once
// per 16 tokens: fp8_gemm_quant_kernel quantises the chunk once into a per-device arena (fp16-widened e4m3 in the K order above,
// scales transposed to [kb][token]), then fp8_gemm_kernel computes [128 weight rows x 128 tokens] tiles with the same arithmetic:
//     grid = row tiles x token tiles (banded raster), one CTA per SM; 384 threads: warps 0-7 = two MMA warpgroups of 64 weight
//     rows x 128 tokens (widen the weights in registers, 8 fp16 wgmma m64n128k16 per 128 of K into a fresh accumulator, then
//     acc = acc + (dot * a_s) * b_s), warps 8-11 the TMA producer warpgroup (4-stage ring: weight box, two activation boxes and
//     the 128 token scales per stage).  No K splits: every output is written once, by one CTA, in kb order.
#include <cuda.h>
#include <cuda_fp8.h>

#include <new>

#include "common.cuh"
#include "handles.cuh"
#include "wgmma.cuh"

namespace ktb {
using namespace wg;

constexpr int kFT = 16;                    // token rows per pass (the MMA's N)
constexpr int kFStages = 4, kFA = 128 * 128, kFB = kFT * 128 * 2, kFMaxKb = 8;   // 64 + 32 KB: two CTAs per SM, 128 KB of weight boxes in flight
constexpr int kFOffB = kFStages * kFA, kFOffS = kFOffB + kFMaxKb * kFB, kFOffMisc = kFOffS + kFT * kFMaxKb * 4;
constexpr int kFConsumerWarps = 8, kFThreads = (kFConsumerWarps + 1) * 32;
struct Fp8Misc {
    unsigned long long a_full[kFStages], a_free[kFStages];
    int last;
};
constexpr int kFSmem = kFOffMisc + (int)sizeof(Fp8Misc) + 1024;

struct Fp8Params {
    const void* x;            // [T][K] hidden type
    void* y;                  // [T][N]
    const float* scale_inv;   // [ceil(N/128)][nkb]
    float* ws;                // [kFT][N] fp32, zero between calls (K splits only)
    unsigned* tickets;        // [row tiles], zero between calls
    const int* bsz;
    const uint8_t* xq;        // [T][K] e4m3 and
    const float* xs;          // [T][nkb] scales from fp8_act_quant_kernel (batches of more than 2 tokens), else null
    int hidden_type, T, K, N, nkb, kb_per_split, ksplit, t0;
};

// act_quant (fp8gemm.py:10-27) for one (token, 128 values) block held 4 values per lane: returns the scale, packs the 4 e4m3 bytes
__device__ __forceinline__ float fp8_quant_block(const float (&v)[4], uint32_t& packed) {
    float am = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
    const float s = __fdiv_rn(am, 448.f);
    packed = 0;
#pragma unroll
    for (int e = 0; e < 4; e++)   // x / s in IEEE fp32, round to nearest even into e4m3 (0 / 0 = NaN like the reference)
        packed |= (uint32_t)__nv_cvt_float_to_fp8(__fdiv_rn(v[e], s), __NV_SATFINITE, __NV_E4M3) << (8 * e);
    return s;
}
__device__ __forceinline__ void fp8_load4(const void* x, long off, int hidden_type, float (&v)[4]) {
    if (hidden_type == KTB200_TYPE_F32) {
        const float4 f = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(x) + off);
        v[0] = f.x; v[1] = f.y; v[2] = f.z; v[3] = f.w;
    } else {
        const uint2 w2 = *reinterpret_cast<const uint2*>(reinterpret_cast<const uint16_t*>(x) + off);
        const uint32_t ww[2] = {w2.x, w2.y};
#pragma unroll
        for (int e = 0; e < 2; e++) {
            if (hidden_type == KTB200_TYPE_BF16) { v[2 * e] = __uint_as_float(ww[e] << 16); v[2 * e + 1] = __uint_as_float(ww[e] & 0xffff0000u); }
            else { v[2 * e] = fp16_bits_to_f32((uint16_t)(ww[e] & 0xffff)); v[2 * e + 1] = fp16_bits_to_f32((uint16_t)(ww[e] >> 16)); }
        }
    }
}
// 4 e4m3 bytes (physical k = 4 q .. 4 q + 3 of a 128 block) of token row t -> the fp16 B tile of that block (see the K order above)
__device__ __forceinline__ void fp8_store_b(uint8_t* bt, int t, int q, uint32_t packed) {
    const int h = q >> 4, c = (q >> 2) & 3, s = q & 3, l0 = 16 * s + 2 * c, l1 = l0 + 8;
    const __half2_raw lo = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(packed & 0xffffu), __NV_E4M3);
    const __half2_raw hi = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(packed >> 16), __NV_E4M3);
    uint8_t* row = bt + h * (kFT * 128) + t * 128;
    *reinterpret_cast<uint32_t*>(row + (((l0 >> 3) ^ (t & 7)) << 4) + (l0 & 7) * 2) = (uint32_t)lo.x | ((uint32_t)lo.y << 16);
    *reinterpret_cast<uint32_t*>(row + (((l1 >> 3) ^ (t & 7)) << 4) + (l1 & 7) * 2) = (uint32_t)hi.x | ((uint32_t)hi.y << 16);
}
__device__ __forceinline__ uint32_t fp8x2_to_f16x2(uint32_t two) {
    const __half2_raw v = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)two, __NV_E4M3);
    return (uint32_t)v.x | ((uint32_t)v.y << 16);
}
// batches of more than 2 tokens: quantise x ONCE (one warp per block) instead of once per row tile
__global__ void __launch_bounds__(256) fp8_act_quant_kernel(const void* x, int hidden_type, int T, int K, uint8_t* xq, float* xs) {
    const int lane = threadIdx.x & 31, blk = blockIdx.x * 8 + (threadIdx.x >> 5), nkb = K / 128;
    griddep_launch_dependents();
    if (blk >= T * nkb) return;
    const int t = blk / nkb, kb = blk - t * nkb;
    float v[4];
    fp8_load4(x, (long)t * K + (long)kb * 128 + lane * 4, hidden_type, v);
    uint32_t packed;
    const float s = fp8_quant_block(v, packed);
    reinterpret_cast<uint32_t*>(xq + (long)t * K + (long)kb * 128)[lane] = packed;
    if (lane == 0) xs[t * nkb + kb] = s;
}

__global__ void __launch_bounds__(kFThreads, 2) fp8_linear_kernel(const __grid_constant__ CUtensorMap wmap, const Fp8Params p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base - raw);
    Fp8Misc& misc = *reinterpret_cast<Fp8Misc*>(smem + kFOffMisc);
    float* a_s = reinterpret_cast<float*>(smem + kFOffS);   // [kFT][kb_per_split]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int row0 = blockIdx.x * 128;
    const int kb0 = blockIdx.y * p.kb_per_split, nk = min(p.kb_per_split, p.nkb - kb0);
    if (tid == 0) {
        for (int s = 0; s < kFStages; s++) { bar_init(smem_u32(&misc.a_full[s]), 1); bar_init(smem_u32(&misc.a_free[s]), kFConsumerWarps); }
        bar_fence_init();
        tma_prefetch_desc(&wmap);
    }
    __syncthreads();
    griddep_launch_dependents();   // a PDL-launched successor may set up and prefetch its own weights while this grid streams

    if (warp == kFConsumerWarps) {
        // ---------------------------------------------------------------- weight boxes: independent of x, start at once
        if (lane == 0) {
            for (int i = 0; i < nk; i++) {
                const int s = i % kFStages;
                bar_wait(smem_u32(&misc.a_free[s]), ((i / kFStages) & 1) ^ 1);
                bar_expect_tx(smem_u32(&misc.a_full[s]), kFA);
                tma_load_2d(base + s * kFA, &wmap, smem_u32(&misc.a_full[s]), (kb0 + i) * 128, row0);
            }
        }
        return;
    }
    // -------------------------------------------------------------------- act_quant for this K range (warps 0-7)
    constexpr int kCT = kFConsumerWarps * 32;
    // rows T .. 15 of the B tiles: zeros (their accumulator columns are never read)
    for (int i = tid; i < nk * (kFB / 16); i += kCT) {
        const int r = (i >> 3) & (kFT - 1);
        if (r >= p.T) *reinterpret_cast<uint4*>(smem + kFOffB + i * 16) = make_uint4(0, 0, 0, 0);
    }
    griddep_wait();   // x (or its quantised copy) comes from the kernel before this one; the weight boxes above did not wait
    if (p.xq) {
        // already quantised by fp8_act_quant_kernel: this CTA's K range into the B tiles, 4 bytes per thread and step
        for (int i = tid; i < p.T * nk * 32; i += kCT) {
            const int q = i & 31, kb = (i >> 5) % nk, t = (i >> 5) / nk;
            fp8_store_b(smem + kFOffB + kb * kFB, t, q, *reinterpret_cast<const uint32_t*>(p.xq + (long)t * p.K + (long)(kb0 + kb) * 128 + q * 4));
        }
        for (int i = tid; i < p.T * nk; i += kCT) a_s[(i / nk) * p.kb_per_split + (i % nk)] = p.xs[(i / nk) * p.nkb + kb0 + (i % nk)];
    } else {
        // one warp per (token, 128 of K), lane owns 4 consecutive values; 8 blocks' loads are issued before the first is reduced
        for (int g0 = warp; g0 < p.T * nk; g0 += kFConsumerWarps * 8) {
            float v[8][4];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int blk = g0 + kFConsumerWarps * u;
                if (blk < p.T * nk) {
                    const int t = blk / nk, kb = blk - t * nk;
                    fp8_load4(p.x, (long)t * p.K + (long)(kb0 + kb) * 128 + lane * 4, p.hidden_type, v[u]);
                }
            }
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const int blk = g0 + kFConsumerWarps * u;
                if (blk < p.T * nk) {   // warp-uniform
                    const int t = blk / nk, kb = blk - t * nk;
                    uint32_t packed;
                    const float s = fp8_quant_block(v[u], packed);
                    fp8_store_b(smem + kFOffB + kb * kFB, t, lane, packed);
                    if (lane == 0) a_s[t * p.kb_per_split + kb] = s;
                }
            }
        }
    }
    fence_async_smem();
    asm volatile("bar.sync 1, %0;" ::"n"(kCT) : "memory");   // B tiles and a_s are read by both warpgroups

    // -------------------------------------------------------------------- MMA + scales: warpgroup g owns weight rows 64 g .. 64 g + 63
    const int g = warp >> 2, r0 = 64 * g + 16 * (warp & 3) + (lane >> 2), c = lane & 3;
    float acc[8], d[8];
#pragma unroll
    for (int q = 0; q < 8; q++) acc[q] = 0.f;
    const float* sinv = p.scale_inv + (long)blockIdx.x * p.nkb + kb0;
    for (int i = 0; i < nk; i++) {
        const int s = i % kFStages;
        const float bs = __ldg(sinv + i);
        bar_wait(smem_u32(&misc.a_full[s]), (i / kFStages) & 1);
        uint4 w[2][2];   // [row r0, r0 + 8][half of the 128 block]: bytes 16 c .. 16 c + 15 of the half
#pragma unroll
        for (int rr = 0; rr < 2; rr++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int r = r0 + 8 * rr;
                w[rr][h] = *reinterpret_cast<const uint4*>(smem + s * kFA + r * 128 + ((((4 * h + c) ^ (r & 7))) << 4));
            }
        uint32_t a[2][4][4];   // all A fragments of the block before the first MMA: no register writes between the MMAs
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int st = 0; st < 4; st++) {
                const uint32_t w0 = st == 0 ? w[0][h].x : st == 1 ? w[0][h].y : st == 2 ? w[0][h].z : w[0][h].w;
                const uint32_t w1 = st == 0 ? w[1][h].x : st == 1 ? w[1][h].y : st == 2 ? w[1][h].z : w[1][h].w;
                a[h][st][0] = fp8x2_to_f16x2(w0 & 0xffffu); a[h][st][1] = fp8x2_to_f16x2(w1 & 0xffffu);
                a[h][st][2] = fp8x2_to_f16x2(w0 >> 16); a[h][st][3] = fp8x2_to_f16x2(w1 >> 16);
            }
        fence();
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int st = 0; st < 4; st++)
                mma_f16_rs_m64n16(d, a[h][st], smem_desc(base + kFOffB + i * kFB + h * (kFT * 128) + st * 32, 16, 1024, kLayoutSw128), (h | st) != 0);
        commit();
        wait<0>();
        fence_regs(d);
        // free the stage only now: the MMAs that consumed the registers loaded from it have completed, so every one of those
        // shared-memory loads has delivered before TMA may overwrite the stage
        __syncwarp();
        if (lane == 0) bar_arrive(smem_u32(&misc.a_free[s]));
#pragma unroll
        for (int q = 0; q < 8; q++) {   // register q: token 8 (q / 4) + 2 (lane % 4) + q % 2, row r0 + 8 (q / 2 % 2)
            const int t = 8 * (q >> 2) + 2 * (lane & 3) + (q & 1);
            if (t < p.T) acc[q] = __fadd_rn(acc[q], __fmul_rn(__fmul_rn(d[q], a_s[t * p.kb_per_split + i]), bs));   // (dot * a_s) * b_s, then +=
        }
    }
    const int live = p.bsz ? max(0, min(p.T, *p.bsz - p.t0)) : p.T;   // rows at or beyond the live batch size stay untouched
    if (p.ksplit == 1) {
#pragma unroll
        for (int q = 0; q < 8; q++) {
            const int t = 8 * (q >> 2) + 2 * (lane & 3) + (q & 1), n = row0 + r0 + 8 * ((q >> 1) & 1);
            if (t < live && n < p.N) store_hidden(p.y, (long)t * p.N + n, p.hidden_type, acc[q]);
        }
    } else {
#pragma unroll
        for (int q = 0; q < 8; q++) {
            const int t = 8 * (q >> 2) + 2 * (lane & 3) + (q & 1), n = row0 + r0 + 8 * ((q >> 1) & 1);
            if (t < p.T && n < p.N) atomicAdd(p.ws + (long)t * p.N + n, acc[q]);
        }
        __threadfence();
        asm volatile("bar.sync 1, %0;" ::"n"(kCT) : "memory");
        if (tid == 0) misc.last = atomicAdd(p.tickets + blockIdx.x, 1u) == (unsigned)(p.ksplit - 1);
        asm volatile("bar.sync 1, %0;" ::"n"(kCT) : "memory");
        if (misc.last) {
            __threadfence();
            for (int i = tid; i < 128 * p.T; i += kCT) {
                const int t = i >> 7, n = row0 + (i & 127);
                if (n < p.N) {
                    const float v = __ldcg(p.ws + (long)t * p.N + n);
                    p.ws[(long)t * p.N + n] = 0.f;
                    if (t < live) store_hidden(p.y, (long)t * p.N + n, p.hidden_type, v);
                }
            }
            if (tid == 0) p.tickets[blockIdx.x] = 0;
        }
    }
}

// ------------------------------------------------------------------------------------------------ prompt route
constexpr int kPT = 128;                                          // tokens per CTA (the MMA's N)
constexpr int kPStages = 4, kPA = 128 * 128, kPB = kPT * 128 * 2, kPS = kPT * 4;   // 16 KB weights + 32 KB fp16 x + 512 B scales
constexpr int kPOffB = kPStages * kPA, kPOffS = kPOffB + kPStages * kPB, kPOffMisc = kPOffS + kPStages * kPS;
constexpr int kPConsumerWarps = 8, kPThreads = (kPConsumerWarps + 4) * 32;
constexpr int kPChunk = 2048;                                     // tokens per GEMM launch: bounds the arena
constexpr int kPBand = 16;                                        // row tiles per raster band: a wave shares weight and x boxes in L2
struct Fp8GemmMisc {
    unsigned long long full[kPStages], free_[kPStages];
};
constexpr int kPSmem = kPOffMisc + (int)sizeof(Fp8GemmMisc) + 1024;

struct Fp8GemmParams {
    void* y;                  // [T][N], already offset to the chunk
    const float* scale_inv;   // [ceil(N/128)][nkb]
    const int* bsz;
    int hidden_type, T, N, nkb, row_tiles, token_tiles, t0;
};

// one warp per (token, 128 of K): fp8_quant_block, then the e4m3 values widened to fp16 at the K positions the GEMM's B tile
// expects (the physical -> logical map of fp8_store_b), scales transposed so that one token tile's 128 scales of a kb are contiguous
__global__ void __launch_bounds__(256) fp8_gemm_quant_kernel(const void* x, int hidden_type, int T, int K, int pitch, uint16_t* xh, float* xs) {
    const int lane = threadIdx.x & 31, blk = blockIdx.x * 8 + (threadIdx.x >> 5), nkb = K / 128;
    griddep_launch_dependents();
    if (blk >= T * nkb) return;
    const int t = blk / nkb, kb = blk - t * nkb;
    float v[4];
    fp8_load4(x, (long)t * K + (long)kb * 128 + lane * 4, hidden_type, v);
    uint32_t packed;
    const float s = fp8_quant_block(v, packed);
    const int l0 = 64 * (lane >> 4) + 16 * (lane & 3) + 2 * ((lane >> 2) & 3);
    uint32_t* row = reinterpret_cast<uint32_t*>(xh + (long)t * K + (long)kb * 128);
    row[l0 >> 1] = fp8x2_to_f16x2(packed & 0xffffu);
    row[(l0 + 8) >> 1] = fp8x2_to_f16x2(packed >> 16);
    if (lane == 0) xs[(long)kb * pitch + t] = s;
}

__global__ void __launch_bounds__(kPThreads, 1) fp8_gemm_kernel(const __grid_constant__ CUtensorMap wmap, const __grid_constant__ CUtensorMap xmap,
                                                                const __grid_constant__ CUtensorMap smap, const Fp8GemmParams p) {
    const int band_ctas = kPBand * p.token_tiles, band = blockIdx.x / band_ctas, in_band = blockIdx.x - band * band_ctas;
    const int band_rows = min(kPBand, p.row_tiles - band * kPBand);
    const int rt = band * kPBand + in_band % band_rows, tt = in_band / band_rows;
    const int live = p.bsz ? max(0, min(p.T, *p.bsz - p.t0)) : p.T;   // bsz was written before the quantiser (a full dependency)
    if (tt * kPT >= live) return;                                    // a token tile wholly beyond the live batch: no MMA, no store
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* smem = smem_raw + (base - raw);
    Fp8GemmMisc& misc = *reinterpret_cast<Fp8GemmMisc*>(smem + kPOffMisc);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        for (int s = 0; s < kPStages; s++) { bar_init(smem_u32(&misc.full[s]), 1); bar_init(smem_u32(&misc.free_[s]), kPConsumerWarps); }
        bar_fence_init();
        tma_prefetch_desc(&wmap); tma_prefetch_desc(&xmap); tma_prefetch_desc(&smap);
    }
    __syncthreads();

    if (warp >= kPConsumerWarps) {
        regs_dec<40>();
        if (warp == kPConsumerWarps && lane == 0) {
            griddep_wait();   // the quantised chunk comes from the kernel before this one
            for (int i = 0; i < p.nkb; i++) {
                const int s = i % kPStages;
                const uint32_t full = smem_u32(&misc.full[s]), bb = base + kPOffB + s * kPB;
                bar_wait(smem_u32(&misc.free_[s]), ((i / kPStages) & 1) ^ 1);
                bar_expect_tx(full, kPA + kPB + kPS);
                tma_load_2d(base + s * kPA, &wmap, full, i * 128, rt * 128);
                tma_load_2d(bb, &xmap, full, i * 128, tt * kPT);
                tma_load_2d(bb + kPT * 128, &xmap, full, i * 128 + 64, tt * kPT);
                tma_load_2d(base + kPOffS + s * kPS, &smap, full, tt * kPT, i);
            }
        }
        return;
    }
    regs_inc<232>();   // 128 x 40 + 256 x 232 <= 64 K registers
    // warpgroup g owns weight rows 64 g .. 64 g + 63 of the tile; register 4 j + e: row r0 + 8 (e / 2), token 8 j + 2 c + e % 2
    const int g = warp >> 2, r0 = 64 * g + 16 * (warp & 3) + (lane >> 2), c = lane & 3;
    float acc[64], d[64];
#pragma unroll
    for (int q = 0; q < 64; q++) acc[q] = 0.f;
    const float* sinv = p.scale_inv + (long)rt * p.nkb;
    for (int i = 0; i < p.nkb; i++) {
        const int s = i % kPStages;
        const float bs = __ldg(sinv + i);
        bar_wait(smem_u32(&misc.full[s]), (i / kPStages) & 1);
        uint4 w[2][2];   // the decode kernel's A fragments: [row r0, r0 + 8][half of the 128 block], bytes 16 c .. 16 c + 15
#pragma unroll
        for (int rr = 0; rr < 2; rr++)
#pragma unroll
            for (int h = 0; h < 2; h++) {
                const int r = r0 + 8 * rr;
                w[rr][h] = *reinterpret_cast<const uint4*>(smem + s * kPA + r * 128 + ((((4 * h + c) ^ (r & 7))) << 4));
            }
        uint32_t a[2][4][4];
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int st = 0; st < 4; st++) {
                const uint32_t w0 = st == 0 ? w[0][h].x : st == 1 ? w[0][h].y : st == 2 ? w[0][h].z : w[0][h].w;
                const uint32_t w1 = st == 0 ? w[1][h].x : st == 1 ? w[1][h].y : st == 2 ? w[1][h].z : w[1][h].w;
                a[h][st][0] = fp8x2_to_f16x2(w0 & 0xffffu); a[h][st][1] = fp8x2_to_f16x2(w1 & 0xffffu);
                a[h][st][2] = fp8x2_to_f16x2(w0 >> 16); a[h][st][3] = fp8x2_to_f16x2(w1 >> 16);
            }
        fence();
        const uint32_t bb = base + kPOffB + s * kPB;
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int st = 0; st < 4; st++)
                mma_f16_rs_m64n128(d, a[h][st], smem_desc(bb + h * (kPT * 128) + st * 32, 16, 1024, kLayoutSw128), (h | st) != 0);
        commit();
        wait<0>();
        fence_regs(d);
        const float* as = reinterpret_cast<const float*>(smem + kPOffS + s * kPS);
#pragma unroll
        for (int j = 0; j < 16; j++) {
            const float2 sc = *reinterpret_cast<const float2*>(as + 8 * j + 2 * c);
#pragma unroll
            for (int e = 0; e < 4; e++)   // (dot * a_s) * b_s, then +=
                acc[4 * j + e] = __fadd_rn(acc[4 * j + e], __fmul_rn(__fmul_rn(d[4 * j + e], (e & 1) ? sc.y : sc.x), bs));
        }
        // the stage is free once the MMAs that read it have completed and its scales are in registers
        __syncwarp();
        if (lane == 0) bar_arrive(smem_u32(&misc.free_[s]));
    }
#pragma unroll
    for (int j = 0; j < 16; j++)
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const int t = tt * kPT + 8 * j + 2 * c + (e & 1), n = rt * 128 + r0 + 8 * (e >> 1);
            if (t < live && n < p.N) store_hidden(p.y, (long)t * p.N + n, p.hidden_type, acc[4 * j + e]);
        }
}

typedef CUresult (*EncodeTiledFn8)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn8 encode_tiled8() {
    static EncodeTiledFn8 fn = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) f = nullptr;
        return (EncodeTiledFn8)f;
    }();
    return fn;
}

// The route: prompt-sized batches go through fp8_gemm_kernel, everything shorter through the decode passes.  Up to 128 tokens
// the GEMM costs one token tile whatever the count, so the crossover is where the decode route's passes (one per 16 tokens)
// overtake it.  Measured at DeepSeek-V3's module shapes with tools/fp8_prefill_probe.py (DESIGN.md §4.6):
//   N <= 2048   (16 row tiles or fewer: few CTAs per token tile)   from 96 tokens (64 is faster on the decode route)
//   K >= 16384  (128 or more K blocks per CTA)                       from 48 tokens (32 is faster on the decode route)
//   otherwise                                                       from 32 tokens, the floor: calls shorter than two decode
//                                                                   passes always take the decode route
static int fp8_prompt_min(int N, int K) { return N <= 2048 ? 96 : K >= 16384 ? 48 : 32; }
static bool fp8_prompt_route(int qlen, int N, int K) { return qlen >= fp8_prompt_min(N, K); }

// One grow-only arena per device, shared by every handle (calls on one device are stream-ordered by the caller):
// [kPChunk or fewer tokens][K] fp16 activations, then [K / 128][pitch] fp32 scales.
struct Fp8Scratch {
    size_t cap = 0;
    void* buf = nullptr;
};
static Fp8Scratch g_fp8[64];

static int fp8_ensure(int dev, int N, int K, size_t need, cudaStream_t s) {
    Fp8Scratch& a = g_fp8[dev & 63];
    if (a.cap >= need) return KTB200_OK;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    KTB_CUDA_CHECK(cudaStreamIsCapturing(s, &cs));
    if (cs != cudaStreamCaptureStatusNone) {
        set_error("fp8_linear: this prompt call needs %zu bytes of prompt scratch on device %d, which holds %zu; the arena cannot grow "
                  "while the stream is capturing: run one eager call of %d or more tokens at in_features >= %d on this device before capture",
                  need, dev, a.cap, fp8_prompt_min(N, K), K);
        return KTB200_ESTATE;
    }
    // grow to a whole chunk at this K, so that one warm-up call of any prompt length covers every later length
    const size_t full = (size_t)kPChunk * K * 2 + (size_t)(K / 128) * kPChunk * sizeof(float);
    KTB_CUDA_CHECK(cudaDeviceSynchronize());   // earlier calls may still be using the arena
    cudaFree(a.buf);
    a = Fp8Scratch();
    KTB_CUDA_CHECK(cudaMalloc(&a.buf, full > need ? full : need));
    a.cap = full > need ? full : need;
    return KTB200_OK;
}
}  // namespace ktb

struct ktb200_fp8_linear {
    int K, N, hidden_type, device, nkb, row_tiles, ksplit, kb_per_split;
    const void* w;
    const float* scale_inv;
    CUtensorMap map;
    float* ws;
    unsigned* tickets;
    uint8_t* xq;   // [kFT][K] e4m3
    float* xs;     // [kFT][nkb]
};

namespace ktb {
// qlen tokens in balanced chunks of whole token tiles (at most kPChunk): per chunk one quantiser launch and one GEMM launch
static int fp8_forward_prompt(ktb200_fp8_linear* l, int qlen, const void* x, void* y, const int* bsz, cudaStream_t s) {
    const int nch = (qlen + kPChunk - 1) / kPChunk;
    const int Tc = ((qlen + nch - 1) / nch + kPT - 1) / kPT * kPT;
    const size_t xh_bytes = (size_t)Tc * l->K * 2, need = xh_bytes + (size_t)l->nkb * Tc * sizeof(float);
    int rc = fp8_ensure(l->device, l->N, l->K, need, s);
    if (rc) return rc;
    EncodeTiledFn8 enc = encode_tiled8();
    uint16_t* xh = reinterpret_cast<uint16_t*>(g_fp8[l->device & 63].buf);
    float* xs = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(xh) + xh_bytes);
    const size_t hb = type_size(l->hidden_type);
    for (int t0 = 0; t0 < qlen; t0 += Tc) {
        const int T = qlen - t0 < Tc ? qlen - t0 : Tc;
        // rows T .. of a token tile and rows N .. of a weight tile are filled with zeros by TMA; no output of theirs is stored
        CUtensorMap xmap, smap;
        const cuuint64_t xdim[2] = {(cuuint64_t)l->K, (cuuint64_t)T}, xstr[1] = {(cuuint64_t)l->K * 2};
        const cuuint64_t sdim[2] = {(cuuint64_t)T, (cuuint64_t)l->nkb}, sstr[1] = {(cuuint64_t)Tc * sizeof(float)};
        const cuuint32_t xbox[2] = {64, kPT}, sbox[2] = {kPT, 1}, estr[2] = {1, 1};
        CUresult cr = enc(&xmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, xh, xdim, xstr, xbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (cr == CUDA_SUCCESS)
            cr = enc(&smap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, xs, sdim, sstr, sbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                     CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (cr != CUDA_SUCCESS) { set_error("fp8_linear: cuTensorMapEncodeTiled failed for the prompt scratch (%d)", (int)cr); return KTB200_ECUDA; }
        Fp8GemmParams p{};
        p.y = reinterpret_cast<uint8_t*>(y) + (size_t)t0 * l->N * hb;
        p.scale_inv = l->scale_inv; p.bsz = bsz; p.t0 = t0;
        p.hidden_type = l->hidden_type; p.T = T; p.N = l->N; p.nkb = l->nkb;
        p.row_tiles = l->row_tiles; p.token_tiles = (T + kPT - 1) / kPT;
        fp8_gemm_quant_kernel<<<(T * l->nkb + 7) / 8, 256, 0, s>>>(reinterpret_cast<const uint8_t*>(x) + (size_t)t0 * l->K * hb, l->hidden_type, T, l->K, Tc,
                                                                   xh, xs);
        KTB_CUDA_CHECK(launch_pdl(fp8_gemm_kernel, dim3(p.row_tiles * p.token_tiles), dim3(kPThreads), (size_t)kPSmem, s, l->map, xmap, smap, p));
        count_launch(2);
    }
    return KTB200_OK;
}
}  // namespace ktb

extern "C" {

int ktb200_fp8_linear_create(int in_features, int out_features, const void* weight_e4m3, const float* weight_scale_inv, int hidden_type, int device,
                             ktb200_fp8_linear** out) {
    using namespace ktb;
    if (!out || !weight_e4m3 || !weight_scale_inv) { set_error("fp8_linear: null argument"); return KTB200_EINVAL; }
    if (in_features <= 0 || out_features <= 0 || in_features % 128) { set_error("fp8_linear: in_features %d must be a positive multiple of 128 (act_quant block)", in_features); return KTB200_EINVAL; }
    if (!is_hidden_type(hidden_type)) { set_error("fp8_linear: bad hidden_type %d", hidden_type); return KTB200_EINVAL; }
    if ((uintptr_t)weight_e4m3 & 15) { set_error("fp8_linear: weight must be 16-byte aligned"); return KTB200_EINVAL; }
    DeviceGuard g(device);
    if (!g.ok) { set_error("cudaSetDevice(%d) failed", device); return KTB200_ECUDA; }
    EncodeTiledFn8 enc = encode_tiled8();
    if (!enc) { set_error("fp8_linear: cuTensorMapEncodeTiled is not available from this driver"); return KTB200_ECUDA; }
    ktb200_fp8_linear* l = new (std::nothrow) ktb200_fp8_linear();
    if (!l) return KTB200_ENOMEM;
    l->K = in_features; l->N = out_features; l->hidden_type = hidden_type; l->device = device; l->w = weight_e4m3; l->scale_inv = weight_scale_inv;
    l->nkb = in_features / 128; l->row_tiles = (out_features + 127) / 128;
    // K splits: at most kFMaxKb blocks of B per CTA, and enough CTAs for two resident waves (2 per SM) when the row tiles are few
    int ks = (4 * num_sms(device) + l->row_tiles - 1) / l->row_tiles;
    const int ks_min = (l->nkb + kFMaxKb - 1) / kFMaxKb;
    if (ks < ks_min) ks = ks_min;
    if (ks > l->nkb) ks = l->nkb;
    l->kb_per_split = (l->nkb + ks - 1) / ks;
    if (l->kb_per_split < 4 && l->nkb >= 4) l->kb_per_split = 4;   // a CTA should at least fill its ring
    l->ksplit = (l->nkb + l->kb_per_split - 1) / l->kb_per_split;
    const cuuint64_t gdim[2] = {(cuuint64_t)in_features, (cuuint64_t)out_features};
    const cuuint64_t gstr[1] = {(cuuint64_t)in_features};
    const cuuint32_t box[2] = {128, 128}, estr[2] = {1, 1};
    const CUresult cr = enc(&l->map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(weight_e4m3), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { set_error("fp8_linear: cuTensorMapEncodeTiled failed (%d)", (int)cr); delete l; return KTB200_ECUDA; }
    l->ws = nullptr; l->tickets = nullptr; l->xq = nullptr; l->xs = nullptr;
    cudaError_t e = cudaMalloc(&l->ws, (size_t)kFT * out_features * sizeof(float));
    if (e == cudaSuccess) e = cudaMemset(l->ws, 0, (size_t)kFT * out_features * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&l->tickets, (size_t)l->row_tiles * sizeof(unsigned));
    if (e == cudaSuccess) e = cudaMemset(l->tickets, 0, (size_t)l->row_tiles * sizeof(unsigned));
    if (e == cudaSuccess) e = cudaMalloc(&l->xq, (size_t)kFT * in_features);
    if (e == cudaSuccess) e = cudaMalloc(&l->xs, (size_t)kFT * l->nkb * sizeof(float));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(fp8_linear_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kFSmem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(fp8_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPSmem);
    if (e != cudaSuccess) { set_error("fp8_linear: %s", cudaGetErrorString(e)); cudaFree(l->ws); cudaFree(l->tickets); cudaFree(l->xq); cudaFree(l->xs); delete l; return KTB200_ENOMEM; }
    *out = l;
    return KTB200_OK;
}

void ktb200_fp8_linear_destroy(ktb200_fp8_linear* l) {
    if (!l) return;
    DeviceGuard g(l->device);
    cudaFree(l->ws); cudaFree(l->tickets); cudaFree(l->xq); cudaFree(l->xs);
    delete l;
}

int ktb200_fp8_linear_forward(ktb200_fp8_linear* l, int qlen, const void* x, void* y, const int* bsz, void* stream) {
    using namespace ktb;
    if (!l || !x || !y) { set_error("fp8_linear: null pointer"); return KTB200_EINVAL; }
    if (qlen <= 0) return KTB200_OK;
    DeviceGuard g(l->device);
    if (fp8_prompt_route(qlen, l->N, l->K)) return fp8_forward_prompt(l, qlen, x, y, bsz, (cudaStream_t)stream);
    const size_t hb = type_size(l->hidden_type);
    for (int t0 = 0; t0 < qlen; t0 += kFT) {   // decode-sized passes: each re-streams the weights
        Fp8Params p{};
        p.x = reinterpret_cast<const uint8_t*>(x) + (size_t)t0 * l->K * hb;
        p.y = reinterpret_cast<uint8_t*>(y) + (size_t)t0 * l->N * hb;
        p.scale_inv = l->scale_inv; p.ws = l->ws; p.tickets = l->tickets; p.bsz = bsz; p.t0 = t0;
        p.hidden_type = l->hidden_type; p.T = qlen - t0 < kFT ? qlen - t0 : kFT; p.K = l->K; p.N = l->N; p.nkb = l->nkb;
        p.kb_per_split = l->kb_per_split; p.ksplit = l->ksplit;
        if (p.T > 2) {   // quantise once, then the GEMM as a programmatic dependent launch: its weight boxes stream while the quantiser drains
            p.xq = l->xq; p.xs = l->xs;
            fp8_act_quant_kernel<<<(p.T * l->nkb + 7) / 8, 256, 0, (cudaStream_t)stream>>>(p.x, l->hidden_type, p.T, l->K, l->xq, l->xs);
            KTB_CUDA_CHECK(launch_pdl(fp8_linear_kernel, dim3(l->row_tiles, l->ksplit), dim3(kFThreads), (size_t)kFSmem, (cudaStream_t)stream, l->map, p));
            count_launch(2);
        } else {
            KTB_CUDA_CHECK(launch_pdl(fp8_linear_kernel, dim3(l->row_tiles, l->ksplit), dim3(kFThreads), (size_t)kFSmem, (cudaStream_t)stream, l->map, p));
            count_launch(1);
        }
    }
    return KTB200_OK;
}

}  // extern "C"
