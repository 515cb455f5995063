// Absorbed-MLA paged decode attention on the Hopper tensor path (wgmma + TMA) and the paged latent KV write.
//
// Replaces MLAWrapper.run / flashinfer BatchMLAPagedAttentionWrapper
// (archive/ktransformers/operators/flashinfer_wrapper.py:117-161, attention.py:419-447) and the Triton split-KV decode
// (archive/ktransformers/operators/triton_attention.py:16-385).  Math (attention.py:395-478, SURVEY Appendix A):
//     s[h,t] = (q_nope[h,:] . ckv[t,:] + q_pe[h,:] . k_pe[t,:]) * sm_scale        576-long dot, bf16 x bf16 -> fp32
//     p      = softmax_t(s)   fp32, online; P is cast to bf16 before P.V            (triton_attention.py:137-141)
//     out[h] = sum_t p[h,t] * ckv[t,:]                                             512 wide
//
// Work decomposition: CTA = (KV split, group of 64 heads, sequence); 3 warpgroups
//     warp 8      TMA producer (the rest of its warpgroup only hands its registers to the other two): paged KV tiles of 32 tokens x 576 columns, 9 boxes of [32 rows x 64 columns] per tile
//                 (cp.async.bulk.tensor, 128-byte swizzle) into a 4-stage ring, one mbarrier per stage
//     warps 0..7  two warpgroups; warpgroup g owns latent columns [256 g, 256 g + 256) of the output.  Each computes
//                 S = Q.K^T (64 heads x 32 tokens, wgmma from shared memory), the online softmax in registers, and
//                 O[:, 256 g ..] += P.V with P straight from registers (the accumulator layout of S is the A-fragment
//                 layout of P.V) and V read MN-major from the same tile (the swizzle is a function of the address only).
// Both warpgroups compute the same S: the alternative, one S shared through shared memory, costs a CTA-wide hand-off per
// tile, while the second S is 36 small MMAs on a tile whose load dominates the time.  The O accumulator (64 x 256 fp32 per
// warpgroup) stays in registers for the whole split.
//
// mla_chunk_tc_kernel is the same CTA for prompt chunks (ktb200_mla_decode_chunk): one query token per CTA, its own causal
// key limit, the tokens of one KV split adjacent in the grid so that they read each tile from L2 (see mla_attend).
//
// mla_ragged_tc_kernel is the same CTA for a ragged batch (ktb200_mla_decode_ragged): sequences with their own query counts
// and lengths in one launch.  Each CTA takes its (query row, head group, tile range, key limit, partial slot) from a work
// list the host planned (ktb200_mla_ragged_plan); mla_ragged_merge_kernel merges each row's own range of slots.
//
// Online softmax with a LAZY reference maximum: p = 2^(x - m_ref), m_ref is only raised (and the head's O row rescaled)
// when the head's running maximum exceeds it by more than 8 — p stays <= 256, exact in bf16/fp32 terms.  Split-KV
// partials (fp32 O, base-2 LSE) are merged by mla_merge_kernel.
#include <cuda_bf16.h>

#include <vector>

#include "common.cuh"
#include "wgmma.cuh"

namespace ktb {

using namespace wg;

constexpr int kDK = 576;             // 512 latent + 64 rope
constexpr int kDV = 512;
constexpr int kHG = 64;              // heads per CTA (wgmma M)
constexpr int kLT = 32;              // kv tokens per tile (N of S, K of P.V)
constexpr int kStages = 4;
constexpr int kMaxSplits = 128;      // mla_merge_kernel: one thread (and one ws[] slot) per split
constexpr int kChunks = kDK / 64;    // 9 column chunks of 64 bf16 = 128 B (one swizzle row)
constexpr int kMlaConsumerWarps = 8, kMlaThreads = kMlaConsumerWarps * 32 + 128;
constexpr int kStageBytes = kLT * kDK * 2;         // 36,864 = 9 regions of 32 rows x 128 B
constexpr int kKRegion = kLT * 128;                // 4,096
constexpr int kQRegion = kHG * 128;                // 8,192
constexpr int kQBytes = kHG * kDK * 2;             // 73,728
constexpr int kOffQ = kStages * kStageBytes;       // 147,456
constexpr int kOffMisc = kOffQ + kQBytes;          // 221,184
constexpr float kRescaleThreshold = 8.f;

struct MlaMisc {
    unsigned long long k_full[kStages], k_empty[kStages];
};
constexpr int kMlaSmem = kOffMisc + (int)sizeof(MlaMisc) + 1024;   // + slack to align the base to 1024 B
static_assert(kMlaSmem <= 232448, "shared memory budget");

struct MlaKParams {
    const __nv_bfloat16* q_nope;   // [B][Hq][512]
    const __nv_bfloat16* q_pe;     // [B][Hq][64]
    const int* page_table;         // [B][max_pages]
    const int* kv_len;             // [B]
    int num_heads, page_size, max_pages, num_splits;
    float scale_log2;              // sm_scale * log2(e)
    float* o_part;                 // [B][splits][Hq][512]
    float* lse_part;               // [B][splits][Hq]  (base-2)
    float* debug;                  // optional: S of the first tile [64][32], see ktb200_debug_mla
    int q_len;                     // mla_chunk_tc_kernel: queries per sequence (q_nope [B][q_len][Hq][512], o_part / lse_part per row)
    const int* plan;               // mla_ragged_tc_kernel: the device work list (kPlanHeader, items, row offsets)
    int max_items, rows;           // mla_ragged_tc_kernel: the plan's item capacity; query rows of q_nope
};

// The ragged work list (ktb200_mla_ragged_plan): int32 header {items, rows, slots, item capacity, row capacity, 0, 0, 0},
// then `item capacity` items of kItemInts {query row, sequence, head group, first tile, end tile, key limit, slot, 0},
// then row_off[row capacity + 1]: the partial slots of row r are [row_off[r], row_off[r + 1]).
constexpr int kPlanHeader = 8, kItemInts = 8;
enum MlaMode { kMlaDecode, kMlaChunk, kMlaRagged };

__device__ __forceinline__ float ex2(float x) {   // 2^x, one MUFU (x = -inf -> 0)
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&v);
}

// kChunk = false: decode, one query per sequence; CTA = (split, head group, sequence), query row b, keys [0, kv_len).
// kChunk = true: a prompt chunk of q_len queries per sequence; CTA = (head group + token * head groups, split, sequence),
// query row b * q_len + i, keys [0, P + i + 1) with P = kv_len - q_len.  Every token of a sequence splits the keys as its
// last token does, so the CTAs of one split (adjacent in the grid) read the same tiles; a token whose limit ends before a
// split's first tile writes that split's neutral element.  Within a CTA every row has the same limit, so the masking of
// the decode path (S = -inf past the limit, V rows past it zeroed in shared memory) is the causal mask.
// kMlaRagged: CTA x = item x of the host-planned work list; the item names the query row, sequence, head group, tile
// range, key limit and partial slot.  CTAs past the plan's item count (the grid is the item capacity) return at once.
template <int kMode>
__device__ __forceinline__ void mla_attend(const CUtensorMap& kv_map, const MlaKParams& p) {
    constexpr bool kChunk = kMode == kMlaChunk;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;           // 128-byte swizzle atoms are 1024-byte aligned
    uint8_t* smem = smem_raw + (base - raw);
    MlaMisc& misc = *reinterpret_cast<MlaMisc*>(smem + kOffMisc);
    int split = 0, hg = 0, tok = 0;
    int b = blockIdx.z;
    if constexpr (kChunk) {
        const int head_groups = (p.num_heads + kHG - 1) / kHG;
        tok = blockIdx.x / head_groups;
        hg = blockIdx.x - tok * head_groups;
        split = blockIdx.y;
    } else if constexpr (kMode == kMlaDecode) {
        split = blockIdx.x;
        hg = blockIdx.y;
    }
    int qrow = kChunk ? b * p.q_len + tok : b;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    int h0 = hg * kHG;
    griddep_launch_dependents();
    griddep_wait();          // q, the newest cache row and kv_len come from the kernels before this one
    int L, tile0, tile1;
    long slot;
    if constexpr (kMode == kMlaRagged) {
        // a plan made for another item capacity reads as empty (its row offsets sit elsewhere); rows past q_nope are skipped
        if ((int)blockIdx.x >= p.plan[0] || p.plan[3] != p.max_items) return;
        const int4* it = reinterpret_cast<const int4*>(p.plan + kPlanHeader + (long)kItemInts * blockIdx.x);
        const int4 u = __ldg(it), v = __ldg(it + 1);
        if (u.x >= p.rows) return;
        qrow = u.x; b = u.y; hg = u.z; tile0 = u.w; tile1 = v.x; L = v.y; slot = v.z;
        h0 = hg * kHG;
    } else {
        L = p.kv_len[b];
        int Lsplit;
        if constexpr (kChunk) {
            // kv_len < q_len cannot be refused on the host (kv_len is device data): the sequence's rows are empty (zeros)
            Lsplit = L < p.q_len ? 0 : L;
            L = L < p.q_len ? 0 : L - p.q_len + tok + 1;
            Lsplit = min(Lsplit, p.max_pages * p.page_size);
            L = min(L, p.max_pages * p.page_size);
        } else {
            if (L > p.max_pages * p.page_size) L = p.max_pages * p.page_size;
            Lsplit = L;
        }
        const int ntiles = (Lsplit + kLT - 1) / kLT;
        const int tiles_per = (ntiles + p.num_splits - 1) / p.num_splits;
        tile0 = split * tiles_per;
        tile1 = min(kChunk ? (L + kLT - 1) / kLT : ntiles, tile0 + tiles_per);
        slot = (long)qrow * p.num_splits + split;
    }
    const int n = tile1 - tile0;
    float* o_out = p.o_part + (slot * p.num_heads + h0) * kDV;
    float* lse_out = p.lse_part + slot * p.num_heads + h0;

    if (n <= 0) {   // empty split: the neutral element of the merge
        for (int i = tid; i < kHG * kDV; i += kMlaThreads)
            if (h0 + i / kDV < p.num_heads) o_out[i] = 0.f;
        if (tid < kHG && h0 + tid < p.num_heads) lse_out[tid] = -INFINITY;
        return;
    }

    // ---- one-time setup -----------------------------------------------------------------------------------------
    auto issue_tile = [&](int j, int s) {
        const int t_base = (tile0 + j) * kLT;
        const int page = p.page_table[(long)b * p.max_pages + t_base / p.page_size];
        const int row = page * p.page_size + t_base % p.page_size;
        const uint32_t bar = smem_u32(&misc.k_full[s]);
        bar_expect_tx(bar, kStageBytes);
#pragma unroll
        for (int c = 0; c < kChunks; c++) tma_load_2d(base + s * kStageBytes + c * kKRegion, &kv_map, bar, c * 64, row);
    };
    if (warp == kMlaConsumerWarps && lane == 0) {
        tma_prefetch_desc(&kv_map);
        for (int s = 0; s < kStages; s++) { bar_init(smem_u32(&misc.k_full[s]), 1); bar_init(smem_u32(&misc.k_empty[s]), kMlaConsumerWarps); }
        bar_fence_init();
        // the first tiles do not depend on anything set up below: request them now
        for (int j = 0; j < n && j < kStages; j++) issue_tile(j, j);
    }
    // Q (64 heads x 576) -> shared memory in the K-major 128-byte-swizzle layout: chunk region c (64 columns) holds 64
    // rows of 128 B; the 16-byte piece j of row r sits at piece (j ^ (r & 7)).  Rows beyond num_heads are zero.
    {
        constexpr int kPieces = kHG * (kDK / 8), kIter = kPieces / kMlaThreads;   // 4608 = 12 x 384
        static_assert(kPieces % kMlaThreads == 0, "Q pieces");
        constexpr int kB = 6;
        static_assert(kIter % kB == 0, "Q batches");
#pragma unroll
        for (int i0 = 0; i0 < kIter; i0 += kB) {
            uint4 v[kB];
#pragma unroll
            for (int u = 0; u < kB; u++) {   // 6 independent 16-byte loads in flight per thread
                const int i = tid + (i0 + u) * kMlaThreads, r = i / (kDK / 8), j = i - r * (kDK / 8);
                v[u] = make_uint4(0, 0, 0, 0);
                if (h0 + r < p.num_heads) {
                    const long hrow = (long)qrow * p.num_heads + h0 + r;
                    v[u] = j < 64 ? __ldg(reinterpret_cast<const uint4*>(p.q_nope + hrow * kDV) + j) : __ldg(reinterpret_cast<const uint4*>(p.q_pe + hrow * 64) + (j - 64));
                }
            }
#pragma unroll
            for (int u = 0; u < kB; u++) {
                const int i = tid + (i0 + u) * kMlaThreads, r = i / (kDK / 8), j = i - r * (kDK / 8);
                const int c = j >> 3, jj = j & 7;
                *reinterpret_cast<uint4*>(smem + kOffQ + c * kQRegion + r * 128 + ((jj ^ (r & 7)) << 4)) = v[u];
            }
        }
    }
    fence_async_smem();
    __syncthreads();

    if (warp >= kMlaConsumerWarps) {
        // ================================================================ TMA producer
        regs_dec<40>();
        if (warp == kMlaConsumerWarps && lane == 0) {
            for (int j = kStages; j < n; j++) {
                const int s = j % kStages;
                bar_wait(smem_u32(&misc.k_empty[s]), ((j / kStages) & 1) ^ 1);
                issue_tile(j, s);
            }
        }
        return;
    }
    // ==================================================================== the two warpgroups
    regs_inc<232>();   // 128 x 40 + 256 x 232 <= 64 K registers
    // thread = rows (heads) ra = 16 (warp % 4) + lane / 4 and ra + 8; accumulator register 4 jb + 2 h + e holds row ra + 8 h,
    // column 8 jb + 2 (lane % 4) + e
    const int g = warp >> 2, wt = tid & 127, ra = 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
    const uint32_t qb = base + kOffQ;
    float o[128];
#pragma unroll
    for (int i = 0; i < 128; i++) o[i] = 0.f;
    float m_ref[2] = {-INFINITY, -INFINITY}, m_run[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // l: this thread's share of the row sum
    for (int j = 0; j < n; j++) {
        const int s = j % kStages;
        const uint32_t kb = base + s * kStageBytes;
        bar_wait(smem_u32(&misc.k_full[s]), (j / kStages) & 1);
        float sv[16];
        fence();
#pragma unroll
        for (int c = 0; c < kChunks; c++)
#pragma unroll
            for (int k = 0; k < 4; k++)
                mma_bf16_m64n32(sv, smem_desc(qb + c * kQRegion + k * 32, 16, 1024, kLayoutSw128), smem_desc(kb + c * kKRegion + k * 32, 16, 1024, kLayoutSw128),
                                (c | k) != 0);
        commit();
        wait<0>();
        fence_regs(sv);
        if (p.debug && j == 0 && g == 0 && split == 0 && hg == 0 && b == 0)
#pragma unroll
            for (int i = 0; i < 16; i++) p.debug[(ra + 8 * ((i >> 1) & 1)) * kLT + 8 * (i >> 2) + cq + (i & 1)] = sv[i];
        const int t_base = (tile0 + j) * kLT;
        float x[16], mt[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 16; i++) {
            x[i] = (t_base + 8 * (i >> 2) + cq + (i & 1) < L) ? sv[i] * p.scale_log2 : -INFINITY;
            mt[(i >> 1) & 1] = fmaxf(mt[(i >> 1) & 1], x[i]);
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
            mt[h] = fmaxf(mt[h], __shfl_xor_sync(0xffffffffu, mt[h], 1));
            mt[h] = fmaxf(mt[h], __shfl_xor_sync(0xffffffffu, mt[h], 2));
            m_run[h] = fmaxf(m_run[h], mt[h]);
            // raise the reference maximum of this head? (never on the first tile: O is still zero)
            if (j == 0) m_ref[h] = m_run[h];
            else if (m_run[h] - m_ref[h] > kRescaleThreshold) {
                const float a = ex2(m_ref[h] - m_run[h]);
                l[h] *= a;
                m_ref[h] = m_run[h];
#pragma unroll
                for (int jb = 0; jb < 32; jb++) { o[4 * jb + 2 * h] *= a; o[4 * jb + 2 * h + 1] *= a; }
            }
        }
        // P in bf16 as the A fragments of the two K = 16 steps: a[kk][i] = (p[8 kk + 2 i], p[8 kk + 2 i + 1])
        uint32_t pa[2][4];
#pragma unroll
        for (int i = 0; i < 16; i += 2) {
            const int h = (i >> 1) & 1;
            const float p0 = ex2(x[i] - m_ref[h]), p1 = ex2(x[i + 1] - m_ref[h]);
            l[h] += p0 + p1;
            pa[i >> 3][(i >> 1) & 3] = pack_bf16(p0, p1);
        }
        // rows of the tile beyond kv_len hold whatever the page contains: P is 0 there, but 0 * NaN is NaN -> zero the V rows
        // of this warpgroup's latent half (the other half is only read by the other warpgroup, S never uses these rows)
        if (t_base + kLT > L) {
            const int valid = L - t_base;
            uint8_t* kt = smem + s * kStageBytes + 4 * g * kKRegion;
            for (int i = wt; i < (kLT - valid) * 32; i += 128) {      // 32 pieces of 16 B per row over the 4 latent chunks
                const int r = valid + i / 32, pc = i % 32;
                *reinterpret_cast<uint4*>(kt + (pc >> 3) * kKRegion + r * 128 + (pc & 7) * 16) = make_uint4(0, 0, 0, 0);
            }
            fence_async_smem();
            asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
        }
        fence();
#pragma unroll
        for (int kk = 0; kk < 2; kk++)
            mma_bf16_rs_m64n256_bt(o, pa[kk], smem_desc(kb + 4 * g * kKRegion + kk * 2048, kKRegion, 1024, kLayoutSw128), 1);
        commit();
        wait<0>();
        fence_regs(o);
        __syncwarp();
        if (lane == 0) bar_arrive(smem_u32(&misc.k_empty[s]));
    }
    // ---- epilogue: O / l -> fp32 partial output, base-2 LSE ---------------------------------------------------------
#pragma unroll
    for (int h = 0; h < 2; h++) {
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
        l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
        const int r = ra + 8 * h;
        if (h0 + r >= p.num_heads) continue;
        if (g == 0 && (lane & 3) == 0) lse_out[r] = m_ref[h] + log2f(l[h]);
        const float inv = 1.f / l[h];
        float* dst = o_out + (long)r * kDV + 256 * g + cq;
#pragma unroll
        for (int jb = 0; jb < 32; jb++) *reinterpret_cast<float2*>(dst + 8 * jb) = make_float2(o[4 * jb + 2 * h] * inv, o[4 * jb + 2 * h + 1] * inv);
    }
}

__global__ void __launch_bounds__(kMlaThreads, 1) mla_decode_tc_kernel(const __grid_constant__ CUtensorMap kv_map, const MlaKParams p) {
    mla_attend<kMlaDecode>(kv_map, p);
}
__global__ void __launch_bounds__(kMlaThreads, 1) mla_chunk_tc_kernel(const __grid_constant__ CUtensorMap kv_map, const MlaKParams p) {
    mla_attend<kMlaChunk>(kv_map, p);
}
__global__ void __launch_bounds__(kMlaThreads, 1) mla_ragged_tc_kernel(const __grid_constant__ CUtensorMap kv_map, const MlaKParams p) {
    mla_attend<kMlaRagged>(kv_map, p);
}

// out[b][h][:] = sum_s w_s * o_part[b][s][h][:],  w_s = 2^(lse_s - max) / sum ; lse (natural log) optional
// 128 threads (4 warps), one per split: ktb200_mla_decode refuses num_kv_splits > kMaxSplits
// out[b][h][:] = sum_s w_s * o_part[b][s][h][:],  w_s = 2^(lse_s - max) / sum ; lse (natural log) optional
// 128 threads (4 warps), one per split: ktb200_mla_decode refuses num_kv_splits > kMaxSplits
static_assert(kMaxSplits == 128, "mla_merge_kernel reduces over exactly 4 warps");
__global__ void __launch_bounds__(128) mla_merge_kernel(const float* o_part, const float* lse_part, int num_splits, int num_heads,
                                                        __nv_bfloat16* out, float* lse_out) {
    __shared__ float ws[kMaxSplits];
    __shared__ float red[8];
    griddep_launch_dependents();
    griddep_wait();
    const int bh = blockIdx.x, b = bh / num_heads, h = bh % num_heads;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float my = tid < num_splits ? lse_part[((long)b * num_splits + tid) * num_heads + h] : -INFINITY;   // num_splits <= kMaxSplits
    float mx = my;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
    const int c = tid * 4;
    __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(out + ((long)b * num_heads + h) * kDV + c);
    if (mx == -INFINITY) {   // kv_len == 0 (e.g. a padded CUDA-graph batch slot): zeros, lse = -inf
        o2[0] = __floats2bfloat162_rn(0.f, 0.f);
        o2[1] = __floats2bfloat162_rn(0.f, 0.f);
        if (lse_out && tid == 0) lse_out[(long)b * num_heads + h] = -INFINITY;
        return;
    }
    const float e = tid < num_splits ? exp2f(my - mx) : 0.f;
    float den = warp_sum(e);
    if (lane == 0) red[4 + warp] = den;
    __syncthreads();
    den = (red[4] + red[5]) + (red[6] + red[7]);
    ws[tid] = e / den;
    __syncthreads();
    float4 acc = make_float4(0, 0, 0, 0);
    const float* src = o_part + ((long)b * num_splits * num_heads + h) * kDV + c;
    const long sstride = (long)num_heads * kDV;
    for (int s0 = 0; s0 < num_splits; s0 += 8) {
        float4 v[8];
#pragma unroll
        for (int u = 0; u < 8; u++)
            if (s0 + u < num_splits) v[u] = __ldcs(reinterpret_cast<const float4*>(src + (s0 + u) * sstride));
#pragma unroll
        for (int u = 0; u < 8; u++)
            if (s0 + u < num_splits) {
                const float w = ws[s0 + u];
                acc.x += w * v[u].x; acc.y += w * v[u].y; acc.z += w * v[u].z; acc.w += w * v[u].w;
            }
    }
    o2[0] = __floats2bfloat162_rn(acc.x, acc.y);
    o2[1] = __floats2bfloat162_rn(acc.z, acc.w);
    if (lse_out && tid == 0) lse_out[(long)b * num_heads + h] = (mx + log2f(den)) * 0.6931471805599453f;
}

// mla_merge_kernel for a ragged plan: one CTA per (row, head) of the launch's `rows` query rows; row r merges its own slots
// [row_off[r], row_off[r + 1]) of o_part [slot][Hq][512] / lse_part [slot][Hq] with the same lane-per-slot code (lanes
// past the row's count at -inf).  Rows past the plan's row count (padded CUDA-graph rows) write zeros and lse -inf.
// A copy rather than a shared body: sharing it changed mla_merge_kernel's instruction schedule.
__global__ void __launch_bounds__(128) mla_ragged_merge_kernel(const float* o_part, const float* lse_part, const int* plan, int max_items,
                                                               int num_heads, __nv_bfloat16* out, float* lse_out) {
    __shared__ float ws[kMaxSplits];
    __shared__ float red[8];
    griddep_launch_dependents();
    griddep_wait();
    const int r = blockIdx.x / num_heads, h = blockIdx.x % num_heads;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int* row_off = plan + kPlanHeader + (long)kItemInts * max_items;
    const bool planned = plan[3] == max_items && r < plan[1];
    const int slot0 = planned ? row_off[r] : 0, count = planned ? row_off[r + 1] - slot0 : 0;   // count <= kMaxSplits
    const float my = tid < count ? lse_part[((long)slot0 + tid) * num_heads + h] : -INFINITY;
    float mx = my;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) red[warp] = mx;
    __syncthreads();
    mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
    const int c = tid * 4;
    __nv_bfloat162* o2 = reinterpret_cast<__nv_bfloat162*>(out + ((long)r * num_heads + h) * kDV + c);
    if (mx == -INFINITY) {
        o2[0] = __floats2bfloat162_rn(0.f, 0.f);
        o2[1] = __floats2bfloat162_rn(0.f, 0.f);
        if (lse_out && tid == 0) lse_out[(long)r * num_heads + h] = -INFINITY;
        return;
    }
    const float e = tid < count ? exp2f(my - mx) : 0.f;
    float den = warp_sum(e);
    if (lane == 0) red[4 + warp] = den;
    __syncthreads();
    den = (red[4] + red[5]) + (red[6] + red[7]);
    ws[tid] = e / den;
    __syncthreads();
    float4 acc = make_float4(0, 0, 0, 0);
    const float* src = o_part + ((long)slot0 * num_heads + h) * kDV + c;
    const long sstride = (long)num_heads * kDV;
    for (int s0 = 0; s0 < count; s0 += 8) {
        float4 v[8];
#pragma unroll
        for (int u = 0; u < 8; u++)
            if (s0 + u < count) v[u] = __ldcs(reinterpret_cast<const float4*>(src + (s0 + u) * sstride));
#pragma unroll
        for (int u = 0; u < 8; u++)
            if (s0 + u < count) {
                const float w = ws[s0 + u];
                acc.x += w * v[u].x; acc.y += w * v[u].y; acc.z += w * v[u].z; acc.w += w * v[u].w;
            }
    }
    o2[0] = __floats2bfloat162_rn(acc.x, acc.y);
    o2[1] = __floats2bfloat162_rn(acc.z, acc.w);
    if (lse_out && tid == 0) lse_out[(long)r * num_heads + h] = (mx + log2f(den)) * 0.6931471805599453f;
}

// StaticCache.update (archive/ktransformers/models/custom_cache.py:147-200): one CTA per token
__global__ void __launch_bounds__(72) mla_kv_write_kernel(__nv_bfloat16* kv, int page_size, const __nv_bfloat16* ckv,
                                                          const __nv_bfloat16* k_pe, const int* page_idx, const int* page_off) {
    const int t = blockIdx.x, i = threadIdx.x;   // 72 x 16 B = 1152 B
    __nv_bfloat16* dst = kv + ((long)page_idx[t] * page_size + page_off[t]) * kDK;
    const uint4 v = (i < 64) ? reinterpret_cast<const uint4*>(ckv + (long)t * kDV)[i] : reinterpret_cast<const uint4*>(k_pe + (long)t * 64)[i - 64];
    reinterpret_cast<uint4*>(dst)[i] = v;
}

static int pick_splits(int batch, int num_heads, int max_kv_tiles, int device) {
    const int groups = batch * ((num_heads + kHG - 1) / kHG);
    int s = (num_sms(device) + groups - 1) / groups;          // one CTA per SM (227 KB of shared memory each)
    const int cap = (max_kv_tiles + 3) / 4;                   // at least 4 tiles (128 tokens) per split
    if (s > cap) s = cap;
    if (s > kMaxSplits) s = kMaxSplits;
    if (s < 1) s = 1;
    return s;
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (libktb200.so links libcudart only)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled() {
    static EncodeTiledFn fn = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) f = nullptr;
        return (EncodeTiledFn)f;
    }();
    return fn;
}

// the paged cache as a 2-D tensor [token rows][576 columns]; a tile never crosses a page (page_size % 32 == 0)
static int encode_kv_map(CUtensorMap* map, const void* kv_cache, long kv_cache_rows, const char* who) {
    EncodeTiledFn enc = encode_tiled();
    if (!enc) { set_error("%s: cuTensorMapEncodeTiled is not available from this driver", who); return KTB200_ECUDA; }
    const cuuint64_t rows = kv_cache_rows > 0 ? (cuuint64_t)kv_cache_rows : (cuuint64_t)1 << 31;
    const cuuint64_t gdim[2] = {(cuuint64_t)kDK, rows};
    const cuuint64_t gstr[1] = {(cuuint64_t)kDK * 2};
    const cuuint32_t box[2] = {64, (cuuint32_t)kLT};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult cr = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(kv_cache), gdim, gstr, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { set_error("%s: cuTensorMapEncodeTiled failed (%d)", who, (int)cr); return KTB200_ECUDA; }
    return KTB200_OK;
}

static float* g_mla_debug = nullptr;

}  // namespace ktb

extern "C" {

size_t ktb200_mla_workspace_bytes(int batch, int num_heads, int max_splits) {
    if (max_splits <= 0) max_splits = ktb::kMaxSplits;
    return (size_t)batch * max_splits * num_heads * (ktb::kDV + 1) * sizeof(float);
}

int ktb200_mla_decode(const ktb200_mla_params* q, void* stream) {
    using namespace ktb;
    if (!q || !q->q_nope || !q->q_pe || !q->kv_cache || !q->page_table || !q->kv_len || !q->out || !q->workspace) { set_error("mla_decode: null pointer"); return KTB200_EINVAL; }
    if (q->batch <= 0) return KTB200_OK;
    if (q->num_heads <= 0 || q->page_size <= 0 || q->page_size % kLT || q->max_pages_per_seq <= 0) {
        set_error("mla_decode: page_size %d must be a positive multiple of %d", q->page_size, kLT);
        return KTB200_EINVAL;
    }
    if (((uintptr_t)q->kv_cache & 15) || ((uintptr_t)q->q_nope & 15) || ((uintptr_t)q->q_pe & 15)) { set_error("mla_decode: q / kv_cache must be 16-byte aligned"); return KTB200_EINVAL; }
    if (q->num_kv_splits > kMaxSplits) {   // the merge kernel weighs at most kMaxSplits partials
        set_error("mla_decode: num_kv_splits %d exceeds the maximum of %d", q->num_kv_splits, kMaxSplits);
        return KTB200_EINVAL;
    }
    int dev = 0;
    KTB_CUDA_CHECK(cudaGetDevice(&dev));
    const int max_tiles = q->max_pages_per_seq * (q->page_size / kLT);
    int splits = q->num_kv_splits > 0 ? q->num_kv_splits : pick_splits(q->batch, q->num_heads, max_tiles, dev);
    if (splits > max_tiles) splits = max_tiles;
    const size_t need = (size_t)q->batch * splits * q->num_heads * (kDV + 1) * sizeof(float);
    if (need > q->workspace_bytes) { set_error("mla_decode: workspace too small (%zu < %zu bytes for %d splits)", q->workspace_bytes, need, splits); return KTB200_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;

    CUtensorMap map;
    if (const int rc = encode_kv_map(&map, q->kv_cache, q->kv_cache_rows, "mla_decode")) return rc;

    MlaKParams p{};
    p.q_nope = (const __nv_bfloat16*)q->q_nope; p.q_pe = (const __nv_bfloat16*)q->q_pe;
    p.page_table = q->page_table; p.kv_len = q->kv_len; p.num_heads = q->num_heads; p.page_size = q->page_size;
    p.max_pages = q->max_pages_per_seq; p.num_splits = splits; p.scale_log2 = q->sm_scale * 1.4426950408889634f;
    p.o_part = (float*)q->workspace;
    p.lse_part = p.o_part + (size_t)q->batch * splits * q->num_heads * kDV;
    p.debug = g_mla_debug;
    static bool attr_set[64] = {};
    if (!attr_set[dev & 63]) {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(mla_decode_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMlaSmem));
        attr_set[dev & 63] = true;
    }
    const int head_groups = (q->num_heads + kHG - 1) / kHG;
    KTB_CUDA_CHECK(launch_pdl(mla_decode_tc_kernel, dim3(splits, head_groups, q->batch), dim3(kMlaThreads), (size_t)kMlaSmem, s, map, p));
    count_launch();
    KTB_CUDA_CHECK(launch_pdl(mla_merge_kernel, dim3(q->batch * q->num_heads), dim3(128), 0, s, (const float*)p.o_part, (const float*)p.lse_part, splits, q->num_heads,
                              (__nv_bfloat16*)q->out, q->lse_out));
    count_launch();
    return KTB200_OK;
}

size_t ktb200_mla_chunk_workspace_bytes(int batch, int q_len, int num_heads, int max_splits) {
    if (batch <= 0 || q_len <= 0 || num_heads <= 0) return 0;
    if (max_splits <= 0) max_splits = ktb::kMaxSplits;
    return (size_t)batch * q_len * max_splits * num_heads * (ktb::kDV + 1) * sizeof(float);
}

int ktb200_mla_decode_chunk(const ktb200_mla_chunk_params* q, void* stream) {
    using namespace ktb;
    if (!q) { set_error("mla_decode_chunk: null params"); return KTB200_EINVAL; }
    if (!q->q_nope || !q->q_pe || !q->kv_cache || !q->page_table || !q->kv_len || !q->out || !q->workspace) { set_error("mla_decode_chunk: null pointer"); return KTB200_EINVAL; }
    if (q->q_len < 1) { set_error("mla_decode_chunk: q_len %d must be at least 1", q->q_len); return KTB200_EINVAL; }
    if (q->batch <= 0) return KTB200_OK;
    if (q->num_heads <= 0 || q->page_size <= 0 || q->page_size % kLT || q->max_pages_per_seq <= 0) {
        set_error("mla_decode_chunk: page_size %d must be a positive multiple of %d (num_heads %d, max_pages_per_seq %d must be positive)",
                  q->page_size, kLT, q->num_heads, q->max_pages_per_seq);
        return KTB200_EINVAL;
    }
    if (((uintptr_t)q->kv_cache & 15) || ((uintptr_t)q->q_nope & 15) || ((uintptr_t)q->q_pe & 15)) { set_error("mla_decode_chunk: q / kv_cache must be 16-byte aligned"); return KTB200_EINVAL; }
    if (q->num_kv_splits > kMaxSplits) {
        set_error("mla_decode_chunk: num_kv_splits %d exceeds the maximum of %d", q->num_kv_splits, kMaxSplits);
        return KTB200_EINVAL;
    }
    const long rows = (long)q->batch * q->q_len;
    const int head_groups = (q->num_heads + kHG - 1) / kHG;
    if (q->batch > 65535 || rows * q->num_heads > 0x7fffffffL) {   // grid z; merge CTAs and query rows are int
        set_error("mla_decode_chunk: batch %d x q_len %d x num_heads %d is too large", q->batch, q->q_len, q->num_heads);
        return KTB200_EINVAL;
    }
    int dev = 0;
    const int max_tiles = q->max_pages_per_seq * (q->page_size / kLT);
    // automatic splits: as decode with every query row counted as a sequence, planned on the chunk's last row
    int splits = q->num_kv_splits;
    if (splits <= 0) {
        KTB_CUDA_CHECK(cudaGetDevice(&dev));
        splits = pick_splits((int)rows, q->num_heads, max_tiles, dev);
    }
    if (splits > max_tiles) splits = max_tiles;
    const size_t need = (size_t)rows * splits * q->num_heads * (kDV + 1) * sizeof(float);
    if (need > q->workspace_bytes) { set_error("mla_decode_chunk: workspace too small (%zu < %zu bytes for %d splits)", q->workspace_bytes, need, splits); return KTB200_EINVAL; }
    if (q->num_kv_splits > 0) KTB_CUDA_CHECK(cudaGetDevice(&dev));
    CUtensorMap map;
    if (const int rc = encode_kv_map(&map, q->kv_cache, q->kv_cache_rows, "mla_decode_chunk")) return rc;

    MlaKParams p{};
    p.q_nope = (const __nv_bfloat16*)q->q_nope; p.q_pe = (const __nv_bfloat16*)q->q_pe;
    p.page_table = q->page_table; p.kv_len = q->kv_len; p.num_heads = q->num_heads; p.page_size = q->page_size;
    p.max_pages = q->max_pages_per_seq; p.num_splits = splits; p.scale_log2 = q->sm_scale * 1.4426950408889634f;
    p.o_part = (float*)q->workspace;
    p.lse_part = p.o_part + (size_t)rows * splits * q->num_heads * kDV;
    p.q_len = q->q_len;
    static bool attr_set[64] = {};
    if (!attr_set[dev & 63]) {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(mla_chunk_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMlaSmem));
        attr_set[dev & 63] = true;
    }
    cudaStream_t s = (cudaStream_t)stream;
    KTB_CUDA_CHECK(launch_pdl(mla_chunk_tc_kernel, dim3(head_groups * q->q_len, splits, q->batch), dim3(kMlaThreads), (size_t)kMlaSmem, s, map, p));
    count_launch();
    // the merge is decode's over batch * q_len query rows
    KTB_CUDA_CHECK(launch_pdl(mla_merge_kernel, dim3((unsigned)(rows * q->num_heads)), dim3(128), 0, s, (const float*)p.o_part, (const float*)p.lse_part, splits,
                              q->num_heads, (__nv_bfloat16*)q->out, q->lse_out));
    count_launch();
    return KTB200_OK;
}

size_t ktb200_mla_ragged_plan_ints(int max_items, int max_rows) {
    if (max_items <= 0 || max_rows < 0) return 0;
    return (size_t)ktb::kPlanHeader + (size_t)ktb::kItemInts * max_items + (size_t)max_rows + 1;
}

size_t ktb200_mla_ragged_workspace_bytes(int max_items, int num_heads) {
    if (max_items <= 0 || num_heads <= 0) return 0;
    const int head_groups = (num_heads + ktb::kHG - 1) / ktb::kHG;   // every slot has one item per head group
    return (size_t)(max_items / head_groups) * num_heads * (ktb::kDV + 1) * sizeof(float);
}

// Host only.  Token i of sequence b (row qo_indptr[b] + i) attends to keys [0, kv_len[b] - q_len_b + i + 1).  Sequence b's
// tiles [0, tiles(kv_len[b])) are cut once into ranges of tiles_per[b]; a token takes the ranges that start below its limit,
// one slot each (row_off), and one item per (range, head group).  Items are listed sequence by sequence, range by range,
// token by token, so the CTAs that read one range are adjacent in the grid.
int ktb200_mla_ragged_plan(const int* qo_indptr, const int* kv_len, int batch, int num_heads, int page_size, int max_pages_per_seq,
                           int num_sms, int num_kv_splits, int max_items, int max_rows, int* plan, size_t plan_ints, int* n_slots,
                           size_t* workspace_bytes) {
    using namespace ktb;
    if (!qo_indptr || !kv_len || !plan) { set_error("mla_ragged_plan: null pointer"); return KTB200_EINVAL; }
    if (batch < 0 || num_heads <= 0 || page_size <= 0 || page_size % kLT || max_pages_per_seq <= 0 || num_sms <= 0) {
        set_error("mla_ragged_plan: page_size %d must be a positive multiple of %d (batch %d >= 0; num_heads %d, max_pages_per_seq %d, num_sms %d positive)",
                  page_size, kLT, batch, num_heads, max_pages_per_seq, num_sms);
        return KTB200_EINVAL;
    }
    if (num_kv_splits > kMaxSplits) { set_error("mla_ragged_plan: num_kv_splits %d exceeds the maximum of %d", num_kv_splits, kMaxSplits); return KTB200_EINVAL; }
    if (max_items <= 0 || max_rows < 0) { set_error("mla_ragged_plan: item capacity %d must be positive and row capacity %d non-negative", max_items, max_rows); return KTB200_EINVAL; }
    const size_t need_ints = ktb200_mla_ragged_plan_ints(max_items, max_rows);
    if (plan_ints < need_ints) { set_error("mla_ragged_plan: plan buffer too small (%zu < %zu ints)", plan_ints, need_ints); return KTB200_EINVAL; }
    const long cap_len = (long)max_pages_per_seq * page_size;
    if (qo_indptr[0] != 0) { set_error("mla_ragged_plan: qo_indptr[0] = %d, must be 0", qo_indptr[0]); return KTB200_EINVAL; }
    for (int b = 0; b < batch; b++) {
        const int q = qo_indptr[b + 1] - qo_indptr[b];
        if (qo_indptr[b + 1] < qo_indptr[b]) { set_error("mla_ragged_plan: qo_indptr is not monotone at %d (%d > %d)", b, qo_indptr[b], qo_indptr[b + 1]); return KTB200_EINVAL; }
        if (kv_len[b] < q) { set_error("mla_ragged_plan: kv_len[%d] = %d is shorter than its q_len %d", b, kv_len[b], q); return KTB200_EINVAL; }
        if (kv_len[b] > cap_len) { set_error("mla_ragged_plan: kv_len[%d] = %d exceeds max_pages_per_seq * page_size = %ld", b, kv_len[b], cap_len); return KTB200_EINVAL; }
    }
    const int rows = batch ? qo_indptr[batch] : 0;
    if (rows > max_rows) { set_error("mla_ragged_plan: %d query rows exceed the row capacity %d", rows, max_rows); return KTB200_EINVAL; }
    const int head_groups = (num_heads + kHG - 1) / kHG;
    auto tiles = [](long len) { return (len + kLT - 1) / kLT; };
    std::vector<long> tiles_per(batch > 0 ? batch : 1, 1);
    auto count_items = [&]() {   // items of the current tiles_per: sum over tokens of the ranges below the limit
        long n = 0;
        for (int b = 0; b < batch; b++) {
            const int q = qo_indptr[b + 1] - qo_indptr[b];
            for (int i = 0; i < q; i++) n += (tiles(kv_len[b] - q + i + 1) + tiles_per[b] - 1) / tiles_per[b];
        }
        return n * head_groups;
    };
    long items = 0;
    if (num_kv_splits > 0) {   // ktb200_mla_decode_chunk's ranges: its split count (clamped to the page table), on kv_len
        const long max_tiles = cap_len / kLT;
        const long s = num_kv_splits < max_tiles ? num_kv_splits : max_tiles;
        for (int b = 0; b < batch; b++) tiles_per[b] = kv_len[b] > 0 ? (tiles(kv_len[b]) + s - 1) / s : 1;
        items = count_items();
    } else {
        // the largest item is at most max(4 tiles, the (row, head group, tile) work over the SMs), at most kMaxSplits ranges
        // per sequence; when that does not fit the item capacity the bound doubles until it does
        long work = 0;
        for (int b = 0; b < batch; b++) {
            const int q = qo_indptr[b + 1] - qo_indptr[b];
            for (int i = 0; i < q; i++) work += tiles(kv_len[b] - q + i + 1);
        }
        work *= head_groups;
        long bound = (work + num_sms - 1) / num_sms;
        if (bound < 4) bound = 4;
        for (;;) {
            bool one_range = true;
            for (int b = 0; b < batch; b++) {
                const long t = tiles(kv_len[b]);
                long s = (t + bound - 1) / bound;
                if (s > kMaxSplits) s = kMaxSplits;
                if (s < 1) s = 1;
                one_range &= s == 1;
                tiles_per[b] = t > 0 ? (t + s - 1) / s : 1;
            }
            items = count_items();
            if (items <= max_items || one_range) break;
            bound *= 2;
        }
    }
    if (items > max_items) { set_error("mla_ragged_plan: %ld work items exceed the item capacity %d", items, max_items); return KTB200_EINVAL; }
    int* item = plan + kPlanHeader;
    int* row_off = plan + kPlanHeader + (long)kItemInts * max_items;
    int slots = 0;
    for (int b = 0; b < batch; b++) {
        const int q = qo_indptr[b + 1] - qo_indptr[b];
        for (int i = 0; i < q; i++) {
            row_off[qo_indptr[b] + i] = slots;
            slots += (int)((tiles(kv_len[b] - q + i + 1) + tiles_per[b] - 1) / tiles_per[b]);
        }
    }
    row_off[rows] = slots;
    long k = 0;
    for (int b = 0; b < batch; b++) {
        const int q = qo_indptr[b + 1] - qo_indptr[b];
        if (q == 0) continue;
        const int past = kv_len[b] - q;
        const long ranges = (tiles(kv_len[b]) + tiles_per[b] - 1) / tiles_per[b];
        for (long r = 0; r < ranges; r++) {
            const long t0 = r * tiles_per[b];
            // the tokens whose limit past + i + 1 reaches into tile t0: i >= t0 * kLT - past
            for (long i = t0 * kLT - past > 0 ? t0 * kLT - past : 0; i < q; i++) {
                const long limit = past + i + 1, t1 = tiles(limit) < t0 + tiles_per[b] ? tiles(limit) : t0 + tiles_per[b];
                const int row = qo_indptr[b] + (int)i;
                for (int g = 0; g < head_groups; g++, k++) {
                    int* it = item + kItemInts * k;
                    it[0] = row; it[1] = b; it[2] = g; it[3] = (int)t0; it[4] = (int)t1; it[5] = (int)limit; it[6] = row_off[row] + (int)r; it[7] = 0;
                }
            }
        }
    }
    const int header[kPlanHeader] = {(int)items, rows, slots, max_items, max_rows, 0, 0, 0};
    for (int i = 0; i < kPlanHeader; i++) plan[i] = header[i];
    if (n_slots) *n_slots = slots;
    if (workspace_bytes) *workspace_bytes = (size_t)slots * num_heads * (kDV + 1) * sizeof(float);
    return KTB200_OK;
}

int ktb200_mla_decode_ragged(const ktb200_mla_ragged_params* q, void* stream) {
    using namespace ktb;
    if (!q) { set_error("mla_decode_ragged: null params"); return KTB200_EINVAL; }
    if (!q->q_nope || !q->q_pe || !q->kv_cache || !q->page_table || !q->plan || !q->out || !q->workspace) { set_error("mla_decode_ragged: null pointer"); return KTB200_EINVAL; }
    if (q->rows < 0 || q->max_items <= 0) { set_error("mla_decode_ragged: item capacity %d must be positive and rows %d non-negative", q->max_items, q->rows); return KTB200_EINVAL; }
    if (q->num_heads <= 0 || q->page_size <= 0 || q->page_size % kLT || q->max_pages_per_seq <= 0) {
        set_error("mla_decode_ragged: page_size %d must be a positive multiple of %d (num_heads %d, max_pages_per_seq %d must be positive)",
                  q->page_size, kLT, q->num_heads, q->max_pages_per_seq);
        return KTB200_EINVAL;
    }
    if (((uintptr_t)q->kv_cache & 15) || ((uintptr_t)q->q_nope & 15) || ((uintptr_t)q->q_pe & 15) || ((uintptr_t)q->plan & 15)) {
        set_error("mla_decode_ragged: q / kv_cache / plan must be 16-byte aligned");
        return KTB200_EINVAL;
    }
    if ((long)q->rows * q->num_heads > 0x7fffffffL) {   // merge CTAs
        set_error("mla_decode_ragged: rows %d x num_heads %d is too large", q->rows, q->num_heads);
        return KTB200_EINVAL;
    }
    const size_t need = ktb200_mla_ragged_workspace_bytes(q->max_items, q->num_heads);
    if (need > q->workspace_bytes) { set_error("mla_decode_ragged: workspace too small (%zu < %zu bytes for %d items)", q->workspace_bytes, need, q->max_items); return KTB200_EINVAL; }
    if (q->rows == 0) return KTB200_OK;
    int dev = 0;
    KTB_CUDA_CHECK(cudaGetDevice(&dev));
    CUtensorMap map;
    if (const int rc = encode_kv_map(&map, q->kv_cache, q->kv_cache_rows, "mla_decode_ragged")) return rc;

    MlaKParams p{};
    p.q_nope = (const __nv_bfloat16*)q->q_nope; p.q_pe = (const __nv_bfloat16*)q->q_pe;
    p.page_table = q->page_table; p.num_heads = q->num_heads; p.page_size = q->page_size;
    p.max_pages = q->max_pages_per_seq; p.scale_log2 = q->sm_scale * 1.4426950408889634f;
    p.o_part = (float*)q->workspace;
    const long slot_cap = q->max_items / ((q->num_heads + kHG - 1) / kHG);
    p.lse_part = p.o_part + slot_cap * q->num_heads * kDV;   // o_part [slot capacity][Hq][512], then lse_part [slot capacity][Hq]
    p.plan = q->plan; p.max_items = q->max_items; p.rows = q->rows;
    static bool attr_set[64] = {};
    if (!attr_set[dev & 63]) {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(mla_ragged_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMlaSmem));
        attr_set[dev & 63] = true;
    }
    cudaStream_t s = (cudaStream_t)stream;
    KTB_CUDA_CHECK(launch_pdl(mla_ragged_tc_kernel, dim3((unsigned)q->max_items), dim3(kMlaThreads), (size_t)kMlaSmem, s, map, p));
    count_launch();
    KTB_CUDA_CHECK(launch_pdl(mla_ragged_merge_kernel, dim3((unsigned)(q->rows * q->num_heads)), dim3(128), 0, s, (const float*)p.o_part,
                              (const float*)p.lse_part, q->plan, q->max_items, q->num_heads, (__nv_bfloat16*)q->out, q->lse_out));
    count_launch();
    return KTB200_OK;
}

// Diagnostics: while set, CTA (split 0, head group 0, sequence 0) of ktb200_mla_decode writes the raw fp32 scores of its
// first tile (S[64 heads][32 tokens], before scaling) to debug_dev[0..2048).
void ktb200_debug_mla(float* debug_dev) { ktb::g_mla_debug = debug_dev; }

int ktb200_mla_kv_write(void* kv_cache, int page_size, const void* ckv, const void* k_pe, const int* page_idx,
                        const int* page_offset, int n_tokens, void* stream) {
    using namespace ktb;
    if (!kv_cache || !ckv || !k_pe || !page_idx || !page_offset) { set_error("mla_kv_write: null pointer"); return KTB200_EINVAL; }
    // 16-byte row pieces
    if ((uintptr_t)kv_cache & 15) { set_error("mla_kv_write: kv_cache must be 16-byte aligned"); return KTB200_EINVAL; }
    if ((uintptr_t)ckv & 15) { set_error("mla_kv_write: ckv must be 16-byte aligned"); return KTB200_EINVAL; }
    if ((uintptr_t)k_pe & 15) { set_error("mla_kv_write: k_pe must be 16-byte aligned"); return KTB200_EINVAL; }
    if (n_tokens <= 0) return KTB200_OK;
    mla_kv_write_kernel<<<n_tokens, 72, 0, (cudaStream_t)stream>>>((__nv_bfloat16*)kv_cache, page_size, (const __nv_bfloat16*)ckv,
                                                                   (const __nv_bfloat16*)k_pe, page_idx, page_offset);
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

}  // extern "C"
