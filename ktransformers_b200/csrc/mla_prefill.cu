// Causal MLA prefill attention on the Hopper tensor path (wgmma + TMA), over the decompressed heads.
//
// The reference's non-absorbed prefill (archive/ktransformers/operators/attention.py:349-478, q_len > 1): the cached latents
// go through kv_b_proj, then flash_attn_func(q, k, v, softmax_scale, causal=True).  With P tokens already cached and
// S = P + q_len, query i of the chunk (position P + i) and key j <= P + i:
//     s[i,j] = (q_nope[i] . k_nope[j] + q_pe[i] . k_pe[j]) * sm_scale     192-long dot, bf16 x bf16 -> fp32
//     p      = softmax_j(s)   fp32, online, base 2; P rounded to bf16 before P.V (as flash_attn_func)
//     out[i] = sum_j p[i,j] v[j]                                          fp32, one division by the row sum, one bf16 rounding
//
// Work decomposition: CTA = (query tile of 128 rows, head, sequence); 3 warpgroups
//     warp 8      TMA producer (the rest of its warpgroup only hands its registers to the other two).  Q once, as 3 boxes
//                 of [128 rows x 64 columns]; then per key tile of 128 keys K (k_nope 2 boxes, k_pe 1 box) and V (2 boxes)
//                 into a 2-stage ring, 128-byte swizzle, one full / empty mbarrier pair per stage.  Every operand is read in
//                 place through a tensor map {64-column box, head, token, sequence} (k_pe, which all heads share, has no head
//                 dimension).  The token extent of the maps is q_len / S: rows past it arrive as zeros, so whatever follows
//                 the live rows in memory never reaches S or P.V.
//     warps 0..7  two warpgroups of 64 query rows.  Each computes S = Q.K^T (64 x 128, wgmma from shared memory), masks the
//                 keys above the diagonal, runs the online softmax in registers and adds P.V with P straight from registers
//                 (the accumulator layout of S is the A-fragment layout of P.V) and V read MN-major from shared memory.
//                 O (64 x 128 fp32) stays in registers.
// Key tiles entirely above a warpgroup's diagonal are skipped (by the producer when above the CTA's last row).  The CTAs of
// the last query tiles, which see the most keys, are launched first.
#include <cuda_bf16.h>
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "wgmma.cuh"

namespace ktb {

using namespace wg;

namespace prefill {

constexpr int kBM = 128;                     // query rows per CTA (two warpgroups of 64)
constexpr int kBN = 128;                     // keys per tile
constexpr int kStages = 2;
constexpr int kConsumerWarps = 8, kThreads = kConsumerWarps * 32 + 128;
constexpr int kRegion = 128 * 128;           // one box: 128 rows x 64 bf16 columns (128 B), 16 KB
static_assert(kBM == 128 && kBN == 128, "a box is 128 rows of Q, K or V");
constexpr int kOffQ = 0;                     // q_nope 0..63 | q_nope 64..127 | q_pe
constexpr int kStageBytes = 5 * kRegion;     // k_nope 0..63 | k_nope 64..127 | k_pe | v 0..63 | v 64..127
constexpr int kOffStage = kOffQ + 3 * kRegion;
constexpr int kOffMisc = kOffStage + kStages * kStageBytes;
struct Misc {
    unsigned long long q_full, full[kStages], empty[kStages];
};
constexpr int kSmem = kOffMisc + (int)sizeof(Misc) + 1024;   // + slack to align the base to 1024 B
static_assert(kSmem <= 232448, "shared memory budget");

struct KParams {
    int q_len, past, num_heads, num_m_tiles;
    float scale_log2;          // sm_scale * log2(e)
    __nv_bfloat16* out;        // [B][q_len][H][128]
};
constexpr int kMaxSeqs = KTB200_MLA_PREFILL_VARLEN_MAX_BATCH;
struct VParams {               // ktb200_mla_prefill_varlen: the sequences travel in the kernel's parameter block
    int num_heads;
    float scale_log2;
    __nv_bfloat16* out;        // [q_rows][H][128]
    int4 seq[kMaxSeqs];        // {q_row, q_len, k_row, kv_len}
};
static_assert(5 * sizeof(CUtensorMap) + sizeof(VParams) <= 32764, "kernel parameters of sm_90 (CUDA >= 12.1)");

__device__ __forceinline__ float ex2(float x) {   // 2^x, one MUFU (x = -inf -> 0)
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&v);
}

}  // namespace prefill

using namespace prefill;

// One CTA: query tile q0 of head h of one sequence.  Dense: sequence b of the 4-D maps {column, head, token, sequence}, its
// q_len / past from the launch.  Varlen: sequence b's {q_row, q_len, k_row, kv_len} from the parameter block, 3-D maps
// {column, head, row}; the rows past its keys belong to another sequence (or to a gap), so they are not zeros: keys at or
// past kv_len are masked (S -inf) and the V rows past kv_len in the crossing tile are zeroed in shared memory.
template <bool kVarlen, class KP>
__device__ __forceinline__ void prefill_cta(const CUtensorMap* qn_map, const CUtensorMap* qp_map, const CUtensorMap* kn_map, const CUtensorMap* kp_map,
                                            const CUtensorMap* v_map, const KP& p) {
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;           // 128-byte swizzle atoms are 1024-byte aligned
    Misc& misc = *reinterpret_cast<Misc*>(smem_raw + (base - raw) + kOffMisc);
    const int h = blockIdx.x % p.num_heads, b = blockIdx.x / p.num_heads;
    int q_len, past, q0, q_row = 0, k_row = 0, kv_end = 0;
    if constexpr (kVarlen) {
        const int4 s = p.seq[b];
        const int m_tiles = (s.y + kBM - 1) / kBM;
        if ((int)blockIdx.y >= m_tiles) return;            // past this sequence's queries (q_len 0: every tile)
        q_len = s.y; past = s.w - s.y; q_row = s.x; k_row = s.z;
        kv_end = s.w;                                       // keys at or past it are another sequence's
        q0 = (m_tiles - 1 - blockIdx.y) * kBM;              // the sequence's heaviest query tiles first
    } else {
        q_len = p.q_len; past = p.past;
        q0 = (p.num_m_tiles - 1 - blockIdx.y) * kBM;        // the heaviest query tiles first
    }
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = (past + min(q0 + kBM, q_len) + kBN - 1) / kBN;   // key tiles up to the CTA's last row

    if (warp == kConsumerWarps && lane == 0) {
        tma_prefetch_desc(qn_map); tma_prefetch_desc(qp_map); tma_prefetch_desc(kn_map); tma_prefetch_desc(kp_map); tma_prefetch_desc(v_map);
        bar_init(smem_u32(&misc.q_full), 1);
        for (int s = 0; s < kStages; s++) { bar_init(smem_u32(&misc.full[s]), 1); bar_init(smem_u32(&misc.empty[s]), kConsumerWarps); }
        bar_fence_init();
    }
    __syncthreads();

    if (warp >= kConsumerWarps) {
        // ================================================================ TMA producer
        regs_dec<40>();
        if (warp == kConsumerWarps && lane == 0) {
            const uint32_t qbar = smem_u32(&misc.q_full);
            bar_expect_tx(qbar, 3 * kRegion);
            if constexpr (kVarlen) {
                tma_load_3d(base + kOffQ, qn_map, qbar, 0, h, q_row + q0);
                tma_load_3d(base + kOffQ + kRegion, qn_map, qbar, 64, h, q_row + q0);
                tma_load_3d(base + kOffQ + 2 * kRegion, qp_map, qbar, 0, h, q_row + q0);
            } else {
                tma_load_4d(base + kOffQ, qn_map, qbar, 0, h, q0, b);
                tma_load_4d(base + kOffQ + kRegion, qn_map, qbar, 64, h, q0, b);
                tma_load_4d(base + kOffQ + 2 * kRegion, qp_map, qbar, 0, h, q0, b);
            }
            for (int j = 0; j < n; j++) {
                const int s = j % kStages, k0 = j * kBN;
                bar_wait(smem_u32(&misc.empty[s]), ((j / kStages) & 1) ^ 1);
                const uint32_t bar = smem_u32(&misc.full[s]), st = base + kOffStage + s * kStageBytes;
                bar_expect_tx(bar, kStageBytes);   // boxes that cross the token extent still count in full (zero-filled)
                if constexpr (kVarlen) {
                    tma_load_3d(st, kn_map, bar, 0, h, k_row + k0);
                    tma_load_3d(st + kRegion, kn_map, bar, 64, h, k_row + k0);
                    tma_load_2d(st + 2 * kRegion, kp_map, bar, 0, k_row + k0);
                    tma_load_3d(st + 3 * kRegion, v_map, bar, 0, h, k_row + k0);
                    tma_load_3d(st + 4 * kRegion, v_map, bar, 64, h, k_row + k0);
                } else {
                    tma_load_4d(st, kn_map, bar, 0, h, k0, b);
                    tma_load_4d(st + kRegion, kn_map, bar, 64, h, k0, b);
                    tma_load_3d(st + 2 * kRegion, kp_map, bar, 0, k0, b);
                    tma_load_4d(st + 3 * kRegion, v_map, bar, 0, h, k0, b);
                    tma_load_4d(st + 4 * kRegion, v_map, bar, 64, h, k0, b);
                }
            }
        }
        return;
    }
    // ==================================================================== the two warpgroups
    regs_inc<232>();   // 128 x 40 + 256 x 232 <= 64 K registers
    // thread = rows ra = 16 (warp % 4) + lane / 4 and ra + 8 of its warpgroup; accumulator register 4 jb + 2 hh + e holds row
    // ra + 8 hh, column 8 jb + 2 (lane % 4) + e
    const int g = warp >> 2, ra = 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
    const int wg_first = past + q0 + 64 * g;       // position of the warpgroup's first query row
    const int pos0 = wg_first + ra;                // position of row ra (row ra + 8: pos0 + 8)
    // varlen: the last key each row sees, the causal limit clamped below kv_end (only rows past q_len reach the clamp)
    int lim[2] = {0, 0};
    if constexpr (kVarlen) { lim[0] = min(pos0, kv_end - 1); lim[1] = min(pos0 + 8, kv_end - 1); }
    const uint32_t qb = base + kOffQ + g * 64 * 128;
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; i++) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // l: this thread's share of the row sum
    bar_wait(smem_u32(&misc.q_full), 0);
    for (int j = 0; j < n; j++) {
        const int s = j % kStages, k0 = j * kBN;
        const uint32_t st = base + kOffStage + s * kStageBytes;
        bar_wait(smem_u32(&misc.full[s]), (j / kStages) & 1);
        // tile 0 always holds key 0, which every row sees: after it each row's maximum is finite
        if (k0 > wg_first + 63) {   // every key above this warpgroup's diagonal
            __syncwarp();
            if (lane == 0) bar_arrive(smem_u32(&misc.empty[s]));
            continue;
        }
        float sv[64];
        fence();
#pragma unroll
        for (int c = 0; c < 3; c++)
#pragma unroll
            for (int k = 0; k < 4; k++)
                mma_bf16_m64n128(sv, smem_desc(qb + c * kRegion + k * 32, 16, 1024, kLayoutSw128), smem_desc(st + c * kRegion + k * 32, 16, 1024, kLayoutSw128),
                                 (c | k) != 0);
        commit();
        wait<0>();
        fence_regs(sv);
        // mask per element before the maximum: key k0 + 8 jb + cq + e is visible to the row at position pos0 + 8 hh iff <= it
        const bool diag = kVarlen ? k0 + kBN - 1 > min(wg_first, kv_end - 1) : k0 + kBN - 1 > wg_first;
        float mt[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 64; i++) {
            const int hh = (i >> 1) & 1;
            float x = sv[i] * p.scale_log2;
            if (diag && k0 + 8 * (i >> 2) + cq + (i & 1) > (kVarlen ? lim[hh] : pos0 + 8 * hh)) x = -INFINITY;
            sv[i] = x;
            mt[hh] = fmaxf(mt[hh], x);
        }
        float a[2];
#pragma unroll
        for (int hh = 0; hh < 2; hh++) {
            mt[hh] = fmaxf(mt[hh], __shfl_xor_sync(0xffffffffu, mt[hh], 1));
            mt[hh] = fmaxf(mt[hh], __shfl_xor_sync(0xffffffffu, mt[hh], 2));
            const float mn = fmaxf(m[hh], mt[hh]);
            a[hh] = ex2(m[hh] - mn);                   // 0 on the first tile (m = -inf), O and l are still zero
            m[hh] = mn;
            l[hh] *= a[hh];
        }
        // P in bf16 as the A fragments of the eight K = 16 steps: pa[kk][i] = (p[8 kk + 2 i], p[8 kk + 2 i + 1])
        uint32_t pa[8][4];
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const int hh = (i >> 1) & 1;
            const float p0 = ex2(sv[i] - m[hh]), p1 = ex2(sv[i + 1] - m[hh]);
            l[hh] += p0 + p1;
            pa[i >> 3][(i >> 1) & 3] = pack_bf16(p0, p1);
        }
#pragma unroll
        for (int jb = 0; jb < 16; jb++) {
            o[4 * jb] *= a[0]; o[4 * jb + 1] *= a[0];
            o[4 * jb + 2] *= a[1]; o[4 * jb + 3] *= a[1];
        }
        if constexpr (kVarlen) {
            // P is 0 at keys >= kv_end, but 0 * NaN is NaN: zero the V rows of the crossing tile past kv_end (rows of 128 B
            // in both 64-column boxes; whole rows, so the swizzle does not matter).  Both warpgroups read every V row, so each
            // zeroes them all before its own P.V; the other's stores write the same zeros.
            if (k0 + kBN > kv_end) {
                const int valid = kv_end - k0;
                uint8_t* vt = smem_raw + (base - raw) + kOffStage + s * kStageBytes + 3 * kRegion;
                for (int i = (tid & 127); i < (kBN - valid) * 16; i += 128) {   // 8 pieces of 16 B per row and box
                    const int r = valid + (i >> 4), pc = i & 15;
                    *reinterpret_cast<uint4*>(vt + (pc >> 3) * kRegion + r * 128 + (pc & 7) * 16) = make_uint4(0, 0, 0, 0);
                }
                fence_async_smem();
                asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
            }
        }
        fence();
#pragma unroll
        for (int kk = 0; kk < 8; kk++)
            mma_bf16_rs_m64n128_bt(o, pa[kk], smem_desc(st + 3 * kRegion + kk * 2048, kRegion, 1024, kLayoutSw128), 1);
        commit();
        wait<0>();
        fence_regs(o);
        __syncwarp();
        if (lane == 0) bar_arrive(smem_u32(&misc.empty[s]));
    }
    // ---- epilogue: O / l -> bf16 -------------------------------------------------------------------------------------
#pragma unroll
    for (int hh = 0; hh < 2; hh++) {
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
        const int row = q0 + 64 * g + ra + 8 * hh;
        if (row >= q_len) continue;
        const float inv = 1.f / l[hh];
        __nv_bfloat16* dst = kVarlen ? p.out + ((long)(q_row + row) * p.num_heads + h) * 128 + cq
                                     : p.out + (((long)b * q_len + row) * p.num_heads + h) * 128 + cq;
#pragma unroll
        for (int jb = 0; jb < 16; jb++) *reinterpret_cast<uint32_t*>(dst + 8 * jb) = pack_bf16(o[4 * jb + 2 * hh] * inv, o[4 * jb + 2 * hh + 1] * inv);
    }
}

__global__ void __launch_bounds__(kThreads, 1) mla_prefill_kernel(const __grid_constant__ CUtensorMap qn_map, const __grid_constant__ CUtensorMap qp_map,
                                                                  const __grid_constant__ CUtensorMap kn_map, const __grid_constant__ CUtensorMap kp_map,
                                                                  const __grid_constant__ CUtensorMap v_map, const KParams p) {
    prefill_cta<false>(&qn_map, &qp_map, &kn_map, &kp_map, &v_map, p);
}

__global__ void __launch_bounds__(kThreads, 1) mla_prefill_varlen_kernel(const __grid_constant__ CUtensorMap qn_map, const __grid_constant__ CUtensorMap qp_map,
                                                                         const __grid_constant__ CUtensorMap kn_map, const __grid_constant__ CUtensorMap kp_map,
                                                                         const __grid_constant__ CUtensorMap v_map, const __grid_constant__ VParams p) {
    prefill_cta<true>(&qn_map, &qp_map, &kn_map, &kp_map, &v_map, p);
}

namespace prefill {

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

// bf16 operand [batch][tokens][heads][cols] (heads == 0: no head dimension; batch == 0: no batch dimension) with element
// strides, as boxes of 64 columns x 128 tokens; tokens past `tokens` read as zeros
static bool encode(EncodeTiledFn enc, CUtensorMap* map, const void* ptr, int cols, int heads, int tokens, int batch, long token_stride,
                   long head_stride, long batch_stride) {
    cuuint64_t gdim[4], gstr[3];
    cuuint32_t box[4], estr[4] = {1, 1, 1, 1};
    int rank = 0;
    gdim[rank] = (cuuint64_t)cols; box[rank++] = 64;
    if (heads > 0) { gdim[rank] = (cuuint64_t)heads; gstr[rank - 1] = (cuuint64_t)head_stride * 2; box[rank++] = 1; }
    gdim[rank] = (cuuint64_t)tokens; gstr[rank - 1] = (cuuint64_t)token_stride * 2; box[rank++] = 128;
    if (batch > 0) { gdim[rank] = (cuuint64_t)batch; gstr[rank - 1] = (cuuint64_t)batch_stride * 2; box[rank++] = 1; }
    return enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, rank, const_cast<void*>(ptr), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// the checks both entries make on head dims, sm_scale, the six operand pointers (q_nope, q_pe, k_nope, v, k_pe, out) and
// the strides; false with the error set
static bool check_operands(const char* who, int nope, int rope, int vdim, int num_heads, float sm_scale, const void* const (&ptrs)[6],
                           const long* strides, const char* const* snames, int n_strides) {
    if (nope != 128 || rope != 64 || vdim != 128) {
        set_error("%s: head dims %d / %d / %d, the kernel takes 128 / 64 / 128", who, nope, rope, vdim);
        return false;
    }
    if (num_heads < 1) { set_error("%s: num_heads %d must be >= 1", who, num_heads); return false; }
    if (!(sm_scale > 0.f) || !isfinite(sm_scale)) { set_error("%s: sm_scale must be a positive finite number", who); return false; }
    static const char* names[6] = {"q_nope", "q_pe", "k_nope", "v", "k_pe", "out"};
    for (int i = 0; i < 6; i++)
        if (!ptrs[i]) { set_error("%s: null pointer (%s)", who, names[i]); return false; }
    for (int i = 0; i < 6; i++)
        if ((uintptr_t)ptrs[i] & 15) { set_error("%s: %s must be 16-byte aligned", who, names[i]); return false; }
    for (int i = 0; i < n_strides; i++)
        if (strides[i] <= 0 || strides[i] % 8) {
            set_error("%s: %s stride %ld must be a positive multiple of 8 elements (16 bytes)", who, snames[i], strides[i]);
            return false;
        }
    return true;
}

// the dynamic shared memory of `kernel` raised to kSmem, once per device
static cudaError_t allow_smem(const void* kernel, bool (&done)[64]) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    if (e == cudaSuccess && !done[dev & 63]) {
        e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
        if (e == cudaSuccess) done[dev & 63] = true;
    }
    return e;
}

}  // namespace prefill
}  // namespace ktb

extern "C" int ktb200_mla_prefill(const ktb200_mla_prefill_params* q, void* stream) {
    using namespace ktb;
    using namespace ktb::prefill;
    if (!q) { set_error("mla_prefill: null parameter struct"); return KTB200_EINVAL; }
    if (q->batch < 1) { set_error("mla_prefill: batch %d and num_heads %d must be >= 1", q->batch, q->num_heads); return KTB200_EINVAL; }
    if (q->q_len < 1 || q->q_len > q->kv_len) { set_error("mla_prefill: need 1 <= q_len (%d) <= kv_len (%d)", q->q_len, q->kv_len); return KTB200_EINVAL; }
    if (q->q_len > 65535 * kBM) { set_error("mla_prefill: q_len %d exceeds %d tokens per call", q->q_len, 65535 * kBM); return KTB200_EINVAL; }
    const void* const ptrs[6] = {q->q_nope, q->q_pe, q->k_nope, q->v, q->k_pe, q->out};
    const long strides[14] = {q->q_nope_token_stride, q->q_nope_head_stride, q->q_nope_batch_stride, q->q_pe_token_stride, q->q_pe_head_stride,
                              q->q_pe_batch_stride, q->k_nope_token_stride, q->k_nope_head_stride, q->k_nope_batch_stride, q->v_token_stride,
                              q->v_head_stride, q->v_batch_stride, q->k_pe_token_stride, q->k_pe_batch_stride};
    static const char* snames[14] = {"q_nope token", "q_nope head", "q_nope batch", "q_pe token", "q_pe head", "q_pe batch", "k_nope token",
                                     "k_nope head", "k_nope batch", "v token", "v head", "v batch", "k_pe token", "k_pe batch"};
    if (!check_operands("mla_prefill", q->qk_nope_head_dim, q->qk_rope_head_dim, q->v_head_dim, q->num_heads, q->sm_scale, ptrs, strides, snames, 14))
        return KTB200_EINVAL;

    EncodeTiledFn enc = encode_tiled();
    if (!enc) { set_error("mla_prefill: cuTensorMapEncodeTiled is not available from this driver"); return KTB200_ECUDA; }
    CUtensorMap qn_map, qp_map, kn_map, kp_map, v_map;
    const int B = q->batch, H = q->num_heads;
    if (!encode(enc, &qn_map, q->q_nope, 128, H, q->q_len, B, q->q_nope_token_stride, q->q_nope_head_stride, q->q_nope_batch_stride) ||
        !encode(enc, &qp_map, q->q_pe, 64, H, q->q_len, B, q->q_pe_token_stride, q->q_pe_head_stride, q->q_pe_batch_stride) ||
        !encode(enc, &kn_map, q->k_nope, 128, H, q->kv_len, B, q->k_nope_token_stride, q->k_nope_head_stride, q->k_nope_batch_stride) ||
        !encode(enc, &kp_map, q->k_pe, 64, 0, q->kv_len, B, q->k_pe_token_stride, 0, q->k_pe_batch_stride) ||
        !encode(enc, &v_map, q->v, 128, H, q->kv_len, B, q->v_token_stride, q->v_head_stride, q->v_batch_stride)) {
        set_error("mla_prefill: cuTensorMapEncodeTiled rejected an operand layout");
        return KTB200_ECUDA;
    }
    static bool attr_set[64] = {};
    KTB_CUDA_CHECK(allow_smem((const void*)mla_prefill_kernel, attr_set));
    KParams p{};
    p.q_len = q->q_len; p.past = q->kv_len - q->q_len; p.num_heads = H;
    p.num_m_tiles = (q->q_len + kBM - 1) / kBM;
    p.scale_log2 = q->sm_scale * 1.4426950408889634f;
    p.out = (__nv_bfloat16*)q->out;
    mla_prefill_kernel<<<dim3(H * B, p.num_m_tiles), kThreads, kSmem, (cudaStream_t)stream>>>(qn_map, qp_map, kn_map, kp_map, v_map, p);
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

extern "C" int ktb200_mla_prefill_varlen(const ktb200_mla_prefill_varlen_params* q, void* stream) {
    using namespace ktb;
    using namespace ktb::prefill;
    if (!q) { set_error("mla_prefill_varlen: null parameter struct"); return KTB200_EINVAL; }
    if (q->batch < 1 || q->batch > kMaxSeqs) { set_error("mla_prefill_varlen: batch %d must be in 1 .. %d", q->batch, kMaxSeqs); return KTB200_EINVAL; }
    if (q->q_rows < 0 || q->k_rows < 0) { set_error("mla_prefill_varlen: q_rows %d and k_rows %d must be >= 0", q->q_rows, q->k_rows); return KTB200_EINVAL; }
    if (!q->seq) { set_error("mla_prefill_varlen: null pointer (seq)"); return KTB200_EINVAL; }
    const void* const ptrs[6] = {q->q_nope, q->q_pe, q->k_nope, q->v, q->k_pe, q->out};
    const long strides[9] = {q->q_nope_token_stride, q->q_nope_head_stride, q->q_pe_token_stride, q->q_pe_head_stride, q->k_nope_token_stride,
                             q->k_nope_head_stride, q->v_token_stride, q->v_head_stride, q->k_pe_token_stride};
    static const char* snames[9] = {"q_nope token", "q_nope head", "q_pe token", "q_pe head", "k_nope token", "k_nope head", "v token", "v head",
                                    "k_pe token"};
    if (!check_operands("mla_prefill_varlen", q->qk_nope_head_dim, q->qk_rope_head_dim, q->v_head_dim, q->num_heads, q->sm_scale, ptrs, strides, snames, 9))
        return KTB200_EINVAL;
    const int B = q->batch, H = q->num_heads;
    if ((long)B * H > 0x7fffffffL) { set_error("mla_prefill_varlen: batch * num_heads %ld exceeds 2^31 - 1", (long)B * H); return KTB200_EINVAL; }
    VParams p{};
    int order[kMaxSeqs], live = 0, max_tiles = 0;
    for (int b = 0; b < B; b++) {
        const int* s = q->seq + 4 * b;
        const int q_row = s[0], q_len = s[1], k_row = s[2], kv_len = s[3];
        if (q_row < 0 || q_len < 0 || k_row < 0 || kv_len < 0) {
            set_error("mla_prefill_varlen: sequence %d {q_row %d, q_len %d, k_row %d, kv_len %d} has a negative value", b, q_row, q_len, k_row, kv_len);
            return KTB200_EINVAL;
        }
        if (q_len > kv_len) { set_error("mla_prefill_varlen: sequence %d needs q_len (%d) <= kv_len (%d)", b, q_len, kv_len); return KTB200_EINVAL; }
        if (q_len > 65535 * kBM) { set_error("mla_prefill_varlen: sequence %d: q_len %d exceeds %d tokens per call", b, q_len, 65535 * kBM); return KTB200_EINVAL; }
        if ((long)q_row + q_len > q->q_rows) {
            set_error("mla_prefill_varlen: sequence %d query rows %d .. %ld are outside q_rows %d", b, q_row, (long)q_row + q_len, q->q_rows);
            return KTB200_EINVAL;
        }
        if ((long)k_row + kv_len > q->k_rows) {
            set_error("mla_prefill_varlen: sequence %d key rows %d .. %ld are outside k_rows %d", b, k_row, (long)k_row + kv_len, q->k_rows);
            return KTB200_EINVAL;
        }
        p.seq[b] = make_int4(q_row, q_len, k_row, kv_len);
        if (q_len > 0) order[live++] = b;
        max_tiles = max(max_tiles, (q_len + kBM - 1) / kBM);
    }
    std::sort(order, order + live, [&](int a, int b) { return p.seq[a].x < p.seq[b].x; });
    for (int i = 1; i < live; i++) {
        const int4 a = p.seq[order[i - 1]], c = p.seq[order[i]];
        if (a.x + a.y > c.x) {
            set_error("mla_prefill_varlen: the output rows of sequences %d and %d overlap", order[i - 1], order[i]);
            return KTB200_EINVAL;
        }
    }
    if (live == 0) return KTB200_OK;   // nothing to write (and no rows to map)

    EncodeTiledFn enc = encode_tiled();
    if (!enc) { set_error("mla_prefill_varlen: cuTensorMapEncodeTiled is not available from this driver"); return KTB200_ECUDA; }
    CUtensorMap qn_map, qp_map, kn_map, kp_map, v_map;
    if (!encode(enc, &qn_map, q->q_nope, 128, H, q->q_rows, 0, q->q_nope_token_stride, q->q_nope_head_stride, 0) ||
        !encode(enc, &qp_map, q->q_pe, 64, H, q->q_rows, 0, q->q_pe_token_stride, q->q_pe_head_stride, 0) ||
        !encode(enc, &kn_map, q->k_nope, 128, H, q->k_rows, 0, q->k_nope_token_stride, q->k_nope_head_stride, 0) ||
        !encode(enc, &kp_map, q->k_pe, 64, 0, q->k_rows, 0, q->k_pe_token_stride, 0, 0) ||
        !encode(enc, &v_map, q->v, 128, H, q->k_rows, 0, q->v_token_stride, q->v_head_stride, 0)) {
        set_error("mla_prefill_varlen: cuTensorMapEncodeTiled rejected an operand layout");
        return KTB200_ECUDA;
    }
    static bool attr_set[64] = {};
    KTB_CUDA_CHECK(allow_smem((const void*)mla_prefill_varlen_kernel, attr_set));
    p.num_heads = H;
    p.scale_log2 = q->sm_scale * 1.4426950408889634f;
    p.out = (__nv_bfloat16*)q->out;
    mla_prefill_varlen_kernel<<<dim3(H * B, max_tiles), kThreads, kSmem, (cudaStream_t)stream>>>(qn_map, qp_map, kn_map, kp_map, v_map, p);
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}
