// The small memory-bound steps between the projections of a DeepSeek decode layer, fused so that a layer is ~14 launches
// instead of ~40 ATen kernels (archive/ktransformers/operators/layernorm.py, RoPE.py and the residual adds of
// models/modeling_deepseek_v3.py DeepseekV3DecoderLayer.forward :1086-1140):
//   ktb200_add_rmsnorm   residual += delta ; out = RMSNorm(residual) * weight          (input_layernorm / post_attention_layernorm)
//   ktb200_mla_prep      q_a / kv_a layernorms are ktb200_add_rmsnorm calls; this kernel does what follows the q_b and kv_a
//                        projections of MLA: kv_a_layernorm on the 512 latent columns, RoPE on k_pe and on every head's
//                        q_pe (de-interleaved pairs, modeling_deepseek_v3.py:339-373), and the paged cache write
//                        (StaticCache.update, custom_cache.py:147-193) — one launch.
// RMSNorm follows DeepseekV3RMSNorm (modeling_deepseek_v3.py:65-80): variance in fp32, normalised value rounded to the
// input dtype, then multiplied by the weight in that dtype.
#include <cuda_bf16.h>

#include "common.cuh"

namespace ktb {

__device__ __forceinline__ float block_sum(float v, float* red) {   // red: >= blockDim.x / 32 floats
    v = warp_sum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float s = lane < nw ? red[lane] : 0.f;   // every warp adds the per-warp sums in the same (butterfly) order
    s = warp_sum(s);
    __syncthreads();
    return s;
}
__device__ __forceinline__ float bf(const __nv_bfloat16 v) { return __bfloat162float(v); }

// one CTA of 1024 threads per row, ONE pass: a thread keeps its <= 4 bf16 pairs in registers (H <= 8192), so the row is
// read once and the kernel is a single load -> block reduction -> store chain (it is launch-latency bound: 14 KB)
constexpr int kNormThreads = 1024, kNormPairs = 4;
__global__ void __launch_bounds__(kNormThreads) add_rmsnorm_kernel(__nv_bfloat16* resid, const __nv_bfloat16* delta, const __nv_bfloat16* weight, float eps,
                                                                   __nv_bfloat16* out, int H, long resid_stride, long delta_stride, long out_stride) {
    __shared__ float red[32];
    griddep_launch_dependents();
    __nv_bfloat162 wv[kNormPairs];
#pragma unroll
    for (int j = 0; j < kNormPairs; j++) {   // the norm weight does not depend on the previous kernel
        const int i = (threadIdx.x + j * kNormThreads) * 2;
        if (i < H) wv[j] = *reinterpret_cast<const __nv_bfloat162*>(weight + i);
    }
    griddep_wait();
    const long t = blockIdx.x;
    __nv_bfloat16* r = resid + t * resid_stride;
    const __nv_bfloat16* d = delta ? delta + t * delta_stride : nullptr;
    __nv_bfloat162 v[kNormPairs];
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < kNormPairs; j++) {
        const int i = (threadIdx.x + j * kNormThreads) * 2;
        if (i < H) {
            v[j] = *reinterpret_cast<const __nv_bfloat162*>(r + i);
            if (d) {
                v[j] = __hadd2(v[j], *reinterpret_cast<const __nv_bfloat162*>(d + i));   // the residual stream itself is bf16 (x = x + attn_out)
                *reinterpret_cast<__nv_bfloat162*>(r + i) = v[j];
            }
            const float2 f = __bfloat1622float2(v[j]);
            ss += f.x * f.x + f.y * f.y;
        }
    }
    const float inv = rsqrtf(block_sum(ss, red) / (float)H + eps);
    __nv_bfloat16* o = out + t * out_stride;
#pragma unroll
    for (int j = 0; j < kNormPairs; j++) {
        const int i = (threadIdx.x + j * kNormThreads) * 2;
        if (i < H) {
            const float2 f = __bfloat1622float2(v[j]);
            *reinterpret_cast<__nv_bfloat162*>(o + i) = __hmul2(wv[j], __floats2bfloat162_rn(f.x * inv, f.y * inv));
        }
    }
}

// grid (tokens), 256 threads: threads 0..63 of warps handle heads round-robin for q_pe; the latent norm uses the whole CTA
__global__ void __launch_bounds__(256) mla_prep_kernel(const __nv_bfloat16* q, int num_heads, int q_head_dim, int nope_dim, const __nv_bfloat16* kva,
                                                       const __nv_bfloat16* kv_norm_w, float eps, const float* cos_t, const float* sin_t,
                                                       __nv_bfloat16* kv_cache, int page_size, const int* page_idx, const int* page_off,
                                                       __nv_bfloat16* q_pe_out) {
    constexpr int R = 64, LAT = 512;
    __shared__ float red[8];
    griddep_launch_dependents();
    griddep_wait();
    const long t = blockIdx.x;
    const float* cs = cos_t + t * R;
    const float* sn = sin_t + t * R;
    // y[i] = x'[i] * cos[i] + rot(x')[i] * sin[i],  x'[i] = x[2i] (i < 32) | x[2(i-32)+1] ;  rot(x')[i] = -x'[i+32] | x'[i-32]
    auto rope = [&](const __nv_bfloat16* x, int i) -> float {
        const int half = R / 2;
        const float a = bf(x[i < half ? 2 * i : 2 * (i - half) + 1]);
        const float b = i < half ? -bf(x[2 * i + 1]) : bf(x[2 * (i - half)]);
        // the reference computes (q * cos) + (rotate_half(q) * sin) in the tensor dtype: each product rounded to bf16, then the sum
        const float p0 = __bfloat162float(__float2bfloat16_rn(a * cs[i])), p1 = __bfloat162float(__float2bfloat16_rn(b * sn[i]));
        return p0 + p1;
    };
    for (int u = threadIdx.x; u < num_heads * R; u += blockDim.x) {
        const int h = u / R, i = u - h * R;
        q_pe_out[(t * num_heads + h) * R + i] = __float2bfloat16_rn(rope(q + (t * num_heads + h) * q_head_dim + nope_dim, i));
    }
    __nv_bfloat16* dst = kv_cache + ((long)page_idx[t] * page_size + page_off[t]) * (LAT + R);
    const __nv_bfloat16* row = kva + t * (LAT + R);
    float ss = 0.f;
    for (int i = threadIdx.x; i < LAT; i += blockDim.x) { const float f = bf(row[i]); ss += f * f; }
    const float inv = rsqrtf(block_sum(ss, red) / (float)LAT + eps);
    for (int i = threadIdx.x; i < LAT; i += blockDim.x) {
        const __nv_bfloat16 hn = __float2bfloat16_rn(bf(row[i]) * inv);
        dst[i] = __hmul(kv_norm_w[i], hn);
    }
    if (threadIdx.x < R) dst[LAT + threadIdx.x] = __float2bfloat16_rn(rope(row + LAT, threadIdx.x));
}

}  // namespace ktb

using namespace ktb;

static bool misaligned(const void* p, uintptr_t bytes) { return ((uintptr_t)p & (bytes - 1)) != 0; }

extern "C" int ktb200_add_rmsnorm(void* residual, const void* delta, const void* weight, float eps, void* out, int n_tokens, int hidden, void* stream) {
    if (!residual || !weight || !out || n_tokens < 0) { set_error("add_rmsnorm: null pointer / negative n_tokens"); return KTB200_EINVAL; }
    if (hidden <= 0 || hidden % 2 || hidden > 2 * kNormPairs * kNormThreads) { set_error("add_rmsnorm: hidden %d must be even and <= 8192 (bf16)", hidden); return KTB200_EINVAL; }
    // bf16x2 loads and stores
    if (misaligned(residual, 4)) { set_error("add_rmsnorm: residual must be 4-byte aligned"); return KTB200_EINVAL; }
    if (misaligned(delta, 4)) { set_error("add_rmsnorm: delta must be 4-byte aligned"); return KTB200_EINVAL; }
    if (misaligned(weight, 4)) { set_error("add_rmsnorm: weight must be 4-byte aligned"); return KTB200_EINVAL; }
    if (misaligned(out, 4)) { set_error("add_rmsnorm: out must be 4-byte aligned"); return KTB200_EINVAL; }
    if (n_tokens == 0) return KTB200_OK;
    KTB_CUDA_CHECK(launch_pdl(add_rmsnorm_kernel, dim3(n_tokens), dim3(kNormThreads), 0, (cudaStream_t)stream, (__nv_bfloat16*)residual, (const __nv_bfloat16*)delta,
                              (const __nv_bfloat16*)weight, eps, (__nv_bfloat16*)out, hidden, (long)hidden, (long)hidden, (long)hidden));
    count_launch();
    return KTB200_OK;
}

extern "C" int ktb200_mla_prep(const void* q, int num_heads, int qk_nope_head_dim, const void* kv_a_out, const void* kv_a_norm_weight, float eps,
                               const float* cos, const float* sin, void* kv_cache, int page_size, const int* page_idx, const int* page_offset,
                               void* q_pe_out, int n_tokens, void* stream) {
    if (!q || !kv_a_out || !kv_a_norm_weight || !cos || !sin || !kv_cache || !page_idx || !page_offset || !q_pe_out || num_heads <= 0 || qk_nope_head_dim <= 0) {
        set_error("mla_prep: null pointer / bad shape");
        return KTB200_EINVAL;
    }
    if (n_tokens <= 0) return KTB200_OK;
    KTB_CUDA_CHECK(launch_pdl(mla_prep_kernel, dim3(n_tokens), dim3(256), 0, (cudaStream_t)stream, (const __nv_bfloat16*)q, num_heads, qk_nope_head_dim + 64,
                              qk_nope_head_dim, (const __nv_bfloat16*)kv_a_out, (const __nv_bfloat16*)kv_a_norm_weight, eps, cos, sin, (__nv_bfloat16*)kv_cache,
                              page_size, page_idx, page_offset, (__nv_bfloat16*)q_pe_out));
    count_launch();
    return KTB200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// The two absorb products of MLA decode (archive/ktransformers/operators/attention.py:428-431, 470-472), batch of
// one-row GEMVs over per-head bf16 weights — HBM-bound (16.8 MB each for DeepSeek-V3), fp32 accumulation:
//   mode 0  q_abs[t][h][c] = sum_d q_nope[t][h][d] * W_UK[h][d][c]     W [heads][D][C] read along c (contiguous)
//   mode 1  o[t][h][v]     = sum_c lat[t][h][c]   * W_UV[h][v][c]     W [heads][V][C] read along c (contiguous): one warp per (h, v)
namespace ktb {

constexpr int kMaxGridZ = 65535;   // the tokens of one absorb launch (gridDim.z)

// grid (C / 512, heads, tokens), 256 threads = 4 groups of 64: a group owns a quarter of the d range, a thread 8 columns of
// the 512-column slab (16-byte loads, 8 rows in flight); the four partial sums meet in shared memory in group order
__global__ void __launch_bounds__(256) absorb_q_kernel(const __nv_bfloat16* q, long q_head_stride, long q_tok_stride, const __nv_bfloat16* W, int D, int Cc,
                                                        __nv_bfloat16* out) {
    __shared__ float qs[512];
    __shared__ float part[4][512];
    griddep_launch_dependents();
    griddep_wait();
    const int h = blockIdx.y, t = blockIdx.z, heads = gridDim.y;
    const __nv_bfloat16* qrow = q + t * q_tok_stride + h * q_head_stride;
    for (int i = threadIdx.x; i < D; i += blockDim.x) qs[i] = bf(qrow[i]);
    __syncthreads();
    const int grp = threadIdx.x >> 6, ct = threadIdx.x & 63;
    const int c = blockIdx.x * 512 + ct * 8;
    float a[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (c < Cc) {
        const int dper = (D + 3) / 4, d0 = grp * dper, d1 = min(D, d0 + dper);
        const __nv_bfloat16* w = W + ((long)h * D) * Cc + c;
#pragma unroll 8
        for (int d = d0; d < d1; d++) {
            const uint4 raw = *reinterpret_cast<const uint4*>(w + (long)d * Cc);
            const __nv_bfloat162* w2 = reinterpret_cast<const __nv_bfloat162*>(&raw);
            const float qd = qs[d];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const float2 f = __bfloat1622float2(w2[i]);
                a[2 * i] = fmaf(qd, f.x, a[2 * i]);
                a[2 * i + 1] = fmaf(qd, f.y, a[2 * i + 1]);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 8; i++) part[grp][ct * 8 + i] = a[i];
    __syncthreads();
    const int cc = threadIdx.x * 2;
    if (blockIdx.x * 512 + cc < Cc) {
        const float s0 = (part[0][cc] + part[1][cc]) + (part[2][cc] + part[3][cc]);
        const float s1 = (part[0][cc + 1] + part[1][cc + 1]) + (part[2][cc + 1] + part[3][cc + 1]);
        *reinterpret_cast<__nv_bfloat162*>(out + ((long)t * heads + h) * Cc + blockIdx.x * 512 + cc) = __floats2bfloat162_rn(s0, s1);
    }
}

// grid (V / 8, heads, tokens), 256 threads = 8 warps: warp w owns output v = 8 * blockIdx.x + w
__global__ void __launch_bounds__(256) absorb_o_kernel(const __nv_bfloat16* lat, const __nv_bfloat16* W, int V, int Cc, __nv_bfloat16* out) {
    griddep_launch_dependents();
    griddep_wait();
    const int h = blockIdx.y, t = blockIdx.z, heads = gridDim.y, lane = threadIdx.x & 31;
    const int v = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (v >= V) return;
    const __nv_bfloat16* x = lat + ((long)t * heads + h) * Cc;
    const __nv_bfloat16* w = W + ((long)h * V + v) * Cc;
    float acc = 0.f;
    for (int c = lane * 8; c < Cc; c += 256) {
        const uint4 wv = *reinterpret_cast<const uint4*>(w + c), xv = *reinterpret_cast<const uint4*>(x + c);
        const __nv_bfloat162* w2 = reinterpret_cast<const __nv_bfloat162*>(&wv);
        const __nv_bfloat162* x2 = reinterpret_cast<const __nv_bfloat162*>(&xv);
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const float2 a = __bfloat1622float2(w2[i]), b = __bfloat1622float2(x2[i]);
            acc = fmaf(a.x, b.x, acc);
            acc = fmaf(a.y, b.y, acc);
        }
    }
    acc = warp_sum(acc);
    if (lane == 0) out[((long)t * heads + h) * V + v] = __float2bfloat16_rn(acc);
}

}  // namespace ktb

extern "C" int ktb200_mla_absorb_q(const void* q, long q_head_stride, long q_token_stride, const void* w_uk, int num_heads, int nope_dim, int kv_lora_rank,
                                   void* q_abs_out, int n_tokens, void* stream) {
    if (!q || !w_uk || !q_abs_out || num_heads <= 0) { set_error("mla_absorb_q: null pointer / bad num_heads"); return KTB200_EINVAL; }
    if (nope_dim <= 0 || nope_dim > 512) { set_error("mla_absorb_q: qk_nope_head_dim %d must be in 1..512", nope_dim); return KTB200_EINVAL; }   // qs[512]
    if (kv_lora_rank <= 0 || kv_lora_rank % 8) { set_error("mla_absorb_q: kv_lora_rank %d must be a positive multiple of 8", kv_lora_rank); return KTB200_EINVAL; }
    if (misaligned(w_uk, 16)) { set_error("mla_absorb_q: w_uk must be 16-byte aligned"); return KTB200_EINVAL; }          // uint4 weight loads
    if (misaligned(q_abs_out, 4)) { set_error("mla_absorb_q: q_abs_out must be 4-byte aligned"); return KTB200_EINVAL; }  // bf16x2 stores
    if (n_tokens <= 0) return KTB200_OK;
    for (int t0 = 0; t0 < n_tokens; t0 += kMaxGridZ) {   // tokens are grid.z: one launch per 65535
        const int nt = n_tokens - t0 < kMaxGridZ ? n_tokens - t0 : kMaxGridZ;
        KTB_CUDA_CHECK(launch_pdl(ktb::absorb_q_kernel, dim3((kv_lora_rank + 511) / 512, num_heads, nt), dim3(256), 0, (cudaStream_t)stream,
                                  (const __nv_bfloat16*)q + t0 * q_token_stride, q_head_stride, q_token_stride, (const __nv_bfloat16*)w_uk, nope_dim,
                                  kv_lora_rank, (__nv_bfloat16*)q_abs_out + (long)t0 * num_heads * kv_lora_rank));
        count_launch();
    }
    return KTB200_OK;
}

extern "C" int ktb200_mla_absorb_o(const void* attn_latent, const void* w_uv, int num_heads, int v_head_dim, int kv_lora_rank, void* out, int n_tokens, void* stream) {
    if (!attn_latent || !w_uv || !out || num_heads <= 0 || v_head_dim <= 0) { set_error("mla_absorb_o: null pointer / bad shape"); return KTB200_EINVAL; }
    if (kv_lora_rank <= 0 || kv_lora_rank % 8) { set_error("mla_absorb_o: kv_lora_rank %d must be a positive multiple of 8", kv_lora_rank); return KTB200_EINVAL; }
    // uint4 loads of both operands
    if (misaligned(attn_latent, 16)) { set_error("mla_absorb_o: attn_latent must be 16-byte aligned"); return KTB200_EINVAL; }
    if (misaligned(w_uv, 16)) { set_error("mla_absorb_o: w_uv must be 16-byte aligned"); return KTB200_EINVAL; }
    if (n_tokens <= 0) return KTB200_OK;
    for (int t0 = 0; t0 < n_tokens; t0 += kMaxGridZ) {
        const int nt = n_tokens - t0 < kMaxGridZ ? n_tokens - t0 : kMaxGridZ;
        KTB_CUDA_CHECK(launch_pdl(ktb::absorb_o_kernel, dim3((v_head_dim + 7) / 8, num_heads, nt), dim3(256), 0, (cudaStream_t)stream,
                                  (const __nv_bfloat16*)attn_latent + (long)t0 * num_heads * kv_lora_rank, (const __nv_bfloat16*)w_uv, v_head_dim,
                                  kv_lora_rank, (__nv_bfloat16*)out + (long)t0 * num_heads * v_head_dim));
        count_launch();
    }
    return KTB200_OK;
}
