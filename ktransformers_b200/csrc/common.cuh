// Shared device helpers for the ktb200 kernels (sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/ktb200.h"

#define QK_K 256
#define SZ_Q8_0 34
#define SZ_Q2_K 84
#define SZ_Q3_K 110
#define SZ_Q4_K 144
#define SZ_Q5_K 176
#define SZ_Q6_K 210
#define SZ_Q8_K 292
#define SZ_IQ4_XS 136
#define SZ_IQ2_XXS 66    // fp16 d + 8 x (4 grid indices | signs + scale) words
#define SZ_IQ1_S 50      // fp16 d + qs[32] + qh[8] (uint16)
#define SZ_IQ1_M 56      // qs[32] + qh[16] + scales[4] (uint16, fp16 d in the top nibbles)
#define SZ_IQ3_XXS 98    // fp16 d + qs[64] + 8 x (signs + scale) words
#define SZ_IQ3_S 110     // fp16 d + qs[64] + qh[8] + signs[32] + scales[4]
#define SZ_IQ2_XS 74     // fp16 d + qs[32] (uint16: 9-bit grid index | 7-bit sign index) + scales[8]
#define SZ_IQ2_S 82      // fp16 d + qs[32] + signs[32] + qh[8] + scales[8]
#define SZ_RAWINT4 144   // 8 bf16 scales + 256 nibbles (rawint4.cuh)

namespace ktb {

// ------------------------------------------------------------------ error plumbing (host)
void set_error(const char* fmt, ...);
void count_launch(int n = 1);
#define KTB_CUDA_CHECK(expr)                                                                 \
    do {                                                                                     \
        cudaError_t _e = (expr);                                                             \
        if (_e != cudaSuccess) {                                                             \
            ktb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            return KTB200_ECUDA;                                                             \
        }                                                                                    \
    } while (0)
#define KTB_LAUNCH_CHECK()                                                                   \
    do {                                                                                     \
        cudaError_t _e = cudaGetLastError();                                                 \
        if (_e != cudaSuccess) {                                                             \
            ktb::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
            return KTB200_ECUDA;                                                             \
        }                                                                                    \
        ktb::count_launch();                                                                 \
    } while (0)

int num_sms(int device);

#ifdef __CUDACC__
// launch with the programmatic-stream-serialization attribute (KTB200_PDL=0 disables it library-wide)
bool pdl_enabled();
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
    cudaLaunchConfig_t lc{};
    lc.gridDim = grid; lc.blockDim = block; lc.dynamicSmemBytes = smem; lc.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    lc.attrs = at; lc.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&lc, kernel, static_cast<KArgs>(args)...);
}
#endif

__host__ __device__ inline long type_size(int t) {
    switch (t) {
        case KTB200_TYPE_F32: return 4;
        case KTB200_TYPE_F16: case KTB200_TYPE_BF16: return 2;
        case KTB200_TYPE_Q8_0: return SZ_Q8_0;
        case KTB200_TYPE_Q2_K: return SZ_Q2_K;
        case KTB200_TYPE_Q3_K: return SZ_Q3_K;
        case KTB200_TYPE_Q4_K: return SZ_Q4_K;
        case KTB200_TYPE_Q5_K: return SZ_Q5_K;
        case KTB200_TYPE_Q6_K: return SZ_Q6_K;
        case KTB200_TYPE_Q8_K: return SZ_Q8_K;
        case KTB200_TYPE_IQ4_XS: return SZ_IQ4_XS;
        case KTB200_TYPE_RAWINT4_G32: return SZ_RAWINT4;
        default: return 0;
    }
}
__host__ __device__ inline long blck_size(int t) {
    switch (t) {
        case KTB200_TYPE_F32: case KTB200_TYPE_F16: case KTB200_TYPE_BF16: return 1;
        case KTB200_TYPE_Q8_0: return 32;
        case KTB200_TYPE_Q2_K: case KTB200_TYPE_Q3_K: case KTB200_TYPE_Q4_K: case KTB200_TYPE_Q5_K:
        case KTB200_TYPE_Q6_K: case KTB200_TYPE_Q8_K: case KTB200_TYPE_IQ4_XS: case KTB200_TYPE_RAWINT4_G32: return QK_K;
        default: return 0;
    }
}
__host__ __device__ inline bool is_kquant(int t) {
    return t == KTB200_TYPE_Q2_K || t == KTB200_TYPE_Q3_K || t == KTB200_TYPE_Q4_K || t == KTB200_TYPE_Q5_K ||
           t == KTB200_TYPE_Q6_K || t == KTB200_TYPE_IQ4_XS;
}
// codebook i-quants: routed experts only (iq.cuh bulk kernels, generic per-pair fallback), no linear /
// MLP / grouped / block / expert-parallel path
__host__ __device__ inline bool is_iquant(int t) {
    return t == KTB200_TYPE_IQ2_XXS || t == KTB200_TYPE_IQ1_S || t == KTB200_TYPE_IQ1_M || t == KTB200_TYPE_IQ3_XXS ||
           t == KTB200_TYPE_IQ3_S || t == KTB200_TYPE_IQ2_XS || t == KTB200_TYPE_IQ2_S;
}
static inline const char* iquant_name(int t) {
    return t == KTB200_TYPE_IQ1_S ? "IQ1_S" : t == KTB200_TYPE_IQ2_XXS ? "IQ2_XXS" : t == KTB200_TYPE_IQ1_M ? "IQ1_M"
         : t == KTB200_TYPE_IQ3_XXS ? "IQ3_XXS" : t == KTB200_TYPE_IQ3_S ? "IQ3_S" : t == KTB200_TYPE_IQ2_XS ? "IQ2_XS"
         : t == KTB200_TYPE_IQ2_S ? "IQ2_S" : "?";
}
// block geometry including the i-quants.  Kept apart from type_size / blck_size, which every kernel inlines for its hidden
// type: a longer switch there would change the code of kernels that never see an i-quant.
__host__ __device__ inline long weight_block_bytes(int t) {
    return t == KTB200_TYPE_IQ2_XXS ? SZ_IQ2_XXS : t == KTB200_TYPE_IQ1_S ? SZ_IQ1_S : t == KTB200_TYPE_IQ1_M ? SZ_IQ1_M
         : t == KTB200_TYPE_IQ3_XXS ? SZ_IQ3_XXS : t == KTB200_TYPE_IQ3_S ? SZ_IQ3_S : t == KTB200_TYPE_IQ2_XS ? SZ_IQ2_XS
         : t == KTB200_TYPE_IQ2_S ? SZ_IQ2_S : type_size(t);
}
__host__ __device__ inline long weight_block_elems(int t) { return is_iquant(t) ? QK_K : blck_size(t); }
// not a K-quant: it has its own kernels (rawint4.cuh) and no path through the generic K-quant ones
__host__ __device__ inline bool is_rawint4(int t) { return t == KTB200_TYPE_RAWINT4_G32; }
__host__ __device__ inline bool is_hidden_type(int t) {
    return t == KTB200_TYPE_F32 || t == KTB200_TYPE_F16 || t == KTB200_TYPE_BF16;
}
__host__ __device__ inline long row_bytes(long n, int t) { return n / blck_size(t) * type_size(t); }

#ifdef __CUDACC__
// ------------------------------------------------------------------ loads
// Streaming 16-byte weight load: read-only path, do not allocate in L1 (each weight byte is used once).
__device__ __forceinline__ uint4 ldg_stream16(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ uint32_t ldg_stream4(const void* p) {
    uint32_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
// Ask the memory system to pull `bytes` (multiple of 16, 16-byte aligned) into L2 ahead of use: one
// instruction, no registers held while the data is in flight (cp.async.bulk.prefetch.L2, sm_90+).
__device__ __forceinline__ void prefetch_l2_bulk(const void* p, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
// Programmatic dependent launch (PDL): a kernel launched with launch_pdl() may start while its predecessor in the stream is
// still running; everything it reads from — or writes over — what the predecessor touches must come after griddep_wait()
// (which returns when the predecessor grid has completed and flushed).  griddep_launch_dependents() lets the successor's
// launch processing begin.  Weight prefetches go before the wait, activations after it.
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ uint16_t ldg_u16(const void* p) { return __ldg(reinterpret_cast<const unsigned short*>(p)); }
__device__ __forceinline__ uint8_t ldg_u8(const void* p) { return __ldg(reinterpret_cast<const unsigned char*>(p)); }

__device__ __forceinline__ int dp4a_s8s8(uint32_t a, uint32_t b, int c) { return __dp4a((int)a, (int)b, c); }
// a holds unsigned bytes (0..255), b signed bytes
__device__ __forceinline__ int dp4a_u8s8(uint32_t a, uint32_t b, int c) {
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// ------------------------------------------------------------------ hidden-type conversions
__device__ __forceinline__ float fp16_bits_to_f32(uint16_t h) { return __half2float(__ushort_as_half(h)); }

// ------------------------------------------------------------------ IQ1_S / IQ1_M / IQ2 / IQ3 arithmetic shared by iq.cuh and grouped.cu
// a super-block's fp32 term (DESIGN.md §2): ((d / 8) * dx) * S with the exact integer S of the super-block; also the term
// (d * dx) * isum of Q3_K and Q6_K (gemv_bulk.cuh BulkQ3K, grouped.cu)
__device__ __forceinline__ float iq_d8(uint16_t d_bits) { return fp16_bits_to_f32(d_bits) * 0.125f; }
// IQ3_XXS's d / 4: the reference's final 0.25 folded into the scale (exact, a power of two)
__device__ __forceinline__ float iq_d4(uint16_t d_bits) { return fp16_bits_to_f32(d_bits) * 0.25f; }
__device__ __forceinline__ float iq_term(float d8, float dx, int isum) { return (d8 * dx) * (float)isum; }
// IQ1_M's fp16 d: the top nibbles of its four scale words (s01 = scales[0] | scales[1] << 16, s23 likewise), scales[0]'s lowest
__device__ __forceinline__ uint16_t iq1m_d_bits(uint32_t s01, uint32_t s23) {
    return (uint16_t)(((s01 >> 12) & 0x000fu) | ((s01 >> 24) & 0x00f0u) | ((s23 >> 4) & 0x0f00u) | ((s23 >> 16) & 0xf000u));
}
// the term of a K-quant with mins (gemv_bulk.cuh BulkQ2K; grouped.cu's Q4_K, Q5_K and Q2_K finish): (d * dx) * isum -
// (dmin * dx) * msum, msum the exact sum of the mins times the activation sums
__device__ __forceinline__ float kq_min_term(float d, float dmin, float dx, int isum, float msum) {
    return (d * dx) * (float)isum - (dmin * dx) * msum;
}
// an IQ2_XXS / IQ2_XS / IQ3_XXS sign pattern (ksigns_iq2xs byte), or an IQ2_S / IQ3_S sign byte, as byte masks: value = (grid ^ m) - m per byte
__device__ __forceinline__ uint2 iq2_sign_masks(uint32_t s) {
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        lo |= ((s >> j) & 1u) ? 0xffu << (8 * j) : 0u;
        hi |= ((s >> (j + 4)) & 1u) ? 0xffu << (8 * j) : 0u;
    }
    return make_uint2(lo, hi);
}

// ggml_compute_fp32_to_bf16 (third_party/llama.cpp/ggml-impl.h:87-104): RNE, NaN quieted,
// fp32 subnormals flushed to signed zero.
__device__ __forceinline__ uint16_t f32_to_bf16_ggml(float f) {
    uint32_t i = __float_as_uint(f);
    if ((i & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((i >> 16) | 64);
    if (!(i & 0x7f800000u)) return (uint16_t)((i & 0x80000000u) >> 16);
    return (uint16_t)((i + (0x7fffu + ((i >> 16) & 1))) >> 16);
}

__device__ __forceinline__ float load_hidden(const void* base, long idx, int hidden_type) {
    if (hidden_type == KTB200_TYPE_BF16) {
        return __uint_as_float(((uint32_t) reinterpret_cast<const uint16_t*>(base)[idx]) << 16);
    } else if (hidden_type == KTB200_TYPE_F16) {
        return __half2float(reinterpret_cast<const __half*>(base)[idx]);
    }
    return reinterpret_cast<const float*>(base)[idx];
}
__device__ __forceinline__ void store_hidden(void* base, long idx, int hidden_type, float v) {
    if (hidden_type == KTB200_TYPE_BF16) {
        reinterpret_cast<uint16_t*>(base)[idx] = f32_to_bf16_ggml(v);
    } else if (hidden_type == KTB200_TYPE_F16) {
        reinterpret_cast<__half*>(base)[idx] = __float2half_rn(v);  // == _cvtss_sh(x, 0), GGML_FP32_TO_FP16
    } else {
        reinterpret_cast<float*>(base)[idx] = v;
    }
}

__device__ __forceinline__ float round_hidden(float v, int hidden_type) {
    if (hidden_type == KTB200_TYPE_BF16) return __uint_as_float(((uint32_t)f32_to_bf16_ggml(v)) << 16);
    if (hidden_type == KTB200_TYPE_F16) return __half2float(__float2half_rn(v));
    return v;
}

// act_fn (operators/llamafile/moe.cpp:134-136) and act_fn_relu (:138-144); IEEE division, accurate expf.
__device__ __forceinline__ float act_silu(float x) { return __fdiv_rn(x, 1.0f + expf(-x)); }
__device__ __forceinline__ float act_relu(float x) { return x > 0.0f ? x : 0.0f; }

// get_scale_min_k4 for the sub-block pair (2j, 2j+1) of a Q4_K/Q5_K block; w0..w2 are the 12 scale
// bytes as three little-endian words.  Returns sc = sc0 | sc1<<8, mn = m0 | m1<<8.
// (third_party/llama.cpp/ggml-quants.c:1891-1899)
__device__ __forceinline__ void scale_min_pair_k4(uint32_t w0, uint32_t w1, uint32_t w2, int j, uint32_t& sc,
                                                  uint32_t& mn) {
    const int sh = (j & 1) * 16;
    const uint32_t a0 = w0 >> sh, a1 = w1 >> sh, a2 = w2 >> sh;
    if (j < 2) {
        sc = a0 & 0x3f3fu;
        mn = a1 & 0x3f3fu;
    } else {
        sc = (a2 & 0x0f0fu) | ((a0 >> 2) & 0x3030u);
        mn = ((a2 >> 4) & 0x0f0fu) | ((a1 >> 2) & 0x3030u);
    }
}
#endif  // __CUDACC__

}  // namespace ktb
