// Activation quantisation to the reference's vec_dot types, bit-exact with the as-built x86
// reference (see oracle/ktoracle.c for the pinned semantics):
//   Q8_K  quantize_row_q8_K_reference  third_party/llama.cpp/ggml-quants.c:3593-3630
//   Q8_0  quantize_row_q8_0 (AVX path) third_party/llama.cpp/ggml-quants.c:936-1000
#pragma once
#include "common.cuh"

namespace ktb {

// One warp quantises one 256-element block held as 8 consecutive floats per lane
// (lane l owns elements 8l .. 8l+7).  Outputs:
//   q8  : 256 int8 written as 2 words per lane at q8_out[2*lane .. 2*lane+1]   (word = 4 int8)
//   d   : block scale (lane 0 writes *d_out)
//   bsums: 16 int16 sums of 16 consecutive q8 (even lanes write bsums_out[lane/2])
//
// Reference semantics reproduced exactly:
//   * `max` is the signed value of the FIRST element with the largest |x| (strict > scan).
//   * iscale = -127.f / max  (IEEE division);  d = 1 / iscale (IEEE division)
//   * q = min(127, nearest_int(iscale * x)) where the multiply and the 1.5*2^23 magic add are ONE
//     fused multiply-add (what gcc emits for the reference on every FMA-capable x86-64 build).
//   * an all-zero block gives d = 0, q = 0 (bsums forced to 0; the reference leaves them stale but
//     they are only ever multiplied by d == 0).
__device__ __forceinline__ void warp_quantize_q8k_block(const float (&x)[8], int lane, uint32_t* q8_out,
                                                        float* d_out, int16_t* bsums_out, int16_t* bs32_out = nullptr) {
    // local first-max scan
    float amax = 0.f, mx = 0.f;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        float ax = fabsf(x[i]);
        if (ax > amax) { amax = ax; mx = x[i]; }
    }
    // warp arg-max, first occurrence: |x| >= 0 orders like its bit pattern, so one REDUX finds the largest magnitude;
    // the lowest lane holding it owns the earliest element (a lane owns 8 consecutive elements and its own scan kept
    // the first), and one shuffle fetches that element's signed value.
    {
        const unsigned gmax = __reduce_max_sync(0xffffffffu, __float_as_uint(amax));
        const int src = __ffs(__ballot_sync(0xffffffffu, __float_as_uint(amax) == gmax)) - 1;
        mx = __shfl_sync(0xffffffffu, mx, src);
        amax = __uint_as_float(gmax);
    }
    uint32_t w0 = 0, w1 = 0;
    int s = 0;
    float d = 0.f;
    if (amax != 0.f) {
        const float iscale = __fdiv_rn(-127.f, mx);
        int q[8];
#pragma unroll
        for (int i = 0; i < 8; i++) {
            float val = __fmaf_rn(iscale, x[i], 12582912.f);
            int v = (int)(__float_as_uint(val) & 0x007fffffu) - 0x00400000;
            q[i] = v < 127 ? v : 127;
            s += q[i];
        }
        w0 = (uint32_t)(q[0] & 0xff) | ((uint32_t)(q[1] & 0xff) << 8) | ((uint32_t)(q[2] & 0xff) << 16) |
             ((uint32_t)(q[3] & 0xff) << 24);
        w1 = (uint32_t)(q[4] & 0xff) | ((uint32_t)(q[5] & 0xff) << 8) | ((uint32_t)(q[6] & 0xff) << 16) |
             ((uint32_t)(q[7] & 0xff) << 24);
        d = __frcp_rn(iscale);   // correctly rounded reciprocal == 1.f / iscale
    }
    q8_out[2 * lane] = w0;
    q8_out[2 * lane + 1] = w1;
    int s2 = s + __shfl_xor_sync(0xffffffffu, s, 1);
    if (bsums_out && (lane & 1) == 0) bsums_out[lane >> 1] = (int16_t)s2;
    if (bs32_out) {   // sums of 32 consecutive q8 (one Q4_K/Q5_K sub-block each), |sum| <= 4064
        const int s4 = s2 + __shfl_xor_sync(0xffffffffu, s2, 2);
        if ((lane & 3) == 0) bs32_out[lane >> 2] = (int16_t)s4;
    }
    if (lane == 0) *d_out = d;
}

// Load the 8 values lane `lane` owns of block `b` of a row (hidden-type or fp32 source).
__device__ __forceinline__ void load_block8(const void* src, long base, int hidden_type, float (&x)[8]) {
    if (hidden_type == KTB200_TYPE_F32) {
        const float4* p = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(src) + base);
        const float4 a = p[0], c = p[1];
        x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = c.x; x[5] = c.y; x[6] = c.z; x[7] = c.w;
    } else {
        const uint4 raw = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint16_t*>(src) + base);
        const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
        for (int i = 0; i < 4; i++) {
            if (hidden_type == KTB200_TYPE_BF16) {
                x[2 * i] = __uint_as_float(w[i] << 16);
                x[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
            } else {
                x[2 * i] = fp16_bits_to_f32((uint16_t)(w[i] & 0xffff));
                x[2 * i + 1] = fp16_bits_to_f32((uint16_t)(w[i] >> 16));
            }
        }
    }
}

// Quantise `nrows` rows of `n` (multiple of 256) values into shared staging arrays, all warps of the CTA
// cooperating.  Row r lives at src + row_off[r-th] ... expressed as src_off + r*src_stride (elements);
// rows r < 32 with bit r of skip_mask are left untouched.  Blocks are dealt round-robin to warps and processed G at a
// time: the G global loads are issued back to back BEFORE any of the shuffle reductions, so the prologue
// pays the memory latency once per group instead of once per block.
//   q8 [nrows][n] int8    dx [nrows][n/256] float    bsums [nrows][n/16] int16
template <int G>
__device__ __forceinline__ void cta_quantize_q8k_rows(const void* src, long src_off, long src_stride, int hidden_type,
                                                      int nrows, int n, unsigned skip_mask, uint8_t* q8, float* dx,
                                                      int16_t* bsums) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int bpr = n / QK_K, total = nrows * bpr;
    for (int g0 = warp; g0 < total; g0 += nwarps * G) {
        float x[G][8];
        bool live[G];
#pragma unroll
        for (int i = 0; i < G; i++) {
            const int gb = g0 + i * nwarps;
            live[i] = gb < total;
            if (live[i]) {
                const int r = gb / bpr, b = gb - r * bpr;
                live[i] = !(r < 32 && ((skip_mask >> r) & 1u));
                if (live[i]) load_block8(src, src_off + (long)r * src_stride + (long)b * QK_K + lane * 8, hidden_type, x[i]);
            }
        }
#pragma unroll
        for (int i = 0; i < G; i++) {
            if (live[i]) {   // warp-uniform
                const int gb = g0 + i * nwarps;
                const int r = gb / bpr, b = gb - r * bpr;
                warp_quantize_q8k_block(x[i], lane, reinterpret_cast<uint32_t*>(q8 + (size_t)r * n) + b * (QK_K / 4),
                                        dx + r * bpr + b, bsums + r * (n / 16) + b * 16);
            }
        }
    }
}

// Q8_0: one warp handles 8 consecutive 32-element blocks? Keep it simple: each lane owns one element of
// a 32-block, a warp quantises one block per step.  q8 [n] int8 (byte array), d [n/32] float (the
// fp16-rounded scale, widened), matching block_q8_0 {half d; int8 qs[32]}.
__device__ __forceinline__ void warp_quantize_q8_0_block(float x, int lane, int8_t* q_out, float* d_out,
                                                         uint16_t* d_bits_out) {
    float amax = fabsf(x);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    const float d = __fdiv_rn(amax, 127.f);
    const float id = (amax != 0.0f) ? __fdiv_rn(127.f, amax) : 0.0f;
    const __half hd = __float2half_rn(d);
    q_out[lane] = (int8_t)__float2int_rn(__fmul_rn(x, id));  // round-to-nearest-even, like _mm256_round_ps
    if (lane == 0) {
        *d_out = __half2float(hd);
        if (d_bits_out) *d_bits_out = __half_as_ushort(hd);
    }
}

}  // namespace ktb
