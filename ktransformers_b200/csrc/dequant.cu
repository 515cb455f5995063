// GGUF block -> dense tensor (load path).  Replaces KTransformersOps.dequantize_* of the reference
// (kt-kernel/cuda/custom_gguf/dequant.cu:23-661: one THREAD per 256-element super-block, scalar byte
// loads).  Here one thread owns one 16-element group, so a warp covers two super-blocks with
// contiguous 32-byte stores per lane; value = fma(d*sc, q, -(dmin*m)) in fp32, then cast — the same
// expression the reference kernels evaluate (dequant.cu:343-413 for Q4_K, 502-595 for Q6_K).
#define KTB_IQ_CODEBOOKS
#include "formats.cuh"

namespace ktb {

template <typename OutT>
__device__ __forceinline__ OutT cast_out(float v);
template <> __device__ __forceinline__ float cast_out<float>(float v) { return v; }
template <> __device__ __forceinline__ __half cast_out<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 cast_out<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

template <typename OutT>
__global__ void __launch_bounds__(256) dequant_k_kernel(const uint8_t* src, int type, int bsz, long n_groups, OutT* out) {
    for (long gi = (long)blockIdx.x * blockDim.x + threadIdx.x; gi < n_groups; gi += (long)gridDim.x * blockDim.x) {
        GroupK g;
        unpack_group16(type, src + (gi >> 4) * bsz, (int)(gi & 15), g);
        const float dl = g.d * (float)g.isc, ml = g.dmin * (float)g.imn;
        OutT* o = out + gi * 16;
#pragma unroll
        for (int w = 0; w < 4; w++)
#pragma unroll
            for (int b = 0; b < 4; b++) {
                const float q = (float)(int8_t)((g.q[w] >> (8 * b)) & 0xff);
                o[4 * w + b] = cast_out<OutT>(__fmaf_rn(dl, q, -ml));
            }
    }
}

// block_q8_0 {half d; int8 qs[32]} (ggml-quants.c:1609-1624): y = qs * d
template <typename OutT>
__global__ void __launch_bounds__(256) dequant_q8_0_kernel(const uint8_t* src, long n, OutT* out) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        const uint8_t* blk = src + (i >> 5) * SZ_Q8_0;
        const float d = fp16_bits_to_f32(ldg_u16(blk));
        out[i] = cast_out<OutT>((float)(int8_t)ldg_u8(blk + 2 + (i & 31)) * d);
    }
}

// RAWINT4_G32 device blocks (rawint4.cuh): thread = one 32-bit word = 8 values, value = (u - 8) * s in fp32, then cast
template <typename OutT>
__global__ void __launch_bounds__(256) dequant_rawint4_kernel(const uint8_t* src, long n_words, OutT* out) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += (long)gridDim.x * blockDim.x) {
        const uint8_t* blk = src + (i >> 5) * SZ_RAWINT4;
        const int wi = (int)(i & 31);                     // word of the block; group wi / 4
        const uint32_t w = *reinterpret_cast<const uint32_t*>(blk + 16 + 4 * wi);
        const float s = __uint_as_float((uint32_t)reinterpret_cast<const uint16_t*>(blk)[wi >> 2] << 16);
#pragma unroll
        for (int v = 0; v < 8; v++) out[i * 8 + v] = cast_out<OutT>((float)((int)((w >> (4 * v)) & 15u) - 8) * s);
    }
}

template <typename InT, typename OutT>
__global__ void __launch_bounds__(256) convert_kernel(const InT* src, long n, OutT* out) {
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
        out[i] = cast_out<OutT>((float)src[i]);
}

template <typename OutT>
static int dequant_to(const void* src, int type, long n, OutT* out, cudaStream_t s) {
    int dev = 0;
    cudaGetDevice(&dev);
    const int max_blocks = num_sms(dev) * 16;
    if (type == KTB200_TYPE_Q8_0) {
        long blocks = (n + 255) / 256;
        if (blocks > max_blocks) blocks = max_blocks;
        dequant_q8_0_kernel<OutT><<<(unsigned)blocks, 256, 0, s>>>(reinterpret_cast<const uint8_t*>(src), n, out);
    } else if (is_kquant(type) || is_iquant(type)) {
        const long ng = n / 16;
        long blocks = (ng + 255) / 256;
        if (blocks > max_blocks) blocks = max_blocks;
        dequant_k_kernel<OutT><<<(unsigned)blocks, 256, 0, s>>>(reinterpret_cast<const uint8_t*>(src), type, (int)weight_block_bytes(type), ng, out);
    } else if (is_rawint4(type)) {
        long blocks = (n / 8 + 255) / 256;
        if (blocks > max_blocks) blocks = max_blocks;
        dequant_rawint4_kernel<OutT><<<(unsigned)blocks, 256, 0, s>>>(reinterpret_cast<const uint8_t*>(src), n / 8, out);
    } else if (type == KTB200_TYPE_F32 || type == KTB200_TYPE_F16 || type == KTB200_TYPE_BF16) {
        long blocks = (n + 255) / 256;
        if (blocks > max_blocks) blocks = max_blocks;
        if (type == KTB200_TYPE_F32) convert_kernel<float, OutT><<<(unsigned)blocks, 256, 0, s>>>(reinterpret_cast<const float*>(src), n, out);
        else if (type == KTB200_TYPE_F16) convert_kernel<__half, OutT><<<(unsigned)blocks, 256, 0, s>>>(reinterpret_cast<const __half*>(src), n, out);
        else convert_kernel<__nv_bfloat16, OutT><<<(unsigned)blocks, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(src), n, out);
    } else {
        set_error("dequantize: unsupported ggml type %d", type);
        return KTB200_EINVAL;
    }
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

}  // namespace ktb

extern "C" int ktb200_dequantize(const void* src, int type, long n, void* out, int out_type, void* stream) {
    using namespace ktb;
    if (!src || !out) { set_error("null pointer"); return KTB200_EINVAL; }
    if (n <= 0) return KTB200_OK;
    const long blk = weight_block_elems(type);
    if (blk == 0 || n % blk) { set_error("dequantize: n=%ld is not a multiple of the block size of type %d", n, type); return KTB200_EINVAL; }
    cudaStream_t s = (cudaStream_t)stream;
    switch (out_type) {
        case KTB200_TYPE_F32: return dequant_to<float>(src, type, n, reinterpret_cast<float*>(out), s);
        case KTB200_TYPE_F16: return dequant_to<__half>(src, type, n, reinterpret_cast<__half*>(out), s);
        case KTB200_TYPE_BF16: return dequant_to<__nv_bfloat16>(src, type, n, reinterpret_cast<__nv_bfloat16*>(out), s);
        default: set_error("dequantize: out_type %d must be F32/F16/BF16", out_type); return KTB200_EINVAL;
    }
}
