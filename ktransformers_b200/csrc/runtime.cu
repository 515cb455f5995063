#include <cstdlib>
// Host-side plumbing shared by all translation units: error string, launch counter, SM count.
#include <cstdarg>
#include <cstdio>
#include <atomic>

#include "gemv_bulk.cuh"

namespace ktb {
bool pdl_enabled() {
    static const bool on = [] { const char* e = getenv("KTB200_PDL"); return !e || atoi(e) != 0; }();
    return on;
}


static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

int num_sms(int device) {
    static int cached[64] = {0};
    if (device < 0 || device >= 64) device = 0;
    if (!cached[device]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || n <= 0) n = 132;
        cached[device] = n;
    }
    return cached[device];
}

}  // namespace ktb

extern "C" {
const char* ktb200_last_error(void) { return ktb::g_err; }
const char* ktb200_version(void) { return "ktb200 0.1 (sm_90a)"; }
long ktb200_type_size(int t) { return ktb::weight_block_bytes(t); }
long ktb200_blck_size(int t) { return ktb::weight_block_elems(t); }
unsigned long long ktb200_launch_count(void) { return ktb::g_launches.load(); }
}

// ---------------------------------------------------------------------------------------------------------------
// Diagnostics: what does a plain read-only stream achieve on this part?  (bench.py --probe; profiles/)
//   mode 0: grid-stride coalesced 16-byte loads, U loads in flight per thread
//   mode 1: every warp reads `chunk`-byte pieces at pseudo-random (hashed) offsets — the access shape of the
//           expert GEMV (one 4 KB weight row per warp at a time)
namespace ktb {
template <int U>
__global__ void __launch_bounds__(256) stream_read_kernel(const uint4* __restrict__ src, long n16, int mode, int chunk16,
                                                          unsigned* sink) {
    unsigned acc = 0;
    if (mode == 0) {
        const long stride = (long)gridDim.x * blockDim.x;
        long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
        for (; i + (U - 1) * stride < n16; i += U * stride) {
            uint4 v[U];
#pragma unroll
            for (int u = 0; u < U; u++) v[u] = ldg_stream16(src + i + u * stride);
#pragma unroll
            for (int u = 0; u < U; u++) acc ^= v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
        }
    } else {
        const int lane = threadIdx.x & 31;
        const long nwarps = (long)gridDim.x * (blockDim.x >> 5), w = (long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
        const long nchunks = n16 / chunk16;
        for (long c = w; c < nchunks; c += nwarps) {
            const long pc = (c * 2654435761L) % nchunks;   // scatter the chunks
            const uint4* p = src + pc * chunk16;
            for (int i = lane; i < chunk16; i += 32 * U) {
                uint4 v[U];
#pragma unroll
                for (int u = 0; u < U; u++) if (i + 32 * u < chunk16) v[u] = ldg_stream16(p + i + 32 * u); else v[u] = make_uint4(0, 0, 0, 0);
#pragma unroll
                for (int u = 0; u < U; u++) acc ^= v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
            }
        }
    }
    if (acc == 0x12345678u) *sink = acc;   // never true in practice: keeps the loads alive
}

// mode 2: the access shape of the bulk-copy kernels without their arithmetic — one CTA per SM, W warps, each with a
// private ring of S slots filled by cp.async.bulk and "consumed" by one 16-byte LDS per lane.  Upper bound for what
// the ring structure itself can stream in a launch of this size.
template <int S>
__global__ void __launch_bounds__(1024, 1) stream_bulk_kernel(const uint8_t* __restrict__ src, long nchunks, int chunk, unsigned* sink) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    const uint32_t bar_u32 = (uint32_t)__cvta_generic_to_shared(smem) + warp * S * 8;
    const int bar_bytes = (W * S * 8 + 15) & ~15;
    uint8_t* ring = smem + bar_bytes + (size_t)warp * S * chunk;
    const uint32_t ring_u32 = (uint32_t)__cvta_generic_to_shared(ring);
    if (lane == 0) {
        for (int s = 0; s < S; s++) mbar_init(bar_u32 + 8 * s, 1);
        mbar_fence_init();
        fence_proxy_async_smem();
    }
    __syncthreads();
    const long c0 = nchunks * blockIdx.x / gridDim.x, c1 = nchunks * (blockIdx.x + 1) / gridDim.x;
    long ci = c0 + warp;
    int slot_i = 0, slot_u = 0;
    uint32_t phase = 0;
    unsigned acc = 0;
    auto issue = [&]() {
        if (ci < c1) {
            if (lane == 0) {
                mbar_expect_tx(bar_u32 + 8 * slot_i, (uint32_t)chunk);
                bulk_g2s(ring_u32 + slot_i * chunk, src + ci * chunk, (uint32_t)chunk, bar_u32 + 8 * slot_i);
            }
            ci += W;
            slot_i = (slot_i + 1 == S) ? 0 : slot_i + 1;
        }
    };
    for (int s = 0; s < S; s++) issue();
    for (long c = c0 + warp; c < c1; c += W) {
        mbar_wait(bar_u32 + 8 * slot_u, (phase >> slot_u) & 1u);
        phase ^= 1u << slot_u;
        const uint4 v = *reinterpret_cast<const uint4*>(ring + slot_u * chunk + lane * 16);
        acc ^= v.x ^ v.y ^ v.z ^ v.w;
        __syncwarp();
        slot_u = (slot_u + 1 == S) ? 0 : slot_u + 1;
        issue();
    }
    if (acc == 0x12345678u) *sink = acc;
}
}  // namespace ktb

extern "C" int ktb200_debug_stream_read(const void* src, long bytes, int mode, int unroll, int ctas_per_sm, int chunk_bytes,
                                        void* stream, float* ms_out) {
    using namespace ktb;
    int dev = 0;
    KTB_CUDA_CHECK(cudaGetDevice(&dev));
    static unsigned* sink = nullptr;
    if (!sink) KTB_CUDA_CHECK(cudaMalloc(&sink, 4));
    cudaStream_t s = (cudaStream_t)stream;
    cudaEvent_t e0, e1;
    KTB_CUDA_CHECK(cudaEventCreate(&e0));
    KTB_CUDA_CHECK(cudaEventCreate(&e1));
    const int grid = num_sms(dev) * (ctas_per_sm > 0 ? ctas_per_sm : 2);
    const long n16 = bytes / 16;
    if (mode == 2) {   // unroll = ring slots, ctas_per_sm = warps per CTA
        const int W = ctas_per_sm > 0 ? (ctas_per_sm > 32 ? 32 : ctas_per_sm) : 16, S = unroll >= 4 ? 4 : (unroll == 3 ? 3 : 2);
        const size_t smem = (((size_t)W * S * 8 + 15) & ~(size_t)15) + (size_t)W * S * chunk_bytes;
        if (chunk_bytes % 16 || smem > 232448 - 256) { set_error("stream probe: ring does not fit"); cudaEventDestroy(e0); cudaEventDestroy(e1); return KTB200_EINVAL; }
        const long nchunks = bytes / chunk_bytes;
        auto k = S == 4 ? stream_bulk_kernel<4> : (S == 3 ? stream_bulk_kernel<3> : stream_bulk_kernel<2>);
        KTB_CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        KTB_CUDA_CHECK(cudaEventRecord(e0, s));
        k<<<num_sms(dev), W * 32, smem, s>>>(reinterpret_cast<const uint8_t*>(src), nchunks, chunk_bytes, sink);
        KTB_LAUNCH_CHECK();
        KTB_CUDA_CHECK(cudaEventRecord(e1, s));
        KTB_CUDA_CHECK(cudaEventSynchronize(e1));
        if (ms_out) cudaEventElapsedTime(ms_out, e0, e1);
        cudaEventDestroy(e0); cudaEventDestroy(e1);
        return KTB200_OK;
    }
    KTB_CUDA_CHECK(cudaEventRecord(e0, s));
    if (unroll >= 8) stream_read_kernel<8><<<grid, 256, 0, s>>>((const uint4*)src, n16, mode, chunk_bytes / 16, sink);
    else if (unroll >= 4) stream_read_kernel<4><<<grid, 256, 0, s>>>((const uint4*)src, n16, mode, chunk_bytes / 16, sink);
    else stream_read_kernel<2><<<grid, 256, 0, s>>>((const uint4*)src, n16, mode, chunk_bytes / 16, sink);
    KTB_LAUNCH_CHECK();
    KTB_CUDA_CHECK(cudaEventRecord(e1, s));
    KTB_CUDA_CHECK(cudaEventSynchronize(e1));
    if (ms_out) cudaEventElapsedTime(ms_out, e0, e1);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return KTB200_OK;
}
