// Expert-parallel token exchange over NVLink peer memory (one process per GPU; every rank maps the others' buffers).
//
// Replaces the two latency-bound NCCL collectives of an expert-parallel decode layer (all-gather of the N tokens,
// reduce-scatter of the N x H fp32 partial sums) with two small hand-written kernels that
// store / load peer memory directly and synchronise with system-scope flags:
//
//   ktb200_ep_all_gather_tokens   rank r stores its token row into row r of EVERY peer's token buffer (14 KB each),
//                                 releases a flag on every peer, waits for the N flags addressed to it, and converts
//                                 the gathered rows to fp32 for the shard's expert kernels in the same launch.
//   ktb200_ep_reduce_own_token    rank r announces "my partial sums are complete", waits for the N announcements, then
//                                 LOADS row r of every peer's partial buffer and adds the N rows in rank order (the same
//                                 order on every rank and every run: deterministic), rounds once to the hidden type and
//                                 adds the (already rounded) shared-expert term: y = round(sum) + y_shared
//                                 (KDeepseekV3MoE.forward, experts.py:984-1011).
//
// Epochs live in device memory and are advanced by the kernels themselves (graph replays need no host parameter).
// Buffer reuse is safe without extra barriers: a peer can only overwrite my token buffer for layer L+1 after passing
// its layer-L reduce barrier, which waits for my layer-L announcement, which my stream orders after my expert kernels
// (the readers of the token buffer); symmetrically my partial buffer is only rewritten after the layer-(L+1) gather
// barrier, which every peer reaches after it finished reading my layer-L partial sums.
#include "common.cuh"

namespace ktb {

constexpr int kEpMaxWorld = 16;

struct EpParams {
    int rank, world, H, hidden_type;
    void* tok[kEpMaxWorld];        // every rank's token buffer [world][H] hidden_type
    float* part[kEpMaxWorld];      // every rank's partial-sum buffer [world][H] fp32
    unsigned* flags[kEpMaxWorld];  // every rank's flag block: [0 .. world) gather flags, [world .. 2 world) reduce flags, [2 world] epochs (2)
};

__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// one CTA; `which` = 0 gather / 1 reduce.  Returns this call's epoch to every thread.
__device__ __forceinline__ unsigned ep_next_epoch(const EpParams& p, int which, unsigned* s_epoch) {
    if (threadIdx.x == 0) {
        unsigned* e = p.flags[p.rank] + 2 * p.world + which;
        *s_epoch = *e + 1;
        *e = *s_epoch;
    }
    __syncthreads();
    return *s_epoch;
}
__device__ __forceinline__ void ep_signal_and_wait(const EpParams& p, int which, unsigned epoch) {
    __threadfence_system();
    __syncthreads();
    if ((int)threadIdx.x < p.world) {
        st_release_sys(p.flags[threadIdx.x] + which * p.world + p.rank, epoch);                   // "rank -> peer threadIdx.x"
        const unsigned* mine = p.flags[p.rank] + which * p.world + threadIdx.x;                     // "peer threadIdx.x -> me"
        while ((int)(ld_acquire_sys(mine) - epoch) < 0) {}
    }
    __syncthreads();
}

__global__ void __launch_bounds__(512) ep_all_gather_kernel(const EpParams p, const void* x_own, float* x_all_f32) {
    __shared__ unsigned s_epoch;
    const unsigned epoch = ep_next_epoch(p, 0, &s_epoch);
    const int row_bytes = p.H * (int)type_size(p.hidden_type);
    const int n16 = row_bytes / 16;
    const uint4* src = reinterpret_cast<const uint4*>(x_own);
    for (int i = threadIdx.x; i < n16 * p.world; i += blockDim.x) {
        const int peer = i / n16, c = i - peer * n16;
        reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(p.tok[peer]) + (size_t)p.rank * row_bytes)[c] = src[c];
    }
    ep_signal_and_wait(p, 0, epoch);
    if (x_all_f32) {
        const void* mine = p.tok[p.rank];
        for (int i = threadIdx.x; i < p.world * p.H; i += blockDim.x) x_all_f32[i] = load_hidden(mine, i, p.hidden_type);
    }
}

__global__ void __launch_bounds__(512) ep_reduce_kernel(const EpParams p, void* y_out, const void* y_shared) {
    __shared__ unsigned s_epoch;
    const unsigned epoch = ep_next_epoch(p, 1, &s_epoch);
    ep_signal_and_wait(p, 1, epoch);     // every rank's partial buffer is complete (written by its previous kernel)
    for (int h = threadIdx.x * 4; h < p.H; h += blockDim.x * 4) {
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int r = 0; r < p.world; r++) {   // rank order: the same sum on every run
            const float4 v = *reinterpret_cast<const float4*>(p.part[r] + (size_t)p.rank * p.H + h);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
        const float a[4] = {acc.x, acc.y, acc.z, acc.w};
#pragma unroll
        for (int i = 0; i < 4; i++) {
            float v = round_hidden(a[i], p.hidden_type);
            if (y_shared) v += load_hidden(y_shared, h + i, p.hidden_type);
            store_hidden(y_out, h + i, p.hidden_type, v);
        }
    }
}

}  // namespace ktb

using namespace ktb;

static int ep_fill(EpParams& p, const ktb200_ep_comm* c) {
    if (!c || c->world < 1 || c->world > kEpMaxWorld || c->rank < 0 || c->rank >= c->world) { set_error("ep: bad rank/world (world <= %d)", kEpMaxWorld); return KTB200_EINVAL; }
    if (c->hidden_size <= 0 || c->hidden_size % 8 || !is_hidden_type(c->hidden_type)) { set_error("ep: hidden_size must be a positive multiple of 8, hidden_type F32/F16/BF16"); return KTB200_EINVAL; }
    p.rank = c->rank; p.world = c->world; p.H = c->hidden_size; p.hidden_type = c->hidden_type;
    for (int r = 0; r < c->world; r++) {
        if (!c->token_bufs[r] || !c->partial_bufs[r] || !c->flag_bufs[r]) { set_error("ep: null peer pointer for rank %d", r); return KTB200_EINVAL; }
        p.tok[r] = c->token_bufs[r]; p.part[r] = c->partial_bufs[r]; p.flags[r] = c->flag_bufs[r];
    }
    return KTB200_OK;
}

extern "C" int ktb200_ep_all_gather_tokens(const ktb200_ep_comm* c, const void* x_own, float* x_all_f32, void* stream) {
    EpParams p{};
    int rc = ep_fill(p, c);
    if (rc) return rc;
    if (!x_own) { set_error("ep: null token"); return KTB200_EINVAL; }
    ep_all_gather_kernel<<<1, 512, 0, (cudaStream_t)stream>>>(p, x_own, x_all_f32);
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

extern "C" int ktb200_ep_reduce_own_token(const ktb200_ep_comm* c, void* y_out, const void* y_shared, void* stream) {
    EpParams p{};
    int rc = ep_fill(p, c);
    if (rc) return rc;
    if (!y_out) { set_error("ep: null output"); return KTB200_EINVAL; }
    ep_reduce_kernel<<<1, 512, 0, (cudaStream_t)stream>>>(p, y_out, y_shared);
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}
