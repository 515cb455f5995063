// Expert-parallel MoE layer for any number of tokens per GPU (prompt chunks through sharded experts over NVLink).
//
// ktb200_moe_ep_forward_tokens (include/ktb200.h) is the EP branch of DeepseekV3MoE.moe_infer
// (archive/ktransformers/models/modeling_deepseek_v3.py:550-605) without its host round trips.  Every rank owns E/world
// experts and holds counts[rank] tokens; counts is the same host array on every rank, so every offset below is known
// everywhere without an exchange.  prefix[s] = counts[0] + .. + counts[s-1].
//
// Per-rank region (ktb200_ep_tokens_layout; R = world * Tmax rows):
//   x     [R][H] hidden type   row prefix[s] + i = token i of source rank s, stored by s only when this rank owns one of
//                              its expert ids, so the gathered rows are one contiguous [sum counts][H] expert input
//   ids   [R][k] int64         same rows, stored by every source into every rank (small)
//   w     [R][k] fp32
//   part  [world][Tmax][H] fp32   part[s][i] = rank s's fp32 routed sum for this rank's token i, stored by s only when s
//                              owns one of the token's ids
//   scratch [min(R, 1024)][H] fp32   local: the shard's expert output of one chunk before it is delivered
//   flags: send[world] | deliver[world] | epoch_send | epoch_deliver | status | arrive_send | arrive_deliver
//
// Phases (phase_mask bits; 7 = the whole layer):
//   1 route + send   gate on the own tokens; ep_tok_send_kernel stores ids / weights everywhere and x rows where they are
//                    needed (16-byte peer stores, one CTA per token); the last CTA to finish bumps epoch_send and releases
//                    send[rank] on every rank.
//   2 experts + deliver   ep_tok_wait_kernel waits for the world send flags; the shard's ordinary expert kernels run on
//                    the gathered rows in place with fp32 output (per-pair kernels below 48 rows / 80 for IQ / 96 for RAWINT4, grouped GEMM above, in
//                    chunks of min(group_max_len, scratch rows)); ep_tok_deliver_kernel stores each needed row into its
//                    owner's part slot; after the last chunk its last CTA bumps epoch_deliver and releases deliver[rank]
//                    on every rank (also when nothing was delivered to that rank).
//   4 combine        first the shared expert on the own tokens (ktb200_mlp_forward, rounded into y_out), then
//                    ep_tok_combine_kernel, on the same stream: it waits for the world deliver flags, adds the part rows of
//                    the owning ranks in rank order, rounds, and adds the shared term: y = round(sum_r part_r) + round(shared).
//
// Buffer reuse across back-to-back layers needs no extra barrier:
//   - rank s stores into rank d's x / ids / w rows for layer L+1 only after its layer-L combine passed, which waited for
//     deliver[d] of layer L; d releases that after its last deliver kernel, which its stream orders after the expert
//     kernels and the deliver kernels, the only readers of those rows.  (The combine reads the routing from the caller's
//     idx_out, never from the message rows, since those may already hold layer L+1.)
//   - rank s stores into owner o's part rows for layer L+1 only after its layer-(L+1) wait passed, which waited for
//     send[o] of layer L+1; o releases that after its layer-L combine, the only reader of its part rows.
//   - every rank releases every flag in every layer, and every wait is for all world flags, so the two arguments hold
//     whatever the routing; the flags are this entry point's own, apart from the one-token kernels' flag blocks.
// Epochs live in the flag words and are advanced by the kernels.  Every wait gives up after 4 s and sets `status`.
#include "common.cuh"
#include "handles.cuh"

namespace ktb {

int moe_forward_f32_out(ktb200_moe* m, int qlen, int k, const int64_t* ids, const float* weights, const void* input, float* output,
                        cudaStream_t s);

constexpr int kTokMaxWorld = 16;
constexpr int kTokScratchRows = 1024;
constexpr int kTokThreads = 256;
constexpr unsigned long long kTokTimeoutNs = 4000000000ull;
enum { kFlagSend = 0, kFlagDeliver = 1 };

struct TokLayout {
    size_t x, ids, w, part, scratch, flags, total;
    long rows, scratch_rows;
};

static TokLayout tok_layout(int world, int tmax, int H, int hidden_type, int k) {
    auto up = [](size_t v) { return (v + 255) & ~(size_t)255; };
    TokLayout L{};
    L.rows = (long)world * tmax;
    L.scratch_rows = L.rows < kTokScratchRows ? L.rows : kTokScratchRows;
    L.x = 0;
    L.ids = up(L.x + (size_t)L.rows * H * type_size(hidden_type));
    L.w = up(L.ids + (size_t)L.rows * k * sizeof(int64_t));
    L.part = up(L.w + (size_t)L.rows * k * sizeof(float));
    L.scratch = up(L.part + (size_t)L.rows * H * sizeof(float));
    L.flags = up(L.scratch + (size_t)L.scratch_rows * H * sizeof(float));
    L.total = up(L.flags + (size_t)(2 * world + 5) * sizeof(unsigned));
    return L;
}

struct TokParams {
    int rank, world, tmax, H, row16, k, per;   // row16: 16-byte words per hidden-type row; per: experts per rank
    int n_experts;
    int prefix[kTokMaxWorld + 1];
    uint8_t* base[kTokMaxWorld];                // every rank's region
    size_t off_x, off_ids, off_w, off_part, off_flags;
};

__device__ __forceinline__ unsigned* tok_flags(const TokParams& p, int r) { return reinterpret_cast<unsigned*>(p.base[r] + p.off_flags); }

__device__ __forceinline__ void tok_st_release_sys(unsigned* a, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(a), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned tok_ld_acquire_sys(const unsigned* a) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(a) : "memory");
    return v;
}
// spin until *a - target >= 0 (wrap-safe); after kTokTimeoutNs give up and set *status
__device__ __forceinline__ void tok_wait_ge(const unsigned* a, unsigned target, unsigned* status) {
    unsigned long long t0 = 0;
    unsigned spins = 0;
    while ((int)(tok_ld_acquire_sys(a) - target) < 0) {
        if ((++spins & 1023u) == 0) {
            unsigned long long t;
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
            if (!t0) t0 = t;
            else if (t - t0 > kTokTimeoutNs) { *status = 1; break; }
        }
    }
}

// bit r set when rank r owns one of the k ids
__device__ __forceinline__ unsigned tok_owner_mask(const int64_t* ids, int k, int per, int n_experts) {
    unsigned m = 0;
    for (int j = 0; j < k; j++) {
        const int64_t e = ids[j];
        if (e >= 0 && e < n_experts) m |= 1u << (int)(e / per);
    }
    return m;
}

// Called by every CTA after its last store of the launch: the CTA that arrives last advances the epoch word `which` and
// releases flag `which` of this rank on every rank.  The fences order every CTA's peer stores before the flag.
__device__ __forceinline__ void tok_arrive_and_release(const TokParams& p, int which) {
    __shared__ int s_last;
    unsigned* mine = tok_flags(p, p.rank);
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        s_last = atomicAdd(mine + 2 * p.world + 3 + which, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __shared__ unsigned s_epoch;
    if (threadIdx.x == 0) {
        mine[2 * p.world + 3 + which] = 0;
        __threadfence_system();
        s_epoch = mine[2 * p.world + which] + 1;
        mine[2 * p.world + which] = s_epoch;
    }
    __syncthreads();
    if ((int)threadIdx.x < p.world) tok_st_release_sys(tok_flags(p, threadIdx.x) + which * p.world + p.rank, s_epoch);
}

// phase 1: one CTA per own token (grid-stride); x goes to the owners of its ids, ids / weights to every rank
__global__ void __launch_bounds__(kTokThreads) ep_tok_send_kernel(const TokParams p, int T, const void* x_own, const int64_t* idx,
                                                                  const float* wts) {
    const int row = p.prefix[p.rank];
    for (int i = blockIdx.x; i < T; i += gridDim.x) {
        const unsigned dest = tok_owner_mask(idx + (long)i * p.k, p.k, p.per, p.n_experts);
        for (int e = threadIdx.x; e < p.world * p.k; e += blockDim.x) {
            const int d = e / p.k, j = e - d * p.k;
            const long o = (long)(row + i) * p.k + j;
            reinterpret_cast<int64_t*>(p.base[d] + p.off_ids)[o] = idx[(long)i * p.k + j];
            reinterpret_cast<float*>(p.base[d] + p.off_w)[o] = wts[(long)i * p.k + j];
        }
        const uint4* src = reinterpret_cast<const uint4*>(x_own) + (long)i * p.row16;
        for (int c = threadIdx.x; c < p.row16; c += blockDim.x) {
            const uint4 v = src[c];
            for (int d = 0; d < p.world; d++)
                if (dest >> d & 1u) reinterpret_cast<uint4*>(p.base[d] + p.off_x)[(long)(row + i) * p.row16 + c] = v;
        }
    }
    tok_arrive_and_release(p, kFlagSend);
}

// phase 2, before the expert kernels: every source's message rows have arrived
__global__ void ep_tok_wait_kernel(const TokParams p) {
    unsigned* mine = tok_flags(p, p.rank);
    if ((int)threadIdx.x < p.world) tok_wait_ge(mine + kFlagSend * p.world + threadIdx.x, mine[2 * p.world + kFlagSend], mine + 2 * p.world + 2);
}

// phase 2, after the expert kernels of gathered rows [g0, g0 + n): row g of the scratch goes to part[rank][i] of its
// source s (g = prefix[s] + i) when this rank owns one of its ids.  `last`: the final chunk, release the deliver flags.
__global__ void __launch_bounds__(kTokThreads) ep_tok_deliver_kernel(const TokParams p, int g0, int n, const float* scratch, int last) {
    const int H4 = p.H / 4;
    const int64_t* ids = reinterpret_cast<const int64_t*>(p.base[p.rank] + p.off_ids);
    for (int j = blockIdx.x; j < n; j += gridDim.x) {
        const int g = g0 + j;
        if (!(tok_owner_mask(ids + (long)g * p.k, p.k, p.per, p.n_experts) >> p.rank & 1u)) continue;
        int s = 0;
        while (g >= p.prefix[s + 1]) s++;
        const int i = g - p.prefix[s];
        float4* dst = reinterpret_cast<float4*>(p.base[s] + p.off_part) + ((long)p.rank * p.tmax + i) * H4;
        const float4* src = reinterpret_cast<const float4*>(scratch) + (long)j * H4;
        for (int c = threadIdx.x; c < H4; c += blockDim.x) dst[c] = src[c];
    }
    if (last) tok_arrive_and_release(p, kFlagDeliver);
}

// phase 4: y[i] = round(sum over owning ranks r, in rank order, of part[r][i]) (+ y[i], the rounded shared term).
// One thread per 4 columns of a row, rows grid-strided; every CTA waits for the world deliver flags first.
__global__ void __launch_bounds__(kTokThreads) ep_tok_combine_kernel(const TokParams p, int T, const int64_t* idx, void* y, int hidden_type,
                                                                     int has_shared) {
    unsigned* mine = tok_flags(p, p.rank);
    if ((int)threadIdx.x < p.world) tok_wait_ge(mine + kFlagDeliver * p.world + threadIdx.x, mine[2 * p.world + kFlagDeliver], mine + 2 * p.world + 2);
    __syncthreads();
    const int H4 = p.H / 4;
    const float4* part = reinterpret_cast<const float4*>(p.base[p.rank] + p.off_part);
    for (long e = (long)blockIdx.x * blockDim.x + threadIdx.x; e < (long)T * H4; e += (long)gridDim.x * blockDim.x) {
        const int i = (int)(e / H4), c = (int)(e - (long)i * H4);
        const unsigned from = tok_owner_mask(idx + (long)i * p.k, p.k, p.per, p.n_experts);
        float a[4] = {0.f, 0.f, 0.f, 0.f};
        for (int r = 0; r < p.world; r++) {
            if (!(from >> r & 1u)) continue;
            const float4 v = part[((long)r * p.tmax + i) * H4 + c];
            a[0] += v.x; a[1] += v.y; a[2] += v.z; a[3] += v.w;
        }
        const long o = (long)i * p.H + 4 * c;
#pragma unroll
        for (int q = 0; q < 4; q++) {
            float v = round_hidden(a[q], hidden_type);
            if (has_shared) v += load_hidden(y, o + q, hidden_type);
            store_hidden(y, o + q, hidden_type, v);
        }
    }
}

}  // namespace ktb

using namespace ktb;

extern "C" long ktb200_ep_tokens_layout(int world, int max_tokens_per_rank, int hidden_size, int hidden_type, int top_k, long* offsets) {
    if (world < 1 || world > kTokMaxWorld || max_tokens_per_rank < 1 || hidden_size <= 0 || hidden_size % 8 || !is_hidden_type(hidden_type) ||
        top_k < 1 || top_k > 32) {
        set_error("ep_tokens_layout: world 1..%d, max_tokens_per_rank >= 1, hidden_size a positive multiple of 8, F32/F16/BF16, top_k 1..32",
                  kTokMaxWorld);
        return -1;
    }
    const TokLayout L = tok_layout(world, max_tokens_per_rank, hidden_size, hidden_type, top_k);
    if (offsets) {
        const size_t o[6] = {L.x, L.ids, L.w, L.part, L.scratch, L.flags};
        for (int i = 0; i < 6; i++) offsets[i] = (long)o[i];
    }
    return (long)L.total;
}

extern "C" int ktb200_moe_ep_forward_tokens(const ktb200_gate_config* gc, ktb200_moe* m, ktb200_mlp* sh, const ktb200_ep_tokens_comm* comm,
                                            const int* counts, const void* x_own, void* y_out, int64_t* idx, float* w, int phase_mask,
                                            void* stream) {
    // communicator and counts first: they need no device
    if (!comm || !counts) { set_error("ep_tokens: null comm or counts"); return KTB200_EINVAL; }
    const int world = comm->world, rank = comm->rank, tmax = comm->max_tokens_per_rank;
    if (world < 1 || world > kTokMaxWorld || rank < 0 || rank >= world) { set_error("ep_tokens: rank %d / world %d (world 1..%d)", rank, world, kTokMaxWorld); return KTB200_EINVAL; }
    if (tmax < 1 || comm->hidden_size <= 0 || comm->hidden_size % 8 || !is_hidden_type(comm->hidden_type) || comm->top_k < 1 || comm->top_k > 32) {
        set_error("ep_tokens: bad comm sizes (max_tokens_per_rank %d, hidden_size %d, hidden_type %d, top_k %d)", tmax, comm->hidden_size,
                  comm->hidden_type, comm->top_k);
        return KTB200_EINVAL;
    }
    if (!comm->bufs) { set_error("ep_tokens: null peer pointer array"); return KTB200_EINVAL; }
    for (int r = 0; r < world; r++) {
        if (!comm->bufs[r]) { set_error("ep_tokens: null peer pointer for rank %d", r); return KTB200_EINVAL; }
        if ((uintptr_t)comm->bufs[r] & 15) { set_error("ep_tokens: the region of rank %d is not 16-byte aligned", r); return KTB200_EINVAL; }
    }
    TokParams p{};
    for (int r = 0; r < world; r++) {
        if (counts[r] < 0 || counts[r] > tmax) { set_error("ep_tokens: counts[%d] = %d outside [0, max_tokens_per_rank = %d]", r, counts[r], tmax); return KTB200_EINVAL; }
        p.prefix[r + 1] = p.prefix[r] + counts[r];
    }
    if (phase_mask < 1 || phase_mask > 7) { set_error("ep_tokens: phase_mask %d (1..7)", phase_mask); return KTB200_EINVAL; }
    const int T = counts[rank], total = p.prefix[world];
    if (T > 0 && (!x_own || !y_out || !idx || !w)) { set_error("ep_tokens: null token / output / routing pointer"); return KTB200_EINVAL; }
    if (T > 0 && ((uintptr_t)x_own & 15)) { set_error("ep_tokens: x_own must be 16-byte aligned (it is read in 16-byte words)"); return KTB200_EINVAL; }
    if (!gc || !m) { set_error("ep_tokens: null gate config or expert handle"); return KTB200_EINVAL; }
    if (!m->loaded || (sh && !sh->loaded)) { set_error("Not Loaded"); return KTB200_ESTATE; }
    const ktb200_moe_config& c = m->cfg;
    const int H = c.hidden_size, k = gc->top_k;
    if (gc->hidden_size != H || gc->hidden_type != c.hidden_type || comm->hidden_size != H || comm->hidden_type != c.hidden_type ||
        (sh && (sh->H != H || sh->hidden_type != c.hidden_type))) {
        set_error("ep_tokens: gate / experts / shared expert / comm disagree on the hidden size or type");
        return KTB200_EINVAL;
    }
    if (k != comm->top_k || k > c.routed_expert_num) { set_error("ep_tokens: top_k %d (comm %d, experts handle %d)", k, comm->top_k, c.routed_expert_num); return KTB200_EINVAL; }
    if ((long)c.expert_num * world != gc->n_experts || c.expert_id_offset != rank * c.expert_num) {
        set_error("ep_tokens: the experts handle must own ids [%d, %d) of %d (expert_num %d, offset %d)", rank * c.expert_num,
                  (rank + 1) * c.expert_num, gc->n_experts, c.expert_num, c.expert_id_offset);
        return KTB200_EINVAL;
    }
    if (c.group_max_len < 1 || (sh && sh->group_max_len < 1)) { set_error("ep_tokens: group_max_len must be positive"); return KTB200_EINVAL; }

    const TokLayout L = tok_layout(world, tmax, H, c.hidden_type, k);
    p.rank = rank; p.world = world; p.tmax = tmax; p.H = H; p.k = k; p.per = c.expert_num; p.n_experts = gc->n_experts;
    p.row16 = (int)((size_t)H * type_size(c.hidden_type) / 16);
    p.off_x = L.x; p.off_ids = L.ids; p.off_w = L.w; p.off_part = L.part; p.off_flags = L.flags;
    for (int r = 0; r < world; r++) p.base[r] = reinterpret_cast<uint8_t*>(comm->bufs[r]);
    uint8_t* mine = p.base[rank];
    DeviceGuard guard(m->device);
    cudaStream_t s = (cudaStream_t)stream;
    const int sms = num_sms(m->device);

    if (phase_mask & 1) {
        if (T > 0) {
            int rc = ktb200_moe_gate_forward(gc, T, x_own, idx, w, nullptr, nullptr, stream);
            if (rc) return rc;
        }
        const int grid = T < 1 ? 1 : (T < 2 * sms ? T : 2 * sms);
        ep_tok_send_kernel<<<grid, kTokThreads, 0, s>>>(p, T, x_own, idx, w);
        KTB_LAUNCH_CHECK();
    }
    if (phase_mask & 2) {
        ep_tok_wait_kernel<<<1, 32, 0, s>>>(p);
        KTB_LAUNCH_CHECK();
        const long chunk = c.group_max_len < L.scratch_rows ? c.group_max_len : L.scratch_rows;
        float* scratch = reinterpret_cast<float*>(mine + L.scratch);
        const int64_t* ids = reinterpret_cast<const int64_t*>(mine + L.ids);
        const float* wts = reinterpret_cast<const float*>(mine + L.w);
        const size_t hb = type_size(c.hidden_type);
        int g0 = 0;
        do {
            const int n = total - g0 < chunk ? total - g0 : (int)chunk;
            if (n > 0) {
                int rc = moe_forward_f32_out(m, n, k, ids + (size_t)g0 * k, wts + (size_t)g0 * k, mine + L.x + (size_t)g0 * H * hb, scratch, s);
                if (rc) return rc;
            }
            const int last = g0 + n >= total;
            const int grid = n < 1 ? 1 : (n < 2 * sms ? n : 2 * sms);
            ep_tok_deliver_kernel<<<grid, kTokThreads, 0, s>>>(p, g0, n, scratch, last);
            KTB_LAUNCH_CHECK();
            g0 += n;
        } while (g0 < total);
    }
    if (phase_mask & 4) {
        for (int t0 = 0; sh && t0 < T; t0 += sh->group_max_len) {
            const int n = T - t0 < sh->group_max_len ? T - t0 : sh->group_max_len;
            const size_t o = (size_t)t0 * H * type_size(c.hidden_type);
            int rc = ktb200_mlp_forward(sh, n, reinterpret_cast<const uint8_t*>(x_own) + o, reinterpret_cast<uint8_t*>(y_out) + o, 0, nullptr, stream);
            if (rc) return rc;
        }
        long grid = ((long)T * (H / 4) + kTokThreads - 1) / kTokThreads;
        if (grid > 4L * sms) grid = 4L * sms;
        if (grid < 1) grid = 1;
        ep_tok_combine_kernel<<<(unsigned)grid, kTokThreads, 0, s>>>(p, T, idx, y_out, c.hidden_type, sh ? 1 : 0);
        KTB_LAUNCH_CHECK();
    }
    return KTB200_OK;
}
