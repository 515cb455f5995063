// The whole MoE block of one decoder layer in ONE persistent launch:
//     router GEMV + grouped top-k  ->  gate/up of the selected (and the shared) experts  ->  down + weighted combine
// Replaces KDeepseekV3MoE.forward (archive/ktransformers/operators/experts.py:972-1012): `topk_idx, topk_weight =
// self.gate(x)` (models/modeling_deepseek_v3.py:430-481), `y = self.experts(x, topk_idx, topk_weight)` (the CPU MOE,
// operators/llamafile/moe.cpp:146-245) and `y += self.shared_experts(identity)`.
//
// Why one kernel: a launch that streams ~100-150 MB pays a fixed cost (launch gap, pipeline ramp, activation prologue,
// tail) on top of the time its bytes take at the sustained rate (profiles/probe_bulk.py measures both for the bare copy
// ring).  Three launches per layer pay that three times.  Here one CTA per SM (cooperative launch, 12 warps, 168
// registers) stays resident for the whole layer.  One grid-wide barrier separates the router from the top-k; gate/up
// hands its output to down through per-Q8_K-block readiness instead.  What overlaps what was decided with
// profiles/block_trace.py (%globaltimer at the phase boundaries of every CTA):
//   * the barrier is split into arrive / wait; the shared expert's first rows are requested in between, never before
//     the arrive: a fence issued with bulk copies in flight waits for them (measured again on H100: one gpu-scope fence
//     per CTA and Q8_K block inside the gate/up stream cost ~10 us per layer);
//   * x is quantised under the barrier (the router reads x itself); the shared expert's gate/up rows are consumed by
//     warps 4.. while warps 0..3 run the top-k;
//   * gate/up is entry-major: every CTA computes a slice of every entry, in work-list order, so the entries complete
//     one after another across the grid.  The producers only store (`inter` starts out as kInterEmpty: a consumer sees
//     each value arrive, no fence or count is needed).  Each Q8_K block is quantised once, by the first CTA to claim
//     it, into a global staging buffer; a CTA's down tiles of entry j start as soon as entry j is staged, while other
//     CTAs may still be computing later entries.  The claims and their fences run on one warp per CTA that streams no
//     down tiles;
//   * the selection runs redundantly in every CTA (128 threads, from the same partial sums in the same order): no
//     second barrier and no global round trip for the ids;
//   * programmatic dependent launch: the router's weight loads are issued before griddepcontrol.wait, so the next
//     layer's launch latency and first DRAM round trip hide under this layer's tail.
//
// Arithmetic, summation orders and rounding are exactly those of the separate kernels (gate.cuh, gemv_bulk.cuh):
// the fused launch is bit-identical to ktb200_moe_gate_forward + ktb200_moe_forward_shared (tests/test_gpu_parity.py).
#include <cstdlib>

#include "gate.cuh"
#include "gemv_bulk.cuh"
#include "handles.cuh"

namespace ktb {

constexpr int kBlockWarps = 15;    // 480 threads -> 128 registers; 15 x 13440-byte rings + staging = 227 KB
constexpr int kBlockWarpsLo = 12;  // 384 threads -> 168 registers (KTB200_BLK_WARPS <= 12)

struct BlockParams {
    GateParams g;                        // router (W, bias, partial scratch, idx / w / logits outputs, x)
    const void *w_gate, *w_up, *w_down;  // routed experts [n_local][...]
    const void *s_gate, *s_up, *s_down;  // shared expert (null: none)
    int n_local, id_offset;              // this shard owns expert ids [id_offset, id_offset + n_local)
    int H, I, k;
    int hidden_type, use_silu;
    float* inter;                        // [T][ns][I] fp32 (moe_block_kernel: kInterEmpty where not written yet)
    void* out;                           // [T][H]
    unsigned* sync;                      // [0] barrier counter, [1] exit counter; both zero between launches
    // moe_block_kernel: ready[(t * ns + slot) * nb + b] of Q8_K block b of `inter`: 1 = a CTA is quantising it into the
    // stage_* buffers, 2 = staged; zero between launches
    unsigned* ready;
    unsigned* status;                    // set to 1 when a readiness wait timed out (the results of that launch are invalid)
    uint8_t* stage_q;                    // [T][ns][nb][QK_K] int8 quants, same values as the shared-memory `aq` staging
    int16_t* stage_bs;                   // [T][ns][nb][KBS] block sums (`abs_`)
    float* stage_d;                      // [T][ns][nb] scales (`adx`)
    int nrows_max;                       // output rows per CTA (stride of the `partial` staging)
    int region_a;                        // bytes of the aliased activation staging
    int ring_bytes;                      // per-warp ring
    int prime_u, prime_d;                // rows / tiles every warp requests BEFORE the router's / the second grid barrier (EP)
    unsigned long long* trace;           // debug: [grid][16] globaltimer stamps of the phase boundaries (null: off)
    const uint8_t* pf[3];                // ranges to pull into L2 while the down phase streams (the NEXT layer's router rows and
    unsigned pf_bytes[3];                // shared-expert gate/up rows: ktb200_moe_block_prefetch_hint); null: none
};

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned ld_acquire_sys_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long ep_now() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
constexpr unsigned long long kEpTimeoutNs = 4000000000ull;
// spin until *p - target >= 0 (wrap-safe), acquiring at system (peer memory) or GPU scope; gives up after kEpTimeoutNs
// and records it in `status`
template <bool SYS>
__device__ __forceinline__ void wait_ge(const unsigned* p, unsigned target, unsigned* status) {
    unsigned long long t0 = 0;
    unsigned spins = 0;
    while ((int)((SYS ? ld_acquire_sys_u32(p) : ld_acquire_u32(p)) - target) < 0) {
        if ((++spins & 1023u) == 0) {
            const unsigned long long t = ep_now();
            if (!t0) t0 = t;
            else if (t - t0 > kEpTimeoutNs) { *status = 1; break; }
        }
    }
}

// Grid-wide barrier over the (co-resident) CTAs, split in two so that work which does not depend on the other CTAs —
// here: requesting the next phase's weights — can be issued in between.  `gen` counts the barriers passed.  The arrive
// side fences BEFORE any of those requests exist (a fence issued with bulk copies in flight waits for them: measured).
__device__ __forceinline__ void grid_arrive(unsigned* counter, unsigned& gen) {
    __syncthreads();
    gen++;
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(counter, 1u);
    }
}
__device__ __forceinline__ void grid_wait(unsigned* counter, unsigned gen) {
    if (threadIdx.x == 0) {
        const unsigned target = gen * gridDim.x;
        while (ld_acquire_u32(counter) < target) {}
    }
    __syncthreads();
}

// Programmatic dependent launch: the next layer's launch is processed, and its CTAs start on SMs as they free up,
// while the tail of this one still runs; everything that depends on the previous kernel comes after griddep_wait().

__device__ __forceinline__ void trace_stamp(const BlockParams& p, int i) {   // from the calling thread
    if (p.trace) p.trace[blockIdx.x * 16 + i] = ep_now();
}
__device__ __forceinline__ void block_stamp(const BlockParams& p, int i) {
    if (threadIdx.x == 0) trace_stamp(p, i);
}

__device__ __forceinline__ float4 load_x4(const void* x, long i4, int type) {
    if (type == KTB200_TYPE_F32) return reinterpret_cast<const float4*>(x)[i4];
    const uint2 v = reinterpret_cast<const uint2*>(x)[i4];
    if (type == KTB200_TYPE_BF16)
        return make_float4(__uint_as_float(v.x << 16), __uint_as_float(v.x & 0xffff0000u), __uint_as_float(v.y << 16),
                           __uint_as_float(v.y & 0xffff0000u));
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&v.x)), b = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
    return make_float4(a.x, a.y, b.x, b.y);
}

// ---------------------------------------------------------------------------------------------------------------
// Shared-memory layout (dynamic):
//   [BlockShared]  ids / weights / work list of the current token
//   [region A]     aliased over the phases:  {x int8 staging | selection scratch}  then  {a int8 staging}
//   [partial]      [nrows_max][ns] fp32 down results before the weighted combine
//   [mbarriers]    W x 3
//   [rings]        W x ring_bytes   (3 gate/up rows or 2 down tiles per warp)
struct BlockShared {
    BlockParams prm;   // the launch parameters, copied once: the cold phases read them with LDS instead of going through
                       // a pointer to the kernel-parameter space after every barrier
    int64_t ids[32];
    float w[32];
    int vs[36];      // work list: slot indices this shard computes (the shared expert, slot k, first)
    int nv;
    unsigned skip;   // bit j: routed slot j is not owned by this shard
    int ent_state[36];   // down: 0 = entry i's `a` not in shared memory, 1 = a warp is copying it, 2 = there
    int last_cta;        // this CTA is the last to leave the launch: it zeroes the barrier and readiness words
};
constexpr int kBlockSharedBytes = (sizeof(BlockShared) + 15) & ~15;

struct BlockLay {
    uint8_t *xq, *aq;
    int16_t *xbs, *abs_;
    float *xdx, *adx, *sel, *partial;
    size_t ring_off;   // mbarriers, then the rings
};
template <int KBS>
__device__ __forceinline__ BlockLay block_layout(const BlockParams& p, uint8_t* smem) {
    const int nblk = p.H / QK_K, nb = p.I / QK_K, ns = p.k + (p.s_gate ? 1 : 0);
    uint8_t* a = smem + kBlockSharedBytes;
    BlockLay L;
    L.xq = a;
    L.xbs = reinterpret_cast<int16_t*>(a + (size_t)nblk * kActBlkStride);
    L.xdx = reinterpret_cast<float*>(a + (size_t)nblk * (kActBlkStride + 16));
    L.sel = reinterpret_cast<float*>(a + (((size_t)nblk * (kActBlkStride + 16 + 4) + 15) & ~(size_t)15));
    L.aq = a;
    L.abs_ = reinterpret_cast<int16_t*>(a + (size_t)ns * nb * kActBlkStride);
    L.adx = reinterpret_cast<float*>(a + (size_t)ns * nb * (kActBlkStride + 2 * KBS));
    L.partial = reinterpret_cast<float*>(a + p.region_a);
    L.ring_off = ((size_t)kBlockSharedBytes + p.region_a + (size_t)p.nrows_max * ns * 4 + 15) & ~(size_t)15;
    return L;
}

// ---- the phases around the two streaming loops, once per token --------------------------------------------------
// x -> Q8_K (padded staging)
__device__ __forceinline__ void blk_quantize_x(int t) {
    extern __shared__ __align__(16) uint8_t smem[];
    const BlockParams& p = reinterpret_cast<const BlockShared*>(smem)->prm;
    const BlockLay L = block_layout<8>(p, smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5, nblk = p.H / QK_K;
    // one block per warp and iteration, the next block's load already in flight (rolled: one copy of the quantiser)
    float cur[8], nxt[8];
    int b = warp;
    if (b < nblk) load_block8(p.g.x, (long)t * p.H + (long)b * QK_K + lane * 8, p.hidden_type, cur);
#pragma unroll 1
    while (b < nblk) {
        const int bn = b + W;
        if (bn < nblk) load_block8(p.g.x, (long)t * p.H + (long)bn * QK_K + lane * 8, p.hidden_type, nxt);
        warp_quantize_q8k_block(cur, lane, reinterpret_cast<uint32_t*>(L.xq + (size_t)b * kActBlkStride), L.xdx + b, nullptr, L.xbs + b * 8);
#pragma unroll
        for (int i = 0; i < 8; i++) cur[i] = nxt[i];
        b = bn;
    }
}

// router partial sums: unit = (expert row e, column split s); same loop and summation order as gate_dot<1> (gate.cuh)
// `waited`: whether this thread already passed griddep_wait() — the router's WEIGHT loads are issued before it (they do
// not depend on the previous kernel), x is read after it.
__device__ __forceinline__ void blk_router(int t, bool& waited) {
    extern __shared__ __align__(16) uint8_t smem[];
    const BlockParams& p = reinterpret_cast<const BlockShared*>(smem)->prm;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    const int E = p.g.E, S = p.g.S, n4 = p.H / 4;
    const int gw = blockIdx.x * W + warp, tw = gridDim.x * W;
    for (int u = gw; u < E * S; u += tw) {
        const int s = u / E, e = u - s * E;
        const int c0 = (int)((long)n4 * s / S), nc4 = (int)((long)n4 * (s + 1) / S) - c0;
        const float4* wrow = reinterpret_cast<const float4*>(p.g.W + (long)e * p.H) + c0;
        const long xbase = (long)t * n4 + c0;
        float acc = 0.f;
        constexpr int NQ = 10;   // float4 in flight per lane: one batch covers H/S up to 1280 columns
        for (int cb = lane; cb < nc4; cb += 32 * NQ) {
            float4 w[NQ], xv[NQ];
#pragma unroll
            for (int q = 0; q < NQ; q++) {
                const int c = cb + 32 * q;
                if (c < nc4) w[q] = __ldg(wrow + c);
            }
            if (!waited) { griddep_wait(); waited = true; }
#pragma unroll
            for (int q = 0; q < NQ; q++) {
                const int c = cb + 32 * q;
                if (c < nc4) xv[q] = load_x4(p.g.x, xbase + c, p.hidden_type);
            }
#pragma unroll
            for (int q = 0; q < NQ; q++) {
                const int c = cb + 32 * q;
                if (c < nc4) {
                    acc = fmaf(w[q].x, xv[q].x, acc);
                    acc = fmaf(w[q].y, xv[q].y, acc);
                    acc = fmaf(w[q].z, xv[q].z, acc);
                    acc = fmaf(w[q].w, xv[q].w, acc);
                }
            }
        }
        const float v = warp_sum(acc);
        if (lane == 0) p.g.partial[((long)t * S + s) * E + e] = v;
    }
    if (!waited) { griddep_wait(); waited = true; }
}

// top-k selection (first 4 warps of EVERY CTA, identical results), work-list compaction, routing outputs (CTA 0)
__device__ __forceinline__ void blk_select(int t) {
    extern __shared__ __align__(16) uint8_t smem[];
    BlockShared& sh = *reinterpret_cast<BlockShared*>(smem);
    const BlockParams& p = sh.prm;
    const BlockLay L = block_layout<8>(p, smem);
    const int k = p.k;
    if ((threadIdx.x >> 5) < kGateWarps) {
        gate_select_token<1>(p.g, t, L.sel, sh.ids, sh.w, blockIdx.x == 0 ? p.g.logits_out : nullptr);
    }
    __syncthreads();
    block_stamp(p, 10);
    if (threadIdx.x == 0) {
        unsigned sk = 0;
        int nv = p.s_gate ? 1 : 0;
        for (int j = 0; j < k; j++) {
            const long e = (long)sh.ids[j] - p.id_offset;
            if (e < 0 || e >= p.n_local) sk |= 1u << j; else sh.vs[nv++] = j;
        }
        sh.nv = nv;
        sh.skip = sk;
    }
    if (blockIdx.x == 0 && threadIdx.x < k) {
        p.g.idx[(long)t * k + threadIdx.x] = sh.ids[threadIdx.x];
        p.g.w[(long)t * k + threadIdx.x] = sh.w[threadIdx.x];
    }
    __syncthreads();
}

// Rows of entry `ie` (index into the work list) this CTA computes in gate/up: slice (blockIdx + ie) mod G of the G equal
// slices of I.  Rotating the slice per entry keeps every CTA's total within one row of I * entries / G.
__device__ __forceinline__ void entry_slice(int I, int ie, int& r0, int& len) {
    const unsigned s = (blockIdx.x + (unsigned)ie) % gridDim.x;
    r0 = (int)((unsigned long long)I * s / gridDim.x);
    len = (int)((unsigned long long)I * (s + 1) / gridDim.x) - r0;
}

// `inter` of the block kernel (ktb200_moe::blk_inter) holds kInterEmpty wherever gate/up has not stored a value yet: a
// consumer sees each value arrive on its own, so the producers store without any fence or count.  The bits are a NaN
// that arithmetic never produces (a NaN result is the canonical 0x7fffffff).
constexpr unsigned kInterEmpty = 0xffffffffu;
__device__ __forceinline__ void st_relaxed_f32(float* p, float v) {
    asm volatile("st.relaxed.gpu.global.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}
__device__ __forceinline__ uint4 ld_relaxed_u4(const void* p) {
    uint4 v;
    asm volatile("ld.relaxed.gpu.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}

// Q8_K block `gb` (readiness word index), already claimed by this warp (ready 0 -> 1): wait until its QK_K values in
// `src` have all arrived, quantise them in exactly the layout of the shared-memory staging, empty them again for the next
// launch and publish the result (ready 2).  Whole warp.
template <int KBS>
__device__ __forceinline__ void quantise_block(const BlockParams& p, long gb, float* src) {
    const int lane = threadIdx.x & 31;
    uint4 v0, v1;
    unsigned long long t0 = 0;
    for (unsigned spins = 1;; spins++) {
        v0 = ld_relaxed_u4(src + lane * 8);
        v1 = ld_relaxed_u4(src + lane * 8 + 4);
        const bool here = v0.x != kInterEmpty && v0.y != kInterEmpty && v0.z != kInterEmpty && v0.w != kInterEmpty &&
                          v1.x != kInterEmpty && v1.y != kInterEmpty && v1.z != kInterEmpty && v1.w != kInterEmpty;
        if (__all_sync(0xffffffffu, here)) break;
        if ((spins & 255u) == 0) {   // bounded like wait_ge
            const unsigned long long t = ep_now();
            if (!t0) t0 = t;
            else if (t - t0 > kEpTimeoutNs) { if (lane == 0) *p.status = 1; break; }
        }
    }
    const float x[8] = {__uint_as_float(v0.x), __uint_as_float(v0.y), __uint_as_float(v0.z), __uint_as_float(v0.w),
                        __uint_as_float(v1.x), __uint_as_float(v1.y), __uint_as_float(v1.z), __uint_as_float(v1.w)};
    warp_quantize_q8k_block(x, lane, reinterpret_cast<uint32_t*>(p.stage_q + gb * QK_K), p.stage_d + gb,
                            KBS == 16 ? p.stage_bs + gb * 16 : nullptr, KBS == 8 ? p.stage_bs + gb * 8 : nullptr);
    const uint4 empty = make_uint4(kInterEmpty, kInterEmpty, kInterEmpty, kInterEmpty);
    reinterpret_cast<uint4*>(src + lane * 8)[0] = empty;
    reinterpret_cast<uint4*>(src + lane * 8)[1] = empty;
    __syncwarp();
    if (lane == 0) {
        __threadfence();
        atomicExch(p.ready + gb, 2u);
    }
}

// Every Q8_K block of (token t, slot) is quantised once per launch, by whichever CTA claims it first.  The warp claims the
// blocks no CTA has claimed yet, one at a time, preferring a different block in every CTA so that the CTAs arriving
// together quantise the blocks of an entry in parallel.  Returns when every block is claimed.  Whole warp.
template <int KBS>
__device__ __forceinline__ void claim_entry(const BlockParams& p, int t, int slot) {
    const int lane = threadIdx.x & 31, ns = p.k + (p.s_gate ? 1 : 0), nb = p.I / QK_K;
    const long g0 = ((long)t * ns + slot) * nb;
    for (int c0 = 0; c0 < nb; c0 += 32) {
        const int nc = min(32, nb - c0), rot = (int)(blockIdx.x % nc);
        for (;;) {
            const unsigned fr = __ballot_sync(0xffffffffu, lane < nc && ld_acquire_u32(p.ready + g0 + c0 + lane) == 0u);
            if (!fr) break;
            const unsigned pref = fr & (~0u << rot);
            const int b = c0 + __ffs(pref ? pref : fr) - 1;
            unsigned won = 0;
            if (lane == 0) won = atomicCAS(p.ready + g0 + b, 0u, 1u) == 0u;
            if (__shfl_sync(0xffffffffu, won, 0)) quantise_block<KBS>(p, g0 + b, p.inter + ((long)t * ns + slot) * p.I + (long)b * QK_K);
        }
    }
}

// Down: entry `ev`'s quantised `a` must be in region A before the first tile of it.  The first warp of the CTA to get here
// waits until every block of the entry is staged and copies it (plain L2 loads: the staging was written in this
// launch); with `need`, a warp that finds another warp doing it waits for that warp, without it returns at once (a
// look-ahead).  Whole warp.
template <int KBS>
__device__ __forceinline__ void entry_to_smem(BlockShared& sh, const BlockLay& L, int t, int ev, bool need) {
    const BlockParams& p = sh.prm;
    const int lane = threadIdx.x & 31;
    volatile int* state = &sh.ent_state[ev];
    int s = lane == 0 ? *state : 0;
    s = __shfl_sync(0xffffffffu, s, 0);
    if (s == 0) {
        if (lane == 0) s = atomicCAS(&sh.ent_state[ev], 0, 1) == 0 ? 3 : 1;
        s = __shfl_sync(0xffffffffu, s, 0);
    }
    if (s == 3) {   // this warp claimed the copy
        const int nb = p.I / QK_K, slot = sh.vs[ev];
        const long g0 = ((long)t * (p.k + (p.s_gate ? 1 : 0)) + slot) * nb;
        for (int b = lane; b < nb; b += 32) wait_ge<false>(p.ready + g0 + b, 2u, p.status);
        __syncwarp();
        const uint4* q = reinterpret_cast<const uint4*>(p.stage_q + g0 * QK_K);
        for (int i = lane; i < nb * (QK_K / 16); i += 32)
            *reinterpret_cast<uint4*>(L.aq + (size_t)(slot * nb + i / (QK_K / 16)) * kActBlkStride + (i % (QK_K / 16)) * 16) = __ldcg(q + i);
        const uint4* bs = reinterpret_cast<const uint4*>(p.stage_bs + g0 * KBS);
        for (int i = lane; i < nb * KBS / 8; i += 32) reinterpret_cast<uint4*>(L.abs_ + slot * nb * KBS)[i] = __ldcg(bs + i);
        for (int i = lane; i < nb; i += 32) L.adx[slot * nb + i] = __ldcg(p.stage_d + g0 + i);
        __syncwarp();
        if (lane == 0) {
            __threadfence_block();
            *state = 2;
            if (ev == 0) trace_stamp(p, 6);
            if (ev == sh.nv - 1) trace_stamp(p, 7);
        }
    } else if (s == 1 && need && lane == 0) {
        while (*state != 2) {}   // bounded: the copying warp's own waits are
    }
    if (lane == 0) __threadfence_block();
    __syncwarp();
}

// weighted accumulation over the k experts IN expert_ids ORDER (moe.cpp:222-236), one FMA per expert; then the
// shared expert as a second rounded term (experts.py:1011)
template <int KBS>
__device__ __forceinline__ void blk_combine(int t) {
    extern __shared__ __align__(16) uint8_t smem[];
    const BlockShared& sh = *reinterpret_cast<const BlockShared*>(smem);
    const BlockParams& p = sh.prm;
    const BlockLay L = block_layout<KBS>(p, smem);
    const int k = p.k, ns = k + (p.s_gate ? 1 : 0);
    const int quads = p.H / 4;
    const int q0 = (int)((long)quads * blockIdx.x / gridDim.x), nrows = ((int)((long)quads * (blockIdx.x + 1) / gridDim.x) - q0) * 4;
    const unsigned skip = sh.skip;
    for (int hl = threadIdx.x; hl < nrows; hl += blockDim.x) {
        float acc = 0.f;
        for (int j = 0; j < k; j++) {
            if ((skip >> j) & 1u) continue;
            acc = __fmaf_rn(L.partial[hl * ns + j], sh.w[j], acc);
        }
        if (p.s_gate) acc = round_hidden(acc, p.hidden_type) + round_hidden(L.partial[hl * ns + k], p.hidden_type);
        store_hidden(p.out, (long)t * p.H + q0 * 4 + hl, p.hidden_type, acc);
    }
}

template <class DownFmt, int MAXW>
__global__ void __launch_bounds__(MAXW * 32, 1) moe_block_kernel(const BlockParams p) {
    // rows per down tile; ring depth in rows (gate/up: 4 with 12 warps, 3 with 15) and in tiles (down)
    constexpr int RW = 4, SU = MAXW <= kBlockWarpsLo ? 4 : 3, SD = 2;
    extern __shared__ __align__(16) uint8_t smem[];
    BlockShared& sh = *reinterpret_cast<BlockShared*>(smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    griddep_launch_dependents();
    bool waited = false;
    int Teff = p.g.T;
    if (p.g.bsz) { griddep_wait(); waited = true; Teff = min(Teff, *p.g.bsz); }   // a device-side batch size is an input too
    const int k = p.k;
    const bool has_shared = p.s_gate != nullptr;
    uint32_t bar_u32, ring_u32;
    {
        const BlockLay L = block_layout<DownFmt::kBs>(p, smem);
        const int bar_bytes = (W * SU * 8 + 15) & ~15;
        bar_u32 = (uint32_t)__cvta_generic_to_shared(smem + L.ring_off) + warp * SU * 8;
        ring_u32 = (uint32_t)__cvta_generic_to_shared(smem + L.ring_off + bar_bytes) + warp * p.ring_bytes;
    }
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < SU; s++) mbar_init(bar_u32 + 8 * s, 1);
        mbar_fence_init();
        fence_proxy_async_smem();
    }
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&p);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&sh.prm);
        for (int i = threadIdx.x; i < (int)(sizeof(BlockParams) / 4); i += blockDim.x) dst[i] = src[i];
    }
    if (threadIdx.x == 0 && has_shared) sh.vs[0] = k;   // the shared expert is always the first entry of the work list
    uint32_t phase = 0;   // bit s = parity the next use of barrier s waits for
    unsigned gen = 0;
    block_stamp(p, 0);

  for (int t = 0; t < Teff; t++) {
    __syncthreads();   // previous token: region A, partial and the work list are free (first token: barriers initialised)
    {
        // ------------------------------------------------------------ gate/up
        // A warp walks a list of units (work-list entry, row) — 2 weight rows (gate, up) each.  A CTA computes one slice of
        // every entry (entry_slice); its list is the concatenation of those slices in entry order.  Two lists per token:
        //   S: the shared expert (entry 0), its slice walked by warps 4.. WHILE warps 0..3 run the top-k (the shared
        //      expert needs no routing);
        //   R: the routed entries, all warps, dealt round-robin.  Every CTA walks the entries in the same order, so they
        //      complete one after another across the grid and the down phase can start on the first while the last are
        //      still being computed.
        const int nblk = p.H / QK_K, row_bytes = nblk * SZ_Q4_K;
        const int ns = k + (has_shared ? 1 : 0);
        int ie = 0, ir = 0, ir0 = 0, ilen = 0, ileft = 0, isub = 0;   // issue cursor (entry, row, its slice), units left to request, rows requested
        int ce = 0, cr = 0, cr0 = 0, clen = 0, cleft = 0, csub = 0;   // consume cursor, units left to finish, rows consumed
        int stride = W, iend = 1;
        int slot_i = 0, slot_u = 0;
        auto advance = [&](int& e, int& r, int& r0, int& len, int n) {   // n units further along the list
            int off = r - r0 + n;
            while (off >= len && e + 1 < iend) { off -= len; e++; entry_slice(p.I, e, r0, len); }
            r = r0 + off;
        };
        auto start_list = [&](int e0, int e1, int first, int count, int stride_) {   // entries [e0, e1), from unit `first`
            iend = e1;
            ie = e0;
            entry_slice(p.I, e0, ir0, ilen);
            ir = ir0;
            advance(ie, ir, ir0, ilen, first);
            ce = ie; cr = ir; cr0 = ir0; clen = ilen;
            ileft = cleft = count > 0 ? count : 0;
            stride = stride_;
        };
        auto issue_u = [&]() {
            if (ileft > 0 && isub - csub < SU) {
                if (lane == 0) {
                    const int s = sh.vs[ie];
                    const bool second = isub & 1;
                    const uint8_t* src;
                    if (s == k) {
                        src = reinterpret_cast<const uint8_t*>(second ? p.s_up : p.s_gate) + (long)ir * row_bytes;
                    } else {
                        const long e = (long)sh.ids[s] - p.id_offset;
                        src = reinterpret_cast<const uint8_t*>(second ? p.w_up : p.w_gate) + (e * p.I + ir) * row_bytes;
                    }
                    const uint32_t bar = bar_u32 + 8 * slot_i;
                    mbar_expect_tx(bar, (uint32_t)row_bytes);
                    bulk_g2s(ring_u32 + slot_i * row_bytes, src, (uint32_t)row_bytes, bar);
                }
                isub++;
                if (!(isub & 1)) {
                    ileft--;
                    advance(ie, ir, ir0, ilen, stride);
                }
                slot_i = (slot_i + 1 == SU) ? 0 : slot_i + 1;
            }
        };
        if (threadIdx.x < 36) sh.ent_state[threadIdx.x] = 0;
        blk_router(t, waited);
        block_stamp(p, 2);
        grid_arrive(p.sync, gen);
        // while the barrier completes: request the shared expert's first rows, then quantise x (the router read x itself)
        if (has_shared && warp >= kGateWarps) {
            int r0, nr;
            entry_slice(p.I, 0, r0, nr);
            const int first = warp - kGateWarps, st = W - kGateWarps;
            start_list(0, 1, first, (nr - first + st - 1) / st, st);
        }
#pragma unroll
        for (int s = 0; s < SU; s++)
            if (s < p.prime_u) issue_u();
        blk_quantize_x(t);
        block_stamp(p, 1);
        grid_wait(p.sync, gen);
        block_stamp(p, 3);
        const BlockLay L = block_layout<DownFmt::kBs>(p, smem);
        const uint8_t* ring = smem + (ring_u32 - (uint32_t)__cvta_generic_to_shared(smem));
#pragma unroll 1
        for (int list = 0; list < 2; list++) {
            if (list == 1) {
                // list 0 (the shared expert) was consumed by warps 4.. while warps 0..3 run the top-k now
                blk_select(t);
                block_stamp(p, 4);
                const int e0 = has_shared ? 1 : 0, nv = sh.nv;
                int total = 0;
                for (int e = e0; e < nv; e++) {
                    int r0, len;
                    entry_slice(p.I, e, r0, len);
                    total += len;
                }
                start_list(e0, nv, warp, (total - warp + W - 1) / W, W);
#pragma unroll
                for (int s = 0; s < SU; s++) issue_u();
            }
            float acc_first = 0.f;
            while (cleft > 0) {
                mbar_wait(bar_u32 + 8 * slot_u, (phase >> slot_u) & 1u);
                phase ^= 1u << slot_u;
                const uint8_t* row0 = ring + slot_u * row_bytes;
                float acc = 0.f;
                if (lane < nblk)
                    acc = q4k_block_dot(row0 + lane * SZ_Q4_K, L.xq + (size_t)lane * kActBlkStride,
                                        *reinterpret_cast<const uint4*>(L.xbs + lane * 8), L.xdx[lane]);
                __syncwarp();
                slot_u = (slot_u + 1 == SU) ? 0 : slot_u + 1;
                csub++;
                issue_u();
                if (csub & 1) { acc_first = acc; continue; }
                float g = acc_first, uu = acc;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    g += __shfl_xor_sync(0xffffffffu, g, o);
                    uu += __shfl_xor_sync(0xffffffffu, uu, o);
                }
                if (lane == 0) st_relaxed_f32(p.inter + ((long)t * ns + sh.vs[ce]) * p.I + cr, (p.use_silu ? act_silu(g) : act_relu(g)) * uu);
                cleft--;
                advance(ce, cr, cr0, clen, stride);
            }
        }
        __syncthreads();   // every warp's gate/up is done: region A (the x staging) is free for `a`
        block_stamp(p, 5);
    }
    {
        // ------------------------------------------------------------ down: row quads [q0, q0 + nquads) of every entry
        const int nb = p.I / QK_K, nrb = RW * nb, item_bytes = nrb * DownFmt::kBlockBytes;
        const int quads = p.H / RW;
        const int q0 = (int)((long)quads * blockIdx.x / gridDim.x), nquads = (int)((long)quads * (blockIdx.x + 1) / gridDim.x) - q0;
        const int nv = sh.nv;
        const int Wd = W - 1;   // warps streaming tiles; warp W - 1 quantises this CTA's share of the Q8_K blocks
        int ni = warp < Wd ? nquads * nv - warp : 0;
        ni = ni > 0 ? (ni + Wd - 1) / Wd : 0;
        int dvi = 0, dq = 0, dss = 0, dcons = 0;   // issue cursor, tiles requested, tiles consumed
        if (ni > 0) { dvi = warp / nquads; dq = warp - dvi * nquads; }
        int evi = dvi, eq = dq;
        int dslot_i = 0, dslot_u = 0;
        auto issue_d = [&]() {
            if (dss < ni && dss - dcons < SD) {
                if (lane == 0) {
                    const int j = sh.vs[dvi];
                    long row = (long)(q0 + dq) * RW;
                    const uint8_t* wbase = reinterpret_cast<const uint8_t*>(p.w_down);
                    if (j == k) wbase = reinterpret_cast<const uint8_t*>(p.s_down);
                    else row += ((long)sh.ids[j] - p.id_offset) * p.H;
                    const uint32_t bar = bar_u32 + 8 * dslot_i;
                    mbar_expect_tx(bar, (uint32_t)item_bytes);
                    bulk_g2s(ring_u32 + dslot_i * item_bytes, wbase + (row >> 2) * item_bytes, (uint32_t)item_bytes, bar);
                }
                dss++;
                dq += Wd;
                while (dq >= nquads) { dq -= nquads; dvi++; }
                dslot_i = (dslot_i + 1 == SD) ? 0 : dslot_i + 1;
            }
        };
        // the tiles depend on the expert ids only: they stream while the first entry's `a` is fetched
#pragma unroll
        for (int s = 0; s < SD; s++) issue_d();
        const BlockLay L = block_layout<DownFmt::kBs>(p, smem);
        if (warp == W - 1) {
            // the quantisation this CTA contributes, in work-list order (this warp has no bulk copies in flight: its
            // fences do not wait for any)
            for (int ev = 0; ev < nv; ev++) claim_entry<DownFmt::kBs>(p, t, sh.vs[ev]);
        }
        if (t == Teff - 1 && warp == W - 1) {
            // the next layer's first bytes (ktb200_moe_block_prefetch_hint) -> L2, this CTA's 1/grid slice of each range in
            // 4 KB pieces: no registers or shared memory held, the down stream keeps its ring
#pragma unroll
            for (int r = 0; r < 3; r++) {
                if (p.pf[r]) {
                    const unsigned per = ((p.pf_bytes[r] / gridDim.x) + 15u) & ~15u;
                    const unsigned lo = per * blockIdx.x, hi = min(p.pf_bytes[r], lo + per);
                    for (unsigned o = lo + lane * 4096u; o < hi; o += 32u * 4096u) prefetch_l2_bulk(p.pf[r] + o, min(4096u, hi - o) & ~15u);
                }
            }
        }

        const uint8_t* ring = smem + (ring_u32 - (uint32_t)__cvta_generic_to_shared(smem));
        const int ns = k + (has_shared ? 1 : 0);
        for (int n = 0; n < ni; n++) {
            if (eq < Wd) {   // this warp's first tile of entry evi; the next entry is copied ahead by whoever gets there first
                entry_to_smem<DownFmt::kBs>(sh, L, t, evi, true);
                if (evi + 1 < nv) entry_to_smem<DownFmt::kBs>(sh, L, t, evi + 1, false);
            }
            mbar_wait(bar_u32 + 8 * dslot_u, (phase >> dslot_u) & 1u);
            phase ^= 1u << dslot_u;
            const uint8_t* sl = ring + dslot_u * item_bytes;
            const int j = sh.vs[evi];
            float res;
            {
                float acc[RW] = {0.f, 0.f, 0.f, 0.f};
                for (int f = lane; f < nrb; f += 32) {   // (row, block) pairs of the tile; 4 x 8 = one per lane for I = 2048
                    const int rw = f / nb, blk = f - rw * nb;
                    const int ab = j * nb + blk;
                    const float val = DownFmt::dot(sl, f, nrb, L.aq + (size_t)ab * kActBlkStride, L.abs_ + ab * DownFmt::kBs, L.adx[ab]);
                    acc[0] += rw == 0 ? val : 0.f; acc[1] += rw == 1 ? val : 0.f; acc[2] += rw == 2 ? val : 0.f; acc[3] += rw == 3 ? val : 0.f;
                }
                res = warp_reduce4(acc[0], acc[1], acc[2], acc[3], lane);
            }
            __syncwarp();
            dslot_u = (dslot_u + 1 == SD) ? 0 : dslot_u + 1;
            dcons++;
            issue_d();
            if ((lane & 7) == 0) L.partial[(eq * RW + (lane >> 3)) * ns + j] = res;
            eq += Wd;
            while (eq >= nquads) { eq -= nquads; evi++; }
        }
        __syncthreads();
        block_stamp(p, 8);
        blk_combine<DownFmt::kBs>(t);
        block_stamp(p, 9);
    }
  }  // tokens

    // leave the barrier and readiness words zeroed for the next launch / graph replay: the last CTA to get here resets
    // them (every other CTA has finished all its reads of them)
    __syncthreads();
    if (threadIdx.x == 0) sh.last_cta = atomicAdd(p.sync + 1, 1u) == gridDim.x - 1;
    __syncthreads();
    if (sh.last_cta) {
        const int nready = Teff * (k + (has_shared ? 1 : 0)) * (p.I / QK_K);
        for (int i = threadIdx.x; i < nready; i += blockDim.x) p.ready[i] = 0;
        if (threadIdx.x == 0) {
            p.sync[0] = 0;
            p.sync[1] = 0;
        }
        __threadfence();
    }
}


// ===================================================================================================================
// Expert-parallel MoE block: ONE persistent launch per layer and GPU, exchange over NVLink peer memory inside it.
//
// Rank r owns experts [id_offset, id_offset + n_local) and one token per layer (decode, one sequence per GPU).  Spec:
// the all-to-all dispatch / combine of archive/ktransformers/models/modeling_deepseek_v3.py:550-605 without its host
// round trips.  Phases (mask bits; tests run them as separate launches to emulate N ranks on one GPU):
//   R (1)  router GEMV + top-k of the OWN token (as in moe_block_kernel: nothing is routed redundantly); the shared
//          expert's gate/up rows stream while the top-k runs; CTA c < world then PUSHES the message
//          {x row, ids int32[k], weights[k]} into row `rank` of peer c's message buffer and releases a system-scope flag.
//   X (2)  wait for the `world` messages; every CTA builds the same list of (token, slot) pairs this shard owns
//          (sorted by token, slot); gate/up over the (pair, row) list; grid barrier; down + weighted sum per token in
//          slot order (chunks of `pa` entries: the activation staging is finite), the shared expert's down rows as an
//          extra entry; every CTA stores its row slice of all `world` partial rows into the owners' partial buffers
//          (row `rank`) and bumps a system-scope counter on each owner.
//   C (4)  wait until all CTAs of all ranks have delivered; y = round(sum over ranks, rank order) + round(shared).
// Buffers are reused every layer without extra barriers: a rank can only send its next token after it finished
// phase C, which needs every rank's phase-X stores, which come after that rank's reads of the messages.
// moe_ep_block_kernel<GU, DownFmt> below (Q2_K / Q3_K gate/up) repeats this exchange (the message push, the pair list, the
// deliver stores, the flag and epoch protocol, phase C and the exit): a change to the protocol is a change to both.
constexpr int kEpWorldMax = 8;
constexpr int kEpPairsMax = 64;

struct EpExtra {
    int rank, world, phase_mask, pa;      // pa: entries per down chunk (activation staging capacity)
    int msg_bytes;                        // message row: H * sizeof(hidden) + 128
    int inter_shared_row;                 // row of `inter` that holds the shared expert's activations (= world * k)
    float* shared_out;                    // [H] fp32: shared expert's down result (before rounding), phase X -> C
    uint8_t* msg[kEpWorldMax];            // every rank's message buffer [world][msg_bytes]
    float* part[kEpWorldMax];             // every rank's partial buffer [world][H] fp32
    unsigned* flags[kEpWorldMax];         // every rank's flag block: tok[world] | cnt[world] | epoch | status
    int ep_off;                           // byte offset of EpShared in dynamic shared memory
};
struct EpParams { BlockParams b; EpExtra x; };

struct EpShared {
    EpExtra x;
    unsigned epoch;
    int np;                               // pairs owned by this shard
    int pair_src[kEpPairsMax];            // source token (= rank that owns it)
    int pair_e[kEpPairsMax];              // local expert index
    float pair_w[kEpPairsMax];
    int tok_slot[2];                      // which tokens' activations sit in the two x staging slots (phase X)
};

__device__ __forceinline__ void st_release_sys_u32(unsigned* p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_release_sys_add(unsigned* p, unsigned v) {
    asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// one token row (hidden type, read at L2: it was written by a peer) -> Q8_K in staging slot `slot`, KBS int16 sums per block
template <int KBS>
__device__ __forceinline__ void ep_quantize_row(const BlockParams& p, const uint8_t* row, uint8_t* slot_base) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5, nblk = p.H / QK_K;
    uint8_t* xq = slot_base;
    int16_t* xbs = reinterpret_cast<int16_t*>(slot_base + (size_t)nblk * kActBlkStride);
    float* xdx = reinterpret_cast<float*>(slot_base + (size_t)nblk * (kActBlkStride + 2 * KBS));
    for (int b = warp; b < nblk; b += W) {
        float x[8];
        const long e0 = (long)b * QK_K + lane * 8;
        if (p.hidden_type == KTB200_TYPE_F32) {
            const float4 a = __ldcg(reinterpret_cast<const float4*>(row) + e0 / 4), c = __ldcg(reinterpret_cast<const float4*>(row) + e0 / 4 + 1);
            x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = c.x; x[5] = c.y; x[6] = c.z; x[7] = c.w;
        } else {
            const uint4 raw = __ldcg(reinterpret_cast<const uint4*>(row) + e0 / 8);
            const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
            for (int i = 0; i < 4; i++) {
                if (p.hidden_type == KTB200_TYPE_BF16) {
                    x[2 * i] = __uint_as_float(w[i] << 16);
                    x[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
                } else {
                    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
                    x[2 * i] = f.x; x[2 * i + 1] = f.y;
                }
            }
        }
        warp_quantize_q8k_block(x, lane, reinterpret_cast<uint32_t*>(xq + (size_t)b * kActBlkStride), xdx + b,
                                KBS == 16 ? xbs + b * 16 : nullptr, KBS == 8 ? xbs + b * 8 : nullptr);
    }
}

template <class DownFmt>
__global__ void __launch_bounds__(kBlockWarpsLo * 32, 1) moe_ep_block_kernel(const EpParams pp) {
    constexpr int RW = 4, SU = 4, SD = 2;
    extern __shared__ __align__(16) uint8_t smem[];
    BlockShared& sh = *reinterpret_cast<BlockShared*>(smem);
    EpShared& es = *reinterpret_cast<EpShared*>(smem + pp.x.ep_off);
    const BlockParams& p = pp.b;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    griddep_launch_dependents();
    bool waited = false;
    const int k = p.k, world = pp.x.world, rank = pp.x.rank, mask = pp.x.phase_mask;
    const bool has_shared = p.s_gate != nullptr;
    const int nblk = p.H / QK_K, row_bytes = nblk * SZ_Q4_K;
    const int nb = p.I / QK_K;
    uint32_t bar_u32, ring_u32;
    {
        const BlockLay L = block_layout<DownFmt::kBs>(p, smem);
        const int bar_bytes = (W * SU * 8 + 15) & ~15;
        bar_u32 = (uint32_t)__cvta_generic_to_shared(smem + L.ring_off) + warp * SU * 8;
        ring_u32 = (uint32_t)__cvta_generic_to_shared(smem + L.ring_off + bar_bytes) + warp * p.ring_bytes;
    }
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < SU; s++) mbar_init(bar_u32 + 8 * s, 1);
        mbar_fence_init();
        fence_proxy_async_smem();
    }
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&pp.b);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&sh.prm);
        for (int i = threadIdx.x; i < (int)(sizeof(BlockParams) / 4); i += blockDim.x) dst[i] = src[i];
        const uint32_t* src2 = reinterpret_cast<const uint32_t*>(&pp.x);
        uint32_t* dst2 = reinterpret_cast<uint32_t*>(&es.x);
        for (int i = threadIdx.x; i < (int)(sizeof(EpExtra) / 4); i += blockDim.x) dst2[i] = src2[i];
    }
    if (threadIdx.x == 0 && has_shared) sh.vs[0] = k;
    __syncthreads();   // the parameter copies in shared memory (read by blk_router & co through sh.prm) and the mbarriers are ready
    uint32_t phase = 0;
    unsigned gen = 0;
    const uint8_t* ring = smem + (ring_u32 - (uint32_t)__cvta_generic_to_shared(smem));
    unsigned* my_flags = pp.x.flags[rank];
    unsigned* status = my_flags + 2 * world + 1;
    // row slice of this CTA (phases X and C)
    const int quads = p.H / RW;
    const int q0 = (int)((long)quads * blockIdx.x / gridDim.x), nquads = (int)((long)quads * (blockIdx.x + 1) / gridDim.x) - q0;
    const int nrows = nquads * RW;
    const int pa = pp.x.pa;
    float* tokacc = reinterpret_cast<float*>(smem + pp.x.ep_off + ((sizeof(EpShared) + 15) & ~(size_t)15));   // [nrows_max][world]
    float* sharedres = tokacc + (size_t)p.nrows_max * kEpWorldMax;                                            // [nrows_max]
    float* partial = sharedres + p.nrows_max;                                                                 // [nrows_max][pa]
    block_stamp(p, 0);

    // gate/up list machinery (as in moe_block_kernel; an entry is either the shared expert or a pair)
    int ie = 0, ir = 0, ileft = 0, isub = 0, ce = 0, cr = 0, cleft = 0, csub = 0, stride = W, slot_i = 0, slot_u = 0;
    bool list_shared = true;
    auto start_list = [&](int e0, int first_row, int count, int stride_) {
        ie = e0 + first_row / p.I; ir = first_row - (first_row / p.I) * p.I;
        ce = ie; cr = ir;
        ileft = cleft = count > 0 ? count : 0;
        stride = stride_;
    };
    auto issue_u = [&]() {
        if (ileft > 0 && isub - csub < SU) {
            if (lane == 0) {
                const bool second = isub & 1;
                const uint8_t* src;
                if (list_shared) src = reinterpret_cast<const uint8_t*>(second ? p.s_up : p.s_gate) + (long)ir * row_bytes;
                else src = reinterpret_cast<const uint8_t*>(second ? p.w_up : p.w_gate) + ((long)es.pair_e[ie] * p.I + ir) * row_bytes;
                const uint32_t bar = bar_u32 + 8 * slot_i;
                mbar_expect_tx(bar, (uint32_t)row_bytes);
                bulk_g2s(ring_u32 + slot_i * row_bytes, src, (uint32_t)row_bytes, bar);
            }
            isub++;
            if (!(isub & 1)) {
                ileft--;
                ir += stride;
                while (ir >= p.I) { ir -= p.I; ie++; }
            }
            slot_i = (slot_i + 1 == SU) ? 0 : slot_i + 1;
        }
    };
    const int x_slot_bytes = ((nblk * (kActBlkStride + 16 + 4)) + 15) & ~15;
    // consume the current list; `first_entry`: entry whose activations sit in x staging slot 0 (the next one in slot 1)
    auto consume_u = [&](int first_entry, long inter_row0) {
        const BlockLay L = block_layout<DownFmt::kBs>(p, smem);
        float acc_first = 0.f;
        while (cleft > 0) {
            mbar_wait(bar_u32 + 8 * slot_u, (phase >> slot_u) & 1u);
            phase ^= 1u << slot_u;
            const uint8_t* row0 = ring + slot_u * row_bytes;
            const uint8_t* xs = L.xq + (list_shared ? 0 : (es.pair_src[ce] == es.tok_slot[0] ? 0 : x_slot_bytes));
            float acc = 0.f;
            if (lane < nblk)
                acc = q4k_block_dot(row0 + lane * SZ_Q4_K, xs + (size_t)lane * kActBlkStride,
                                    *reinterpret_cast<const uint4*>(xs + (size_t)nblk * kActBlkStride + lane * 16),
                                    reinterpret_cast<const float*>(xs + (size_t)nblk * (kActBlkStride + 16))[lane]);
            __syncwarp();
            slot_u = (slot_u + 1 == SU) ? 0 : slot_u + 1;
            csub++;
            issue_u();
            if (csub & 1) { acc_first = acc; continue; }
            float g = acc_first, uu = acc;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                g += __shfl_xor_sync(0xffffffffu, g, o);
                uu += __shfl_xor_sync(0xffffffffu, uu, o);
            }
            if (lane == 0) p.inter[(inter_row0 + (list_shared ? 0 : ce)) * p.I + cr] = (p.use_silu ? act_silu(g) : act_relu(g)) * uu;
            cleft--;
            cr += stride;
            while (cr >= p.I) { cr -= p.I; ce++; }
        }
        (void)first_entry;
    };

    // =============================================================================================== phase R
    if (mask & 1) {
        blk_router(0, waited);
        block_stamp(p, 2);
        grid_arrive(p.sync, gen);
        list_shared = true;
        if (has_shared && warp >= kGateWarps) {
            const int ur0 = (int)((long)p.I * blockIdx.x / gridDim.x), nr = (int)((long)p.I * (blockIdx.x + 1) / gridDim.x) - ur0;
            const int first = warp - kGateWarps, st = W - kGateWarps;
            start_list(0, ur0 + first, (nr - first + st - 1) / st, st);
        }
#pragma unroll
        for (int s = 0; s < SU; s++)
            if (s < p.prime_u) issue_u();
        blk_quantize_x(0);
        grid_wait(p.sync, gen);
        block_stamp(p, 3);
        consume_u(0, pp.x.inter_shared_row);   // warps 4..: the shared expert's rows of this CTA (no-op for warps 0..3)
        blk_select(0);                          // warps 0..3 (barriers inside: all threads call it)
        block_stamp(p, 4);
        // push {x, ids, w} to peer `blockIdx.x`
        if ((int)blockIdx.x < world) {
            if (!waited) { griddep_wait(); waited = true; }
            const int peer = blockIdx.x;
            uint8_t* dst = pp.x.msg[peer] + (size_t)rank * pp.x.msg_bytes;
            const int xb = p.H * (int)type_size(p.hidden_type);
            const uint4* src = reinterpret_cast<const uint4*>(p.g.x);
            for (int i = threadIdx.x; i < xb / 16; i += blockDim.x) reinterpret_cast<uint4*>(dst)[i] = src[i];
            if ((int)threadIdx.x < k) {
                reinterpret_cast<int*>(dst + xb)[threadIdx.x] = (int)sh.ids[threadIdx.x];
                reinterpret_cast<float*>(dst + xb + 64)[threadIdx.x] = sh.w[threadIdx.x];
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                unsigned ep = *reinterpret_cast<volatile unsigned*>(my_flags + 2 * world) + 1;
                __threadfence_system();
                st_release_sys_u32(pp.x.flags[peer] + rank, ep);
            }
        }
    }
    if (!waited) { griddep_wait(); waited = true; }
    if (threadIdx.x == 0) es.epoch = *reinterpret_cast<volatile unsigned*>(my_flags + 2 * world) + 1;
    __syncthreads();
    const unsigned epoch = es.epoch;

    // =============================================================================================== phase X
    if (mask & 2) {
        if ((int)threadIdx.x < world) wait_ge<true>(my_flags + threadIdx.x, epoch, status);
        __syncthreads();
        block_stamp(p, 5);
        const uint8_t* mymsg = pp.x.msg[rank];
        const int xb = p.H * (int)type_size(p.hidden_type);
        if (threadIdx.x == 0) {   // the pairs this shard owns, by (token, slot): identical in every CTA
            int np = 0;
            for (int t = 0; t < world; t++) {
                const uint8_t* m = mymsg + (size_t)t * pp.x.msg_bytes + xb;
                for (int j = 0; j < k; j++) {
                    const int e = __ldcg(reinterpret_cast<const int*>(m) + j) - p.id_offset;
                    if (e >= 0 && e < p.n_local && np < kEpPairsMax) {
                        es.pair_src[np] = t; es.pair_e[np] = e; es.pair_w[np] = __ldcg(reinterpret_cast<const float*>(m + 64) + j);
                        np++;
                    }
                }
            }
            es.np = np;
        }
        __syncthreads();
        const int np = es.np;
        // ------------------------------------------------------------ gate/up over (pair, row) units
        const long total = (long)np * p.I;
        const int u0 = (int)(total * blockIdx.x / gridDim.x), u1 = (int)(total * (blockIdx.x + 1) / gridDim.x);
        if (u1 > u0) {
            const int pe0 = u0 / p.I, pe1 = (u1 - 1) / p.I;       // at most two pairs: total / grid < I
            if (threadIdx.x == 0) { es.tok_slot[0] = es.pair_src[pe0]; es.tok_slot[1] = es.pair_src[pe1]; }
            const BlockLay L = block_layout<DownFmt::kBs>(p, smem);
            ep_quantize_row<8>(p, mymsg + (size_t)es.pair_src[pe0] * pp.x.msg_bytes, L.xq);
            if (es.pair_src[pe1] != es.pair_src[pe0]) ep_quantize_row<8>(p, mymsg + (size_t)es.pair_src[pe1] * pp.x.msg_bytes, L.xq + x_slot_bytes);
        }
        __syncthreads();
        list_shared = false;
        start_list(0, u0 + warp, (u1 - u0 - warp + W - 1) / W, W);
#pragma unroll
        for (int s = 0; s < SU; s++) issue_u();
        consume_u(0, 0);
        block_stamp(p, 6);

        // ------------------------------------------------------------ down
        const int nrb = RW * nb, item_bytes = nrb * DownFmt::kBlockBytes;
        const int nent = np + (has_shared ? 1 : 0);   // entry 0 = shared expert (if any), then the pairs
        for (int i = threadIdx.x; i < nrows * world; i += blockDim.x) tokacc[i] = 0.f;
        grid_arrive(p.sync, gen);
        int dvi = 0, dq = 0, dss = 0, dcons = 0, ni = 0, evi = 0, eq = 0, dslot_i = 0, dslot_u = 0, c0 = 0;
        auto issue_d = [&]() {
            if (dss < ni && dss - dcons < SD) {
                if (lane == 0) {
                    const int ent = c0 + dvi;
                    long row = (long)(q0 + dq) * RW;
                    const uint8_t* wbase = reinterpret_cast<const uint8_t*>(p.w_down);
                    if (has_shared && ent == 0) wbase = reinterpret_cast<const uint8_t*>(p.s_down);
                    else row += (long)es.pair_e[ent - (has_shared ? 1 : 0)] * p.H;
                    const uint32_t bar = bar_u32 + 8 * dslot_i;
                    mbar_expect_tx(bar, (uint32_t)item_bytes);
                    bulk_g2s(ring_u32 + dslot_i * item_bytes, wbase + (row >> 2) * item_bytes, (uint32_t)item_bytes, bar);
                }
                dss++;
                dq += W;
                while (dq >= nquads) { dq -= nquads; dvi++; }
                dslot_i = (dslot_i + 1 == SD) ? 0 : dslot_i + 1;
            }
        };
        auto start_chunk = [&](int c0_, int cn) {
            c0 = c0_;
            ni = nquads * cn - warp;
            ni = ni > 0 ? (ni + W - 1) / W : 0;
            dss = dcons = 0;
            dvi = ni > 0 ? warp / nquads : 0; dq = ni > 0 ? warp - dvi * nquads : 0;
            evi = dvi; eq = dq;
        };
        start_chunk(0, min(pa, nent));
#pragma unroll
        for (int s = 0; s < SD; s++)
            if (s < p.prime_d) issue_d();
        grid_wait(p.sync, gen);
        block_stamp(p, 7);
        for (int cbase = 0; cbase < nent; cbase += pa) {
            const int cn = min(pa, nent - cbase);
            if (cbase) start_chunk(cbase, cn);
            // activations of the chunk's entries -> Q8_K (region A is free: gate/up is done everywhere after the barrier)
            {
                const BlockLay L = block_layout<DownFmt::kBs>(p, smem);
                uint8_t* aq = L.aq;
                int16_t* abs_ = reinterpret_cast<int16_t*>(aq + (size_t)pa * nb * kActBlkStride);
                float* adx = reinterpret_cast<float*>(aq + (size_t)pa * nb * (kActBlkStride + 2 * DownFmt::kBs));
                for (int gb = warp; gb < cn * nb; gb += W) {
                    const int r = gb / nb, b = gb - r * nb;
                    const int ent = cbase + r;
                    const long irow = (has_shared && ent == 0) ? pp.x.inter_shared_row : ent - (has_shared ? 1 : 0);
                    const float4* src = reinterpret_cast<const float4*>(p.inter + irow * p.I + (long)b * QK_K + lane * 8);
                    const float4 v0 = __ldcg(src), v1 = __ldcg(src + 1);
                    float x[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
                    warp_quantize_q8k_block(x, lane, reinterpret_cast<uint32_t*>(aq + (size_t)gb * kActBlkStride), adx + gb,
                                            DownFmt::kBs == 16 ? abs_ + gb * 16 : nullptr, DownFmt::kBs == 8 ? abs_ + gb * 8 : nullptr);
                }
#pragma unroll
                for (int s = 0; s < SD; s++) issue_d();
                __syncthreads();
                for (int n = 0; n < ni; n++) {
                    mbar_wait(bar_u32 + 8 * dslot_u, (phase >> dslot_u) & 1u);
                    phase ^= 1u << dslot_u;
                    const uint8_t* sl = ring + dslot_u * item_bytes;
                    float res;
                    {
                        float acc[RW] = {0.f, 0.f, 0.f, 0.f};
                        for (int f = lane; f < nrb; f += 32) {
                            const int rw = f / nb, blk = f - rw * nb;
                            const int ab = evi * nb + blk;
                            const float val = DownFmt::dot(sl, f, nrb, aq + (size_t)ab * kActBlkStride, abs_ + ab * DownFmt::kBs, adx[ab]);
                            acc[0] += rw == 0 ? val : 0.f; acc[1] += rw == 1 ? val : 0.f; acc[2] += rw == 2 ? val : 0.f; acc[3] += rw == 3 ? val : 0.f;
                        }
                        res = warp_reduce4(acc[0], acc[1], acc[2], acc[3], lane);
                    }
                    __syncwarp();
                    dslot_u = (dslot_u + 1 == SD) ? 0 : dslot_u + 1;
                    dcons++;
                    issue_d();
                    if ((lane & 7) == 0) partial[(eq * RW + (lane >> 3)) * pa + evi] = res;
                    eq += W;
                    while (eq >= nquads) { eq -= nquads; evi++; }
                }
                __syncthreads();
                // weighted accumulation per token in (token, slot) order with one FMA per pair (moe.cpp:222-236)
                for (int hl = threadIdx.x; hl < nrows; hl += blockDim.x) {
                    for (int r = 0; r < cn; r++) {
                        const int ent = cbase + r;
                        if (has_shared && ent == 0) { sharedres[hl] = partial[hl * pa + r]; continue; }
                        const int pi = ent - (has_shared ? 1 : 0);
                        float* a = tokacc + hl * world + es.pair_src[pi];
                        *a = __fmaf_rn(partial[hl * pa + r], es.pair_w[pi], *a);
                    }
                }
                __syncthreads();
            }
        }
        block_stamp(p, 8);
        // ------------------------------------------------------------ deliver: my rows of every token's partial sum
        for (int i = threadIdx.x; i < nquads * world; i += blockDim.x) {
            const int t = i / nquads, qd = i - t * nquads;
            const float4 v = make_float4(tokacc[(qd * 4 + 0) * world + t], tokacc[(qd * 4 + 1) * world + t], tokacc[(qd * 4 + 2) * world + t],
                                         tokacc[(qd * 4 + 3) * world + t]);
            *reinterpret_cast<float4*>(pp.x.part[t] + (size_t)rank * p.H + (size_t)(q0 + qd) * 4) = v;
        }
        if (has_shared)
            for (int hl = threadIdx.x; hl < nrows; hl += blockDim.x) pp.x.shared_out[q0 * 4 + hl] = sharedres[hl];
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence_system();
            for (int t = 0; t < world; t++) red_release_sys_add(pp.x.flags[t] + world + rank, 1u);
        }
    }

    // =============================================================================================== phase C
    if (mask & 4) {
        if ((int)threadIdx.x < world) wait_ge<true>(my_flags + world + threadIdx.x, epoch * gridDim.x, status);
        __syncthreads();
        block_stamp(p, 9);
        const float* mine = pp.x.part[rank];
        for (int hl = threadIdx.x; hl < nrows; hl += blockDim.x) {
            const int row = q0 * 4 + hl;
            float acc = 0.f;
            for (int r = 0; r < world; r++) acc += __ldcg(mine + (size_t)r * p.H + row);   // rank order: deterministic
            float v = round_hidden(acc, p.hidden_type);
            if (has_shared) v += round_hidden(__ldcg(pp.x.shared_out + row), p.hidden_type);
            store_hidden(p.out, row, p.hidden_type, v);
        }
        block_stamp(p, 10);
    }

    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned prev = atomicAdd(p.sync + 1, 1u);
        if (prev == gridDim.x - 1) {
            p.sync[0] = 0;
            p.sync[1] = 0;
            if (mask & 4) my_flags[2 * world] = epoch;
            __threadfence();
        }
    }
}

// The same layer for Q2_K / Q3_K routed gate/up (GU = BulkQ2K | BulkQ3K, gate and up of one type) and any bulk down item
// (BulkQ2K | BulkQ3K | BulkQ4K | BulkQ6K4T): llama.cpp's Q2_K, Q3_K_S and Q3_K_M files.  Phases, messages, flags, epochs and
// the reuse argument are those of the kernel above, and the code that implements them repeats that kernel's (kept apart so
// that the Q4_K instantiations compile to the same instructions as before): a change to the protocol is a change to both.
// What differs:
//   * a gate/up unit is rows 2r, 2r+1 of gate and of up (the unit of rows_bulk_iq_kernel, iq.cuh: single Q2_K / Q3_K rows are
//     not 16-byte sized), two bulk copies on one mbarrier; the per-lane loop and the reduction are that kernel's, so `inter`
//     equals the per-pair kernels' output bit for bit;
//   * the shared expert is not in the launch (its types need not be the routed ones): the launcher runs ktb200_mlp_forward
//     into y first, with the combine phase, and p.s_gate != null says y holds that rounded term.  Phase C computes
//     y = round(sum over ranks, rank order) + y, as ep_tok_combine_kernel does; phase R streams nothing beside the router;
//   * warps per CTA and the down chunk `pa` come from the shared-memory plan (ep_kq_plan).
// Dynamic shared memory: [BlockShared][region A][EpShared | tokacc [nrows_max][kEpWorldMax] | partial [nrows_max][pa]]
// [mbarriers W x 2][rings W x ring_bytes].  Region A holds in turn the router's selection scratch (blk_select's layout), the
// Q8_K rows of up to two tokens (GU's sums) and the Q8_K `a` of pa entries (DownFmt's sums).
constexpr int kEpKqSlots = 2;   // ring slots per warp, gate/up units and down items alike
template <int KBS>
__host__ __device__ constexpr int ep_x_slot_bytes(int nblk) { return (nblk * (kActBlkStride + 2 * KBS + 4) + 15) & ~15; }

template <class GU, class DownFmt>
__global__ void __launch_bounds__(kBlockWarpsLo * 32, 1) moe_ep_block_kernel(const EpParams pp) {
    constexpr int RW = 4, S = kEpKqSlots;
    extern __shared__ __align__(16) uint8_t smem[];
    BlockShared& sh = *reinterpret_cast<BlockShared*>(smem);
    EpShared& es = *reinterpret_cast<EpShared*>(smem + pp.x.ep_off);
    const BlockParams& p = pp.b;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    griddep_launch_dependents();
    bool waited = false;
    const int k = p.k, world = pp.x.world, rank = pp.x.rank, mask = pp.x.phase_mask;
    const bool has_shared = p.s_gate != nullptr;
    const int nblk = p.H / QK_K, nb = p.I / QK_K;
    const int pa = pp.x.pa;
    float* tokacc = reinterpret_cast<float*>(smem + pp.x.ep_off + ((sizeof(EpShared) + 15) & ~(size_t)15));   // [nrows_max][world]
    float* partial = tokacc + (size_t)p.nrows_max * kEpWorldMax;                                            // [nrows_max][pa]
    uint32_t bar_u32, ring_u32;
    {
        const size_t off = (reinterpret_cast<uint8_t*>(partial + (size_t)p.nrows_max * pa) - smem + 15) & ~(size_t)15;
        bar_u32 = (uint32_t)__cvta_generic_to_shared(smem + off) + warp * S * 8;
        ring_u32 = (uint32_t)__cvta_generic_to_shared(smem + off + ((W * S * 8 + 15) & ~15)) + warp * p.ring_bytes;
    }
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < S; s++) mbar_init(bar_u32 + 8 * s, 1);
        mbar_fence_init();
        fence_proxy_async_smem();
    }
    {
        const uint32_t* src = reinterpret_cast<const uint32_t*>(&pp.b);
        uint32_t* dst = reinterpret_cast<uint32_t*>(&sh.prm);
        for (int i = threadIdx.x; i < (int)(sizeof(BlockParams) / 4); i += blockDim.x) dst[i] = src[i];
        const uint32_t* src2 = reinterpret_cast<const uint32_t*>(&pp.x);
        uint32_t* dst2 = reinterpret_cast<uint32_t*>(&es.x);
        for (int i = threadIdx.x; i < (int)(sizeof(EpExtra) / 4); i += blockDim.x) dst2[i] = src2[i];
    }
    __syncthreads();   // the parameter copies in shared memory (read by blk_router & co through sh.prm) and the mbarriers are ready
    uint32_t phase = 0;   // bit s = parity the next use of barrier s waits for
    unsigned gen = 0;
    const uint8_t* ring = smem + (ring_u32 - (uint32_t)__cvta_generic_to_shared(smem));
    unsigned* my_flags = pp.x.flags[rank];
    unsigned* status = my_flags + 2 * world + 1;
    // row slice of this CTA (phases X and C)
    const int quads = p.H / RW;
    const int q0 = (int)((long)quads * blockIdx.x / gridDim.x), nquads = (int)((long)quads * (blockIdx.x + 1) / gridDim.x) - q0;
    const int nrows = nquads * RW;
    uint8_t* region_a = smem + kBlockSharedBytes;
    block_stamp(p, 0);

    // =============================================================================================== phase R
    if (mask & 1) {
        blk_router(0, waited);
        block_stamp(p, 2);
        grid_arrive(p.sync, gen);
        grid_wait(p.sync, gen);
        block_stamp(p, 3);
        blk_select(0);
        block_stamp(p, 4);
        // push {x, ids, w} to peer `blockIdx.x`
        if ((int)blockIdx.x < world) {
            const int peer = blockIdx.x;
            uint8_t* dst = pp.x.msg[peer] + (size_t)rank * pp.x.msg_bytes;
            const int xb = p.H * (int)type_size(p.hidden_type);
            const uint4* src = reinterpret_cast<const uint4*>(p.g.x);
            for (int i = threadIdx.x; i < xb / 16; i += blockDim.x) reinterpret_cast<uint4*>(dst)[i] = src[i];
            if ((int)threadIdx.x < k) {
                reinterpret_cast<int*>(dst + xb)[threadIdx.x] = (int)sh.ids[threadIdx.x];
                reinterpret_cast<float*>(dst + xb + 64)[threadIdx.x] = sh.w[threadIdx.x];
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                unsigned ep = *reinterpret_cast<volatile unsigned*>(my_flags + 2 * world) + 1;
                __threadfence_system();
                st_release_sys_u32(pp.x.flags[peer] + rank, ep);
            }
        }
    }
    if (!waited) { griddep_wait(); waited = true; }
    if (threadIdx.x == 0) es.epoch = *reinterpret_cast<volatile unsigned*>(my_flags + 2 * world) + 1;
    __syncthreads();
    const unsigned epoch = es.epoch;

    // =============================================================================================== phase X
    if (mask & 2) {
        if ((int)threadIdx.x < world) wait_ge<true>(my_flags + threadIdx.x, epoch, status);
        __syncthreads();
        block_stamp(p, 5);
        const uint8_t* mymsg = pp.x.msg[rank];
        const int xb = p.H * (int)type_size(p.hidden_type);
        if (threadIdx.x == 0) {   // the pairs this shard owns, by (token, slot): identical in every CTA
            int np = 0;
            for (int t = 0; t < world; t++) {
                const uint8_t* m = mymsg + (size_t)t * pp.x.msg_bytes + xb;
                for (int j = 0; j < k; j++) {
                    const int e = __ldcg(reinterpret_cast<const int*>(m) + j) - p.id_offset;
                    if (e >= 0 && e < p.n_local && np < kEpPairsMax) {
                        es.pair_src[np] = t; es.pair_e[np] = e; es.pair_w[np] = __ldcg(reinterpret_cast<const float*>(m + 64) + j);
                        np++;
                    }
                }
            }
            es.np = np;
        }
        __syncthreads();
        const int np = es.np;
        // ------------------------------------------------------------ gate/up over (pair, row pair) units
        const int nru = p.I / 2, row_bytes = nblk * GU::kBlockBytes, unit_bytes = 2 * row_bytes;
        const int x_slot = ep_x_slot_bytes<GU::kBs>(nblk);
        const long total = (long)np * nru;
        const int u0 = (int)(total * blockIdx.x / gridDim.x), u1 = (int)(total * (blockIdx.x + 1) / gridDim.x);
        if (u1 > u0) {
            const int pe0 = u0 / nru, pe1 = (u1 - 1) / nru;       // at most two pairs: total / grid < I / 2
            if (threadIdx.x == 0) { es.tok_slot[0] = es.pair_src[pe0]; es.tok_slot[1] = es.pair_src[pe1]; }
            ep_quantize_row<GU::kBs>(p, mymsg + (size_t)es.pair_src[pe0] * pp.x.msg_bytes, region_a);
            if (es.pair_src[pe1] != es.pair_src[pe0]) ep_quantize_row<GU::kBs>(p, mymsg + (size_t)es.pair_src[pe1] * pp.x.msg_bytes, region_a + x_slot);
        }
        __syncthreads();
        const int nu = warp_units(u0, u1, warp, W);
        UnitCursor ic;
        if (nu > 0) ic.start(u0 + warp, nru);
        UnitCursor cc = ic;
        int iss = 0, slot_i = 0, slot_u = 0;
        auto issue_u = [&]() {
            if (iss < nu) {
                if (lane == 0) {
                    const long off = ((long)es.pair_e[ic.pi] * p.I + 2L * ic.r) * row_bytes;
                    const uint32_t bar = bar_u32 + 8 * slot_i, dst = ring_u32 + slot_i * 2 * unit_bytes;
                    mbar_expect_tx(bar, 2u * unit_bytes);
                    bulk_g2s(dst, reinterpret_cast<const uint8_t*>(p.w_gate) + off, (uint32_t)unit_bytes, bar);
                    bulk_g2s(dst + unit_bytes, reinterpret_cast<const uint8_t*>(p.w_up) + off, (uint32_t)unit_bytes, bar);
                }
                iss++;
                ic.step(W, nru);
                slot_i = (slot_i + 1 == S) ? 0 : slot_i + 1;
            }
        };
#pragma unroll
        for (int s = 0; s < S; s++) issue_u();
        for (int n = 0; n < nu; n++) {
            mbar_wait(bar_u32 + 8 * slot_u, (phase >> slot_u) & 1u);
            phase ^= 1u << slot_u;
            const uint8_t* sl = ring + slot_u * 2 * unit_bytes;
            const uint8_t* at = region_a + (es.pair_src[cc.pi] == es.tok_slot[0] ? 0 : x_slot);
            const int16_t* bs = reinterpret_cast<const int16_t*>(at + (size_t)nblk * kActBlkStride);
            const float* dx = reinterpret_cast<const float*>(at + (size_t)nblk * (kActBlkStride + 2 * GU::kBs));
            float g0 = 0.f, g1 = 0.f, v0 = 0.f, v1 = 0.f;
            for (int f = lane; f < 2 * nblk; f += 32) {   // (row, block) of the unit: f = rw * nblk + blk
                const int rw = f >= nblk, blk = f - rw * nblk;
                const uint8_t* aq = at + (size_t)blk * kActBlkStride;
                const float g = GU::block_dot(sl + f * GU::kBlockBytes, aq, bs + blk * GU::kBs, dx[blk]);
                const float u = GU::block_dot(sl + unit_bytes + f * GU::kBlockBytes, aq, bs + blk * GU::kBs, dx[blk]);
                if (rw) { g1 += g; v1 += u; } else { g0 += g; v0 += u; }
            }
            const float r = warp_reduce4(g0, g1, v0, v1, lane);   // lane 0: g0, 8: g1, 16: u0, 24: u1
            __syncwarp();
            slot_u = (slot_u + 1 == S) ? 0 : slot_u + 1;
            issue_u();
            const float gs = __shfl_sync(0xffffffffu, r, 8 * (lane & 1)), us = __shfl_sync(0xffffffffu, r, 16 + 8 * (lane & 1));
            if (lane < 2) p.inter[(long)cc.pi * p.I + 2L * cc.r + lane] = (p.use_silu ? act_silu(gs) : act_relu(gs)) * us;
            cc.step(W, nru);
        }
        block_stamp(p, 6);

        // ------------------------------------------------------------ down (entries = the pairs, in chunks of pa)
        const int nrb = RW * nb, item_bytes = nrb * DownFmt::kBlockBytes;
        for (int i = threadIdx.x; i < nrows * world; i += blockDim.x) tokacc[i] = 0.f;
        grid_arrive(p.sync, gen);
        int dvi = 0, dq = 0, dss = 0, dcons = 0, ni = 0, evi = 0, eq = 0, dslot_i = 0, dslot_u = 0, c0 = 0;
        auto issue_d = [&]() {
            if (dss < ni && dss - dcons < S) {
                if (lane == 0) {
                    const long row = (long)(q0 + dq) * RW + (long)es.pair_e[c0 + dvi] * p.H;
                    const uint32_t bar = bar_u32 + 8 * dslot_i;
                    mbar_expect_tx(bar, (uint32_t)item_bytes);
                    bulk_g2s(ring_u32 + dslot_i * item_bytes, reinterpret_cast<const uint8_t*>(p.w_down) + (row >> 2) * item_bytes,
                             (uint32_t)item_bytes, bar);
                }
                dss++;
                dq += W;
                while (dq >= nquads) { dq -= nquads; dvi++; }
                dslot_i = (dslot_i + 1 == S) ? 0 : dslot_i + 1;
            }
        };
        auto start_chunk = [&](int c0_, int cn) {
            c0 = c0_;
            ni = nquads * cn - warp;
            ni = ni > 0 ? (ni + W - 1) / W : 0;
            dss = dcons = 0;
            dvi = ni > 0 ? warp / nquads : 0; dq = ni > 0 ? warp - dvi * nquads : 0;
            evi = dvi; eq = dq;
        };
        start_chunk(0, min(pa, np));
#pragma unroll
        for (int s = 0; s < S; s++)
            if (s < p.prime_d) issue_d();
        grid_wait(p.sync, gen);
        block_stamp(p, 7);
        uint8_t* aq = region_a;
        int16_t* abs_ = reinterpret_cast<int16_t*>(aq + (size_t)pa * nb * kActBlkStride);
        float* adx = reinterpret_cast<float*>(aq + (size_t)pa * nb * (kActBlkStride + 2 * DownFmt::kBs));
        for (int cbase = 0; cbase < np; cbase += pa) {
            const int cn = min(pa, np - cbase);
            if (cbase) start_chunk(cbase, cn);
            // activations of the chunk's pairs -> Q8_K (region A is free: gate/up is done everywhere after the barrier)
            for (int gb = warp; gb < cn * nb; gb += W) {
                const int r = gb / nb, b = gb - r * nb;
                const float4* src = reinterpret_cast<const float4*>(p.inter + (long)(cbase + r) * p.I + (long)b * QK_K + lane * 8);
                const float4 v0 = __ldcg(src), v1 = __ldcg(src + 1);
                float x[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
                warp_quantize_q8k_block(x, lane, reinterpret_cast<uint32_t*>(aq + (size_t)gb * kActBlkStride), adx + gb,
                                        DownFmt::kBs == 16 ? abs_ + gb * 16 : nullptr, DownFmt::kBs == 8 ? abs_ + gb * 8 : nullptr);
            }
#pragma unroll
            for (int s = 0; s < S; s++) issue_d();
            __syncthreads();
            for (int n = 0; n < ni; n++) {
                mbar_wait(bar_u32 + 8 * dslot_u, (phase >> dslot_u) & 1u);
                phase ^= 1u << dslot_u;
                const uint8_t* sl = ring + dslot_u * item_bytes;
                float res;
                {
                    float acc[RW] = {0.f, 0.f, 0.f, 0.f};
                    for (int f = lane; f < nrb; f += 32) {
                        const int rw = f / nb, blk = f - rw * nb;
                        const int ab = evi * nb + blk;
                        const float val = DownFmt::dot(sl, f, nrb, aq + (size_t)ab * kActBlkStride, abs_ + ab * DownFmt::kBs, adx[ab]);
                        acc[0] += rw == 0 ? val : 0.f; acc[1] += rw == 1 ? val : 0.f; acc[2] += rw == 2 ? val : 0.f; acc[3] += rw == 3 ? val : 0.f;
                    }
                    res = warp_reduce4(acc[0], acc[1], acc[2], acc[3], lane);
                }
                __syncwarp();
                dslot_u = (dslot_u + 1 == S) ? 0 : dslot_u + 1;
                dcons++;
                issue_d();
                if ((lane & 7) == 0) partial[(eq * RW + (lane >> 3)) * pa + evi] = res;
                eq += W;
                while (eq >= nquads) { eq -= nquads; evi++; }
            }
            __syncthreads();
            // weighted accumulation per token in (token, slot) order with one FMA per pair (moe.cpp:222-236)
            for (int hl = threadIdx.x; hl < nrows; hl += blockDim.x) {
                for (int r = 0; r < cn; r++) {
                    const int pi = cbase + r;
                    float* a = tokacc + hl * world + es.pair_src[pi];
                    *a = __fmaf_rn(partial[hl * pa + r], es.pair_w[pi], *a);
                }
            }
            __syncthreads();
        }
        block_stamp(p, 8);
        // ------------------------------------------------------------ deliver: my rows of every token's partial sum
        for (int i = threadIdx.x; i < nquads * world; i += blockDim.x) {
            const int t = i / nquads, qd = i - t * nquads;
            const float4 v = make_float4(tokacc[(qd * 4 + 0) * world + t], tokacc[(qd * 4 + 1) * world + t], tokacc[(qd * 4 + 2) * world + t],
                                         tokacc[(qd * 4 + 3) * world + t]);
            *reinterpret_cast<float4*>(pp.x.part[t] + (size_t)rank * p.H + (size_t)(q0 + qd) * 4) = v;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence_system();
            for (int t = 0; t < world; t++) red_release_sys_add(pp.x.flags[t] + world + rank, 1u);
        }
    }

    // =============================================================================================== phase C
    if (mask & 4) {
        if ((int)threadIdx.x < world) wait_ge<true>(my_flags + world + threadIdx.x, epoch * gridDim.x, status);
        __syncthreads();
        block_stamp(p, 9);
        const float* mine = pp.x.part[rank];
        for (int hl = threadIdx.x; hl < nrows; hl += blockDim.x) {
            const int row = q0 * 4 + hl;
            float acc = 0.f;
            for (int r = 0; r < world; r++) acc += __ldcg(mine + (size_t)r * p.H + row);   // rank order: deterministic
            float v = round_hidden(acc, p.hidden_type);
            if (has_shared) v += load_hidden(p.out, row, p.hidden_type);   // the rounded shared term ktb200_mlp_forward stored
            store_hidden(p.out, row, p.hidden_type, v);
        }
        block_stamp(p, 10);
    }

    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned prev = atomicAdd(p.sync + 1, 1u);
        if (prev == gridDim.x - 1) {
            p.sync[0] = 0;
            p.sync[1] = 0;
            if (mask & 4) my_flags[2 * world] = epoch;
            __threadfence();
        }
    }
}

static unsigned long long* g_btrace = nullptr;

static int env_fused() {
    static int v = [] { const char* e = getenv("KTB200_FUSED"); return e ? atoi(e) : 1; }();
    return v;
}

}  // namespace ktb

using namespace ktb;

extern "C" int ktb200_moe_block_forward(const ktb200_gate_config* gc, ktb200_moe* m, ktb200_mlp* sh, int qlen, const void* input,
                                        void* output, int64_t* idx, float* w, const int* bsz, void* stream) {
    if (!gc || !m || !input || !output || !idx || !w) { set_error("null pointer"); return KTB200_EINVAL; }
    if (!m->loaded) { set_error("Not Loaded"); return KTB200_ESTATE; }
    if (sh && !sh->loaded) { set_error("shared expert: Not Loaded"); return KTB200_ESTATE; }
    if (qlen <= 0) return KTB200_OK;
    const ktb200_moe_config& c = m->cfg;
    const int k = gc->top_k;
    if (gc->hidden_size != c.hidden_size || gc->hidden_type != c.hidden_type) { set_error("moe_block: gate and experts disagree on the hidden size / type"); return KTB200_EINVAL; }
    if (k <= 0 || k > c.routed_expert_num) { set_error("moe_block: top_k=%d outside (0, routed_expert_num=%d]", k, c.routed_expert_num); return KTB200_EINVAL; }
    if (qlen > c.group_max_len) { set_error("forward: qlen=%d exceeds group_max_len=%d", qlen, c.group_max_len); return KTB200_EINVAL; }

    // ---- can the fused kernel take it?  otherwise: the separate launches (same results)
    const FmtId fd = pick_fmt(c.down_type, m->down_layout);
    const bool sh_ok = !sh || (sh->H == c.hidden_size && sh->I == c.intermediate_size && sh->hidden_type == c.hidden_type &&
                               sh->gate_type == c.gate_type && sh->up_type == c.up_type && sh->down_type == c.down_type &&
                               sh->gu_soa == m->gu_soa && sh->down_layout == m->down_layout && c.use_silu);
    const int nblk = c.hidden_size / QK_K, nb = c.intermediate_size / QK_K;
    bool fused = env_fused() && qlen <= kBlockMaxTokens && sh_ok && c.gate_type == KTB200_TYPE_Q4_K && c.up_type == KTB200_TYPE_Q4_K &&
                 (fd == FMT_Q6K4T || fd == FMT_Q4K) && nblk >= 16 && nblk <= 32 && c.hidden_size % 4 == 0 && k <= 31 &&
                 gc->n_experts <= kGateThreads * kGateEPT && gc->n_experts > 0 && gc->n_group >= 1 && gc->n_group <= 32 &&
                 gc->n_experts % gc->n_group == 0 && gc->topk_group >= 1 && gc->topk_group <= gc->n_group && gc->weight &&
                 gc->scoring >= 0 && gc->scoring <= 1 && gc->topk_method >= 0 && gc->topk_method <= 2 && k <= gc->n_experts;
    DeviceGuard guard(m->device);
    const int dev = m->device;
    cudaStream_t s = (cudaStream_t)stream;
    BlockParams p{};
    size_t smem = 0;
    int W = 0, G = 0;
    if (fused) {
        const int ns = k + (sh ? 1 : 0);
        const int kbs = fd == FMT_Q6K4T ? 16 : 8, bbytes = fd == FMT_Q6K4T ? SZ_Q6_K : SZ_Q4_K;
        const size_t item = (size_t)4 * nb * bbytes, row = (size_t)nblk * SZ_Q4_K;
        G = num_sms(dev);
        if (G > c.intermediate_size) G = c.intermediate_size;
        if (G > c.hidden_size / 4) G = c.hidden_size / 4;
        const int quads = c.hidden_size / 4;
        p.nrows_max = ((quads + G - 1) / G) * 4;
        const size_t xq = (((size_t)nblk * (kActBlkStride + 16 + 4) + 15) & ~(size_t)15) + ((size_t)2 * gc->n_experts + 32 + 4 * kGateWarps) * 4;
        const size_t aqb = (size_t)ns * nb * (kActBlkStride + 2 * kbs + 4);
        p.region_a = (int)(((xq > aqb ? xq : aqb) + 15) & ~(size_t)15);
        size_t base = (size_t)kBlockSharedBytes + p.region_a + (size_t)p.nrows_max * ns * 4;
        base = (base + 15) & ~(size_t)15;
        // 12 warps x (4 rows | 2 tiles) with 168 registers by default; KTB200_BLK_WARPS=15: 15 warps x (3 rows | 2 tiles), 128 registers
        static const int want_w = [] { const char* e = getenv("KTB200_BLK_WARPS"); return e ? atoi(e) : kBlockWarpsLo; }();
        const int su = want_w > kBlockWarpsLo ? 3 : 4;
        size_t ring = su * row > 2 * item ? su * row : 2 * item;
        p.ring_bytes = (int)ring;
        W = base + 64 < 232448 - 1024 ? (int)((232448 - 1024 - base - 16) / (ring + 8 * su)) : 0;
        if (W > (want_w > kBlockWarpsLo ? kBlockWarps : kBlockWarpsLo)) W = want_w > kBlockWarpsLo ? kBlockWarps : kBlockWarpsLo;
        if (want_w >= 8 && W > want_w) W = want_w;
        if (want_w > kBlockWarpsLo && W <= kBlockWarpsLo) W = 0;   // the 3-row ring needs the 15-warp kernel
        smem = base + (((size_t)W * su * 8 + 15) & ~(size_t)15) + (size_t)W * ring;
        if (W < 8 || c.hidden_size % 4 || item % 16 || c.intermediate_size < 1) fused = false;
    }
    if (!fused) {
        int rc = ktb200_moe_gate_forward(gc, qlen, input, idx, w, nullptr, bsz, stream);
        if (rc) return rc;
        return ktb200_moe_forward_shared(m, sh, qlen, k, idx, w, input, output, bsz, stream);
    }

    const int S = gate_splits(gc->n_experts, gc->hidden_size, num_sms(dev));
    p.g = GateParams{gc->weight, input, gc->hidden_type, gc->n_experts, gc->hidden_size, qlen, S, k, gc->n_group, gc->topk_group,
                     gc->scoring, gc->topk_method, gc->norm_topk_prob, gc->routed_scaling_factor, gc->bias, m->blk_partial, nullptr,
                     idx, w, bsz, nullptr};
    p.w_gate = c.gate_proj; p.w_up = c.up_proj; p.w_down = c.down_proj;
    p.s_gate = sh ? sh->gate : nullptr; p.s_up = sh ? sh->up : nullptr; p.s_down = sh ? sh->down : nullptr;
    p.n_local = c.expert_num; p.id_offset = c.expert_id_offset;
    p.H = c.hidden_size; p.I = c.intermediate_size; p.k = k; p.hidden_type = c.hidden_type; p.use_silu = c.use_silu;
    const unsigned flip = m->blk_flip++ & 1u;
    p.inter = m->blk_inter; p.out = output; p.sync = m->blk_sync + 2 * flip; p.trace = g_btrace;
    p.status = m->blk_sync + kBlkStatusWord;
    p.ready = m->blk_sync + kBlkReadyWord + flip * blk_ready_words(c);
    p.stage_q = m->blk_stage;
    p.stage_bs = reinterpret_cast<int16_t*>(m->blk_stage + blk_ready_words(c) * (size_t)QK_K);
    p.stage_d = reinterpret_cast<float*>(m->blk_stage + blk_ready_words(c) * (size_t)(QK_K + 32));
    for (int r = 0; r < 3; r++) { p.pf[r] = (const uint8_t*)m->pf[r]; p.pf_bytes[r] = (unsigned)m->pf_bytes[r]; }
    static const int prime_u = [] { const char* e = getenv("KTB200_BLK_PRIME_U"); return e ? atoi(e) : 3; }();
    p.prime_u = prime_u;

    void* args[] = {&p};
    const void* fn;
    if (W > kBlockWarpsLo) fn = fd == FMT_Q6K4T ? (const void*)moe_block_kernel<BulkQ6K4T, kBlockWarps> : (const void*)moe_block_kernel<BulkQ4K, kBlockWarps>;
    else fn = fd == FMT_Q6K4T ? (const void*)moe_block_kernel<BulkQ6K4T, kBlockWarpsLo> : (const void*)moe_block_kernel<BulkQ4K, kBlockWarpsLo>;
    static const int coop = [] { const char* e = getenv("KTB200_BLK_COOP"); return e ? atoi(e) : 1; }();
    static const int pdl = [] { const char* e = getenv("KTB200_BLK_PDL"); return e ? atoi(e) : 1; }();
    auto separate = [&]() -> int {   // the same results from the separate launches (no grid barrier: nothing can hang)
        int rc = ktb200_moe_gate_forward(gc, qlen, input, idx, w, nullptr, bsz, stream);
        if (rc) return rc;
        return ktb200_moe_forward_shared(m, sh, qlen, k, idx, w, input, output, bsz, stream);
    };
    {   // once per (variant, device): raise the dynamic shared-memory limit and check that the G CTAs CAN be co-resident —
        // the spin grid barriers need all of them on the SMs at the same time (1 CTA / SM at this shared-memory size)
        static size_t limit[4][64] = {};
        static int resident[4][64] = {};
        const int v = (W > kBlockWarpsLo ? 2 : 0) + (fd == FMT_Q6K4T ? 1 : 0);
        if (limit[v][dev & 63] < smem) {
            KTB_CUDA_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            int per_sm = 0;
            KTB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, W * 32, smem));
            resident[v][dev & 63] = per_sm * num_sms(dev);
            limit[v][dev & 63] = smem;
        }
        if (resident[v][dev & 63] < G) return separate();
    }
    // Launch attributes.  Cooperative (library default): the driver guarantees co-residency of the G <= #SM CTAs or REFUSES
    // the launch (cudaErrorCooperativeLaunchTooLarge: MPS thread percentage, green contexts ...) — then the separate
    // launches run.  KTB200_BLK_COOP=0 is the caller's statement that this process decodes on one stream and owns the
    // GPU (bench.py): a plain grid of G <= occupancy * #SM CTAs (checked above) is co-resident as soon as the previous
    // kernel's CTAs exit.  Programmatic stream serialization (KTB200_BLK_PDL=0 to disable): see griddep_wait().
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(G); lc.blockDim = dim3(W * 32); lc.dynamicSmemBytes = smem; lc.stream = s;
    cudaLaunchAttribute at[2];
    int na = 0;
    if (coop) { at[na].id = cudaLaunchAttributeCooperative; at[na].val.cooperative = 1; na++; }
    if (pdl) { at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[na].val.programmaticStreamSerializationAllowed = 1; na++; }
    lc.attrs = at; lc.numAttrs = na;
    cudaError_t le = cudaLaunchKernelExC(&lc, fn, args);
    if (le != cudaSuccess && coop && pdl && (le == cudaErrorNotSupported || le == cudaErrorInvalidValue)) {
        // cooperative + programmatic together are not accepted by every driver: keep the co-residency guarantee, drop the overlap
        (void)cudaGetLastError();
        lc.numAttrs = 1;
        le = cudaLaunchKernelExC(&lc, fn, args);
    }
    if (le == cudaErrorCooperativeLaunchTooLarge) {   // the driver cannot make the grid co-resident right now
        (void)cudaGetLastError();
        return separate();
    }
    if (le != cudaSuccess) { set_error("moe_block launch failed: %s", cudaGetErrorString(le)); return KTB200_ECUDA; }
    count_launch(1);
    return KTB200_OK;
}

extern "C" long ktb200_ep_msg_bytes(int hidden_size, int hidden_type) { return (long)hidden_size * type_size(hidden_type) + 128; }

namespace ktb {
// the router configurations the persistent kernels' grouped top-k (gate_select_token) takes
static bool ep_gate_ok(const ktb200_gate_config* gc, int k) {
    return gc->n_experts <= kGateThreads * kGateEPT && gc->n_experts > 0 && gc->n_group >= 1 && gc->n_group <= 32 &&
           gc->n_experts % gc->n_group == 0 && gc->topk_group >= 1 && gc->topk_group <= gc->n_group && gc->weight && gc->scoring >= 0 &&
           gc->scoring <= 1 && gc->topk_method >= 0 && gc->topk_method <= 2 && k <= gc->n_experts;
}

// Fills everything of an expert-parallel launch but the plan (nrows_max, region_a, ring_bytes, pa, ep_off).
static int ep_block_params(EpParams& pp, const ktb200_gate_config* gc, ktb200_moe* m, ktb200_mlp* sh, const ktb200_ep_comm* comm,
                           const void* x_own, void* y_out, int64_t* idx, float* w, int phase_mask) {
    const ktb200_moe_config& c = m->cfg;
    const int k = gc->top_k, world = comm->world;
    BlockParams& p = pp.b;
    const int S = gate_splits(gc->n_experts, gc->hidden_size, num_sms(m->device));
    p.g = GateParams{gc->weight, x_own, gc->hidden_type, gc->n_experts, gc->hidden_size, 1, S, k, gc->n_group, gc->topk_group,
                     gc->scoring, gc->topk_method, gc->norm_topk_prob, gc->routed_scaling_factor, gc->bias, m->blk_partial, nullptr,
                     idx, w, nullptr, nullptr};
    p.w_gate = c.gate_proj; p.w_up = c.up_proj; p.w_down = c.down_proj;
    p.s_gate = sh ? sh->gate : nullptr; p.s_up = sh ? sh->up : nullptr; p.s_down = sh ? sh->down : nullptr;
    p.n_local = c.expert_num; p.id_offset = c.expert_id_offset;
    p.H = c.hidden_size; p.I = c.intermediate_size; p.k = k; p.hidden_type = c.hidden_type; p.use_silu = c.use_silu;
    p.inter = m->inter; p.out = y_out; p.sync = m->blk_sync + 2 * (m->blk_flip++ & 1u); p.trace = g_btrace;
    p.prime_u = 3; p.prime_d = 2;
    pp.x.rank = comm->rank; pp.x.world = world; pp.x.phase_mask = phase_mask;
    pp.x.msg_bytes = (int)ktb200_ep_msg_bytes(c.hidden_size, c.hidden_type);
    pp.x.inter_shared_row = world * k;
    pp.x.shared_out = m->blk_partial + 16384;
    for (int r = 0; r < world; r++) {
        if (!comm->token_bufs[r] || !comm->partial_bufs[r] || !comm->flag_bufs[r]) { set_error("ep_block: null peer pointer for rank %d", r); return KTB200_EINVAL; }
        pp.x.msg[r] = (uint8_t*)comm->token_bufs[r]; pp.x.part[r] = comm->partial_bufs[r]; pp.x.flags[r] = comm->flag_bufs[r];
    }
    return KTB200_OK;
}

// Once per (variant, device): raise the kernel's dynamic shared-memory limit and check that the G CTAs can be co-resident
// (the grid barriers spin on all of them).  Variants: 0 / 1 the Q4_K kernels (Q4_K / Q6_K down), 2 .. 9 the Q2_K / Q3_K ones.
static int ep_block_resident(const void* fn, int variant, int G, int W, size_t smem, int dev) {
    static size_t limit[10][64] = {};
    static int resident[10][64] = {};
    if (limit[variant][dev & 63] < smem) {
        KTB_CUDA_CHECK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int per_sm = 0;
        KTB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, W * 32, smem));
        resident[variant][dev & 63] = per_sm * num_sms(dev);
        limit[variant][dev & 63] = smem;
    }
    if (resident[variant][dev & 63] < G) { set_error("ep_block: %d CTAs cannot be co-resident on this device", G); return KTB200_EINVAL; }
    return KTB200_OK;
}

// Cooperative launch with programmatic stream serialization (the cooperative attribute alone where a driver refuses both).
static int ep_block_launch(const void* fn, int G, int W, size_t smem, EpParams& pp, cudaStream_t s) {
    static const int coop = [] { const char* e = getenv("KTB200_BLK_COOP"); return e ? atoi(e) : 1; }();
    static const int pdl = [] { const char* e = getenv("KTB200_BLK_PDL"); return e ? atoi(e) : 1; }();
    void* args[] = {&pp};
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(G); lc.blockDim = dim3(W * 32); lc.dynamicSmemBytes = smem; lc.stream = s;
    cudaLaunchAttribute at[2];
    int na = 0;
    if (coop) { at[na].id = cudaLaunchAttributeCooperative; at[na].val.cooperative = 1; na++; }
    if (pdl) { at[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; at[na].val.programmaticStreamSerializationAllowed = 1; na++; }
    lc.attrs = at; lc.numAttrs = na;
    cudaError_t le = cudaLaunchKernelExC(&lc, fn, args);
    if (le != cudaSuccess && coop && pdl && (le == cudaErrorNotSupported || le == cudaErrorInvalidValue)) {
        (void)cudaGetLastError();
        lc.numAttrs = 1;
        le = cudaLaunchKernelExC(&lc, fn, args);
    }
    if (le != cudaSuccess) { set_error("ep_block launch failed: %s", cudaGetErrorString(le)); return KTB200_ECUDA; }
    count_launch(1);
    return KTB200_OK;
}

// Shared-memory plan of moe_ep_block_kernel<GU, D> (layout at the kernel): the most warps (12 down to 4), then for them the
// largest down chunk pa (16 down to 2), within the opt-in limit.  False when no such pair fits.
struct EpKqPlan { int W, pa; size_t region_a, ep_off, smem; };
static bool ep_kq_plan(int nblk, int nb, int n_experts, int gu_kbs, int gu_block, int d_kbs, int d_block, int nrows_max, EpKqPlan& pl) {
    const size_t cap = 232448 - 1024;
    const size_t unit = (size_t)2 * nblk * gu_block, item = (size_t)4 * nb * d_block;
    const size_t ring = kEpKqSlots * (2 * unit > item ? 2 * unit : item);
    // blk_select's scratch sits behind one Q8_K row of 8 sums per block; two rows of GU's layout; pa entries of D's
    const size_t sel = ep_x_slot_bytes<8>(nblk) + ((size_t)2 * n_experts + 32 + 4 * kGateWarps) * 4;
    const size_t x2 = (size_t)2 * (((size_t)nblk * (kActBlkStride + 2 * gu_kbs + 4) + 15) & ~(size_t)15);
    for (int W = kBlockWarpsLo; W >= 4; W--) {
        for (int pa = 16; pa >= 2; pa--) {
            size_t ra = sel > x2 ? sel : x2;
            const size_t aqb = (size_t)pa * nb * (kActBlkStride + 2 * d_kbs + 4);
            if (aqb > ra) ra = aqb;
            ra = (ra + 15) & ~(size_t)15;
            const size_t ep_off = ((size_t)kBlockSharedBytes + ra + 15) & ~(size_t)15;
            size_t off = ep_off + ((sizeof(EpShared) + 15) & ~(size_t)15) + (size_t)nrows_max * (kEpWorldMax + pa) * 4;
            off = (off + 15) & ~(size_t)15;
            const size_t smem = off + (((size_t)W * kEpKqSlots * 8 + 15) & ~(size_t)15) + (size_t)W * ring;
            if (smem <= cap) { pl = EpKqPlan{W, pa, ra, ep_off, smem}; return true; }
        }
    }
    return false;
}

static const char* kq_name(int t) {
    return t == KTB200_TYPE_Q2_K ? "Q2_K" : t == KTB200_TYPE_Q3_K ? "Q3_K" : t == KTB200_TYPE_Q4_K ? "Q4_K" : "Q6_K";
}

template <class GU>
static const void* ep_kq_kernel(int down_fmt, int down_type) {
    if (down_fmt == FMT_Q4K) return (const void*)moe_ep_block_kernel<GU, BulkQ4K>;
    if (down_fmt == FMT_Q6K4T) return (const void*)moe_ep_block_kernel<GU, BulkQ6K4T>;
    return down_type == KTB200_TYPE_Q2_K ? (const void*)moe_ep_block_kernel<GU, BulkQ2K> : (const void*)moe_ep_block_kernel<GU, BulkQ3K>;
}

// Q2_K / Q3_K routed gate/up (ktb200_moe_ep_block_forward has checked the arguments every configuration shares)
static int ep_block_kq_forward(const ktb200_gate_config* gc, ktb200_moe* m, ktb200_mlp* sh, const ktb200_ep_comm* comm, const void* x_own,
                               void* y_out, int64_t* idx, float* w, int phase_mask, void* stream, FmtId fd) {
    const ktb200_moe_config& c = m->cfg;
    const int k = gc->top_k, world = comm->world;
    const int nblk = c.hidden_size / QK_K, nb = c.intermediate_size / QK_K;
    const bool q2 = c.gate_type == KTB200_TYPE_Q2_K;
    if (sh && (sh->H != c.hidden_size || sh->hidden_type != c.hidden_type)) {
        set_error("ep_block: the shared expert's hidden size / type differ from the routed experts'"); return KTB200_EINVAL;
    }
    if (!ep_gate_ok(gc, k) || nblk % BulkQ2K::kNblkMultiple || nblk < 4 || c.hidden_size > 16384 || c.hidden_size % 16) {
        set_error("ep_block: unsupported configuration (Q2_K / Q3_K gate/up rows need a multiple of 1024 columns, at most 16384)");
        return KTB200_EINVAL;
    }
    const int d_kbs = fd == FMT_Q6K4T ? BulkQ6K4T::kBs : fd == FMT_Q4K ? BulkQ4K::kBs : c.down_type == KTB200_TYPE_Q2_K ? BulkQ2K::kBs : BulkQ3K::kBs;
    const int d_block = fd == FMT_Q6K4T ? SZ_Q6_K : fd == FMT_Q4K ? SZ_Q4_K : c.down_type == KTB200_TYPE_Q2_K ? SZ_Q2_K : SZ_Q3_K;
    if ((size_t)4 * nb * d_block % 16) { set_error("ep_block: %s down rows of %d blocks: a 4-row item is not 16-byte sized", kq_name(c.down_type), nb); return KTB200_EINVAL; }
    const int dev = m->device;
    int G = num_sms(dev);
    if (G > c.intermediate_size / 2) G = c.intermediate_size / 2;
    if (G > c.hidden_size / 4) G = c.hidden_size / 4;
    if (world * k >= G) { set_error("ep_block: grid too small for %d pairs", world * k); return KTB200_EINVAL; }
    EpParams pp{};
    BlockParams& p = pp.b;
    p.nrows_max = ((c.hidden_size / 4 + G - 1) / G) * 4;
    EpKqPlan pl;
    if (!ep_kq_plan(nblk, nb, gc->n_experts, q2 ? BulkQ2K::kBs : BulkQ3K::kBs, q2 ? SZ_Q2_K : SZ_Q3_K, d_kbs, d_block, p.nrows_max, pl)) {
        set_error("ep_block: %s gate/up rows of %d columns and %s down rows of %d columns leave no room for 4 warps and 2 down "
                  "entries in shared memory", kq_name(c.gate_type), c.hidden_size, kq_name(c.down_type), c.intermediate_size);
        return KTB200_EINVAL;
    }
    int rc = ep_block_params(pp, gc, m, sh, comm, x_own, y_out, idx, w, phase_mask);
    if (rc) return rc;
    const size_t unit = (size_t)2 * nblk * (q2 ? SZ_Q2_K : SZ_Q3_K), item = (size_t)4 * nb * d_block;
    p.ring_bytes = (int)(kEpKqSlots * (2 * unit > item ? 2 * unit : item));
    p.region_a = (int)pl.region_a;
    pp.x.pa = pl.pa;
    pp.x.ep_off = (int)pl.ep_off;
    const void* fn = q2 ? ep_kq_kernel<BulkQ2K>(fd, c.down_type) : ep_kq_kernel<BulkQ3K>(fd, c.down_type);
    const int variant = 2 + (q2 ? 0 : 4) + (fd == FMT_Q4K ? 0 : fd == FMT_Q6K4T ? 1 : c.down_type == KTB200_TYPE_Q2_K ? 2 : 3);
    rc = ep_block_resident(fn, variant, G, pl.W, pl.smem, dev);
    if (rc) return rc;
    // the shared expert's rounded output goes into y first, with the combine phase (whose sum adds to it)
    if (sh && (phase_mask & 4)) {
        rc = ktb200_mlp_forward(sh, 1, x_own, y_out, 0, nullptr, stream);
        if (rc) return rc;
    }
    return ep_block_launch(fn, G, pl.W, pl.smem, pp, (cudaStream_t)stream);
}
}  // namespace ktb

extern "C" int ktb200_moe_ep_block_forward(const ktb200_gate_config* gc, ktb200_moe* m, ktb200_mlp* sh, const ktb200_ep_comm* comm,
                                           const void* x_own, void* y_out, int64_t* idx, float* w, int phase_mask, void* stream) {
    if (!gc || !m || !comm || !x_own || !y_out || !idx || !w) { set_error("ep_block: null pointer"); return KTB200_EINVAL; }
    if (!m->loaded || (sh && !sh->loaded)) { set_error("Not Loaded"); return KTB200_ESTATE; }
    const ktb200_moe_config& c = m->cfg;
    const int k = gc->top_k, world = comm->world, rank = comm->rank;
    if (world < 1 || world > kEpWorldMax || rank < 0 || rank >= world) { set_error("ep_block: world must be 1..%d", kEpWorldMax); return KTB200_EINVAL; }
    if (phase_mask <= 0 || phase_mask > 7) phase_mask = 7;
    if (gc->hidden_size != c.hidden_size || gc->hidden_type != c.hidden_type || comm->hidden_size != c.hidden_size || comm->hidden_type != c.hidden_type) {
        set_error("ep_block: gate / experts / comm disagree on the hidden size or type"); return KTB200_EINVAL;
    }
    if (k <= 0 || k > c.routed_expert_num || k > 16 || world * k > kEpPairsMax) { set_error("ep_block: top_k=%d (<= 16, world * top_k <= %d)", k, kEpPairsMax); return KTB200_EINVAL; }
    if (c.group_max_len < world) { set_error("ep_block: group_max_len=%d must be >= world=%d (scratch rows)", c.group_max_len, world); return KTB200_EINVAL; }
    if (is_rawint4(c.gate_type)) { set_error("ep_block: RAWINT4_G32 experts are not supported by the expert-parallel kernel"); return KTB200_EINVAL; }
    for (int t : {c.gate_type, c.up_type, c.down_type})
        if (is_iquant(t)) { set_error("ep_block: %s experts are not supported by the expert-parallel kernel", iquant_name(t)); return KTB200_EINVAL; }
    const FmtId fd = pick_fmt(c.down_type, m->down_layout);
    DeviceGuard guard(m->device);
    if ((c.gate_type == KTB200_TYPE_Q2_K || c.gate_type == KTB200_TYPE_Q3_K) && c.up_type == c.gate_type &&
        (fd == FMT_Q4K || fd == FMT_Q6K4T || c.down_type == KTB200_TYPE_Q2_K || c.down_type == KTB200_TYPE_Q3_K))
        return ep_block_kq_forward(gc, m, sh, comm, x_own, y_out, idx, w, phase_mask, stream, fd);
    const bool sh_ok = !sh || (sh->H == c.hidden_size && sh->I == c.intermediate_size && sh->hidden_type == c.hidden_type &&
                               sh->gate_type == c.gate_type && sh->up_type == c.up_type && sh->down_type == c.down_type &&
                               sh->gu_soa == m->gu_soa && sh->down_layout == m->down_layout && c.use_silu);
    const int nblk = c.hidden_size / QK_K, nb = c.intermediate_size / QK_K;
    const bool ok = sh_ok && c.gate_type == KTB200_TYPE_Q4_K && c.up_type == KTB200_TYPE_Q4_K && (fd == FMT_Q6K4T || fd == FMT_Q4K) && nblk >= 16 &&
                    nblk <= 32 && c.hidden_size % 16 == 0 && ep_gate_ok(gc, k) && c.hidden_size <= 16384;
    if (!ok) { set_error("ep_block: unsupported configuration (needs Q4_K gate/up rows of 4096..8192 columns, Q6_K/Q4_K down, shared expert of the same shapes)"); return KTB200_EINVAL; }
    const int dev = m->device;
    EpParams pp{};
    BlockParams& p = pp.b;
    const int ns = k + (sh ? 1 : 0);
    const int kbs = fd == FMT_Q6K4T ? 16 : 8, bbytes = fd == FMT_Q6K4T ? SZ_Q6_K : SZ_Q4_K;
    const size_t item = (size_t)4 * nb * bbytes, row = (size_t)nblk * SZ_Q4_K;
    int G = num_sms(dev);
    if (G > c.intermediate_size) G = c.intermediate_size;
    if (G > c.hidden_size / 4) G = c.hidden_size / 4;
    if (world * k >= G || item % 16) { set_error("ep_block: grid too small for %d pairs", world * k); return KTB200_EINVAL; }
    const int quads = c.hidden_size / 4;
    p.nrows_max = ((quads + G - 1) / G) * 4;
    const int W = kBlockWarpsLo, su = 4;
    const size_t ring = su * row > 2 * item ? su * row : 2 * item;
    p.ring_bytes = (int)ring;
    const size_t x_slot = (((size_t)nblk * (kActBlkStride + 16 + 4)) + 15) & ~(size_t)15;
    const size_t sel = ((size_t)2 * gc->n_experts + 32 + 4 * kGateWarps) * 4;
    size_t smem = 0;
    int pa = 0;
    for (int cand = 16; cand >= 2; cand--) {
        size_t ra = x_slot + sel > 2 * x_slot ? x_slot + sel : 2 * x_slot;
        const size_t aqb = (size_t)cand * nb * (kActBlkStride + 2 * kbs + 4);
        if (aqb > ra) ra = aqb;
        ra = (ra + 15) & ~(size_t)15;
        size_t off = ((size_t)kBlockSharedBytes + ra + (size_t)p.nrows_max * ns * 4 + 15) & ~(size_t)15;   // == BlockLay::ring_off
        off += (((size_t)W * su * 8 + 15) & ~(size_t)15) + (size_t)W * ring;
        off = (off + 15) & ~(size_t)15;
        const size_t tail = ((sizeof(EpShared) + 15) & ~(size_t)15) + (size_t)p.nrows_max * (kEpWorldMax + 1 + cand) * 4;
        if (off + tail <= 232448 - 1024) { pa = cand; p.region_a = (int)ra; pp.x.ep_off = (int)off; smem = off + tail; break; }
    }
    if (pa < 2) { set_error("ep_block: shared memory budget"); return KTB200_EINVAL; }
    const int rc = ep_block_params(pp, gc, m, sh, comm, x_own, y_out, idx, w, phase_mask);
    if (rc) return rc;
    pp.x.pa = pa;
    const void* fn = fd == FMT_Q6K4T ? (const void*)moe_ep_block_kernel<BulkQ6K4T> : (const void*)moe_ep_block_kernel<BulkQ4K>;
    const int rr = ep_block_resident(fn, fd == FMT_Q6K4T ? 1 : 0, G, W, smem, dev);
    if (rr) return rr;
    return ep_block_launch(fn, G, W, smem, pp, (cudaStream_t)stream);
}

// Prefetch hint: while this handle's block kernel streams its down projection, pull up to three byte ranges into L2 — the
// caller passes what the NEXT layer's launch reads first (its router weight, its shared expert's gate / up tensors).
// While the down stream already saturates HBM the prefetch competes with it, so bench.py leaves it off (KTB200_BENCH_PREFETCH);
// kept for callers whose next layer is not back to back.
extern "C" int ktb200_moe_block_prefetch_hint(ktb200_moe* m, const void* const* ptrs, const size_t* bytes, int n) {
    if (!m || n < 0 || n > 3 || (n && (!ptrs || !bytes))) { set_error("prefetch_hint: up to 3 ranges"); return KTB200_EINVAL; }
    for (int r = 0; r < 3; r++) {
        m->pf[r] = r < n ? ptrs[r] : nullptr;
        m->pf_bytes[r] = r < n ? (bytes[r] > 0xfffffff0u ? 0xfffffff0u : bytes[r]) : 0;
        if (r < n && ((uintptr_t)ptrs[r] & 15)) { set_error("prefetch_hint: ranges must be 16-byte aligned"); m->pf[r] = nullptr; return KTB200_EINVAL; }
    }
    return KTB200_OK;
}

// Host-buffer form of the same call (the shape of the reference's CPU operator: pinned host tensors in, host tensors
// out, cpuinfer.submit + sync — experts.py:293-318): H2D of the tokens, the block, D2H of the result and the routing.
extern "C" int ktb200_moe_block_forward_host(const ktb200_gate_config* gc, ktb200_moe* m, ktb200_mlp* sh, int qlen, const void* input,
                                             void* output, int64_t* idx, float* w, void* stream) {
    if (!gc || !m || !input || !output) { set_error("null pointer"); return KTB200_EINVAL; }
    if (qlen <= 0) return KTB200_OK;
    const ktb200_moe_config& c = m->cfg;
    const int k = gc->top_k;
    if (qlen > c.group_max_len || k <= 0 || k > c.routed_expert_num) { set_error("forward_host: qlen/k out of range"); return KTB200_EINVAL; }
    DeviceGuard guard(m->device);
    cudaStream_t s = (cudaStream_t)stream;
    const size_t hid = (size_t)qlen * c.hidden_size * type_size(c.hidden_type);
    KTB_CUDA_CHECK(cudaMemcpyAsync(m->in_d, input, hid, cudaMemcpyHostToDevice, s));
    // a pinned (mapped) output buffer is written by the kernel's own stores — the device-to-host transfer without a copy-engine
    // launch behind the kernel; pageable memory takes the staged copy
    void* out_dev = m->out_d;
    cudaPointerAttributes pa;
    if (cudaPointerGetAttributes(&pa, output) == cudaSuccess && pa.type == cudaMemoryTypeHost && pa.devicePointer) out_dev = pa.devicePointer;
    else (void)cudaGetLastError();
    int rc = ktb200_moe_block_forward(gc, m, sh, qlen, m->in_d, out_dev, m->ids_d, m->w_d, nullptr, stream);
    if (rc) return rc;
    if (out_dev == m->out_d) KTB_CUDA_CHECK(cudaMemcpyAsync(output, m->out_d, hid, cudaMemcpyDeviceToHost, s));
    if (idx) KTB_CUDA_CHECK(cudaMemcpyAsync(idx, m->ids_d, (size_t)qlen * k * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    if (w) KTB_CUDA_CHECK(cudaMemcpyAsync(w, m->w_d, (size_t)qlen * k * sizeof(float), cudaMemcpyDeviceToHost, s));
    KTB_CUDA_CHECK(cudaStreamSynchronize(s));
    return KTB200_OK;
}

// Diagnostics (profiles/block_trace.py): when set, thread 0 of every CTA of the following ktb200_moe_block_forward
// launches writes %globaltimer at the phase boundaries into trace[cta][16] (device memory, >= num_SMs*16 u64).
extern "C" void ktb200_debug_block_trace(unsigned long long* trace_dev) { g_btrace = trace_dev; }

extern "C" long ktb200_debug_block_sync_words(ktb200_moe* m, unsigned* host_out, long n) {
    if (!m) { set_error("null handle"); return -1; }
    const long total = (long)(kBlkReadyWord + 2 * blk_ready_words(m->cfg));
    DeviceGuard guard(m->device);
    if (host_out && n > 0) {
        if (cudaDeviceSynchronize() != cudaSuccess ||
            cudaMemcpy(host_out, m->blk_sync, (size_t)(n < total ? n : total) * sizeof(unsigned), cudaMemcpyDeviceToHost) != cudaSuccess) {
            set_error("debug_block_sync_words: %s", cudaGetErrorString(cudaGetLastError()));
            return -1;
        }
    }
    return total;
}
