// The scaffolding the bulk-copy ring kernels share (gemv_bulk.cuh, iq.cuh, rawint4.cuh, dense_bulk.cuh): the mbarrier / bulk-copy
// PTX, the per-warp ring of slots, the warp's share of a CTA's units, the per-chunk (token, slot) work lists and the Q8_K
// activation staging loop.  Everything is forceinline with plain-integer cursors, so nvcc's scalar replacement leaves no
// structs or lambdas in the kernels.  The instructions are not those of the earlier hand-written copies: ptxas allocates a few
// registers more or fewer per instantiation (DESIGN.md §4.2), with no spills.
#pragma once
#include "gemv_pipe.cuh"

namespace ktb {

constexpr int kActBlkStride = QK_K + 16;   // int8 activation blocks padded to 272 B: 8 lanes x LDS.128 hit 32 distinct banks
constexpr int kBulkMaxChunkTokens = 16;    // down kernels: tokens per chunk (s_first has one entry more)

// ---------------------------------------------------------------------------------------------------------------
// mbarrier / bulk-copy PTX
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// global -> shared bulk copy (size and both addresses multiples of 16 B); completion is signalled on `bar`
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
                 "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}" ::"r"(bar),
        "r"(parity)
        : "memory");
}

// ---------------------------------------------------------------------------------------------------------------
// A warp's private ring of SLOTS slots of `slot_bytes`, each filled by bulk copies and tracked by one mbarrier.  Dynamic shared
// memory from byte `head` (rounded up to 16): [W x SLOTS mbarriers, padded to 16 B] [W x SLOTS slots], warp by warp.  This is
// the layout plan_ring (moe.cu) sizes; a change here is a change there.  The issue and use cursors advance in lock step over
// the whole launch: SLOTS - 1 slots are in flight behind the one being consumed.
template <int SLOTS>
struct BulkRing {
    uint8_t* ring;            // the warp's first slot
    uint32_t bar, ring_u32;   // shared-window addresses of the warp's first mbarrier and first slot
    int slot_bytes;
    int slot_i = 0, slot_u = 0;   // next slot to fill / to consume
    uint32_t phase = 0;           // bit s = parity the next use of slot s waits for

    __device__ __forceinline__ BulkRing(uint8_t* smem, size_t head, int slot_bytes_, int lane, int warp, int W)
        : slot_bytes(slot_bytes_) {
        const size_t off = (head + 15) & ~(size_t)15;
        const int bar_bytes = (W * SLOTS * 8 + 15) & ~15;
        bar = (uint32_t)__cvta_generic_to_shared(smem + off) + warp * SLOTS * 8;
        ring = smem + off + bar_bytes + (size_t)warp * SLOTS * slot_bytes;
        ring_u32 = (uint32_t)__cvta_generic_to_shared(ring);
        if (lane == 0) {
#pragma unroll
            for (int s = 0; s < SLOTS; s++) mbar_init(bar + 8 * s, 1);
            mbar_fence_init();
            fence_proxy_async_smem();
        }
    }
    // Fill the next slot with `ncopy` (1 or 2, a constant at every call) bulk copies of `bytes` each, copy c from src(c) into
    // part c of the slot (gate and up rows side by side).  Lane 0 alone evaluates src and issues; every lane moves the cursor on.
    template <class SrcFn>
    __device__ __forceinline__ void issue(int lane, int ncopy, uint32_t bytes, SrcFn&& src) {
        if (lane == 0) {
            const void* s0 = src(0);
            const void* s1 = ncopy > 1 ? src(1) : nullptr;
            const uint32_t b = bar + 8 * slot_i, dst = ring_u32 + slot_i * slot_bytes;
            mbar_expect_tx(b, ncopy * bytes);
            bulk_g2s(dst, s0, bytes, b);
            if (ncopy > 1) bulk_g2s(dst + bytes, s1, bytes, b);
        }
        slot_i = (slot_i + 1 == SLOTS) ? 0 : slot_i + 1;
    }
    // wait for the slot to consume; returns its address
    __device__ __forceinline__ const uint8_t* wait() {
        mbar_wait(bar + 8 * slot_u, (phase >> slot_u) & 1u);
        phase ^= 1u << slot_u;
        return ring + slot_u * slot_bytes;
    }
    // every lane is done reading the slot: hand it back to the copy engine
    __device__ __forceinline__ void release() {
        __syncwarp();
        slot_u = (slot_u + 1 == SLOTS) ? 0 : slot_u + 1;
    }
};

// ---------------------------------------------------------------------------------------------------------------
// Work split: a CTA owns the contiguous units [u0, u1), warp w of W takes u0 + w, u0 + w + W, ...  Units are pair-major
// (unit = pair * per + row), and a cursor walks them as (pair, row) with one division at the start.
__device__ __forceinline__ int warp_units(int u0, int u1, int warp, int W) {
    const int nu = u1 - u0 - warp;
    return nu > 0 ? (nu + W - 1) / W : 0;
}
struct UnitCursor {
    int pi = 0, r = 0;   // pair index, row (or row group) within the pair
    __device__ __forceinline__ void start(int u, int per) { pi = u / per; r = u - pi * per; }
    __device__ __forceinline__ void step(int W, int per) {
        r += W;
        while (r >= per) { r -= per; pi++; }
    }
};

// expert of slot s of token t relative to this launch's shard (0 without ids); owned when in [0, n_experts)
template <class P>
__device__ __forceinline__ long pair_expert(const P& p, long t, int s) {
    return p.ids ? (long)p.ids[t * p.slots + s] - p.id_offset : 0;
}

// Gate/up work list of tokens t0 .. t0 + nt - 1 (thread 0): every owned (token in chunk << 8 | slot) pair in token order, each
// token followed by the shared-expert slot `slots` when `shared` and p.shared_token is < 0 or that token.  Returns the count.
template <class P>
__device__ __forceinline__ int gateup_pairs(const P& p, int t0, int nt, bool shared, int* pairs) {
    int np = 0;
    for (int tl = 0; tl < nt; tl++) {
        for (int s = 0; s < p.slots; s++) {
            const long e = pair_expert(p, t0 + tl, s);
            if (e >= 0 && e < p.n_experts) pairs[np++] = (tl << 8) | s;
        }
        if (shared && (p.shared_token < 0 || p.shared_token == t0 + tl)) pairs[np++] = (tl << 8) | p.slots;
    }
    return np;
}

// Down work list (thread 0): the greedy chunk from token t0, as many tokens (<= kBulkMaxChunkTokens, at least one) as have
// together at most `pcap` owned pairs, the shared slot k = slots last in a token when `shared` and p.shared_token is < 0 or that
// token.  first[tl] = first pair of token tl, first[nt] = np.  Returns nt.
template <class P>
__device__ __forceinline__ int down_pairs(const P& p, int t0, int Teff, int pcap, bool shared, int* pairs, int* first, int& np) {
    const int k = p.slots;
    int nt = 0;
    np = 0;
    while (t0 + nt < Teff && nt < kBulkMaxChunkTokens) {
        const bool sh_here = shared && (p.shared_token < 0 || p.shared_token == t0 + nt);
        int cnt = sh_here ? 1 : 0;
        for (int j = 0; j < k; j++) {
            const long e = pair_expert(p, t0 + nt, j);
            cnt += (e >= 0 && e < p.n_experts) ? 1 : 0;
        }
        if (nt > 0 && np + cnt > pcap) break;
        first[nt] = np;
        for (int j = 0; j < k; j++) {
            const long e = pair_expert(p, t0 + nt, j);
            if (e >= 0 && e < p.n_experts) pairs[np++] = (nt << 8) | j;
        }
        if (sh_here) pairs[np++] = (nt << 8) | k;
        nt++;
    }
    first[nt] = np;
    return nt;
}

// ---------------------------------------------------------------------------------------------------------------
// Q8_K staging of activation blocks 0 .. n-1, block g on warp g % W; each lane loads its 8 values of the warp's next block while
// the current one is quantised.  src(g) = element offset of block g in x; dst(g) = where its padded int8 values, kBs int16 sums
// and scale go.
struct StagedBlock { uint8_t* q8; int16_t* bs; float* dx; };
template <int kBs, class SrcFn, class DstFn>
__device__ __forceinline__ void stage_q8k(const void* x, int hidden_type, int n, int lane, int warp, int W, SrcFn&& src,
                                          DstFn&& dst) {
    float cur[8], nxt[8];
    int g = warp;
    if (g < n) load_block8(x, src(g) + lane * 8, hidden_type, cur);
#pragma unroll 1
    while (g < n) {
        const int gn = g + W;
        if (gn < n) load_block8(x, src(gn) + lane * 8, hidden_type, nxt);
        const StagedBlock d = dst(g);
        warp_quantize_q8k_block(cur, lane, reinterpret_cast<uint32_t*>(d.q8), d.dx, kBs == 16 ? d.bs : nullptr,
                                kBs == 8 ? d.bs : nullptr);
#pragma unroll
        for (int i = 0; i < 8; i++) cur[i] = nxt[i];
        g = gn;
    }
}
// The activation rows t0 .. t0 + nt - 1 of x ([T][ncols]); row tl is staged at smem + tl * act_tok as
// q8 [nblk][272] | int16 sums [nblk][kBs] | scales [nblk]
template <int kBs>
__device__ __forceinline__ void stage_q8k_rows(const void* x, int hidden_type, int t0, int nt, int ncols, uint8_t* smem,
                                               size_t act_tok, int lane, int warp, int W) {
    const int nblk = ncols / QK_K;
    stage_q8k<kBs>(
        x, hidden_type, nt * nblk, lane, warp, W, [&](int g) { return (long)(t0 + g / nblk) * ncols + (long)(g % nblk) * QK_K; },
        [&](int g) {
            const int tl = g / nblk, b = g - tl * nblk;
            uint8_t* at = smem + (size_t)tl * act_tok;
            return StagedBlock{at + (size_t)b * kActBlkStride, reinterpret_cast<int16_t*>(at + (size_t)nblk * kActBlkStride) + b * kBs,
                               reinterpret_cast<float*>(at + (size_t)nblk * (kActBlkStride + 2 * kBs)) + b};
        });
}

}  // namespace ktb
