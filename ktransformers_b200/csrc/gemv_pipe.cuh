// Software-pipelined variant of rows_kernel for long raw-block rows (Q4_K / Q5_K gate+up of a 7168-wide model).
//
// ncu on rows_kernel shows every warp parked on long-scoreboard (global-load) stalls: the bytes a warp can keep in
// flight are bounded by the registers that hold them.  Here the weight rows travel global -> shared memory with
// cp.async (LDGSTS: no register staging): every warp owns a private 2-slot ring, streams the NEXT unit (one gate
// row + one up row, 8 KB) into one slot while it computes on the other, and reads weights back with conflict-free
// LDS.128.  No cross-warp synchronisation in the steady state; 12 warps x 8 KB = 96 KB in flight per SM instead
// of ~32 KB.  Arithmetic, lane mapping and epilogue are those of rows_kernel (same Fmt::dot).
#pragma once
#include "gemv.cuh"

namespace ktb {

__device__ __forceinline__ void cp_async16_cg(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit_group() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <class Fmt, bool PAIR, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 1) rows_pipe_kernel(const RowsParams p, int act_bytes, int slot_bytes) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int t = blockIdx.y;
    if (p.bsz && t >= *p.bsz) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nblk = p.ncols / QK_K;
    const int row_bytes = nblk * Fmt::kBlockBytes;
    constexpr int NM = PAIR ? 2 : 1;
    uint8_t* q8 = smem;
    float* dx = reinterpret_cast<float*>(smem + p.ncols);
    int16_t* bsums = reinterpret_cast<int16_t*>(smem + p.ncols + ((nblk * 4 + 15) & ~15));   // 16-byte aligned
    uint8_t* ring = smem + act_bytes + (size_t)warp * 2 * slot_bytes;
    const uint32_t ring_u32 = (uint32_t)__cvta_generic_to_shared(ring);
    const ActQ8K act{q8, dx, bsums};
    const typename Fmt::Lane L = Fmt::lane(lane);

    const int nslots = p.slots + (p.x0 ? 1 : 0);
    const int total = nslots * p.rows;
    const int u0 = (int)((long)total * blockIdx.x / gridDim.x), u1 = (int)((long)total * (blockIdx.x + 1) / gridDim.x);

    auto unit_rows = [&](int u, const uint8_t* (&r)[NM]) -> bool {
        if (u >= u1) return false;
        const int s = u / p.rows, rr = u - s * p.rows;
        if (s == p.slots) {
            r[0] = reinterpret_cast<const uint8_t*>(p.x0) + (long)rr * row_bytes;
            if (PAIR) r[NM - 1] = reinterpret_cast<const uint8_t*>(p.x1) + (long)rr * row_bytes;
            return true;
        }
        const long e = p.ids ? (long)p.ids[(long)t * p.slots + s] - p.id_offset : 0;
        if (e < 0 || e >= p.n_experts) return false;
        r[0] = reinterpret_cast<const uint8_t*>(p.w0) + (e * p.rows + rr) * row_bytes;
        if (PAIR) r[NM - 1] = reinterpret_cast<const uint8_t*>(p.w1) + (e * p.rows + rr) * row_bytes;
        return true;
    };
    // stream one unit into ring slot `slot`; always commits a group so the per-thread group count stays in step
    auto issue = [&](int u, int slot) -> bool {
        const uint8_t* r[NM];
        const bool ok = unit_rows(u, r);
        if (ok) {
#pragma unroll
            for (int m = 0; m < NM; m++) {
                const uint32_t dst = ring_u32 + slot * slot_bytes + m * row_bytes;
                for (int c = lane * 16; c < row_bytes; c += 32 * 16) cp_async16_cg(dst + c, r[m] + c);
            }
        }
        cp_async_commit_group();
        return ok;
    };

    int u = u0 + warp;
    bool cur_ok = issue(u, 0);   // first unit streams in while the activation row is quantised
    cta_quantize_q8k_rows<4>(p.x, (long)t * p.ncols, 0, p.hidden_type, 1, p.ncols, 0u, q8, dx, bsums);
    __syncthreads();

    const int nsteps = (nblk + Fmt::kBlocksPerStep - 1) / Fmt::kBlocksPerStep;
    for (int it = 0; u < u1; u += WARPS, it++) {
        const int slot = it & 1;
        const bool next_ok = issue(u + WARPS, slot ^ 1);
        cp_async_wait_group<1>();   // everything but the group just committed has landed (this thread's copies)
        __syncwarp();               // ... and the other lanes' copies of this slot are visible
        float acc[NM];
#pragma unroll
        for (int m = 0; m < NM; m++) acc[m] = 0.f;
        if (cur_ok) {
            const uint8_t* row0 = ring + slot * slot_bytes;
#pragma unroll 2
            for (int s = 0; s < nsteps; s++) {
                const int blk = s * Fmt::kBlocksPerStep + L.blk;
                if (blk < nblk) {
                    typename Fmt::Regs R[NM];
#pragma unroll
                    for (int m = 0; m < NM; m++) Fmt::load_smem(row0 + m * row_bytes, blk, L, R[m]);
                    typename Fmt::Act A;
                    Fmt::load_act(act, blk, L, A);
#pragma unroll
                    for (int m = 0; m < NM; m++) acc[m] += Fmt::dot(R[m], A, L);
                }
            }
        }
        float g = warp_sum(acc[0]);
        const float uu = PAIR ? warp_sum(acc[NM - 1]) : 0.f;
        if (lane == 0) {
            if (PAIR) {
                p.out_f32[(long)t * total + u] = cur_ok ? (p.use_silu ? act_silu(g) : act_relu(g)) * uu : 0.f;
            } else {
                if (!cur_ok) g = 0.f;
                if (p.bias) g += p.bias[u % p.rows];
                if (p.out_f32) p.out_f32[(long)t * total + u] = g;
                if (p.out_hidden) store_hidden(p.out_hidden, (long)t * total + u, p.hidden_type, g);
            }
        }
        __syncwarp();               // all lanes are done with `slot` before the next iteration refills it
        cur_ok = next_ok;
    }
    cp_async_wait_group<0>();
}

}  // namespace ktb

namespace ktb {

// Pipelined reduce_kernel for Q6_K (8-row SoA) down projections.  Work item = (slot j, 4 consecutive rows):
// in the SoA layout the item is four contiguous pieces (ql 4x128nb | qh 4x64nb | scales 4x16nb | d 4x2nb),
// streamed into a warp-private 2-slot ring with cp.async while the previous item is reduced from shared memory.
// CTA row ranges are multiples of 4 rows; requires rows % 4 == 0 and nb even.
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 1) reduce_pipe_q6k8_kernel(const ReduceParams p, int slot_bytes) {
    using Fmt = FmtQ6K8;
    constexpr int RW = 4;
    extern __shared__ __align__(16) uint8_t smem[];
    const int t = blockIdx.y;
    if (p.bsz && t >= *p.bsz) return;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nb = p.ncols / QK_K;
    const int k = p.slots;
    const int ns = k + (p.xw ? 1 : 0);
    // staging: q8 [ns][ncols] | dx [ns][nb] | bsums [ns][ncols/16] | partial [rows_local][ns] | ring
    uint8_t* q8 = smem;
    float* dx = reinterpret_cast<float*>(smem + (size_t)ns * p.ncols);
    int16_t* bsums = reinterpret_cast<int16_t*>(smem + (size_t)ns * p.ncols + (size_t)ns * nb * 4);
    float* partial = reinterpret_cast<float*>(smem + (size_t)ns * p.ncols + (size_t)ns * nb * 4 + (size_t)ns * (p.ncols / 16) * 2);
    const int quads = p.rows / RW;
    const int q0 = (int)((long)quads * blockIdx.x / gridDim.x), q1 = (int)((long)quads * (blockIdx.x + 1) / gridDim.x);
    const int r0 = q0 * RW, nrows = (q1 - q0) * RW;
    const int nquads = q1 - q0;
    size_t off = (size_t)ns * p.ncols + (size_t)ns * nb * 4 + (size_t)ns * (p.ncols / 16) * 2 + (size_t)(nrows > 0 ? nrows : 1) * ns * 4;
    off = (off + 15) & ~(size_t)15;
    uint8_t* ring = smem + off + (size_t)warp * 2 * slot_bytes;
    const uint32_t ring_u32 = (uint32_t)__cvta_generic_to_shared(ring);

    const unsigned skip = skip_mask32(p, t);
    const int total = nquads * ns;   // item = j * nquads + quad
    const int s_ql = 4 * 128 * nb, s_qh = 4 * 64 * nb, s_sc = 4 * 16 * nb, s_d = 4 * 2 * nb;

    auto issue = [&](int item, int slot) -> bool {
        bool ok = item < total;
        if (ok) {
            const int j = item / nquads, quad = item - j * nquads;
            const uint8_t* wbase = reinterpret_cast<const uint8_t*>(p.w);
            long row = r0 + quad * RW;
            if (j == k) wbase = reinterpret_cast<const uint8_t*>(p.xw);
            else if (slot_skipped(p, t, skip, j)) ok = false;
            else row += (p.ids ? (long)p.ids[(long)t * k + j] - p.id_offset : 0L) * p.rows;
            if (ok) {
                const long G = row >> 3, r8 = row & 7;
                const uint8_t* g = wbase + G * (8 * SZ_Q6_K) * nb;
                const uint32_t dst = ring_u32 + slot * slot_bytes;
                const uint8_t* src[4] = {g + r8 * 128 * nb, g + 1024L * nb + r8 * 64 * nb, g + 1536L * nb + r8 * 16 * nb, g + 1664L * nb + r8 * 2 * nb};
                const int len[4] = {s_ql, s_qh, s_sc, s_d};
                int o = 0;
#pragma unroll
                for (int s = 0; s < 4; s++) {
                    for (int c = lane * 16; c < len[s]; c += 32 * 16) cp_async16_cg(dst + o + c, src[s] + c);
                    o += len[s];
                }
            }
        }
        cp_async_commit_group();
        return ok;
    };

    int item = warp;
    bool cur_ok = issue(item, 0);   // weights do not depend on phase 1: stream the first item during the prologue
    cta_quantize_q8k_rows<4>(p.a, (long)t * ns * p.ncols, p.ncols, KTB200_TYPE_F32, ns, p.ncols, skip, q8, dx, bsums);
    __syncthreads();

    const Fmt::Lane L = Fmt::lane(lane);
    const int nsteps = (nb + Fmt::kBlocksPerStep - 1) / Fmt::kBlocksPerStep;
    for (int it = 0; item < total; item += WARPS, it++) {
        const int slot = it & 1;
        const bool next_ok = issue(item + WARPS, slot ^ 1);
        cp_async_wait_group<1>();
        __syncwarp();
        const int j = item / nquads, quad = item - j * nquads;
        float res = 0.f;
        if (cur_ok) {
            const uint8_t* sl = ring + slot * slot_bytes;
            Fmt::Row rp[RW];
#pragma unroll
            for (int rw = 0; rw < RW; rw++)
                rp[rw] = Fmt::Row{sl + rw * 128 * nb, sl + s_ql + rw * 64 * nb, sl + s_ql + s_qh + rw * 16 * nb, sl + s_ql + s_qh + s_sc + rw * 2 * nb};
            const ActQ8K act{q8 + (size_t)j * p.ncols, dx + j * nb, bsums + j * (p.ncols / 16)};
            float acc[RW] = {0.f, 0.f, 0.f, 0.f};
            for (int s = 0; s < nsteps; s++) {
                const int blk = s * Fmt::kBlocksPerStep + L.blk;
                if (blk < nb) {
                    Fmt::Act A;
                    Fmt::load_act(act, blk, L, A);
#pragma unroll
                    for (int rw = 0; rw < RW; rw++) {
                        Fmt::Regs R;
                        Fmt::load_smem(rp[rw], blk, L, R);
                        acc[rw] += Fmt::dot(R, A, L);
                    }
                }
            }
            res = warp_reduce4(acc[0], acc[1], acc[2], acc[3], lane);
        }
        if ((lane & 7) == 0) partial[(quad * RW + (lane >> 3)) * ns + j] = res;
        __syncwarp();
        cur_ok = next_ok;
    }
    cp_async_wait_group<0>();
    __syncthreads();
    for (int hl = threadIdx.x; hl < nrows; hl += WARPS * 32) {
        float acc = 0.f;
        for (int j = 0; j < k; j++) {
            if (slot_skipped(p, t, skip, j)) continue;
            const float d = partial[hl * ns + j];
            acc = p.weights ? __fmaf_rn(d, p.weights[(long)t * k + j], acc) : acc + d;
        }
        const long o = (long)t * p.rows + r0 + hl;
        if (p.xw) acc = round_hidden(acc, p.hidden_type) + round_hidden(partial[hl * ns + k], p.hidden_type);
        if (p.accumulate) acc = load_hidden(p.out, o, p.hidden_type) + round_hidden(acc, p.hidden_type);
        store_hidden(p.out, o, p.hidden_type, acc);
    }
}

}  // namespace ktb
