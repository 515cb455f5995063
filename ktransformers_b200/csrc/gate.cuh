// Device code of the MoE router (shared by gate.cu and the fused MoE-block kernel, moe_block.cu).
#pragma once
#include "common.cuh"

namespace ktb {

constexpr int kGateWarps = 4;
constexpr int kGateThreads = kGateWarps * 32;
constexpr int kGateTokTile = 8;

struct GateParams {
    const float* W;
    const void* x;
    int hidden_type, E, H, T, S;
    int top_k, n_group, topk_group, scoring, topk_method, norm_topk_prob;
    float routed_scaling_factor;
    const float* bias;
    float* partial;      // [T][S][E]
    float* logits_out;   // optional [T][E]
    int64_t* idx;
    float* w;
    const int* bsz;
    unsigned* ticket;
};

// Column splits of the router GEMV: as many (row, split) units as fit ONE wave of the persistent MoE-block kernel
// (12 warps on every SM; a second wave doubles the router's latency), at least 64 float4 per unit.
// ktb200_moe_gate_forward and the fused kernel use the SAME S: their partial sums are bit-identical.
static inline int gate_splits(int E, int H, int nsms) {
    int S = nsms * 12 / E;
    if (S < 1) S = 1;
    if (S > 8) S = 8;
    while (S > 1 && H / 4 / S < 64) S--;
    return S;
}

constexpr int kGateEPT = 4;   // experts per thread of the selecting CTA (E <= 512)

// The router configurations gate_select_token takes: the one check of ktb200_moe_gate_forward, ktb200_moe_block_forward and
// ktb200_moe_ep_block_forward (host only; it reads no device memory).  False, with the error set, otherwise.
//   - noaux_tc scores a group by its two best experts: a group of one expert would score -inf, and the groups would then be
//     chosen by index, not by score (the reference's topk(2) over a group of one raises).
//   - top_k may not exceed the experts the group mask leaves, or masked experts would be chosen.
static inline bool gate_config_ok(const ktb200_gate_config* c) {
    if (c->n_experts <= 0 || c->n_experts > kGateThreads * kGateEPT || c->hidden_size <= 0 || c->hidden_size % 4 || c->top_k <= 0 ||
        c->top_k > 32 || c->top_k > c->n_experts) {
        set_error("gate: bad shape (E=%d H=%d top_k=%d; E<=%d, top_k<=32, H%%4==0)", c->n_experts, c->hidden_size, c->top_k,
                  kGateThreads * kGateEPT);
        return false;
    }
    if (c->n_group < 1 || c->n_group > 32 || c->n_experts % c->n_group || c->topk_group < 1 || c->topk_group > c->n_group) {
        set_error("gate: bad grouping (n_group=%d topk_group=%d)", c->n_group, c->topk_group);
        return false;
    }
    if (c->scoring < 0 || c->scoring > 1 || c->topk_method < 0 || c->topk_method > 2) { set_error("gate: bad scoring/topk_method"); return false; }
    const int gs = c->n_experts / c->n_group;
    if (c->topk_method == 0 && c->n_group > 1 && gs < 2) {
        set_error("gate: noaux_tc needs at least 2 experts per group (E=%d n_group=%d)", c->n_experts, c->n_group);
        return false;
    }
    if (c->topk_method != 1 && c->n_group > 1 && c->top_k > c->topk_group * gs) {
        set_error("gate: top_k=%d exceeds the %d experts of topk_group=%d groups", c->top_k, c->topk_group * gs, c->topk_group);
        return false;
    }
    if (!is_hidden_type(c->hidden_type) || !c->weight) { set_error("gate: bad hidden_type or null weight"); return false; }
    return true;
}

// order-preserving float -> uint32 key
__device__ __forceinline__ unsigned fkey(float f) {
    const unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float fkey_inv(unsigned k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Selection for ONE token by the whole CTA (kGateThreads threads).  Shared scratch (floats):
//   scores[E] | choice[E] | gsc[32] | wbest[2*kGateWarps] | red[2*kGateWarps]
// BAR = 0: the CTA is exactly kGateThreads threads and synchronises with __syncthreads(); BAR > 0: the first
// kGateThreads threads of a larger CTA run the selection and synchronise on named barrier BAR (fused MoE-block kernel).
// idx_out / w_out: where token t's top_k (id, weight) pairs go ([top_k] each; global or shared memory).
template <int BAR>
__device__ __forceinline__ void gate_sync() {
    if (BAR == 0) __syncthreads();
    else asm volatile("bar.sync %0, %1;" ::"n"(BAR), "n"(kGateThreads) : "memory");
}
// (the fields the selection reads, copied into registers once: the named barriers below are memory clobbers, and a
// params struct reached through a pointer would be re-read from memory after every one of them)
struct GateSel {
    int E, S, top_k, n_group, topk_group, scoring, topk_method, norm_topk_prob;
    float routed_scaling_factor;
    const float* bias;
    const float* partial;
};
template <int BAR>
__device__ void gate_select_token(const GateParams& pin, int t, float* sm, int64_t* idx_out, float* w_out, float* logits_out) {
    const GateSel p{pin.E, pin.S, pin.top_k, pin.n_group, pin.topk_group, pin.scoring, pin.topk_method, pin.norm_topk_prob,
                    pin.routed_scaling_factor, pin.bias, pin.partial};
    const int E = p.E, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    float* scores = sm;
    float* choice = sm + E;
    float* gsc = choice + E;
    unsigned* wbest = reinterpret_cast<unsigned*>(gsc + 32);
    float* red = reinterpret_cast<float*>(wbest + 2 * kGateWarps);

    // logits = sum of the S partials in fixed order; thread owns experts e = tid + 128*i
    // (all S <= 8 loads are issued before the first add: one L2 round trip instead of S)
    float v[kGateEPT], pv[8][kGateEPT];
#pragma unroll
    for (int s = 0; s < 8; s++) {
        const float* pp = p.partial + ((long)t * p.S + s) * E;
#pragma unroll
        for (int i = 0; i < kGateEPT; i++) {
            const int e = tid + kGateThreads * i;
            pv[s][i] = (s < p.S && e < E) ? __ldcg(pp + e) : 0.f;   // written by other SMs in this launch: read at L2
        }
    }
    float bv[kGateEPT];   // e_score_correction_bias, requested together with the partial sums
#pragma unroll
    for (int i = 0; i < kGateEPT; i++) {
        const int e = tid + kGateThreads * i;
        bv[i] = (p.topk_method == 0 && p.bias && e < E) ? __ldg(p.bias + e) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < kGateEPT; i++) {
        v[i] = 0.f;
#pragma unroll
        for (int s = 0; s < 8; s++)
            if (s < p.S) v[i] += pv[s][i];
    }
    if (logits_out) {
#pragma unroll
        for (int i = 0; i < kGateEPT; i++) {
            const int e = tid + kGateThreads * i;
            if (e < E) logits_out[(long)t * E + e] = v[i];
        }
    }
    if (p.scoring == 0) {  // sigmoid
#pragma unroll
        for (int i = 0; i < kGateEPT; i++) v[i] = __fdiv_rn(1.0f, 1.0f + expf(-v[i]));
    } else {               // softmax(dim=-1, fp32): block max, block sum
        float m = -INFINITY;
#pragma unroll
        for (int i = 0; i < kGateEPT; i++) if (tid + kGateThreads * i < E) m = fmaxf(m, v[i]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (lane == 0) red[warp] = m;
        gate_sync<BAR>();
        m = red[0];
        for (int w = 1; w < kGateWarps; w++) m = fmaxf(m, red[w]);
        float sum = 0.f;
#pragma unroll
        for (int i = 0; i < kGateEPT; i++) {
            v[i] = (tid + kGateThreads * i < E) ? expf(v[i] - m) : 0.f;
            sum += v[i];
        }
        sum = warp_sum(sum);
        if (lane == 0) red[kGateWarps + warp] = sum;
        gate_sync<BAR>();
        sum = 0.f;
        for (int w = 0; w < kGateWarps; w++) sum += red[kGateWarps + w];
#pragma unroll
        for (int i = 0; i < kGateEPT; i++) v[i] = __fdiv_rn(v[i], sum);
    }
    float c[kGateEPT];   // selection scores
#pragma unroll
    for (int i = 0; i < kGateEPT; i++) {
        const int e = tid + kGateThreads * i;
        c[i] = -INFINITY;
        if (e < E) {
            c[i] = v[i] + bv[i];
            scores[e] = v[i];
            choice[e] = c[i];
        }
    }
    gate_sync<BAR>();

    // group selection (noaux_tc: sum of the group's top-2 biased scores; group_limited_greedy: group max)
    if (p.n_group > 1 && p.topk_method != 1) {
        const int gs = E / p.n_group;
        for (int g = warp; g < p.n_group; g += kGateWarps) {   // one warp per group
            float a1 = -INFINITY, a2 = -INFINITY;
            for (int i = lane; i < gs; i += 32) {
                const float x = choice[g * gs + i];
                if (x > a1) { a2 = a1; a1 = x; } else if (x > a2) { a2 = x; }
            }
            const unsigned k1 = fkey(a1);
            const unsigned mx1 = __reduce_max_sync(0xffffffffu, k1);
            const int wl = __ffs(__ballot_sync(0xffffffffu, k1 == mx1)) - 1;
            const unsigned mx2 = __reduce_max_sync(0xffffffffu, lane == wl ? fkey(a2) : k1);
            if (lane == 0) gsc[g] = (p.topk_method == 0) ? (fkey_inv(mx1) + fkey_inv(mx2)) : fkey_inv(mx1);
        }
        gate_sync<BAR>();
        const float fill = (p.topk_method == 0) ? -INFINITY : 0.0f;  // V3 masks with -inf, V2 with 0.0
#pragma unroll
        for (int i = 0; i < kGateEPT; i++) {
            const int e = tid + kGateThreads * i;
            if (e < E) {
                const int g = e / gs;
                const float mine = gsc[g];
                int rank = 0;  // higher first, ties -> lower index
                for (int o = 0; o < p.n_group; o++) {
                    const float og = gsc[o];
                    rank += (og > mine || (og == mine && o < g)) ? 1 : 0;
                }
                if (rank >= p.topk_group) { c[i] = fill; choice[e] = fill; }
            }
        }
        gate_sync<BAR>();
    }

    // top-k by iterative arg-max, ties -> lowest expert index.  ONE warp does it from registers (lane owns experts
    // lane + 32*i): two REDUX per pick and no block-level barrier inside the loop.
    if (warp == 0) {
        constexpr int EPL = kGateThreads * kGateEPT / 32;
        unsigned ck[EPL];   // order-preserving keys of the selection scores; 0 = absent / already picked
#pragma unroll
        for (int i = 0; i < EPL; i++) {
            const int e = lane + 32 * i;
            ck[i] = (e < E) ? fkey(choice[e]) : 0u;
        }
        float wsum = 0.f, myw = 0.f;
        long myidx = 0;
        for (int it = 0; it < p.top_k; it++) {
            unsigned bk = 0;
            int bi = 0x7fffffff;
#pragma unroll
            for (int i = 0; i < EPL; i++)
                if (ck[i] > bk) { bk = ck[i]; bi = lane + 32 * i; }
            const unsigned mx = __reduce_max_sync(0xffffffffu, bk);
            int win = __reduce_min_sync(0xffffffffu, (bk == mx) ? bi : 0x7fffffff);
            if (win == 0x7fffffff || win < 0 || win >= E) win = 0;  // degenerate (all NaN)
            // V3 gathers the weight from the un-biased scores; V2 group_limited takes the (masked) score itself
            const float wv = (p.topk_method == 2) ? choice[win] : scores[win];
#pragma unroll
            for (int i = 0; i < EPL; i++)
                if (lane + 32 * i == win) ck[i] = 0u;
            if (lane == it) { myw = wv; myidx = win; }
            wsum += wv;
        }
        // V3 (modeling_deepseek_v3.py:474-479): normalise (if top_k>1 && norm_topk_prob) THEN always scale;
        // V2 (modeling_deepseek.py:455-459): normalise XOR scale.
        if (lane < p.top_k) {
            float w = myw;
            const bool do_norm = p.top_k > 1 && p.norm_topk_prob;
            if (do_norm) w = __fdiv_rn(w, wsum + 1e-20f);
            if (p.topk_method == 0 || !do_norm) w = w * p.routed_scaling_factor;
            idx_out[lane] = myidx;
            w_out[lane] = w;
        }
    }
    gate_sync<BAR>();
}

template <int NT>
__device__ __forceinline__ void gate_dot(const GateParams& p, const float4* wrow, const float* xs, int nc4, int lane, int t0, int e,
                                         int s, int S, int nt = NT) {
    float acc[NT];
#pragma unroll
    for (int i = 0; i < NT; i++) acc[i] = 0.f;
    for (int cb = lane; cb < nc4; cb += 32 * 8) {
        float4 w[8];
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int c = cb + 32 * u;
            if (c < nc4) w[u] = __ldg(wrow + c);
        }
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int c = cb + 32 * u;
            if (c < nc4) {
#pragma unroll
                for (int i = 0; i < NT; i++) {
                    const float4 xv = reinterpret_cast<const float4*>(xs + (size_t)(i < nt ? i : 0) * nc4 * 4)[c];
                    acc[i] = fmaf(w[u].x, xv.x, acc[i]);
                    acc[i] = fmaf(w[u].y, xv.y, acc[i]);
                    acc[i] = fmaf(w[u].z, xv.z, acc[i]);
                    acc[i] = fmaf(w[u].w, xv.w, acc[i]);
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < NT; i++) {
        const float v = warp_sum(acc[i]);
        if (i < nt && lane == 0) p.partial[((long)(t0 + i) * S + s) * p.E + e] = v;
    }
}

}  // namespace ktb
