// DeepSeek MoEGate routing on the GPU.  Replaces MoEGate.forward
// (archive/ktransformers/models/modeling_deepseek_v3.py:430-481 for V3 sigmoid/noaux_tc,
//  archive/ktransformers/models/modeling_deepseek.py:411-459 for V2 softmax greedy/group_limited_greedy),
// which the reference runs as ~10 ATen kernels per layer (fp32 F.linear, sigmoid, two topk, scatter,
// masked_fill, gather, sum, div, mul).
//
// ONE kernel:
//   phase 1  fp32 GEMV  logits[t][e] = x_t(fp32) . W[e]   (HBM-bound: E*H*4 bytes).  A CTA of 4 warps owns 4
//            expert rows x one column split; each warp streams its row slice with 16-byte loads (8 in flight
//            per lane) against the token slice staged in shared memory, and writes one partial sum per
//            (token, expert, split).  Partials are added in fixed split order: deterministic, no float atomics.
//   phase 2  the LAST CTA to finish (atomic ticket, self-resetting, graph-replay safe) selects, all 128 threads
//            per token — scoring, bias, group top-2 / max, group top-k, expert top-k by iterative arg-max with
//            REDUX max/min (ties -> lowest index), gather, normalise, scale.
#include "gate.cuh"
#include "handles.cuh"

namespace ktb {

__global__ void __launch_bounds__(kGateThreads) gate_kernel(const GateParams p) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    float* xs = reinterpret_cast<float*>(smem_raw);   // [tok tile][slice cols]  (phase 1) / scores+choice (phase 2)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int Teff = p.T;
    if (p.bsz) Teff = max(0, min(p.T, *p.bsz));   // a negative device batch size selects nothing, like 0
    const int s = blockIdx.y, S = p.S;
    const int n4 = p.H / 4;
    const int c0 = (int)((long)n4 * s / S), c1 = (int)((long)n4 * (s + 1) / S);   // float4 column range of this split
    const int nc4 = c1 - c0;
    const int e = blockIdx.x * kGateWarps + warp;
    const float4* wrow = reinterpret_cast<const float4*>(p.W + (long)(e < p.E ? e : 0) * p.H) + c0;

    for (int t0 = 0; t0 < Teff; t0 += kGateTokTile) {
        const int nt = min(kGateTokTile, Teff - t0);
        __syncthreads();
        for (int tt = 0; tt < nt; tt++)
            for (int c = threadIdx.x; c < nc4 * 4; c += kGateThreads)
                xs[tt * nc4 * 4 + c] = load_hidden(p.x, (long)(t0 + tt) * p.H + 4L * c0 + c, p.hidden_type);
        __syncthreads();
        if (e < p.E) {
            switch (nt) {   // compile-time token counts: no predicated-off FMAs for the common bs=1 decode
                case 1: gate_dot<1>(p, wrow, xs, nc4, lane, t0, e, s, S); break;
                case 2: gate_dot<2>(p, wrow, xs, nc4, lane, t0, e, s, S); break;
                case 3: case 4: gate_dot<4>(p, wrow, xs, nc4, lane, t0, e, s, S, nt); break;
                default: gate_dot<kGateTokTile>(p, wrow, xs, nc4, lane, t0, e, s, S, nt); break;
            }
        }
    }

    // ---- the last CTAs to finish select: one token each (round-robin), in parallel ----------------------------------
    // ticket[0] counts finished CTAs, ticket[1] finished selectors; both are zero again when the launch ends
    // (graph-replay safe).  A selector that is not the very last CTA spins until all partial sums are written: the whole
    // grid is resident (<= 16 small CTAs per SM), so the CTAs it waits for are running.
    __shared__ int s_sel;
    const unsigned total = gridDim.x * gridDim.y;
    const int nsel = min(Teff, (int)min(total, 16u));
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned prev = atomicAdd(p.ticket, 1u);
        s_sel = nsel > 0 ? (int)prev - (int)(total - nsel) : -1;
        if (nsel == 0 && prev == total - 1) p.ticket[0] = 0;   // device-side batch size 0: nothing to select
        if (s_sel >= 0) {
            unsigned v;
            do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p.ticket) : "memory"); } while (v < total);
        }
    }
    __syncthreads();
    if (s_sel < 0) return;
    __threadfence();
    for (int t = s_sel; t < Teff; t += nsel) gate_select_token<0>(p, t, xs, p.idx + (long)t * p.top_k, p.w + (long)t * p.top_k, p.logits_out);
    if (threadIdx.x == 0) {
        const unsigned done = atomicAdd(p.ticket + 1, 1u);
        if (done == (unsigned)nsel - 1) { p.ticket[0] = 0; p.ticket[1] = 0; }
    }
}

// per-device scratch: partial sums + ticket
static float* g_partial[64] = {nullptr};
static size_t g_partial_cap[64] = {0};
static unsigned* g_ticket[64] = {nullptr};

}  // namespace ktb

extern "C" int ktb200_moe_gate_forward(const ktb200_gate_config* c, int qlen, const void* x, int64_t* idx, float* w,
                                       float* logits, const int* bsz, void* stream) {
    using namespace ktb;
    if (!c || !x || !idx || !w) { set_error("null pointer"); return KTB200_EINVAL; }
    if (qlen <= 0) return KTB200_OK;
    if (!gate_config_ok(c)) return KTB200_EINVAL;
    int dev = 0;
    KTB_CUDA_CHECK(cudaGetDevice(&dev));
    const int d = dev & 63;
    cudaStream_t s = (cudaStream_t)stream;
    const int row_ctas = (c->n_experts + kGateWarps - 1) / kGateWarps;
    const int S = gate_splits(c->n_experts, c->hidden_size, num_sms(dev));
    const size_t need = (size_t)qlen * c->n_experts * S * sizeof(float);
    if (need > g_partial_cap[d] || !g_ticket[d]) {
        // grow-only scratch.  Growing is synchronous and cannot be captured: on a capturing stream return before any device
        // work and name the warm-up (one eager call at this qlen or more, with this router, on this device)
        cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
        KTB_CUDA_CHECK(cudaStreamIsCapturing(s, &cs));
        if (cs != cudaStreamCaptureStatusNone) {
            set_error("gate: this call needs %zu bytes of router scratch on device %d, which holds %zu%s; the scratch cannot grow while "
                      "the stream is capturing: run one eager ktb200_moe_gate_forward call of %d or more tokens with n_experts %d and "
                      "hidden_size %d on this device before capture", need, dev, g_partial_cap[d], g_ticket[d] ? "" : " (first call)", qlen,
                      c->n_experts, c->hidden_size);
            return KTB200_ESTATE;
        }
        if (need > g_partial_cap[d]) {
            KTB_CUDA_CHECK(cudaDeviceSynchronize());   // earlier calls may still be using the scratch
            cudaFree(g_partial[d]);
            g_partial[d] = nullptr;
            g_partial_cap[d] = 0;
            const size_t cap = need < (1u << 20) ? (1u << 20) : need;
            KTB_CUDA_CHECK(cudaMalloc(&g_partial[d], cap));
            g_partial_cap[d] = cap;
        }
        if (!g_ticket[d]) {
            KTB_CUDA_CHECK(cudaMalloc(&g_ticket[d], 2 * sizeof(unsigned)));
            KTB_CUDA_CHECK(cudaMemset(g_ticket[d], 0, 2 * sizeof(unsigned)));
        }
    }
    GateParams p{c->weight, x, c->hidden_type, c->n_experts, c->hidden_size, qlen, S, c->top_k, c->n_group, c->topk_group,
                 c->scoring, c->topk_method, c->norm_topk_prob, c->routed_scaling_factor, c->bias, g_partial[d], logits,
                 idx, w, bsz, g_ticket[d]};
    const int nc4_max = c->hidden_size / 4 / S + 1;
    const int nt = qlen < kGateTokTile ? qlen : kGateTokTile;
    size_t smem = (size_t)nt * nc4_max * 16;
    const size_t smem_sel = ((size_t)2 * c->n_experts + 32 + 4 * kGateWarps) * sizeof(float);
    if (smem_sel > smem) smem = smem_sel;
    if (smem > 48 * 1024) KTB_CUDA_CHECK(cudaFuncSetAttribute(gate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    gate_kernel<<<dim3(row_ctas, S), kGateThreads, smem, s>>>(p);
    KTB_LAUNCH_CHECK();
    return KTB200_OK;
}

extern "C" int ktb200_debug_gate_ticket(int device, unsigned* host_out) {
    using namespace ktb;
    if (!host_out) { set_error("debug_gate_ticket: null pointer"); return KTB200_EINVAL; }
    const int d = device & 63;
    if (!g_ticket[d]) { set_error("debug_gate_ticket: no router call has run on device %d", device); return KTB200_ESTATE; }
    DeviceGuard guard(device);
    KTB_CUDA_CHECK(cudaDeviceSynchronize());
    KTB_CUDA_CHECK(cudaMemcpy(host_out, g_ticket[d], 2 * sizeof(unsigned), cudaMemcpyDeviceToHost));
    return KTB200_OK;
}
