// Internal (not part of the C-ABI): the opaque handles behind include/ktb200.h and the weight-format ids the
// dispatchers in moe.cu / moe_block.cu agree on.
#pragma once
#include "common.cuh"

namespace ktb {
enum FmtId { FMT_Q4K, FMT_Q5K, FMT_Q6K8, FMT_Q6K4T, FMT_GENK, FMT_RAWINT4, FMT_NONE };
// how a Q6_K tensor was re-laid at load time
enum Q6Layout { LAYOUT_RAW = 0, LAYOUT_SOA8 = 1, LAYOUT_T4 = 2 };

static inline FmtId pick_fmt(int type, int layout) {
    if (type == KTB200_TYPE_Q4_K) return FMT_Q4K;
    if (type == KTB200_TYPE_Q5_K) return FMT_Q5K;
    if (type == KTB200_TYPE_Q6_K && layout == LAYOUT_SOA8) return FMT_Q6K8;
    if (type == KTB200_TYPE_Q6_K && layout == LAYOUT_T4) return FMT_Q6K4T;
    if (is_kquant(type) || is_iquant(type)) return FMT_GENK;
    if (is_rawint4(type)) return FMT_RAWINT4;
    return FMT_NONE;
}
}  // namespace ktb

// ------------------------------------------------------------------------------------------
struct ktb200_mlp {
    int H, I, gate_type, up_type, down_type, hidden_type, group_max_len, device;
    const void *gate, *up, *down;
    bool loaded, gu_soa;
    int down_layout;   // Q6Layout of the down tensor
    float* inter;
};

struct ktb200_moe {
    ktb200_moe_config cfg;
    int device;
    bool loaded;
    bool gu_soa;
    int down_layout;   // Q6Layout of the down tensor
    float* inter;      // [group_max_len * k][I]
    // host-call staging
    int64_t* ids_d;
    float* w_d;
    void* in_d;
    void* out_d;
    // scratch of the persistent MoE-block kernel (moe_block.cu): router partial sums [8 tokens][8 splits][512 experts];
    // blk_sync: two pairs of grid-barrier words, a status word, then two sets of per-Q8_K-block readiness words
    // (blk_ready_words each), pairs and sets used alternately (zero between launches); blk_inter: the kernel's fp32
    // intermediate [8 tokens][top-k + 1][I], all ones between launches (moe_block.cu: kInterEmpty); blk_stage: it
    // quantised, [blk_ready_words] x (QK_K int8 | 16 int16 block sums | fp32 scale), as three arrays
    float* blk_partial;
    unsigned* blk_sync;
    unsigned blk_flip;
    float* blk_inter;
    uint8_t* blk_stage;
    const void* pf[3];       // ktb200_moe_block_prefetch_hint: ranges the block kernel pulls into L2 during its down phase
    size_t pf_bytes[3];
};

namespace ktb {
constexpr int kBlockMaxTokens = 8;   // tokens one persistent MoE-block launch takes
constexpr int kBlkStatusWord = 4, kBlkReadyWord = 8;   // offsets in ktb200_moe::blk_sync
// readiness words of one set: [tokens][slots: top-k + the shared expert][Q8_K blocks of I]
static inline size_t blk_ready_words(const ktb200_moe_config& c) {
    const int t = c.group_max_len < kBlockMaxTokens ? c.group_max_len : kBlockMaxTokens;
    return (size_t)t * (c.routed_expert_num + 1) * (c.intermediate_size / QK_K);
}

// the Q8_K activation buffers of the grouped path's per-device arena (grouped.cu), lent to the tiled linear GEMM
struct GrpX {
    int8_t* q;     // [tokens][K]
    float* d;      // [tokens][K / 256]
    int16_t* bs;   // [tokens][K / 16]
};
int grp_prompt_x(int dev, size_t need, size_t grow, cudaStream_t s, GrpX* out);
int grp_prompt_quant(const void* x, int hidden_type, int T, int K, const GrpX& b, cudaStream_t s);
// the prompt route of the GGUF dense linear (gguf_gemm.cu): ktb200_linear_prompt_min, ktb200_linear_forward_prompt
int gguf_prompt_min(int type, int layout, int K, int N);
int gguf_forward_prompt(const void* w, int type, int layout, int K, int N, int hidden_type, int dev, int qlen, const void* x, void* y,
                        const float* bias, const int* bsz, cudaStream_t s);
}  // namespace ktb

struct DeviceGuard {
    int prev;
    bool ok;
    explicit DeviceGuard(int dev) : prev(0), ok(true) {
        if (cudaGetDevice(&prev) != cudaSuccess) ok = false;
        if (ok && prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
    }
    ~DeviceGuard() { cudaSetDevice(prev); }
};

