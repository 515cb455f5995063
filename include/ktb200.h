/* ktb200 — H100-native (sm_90a) drop-in for kt-kernel's quantized-MoE decode hot path.
 *
 * C-ABI boundary: plain pointers and sizes only, no torch / pybind types.  Every entry point
 * names the reference interface it replaces.  All `*_dev` pointers are CUDA device pointers on the
 * device the handle was created for; `stream` is a cudaStream_t passed as void*.  All calls are
 * stream-ordered, never synchronise the device (except the *_host convenience calls and where
 * stated) and never call back into Python, so they can be captured into a CUDA graph.
 *
 * Ownership (same contract as the reference, kt-kernel/ext_bindings.cpp:167-177 DEF_PTR_PROPERTY,
 * archive/ktransformers/operators/experts.py:183-218): the caller owns every tensor; the library
 * receives raw pointers and never frees them.  Weight tensors must stay alive as long as the
 * handle; `*_load_weights` may permute bytes of a weight tensor IN PLACE (see below), exactly like
 * the reference's load_weights re-packs into its own layout (llamafile/moe.hpp:194-251).
 *
 * Errors: every function returns 0 on success or a negative KTB200_E* code; ktb200_last_error()
 * returns a thread-local message (reference: C++ exceptions -> Python, moe-tp.hpp:203-205,
 * ext_bindings.cpp:88-92 invalid ggml_type -> ValueError).  Expert ids < 0 or >= expert_num are
 * silently skipped (kt-kernel/operators/common.hpp:255-258 should_skip_expert).
 */
#ifndef KTB200_H
#define KTB200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define KTB200_OK 0
#define KTB200_EINVAL (-1)   /* bad argument / unsupported ggml type */
#define KTB200_ECUDA (-2)    /* CUDA runtime error */
#define KTB200_ESTATE (-3)   /* e.g. forward before load_weights ("Not Loaded", moe-tp.hpp:203-205) */
#define KTB200_ENOMEM (-4)

/* ggml type ids, identical to the reference (third_party/llama.cpp/ggml.h:349-380). */
enum ktb200_ggml_type {
    KTB200_TYPE_F32 = 0, KTB200_TYPE_F16 = 1, KTB200_TYPE_Q8_0 = 8, KTB200_TYPE_Q2_K = 10,
    KTB200_TYPE_Q3_K = 11, KTB200_TYPE_Q4_K = 12, KTB200_TYPE_Q5_K = 13, KTB200_TYPE_Q6_K = 14,
    KTB200_TYPE_Q8_K = 15, KTB200_TYPE_IQ4_XS = 23, KTB200_TYPE_BF16 = 30,
    /* ggml's codebook i-quants (DeepSeek-V3's and R1's 1.5-3-bit GGUF experts), raw ggml blocks of 256 values:
     *   IQ2_XXS  66 B: fp16 d, then per 32-value sub-block two 32-bit words: four 8-bit indices into iq2xxs_grid, then
     *            four 7-bit indices into ksigns_iq2xs and the 4-bit scale s in bits 28..31; value = d*(2s+1)/8 * grid * sign
     *   IQ1_S    50 B: fp16 d, qs[32], qh uint16[8]; sub-block ib has ls = 2*((qh>>12)&7)+1, delta = qh bit 15 ? -1/8 : +1/8,
     *            group l = iq1s_grid[qs[4ib+l] | ((qh >> 3l) & 7) << 8]; value = d*ls*(grid + delta)
     *   IQ1_M    56 B: qs[32], qh[16], scales uint16[4]; 8-value group l (0..31) has the nibble of qh byte l/2 (low for even
     *            l): bits 0-2 the high bits of its iq1s_grid index qs[l] | (nibble & 7) << 8, bit 3 the sign of its
     *            delta (+-1/8); 16-value half h (0..15) has ls = 2*((scales[h/4] >> 3(h%4)) & 7)+1; the fp16 d is the
     *            four top nibbles, scales[0] >> 12 lowest; value = d*ls*(grid + delta)
     *   IQ3_XXS  98 B: fp16 d, qs[64], then per 32-value sub-block ib one 32-bit word: four 7-bit indices into ksigns_iq2xs
     *            (bits 7l..7l+6 for values 8l..8l+7) and the 4-bit scale s in bits 28..31; 4-value group g (0..7) of ib is
     *            iq3xxs_grid[qs[8ib+g]]; value = d*(2s+1)/4 * grid * sign
     *   IQ3_S   110 B: fp16 d, qs[64], qh[8], signs[32], scales[4]; 4-value group j (0..63) is iq3s_grid[qs[j] | (bit j%8
     *            of qh[j/8]) << 8], bit i of signs[k] negates value 8k+i, sub-block ib has s = nibble ib%2 (low for
     *            even ib) of scales[ib/2]; value = d*(2s+1) * grid * sign
     *   IQ2_XS   74 B: fp16 d, qs uint16[32], scales[8]; 8-value group l (0..31) is iq2xs_grid[qs[l] & 511] with the signs
     *            ksigns_iq2xs[qs[l] >> 9]; 16-value half h (0..15) has s = nibble h%2 (low for even h) of scales[h/2];
     *            value = d*(2s+1)/8 * grid * sign
     *   IQ2_S    82 B: fp16 d, qs[32], signs[32], qh[8], scales[8]; 8-value group l (0..31) is iq2s_grid[qs[l] | ((qh[l/4]
     *            >> 2(l%4)) & 3) << 8], bit i of signs[l] negates its value i; s per 16 values as IQ2_XS;
     *            value = d*(2s+1)/8 * grid * sign
     * vec_dot_type Q8_K.  Routed experts only (ktb200_moe_create, any mix with the K-quants); linears, MLP handles and the
     * one-token expert-parallel entry points reject them.  ktb200_moe_forward runs them per (token, expert) pair below 80
     * tokens and on the grouped tensor-core GEMM from 80 (gate, up and down each in its own format).  The codebooks are
     * ktransformers_b200/csrc/iq_tables.h, iq3_tables.h and iq2_tables.h. */
    KTB200_TYPE_IQ2_XXS = 16, KTB200_TYPE_IQ2_XS = 17, KTB200_TYPE_IQ3_XXS = 18, KTB200_TYPE_IQ1_S = 19, KTB200_TYPE_IQ3_S = 21,
    KTB200_TYPE_IQ2_S = 22, KTB200_TYPE_IQ1_M = 29,
    /* Not a ggml type: ggml's ids stay below 64, so 256 cannot collide with one.
     * Symmetric INT4 in groups of 32 with bf16 scales (compressed-tensors "pack-quantized", kt-kernel's RAWINT4; Kimi-K2's
     * routed experts), in the device layout ktb200_rawint4_pack writes: 144 B per 256 values of a row,
     *   bytes 0..15          eight bf16 group scales
     *   bytes 16+16j..31+16j group j = four 32-bit words, word w holds columns 8w..8w+7 of the group, column 8w+i in
     *                        bits 4i..4i+3 as u = q + 8 (the compressed-tensors words unchanged)
     * value = (u - 8) * scale.  Routed experts only (ktb200_moe_*): linears and MLP handles reject it.  ktb200_moe_forward
     * runs them per (token, expert) pair below 96 tokens and on the grouped tensor-core GEMM from 96 (bf16 planes of the
     * activations against u - 8, DESIGN.md §4.5). */
    KTB200_TYPE_RAWINT4_G32 = 256
};

const char* ktb200_last_error(void);
const char* ktb200_version(void);
/* bytes per block / elements per block of a ggml type (0 when unsupported):
 * ggml_type_size / ggml_blck_size, archive/ktransformers/util/custom_gguf.py:72-102 */
long ktb200_type_size(int ggml_type);
long ktb200_blck_size(int ggml_type);
/* number of kernels this library has launched since load (bench.py's gpu_launches claim). */
unsigned long long ktb200_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Routed experts.  Replaces cpuinfer_ext.moe.MOEConfig / MOE
 *   archive/csrc/ktransformers_ext/ext_bindings.cpp:683-695 (MOEConfig ctor), :554-567 (forward)
 *   archive/csrc/ktransformers_ext/operators/llamafile/moe.h:27-48, moe.cpp:146-380
 * and kt_kernel_ext.moe.MOEConfig / MOE (kt-kernel/ext_bindings.cpp:746-831, 447-471).
 * Field names and meaning are the reference's; `stride`, `group_min_len` are accepted for source
 * compatibility and ignored (they are CPU work-splitting knobs).
 * ------------------------------------------------------------------------------------------ */
typedef struct ktb200_moe_config {
    int expert_num;          /* E: experts resident behind gate/up/down pointers */
    int routed_expert_num;   /* k: experts per token (num_experts_per_tok) */
    int hidden_size;         /* H */
    int intermediate_size;   /* I */
    int stride;              /* ignored */
    int group_min_len;       /* ignored */
    int group_max_len;       /* max tokens per forward call (scratch is sized for it) */
    int use_silu;            /* 1: silu(g)*u (moe.cpp:134-136), 0: relu(g)*u (:138-144) */
    const void* gate_proj;   /* DEVICE ptr, ggml blocks, row-major [E][I][H]  */
    const void* up_proj;     /* DEVICE ptr, [E][I][H] */
    const void* down_proj;   /* DEVICE ptr, [E][H][I] */
    int gate_type, up_type, down_type;   /* ggml types of the three tensors */
    int hidden_type;         /* F32 / F16 / BF16: dtype of input and output rows */
    int expert_id_offset;    /* expert-parallel shard: this handle owns global ids
                                [offset, offset+expert_num); others are skipped */
} ktb200_moe_config;

typedef struct ktb200_moe ktb200_moe;

int ktb200_moe_create(const ktb200_moe_config* cfg, int device, ktb200_moe** out);
void ktb200_moe_destroy(ktb200_moe* moe);

/* Replaces MOE::load_weights / load_weights_task (kt-kernel/ext_bindings.cpp:447-471).
 * Q6_K tensors are permuted IN PLACE, once, into the 16-byte-aligned "8-row SoA" layout that the
 * sm_90a kernels stream (DESIGN.md §3); other types are consumed as raw ggml blocks.
 * Byte count is unchanged.  Idempotent per handle. */
int ktb200_moe_load_weights(ktb200_moe* moe, void* stream);

/* Replaces MOE::warm_up (moe.cpp:119-132): runs one token through every expert slot. */
int ktb200_moe_warm_up(ktb200_moe* moe, void* stream);

/* Replaces MOE::forward(qlen, k, expert_ids, weights, input, output, batch_size_tensor)
 * (moe.cpp:367-380; kt-kernel forward_task(qlen_ptr,k,ids,w,in,out), ext_bindings.cpp:235-239).
 *   expert_ids_dev [qlen][k] int64 (kt-kernel) — the archive's uint64 has the same bits
 *   weights_dev    [qlen][k] float (already scaled by routed_scaling_factor)
 *   input_dev/output_dev [qlen][H] of hidden_type
 *   bsz_tensor_dev optional device int*: when non-null the effective qlen is min(qlen, *bsz) read ON
 *     DEVICE (the reference reads batch_size_tensor[0] on the host, moe.cpp:368) so one captured
 *     graph serves a variable batch; rows >= *bsz are left untouched.
 * Arithmetic: identical to the reference CPU path — activations quantised to the weight type's
 * vec_dot_type (Q8_K / Q8_0) with the reference's rounding, integer dot products, fp32 scales,
 * fp32 accumulation over experts in expert_ids order, output rounded like ggml from_float.
 * RAWINT4_G32 experts are W4A16 instead: fp32 activations against (u - 8) * scale, fp32 sums (DESIGN.md §2).
 * Routes: per-pair GEMV kernels for short batches; from 48 tokens (Q2_K..Q6_K experts; 80 for a handle with an i-quant
 * tensor, 96 for RAWINT4; KTB200_GROUPED_MIN overrides) the grouped tensor-core GEMMs, which read each expert once per 32-token tile and grow a
 * per-device scratch arena on first use. */
int ktb200_moe_forward(ktb200_moe* moe, int qlen, int k, const int64_t* expert_ids_dev,
                       const float* weights_dev, const void* input_dev, void* output_dev,
                       const int* bsz_tensor_dev, void* stream);

/* Same call with HOST buffers (pinned or pageable), the shape of the reference's own call where
 * ids/weights/input/output live in host memory (experts.py:297-313): H2D copies, forward, D2H copy,
 * then stream synchronise.  This is what bench.py's e2e number times. */
int ktb200_moe_forward_host(ktb200_moe* moe, int qlen, int k, const int64_t* expert_ids,
                            const float* weights, const void* input, void* output, void* stream);

/* Profiling aid for bench.py's roofline leg: same as ktb200_moe_forward, but brackets the two kernels
 * (phase 1: gate/up GEMV + activation, phase 2: down GEMV + weighted sum) with CUDA events on `stream`,
 * synchronises, and returns their durations in milliseconds.  Not capturable. */
int ktb200_moe_forward_timed(ktb200_moe* moe, int qlen, int k, const int64_t* expert_ids_dev,
                             const float* weights_dev, const void* input_dev, void* output_dev, void* stream,
                             float* ms_gate_up, float* ms_down);

/* scratch the forward uses (device, fp32 [group_max_len*k][I]) — exposed for tests / fusion */
float* ktb200_moe_intermediate(ktb200_moe* moe);

/* ------------------------------------------------------------------------------------------
 * FP8 (e4m3, 128 x 128 block scales) linear — DeepSeek-V3's native checkpoint format.  Replaces KLinearFP8
 * (archive/ktransformers/operators/linear.py:388-435) = act_quant + fp8_gemm of
 * archive/ktransformers/ktransformers_ext/triton/fp8gemm.py:10-47, 104-192 (BASELINE configs 3 / 5: FP8 linears beside GGUF experts).
 * weight: DEVICE ptr, e4m3 bytes [out][in] (16-byte aligned, in % 128 == 0); weight_scale_inv: DEVICE fp32 [ceil(out/128)][in/128].
 * forward: x [qlen][in] -> y [qlen][out] in hidden_type (x is quantised per token and 128 values inside the kernel, exactly like
 * act_quant; rows >= *bsz untouched).  An all-zero 128-block of x yields NaN outputs, as it does in the reference (0 / 0).
 * TMA + fp16 wgmma on e4m3 weights widened in registers; stream-ordered; everything is allocated at create -> CUDA-graph capturable.
 * ------------------------------------------------------------------------------------------ */
typedef struct ktb200_fp8_linear ktb200_fp8_linear;
int ktb200_fp8_linear_create(int in_features, int out_features, const void* weight_e4m3_dev, const float* weight_scale_inv_dev, int hidden_type, int device,
                             ktb200_fp8_linear** out);
void ktb200_fp8_linear_destroy(ktb200_fp8_linear* l);
/* Two routes, chosen from qlen and the shape; the results agree within the oracle's bound (DESIGN.md §4.6).
 *   qlen below 32 / 48 / 96 tokens (32 by default, 48 for in >= 16384, 96 for out <= 2048): decode passes of 16 tokens, each
 *     streaming the weights; allocation-free, capturable as above.
 *   from there on: the tokens are quantised once per chunk of at most 2048 into a grow-only per-device scratch arena shared by
 *     every handle, and a tiled GEMM (128 weight rows x 128 tokens per CTA) reads each weight once per chunk.  Deterministic (no
 *     K splits, no atomics).  A call that would have to grow the arena while its stream is capturing returns KTB200_ESTATE
 *     before any device work: run one eager call on the prompt route at this in_features (or larger) on the device before
 *     capture.  Calls on one device must be stream-ordered with each other (they share the arena). */
int ktb200_fp8_linear_forward(ktb200_fp8_linear* l, int qlen, const void* x, void* y, const int* bsz, void* stream);

/* ------------------------------------------------------------------------------------------
 * Dense quantised linear and gated MLP (shared experts / dense layers / projections / lm_head).
 * Replaces cpuinfer_ext.linear.Linear / mlp.MLP (archive ext_bindings.cpp, operators/llamafile/
 * linear.cpp:37-70, mlp.cpp:47-125) and the dequant->Marlin path of KLinearMarlin
 * (archive/ktransformers/operators/linear.py:595-721).  Weight: DEVICE ptr, ggml blocks [out][in].
 * ------------------------------------------------------------------------------------------ */
typedef struct ktb200_linear ktb200_linear;
int ktb200_linear_create(int in_size, int out_size, const void* proj_dev, int proj_type, int hidden_type,
                         int group_max_len, int device, ktb200_linear** out);
void ktb200_linear_destroy(ktb200_linear* lin);
int ktb200_linear_load_weights(ktb200_linear* lin, void* stream);
/* y[qlen][out] = x[qlen][in] * W^T ; bias_dev optional fp32 [out] added before rounding */
int ktb200_linear_forward(ktb200_linear* lin, int qlen, const void* input_dev, void* output_dev,
                          const float* bias_dev, const int* bsz_tensor_dev, void* stream);
/* The prompt route: ktb200_linear_forward's contract at any qlen >= 1, on a tiled integer tensor-core GEMM that reads each
 * weight once per chunk of at most 2048 tokens (DESIGN.md §4.17).  Q4_K weights, and Q6_K weights in the 8-row layout
 * ktb200_linear_load_weights gives them when out_size % 8 == 0; any other handle returns KTB200_EINVAL.  Its activation
 * scratch is a grow-only per-device arena: a call that would have to grow it while the stream is capturing returns
 * KTB200_ESTATE before any device work, so run one eager call of the largest in_size before capture. */
int ktb200_linear_forward_prompt(ktb200_linear* lin, int qlen, const void* input_dev, void* output_dev,
                                 const float* bias_dev, const int* bsz_tensor_dev, void* stream);
/* the qlen from which ktb200_linear_forward_prompt is the faster route for this handle (a function of its weight type,
 * layout and shape, measured on an H100), 0 when it does not take the handle */
int ktb200_linear_prompt_min(const ktb200_linear* lin);

typedef struct ktb200_mlp ktb200_mlp;
int ktb200_mlp_create(int hidden_size, int intermediate_size, const void* gate_dev, const void* up_dev,
                      const void* down_dev, int gate_type, int up_type, int down_type, int hidden_type,
                      int group_max_len, int device, ktb200_mlp** out);
void ktb200_mlp_destroy(ktb200_mlp* mlp);
int ktb200_mlp_load_weights(ktb200_mlp* mlp, void* stream);
/* out = down(silu(gate x) * up x); when accumulate != 0, out += result (fp32 add before rounding):
 * fuses KDeepseekV3MoE's `y += shared_experts(identity)` (experts.py:984-1011). */
int ktb200_mlp_forward(ktb200_mlp* mlp, int qlen, const void* input_dev, void* output_dev, int accumulate,
                       const int* bsz_tensor_dev, void* stream);

/* KDeepseekV3MoE.forward in one call (experts.py:974-1012): out = round(experts(x)) + round(shared_experts(x)),
 * each term rounded to hidden_type first, exactly like `y = experts(...); y += shared_experts(identity)` on
 * hidden-type tensors.  When the shared expert has the routed experts' shapes and ggml types (DeepSeek-V3) it is
 * computed as an extra slot INSIDE the two routed launches; otherwise it runs as a separate ktb200_mlp_forward.
 * `shared` may be NULL (== ktb200_moe_forward). */
int ktb200_moe_forward_shared(ktb200_moe* moe, ktb200_mlp* shared, int qlen, int k, const int64_t* expert_ids_dev,
                              const float* weights_dev, const void* input_dev, void* output_dev,
                              const int* bsz_tensor_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Activation quantisation exposed for parity tests: from_float(x, Q8_K | Q8_0)
 * (operators/llamafile/conversion.h:27-36 -> ggml-quants.c:3593-3630, :936-1000).
 * out_dev receives packed ggml blocks (292 B / 256 el for Q8_K, 34 B / 32 el for Q8_0).
 * ------------------------------------------------------------------------------------------ */
int ktb200_quantize_activations(const void* x_dev, int hidden_type, long n_rows, long n_cols, int act_type,
                                void* out_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * GGUF block dequantisation (load path).  Replaces KTransformersOps.dequantize_{q8_0,q2_k,q3_k,
 * q4_k,q5_k,q6_k,iq4_xs}(data, num_bytes, blk_size, ele_per_blk, device, dtype)
 * (kt-kernel/cuda/custom_gguf/dequant.cu:343-413, 502-595, 759-789).  src_dev is RAW ggml blocks.
 * out_type: F32 / F16 / BF16.
 * ------------------------------------------------------------------------------------------ */
int ktb200_dequantize(const void* src_dev, int ggml_type, long n_elements, void* out_dev, int out_type,
                      void* stream);

/* Load-time conversion of compressed-tensors pack-quantized INT4 (num_bits 4, group 32, symmetric) into the
 * KTB200_TYPE_RAWINT4_G32 device layout (see the type enum):
 *   packed_dev    int32 [n_rows][n_cols/8]  (`weight_packed`: value i of a word in bits 4i..4i+3, stored as q + 8)
 *   scale_bf16_dev bf16  [n_rows][n_cols/32] (`weight_scale`)
 *   out_dev       caller-owned, n_rows * n_cols / 256 * 144 bytes, 16-byte aligned.
 * Stacked experts are more rows.  KTB200_EINVAL when n_cols % 256 != 0.  Stream-ordered, no allocation. */
int ktb200_rawint4_pack(const int32_t* packed_dev, const uint16_t* scale_bf16_dev, long n_rows, long n_cols, void* out_dev,
                        void* stream);

/* ------------------------------------------------------------------------------------------
 * Router.  Replaces MoEGate.forward (archive/ktransformers/models/modeling_deepseek_v3.py:430-481,
 * reached through KMoEGate, operators/gate.py:91-127) and, for softmax scoring,
 * topk_softmax (kt-kernel/cuda/moe/moe_topk_softmax_kernels.cu:405-462).
 *   logits = x(fp32) . W^T (fp32) ; scores = sigmoid | softmax ; noaux_tc: s' = scores + bias,
 *   group score = sum of top-2 s' in the group, keep topk_group groups, top_k experts by s',
 *   weights = scores[idx] (normalised if norm_topk_prob) * routed_scaling_factor.
 * ------------------------------------------------------------------------------------------ */
typedef struct ktb200_gate_config {
    int n_experts;             /* n_routed_experts */
    int hidden_size;
    int top_k;
    int n_group;               /* 1 = no grouping */
    int topk_group;
    int scoring;               /* 0 sigmoid (V3), 1 softmax (V2) */
    int topk_method;           /* 0 noaux_tc (V3), 1 greedy, 2 group_limited_greedy (V2) */
    int norm_topk_prob;
    float routed_scaling_factor;
    const float* weight;       /* DEVICE fp32 [n_experts][hidden] */
    const float* bias;         /* DEVICE fp32 [n_experts] e_score_correction_bias, or NULL */
    int hidden_type;           /* dtype of x */
} ktb200_gate_config;
/* idx_dev int64 [qlen][top_k] (order: descending biased score, like torch.topk sorted=True — the
 * reference uses sorted=False whose order is unspecified; tests compare as sets), w_dev fp32.
 * logits_dev optional fp32 [qlen][n_experts] scratch/out (NULL -> internal).
 * With bsz_tensor_dev, rows >= max(0, min(qlen, *bsz)) are not written (a negative value selects nothing, like 0).
 * Scratch: one grow-only partial-sum buffer per device (qlen * n_experts * column splits * 4 bytes, at least 1 MB) and a
 * ticket, allocated by the first call and grown by a call that needs more.  Growing cannot be captured: a call on a
 * capturing stream that would allocate or grow returns KTB200_ESTATE before any device work, with a message naming the
 * warm-up — one eager call with the same router and at least as many tokens on that device before capture. */
int ktb200_moe_gate_forward(const ktb200_gate_config* cfg, int qlen, const void* x_dev, int64_t* idx_dev,
                            float* w_dev, float* logits_dev, const int* bsz_tensor_dev, void* stream);

/* Expert-parallel shard form of ktb200_moe_forward_shared: `partial_out` [qlen][hidden] receives the routed partial sums
 * of the experts this shard owns (hidden_type of the moe handle, fp32 for an exact cross-rank sum), and the shared
 * expert is computed for token `own_token` ONLY, as an extra slot of the same two launches; its result goes, rounded
 * to the shared handle's hidden_type, to shared_out [hidden] (it is the second, separately rounded term of
 * `y = experts(x); y += shared_experts(x)`, experts.py:984-1011, to be added after the cross-rank reduction).
 * Needs the bulk-copy kernels (Q4_K gate/up rows of >= 16 super-blocks, tile-layout Q6_K or Q4_K down) and a shared
 * expert with the routed experts' shapes and weight types; KTB200_EINVAL otherwise (run the two calls separately). */
int ktb200_moe_forward_ep(ktb200_moe* moe, ktb200_mlp* shared, int qlen, int k, const int64_t* expert_ids_dev,
                          const float* weights_dev, const void* input_dev, void* partial_out_dev, int own_token,
                          void* shared_out_dev, const int* bsz_tensor_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * The whole MoE block of a decoder layer in ONE call — KDeepseekV3MoE.forward
 * (archive/ktransformers/operators/experts.py:972-1012):
 *     topk_idx, topk_weight = self.gate(hidden_states)          (models/modeling_deepseek_v3.py:430-481)
 *     y = self.experts(hidden_states, topk_idx, topk_weight)    (CPU MOE: operators/llamafile/moe.cpp:146-245)
 *     y += self.shared_experts(identity)                        (n_shared_experts is not None)
 * For decode batches (qlen <= 8) of Q4_K gate/up + Q6_K or Q4_K down experts with rows of 4096..8192 columns this is
 * ONE persistent cooperative launch (router GEMV, grid barrier, top-k in every CTA, gate/up, grid barrier, down +
 * combine; weights stream through the copy engine across the barriers); any other configuration runs as
 * ktb200_moe_gate_forward + ktb200_moe_forward_shared.  Results are bit-identical between the two.
 * idx_dev int64 [qlen][top_k] and w_dev fp32 [qlen][top_k] receive the routing (as from ktb200_moe_gate_forward).
 * `shared` may be NULL.  Capturable as is (its scratch belongs to the moe handle); when it falls back to the separate
 * launches, ktb200_moe_gate_forward's first-call allocation rule applies.
 * ------------------------------------------------------------------------------------------ */
int ktb200_moe_block_forward(const ktb200_gate_config* gate, ktb200_moe* moe, ktb200_mlp* shared, int qlen,
                             const void* input_dev, void* output_dev, int64_t* idx_dev, float* w_dev,
                             const int* bsz_tensor_dev, void* stream);
/* Optional chaining hint for back-to-back layers: during this handle's down-projection phase the block kernel also pulls up
 * to 3 byte ranges (16-byte aligned) into L2 — pass what the NEXT layer's launch reads first (its router weight, its shared
 * expert's gate and up tensors), so that the next launch's latency-bound first microseconds hit L2.  n = 0 clears it. */
int ktb200_moe_block_prefetch_hint(ktb200_moe* moe, const void* const* ptrs, const size_t* bytes, int n);
/* HOST-buffer form (pinned host tensors in / out like the reference's CPU operator, experts.py:293-318): copies the
 * tokens up, runs the block, copies output (+ routing when idx_host / w_host are non-NULL) back, synchronises. */
int ktb200_moe_block_forward_host(const ktb200_gate_config* gate, ktb200_moe* moe, ktb200_mlp* shared, int qlen,
                                  const void* input_host, void* output_host, int64_t* idx_host, float* w_host, void* stream);

/* ------------------------------------------------------------------------------------------
 * Expert-parallel token exchange over NVLink peer memory (one process per GPU).  The reference shards experts over
 * devices with `gpu_experts_mask` and exchanges activations through torch / NCCL (kt-kernel/python/experts_base.py:
 * 377-483, archive/ktransformers/operators/experts.py:143-318 for the CPU<->GPU hand-off); here every rank maps the
 * others' buffers (CUDA IPC / torch symmetric memory: the caller owns the allocation and the mapping) and two small
 * kernels move one decode layer's tokens and partial sums with direct peer stores / loads and system-scope flags.
 *   token_bufs[r]   : rank r's token buffer   [world][hidden] hidden_type   (this rank writes row `rank` of every one)
 *   partial_bufs[r] : rank r's partial buffer [world][hidden] fp32          (this rank reads row `rank` of every one)
 *   flag_bufs[r]    : rank r's flag block, 2*world + 2 uint32, zero-initialised once
 * all three are HOST arrays of `world` DEVICE pointers valid on this rank.  Every rank must issue the same sequence of
 * calls (they are barriers).  Graph-capturable; epochs live in the flag block.
 * ------------------------------------------------------------------------------------------ */
typedef struct ktb200_ep_comm {
    int rank, world, hidden_size, hidden_type;
    void* const* token_bufs;
    float* const* partial_bufs;
    unsigned* const* flag_bufs;
} ktb200_ep_comm;
/* all-gather: x_own [hidden] -> row `rank` of every rank's token buffer; returns when all `world` rows of THIS rank's
 * buffer are complete; x_all_f32 (optional, [world][hidden]) receives them converted to fp32. */
int ktb200_ep_all_gather_tokens(const ktb200_ep_comm* comm, const void* x_own_dev, float* x_all_f32_dev, void* stream);
/* reduce-scatter + epilogue: y_out[hidden] = round_hidden(sum over ranks r of partial_bufs[r][rank][:]) (+ y_shared,
 * the already rounded shared-expert term, optional).  Call after the kernels that wrote this rank's partial buffer. */
int ktb200_ep_reduce_own_token(const ktb200_ep_comm* comm, void* y_out_dev, const void* y_shared_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Expert-parallel MoE block in ONE launch per layer and GPU (decode, one token per GPU): KDeepseekV3MoE.forward
 * (archive/ktransformers/operators/experts.py:972-1012) with the dispatch / combine exchange of
 * archive/ktransformers/models/modeling_deepseek_v3.py:550-605 done INSIDE the kernel over NVLink peer memory:
 *   router + top-k of the rank's own token  ->  the message {x, ids, weights} is stored into every peer's buffer  ->
 *   every rank runs the (token, expert) pairs it owns (gate/up, grid barrier, down, weighted sum per token in slot order)
 *   ->  stores its row slices of all partial sums into the token owners' buffers  ->  each owner adds the `world` partial
 *   rows in rank order, rounds, and adds the rounded shared-expert term (computed locally for its own token).
 * `comm` as for ktb200_ep_all_gather_tokens, except that token_bufs[r] are MESSAGE buffers of
 * world * ktb200_ep_msg_bytes(hidden, type) bytes; flag blocks (2*world + 2 uint32) start zeroed and are private to this
 * call sequence.  Every rank must issue the same sequence of calls.  moe->group_max_len >= world.  idx_dev / w_dev
 * receive the own token's routing.  phase_mask: 7 = the whole layer (production); 1 / 2 / 4 run the route+send, the
 * experts+deliver and the combine phase as separate launches (tests emulate N ranks on one GPU with them).
 * Accepted expert types (gate / up / down, gate and up of one type): Q4_K / Q4_K / {Q4_K, Q6_K}, with a shared expert of the
 * same types and shapes; and {Q2_K, Q3_K} gate / up with {Q2_K, Q3_K, Q4_K, Q6_K} down (llama.cpp's Q2_K, Q3_K_S and Q3_K_M
 * files; hidden_size a multiple of 1024 up to 16384, an even number of blocks per down row for Q3_K).  With Q2_K / Q3_K the
 * shared expert may be of any types ktb200_mlp_forward takes: with the combine phase (phase_mask bit 4) its rounded output is
 * written into y_out on `stream` first, and the kernel adds the cross-rank sum to it; so y_out must not alias x_own (the
 * router still reads x_own after that write).
 * KTB200_EINVAL when the configuration is not the persistent kernel's (see ktb200_moe_block_forward): other type sets (mixed
 * Q2_K / Q3_K gate / up, Q5_K, the i-quants, RAWINT4), or a shape that does not fit shared memory.
 * ------------------------------------------------------------------------------------------ */
long ktb200_ep_msg_bytes(int hidden_size, int hidden_type);
int ktb200_moe_ep_block_forward(const ktb200_gate_config* gate, ktb200_moe* moe, ktb200_mlp* shared, const ktb200_ep_comm* comm,
                                const void* x_own_dev, void* y_out_dev, int64_t* idx_dev, float* w_dev, int phase_mask, void* stream);

/* ------------------------------------------------------------------------------------------
 * Expert-parallel MoE layer for ANY number of tokens per GPU (prompt chunks, mixed batches): KDeepseekV3MoE.forward with the
 * EP branch of DeepseekV3MoE.moe_infer (archive/ktransformers/models/modeling_deepseek_v3.py:550-605), no host round trips.
 * Rank r holds counts[r] tokens (0 allowed) and owns experts [r*E/world, (r+1)*E/world).  Every token's output is what the
 * single-GPU layer computes, up to the order of the fp32 cross-rank sum:
 *   y[t] = round(sum over ranks r in rank order of partial_r[t]) + round(shared(x[t]))
 * partial_r[t] = the fp32 weighted sum of t's experts that rank r owns, in expert_ids order (the shard's ordinary expert
 * kernels, so every expert format ktb200_moe_forward runs is taken, RAWINT4 and the i-quants included).
 * Each rank's region (symmetric: the same layout on every rank, mapped by every peer) holds the message rows {x, ids, weights}
 * per source rank, the fp32 partial rows [world][max_tokens_per_rank][hidden] of its own tokens, a local fp32 scratch and
 * flag words of its own; it starts zeroed and serves every layer (epochs live in it).  ktb200_ep_tokens_layout returns its
 * size in bytes and, when `offsets` is non-NULL, the byte offsets of {x, ids, weights, partial, scratch, flags}; -1 on bad
 * sizes.  flags: send[world] | deliver[world] | 2 epochs | status (1: a peer wait gave up after 4 s) | 2 arrival counters.
 * ------------------------------------------------------------------------------------------ */
typedef struct ktb200_ep_tokens_comm {
    int rank, world, max_tokens_per_rank, hidden_size, hidden_type, top_k;
    void* const* bufs;   /* HOST array of `world` DEVICE pointers valid on this rank: every rank's region */
} ktb200_ep_tokens_comm;
long ktb200_ep_tokens_layout(int world, int max_tokens_per_rank, int hidden_size, int hidden_type, int top_k, long* offsets);
/* counts: HOST int[world], identical on every rank.  x_own / y_out [counts[rank]][hidden] hidden_type; idx_out int64 and
 * w_out fp32 [counts[rank]][top_k] receive the own tokens' routing and must stay untouched until the combine phase.
 * `moe` owns ids [rank * expert_num, (rank + 1) * expert_num) of the gate's n_experts; `shared` may be NULL.
 * phase_mask: 7 = the whole layer; 1 = route + send, 2 = experts + deliver, 4 = shared expert + combine, as separate calls
 * (one GPU can emulate N ranks with them).  Every rank must issue the same sequence of calls.  Eager only (the gate and the
 * grouped expert GEMMs allocate on first use), not capturable.  KTB200_EINVAL before any device work for counts outside
 * [0, max_tokens_per_rank], rank / world out of range, null or not 16-byte aligned peer regions, an x_own that is not 16-byte
 * aligned, and handles whose sizes, types or shard do not fit. */
int ktb200_moe_ep_forward_tokens(const ktb200_gate_config* gate, ktb200_moe* moe, ktb200_mlp* shared, const ktb200_ep_tokens_comm* comm,
                                 const int* counts, const void* x_own_dev, void* y_out_dev, int64_t* idx_dev, float* w_dev, int phase_mask,
                                 void* stream);

/* ------------------------------------------------------------------------------------------
 * Absorbed-MLA paged decode attention.  Replaces MLAWrapper.run / BatchMLAPagedAttentionWrapper
 * (archive/ktransformers/operators/flashinfer_wrapper.py:117-161; attention.py:419-447) and the
 * Triton split-KV decode (triton_attention.py:358-385).
 *   q_nope [B][Hq][512] , q_pe [B][Hq][64]  (bf16)      ; kv cache [pages][page_size][576] bf16
 *   (512 latent ‖ 64 rope), page_table int32 [B][max_pages], kv_len int32 [B]
 *   out [B][Hq][512] bf16 ; lse_out optional fp32 [B][Hq] (natural log)
 * ------------------------------------------------------------------------------------------ */
typedef struct ktb200_mla_params {
    int batch, num_heads, page_size, max_pages_per_seq, num_kv_splits; /* splits <=0: auto; > 128: KTB200_EINVAL */
    float sm_scale;
    const void* q_nope; const void* q_pe; const void* kv_cache;
    const int* page_table; const int* kv_len;
    void* out; float* lse_out;
    void* workspace; size_t workspace_bytes;  /* device scratch for split partials */
    long kv_cache_rows;                       /* pages * page_size of the cache allocation (bounds the TMA tensor map); 0: unknown */
} ktb200_mla_params;
size_t ktb200_mla_workspace_bytes(int batch, int num_heads, int max_splits);
int ktb200_mla_decode(const ktb200_mla_params* p, void* stream);
/* Diagnostics: while non-NULL, one CTA of ktb200_mla_decode dumps the raw scores of its first tile (>= 2048 floats). */
void ktb200_debug_mla(float* debug_dev);
/* ------------------------------------------------------------------------------------------
 * Absorbed-MLA attention of a prompt chunk over the paged latent cache (the reference's absorb_for_prefill path,
 * q_len > 1 through the absorbed branch): no kv_b_proj decompression, the keys straight from the cache.
 *   q_nope [B][q_len][Hq][512], q_pe [B][q_len][Hq][64] (bf16; the ktb200_mla_absorb_q output and the roped q_pe)
 *   kv cache, page_table, kv_cache_rows, sm_scale, num_kv_splits as ktb200_mla_params
 *   kv_len int32 [B]: each sequence's length AFTER the chunk was written to the cache
 *   out [B][q_len][Hq][512] bf16 ; lse_out optional fp32 [B][q_len][Hq] (natural log)
 * Causal, bottom-right aligned as ktb200_mla_prefill: with P = kv_len[b] - q_len, query i attends to keys j <= P + i.
 * The arithmetic is ktb200_mla_decode's; at q_len == 1 the output equals it bit for bit.  Splits are planned on each
 * sequence's last query; automatic splits never exceed ceil(SMs / (batch * q_len * ceil(Hq / 64))) nor 128.
 * KTB200_EINVAL (before any device work) for q_len < 1, null pointers, batch > 65535 or batch * q_len * Hq >= 2^31, a
 * workspace smaller than ktb200_mla_chunk_workspace_bytes for the splits used, and whatever ktb200_mla_decode refuses.
 * kv_len is device data: a sequence with kv_len[b] < q_len is not refused but treated as empty (zeros, lse -inf).
 * ------------------------------------------------------------------------------------------ */
typedef struct ktb200_mla_chunk_params {
    int batch, q_len, num_heads, page_size, max_pages_per_seq, num_kv_splits; /* splits <=0: auto; > 128: KTB200_EINVAL */
    float sm_scale;
    const void* q_nope; const void* q_pe; const void* kv_cache;
    const int* page_table; const int* kv_len;
    void* out; float* lse_out;
    void* workspace; size_t workspace_bytes;
    long kv_cache_rows;
} ktb200_mla_chunk_params;
/* bytes of split partials for batch * q_len query rows; max_splits <= 0: the 128-split maximum; 0 for a non-positive size */
size_t ktb200_mla_chunk_workspace_bytes(int batch, int q_len, int num_heads, int max_splits);
int ktb200_mla_decode_chunk(const ktb200_mla_chunk_params* p, void* stream);
/* ------------------------------------------------------------------------------------------
 * Absorbed-MLA attention of a ragged batch (the reference's BatchMLAPagedAttentionWrapper with a ragged qo_indptr): decode
 * tokens and prompt chunks of sequences at their own positions in one call.  Planned on the host, run on the device:
 *
 * ktb200_mla_ragged_plan (host only, no CUDA call) fills the caller's host buffer `plan` with a work list:
 *   qo_indptr int32 [batch + 1] (HOST): sequence b owns query rows [qo_indptr[b], qo_indptr[b + 1]); q_len_b may be 0
 *   kv_len int32 [batch] (HOST): each sequence's length AFTER this step's tokens were written to the cache
 *   Token i of sequence b attends to keys j < kv_len[b] - q_len_b + i + 1 (bottom-right aligned, as ktb200_mla_decode_chunk).
 *   An item is (query row, 64-head group, tile range, partial slot).  Each sequence's keys are cut once into ranges of
 *   tiles_per[b] tiles of 32 tokens that all its tokens share; a token gets one slot and one item per head group for every
 *   range that starts below its limit.  num_kv_splits > 0: tiles_per[b] = ceil(tiles(kv_len[b]) / splits), the splits clamped
 *   to max_pages_per_seq * page_size / 32, exactly the ranges of ktb200_mla_decode_chunk (and ktb200_mla_decode at q_len 1)
 *   with that split count.  num_kv_splits <= 0: per sequence, the largest item is at most max(4, ceil(W / num_sms)) tiles,
 *   W the (row, head group, tile) work of the whole batch, with at most 128 ranges per sequence; if the items then exceed
 *   max_items, the bound doubles until they fit.
 *   plan_ints >= ktb200_mla_ragged_plan_ints(max_items, max_rows).  n_slots / workspace_bytes (optional) receive the partial
 *   slots and the workspace bytes this plan uses.
 *   KTB200_EINVAL, nothing written, for null pointers, batch < 0, num_heads / max_pages_per_seq / num_sms <= 0, a page_size
 *   that is not a positive multiple of 32, num_kv_splits > 128, qo_indptr[0] != 0 or decreasing, kv_len[b] < q_len_b,
 *   kv_len[b] > max_pages_per_seq * page_size, more rows than max_rows, more items than max_items, a small buffer.
 *
 * ktb200_mla_decode_ragged runs a plan copied to the device (the same int32 buffer, 16-byte aligned):
 *   q_nope [rows][Hq][512], q_pe [rows][Hq][64] (bf16): query rows in qo_indptr order; rows >= the plan's rows
 *   kv cache, page_table [batch][max_pages_per_seq], kv_cache_rows, sm_scale as ktb200_mla_params
 *   out [rows][Hq][512] bf16 ; lse_out optional fp32 [rows][Hq] (natural log): rows past the plan's rows get zeros, lse -inf
 *   max_items: the plan's item capacity.  One CTA per item of the capacity (those past the plan's items return at once), so
 *   a call captured in a CUDA graph serves every later plan of the same capacities; a plan made for another item capacity
 *   reads as empty.  num_heads, page_size, max_pages_per_seq must be those the plan was made with.
 *   The arithmetic is ktb200_mla_decode's.  KTB200_EINVAL (before any device work) for null pointers, rows < 0,
 *   max_items <= 0, rows * Hq >= 2^31, a workspace smaller than ktb200_mla_ragged_workspace_bytes(max_items, Hq), an
 *   unaligned plan, and whatever ktb200_mla_decode_chunk refuses.
 * ------------------------------------------------------------------------------------------ */
typedef struct ktb200_mla_ragged_params {
    int rows, max_items, num_heads, page_size, max_pages_per_seq;
    float sm_scale;
    const void* q_nope; const void* q_pe; const void* kv_cache;
    const int* page_table; const int* plan;
    void* out; float* lse_out;
    void* workspace; size_t workspace_bytes;
    long kv_cache_rows;
} ktb200_mla_ragged_params;
/* int32 elements of a plan: 8 header + 8 per item + max_rows + 1 row offsets; 0 for max_items <= 0 or max_rows < 0 */
size_t ktb200_mla_ragged_plan_ints(int max_items, int max_rows);
/* bytes of split partials for any plan of max_items items (max_items / ceil(Hq / 64) slots); 0 for a non-positive size */
size_t ktb200_mla_ragged_workspace_bytes(int max_items, int num_heads);
int ktb200_mla_ragged_plan(const int* qo_indptr, const int* kv_len, int batch, int num_heads, int page_size, int max_pages_per_seq,
                           int num_sms, int num_kv_splits, int max_items, int max_rows, int* plan, size_t plan_ints, int* n_slots,
                           size_t* workspace_bytes);
int ktb200_mla_decode_ragged(const ktb200_mla_ragged_params* p, void* stream);
/* ------------------------------------------------------------------------------------------
 * Causal MLA prefill attention over the decompressed heads (the non-absorbed prefill of
 * archive/ktransformers/operators/attention.py:349-478: kv_b_proj, then flash_attn_func(..., causal=True)).
 * With P = kv_len - q_len tokens already cached, query i of the chunk sits at position P + i and attends to keys j <= P + i:
 *   s = (q_nope . k_nope_j + q_pe . k_pe_j) * sm_scale  (fp32), online softmax in fp32, P rounded to bf16 before P.V,
 *   out [batch][q_len][num_heads][128] bf16 (contiguous) = (sum_j P_j v_j) / sum_j P_j.
 * Operands (bf16) are read in place; strides are in elements, token / head / batch:
 *   q_nope [.][q_len][num_heads][128], q_pe [.][q_len][num_heads][64]   (e.g. the q_b output view and the roped q_pe)
 *   k_nope, v [.][kv_len][num_heads][128]                               (e.g. the two halves of each head of kv_b_proj's output)
 *   k_pe [.][kv_len][64], shared by all heads                           (e.g. columns 512..575 of the latent cache rows)
 * Head dims must be 128 / 64 / 128.  Every pointer must be 16-byte aligned and every stride a multiple of 8 elements.
 * KTB200_EINVAL (before any device work) for q_len < 1, q_len > kv_len, batch or num_heads < 1, sm_scale <= 0, null
 * pointers, other head dims or misalignment.
 * ------------------------------------------------------------------------------------------ */
typedef struct ktb200_mla_prefill_params {
    int batch, q_len, kv_len, num_heads;
    int qk_nope_head_dim, qk_rope_head_dim, v_head_dim;
    float sm_scale;
    const void* q_nope; long q_nope_token_stride, q_nope_head_stride, q_nope_batch_stride;
    const void* q_pe; long q_pe_token_stride, q_pe_head_stride, q_pe_batch_stride;
    const void* k_nope; long k_nope_token_stride, k_nope_head_stride, k_nope_batch_stride;
    const void* v; long v_token_stride, v_head_stride, v_batch_stride;
    const void* k_pe; long k_pe_token_stride, k_pe_batch_stride;
    void* out;
} ktb200_mla_prefill_params;
int ktb200_mla_prefill(const ktb200_mla_prefill_params* p, void* stream);
/* ------------------------------------------------------------------------------------------
 * Causal MLA prefill over decompressed heads for a batch of sequences of their own lengths (varlen): ktb200_mla_prefill's
 * arithmetic, head dims, alignment and stride rules, with rows in place of the batch dimension.
 *   seq int32 [batch][4] (HOST) = {q_row, q_len, k_row, kv_len}: sequence b's queries are rows q_row .. q_row + q_len - 1
 *   of q_nope / q_pe, its keys rows k_row .. k_row + kv_len - 1 of k_nope / v / k_pe.  With P = kv_len - q_len, query i
 *   sits at position P + i and attends to keys j <= P + i (bottom-right aligned); its output is row q_row + i of
 *   out [q_rows][num_heads][128] bf16 (contiguous).  No other row of out is written; q_len = 0 writes nothing.
 *   q_nope [q_rows][num_heads][128], q_pe [q_rows][num_heads][64], k_nope / v [k_rows][num_heads][128], k_pe [k_rows][64]
 *   (strides in elements, token / head); rows outside the named ranges are never used, whatever they hold.
 * Each sequence's output equals ktb200_mla_prefill on that sequence alone (batch 1) bit for bit.  The sequences travel in
 * the kernel's parameter block: no allocation, no synchronisation, stream-ordered.
 * KTB200_EINVAL (before any device work) for whatever ktb200_mla_prefill refuses, batch outside 1 ..
 * KTB200_MLA_PREFILL_VARLEN_MAX_BATCH, a null seq, negative values, q_len > kv_len, q_len > 65535 * 128, a row range outside
 * q_rows / k_rows, and two sequences whose output rows overlap.
 * ------------------------------------------------------------------------------------------ */
#define KTB200_MLA_PREFILL_VARLEN_MAX_BATCH 1024
typedef struct ktb200_mla_prefill_varlen_params {
    int batch, q_rows, k_rows, num_heads;
    int qk_nope_head_dim, qk_rope_head_dim, v_head_dim;
    float sm_scale;
    const int* seq;
    const void* q_nope; long q_nope_token_stride, q_nope_head_stride;
    const void* q_pe; long q_pe_token_stride, q_pe_head_stride;
    const void* k_nope; long k_nope_token_stride, k_nope_head_stride;
    const void* v; long v_token_stride, v_head_stride;
    const void* k_pe; long k_pe_token_stride;
    void* out;
} ktb200_mla_prefill_varlen_params;
int ktb200_mla_prefill_varlen(const ktb200_mla_prefill_varlen_params* p, void* stream);
/* Debug aid of the grouped (prefill) expert GEMM: when non-null, CTA 0 of the gate and down GEMMs writes clock64 stamps of its
 * first 96 stages, [kernel 2][role 3 = producer, MMA warpgroup, unused][stage 96][4] int64 (tools/grouped_probe.py prints them). */
void ktb200_debug_grouped(long long* trace_dev);

/* ------------------------------------------------------------------------------------------
 * The memory-bound steps between the projections of a DeepSeek decode layer (bf16), fused:
 *   ktb200_add_rmsnorm: residual[t] += delta[t] (delta may be NULL); out[t] = DeepseekV3RMSNorm(residual[t]) * weight
 *     (archive/ktransformers/models/modeling_deepseek_v3.py:65-80 and the residual adds of DeepseekV3DecoderLayer.forward;
 *      operators/layernorm.py).  Also used for q_a_layernorm (delta NULL, residual == the projection output, untouched).
 *   ktb200_mla_prep: after the q_b and kv_a projections of MLA — kv_a_layernorm on the 512 latent columns, RoPE
 *     (de-interleaved pairs, modeling_deepseek_v3.py:339-373) on k_pe and on every head's q_pe, and the paged cache write
 *     (custom_cache.py:147-193): q [T][heads][nope+64], kv_a_out [T][576], cos/sin fp32 [T][64], page_idx/page_offset
 *     int32 [T]; q_pe_out [T][heads][64].
 * Both take dense rows: residual, delta and out are [T][hidden], q is [T][heads][nope+64] and kv_a_out is [T][576], each
 * row right after the previous one.  A view of one projection output whose rows are wider (q_a and kv_a stacked in one
 * [T][q_lora + 576] buffer) is therefore only valid at T = 1.
 * add_rmsnorm: hidden even and <= 8192; residual, delta, weight and out 4-byte aligned (bf16 pairs), else KTB200_EINVAL
 * before any device work (n_tokens = 0 included).
 * ------------------------------------------------------------------------------------------ */
int ktb200_add_rmsnorm(void* residual_dev, const void* delta_dev, const void* weight_dev, float eps, void* out_dev, int n_tokens,
                       int hidden, void* stream);
int ktb200_mla_prep(const void* q_dev, int num_heads, int qk_nope_head_dim, const void* kv_a_out_dev, const void* kv_a_norm_weight_dev,
                    float eps, const float* cos_dev, const float* sin_dev, void* kv_cache_dev, int page_size, const int* page_idx_dev,
                    const int* page_offset_dev, void* q_pe_out_dev, int n_tokens, void* stream);

/* The two absorb products of MLA decode (attention.py:428-431, 470-472): batches of one-row GEMVs over the per-head bf16
 * halves of kv_b_proj — q_abs[t][h][:] = q_nope[t][h][:] . W_UK[h] ([heads][nope][512]; q addressed by element strides so the
 * q_nope slice of the q_b output needs no copy) and out[t][h][:] = attn_latent[t][h][:] . W_UV[h]^T ([heads][v][512]).
 * qk_nope_head_dim <= 512, kv_lora_rank a multiple of 8.  absorb_q: w_uk 16-byte aligned, q_abs_out 4-byte aligned;
 * absorb_o: attn_latent and w_uv 16-byte aligned.  Other arguments give KTB200_EINVAL before any device work
 * (n_tokens = 0 included).  Any n_tokens runs (one launch per 65535 tokens). */
int ktb200_mla_absorb_q(const void* q_dev, long q_head_stride, long q_token_stride, const void* w_uk_dev, int num_heads, int qk_nope_head_dim,
                        int kv_lora_rank, void* q_abs_out_dev, int n_tokens, void* stream);
int ktb200_mla_absorb_o(const void* attn_latent_dev, const void* w_uv_dev, int num_heads, int v_head_dim, int kv_lora_rank, void* out_dev,
                        int n_tokens, void* stream);

/* paged latent KV write: StaticCache.update (archive/ktransformers/models/custom_cache.py:147-200)
 * kv_cache[page_idx[t]][page_offset[t]][0:512] = ckv[t], [512:576] = k_pe[t]; kv_cache, ckv and k_pe 16-byte aligned
 * (KTB200_EINVAL otherwise) */
int ktb200_mla_kv_write(void* kv_cache, int page_size, const void* ckv, const void* k_pe, const int* page_idx,
                        const int* page_offset, int n_tokens, void* stream);

/* Diagnostics (bench.py --probe): time a plain read-only stream over `bytes` of device memory.
 * mode 0 = grid-stride coalesced 16-byte loads; mode 1 = every warp reads chunk_bytes pieces at hashed offsets
 * (the access shape of the expert GEMV).  Establishes the practical read ceiling next to MEASURED_PEAKS' copy figure. */
int ktb200_debug_stream_read(const void* src_dev, long bytes, int mode, int unroll, int ctas_per_sm, int chunk_bytes,
                             void* stream, float* ms_out);
/* mode 2 of the probe above: the bulk-copy ring of the expert kernels without arithmetic (unroll = ring slots,
 * ctas_per_sm = warps per CTA).
 * Phase trace of ktb200_moe_block_forward (profiles/block_trace.py): while trace_dev != NULL, thread 0 of every CTA
 * writes %globaltimer at the phase boundaries into trace_dev[cta][16] (uint64, >= num_SMs * 16 entries). */
void ktb200_debug_block_trace(unsigned long long* trace_dev);
/* The synchronisation words of the handle's MoE-block launches, copied to host memory after a device synchronise: grid
 * barrier words [0..3], the timeout status word [4], then the per-Q8_K-block readiness words.  Every word is 0 between
 * launches.  Copies min(n, total) words to host_out (may be NULL) and returns the total, or -1 on error. */
long ktb200_debug_block_sync_words(ktb200_moe* moe, unsigned* host_out, long n);
/* The router's two ticket words on `device` (finished CTAs, finished selectors), copied to host_out[2] after a device
 * synchronise.  Both are 0 between ktb200_moe_gate_forward launches.  KTB200_ESTATE before the first router call there. */
int ktb200_debug_gate_ticket(int device, unsigned* host_out);

#ifdef __cplusplus
}
#endif
#endif /* KTB200_H */
