"""GGUF constants and HF->GGUF tensor-name translation.

Behavioural mirror of archive/ktransformers/util/custom_gguf.py (constants :34-131, name
translation :665-746).  Block geometry per ggml type is (elements per block, bytes per block).
"""
from __future__ import annotations

import re
from enum import IntEnum

import numpy as np
import torch


class GGMLQuantizationType(IntEnum):
    F32 = 0
    F16 = 1
    Q4_0 = 2
    Q4_1 = 3
    Q5_0 = 6
    Q5_1 = 7
    Q8_0 = 8
    Q8_1 = 9
    Q2_K = 10
    Q3_K = 11
    Q4_K = 12
    Q5_K = 13
    Q6_K = 14
    Q8_K = 15
    IQ2_XXS = 16
    IQ2_XS = 17
    IQ3_XXS = 18
    IQ1_S = 19
    IQ4_NL = 20
    IQ3_S = 21
    IQ2_S = 22
    IQ4_XS = 23
    I8 = 24
    I16 = 25
    I32 = 26
    I64 = 27
    F64 = 28
    IQ1_M = 29
    BF16 = 30


QK_K = 256
# (elements per block, bytes per block)
GGML_QUANT_SIZES = {
    GGMLQuantizationType.F32: (1, 4), GGMLQuantizationType.F16: (1, 2), GGMLQuantizationType.BF16: (1, 2),
    GGMLQuantizationType.Q4_0: (32, 18), GGMLQuantizationType.Q4_1: (32, 20), GGMLQuantizationType.Q5_0: (32, 22),
    GGMLQuantizationType.Q5_1: (32, 24), GGMLQuantizationType.Q8_0: (32, 34), GGMLQuantizationType.Q8_1: (32, 40),
    GGMLQuantizationType.Q2_K: (256, 84), GGMLQuantizationType.Q3_K: (256, 110), GGMLQuantizationType.Q4_K: (256, 144),
    GGMLQuantizationType.Q5_K: (256, 176), GGMLQuantizationType.Q6_K: (256, 210), GGMLQuantizationType.Q8_K: (256, 292),
    GGMLQuantizationType.IQ2_XXS: (256, 66), GGMLQuantizationType.IQ2_XS: (256, 74), GGMLQuantizationType.IQ3_XXS: (256, 98),
    GGMLQuantizationType.IQ1_S: (256, 50), GGMLQuantizationType.IQ4_NL: (32, 18), GGMLQuantizationType.IQ3_S: (256, 110),
    GGMLQuantizationType.IQ2_S: (256, 82), GGMLQuantizationType.IQ4_XS: (256, 136), GGMLQuantizationType.I8: (1, 1),
    GGMLQuantizationType.I16: (1, 2), GGMLQuantizationType.I32: (1, 4), GGMLQuantizationType.I64: (1, 8),
    GGMLQuantizationType.F64: (1, 8), GGMLQuantizationType.IQ1_M: (256, 56),
}
GGML_NAMES = {int(t): t.name for t in GGMLQuantizationType}
GGML_TYPES = {t.name: int(t) for t in GGMLQuantizationType}
GGML_ELEMENTS_PER_BLOCK = {t.name: GGML_QUANT_SIZES[t][0] for t in GGML_QUANT_SIZES}
GGML_BLOCK_SIZES = {t.name: GGML_QUANT_SIZES[t][1] for t in GGML_QUANT_SIZES}

# types the sm_90a kernels consume / dequantise directly
B200_WEIGHT_TYPES = {"Q2_K", "Q3_K", "Q4_K", "Q5_K", "Q6_K", "IQ4_XS"}
# routed experts also take ggml's codebook i-quants (DeepSeek-R1's 1.5-2-bit GGUF files); linears and MLPs do not
B200_EXPERT_TYPES = B200_WEIGHT_TYPES | {"IQ1_S", "IQ2_XXS"}
# what the routed-expert loaders accept: kept apart from B200_EXPERT_TYPES, whose value callers and tests rely on
B200_ROUTED_EXPERT_TYPES = B200_EXPERT_TYPES | {"IQ1_M"}
B200_DEQUANT_TYPES = B200_ROUTED_EXPERT_TYPES | {"Q8_0", "F32", "F16", "BF16"}
# the (gate/up, down) type sets the single-launch expert-parallel kernel takes (gate and up of one type): Q4_K gate/up with
# Q4_K or Q6_K down, and Q2_K or Q3_K gate/up with Q2_K, Q3_K, Q4_K or Q6_K down (llama.cpp's Q2_K, Q3_K_S and Q3_K_M files)
B200_EP_TYPE_SETS = {("Q4_K", "Q4_K"), ("Q4_K", "Q6_K")} | {(gu, d) for gu in ("Q2_K", "Q3_K") for d in ("Q2_K", "Q3_K", "Q4_K", "Q6_K")}

TORCH_TO_GGML_HIDDEN = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 30}

# GGUF metadata value types
DATA_TYPES = {"uint8": 0, "int8": 1, "uint16": 2, "int16": 3, "uint32": 4, "int32": 5, "float32": 6, "bool": 7,
              "string": 8, "array": 9, "uint64": 10, "int64": 11, "float64": 12}


def quant_shape_to_byte_shape(shape, ggml_type) -> tuple:
    epb, bpb = GGML_QUANT_SIZES[GGMLQuantizationType(ggml_type)]
    if shape[-1] % epb != 0:
        raise ValueError(f"Quantized tensor row size ({shape[-1]}) is not a multiple of {GGML_NAMES[int(ggml_type)]} block size ({epb})")
    return (*shape[:-1], shape[-1] // epb * bpb)


# ---- HF module path -> GGUF tensor name ------------------------------------------------------------
_EXPERT_RE = re.compile(r"(?:model\.layers|blk)\.(\d+)\.mlp\.experts\.(\d+)\.(gate_proj|up_proj|down_proj)")
_MIXTRAL_RE = re.compile(r"model\.layers\.(\d+)\.block_sparse_moe\.experts\.(\d+)\.(w\d)\.weight")
_MIXTRAL_W = {"w1": "ffn_gate", "w2": "ffn_down", "w3": "ffn_up"}
_PROJ = {"gate_proj": "ffn_gate_exps", "up_proj": "ffn_up_exps", "down_proj": "ffn_down_exps"}

# ordered: earlier entries must win over later, more general ones
_RENAMES = [
    ("lm_head.", "output."), ("model.embed_tokens.", "token_embd."), ("model.norm.", "output_norm."),
    ("model.layers.", "blk."), (".input_layernorm", ".attn_norm"), (".mlp.down_proj", ".ffn_down"),
    (".mlp.gate_proj", ".ffn_gate"), (".mlp.up_proj", ".ffn_up"), (".post_attention_layernorm", ".ffn_norm"),
    (".self_attn.q_proj", ".attn_q"), (".self_attn.k_proj", ".attn_k"), (".self_attn.v_proj", ".attn_v"),
    (".self_attn.o_proj", ".attn_output"), (".self_attn.qkv_proj", ".attn_qkv"),
    (".self_attn.kv_a_proj_with_mqa", ".attn_kv_a_mqa"), (".self_attn.kv_a_layernorm", ".attn_kv_a_norm"),
    (".self_attn.kv_b_proj", ".attn_kv_b"), (".self_attn.q_a_proj", ".attn_q_a"),
    (".self_attn.q_a_layernorm", ".attn_q_a_norm"), (".self_attn.q_b_proj", ".attn_q_b"),
    (".self_attn.q_norm", ".attn_q_norm"), (".self_attn.k_norm", ".attn_k_norm"),
    (".shared_expert.", ".shared_experts."), (".shared_expert_", ".shared_experts_"), (".gate_up_proj.", ".up_proj"),
    (".mlp.shared_experts.down_proj", ".ffn_down_shexp"), (".mlp.gate.e_score_correction_bias", ".exp_probs_b.bias"),
    (".mlp.gate", ".ffn_gate_inp"), (".mlp.shared_experts.gate_proj", ".ffn_gate_shexp"),
    (".mlp.shared_experts.up_proj", ".ffn_up_shexp"), (".mlp.shared_experts_gate", ".ffn_gate_inp_shexp"),
    (".mlp.experts", ""), (".block_sparse_moe.gate.", ".ffn_gate_inp."), (".block_sparse_moe.experts", ""),
    (".feed_forward.experts", ""), (".feed_forward.router", ".ffn_gate_inp"),
    (".feed_forward.shared_experts.down_proj", ".ffn_down_shexp"),
    (".feed_forward.shared_experts.gate_proj", ".ffn_gate_shexp"),
    (".feed_forward.shared_experts.up_proj", ".ffn_up_shexp"),
]


def translate_name_to_gguf(name: str) -> str:
    """HF parameter/module path -> GGUF tensor name (same mapping as the reference, :665-746)."""
    name = _MIXTRAL_RE.sub(lambda m: f"blk.{m.group(1)}.{_MIXTRAL_W[m.group(3)]}.{m.group(2)}.weight", name)
    for s in ("gate", "up", "down"):
        name = name.replace(f".ffn_{s}_exp.", f".ffn_{s}_exps.")
    m = _EXPERT_RE.match(name)
    if m:
        layer, expert, proj = m.groups()
        return f"blk.{layer}.{expert}.{_PROJ[proj]}"
    for old, new in _RENAMES:
        name = name.replace(old, new)
    return name


def dequantize_cpu(data: np.ndarray, ggml_type: int) -> np.ndarray:
    """CPU dequantisation for tensors a rule places on the CPU (rare on this path).  Uses the `gguf`
    package's reference implementation; the GPU path never calls this."""
    t = GGMLQuantizationType(ggml_type)
    if t == GGMLQuantizationType.F32:
        return np.frombuffer(data, dtype=np.float32)
    if t == GGMLQuantizationType.F16:
        return np.frombuffer(data, dtype=np.float16)
    if t == GGMLQuantizationType.BF16:
        return np.frombuffer(data, dtype=np.int16)
    try:
        import gguf
    except ImportError as e:  # pragma: no cover
        raise NotImplementedError(f"CPU dequantisation of {t.name} needs the `gguf` package") from e
    return gguf.quants.dequantize(np.frombuffer(data, dtype=np.uint8), gguf.GGMLQuantizationType(int(t)))
