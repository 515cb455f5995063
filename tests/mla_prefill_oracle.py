"""TEST INFRASTRUCTURE ONLY — float64 numpy restatement of causal MLA prefill attention over decompressed heads.

Reference math: the non-absorbed prefill of archive/ktransformers/operators/attention.py:349-478 (kv_b_proj, then
flash_attn_func(q, k, v, softmax_scale, causal=True) with k = k_nope ‖ k_pe expanded per head and v padded to 192), which
models/modeling_deepseek_v3.DeepseekV3Attention.forward restates in torch.  With S keys and q_len queries, query i sits at
position S - q_len + i and sees keys j <= S - q_len + i (the bottom-right causal mask):
    s[i,j] = (q_nope[i] . k_nope[j] + q_pe[i] . k_pe[j]) * sm_scale ;  out[i] = softmax_j(s) . v
`p_bf16=True` rounds exp(s - max) to bf16 before the product with v and divides by the unrounded sum, as the kernels do
(P in bf16 before P.V, fp32 row sums).
"""
from __future__ import annotations

import numpy as np


def bf16_round(x: np.ndarray) -> np.ndarray:
    """Round to the nearest bf16 value (ties to even), returned as float32."""
    i = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    r = ((i + (0x7FFF + ((i >> 16) & 1))) >> 16).astype(np.uint32) << 16
    return r.view(np.float32)


def mla_prefill(q_nope, q_pe, k_nope, k_pe, v, sm_scale, p_bf16: bool = False):
    """q_nope [B,q,H,128], q_pe [B,q,H,64], k_nope [B,S,H,128], k_pe [B,S,64], v [B,S,H,128] -> out [B,q,H,128] float64."""
    q_nope, q_pe, k_nope, k_pe, v = (np.asarray(a, np.float64) for a in (q_nope, q_pe, k_nope, k_pe, v))
    B, q_len, H, _ = q_nope.shape
    S = k_nope.shape[1]
    s = (q_nope.transpose(0, 2, 1, 3) @ k_nope.transpose(0, 2, 3, 1) + q_pe.transpose(0, 2, 1, 3) @ k_pe.transpose(0, 2, 1)[:, None]) * sm_scale
    mask = np.arange(S)[None, :] > (S - q_len + np.arange(q_len))[:, None]
    s = np.where(mask[None, None], -np.inf, s)
    m = s.max(-1, keepdims=True)
    e = np.exp(s - m)
    den = e.sum(-1, keepdims=True)
    if p_bf16:
        e = bf16_round(e.astype(np.float32)).astype(np.float64)
    return ((e / den) @ v.transpose(0, 2, 1, 3)).transpose(0, 2, 1, 3)
