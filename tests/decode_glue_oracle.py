"""TEST INFRASTRUCTURE ONLY — float64 numpy restatement of the small kernels between the projections of a DeepSeek decode
layer (csrc/elementwise.cu): residual add + RMSNorm, MLA prep (kv_a norm, RoPE of k_pe and q_pe, paged cache row) and the
two absorb products.

Reference math: DeepseekV3RMSNorm and apply_rotary_pos_emb (models/modeling_deepseek_v3.py, restating the reference's
modeling_deepseek_v3.py:65-80 and :339-373), the residual adds of DeepseekV3DecoderLayer.forward, StaticCache.update
(custom_cache.py:147-193) and the absorbed decode's q_nope . W_UK / latent . W_UV^T (attention.py:428-431, 470-472).
Inputs are bf16 values held in float arrays; every result is float64 with the module's bf16 rounding points applied
explicitly (`bf16`, round to nearest even from float64).  tests/test_decode_glue.py pins `rope` and `add_rmsnorm` to the
module code on CPU bf16 tensors.
"""
from __future__ import annotations

import numpy as np

ROPE, LATENT = 64, 512


def bf16(x) -> np.ndarray:
    """Round to the nearest bf16 value (ties to even) directly from float64; overflow gives +-inf."""
    x = np.asarray(x, np.float64)
    m, e = np.frexp(x)                                    # x = m * 2^e, 0.5 <= |m| < 1: bf16 keeps 8 significant bits
    r = np.ldexp(np.rint(m * 256.0), e - 8)
    sub = np.abs(x) < 2.0 ** -126                         # bf16 subnormals: multiples of 2^-133
    r = np.where(sub, np.rint(x * 2.0 ** 133) * 2.0 ** -133, r)
    return np.where(np.abs(r) > 3.3895313892515355e38, np.copysign(np.inf, x), r)


def add_rmsnorm(res, delta, w, eps):
    """-> (r, out): r = bf16(res + delta) (res when delta is None), out = bf16(w * bf16(r / sqrt(mean(r^2) + eps)))"""
    r = np.asarray(res, np.float64)
    if delta is not None:
        r = bf16(r + np.asarray(delta, np.float64))
    inv = 1.0 / np.sqrt(np.mean(r * r, axis=-1, keepdims=True) + eps)
    return r, bf16(np.asarray(w, np.float64) * bf16(r * inv))


def deinterleave(x):
    """the permutation apply_rotary_pos_emb applies first: pairs (x[2i], x[2i+1]) -> x[0::2] || x[1::2]"""
    x = np.asarray(x, np.float64)
    return np.concatenate([x[..., 0::2], x[..., 1::2]], axis=-1)


def rope(x64, cos, sin, fp32_products=False):
    """apply_rotary_pos_emb on the last axis (64 wide): x' = deinterleave(x), rot(x') = (-x'[32:], x'[:32]),
    bf16(bf16(x' cos) + bf16(rot(x') sin)); cos / sin broadcast against x64.  With bf16 tables the products are exact in
    fp32; with fp32 tables ktb200_mla_prep rounds each product to fp32 before bf16 (`fp32_products=True` does the same)."""
    xp = deinterleave(x64)
    half = xp.shape[-1] // 2
    rot = np.concatenate([-xp[..., half:], xp[..., :half]], axis=-1)
    p0, p1 = xp * np.asarray(cos, np.float64), rot * np.asarray(sin, np.float64)
    if fp32_products:
        p0, p1 = p0.astype(np.float32).astype(np.float64), p1.astype(np.float32).astype(np.float64)
    return bf16(bf16(p0) + bf16(p1))


def mla_prep(q, nope, kva, kv_norm_w, eps, cos, sin, page_idx, page_off, fp32_products=False):
    """q [T][heads][nope + 64], kva [T][576], cos / sin [T][64], page_idx / page_off [T] ->
    (q_pe_out [T][heads][64], {(page_idx[t], page_off[t]): cache row [576] = kv_a_norm(kva[t][:512]) || rope(kva[t][512:])})"""
    q, kva = np.asarray(q, np.float64), np.asarray(kva, np.float64)
    cos, sin = np.asarray(cos, np.float64), np.asarray(sin, np.float64)
    q_pe = rope(q[..., nope:nope + ROPE], cos[:, None], sin[:, None], fp32_products)
    _, lat = add_rmsnorm(kva[:, :LATENT], None, kv_norm_w, eps)
    k_pe = rope(kva[:, LATENT:], cos, sin, fp32_products)
    rows = np.concatenate([lat, k_pe], axis=-1)
    return q_pe, {(int(p), int(o)): rows[t] for t, (p, o) in enumerate(zip(page_idx, page_off))}


def absorb_q(q, w_uk):
    """q_nope [T][heads][D], W_UK [heads][D][C] -> (einsum("thd,hdc->thc"), sum_d |q W|), both float64"""
    q, w = np.asarray(q, np.float64), np.asarray(w_uk, np.float64)
    qt = q.transpose(1, 0, 2)
    return (qt @ w).transpose(1, 0, 2), (np.abs(qt) @ np.abs(w)).transpose(1, 0, 2)


def absorb_o(lat, w_uv):
    """latents [T][heads][C], W_UV [heads][V][C] -> (einsum("thc,hvc->thv"), sum_c |lat W|), both float64"""
    lat, w = np.asarray(lat, np.float64), np.asarray(w_uv, np.float64)
    lt, wt = lat.transpose(1, 0, 2), w.transpose(0, 2, 1)
    return (lt @ wt).transpose(1, 0, 2), (np.abs(lt) @ np.abs(wt)).transpose(1, 0, 2)
