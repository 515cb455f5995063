"""Test-only numpy restatement of the RAWINT4_G32 format and of the routed-expert arithmetic the kernels implement.

Written from the compressed-tensors "pack-quantized" description (num_bits 4, group 32, symmetric), not from the library:
  weight_packed int32 [rows][cols/8]: column 8w+i of a row in bits 4i..4i+3 of word w, stored as q + 8
  weight_scale  bf16  [rows][cols/32]
  weight = q * scale = (u - 8) * scale
The MoE is computed in float64 over the experts that are hit: out[t] = sum_j w[t,j] * down_e(silu(gate_e x) * up_e x).
"""
from __future__ import annotations

import numpy as np


def bf16_bits_to_f64(b: np.ndarray) -> np.ndarray:
    return (np.asarray(b, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def f32_to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """round to nearest even (finite inputs)"""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def unpack(packed: np.ndarray) -> np.ndarray:
    """weight_packed [..., cols/8] int32 -> q [..., cols] int8 in -8..7"""
    w = np.asarray(packed).view(np.uint32)
    nib = (w[..., :, None] >> (4 * np.arange(8, dtype=np.uint32))) & 0xF       # [..., cols/8, 8]: column 8w+i
    return (nib.astype(np.int16) - 8).astype(np.int8).reshape(*w.shape[:-1], w.shape[-1] * 8)


def pack(q: np.ndarray) -> np.ndarray:
    """q [..., cols] int8 in -8..7 -> weight_packed int32 (the inverse of unpack)"""
    u = (np.asarray(q).astype(np.int16) + 8).astype(np.uint32).reshape(*q.shape[:-1], q.shape[-1] // 8, 8)
    return (u << (4 * np.arange(8, dtype=np.uint32))).sum(axis=-1, dtype=np.uint32).view(np.int32)


def dequant(packed: np.ndarray, scale_bits: np.ndarray) -> np.ndarray:
    """float64 [..., rows, cols]"""
    q = unpack(packed).astype(np.float64)
    s = bf16_bits_to_f64(scale_bits)
    return (q.reshape(*s.shape, 32) * s[..., None]).reshape(q.shape)


def device_layout(packed: np.ndarray, scale_bits: np.ndarray) -> np.ndarray:
    """The KTB200_TYPE_RAWINT4_G32 blocks of [rows][cols] (include/ktb200.h): per 256 columns, 16 bytes of the eight bf16
    scales, then the 32 packed words unchanged.  uint8 [rows * cols/256 * 144]."""
    p = np.ascontiguousarray(packed).view(np.uint32)
    s = np.ascontiguousarray(scale_bits).astype(np.uint16)
    rows, nb = p.reshape(-1, p.shape[-1]).shape[0], p.shape[-1] // 32
    words = p.reshape(rows, nb, 32).view(np.uint8).reshape(rows, nb, 128)
    scl = s.reshape(rows, nb, 8).view(np.uint8).reshape(rows, nb, 16)
    return np.concatenate([scl, words], axis=2).reshape(-1)


def silu(x):
    return x / (1.0 + np.exp(-x))


def moe_forward(x: np.ndarray, ids: np.ndarray, weights: np.ndarray, expert, n_experts: int, id_offset: int = 0,
                use_silu: bool = True) -> np.ndarray:
    """x float [T][H], ids [T][k], weights [T][k]; expert(e) -> (gate [I][H], up [I][H], down [H][I]) float64 for local
    expert e.  Ids outside [id_offset, id_offset + n_experts) are skipped.  Returns float64 [T][H]."""
    x = np.asarray(x, dtype=np.float64)
    T, k = ids.shape
    local = ids.astype(np.int64) - id_offset
    out = np.zeros_like(x)
    for e in np.unique(local):
        if e < 0 or e >= n_experts:
            continue
        g, u, d = expert(int(e))
        tok, slot = np.nonzero(local == e)
        xe = x[tok]
        h = xe @ g.T
        a = (silu(h) if use_silu else np.maximum(h, 0.0)) * (xe @ u.T)
        y = a @ d.T
        np.add.at(out, tok, y * weights[tok, slot, None].astype(np.float64))
    return out
