"""Test-only numpy restatement of the IQ3_XXS and IQ3_S formats and of the arithmetic the expert kernels implement for them.

block_iq3_xxs (include/ktb200.h), 98 B per 256 values: fp16 d, qs[64] (8-bit indices into the 256 x 4 iq3xxs_grid, values
4..62), then one 32-bit word per 32-value sub-block: four 7-bit indices into ksigns_iq2xs and the 4-bit scale s in bits 28..31;
value = d (2s + 1) / 4 * grid * sign.

block_iq3_s, 110 B: fp16 d, qs[64], qh[8] (bit j % 8 of qh[j / 8] is bit 8 of the iq3s_grid index of 4-value group j; 512 x 4
entries, values 1..15), signs[32] (bit i of signs[k] negates value 8k + i), scales[4] (sub-block ib: nibble ib % 2 of
scales[ib / 2], low nibble for even ib); value = d (2s + 1) * grid * sign.

`dequant` restates gguf-py's dequantisers in their fp32 operation order; `superblock_ints` gives the exact integer
S = sum_ib (2s + 1) * sum (+-grid) q8 of ggml_vec_dot_iq3_xxs_q8_K / ggml_vec_dot_iq3_s_q8_K, `superblock_terms` the
kernels' fp32 term per super-block ((d / 4) dx S and (d dx) S) and `vec_dot` the reference's fp32 sum.
"""
from __future__ import annotations

import numpy as np
from gguf import quants

from iq_oracle import KSIGNS, q8k_fields

IQ3_XXS, IQ3_S = 18, 21
BLOCK_BYTES = {IQ3_XXS: 98, IQ3_S: 110}


def _grid(cls):
    cls.init_grid()
    return np.asarray(cls.grid).reshape(cls.grid_shape).astype(np.int64)


IQ3XXS_GRID = _grid(quants.IQ3_XXS)                                            # [256][4], 4 .. 62
IQ3S_GRID = _grid(quants.IQ3_S)                                                # [512][4], 1 .. 15


def random_blocks(t: int, n_blocks: int, rng: np.random.Generator, d_scale: float = 1.0) -> np.ndarray:
    """any bit pattern is a valid block: random bytes with a sane fp16 `d` (uniform in [0.75, 1.25) * d_scale)"""
    b = rng.integers(0, 256, size=(n_blocks, BLOCK_BYTES[t]), dtype=np.uint8)
    d = ((rng.random(n_blocks) * 0.5 + 0.75) * d_scale).astype(np.float16)
    b[:, 0:2] = d.view(np.uint8).reshape(n_blocks, 2)
    return b


def fields(t: int, blocks):
    """d [n] fp32, ls [n][8] (2s + 1 per 32-value sub-block), values [n][8][32] (+-grid, the sign applied)"""
    b = np.asarray(blocks, np.uint8).reshape(-1, BLOCK_BYTES[t])
    d = b[:, 0:2].copy().view(np.float16).astype(np.float32).reshape(-1)
    qs = b[:, 2:66].astype(np.int64)                                            # [n][64]
    if t == IQ3_XXS:
        aux = b[:, 66:98].copy().view(np.uint32).astype(np.int64)              # [n][8]
        ls = 2 * (aux >> 28) + 1
        signs = KSIGNS[(aux[:, :, None] >> (7 * np.arange(4))) & 127]          # [n][8][4]: values 8l .. 8l + 7
        neg = ((signs[..., None] >> np.arange(8)) & 1).reshape(-1, 8, 32)
        grid = IQ3XXS_GRID[qs].reshape(-1, 8, 32)
    else:
        qh = b[:, 66:74].astype(np.int64)                                       # [n][8]
        idx = qs | (((qh[:, :, None] >> np.arange(8)) & 1).reshape(-1, 64) << 8)
        grid = IQ3S_GRID[idx].reshape(-1, 8, 32)
        sg = b[:, 74:106].astype(np.int64)                                      # [n][32]
        neg = ((sg[:, :, None] >> np.arange(8)) & 1).reshape(-1, 8, 32)
        sc = b[:, 106:110].astype(np.int64)
        ls = 2 * ((sc[:, :, None] >> (4 * np.arange(2))) & 15).reshape(-1, 8) + 1
    return d, ls, np.where(neg == 1, -grid, grid)


def dequant(t: int, blocks) -> np.ndarray:
    """gguf-py's order: IQ3_XXS db = d * (0.5 + s) * 0.5, IQ3_S db = d * (1 + 2s); value = db * grid * sign (fp32)"""
    d, ls, v = fields(t, blocks)
    s = ((ls - 1) // 2).astype(np.float32)
    if t == IQ3_XXS:
        db = ((d[:, None] * (np.float32(0.5) + s)) * np.float32(0.5)).astype(np.float32)
    else:
        db = (d[:, None] * (np.float32(1) + np.float32(2) * s)).astype(np.float32)
    return (db[:, :, None] * v.astype(np.float32)).astype(np.float32).reshape(-1)


def superblock_ints(t: int, w_blocks, q8) -> np.ndarray:
    """S = sum_ib ls_ib * sum (+-grid) q8, the reference's bsum"""
    _, ls, v = fields(t, w_blocks)
    q = q8k_fields(q8)[1].reshape(-1, 8, 32)
    return (ls * (v * q).sum(axis=2)).sum(axis=1)


def superblock_terms(t: int, w_blocks, q8) -> np.ndarray:
    """the kernels' fp32 term per super-block: IQ3_XXS ((d / 4) dx) S, IQ3_S (d dx) S"""
    d = fields(t, w_blocks)[0]
    if t == IQ3_XXS:
        d = (d * np.float32(0.25)).astype(np.float32)
    dx = q8k_fields(q8)[0]
    return ((d * dx).astype(np.float32) * superblock_ints(t, w_blocks, q8).astype(np.float32)).astype(np.float32)


def vec_dot(t: int, w_blocks, q8) -> np.float32:
    """ggml_vec_dot_iq3_xxs_q8_K / ggml_vec_dot_iq3_s_q8_K (scalar branch): fp32 sum of (d dx) S over super-blocks in order;
    IQ3_XXS scales the total by 0.25 once"""
    d, dx = fields(t, w_blocks)[0], q8k_fields(q8)[0]
    acc = np.float32(0)
    for v in ((d * dx).astype(np.float32) * superblock_ints(t, w_blocks, q8).astype(np.float32)).astype(np.float32):
        acc = np.float32(acc + v)
    return np.float32(acc * np.float32(0.25)) if t == IQ3_XXS else acc
