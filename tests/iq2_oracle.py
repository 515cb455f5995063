"""Test-only numpy restatement of the IQ2_XS and IQ2_S formats and of the arithmetic the expert kernels implement for them.

block_iq2_xs (include/ktb200.h), 74 B per 256 values: fp16 d, qs uint16[32] (8-value group l: bits 0..8 index the 512 x 8
iq2xs_grid, values 8 / 25 / 43; bits 9..15 index ksigns_iq2xs), scales[8] (32-value sub-block ib: the low nibble scales values
0..15, the high nibble values 16..31); value = d (2s + 1) / 8 * grid * sign.

block_iq2_s, 82 B: fp16 d, qs[32], signs[32], qh[8], scales[8]; 8-value group l is iq2s_grid[qs[l] | ((qh[l / 4] >> 2 (l % 4))
& 3) << 8] (1024 x 8 entries, values 8 / 25 / 43), bit i of signs[l] negates its value i, the scales as IQ2_XS.

`dequant` restates gguf-py's dequantisers in their fp32 operation order; `superblock_ints` gives the exact integer
S = sum_ib (ls1 * sum_(first 16) (+-grid) q8 + ls2 * sum_(second 16) (+-grid) q8) of ggml_vec_dot_iq2_xs_q8_K /
ggml_vec_dot_iq2_s_q8_K, `superblock_terms` the kernels' fp32 term per super-block ((d / 8) dx S) and `vec_dot` the
reference's fp32 sum.
"""
from __future__ import annotations

import numpy as np
from gguf import quants

from iq_oracle import KSIGNS, q8k_fields

IQ2_XS, IQ2_S = 17, 22
BLOCK_BYTES = {IQ2_XS: 74, IQ2_S: 82}


def _grid(cls):
    cls.init_grid()
    return np.asarray(cls.grid).reshape(cls.grid_shape).astype(np.int64)


IQ2XS_GRID = _grid(quants.IQ2_XS)                                              # [512][8], 8 / 25 / 43
IQ2S_GRID = _grid(quants.IQ2_S)                                                # [1024][8], 8 / 25 / 43


def random_blocks(t: int, n_blocks: int, rng: np.random.Generator, d_scale: float = 1.0) -> np.ndarray:
    """any bit pattern is a valid block: random bytes with a sane fp16 `d` (uniform in [0.75, 1.25) * d_scale)"""
    b = rng.integers(0, 256, size=(n_blocks, BLOCK_BYTES[t]), dtype=np.uint8)
    d = ((rng.random(n_blocks) * 0.5 + 0.75) * d_scale).astype(np.float16)
    b[:, 0:2] = d.view(np.uint8).reshape(n_blocks, 2)
    return b


def grid_indices(t: int, blocks) -> np.ndarray:
    """[n][32] the grid index of every 8-value group"""
    b = np.asarray(blocks, np.uint8).reshape(-1, BLOCK_BYTES[t])
    if t == IQ2_XS:
        return b[:, 2:66].copy().view(np.uint16).astype(np.int64) & 511
    qh = b[:, 66:74].astype(np.int64)
    return b[:, 2:34].astype(np.int64) | (((qh[:, :, None] >> (2 * np.arange(4))) & 3).reshape(-1, 32) << 8)


def fields(t: int, blocks):
    """d [n] fp32, ls [n][16] (2s + 1 per 16 values), values [n][16][16] (+-grid, the sign applied)"""
    b = np.asarray(blocks, np.uint8).reshape(-1, BLOCK_BYTES[t])
    d = b[:, 0:2].copy().view(np.float16).astype(np.float32).reshape(-1)
    idx = grid_indices(t, b)
    if t == IQ2_XS:
        signs = KSIGNS[b[:, 2:66].copy().view(np.uint16).astype(np.int64) >> 9]  # [n][32]
        grid = IQ2XS_GRID[idx]
        sc = b[:, 66:74].astype(np.int64)
    else:
        signs = b[:, 34:66].astype(np.int64)
        grid = IQ2S_GRID[idx]
        sc = b[:, 74:82].astype(np.int64)
    neg = (signs[:, :, None] >> np.arange(8)) & 1                               # [n][32][8]
    ls = 2 * ((sc[:, :, None] >> (4 * np.arange(2))) & 15).reshape(-1, 16) + 1
    return d, ls, np.where(neg == 1, -grid, grid).reshape(-1, 16, 16)


def dequant(t: int, blocks) -> np.ndarray:
    """gguf-py's order: db = d * (0.5 + s) * 0.25, value = db * grid * sign (fp32)"""
    d, ls, v = fields(t, blocks)
    s = ((ls - 1) // 2).astype(np.float32)
    db = ((d[:, None] * (np.float32(0.5) + s)) * np.float32(0.25)).astype(np.float32)
    return (db[:, :, None] * v.astype(np.float32)).astype(np.float32).reshape(-1)


def superblock_ints(t: int, w_blocks, q8) -> np.ndarray:
    """S = sum over the 16-value halves of ls_h * sum (+-grid) q8, the reference's bsum"""
    _, ls, v = fields(t, w_blocks)
    q = q8k_fields(q8)[1].reshape(-1, 16, 16)
    return (ls * (v * q).sum(axis=2)).sum(axis=1)


def superblock_terms(t: int, w_blocks, q8) -> np.ndarray:
    """the kernels' fp32 term per super-block: ((d / 8) dx) S"""
    d = (fields(t, w_blocks)[0] * np.float32(0.125)).astype(np.float32)
    dx = q8k_fields(q8)[0]
    return ((d * dx).astype(np.float32) * superblock_ints(t, w_blocks, q8).astype(np.float32)).astype(np.float32)


def vec_dot(t: int, w_blocks, q8) -> np.float32:
    """ggml_vec_dot_iq2_xs_q8_K / ggml_vec_dot_iq2_s_q8_K (scalar branch): fp32 sum of (d dx) S over super-blocks in order,
    times 0.125 once"""
    d, dx = fields(t, w_blocks)[0], q8k_fields(q8)[0]
    acc = np.float32(0)
    for v in ((d * dx).astype(np.float32) * superblock_ints(t, w_blocks, q8).astype(np.float32)).astype(np.float32):
        acc = np.float32(acc + v)
    return np.float32(acc * np.float32(0.125))
