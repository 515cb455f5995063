"""Test-only numpy restatement of the IQ1_M format and of the arithmetic the expert kernels implement for it.

block_iq1_m (include/ktb200.h), 56 B per 256 values: qs[32], qh[16] (one nibble per 8-value group: bits 0-2 the high bits of
the iq1s_grid index, bit 3 the sign of the group's delta), scales uint16[4] (a 3-bit scale per 16-value half, ls = 2s + 1; the
fp16 d in the four top nibbles).  `dequant` restates ggml's dequantiser in gguf-py's fp32 operation order; `superblock_ints`
gives the exact integer S = sum_h ls_h * sum (8 grid + delta) q8 = 8 sumi1 + sumi2 of ggml_vec_dot_iq1_m_q8_K's
(d dx) (sumi1 + 0.125 sumi2), and `vec_dot` its fp32 sum over super-blocks.
"""
from __future__ import annotations

import numpy as np

from iq_oracle import IQ1S_GRID, q8k_fields

IQ1_M = 29
BLOCK_BYTES = 56


def random_blocks(n_blocks: int, rng: np.random.Generator, d_scale: float = 1.0) -> np.ndarray:
    """random bytes (every bit pattern is a valid block) with a sane fp16 d (uniform in [0.75, 1.25) * d_scale) written into
    the four top nibbles of the scale words"""
    b = rng.integers(0, 256, size=(n_blocks, BLOCK_BYTES), dtype=np.uint8)
    d = ((rng.random(n_blocks) * 0.5 + 0.75) * d_scale).astype(np.float16).view(np.uint16)
    sc = b[:, 48:56].copy().view(np.uint16) & np.uint16(0x0FFF)
    for w in range(4):
        sc[:, w] |= ((d >> np.uint16(4 * w)) & np.uint16(0xF)) << np.uint16(12)
    b[:, 48:56] = sc.view(np.uint8)
    return b


def fields(blocks):
    """d [n] fp32, ls [n][16] (16-value halves), delta [n][32] (+-1 per 8-value group), grid [n][32][8] in {-1, 0, 1}"""
    b = np.asarray(blocks, np.uint8).reshape(-1, BLOCK_BYTES)
    sc = b[:, 48:56].copy().view(np.uint16).astype(np.int64)                  # [n][4]
    dbits = (sc[:, 0] >> 12) | ((sc[:, 1] >> 8) & 0xF0) | ((sc[:, 2] >> 4) & 0xF00) | (sc[:, 3] & 0xF000)
    d = dbits.astype(np.uint16).view(np.float16).astype(np.float32)
    ls = 2 * ((sc[:, :, None] >> (3 * np.arange(4))) & 7).reshape(-1, 16) + 1
    qh = b[:, 32:48].astype(np.int64)
    nib = ((qh[:, :, None] >> (4 * np.arange(2))) & 15).reshape(-1, 32)      # group l: byte l / 2, low nibble for even l
    idx = b[:, 0:32].astype(np.int64) | ((nib & 7) << 8)
    delta = np.where(nib & 8, -1, 1)
    return d, ls, delta, IQ1S_GRID[idx]


def dequant(blocks) -> np.ndarray:
    """dl = d * ls; value = dl * (grid + delta / 8) in fp32 (gguf-py's and ggml's order)"""
    d, ls, delta, grid = fields(blocks)
    dl = (d[:, None] * ls.astype(np.float32)).astype(np.float32)                               # [n][16]
    g = grid.astype(np.float32) + (delta * 0.125).astype(np.float32)[:, :, None]                # [n][32][8]
    return (dl.reshape(-1, 16, 1, 1) * g.reshape(-1, 16, 2, 8)).astype(np.float32).reshape(-1)


def _sums(w_blocks, q8):
    _, ls, delta, grid = fields(w_blocks)
    q = q8k_fields(q8)[1].reshape(-1, 32, 8)
    sg = (grid * q).sum(axis=2).reshape(-1, 16, 2).sum(axis=2)               # sum grid * q8 per half
    sd = (delta * q.sum(axis=2)).reshape(-1, 16, 2).sum(axis=2)              # sum delta * q8 per half
    return ls, sg, sd


def superblock_ints(w_blocks, q8) -> np.ndarray:
    """S = sum_h ls_h * sum (8 grid + delta) q8 per super-block"""
    ls, sg, sd = _sums(w_blocks, q8)
    return (ls * (8 * sg + sd)).sum(axis=1)


def superblock_terms(w_blocks, q8) -> np.ndarray:
    """each super-block's fp32 term as the reference forms it: (d dx) (sumi1 + 0.125 sumi2)"""
    d = fields(w_blocks)[0]
    dx = q8k_fields(q8)[0]
    ls, sg, sd = _sums(w_blocks, q8)
    sumi1, sumi2 = (ls * sg).sum(axis=1), (ls * sd).sum(axis=1)
    inner = (sumi1.astype(np.float32) + np.float32(0.125) * sumi2.astype(np.float32)).astype(np.float32)
    return ((d * dx).astype(np.float32) * inner).astype(np.float32)


def vec_dot(w_blocks, q8) -> np.float32:
    """ggml_vec_dot_iq1_m_q8_K (scalar branch): fp32 sum of the terms in order"""
    acc = np.float32(0)
    for v in superblock_terms(w_blocks, q8):
        acc = np.float32(acc + v)
    return acc
