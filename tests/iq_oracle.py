"""Test-only numpy restatement of the IQ1_S and IQ2_XXS formats and of the arithmetic the expert kernels implement.

Formats (include/ktb200.h): 256-value super-blocks whose 8-value groups index a codebook.  The codebooks come from
gguf-py (the same tables tests/golden/make_iq_tables.py writes into the CUDA header).  `dequant_*` restate ggml's
dequantisers in the same fp32 operation order; `superblock_ints` gives the exact integers of the reference's
`ggml_vec_dot_iq*_q8_K` and `vec_dot` its fp32 sum, so each can be checked against the other and against float64.
Activations are quantised to Q8_K by the C oracle's bit-exact quantiser (oracle/ktoracle.c).
"""
from __future__ import annotations

import numpy as np
from gguf import quants

IQ2_XXS, IQ1_S = 16, 19
BLOCK_BYTES = {IQ2_XXS: 66, IQ1_S: 50}
Q8K_BYTES = 292


def _grid(cls):
    cls.init_grid()
    return np.asarray(cls.grid).reshape(cls.grid_shape).astype(np.int64)


IQ1S_GRID = _grid(quants.IQ1_S)                                               # [2048][8] in {-1, 0, 1}
IQ2XXS_GRID = _grid(quants.IQ2_XXS)                                           # [256][8] in {8, 25, 43}
KSIGNS = np.frombuffer(quants.IQ2_XXS.ksigns, dtype=np.uint8).astype(np.int64)  # [128]


# ------------------------------------------------------------------------------------------------ random blocks
def random_blocks(t: int, n_blocks: int, rng: np.random.Generator, d_scale: float = 1.0) -> np.ndarray:
    """any bit pattern is a valid block: random bytes with a sane fp16 `d` (uniform in [0.75, 1.25) * d_scale)"""
    b = rng.integers(0, 256, size=(n_blocks, BLOCK_BYTES[t]), dtype=np.uint8)
    d = ((rng.random(n_blocks) * 0.5 + 0.75) * d_scale).astype(np.float16)
    b[:, 0:2] = d.view(np.uint8).reshape(n_blocks, 2)
    return b


def _fields_iq1s(blocks):
    b = np.asarray(blocks, np.uint8).reshape(-1, 50)
    d = b[:, 0:2].copy().view(np.float16).astype(np.float32).reshape(-1)
    qs = b[:, 2:34].astype(np.int64)                                          # [n][32]
    qh = b[:, 34:50].copy().view(np.uint16).astype(np.int64)                  # [n][8]
    ls = 2 * ((qh >> 12) & 7) + 1
    delta = np.where(qh & 0x8000, -1, 1)
    idx = qs.reshape(-1, 8, 4) | (((qh[:, :, None] >> (3 * np.arange(4))) & 7) << 8)   # [n][8 sub-blocks][4 groups]
    grid = IQ1S_GRID[idx]                                                     # [n][8][4][8]
    return d, ls, delta, grid


def _fields_iq2xxs(blocks):
    b = np.asarray(blocks, np.uint8).reshape(-1, 66)
    d = b[:, 0:2].copy().view(np.float16).astype(np.float32).reshape(-1)
    words = b[:, 2:66].copy().view(np.uint32).astype(np.int64).reshape(-1, 8, 2)
    idx = b[:, 2:66].reshape(-1, 8, 8)[:, :, 0:4].astype(np.int64)            # [n][8][4]
    aux1 = words[:, :, 1]
    ls = 2 * (aux1 >> 28) + 1
    signs = KSIGNS[(aux1[:, :, None] >> (7 * np.arange(4))) & 127]            # [n][8][4]
    sgn = np.where((signs[..., None] >> np.arange(8)) & 1, -1, 1)             # [n][8][4][8]
    grid = IQ2XXS_GRID[idx] * sgn
    return d, ls, grid


# ------------------------------------------------------------------------------------------------ dequantisation
def dequant_iq1_s(blocks) -> np.ndarray:
    """dl = d * ls; value = dl * (grid + delta), delta = +-0.125 (fp32, gguf-py's and ggml's order)"""
    d, ls, delta, grid = _fields_iq1s(blocks)
    dl = (d[:, None] * ls.astype(np.float32)).astype(np.float32)
    v = dl[:, :, None, None] * (grid.astype(np.float32) + (delta * 0.125).astype(np.float32)[:, :, None, None])
    return v.astype(np.float32).reshape(-1)


def dequant_iq2_xxs(blocks) -> np.ndarray:
    """db = d * (0.5 + s) * 0.25; value = db * grid * sign (fp32)"""
    d, ls, grid = _fields_iq2xxs(blocks)
    s = ((ls - 1) // 2).astype(np.float32)
    db = ((d[:, None] * (np.float32(0.5) + s)) * np.float32(0.25)).astype(np.float32)
    return (db[:, :, None, None] * grid.astype(np.float32)).astype(np.float32).reshape(-1)


def dequant(t: int, blocks) -> np.ndarray:
    return dequant_iq1_s(blocks) if t == IQ1_S else dequant_iq2_xxs(blocks)


# ------------------------------------------------------------------------------------------------ Q8_K activations
def q8k_fields(q8):
    """block_q8_K {float d; int8 qs[256]; int16 bsums[16]} -> d [n], qs [n][256], bsums [n][16]"""
    b = np.asarray(q8, np.uint8).reshape(-1, Q8K_BYTES)
    d = b[:, 0:4].copy().view(np.float32).reshape(-1)
    qs = b[:, 4:260].copy().view(np.int8).astype(np.int64)
    bs = b[:, 260:292].copy().view(np.int16).astype(np.int64)
    return d, qs, bs


def q8k_to_f64(q8) -> np.ndarray:
    d, qs, _ = q8k_fields(q8)
    return (d.astype(np.float64)[:, None] * qs).reshape(-1)


# ------------------------------------------------------------------------------------------------ dot products
def superblock_ints(t: int, w_blocks, q8) -> np.ndarray:
    """the exact per-super-block integer of the reference's vec_dot: IQ1_S  S = sum ls * sum (8 grid + delta) q8
    (= 8 sumi + sumi1), IQ2_XXS  bsum = sum ls * sum (+-grid) q8"""
    _, qs, bs = q8k_fields(q8)
    q = qs.reshape(-1, 8, 4, 8)
    if t == IQ1_S:
        _, ls, delta, grid = _fields_iq1s(w_blocks)
        sumi = (grid * q).sum(axis=(2, 3))                                   # [n][8]
        b32 = bs.reshape(-1, 8, 2).sum(axis=2)                                # bsums[2ib] + bsums[2ib+1]
        return (ls * (8 * sumi + delta * b32)).sum(axis=1)
    _, ls, grid = _fields_iq2xxs(w_blocks)
    return (ls * (grid * q).sum(axis=(2, 3))).sum(axis=1)


def superblock_terms(t: int, w_blocks, q8) -> np.ndarray:
    """each super-block's fp32 term as the reference forms it"""
    dx = q8k_fields(q8)[0]
    dw = np.asarray(w_blocks, np.uint8).reshape(-1, BLOCK_BYTES[t])[:, 0:2].copy().view(np.float16).astype(np.float32).reshape(-1)
    d = (dw * dx).astype(np.float32)
    if t == IQ1_S:
        _, ls, delta, grid = _fields_iq1s(w_blocks)
        _, qs, bs = q8k_fields(q8)
        sumi = (ls * (grid * qs.reshape(-1, 8, 4, 8)).sum(axis=(2, 3))).sum(axis=1)
        sumi1 = (ls * delta * bs.reshape(-1, 8, 2).sum(axis=2)).sum(axis=1)
        inner = (sumi.astype(np.float32) + np.float32(0.125) * sumi1.astype(np.float32)).astype(np.float32)
        return (d * inner).astype(np.float32)
    return (d * superblock_ints(t, w_blocks, q8).astype(np.float32)).astype(np.float32)


def vec_dot(t: int, w_blocks, q8) -> np.float32:
    """ggml_vec_dot_iq1_s_q8_K / ggml_vec_dot_iq2_xxs_q8_K (scalar branch): fp32 sum over super-blocks in order;
    IQ2_XXS scales the total by 0.125 once"""
    acc = np.float32(0)
    for v in superblock_terms(t, w_blocks, q8):
        acc = np.float32(acc + v)
    return np.float32(acc * np.float32(0.125)) if t == IQ2_XXS else acc


# ------------------------------------------------------------------------------------------------ routed experts
def silu(x):
    return x / (1.0 + np.exp(-x))


def moe_forward(oracle, x_f32: np.ndarray, ids: np.ndarray, w: np.ndarray, expert, E: int, use_silu: bool = True) -> np.ndarray:
    """float64 routed experts over Q8_K activations: x and the fp32 intermediate are quantised by the C oracle's Q8_K
    quantiser, weights are dequantised exactly (expert(e) -> float64 gate [I][H], up [I][H], down [H][I]), all sums are
    float64.  Ids outside [0, E) are skipped.  Returns float64 [T][H]."""
    T, k = ids.shape
    H = x_f32.shape[1]
    out = np.zeros((T, H), np.float64)
    xq = [q8k_to_f64(oracle.from_float(x_f32[t].astype(np.float32), 15)) for t in range(T)]
    # expert by expert, so that one expert's float64 weights are resident at a time (352 MB at V3 shapes)
    for e in sorted({int(v) for v in ids.reshape(-1) if 0 <= int(v) < E}):
        g, u, dn = expert(e)
        for t, j in zip(*np.nonzero(ids == e)):
            gv, uv = g @ xq[t], u @ xq[t]
            a = (silu(gv) if use_silu else np.maximum(gv, 0.0)) * uv
            aq = q8k_to_f64(oracle.from_float(a.astype(np.float32), 15))
            out[t] += float(w[t, j]) * (dn @ aq)
        del g, u, dn
    return out
