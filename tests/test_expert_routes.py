"""Routed experts (ktb200_moe_forward / _forward_shared) on every kernel route the launchers pick under default settings, at
model shapes and prompt-sized batches, against the float64 oracle.

The routed experts go through the launchers of tests/test_linear_routes.py (csrc/moe.cu: launch_rows<true>, launch_reduce),
with expert ids, k slots and the fused shared-expert slot.  A handle takes the grouped tensor-core GEMM (grouped.cu) from
grouped_min_qlen tokens when grouped_ok accepts it; every other handle -- any IQ4_XS tensor, Q6_K gate/up, Q6_K down outside
the tile layout, k > 32, E > 1023 -- runs the per-pair kernels for whole prompt chunks (KExpertsB200.MAX_TOKENS = 1024).

  1. Route table: `expert_route` restates the choice of ktb200_moe_forward: grouped or per pair, the load-time Q6_K layout,
     the launch_rows<true> and launch_reduce cascades, when the shared expert rides in the routed launches, and
     reduce_kernel's shared-memory plan at T.  The shared-memory planners are restated only where they decide a route.  The
     case lists reach every reachable route on both sides of each switch; the GPU census holds every launch to its row.
  2. References: _moe_ref (tests/test_iq_grouped.py, float64 over the oracle's Q8_K activations) on oracle_rows of each call
     (tokens are independent), held to _check's bound (tests/test_iq_experts.py) and each token to ROW_TOL of its own largest
     output; the fused shared expert is one more expert of weight 1 in the reference.
  3. Where the T-token call and a 1-token call run the same kernels, every checked row of the T-token call is bit-identical to
     that token run alone: no per-pair kernel's fp32 order depends on T (gx and the token chunks split rows, tokens and
     (token, slot) pairs between CTAs and warps, never one dot product or one row's sum over the slots).

Worst measured errors print with `pytest -s`; DESIGN §4.2 keeps the route table and the values measured on an H100.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from ktransformers_b200 import native
from oracle.bindings import f32_to_bf16_bits
from test_iq_experts import FP_TOL, ROUND_REL, _check, _Experts, _ids, _to_f64, _x
from test_iq_grouped import _moe_ref
from test_linear_routes import _bulk_down_warps, _rows_kernel, mlp_routes, oracle_rows, tokens

Q2K, Q3K, Q4K, Q5K, Q6K = native.GGML_Q2_K, native.GGML_Q3_K, native.GGML_Q4_K, native.GGML_Q5_K, native.GGML_Q6_K
IQ4, IQ1 = native.GGML_IQ4_XS, native.GGML_IQ1_S
F32, BF16 = native.GGML_F32, native.GGML_BF16
QK = 256
H100_SMS = 132
HERE = os.path.dirname(os.path.abspath(__file__))

# ------------------------------------------------------------------------------------------------ constants of the headers
SMEM_CAP = 232448 - 512          # kSmemCap (moe.cu)
ACT_BLK_STRIDE = QK + 16         # kActBlkStride (bulk_ring.cuh)
BULK_MAX_WARPS = 18              # kBulkMaxWarps (gemv_bulk.cuh): rows_bulk_q4k_kernel
BULK_MAX_WARPS_DOWN = 16         # kBulkMaxWarpsDown (gemv_bulk.cuh): reduce_bulk_kernel
IQ_MAX_WARPS = 16                # kIqMaxWarps (iq.cuh): rows_bulk_iq_kernel
GATE_UP_SPARE = 48               # kGateUpSpare (moe.cu)
GEMV_CTAS_PER_SM = 2             # kGemvCtasPerSm (gemv.cuh): rows_kernel / reduce_kernel grids
PIPE_SMEM = 220 * 1024           # launch_rows_pipe, launch_reduce_pipe_q6k8, launch_reduce_fmt
Q6K4T_PLAN_SLOTS = 3             # kQ6K4TPlanSlots (moe.cu)
GROUPED_TILE = 128               # kGM (grouped.cu)
BLOCK_BYTES = {Q2K: 84, Q3K: 110, Q4K: 144, Q5K: 176, Q6K: 210, IQ4: 136, IQ1: 50}
BLOCKS_PER_STEP = {"FmtQ4K": 4, "FmtQ5K": 4, "FmtQ6K8": 8, "FmtGenK": 2}   # Fmt::kBlocksPerStep (formats.cuh)
# bulk-copy formats: name, kBs, kTableBytes, kSharedSlot, kNblkMultiple (gemv_bulk.cuh, iq.cuh)
BULK = {Q2K: ("BulkQ2K", 16, 0, True, 4), Q3K: ("BulkQ3K", 8, 0, True, 4), IQ1: ("BulkIQ1S", 8, 2048 * 8, False, 4)}
GROUPED_TYPES = {Q4K, Q5K, Q3K, Q2K, IQ1}                # grouped_fmt >= 0 on the raw layout (Q6_K: down tiles only)
CODEBOOK_IQ = {IQ1}                                      # is_iquant: the grouped threshold is 80 (IQ4_XS is a K-quant here)
TYPE_NAME = {Q2K: "Q2_K", Q3K: "Q3_K", Q4K: "Q4_K", Q5K: "Q5_K", Q6K: "Q6_K", IQ4: "IQ4_XS", IQ1: "IQ1_S"}


# ------------------------------------------------------------------------------------------------ restated planners
def _ring_warps(unit, slot_bytes, slots, max_warps, table=0):
    """plan_ring at its smallest chunk (one unit): the warps that fit.  A larger chunk is taken only while room_warps still
    fit, so the plan launches exactly when this is >= min_warps."""
    cap = SMEM_CAP - table
    h = (unit + 15) & ~15
    return 0 if h + 16 >= cap else min((cap - h - 16) // (slots * (slot_bytes + 8)), max_warps)


def _down_warps(rows, nb, act_pair, item, slots, ns, sms, table=0):
    """plan_down at pcap = ns (the chunk it falls back to): warps of reduce_bulk_kernel, 0 when the item shape is refused"""
    if rows % 4 or ns > 200 or item % 16:
        return 0
    quads = rows // 4
    nrows_max = -(-quads // max(1, min(sms, quads))) * 4
    return _ring_warps(ns * (act_pair + nrows_max * 4 + 4), item, slots, BULK_MAX_WARPS_DOWN, table)


def _pipe_warps(H, block_bytes):
    """launch_rows_pipe<Fmt, true>: 12 or 8 warps of 2 slots of a (gate | up) row pair, 0 when it declines"""
    nblk = H // QK
    slot = 2 * nblk * block_bytes
    act = (H + ((nblk * 4 + 15) & ~15) + H // 8 + 15) & ~15
    if slot < 4096:
        return 0
    return next((w for w in (12, 8) if act + w * 2 * slot <= PIPE_SMEM), 0)


def q6k4t_eligible(H, I, ns_max, sms):
    """load time: a Q6_K down tensor takes the 4-row tile layout (and then only reduce_bulk_kernel<BulkQ6K4T>)"""
    nb = I // QK
    return nb % 2 == 0 and H % 4 == 0 and _down_warps(H, nb, nb * (ACT_BLK_STRIDE + 32 + 4), 4 * nb * 210, Q6K4T_PLAN_SLOTS,
                                                      ns_max, sms) >= 4


def down_layout(dt, H, I, ns_max, sms, mlp=False):
    """ktb200_moe_load_weights (ns_max = k + 1) / ktb200_mlp_load_weights (ns_max = 17)"""
    if dt != Q6K:
        return "raw"
    if q6k4t_eligible(H, I, ns_max, sms):
        return "t4"
    if H % 8 == 0 and (not mlp or 8 * 210 * (I // QK) <= 200 * 1024):
        return "soa8"
    return "raw"


def reduce_plan(H, I, ns, T, sms, fixed=True):
    """launch_reduce_fmt: (gx, shared bytes), None when it refuses the call.  fixed=False: the plan before gx was raised to
    fit, which refused any call whose row share did not fit at gx = ceil(2 SMs / T)"""
    per_slot = I + I // QK * 4 + I // 8
    gx = max(1, min(-(-GEMV_CTAS_PER_SM * sms // T), H))
    rows_fit = (PIPE_SMEM - per_slot * ns) // (ns * 4) - 1 if per_slot * ns < PIPE_SMEM else 0
    if fixed:
        if rows_fit < 1:
            return None
        gx = max(gx, -(-H // rows_fit))
    smem = per_slot * ns + (-(-H // gx) + 1) * ns * 4
    return (gx, smem) if smem <= PIPE_SMEM else None


def q6k8_pipe_fits(H, I, ns, T, sms):
    """launch_reduce_pipe_q6k8 on a Q6_K down tensor in the 8-row SoA layout"""
    nb = I // QK
    if H % 4 or nb % 2 or 840 * nb < 4096:
        return False
    quads = H // 4
    gx = max(1, min(-(-sms // T), quads))
    nrows_max = (-(-quads // gx) + 1) * 4
    return ns * I + ns * nb * 4 + ns * (I // 16) * 2 + nrows_max * ns * 4 + 16 + 24 * 840 * nb <= PIPE_SMEM


def _fmt(t, soa):
    return {Q4K: "FmtQ4K", Q5K: "FmtQ5K"}.get(t, "FmtQ6K8" if t == Q6K and soa else "FmtGenK")


def gate_up_route(gt, ut, H, I, k, fused, sms):
    """launch_rows<true>: the IQ / Q2_K / Q3_K bulk kernel, the Q4_K bulk kernel, the Q5_K pipe, the Q4K32 pipe, rows_kernel"""
    nblk = H // QK
    soa = gt == ut == Q6K and I % 8 == 0
    f = _fmt(gt, soa) if _fmt(gt, soa) == _fmt(ut, soa) else "FmtGenK"   # mixed gate/up types: the generic kernels
    nslots = k + fused
    if f == "FmtGenK" and gt == ut and gt in BULK:
        name, bs, table, shared_slot, mult = BULK[gt]
        if nblk % mult == 0 and I % 2 == 0 and k <= 200 and (shared_slot or not fused):
            act_tok = (nblk * (ACT_BLK_STRIDE + 2 * bs + 4) + 15) & ~15
            if _ring_warps(act_tok + nslots * 4, 4 * nblk * BLOCK_BYTES[gt], 2, IQ_MAX_WARPS, table) >= 4:
                return f"rows_bulk_iq_kernel<ktb::{name},"
    if f == "FmtQ4K" and nblk >= 16 and nslots <= 200:
        act_tok = (nblk * ACT_BLK_STRIDE + nblk * 16 + nblk * 4 + 15) & ~15
        if _ring_warps(act_tok + nslots * 4, nblk * 144, 3, BULK_MAX_WARPS) >= 4:
            return "rows_bulk_q4k_kernel<true,"
    if f == "FmtQ5K" and _pipe_warps(H, 176):
        return "rows_pipe_kernel<ktb::FmtQ5K,true,"
    if f == "FmtQ4K" and _pipe_warps(H, 144):
        return "rows_pipe_kernel<ktb::FmtQ4K32,true,"
    return _rows_kernel(f, True, nblk)


def down_route(dt, H, I, k, T, fused, layout, sms, fixed=True):
    """launch_reduce: the tile layout, BulkQ4K, the IQ / Q2_K / Q3_K bulk kernel, the Q6K8 pipe, reduce_kernel<Fmt, NB>
    (None: the call is refused)"""
    nb, ns = I // QK, k + fused
    if layout == "t4":
        return "reduce_bulk_kernel<ktb::BulkQ6K4T,"
    if dt == Q4K and _down_warps(H, nb, nb * (ACT_BLK_STRIDE + 16 + 4), 4 * nb * 144, 2, ns, sms) >= 2:
        return "reduce_bulk_kernel<ktb::BulkQ4K,"
    if dt in BULK and (BULK[dt][3] or not fused):
        name, bs, table = BULK[dt][:3]
        if _down_warps(H, nb, nb * (ACT_BLK_STRIDE + 2 * bs + 4), 4 * nb * BLOCK_BYTES[dt], 2, ns, sms, table) >= 2:
            return f"reduce_bulk_kernel<ktb::{name},"
    f = {Q4K: "FmtQ4K", Q5K: "FmtQ5K"}.get(dt, "FmtQ6K8" if layout == "soa8" else "FmtGenK")
    if f == "FmtQ6K8" and q6k8_pipe_fits(H, I, ns, T, sms):
        return "reduce_pipe_q6k8_kernel<"
    if reduce_plan(H, I, ns, T, sms, fixed) is None:
        return None
    nsteps = -(-nb // BLOCKS_PER_STEP[f])
    return f"reduce_kernel<ktb::{f},{(2 if f == 'FmtQ4K' else 1) if nsteps >= 2 else 1}>"


def grouped_min_qlen(types):
    return 80 if any(t in CODEBOOK_IQ for t in types) else 48


def grouped_ok(types, layout, H, I, E, k):
    gt, ut, dt = types
    return (gt in GROUPED_TYPES and ut in GROUPED_TYPES and (dt in GROUPED_TYPES or layout == "t4") and H % GROUPED_TILE == 0
            and I % GROUPED_TILE == 0 and E <= 1023 and k <= 32)


def fuses(types, H, I, kmax, sms):
    """the shared expert (an MLP of the routed types and shape) rides in the routed launches when its down layout is the
    routed one (gate/up SoA follows the same rule on both)"""
    return down_layout(types[2], H, I, kmax + 1, sms) == down_layout(types[2], H, I, 17, sms, mlp=True)


def expert_route(types, H, I, k, T, shared=False, sms=H100_SMS, E=16, fixed=True, kmax=None):
    """kernel name prefixes ktb200_moe_forward(_shared) launches for k slots per token, in order, on a handle of
    routed_expert_num = kmax (default k; the load-time Q6_K layout is planned for kmax + 1 slots); "grouped" stands for one
    1024-token chunk of the grouped GEMM (10 launches); None when the call is refused"""
    gt, ut, dt = types
    kmax = kmax or k
    layout = down_layout(dt, H, I, kmax + 1, sms)
    mlp = tuple(mlp_routes(gt, ut, dt, H, I, sms)) if shared and not fuses(types, H, I, kmax, sms) else ()
    if T >= grouped_min_qlen(types) and grouped_ok(types, layout, H, I, E, k):
        return ("grouped",) * -(-T // 1024) + (tuple(mlp_routes(gt, ut, dt, H, I, sms)) if shared else ())
    fused = bool(shared and not mlp)
    dn = down_route(dt, H, I, k, T, fused, layout, sms, fixed)
    return None if dn is None else (gate_up_route(gt, ut, H, I, k, fused, sms), dn) + mlp


def gx_steps(sms, n=4):
    """token counts on both sides of reduce_kernel's first n grid steps: gx = ceil(2 SMs / T) falls to g at T = ceil(2 SMs / g)"""
    return sorted({t for g in range(1, n + 1) for t in (-(-GEMV_CTAS_PER_SM * sms // g) - 1, -(-GEMV_CTAS_PER_SM * sms // g))})


# ------------------------------------------------------------------------------------------------ cases
SHAPES = {"v3": (7168, 2048, 8), "qwen3-235b": (4096, 1536, 8), "qwen3-30b": (2048, 768, 8), "v2": (5120, 1536, 6)}
FILES = {"q4_k_m": (Q4K, Q4K, Q6K), "q4_k_m-q4k_down": (Q4K, Q4K, Q4K), "q5_k_m": (Q5K, Q5K, Q6K), "q6_k": (Q6K, Q6K, Q6K),
         "iq4_xs": (IQ4, IQ4, IQ4), "q3_k_m": (Q3K, Q3K, Q4K)}
TS = tuple(sorted({1, 8, 9, 47, 48, 79, 80, 1024, *gx_steps(H100_SMS)}))
CASES = {
    # name: (types, H, I, k, shared expert).  Every file at every model shape, then route edges.
    **{f"{f}-{s}": (t, *SHAPES[s], False) for f, t in FILES.items() for s in SHAPES},
    **{f"{f}-v3-shared": (t, *SHAPES["v3"], True) for f, t in FILES.items()},
    "q5_k_m-qwen3-30b-shared": ((Q5K, Q5K, Q6K), 2048, 768, 8, True),
    "mixed-q4k_q5k_q4k-v3": ((Q4K, Q5K, Q4K), 7168, 2048, 8, False),
    "mixed-q4k_q5k_q4k-v3-shared": ((Q4K, Q5K, Q4K), 7168, 2048, 8, True),
    "q4k-pipe-3840x1536": ((Q4K, Q4K, Q4K), 3840, 1536, 8, False),
    "q5k_x3-qwen3-30b": ((Q5K, Q5K, Q5K), 2048, 768, 8, False),
    "q4k-down-nb50-2048x12800": ((Q4K, Q4K, Q4K), 2048, 12800, 8, False),
    "q2k_q2k_q3k-v3": ((Q2K, Q2K, Q3K), 7168, 2048, 8, False),
    "iq1_s-v3": ((IQ1, IQ1, IQ1), 7168, 2048, 8, False),
    "q6k-pipe-1024x1536-k40-of-100": ((Q4K, Q4K, Q6K), 1024, 1536, 40, False),
}
# routed_expert_num of a case's handle where it exceeds the call's k: the Q6_K down layout is planned for 101 slots (8-row
# SoA), and a 40-slot call then fits reduce_pipe_q6k8_kernel
KMAX = {"q6k-pipe-1024x1536-k40-of-100": 100}
# the pipe kernel's plan holds up to the token count where its row share stops fitting: both sides of it as well
_PIPE_LAST = max(T for T in range(1, 1025) if q6k8_pipe_fits(1024, 1536, 40, T, H100_SMS))
CASE_TS = {name: tuple(sorted(set(TS) | ({_PIPE_LAST, _PIPE_LAST + 1} if name in KMAX else set()))) for name in CASES}


def case_route(name, T, **kw):
    types, H, I, k, sh = CASES[name]
    return expert_route(types, H, I, k, T, sh, kmax=KMAX.get(name), **kw)


CENSUS_TS = {name: (1, 9, 47, 48, 264) if name.startswith(("q2k", "iq1", "q3_k_m")) else CASE_TS[name] for name in CASES}

# the routes the case lists must reach (DESIGN §4.2)
GATE_UP_ROUTES = ("rows_bulk_q4k_kernel<true,", "rows_pipe_kernel<ktb::FmtQ5K,true,", "rows_pipe_kernel<ktb::FmtQ4K32,true,",
                  "rows_kernel<ktb::FmtQ4K,true,", "rows_kernel<ktb::FmtQ5K,true,", "rows_kernel<ktb::FmtQ6K8,true,",
                  "rows_kernel<ktb::FmtGenK,true,", "rows_bulk_iq_kernel<ktb::BulkQ2K,", "rows_bulk_iq_kernel<ktb::BulkQ3K,",
                  "rows_bulk_iq_kernel<ktb::BulkIQ1S,")
DOWN_ROUTES = ("reduce_bulk_kernel<ktb::BulkQ6K4T,", "reduce_bulk_kernel<ktb::BulkQ4K,", "reduce_bulk_kernel<ktb::BulkQ3K,",
               "reduce_bulk_kernel<ktb::BulkIQ1S,", "reduce_kernel<ktb::FmtQ4K,2>", "reduce_kernel<ktb::FmtQ5K,1>",
               "reduce_kernel<ktb::FmtQ6K8,1>", "reduce_kernel<ktb::FmtGenK,1>", "reduce_pipe_q6k8_kernel<")

# real files at real shapes: (gate/up, down) at 1 token, at 9 tokens, and at 264 tokens (None: the grouped GEMM)
PINNED = {
    "q4_k_m-v3": ("rows_bulk_q4k_kernel<true,", "reduce_bulk_kernel<ktb::BulkQ6K4T,", None),
    "q4_k_m-qwen3-235b": ("rows_bulk_q4k_kernel<true,", "reduce_bulk_kernel<ktb::BulkQ6K4T,", None),
    "q4_k_m-qwen3-30b": ("rows_kernel<ktb::FmtQ4K,true,2,", "reduce_kernel<ktb::FmtQ6K8,1>", "per pair"),
    "q4_k_m-v2": ("rows_bulk_q4k_kernel<true,", "reduce_bulk_kernel<ktb::BulkQ6K4T,", None),
    "q4_k_m-q4k_down-v3": ("rows_bulk_q4k_kernel<true,", "reduce_bulk_kernel<ktb::BulkQ4K,", None),
    "q4_k_m-q4k_down-qwen3-235b": ("rows_bulk_q4k_kernel<true,", "reduce_bulk_kernel<ktb::BulkQ4K,", None),
    "q4_k_m-q4k_down-qwen3-30b": ("rows_kernel<ktb::FmtQ4K,true,2,", "reduce_bulk_kernel<ktb::BulkQ4K,", None),
    "q4_k_m-q4k_down-v2": ("rows_bulk_q4k_kernel<true,", "reduce_bulk_kernel<ktb::BulkQ4K,", None),
    "q5_k_m-v3": ("rows_pipe_kernel<ktb::FmtQ5K,true,", "reduce_bulk_kernel<ktb::BulkQ6K4T,", None),
    "q5_k_m-qwen3-235b": ("rows_pipe_kernel<ktb::FmtQ5K,true,", "reduce_bulk_kernel<ktb::BulkQ6K4T,", None),
    "q5_k_m-qwen3-30b": ("rows_kernel<ktb::FmtQ5K,true,2,", "reduce_kernel<ktb::FmtQ6K8,1>", "per pair"),
    "q5_k_m-v2": ("rows_pipe_kernel<ktb::FmtQ5K,true,", "reduce_bulk_kernel<ktb::BulkQ6K4T,", None),
    "q6_k-v3": ("rows_kernel<ktb::FmtQ6K8,true,1,", "reduce_bulk_kernel<ktb::BulkQ6K4T,", "per pair"),
    "q6_k-qwen3-235b": ("rows_kernel<ktb::FmtQ6K8,true,2,", "reduce_bulk_kernel<ktb::BulkQ6K4T,", "per pair"),
    "q6_k-qwen3-30b": ("rows_kernel<ktb::FmtQ6K8,true,4,", "reduce_kernel<ktb::FmtQ6K8,1>", "per pair"),
    "q6_k-v2": ("rows_kernel<ktb::FmtQ6K8,true,2,", "reduce_bulk_kernel<ktb::BulkQ6K4T,", "per pair"),
    "iq4_xs-v3": ("rows_kernel<ktb::FmtGenK,true,1,", "reduce_kernel<ktb::FmtGenK,1>", "per pair"),
    "iq4_xs-qwen3-235b": ("rows_kernel<ktb::FmtGenK,true,1,", "reduce_kernel<ktb::FmtGenK,1>", "per pair"),
    "iq4_xs-qwen3-30b": ("rows_kernel<ktb::FmtGenK,true,1,", "reduce_kernel<ktb::FmtGenK,1>", "per pair"),
    "iq4_xs-v2": ("rows_kernel<ktb::FmtGenK,true,1,", "reduce_kernel<ktb::FmtGenK,1>", "per pair"),
    "q3_k_m-v3": ("rows_bulk_iq_kernel<ktb::BulkQ3K,", "reduce_bulk_kernel<ktb::BulkQ4K,", None),
    "q3_k_m-qwen3-235b": ("rows_bulk_iq_kernel<ktb::BulkQ3K,", "reduce_bulk_kernel<ktb::BulkQ4K,", None),
    "q3_k_m-qwen3-30b": ("rows_bulk_iq_kernel<ktb::BulkQ3K,", "reduce_bulk_kernel<ktb::BulkQ4K,", None),
    "q3_k_m-v2": ("rows_bulk_iq_kernel<ktb::BulkQ3K,", "reduce_bulk_kernel<ktb::BulkQ4K,", None),
}


# ------------------------------------------------------------------------------------------------ CPU
def _routes():
    return {(name, T): case_route(name, T) for name in CASES for T in CASE_TS[name]}


def test_route_table_covers_every_route():
    per_pair = [r for r in _routes().values() if r and r[0] != "grouped"]
    for want in GATE_UP_ROUTES:
        assert any(r[0].startswith(want) for r in per_pair), want
    for want in DOWN_ROUTES:
        assert any(r[1].startswith(want) for r in per_pair), want
    assert any(r and r[0] == "grouped" for r in _routes().values())
    assert all(r is not None for r in _routes().values()), "a case the launcher refuses"
    # the fused shared slot on every kernel that has one, and the separate MLP launches where the layouts differ
    fused = {r[0].split("<")[0] + "/" + r[1].split("<")[0] for (n, _), r in _routes().items()
             if CASES[n][4] and r and r[0] != "grouped" and len(r) == 2}
    assert {"rows_bulk_q4k_kernel/reduce_bulk_kernel", "rows_kernel/reduce_kernel", "rows_pipe_kernel/reduce_bulk_kernel"} <= fused, fused


def test_token_counts_straddle_every_switch():
    assert {263, 264, 131, 132}.issubset(TS) and {1, 8, 9, 47, 48, 79, 80, 1024}.issubset(TS)
    for name, (types, H, I, k, sh) in CASES.items():
        ts = CASE_TS[name]
        rs = [case_route(name, T) for T in ts]
        for a, b, ra, rb in zip(ts, ts[1:], rs, rs[1:]):
            assert ra == rb or b == a + 1, f"{name}: the route changes between {a} and {b} tokens"
    # reduce_kernel's grid: gx = ceil(2 SMs / T) takes a new value between each straddling pair
    steps = gx_steps(H100_SMS)
    for a, b in zip(steps[::2], steps[1::2]):
        assert b == a + 1 and reduce_plan(7168, 2048, 8, a, H100_SMS, False) != reduce_plan(7168, 2048, 8, b, H100_SMS, False)


def test_pinned_files():
    for name, (gu, dn, big) in PINNED.items():
        types, H, I, k, _ = CASES[name]
        for T in (1, 9):
            assert expert_route(types, H, I, k, T) == (gu, dn), (name, T)
        r = expert_route(types, H, I, k, 264)
        assert (r[0] == "grouped") == (big is None), (name, r)
        if big is not None:
            assert r == (gu, dn), (name, r)
    # the shared expert rides along at V3 for every file: its 17-slot tile plan and the 9-slot routed plan agree
    for f in FILES:
        assert len(expert_route(FILES[f], 7168, 2048, 8, 9, True)) == 2, f


def test_reduce_plan_keeps_every_launch_that_fit():
    """the restated plan: the raised gx differs from the old one only where the old plan refused the call; where it did not
    fit, IQ4_XS at V3 refused every call of >= 264 tokens (248,096 B of shared memory at gx = 1) and every such call now
    launches.  This checks the restatement against itself; the launcher's own plan is checked on the GPU, by the sweep's
    IQ4_XS calls of 263, 264 and 1024 tokens and the KTMoEWrapper chunk of 1024 tokens."""
    for H, I, _ in SHAPES.values():
        for ns in (1, 6, 7, 8, 9, 16, 33, 41):
            for T in list(range(1, 300)) + [511, 512, 1024, 4096]:
                old, new = reduce_plan(H, I, ns, T, H100_SMS, fixed=False), reduce_plan(H, I, ns, T, H100_SMS)
                if old is not None:
                    assert new == old, (H, I, ns, T)
                else:
                    assert new is not None and new[1] <= PIPE_SMEM, (H, I, ns, T)
    assert reduce_plan(7168, 2048, 8, 264, H100_SMS, fixed=False) is None
    assert reduce_plan(7168, 2048, 8, 263, H100_SMS, fixed=False) == (2, 133408)
    assert reduce_plan(7168, 2048, 8, 264, H100_SMS) == (2, 133408)
    assert reduce_plan(7168, 2048, 9, 1024, H100_SMS) == (2, 21024 + 3585 * 36)
    for name in CASES:
        for T in CASE_TS[name]:
            if case_route(name, T) != case_route(name, T, fixed=False):
                assert case_route(name, T, fixed=False) is None and T >= 264, (name, T)
    # 96 slots of 2048 columns leave room for one row per CTA; 97 do not
    assert reduce_plan(7168, 2048, 96, 1, H100_SMS) == (7168, 96 * 2336 + 2 * 96 * 4)
    assert reduce_plan(7168, 2048, 97, 1, H100_SMS) is None


def test_down_planner_is_test_linear_routes_one():
    """_down_warps at pcap = ns is _bulk_down_warps of tests/test_linear_routes.py for the formats without tables"""
    for H, I, k in SHAPES.values():
        nb = I // QK
        for ns in (k, k + 1, 17):
            assert _down_warps(H, nb, nb * 308, 4 * nb * 210, 3, ns, H100_SMS) == _bulk_down_warps(H, I, 210, 16, 3, ns, H100_SMS)
            assert _down_warps(H, nb, nb * 292, 4 * nb * 144, 2, ns, H100_SMS) == _bulk_down_warps(H, I, 144, 8, 2, ns, H100_SMS)


def test_rarely_reached_routes():
    """reduce_pipe_q6k8_kernel: wherever its 24 ring slots and the staging of k slots fit (nb 6, 8 or 10, at the smallest
    row share, T = 1), a handle of routed_expert_num = k laid its Q6_K down tensor out in 4-row tiles at load time (planned
    for k + 1 slots), so calls with k == routed_expert_num -- every caller in this project -- never reach it.  A call with
    fewer slots than the handle's routed_expert_num can: the layout is planned for routed_expert_num + 1 slots
    (q6k-pipe-1024x1536-k40-of-100 in the case list).  reduce_kernel<FmtQ4K, 1> (one step per row: nb <= 4): the BulkQ4K
    plan fits every such shape up to 128 slots per token (H <= 16384); only calls of more slots at I = 1024 reach it, far
    beyond any model's top-k, and no case forces it."""
    for H in range(256, 16384 + 1, 256):
        for nb in (6, 8, 10):
            for k in range(1, 201):
                if q6k8_pipe_fits(H, nb * QK, k, 1, H100_SMS):
                    assert down_layout(Q6K, H, nb * QK, k + 1, H100_SMS) == "t4", (H, nb, k)
        for nb in range(1, 5):
            for ns in range(1, 129):
                assert _down_warps(H, nb, nb * 292, 4 * nb * 144, 2, ns, H100_SMS) >= 2, (H, nb, ns)
    assert down_layout(Q6K, 1024, 1536, 101, H100_SMS) == "soa8" and q6k8_pipe_fits(1024, 1536, 40, 1, H100_SMS)
    assert down_route(Q4K, 7168, 1024, 160, 1, False, "raw", H100_SMS) == "reduce_kernel<ktb::FmtQ4K,1>"


def test_k_over_32_is_per_pair():
    assert expert_route((Q5K, Q5K, Q5K), 2048, 512, 40, 264) == ("rows_kernel<ktb::FmtQ5K,true,2,", "reduce_kernel<ktb::FmtQ5K,1>")
    for T in (1, 3, 9):
        assert case_route("q6k-pipe-1024x1536-k40-of-100", T)[1] == "reduce_pipe_q6k8_kernel<", T
    assert case_route("q6k-pipe-1024x1536-k40-of-100", 264)[1] == "reduce_kernel<ktb::FmtQ6K8,1>"


# ------------------------------------------------------------------------------------------------ GPU helpers
def _stream():
    return torch.cuda.current_stream().cuda_stream


class _SharedMlp:
    """a shared expert (ktb200_mlp) of the routed types on its own weights, for prompt chunks up to max_tokens"""

    def __init__(self, types, H, I, hidden_type, seed, max_tokens=1024):
        from ktransformers_b200.util.synth import synth_blocks
        self.types, self.H, self.I = types, H, I
        self.w = [synth_blocks(t, r * c, "cuda", seed + i) for i, (t, r, c) in enumerate(zip(types, (I, I, H), (H, H, I)))]
        self.host = [b.cpu().numpy() for b in self.w]
        self.lib, self.h = native.lib(), C.c_void_p()
        native.check(self.lib.ktb200_mlp_create(H, I, *(t.data_ptr() for t in self.w), *types, hidden_type, max_tokens,
                                                torch.cuda.current_device(), C.byref(self.h)))
        native.check(self.lib.ktb200_mlp_load_weights(self.h, _stream()))

    def mats(self, oracle):
        return tuple(oracle.to_float(h, t, r * c).astype(np.float64).reshape(r, c)
                     for h, t, r, c in zip(self.host, self.types, (self.I, self.I, self.H), (self.H, self.H, self.I)))

    def close(self):
        self.lib.ktb200_mlp_destroy(self.h)


def _expert_fn(oracle, ex, shared=None):
    """float64 (gate, up, down) of expert e from the host copies (the C oracle's dequantiser); e == E: the shared expert"""
    def expert(e):
        if e == ex.E:
            return shared
        return tuple(oracle.to_float(np.ascontiguousarray(h[e]), t, r * c).astype(np.float64).reshape(r, c)
                     for h, t, (r, c) in zip(ex.host, ex.types, ((ex.I, ex.H), (ex.I, ex.H), (ex.H, ex.I))))
    return expert


def _edge_ids(T, E, k, rng):
    """random distinct ids, then: expert 1 in every token (crowded; a duplicate where the row already had it), -1 and E,
    E + 3, and expert 2 picked by nobody (k > E: ids drawn with repeats)"""
    ids = _ids(T, E, k, rng) if k <= E else rng.integers(0, E, (T, k)).astype(np.int64)
    ids[ids == 2] = 3
    ids[:, 0] = 1
    ids[0, k - 1] = -1
    ids[T - 1, 1] = E
    if T > 2:
        ids[T // 2, 2] = E + 3
    return ids


def _reference(oracle, ex, x_rows, ids_rows, w_rows, shared_mats=None):
    """float64 routed (+ shared) sums of the given tokens; invalid ids are skipped, the shared expert is expert E, weight 1"""
    E = ex.E
    ids = np.where((ids_rows >= 0) & (ids_rows < E), ids_rows, -1)
    w = w_rows
    if shared_mats is not None:
        ids = np.concatenate([ids, np.full((len(ids), 1), E)], 1)
        w = np.concatenate([w, np.ones((len(w), 1), np.float32)], 1)
    return _moe_ref(oracle, [(x_rows, ids, w)], _expert_fn(oracle, ex, shared_mats), E + 1)[0]


# Each token against its own largest output as well (tokens() spreads the token scales over three decades, so _check's bound
# on the largest token of a call leaves the small ones loose).  One int8 step of the requantised act(g) * u -- the kernel's
# fp32 g and u and the float64 reference's land on opposite sides of a rounding edge -- moves a token by up to about 2e-3 of
# its own largest output at these shapes (measured: 1.7e-3, IQ4_XS at V3); every other token of the sweep stays within 5e-4.
ROW_TOL = 4 * FP_TOL


def _check_fused(got, ref_routed, ref_shared, hidden_type, what, tol=FP_TOL):
    """_check's bound with the fused result's two roundings: hidden(hidden(routed) + hidden(shared))"""
    ref = ref_routed + ref_shared
    err = np.abs(_to_f64(got, hidden_type) - ref)
    r = ROUND_REL[hidden_type]
    bound = tol * np.abs(ref).max() + r * (np.abs(ref) + np.abs(ref_routed) + np.abs(ref_shared))
    assert (err <= bound).all(), (what, (err - bound).max(), err.max(), np.abs(ref).max())
    return float((err / np.abs(ref).max()).max())


def _forward(m, ids, w, x, mlp=None, bsz=None, out=None):
    from gpu_util import moe_forward_shared
    if mlp is None:
        return m.forward(ids, w, x, bsz=bsz, out=out)
    return moe_forward_shared(m, mlp, ids, w, x)


# ------------------------------------------------------------------------------------------------ GPU: census
def _route_census():
    """every case runs the kernels its row of the table names, in order, and the kernels seen cover every route"""
    from test_linear_routes import _census
    torch.cuda.set_device(0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    keep, calls = [], []
    for name, (types, H, I, k, sh) in CASES.items():
        ex = _Experts(16, H, I, *types, 7)
        m = ex.moe(KMAX.get(name, k), BF16, max_tokens=max(CENSUS_TS[name]))
        mlp = _SharedMlp(types, H, I, BF16, 70) if sh else None
        keep.append((ex, m, mlp))
        rng = np.random.default_rng(1)
        for T in CENSUS_TS[name]:
            ids = torch.from_numpy(_edge_ids(T, 16, k, rng)).cuda()
            w = torch.rand((T, k), device="cuda")
            x = (torch.randn((T, H), device="cuda") / 10).to(torch.bfloat16)
            out = torch.zeros((T, H), dtype=torch.bfloat16, device="cuda")
            fn = native.lib().ktb200_moe_forward_shared

            def call(m=m, mlp=mlp, T=T, k=k, ids=ids, w=w, x=x, out=out, fn=fn):
                native.check(fn(m.h, mlp.h if mlp else None, T, k, ids.data_ptr(), w.data_ptr(), x.data_ptr(), out.data_ptr(),
                                None, _stream()))
            calls.append(((name, T), case_route(name, T, sms=sms), call))
    # the grouped chunks by their launch count (their kernels: tests/test_iq_grouped.py, test_kquant_grouped.py), the per-pair
    # calls under the profiler, each launch held to its row
    per_pair = []
    for (name, T), want, call in calls:
        if want[0] == "grouped":
            n0 = native.launch_count()
            call()
            torch.cuda.synchronize()
            assert native.launch_count() - n0 == 10 * want.count("grouped") + len(want) - want.count("grouped"), (name, T, want)
        else:
            per_pair.append(((name, T), want, call))
    seen_gu, seen_dn = set(), set()
    for (name, T), want, n, names in _census(per_pair):
        assert n == len(want) and all(w in s for w, s in zip(want, names)), f"{name} T={T}: {names} ({n} launches), table: {want}"
        seen_gu.add(want[0]); seen_dn.add(want[1])
    for ex, m, mlp in keep:
        m.close()
        if mlp:
            mlp.close()
    for r in GATE_UP_ROUTES:
        assert any(g.startswith(r) for g in seen_gu), r
    for r in DOWN_ROUTES:
        assert any(d.startswith(r) for d in seen_dn), r
    print(f"\nkernels seen: gate/up {sorted(seen_gu)}; down {sorted(seen_dn)}")


@pytest.mark.gpu
def test_route_census():
    """_route_census in an interpreter of its own: after other tests' profiler sessions in the same process, torch.profiler
    can miss a kernel of the session"""
    root = os.path.dirname(HERE)
    code = ("import sys; sys.path[:0] = sys.argv[1:]; import test_expert_routes as t\n"
            "try:\n    t._route_census(); print('OK')\nexcept AssertionError as e:\n    print(e); sys.exit(1)")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, root, HERE]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, cwd=root)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-3000:] + r.stderr[-3000:]


# ------------------------------------------------------------------------------------------------ GPU: oracle sweep
# routes no dedicated file covers, at model shapes over 16 resident experts: (case, token counts)
SWEEP = {
    "q4_k_m-v3": (1, 9, 47),
    "q4_k_m-q4k_down-v3": (1, 9, 47),
    "q4_k_m-qwen3-30b": (1, 9, 47),
    "q5_k_m-v3": (1, 9, 47),
    "q5_k_m-qwen3-30b": (1, 9, 47),
    "q6_k-v3": (1, 9, 264, 1024),
    "iq4_xs-v3": (1, 9, 263, 264, 1024),
    "iq4_xs-v2": (1, 9, 264),
    "mixed-q4k_q5k_q4k-v3": (1, 9, 264),
    "q5k_x3-qwen3-30b": (1, 9, 264),
    "q4k-down-nb50-2048x12800": (1, 9, 47),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SWEEP))
def test_experts_vs_oracle(oracle, name):
    types, H, I, k, _ = CASES[name]
    E = 16
    ex = _Experts(E, H, I, *types, 11)
    Tmax = max(SWEEP[name])
    worst = {}
    for hid in (F32, BF16):
        m = _moe_copy(ex, k, hid, E, 0, 0, Tmax)
        mlp = _SharedMlp(types, H, I, hid, 50 + hid, max_tokens=Tmax)
        sh_mats = mlp.mats(oracle)
        for T in SWEEP[name]:
            rng = np.random.default_rng(T + hid)
            ids, w = _edge_ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
            xf = tokens(T, H, T + 3)
            xc = f32_to_bf16_bits(xf) if hid == BF16 else xf
            rows = oracle_rows(T, T)
            ref = _reference(oracle, ex, xf[rows], ids[rows], w[rows])
            ref_sh = _reference(oracle, ex, xf[rows], np.full((len(rows), 1), -1), np.zeros((len(rows), 1), np.float32), sh_mats)
            for shared in (False, True):
                what = f"{name} {'BF16' if hid == BF16 else 'F32'} T={T} shared={shared}"
                route = expert_route(types, H, I, k, T, shared)
                n0 = native.launch_count()
                got = _forward(m, ids, w, xc, mlp if shared else None)
                assert native.launch_count() - n0 == sum(10 if r == "grouped" else 1 for r in route), what
                # the call's checked tokens against their largest output, then each token against its own (ROW_TOL)
                if shared:
                    _check_fused(got[rows], ref, ref_sh, hid, what)
                else:
                    _check(got[rows], ref, hid, what)
                e = 0.0
                for i, r in enumerate(rows):
                    sh_i = ref_sh[i:i + 1] if shared else np.zeros_like(ref[i:i + 1])
                    e = max(e, _check_fused(got[r:r + 1], ref[i:i + 1], sh_i, hid, f"{what} token {r}", tol=ROW_TOL))
                worst[what.split(" T=")[0]] = max(worst.get(what.split(" T=")[0], 0.0), e)
                # the same kernels at 1 token: each checked token alone gives the same bits
                if T > 1 and route == expert_route(types, H, I, k, 1, shared):
                    for r in (rows[0], rows[len(rows) // 2], rows[-1]):
                        one = _forward(m, ids[r:r + 1], w[r:r + 1], xc[r:r + 1], mlp if shared else None)
                        assert np.array_equal(one[0], got[r]), f"{what}: token {r} alone differs"
            # rows at and beyond the device batch size keep their bytes
            if T > 1:
                from gpu_util import TORCH_HID
                keep = torch.full((T, H), 1536.0, dtype=TORCH_HID[hid], device="cuda")
                part = m.forward(ids, w, xc, bsz=T - 1, out=keep)
                full = m.forward(ids, w, xc)
                assert np.array_equal(part[:T - 1], full[:T - 1]) and (_to_f64(part[T - 1:], hid) == 1536.0).all(), name
        mlp.close()
        m.close()
    print(f"\nworst {name}: " + "; ".join(f"{k_} {v:.3g}" for k_, v in worst.items()) + " of the token's max|ref|")


def _moe_copy(ex, k, hid, E, lo, offset, max_tokens):
    """a handle on its own copy of experts lo .. lo + E - 1 (a Q6_K tensor is re-laid in place when a handle loads)"""
    from gpu_util import Moe
    sl = [b.view(ex.E, -1)[lo:lo + E].clone().reshape(-1) for b in ex.w]
    return Moe(E, k, ex.H, ex.I, *sl, *ex.types, hid, max_tokens=max_tokens, offset=offset)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["iq4_xs-v3", "q6_k-v3", "q5_k_m-qwen3-30b"])
def test_expert_id_offset_shards(oracle, name):
    """two shards of 8 experts (expert_id_offset 0 and 8) see the same ids; their sum is the unsharded layer's output"""
    types, H, I, k, _ = CASES[name]
    ex = _Experts(16, H, I, *types, 13)
    T = 264
    rng = np.random.default_rng(5)
    ids, w = _edge_ids(T, 16, k, rng), rng.random((T, k)).astype(np.float32)
    x = tokens(T, H, 6)
    parts = []
    for lo in (0, 8):
        m = _moe_copy(ex, k, F32, 8, lo, lo, T)
        parts.append(m.forward(ids, w, x).astype(np.float64))
        m.close()
    rows = oracle_rows(T, 7)
    _check((parts[0] + parts[1])[rows].astype(np.float32), _reference(oracle, ex, x[rows], ids[rows], w[rows]), F32, name)


GUARD_CASES = {
    # name: (types, H, I, routed_expert_num, down kernel)
    "q5k-reduce_kernel": ((Q5K, Q5K, Q5K), 2048, 512, 40, "reduce_kernel<ktb::FmtQ5K,1>"),
    "q6k-reduce_pipe_q6k8": ((Q4K, Q4K, Q6K), 1024, 1536, 100, "reduce_pipe_q6k8_kernel<"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GUARD_CASES))
def test_k_over_32_skips_ids_outside_the_shard(oracle, name):
    """k = 40 on the per-pair kernels, down on each kernel that stages a skip mask: ids -1 and E in slots >= 32 are skipped.
    The experts sit in one allocation of E + 2 between two guard experts whose every byte is 0xff (every fp16 scale NaN,
    whatever layout the down tensor is given at load time), so a slot that is not skipped reads a guard expert and turns its
    token's output NaN, without reading outside the allocation."""
    from gpu_util import Moe
    from ktransformers_b200.util.synth import synth_blocks
    types, H, I, kmax, down = GUARD_CASES[name]
    E, k, T = 16, 40, 3
    full = [synth_blocks(t, (E + 2) * r * c, "cuda", 20 + i).view(E + 2, -1)
            for i, (t, r, c) in enumerate(zip(types, (I, I, H), (H, H, I)))]
    for t in full:
        t[0].fill_(0xff)
        t[E + 1].fill_(0xff)
    ex = _Experts.__new__(_Experts)
    ex.E, ex.H, ex.I, ex.types = E, H, I, types
    ex.host = [t[1:E + 1].cpu().numpy() for t in full]
    m = Moe(E, kmax, H, I, *(t[1:E + 1].reshape(-1) for t in full), *types, F32, max_tokens=T)
    rng = np.random.default_rng(3)
    ids = rng.integers(0, E, (T, k)).astype(np.int64)
    ids[0, 32], ids[1, 39], ids[2, 33], ids[2, 38] = -1, E, -1, E
    ids[0, 5] = -1                                                   # one below 32 as well
    w = rng.random((T, k)).astype(np.float32) / k
    x = tokens(T, H, 4)
    assert expert_route(types, H, I, k, T, kmax=kmax)[1] == down
    got = m.forward(ids, w, x)
    assert np.isfinite(got).all(), f"NaN in tokens {sorted(set(np.nonzero(~np.isfinite(got))[0].tolist()))}: a slot >= 32 read a guard expert"
    _check(got, _reference(oracle, ex, x, ids, w), F32, name)
    m.close()


@pytest.mark.gpu
def test_ktmoe_wrapper_iq4_xs_v3_prompt_chunk(oracle):
    """KTMoEWrapper(method="B200_GGUF"): IQ4_XS experts at V3's shape serve a 1024-token chunk (per pair: grouped_ok declines
    IQ4_XS; down on reduce_kernel<FmtGenK> at 2 CTAs per token) against the float64 reference"""
    from ktransformers_b200.kt_moe_wrapper import KTMoEWrapper
    E, k, H, I, T = 16, 8, 7168, 2048, 1024
    ex = _Experts(E, H, I, IQ4, IQ4, IQ4, 17)
    wr = KTMoEWrapper(layer_idx=0, num_experts=E, num_experts_per_tok=k, hidden_size=H, moe_intermediate_size=I,
                      gpu_experts_mask=None, method="B200_GGUF", chunked_prefill_size=T)
    wr.load_weights_from_tensors(*(torch.from_numpy(h.reshape(E, r, -1)) for h, r in zip(ex.host, (I, I, H))),
                                 torch.arange(E), ggml_types=(IQ4, IQ4, IQ4))
    rng = np.random.default_rng(23)
    ids, w = _edge_ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    ids = np.where(ids >= E, -1, ids)             # the wrapper takes router ids: in range, or -1
    xb, xf = _x(T, H, 24, BF16)
    x = torch.from_numpy(xb.view(np.int16)).view(torch.bfloat16).cuda()
    n0 = native.launch_count()
    out = wr.forward(x, torch.from_numpy(ids).cuda(), torch.from_numpy(w).cuda())
    torch.cuda.synchronize()
    assert native.launch_count() - n0 >= 2
    got = out.cpu().view(torch.int16).numpy().view(np.uint16)
    rows = oracle_rows(T, 25)
    _check(got[rows], _reference(oracle, ex, xf[rows], ids[rows], w[rows]), BF16, "KTMoEWrapper IQ4_XS V3 1024")
