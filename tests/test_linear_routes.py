"""The GGUF dense linear (ktb200_linear_forward) and MLP (ktb200_mlp_forward) at prompt-sized batches, on every kernel
route the launchers (csrc/moe.cu: launch_rows, launch_reduce) pick under default settings.

With the shipped rule files every KTransformersLinear runs in GENERATE mode, so KLinearB200 serves every token of a prompt
chunk: the MLA projections at T = bsz * q_len, the dense MLP layers, the shared experts.  The launchers switch kernels by
weight type, shape and T (dense Q4_K linears at 8 tokens, kDenseMaxTokens), and the bulk-copy kernel walks T in token
chunks of <= 8.

  1. Route table: `linear_route` / `mlp_routes` restate the launchers' conditions (not their shared-memory plans, except the
     load-time Q6_K tile-layout decision); the case lists are generated to reach every route on both sides of each switch.
     The GPU census runs every case under torch.profiler and holds each launch to the kernel its row names.
  2. References (rows of a linear are independent):
       * the C oracle on a subset of tokens (token 0, the first 17 tokens — every chunk edge among them — the last token and
         16 seeded random ones);
       * a float64 restatement on EVERY token: activations quantised to Q8_K by the oracle and dequantised, times the
         oracle's dequantised weights, in float64.  Its CPU test pins it to the C oracle for all six weight types.
  3. Bounds.  A linear has no requantisation: activation quantisation is byte-exact, block dots are exact integers, only the
     fp32 order of at most nblk block terms is free (DESIGN §2).  So F32 outputs are held to the oracle per row within
     F32_REL * max|row| and to the float64 restatement within F32_REL * (|W| . |x_q|) per element; BF16 outputs within one
     ulp of the oracle plus F32_REL * max|row| (an element much smaller than its row may move by several of its own ulps
     within the F32 bound), >= 99 % bit-identical; F16 outputs bit-identical to the F32 output on the widened input,
     rounded.
     The MLP requantises its intermediate (int8 knife edges), so it keeps the suite's FP_TOL / assert_bf16_close bounds, on
     weights from the CPU generator (see test_moe_with_shared_expert_prefill_sized_batch).

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
from ktransformers_b200.util.synth import synth_blocks
from oracle.bindings import (BF16, F16, F32, IQ4_XS, Q2_K, Q3_K, Q4_K, Q5_K, Q6_K, Q8_K, TYPE_NAMES, bf16_to_f32,
                             f32_to_bf16_bits)

QK = 256
H100_SMS = 132
F32_REL = 1e-5
KERNEL_TYPES = (Q2_K, Q3_K, Q4_K, Q5_K, Q6_K, IQ4_XS)


# ------------------------------------------------------------------------------------------------ route table
BLOCKS_PER_STEP = {"FmtQ4K": 4, "FmtQ5K": 4, "FmtQ6K8": 8, "FmtGenK": 2}   # Fmt::kBlocksPerStep (formats.cuh)
SMEM_CAP = 232448 - 512                                                      # kSmemCap (moe.cu)


def _rows_kernel(fmt, pair, nblk):
    """launch_rows_fmt: 4 rows per warp for one step per row, 2 for two or three, 1 from four"""
    nsteps = -(-nblk // BLOCKS_PER_STEP[fmt])
    rw = 1 if nsteps >= 4 else (2 if nsteps >= 2 else 4)
    return f"rows_kernel<ktb::{fmt},{'true' if pair else 'false'},{rw},"


def _dense_q4k_takes(nblk, T):
    """launch_dense_q4k: <= 8 tokens; rows of <= 32 blocks, or split into equal segments of <= 32 blocks"""
    return T <= 8 and (nblk <= 32 or nblk % -(-nblk // 32) == 0)


def linear_route(t, n_in, n_out, T):
    """name prefix (spaces removed) of the kernel ktb200_linear_forward launches"""
    nblk = n_in // QK
    if t == Q4_K:
        if _dense_q4k_takes(nblk, T):
            return "dense_q4k_kernel<"
        if nblk >= 16:                                # launch_rows_bulk_q4k: >= 16 blocks per row
            return "rows_bulk_q4k_kernel<false,"
        return _rows_kernel("FmtQ4K", False, nblk)     # rows under 16 blocks are under the pipe kernel's 4096 bytes
    if t == Q5_K:                                      # launch_rows_pipe: rows of >= 4096 bytes
        return "rows_pipe_kernel<ktb::FmtQ5K,false," if nblk * 176 >= 4096 else _rows_kernel("FmtQ5K", False, nblk)
    if t == Q6_K and n_out % 8 == 0 and 8 * 210 * nblk <= 200 * 1024:   # ktb200_linear_load_weights: 8-row SoA repack
        return _rows_kernel("FmtQ6K8", False, nblk)
    return _rows_kernel("FmtGenK", False, nblk)


def _bulk_down_warps(rows, ncols, block_bytes, bs, slots, pcap, sms):
    """plan_down: warps of reduce_bulk_kernel for `pcap` staged pairs (0: does not fit)"""
    nb = ncols // QK
    item = 4 * nb * block_bytes
    if rows % 4 or item % 16 or pcap > 200:
        return 0
    quads = rows // 4
    gx = max(1, min(sms, quads))
    nrows_max = -(-quads // gx) * 4
    base = (pcap * nb * (QK + 16 + 2 * bs + 4) + nrows_max * pcap * 4 + pcap * 4 + 15) & ~15
    if base + 16 >= SMEM_CAP:
        return 0
    return min((SMEM_CAP - base - 16) // (slots * (item + 8)), 16)


def mlp_routes(gt, ut, dt, H, I, sms=H100_SMS):
    """(gate/up kernel, down kernel) name prefixes of ktb200_mlp_forward"""
    nblk, nb = H // QK, I // QK
    soa = gt == ut == Q6_K and I % 8 == 0
    fmt = {Q4_K: "FmtQ4K", Q5_K: "FmtQ5K"}

    def pick(t):
        return fmt.get(t, "FmtQ6K8" if t == Q6_K and soa else "FmtGenK")
    fg = pick(gt) if pick(gt) == pick(ut) else "FmtGenK"
    if fg == "FmtQ4K" and nblk >= 16:
        gu = "rows_bulk_q4k_kernel<true,"
    elif fg == "FmtQ4K" and 2 * nblk * 144 >= 4096:
        gu = "rows_pipe_kernel<ktb::FmtQ4K32,true,"
    elif fg == "FmtQ5K" and 2 * nblk * 176 >= 4096:
        gu = "rows_pipe_kernel<ktb::FmtQ5K,true,"
    else:
        gu = _rows_kernel(fg, True, nblk)
    # ktb200_mlp_load_weights: Q6_K down in 4-row tiles when the bulk kernel fits 17 slots, else 8-row SoA
    if dt == Q6_K and nb % 2 == 0 and _bulk_down_warps(H, I, 210, 16, 3, 17, sms) >= 4:
        dn = "reduce_bulk_kernel<ktb::BulkQ6K4T,"
    elif dt == Q6_K and H % 8 == 0 and 8 * 210 * nb <= 200 * 1024:
        # launch_reduce_pipe_q6k8: nb even, and 12 warps x 2 slots of 840 * nb bytes in 220 KB
        pipe = H % 4 == 0 and nb % 2 == 0 and 840 * nb >= 4096 and 24 * 840 * nb <= 220 * 1024
        dn = "reduce_pipe_q6k8_kernel<" if pipe else "reduce_kernel<ktb::FmtQ6K8,"
    elif dt == Q4_K and _bulk_down_warps(H, I, 144, 8, 2, 1, sms) >= 2:
        dn = "reduce_bulk_kernel<ktb::BulkQ4K,"
    else:
        dn = f"reduce_kernel<ktb::{ {Q4_K: 'FmtQ4K', Q5_K: 'FmtQ5K'}.get(dt, 'FmtGenK') },"
    return gu, dn


# ------------------------------------------------------------------------------------------------ cases
TS = (1, 8, 9, 16, 17, 33, 64, 839, 841, 1024, 4096)   # 840 = lcm(2..8): 839 / 841 leave tails of tc - 1 / 1 for every tc
LINEAR = {
    # name: (weight type, in, out, token counts, F16 too).  DeepSeek-V3's projections first, then route edges.
    "q4k-q_a-7168x1536": (Q4_K, 7168, 1536, TS, True),
    "q4k-q_b-1536x24576": (Q4_K, 1536, 24576, TS, True),
    "q4k-kv_a-7168x576": (Q4_K, 7168, 576, TS, False),
    "q4k-o_proj-16384x7168": (Q4_K, 16384, 7168, (8, 9, 17, 841, 4096), False),
    "q4k-gate_up-7168x18432": (Q4_K, 7168, 18432, (8, 9, 841, 4096), False),
    "q4k-down-18432x7168": (Q4_K, 18432, 7168, (8, 9, 841, 4096), False),
    "q4k-shared_down-2048x7168": (Q4_K, 2048, 7168, (1, 8, 9, 17, 841, 4096), False),
    "q4k-odd_nblk-8448x512": (Q4_K, 8448, 512, (1, 8, 9, 16, 17, 33, 839, 841), True),
    "q4k-one_block-256x777": (Q4_K, 256, 777, (1, 8, 9, 17, 841, 1024), False),
    "q4k-nblk13-3328x2051": (Q4_K, 3328, 2051, (1, 8, 9, 33, 841), False),
    "q5k-pipe-7168x1536": (Q5_K, 7168, 1536, (1, 8, 9, 33, 841, 4096), True),
    "q5k-1536x512": (Q5_K, 1536, 512, (1, 9, 33, 841), False),
    "q6k-soa-2048x7168": (Q6_K, 2048, 7168, (1, 9, 33, 841), False),
    "q6k-generic-1536x2051": (Q6_K, 1536, 2051, (1, 9, 841), False),
    "q2k-7168x1536": (Q2_K, 7168, 1536, (1, 9, 841), False),
    "q3k-7168x576": (Q3_K, 7168, 576, (1, 9, 841), False),
    "iq4xs-7168x1536": (IQ4_XS, 7168, 1536, (1, 9, 841), False),
}
F16_TS = (9, 33, 841)

MLP_MAX_TOKENS = 64
MLP_TS = (9, 33, 63, MLP_MAX_TOKENS)
MLP = {
    # name: (H, I, gate, up, down)
    "q4k-bulk_q6k-tiles-4096x1024": (4096, 1024, Q4_K, Q4_K, Q6_K),
    "q5k-pipe_q6k-soa-4096x768": (4096, 768, Q5_K, Q5_K, Q6_K),
    "q6k-soa_q6k-soa-1024x4096": (1024, 4096, Q6_K, Q6_K, Q6_K),
    "mixed-generic_q4k-bulk-2048x1024": (2048, 1024, Q4_K, Q5_K, Q4_K),
    "q2k-generic_q5k-1024x1024": (1024, 1024, Q2_K, Q2_K, Q5_K),
    "q4k-pipe_iq4xs-3840x512": (3840, 512, Q4_K, Q4_K, IQ4_XS),
    "q4k-rows_q3k-1024x512": (1024, 512, Q4_K, Q4_K, Q3_K),
    "v3-dense-7168x18432": (7168, 18432, Q4_K, Q4_K, Q6_K),
}

# the routes the case lists must reach (DESIGN §4.2)
LINEAR_ROUTES = ("dense_q4k_kernel<", "rows_bulk_q4k_kernel<false,", "rows_kernel<ktb::FmtQ4K,false,1,",
                 "rows_kernel<ktb::FmtQ4K,false,2,", "rows_kernel<ktb::FmtQ4K,false,4,", "rows_pipe_kernel<ktb::FmtQ5K,false,",
                 "rows_kernel<ktb::FmtQ5K,false,", "rows_kernel<ktb::FmtQ6K8,false,", "rows_kernel<ktb::FmtGenK,false,")
GENERIC_TYPES = (Q2_K, Q3_K, Q6_K, IQ4_XS)
MLP_GATE_UP_ROUTES = ("rows_bulk_q4k_kernel<true,", "rows_pipe_kernel<ktb::FmtQ5K,true,", "rows_pipe_kernel<ktb::FmtQ4K32,true,",
                      "rows_kernel<ktb::FmtQ6K8,true,", "rows_kernel<ktb::FmtGenK,true,", "rows_kernel<ktb::FmtQ4K,true,")
MLP_DOWN_ROUTES = ("reduce_bulk_kernel<ktb::BulkQ6K4T,", "reduce_kernel<ktb::FmtQ6K8,", "reduce_bulk_kernel<ktb::BulkQ4K,",
                   "reduce_kernel<ktb::FmtQ5K,", "reduce_kernel<ktb::FmtGenK,")


# ------------------------------------------------------------------------------------------------ references
def q8k_values(oracle, x32):
    """float64 values of the Q8_K activations (oracle quantiser): d * q per element"""
    T, n = x32.shape
    q = oracle.from_float(np.ascontiguousarray(x32).reshape(-1), Q8_K).reshape(-1, 292)
    d = q[:, :4].copy().view(np.float32).astype(np.float64)
    return (q[:, 4:260].view(np.int8).astype(np.float64) * d).reshape(T, n)


def restated(w64, xq64):
    """float64 y = x_q . W^T and the magnitude |x_q| . |W|^T that bounds the fp32 rounding of each element"""
    return xq64 @ w64.T, xq64.abs() @ w64.abs().T


def oracle_rows(T, seed):
    """token 0, the first 17 tokens (every chunk edge of chunks of 1..8), the last token and 16 seeded random ones"""
    rows = set(range(min(T, 17))) | {T - 1}
    rows |= set(np.random.default_rng(seed).choice(T, size=min(T, 16), replace=False).tolist())
    return np.array(sorted(rows))


def tokens(T, n, seed):
    """bf16-representable activations with per-token scales over three decades (F32 and BF16 calls see the same values)"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((T, n), dtype=np.float32) * np.exp(rng.uniform(-4, 2, (T, 1))).astype(np.float32) / 10
    return bf16_to_f32(f32_to_bf16_bits(x))


# ------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("t", KERNEL_TYPES, ids=[TYPE_NAMES[t] for t in KERNEL_TYPES])
def test_restatement_matches_oracle(oracle, t):
    """the float64 restatement against the C oracle's F32 linear, within the bound the GPU tests use"""
    n_in, n_out, T = 1024, 96, 6
    w = synth_blocks(t, n_out * n_in, "cpu", 7).numpy()
    x = tokens(T, n_in, t)
    x[2] = 0                                        # an all-zero row: d = 0
    x[3, :256] *= 1e-30                             # a block far below the others
    want = oracle.linear_forward(n_in, n_out, w, t, F32, x).astype(np.float64)
    w64 = torch.from_numpy(oracle.to_float(w, t, n_out * n_in).reshape(n_out, n_in)).double()
    ref, mag = (a.numpy() for a in restated(w64, torch.from_numpy(q8k_values(oracle, x))))
    assert not want[2].any() and not ref[2].any()
    err = np.abs(want - ref) / np.maximum(mag, 1e-300)
    assert err.max() <= F32_REL, err.max()
    assert np.abs(ref).max() > 0


def test_q8k_values_are_the_oracle_activations(oracle):
    """d * q of every block reproduces the oracle's own dot product against an all-ones F32 weight row"""
    x = tokens(3, 512, 1)
    xq = q8k_values(oracle, x)
    for i in range(3):
        q = oracle.from_float(x[i], Q8_K).reshape(-1, 292)
        for b in range(2):
            assert np.array_equal(xq[i, b * 256:(b + 1) * 256] / q[b, :4].copy().view(np.float32)[0], q[b, 4:260].view(np.int8))


def test_route_table_covers_every_route():
    routes = {(t, linear_route(t, i, o, T)) for t, i, o, ts, _ in LINEAR.values() for T in ts}
    for r in LINEAR_ROUTES:
        assert any(rr.startswith(r) for _, rr in routes), r
    for t in GENERIC_TYPES:
        assert any(tt == t and rr.startswith("rows_kernel<ktb::FmtGenK,") for tt, rr in routes), TYPE_NAMES[t]
    mlp = [mlp_routes(g, u, d, H, I) for H, I, g, u, d in MLP.values()]
    for r in MLP_GATE_UP_ROUTES:
        assert any(gu.startswith(r) for gu, _ in mlp), r
    for r in MLP_DOWN_ROUTES:
        assert any(dn.startswith(r) for _, dn in mlp), r


def test_token_counts_straddle_every_switch():
    for name, (t, i, o, ts, _) in LINEAR.items():
        rs = [linear_route(t, i, o, T) for T in ts]
        for a, b, ra, rb in zip(ts, ts[1:], rs, rs[1:]):
            assert ra == rb or b == a + 1, f"{name}: the route changes between {a} and {b} tokens"
        if t == Q4_K and _dense_q4k_takes(i // QK, 8):
            assert 8 in ts and 9 in ts, name
    for T in (839, 841):
        assert {T % tc for tc in range(2, 9)} == ({tc - 1 for tc in range(2, 9)} if T == 839 else {1})


def test_mlp_never_takes_the_q6k_soa_pipe():
    """Under default settings the MLP's Q6_K down projection takes the 4-row tile layout wherever the SoA pipe kernel
    would fit (nb even and <= 10 blocks), so reduce_pipe_q6k8_kernel serves routed experts only."""
    for H in range(256, 16384 + 1, 256):
        for I in range(256, 24576 + 1, 256):
            assert not mlp_routes(Q6_K, Q6_K, Q6_K, H, I)[1].startswith("reduce_pipe_q6k8_kernel<"), (H, I)


# ------------------------------------------------------------------------------------------------ GPU helpers
def _stream():
    return torch.cuda.current_stream().cuda_stream


TORCH_HID = {F32: torch.float32, F16: torch.float16, BF16: torch.bfloat16}


class Linear:
    """a ktb200_linear handle on its own copy of the weights (Q6_K handles re-lay them out in place)"""

    def __init__(self, t, n_in, n_out, w, hid):
        self.lib, self.n_out, self.hid = native.lib(), n_out, hid
        self.w = w.clone()
        self.h = C.c_void_p()
        native.check(self.lib.ktb200_linear_create(n_in, n_out, self.w.data_ptr(), t, hid, 1024, torch.cuda.current_device(),
                                                   C.byref(self.h)))
        native.check(self.lib.ktb200_linear_load_weights(self.h, _stream()))

    def __call__(self, x, bias=None):
        """x: cuda tensor [T][in] of the hidden type; rows the kernel does not write stay NaN"""
        y = torch.full((x.shape[0], self.n_out), float("nan"), dtype=TORCH_HID[self.hid], device="cuda")
        native.check(self.lib.ktb200_linear_forward(self.h, x.shape[0], x.data_ptr(), y.data_ptr(),
                                                    bias.data_ptr() if bias is not None else None, None, _stream()))
        return y

    def close(self):
        self.lib.ktb200_linear_destroy(self.h)


class Mlp:
    def __init__(self, H, I, g, u, d, gt, ut, dt, hid):
        self.lib, self.H, self.hid = native.lib(), H, hid
        self.keep = (g.clone(), u.clone(), d.clone())
        self.h = C.c_void_p()
        native.check(self.lib.ktb200_mlp_create(H, I, *(t.data_ptr() for t in self.keep), gt, ut, dt, hid, MLP_MAX_TOKENS,
                                                torch.cuda.current_device(), C.byref(self.h)))
        native.check(self.lib.ktb200_mlp_load_weights(self.h, _stream()))

    def __call__(self, x, prev=None):
        y = prev.clone() if prev is not None else torch.full((x.shape[0], self.H), float("nan"), dtype=TORCH_HID[self.hid], device="cuda")
        native.check(self.lib.ktb200_mlp_forward(self.h, x.shape[0], x.data_ptr(), y.data_ptr(), int(prev is not None), None, _stream()))
        return y

    def close(self):
        self.lib.ktb200_mlp_destroy(self.h)


def _census(calls):
    """run `calls` [(label, expected kernel prefixes in launch order, fn)] in ONE torch.profiler session (many short sessions
    in one process can come back without kernels) and return [(label, expected, launches counted, kernel names)]"""
    from torch.profiler import ProfilerActivity, profile
    counts = []
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _, _, fn in calls:
            n0 = native.launch_count()
            fn()
            torch.cuda.synchronize()
            counts.append(native.launch_count() - n0)
    names = [e.name.replace(" ", "") for e in sorted((e for e in prof.events() if "ktb::" in e.name), key=lambda e: e.time_range.start)]
    assert len(names) == sum(counts), f"{len(names)} library kernels recorded, {sum(counts)} launched"
    out, i = [], 0
    for (label, want, _), n in zip(calls, counts):
        out.append((label, want, n, names[i:i + n]))
        i += n
    return out


def _bf16_bits(t):
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


def _weights(t, n, seed):
    return synth_blocks(t, n, device="cuda", seed=seed)


def _cpu_weights(t, n, seed):
    return synth_blocks(t, n, device="cpu", seed=seed).cuda()


# ------------------------------------------------------------------------------------------------ GPU: census
def _route_census():
    """every case runs the kernel its row of the table names, and the kernels seen cover every row"""
    torch.cuda.set_device(0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    keep, calls = [], []
    for name, (t, n_in, n_out, ts, _) in LINEAR.items():
        lin = Linear(t, n_in, n_out, _weights(t, n_out * n_in, 3), F32)
        keep.append(lin)
        for T in ts:
            x = torch.randn((T, n_in), device="cuda") / 10
            calls.append(((name, t, T), (linear_route(t, n_in, n_out, T),), lambda lin=lin, x=x: lin(x)))
    for name, (H, I, gt, ut, dt) in MLP.items():
        m = Mlp(H, I, _weights(gt, I * H, 4), _weights(ut, I * H, 5), _weights(dt, H * I, 6), gt, ut, dt, F32)
        keep.append(m)
        for T in MLP_TS:
            x = torch.randn((T, H), device="cuda") / 10
            calls.append(((name, "mlp", T), mlp_routes(gt, ut, dt, H, I, sms), lambda m=m, x=x: m(x)))
    seen, seen_gu, seen_dn = set(), set(), set()
    for (name, t, T), want, n, names in _census(calls):
        assert n == len(want) and all(w in k for w, k in zip(want, names)), f"{name} T={T}: {names} ({n} launches), table: {want}"
        if t == "mlp":
            seen_gu.add(want[0]); seen_dn.add(want[1])
        else:
            seen.add((t, want[0]))
    for h in keep:
        h.close()
    for r in LINEAR_ROUTES:
        assert any(rr.startswith(r) for _, rr in seen), r
    for g in GENERIC_TYPES:
        assert any(tt == g and "FmtGenK" in rr for tt, rr in seen), TYPE_NAMES[g]
    for r in MLP_GATE_UP_ROUTES:
        assert any(g.startswith(r) for g in seen_gu), r
    for r in MLP_DOWN_ROUTES:
        assert any(d.startswith(r) for d in seen_dn), r
    print(f"\nkernels seen: linear {sorted(r for _, r in seen)}; mlp gate/up {sorted(seen_gu)}; mlp down {sorted(seen_dn)}")


@pytest.mark.gpu
def test_route_census():
    """_route_census in an interpreter of its own: after other tests' profiler sessions in the same process, torch.profiler
    can miss a kernel of the session"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = ("import sys; sys.path[:0] = sys.argv[1:]; import test_linear_routes as t\n"
            "try:\n    t._route_census(); print('OK')\nexcept AssertionError as e:\n    print(e); sys.exit(1)")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, root, os.path.join(root, "tests")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-2000:] + r.stderr[-2000:]


# ------------------------------------------------------------------------------------------------ GPU: linear
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(LINEAR))
def test_linear_vs_oracle_and_float64(oracle, name):
    t, n_in, n_out, ts, with_f16 = LINEAR[name]
    w = _weights(t, n_out * n_in, n_in + n_out)
    w_np = w.cpu().numpy()
    w64 = torch.from_numpy(oracle.to_float(w_np, t, n_out * n_in).reshape(n_out, n_in)).cuda().double()
    hids = (F32, BF16, F16) if with_f16 else (F32, BF16)
    lin = {h: Linear(t, n_in, n_out, w, h) for h in hids}
    bias = torch.from_numpy(np.random.default_rng(n_out).standard_normal(n_out).astype(np.float32)).cuda()
    worst = {"f32/oracle": 0.0, "f32/f64": 0.0, "bf16/f64": 0.0, "bf16 identical": 1.0}
    for T in ts:
        x = tokens(T, n_in, T * 7 + n_in)
        x_d = torch.from_numpy(x).cuda()
        ref, mag = restated(w64, torch.from_numpy(q8k_values(oracle, x)).cuda())
        rows = oracle_rows(T, T)
        want = oracle.linear_forward(n_in, n_out, w_np, t, F32, x[rows])
        for b in (None, bias):
            what = f"{name} T={T} bias={b is not None}"
            v = ref + b.double() if b is not None else ref
            # F32: every element against the float64 restatement, the oracle's rows per row
            y = lin[F32](x_d, b)
            e64 = ((y.double() - v).abs() - 2.0 ** -24 * v.abs()) / mag.clamp_min(1e-300)
            worst["f32/f64"] = max(worst["f32/f64"], float(e64.max()))
            assert float(e64.max()) <= F32_REL, f"{what}: F32 vs float64 {float(e64.max()):.3g} x |W|.|x_q| at {divmod(int(e64.argmax()), n_out)}"
            got = y[torch.from_numpy(rows).cuda()].cpu().numpy()
            wb = want + b.cpu().numpy() if b is not None else want
            eo = np.abs(got - wb).max(1) / np.maximum(np.abs(wb).max(1), 1e-30)
            worst["f32/oracle"] = max(worst["f32/oracle"], float(eo.max()))
            assert eo.max() <= F32_REL, f"{what}: F32 vs oracle {eo.max():.3g} of the row's max at token {rows[eo.argmax()]}"
            # BF16 on the same (bf16-exact) values: one ulp of the oracle's rounded output, >= 99 % identical
            yb = lin[BF16](x_d.to(torch.bfloat16), b)
            eb = ((yb.double() - v).abs() - 2.0 ** -8 * v.abs()) / mag.clamp_min(1e-300)
            worst["bf16/f64"] = max(worst["bf16/f64"], float(eb.max()))
            assert float(eb.max()) <= F32_REL, f"{what}: BF16 vs float64 beyond rounding at {divmod(int(eb.argmax()), n_out)}"
            gb, wbb = _bf16_bits(yb[torch.from_numpy(rows).cuda()]), f32_to_bf16_bits(wb)
            a, c = bf16_to_f32(gb), bf16_to_f32(wbb)
            tol = 2.0 ** -7 * np.maximum(np.abs(a), np.abs(c)) + F32_REL * np.abs(c).max(1, keepdims=True)
            assert (np.abs(a - c) <= tol).all(), f"{what}: BF16 more than one ulp (+ the F32 bound) from the oracle"
            same = float((gb == wbb).mean())
            worst["bf16 identical"] = min(worst["bf16 identical"], same)
            assert same >= 0.99, f"{what}: BF16 {same:.4f} bit-identical to the oracle"
            # F16: exactly the F32 output on the widened input, rounded
            if F16 in lin and T in F16_TS:
                xh = x_d.to(torch.float16)
                yh, y32 = lin[F16](xh, b), lin[F32](xh.float(), b)
                assert torch.equal(yh.view(torch.int16), y32.to(torch.float16).view(torch.int16)), f"{what}: F16 != rounded F32"
        del ref, mag
    for h in lin.values():
        h.close()
    print(f"\nworst {name}: F32 vs oracle {worst['f32/oracle']:.3g} of the row max; F32 vs float64 {worst['f32/f64']:.3g} x |W|.|x_q|; "
          f"BF16 vs float64 beyond rounding {worst['bf16/f64']:.3g} x |W|.|x_q|; BF16 identical to the oracle {worst['bf16 identical']:.4f}")


# ------------------------------------------------------------------------------------------------ GPU: MLP
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(MLP))
def test_mlp_vs_oracle(oracle, name):
    from test_gpu_parity import FP_TOL, assert_bf16_close
    H, I, gt, ut, dt = MLP[name]
    seed = H + I + 100 * dt
    g, u, d = _cpu_weights(gt, I * H, seed + 1), _cpu_weights(ut, I * H, seed + 2), _cpu_weights(dt, H * I, seed + 3)
    g_np, u_np, d_np = g.cpu().numpy(), u.cpu().numpy(), d.cpu().numpy()
    for hid in (F32, BF16):
        m = Mlp(H, I, g, u, d, gt, ut, dt, hid)
        for T in MLP_TS:
            rng = np.random.default_rng(T + hid)
            x32 = (rng.standard_normal((T, H)) / 10).astype(np.float32)
            prev32 = rng.standard_normal((T, H)).astype(np.float32)
            rows = oracle_rows(T, T) if 3 * H * I * T > 2e9 else np.arange(T)
            r_d = torch.from_numpy(rows).cuda()
            if hid == F32:
                x_d = torch.from_numpy(x32).cuda()
                want = oracle.mlp_forward(H, I, g_np, u_np, d_np, gt, ut, dt, F32, x32[rows])
                got = m(x_d)[r_d].cpu().numpy()
                err = float(np.abs(got - want).max() / np.abs(want).max())
                assert err < FP_TOL, f"{name} T={T}: {err:.3g}"
                got = m(x_d, torch.from_numpy(prev32).cuda())[r_d].cpu().numpy()
                err = float(np.abs(got - (prev32[rows] + want)).max() / np.abs(prev32[rows] + want).max())
                assert err < FP_TOL, f"{name} T={T} accumulate: {err:.3g}"
            else:
                xb, pb = f32_to_bf16_bits(x32), f32_to_bf16_bits(prev32)
                x_d = torch.from_numpy(xb.view(np.int16)).view(torch.bfloat16).cuda()
                want = oracle.mlp_forward(H, I, g_np, u_np, d_np, gt, ut, dt, BF16, xb[rows])
                assert_bf16_close(_bf16_bits(m(x_d)[r_d]), want)
                got = _bf16_bits(m(x_d, torch.from_numpy(pb.view(np.int16)).view(torch.bfloat16).cuda())[r_d])
                assert_bf16_close(got, f32_to_bf16_bits(bf16_to_f32(pb[rows]) + bf16_to_f32(want)))
        m.close()
