#!/usr/bin/env python
"""How fast can a launch of the expert kernels' SIZE stream its bytes, arithmetic removed?
(a) the bulk-copy ring of gemv_bulk.cuh (cp.async.bulk + mbarrier, W warps x S slots per SM), (b) plain LDG.128.
One launch reads 148.6 MB (gate/up: 36864 rows of 4032 B) or 108.4 MB (down: 16128 items of 6720 B) at a fresh offset
of an 8 GiB buffer (no L2 reuse).  Usage: python profiles/probe_bulk.py > probe_bulk.txt"""
import ctypes as C
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from ktransformers_b200 import native

lib = native.lib()
buf = torch.randint(0, 255, (8 << 30,), dtype=torch.uint8, device="cuda")
ms = C.c_float()
s = torch.cuda.current_stream().cuda_stream


def run(mode, a, b, chunk, nbytes, reps=24):
    ts = []
    span = (nbytes + 4095) // 4096 * 4096
    for r in range(reps):
        off = (r * span) % (buf.numel() - span)
        native.check(lib.ktb200_debug_stream_read(buf.data_ptr() + off, nbytes, mode, a, b, chunk, s, C.byref(ms)))
        ts.append(ms.value * 1e3)
    ts = ts[4:]
    return min(ts), statistics.median(ts)


print("kind            chunk   W  S    min_us  med_us  GB/s(med)")
for label, chunk, n in (("gate/up", 4032, 36864), ("down", 6720, 16128)):
    nbytes = chunk * n
    for W, S in ((12, 2), (12, 4), (16, 3), (18, 2), (18, 3), (24, 2), (27, 2), (32, 1), (15, 2), (10, 3), (16, 2), (8, 4)):
        if W * S * (chunk + 8) + 64 > 232448 - 256 or S < 2:
            continue
        lo, med = run(2, S, W, chunk, nbytes)
        print(f"bulk {label:8s} {chunk:6d} {W:3d} {S:2d} {lo:9.2f} {med:7.2f} {nbytes / med / 1e3:9.1f}", flush=True)
    for unroll, cps in ((4, 4), (8, 4), (8, 8)):
        lo, med = run(1, unroll, cps, chunk, nbytes)
        print(f"ldg  {label:8s} {chunk:6d} u{unroll} c{cps} {lo:9.2f} {med:7.2f} {nbytes / med / 1e3:9.1f}", flush=True)
