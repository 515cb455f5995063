#!/usr/bin/env python
"""What read bandwidth does a plain streaming kernel reach on this GPU?  (context for the roofline fractions)
Usage: python profiles/probe_read.py > probe_read.txt"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from ktransformers_b200 import native

lib = native.lib()
buf = torch.randint(0, 255, (8 << 30,), dtype=torch.uint8, device="cuda")   # 8 GiB >> L2
ms = C.c_float()
s = torch.cuda.current_stream().cuda_stream
print("mode unroll ctas/sm chunk  GB/s")
for mode, chunk in ((0, 0), (1, 4032), (1, 8064), (1, 1680), (1, 65536)):
    for unroll in (2, 4, 8):
        for cps in (2, 4, 8):
            best = 0.0
            for rep in range(3):
                native.check(lib.ktb200_debug_stream_read(buf.data_ptr(), buf.numel(), mode, unroll, cps, chunk if chunk else 16, s, C.byref(ms)))
                n = buf.numel() if mode == 0 else buf.numel() // chunk * chunk
                best = max(best, n / (ms.value * 1e-3) / 1e9)
            print(f"{mode:4d} {unroll:6d} {cps:7d} {chunk:6d} {best:8.1f}", flush=True)
# torch reference points
x = torch.empty(2 << 30, dtype=torch.uint8, device="cuda"); y = torch.empty_like(x)
for name, fn, nbytes in (("copy (r+w)", lambda: y.copy_(x), 2 * x.numel()), ("sum (read)", lambda: x.view(torch.int32).sum(), x.numel())):
    fn(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        fn()
    e1.record(); torch.cuda.synchronize()
    print(f"torch {name}: {nbytes * 5 / (e0.elapsed_time(e1) * 1e-3) / 1e9:.1f} GB/s")
