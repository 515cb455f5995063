#!/usr/bin/env python
"""Where does the time go inside the persistent MoE-block kernel?  Thread 0 of every CTA stamps %globaltimer at the
phase boundaries (ktb200_debug_block_trace); this prints, per boundary, when the first / median / last CTA passed it,
relative to the first CTA's start.  DeepSeek-V3 shapes, bs=1.  Usage on the GPU box:
    python profiles/block_trace.py > block_trace.txt"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from ktransformers_b200 import native
from ktransformers_b200.util.synth import synth_blocks

lib = native.lib()
E, K, H, I = 256, 8, 7168, 2048
Q4_K, Q6_K, BF16 = 12, 14, 30
S = lambda: torch.cuda.current_stream().cuda_stream
layers = []
for l in range(3):
    g, u, d = synth_blocks(Q4_K, E * I * H, device="cuda", seed=3 * l), synth_blocks(Q4_K, E * I * H, device="cuda", seed=3 * l + 1), synth_blocks(Q6_K, E * H * I, device="cuda", seed=3 * l + 2)
    sg, su, sd = synth_blocks(Q4_K, I * H, device="cuda", seed=100 + l), synth_blocks(Q4_K, I * H, device="cuda", seed=200 + l), synth_blocks(Q6_K, H * I, device="cuda", seed=300 + l)
    cfg = native.MoeConfig(E, K, H, I, 64, 10, 8, 1, g.data_ptr(), u.data_ptr(), d.data_ptr(), Q4_K, Q4_K, Q6_K, BF16, 0)
    moe = C.c_void_p(); native.check(lib.ktb200_moe_create(C.byref(cfg), 0, C.byref(moe))); native.check(lib.ktb200_moe_load_weights(moe, S()))
    mlp = C.c_void_p(); native.check(lib.ktb200_mlp_create(H, I, sg.data_ptr(), su.data_ptr(), sd.data_ptr(), Q4_K, Q4_K, Q6_K, BF16, 8, 0, C.byref(mlp)))
    native.check(lib.ktb200_mlp_load_weights(mlp, S()))
    W = torch.randn(E, H, device="cuda"); b = torch.randn(E, device="cuda")
    gc = native.GateConfig(E, H, K, 8, 4, 0, 0, 1, 2.5, W.data_ptr(), b.data_ptr(), BF16)
    layers.append((gc, moe, mlp, (g, u, d, sg, su, sd, W, b)))
x = (torch.randn(1, H, device="cuda") / 100).to(torch.bfloat16)
y = torch.zeros(1, H, dtype=torch.bfloat16, device="cuda")
ids = torch.zeros(1, K, dtype=torch.int64, device="cuda"); wts = torch.zeros(1, K, device="cuda")
n_sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count   # one CTA per SM
trace = torch.zeros(n_sm * 16, dtype=torch.int64, device="cuda")
names = ["start", "x quantised (under barrier 1)", "router partials written", "grid barrier 1 passed", "top-k selected",
         "gate/up done (CTA)", "entry 0 ready (its a in smem)", "last entry ready (its a in smem)", "down tiles done (CTA)", "combined + stored",
         "  (top-k done, before the work-list build)"]
acc = []
for rep in range(12):
    gc, moe, mlp, _ = layers[rep % 3]
    lib.ktb200_debug_block_trace(trace.data_ptr())
    native.check(lib.ktb200_moe_block_forward(C.byref(gc), moe, mlp, 1, x.data_ptr(), y.data_ptr(), ids.data_ptr(), wts.data_ptr(), None, S()))
    torch.cuda.synchronize()
    t = trace.cpu().numpy().reshape(n_sm, 16)[:, :11].astype(np.float64)
    t -= t[:, 0].min()
    if rep >= 3:
        acc.append(t)
lib.ktb200_debug_block_trace(None)
t = np.mean(acc, axis=0) / 1e3
print(f"{'boundary':42s} {'first':>8s} {'median':>8s} {'last':>8s}   (us after the first CTA started; mean of {len(acc)} launches)")
for i in sorted(range(len(names)), key=lambda i: np.median(t[:, i])):
    print(f"{names[i]:42s} {t[:, i].min():8.2f} {np.median(t[:, i]):8.2f} {t[:, i].max():8.2f}")
