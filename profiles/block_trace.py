#!/usr/bin/env python
"""Where does the time go inside the persistent MoE-block kernel?  Thread 0 of every CTA stamps %globaltimer at the
phase boundaries (ktb200_debug_block_trace); this prints, per boundary, when the first / median / last CTA passed it,
relative to the first CTA's start.  DeepSeek-V3 shapes, bs=1.  Usage on the GPU box:
    python profiles/block_trace.py > block_trace.txt            # eager, synchronised, cooperative launches
    python profiles/block_trace.py --graph > block_trace.txt    # bench.py's mode: 58 layers in one CUDA graph, PDL

--graph captures 58 launches over 4 resident layer sets in one CUDA graph with KTB200_BLK_COOP=0 (plain grid +
programmatic dependent launch), every launch with its own stamp buffer, and reads the stamps of one replay after warm-up.
Launches 1..57 are also reported relative to the moment the previous launch's last CTA finished (its combined output
stored): under PDL a CTA starts while the previous layer's tail still runs, so "after start" alone hides the overlap."""
import argparse
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap = argparse.ArgumentParser()
ap.add_argument("--graph", action="store_true", help="58 launches in one CUDA graph with PDL, as bench.py times them")
args = ap.parse_args()
if args.graph:
    os.environ["KTB200_BLK_COOP"] = "0"   # read once, at the first launch
import numpy as np
import torch

from ktransformers_b200 import native
from ktransformers_b200.util.synth import synth_blocks

lib = native.lib()
E, K, H, I = 256, 8, 7168, 2048
Q4_K, Q6_K, BF16 = 12, 14, 30
N_LAYERS = 58
S = lambda: torch.cuda.current_stream().cuda_stream
layers = []
for l in range(4 if args.graph else 3):
    g, u, d = synth_blocks(Q4_K, E * I * H, device="cuda", seed=3 * l), synth_blocks(Q4_K, E * I * H, device="cuda", seed=3 * l + 1), synth_blocks(Q6_K, E * H * I, device="cuda", seed=3 * l + 2)
    sg, su, sd = synth_blocks(Q4_K, I * H, device="cuda", seed=100 + l), synth_blocks(Q4_K, I * H, device="cuda", seed=200 + l), synth_blocks(Q6_K, H * I, device="cuda", seed=300 + l)
    cfg = native.MoeConfig(E, K, H, I, 64, 10, 8, 1, g.data_ptr(), u.data_ptr(), d.data_ptr(), Q4_K, Q4_K, Q6_K, BF16, 0)
    moe = C.c_void_p(); native.check(lib.ktb200_moe_create(C.byref(cfg), 0, C.byref(moe))); native.check(lib.ktb200_moe_load_weights(moe, S()))
    mlp = C.c_void_p(); native.check(lib.ktb200_mlp_create(H, I, sg.data_ptr(), su.data_ptr(), sd.data_ptr(), Q4_K, Q4_K, Q6_K, BF16, 8, 0, C.byref(mlp)))
    native.check(lib.ktb200_mlp_load_weights(mlp, S()))
    W = torch.randn(E, H, device="cuda"); b = (0.01 if args.graph else 1.0) * torch.randn(E, device="cuda")
    gc = native.GateConfig(E, H, K, 8, 4, 0, 0, 1, 2.5, W.data_ptr(), b.data_ptr(), BF16)
    layers.append((gc, moe, mlp, (g, u, d, sg, su, sd, W, b)))
x = (torch.randn(1, H, device="cuda") / 100).to(torch.bfloat16)
n_sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count   # one CTA per SM
names = ["start", "x quantised (under barrier 1)", "router partials written", "grid barrier 1 passed", "top-k selected",
         "gate/up done (CTA)", "entry 0 ready (its a in smem)", "last entry ready (its a in smem)", "down tiles done (CTA)", "combined + stored",
         "  (top-k done, before the work-list build)", "first routed gate/up row landed (warp 0)"]
NS = len(names)
PRELUDE = [0, 2, 1, 3, 10, 4, 11]


def table(t, title):
    print(f"{'boundary':46s} {'first':>8s} {'median':>8s} {'last':>8s}   ({title})")
    for i in sorted(range(NS), key=lambda i: np.median(t[:, i])):
        print(f"{names[i]:46s} {t[:, i].min():8.2f} {np.median(t[:, i]):8.2f} {t[:, i].max():8.2f}")


if not args.graph:
    y = torch.zeros(1, H, dtype=torch.bfloat16, device="cuda")
    ids = torch.zeros(1, K, dtype=torch.int64, device="cuda"); wts = torch.zeros(1, K, device="cuda")
    trace = torch.zeros(n_sm * 16, dtype=torch.int64, device="cuda")
    acc = []
    for rep in range(12):
        gc, moe, mlp, _ = layers[rep % 3]
        lib.ktb200_debug_block_trace(trace.data_ptr())
        native.check(lib.ktb200_moe_block_forward(C.byref(gc), moe, mlp, 1, x.data_ptr(), y.data_ptr(), ids.data_ptr(), wts.data_ptr(), None, S()))
        torch.cuda.synchronize()
        t = trace.cpu().numpy().reshape(n_sm, 16)[:, :NS].astype(np.float64)
        t -= t[:, 0].min()
        if rep >= 3:
            acc.append(t)
    lib.ktb200_debug_block_trace(None)
    table(np.mean(acc, axis=0) / 1e3, f"us after the first CTA started; mean of {len(acc)} eager launches")
    sys.exit(0)

# ---- graph mode: bench.py's 58 back-to-back launches, one stamp buffer per launch
y = torch.zeros(N_LAYERS, 1, H, dtype=torch.bfloat16, device="cuda")
ids = torch.zeros(N_LAYERS, 1, K, dtype=torch.int64, device="cuda"); wts = torch.zeros(N_LAYERS, 1, K, device="cuda")
trace = torch.zeros(N_LAYERS, n_sm, 16, dtype=torch.int64, device="cuda")


def step(traced):
    for l in range(N_LAYERS):
        gc, moe, mlp, _ = layers[l % 4]
        lib.ktb200_debug_block_trace(trace[l].data_ptr() if traced else None)   # read at launch: baked into the captured node
        native.check(lib.ktb200_moe_block_forward(C.byref(gc), moe, mlp, 1, x.data_ptr(), y[l].data_ptr(), ids[l].data_ptr(), wts[l].data_ptr(), None, S()))
    lib.ktb200_debug_block_trace(None)


step(False)
torch.cuda.synchronize()
side = torch.cuda.Stream()
side.wait_stream(torch.cuda.current_stream())
with torch.cuda.stream(side):
    step(True)
torch.cuda.current_stream().wait_stream(side)
torch.cuda.synchronize()
gr = torch.cuda.CUDAGraph()
with torch.cuda.graph(gr):
    step(True)
for _ in range(5):
    gr.replay()
torch.cuda.synchronize()
trace.zero_()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); gr.replay(); e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1)
tr = trace.cpu().numpy()[:, :, :NS].astype(np.float64)
print(f"# {torch.cuda.get_device_name()}: one replay of {N_LAYERS} launches in {ms:.3f} ms = {1e3 * ms / N_LAYERS:.1f} us per launch (stamps on)")
rel_start = np.mean([tr[l] - tr[l, :, 0].min() for l in range(1, N_LAYERS)], axis=0) / 1e3
table(rel_start, f"us after this launch's first CTA started; mean of launches 1..{N_LAYERS - 1} of one replay")
print()
rel_prev = np.mean([tr[l] - tr[l - 1, :, 9].max() for l in range(1, N_LAYERS)], axis=0) / 1e3
table(rel_prev, f"us after the previous launch's last CTA stored its output; mean of launches 1..{N_LAYERS - 1}")
print()
per = np.array([tr[l, :, 9].max() - tr[l - 1, :, 9].max() for l in range(1, N_LAYERS)]) / 1e3
print(f"last-CTA-done to last-CTA-done per launch: median {np.median(per):.2f} us, min {per.min():.2f}, max {per.max():.2f}")
print("prelude split (median CTA, us after the previous launch's last CTA):")
for i in PRELUDE:
    print(f"  {names[i].strip():46s} {np.median(rel_prev[:, i]):8.2f}")
