#!/usr/bin/env python
"""Where does the time go inside the expert-parallel MoE block kernel (ktb200_moe_ep_block_forward)?  Thread 0 of every
CTA stamps %globaltimer at the phase boundaries; every rank prints when its first / median / last CTA passed each
boundary relative to its own first CTA's start, plus the number of (token, expert) pairs it owned.  DeepSeek-V3 shapes,
one token per GPU.  Usage on the GPU box (N GPUs):
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 profiles/ep_trace.py > ep_trace_nN.txt"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

from ktransformers_b200 import native
from ktransformers_b200.operators.expert_parallel import PeerExchange
from ktransformers_b200.util.synth import synth_blocks

rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(lr)
dev = torch.device("cuda", lr)
dist.init_process_group("nccl", device_id=dev)
lib = native.lib()
E, K, H, I = 256, 8, 7168, 2048
El = E // world
Q4_K, Q6_K, BF16 = 12, 14, 30
S = lambda: torch.cuda.current_stream().cuda_stream
layers = []
for l in range(3):
    sd_ = 1000 * l + 17 * rank
    g, u, d = synth_blocks(Q4_K, El * I * H, device=dev, seed=sd_), synth_blocks(Q4_K, El * I * H, device=dev, seed=sd_ + 1), synth_blocks(Q6_K, El * H * I, device=dev, seed=sd_ + 2)
    sg, su, sd = synth_blocks(Q4_K, I * H, device=dev, seed=100 + l), synth_blocks(Q4_K, I * H, device=dev, seed=200 + l), synth_blocks(Q6_K, H * I, device=dev, seed=300 + l)
    cfg = native.MoeConfig(El, K, H, I, 64, 10, 8, 1, g.data_ptr(), u.data_ptr(), d.data_ptr(), Q4_K, Q4_K, Q6_K, BF16, rank * El)
    moe = C.c_void_p(); native.check(lib.ktb200_moe_create(C.byref(cfg), lr, C.byref(moe))); native.check(lib.ktb200_moe_load_weights(moe, S()))
    mlp = C.c_void_p(); native.check(lib.ktb200_mlp_create(H, I, sg.data_ptr(), su.data_ptr(), sd.data_ptr(), Q4_K, Q4_K, Q6_K, BF16, 8, lr, C.byref(mlp)))
    native.check(lib.ktb200_mlp_load_weights(mlp, S()))
    gen = torch.Generator(device=dev); gen.manual_seed(1000 * l + 9)
    W = torch.randn(E, H, device=dev, generator=gen); b = 0.01 * torch.randn(E, device=dev, generator=gen)   # balanced routing (see bench.py)
    gc = native.GateConfig(E, H, K, 8, 4, 0, 0, 1, 2.5, W.data_ptr(), b.data_ptr(), BF16)
    layers.append((gc, moe, mlp, (g, u, d, sg, su, sd, W, b)))
ex = PeerExchange(H, BF16, dev)
gx = torch.Generator(device=dev); gx.manual_seed(77 + rank)
y = torch.zeros(1, H, dtype=torch.bfloat16, device=dev)
ids = torch.zeros(1, K, dtype=torch.int64, device=dev); wts = torch.zeros(1, K, device=dev)
n_sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count   # one CTA per SM
trace = torch.zeros(n_sm * 16, dtype=torch.int64, device=dev)
names = ["start", "-", "router partials written", "grid barrier 1 passed", "top-k done, shared gate/up consumed", "all tokens arrived (peer flags)",
         "gate/up done (CTA)", "grid barrier 2 passed", "down done (CTA)", "all partial rows arrived (peer counters)", "combined + stored"]
acc, pairs = [], []
for rep in range(14):
    gc, moe, mlp, _ = layers[rep % 3]
    x = (torch.randn(1, H, device=dev, generator=gx) / 100).to(torch.bfloat16)
    torch.cuda.synchronize(); dist.barrier()
    lib.ktb200_debug_block_trace(trace.data_ptr())
    native.check(lib.ktb200_moe_ep_block_forward(C.byref(gc), moe, mlp, C.byref(ex.comm), x.data_ptr(), y.data_ptr(), ids.data_ptr(), wts.data_ptr(), 7, S()))
    torch.cuda.synchronize()
    all_ids = torch.zeros(world, K, dtype=torch.int64, device=dev); dist.all_gather_into_tensor(all_ids, ids)
    t = trace.cpu().numpy().reshape(n_sm, 16)[:, :11].astype(np.float64)
    t -= t[:, 0].min()
    if rep >= 4:
        acc.append(t)
        pairs.append(int(((all_ids >= rank * El) & (all_ids < (rank + 1) * El)).sum()))
lib.ktb200_debug_block_trace(None)
assert not ex.timed_out()
t = np.mean(acc, axis=0) / 1e3
out = [f"rank {rank}/{world}: owned pairs per layer {pairs} (mean {np.mean(pairs):.1f})",
       f"{'boundary':44s} {'first':>8s} {'median':>8s} {'last':>8s}   (us after this rank's first CTA started; mean of {len(acc)} launches)"]
for i in range(len(names)):
    if names[i] != "-":
        out.append(f"{names[i]:44s} {t[:, i].min():8.2f} {np.median(t[:, i]):8.2f} {t[:, i].max():8.2f}")
for r in range(world):
    dist.barrier()
    if r == rank and (rank < 2 or rank == world - 1):
        print("\n".join(out), flush=True)
dist.barrier()
torch.cuda.synchronize()
os._exit(0)
