"""Times the multi-token expert-parallel MoE layer at world 1 against the single-GPU layer, DeepSeek-V3 shapes
(E 256, H 7168, I 2048, top-k 8, n_group 8, topk_group 4; Q4_K gate/up, Q6_K down; a Q4_K/Q4_K/Q6_K shared expert; bf16).

For T = 1, 8, 64, 512, 1024 tokens, CUDA events over ITERS calls after warm-up:
  - single:  ktb200_moe_gate_forward + ktb200_moe_forward_shared (the fused shared slot where it applies);
  - ep_w1:   ktb200_moe_ep_forward_tokens, phase 7, world 1 (route + send, experts with fp32 output + deliver, shared
             expert + combine): the exchange's cost on top of the experts, with no peer to wait for;
  - and the largest |difference| between the two outputs (0 when the shared expert is not fused: both are the two rounded
    terms of the same kernels).
The NVLink rate of the send and deliver kernels needs two or more GPUs and is not measured here.
Prints the card name and power limit (read-only nvidia-smi query) and one JSON line.

    python tools/ep_tokens_probe.py [--out FILE]
"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ktransformers_b200 import native  # noqa: E402
from ktransformers_b200.util.synth import synth_blocks  # noqa: E402

E, H, I, K, NG, TG = 256, 7168, 2048, 8, 8, 4
Q4_K, Q6_K, BF16 = 12, 14, 30
TOKENS = [1, 8, 64, 512, 1024]
ITERS = int(os.environ.get("ITERS", 20))


def timed(fn, iters=ITERS, warm=3):
    for _ in range(warm):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    lib, dev = native.lib(), torch.cuda.current_device()
    s = torch.cuda.current_stream().cuda_stream
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[dev]
    Tmax = max(TOKENS)
    gate_w, up_w = synth_blocks(Q4_K, E * I * H, "cuda", 1), synth_blocks(Q4_K, E * I * H, "cuda", 2)
    down_w = synth_blocks(Q6_K, E * H * I, "cuda", 3)
    sg, su, sd = synth_blocks(Q4_K, I * H, "cuda", 4), synth_blocks(Q4_K, I * H, "cuda", 5), synth_blocks(Q6_K, H * I, "cuda", 6)
    cfg = native.MoeConfig(E, K, H, I, 64, 10, Tmax, 1, gate_w.data_ptr(), up_w.data_ptr(), down_w.data_ptr(), Q4_K, Q4_K, Q6_K, BF16, 0)
    moe, mlp = C.c_void_p(), C.c_void_p()
    native.check(lib.ktb200_moe_create(C.byref(cfg), dev, C.byref(moe)))
    native.check(lib.ktb200_moe_load_weights(moe, s))
    native.check(lib.ktb200_mlp_create(H, I, sg.data_ptr(), su.data_ptr(), sd.data_ptr(), Q4_K, Q4_K, Q6_K, BF16, Tmax, dev, C.byref(mlp)))
    native.check(lib.ktb200_mlp_load_weights(mlp, s))
    rng = np.random.default_rng(0)
    Wr = torch.from_numpy(rng.standard_normal((E, H)).astype(np.float32)).cuda()
    bias = torch.from_numpy((rng.standard_normal(E) / 100).astype(np.float32)).cuda()
    gate = native.GateConfig(E, H, K, NG, TG, 0, 0, 1, 2.5, Wr.data_ptr(), bias.data_ptr(), BF16)
    nbytes, off = native.ep_tokens_layout(1, Tmax, H, BF16, K)
    region = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    comm = native.EpTokensComm.make(0, 1, Tmax, H, BF16, K, [region.data_ptr()])
    rows = []
    for T in TOKENS:
        x = (torch.randn(T, H, device="cuda") / 10).to(torch.bfloat16)
        idx = torch.zeros((T, K), dtype=torch.int64, device="cuda")
        w = torch.zeros((T, K), dtype=torch.float32, device="cuda")
        y1, y2 = torch.zeros_like(x), torch.zeros_like(x)
        counts = (C.c_int * 1)(T)

        def single():
            native.check(lib.ktb200_moe_gate_forward(C.byref(gate), T, x.data_ptr(), idx.data_ptr(), w.data_ptr(), None, None, s))
            native.check(lib.ktb200_moe_forward_shared(moe, mlp, T, K, idx.data_ptr(), w.data_ptr(), x.data_ptr(), y1.data_ptr(), None, s))

        def ep_w1():
            native.check(lib.ktb200_moe_ep_forward_tokens(C.byref(gate), moe, mlp, C.byref(comm), counts, x.data_ptr(), y2.data_ptr(),
                                                          idx.data_ptr(), w.data_ptr(), 7, s))
        t_single, t_ep = timed(single), timed(ep_w1)
        single(); ep_w1()
        torch.cuda.synchronize()
        status = int(region[off["flags"]:].view(torch.int32)[2 + 2])
        rows.append({"T": T, "single_ms": round(t_single, 4), "ep_world1_ms": round(t_ep, 4),
                     "overhead_ms": round(t_ep - t_single, 4), "ratio": round(t_ep / t_single, 3),
                     "max_abs_diff": float((y1.float() - y2.float()).abs().max()), "status": status})
        print(rows[-1], flush=True)
    res = {"probe": "ep_tokens world 1 vs single-GPU layer", "card": card, "shapes": dict(E=E, H=H, I=I, k=K), "rows": rows,
           "nvlink": "not measured (needs two or more GPUs)"}
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    lib.ktb200_moe_destroy(moe)
    lib.ktb200_mlp_destroy(mlp)


if __name__ == "__main__":
    main()
