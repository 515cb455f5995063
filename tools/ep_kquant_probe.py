"""Times one-token expert-parallel decode of Q2_K / Q3_K experts at world 1, DeepSeek-V3 shapes (E 256, H 7168, I 2048, top-k 8,
n_group 8, topk_group 4; a Q4_K/Q4_K/Q6_K shared expert; bf16), for the Q2_K file's Q2_K/Q2_K/Q3_K and the Q3_K_M file's
Q3_K/Q3_K/Q4_K experts.  Three paths, alternated in ROUNDS rounds of CUDA events over ITERS calls after warm-up (median):
  - ep_block:   ktb200_moe_ep_block_forward, phase 7: the shared expert's ktb200_mlp_forward, then moe_ep_block_kernel<GU, D>;
  - ep_tokens:  ktb200_moe_ep_forward_tokens with counts [1], phase 7 (the fallback the one-launch kernel replaces);
  - unsharded:  ktb200_moe_block_forward on the same handles (gate, then the per-pair kernels: separate launches).
Achieved bytes/s are over the algorithmic bytes: the router's fp32 weight, the gate/up/down rows of the distinct selected
experts and the shared expert's tensors.  The exchange over NVLink needs two or more GPUs and is not measured here.
Prints the card name and power limit (read-only nvidia-smi query) and one JSON line.

    python tools/ep_kquant_probe.py [--out FILE]
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
Q2_K, Q3_K, Q4_K, Q6_K, BF16 = 10, 11, 12, 14, 30
BLOCK_BYTES = {Q2_K: 84, Q3_K: 110, Q4_K: 144, Q6_K: 210}
SETS = [(Q2_K, Q2_K, Q3_K), (Q3_K, Q3_K, Q4_K)]
NAMES = {Q2_K: "Q2_K", Q3_K: "Q3_K", Q4_K: "Q4_K", Q6_K: "Q6_K"}
ITERS = int(os.environ.get("ITERS", 50))
ROUNDS = int(os.environ.get("ROUNDS", 5))


def timed(fn, iters=ITERS):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def tensor_bytes(t, rows, cols):
    return rows * cols // 256 * BLOCK_BYTES[t]


def main():
    out_path = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    lib, dev = native.lib(), torch.cuda.current_device()
    s = torch.cuda.current_stream().cuda_stream
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[dev]
    sg, su, sd = synth_blocks(Q4_K, I * H, "cuda", 4), synth_blocks(Q4_K, I * H, "cuda", 5), synth_blocks(Q6_K, H * I, "cuda", 6)
    mlp = C.c_void_p()
    native.check(lib.ktb200_mlp_create(H, I, sg.data_ptr(), su.data_ptr(), sd.data_ptr(), Q4_K, Q4_K, Q6_K, BF16, 8, dev, C.byref(mlp)))
    native.check(lib.ktb200_mlp_load_weights(mlp, s))
    rng = np.random.default_rng(0)
    Wr = torch.from_numpy(rng.standard_normal((E, H)).astype(np.float32)).cuda()
    bias = torch.from_numpy((rng.standard_normal(E) / 100).astype(np.float32)).cuda()
    gate = native.GateConfig(E, H, K, NG, TG, 0, 0, 1, 2.5, Wr.data_ptr(), bias.data_ptr(), BF16)
    # one-token kernel buffers (message, partial, flags) and the multi-token region, world 1
    msg = torch.zeros(lib.ktb200_ep_msg_bytes(H, BF16), dtype=torch.uint8, device="cuda")
    part = torch.zeros((1, H), dtype=torch.float32, device="cuda")
    flags = torch.zeros(4, dtype=torch.int32, device="cuda")
    comm = native.EpComm.make(0, 1, H, BF16, [msg.data_ptr()], [part.data_ptr()], [flags.data_ptr()])
    nbytes, off = native.ep_tokens_layout(1, 8, H, BF16, K)
    region = torch.zeros(nbytes, dtype=torch.uint8, device="cuda")
    tok_comm = native.EpTokensComm.make(0, 1, 8, H, BF16, K, [region.data_ptr()])
    counts = (C.c_int * 1)(1)
    rows = []
    for gt, ut, dt in SETS:
        gate_w, up_w, down_w = (synth_blocks(gt, E * I * H, "cuda", 1), synth_blocks(ut, E * I * H, "cuda", 2),
                                synth_blocks(dt, E * H * I, "cuda", 3))
        cfg = native.MoeConfig(E, K, H, I, 64, 10, 8, 1, gate_w.data_ptr(), up_w.data_ptr(), down_w.data_ptr(), gt, ut, dt, BF16, 0)
        moe = C.c_void_p()
        native.check(lib.ktb200_moe_create(C.byref(cfg), dev, C.byref(moe)))
        native.check(lib.ktb200_moe_load_weights(moe, s))
        x = (torch.randn(1, H, device="cuda") / 10).to(torch.bfloat16)
        idx = torch.zeros((1, K), dtype=torch.int64, device="cuda")
        w = torch.zeros((1, K), dtype=torch.float32, device="cuda")
        ys = {n: torch.zeros_like(x) for n in ("ep_block", "ep_tokens", "unsharded")}
        paths = {
            "ep_block": lambda: native.check(lib.ktb200_moe_ep_block_forward(C.byref(gate), moe, mlp, C.byref(comm), x.data_ptr(),
                                                                             ys["ep_block"].data_ptr(), idx.data_ptr(), w.data_ptr(), 7, s)),
            "ep_tokens": lambda: native.check(lib.ktb200_moe_ep_forward_tokens(C.byref(gate), moe, mlp, C.byref(tok_comm), counts,
                                                                               x.data_ptr(), ys["ep_tokens"].data_ptr(), idx.data_ptr(),
                                                                               w.data_ptr(), 7, s)),
            "unsharded": lambda: native.check(lib.ktb200_moe_block_forward(C.byref(gate), moe, mlp, 1, x.data_ptr(), ys["unsharded"].data_ptr(),
                                                                           idx.data_ptr(), w.data_ptr(), None, s)),
        }
        for fn in paths.values():   # warm-up: attributes, first launches
            for _ in range(3):
                fn()
        times = {n: [] for n in paths}
        for _ in range(ROUNDS):
            for n, fn in paths.items():
                times[n].append(timed(fn))
        med = {n: float(np.median(v)) for n, v in times.items()}
        for fn in paths.values():
            fn()
        torch.cuda.synchronize()
        n_exp = len(set(idx[0].tolist()))
        algo = (E * H * 4 + n_exp * (tensor_bytes(gt, I, H) + tensor_bytes(ut, I, H) + tensor_bytes(dt, H, I)) +
                tensor_bytes(Q4_K, I, H) * 2 + tensor_bytes(Q6_K, H, I) + 2 * H * 2)
        row = {"set": "/".join(NAMES[t] for t in (gt, ut, dt)), "distinct_experts": n_exp, "algorithmic_bytes": algo}
        for n in paths:
            row[f"{n}_ms"] = round(med[n], 4)
            row[f"{n}_spread_ms"] = round(float(max(times[n]) - min(times[n])), 4)
            row[f"{n}_GBps"] = round(algo / med[n] / 1e6, 1)
        row["ep_block_vs_ep_tokens_ms"] = round(med["ep_block"] - med["ep_tokens"], 4)
        row["ep_block_equals_ep_tokens"] = bool(torch.equal(ys["ep_block"], ys["ep_tokens"]))
        row["status"] = [int(flags[3]), int(region[off["flags"]:].view(torch.int32)[4])]
        rows.append(row)
        print(row, flush=True)
        lib.ktb200_moe_destroy(moe)
        del gate_w, up_w, down_w
    res = {"probe": "Q2_K / Q3_K expert-parallel decode, world 1", "card": card, "shapes": dict(E=E, H=H, I=I, k=K),
           "iters": ITERS, "rounds": ROUNDS, "rows": rows, "nvlink": "not measured (needs two or more GPUs)"}
    print(json.dumps(res))
    if out_path:
        with open(out_path, "w") as f:
            json.dump(res, f, indent=1)
    lib.ktb200_mlp_destroy(mlp)


if __name__ == "__main__":
    main()
