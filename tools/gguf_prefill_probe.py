"""Times the routes of the GGUF dense linear at DeepSeek-V3's Q4_K / Q6_K module shapes and prompt sizes, to place the prompt
threshold (csrc/gguf_gemm.cu gguf_prompt_min, DESIGN.md §4.17):
  gemv    ktb200_linear_forward with T tokens: the decode GEMVs (one weight pass per token chunk of at most 8, one token at
          in_features 16384 / 18432; Q6_K tokens in grid.y);
  gemm    ktb200_linear_forward_prompt with T tokens: the quantiser and gguf_gemm_kernel per chunk of at most 2048, below the
          threshold too;
  torch   at 1024 and 4096 tokens, torch.matmul of the bf16 activations by a bf16 weight of the same shape: KLinearTorch's work
          on its dequantised copy, without the cost of building that copy.
CUDA events; the routes alternate in every round; median and spread (max - min) over the rounds.  TOPS count 2 T K N over the
call time (the quantiser included); the share is of the H100 SXM data-sheet dense INT8 rate (1,979 TOPS).  The card's name
and power limit are read (read-only nvidia-smi query) in the same run.
    python tools/gguf_prefill_probe.py [--rounds 5] [--json out.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ktransformers_b200 import native  # noqa: E402
from ktransformers_b200.util.synth import synth_blocks  # noqa: E402

Q4_K, Q6_K, BF16 = 12, 14, 30
SHAPES = [("q_a", Q4_K, 7168, 1536), ("kv_a", Q4_K, 7168, 576), ("q_b", Q4_K, 1536, 24576), ("o_proj", Q4_K, 16384, 7168),
          ("dense gate/up", Q4_K, 7168, 18432), ("dense down", Q6_K, 18432, 7168), ("shared gate/up", Q4_K, 7168, 2048),
          ("shared down", Q6_K, 2048, 7168), ("lm_head", Q6_K, 7168, 129280)]
TS = [8, 16, 24, 32, 48, 64, 96, 128, 256, 1024, 4096]
TORCH_TS = (1024, 4096)
PEAK = 1979e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window-ms", type=float, default=3.0, help="least time per timed sample (calls are repeated inside it)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "the probe times the GPU"
    lib = native.lib()
    s = torch.cuda.current_stream().cuda_stream
    dev = card()
    print(f"card: {dev}", flush=True)
    rows = []
    for name, t, K, N in SHAPES:
        w = synth_blocks(t, N * K, device="cuda", seed=K + N)
        h = C.c_void_p()
        native.check(lib.ktb200_linear_create(K, N, w.data_ptr(), t, BF16, 1024, torch.cuda.current_device(), C.byref(h)))
        native.check(lib.ktb200_linear_load_weights(h, s))
        pm = lib.ktb200_linear_prompt_min(h)
        g = torch.Generator(device="cuda").manual_seed(K + N)
        x = (torch.randn(max(TS), K, device="cuda", generator=g) / 10).bfloat16()
        y = torch.empty(max(TS), N, dtype=torch.bfloat16, device="cuda")
        wd = torch.randn(N, K, device="cuda", generator=g).bfloat16()

        def gemv(T):
            native.check(lib.ktb200_linear_forward(h, T, x.data_ptr(), y.data_ptr(), None, None, s))

        def gemm(T):
            native.check(lib.ktb200_linear_forward_prompt(h, T, x.data_ptr(), y.data_ptr(), None, None, s))

        def mm(T):
            torch.matmul(x[:T], wd.T, out=y[:T])

        for T in TS:
            fns = (gemv, gemm, mm) if T in TORCH_TS else (gemv, gemm)
            reps = {}
            for fn in fns:   # warm-up (arena growth, module load), then the repeat count for a window of window_ms
                fn(T)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
                e0.record(); fn(T); e1.record(); torch.cuda.synchronize()
                reps[fn] = max(1, int(args.window_ms / max(e0.elapsed_time(e1), 1e-3)) + 1)
            ms = {fn: [] for fn in fns}
            for r in range(args.rounds):
                for fn in (fns if r % 2 == 0 else fns[::-1]):
                    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
                    e0.record()
                    for _ in range(reps[fn]):
                        fn(T)
                    e1.record(); torch.cuda.synchronize()
                    ms[fn].append(e0.elapsed_time(e1) / reps[fn])
            med = {fn: sorted(v)[len(v) // 2] for fn, v in ms.items()}
            spr = {fn: max(v) - min(v) for fn, v in ms.items()}
            picked, other = (gemm, gemv) if pm and T >= pm else (gemv, gemm)
            ok = med[picked] <= med[other] + max(spr[picked], spr[other])
            ops = 2.0 * T * K * N
            row = dict(module=name, type="Q4_K" if t == Q4_K else "Q6_K", K=K, N=N, T=T, prompt_min=pm, gemv_ms=med[gemv], gemv_spread_ms=spr[gemv],
                       gemm_ms=med[gemm], gemm_spread_ms=spr[gemm], route="gemm" if picked is gemm else "gemv", picked_not_slower=ok,
                       gemv_tops=ops / med[gemv] / 1e9, gemm_tops=ops / med[gemm] / 1e9)
            line = (f"{name:15s} {row['type']} {K:6d}->{N:6d} T={T:5d}  gemv {med[gemv]:9.3f} ms ±{spr[gemv]:.3f} {row['gemv_tops']:6.1f} TOPS"
                    f"   gemm {med[gemm]:8.3f} ms ±{spr[gemm]:.3f} {row['gemm_tops']:6.1f} TOPS ({row['gemm_tops'] * 1e12 / PEAK:5.1%})")
            if mm in med:
                row.update(torch_ms=med[mm], torch_spread_ms=spr[mm], torch_tflops=ops / med[mm] / 1e9)
                line += f"   torch bf16 {med[mm]:8.3f} ms ±{spr[mm]:.3f}"
            rows.append(row)
            # 'floor': calls of fewer than 16 tokens keep the GEMV whatever the shape
            print(line + f"   picks {row['route']:4s} {'ok' if ok else 'floor' if T < 16 else 'SLOWER'}", flush=True)
        lib.ktb200_linear_destroy(h)
        del w, x, y, wd
        torch.cuda.empty_cache()
    print("shares are of 1,979 TOPS (data-sheet dense INT8 of an H100 SXM at 700 W)")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": dev, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
