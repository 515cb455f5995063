"""Times the two routes of ktb200_fp8_linear_forward at DeepSeek-V3's FP8 module shapes and prompt sizes, to place the route
threshold (csrc/fp8_linear.cu fp8_prompt_route, DESIGN.md §4.6):
  decode  the entry called in 16-token slices: every slice is below the threshold, so this is exactly what the decode route
          does with a prompt (one weight pass and two launches per 16 tokens);
  gemm    one call of T tokens through fp8_gemm_kernel.  Below the threshold a single call would take the decode route, so
          there the GEMM is timed as a call at the threshold with a device batch size of T: token tiles beyond T exit at once,
          and the live tile costs what it costs at T (a token tile is 128 wide either way).
CUDA events; the two routes alternate in every round; median and spread (max - min) over the rounds.  Achieved TFLOP/s count
2 T K N over the call time; the share is of the H100 SXM data-sheet dense fp16 rate (989 TFLOP/s) — the bound at these sizes is
compute.  The card's name and power limit are read (read-only nvidia-smi query) in the same run.
    python tools/fp8_prefill_probe.py [--rounds 5] [--json out.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ktransformers_b200 import native  # noqa: E402

SHAPES = [("q_a", 7168, 1536), ("kv_a", 7168, 576), ("q_b", 1536, 24576), ("o_proj", 16384, 7168),
          ("dense gate/up", 7168, 18432), ("dense down", 18432, 7168), ("shared gate/up", 7168, 2048), ("shared down", 2048, 7168)]
TS = [16, 24, 32, 48, 64, 96, 128, 256, 1024, 4096]
# one MoE layer's seven FP8 linears: q_a, kv_a, q_b, o_proj, the shared expert's gate, up and down
LAYER = {"q_a": 1, "kv_a": 1, "q_b": 1, "o_proj": 1, "shared gate/up": 2, "shared down": 1}
PEAK = 989e12
BF16 = 30


def prompt_min(N, K):
    """restates fp8_prompt_min (csrc/fp8_linear.cu): the smallest qlen that takes the GEMM route"""
    return 96 if N <= 2048 else 48 if K >= 16384 else 32


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
    for name, K, N in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(K + N)
        w = (torch.randn(N, K, device="cuda", generator=g) * 0.5).to(torch.float8_e4m3fn).view(torch.uint8)
        ws = torch.rand(((N + 127) // 128, K // 128), device="cuda", generator=g) * 0.01 + 0.001
        h = C.c_void_p()
        native.check(lib.ktb200_fp8_linear_create(K, N, w.data_ptr(), ws.data_ptr(), BF16, 0, C.byref(h)))
        Tmax = max(max(TS), prompt_min(N, K))
        x = (torch.randn(Tmax, K, device="cuda", generator=g) / 10).bfloat16()
        y = torch.zeros(Tmax, N, dtype=torch.bfloat16, device="cuda")
        bsz = torch.zeros(1, dtype=torch.int32, device="cuda")
        xb, yb = x.element_size() * K, y.element_size() * N

        def decode(T):
            for t0 in range(0, T, 16):
                native.check(lib.ktb200_fp8_linear_forward(h, min(16, T - t0), x.data_ptr() + t0 * xb, y.data_ptr() + t0 * yb, None, s))

        def gemm(T):
            q = max(T, prompt_min(N, K))
            native.check(lib.ktb200_fp8_linear_forward(h, q, x.data_ptr(), y.data_ptr(), bsz.data_ptr() if q > T else None, s))

        for T in TS:
            bsz.fill_(T)
            reps = {}
            for fn in (decode, gemm):   # warm-up (arena growth, module load), then the repeat count for a window of window_ms
                fn(T)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
                e0.record(); fn(T); e1.record(); torch.cuda.synchronize()
                reps[fn] = max(1, int(args.window_ms / max(e0.elapsed_time(e1), 1e-3)) + 1)
            ms = {decode: [], gemm: []}
            for r in range(args.rounds):
                for fn in ((decode, gemm) if r % 2 == 0 else (gemm, decode)):
                    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
                    e0.record()
                    for _ in range(reps[fn]):
                        fn(T)
                    e1.record(); torch.cuda.synchronize()
                    ms[fn].append(e0.elapsed_time(e1) / reps[fn])
            med = {fn: sorted(v)[len(v) // 2] for fn, v in ms.items()}
            spr = {fn: max(v) - min(v) for fn, v in ms.items()}
            picked, other = (gemm, decode) if T >= prompt_min(N, K) else (decode, gemm)
            ok = med[picked] <= med[other] + max(spr[picked], spr[other])
            fl = 2.0 * T * K * N
            row = dict(module=name, K=K, N=N, T=T, decode_ms=med[decode], decode_spread_ms=spr[decode], gemm_ms=med[gemm],
                       gemm_spread_ms=spr[gemm], route="gemm" if picked is gemm else "decode", picked_not_slower=ok,
                       decode_tflops=fl / med[decode] / 1e9, gemm_tflops=fl / med[gemm] / 1e9)
            rows.append(row)   # 'floor': below 32 tokens the decode route is kept whatever the shape
            print(f"{name:15s} {K:6d}->{N:6d} T={T:5d}  decode {med[decode]:8.3f} ms ±{spr[decode]:.3f} {row['decode_tflops']:6.1f} TF/s"
                  f" ({row['decode_tflops'] * 1e12 / PEAK:5.1%})   gemm {med[gemm]:8.3f} ms ±{spr[gemm]:.3f} {row['gemm_tflops']:6.1f} TF/s"
                  f" ({row['gemm_tflops'] * 1e12 / PEAK:5.1%})   picks {row['route']:6s} {'ok' if ok else 'floor' if T < 32 else 'SLOWER'}", flush=True)
        lib.ktb200_fp8_linear_destroy(h)
        del w, ws, x, y
        torch.cuda.empty_cache()
    for route in ("decode", "gemm"):
        tot = sum(LAYER[r["module"]] * r[f"{route}_ms"] for r in rows if r["T"] == 4096 and r["module"] in LAYER)
        print(f"one MoE layer's seven FP8 linears at 4096 tokens, {route} route: {tot:.2f} ms")
    print("shares are of 989 TFLOP/s (data-sheet dense fp16 of an H100 SXM at 700 W): the bound at these sizes is compute")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"card": dev, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
