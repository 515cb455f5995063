"""Times causal MLA prefill at DeepSeek-V3 shapes (H = 128 heads, q_lora_rank 1536, hidden 7168), one sequence.

For each (P, q_len) chunk (P tokens already cached):
  - kernel: ktb200_mla_prefill alone, CUDA events over ITERS launches after warm-up;
  - decompress: kv_b_proj (dense bf16, 512 -> 128 x 256) over the S = P + q_len cached latents;
  - operator: KDeepseekV2Attention.forward for the chunk (projections, RoPE, cache write, decompression, kernel, o_proj);
  - the causal FLOP count 2 H (192 + 128) sum_i (P + i + 1), the kernel's TFLOP/s and its share of the 989 TFLOP/s bf16
    dense data-sheet rate of the H100 SXM (a bound from shapes; a card with a lower power limit clocks lower);
  - at P = 0, torch's scaled_dot_product_attention (causal, k = k_nope | k_pe expanded per head, v padded to 192 as the
    reference pads for flash_attn_func) on the same inputs: its time and the largest difference from the kernel's output.
Prints the card name and power limit (read-only nvidia-smi query) and one JSON line.

    python tools/mla_prefill_probe.py [--out FILE]
"""
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ktransformers_b200 import native  # noqa: E402

H = 128
CHUNKS = [(0, 1024), (0, 4096), (3072, 1024)]
ITERS = int(os.environ.get("ITERS", 50))
PEAK_TFLOPS = 989.0
SCALE = (128 + 64) ** -0.5


def timed(fn, iters=ITERS, warm=5):
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


def causal_flops(past, q_len):
    return 2 * H * (192 + 128) * sum(past + i + 1 for i in range(q_len))


def main():
    from ktransformers_b200.models.custom_cache import StaticCache
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Attention, DeepseekV3Config
    from ktransformers_b200.operators.attention import KDeepseekV2Attention
    assert torch.cuda.is_available(), "the probe measures on the GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print("card:", card)
    torch.manual_seed(0)
    cfg = DeepseekV3Config(num_hidden_layers=1)   # V3 shapes
    plain = DeepseekV3Attention(cfg, layer_idx=0).to(device="cuda", dtype=torch.bfloat16)
    op = KDeepseekV2Attention("blk.0.self_attn", None, cfg, plain, "cuda", "cuda")
    lib, stream = native.lib(), lambda: torch.cuda.current_stream().cuda_stream
    rows = []
    for past, q_len in CHUNKS:
        S = past + q_len
        q = (torch.randn(1, q_len, H, 192, device="cuda")).to(torch.bfloat16)
        q_pe = (torch.randn(1, q_len, H, 64, device="cuda")).to(torch.bfloat16)
        lat = (torch.randn(1, S, 576, device="cuda")).to(torch.bfloat16)
        kv = plain.kv_b_proj(lat[..., :512]).view(1, S, H, 256)
        out = torch.empty(1, q_len, H, 128, dtype=torch.bfloat16, device="cuda")
        qn, kn, v, kp = q[..., :128], kv[..., :128], kv[..., 128:], lat[..., 512:]
        p = native.MlaPrefillParams(1, q_len, S, H, 128, 64, 128, SCALE, qn.data_ptr(), qn.stride(1), qn.stride(2), qn.stride(0),
                                    q_pe.data_ptr(), q_pe.stride(1), q_pe.stride(2), q_pe.stride(0),
                                    kn.data_ptr(), kn.stride(1), kn.stride(2), kn.stride(0), v.data_ptr(), v.stride(1), v.stride(2), v.stride(0),
                                    kp.data_ptr(), kp.stride(1), kp.stride(0), out.data_ptr())
        kernel_ms = timed(lambda: native.check(lib.ktb200_mla_prefill(C.byref(p), stream())))
        decompress_ms = timed(lambda: plain.kv_b_proj(lat[..., :512]))
        # the operator on a cache that already holds P tokens: the host counter is rewound before each call
        cache = StaticCache(cfg, max_batch_size=1, max_cache_len=S, device="cuda")
        x = (torch.randn(1, S, cfg.hidden_size, device="cuda") * 0.5).to(torch.bfloat16)
        pos = torch.arange(S, device="cuda")
        if past:
            op(x[:, :past], position_ids=pos[None, :past], past_key_value=cache, cache_position=pos[:past])

        def chunk():
            cache.past_tokens[0] = past
            op(x[:, past:], position_ids=pos[None, past:], past_key_value=cache, cache_position=pos[past:])
        operator_ms = timed(chunk, iters=max(5, ITERS // 5))
        fl = causal_flops(past, q_len)
        r = {"P": past, "q_len": q_len, "kernel_ms": round(kernel_ms, 4), "decompress_ms": round(decompress_ms, 4),
             "operator_ms": round(operator_ms, 4), "tflop": round(fl / 1e12, 4), "kernel_tflops": round(fl / kernel_ms / 1e9, 1),
             "bound_ms_at_989": round(fl / PEAK_TFLOPS / 1e9, 4), "share_of_bound": round(fl / PEAK_TFLOPS / 1e9 / kernel_ms, 3)}
        if past == 0:
            import torch.nn.functional as F
            qs = torch.cat([q[..., :128], q_pe], -1).transpose(1, 2)
            ks = torch.cat([kn, kp[:, :, None].expand(1, S, H, 64)], -1).transpose(1, 2)
            vs = torch.nn.functional.pad(v, (0, 64)).transpose(1, 2)
            sdpa = lambda: F.scaled_dot_product_attention(qs, ks, vs, is_causal=True, scale=SCALE)
            r["sdpa_ms"] = round(timed(sdpa), 4)
            ref = sdpa()[..., :128].transpose(1, 2).float()
            native.check(lib.ktb200_mla_prefill(C.byref(p), stream()))
            torch.cuda.synchronize()
            r["max_abs_diff_vs_sdpa"] = float((out.float() - ref).abs().max())
            r["max_abs_sdpa"] = float(ref.abs().max())
        print(r)
        rows.append(r)
    res = {"card": card, "heads": H, "iters": ITERS, "chunks": rows}
    line = json.dumps(res)
    print(line)
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
