"""Times the two prompt-chunk attention paths of KDeepseekV2Attention at DeepSeek-V3 shapes (H = 128 heads), one sequence
with P tokens already cached and a chunk of q_len new ones:

  - absorbed (absorb_for_prefill): ktb200_mla_absorb_q + ktb200_mla_decode_chunk over the paged latent cache + ktb200_mla_absorb_o;
  - non-absorbed (the default): kv_b_proj (dense bf16, 512 -> 128 x 256) over the S = P + q_len cached latents, then
    ktb200_mla_prefill; its peak extra allocation (the decompressed S x 128 x 256 buffer) is reported too.

Both produce the [q_len, 128, 128] per-head attention output that o_proj reads.  CUDA events over ITERS calls (at least
~50 ms of work per window) after warm-up; the two paths alternate over ROUNDS rounds and the median window is kept.
Non-absorbed cases whose buffer does not fit in free memory are skipped.  Prints the card name and power limit (read-only
nvidia-smi query), one line per case and one JSON line.

    python tools/mla_chunk_probe.py [--out FILE]     (QLENS / PASTS / ROUNDS: comma lists / count in the environment)
"""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ktransformers_b200 import native  # noqa: E402

H, PAGE = 128, 64
QLENS = [int(x) for x in os.environ.get("QLENS", "1,2,4,8,16,64,128,256,1024").split(",")]
PASTS = [int(x) for x in os.environ.get("PASTS", "0,4096,32768,131072").split(",")]
ROUNDS = int(os.environ.get("ROUNDS", 3))
SCALE = (128 + 64) ** -0.5


def window(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def iters_for(fn):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    t = window(fn, 1)
    return max(1, min(200, int(50.0 / max(t, 1e-3))))


def main():
    assert torch.cuda.is_available(), "the probe measures on the GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print("card:", card)
    lib, stream = native.lib(), lambda: torch.cuda.current_stream().cuda_stream
    g = torch.Generator(device="cuda").manual_seed(0)
    rnd = lambda *s, scale=1.0: (torch.randn(*s, generator=g, device="cuda") * scale).to(torch.bfloat16)
    w_kvb = rnd(H * 256, 512, scale=512 ** -0.5)                       # kv_b_proj weight: per head 128 rows W_UK, 128 rows W_UV
    w_uk = w_kvb.view(H, 256, 512)[:, :128].contiguous()
    w_uv = w_kvb.view(H, 256, 512)[:, 128:].contiguous()
    max_S = max(PASTS) + max(QLENS)
    pages = -(-max_S // PAGE)
    cache = rnd(pages, PAGE, 576)
    pt = torch.arange(pages, dtype=torch.int32, device="cuda").view(1, pages)
    rows = []
    for past in PASTS:
        for q_len in QLENS:
            S = past + q_len
            q = rnd(1, q_len, H, 192)
            q_pe = rnd(1, q_len, H, 64)
            kl = torch.tensor([S], dtype=torch.int32, device="cuda")
            q_abs = torch.empty(q_len, H, 512, dtype=torch.bfloat16, device="cuda")
            lat = torch.empty(q_len, H, 512, dtype=torch.bfloat16, device="cuda")
            o_abs = torch.empty(q_len, H, 128, dtype=torch.bfloat16, device="cuda")
            splits = min(128, -(-torch.cuda.get_device_properties(0).multi_processor_count // (q_len * 2)))
            ws_bytes = lib.ktb200_mla_chunk_workspace_bytes(1, q_len, H, splits)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
            cp = native.MlaChunkParams(1, q_len, H, PAGE, pages, 0, SCALE, q_abs.data_ptr(), q_pe.data_ptr(), cache.data_ptr(),
                                       pt.data_ptr(), kl.data_ptr(), lat.data_ptr(), None, ws.data_ptr(), ws_bytes, pages * PAGE)

            def absorbed():
                native.check(lib.ktb200_mla_absorb_q(q.data_ptr(), 192, H * 192, w_uk.data_ptr(), H, 128, 512, q_abs.data_ptr(), q_len, stream()))
                native.check(lib.ktb200_mla_decode_chunk(C.byref(cp), stream()))
                native.check(lib.ktb200_mla_absorb_o(lat.data_ptr(), w_uv.data_ptr(), H, 128, 512, o_abs.data_ptr(), q_len, stream()))

            rows_lat = cache.view(1, -1, 576)[:, :S]
            o_pre = torch.empty(1, q_len, H, 128, dtype=torch.bfloat16, device="cuda")
            qn = q[..., :128]
            kp = rows_lat[..., 512:]

            def non_absorbed():
                kv = torch.nn.functional.linear(rows_lat[..., :512], w_kvb).view(1, S, H, 256)
                kn, v = kv[..., :128], kv[..., 128:]
                p = native.MlaPrefillParams(1, q_len, S, H, 128, 64, 128, SCALE, qn.data_ptr(), qn.stride(1), qn.stride(2), qn.stride(0),
                                            q_pe.data_ptr(), q_pe.stride(1), q_pe.stride(2), q_pe.stride(0),
                                            kn.data_ptr(), kn.stride(1), kn.stride(2), kn.stride(0), v.data_ptr(), v.stride(1), v.stride(2), v.stride(0),
                                            kp.data_ptr(), kp.stride(1), kp.stride(0), o_pre.data_ptr())
                native.check(lib.ktb200_mla_prefill(C.byref(p), stream()))

            buf = S * H * 256 * 2
            fits = buf < 0.7 * torch.cuda.mem_get_info()[0]
            r = {"P": past, "q_len": q_len, "splits_bound": splits}
            ia = iters_for(absorbed)
            if fits:
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                non_absorbed()
                torch.cuda.synchronize()
                r["non_absorbed_peak_bytes"] = torch.cuda.max_memory_allocated() - base
                ib = iters_for(non_absorbed)
                r["max_abs_diff"] = float((o_abs.float() - o_pre[0].float()).abs().max())   # the two paths round differently
                r["max_abs"] = float(o_pre.float().abs().max())
            ta, tb = [], []
            for _ in range(ROUNDS):
                ta.append(window(absorbed, ia))
                if fits:
                    tb.append(window(non_absorbed, ib))
            r["absorbed_ms"] = round(statistics.median(ta), 4)
            r["absorbed_spread"] = round((max(ta) - min(ta)) / statistics.median(ta), 3)
            if fits:
                r["non_absorbed_ms"] = round(statistics.median(tb), 4)
                r["non_absorbed_spread"] = round((max(tb) - min(tb)) / statistics.median(tb), 3)
                r["absorbed_over_non_absorbed"] = round(r["absorbed_ms"] / r["non_absorbed_ms"], 3)
            else:
                r["non_absorbed"] = f"skipped: a {buf / 2**30:.1f} GiB buffer does not fit"
            print(r, flush=True)
            rows.append(r)
            del ws
            torch.cuda.empty_cache()
    res = {"card": card, "heads": H, "rounds": ROUNDS, "cases": rows}
    line = json.dumps(res)
    print(line)
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
