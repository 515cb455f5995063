"""Ragged absorbed-MLA attention (ktb200_mla_decode_ragged) against the launches a ragged batch needs today, on one GPU.

(a) a mixed batch: 7 decode rows at 4096..32768 cached tokens and one 512-token prompt chunk at P = 0, as one ragged call
    against ktb200_mla_decode (the 7 rows) followed by ktb200_mla_decode_chunk (the chunk), on the same data;
(b) a skewed decode batch: one sequence at 131072 tokens and 65 at 1024, the ragged planner against ktb200_mla_decode's
    single split count (pick_splits).
V3 shapes (128 heads, 512 + 64 latent, pages of 64).  CUDA-event windows of >= 50 ms, the median of 3 alternating rounds.
The card's name and power limit are read in the same run.  The host planner's time is reported too (it runs once per step).

    python tools/mla_ragged_probe.py [--out results.json]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ktransformers_b200 import native  # noqa: E402

H, PAGE, SCALE = 128, 64, (128 + 64) ** -0.5


def timed(fn, min_ms=50.0):
    fn()
    torch.cuda.synchronize()
    n = 1
    while True:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(n):
            fn()
        b.record()
        b.synchronize()
        ms = a.elapsed_time(b)
        if ms >= min_ms:
            return ms / n
        n *= 2


def median_alternating(fns, rounds=3):
    res = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            res[k].append(timed(f))
    return {k: float(np.median(v)) for k, v in res.items()}


class Batch:
    """sequences with their own lengths over one cache of consecutive pages; bf16 queries for every row"""

    def __init__(self, q_lens, kv_len, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.q_lens, self.kv_len = np.array(q_lens, np.int32), np.array(kv_len, np.int32)
        self.B = len(q_lens)
        self.width = int(-(-self.kv_len.max() // PAGE))
        pages = int(sum(-(-int(k) // PAGE) for k in self.kv_len))
        self.cache = torch.randn((pages, PAGE, 576), generator=g, device="cuda").to(torch.bfloat16)
        pt, start = np.zeros((self.B, self.width), np.int32), 0
        for b in range(self.B):
            n = -(-int(self.kv_len[b]) // PAGE)
            pt[b, :n] = np.arange(start, start + n)
            start += n
        self.pt = torch.from_numpy(pt).cuda()
        self.rows = int(self.q_lens.sum())
        self.qo = np.r_[0, np.cumsum(self.q_lens)].astype(np.int32)
        self.qn = (torch.randn((self.rows, H, 512), generator=g, device="cuda") * 0.5).to(torch.bfloat16)
        self.qp = (torch.randn((self.rows, H, 64), generator=g, device="cuda") * 0.5).to(torch.bfloat16)

    def ragged(self, max_items=8192):
        lib = native.lib()
        n = lib.ktb200_mla_ragged_plan_ints(max_items, self.rows)
        buf = np.zeros(n, np.int32)
        sms = torch.cuda.get_device_properties(0).multi_processor_count

        def do_plan():
            native.check(lib.ktb200_mla_ragged_plan(self.qo.ctypes.data, self.kv_len.ctypes.data, self.B, H, PAGE, self.width, sms, 0,
                                                    max_items, self.rows, buf.ctypes.data, n, None, None))
        t0 = time.perf_counter()
        for _ in range(20):
            do_plan()
        plan_us = (time.perf_counter() - t0) / 20 * 1e6
        plan_d = torch.from_numpy(buf).cuda()
        ws_bytes = lib.ktb200_mla_ragged_workspace_bytes(max_items, H)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
        out = torch.empty_like(self.qn)
        p = native.MlaRaggedParams(self.rows, max_items, H, PAGE, self.width, SCALE, self.qn.data_ptr(), self.qp.data_ptr(), self.cache.data_ptr(),
                                   self.pt.data_ptr(), plan_d.data_ptr(), out.data_ptr(), None, ws.data_ptr(), ws_bytes, 0)
        s = torch.cuda.current_stream().cuda_stream
        keep = (plan_d, ws, out, p)
        return (lambda: native.check(lib.ktb200_mla_decode_ragged(C.byref(keep[3]), s))), plan_us, int(buf[0]), out

    def decode(self, seqs):
        """ktb200_mla_decode over the q_len-1 sequences `seqs` (their rows in order), automatic splits"""
        lib = native.lib()
        rows = [int(self.qo[b]) for b in seqs]
        qn, qp = self.qn[rows].contiguous(), self.qp[rows].contiguous()
        pt, kl = self.pt[list(seqs)].contiguous(), torch.from_numpy(self.kv_len[list(seqs)]).cuda()
        ws_bytes = lib.ktb200_mla_workspace_bytes(len(seqs), H, 0)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
        out = torch.empty_like(qn)
        p = native.MlaParams(len(seqs), H, PAGE, self.width, 0, SCALE, qn.data_ptr(), qp.data_ptr(), self.cache.data_ptr(), pt.data_ptr(),
                             kl.data_ptr(), out.data_ptr(), None, ws.data_ptr(), ws_bytes, 0)
        s = torch.cuda.current_stream().cuda_stream
        keep = (qn, qp, pt, kl, ws, out, p)
        return (lambda: native.check(lib.ktb200_mla_decode(C.byref(keep[-1]), s))), out

    def chunk(self, b):
        lib = native.lib()
        q = int(self.q_lens[b])
        qn, qp = self.qn[self.qo[b]:self.qo[b + 1]].contiguous(), self.qp[self.qo[b]:self.qo[b + 1]].contiguous()
        pt, kl = self.pt[b:b + 1].contiguous(), torch.from_numpy(self.kv_len[b:b + 1]).cuda()
        ws_bytes = lib.ktb200_mla_chunk_workspace_bytes(1, q, H, 0)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
        out = torch.empty_like(qn)
        p = native.MlaChunkParams(1, q, H, PAGE, self.width, 0, SCALE, qn.data_ptr(), qp.data_ptr(), self.cache.data_ptr(), pt.data_ptr(),
                                  kl.data_ptr(), out.data_ptr(), None, ws.data_ptr(), ws_bytes, 0)
        s = torch.cuda.current_stream().cuda_stream
        keep = (qn, qp, pt, kl, ws, out, p)
        return (lambda: native.check(lib.ktb200_mla_decode_chunk(C.byref(keep[-1]), s))), out


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0) + ", power limit not read"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the probe times the GPU; there is nothing to measure without one"
    res = {"card": card()}
    # (a) mixed: 7 decode rows and a 512-token chunk at P = 0 (third)
    mixed = Batch([1, 1, 512, 1, 1, 1, 1, 1], [4096, 8192, 512, 12288, 16384, 20480, 24576, 32768], 1)
    rag, plan_us, items, r_out = mixed.ragged()
    dec, d_out = mixed.decode([0, 1, 3, 4, 5, 6, 7])
    chk, c_out = mixed.chunk(2)
    two = lambda: (dec(), chk())
    t = median_alternating({"ragged": rag, "decode+chunk": two})
    torch.cuda.synchronize()
    dec_rows = [int(mixed.qo[b]) for b in (0, 1, 3, 4, 5, 6, 7)]
    diff = max((r_out[dec_rows].float() - d_out.float()).abs().max().item(),
               (r_out[int(mixed.qo[2]):int(mixed.qo[3])].float() - c_out.float()).abs().max().item())
    res["mixed"] = {"ragged_ms": t["ragged"], "decode_then_chunk_ms": t["decode+chunk"], "plan_us": plan_us, "items": items,
                    "max_abs_diff": diff}
    # (b) skewed decode: one at 131072, 65 at 1024
    skew = Batch([1] * 66, [131072] + [1024] * 65, 2)
    rag, plan_us, items, r_out = skew.ragged()
    dec, d_out = skew.decode(list(range(66)))
    t = median_alternating({"ragged": rag, "decode": dec})
    torch.cuda.synchronize()
    res["skewed"] = {"ragged_ms": t["ragged"], "decode_pick_splits_ms": t["decode"], "plan_us": plan_us, "items": items,
                     "max_abs_diff": (r_out.float() - d_out.float()).abs().max().item()}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
