"""GPU probe for ktb200_mla_decode (wgmma path): stage-by-stage numerics (raw scores of the first tile through
ktb200_debug_mla, then output / LSE against the numpy oracle) and timing over context lengths.
    python tools/mla_probe.py [--time]
"""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import gpu_util as G  # noqa: E402
from ktransformers_b200 import native  # noqa: E402
from oracle import mla_oracle  # noqa: E402

lib = native.lib()


def case(B, Hq, page, lens, seed=0):
    rng = np.random.default_rng(seed)
    maxp = max((l + page - 1) // page for l in lens)
    npg = B * maxp + 3
    kv = mla_oracle.bf16_round(rng.standard_normal((npg, page, 576)).astype(np.float32))
    pt = rng.permutation(npg)[: B * maxp].reshape(B, maxp).astype(np.int32)
    qn = mla_oracle.bf16_round((rng.standard_normal((B, Hq, 512)) * 0.5).astype(np.float32))
    qp = mla_oracle.bf16_round((rng.standard_normal((B, Hq, 64)) * 0.5).astype(np.float32))
    return qn, qp, kv, pt, np.array(lens, np.int32)


def numerics():
    dbg = torch.zeros(8192, dtype=torch.float32, device="cuda")
    for B, Hq, page, lens, splits in ((1, 128, 64, [32], 1), (1, 128, 64, [64], 1), (1, 128, 64, [100], 1), (1, 16, 32, [200], 2),
                                     (2, 128, 64, [640, 2049], 0), (1, 128, 64, [4096], 0), (1, 128, 64, [65536], 0)):
        qn, qp, kv, pt, kl = case(B, Hq, page, lens, seed=sum(lens))
        scale = (128 + 64) ** -0.5
        dbg.zero_()
        lib.ktb200_debug_mla(dbg.data_ptr())
        out, lse = G.mla_decode(qn, qp, kv, pt, kl, scale, num_kv_splits=splits)
        lib.ktb200_debug_mla(None)
        rows = mla_oracle.gather_kv(kv, pt[0], int(kl[0]), page)
        nt = min(32, rows.shape[0])
        q = np.concatenate([qn[0], qp[0]], -1)[:64]                      # first head group
        s_ref = q.astype(np.float64) @ rows[:nt].astype(np.float64).T    # [heads<=64][nt]
        s_got = dbg.cpu().numpy()[: 64 * 32].reshape(64, 32)[: q.shape[0], :nt]
        want, want_lse = mla_oracle.mla_decode(qn, qp, kv, pt, kl, scale, p_bf16=True)
        mag = np.abs(want).max()
        print(f"B={B} Hq={Hq} page={page} lens={lens} splits={splits}: S err {np.abs(s_got - s_ref).max():.3e} (|S| {np.abs(s_ref).max():.2f}) "
              f"out err {np.abs(out - want).max() / mag:.3e} lse err {np.abs(lse - want_lse).max():.3e} finite={np.isfinite(out).all()}", flush=True)
        if np.abs(s_got - s_ref).max() > 1e-2 * np.abs(s_ref).max():
            bad = np.argwhere(np.abs(s_got - s_ref) > 1e-2 * np.abs(s_ref).max())
            print("   first bad S entries (head, token):", bad[:8].tolist(), "got", s_got[tuple(bad[0])], "want", s_ref[tuple(bad[0])])
            print("   S got row0[:8]", s_got[0, :8], "want", s_ref[0, :8])


def timing():
    page = 64
    for B, L in ((1, 1024), (1, 4096), (1, 32768), (1, 131072), (8, 4096), (8, 32768)):
        npg = B * (L // page)
        kv = torch.randn((npg, page, 576), device="cuda", dtype=torch.bfloat16)
        pt = torch.arange(npg, dtype=torch.int32, device="cuda").reshape(B, -1).contiguous()
        kl = torch.full((B,), L, dtype=torch.int32, device="cuda")
        qn = (torch.randn((B, 128, 512), device="cuda") * 0.5).to(torch.bfloat16)
        qp = (torch.randn((B, 128, 64), device="cuda") * 0.5).to(torch.bfloat16)
        out = torch.zeros((B, 128, 512), dtype=torch.bfloat16, device="cuda")
        wsb = lib.ktb200_mla_workspace_bytes(B, 128, 0)
        ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
        p = native.MlaParams(B, 128, page, pt.shape[1], 0, 0.072, qn.data_ptr(), qp.data_ptr(), kv.data_ptr(), pt.data_ptr(), kl.data_ptr(),
                             out.data_ptr(), None, ws.data_ptr(), wsb, npg * page)
        flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
        s = torch.cuda.current_stream().cuda_stream
        for _ in range(3):
            native.check(lib.ktb200_mla_decode(C.byref(p), s))
        torch.cuda.synchronize()
        ts = []
        for _ in range(10):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            native.check(lib.ktb200_mla_decode(C.byref(p), s))
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ms = float(np.median(ts))
        byts = B * L * 1152
        flops = B * L * 278528
        print(f"B={B} L={L}: {ms * 1e3:.1f} us  {byts / ms / 1e6:.0f} GB/s  {flops / ms / 1e9:.0f} TFLOP/s", flush=True)


if __name__ == "__main__":
    numerics()
    if "--time" in sys.argv:
        timing()
