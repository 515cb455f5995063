"""Times the grouped (prefill) MoE path at DeepSeek-V3 shapes: tokens/s at qlen in {64, 256, 1024, 4096}, against the per-pair kernels."""
import ctypes as C, os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ktransformers_b200 import native
from ktransformers_b200.util.synth import synth_blocks
Q4_K, Q6_K, BF16 = 12, 14, 30
lib = native.lib()
E, k, H, I = int(os.environ.get("E", 256)), 8, 7168, 2048
gate, up, down = synth_blocks(Q4_K, E * I * H, "cuda", 1), synth_blocks(Q4_K, E * I * H, "cuda", 2), synth_blocks(Q6_K, E * H * I, "cuda", 3)
cfg = native.MoeConfig(E, k, H, I, 64, 10, 4096, 1, gate.data_ptr(), up.data_ptr(), down.data_ptr(), Q4_K, Q4_K, Q6_K, BF16, 0)
h = C.c_void_p(); native.check(lib.ktb200_moe_create(C.byref(cfg), 0, C.byref(h)))
s = torch.cuda.current_stream().cuda_stream
native.check(lib.ktb200_moe_load_weights(h, s))
g = torch.Generator(device="cuda").manual_seed(0)
for qlen in [int(v) for v in os.environ.get("QLENS", "64,256,1024,4096").split(",")]:
    x = (torch.randn(qlen, H, device="cuda", generator=g) / 100).bfloat16()
    ids = torch.stack([torch.randperm(E, device="cuda", generator=g)[:k] for _ in range(qlen)]).long()
    w = torch.rand(qlen, k, device="cuda", generator=g)
    out = torch.zeros_like(x)
    def run(): native.check(lib.ktb200_moe_forward(h, qlen, k, ids.data_ptr(), w.data_ptr(), x.data_ptr(), out.data_ptr(), None, s))
    for _ in range(2): run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    n = 5
    e0.record()
    for _ in range(n): run()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / n
    flops = 2.0 * qlen * k * 3 * H * I
    print(f"qlen {qlen}: {ms:.3f} ms  {qlen / ms * 1e3:.0f} tok/s  {flops / ms / 1e9:.1f} TFLOP/s-equivalent  (KTB200_GROUPED_MIN={os.environ.get('KTB200_GROUPED_MIN', '48')})", flush=True)

if os.environ.get("TRACE"):
    tr = torch.zeros(2 * 3 * 96 * 4, dtype=torch.int64, device="cuda")
    lib.ktb200_debug_grouped(tr.data_ptr()); run(); torch.cuda.synchronize(); lib.ktb200_debug_grouped(None)
    t = tr.cpu().numpy().reshape(2, 3, 96, 4)
    for kname, kk in (("gate (Q4_K)", 0), ("down (Q6_K)", 1)):
        t0 = t[kk, 0, 0, 0]
        print(f"--- {kname}: cycles since the producer's first stage; P = wait_group done / smem_free seen / arrived, M = before ab_full / ab_full seen / MMAs + scale-and-add done / arrived")
        for st in range(0, 40):
            P, M = t[kk, 0, st] - t0, t[kk, 1, st] - t0
            print(f"st {st:2d}  P {P[0]:6d} {P[1]:6d} {P[2]:6d} {P[3]:6d} | M {M[0]:6d} {M[1]:6d} {M[2]:6d} {M[3]:6d}")
