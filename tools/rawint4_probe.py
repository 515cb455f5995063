"""Times RAWINT4_G32 routed-expert decode at Kimi-K2 shapes beside the Q4_K per-pair path on the same expert ids.

E=384, H=7168, I=2048, k=8.  One RAWINT4 expert (gate + up + down) and one all-Q4_K expert both take 24,772,608 B, so the
two formats stream identical bytes.  SETS resident layer sets per format (9.5 GB each) are cycled inside one CUDA graph, so
consecutive layers never find their experts in the 50 MB L2.  Reported per batch size (1 and 8): us per layer, algorithmic
bytes (U x 24,772,608 B, U = unique experts hit per layer), GB/s and the fraction of the H100 SXM data-sheet 3.35 TB/s.
ROUNDS alternating rounds show the run-to-run spread.  Prints the card name and power limit (read-only nvidia-smi query).

    python tools/rawint4_probe.py [--out FILE]
"""
import ctypes as C
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ktransformers_b200 import native  # noqa: E402
from ktransformers_b200.util.synth import synth_blocks  # noqa: E402

E, K, H, I = 384, 8, 7168, 2048
EXPERT_BYTES = 3 * I * H // 256 * 144
SETS = int(os.environ.get("SETS", 2))
ROUNDS = int(os.environ.get("ROUNDS", 3))
REPLAYS = int(os.environ.get("REPLAYS", 20))
BF16, Q4_K, I4 = native.GGML_BF16, native.GGML_Q4_K, native.RAWINT4_G32
lib = native.lib()
stream = lambda: torch.cuda.current_stream().cuda_stream


def rawint4_set(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = []
    for rows, cols in ((I, H), (I, H), (H, I)):
        packed = torch.randint(0, 256, (E * rows * cols // 2,), dtype=torch.uint8, device="cuda", generator=g).view(torch.int32)
        scale = (torch.rand(E * rows * cols // 32, device="cuda", generator=g) * 0.02 + 0.005).to(torch.bfloat16)
        blocks = torch.empty(E * rows * cols // 256 * 144, dtype=torch.uint8, device="cuda")
        native.check(lib.ktb200_rawint4_pack(packed.data_ptr(), scale.data_ptr(), E * rows, cols, blocks.data_ptr(), stream()))
        del packed, scale
        out.append(blocks)
    return out, (I4, I4, I4)


def q4k_set(seed):
    return [synth_blocks(Q4_K, E * I * H, "cuda", seed + i) for i in range(3)], (Q4_K, Q4_K, Q4_K)


def handle(tensors, types, max_tokens):
    cfg = native.MoeConfig(E, K, H, I, 64, 10, max_tokens, 1, *(t.data_ptr() for t in tensors), *types, BF16, 0)
    h = C.c_void_p()
    native.check(lib.ktb200_moe_create(C.byref(cfg), 0, C.byref(h)))
    native.check(lib.ktb200_moe_load_weights(h, stream()))
    return h


def graph_of(handles, bs, ids, w, x, out):
    def run():
        for h, i in zip(handles, ids):
            native.check(lib.ktb200_moe_forward(h, bs, K, i.data_ptr(), w.data_ptr(), x.data_ptr(), out.data_ptr(), None, stream()))
    run()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        run()
    g.replay()
    torch.cuda.synchronize()
    return g


def time_graph(g, layers):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(REPLAYS):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (REPLAYS * layers)


def main():
    lines = []
    say = lambda s: (print(s, flush=True), lines.append(s))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    say(f"card: {q.stdout.strip() or 'nvidia-smi unavailable'}; torch: {torch.cuda.get_device_name(0)}")
    say(f"K2 shapes E={E} H={H} I={I} k={K}, {SETS} resident layer sets per format, {EXPERT_BYTES} B per expert, "
        f"{REPLAYS} graph replays x {ROUNDS} alternating rounds")
    sets = {"RAWINT4": [rawint4_set(100 + 10 * s) for s in range(SETS)], "Q4_K": [q4k_set(200 + 10 * s) for s in range(SETS)]}
    handles = {f: [handle(t, ty, 8) for t, ty in sets[f]] for f in sets}
    gen = torch.Generator(device="cuda").manual_seed(0)
    for bs in (1, 8):
        ids = [torch.stack([torch.randperm(E, device="cuda", generator=gen)[:K] for _ in range(bs)]).long() for _ in range(SETS)]
        U = sum(int(torch.unique(i).numel()) for i in ids) / SETS
        w = torch.rand(bs, K, device="cuda", generator=gen)
        x = (torch.randn(bs, H, device="cuda", generator=gen) * 0.5).bfloat16()
        out = torch.zeros_like(x)
        graphs = {f: graph_of(handles[f], bs, ids, w, x, out) for f in handles}
        res = {f: [] for f in graphs}
        for _ in range(ROUNDS):
            for f in graphs:
                res[f].append(time_graph(graphs[f], SETS))
        for f, us in res.items():
            best, med = min(us), sorted(us)[len(us) // 2]
            gbs = U * EXPERT_BYTES / (med * 1e-6) / 1e9
            say(f"bs={bs} {f:8s} U={U:5.1f} bytes/layer={U * EXPERT_BYTES / 1e6:8.1f} MB  us/layer median {med:7.1f} "
                f"(min {best:7.1f}, max {max(us):7.1f})  {gbs:7.1f} GB/s  {gbs / 3350:5.3f} of 3.35 TB/s")
        del graphs
    for f in handles:
        for h in handles[f]:
            lib.ktb200_moe_destroy(h)
    if "--out" in sys.argv:
        path = sys.argv[sys.argv.index("--out") + 1]
        os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
        with open(path, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
