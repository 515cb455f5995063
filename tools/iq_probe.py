"""Times IQ1_S / IQ2_XXS routed-expert decode at DeepSeek-V3/R1 shapes beside the Q4_K/Q4_K/Q6_K path on the same expert ids.

E=256, H=7168, I=2048, k=8.  Three formats (gate/up/down): IQ1_S x3 (8,601,600 B per expert), IQ1_S/IQ1_S/IQ2_XXS
(9,519,104 B) and Q4_K/Q4_K/Q6_K (28,557,312 B, bench.py's mix).  SETS resident layer sets per format are cycled inside one
CUDA graph, so consecutive layers never find their experts in the 50 MB L2 (the smallest set is 2.2 GB).  Reported per batch
size (1 and 8): us per layer, algorithmic bytes (U x bytes per expert, U = unique experts hit per layer), GB/s and the
fraction of the H100 SXM data-sheet 3.35 TB/s.  ROUNDS alternating rounds show the run-to-run spread.  Prints the card name
and power limit (read-only nvidia-smi query).

    python tools/iq_probe.py [--out FILE]
"""
import ctypes as C
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ktransformers_b200 import native  # noqa: E402
from ktransformers_b200.util.synth import synth_blocks  # noqa: E402

E, K, H, I = 256, 8, 7168, 2048
SETS = int(os.environ.get("SETS", 2))
ROUNDS = int(os.environ.get("ROUNDS", 3))
REPLAYS = int(os.environ.get("REPLAYS", 20))
BF16, Q4_K, Q6_K = native.GGML_BF16, native.GGML_Q4_K, native.GGML_Q6_K
IQ1, IQ2 = native.GGML_IQ1_S, native.GGML_IQ2_XXS
FORMATS = {"IQ1_Sx3": (IQ1, IQ1, IQ1), "IQ1_S/IQ2_XXS": (IQ1, IQ1, IQ2), "Q4_K/Q6_K": (Q4_K, Q4_K, Q6_K)}
lib = native.lib()
stream = lambda: torch.cuda.current_stream().cuda_stream


def expert_bytes(types):
    return sum(I * H // 256 * int(lib.ktb200_type_size(t)) for t in types)


def iq_blocks(t, n_elems, seed):
    """random bytes (any pattern is a valid block) with a sane fp16 d"""
    bb = int(lib.ktb200_type_size(t))
    g = torch.Generator(device="cuda").manual_seed(seed)
    b = torch.randint(0, 256, (n_elems // 256, bb), dtype=torch.uint8, device="cuda", generator=g)
    d = ((torch.rand(n_elems // 256, device="cuda", generator=g) * 0.5 + 0.75) / (64 if t == IQ1 else 512)).half()
    b[:, 0:2] = d.view(torch.uint8).view(-1, 2)
    return b.reshape(-1)


def layer_set(types, seed):
    out = []
    for i, (t, (rows, cols)) in enumerate(zip(types, ((I, H), (I, H), (H, I)))):
        out.append(iq_blocks(t, E * rows * cols, seed + i) if t in (IQ1, IQ2) else synth_blocks(t, E * rows * cols, "cuda", seed + i))
    return out


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
    say(f"V3 shapes E={E} H={H} I={I} k={K}, {SETS} resident layer sets per format, {REPLAYS} graph replays x {ROUNDS} alternating rounds")
    sets = {f: [layer_set(ty, 100 * (j + 1) + 10 * s) for s in range(SETS)] for j, (f, ty) in enumerate(FORMATS.items())}
    handles = {f: [handle(t, FORMATS[f], 8) for t in sets[f]] for f in sets}
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
            eb = expert_bytes(FORMATS[f])
            best, med = min(us), sorted(us)[len(us) // 2]
            gbs = U * eb / (med * 1e-6) / 1e9
            say(f"bs={bs} {f:14s} U={U:5.1f} bytes/layer={U * eb / 1e6:7.1f} MB  us/layer median {med:8.1f} "
                f"(min {best:8.1f}, max {max(us):8.1f})  {gbs:7.1f} GB/s  {gbs / 3350:5.3f} of 3.35 TB/s")
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
