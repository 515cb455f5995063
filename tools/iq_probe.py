"""Times low-bit routed-expert decode at DeepSeek-V3/R1 shapes beside the Q4_K/Q4_K/Q6_K path on the same expert ids.

E=256, H=7168, I=2048, k=8.  Formats (gate/up/down), chosen with FORMATS (comma-separated names, default the first three):
IQ1_S x3 (8,601,600 B per expert), IQ1_S/IQ1_S/IQ2_XXS (9,519,104 B), Q4_K/Q4_K/Q6_K (28,557,312 B, bench.py's mix),
IQ1_M/IQ1_M/IQ2_XXS (10,207,232 B, the 1.73-bit R1 files' experts), IQ1_M x3 (9,633,792 B), llama.cpp's 3-bit i-quant
mixes IQ3_XXS x3 (16,859,136 B), IQ3_XXS/IQ3_XXS/IQ3_S (17,547,264 B) and IQ3_S x3 (18,923,520 B), the 2-bit i-quant mixes
IQ2_XS x3 (12,730,368 B), IQ2_XS/IQ2_XS/IQ2_S (13,189,056 B) and IQ2_S x3 (14,106,624 B), and
llama.cpp's K-quant mixes Q2_K/Q2_K/Q3_K (15,941,632 B), Q3_K/Q3_K/Q4_K (20,873,216 B) and Q3_K x3 (18,923,520 B).  SETS
resident layer sets per format are cycled inside one CUDA graph, so consecutive layers never find their experts in the 50 MB
L2 (the smallest set is 2.2 GB).  Reported per batch size (1 and 8): us per layer, algorithmic bytes (U x bytes per expert,
U = unique experts hit per layer), GB/s and the fraction of the H100 SXM data-sheet 3.35 TB/s.  ROUNDS alternating rounds
show the run-to-run spread.  Prints the card name and power limit (read-only nvidia-smi query).

BASELINE_LIB names another build of libktb200.so: then this build and that one run as two arms, each in an interpreter of its
own (PROBE_LIB selects a worker's library), alternating REPS times on the same seeded weights, ids and inputs.  The summary
gives both arms' median over all rounds and checks that their outputs agree within assert_bf16_close's bound.

    python tools/iq_probe.py [--out FILE]
    FORMATS=Q2_K/Q2_K/Q3_K,Q3_K/Q3_K/Q4_K,Q3_Kx3,Q4_K/Q6_K BASELINE_LIB=/path/to/parent/libktb200.so python tools/iq_probe.py
"""
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ktransformers_b200 import native  # noqa: E402

if os.environ.get("PROBE_LIB"):
    native.LIB_PATH = os.environ["PROBE_LIB"]
from ktransformers_b200.util.synth import synth_blocks  # noqa: E402

E, K, H, I = 256, 8, 7168, 2048
SETS = int(os.environ.get("SETS", 2))
ROUNDS = int(os.environ.get("ROUNDS", 3))
REPLAYS = int(os.environ.get("REPLAYS", 20))
BF16, Q4_K, Q6_K = native.GGML_BF16, native.GGML_Q4_K, native.GGML_Q6_K
Q2_K, Q3_K = native.GGML_Q2_K, native.GGML_Q3_K
IQ1, IQ2, IQ1M = native.GGML_IQ1_S, native.GGML_IQ2_XXS, native.GGML_IQ1_M
IQ3XXS, IQ3S = native.GGML_IQ3_XXS, native.GGML_IQ3_S
IQ2XS, IQ2S = native.GGML_IQ2_XS, native.GGML_IQ2_S
ALL_FORMATS = {"IQ1_Sx3": (IQ1, IQ1, IQ1), "IQ1_S/IQ2_XXS": (IQ1, IQ1, IQ2), "Q4_K/Q6_K": (Q4_K, Q4_K, Q6_K),
               "IQ1_M/IQ1_M/IQ2_XXS": (IQ1M, IQ1M, IQ2), "IQ1_Mx3": (IQ1M, IQ1M, IQ1M),
               "IQ3_XXSx3": (IQ3XXS, IQ3XXS, IQ3XXS), "IQ3_XXS/IQ3_XXS/IQ3_S": (IQ3XXS, IQ3XXS, IQ3S), "IQ3_Sx3": (IQ3S, IQ3S, IQ3S),
               "IQ2_XSx3": (IQ2XS, IQ2XS, IQ2XS), "IQ2_XS/IQ2_XS/IQ2_S": (IQ2XS, IQ2XS, IQ2S), "IQ2_Sx3": (IQ2S, IQ2S, IQ2S),
               "Q2_K/Q2_K/Q3_K": (Q2_K, Q2_K, Q3_K), "Q3_K/Q3_K/Q4_K": (Q3_K, Q3_K, Q4_K), "Q3_Kx3": (Q3_K, Q3_K, Q3_K)}
FORMATS = {f: ALL_FORMATS[f] for f in os.environ.get("FORMATS", "IQ1_Sx3,IQ1_S/IQ2_XXS,Q4_K/Q6_K").split(",")}
lib = native.lib()
stream = lambda: torch.cuda.current_stream().cuda_stream


def expert_bytes(types):
    return sum(I * H // 256 * int(lib.ktb200_type_size(t)) for t in types)


def iq1m_set_d(b, d):
    """IQ1_M keeps its fp16 d in the top nibbles of the four scale words (bytes 49, 51, 53, 55), lowest nibble first"""
    bits = d.view(torch.int16).to(torch.int32) & 0xFFFF
    for w in range(4):
        b[:, 49 + 2 * w] = ((b[:, 49 + 2 * w].to(torch.int32) & 0x0F) | (((bits >> (4 * w)) & 0xF) << 4)).to(torch.uint8)


def iq_blocks(t, n_elems, seed):
    """random bytes (any pattern is a valid block) with a sane fp16 d"""
    bb = int(lib.ktb200_type_size(t))
    g = torch.Generator(device="cuda").manual_seed(seed)
    b = torch.randint(0, 256, (n_elems // 256, bb), dtype=torch.uint8, device="cuda", generator=g)
    d = ((torch.rand(n_elems // 256, device="cuda", generator=g) * 0.5 + 0.75) / (512 if t in (IQ2, IQ2XS, IQ2S) else 1024 if t in (IQ3XXS, IQ3S) else 64)).half()
    if t == IQ1M:
        iq1m_set_d(b, d)
    else:
        b[:, 0:2] = d.view(torch.uint8).view(-1, 2)
    return b.reshape(-1)


def layer_set(types, seed):
    out = []
    for i, (t, (rows, cols)) in enumerate(zip(types, ((I, H), (I, H), (H, I)))):
        out.append(iq_blocks(t, E * rows * cols, seed + i) if t in (IQ1, IQ2, IQ1M, IQ3XXS, IQ3S, IQ2XS, IQ2S) else synth_blocks(t, E * rows * cols, "cuda", seed + i))
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


def measure(say, outdir=None):
    """time every format at bs 1 and 8; returns {"format bs": [us per round]}, and saves each output under outdir"""
    say(f"V3 shapes E={E} H={H} I={I} k={K}, {SETS} resident layer sets per format, {REPLAYS} graph replays x {ROUNDS} alternating rounds")
    allres = {}
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
        for f, g in graphs.items():   # the last layer set's output for the seeded inputs, after a replay of this format's graph
            g.replay()
            torch.cuda.synchronize()
            if outdir:
                np.save(os.path.join(outdir, f"{f.replace('/', '_')}_{bs}.npy"), out.view(torch.int16).cpu().numpy())
        for f, us in res.items():
            allres[f"{f} {bs}"] = us
            eb = expert_bytes(FORMATS[f])
            best, med = min(us), sorted(us)[len(us) // 2]
            gbs = U * eb / (med * 1e-6) / 1e9
            say(f"bs={bs} {f:14s} U={U:5.1f} bytes/layer={U * eb / 1e6:7.1f} MB  us/layer median {med:8.1f} "
                f"(min {best:8.1f}, max {max(us):8.1f})  {gbs:7.1f} GB/s  {gbs / 3350:5.3f} of 3.35 TB/s")
        del graphs
    for f in handles:
        for h in handles[f]:
            lib.ktb200_moe_destroy(h)
    return allres


def bf16_close(got, want):
    """tests/test_gpu_parity.py assert_bf16_close: within 2^-7 of the larger magnitude + 1e-3 of max |want|, > 97 % bit-identical"""
    a = (got.astype(np.uint32) << 16).view(np.float32)
    b = (want.astype(np.uint32) << 16).view(np.float32)
    ok = np.abs(a - b) <= 2.0 ** -7 * np.maximum(np.abs(a), np.abs(b)) + 1e-3 * np.abs(b).max()
    return bool(ok.all()) and float((got == want).mean()) > 0.97, float((got == want).mean())


def compare_builds(say):
    """this build against BASELINE_LIB, each arm in an interpreter of its own, alternating REPS times"""
    reps = int(os.environ.get("REPS", 2))
    arms = {"this build": native.LIB_PATH, "baseline": os.environ["BASELINE_LIB"]}
    tmp = tempfile.mkdtemp(prefix="iq_probe_")
    times = {a: {} for a in arms}
    for rep in range(reps):
        for arm, path in arms.items():
            d = os.path.join(tmp, arm.replace(" ", "_"))
            os.makedirs(d, exist_ok=True)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", d], env=dict(os.environ, PROBE_LIB=path),
                               capture_output=True, text=True)
            if r.returncode:
                print(r.stdout[-2000:], r.stderr[-3000:])
                raise SystemExit(f"{arm}: worker failed")
            for l in r.stdout.splitlines():
                if l.startswith("RESULT "):
                    for key, us in json.loads(l[7:]).items():
                        times[arm].setdefault(key, []).extend(us)
                else:
                    say(f"[{arm}, rep {rep}] {l}")
    ok = True
    say(f"summary: median us per layer over {reps} alternating reps x {ROUNDS} rounds (min-max in brackets)")
    for key in times["this build"]:
        f, bs = key.rsplit(" ", 1)
        name = f"{f.replace('/', '_')}_{bs}.npy"
        a, b = (np.load(os.path.join(tmp, x, name)).view(np.uint16) for x in ("this_build", "baseline"))
        close, same = bf16_close(a, b)
        ok &= close
        med = {arm: sorted(times[arm][key])[len(times[arm][key]) // 2] for arm in arms}
        rng = {arm: f"{min(times[arm][key]):.1f}-{max(times[arm][key]):.1f}" for arm in arms}
        say(f"bs={bs} {f:16s} this build {med['this build']:8.1f} [{rng['this build']}]  baseline {med['baseline']:8.1f} "
            f"[{rng['baseline']}]  speed-up {med['baseline'] / med['this build']:5.2f}x  outputs "
            f"{'within' if close else 'OUTSIDE'} bf16 bound ({same:.2%} bit-identical)")
    say("all outputs agree" if ok else "OUTPUT MISMATCH")
    return ok


def main():
    if len(sys.argv) > 2 and sys.argv[1] == "--worker":
        print("RESULT " + json.dumps(measure(print, sys.argv[2])), flush=True)
        return
    lines = []
    say = lambda s: (print(s, flush=True), lines.append(s))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    say(f"card: {q.stdout.strip() or 'nvidia-smi unavailable'}; torch: {torch.cuda.get_device_name(0)}")
    ok = compare_builds(say) if os.environ.get("BASELINE_LIB") else bool(measure(say))
    if "--out" in sys.argv:
        path = sys.argv[sys.argv.index("--out") + 1]
        os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
        with open(path, "w") as f:
            f.write("\n".join(lines) + "\n")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
