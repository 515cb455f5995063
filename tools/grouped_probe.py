"""Times the grouped (prefill) MoE path at DeepSeek-V3 shapes (E 256, H 7168, I 2048, k 8, BF16) against the per-pair kernels,
for the expert type sets Q4_K/Q4_K/Q6_K, DeepSeek-R1's IQ1_S x3, IQ1_S/IQ1_S/IQ2_XXS, IQ1_M x3 ("iq1mx3") and IQ1_M/IQ1_M/IQ2_XXS
("iq1m_iq1m_iq2"), the 3-bit i-quant sets IQ3_XXS x3 ("iq3xxsx3"), IQ3_XXS/IQ3_XXS/IQ3_S ("iq3xxs_iq3xxs_iq3s") and IQ3_S x3
("iq3sx3"), the 2-bit i-quant sets IQ2_XS x3 ("iq2xsx3"), IQ2_XS/IQ2_XS/IQ2_S ("iq2xs_iq2xs_iq2s") and IQ2_S x3 ("iq2sx3"), and
the K-quant mixes "q5k" (Q5_K/Q5_K/Q6_K,
Q5_K_M), "q3k" (Q3_K/Q3_K/Q4_K, Q3_K_M), "q2k" (Q2_K/Q2_K/Q3_K, Q2_K) and "q2k_q6k" (Q2_K/Q2_K/Q6_K: the per-pair kernels refuse
a Q3_K down projection at these shapes, so this set gives Q2_K gate / up a per-pair time); and set "i4" at Kimi-K2's shapes
(RAWINT4_G32 x3, E 384, 60 MoE layers), packed with ktb200_rawint4_pack from seeded words and scales as tools/rawint4_probe.py.

Every (type set, arm) runs in an interpreter of its own on the same seeded weights and inputs: arm "grouped" as shipped,
arm "per-pair" with KTB200_GROUPED_MIN above every qlen (the threshold is read once per process), and, when BASELINE_LIB names
another build of libktb200.so, arm "baseline" = the grouped path of that build.  Arms alternate, REPS times; the table gives
the fastest repetition, ms per layer, tok/s over the model's MoE layers (V3/R1 58, K2 60), and the share of the HBM bound for the bytes the grouped GEMMs
read (every expert's three matrices once per 32-token tile of its tokens, at 3.35 TB/s).  Outputs are compared at every timed
size: per-pair against grouped within assert_bf16_close's bound, baseline against grouped bit for bit where both builds run
the same kernels (else within that bound).

    python tools/grouped_probe.py                       TYPES=q4k,iq1x3,iq1_iq1_iq2  QLENS=48,64,256,1024,4096  REPS=2
    TYPES=q5k,q3k,q2k python tools/grouped_probe.py
    TYPES=i4 QLENS=8,16,24,32,48,64,128,256,1024,4096 python tools/grouped_probe.py
    TRACE=1 python tools/grouped_probe.py               clock64 stamps of the gate and down GEMMs' CTA 0 (grouped arm)
"""
import json, os, subprocess, sys, tempfile
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
Q2_K, Q3_K, Q4_K, Q5_K, Q6_K, IQ2_XXS, IQ1_S, IQ1_M, BF16, I4 = 10, 11, 12, 13, 14, 16, 19, 29, 30, 256
IQ3_XXS, IQ3_S = 18, 21
IQ2_XS, IQ2_S = 17, 22
TYPE_SETS = {"q4k": (Q4_K, Q4_K, Q6_K), "iq1x3": (IQ1_S,) * 3, "iq1_iq1_iq2": (IQ1_S, IQ1_S, IQ2_XXS), "i4": (I4,) * 3,
             "iq1mx3": (IQ1_M,) * 3, "iq1m_iq1m_iq2": (IQ1_M, IQ1_M, IQ2_XXS), "q5k": (Q5_K, Q5_K, Q6_K), "q3k": (Q3_K, Q3_K, Q4_K), "q2k": (Q2_K, Q2_K, Q3_K), "q2k_q6k": (Q2_K, Q2_K, Q6_K),
             "iq3xxsx3": (IQ3_XXS,) * 3, "iq3xxs_iq3xxs_iq3s": (IQ3_XXS, IQ3_XXS, IQ3_S), "iq3sx3": (IQ3_S,) * 3,
             "iq2xsx3": (IQ2_XS,) * 3, "iq2xs_iq2xs_iq2s": (IQ2_XS, IQ2_XS, IQ2_S), "iq2sx3": (IQ2_S,) * 3}
NAMES = {Q2_K: "Q2_K", Q3_K: "Q3_K", Q4_K: "Q4_K", Q5_K: "Q5_K", Q6_K: "Q6_K", IQ1_S: "IQ1_S", IQ1_M: "IQ1_M", IQ2_XXS: "IQ2_XXS",
         I4: "RAWINT4_G32", IQ3_XXS: "IQ3_XXS", IQ3_S: "IQ3_S", IQ2_XS: "IQ2_XS", IQ2_S: "IQ2_S"}
BLOCK = {Q2_K: 84, Q3_K: 110, Q4_K: 144, Q5_K: 176, Q6_K: 210, IQ1_S: 50, IQ1_M: 56, IQ2_XXS: 66, I4: 144, IQ3_XXS: 98, IQ3_S: 110, IQ2_XS: 74, IQ2_S: 82}
KERNEL = {Q4_K: "grouped_gemm_kernel<0>", Q6_K: "grouped_gemm_kernel<1>", IQ1_S: "grouped_gemm_kernel<2>", IQ2_XXS: "grouped_gemm_kernel<3>",
          I4: "grouped_i4_kernel<1> (gate, BF16) / <3> (down)", Q5_K: "grouped_gemm_kernel<5>", Q3_K: "grouped_gemm_kernel<6>",
          Q2_K: "grouped_gemm_kernel<7>", IQ1_M: "grouped_gemm_kernel<8>", IQ3_XXS: "grouped_gemm_kernel<9>", IQ3_S: "grouped_gemm_kernel<10>",
          IQ2_XS: "grouped_gemm_kernel<11>", IQ2_S: "grouped_gemm_kernel<12>"}
k, H, I, HBM = 8, 7168, 2048, 3.35e12
# (experts, MoE layers) per type set: DeepSeek-V3/R1 256 and 58, Kimi-K2 384 and 60; E in the environment overrides the experts
SHAPE = {"i4": (384, 60)}
set_e = lambda tset: int(os.environ.get("E", SHAPE.get(tset, (256, 58))[0]))
set_layers = lambda tset: SHAPE.get(tset, (256, 58))[1]


def weights(t, n, seed, cols=H):
    """seeded raw blocks on the device: synth_blocks for the K-quants; random bytes with d in [0.75, 1.25) / 64 (IQ1_S, IQ1_M), / 512
    (IQ2_XXS, IQ2_XS, IQ2_S) or / 1024 (IQ3_XXS, IQ3_S) for the i-quants (every bit pattern is a valid i-quant block); RAWINT4 packed from random words and bf16 scales
    in [0.005, 0.025) (tools/rawint4_probe.py)"""
    if t == I4:
        from ktransformers_b200 import native
        g = torch.Generator(device="cuda").manual_seed(seed)
        packed = torch.randint(0, 256, (n // 2,), dtype=torch.uint8, device="cuda", generator=g).view(torch.int32)
        scale = (torch.rand(n // 32, device="cuda", generator=g) * 0.02 + 0.005).to(torch.bfloat16)
        blocks = torch.empty(n // 256 * 144, dtype=torch.uint8, device="cuda")
        native.check(native.lib().ktb200_rawint4_pack(packed.data_ptr(), scale.data_ptr(), n // cols, cols, blocks.data_ptr(),
                                                      torch.cuda.current_stream().cuda_stream))
        return blocks
    if t in (Q2_K, Q3_K, Q4_K, Q5_K, Q6_K):
        from ktransformers_b200.util.synth import synth_blocks
        return synth_blocks(t, n, "cuda", seed)
    g = torch.Generator(device="cuda").manual_seed(seed)
    b = torch.randint(0, 256, (n // 256, BLOCK[t]), dtype=torch.uint8, device="cuda", generator=g)
    d = ((torch.rand(n // 256, device="cuda", generator=g) * 0.5 + 0.75) / (512 if t in (IQ2_XXS, IQ2_XS, IQ2_S) else 1024 if t in (IQ3_XXS, IQ3_S) else 64)).half()
    if t == IQ1_M:   # d in the top nibbles of the four scale words (bytes 49, 51, 53, 55), lowest nibble first
        bits = d.view(torch.int16).to(torch.int32) & 0xFFFF
        for w in range(4):
            b[:, 49 + 2 * w] = ((b[:, 49 + 2 * w].to(torch.int32) & 0x0F) | (((bits >> (4 * w)) & 0xF) << 4)).to(torch.uint8)
    else:
        b[:, 0:2] = d.view(torch.uint8).view(-1, 2)
    return b.reshape(-1)


def worker(tset, qlens, outdir):
    import ctypes as C
    from ktransformers_b200 import native
    if os.environ.get("PROBE_LIB"):
        native.LIB_PATH = os.environ["PROBE_LIB"]
    lib = native.lib()
    gt, ut, dt = TYPE_SETS[tset]
    E = set_e(tset)
    w3 = [weights(t, E * I * H, s, c) for t, s, c in ((gt, 1, H), (ut, 2, H), (dt, 3, I))]
    cfg = native.MoeConfig(E, k, H, I, 64, 10, max(qlens), 1, *(t.data_ptr() for t in w3), gt, ut, dt, BF16, 0)
    h = C.c_void_p()
    native.check(lib.ktb200_moe_create(C.byref(cfg), 0, C.byref(h)))
    s = torch.cuda.current_stream().cuda_stream
    native.check(lib.ktb200_moe_load_weights(h, s))
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {}
    for qlen in qlens:
        x = (torch.randn(qlen, H, device="cuda", generator=g) / 100).bfloat16()
        ids = torch.stack([torch.randperm(E, device="cuda", generator=g)[:k] for _ in range(qlen)]).long()
        w = torch.rand(qlen, k, device="cuda", generator=g)
        out = torch.zeros_like(x)

        def run():
            native.check(lib.ktb200_moe_forward(h, qlen, k, ids.data_ptr(), w.data_ptr(), x.data_ptr(), out.data_ptr(), None, s))
        for _ in range(2):
            run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        n = 5
        e0.record()
        for _ in range(n):
            run()
        e1.record()
        torch.cuda.synchronize()
        counts = torch.bincount(ids.reshape(-1), minlength=E)
        res[qlen] = {"ms": e0.elapsed_time(e1) / n, "tiles": ((counts + 31) // 32).tolist()}
        np.save(os.path.join(outdir, f"{qlen}.npy"), out.view(torch.int16).cpu().numpy())
    if os.environ.get("TRACE"):
        tr = torch.zeros(2 * 3 * 96 * 4, dtype=torch.int64, device="cuda")
        lib.ktb200_debug_grouped(tr.data_ptr()); run(); torch.cuda.synchronize(); lib.ktb200_debug_grouped(None)
        t = tr.cpu().numpy().reshape(2, 3, 96, 4)
        for kname, kk in ((f"gate ({NAMES[gt]}, {KERNEL[gt]})", 0), (f"down ({NAMES[dt]}, {KERNEL[dt]})", 1)):
            t0 = t[kk, 0, 0, 0]
            print(f"--- {kname}, qlen {qlen}: cycles since the producer's first stage; P = wait_group done / smem_free seen / arrived, "
                  f"M = before ab_full / ab_full seen / MMAs + scale-and-add done / arrived")
            for st in range(0, 40):
                P, M = t[kk, 0, st] - t0, t[kk, 1, st] - t0
                print(f"st {st:2d}  P {P[0]:6d} {P[1]:6d} {P[2]:6d} {P[3]:6d} | M {M[0]:6d} {M[1]:6d} {M[2]:6d} {M[3]:6d}")
    lib.ktb200_moe_destroy(h)
    print("RESULT " + json.dumps(res), flush=True)


def bf16_close(got, want):
    """tests/test_gpu_parity.py assert_bf16_close: within 2^-7 of the larger magnitude + 1e-3 of max |want|, > 97 % bit-identical"""
    a = (got.astype(np.uint32) << 16).view(np.float32)
    b = (want.astype(np.uint32) << 16).view(np.float32)
    ok = np.abs(a - b) <= 2.0 ** -7 * np.maximum(np.abs(a), np.abs(b)) + 1e-3 * np.abs(b).max()
    return bool(ok.all()) and float((got == want).mean()) > 0.97, float((got == want).mean())


def main():
    tsets = os.environ.get("TYPES", "q4k,iq1x3,iq1_iq1_iq2").split(",")
    qlens = [int(v) for v in os.environ.get("QLENS", "48,64,256,1024,4096").split(",")]
    reps = int(os.environ.get("REPS", 2))
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print(f"card: {torch.cuda.get_device_name(0)}; nvidia-smi name, power limit, max SM clock: {smi.stdout.strip()}", flush=True)
    arms = {"grouped": {}, "per-pair": {"KTB200_GROUPED_MIN": str(max(qlens) + 1)}}
    if os.environ.get("BASELINE_LIB"):
        arms["baseline"] = {"PROBE_LIB": os.environ["BASELINE_LIB"]}
    tmp = tempfile.mkdtemp(prefix="grouped_probe_")
    ok = True
    for tset in tsets:
        best, refused = {}, {}
        for rep in range(reps):
            for arm, env in arms.items():
                d = os.path.join(tmp, tset, arm)
                os.makedirs(d, exist_ok=True)
                env = dict(os.environ, **env)
                if arm != "grouped" or rep:
                    env.pop("TRACE", None)
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", tset, ",".join(map(str, qlens)), d],
                                   env=env, capture_output=True, text=True)
                lines = r.stdout.splitlines()
                if r.returncode:
                    err = [l[12:] for l in r.stderr.splitlines() if l.startswith("ValueError: ")]
                    if arm != "grouped" and err:   # the library refuses the handle on this arm's route (per-pair kernels)
                        refused[arm] = err[-1]
                        print(f"{tset} {arm}: refused: {err[-1]}")
                        continue
                    print(r.stdout[-2000:], r.stderr[-3000:])
                    raise SystemExit(f"{tset} {arm}: worker failed")
                print("\n".join(l for l in lines if not l.startswith("RESULT ")), end="" if len(lines) < 2 else "\n")
                res = json.loads(next(l for l in lines if l.startswith("RESULT "))[7:])
                for q, v in res.items():
                    b = best.setdefault((arm, int(q)), v)
                    b["ms"] = min(b["ms"], v["ms"])
                    b.setdefault("all", []).append(v["ms"])
        gt, ut, dt = TYPE_SETS[tset]
        E, LAYERS = set_e(tset), set_layers(tset)
        eb = [I * H // 256 * BLOCK[t] for t in (gt, ut, dt)]
        print(f"\n{NAMES[gt]}/{NAMES[ut]}/{NAMES[dt]}  (E {E}, H {H}, I {I}, k {k}, BF16; ms per layer = fastest of {reps}, all reps in brackets)")
        tl = f"tok/s/{LAYERS}L"
        print(f"{'qlen':>6} | {'grouped ms':>22} {tl:>9} {'HBM share':>9} | {'per-pair ms':>22} {tl:>9} | {'speed-up':>8} | outputs")
        for q in qlens:
            gr, pp = best[("grouped", q)], best.get(("per-pair", q))
            tile_bytes = sum(gr["tiles"]) * sum(eb)
            a = np.load(os.path.join(tmp, tset, "grouped", f"{q}.npy")).view(np.uint16)
            if pp:
                close, exact = bf16_close(np.load(os.path.join(tmp, tset, "per-pair", f"{q}.npy")).view(np.uint16), a)
                cmp = f"per-pair {'within' if close else 'OUTSIDE'} bf16 bound ({exact:.2%} bit-identical)"
                ok &= close
            else:
                cmp = f"per-pair refused ({refused['per-pair']})"
            if "baseline" in refused:
                cmp += "; baseline refused"
            elif "baseline" in arms:
                # bit-identical where both builds take the same kernels; otherwise (a route the baseline build lacks) the
                # per-pair bound
                bl = best[("baseline", q)]
                c = np.load(os.path.join(tmp, tset, "baseline", f"{q}.npy")).view(np.uint16)
                same = np.array_equal(c, a)
                close = same or bf16_close(c, a)[0]
                ok &= close
                verdict = "bit-identical" if same else "within bf16 bound" if close else "OUTSIDE bf16 bound"
                cmp += f"; baseline {verdict}, {bl['ms']:.3f} ms [{' '.join(f'{v:.3f}' for v in bl['all'])}]"
            fmt = lambda v: f"{v['ms']:8.3f} [{' '.join(f'{x:.2f}' for x in v['all'])}]"
            ppc = f"{fmt(pp):>22} {q / (LAYERS * pp['ms']) * 1e3:9.0f} | {pp['ms'] / gr['ms']:7.2f}x" if pp else f"{'-':>22} {'-':>9} | {'-':>8}"
            print(f"{q:6d} | {fmt(gr):>22} {q / (LAYERS * gr['ms']) * 1e3:9.0f} {tile_bytes / HBM * 1e3 / gr['ms']:9.1%} | {ppc} | {cmp}", flush=True)
    print("all outputs agree" if ok else "OUTPUT MISMATCH")
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--worker":
        worker(sys.argv[2], [int(v) for v in sys.argv[3].split(",")], sys.argv[4])
    else:
        main()
