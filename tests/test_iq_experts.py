"""IQ1_S and IQ2_XXS routed experts (ggml codebook i-quants): codebook header, format and dot-product pins against
gguf-py and the reference's integer formulas, C-ABI and host checks, and the sm_90a kernels against the float64 oracle
in tests/iq_oracle.py."""
import ctypes as C
import importlib.util
import os
import types

import numpy as np
import pytest
import torch

import iq_oracle as oq
from ktransformers_b200 import native

IQ1, IQ2 = native.GGML_IQ1_S, native.GGML_IQ2_XXS
Q4K, Q6K = native.GGML_Q4_K, native.GGML_Q6_K
F32, F16, BF16 = native.GGML_F32, native.GGML_F16, native.GGML_BF16
FP_TOL = 1e-3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------ codebook header (CPU)
def test_generator_reproduces_header():
    spec = importlib.util.spec_from_file_location("make_iq_tables", os.path.join(ROOT, "tests", "golden", "make_iq_tables.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    with open(os.path.join(ROOT, "ktransformers_b200", "csrc", "iq_tables.h"), newline="") as f:
        assert f.read() == mod.render()


def test_tables_match_ggml_constants():
    # first entries of ggml's iq1s_grid (0xffffffffffffffff, 0xffffffffffffff01) and iq2xxs_grid (0x0808080808080808),
    # and ksigns_iq2xs: bit 7 = parity of the low 7 bits
    assert (oq.IQ1S_GRID[0] == -1).all() and list(oq.IQ1S_GRID[1]) == [1] + [-1] * 7
    assert (oq.IQ2XXS_GRID[0] == 8).all()
    k = np.arange(128)
    par = np.array([bin(i).count("1") & 1 for i in k])
    assert np.array_equal(oq.KSIGNS, k | (par << 7))


# ------------------------------------------------------------------------------------------------ format (CPU)
def _blocks(t, n, seed):
    return oq.random_blocks(t, n, np.random.default_rng(seed))


def test_random_blocks_cover_every_field():
    b1 = _blocks(IQ1, 512, 1)
    qh = b1[:, 34:50].copy().view(np.uint16)
    assert set(((qh >> 12) & 7).reshape(-1).tolist()) == set(range(8))
    assert set((qh >> 15).reshape(-1).tolist()) == {0, 1}
    for l in range(4):
        assert set(((qh >> (3 * l)) & 7).reshape(-1).tolist()) == set(range(8))
    b2 = _blocks(IQ2, 512, 2)
    aux1 = b2[:, 2:66].copy().view(np.uint32).reshape(-1, 8, 2)[:, :, 1]
    assert set((aux1 >> 28).reshape(-1).tolist()) == set(range(16))
    for l in range(4):
        assert set(((aux1 >> (7 * l)) & 127).reshape(-1).tolist()) == set(range(128))


@pytest.mark.parametrize("t", [IQ1, IQ2])
def test_oracle_dequant_matches_gguf_bit_for_bit(t):
    import gguf
    b = _blocks(t, 512, 3 + t)
    ref = gguf.quants.dequantize(b.reshape(-1), gguf.GGMLQuantizationType(t))
    got = oq.dequant(t, b)
    assert np.array_equal(got.view(np.uint32), ref.astype(np.float32).view(np.uint32))


def _q8(n_blocks, seed):
    from oracle.bindings import Oracle
    x = np.random.default_rng(seed).standard_normal(n_blocks * 256).astype(np.float32)
    return Oracle().from_float(x, 15)


@pytest.mark.parametrize("t", [IQ1, IQ2])
def test_superblock_term_is_the_integer_formula(t):
    w, q8 = _blocks(t, 256, 10 + t), _q8(256, 11 + t)
    S = oq.superblock_ints(t, w, q8)
    assert np.abs(S).max() < 2 ** 22
    dw = w[:, 0:2].copy().view(np.float16).astype(np.float32).reshape(-1)
    d = (dw * oq.q8k_fields(q8)[0]).astype(np.float32)
    if t == IQ1:
        # (d dx) (sumi + 0.125 sumi1) == (d dx) (S / 8) exactly: S/8 is representable
        assert np.array_equal(oq.superblock_terms(t, w, q8), (d * (S.astype(np.float32) / np.float32(8))).astype(np.float32))
    else:
        assert np.array_equal(oq.superblock_terms(t, w, q8), (d * S.astype(np.float32)).astype(np.float32))


@pytest.mark.parametrize("t", [IQ1, IQ2])
def test_vec_dot_within_fp32_rounding_of_float64(t):
    rng = np.random.default_rng(20 + t)
    for _ in range(8):
        nb = 28
        w, q8 = oq.random_blocks(t, nb, rng), _q8(nb, int(rng.integers(1 << 30)))
        got = float(oq.vec_dot(t, w, q8))
        ref = float(np.dot(oq.dequant(t, w).astype(np.float64), oq.q8k_to_f64(q8)))
        terms = np.abs(oq.superblock_terms(t, w, q8).astype(np.float64)).sum()
        assert abs(got - ref) <= 4 * nb * 2 ** -24 * max(terms, 1e-30), (got, ref)


# ------------------------------------------------------------------------------------------------ C-ABI and host (CPU)
def test_type_size_and_block():
    lib = native.lib()
    assert lib.ktb200_type_size(IQ1) == 50 and lib.ktb200_blck_size(IQ1) == 256
    assert lib.ktb200_type_size(IQ2) == 66 and lib.ktb200_blck_size(IQ2) == 256


def test_type_sets():
    from ktransformers_b200.util import custom_gguf as cg
    assert cg.B200_WEIGHT_TYPES == {"Q2_K", "Q3_K", "Q4_K", "Q5_K", "Q6_K", "IQ4_XS"}
    assert cg.B200_EXPERT_TYPES == cg.B200_WEIGHT_TYPES | {"IQ1_S", "IQ2_XXS"}
    assert {"IQ1_S", "IQ2_XXS"} <= cg.B200_DEQUANT_TYPES


@pytest.mark.parametrize("t,name", [(IQ1, "IQ1_S"), (IQ2, "IQ2_XXS")])
def test_linear_and_mlp_reject_with_type_name(t, name):
    lib = native.lib()
    h = C.c_void_p()
    assert lib.ktb200_linear_create(512, 256, 1 << 20, t, BF16, 16, 0, C.byref(h)) == native.EINVAL
    assert name in lib.ktb200_last_error().decode()
    assert lib.ktb200_mlp_create(512, 256, 1 << 20, 1 << 20, 1 << 20, Q4K, Q4K, t, BF16, 16, 0, C.byref(h)) == native.EINVAL
    assert name in lib.ktb200_last_error().decode()


def test_moe_create_rejects_shapes():
    lib = native.lib()
    h = C.c_void_p()
    cfg = native.MoeConfig(8, 2, 7000, 2048, 64, 10, 16, 1, 1 << 20, 1 << 20, 1 << 20, IQ1, IQ1, IQ2, BF16, 0)
    assert lib.ktb200_moe_create(C.byref(cfg), 0, C.byref(h)) == native.EINVAL and not h.value


@pytest.mark.parametrize("expert_types", [(IQ1, IQ1, IQ2), (Q4K, Q4K, IQ1), (native.RAWINT4_G32,) * 3, (native.GGML_Q5_K, native.GGML_Q5_K, Q6K)])
def test_attach_expert_parallel_refuses(expert_types):
    from ktransformers_b200.operators.expert_parallel import attach_expert_parallel

    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self._block_handles = None
            self.key = "blk.3"
            self.experts = types_ns

    types_ns = _ExpertsNs(*expert_types)
    model = torch.nn.Sequential(Block())
    with pytest.raises(ValueError, match="expert-parallel"):
        attach_expert_parallel(model, 512, BF16, "cpu")


class _ExpertsNs:
    def __init__(self, g, u, d):
        self.generate_experts = types.SimpleNamespace(gate_type=g, up_type=u, down_type=d)


# ------------------------------------------------------------------------------------------------ GPU helpers
def _dev_blocks(t, n_elems, seed, scale=None):
    """random blocks of any supported expert type on the device"""
    if t in (IQ1, IQ2):
        d = scale if scale is not None else (1 / 64 if t == IQ1 else 1 / 512)
        return torch.from_numpy(oq.random_blocks(t, n_elems // 256, np.random.default_rng(seed), d).reshape(-1)).cuda()
    from ktransformers_b200.util.synth import synth_blocks
    return synth_blocks(t, n_elems, "cuda", seed)


def _dequant_f64(t, blocks_np, rows, cols):
    import gguf
    return gguf.quants.dequantize(blocks_np, gguf.GGMLQuantizationType(t)).astype(np.float64).reshape(rows, cols)


class _Experts:
    def __init__(self, E, H, I, gt, ut, dt, seed):
        self.E, self.H, self.I, self.types = E, H, I, (gt, ut, dt)
        self.w = [_dev_blocks(t, E * r * c, seed + i) for i, (t, r, c) in enumerate(((gt, I, H), (ut, I, H), (dt, H, I)))]
        # host copies in ggml layout: loading a handle re-tiles Q6_K tensors in place on the device
        self.host = [b.cpu().numpy().reshape(E, -1) for b in self.w]

    def expert(self, e):
        return tuple(_dequant_f64(t, h[e], r, c)
                     for h, t, (r, c) in zip(self.host, self.types, ((self.I, self.H), (self.I, self.H), (self.H, self.I))))

    def moe(self, k, hidden_type, max_tokens=64, use_silu=1, E=None, lo=0, offset=0):
        from gpu_util import Moe
        E = E or self.E
        sl = [b.view(self.E, -1)[lo:lo + E].reshape(-1) for b in self.w]
        return Moe(E, k, self.H, self.I, *sl, *self.types, hidden_type, max_tokens=max_tokens, use_silu=use_silu, offset=offset)


def _x(T, H, seed, hidden_type):
    """(kernel input in its numpy carrier, the same values as float32)"""
    x = np.random.default_rng(seed).standard_normal((T, H)).astype(np.float32)
    if hidden_type == BF16:
        from oracle.bindings import f32_to_bf16_bits, bf16_to_f32
        b = f32_to_bf16_bits(x)
        return b, bf16_to_f32(b)
    if hidden_type == F16:
        h = x.astype(np.float16)
        return h, h.astype(np.float32)
    return x, x


def _to_f64(got, hidden_type):
    if hidden_type == BF16:
        from oracle.bindings import bf16_to_f32
        return bf16_to_f32(got).astype(np.float64)
    return got.astype(np.float64)


# half an ulp of the output type, relative: BF16 / F16 outputs are the fp32 result rounded once more
ROUND_REL = {F32: 0.0, F16: 2.0 ** -11, BF16: 2.0 ** -8}


def _check(got, ref, hidden_type, what=""):
    """|got - ref| <= FP_TOL * max|ref| plus the rounding of the output to the hidden type"""
    err = np.abs(_to_f64(got, hidden_type) - ref)
    bound = FP_TOL * np.abs(ref).max() + ROUND_REL[hidden_type] * np.abs(ref)
    assert (err <= bound).all(), (what, (err - bound).max(), err.max(), np.abs(ref).max())


def _ids(T, E, k, rng):
    return np.stack([rng.permutation(E)[:k] for _ in range(T)]).astype(np.int64)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("t", [IQ1, IQ2])
def test_dequantize_bit_exact(t):
    from gpu_util import dequantize
    import gguf
    b = oq.random_blocks(t, 600, np.random.default_rng(30 + t))
    ref = gguf.quants.dequantize(b.reshape(-1), gguf.GGMLQuantizationType(t)).astype(np.float32)
    n = ref.size
    assert np.array_equal(dequantize(b.reshape(-1), t, n, F32).numpy().view(np.uint32), ref.view(np.uint32))
    assert torch.equal(dequantize(b.reshape(-1), t, n, BF16), torch.from_numpy(ref).to(torch.bfloat16))
    assert torch.equal(dequantize(b.reshape(-1), t, n, F16), torch.from_numpy(ref).to(torch.float16))


TYPE_MIXES = {
    "iq1x3": (IQ1, IQ1, IQ1), "iq2x3": (IQ2, IQ2, IQ2), "iq1_iq1_iq2": (IQ1, IQ1, IQ2),
    "iq1_iq1_q6k": (IQ1, IQ1, Q6K), "iq2_iq2_q4k": (IQ2, IQ2, Q4K), "q4k_q4k_iq1": (Q4K, Q4K, IQ1),
    "q4k_q4k_iq2": (Q4K, Q4K, IQ2), "iq1_iq2_iq1": (IQ1, IQ2, IQ1), "q4k_iq1_q6k": (Q4K, IQ1, Q6K),
}


@pytest.mark.gpu
@pytest.mark.parametrize("mix", sorted(TYPE_MIXES))
@pytest.mark.parametrize("qlen", [1, 3, 8, 47, 64])
def test_moe_forward_type_mixes(oracle, mix, qlen):
    E, k, H, I = 8, 4, 1024, 512
    ex = _Experts(E, H, I, *TYPE_MIXES[mix], 100 + qlen)
    m = ex.moe(k, F32)
    rng = np.random.default_rng(qlen)
    ids, w = _ids(qlen, E, k, rng), rng.random((qlen, k)).astype(np.float32)
    x, xf = _x(qlen, H, qlen, F32)
    _check(m.forward(ids, w, x), oq.moe_forward(oracle, xf, ids, w, ex.expert, E), F32, mix)
    m.close()


# (H, I): which kernels a same-type all-IQ handle takes
PATHS = {(1024, 512): ("rows_bulk_iq_kernel", "reduce_bulk_kernel<ktb::BulkIQ"),     # both on the bulk-copy ring
         (2048, 1024): ("rows_bulk_iq_kernel", "reduce_bulk_kernel<ktb::BulkIQ"),    # the same with 8 / 4 blocks per row
         (512, 256): ("rows_kernel<ktb::FmtGenK", "reduce_kernel<ktb::FmtGenK")}     # 2 blocks per row, 1 per down row
KERNEL_MIXES = ["iq1x3", "iq2x3"]

# every (mix, shape) of test_kernels_that_ran in ONE torch.profiler session, in an interpreter of its own: after other
# profiler sessions in the same process a session can come back without some of its kernels.  Kernels are attributed to
# the call that launched them by launch order.
_CENSUS = r"""
import json, sys
import numpy as np, torch
sys.path[:0] = sys.argv[1:]
from torch.profiler import ProfilerActivity, profile
from ktransformers_b200 import native
from test_iq_experts import KERNEL_MIXES, PATHS, TYPE_MIXES, _Experts, _ids, _x
cases = []
for mix in KERNEL_MIXES:
    for H, I in sorted(PATHS):
        ex = _Experts(8, H, I, *TYPE_MIXES[mix], 60)
        rng = np.random.default_rng(61)
        cases.append((f"{mix} {H} {I}", ex, ex.moe(4, 0), _ids(3, 8, 4, rng), rng.random((3, 4)).astype(np.float32), _x(3, H, 62, 0)[0]))
torch.cuda.synchronize()
counts = []
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _, _, m, ids, w, x in cases:
        n0 = native.launch_count()
        m.forward(ids, w, x)
        torch.cuda.synchronize()
        counts.append(native.launch_count() - n0)
names = [e.name for e in sorted((e for e in prof.events() if "ktb::" in e.name), key=lambda e: e.time_range.start)]
assert len(names) == sum(counts), f"{len(names)} library kernels recorded, {sum(counts)} launched: {names}"
res, i = {}, 0
for (key, *_), n in zip(cases, counts):
    res[key] = (n, names[i:i + n])
    i += n
print("CENSUS " + json.dumps(res))
"""


@pytest.fixture(scope="module")
def kernel_census():
    import json
    import subprocess
    import sys
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CENSUS, os.path.join(ROOT, "tests"), ROOT]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return json.loads(next(l for l in r.stdout.splitlines() if l.startswith("CENSUS "))[7:])


@pytest.mark.gpu
@pytest.mark.parametrize("shape", sorted(PATHS))
@pytest.mark.parametrize("mix", KERNEL_MIXES)
def test_kernels_that_ran(oracle, kernel_census, shape, mix):
    """the bulk-copy kernels take shapes whose 2-row units / 4-row items are 16-byte aligned; other shapes the generic ones
    (kernel names from the census above; the launch count and the result checked here as well)"""
    H, I = shape
    E, k, T = 8, 4, 3
    ex = _Experts(E, H, I, *TYPE_MIXES[mix], 60)
    m = ex.moe(k, F32)
    rng = np.random.default_rng(61)
    ids, w = _ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    x, xf = _x(T, H, 62, F32)
    launched, names = kernel_census[f"{mix} {H} {I}"]
    assert launched == 2
    n0 = native.launch_count()
    got = m.forward(ids, w, x)
    assert native.launch_count() - n0 == 2
    fmt = "BulkIQ1S" if mix == "iq1x3" else "BulkIQ2XXS"
    gu, dn = PATHS[shape]
    assert any(gu in n and (fmt in n or "FmtGenK" in n) for n in names), names
    assert any(dn in n for n in names), names
    if gu == "rows_bulk_iq_kernel":
        assert any(fmt in n for n in names) and not any("FmtGenK" in n for n in names), names
    _check(got, oq.moe_forward(oracle, xf, ids, w, ex.expert, E), F32)
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("hidden_type", [F32, F16, BF16])
@pytest.mark.parametrize("use_silu", [1, 0])
@pytest.mark.parametrize("qlen", [1, 8])
def test_moe_forward_hidden_types_and_activations(oracle, hidden_type, use_silu, qlen):
    E, k, H, I = 8, 3, 1024, 256
    ex = _Experts(E, H, I, IQ1, IQ1, IQ2, 7)
    m = ex.moe(k, hidden_type, use_silu=use_silu)
    rng = np.random.default_rng(40 + qlen)
    ids, w = _ids(qlen, E, k, rng), rng.random((qlen, k)).astype(np.float32)
    x, xf = _x(qlen, H, 41, hidden_type)
    _check(m.forward(ids, w, x), oq.moe_forward(oracle, xf, ids, w, ex.expert, E, bool(use_silu)), hidden_type)
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["iq1x3", "iq1_iq1_iq2"])
def test_moe_forward_v3_shapes(oracle, mix):
    """DeepSeek-V3/R1 routed experts: E=256, H=7168, I=2048, k=8; qlen 8 over 16 experts and qlen 1; BF16 hidden"""
    E, k, H, I = 256, 8, 7168, 2048
    ex = _Experts(E, H, I, *TYPE_MIXES[mix], 2026)
    rng = np.random.default_rng(8)
    hit = rng.permutation(E)[:16]
    ids = np.stack([rng.permutation(hit)[:k] for _ in range(8)]).astype(np.int64)
    w = rng.random((8, k)).astype(np.float32)
    x, xf = _x(8, H, 9, BF16)
    ref = oq.moe_forward(oracle, xf, ids, w, ex.expert, E)
    m = ex.moe(k, BF16, max_tokens=8)
    _check(m.forward(ids, w, x), ref, BF16, "qlen 8")
    _check(m.forward(ids[:1], w[:1], x[:1]), ref[:1], BF16, "qlen 1")
    m.close()


@pytest.mark.gpu
def test_expert_id_offset_shards_and_skipped_ids(oracle):
    E, k, H, I, T = 8, 4, 512, 256, 5
    ex = _Experts(E, H, I, IQ1, IQ1, IQ2, 9)
    rng = np.random.default_rng(3)
    ids, w = _ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    ids[0, 1], ids[2, 0], ids[3, 3] = -1, E, E + 7
    x, xf = _x(T, H, 4, F32)
    full = ex.moe(k, F32).forward(ids, w, x)
    parts = [ex.moe(k, F32, E=4, lo=lo, offset=lo).forward(ids, w, x) for lo in (0, 4)]
    ref = oq.moe_forward(oracle, xf, ids, w, ex.expert, E)
    _check(full, ref, F32)
    assert np.abs((parts[0] + parts[1]).astype(np.float64) - full).max() <= 1e-6 * np.abs(ref).max()


@pytest.mark.gpu
def test_rows_beyond_bsz_untouched_eager_and_graph():
    from gpu_util import stream
    E, k, H, I, T = 8, 4, 512, 256, 8
    ex = _Experts(E, H, I, IQ1, IQ2, IQ1, 5)   # mixed gate/up: the generic per-pair kernels
    m = ex.moe(k, BF16)
    rng = np.random.default_rng(1)
    ids = torch.from_numpy(_ids(T, E, k, rng)).cuda()
    w = torch.from_numpy(rng.random((T, k)).astype(np.float32)).cuda()
    x = torch.randn((T, H), device="cuda").to(torch.bfloat16)
    bsz = torch.tensor([5], dtype=torch.int32, device="cuda")
    lib = native.lib()

    def call(out):
        native.check(lib.ktb200_moe_forward(m.h, T, k, ids.data_ptr(), w.data_ptr(), x.data_ptr(), out.data_ptr(), bsz.data_ptr(),
                                            torch.cuda.current_stream().cuda_stream))

    full = torch.zeros((T, H), dtype=torch.bfloat16, device="cuda")
    native.check(lib.ktb200_moe_forward(m.h, T, k, ids.data_ptr(), w.data_ptr(), x.data_ptr(), full.data_ptr(), None, stream()))
    out = torch.full((T, H), 1234.5, dtype=torch.bfloat16, device="cuda")
    call(out)
    torch.cuda.synchronize()
    assert torch.equal(out[:5], full[:5]) and (out[5:] == 1234.5).all()
    # one capture, replayed with a smaller batch
    s = torch.cuda.Stream()
    out2 = torch.full((T, H), 1234.5, dtype=torch.bfloat16, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            call(out2)
    torch.cuda.synchronize()
    out2.fill_(1234.5)
    bsz.fill_(3)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out2[:3], full[:3]) and (out2[3:] == 1234.5).all()
    m.close()


def _q4k_mlp(H, I, hidden_type):
    from gpu_util import Mlp
    from ktransformers_b200.util.synth import synth_blocks
    return Mlp(H, I, synth_blocks(Q4K, I * H, "cuda", 1), synth_blocks(Q4K, I * H, "cuda", 2), synth_blocks(Q4K, H * I, "cuda", 3),
               Q4K, Q4K, Q4K, hidden_type)


@pytest.mark.gpu
def test_forward_shared_with_q4k_shared_expert():
    from gpu_util import moe_forward_shared, mlp_forward
    from ktransformers_b200.util.synth import synth_blocks
    E, k, H, I, T = 8, 4, 4096, 512, 3
    ex = _Experts(E, H, I, IQ1, IQ1, IQ2, 12)
    m = ex.moe(k, F32)
    mlp = _q4k_mlp(H, I, F32)
    rng = np.random.default_rng(13)
    ids, w = _ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    x, _ = _x(T, H, 14, F32)
    routed = m.forward(ids, w, x)
    shared = mlp_forward(H, I, *mlp.keep, Q4K, Q4K, Q4K, F32, x)
    assert np.array_equal(moe_forward_shared(m, mlp, ids, w, x), (routed + shared).astype(np.float32))
    mlp.close()
    m.close()


@pytest.mark.gpu
def test_moe_block_forward_takes_the_separate_launches():
    from gpu_util import Gate, moe_block_forward, gate_forward, moe_forward_shared
    E, k, H, I, T = 16, 4, 4096, 512, 3
    ex = _Experts(E, H, I, IQ1, IQ1, IQ2, 11)
    m = ex.moe(k, BF16)
    mlp = _q4k_mlp(H, 256, BF16)
    rng = np.random.default_rng(5)
    W, b = rng.standard_normal((E, H)).astype(np.float32), rng.standard_normal(E).astype(np.float32)
    gate = Gate(W, b, k, 1, 1, hidden_type=BF16)
    x, _ = _x(T, H, 6, BF16)
    out, idx, wt = moe_block_forward(gate, m, mlp, x)
    idx2, wt2, _ = gate_forward(x, W, b, k, 1, 1, hidden_type=BF16)
    assert np.array_equal(idx, idx2) and np.array_equal(wt, wt2)
    assert np.array_equal(out, moe_forward_shared(m, mlp, idx2, wt2, x))
    mlp.close()
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("types,name", [((IQ1, IQ1, IQ1), "IQ1_S"), ((Q4K, Q4K, IQ2), "IQ2_XXS")])
def test_forward_ep_refuses(types, name):
    E, k, H, I = 8, 2, 4096, 512
    m = _Experts(E, H, I, *types, 13).moe(k, BF16)
    mlp = _q4k_mlp(H, I, BF16)
    ids = torch.zeros((1, k), dtype=torch.int64, device="cuda")
    wt = torch.ones((1, k), device="cuda")
    x = torch.zeros((1, H), dtype=torch.bfloat16, device="cuda")
    part, sh = torch.zeros((1, H), device="cuda"), torch.zeros((H,), dtype=torch.bfloat16, device="cuda")
    rc = native.lib().ktb200_moe_forward_ep(m.h, mlp.h, 1, k, ids.data_ptr(), wt.data_ptr(), x.data_ptr(), part.data_ptr(), 0,
                                            sh.data_ptr(), None, torch.cuda.current_stream().cuda_stream)
    assert rc == native.EINVAL and name in native.lib().ktb200_last_error().decode()
    mlp.close()
    m.close()


def _wrapper(**kw):
    from ktransformers_b200.kt_moe_wrapper import KTMoEWrapper
    args = dict(layer_idx=0, num_experts=8, num_experts_per_tok=3, hidden_size=512, moe_intermediate_size=256,
                gpu_experts_mask=None, method="B200_GGUF", chunked_prefill_size=16)
    args.update(kw)
    return KTMoEWrapper(**args)


def _wrapper_check(oracle, wr, blocks, p2l, mask, E, k, H, I, types):
    rng = np.random.default_rng(22)
    T = 5
    ids, w = _ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    xb, xf = _x(T, H, 23, BF16)
    x = torch.from_numpy(xb.view(np.int16)).view(torch.bfloat16).cuda()
    out = wr.forward(x, torch.from_numpy(ids).cuda(), torch.from_numpy(w).cuda())
    torch.cuda.synchronize()
    got = out.cpu().view(torch.int16).numpy().view(np.uint16)

    def expert(pslot):
        le = int(p2l[pslot])
        return tuple(_dequant_f64(t, blocks[n][le].reshape(-1), r, c)
                     for n, t, (r, c) in zip(("gate", "up", "down"), types, ((I, H), (I, H), (H, I))))
    ids_m = np.where(mask.numpy()[ids], -1, ids)
    _check(got, oq.moe_forward(oracle, xf, ids_m, w, expert, E), BF16)


@pytest.mark.gpu
def test_ktmoe_wrapper_from_tensors(oracle):
    E, k, H, I = 8, 3, 512, 256
    types = (IQ1, IQ1, IQ2)
    rng = np.random.default_rng(21)
    blocks = {n: oq.random_blocks(t, E * r * c // 256, rng, 1 / 64 if t == IQ1 else 1 / 512).reshape(E, r, -1)
              for n, t, (r, c) in zip(("gate", "up", "down"), types, ((I, H), (I, H), (H, I)))}
    p2l = torch.tensor([3, 0, 7, 1, 6, 2, 5, 4])
    mask = torch.zeros(E, dtype=torch.bool)
    mask[[2, 5]] = True
    wr = _wrapper(gpu_experts_mask=mask)
    wr.load_weights_from_tensors(*(torch.from_numpy(blocks[n]) for n in ("gate", "up", "down")), p2l, ggml_types=types)
    _wrapper_check(oracle, wr, blocks, p2l, mask, E, k, H, I, types)


@pytest.mark.gpu
def test_ktmoe_wrapper_from_gguf(oracle, tmp_path):
    import gguf
    E, k, H, I = 8, 3, 512, 256
    types = (IQ1, IQ2, IQ1)
    rng = np.random.default_rng(31)
    wtr = gguf.GGUFWriter(str(tmp_path / "iq.gguf"), "deepseek2")
    blocks = {}
    for n, t, (r, c) in zip(("gate", "up", "down"), types, ((I, H), (I, H), (H, I))):
        blocks[n] = oq.random_blocks(t, E * r * c // 256, rng, 1 / 64 if t == IQ1 else 1 / 512).reshape(E, r, -1)
        wtr.add_tensor(f"blk.0.ffn_{n}_exps.weight", blocks[n], raw_dtype=gguf.GGMLQuantizationType(t))
    wtr.write_header_to_file()
    wtr.write_kv_data_to_file()
    wtr.write_tensors_to_file()
    wtr.close()
    p2l = torch.tensor([1, 0, 3, 2, 5, 4, 7, 6])
    mask = torch.zeros(E, dtype=torch.bool)
    mask[[0, 6]] = True
    wr = _wrapper(gpu_experts_mask=mask, weight_path=str(tmp_path), key_template="blk.{layer}")
    wr.load_weights(p2l)
    _wrapper_check(oracle, wr, blocks, p2l, mask, E, k, H, I, types)
