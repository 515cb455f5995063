"""IQ3_XXS and IQ3_S routed experts (ggml types 18 and 21, the experts of llama.cpp's 3-bit i-quant DeepSeek files): format and
dot-product pins against gguf-py and the reference's integer formula, C-ABI and host checks, and the sm_90a kernels (the bulk-copy
decode kernels, the generic per-pair kernels, grouped_gemm_kernel<9> and <10>) against the float64 oracle, through every caller."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import iq3_oracle as o3
import iq_oracle as oq
import test_iq_experts as tie
from ktransformers_b200 import native
from test_iq_experts import _check, _ids, _q4k_mlp, _x
from test_iq_grouped import IQ_MIN, _hard_ids, _moe_ref

IQ3XXS, IQ3S, IQ2 = native.GGML_IQ3_XXS, native.GGML_IQ3_S, native.GGML_IQ2_XXS
IQ3 = (IQ3XXS, IQ3S)
NAMES = {IQ3XXS: "IQ3_XXS", IQ3S: "IQ3_S"}
Q4K, Q6K = native.GGML_Q4_K, native.GGML_Q6_K
F32, F16, BF16 = native.GGML_F32, native.GGML_F16, native.GGML_BF16
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ------------------------------------------------------------------------------------------------ format (CPU)
def test_random_blocks_cover_every_field():
    b = o3.random_blocks(IQ3XXS, 512, np.random.default_rng(1))
    aux = b[:, 66:98].copy().view(np.uint32)
    assert set((aux >> 28).reshape(-1).tolist()) == set(range(16))
    for l in range(4):
        assert set(((aux >> (7 * l)) & 127).reshape(-1).tolist()) == set(range(128))
    assert set(b[:, 2:66].reshape(-1).tolist()) == set(range(256))
    b = o3.random_blocks(IQ3S, 512, np.random.default_rng(2))
    idx = b[:, 2:66].astype(np.int64) | (((b[:, 66:74, None] >> np.arange(8)) & 1).reshape(-1, 64).astype(np.int64) << 8)
    assert set(idx.reshape(-1).tolist()) == set(range(512))
    for sh in (0, 4):
        assert set(((b[:, 106:110] >> sh) & 15).reshape(-1).tolist()) == set(range(16))
    assert set(b[:, 74:106].reshape(-1).tolist()) == set(range(256))
    for t in IQ3:
        d = o3.fields(t, o3.random_blocks(t, 64, np.random.default_rng(t)))[0]
        assert (d >= 0.75).all() and (d < 1.25).all()


@pytest.mark.parametrize("t", IQ3)
def test_oracle_dequant_matches_gguf_bit_for_bit(t):
    import gguf
    b = o3.random_blocks(t, 512, np.random.default_rng(3 + t))
    ref = gguf.quants.dequantize(b.reshape(-1), gguf.GGMLQuantizationType(t)).astype(np.float32)
    assert np.array_equal(o3.dequant(t, b).view(np.uint32), ref.view(np.uint32))


def test_generator_reproduces_header():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_iq3_tables", os.path.join(ROOT, "tests", "golden", "make_iq3_tables.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    with open(os.path.join(ROOT, "ktransformers_b200", "csrc", "iq3_tables.h"), newline="") as f:
        assert f.read() == mod.render()


def test_codebooks_match_ggml_constants():
    # first and last entries of ggml's iq3xxs_grid (0x04040404, 0x3e341c04) and iq3s_grid (0x01010101, 0x0f0f0101)
    assert list(o3.IQ3XXS_GRID[0]) == [4, 4, 4, 4] and list(o3.IQ3XXS_GRID[255]) == [4, 28, 52, 62]
    assert list(o3.IQ3S_GRID[0]) == [1, 1, 1, 1] and list(o3.IQ3S_GRID[511]) == [1, 1, 15, 15]
    assert o3.IQ3XXS_GRID.min() == 4 and o3.IQ3XXS_GRID.max() == 62 and o3.IQ3S_GRID.min() == 1 and o3.IQ3S_GRID.max() == 15
    assert (o3.IQ3XXS_GRID % 2 == 0).all() and (o3.IQ3S_GRID % 2 == 1).all()


def _q8(n_blocks, seed):
    from oracle.bindings import Oracle
    x = np.random.default_rng(seed).standard_normal(n_blocks * 256).astype(np.float32)
    return Oracle().from_float(x, 15)


@pytest.mark.parametrize("t", IQ3)
def test_superblock_term_is_the_integer_formula(t):
    """IQ3_XXS: ((d / 4) dx) S == 0.25 ((d dx) S) exactly (a power-of-two scale); IQ3_S: (d dx) S; S the exact integer"""
    w, q8 = o3.random_blocks(t, 256, np.random.default_rng(10 + t)), _q8(256, 11 + t)
    S = o3.superblock_ints(t, w, q8)
    assert np.abs(S).max() < 2 ** 24
    _, ls, v = o3.fields(t, w)
    q = oq.q8k_fields(q8)[1].reshape(-1, 8, 32)
    assert np.array_equal(S, sum(ls[:, ib] * (v[:, ib] * q[:, ib]).sum(axis=1) for ib in range(8)))
    dd = (o3.fields(t, w)[0] * oq.q8k_fields(q8)[0]).astype(np.float32)
    ref = (dd * S.astype(np.float32)).astype(np.float32)
    if t == IQ3XXS:
        ref = (ref * np.float32(0.25)).astype(np.float32)
    assert np.array_equal(o3.superblock_terms(t, w, q8), ref)


@pytest.mark.parametrize("t", IQ3)
def test_vec_dot_within_fp32_rounding_of_float64(t):
    rng = np.random.default_rng(20 + t)
    for _ in range(8):
        nb = 28
        w, q8 = o3.random_blocks(t, nb, rng), _q8(nb, int(rng.integers(1 << 30)))
        got = float(o3.vec_dot(t, w, q8))
        ref = float(np.dot(o3.dequant(t, w).astype(np.float64), oq.q8k_to_f64(q8)))
        terms = np.abs(o3.superblock_terms(t, w, q8).astype(np.float64)).sum()
        assert abs(got - ref) <= 4 * nb * 2 ** -24 * max(terms, 1e-30), (got, ref)


# ------------------------------------------------------------------------------------------------ C-ABI and host (CPU)
def test_type_size_and_block():
    lib = native.lib()
    assert lib.ktb200_type_size(IQ3XXS) == 98 and lib.ktb200_blck_size(IQ3XXS) == 256
    assert lib.ktb200_type_size(IQ3S) == 110 and lib.ktb200_blck_size(IQ3S) == 256


def test_type_sets():
    from ktransformers_b200.util import custom_gguf as cg
    assert cg.B200_WEIGHT_TYPES == {"Q2_K", "Q3_K", "Q4_K", "Q5_K", "Q6_K", "IQ4_XS"}
    assert cg.B200_EXPERT_TYPES == cg.B200_WEIGHT_TYPES | {"IQ1_S", "IQ2_XXS"}
    assert cg.B200_ROUTED_EXPERT_TYPES == cg.B200_EXPERT_TYPES | {"IQ1_M"}
    assert cg.B200_EXPERT_LOAD_TYPES == cg.B200_ROUTED_EXPERT_TYPES | {"IQ3_XXS", "IQ3_S"}
    assert {"IQ3_XXS", "IQ3_S"} <= cg.B200_DEQUANT_TYPES


@pytest.mark.parametrize("t", IQ3)
def test_linear_and_mlp_reject_with_type_name(t):
    lib = native.lib()
    h = C.c_void_p()
    assert lib.ktb200_linear_create(512, 256, 1 << 20, t, BF16, 16, 0, C.byref(h)) == native.EINVAL
    assert NAMES[t] in lib.ktb200_last_error().decode()
    assert lib.ktb200_mlp_create(512, 256, 1 << 20, 1 << 20, 1 << 20, Q4K, Q4K, t, BF16, 16, 0, C.byref(h)) == native.EINVAL
    assert NAMES[t] in lib.ktb200_last_error().decode()


@pytest.mark.parametrize("types", [(IQ3XXS, IQ3XXS, IQ3S), (IQ3S, IQ3S, IQ3S)])
def test_moe_create_accepts_the_types(types):
    """validation runs before any CUDA call: an IQ3 handle with a bad shape fails on the shape, not on the type"""
    lib = native.lib()
    h = C.c_void_p()
    cfg = native.MoeConfig(8, 2, 7000, 2048, 64, 10, 16, 1, 1 << 20, 1 << 20, 1 << 20, *types, BF16, 0)
    assert lib.ktb200_moe_create(C.byref(cfg), 0, C.byref(h)) == native.EINVAL and not h.value
    err = lib.ktb200_last_error().decode()
    assert "unsupported ggml weight type" not in err and "multiples of 256" in err


@pytest.mark.parametrize("expert_types", [(IQ3XXS, IQ3XXS, IQ3S), (IQ3S, IQ3S, IQ3S), (Q4K, Q4K, IQ3XXS)])
def test_attach_expert_parallel_refuses(expert_types):
    from ktransformers_b200.operators.expert_parallel import attach_expert_parallel

    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self._block_handles = None
            self.key = "blk.3"
            self.experts = tie._ExpertsNs(*expert_types)

    with pytest.raises(ValueError, match="expert-parallel"):
        attach_expert_parallel(torch.nn.Sequential(Block()), 512, BF16, "cpu")


# ------------------------------------------------------------------------------------------------ GPU helpers
D_SCALE = 1 / 1024   # |value| <= 62 * 31 / 4 (IQ3_XXS), 15 * 31 (IQ3_S) times d


def _dev_blocks(t, n_elems, seed):
    if t in IQ3:
        return torch.from_numpy(o3.random_blocks(t, n_elems // 256, np.random.default_rng(seed), D_SCALE).reshape(-1)).cuda()
    return tie._dev_blocks(t, n_elems, seed)


class _Experts(tie._Experts):
    def __init__(self, E, H, I, gt, ut, dt, seed):
        self.E, self.H, self.I, self.types = E, H, I, (gt, ut, dt)
        self.w = [_dev_blocks(t, E * r * c, seed + i) for i, (t, r, c) in enumerate(((gt, I, H), (ut, I, H), (dt, H, I)))]
        self.host = [b.cpu().numpy().reshape(E, -1) for b in self.w]


def _host_blocks(t, n, rng):
    return o3.random_blocks(t, n, rng, D_SCALE) if t in IQ3 else oq.random_blocks(t, n, rng, 1 / 512)


TYPE_MIXES = {"iq3xxsx3": (IQ3XXS, IQ3XXS, IQ3XXS), "iq3xxs_iq3xxs_iq3s": (IQ3XXS, IQ3XXS, IQ3S), "iq3sx3": (IQ3S, IQ3S, IQ3S),
              "iq3xxs_iq3xxs_q4k": (IQ3XXS, IQ3XXS, Q4K), "iq3s_iq3s_q6k": (IQ3S, IQ3S, Q6K), "q4k_q4k_iq3s": (Q4K, Q4K, IQ3S),
              "iq3xxs_iq3s_iq3xxs": (IQ3XXS, IQ3S, IQ3XXS), "iq3xxs_iq3xxs_iq2": (IQ3XXS, IQ3XXS, IQ2)}
# grouped_gemm_kernel<FMT> of a weight type (Q6_K: down tensors in the 4-row tile layout)
GFMT = {Q4K: 0, Q6K: 1, IQ2: 3, IQ3XXS: 9, IQ3S: 10}


# ------------------------------------------------------------------------------------------------ GPU: formats and decode
@pytest.mark.gpu
@pytest.mark.parametrize("t", IQ3)
def test_dequantize_bit_exact(t):
    from gpu_util import dequantize
    import gguf
    b = o3.random_blocks(t, 600, np.random.default_rng(30 + t))
    ref = gguf.quants.dequantize(b.reshape(-1), gguf.GGMLQuantizationType(t)).astype(np.float32)
    n = ref.size
    assert np.array_equal(dequantize(b.reshape(-1), t, n, F32).numpy().view(np.uint32), ref.view(np.uint32))
    assert torch.equal(dequantize(b.reshape(-1), t, n, BF16), torch.from_numpy(ref).to(torch.bfloat16))
    assert torch.equal(dequantize(b.reshape(-1), t, n, F16), torch.from_numpy(ref).to(torch.float16))


@pytest.mark.gpu
def test_gguf_loader_dequantizes_on_the_gpu(tmp_path):
    """GGUFLoader.load_gguf_tensor(device="cuda") of IQ3 tensors: ktb200_dequantize, bit for bit gguf-py"""
    import gguf
    from ktransformers_b200.util.custom_loader import GGUFLoader
    rng = np.random.default_rng(33)
    wtr = gguf.GGUFWriter(str(tmp_path / "iq3.gguf"), "deepseek2")
    names = {IQ3XXS: "blk.0.ffn_gate_exps.weight", IQ3S: "blk.0.ffn_down_exps.weight"}
    blocks = {t: o3.random_blocks(t, 64 * 4, rng).reshape(64, -1) for t in IQ3}
    for t, b in blocks.items():
        wtr.add_tensor(names[t], b, raw_dtype=gguf.GGMLQuantizationType(t))
    wtr.write_header_to_file()
    wtr.write_kv_data_to_file()
    wtr.write_tensors_to_file()
    wtr.close()
    ld = GGUFLoader(str(tmp_path))
    for t, b in blocks.items():
        got = ld.load_gguf_tensor(names[t], device="cuda", target_dtype=torch.float32).cpu().numpy().reshape(-1)
        ref = gguf.quants.dequantize(b.reshape(-1), gguf.GGMLQuantizationType(t)).astype(np.float32).reshape(-1)
        assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), NAMES[t]


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
    n0 = native.launch_count()
    got = m.forward(ids, w, x)
    assert native.launch_count() - n0 == 2
    _check(got, oq.moe_forward(oracle, xf, ids, w, ex.expert, E), F32, mix)
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("hidden_type", [F32, F16, BF16])
@pytest.mark.parametrize("use_silu", [1, 0])
@pytest.mark.parametrize("qlen", [1, 8])
def test_moe_forward_hidden_types_and_activations(oracle, hidden_type, use_silu, qlen):
    E, k, H, I = 8, 3, 1024, 256
    ex = _Experts(E, H, I, IQ3XXS, IQ3XXS, IQ3S, 7)
    m = ex.moe(k, hidden_type, use_silu=use_silu)
    rng = np.random.default_rng(40 + qlen)
    ids, w = _ids(qlen, E, k, rng), rng.random((qlen, k)).astype(np.float32)
    x, xf = _x(qlen, H, 41, hidden_type)
    _check(m.forward(ids, w, x), oq.moe_forward(oracle, xf, ids, w, ex.expert, E, bool(use_silu)), hidden_type)
    m.close()


# which kernels ran: decode at 3 tokens (H, I = 1024, 512: 4 blocks per gate/up row, 2 per down row, the bulk kernels' shapes),
# the grouped GEMM at 80 tokens; torch.profiler in an interpreter of its own (after other profiler sessions in one process a
# session can miss kernels)
CENSUS_DECODE = [("iq3xxsx3", 1024, 512), ("iq3sx3", 1024, 512), ("iq3xxs_iq3xxs_iq3s", 1024, 512), ("iq3xxs_iq3s_iq3xxs", 1024, 512)]
BULK = {IQ3XXS: "BulkIQ3XXS", IQ3S: "BulkIQ3S"}
_CENSUS = r"""
import json, sys
import numpy as np, torch
sys.path[:0] = sys.argv[1:]
from torch.profiler import ProfilerActivity, profile
from test_iq3_experts import CENSUS_DECODE, IQ_MIN, TYPE_MIXES, _Experts, _ids, _x
from ktransformers_b200 import native
def session(run):
    # even in this interpreter a session after others can miss kernels: repeat it (3 tries) until it recorded as
    # many of the library's kernels as the library launched
    for _ in range(3):
        n0 = native.launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run()
            torch.cuda.synchronize()
        seen = sum(e.device_type == torch.autograd.DeviceType.CUDA and 'ktb::' in e.name for e in prof.events())
        if seen >= native.launch_count() - n0:
            break
    return prof.key_averages()
res = {}
for mix, H, I in CENSUS_DECODE:
    ex = _Experts(8, H, I, *TYPE_MIXES[mix], 60)
    m = ex.moe(4, 0)
    rng = np.random.default_rng(61)
    ids, w, x = _ids(3, 8, 4, rng), rng.random((3, 4)).astype(np.float32), _x(3, H, 62, 0)[0]
    m.forward(ids, w, x)
    res[f"decode {mix} {H} {I}"] = sorted({e.key for e in session(lambda: m.forward(ids, w, x)) if "ktb::" in e.key})
    m.close()
for mix in sorted(TYPE_MIXES):
    ex = _Experts(8, 1024, 512, *TYPE_MIXES[mix], 5)
    m = ex.moe(4, 0, max_tokens=IQ_MIN)
    rng = np.random.default_rng(0)
    ids, w, x = _ids(IQ_MIN, 8, 4, rng), rng.random((IQ_MIN, 4)).astype(np.float32), _x(IQ_MIN, 1024, 1, 0)[0]
    m.forward(ids, w, x)
    res[f"grouped {mix}"] = sorted({e.key for e in session(lambda: m.forward(ids, w, x)) if "kernel" in e.key})
    m.close()
print("CENSUS " + json.dumps(res))
"""


@pytest.fixture(scope="module")
def kernel_census():
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CENSUS, HERE, ROOT]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return json.loads(next(l for l in r.stdout.splitlines() if l.startswith("CENSUS "))[7:])


@pytest.mark.gpu
@pytest.mark.parametrize("case", CENSUS_DECODE)
def test_decode_kernels_that_ran(kernel_census, case):
    """same-type IQ3 gate/up on rows_bulk_iq_kernel<BulkIQ3XXS / BulkIQ3S>, IQ3 down on reduce_bulk_kernel of its format;
    mixed gate/up types on the generic kernels"""
    mix, H, I = case
    gt, ut, dt = TYPE_MIXES[mix]
    names = kernel_census[f"decode {mix} {H} {I}"]
    assert len(names) == 2, names
    if gt == ut:
        assert any("rows_bulk_iq_kernel" in n and BULK[gt] + "," in n for n in names), names
        assert not any("FmtGenK" in n for n in names), names
    else:
        assert any("rows_kernel<ktb::FmtGenK" in n for n in names), names
    assert any("reduce_bulk_kernel" in n and BULK[dt] + "," in n for n in names), names


@pytest.mark.gpu
@pytest.mark.parametrize("mix", sorted(TYPE_MIXES))
def test_grouped_kernels_that_ran_at_80_tokens(kernel_census, mix):
    names = kernel_census[f"grouped {mix}"]
    ran = {n.split("grouped_gemm_kernel<")[1].split(">")[0] for n in names if "grouped_gemm_kernel<" in n}
    assert ran == {str(GFMT[t]) for t in TYPE_MIXES[mix]}, (mix, names)
    assert not any(s in n for n in names for s in ("rows_", "reduce_", "FmtGenK", "BulkIQ")), (mix, names)


# ------------------------------------------------------------------------------------------------ GPU: grouped
def _check_requant(got, ref, what):
    """F32 outputs within 2e-3 of max|ref|: the kernels' fp32 act(g) * u and the oracle's float64 one can round to different
    Q8_K bytes of a down input (one step of max|a| / 127 of a block).  With IQ3's scales 2s + 1 spread over 1..31, random
    blocks give act(g) * u a wide range, so over 80-300 tokens a few such steps reach about 1e-3 of max|ref|."""
    err = np.abs(got.astype(np.float64) - ref)
    assert err.max() <= 2e-3 * np.abs(ref).max(), (what, err.max(), np.abs(ref).max())


@pytest.mark.gpu
@pytest.mark.parametrize("mix", sorted(TYPE_MIXES))
def test_grouped_type_mixes_vs_oracle(oracle, mix):
    E, k, H, I = 8, 4, 1024, 512
    ex = _Experts(E, H, I, *TYPE_MIXES[mix], 300)
    m = ex.moe(k, F32, max_tokens=300)
    rng = np.random.default_rng(len(mix))
    cases = []
    for qlen in (IQ_MIN - 1, IQ_MIN, 131, 300):
        ids, w = _hard_ids(qlen, E, k, rng), rng.random((qlen, k)).astype(np.float32)
        cases.append((_x(qlen, H, qlen, F32)[0], ids, w))
    refs = _moe_ref(oracle, cases, ex.expert, E)
    for (x, ids, w), ref in zip(cases, refs):
        n0 = native.launch_count()
        got = m.forward(ids, w, x)
        assert native.launch_count() - n0 == (10 if len(ids) >= IQ_MIN else 2), "grouped from IQ_MIN tokens, per pair below"
        _check_requant(got, ref, (mix, x.shape[0]))
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["iq3xxsx3", "iq3sx3", "iq3xxs_iq3xxs_iq3s"])
def test_grouped_matches_per_pair_kernels(mix):
    """the tolerance rule of test_iq_grouped.test_grouped_matches_per_pair_kernels: the same integer per super-block on both
    routes, the fp32 order of the terms differs, and a Q8_K rounding edge of act(g) * u can move one int8 of a down input"""
    E, k, H, I, T = 8, 4, 2048, 768, 200
    ex = _Experts(E, H, I, *TYPE_MIXES[mix], 31)
    m = ex.moe(k, F32, max_tokens=256)
    rng = np.random.default_rng(9)
    ids, w = _ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    x = _x(T, H, 10, F32)[0]
    n0 = native.launch_count()
    big = m.forward(ids, w, x)
    assert native.launch_count() - n0 == 10
    small = np.concatenate([m.forward(ids[i:i + 40], w[i:i + 40], x[i:i + 40]) for i in range(0, T, 40)])
    row = np.abs(big.astype(np.float64) - small).max(axis=1) / np.abs(small).max()
    assert (row < 1e-5).mean() >= 0.95, np.sort(row)[-12:]
    assert row.max() < 1e-3, row.max()
    m.close()


@pytest.mark.gpu
def test_r1_shapes(oracle):
    """DeepSeek-R1 routed experts (H 7168, I 2048, k 8, BF16) over 16 experts: decode at 1 and 8 tokens, the grouped GEMM at 300,
    and at 1100 over two 1024-token chunks"""
    E, k, H, I = 16, 8, 7168, 2048
    ex = _Experts(E, H, I, IQ3XXS, IQ3XXS, IQ3S, 2028)
    rng = np.random.default_rng(12)
    cases = []
    for qlen in (1, 8, 300, 1100):
        ids = np.stack([rng.permutation(E)[:k] for _ in range(qlen)]).astype(np.int64)
        cases.append((_x(qlen, H, qlen, BF16), ids, rng.random((qlen, k)).astype(np.float32)))
    refs = _moe_ref(oracle, [(xf, ids, w) for (_, xf), ids, w in cases], ex.expert, E)
    m = ex.moe(k, BF16, max_tokens=1100)
    for ((x, _), ids, w), ref in zip(cases, refs):
        n0 = native.launch_count()
        got = m.forward(ids, w, x)
        assert native.launch_count() - n0 == (2 if len(ids) < IQ_MIN else 10 * -(-len(ids) // 1024))
        _check(got, ref, BF16, len(ids))
    m.close()


# ------------------------------------------------------------------------------------------------ GPU: callers
@pytest.mark.gpu
def test_rows_beyond_bsz_untouched_eager_and_graph():
    """decode sizes: rows >= bsz keep their bytes and rows < bsz equal the full call, eagerly and across graph replays"""
    E, k, H, I, T = 8, 4, 1024, 512, 8
    ex = _Experts(E, H, I, IQ3S, IQ3S, IQ3XXS, 5)
    m = ex.moe(k, BF16)
    rng = np.random.default_rng(1)
    ids = torch.from_numpy(_ids(T, E, k, rng)).cuda()
    w = torch.from_numpy(rng.random((T, k)).astype(np.float32)).cuda()
    x = torch.randn((T, H), device="cuda").to(torch.bfloat16)
    bsz = torch.tensor([5], dtype=torch.int32, device="cuda")
    lib = native.lib()

    def call(out, b):
        native.check(lib.ktb200_moe_forward(m.h, T, k, ids.data_ptr(), w.data_ptr(), x.data_ptr(), out.data_ptr(), b,
                                            torch.cuda.current_stream().cuda_stream))

    full = torch.zeros((T, H), dtype=torch.bfloat16, device="cuda")
    call(full, None)
    out = torch.full((T, H), 1234.5, dtype=torch.bfloat16, device="cuda")
    call(out, bsz.data_ptr())
    torch.cuda.synchronize()
    assert torch.equal(out[:5], full[:5]) and (out[5:] == 1234.5).all()
    s = torch.cuda.Stream()
    out2 = torch.full((T, H), 1234.5, dtype=torch.bfloat16, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            call(out2, bsz.data_ptr())
    torch.cuda.synchronize()
    for b in (3, 8, 1):
        out2.fill_(1234.5)
        bsz.fill_(b)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out2[:b], full[:b]) and (out2[b:] == 1234.5).all(), b
    m.close()


@pytest.mark.gpu
def test_expert_id_offset_shards_and_skipped_ids(oracle):
    E, k, H, I, T = 8, 4, 512, 256, 5
    ex = _Experts(E, H, I, IQ3XXS, IQ3XXS, IQ3S, 9)
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
def test_forward_shared_with_q4k_shared_expert():
    from gpu_util import moe_forward_shared, mlp_forward
    E, k, H, I, T = 8, 4, 4096, 512, 3
    ex = _Experts(E, H, I, IQ3XXS, IQ3XXS, IQ3S, 12)
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
    ex = _Experts(E, H, I, IQ3S, IQ3S, IQ3S, 11)
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
@pytest.mark.parametrize("types", [(IQ3XXS, IQ3XXS, IQ3XXS), (IQ3S, IQ3S, IQ3S), (Q4K, Q4K, IQ3S)])
def test_forward_ep_refuses(types):
    E, k, H, I = 8, 2, 4096, 512
    m = _Experts(E, H, I, *types, 13).moe(k, BF16)
    mlp = _q4k_mlp(H, I, BF16)
    ids = torch.zeros((1, k), dtype=torch.int64, device="cuda")
    wt = torch.ones((1, k), device="cuda")
    x = torch.zeros((1, H), dtype=torch.bfloat16, device="cuda")
    part, sh = torch.zeros((1, H), device="cuda"), torch.zeros((H,), dtype=torch.bfloat16, device="cuda")
    rc = native.lib().ktb200_moe_forward_ep(m.h, mlp.h, 1, k, ids.data_ptr(), wt.data_ptr(), x.data_ptr(), part.data_ptr(), 0,
                                            sh.data_ptr(), None, torch.cuda.current_stream().cuda_stream)
    assert rc == native.EINVAL and NAMES[next(t for t in types if t in IQ3)] in native.lib().ktb200_last_error().decode()
    mlp.close()
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("T", [5, 256])
def test_ktmoe_wrapper_from_gguf(oracle, tmp_path, T):
    """KTMoEWrapper(method="B200_GGUF") from a GGUF with raw IQ3_XXS / IQ3_S tensors, a physical-to-logical map and a gpu_experts_mask,
    at a decode batch and over a prefill"""
    import gguf
    from test_iq_experts import _dequant_f64
    E, k, H, I = 8, 3, 512, 256
    types = (IQ3XXS, IQ3XXS, IQ3S)
    rng = np.random.default_rng(31)
    wtr = gguf.GGUFWriter(str(tmp_path / "iq3.gguf"), "deepseek2")
    blocks = {}
    for n, t, (r, c) in zip(("gate", "up", "down"), types, ((I, H), (I, H), (H, I))):
        blocks[n] = _host_blocks(t, E * r * c // 256, rng).reshape(E, r, -1)
        wtr.add_tensor(f"blk.0.ffn_{n}_exps.weight", blocks[n], raw_dtype=gguf.GGMLQuantizationType(t))
    wtr.write_header_to_file()
    wtr.write_kv_data_to_file()
    wtr.write_tensors_to_file()
    wtr.close()
    p2l = torch.tensor([1, 0, 3, 2, 5, 4, 7, 6])
    mask = torch.zeros(E, dtype=torch.bool)
    mask[[0, 6]] = True
    wr = tie._wrapper(gpu_experts_mask=mask, weight_path=str(tmp_path), key_template="blk.{layer}", chunked_prefill_size=T)
    wr.load_weights(p2l)
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
    _check(got, _moe_ref(oracle, [(xf, ids_m, w)], expert, E)[0], BF16)


def _iq_blocks(t, n, seed):
    if t in IQ3 or t == IQ2:
        return _dev_blocks(t, n, seed)
    from ktransformers_b200.util.synth import synth_blocks
    return synth_blocks(t, n, "cuda", seed)


@pytest.mark.gpu
@pytest.mark.parametrize("world,counts", [(1, [100]), (2, [300, 79])])
def test_grouped_ep_tokens_loopback(world, counts):
    """the multi-token expert-parallel layer with IQ3 experts: world 1 bit for bit the unsharded layer, world 2 within fp32
    re-association; phase 2 on the grouped GEMM from 80 gathered rows"""
    from test_ep_tokens import _Loopback
    lb = _Loopback(world, 16, 4, 2048, 512, BF16, 300, types=(IQ3XXS, IQ3XXS, IQ3S), shared=True, seed=93, make=_iq_blocks)
    xs = lb.tokens(counts, np.random.default_rng(19))
    ys, idx, w, launches = lb.run(counts, xs)
    lb.check(counts, xs, ys, idx, w)
    lb.close()
