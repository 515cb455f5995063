"""IQ1_M routed experts (ggml type 29, the experts of DeepSeek-R1's 1.73-bit GGUF files): format and dot-product pins against
gguf-py and the reference's integer formula, C-ABI and host checks, and the sm_90a kernels (the bulk-copy decode kernels, the
generic per-pair kernels, grouped_gemm_kernel<8>) against the float64 oracle, through every caller."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import iq1m_oracle as om
import iq_oracle as oq
import test_iq_experts as tie
from ktransformers_b200 import native
from test_iq_experts import _check, _ids, _q4k_mlp, _x
from test_iq_grouped import IQ_MIN, _hard_ids, _moe_ref

IQ1M, IQ1, IQ2 = native.GGML_IQ1_M, native.GGML_IQ1_S, native.GGML_IQ2_XXS
Q4K, Q6K = native.GGML_Q4_K, native.GGML_Q6_K
F32, F16, BF16 = native.GGML_F32, native.GGML_F16, native.GGML_BF16
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ------------------------------------------------------------------------------------------------ format (CPU)
def test_random_blocks_cover_every_field():
    b = om.random_blocks(512, np.random.default_rng(1))
    sc = b[:, 48:56].copy().view(np.uint16)
    for h in range(4):
        assert set(((sc >> (3 * h)) & 7).reshape(-1).tolist()) == set(range(8))
    qh = b[:, 32:48]
    for nib in (qh & 15, qh >> 4):
        assert set((nib >> 3).reshape(-1).tolist()) == {0, 1}
        assert set((nib & 7).reshape(-1).tolist()) == set(range(8))
    d = om.fields(b)[0]
    assert (d >= 0.75).all() and (d < 1.25).all()
    assert len({int(w) >> 12 for w in sc[:, 0]}) > 1 and len({int(w) >> 12 for w in sc[:, 3]}) == 1   # low nibbles vary, the exponent's not


def test_oracle_dequant_matches_gguf_bit_for_bit():
    import gguf
    b = om.random_blocks(512, np.random.default_rng(3))
    ref = gguf.quants.dequantize(b.reshape(-1), gguf.GGMLQuantizationType.IQ1_M).astype(np.float32)
    assert np.array_equal(om.dequant(b).view(np.uint32), ref.view(np.uint32))


def _q8(n_blocks, seed):
    from oracle.bindings import Oracle
    x = np.random.default_rng(seed).standard_normal(n_blocks * 256).astype(np.float32)
    return Oracle().from_float(x, 15)


def test_superblock_term_is_the_integer_formula():
    """(d dx) (sumi1 + 0.125 sumi2) == ((d / 8) dx) S exactly, S = 8 sumi1 + sumi2 with |S| < 2^23"""
    w, q8 = om.random_blocks(256, np.random.default_rng(10)), _q8(256, 11)
    S = om.superblock_ints(w, q8)
    assert np.abs(S).max() < 2 ** 23
    d8 = (om.fields(w)[0] * np.float32(0.125)).astype(np.float32)
    want = ((d8 * oq.q8k_fields(q8)[0]).astype(np.float32) * S.astype(np.float32)).astype(np.float32)
    assert np.array_equal(om.superblock_terms(w, q8), want)


def test_vec_dot_within_fp32_rounding_of_float64():
    rng = np.random.default_rng(20)
    for _ in range(8):
        nb = 28
        w, q8 = om.random_blocks(nb, rng), _q8(nb, int(rng.integers(1 << 30)))
        got = float(om.vec_dot(w, q8))
        ref = float(np.dot(om.dequant(w).astype(np.float64), oq.q8k_to_f64(q8)))
        terms = np.abs(om.superblock_terms(w, q8).astype(np.float64)).sum()
        assert abs(got - ref) <= 4 * nb * 2 ** -24 * max(terms, 1e-30), (got, ref)


# ------------------------------------------------------------------------------------------------ C-ABI and host (CPU)
def test_type_size_and_block():
    lib = native.lib()
    assert lib.ktb200_type_size(IQ1M) == 56 and lib.ktb200_blck_size(IQ1M) == 256


def test_type_sets():
    from ktransformers_b200.util import custom_gguf as cg
    assert "IQ1_M" in cg.B200_ROUTED_EXPERT_TYPES and cg.B200_ROUTED_EXPERT_TYPES == cg.B200_EXPERT_TYPES | {"IQ1_M"}
    assert "IQ1_M" not in cg.B200_WEIGHT_TYPES and "IQ1_M" in cg.B200_DEQUANT_TYPES


def test_linear_and_mlp_reject_with_type_name():
    lib = native.lib()
    h = C.c_void_p()
    assert lib.ktb200_linear_create(512, 256, 1 << 20, IQ1M, BF16, 16, 0, C.byref(h)) == native.EINVAL
    assert "IQ1_M" in lib.ktb200_last_error().decode()
    assert lib.ktb200_mlp_create(512, 256, 1 << 20, 1 << 20, 1 << 20, Q4K, Q4K, IQ1M, BF16, 16, 0, C.byref(h)) == native.EINVAL
    assert "IQ1_M" in lib.ktb200_last_error().decode()


def test_moe_create_accepts_the_type():
    """validation runs before any CUDA call: an IQ1_M handle with a bad shape fails on the shape, not on the type"""
    lib = native.lib()
    h = C.c_void_p()
    cfg = native.MoeConfig(8, 2, 7000, 2048, 64, 10, 16, 1, 1 << 20, 1 << 20, 1 << 20, IQ1M, IQ1M, IQ2, BF16, 0)
    assert lib.ktb200_moe_create(C.byref(cfg), 0, C.byref(h)) == native.EINVAL and not h.value
    err = lib.ktb200_last_error().decode()
    assert "unsupported ggml weight type" not in err and "multiples of 256" in err


@pytest.mark.parametrize("expert_types", [(IQ1M, IQ1M, IQ2), (Q4K, Q4K, IQ1M)])
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
def _dev_blocks(t, n_elems, seed):
    if t == IQ1M:
        return torch.from_numpy(om.random_blocks(n_elems // 256, np.random.default_rng(seed), 1 / 64).reshape(-1)).cuda()
    return tie._dev_blocks(t, n_elems, seed)


class _Experts(tie._Experts):
    def __init__(self, E, H, I, gt, ut, dt, seed):
        self.E, self.H, self.I, self.types = E, H, I, (gt, ut, dt)
        self.w = [_dev_blocks(t, E * r * c, seed + i) for i, (t, r, c) in enumerate(((gt, I, H), (ut, I, H), (dt, H, I)))]
        self.host = [b.cpu().numpy().reshape(E, -1) for b in self.w]


def _host_blocks(t, n, rng):
    return om.random_blocks(n, rng, 1 / 64) if t == IQ1M else oq.random_blocks(t, n, rng, 1 / 64 if t == IQ1 else 1 / 512)


TYPE_MIXES = {"iq1mx3": (IQ1M, IQ1M, IQ1M), "iq1m_iq1m_iq2": (IQ1M, IQ1M, IQ2), "iq1m_iq1m_q6k": (IQ1M, IQ1M, Q6K),
              "q4k_q4k_iq1m": (Q4K, Q4K, IQ1M), "iq1m_iq1s_iq1m": (IQ1M, IQ1, IQ1M)}
# grouped_gemm_kernel<FMT> of a weight type (Q6_K: down tensors in the 4-row tile layout)
GFMT = {Q4K: 0, Q6K: 1, IQ1: 2, IQ2: 3, IQ1M: 8}


# ------------------------------------------------------------------------------------------------ GPU: formats and decode
@pytest.mark.gpu
def test_dequantize_bit_exact():
    from gpu_util import dequantize
    import gguf
    b = om.random_blocks(600, np.random.default_rng(30))
    ref = gguf.quants.dequantize(b.reshape(-1), gguf.GGMLQuantizationType.IQ1_M).astype(np.float32)
    n = ref.size
    assert np.array_equal(dequantize(b.reshape(-1), IQ1M, n, F32).numpy().view(np.uint32), ref.view(np.uint32))
    assert torch.equal(dequantize(b.reshape(-1), IQ1M, n, BF16), torch.from_numpy(ref).to(torch.bfloat16))
    assert torch.equal(dequantize(b.reshape(-1), IQ1M, n, F16), torch.from_numpy(ref).to(torch.float16))


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
    ex = _Experts(E, H, I, IQ1M, IQ1M, IQ2, 7)
    m = ex.moe(k, hidden_type, use_silu=use_silu)
    rng = np.random.default_rng(40 + qlen)
    ids, w = _ids(qlen, E, k, rng), rng.random((qlen, k)).astype(np.float32)
    x, xf = _x(qlen, H, 41, hidden_type)
    _check(m.forward(ids, w, x), oq.moe_forward(oracle, xf, ids, w, ex.expert, E, bool(use_silu)), hidden_type)
    m.close()


# which kernels ran: decode at 3 tokens (H, I = 1024, 512 and 512, 256: the bulk kernels take every IQ1_M shape), the
# grouped GEMM at 80 tokens; torch.profiler in an interpreter of its own (after other profiler sessions in one process a session
# can miss kernels)
CENSUS_DECODE = [("iq1mx3", 1024, 512), ("iq1mx3", 512, 256), ("iq1m_iq1s_iq1m", 1024, 512)]
_CENSUS = r"""
import json, sys
import numpy as np, torch
sys.path[:0] = sys.argv[1:]
from torch.profiler import ProfilerActivity, profile
from test_iq1m_experts import CENSUS_DECODE, IQ_MIN, TYPE_MIXES, _Experts, _ids, _x
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
    """same-type IQ1_M gate/up on rows_bulk_iq_kernel<BulkIQ1M>, IQ1_M down on reduce_bulk_kernel<BulkIQ1M>; mixed gate/up
    types on the generic kernels"""
    mix, H, I = case
    names = kernel_census[f"decode {mix} {H} {I}"]
    assert len(names) == 2, names
    if TYPE_MIXES[mix][0] == TYPE_MIXES[mix][1]:
        assert any("rows_bulk_iq_kernel" in n and "BulkIQ1M" in n for n in names), names
    else:
        assert any("rows_kernel<ktb::FmtGenK" in n for n in names), names
    assert any("reduce_bulk_kernel" in n and "BulkIQ1M" in n for n in names), names


@pytest.mark.gpu
@pytest.mark.parametrize("mix", sorted(TYPE_MIXES))
def test_grouped_kernels_that_ran_at_80_tokens(kernel_census, mix):
    names = kernel_census[f"grouped {mix}"]
    ran = {n.split("grouped_gemm_kernel<")[1][0] for n in names if "grouped_gemm_kernel<" in n}
    assert ran == {str(GFMT[t]) for t in TYPE_MIXES[mix]}, (mix, names)
    assert not any(s in n for n in names for s in ("rows_", "reduce_", "FmtGenK", "BulkIQ")), (mix, names)


# ------------------------------------------------------------------------------------------------ GPU: grouped
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
        _check(got, ref, F32, (mix, x.shape[0]))
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["iq1mx3", "iq1m_iq1m_iq2"])
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
    ex = _Experts(E, H, I, IQ1M, IQ1M, IQ2, 2028)
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
    ex = _Experts(E, H, I, IQ1M, IQ1M, IQ2, 5)
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
    ex = _Experts(E, H, I, IQ1M, IQ1M, IQ1M, 9)
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
    ex = _Experts(E, H, I, IQ1M, IQ1M, IQ2, 12)
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
    ex = _Experts(E, H, I, IQ1M, IQ1M, IQ2, 11)
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
@pytest.mark.parametrize("types", [(IQ1M, IQ1M, IQ1M), (Q4K, Q4K, IQ1M)])
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
    assert rc == native.EINVAL and "IQ1_M" in native.lib().ktb200_last_error().decode()
    mlp.close()
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("T", [5, 256])
def test_ktmoe_wrapper_from_gguf(oracle, tmp_path, T):
    """KTMoEWrapper(method="B200_GGUF") from a GGUF with raw IQ1_M tensors, a physical-to-logical map and a gpu_experts_mask,
    at a decode batch and over a prefill"""
    import gguf
    from test_iq_experts import _dequant_f64
    E, k, H, I = 8, 3, 512, 256
    types = (IQ1M, IQ1M, IQ2)
    rng = np.random.default_rng(31)
    wtr = gguf.GGUFWriter(str(tmp_path / "iq1m.gguf"), "deepseek2")
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
    if t in (IQ1M, IQ1, IQ2):
        return _dev_blocks(t, n, seed)
    from ktransformers_b200.util.synth import synth_blocks
    return synth_blocks(t, n, "cuda", seed)


@pytest.mark.gpu
@pytest.mark.parametrize("world,counts", [(1, [100]), (2, [300, 79])])
def test_grouped_ep_tokens_loopback(world, counts):
    """the multi-token expert-parallel layer with IQ1_M experts: world 1 bit for bit the unsharded layer, world 2 within fp32
    re-association; phase 2 on the grouped GEMM from 80 gathered rows"""
    from test_ep_tokens import _Loopback
    lb = _Loopback(world, 16, 4, 2048, 512, BF16, 300, types=(IQ1M, IQ1M, IQ2), shared=True, seed=93, make=_iq_blocks)
    xs = lb.tokens(counts, np.random.default_rng(19))
    ys, idx, w, launches = lb.run(counts, xs)
    lb.check(counts, xs, ys, idx, w)
    lb.close()
