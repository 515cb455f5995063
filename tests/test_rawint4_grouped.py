"""RAWINT4_G32 routed experts (Kimi-K2's compressed-tensors INT4) on the grouped tensor-core GEMM (grouped_i4_kernel<NP>,
csrc/grouped.cu): prompts of I4_MIN tokens and more read each expert once per 32-token tile.  W4A16 with nothing quantised:
u - 8 and exact bf16 planes of the activations on the bf16 tensor path, so the float64 oracle of tests/int4_oracle.py and
the tolerances of tests/test_rawint4.py apply unchanged.  Checked through every caller: ktb200_moe_forward / _shared, the
device batch size and CUDA graphs, KTMoEWrapper and phase 2 of the expert-parallel layer; and with crafted inputs whose exact
result only comes out when every bf16 plane is summed."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import int4_oracle as o4
from ktransformers_b200 import native
from test_iq_grouped import _hard_ids
from test_rawint4 import _check, _Experts, _pack, _x

I4 = native.RAWINT4_G32
Q4K = native.GGML_Q4_K
F32, F16, BF16 = native.GGML_F32, native.GGML_F16, native.GGML_BF16
HERE = os.path.dirname(os.path.abspath(__file__))
I4_MIN = 96     # qlen from which a RAWINT4 handle takes the grouped path (csrc/moe.cu grouped_min_qlen)


def _moe(ex, k, hidden_type, max_tokens, use_silu=1):
    """test_rawint4._Experts.moe with an activation switch"""
    from gpu_util import Moe
    sl = [ex.blocks[n] for n in ("gate", "up", "down")]
    return Moe(ex.E, k, ex.H, ex.I, *sl, I4, I4, I4, hidden_type, max_tokens=max_tokens, use_silu=use_silu)


def _counted(m, *args, **kw):
    n0 = native.launch_count()
    r = m.forward(*args, **kw)
    return r, native.launch_count() - n0


# ------------------------------------------------------------------------------------------------ CPU
def test_exact_inputs_have_three_planes():
    """the crafted activations of test_exactness_every_plane_counts need all three bf16 planes: hi = 1, mid = 2^-10, lo = 2^-20"""
    x = _exact_x(4, 256)[:, 32:].astype(np.float64)
    hi = o4.bf16_bits_to_f64(o4.f32_to_bf16_bits(x))
    mid = o4.bf16_bits_to_f64(o4.f32_to_bf16_bits((x - hi).astype(np.float32)))
    lo = x - hi - mid
    assert (np.abs(mid) > 0).all() and (np.abs(lo) > 0).all()
    assert np.array_equal(o4.bf16_bits_to_f64(o4.f32_to_bf16_bits(lo.astype(np.float32))), lo)


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_grouped_vs_oracle_on_both_sides_of_the_threshold():
    E, k, H, I = 8, 4, 1024, 512
    ex = _Experts(E, H, I, 300)
    m = ex.moe(k, F32, max_tokens=300)
    rng = np.random.default_rng(4)
    for qlen in (I4_MIN - 1, I4_MIN, 131, 300):
        ids, w = _hard_ids(qlen, E, k, rng), rng.random((qlen, k)).astype(np.float32)
        x, x64 = _x(qlen, H, qlen, F32)
        got, n = _counted(m, ids, w, x)
        assert n == (10 if qlen >= I4_MIN else 2), "grouped from I4_MIN tokens, per pair below"
        _check(got, o4.moe_forward(x64, ids, w, ex.expert, E), F32)
    m.close()


_CENSUS = r"""
import json, sys
import numpy as np, torch
sys.path[:0] = sys.argv[2:]
from torch.profiler import ProfilerActivity, profile
from test_rawint4 import _Experts, _x
T = int(sys.argv[1])
res = {}
ex = _Experts(8, 1024, 512, 5)
for ht in (0, 30):
    m = ex.moe(4, ht, max_tokens=T)
    rng = np.random.default_rng(0)
    ids = np.stack([rng.permutation(8)[:4] for _ in range(T)]).astype(np.int64)
    w = rng.random((T, 4)).astype(np.float32)
    x = _x(T, 1024, 1, ht)[0]
    m.forward(ids, w, x)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.forward(ids, w, x)
        torch.cuda.synchronize()
    res[ht] = [e.key for e in prof.key_averages() if "kernel" in e.key for _ in range(e.count)]
    m.close()
print("CENSUS " + json.dumps(res))
"""


@pytest.mark.gpu
def test_kernels_that_ran_at_the_threshold():
    """F32: gate, up and down on grouped_i4_kernel<3>; BF16: gate and up on <1>, down on <3>; no per-pair RAWINT4 kernel
    (torch.profiler in an interpreter of its own, as test_iq_grouped's census)"""
    root = os.path.dirname(HERE)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CENSUS, str(I4_MIN), HERE, root]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(next(l for l in r.stdout.splitlines() if l.startswith("CENSUS "))[7:])
    for ht, want in ((str(F32), ["3", "3", "3"]), (str(BF16), ["1", "1", "3"])):
        names = res[ht]
        ran = sorted(n.split("grouped_i4_kernel<")[1][0] for n in names if "grouped_i4_kernel<" in n)
        assert ran == sorted(want), (ht, names)
        assert not any(s in n for n in names for s in ("rows_bulk_i4", "reduce_bulk_kernel<ktb::BulkI4", "grouped_gemm_kernel")), (ht, names)


@pytest.mark.gpu
@pytest.mark.parametrize("hidden_type", [F32, F16, BF16])
@pytest.mark.parametrize("use_silu", [1, 0])
def test_grouped_hidden_types_and_activations(hidden_type, use_silu):
    """against the oracle (F16 with test_hidden_types' bound), and F16 / BF16 bit for bit the F32 call on the widened input,
    rounded: the planes depend on the fp32 value only"""
    from test_hidden_types import assert_f16_close, assert_same_bits, to_h, widen
    E, k, H, I, T = 8, 3, 1024, 256, max(I4_MIN, 40)
    ex = _Experts(E, H, I, 7)
    rng = np.random.default_rng(40)
    ids, w = _hard_ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    x32 = rng.standard_normal((T, H)).astype(np.float32)
    xh = to_h(x32, hidden_type)
    m = _moe(ex, k, hidden_type, T, use_silu)
    got, n = _counted(m, ids, w, xh)
    assert n == 10
    ref = o4.moe_forward(widen(xh, hidden_type).astype(np.float64), ids, w, ex.expert, E, use_silu=bool(use_silu))
    if hidden_type == F16:
        assert_f16_close(got, to_h(ref.astype(np.float32), F16))
    else:
        _check(got, ref, hidden_type)
    if hidden_type != F32:
        m32 = _moe(ex, k, F32, T, use_silu)
        want, n32 = _counted(m32, ids, w, widen(xh, hidden_type))
        assert n32 == n
        assert_same_bits(got, to_h(want, hidden_type), f"RAWINT4 grouped {hidden_type}")
        m32.close()
    m.close()


FINE = 1.0 + 2.0 ** -10 + 2.0 ** -20    # bf16 planes hi = 1, mid = 2^-10, lo = 2^-20


def _exact_x(T, H):
    """token t: 2^(t % 3) in group 0 of its row, FINE * 2^(t % 3) in every other 32-value group"""
    x = np.full((T, H), FINE, np.float32)
    x[:, :32] = 1.0
    return x * (2.0 ** (np.arange(T) % 3)).astype(np.float32)[:, None]


def _group_experts(qs, rows, cols, scale_exp):
    """expert e: every row holds q = qs[e][j] in group j (power-of-two q, or 0) and the bf16 scale 2^scale_exp"""
    q = np.stack([np.repeat(np.asarray(qe, np.int8), 32)[None, :].repeat(rows, axis=0) for qe in qs])
    assert q.shape[2] == cols
    s = torch.full((len(qs), rows, cols // 32), 2.0 ** scale_exp, dtype=torch.bfloat16, device="cuda")
    return _pack(torch.from_numpy(o4.pack(q)).cuda(), s), q.astype(np.float64) * 2.0 ** scale_exp


@pytest.mark.gpu
def test_exactness_every_plane_counts():
    """Crafted experts whose every partial sum is an fp32 number, so the output is the float64 value within 2 fp32 ulps.
    Each matrix reads one group: expert 0 gate reads the FINE group 1 and up the coarse group 0, expert 1 the other way
    round, so each of gate and up sees all three planes; a = relu(g) * u is then FINE times a power of two, and down reads
    it in one group.  A dropped mid or lo plane of gate, up or down moves the output by 2^-20 relative or more (>= 4 ulps)."""
    E, k, H, I = 2, 1, 256, 256
    T = max(I4_MIN, 64)
    z = [0] * 8
    gb, gw = _group_experts([[0, 2] + z[2:], [1] + z[1:]], I, H, -4)
    ub, uw = _group_experts([[-4] + z[1:], [0, 2] + z[2:]], I, H, -5)
    db, dw = _group_experts([[0, 0, -2] + z[3:], z[:5] + [1] + z[6:]], H, I, -6)
    from gpu_util import Moe
    m = Moe(E, k, H, I, gb, ub, db, I4, I4, I4, F32, max_tokens=T, use_silu=0)
    x = _exact_x(T, H)
    ids = (np.arange(T) % E).reshape(T, 1).astype(np.int64)
    w = np.ones((T, 1), np.float32)
    got, n = _counted(m, ids, w, x)
    assert n == 10
    x64 = x.astype(np.float64)
    want = np.zeros((T, H))
    for e in range(E):
        t = ids[:, 0] == e
        a = np.maximum(x64[t] @ gw[e].T, 0.0) * (x64[t] @ uw[e].T)
        assert np.array_equal(a.astype(np.float32), a)   # exact in fp32: the kernels' fp32 a is this value
        want[t] = a @ dw[e].T
    assert np.array_equal(want.astype(np.float32), want) and (want != 0).all()
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    err = np.abs(got.astype(np.float64) - want)
    assert (err <= 2 * ulp).all(), float((err / ulp).max())
    m.close()


@pytest.mark.gpu
def test_grouped_matches_per_pair_kernels():
    """same handle, 200 tokens grouped in one call against 40-token per-pair calls: the same fp32 terms summed in another
    order, and no requantisation that could turn an order difference into a step"""
    E, k, H, I, T = 8, 4, 2048, 768, 200
    ex = _Experts(E, H, I, 31)
    m = ex.moe(k, F32, max_tokens=256)
    rng = np.random.default_rng(9)
    ids, w = _hard_ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    x = _x(T, H, 10, F32)[0]
    big, n = _counted(m, ids, w, x)
    assert n == 10
    n0 = native.launch_count()
    step = min(40, I4_MIN - 1)   # per-pair calls: below the threshold
    small = np.concatenate([m.forward(ids[i:i + step], w[i:i + step], x[i:i + step]) for i in range(0, T, step)])
    assert native.launch_count() - n0 == 2 * -(-T // step), "per-pair kernels below the threshold"
    row = np.abs(big.astype(np.float64) - small).max(axis=1) / np.abs(small).max()
    assert row.max() < 1e-5, np.sort(row)[-8:]
    m.close()


@pytest.mark.gpu
def test_grouped_k2_shapes():
    """Kimi-K2 routed experts (E 384, H 7168, I 2048, k 8, BF16) over 16 experts; 1100 tokens span two 1024-token chunks"""
    E, k, H, I = 384, 8, 7168, 2048
    ex = _Experts(E, H, I, 2026)
    rng = np.random.default_rng(11)
    hit = rng.permutation(E)[:16]
    m = ex.moe(k, BF16, max_tokens=1100)
    for qlen in (300, 1100):
        ids = np.stack([rng.permutation(hit)[:k] for _ in range(qlen)]).astype(np.int64)
        w = rng.random((qlen, k)).astype(np.float32)
        x, x64 = _x(qlen, H, qlen, BF16)
        got, n = _counted(m, ids, w, x)
        assert n == 10 * -(-qlen // 1024)
        _check(got, o4.moe_forward(x64, ids, w, ex.expert, E), BF16)
    m.close()


@pytest.mark.gpu
def test_grouped_rows_beyond_bsz_untouched_eager_and_graph():
    """rows >= bsz keep their bytes and rows < bsz equal the full call, eagerly and across graph replays; the grouped scratch
    grows on first use, so a warm-up call at the captured qlen comes first"""
    E, k, H, I, T = 8, 4, 1024, 512, 100
    ex = _Experts(E, H, I, 5)
    m = ex.moe(k, BF16, max_tokens=T)
    rng = np.random.default_rng(1)
    ids = torch.from_numpy(np.stack([rng.permutation(E)[:k] for _ in range(T)]).astype(np.int64)).cuda()
    w = torch.from_numpy(rng.random((T, k)).astype(np.float32)).cuda()
    x = torch.randn((T, H), device="cuda").to(torch.bfloat16)
    bsz = torch.tensor([60], dtype=torch.int32, device="cuda")
    lib = native.lib()

    def call(out, b):
        native.check(lib.ktb200_moe_forward(m.h, T, k, ids.data_ptr(), w.data_ptr(), x.data_ptr(), out.data_ptr(), b,
                                            torch.cuda.current_stream().cuda_stream))

    full = torch.zeros((T, H), dtype=torch.bfloat16, device="cuda")
    call(full, None)
    out = torch.full((T, H), 1234.5, dtype=torch.bfloat16, device="cuda")
    n0 = native.launch_count()
    call(out, bsz.data_ptr())
    torch.cuda.synchronize()
    assert native.launch_count() - n0 == 10
    assert torch.equal(out[:60], full[:60]) and (out[60:] == 1234.5).all()
    s = torch.cuda.Stream()
    out2 = torch.full((T, H), 1234.5, dtype=torch.bfloat16, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            call(out2, bsz.data_ptr())
    torch.cuda.synchronize()
    for b in (30, 100, 1):
        out2.fill_(1234.5)
        bsz.fill_(b)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out2[:b], full[:b]) and (out2[b:] == 1234.5).all(), b
    m.close()


@pytest.mark.gpu
def test_grouped_forward_shared_with_q4k_shared_expert():
    """ktb200_moe_forward_shared: the grouped routed experts, then the Q4_K shared MLP accumulating into the same rows, bit
    for bit the two calls made one after the other"""
    import ctypes as C
    import types
    from gpu_util import dev, moe_forward_shared, stream
    from ktransformers_b200.util.synth import synth_blocks
    E, k, H, I, T = 8, 4, 1024, 512, max(I4_MIN, 64)
    ex = _Experts(E, H, I, 12)
    m = ex.moe(k, F32, max_tokens=T)
    lib = native.lib()
    sw = [synth_blocks(Q4K, I * H, "cuda", s) for s in (1, 2, 3)]
    h = C.c_void_p()
    native.check(lib.ktb200_mlp_create(H, I, *(t.data_ptr() for t in sw), Q4K, Q4K, Q4K, F32, T, torch.cuda.current_device(), C.byref(h)))
    native.check(lib.ktb200_mlp_load_weights(h, stream()))
    rng = np.random.default_rng(13)
    ids, w = _hard_ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    x, x64 = _x(T, H, 14, F32)
    routed, n = _counted(m, ids, w, x)
    assert n == 10
    _check(routed, o4.moe_forward(x64, ids, w, ex.expert, E), F32)
    total = moe_forward_shared(m, types.SimpleNamespace(h=h), ids, w, x)
    x_d, acc = dev(x), torch.from_numpy(routed).cuda()
    native.check(lib.ktb200_mlp_forward(h, T, x_d.data_ptr(), acc.data_ptr(), 1, None, stream()))
    torch.cuda.synchronize()
    assert np.array_equal(total, acc.cpu().numpy())
    assert not np.array_equal(total, routed)
    lib.ktb200_mlp_destroy(h)
    m.close()


@pytest.mark.gpu
def test_grouped_expert_id_offset_shards_sum_to_full():
    E, k, H, I, T = 8, 4, 512, 256, max(I4_MIN, 48)
    ex = _Experts(E, H, I, 9)
    rng = np.random.default_rng(3)
    ids, w = _hard_ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    x, x64 = _x(T, H, 4, F32)
    full, n = _counted(ex.moe(k, F32, max_tokens=T), ids, w, x)
    assert n == 10
    parts = []
    for lo in (0, 4):
        p, n = _counted(ex.moe(k, F32, max_tokens=T, E=4, lo=lo, offset=lo), ids, w, x)
        assert n == 10
        parts.append(p)
    ref = o4.moe_forward(x64, ids, w, ex.expert, E)
    _check(parts[0] + parts[1], ref, F32)
    assert np.abs((parts[0] + parts[1]).astype(np.float64) - full).max() <= 1e-6 * np.abs(ref).max()


@pytest.mark.gpu
def test_grouped_ktmoe_wrapper_prefill(tmp_path):
    """KTMoEWrapper(method="B200_RAWINT4") from a compressed-tensors directory, with a gpu_experts_mask and a physical-to-logical
    map, over a 256-token prefill"""
    from ktransformers_b200.kt_moe_wrapper import KTMoEWrapper
    from test_rawint4 import _write_ct_dir
    E, k, H, I, T = 8, 3, 512, 256, 256
    ref = _write_ct_dir(str(tmp_path), E, H, I, seed=21)
    p2l = torch.tensor([3, 0, 7, 1, 6, 2, 5, 4])
    mask = torch.zeros(E, dtype=torch.bool)
    mask[[2, 5]] = True
    wr = KTMoEWrapper(layer_idx=0, num_experts=E, num_experts_per_tok=k, hidden_size=H, moe_intermediate_size=I,
                      gpu_experts_mask=mask, method="B200_RAWINT4", weight_path=str(tmp_path), chunked_prefill_size=T)
    wr.load_weights(p2l)
    rng = np.random.default_rng(22)
    ids = np.stack([rng.permutation(E)[:k] for _ in range(T)]).astype(np.int64)
    w = rng.random((T, k)).astype(np.float32)
    xb, x64 = _x(T, H, 23, BF16)
    x = torch.from_numpy(xb.view(np.int16)).view(torch.bfloat16).cuda()
    n0 = native.launch_count()
    out = wr.forward(x, torch.from_numpy(ids).cuda(), torch.from_numpy(w).cuda())
    torch.cuda.synchronize()
    assert native.launch_count() - n0 >= 10
    got = out.cpu().view(torch.int16).numpy().view(np.uint16)

    def expert(pslot):
        le = int(p2l[pslot])
        return tuple(o4.dequant(ref[n][0][le], ref[n][1][le].view(torch.int16).numpy().view(np.uint16)) for n in ("gate", "up", "down"))
    ids_m = np.where(mask.numpy()[ids], -1, ids)
    _check(got, o4.moe_forward(x64, ids_m, w, expert, E), BF16)


def _i4_blocks(t, n, seed):
    """RAWINT4 routed tensors packed from random words and scales; the shared expert's Q4_K / Q6_K from synth_blocks"""
    if t == I4:
        g = torch.Generator(device="cuda").manual_seed(seed)
        # rows of 512 columns: a block-aligned split of every real row, so the packed layout is the same
        packed = torch.randint(0, 256, (n // 2,), dtype=torch.uint8, generator=g, device="cuda").view(torch.int32).view(-1, 64)
        scale = (torch.rand((n // 32,), generator=g, device="cuda") * 0.04 + 0.01).to(torch.bfloat16)
        return _pack(packed, scale)
    from ktransformers_b200.util.synth import synth_blocks
    return synth_blocks(t, n, "cuda", seed)


@pytest.mark.gpu
@pytest.mark.parametrize("world,counts", [(2, [300, I4_MIN - 1]), (4, [300, 0, I4_MIN - 1, I4_MIN]), (4, [8, 8, 7, 8])])
def test_grouped_ep_tokens_loopback(world, counts):
    """phase 2 of ktb200_moe_ep_forward_tokens runs the shard's grouped RAWINT4 GEMMs on the gathered rows (F32 out) from
    I4_MIN rows, the per-pair kernels below, against the unsharded layer"""
    from test_ep_tokens import _Loopback
    lb = _Loopback(world, 16, 4, 2048, 512, BF16, 300, types=(I4, I4, I4), shared=True, seed=91, make=_i4_blocks)
    xs = lb.tokens(counts, np.random.default_rng(19))
    ys, idx, w, launches = lb.run(counts, xs)
    lb.check(counts, xs, ys, idx, w)
    gathered = sum(counts) > 100    # 300 tokens x 4 slots over 16 experts reach every shard; fewer than I4_MIN rows otherwise
    assert all((launches[(2, r)] - 2 >= 10) == gathered for r in range(world)), launches
    lb.close()
