"""Q5_K, Q3_K and Q2_K routed experts on the grouped tensor-core GEMM (grouped_gemm_kernel<5> / <6> / <7>, csrc/grouped.cu):
prompts from the K-quant threshold up read each expert once per 32-token tile.  These are the expert tensors of llama.cpp's
Q5_K_M (Q5_K gate / up, Q6_K down), Q3_K_M / Q3_K_L (Q3_K gate / up, Q4_K or Q5_K down) and Q2_K-style mixes (Q2_K / Q3_K).
Checked against the float64 oracle with the tolerances of tests/test_iq_experts.py, against the per-pair kernels, and through
every caller (ktb200_moe_forward / _shared, the device batch size and CUDA graphs, KTMoEWrapper, the expert-parallel layer's
phase 2)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import iq_oracle as oq
from ktransformers_b200 import native
from test_iq_experts import _check, _dequant_f64, _Experts, _ids, _x
from test_iq_grouped import _hard_ids, _moe_ref

Q2K, Q3K, Q4K, Q5K, Q6K = native.GGML_Q2_K, native.GGML_Q3_K, native.GGML_Q4_K, native.GGML_Q5_K, native.GGML_Q6_K
IQ1 = native.GGML_IQ1_S
F32, F16, BF16 = native.GGML_F32, native.GGML_F16, native.GGML_BF16
HERE = os.path.dirname(os.path.abspath(__file__))
# grouped_gemm_kernel<FMT> of a weight type (Q6_K: down tensors in the 4-row tile layout)
GFMT = {Q4K: 0, Q6K: 1, IQ1: 2, Q5K: 5, Q3K: 6, Q2K: 7}
KQ_MIN = 48     # qlen from which a K-quant handle takes the grouped path (csrc/moe.cu grouped_min_qlen)
IQ_MIN = 80     # the same for a handle with an i-quant tensor

KQ_MIXES = {
    "q5k_q5k_q6k": (Q5K, Q5K, Q6K), "q3k_q3k_q4k": (Q3K, Q3K, Q4K), "q2k_q2k_q3k": (Q2K, Q2K, Q3K),
    "q5kx3": (Q5K, Q5K, Q5K), "q3kx3": (Q3K, Q3K, Q3K), "q2k_q2k_q6k": (Q2K, Q2K, Q6K),
    "q4k_q5k_q6k": (Q4K, Q5K, Q6K), "q3k_q2k_q5k": (Q3K, Q2K, Q5K), "q2k_q3k_iq1": (Q2K, Q3K, IQ1),
}


def _min(types):
    return IQ_MIN if IQ1 in types else KQ_MIN


def _small_x(T, H, seed, hidden_type):
    """_x / 16: the outputs of the synthetic K-quant experts then stay well inside the F16 range"""
    x = np.random.default_rng(seed).standard_normal((T, H)).astype(np.float32) / 16
    if hidden_type == BF16:
        from oracle.bindings import f32_to_bf16_bits, bf16_to_f32
        b = f32_to_bf16_bits(x)
        return b, bf16_to_f32(b)
    if hidden_type == F16:
        h = x.astype(np.float16)
        return h, h.astype(np.float32)
    return x, x


def _cpu_blocks(t, n, seed):
    from ktransformers_b200.util.synth import synth_blocks
    return synth_blocks(t, n, "cpu", seed).numpy()


# ------------------------------------------------------------------------------------------------ CPU
def test_batched_reference_is_the_oracle(oracle):
    """_moe_ref (gguf-py dequantisation, the oracle's Q8_K quantiser) against iq_oracle.moe_forward for every new type, on a
    small case with every kind of id"""
    rng = np.random.default_rng(2)
    E, k, H, I, T = 4, 3, 512, 256, 9
    types = (Q5K, Q3K, Q2K)
    blocks = [_cpu_blocks(t, E * r * c, 5 + i).reshape(E, -1) for i, (t, (r, c)) in enumerate(zip(types, ((I, H), (I, H), (H, I))))]

    def expert(e):
        return tuple(_dequant_f64(t, b[e], r, c) for b, t, (r, c) in zip(blocks, types, ((I, H), (I, H), (H, I))))
    ids = _ids(T, E, k, rng)
    ids[2, 1], ids[4, 0], ids[5] = -1, E, [1, 1, 1]
    w = rng.random((T, k)).astype(np.float32)
    x = rng.standard_normal((T, H)).astype(np.float32)
    for silu in (True, False):
        want = oq.moe_forward(oracle, x, ids, w, expert, E, silu)
        got = _moe_ref(oracle, [(x, ids, w)], expert, E, silu)[0]
        assert np.abs(want).max() > 0
        assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("mix", sorted(KQ_MIXES))
def test_grouped_type_mixes_vs_oracle(oracle, mix):
    E, k, H, I = 8, 4, 1024, 512
    types = KQ_MIXES[mix]
    ex = _Experts(E, H, I, *types, 300)
    m = ex.moe(k, F32, max_tokens=300)
    rng = np.random.default_rng(len(mix))
    lo = _min(types)
    cases = []
    for qlen in (lo - 1, lo, 131, 300):
        ids, w = _hard_ids(qlen, E, k, rng), rng.random((qlen, k)).astype(np.float32)
        cases.append((_x(qlen, H, qlen, F32)[0], ids, w))
    refs = _moe_ref(oracle, cases, ex.expert, E)
    for (x, ids, w), ref in zip(cases, refs):
        n0 = native.launch_count()
        got = m.forward(ids, w, x)
        assert native.launch_count() - n0 == (10 if len(ids) >= lo else 2), "grouped from the threshold, per pair below"
        _check(got, ref, F32, (mix, x.shape[0]))
    m.close()


_CENSUS = r"""
import json, sys
import numpy as np, torch
sys.path[:0] = sys.argv[1:]
from torch.profiler import ProfilerActivity, profile
from test_iq_experts import _Experts, _ids, _x
from test_kquant_grouped import KQ_MIXES, _min
res = {}
for mix in sorted(KQ_MIXES):
    T = _min(KQ_MIXES[mix])
    ex = _Experts(8, 1024, 512, *KQ_MIXES[mix], 5)
    m = ex.moe(4, 0, max_tokens=T)
    rng = np.random.default_rng(0)
    ids, w = _ids(T, 8, 4, rng), rng.random((T, 4)).astype(np.float32)
    x = _x(T, 1024, 1, 0)[0]
    m.forward(ids, w, x)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.forward(ids, w, x)
        torch.cuda.synchronize()
    res[mix] = sorted({e.key for e in prof.key_averages() if "kernel" in e.key})
    m.close()
print("CENSUS " + json.dumps(res))
"""


@pytest.mark.gpu
def test_kernels_that_ran_at_the_threshold():
    """every mix runs gate, up and down on grouped_gemm_kernel<FMT of the tensor's type> and nothing per pair (torch.profiler
    in an interpreter of its own: it can miss kernels after other tests' profiler sessions in one process)"""
    root = os.path.dirname(HERE)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CENSUS, HERE, root]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(next(l for l in r.stdout.splitlines() if l.startswith("CENSUS "))[7:])
    assert sorted(res) == sorted(KQ_MIXES)
    for mix, names in res.items():
        ran = {n.split("grouped_gemm_kernel<")[1][0] for n in names if "grouped_gemm_kernel<" in n}
        assert ran == {str(GFMT[t]) for t in KQ_MIXES[mix]}, (mix, names)
        assert not any(s in n for n in names for s in ("rows_", "reduce_", "FmtGenK", "BulkIQ")), (mix, names)


@pytest.mark.gpu
@pytest.mark.parametrize("hidden_type", [F32, F16, BF16])
@pytest.mark.parametrize("use_silu", [1, 0])
def test_grouped_hidden_types_and_activations(oracle, hidden_type, use_silu):
    E, k, H, I, T = 8, 3, 1024, 256, KQ_MIN
    ex = _Experts(E, H, I, Q2K, Q5K, Q3K, 7)
    m = ex.moe(k, hidden_type, max_tokens=T, use_silu=use_silu)
    rng = np.random.default_rng(40)
    ids, w = _ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    x, xf = _small_x(T, H, 41, hidden_type)
    n0 = native.launch_count()
    got = m.forward(ids, w, x)
    assert native.launch_count() - n0 == 10
    _check(got, _moe_ref(oracle, [(xf, ids, w)], ex.expert, E, bool(use_silu))[0], hidden_type)
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["q5k_q5k_q6k", "q3k_q3k_q4k", "q2k_q2k_q3k"])
def test_grouped_matches_per_pair_kernels(mix):
    """The same integer per super-block on both routes; only the fp32 order of the per-super-block terms differs.  That
    moves gate / up outputs in their last bits, and where one lies on a rounding edge of the Q8_K requantisation of
    act(g) * u, one int8 of that token's down input moves by one unit.  So almost every token agrees within 1e-5 of
    max |out|, and every token within a few such units."""
    # a Q6_K down tensor takes the tile layout (so the grouped path) only with an even number of super-blocks per row
    E, k, H, I, T = 8, 4, 2048, 1024 if Q6K in KQ_MIXES[mix] else 768, 200
    ex = _Experts(E, H, I, *KQ_MIXES[mix], 31)
    m = ex.moe(k, F32, max_tokens=256)
    rng = np.random.default_rng(9)
    ids, w = _ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    x = _x(T, H, 10, F32)[0]
    n0 = native.launch_count()
    big = m.forward(ids, w, x)
    assert native.launch_count() - n0 == 10
    step = min(40, KQ_MIN - 1)
    small = np.concatenate([m.forward(ids[i:i + step], w[i:i + step], x[i:i + step]) for i in range(0, T, step)])
    assert native.launch_count() - n0 - 10 <= 2 * -(-T // step), "per-pair kernels for the short calls"
    row = np.abs(big.astype(np.float64) - small).max(axis=1) / np.abs(small).max()
    assert (row < 1e-5).mean() >= 0.95, np.sort(row)[-12:]
    assert row.max() < 1e-3, row.max()
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["q5k_q5k_q6k", "q3k_q3k_q4k", "q2k_q2k_q3k"])
def test_grouped_v3_shapes(oracle, mix):
    """DeepSeek-V3 routed experts (E 256, H 7168, I 2048, k 8, BF16) over 16 experts; 1100 tokens span two 1024-token chunks"""
    E, k, H, I = 256, 8, 7168, 2048
    ex = _Experts(E, H, I, *KQ_MIXES[mix], 2027)
    rng = np.random.default_rng(11)
    hit = rng.permutation(E)[:16]
    cases = []
    for qlen in (300, 1100):
        ids = np.stack([rng.permutation(hit)[:k] for _ in range(qlen)]).astype(np.int64)
        cases.append((_x(qlen, H, qlen, BF16), ids, rng.random((qlen, k)).astype(np.float32)))
    refs = _moe_ref(oracle, [(xf, ids, w) for (_, xf), ids, w in cases], ex.expert, E)
    m = ex.moe(k, BF16, max_tokens=1100)
    for ((x, _), ids, w), ref in zip(cases, refs):
        n0 = native.launch_count()
        got = m.forward(ids, w, x)
        assert native.launch_count() - n0 == 10 * -(-len(ids) // 1024)
        _check(got, ref, BF16, (mix, len(ids)))
    m.close()


@pytest.mark.gpu
def test_grouped_rows_beyond_bsz_untouched_eager_and_graph():
    """rows >= bsz keep their bytes and rows < bsz equal the full call, eagerly and across graph replays; the grouped scratch
    grows on first use, so a warm-up call at the captured qlen comes first"""
    E, k, H, I, T = 8, 4, 1024, 512, 100
    ex = _Experts(E, H, I, Q3K, Q2K, Q5K, 5)
    m = ex.moe(k, BF16, max_tokens=T)
    rng = np.random.default_rng(1)
    ids = torch.from_numpy(_ids(T, E, k, rng)).cuda()
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
def test_grouped_forward_shared_with_q4k_shared_expert(oracle):
    """ktb200_moe_forward_shared: the grouped routed experts (against the oracle), then the Q4_K shared MLP accumulating into
    the same rows, bit for bit the two calls made one after the other"""
    import ctypes as C
    import types
    from gpu_util import dev, moe_forward_shared, stream
    from ktransformers_b200.util.synth import synth_blocks
    E, k, H, I, T = 8, 4, 1024, 512, KQ_MIN
    ex = _Experts(E, H, I, Q2K, Q2K, Q3K, 12)
    m = ex.moe(k, F32, max_tokens=T)
    lib = native.lib()
    sw = [synth_blocks(Q4K, I * H, "cuda", s) for s in (1, 2, 3)]
    h = C.c_void_p()
    native.check(lib.ktb200_mlp_create(H, I, *(t.data_ptr() for t in sw), Q4K, Q4K, Q4K, F32, T, torch.cuda.current_device(), C.byref(h)))
    native.check(lib.ktb200_mlp_load_weights(h, stream()))
    rng = np.random.default_rng(13)
    ids, w = _ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    x, xf = _x(T, H, 14, F32)
    n0 = native.launch_count()
    routed = m.forward(ids, w, x)
    assert native.launch_count() - n0 == 10
    _check(routed, _moe_ref(oracle, [(xf, ids, w)], ex.expert, E)[0], F32)
    total = moe_forward_shared(m, types.SimpleNamespace(h=h), ids, w, x)
    x_d, acc = dev(x), torch.from_numpy(routed).cuda()
    native.check(lib.ktb200_mlp_forward(h, T, x_d.data_ptr(), acc.data_ptr(), 1, None, stream()))
    torch.cuda.synchronize()
    assert np.array_equal(total, acc.cpu().numpy())
    assert not np.array_equal(total, routed)
    lib.ktb200_mlp_destroy(h)
    m.close()


@pytest.mark.gpu
def test_grouped_ktmoe_wrapper_prefill(oracle):
    """KTMoEWrapper(method="B200_GGUF") with Q5_K / Q3_K / Q2_K experts and a gpu_experts_mask over a 256-token prefill"""
    from ktransformers_b200.kt_moe_wrapper import KTMoEWrapper
    E, k, H, I, T = 8, 3, 512, 256, 256
    types = (Q5K, Q3K, Q2K)
    rng = np.random.default_rng(21)
    blocks = {n: _cpu_blocks(t, E * r * c, 30 + i).reshape(E, r, -1)
              for i, (n, t, (r, c)) in enumerate(zip(("gate", "up", "down"), types, ((I, H), (I, H), (H, I))))}
    p2l = torch.tensor([3, 0, 7, 1, 6, 2, 5, 4])
    mask = torch.zeros(E, dtype=torch.bool)
    mask[[2, 5]] = True
    wr = KTMoEWrapper(layer_idx=0, num_experts=E, num_experts_per_tok=k, hidden_size=H, moe_intermediate_size=I,
                      gpu_experts_mask=mask, method="B200_GGUF", chunked_prefill_size=T)
    wr.load_weights_from_tensors(*(torch.from_numpy(blocks[n]) for n in ("gate", "up", "down")), p2l, ggml_types=types)
    ids, w = _ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    xb, xf = _x(T, H, 23, BF16)
    x = torch.from_numpy(xb.view(np.int16)).view(torch.bfloat16).cuda()
    n0 = native.launch_count()
    out = wr.forward(x, torch.from_numpy(ids).cuda(), torch.from_numpy(w).cuda())
    torch.cuda.synchronize()
    assert native.launch_count() - n0 >= 10
    got = out.cpu().view(torch.int16).numpy().view(np.uint16)

    def expert(pslot):
        le = int(p2l[pslot])
        return tuple(_dequant_f64(t, blocks[n][le].reshape(-1), r, c)
                     for n, t, (r, c) in zip(("gate", "up", "down"), types, ((I, H), (I, H), (H, I))))
    ids_m = np.where(mask.numpy()[ids], -1, ids)
    _check(got, _moe_ref(oracle, [(xf, ids_m, w)], expert, E)[0], BF16)


@pytest.mark.gpu
@pytest.mark.parametrize("world,counts", [(2, [300, KQ_MIN - 1]), (4, [300, 0, KQ_MIN - 1, KQ_MIN]), (2, [20, KQ_MIN - 21]),
                                          (4, [12, 12, 12, KQ_MIN - 36])])
def test_grouped_ep_tokens_loopback(world, counts):
    """phase 2 of ktb200_moe_ep_forward_tokens runs the shard's grouped K-quant GEMMs on the gathered rows (F32 out) from
    KQ_MIN rows, the per-pair kernels below, against the unsharded layer"""
    from test_ep_tokens import _Loopback
    lb = _Loopback(world, 16, 4, 2048, 512, BF16, 300, types=(Q2K, Q2K, Q3K), shared=True, seed=91)
    xs = lb.tokens(counts, np.random.default_rng(19))
    ys, idx, w, launches = lb.run(counts, xs)
    lb.check(counts, xs, ys, idx, w)
    gathered = sum(counts) >= KQ_MIN
    assert all((launches[(2, r)] - 2 >= 10) == gathered for r in range(world)), launches
    lb.close()
