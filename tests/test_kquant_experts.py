"""Q2_K and Q3_K routed experts on the bulk-copy decode kernels: gate/up on rows_bulk_iq_kernel<BulkQ2K | BulkQ3K> (csrc/iq.cuh)
and down on reduce_bulk_kernel<BulkQ2K | BulkQ3K> (csrc/gemv_bulk.cuh), below the grouped threshold.  These are the expert
tensors of llama.cpp's Q2_K (Q2_K gate / up, Q3_K down), Q3_K_S (Q3_K x3) and Q3_K_M / Q3_K_L (Q3_K gate / up, Q4_K or Q5_K
down) files.  Checked against the float64 oracle with the tolerances of tests/test_iq_experts.py, against the grouped GEMM at
the same qlen, and through every caller (ktb200_moe_forward / _shared, the block entry point's fallback, the device batch
size and CUDA graphs, expert_id_offset shards, KTMoEWrapper)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import iq_oracle as oq
from ktransformers_b200 import native
from test_iq_experts import _check, _dequant_f64, _Experts, _ids, _wrapper, _wrapper_check, _x
from test_iq_grouped import _moe_ref
from test_kquant_grouped import _cpu_blocks, _small_x

Q2K, Q3K, Q4K, Q5K, Q6K = native.GGML_Q2_K, native.GGML_Q3_K, native.GGML_Q4_K, native.GGML_Q5_K, native.GGML_Q6_K
F32, F16, BF16 = native.GGML_F32, native.GGML_F16, native.GGML_BF16
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

MIXES = {
    "q2k_q2k_q3k": (Q2K, Q2K, Q3K), "q3k_q3k_q4k": (Q3K, Q3K, Q4K), "q3kx3": (Q3K, Q3K, Q3K), "q2kx3": (Q2K, Q2K, Q2K),
    "q3k_q3k_q5k": (Q3K, Q3K, Q5K), "q4k_q4k_q3k": (Q4K, Q4K, Q3K), "q2k_q2k_q6k": (Q2K, Q2K, Q6K),
}
BULK = {Q2K: "BulkQ2K", Q3K: "BulkQ3K"}


def bulk_route(types, H, I, routed=True, shared=None):
    """Restatement of csrc/moe.cu's choice below the grouped threshold for the Q2_K / Q3_K tensors of a handle: the bulk-copy
    item format of (gate/up, down), None where the generic FmtGenK kernels run (or the tensor is of another type).
    routed: a routed-expert launch (expert ids); shared: None, "all" (a shared expert of every token rides in the launch) or
    "token" (the expert-parallel layer's shared expert of one token).  The shared-memory planners find room at every shape
    used here."""
    gt, ut, dt = types
    nblk, nb = H // 256, I // 256
    ok = routed and shared != "token"
    gu = BULK.get(gt) if ok and gt == ut and nblk % 4 == 0 and I % 2 == 0 else None
    dn = BULK.get(dt) if ok and H % 4 == 0 and (dt == Q2K or nb % 2 == 0) else None
    return gu, dn


def _decode_ids(T, E, k, rng):
    """distinct random ids, then: expert 1 in every token (a crowded expert, a duplicate where the row already had it), an id
    below and one above the shard, and expert 2 picked by nobody"""
    ids = _ids(T, E, k, rng)
    ids[ids == 2] = 3
    ids[:, 0] = 1
    ids[0, k - 1] = -1
    if T > 1:
        ids[T - 1, 1] = E + 3
    return ids


# ------------------------------------------------------------------------------------------------ CPU
def test_route_predicate():
    v3 = (7168, 2048)
    assert bulk_route((Q2K, Q2K, Q3K), *v3) == ("BulkQ2K", "BulkQ3K")
    assert bulk_route((Q3K, Q3K, Q4K), *v3) == ("BulkQ3K", None)
    assert bulk_route((Q3K, Q3K, Q3K), *v3) == ("BulkQ3K", "BulkQ3K")
    assert bulk_route((Q4K, Q4K, Q3K), *v3) == (None, "BulkQ3K")
    assert bulk_route((Q2K, Q3K, Q3K), *v3) == (None, "BulkQ3K"), "mixed gate / up"
    assert bulk_route((Q2K, Q2K, Q3K), 1280, 512) == (None, "BulkQ3K"), "5 blocks per gate row"
    assert bulk_route((Q3K, Q3K, Q3K), 512, 768) == (None, None), "2 blocks per gate row, 3 per down row"
    assert bulk_route((Q2K, Q2K, Q2K), 1024, 768) == ("BulkQ2K", "BulkQ2K"), "Q2_K items are aligned at any nb"
    assert bulk_route((Q2K, Q2K, Q3K), *v3, routed=False) == (None, None), "MLPs and linears"
    assert bulk_route((Q2K, Q2K, Q3K), *v3, shared="all") == ("BulkQ2K", "BulkQ3K")
    assert bulk_route((Q2K, Q2K, Q3K), *v3, shared="token") == (None, None)


@pytest.mark.parametrize("seed", [1, 2])
def test_decode_ids_cover_the_cases(seed):
    E, k = 8, 4
    for T in (1, 2, 8, 9, 47):
        ids = _decode_ids(T, E, k, np.random.default_rng(seed))
        assert (ids[:, 0] == 1).all() and (ids == -1).any() and not (ids == 2).any()
        if T > 1:
            assert (ids >= E).any()
        if T >= 8:
            valid = [r[(r >= 0) & (r < E)].tolist() for r in ids]
            assert any(len(set(v)) < len(v) for v in valid), "a duplicate id"


# ------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("mix", sorted(MIXES))
def test_type_mixes_vs_oracle(oracle, mix):
    E, k, H, I = 8, 4, 1024, 512
    ex = _Experts(E, H, I, *MIXES[mix], 400)
    m = ex.moe(k, F32, max_tokens=47)
    rng = np.random.default_rng(len(mix))
    cases = []
    for qlen in (1, 2, 8, 9, 47):
        cases.append((_x(qlen, H, qlen, F32)[0], _decode_ids(qlen, E, k, rng), rng.random((qlen, k)).astype(np.float32)))
    for (x, ids, w), ref in zip(cases, _moe_ref(oracle, cases, ex.expert, E)):
        n0 = native.launch_count()
        got = m.forward(ids, w, x)
        assert native.launch_count() - n0 == 2
        _check(got, ref, F32, (mix, len(ids)))
    m.close()


# every census case in ONE torch.profiler session, in an interpreter of its own (as tests/test_iq_experts.py: a session can
# come back without some kernels after other sessions in the same process); kernels are attributed to calls by launch order
CENSUS_CASES = {   # name: (types, H, I, fused shared expert of the routed types)
    **{m: (t, 1024, 512, False) for m, t in MIXES.items()},
    "q2k_q2k_q3k H1280": ((Q2K, Q2K, Q3K), 1280, 512, False),
    "q3kx3 H512 I768": ((Q3K, Q3K, Q3K), 512, 768, False),
    "q2k_q3k_q3k mixed": ((Q2K, Q3K, Q3K), 1024, 512, False),
    "q2k_q2k_q3k shared": ((Q2K, Q2K, Q3K), 1024, 512, True),
}
_CENSUS = r"""
import json, sys
import numpy as np, torch
sys.path[:0] = sys.argv[1:]
from torch.profiler import ProfilerActivity, profile
from ktransformers_b200 import native
from gpu_util import Mlp, moe_forward_shared
from test_iq_experts import _Experts, _ids, _x
from test_kquant_experts import CENSUS_CASES
cases = []
for key, (types, H, I, sh) in sorted(CENSUS_CASES.items()):
    ex = _Experts(8, H, I, *types, 70)
    rng = np.random.default_rng(71)
    mlp = Mlp(H, I, *(b.view(8, -1)[7].clone() for b in ex.w), *types, 0) if sh else None
    cases.append((key, ex.moe(4, 0), mlp, _ids(3, 8, 4, rng), rng.random((3, 4)).astype(np.float32), _x(3, H, 72, 0)[0]))
torch.cuda.synchronize()
counts = []
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _, m, mlp, ids, w, x in cases:
        n0 = native.launch_count()
        moe_forward_shared(m, mlp, ids, w, x) if mlp is not None else m.forward(ids, w, x)
        torch.cuda.synchronize()
        counts.append(native.launch_count() - n0)
names = [e.name for e in sorted((e for e in prof.events() if "ktb::" in e.name), key=lambda e: e.time_range.start)]
assert len(names) == sum(counts), f"{len(names)} library kernels recorded, {sum(counts)} launched: {names}"
res, i = {}, 0
for (key, *_), n in zip(cases, counts):
    res[key] = names[i:i + n]
    i += n
print("CENSUS " + json.dumps(res))
"""


@pytest.fixture(scope="module")
def kernel_census():
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CENSUS, HERE, ROOT]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return json.loads(next(l for l in r.stdout.splitlines() if l.startswith("CENSUS "))[7:])


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CENSUS_CASES))
def test_kernels_that_ran(kernel_census, case):
    """two launches; the new instantiations where bulk_route says so, FmtGenK for every Q2_K / Q3_K tensor it does not"""
    types, H, I, sh = CENSUS_CASES[case]
    names = kernel_census[case]
    assert len(names) == 2, names
    gu, dn = bulk_route(types, H, I, shared="all" if sh else None)
    gate_up = [n for n in names if "rows_" in n]
    down = [n for n in names if "reduce_" in n]
    assert len(gate_up) == 1 and len(down) == 1, names
    if gu:
        assert f"rows_bulk_iq_kernel<ktb::{gu}," in gate_up[0], names
    elif types[0] in BULK:
        assert "rows_kernel<ktb::FmtGenK," in gate_up[0], names
    if dn:
        assert f"reduce_bulk_kernel<ktb::{dn}," in down[0], names
    elif types[2] in BULK:
        assert "reduce_kernel<ktb::FmtGenK," in down[0], names


@pytest.mark.gpu
@pytest.mark.parametrize("hidden_type", [F32, F16, BF16])
@pytest.mark.parametrize("use_silu", [1, 0])
def test_hidden_types_and_activations(oracle, hidden_type, use_silu):
    E, k, H, I = 8, 3, 1024, 512
    ex = _Experts(E, H, I, Q2K, Q2K, Q3K, 7)
    m = ex.moe(k, hidden_type, use_silu=use_silu)
    rng = np.random.default_rng(40)
    for qlen in (1, 8):
        ids, w = _ids(qlen, E, k, rng), rng.random((qlen, k)).astype(np.float32)
        x, xf = _small_x(qlen, H, 41 + qlen, hidden_type)
        _check(m.forward(ids, w, x), _moe_ref(oracle, [(xf, ids, w)], ex.expert, E, bool(use_silu))[0], hidden_type, qlen)
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["q2k_q2k_q3k", "q3k_q3k_q4k", "q3kx3"])
def test_v3_shapes(oracle, mix):
    """DeepSeek-V3 routed experts (E 256, H 7168, I 2048, k 8, BF16) over 16 experts at decode and short-prompt sizes"""
    E, k, H, I = 256, 8, 7168, 2048
    ex = _Experts(E, H, I, *MIXES[mix], 2028)
    rng = np.random.default_rng(12)
    hit = rng.permutation(E)[:16]
    cases = []
    for qlen in (1, 8, 47):
        ids = np.stack([rng.permutation(hit)[:k] for _ in range(qlen)]).astype(np.int64)
        cases.append((_x(qlen, H, qlen, BF16), ids, rng.random((qlen, k)).astype(np.float32)))
    refs = _moe_ref(oracle, [(xf, ids, w) for (_, xf), ids, w in cases], ex.expert, E)
    m = ex.moe(k, BF16, max_tokens=47)
    for ((x, _), ids, w), ref in zip(cases, refs):
        n0 = native.launch_count()
        got = m.forward(ids, w, x)
        assert native.launch_count() - n0 == 2
        _check(got, ref, BF16, (mix, len(ids)))
    m.close()


@pytest.mark.gpu
def test_rows_beyond_bsz_untouched_eager_and_graph():
    """rows >= *bsz keep their NaN sentinels and rows < *bsz equal the full call, eagerly and across graph replays"""
    E, k, H, I, T = 8, 4, 1024, 512, 8
    ex = _Experts(E, H, I, Q2K, Q2K, Q3K, 5)
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
    out = torch.full((T, H), float("nan"), dtype=torch.bfloat16, device="cuda")
    n0 = native.launch_count()
    call(out, bsz.data_ptr())
    torch.cuda.synchronize()
    assert native.launch_count() - n0 == 2
    assert torch.equal(out[:5], full[:5]) and out[5:].isnan().all()
    s = torch.cuda.Stream()
    out2 = torch.full((T, H), float("nan"), dtype=torch.bfloat16, device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            call(out2, bsz.data_ptr())
    torch.cuda.synchronize()
    for b in (3, 8, 1):
        out2.fill_(float("nan"))
        bsz.fill_(b)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out2[:b], full[:b]) and out2[b:].isnan().all(), b
    m.close()


@pytest.mark.gpu
def test_shared_expert_of_routed_types_rides_in_the_launches(oracle):
    """a Q2_K/Q2_K/Q3_K shared expert of routed shape is slot k of the same two launches (the census shows them on the new
    kernels): routed experts plus the shared expert's MLP against the oracle"""
    from gpu_util import Mlp, moe_forward_shared
    E, k, H, I = 8, 4, 1024, 512
    types = (Q2K, Q2K, Q3K)
    ex = _Experts(E, H, I, *types, 15)
    sh = [b.view(E, -1)[6].clone() for b in ex.w]   # expert 6's tensors as the shared expert
    m = ex.moe(k, F32)
    mlp = Mlp(H, I, *sh, *types, F32)
    rng = np.random.default_rng(16)
    for T in (1, 8):
        ids, w = _ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
        x, xf = _x(T, H, 17 + T, F32)
        n0 = native.launch_count()
        got = moe_forward_shared(m, mlp, ids, w, x)
        assert native.launch_count() - n0 == 2
        routed = _moe_ref(oracle, [(xf, ids, w)], ex.expert, E)[0]
        shared = _moe_ref(oracle, [(xf, np.zeros((T, 1), np.int64), np.ones((T, 1), np.float32))], lambda e: ex.expert(6), 1)[0]
        _check(got, routed + shared, F32, T)
    mlp.close()
    m.close()


@pytest.mark.gpu
def test_q4k_shared_expert_runs_separately():
    from gpu_util import Mlp, mlp_forward, moe_forward_shared
    from ktransformers_b200.util.synth import synth_blocks
    E, k, H, I, T = 8, 4, 1024, 512, 3
    ex = _Experts(E, H, I, Q2K, Q2K, Q3K, 12)
    m = ex.moe(k, F32)
    sw = [synth_blocks(Q4K, I * H, "cuda", s) for s in (1, 2, 3)]
    mlp = Mlp(H, I, *sw, Q4K, Q4K, Q4K, F32)
    rng = np.random.default_rng(13)
    ids, w = _ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    x, _ = _x(T, H, 14, F32)
    routed = m.forward(ids, w, x)
    shared = mlp_forward(H, I, *sw, Q4K, Q4K, Q4K, F32, x)
    assert np.array_equal(moe_forward_shared(m, mlp, ids, w, x), (routed + shared).astype(np.float32))
    mlp.close()
    m.close()


@pytest.mark.gpu
def test_expert_id_offset_shards_and_skipped_ids(oracle):
    E, k, H, I, T = 8, 4, 1024, 512, 5
    ex = _Experts(E, H, I, Q2K, Q2K, Q3K, 9)
    rng = np.random.default_rng(3)
    ids, w = _ids(T, E, k, rng), rng.random((T, k)).astype(np.float32)
    ids[0, 1], ids[2, 0], ids[3, 3] = -1, E, E + 7
    x, xf = _x(T, H, 4, F32)
    full = ex.moe(k, F32).forward(ids, w, x)
    parts = [ex.moe(k, F32, E=4, lo=lo, offset=lo).forward(ids, w, x) for lo in (0, 4)]
    ref = _moe_ref(oracle, [(xf, ids, w)], ex.expert, E)[0]
    _check(full, ref, F32)
    assert np.abs((parts[0] + parts[1]).astype(np.float64) - full).max() <= 1e-6 * np.abs(ref).max()


def _kq_blocks(types, E, H, I, seed):
    return {n: _cpu_blocks(t, E * r * c, seed + i).reshape(E, r, -1)
            for i, (n, t, (r, c)) in enumerate(zip(("gate", "up", "down"), types, ((I, H), (I, H), (H, I))))}


@pytest.mark.gpu
def test_ktmoe_wrapper_from_tensors(oracle):
    E, k, H, I = 8, 3, 1024, 512
    types = (Q2K, Q2K, Q3K)
    blocks = _kq_blocks(types, E, H, I, 50)
    p2l = torch.tensor([3, 0, 7, 1, 6, 2, 5, 4])
    mask = torch.zeros(E, dtype=torch.bool)
    mask[[2, 5]] = True
    wr = _wrapper(gpu_experts_mask=mask, hidden_size=H, moe_intermediate_size=I)
    wr.load_weights_from_tensors(*(torch.from_numpy(blocks[n]) for n in ("gate", "up", "down")), p2l, ggml_types=types)
    _wrapper_check(oracle, wr, blocks, p2l, mask, E, k, H, I, types)


@pytest.mark.gpu
def test_ktmoe_wrapper_from_gguf(oracle, tmp_path):
    import gguf
    E, k, H, I = 8, 3, 1024, 512
    types = (Q3K, Q3K, Q3K)
    blocks = _kq_blocks(types, E, H, I, 60)
    wtr = gguf.GGUFWriter(str(tmp_path / "kq.gguf"), "deepseek2")
    for n, t in zip(("gate", "up", "down"), types):
        wtr.add_tensor(f"blk.0.ffn_{n}_exps.weight", blocks[n], raw_dtype=gguf.GGMLQuantizationType(t))
    wtr.write_header_to_file()
    wtr.write_kv_data_to_file()
    wtr.write_tensors_to_file()
    wtr.close()
    p2l = torch.tensor([1, 0, 3, 2, 5, 4, 7, 6])
    mask = torch.zeros(E, dtype=torch.bool)
    mask[[0, 6]] = True
    wr = _wrapper(gpu_experts_mask=mask, hidden_size=H, moe_intermediate_size=I, weight_path=str(tmp_path),
                  key_template="blk.{layer}")
    wr.load_weights(p2l)
    _wrapper_check(oracle, wr, blocks, p2l, mask, E, k, H, I, types)


@pytest.mark.gpu
def test_moe_block_forward_takes_the_separate_launches():
    """the persistent block kernel takes Q4_K gate / up only: the block entry point falls back to the router and
    ktb200_moe_forward_shared, bit for bit"""
    from gpu_util import Gate, Mlp, gate_forward, moe_block_forward, moe_forward_shared
    E, k, H, I, T = 16, 4, 1024, 512, 3
    types = (Q2K, Q2K, Q3K)
    ex = _Experts(E, H, I, *types, 11)
    m = ex.moe(k, BF16)
    mlp = Mlp(H, I, *(b.view(E, -1)[0].clone() for b in ex.w), *types, BF16)
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
def test_forward_ep_keeps_refusing():
    """the expert-parallel layer's per-token shared slot has no Q2_K / Q3_K kernel: the same error as before"""
    from gpu_util import Mlp
    E, k, H, I = 8, 2, 1024, 512
    types = (Q2K, Q2K, Q3K)
    ex = _Experts(E, H, I, *types, 13)
    m = ex.moe(k, BF16)
    mlp = Mlp(H, I, *(b.view(E, -1)[0].clone() for b in ex.w), *types, BF16)
    ids = torch.zeros((1, k), dtype=torch.int64, device="cuda")
    wt = torch.ones((1, k), device="cuda")
    x = torch.zeros((1, H), dtype=torch.bfloat16, device="cuda")
    part, sh = torch.zeros((1, H), device="cuda"), torch.zeros((H,), dtype=torch.bfloat16, device="cuda")
    rc = native.lib().ktb200_moe_forward_ep(m.h, mlp.h, 1, k, ids.data_ptr(), wt.data_ptr(), x.data_ptr(), part.data_ptr(), 0,
                                            sh.data_ptr(), None, torch.cuda.current_stream().cuda_stream)
    assert rc == native.EINVAL and "per-token shared slot" in native.lib().ktb200_last_error().decode()
    mlp.close()
    m.close()


_ROUTE_RUN = r"""
import sys
import numpy as np
sys.path[:0] = sys.argv[1:3]
from ktransformers_b200 import native
from test_iq_experts import _Experts, _ids, _x
from test_kquant_experts import MIXES
mix, T, path = sys.argv[3], int(sys.argv[4]), sys.argv[5]
ex = _Experts(8, 2048, 1024, *MIXES[mix], 31)
m = ex.moe(4, 0, max_tokens=T)
rng = np.random.default_rng(9)
ids, w = _ids(T, 8, 4, rng), rng.random((T, 4)).astype(np.float32)
n0 = native.launch_count()
np.save(path, m.forward(ids, w, _x(T, 2048, 10, 0)[0]))
print("LAUNCHES", native.launch_count() - n0)
"""


@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["q2k_q2k_q3k", "q3k_q3k_q4k"])
def test_per_pair_matches_grouped_at_the_same_qlen(mix, tmp_path):
    """40 tokens through the grouped GEMM (KTB200_GROUPED_MIN=1) and through the per-pair kernels (the threshold above 40),
    in two interpreters (the threshold is read once per process).  The same integer per super-block on both routes; only the
    fp32 order of the per-super-block terms differs, so almost every token agrees within 1e-5 of max |out| and, where a gate /
    up output lies on a rounding edge of the Q8_K requantisation of act(g) * u, every token within a few such units."""
    T = 40
    outs = {}
    for arm, env_min in (("grouped", "1"), ("per-pair", "1000")):
        env = dict(os.environ, KTB200_GROUPED_MIN=env_min)
        cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _ROUTE_RUN, HERE, ROOT, mix, str(T),
                                                                                 str(tmp_path / f"{arm}.npy")]
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env=env)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
        launches = int(next(l for l in r.stdout.splitlines() if l.startswith("LAUNCHES "))[9:])
        assert launches == (10 if arm == "grouped" else 2), (arm, launches)
        outs[arm] = np.load(tmp_path / f"{arm}.npy").astype(np.float64)
    row = np.abs(outs["grouped"] - outs["per-pair"]).max(axis=1) / np.abs(outs["per-pair"]).max()
    assert (row < 1e-5).mean() >= 0.95, np.sort(row)[-12:]
    assert row.max() < 1e-3, row.max()
