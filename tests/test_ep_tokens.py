"""ktb200_moe_ep_forward_tokens: the expert-parallel MoE layer for any number of tokens per rank (include/ktb200.h).

CPU: argument checks, region arithmetic, the per-step count exchange under gloo.
GPU, one H100, loopback: `world` shard handles with their own regions in one device's memory; phases 1, 2 and 4 run rank by
rank (a legal schedule of the real concurrent execution), phase 7 at world 1.  World 1 is bit-identical to the gate followed
by ktb200_moe_forward and ktb200_mlp_forward as two rounded terms; world > 1 has the same routing bits and output within fp32
re-association of the cross-rank sum.  Rows a rank does not need start as NaN and must keep their bits."""
import copy
import ctypes as C
import functools
import os
import socket
import types

import numpy as np
import pytest
import torch

from ktransformers_b200 import native

Q4_K, Q6_K, IQ1_S, F32, F16, BF16 = 12, 14, 19, 0, 1, 30


# ------------------------------------------------------------------------------------------------ CPU
def test_ep_tokens_argument_checks_need_no_gpu():
    lib = native.lib()
    ok = dict(rank=0, world=2, tmax=4, H=256, ht=BF16, k=2, bufs=[16, 32])

    def call(counts=(1, 2), phase=7, x=16, **kw):
        a = dict(ok, **kw)
        comm = native.EpTokensComm.make(a["rank"], a["world"], a["tmax"], a["H"], a["ht"], a["k"], a["bufs"])
        cnt = (C.c_int * len(counts))(*counts)
        return lib.ktb200_moe_ep_forward_tokens(None, None, None, C.byref(comm), cnt, x, 16, 16, 16, phase, None)

    cases = [(dict(rank=2), "rank"), (dict(world=0, bufs=[]), "world"), (dict(world=17, bufs=[16] * 17), "world"),
             (dict(bufs=[16, 0]), "null peer pointer for rank 1"), (dict(bufs=[16, 40]), "rank 1 is not 16-byte aligned"),
             (dict(x=24), "x_own must be 16-byte aligned"), (dict(tmax=0), "max_tokens_per_rank"),
             (dict(H=250), "hidden_size"), (dict(ht=Q4_K), "hidden_type"), (dict(k=0), "top_k")]
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            native.check(call(**kw))
    for counts in ((5, 0), (0, -1)):
        with pytest.raises(ValueError, match=r"counts\[\d\] = -?\d+ outside \[0, max_tokens_per_rank = 4\]"):
            native.check(call(counts))
    with pytest.raises(ValueError, match="phase_mask"):
        native.check(call(phase=8))
    with pytest.raises(ValueError, match="null gate config or expert handle"):     # everything else valid: the handles come next
        native.check(call())
    with pytest.raises(ValueError, match="null comm or counts"):
        native.check(lib.ktb200_moe_ep_forward_tokens(None, None, None, None, None, 16, 16, 16, 16, 7, None))


def test_ep_tokens_region_arithmetic():
    up = lambda n: (n + 255) // 256 * 256  # noqa: E731
    for world, tmax, H, ht, k in ((1, 1, 256, BF16, 1), (2, 5, 512, F16, 4), (8, 1024, 7168, BF16, 8), (3, 7, 2048, F32, 6)):
        n, off = native.ep_tokens_layout(world, tmax, H, ht, k)
        R, hb = world * tmax, {F32: 4, F16: 2, BF16: 2}[ht]
        assert off["x"] == 0
        assert off["ids"] == up(R * H * hb)
        assert off["weights"] == off["ids"] + up(R * k * 8)
        assert off["partial"] == off["weights"] + up(R * k * 4)
        assert off["scratch"] == off["partial"] + up(R * H * 4)
        assert off["flags"] == off["scratch"] + up(min(R, 1024) * H * 4)
        assert n == off["flags"] + up(4 * (2 * world + 5))
    n, off = native.ep_tokens_layout(8, 1024, 7168, BF16, 8)
    assert off["scratch"] - off["partial"] == 8 * 1024 * 7168 * 4          # 235 MB of partial rows at V3 prefill sizes
    for bad in ((0, 4, 256, BF16, 2), (17, 4, 256, BF16, 2), (2, 0, 256, BF16, 2), (2, 4, 252, BF16, 2), (2, 4, 256, Q4_K, 2),
                (2, 4, 256, BF16, 33)):
        with pytest.raises(ValueError):
            native.ep_tokens_layout(*bad)


def test_peer_exchange_region_offsets():
    from ktransformers_b200.operators.expert_parallel import exchange_layout
    lib = native.lib()
    for world, H, ht, k, tmax in ((2, 4096, BF16, 4, 64), (8, 7168, BF16, 8, 128)):
        lay = exchange_layout(world, H, ht, k, tmax)
        msg = world * lib.ktb200_ep_msg_bytes(H, ht)
        assert lay["message"] == 0 and lay["partial"] >= msg and lay["partial"] % 256 == 0
        assert lay["flags"] >= lay["partial"] + world * H * 4 and lay["flags"] % 256 == 0
        assert lay["tokens"] >= lay["flags"] + 4 * (2 * world + 2) and lay["tokens"] % 256 == 0
        n, off = native.ep_tokens_layout(world, tmax, H, ht, k)
        assert lay["token_regions"] == off and lay["bytes"] == lay["tokens"] + n


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _count_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from ktransformers_b200.operators.expert_parallel import StepTokenCounts
        st = StepTokenCounts(layers_per_step=2)
        got = []
        for step, n in enumerate(([5, 0, 47], [1, 1, 1])):
            got.append(st.begin_step(n[rank]))
            assert list(st.take(n[rank])) == n and list(st.take(n[rank])) == n     # one take per layer
            assert st.take(n[rank]) is None                                          # expired: the next step announced nothing
        st.begin_step(n[rank])
        try:
            st.take(99)
            got.append("no error")
        except RuntimeError as e:
            got.append("begin_step" in str(e))
        st.end_step()
        got.append(st.take(1))
        q.put((rank, got))
    finally:
        dist.destroy_process_group()


def test_step_token_counts_one_gloo_all_gather_per_step():
    import torch.multiprocessing as mp
    world, port = 3, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ps = [ctx.Process(target=_count_worker, args=(r, world, port, q)) for r in range(world)]
    for p in ps:
        p.start()
    res = dict(q.get(timeout=120) for _ in range(world))
    for p in ps:
        p.join(timeout=60)
    for r in range(world):
        assert res[r] == [[5, 0, 47], [1, 1, 1], True, None], res[r]


# ------------------------------------------------------------------------------------------------ GPU helpers
def _bits(t):
    return t.view(torch.int16).cpu().numpy().view(np.uint16) if t.dtype == torch.bfloat16 else t.cpu().numpy()


def _assert_close(got, want, ht):
    """fp32 re-association of the cross-rank sum: within 2 units of the hidden type's last place, mostly exact"""
    if ht == BF16:
        a = (got.astype(np.uint32) << 16).view(np.float32)
        b = (want.astype(np.uint32) << 16).view(np.float32)
        eps, exact = 2.0 ** -7, 0.9
    else:
        a, b = got.astype(np.float32), want.astype(np.float32)
        eps, exact = (2.0 ** -10, 0.5) if ht == F16 else (2.0 ** -20, 0.0)
    assert np.isfinite(a).all()
    assert (np.abs(a - b) <= 2 * eps * np.maximum(np.abs(a), np.abs(b)) + 1e-3 * np.abs(b).max()).all()
    assert (got == want).mean() >= exact, (got == want).mean()


def _mlp_accumulate(mlp, group_max_len, x, y):
    """y += round(shared(x)) with ktb200_mlp_forward, in chunks of the handle's group_max_len (rows are independent)"""
    for t0 in range(0, x.shape[0], group_max_len):
        xs, ys = x[t0:t0 + group_max_len], y[t0:t0 + group_max_len]
        native.check(native.lib().ktb200_mlp_forward(mlp, xs.shape[0], xs.data_ptr(), ys.data_ptr(), 1, None,
                                                     torch.cuda.current_stream().cuda_stream))


class _Loopback:
    """`world` shard handles on one GPU with one region each, laid out like PeerExchange (the one-token block's buffers
    first, then the multi-token region); everything the layer must not write starts as NaN bytes."""

    def __init__(self, world, E, k, H, I, ht, tmax, types=(Q4_K, Q4_K, Q6_K), shared=True, seed=0, ng=4, tg=2, make=None):
        import gpu_util as G
        from ktransformers_b200.operators.expert_parallel import exchange_layout
        self.G, self.world, self.E, self.k, self.H, self.I, self.ht, self.tmax = G, world, E, k, H, I, ht, tmax
        make = make or (lambda t, n, s: __import__("ktransformers_b200.util.synth", fromlist=["x"]).synth_blocks(t, n, "cuda", s))
        gt, ut, dt = types
        full = [make(gt, E * I * H, seed + 1), make(ut, E * I * H, seed + 2), make(dt, E * H * I, seed + 3)]
        sgs = (make(Q4_K, I * H, seed + 4), make(Q4_K, I * H, seed + 5), make(Q6_K, H * I, seed + 6)) if shared else None
        rng = np.random.default_rng(seed)
        self.Wr, self.bias = rng.standard_normal((E, H)).astype(np.float32), rng.standard_normal(E).astype(np.float32)
        self.gate = G.Gate(self.Wr, self.bias, k, ng, tg, hidden_type=ht)
        self.gate_args = (k, ng, tg)
        self.full = G.Moe(E, k, H, I, *(t.clone() for t in full), gt, ut, dt, ht, max_tokens=tmax)
        self.full_mlp = G.Mlp(H, I, *(t.clone() for t in sgs), Q4_K, Q4_K, Q6_K, ht) if shared else None
        El = E // world
        self.shards, self.mlps = [], []
        for r in range(world):
            sl = [t.view(E, -1)[r * El:(r + 1) * El].reshape(-1).clone() for t in full]
            self.shards.append(G.Moe(El, k, H, I, *sl, gt, ut, dt, ht, max_tokens=tmax, offset=r * El))
            self.mlps.append(G.Mlp(H, I, *(t.clone() for t in sgs), Q4_K, Q4_K, Q6_K, ht) if shared else None)
        self.lay = exchange_layout(world, H, ht, k, tmax)
        self.buf = [torch.full((self.lay["bytes"],), 0xFF, dtype=torch.uint8, device="cuda") for _ in range(world)]
        o_tok, off = self.lay["tokens"], self.lay["token_regions"]
        for b in self.buf:        # flag words start zeroed
            b[self.lay["flags"]:self.lay["tokens"]].zero_()
            b[o_tok + off["flags"]:].zero_()
        base = [b.data_ptr() for b in self.buf]
        self.comms = [native.EpTokensComm.make(r, world, tmax, H, ht, k, [p + o_tok for p in base]) for r in range(world)]
        self.block_comms = [native.EpComm.make(r, world, H, ht, base, [p + self.lay["partial"] for p in base],
                                               [p + self.lay["flags"] for p in base]) for r in range(world)]
        self.hb = {F32: 4, F16: 2, BF16: 2}[ht]

    def region(self, r, name, dtype, shape):
        o = self.lay["tokens"] + self.lay["token_regions"][name]
        n = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
        return self.buf[r][o:o + n].view(dtype).view(*shape)

    def status(self, r):
        return int(self.region(r, "flags", torch.int32, (2 * self.world + 5,))[2 * self.world + 2])

    def tokens(self, counts, rng):
        G = self.G
        xs = []
        for c in counts:
            x = (rng.standard_normal((c, self.H)) / 10).astype(np.float32)
            xs.append(G.dev(x).to(G.TORCH_HID[self.ht]))
        return xs

    def run(self, counts, xs, masks=None, check_launches=False):
        lib, G = native.lib(), self.G
        cnt = (C.c_int * self.world)(*counts)
        ys = [torch.zeros_like(x) for x in xs]
        idx = [torch.zeros((c, self.k), dtype=torch.int64, device="cuda") for c in counts]
        w = [torch.zeros((c, self.k), dtype=torch.float32, device="cuda") for c in counts]
        masks = masks or ((7,) if self.world == 1 else (1, 2, 4))
        launches = {}
        for mask in masks:
            for r in range(self.world):
                n0 = native.launch_count()
                native.check(lib.ktb200_moe_ep_forward_tokens(C.byref(self.gate.cfg), self.shards[r].h, self.mlps[r].h if self.mlps[r] else None,
                                                              C.byref(self.comms[r]), cnt, xs[r].data_ptr(), ys[r].data_ptr(), idx[r].data_ptr(),
                                                              w[r].data_ptr(), mask, G.stream()))
                launches[(mask, r)] = native.launch_count() - n0
        torch.cuda.synchronize()
        return ys, idx, w, launches

    def reference(self, x):
        """gate, then ktb200_moe_forward over all experts and ktb200_mlp_forward added as a second rounded term"""
        lib, G = native.lib(), self.G
        T = x.shape[0]
        idx = torch.zeros((T, self.k), dtype=torch.int64, device="cuda")
        w = torch.zeros((T, self.k), dtype=torch.float32, device="cuda")
        y = torch.zeros_like(x)
        if T:
            native.check(lib.ktb200_moe_gate_forward(C.byref(self.gate.cfg), T, x.data_ptr(), idx.data_ptr(), w.data_ptr(), None, None, G.stream()))
            native.check(lib.ktb200_moe_forward(self.full.h, T, self.k, idx.data_ptr(), w.data_ptr(), x.data_ptr(), y.data_ptr(), None, G.stream()))
            if self.full_mlp is not None:
                _mlp_accumulate(self.full_mlp.h, 64, x, y)
        torch.cuda.synchronize()
        return y, idx, w

    def check(self, counts, xs, ys, idx, w):
        El = self.E // self.world
        total = sum(counts)
        prefix = np.concatenate([[0], np.cumsum(counts)]).astype(int)
        all_ids = [i.cpu().numpy() for i in idx]
        for r in range(self.world):
            assert self.status(r) == 0, "a peer wait timed out"
            want, widx, ww = self.reference(xs[r])
            assert torch.equal(idx[r], widx) and torch.equal(w[r], ww)
            got = _bits(ys[r])
            if self.world == 1:
                assert np.array_equal(got, _bits(want))
            elif counts[r]:
                _assert_close(got, _bits(want), self.ht)
                if self.full_mlp is None:
                    assert np.array_equal(got, self.rank_order_sum(r, counts[r], all_ids[r]))
        # buffer discipline: rows nobody needed keep their NaN bytes; every needed row was written
        row_b = self.H * self.hb
        for d in range(self.world):
            x_rows = self.region(d, "x", torch.uint8, (self.world * self.tmax, row_b))
            part = self.region(d, "partial", torch.int32, (self.world, self.tmax, self.H))
            for s in range(self.world):
                for i in range(counts[s]):
                    owners = {int(e) // El for e in all_ids[s][i] if 0 <= e < self.E}
                    untouched = bool((x_rows[prefix[s] + i] == 0xFF).all())
                    assert untouched == (d not in owners), (d, s, i)
            assert bool((x_rows[total:] == 0xFF).all())
            for s in range(self.world):
                for i in range(self.tmax):
                    owners = {int(e) // El for e in all_ids[d][i] if 0 <= e < self.E} if i < counts[d] else set()
                    untouched = bool((part[s, i] == -1).all())
                    assert untouched == (s not in owners), (d, s, i)

    def rank_order_sum(self, d, T, ids):
        """rank d's output recomputed from the partial rows its owners delivered: fp32 sum in rank order, one rounding"""
        El = self.E // self.world
        part = self.region(d, "partial", torch.float32, (self.world, self.tmax, self.H)).cpu().numpy()
        acc = np.zeros((T, self.H), np.float32)
        for i in range(T):
            owners = {int(e) // El for e in ids[i] if 0 <= e < self.E}
            for r in range(self.world):
                if r in owners:
                    acc[i] += part[r, i]
        if self.ht == BF16:
            u = acc.view(np.uint32).astype(np.uint64)
            return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
        return acc.astype(np.float16) if self.ht == F16 else acc

    def close(self):
        for h in self.shards + [self.full] + [m for m in self.mlps + [self.full_mlp] if m is not None]:
            h.close()


# ------------------------------------------------------------------------------------------------ GPU: C-ABI loopback
CASES = [
    # world, counts, hidden type, shared expert
    (1, [5], BF16, True),
    (1, [64], BF16, True),              # grouped tensor-core path, the same kernels as the single-GPU call
    (1, [0], BF16, True),
    (2, [0, 1], BF16, True),
    (2, [47, 48], F16, False),
    (2, [20, 27], BF16, True),          # 47 gathered rows: per-pair kernels, while ...
    (2, [20, 28], F32, True),           # ... 48 gathered rows take the grouped GEMM
    (4, [1, 0, 47, 48], BF16, True),
    (8, [9, 30, 0, 17, 1, 5, 3, 2], BF16, False),   # no shared term, up to 4 owners a token: pinned bit for bit to the rank-order sum
    (8, [3, 0, 1, 5, 2, 0, 7, 4], F32, True),
    (8, [0, 0, 0, 0, 0, 0, 0, 0], BF16, False),
]


@pytest.mark.gpu
@pytest.mark.parametrize("world,counts,ht,shared", CASES)
def test_ep_tokens_loopback_matches_single_gpu(world, counts, ht, shared):
    lb = _Loopback(world, 32, 4, 2048, 512, ht, 64, shared=shared, seed=10 * world + sum(counts))
    rng = np.random.default_rng(len(counts) + sum(counts))
    xs = lb.tokens(counts, rng)
    ys, idx, w, launches = lb.run(counts, xs)
    lb.check(counts, xs, ys, idx, w)
    total = sum(counts)
    if world > 1:
        for r in range(world):
            assert launches[(1, r)] == (1 if counts[r] else 0) + 1       # gate (none for 0 tokens) + send
            expert = launches[(2, r)] - 2                                 # minus wait + deliver
            assert expert == (0 if total == 0 else 2) if total < 48 else expert >= 10, expert   # per-pair gate/up + down | grouped
            assert launches[(4, r)] == (2 * -(-counts[r] // 64) if shared else 0) + 1      # shared-expert MLP chunks + combine
    lb.close()


@pytest.mark.gpu
def test_ep_tokens_v3_shapes_tmax_1024():
    """E 256, H 7168, I 2048, k 8, n_group 8, topk_group 4 at world 8: 1923 gathered rows (chunked by group_max_len 1024)"""
    counts = [1024, 3, 0, 200, 48, 47, 1, 600]
    lb = _Loopback(8, 256, 8, 7168, 2048, BF16, 1024, shared=True, seed=3, ng=8, tg=4)
    xs = lb.tokens(counts, np.random.default_rng(5))
    ys, idx, w, _ = lb.run(counts, xs)
    lb.check(counts, xs, ys, idx, w)
    lb.close()


def _iq1s_blocks(t, n, seed):
    if t == IQ1_S:
        import iq_oracle as oq
        return torch.from_numpy(oq.random_blocks(IQ1_S, n // 256, np.random.default_rng(seed), 1 / 64).reshape(-1)).cuda()
    from ktransformers_b200.util.synth import synth_blocks
    return synth_blocks(t, n, "cuda", seed)


@pytest.mark.gpu
@pytest.mark.parametrize("world,counts", [(1, [9]), (2, [9, 40])])
def test_ep_tokens_iq1s_experts(world, counts):
    """the shard runs its ordinary kernels, so formats the one-token kernel refuses work here"""
    lb = _Loopback(world, 16, 4, 2048, 512, BF16, 64, types=(IQ1_S, IQ1_S, IQ1_S), shared=True, seed=77, make=_iq1s_blocks)
    xs = lb.tokens(counts, np.random.default_rng(9))
    ys, idx, w, _ = lb.run(counts, xs)
    lb.check(counts, xs, ys, idx, w)
    lb.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
def test_ep_tokens_back_to_back_layers_interleaved_with_one_token_block(world):
    """3 layers reuse the regions without extra barriers; between them the one-launch decode kernel runs on the same
    allocations (its own message / partial / flag words), and neither disturbs the other."""
    import gpu_util as G
    from test_gpu_parity import assert_bf16_close
    lb = _Loopback(world, 32, 4, 4096, 512, BF16, 32, shared=True, seed=200 + world)
    lib = native.lib()
    rng = np.random.default_rng(world)
    for layer in range(3):
        for r in range(world):          # fresh sentinels: rows written by the previous layer stay written
            o = lb.lay["tokens"]
            lb.buf[r][o:o + lb.lay["token_regions"]["scratch"]].fill_(0xFF)
        counts = [int(c) for c in rng.integers(0, 32, world)]
        xs = lb.tokens(counts, rng)
        ys, idx, w, _ = lb.run(counts, xs)
        lb.check(counts, xs, ys, idx, w)
        x1 = lb.tokens([1] * world, rng)
        y1 = [torch.zeros_like(x) for x in x1]
        i1 = [torch.zeros((1, lb.k), dtype=torch.int64, device="cuda") for _ in range(world)]
        w1 = [torch.zeros((1, lb.k), dtype=torch.float32, device="cuda") for _ in range(world)]
        for mask in (1, 2, 4):
            for r in range(world):
                native.check(lib.ktb200_moe_ep_block_forward(C.byref(lb.gate.cfg), lb.shards[r].h, lb.mlps[r].h, C.byref(lb.block_comms[r]),
                                                             x1[r].data_ptr(), y1[r].data_ptr(), i1[r].data_ptr(), w1[r].data_ptr(), mask, G.stream()))
        torch.cuda.synchronize()
        for r in range(world):
            want, _, _ = lb.reference(x1[r])
            assert_bf16_close(_bits(y1[r]), _bits(want), min_exact=0.9, ulps=2)
            assert int(lb.buf[r][lb.lay["flags"]:lb.lay["tokens"]].view(torch.int32)[2 * world + 1]) == 0
    lb.close()


# ------------------------------------------------------------------------------------------------ GPU: operator
@pytest.mark.gpu
def test_sharded_v3_moe_blocks_match_unsharded_prompt_chunk(tmp_path):
    """N KDeepseekV3MoE blocks with sharded KExpertsB200 experts, driven phase by phase through ep_tokens_forward, give the
    unsharded block's output on the same prompt chunk; without an exchange a sharded block raises."""
    from test_gpu_operators import _write_gguf, H, I, E, K
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Config, DeepseekV3MoEOnlyForCausalLM
    from ktransformers_b200.operators.experts import KExpertsB200
    from ktransformers_b200.optimize.optimize import optimize_and_load_gguf
    import ktransformers_b200.optimize.optimize as opt
    _write_gguf(str(tmp_path / "tiny.gguf"))
    rule = os.path.join(os.path.dirname(opt.__file__), "optimize_rules", "DeepSeek-V3-Chat-b200.yaml")
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        cfg = DeepseekV3Config(hidden_size=H, intermediate_size=I, moe_intermediate_size=I, n_routed_experts=E, n_shared_experts=1,
                               num_experts_per_tok=K, n_group=2, topk_group=1, num_hidden_layers=2, first_k_dense_replace=1)
        with torch.device("meta"):
            model = DeepseekV3MoEOnlyForCausalLM(cfg)
        optimize_and_load_gguf(model, rule, str(tmp_path), cfg, default_device="cuda")
        moe = model.model.layers[1].mlp
        gen = moe.experts.generate_experts
        world, tmax = 2, 64
        lay_b, off = native.ep_tokens_layout(world, tmax, H, BF16, K)
        bufs = [torch.zeros(lay_b, dtype=torch.uint8, device="cuda") for _ in range(world)]
        blocks = []
        for r in range(world):
            # a copy of the block whose wrapped module has its own experts (attributes resolve on orig_module)
            b = copy.copy(moe)
            b._modules = dict(moe._modules)
            orig = copy.copy(moe.orig_module)
            orig._modules = dict(moe.orig_module._modules)
            ex = copy.copy(moe.experts)
            ex.generate_experts = KExpertsB200(gen.key, gen.gguf_loader, gen.config, E, device="cuda", expert_parallel_rank=r,
                                               expert_parallel_size=world, hidden_dtype=torch.bfloat16)
            ex.generate_experts.load()
            orig._modules["experts"] = ex
            b.orig_module = orig
            assert b.experts.generate_experts.ep_size == world and moe.experts.generate_experts.ep_size == 1
            blocks.append(b)
        x = (torch.randn(1, 12, H, device="cuda") / 10).to(torch.bfloat16)
        with pytest.raises(RuntimeError, match="no expert-parallel exchange"):
            blocks[0](x)
        counts = [12, 5]
        xs = [x, (torch.randn(1, 5, H, device="cuda") / 10).to(torch.bfloat16)]
        cnt = (C.c_int * world)(*counts)
        for r, b in enumerate(blocks):
            b.ep_exchange = types.SimpleNamespace(
                tok_comm=native.EpTokensComm.make(r, world, tmax, H, BF16, K, [t.data_ptr() for t in bufs]),
                take_step_counts=lambda n, r=r: cnt if cnt[r] == n else None)
        from test_gpu_parity import assert_bf16_close
        lib = native.lib()
        wants = []
        for r in range(world):
            # the unsharded block's two rounded terms: routed experts over all E, then the shared expert's MLP handle
            xr = xs[r].reshape(-1, H).contiguous()
            ridx, rwt = moe.gate(xs[r])
            ridx, rwt = ridx.reshape(-1, K).contiguous(), rwt.reshape(-1, K).float().contiguous()
            want = torch.zeros_like(xr)
            native.check(lib.ktb200_moe_forward(gen.handle, xr.shape[0], K, ridx.data_ptr(), rwt.data_ptr(), xr.data_ptr(), want.data_ptr(),
                                                None, torch.cuda.current_stream().cuda_stream))
            _mlp_accumulate(moe._ktb_mlp, moe.BLOCK_MAX_TOKENS, xr, want)
            torch.cuda.synchronize()
            wants.append((want, ridx, rwt))

        def check(ys):
            for r in range(world):
                want, ridx, rwt = wants[r]
                idx, wt = blocks[r].last_topk
                assert torch.equal(idx, ridx) and torch.equal(wt, rwt)
                assert_bf16_close(_bits(ys[r].reshape(-1, H)), _bits(want), min_exact=0.9, ulps=2)
                assert int(bufs[r][off["flags"]:].view(torch.int32)[2 * world + 2]) == 0

        n0 = native.launch_count()
        for mask in (1, 2):
            for r, b in enumerate(blocks):
                assert b.ep_tokens_forward(xs[r], mask) is None
        ys = [b.ep_tokens_forward(xs[r], 4) for r, b in enumerate(blocks)]
        torch.cuda.synchronize()
        assert native.launch_count() - n0 == world * (2 + 4) + sum(2 * -(-c // 8) + 1 for c in counts)
        check(ys)

        # KDeepseekV3MoEV2.forward with a bsz_tensor on the same sharded blocks: it takes the expert-parallel path and computes
        # every row (the padding rows beyond bsz too, as documented); its phases are driven through ep_tokens_forward
        from ktransformers_b200.operators.experts import KDeepseekV3MoEV2
        bsz = torch.tensor([3], dtype=torch.int32, device="cuda")
        for b in blocks:
            b.__class__ = KDeepseekV3MoEV2
        for mask in (1, 2, 4):
            for b in blocks:
                b.ep_tokens_forward = functools.partial(KDeepseekV3MoEV2.ep_tokens_forward, b, phase_mask=mask)
            ys = [b(xs[r], bsz) for r, b in enumerate(blocks)]
        torch.cuda.synchronize()
        check(ys)
    finally:
        torch.set_default_dtype(old)
