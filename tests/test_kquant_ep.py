"""Expert-parallel decode for Q2_K and Q3_K routed experts: ktb200_moe_ep_block_forward's moe_ep_block_kernel<GU, D>
(csrc/moe_block.cu) for gate/up GU in {Q2_K, Q3_K} and down D in {Q2_K, Q3_K, Q4_K, Q6_K}, the expert tensors of llama.cpp's
Q2_K, Q3_K_S and Q3_K_M DeepSeek files, and attach_expert_parallel's table of accepted sets.

GPU, one H100, loopback as in tests/test_ep_tokens.py: `world` shard handles with their own buffers in one device's memory, the
phases run rank by rank.  Every rank's output must be bit-identical to ktb200_moe_ep_forward_tokens on the same shards with one
token per rank (same per-pair arithmetic, same fp32 cross-rank sum in rank order, same shared-expert term) and close to the
unsharded layer (gate, ktb200_moe_forward over all experts, ktb200_mlp_forward as a second rounded term)."""
import ctypes as C
import functools
import types

import numpy as np
import pytest
import torch

from ktransformers_b200 import native

Q2K, Q3K, Q4K, Q5K, Q6K = native.GGML_Q2_K, native.GGML_Q3_K, native.GGML_Q4_K, native.GGML_Q5_K, native.GGML_Q6_K
F32, F16, BF16 = native.GGML_F32, native.GGML_F16, native.GGML_BF16
IQ1, IQ2, IQ1M = native.GGML_IQ1_S, native.GGML_IQ2_XXS, native.GGML_IQ1_M

NEW_SETS = [(gu, gu, d) for gu in (Q2K, Q3K) for d in (Q2K, Q3K, Q4K, Q6K)]
NAME = {Q2K: "q2k", Q3K: "q3k", Q4K: "q4k", Q6K: "q6k"}


def _set_id(t):
    return "_".join(NAME[x] for x in t)


# ------------------------------------------------------------------------------------------------ CPU
def _attach(expert_types, monkeypatch):
    """attach_expert_parallel on a one-block model whose experts have `expert_types`; the exchange itself is stubbed out"""
    from ktransformers_b200.operators import expert_parallel as ep

    class Block(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self._block_handles = None
            self.key = "blk.3"
            self.experts = types.SimpleNamespace(generate_experts=types.SimpleNamespace(
                gate_type=expert_types[0], up_type=expert_types[1], down_type=expert_types[2]))

    monkeypatch.setattr(ep.dist, "get_world_size", lambda group=None: 1)
    monkeypatch.setattr(ep, "PeerExchange", lambda *a, **kw: "exchange")
    model = torch.nn.Sequential(Block())
    assert ep.attach_expert_parallel(model, 512, BF16, "cpu") == "exchange"
    return model[0].ep_exchange


@pytest.mark.parametrize("expert_types", NEW_SETS + [(Q4K, Q4K, Q4K), (Q4K, Q4K, Q6K)], ids=_set_id)
def test_attach_expert_parallel_accepts(expert_types, monkeypatch):
    assert _attach(expert_types, monkeypatch) == "exchange"


@pytest.mark.parametrize("expert_types", [(Q2K, Q3K, Q3K), (Q3K, Q2K, Q4K), (Q3K, Q3K, Q5K), (Q4K, Q4K, Q2K), (Q4K, Q4K, Q3K),
                                          (Q2K, Q2K, IQ1), (Q5K, Q5K, Q6K), (IQ1, IQ1, IQ2), (Q4K, Q4K, IQ1), (IQ1M, IQ1M, IQ2),
                                          (Q4K, Q4K, IQ1M), (native.RAWINT4_G32,) * 3])
def test_attach_expert_parallel_refuses(expert_types, monkeypatch):
    with pytest.raises(ValueError, match="expert-parallel"):
        _attach(expert_types, monkeypatch)


def test_accepted_sets_table():
    from ktransformers_b200.util.custom_gguf import B200_EP_TYPE_SETS
    names = {Q2K: "Q2_K", Q3K: "Q3_K", Q4K: "Q4_K", Q6K: "Q6_K"}
    assert B200_EP_TYPE_SETS == {("Q4_K", "Q4_K"), ("Q4_K", "Q6_K")} | {(names[g], names[d]) for g, _, d in NEW_SETS}


# ------------------------------------------------------------------------------------------------ GPU helpers
def _bits(t):
    return t.view(torch.int16).cpu().numpy().view(np.uint16) if t.dtype == torch.bfloat16 else t.cpu().numpy()


def _loopback(world, E, k, H, I, ht, types_, shared, seed, ng=4, tg=2, use_silu=1, hot=None):
    """test_ep_tokens._Loopback with the shared expert of types `shared` (None: none) and routed experts of `types_`.
    hot: an expert id whose router bias is raised so that every rank's token picks it (a crowded expert)."""
    import gpu_util as G
    from test_ep_tokens import _Loopback
    orig = G.Moe
    G.Moe = functools.partial(orig, use_silu=use_silu)
    try:
        lb = _Loopback(world, E, k, H, I, ht, max(world, 8), types=types_, shared=False, seed=seed, ng=ng, tg=tg)
    finally:
        G.Moe = orig
    if hot is not None:
        lb.bias[hot] += 100.0
        lb.gate = G.Gate(lb.Wr, lb.bias, k, ng, tg, hidden_type=ht)
    if shared is not None:
        from ktransformers_b200.util.synth import synth_blocks
        sgs = [synth_blocks(t, I * H, "cuda", seed + 40 + i) for i, t in enumerate(shared)]
        lb.full_mlp = G.Mlp(H, I, *(t.clone() for t in sgs), *shared, ht)
        lb.mlps = [G.Mlp(H, I, *(t.clone() for t in sgs), *shared, ht) for _ in range(world)]
    return lb


def _run_block(lb, xs):
    """one token per rank through ktb200_moe_ep_block_forward: phase 7 at world 1, else 1, 2, 4 rank by rank"""
    import gpu_util as G
    lib = native.lib()
    ys = [torch.zeros_like(x) for x in xs]
    idx = [torch.zeros((1, lb.k), dtype=torch.int64, device="cuda") for _ in xs]
    w = [torch.zeros((1, lb.k), dtype=torch.float32, device="cuda") for _ in xs]
    for mask in ((7,) if lb.world == 1 else (1, 2, 4)):
        for r in range(lb.world):
            native.check(lib.ktb200_moe_ep_block_forward(C.byref(lb.gate.cfg), lb.shards[r].h, lb.mlps[r].h if lb.mlps[r] else None,
                                                         C.byref(lb.block_comms[r]), xs[r].data_ptr(), ys[r].data_ptr(),
                                                         idx[r].data_ptr(), w[r].data_ptr(), mask, G.stream()))
    torch.cuda.synchronize()
    return ys, idx, w


def _block_status(lb, r):
    return int(lb.buf[r][lb.lay["flags"]:lb.lay["tokens"]].view(torch.int32)[2 * lb.world + 1])


def _close(got, want, ht):
    from test_gpu_parity import assert_bf16_close
    from test_ep_tokens import _assert_close
    if ht == BF16:
        assert_bf16_close(got, want, min_exact=0.9, ulps=2)
    else:
        _assert_close(got, want, ht)


def _check_against_tokens_and_unsharded(lb, xs):
    """the one-launch layer == ep_forward_tokens with counts [1] * world, bit for bit; both close to the unsharded layer"""
    ys, idx, w = _run_block(lb, xs)
    yt, it, wt, _ = lb.run([1] * lb.world, xs)
    for r in range(lb.world):
        assert _block_status(lb, r) == 0 and lb.status(r) == 0, "a peer wait timed out"
        assert torch.equal(idx[r], it[r]) and torch.equal(w[r], wt[r])
        assert np.array_equal(_bits(ys[r]), _bits(yt[r])), (r, float((ys[r].float() - yt[r].float()).abs().max()))
        want, widx, ww = lb.reference(xs[r])
        assert torch.equal(idx[r], widx) and torch.equal(w[r], ww)
        _close(_bits(ys[r]), _bits(want), lb.ht)
    return ys, idx


# ------------------------------------------------------------------------------------------------ GPU
SHARED = {"none": None, "q4k_q6k": (Q4K, Q4K, Q6K), "routed": "routed"}


@pytest.mark.gpu
@pytest.mark.parametrize("shared", list(SHARED))
@pytest.mark.parametrize("world", [1, 2, 4, 8])
@pytest.mark.parametrize("types_", NEW_SETS, ids=_set_id)
def test_ep_block_kquant_loopback(types_, world, shared):
    """H 4096 (16 blocks a row, a multiple of 4), I 512, E 32, k 4.  Expert 5 is raised in the router so that every token picks
    it (a crowded expert: world pairs on one expert of one shard); at world > 1 most ids lie outside any given shard."""
    sh = types_ if SHARED[shared] == "routed" else SHARED[shared]
    lb = _loopback(world, 32, 4, 4096, 512, BF16, types_, sh, seed=7 * world + types_[0] + types_[2], hot=5)
    rng = np.random.default_rng(world * 31 + types_[2])
    for _ in range(2):   # the second layer reuses the buffers (epochs advance)
        xs = lb.tokens([1] * world, rng)
        _, idx = _check_against_tokens_and_unsharded(lb, xs)
        assert all(5 in i[0].tolist() for i in idx)
    lb.close()


@pytest.mark.gpu
@pytest.mark.parametrize("use_silu", [1, 0])
@pytest.mark.parametrize("ht", [BF16, F16, F32])
@pytest.mark.parametrize("types_", [(Q2K, Q2K, Q3K), (Q3K, Q3K, Q4K)], ids=_set_id)
def test_ep_block_kquant_hidden_types_and_activation(types_, ht, use_silu):
    lb = _loopback(2, 32, 4, 4096, 512, ht, types_, (Q4K, Q4K, Q6K), seed=90 + ht, use_silu=use_silu)
    xs = lb.tokens([1, 1], np.random.default_rng(ht + 3 * use_silu))
    _check_against_tokens_and_unsharded(lb, xs)
    lb.close()


@pytest.mark.gpu
@pytest.mark.parametrize("types_", [(Q2K, Q2K, Q3K), (Q3K, Q3K, Q4K)], ids=_set_id)
def test_ep_block_kquant_v3_shapes_world_8(types_):
    """H 7168, I 2048, k 8, 8 groups / top 4, 256 experts in 8 shards of 32, a Q4_K / Q6_K shared expert"""
    lb = _loopback(8, 256, 8, 7168, 2048, BF16, types_, (Q4K, Q4K, Q6K), seed=11, ng=8, tg=4)
    xs = lb.tokens([1] * 8, np.random.default_rng(12))
    _check_against_tokens_and_unsharded(lb, xs)
    lb.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4])
def test_ep_block_kquant_back_to_back_with_ep_tokens_layers(world):
    """3 one-token layers interleaved with multi-token ep_forward_tokens layers on the same allocations"""
    lb = _loopback(world, 32, 4, 4096, 512, BF16, (Q2K, Q2K, Q3K), (Q4K, Q4K, Q6K), seed=300 + world)
    rng = np.random.default_rng(world)
    for layer in range(3):
        for r in range(world):          # fresh sentinels: rows written by the previous layer stay written
            o = lb.lay["tokens"]
            lb.buf[r][o:o + lb.lay["token_regions"]["scratch"]].fill_(0xFF)
        counts = [int(c) for c in rng.integers(0, 8, world)]
        xs = lb.tokens(counts, rng)
        ys, idx, w, _ = lb.run(counts, xs)
        lb.check(counts, xs, ys, idx, w)
        _check_against_tokens_and_unsharded(lb, lb.tokens([1] * world, rng))
    lb.close()


@pytest.mark.gpu
@pytest.mark.parametrize("types_", [(Q2K, Q2K, Q3K), (Q3K, Q3K, Q6K)], ids=_set_id)
def test_ep_block_kquant_cuda_graph_replays_match_eager(types_):
    import gpu_util as G
    lb = _loopback(1, 32, 4, 4096, 512, BF16, types_, (Q4K, Q4K, Q6K), seed=21)
    lib = native.lib()
    xs = lb.tokens([1], np.random.default_rng(22))
    eager, _, _ = _run_block(lb, xs)
    y = torch.zeros_like(xs[0])
    idx = torch.zeros((1, lb.k), dtype=torch.int64, device="cuda")
    w = torch.zeros((1, lb.k), dtype=torch.float32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            native.check(lib.ktb200_moe_ep_block_forward(C.byref(lb.gate.cfg), lb.shards[0].h, lb.mlps[0].h, C.byref(lb.block_comms[0]),
                                                         xs[0].data_ptr(), y.data_ptr(), idx.data_ptr(), w.data_ptr(), 7, G.stream()))
    torch.cuda.current_stream().wait_stream(s)
    for _ in range(8):
        y.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(_bits(y), _bits(eager[0]))
        assert _block_status(lb, 0) == 0
    del g
    lb.close()


@pytest.mark.gpu
def test_ep_block_kquant_launch_census():
    """a one-token step of a Q2_K set is one moe_ep_block_kernel launch plus the shared MLP's, and no ep_tok_* kernel"""
    lb = _loopback(1, 32, 4, 4096, 512, BF16, (Q2K, Q2K, Q3K), (Q4K, Q4K, Q6K), seed=31)
    xs = lb.tokens([1], np.random.default_rng(32))
    _run_block(lb, xs)                        # warm-up: attributes, first launches
    n0 = native.launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        _run_block(lb, xs)
    launches = native.launch_count() - n0
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    kernels = [n for n in names if "ktb::" in n]          # the library's kernels (not the harness's tensor fills)
    assert sum("moe_ep_block_kernel" in n for n in kernels) == 1, kernels
    assert not any("ep_tok_" in n for n in kernels), kernels
    assert len(kernels) == launches, (kernels, launches)
    n0 = native.launch_count()
    lib = native.lib()
    lb.mlps[0] and native.check(lib.ktb200_mlp_forward(lb.mlps[0].h, 1, xs[0].data_ptr(), torch.zeros_like(xs[0]).data_ptr(), 0, None,
                                                       torch.cuda.current_stream().cuda_stream))
    assert launches == 1 + native.launch_count() - n0
    lb.close()


# ------------------------------------------------------------------------------------------------ GPU: operator
def _write_q2k_gguf(path, E, H, I):
    """a two-layer DeepSeek GGUF: a dense Q4_K / Q6_K MLP in layer 0; in layer 1 Q2_K / Q2_K / Q3_K routed experts (llama.cpp's
    Q2_K file) and a Q4_K / Q4_K / Q6_K shared expert"""
    import gguf
    from ktransformers_b200.util.synth import synth_blocks
    rng = np.random.default_rng(17)
    w = gguf.GGUFWriter(path, "deepseek2")
    seed = [300]

    def add_q(name, shape, qt):
        seed[0] += 1
        q = synth_blocks(int(qt), int(np.prod(shape)), "cpu", seed[0]).numpy()
        w.add_tensor(name, q.reshape(*shape[:-1], -1), raw_dtype=qt)

    T = gguf.GGMLQuantizationType
    for n in ("gate", "up"):
        add_q(f"blk.0.ffn_{n}.weight", (I, H), T.Q4_K)
        add_q(f"blk.1.ffn_{n}_exps.weight", (E, I, H), T.Q2_K)
        add_q(f"blk.1.ffn_{n}_shexp.weight", (I, H), T.Q4_K)
    add_q("blk.0.ffn_down.weight", (H, I), T.Q6_K)
    add_q("blk.1.ffn_down_exps.weight", (E, H, I), T.Q3_K)
    add_q("blk.1.ffn_down_shexp.weight", (H, I), T.Q6_K)
    w.add_tensor("blk.1.ffn_gate_inp.weight", rng.standard_normal((E, H)).astype(np.float32))
    w.add_tensor("blk.1.exp_probs_b.bias", rng.standard_normal((E,)).astype(np.float32))
    w.write_header_to_file(); w.write_kv_data_to_file(); w.write_tensors_to_file(); w.close()


class _LoopbackExchange:
    """One rank's stand-in for PeerExchange in a one-GPU loopback: the same comm / tok_comm / step-count interface over
    buffers laid out by exchange_layout (regions of every rank in one device's memory)."""

    def __init__(self, rank, world, bufs, lay, H, K, tmax):
        base = [b.data_ptr() for b in bufs]
        self.comm = native.EpComm.make(rank, world, H, BF16, base, [p + lay["partial"] for p in base], [p + lay["flags"] for p in base])
        self.tok_comm = native.EpTokensComm.make(rank, world, tmax, H, BF16, K, [p + lay["tokens"] for p in base])
        self.rank, self.counts = rank, None

    def begin_step(self, counts):          # the host counts every rank announced for this step (a gloo all-gather in PeerExchange)
        self.counts = (C.c_int * len(counts))(*counts)

    def take_step_counts(self, n_tokens):
        c, self.counts = self.counts, None
        assert c is None or c[self.rank] == n_tokens
        return c


class _DeferredBlockCalls:
    """`native` as the operator module sees it, except that ktb200_moe_ep_block_forward (which the operator issues with
    phase mask 7) is recorded: the test replays every rank's recorded call as phases 1, 2 and 4, rank by rank, the legal
    one-GPU schedule of N concurrent ranks."""

    def __init__(self, real):
        self._real, self.calls = real, []
        outer = self

        class _Lib:
            def __getattr__(self, name):
                return getattr(real.lib(), name)

            def ktb200_moe_ep_block_forward(self, *args):
                assert args[-2] == 7
                outer.calls.append(args)
                return 0
        self._lib = _Lib()

    def lib(self):
        return self._lib

    def __getattr__(self, name):
        return getattr(self._real, name)

    def replay(self):
        for mask in (1, 2, 4):
            for a in self.calls:
                native.check(native.lib().ktb200_moe_ep_block_forward(*a[:-2], mask, a[-1]))
        self.calls = []


@pytest.mark.gpu
def test_sharded_q2k_moe_blocks_through_attach_expert_parallel(tmp_path, monkeypatch):
    """N = 2 KDeepseekV3MoE blocks whose Q2_K / Q2_K / Q3_K experts are sharded (KExpertsB200 expert_parallel_rank / size),
    each given its exchange by attach_expert_parallel.  One-token steps go through KDeepseekV3MoE.forward, which issues the
    one-launch kernel with the block's shared-expert MLP handle; one multi-token step (begin_step) goes through the
    multi-token layer.  Every rank's output matches the unsharded block: its routed experts over all E, then the shared
    expert's MLP as a second rounded term."""
    import copy
    from test_gpu_parity import assert_bf16_close
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Config, DeepseekV3MoEOnlyForCausalLM
    from ktransformers_b200.operators import experts as experts_mod
    from ktransformers_b200.operators import expert_parallel as ep
    from ktransformers_b200.operators.experts import KExpertsB200
    from ktransformers_b200.optimize.optimize import optimize_and_load_gguf
    import ktransformers_b200.optimize.optimize as opt
    import os
    E, H, I, K, world, tmax = 8, 4096, 512, 4, 2, 16
    _write_q2k_gguf(str(tmp_path / "q2k.gguf"), E, H, I)
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
        assert (gen.gate_type, gen.up_type, gen.down_type) == (Q2K, Q2K, Q3K)
        lay = ep.exchange_layout(world, H, BF16, K, tmax)
        bufs = [torch.zeros(lay["bytes"], dtype=torch.uint8, device="cuda") for _ in range(world)]
        blocks = []
        for r in range(world):
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
            # attach_expert_parallel checks the expert types and hands the block its exchange (a loopback one here)
            monkeypatch.setattr(ep.dist, "get_world_size", lambda group=None: world)
            monkeypatch.setattr(ep, "PeerExchange", lambda *a, r=r, **kw: _LoopbackExchange(r, world, bufs, lay, H, K, tmax))
            assert isinstance(ep.attach_expert_parallel(torch.nn.Sequential(b), H, BF16, "cuda"), _LoopbackExchange)
            blocks.append(b)
        lib = native.lib()

        def unsharded(x):
            xr = x.reshape(-1, H).contiguous()
            ridx, rwt = moe.gate(x)
            ridx, rwt = ridx.reshape(-1, K).contiguous(), rwt.reshape(-1, K).float().contiguous()
            want = torch.zeros_like(xr)
            native.check(lib.ktb200_moe_forward(gen.handle, xr.shape[0], K, ridx.data_ptr(), rwt.data_ptr(), xr.data_ptr(), want.data_ptr(),
                                                None, torch.cuda.current_stream().cuda_stream))
            from test_ep_tokens import _mlp_accumulate
            _mlp_accumulate(moe._ktb_mlp, moe.BLOCK_MAX_TOKENS, xr, want)
            torch.cuda.synchronize()
            return want, ridx, rwt

        def check(xs, ys):
            for r in range(world):
                want, ridx, rwt = unsharded(xs[r])
                idx, wt = blocks[r].last_topk
                assert torch.equal(idx, ridx) and torch.equal(wt, rwt)
                assert_bf16_close(_bits(ys[r].reshape(-1, H)), _bits(want), min_exact=0.9, ulps=2)
                assert int(bufs[r][lay["flags"]:lay["tokens"]].view(torch.int32)[2 * world + 1]) == 0
                assert int(bufs[r][lay["tokens"] + lay["token_regions"]["flags"]:].view(torch.int32)[2 * world + 2]) == 0

        deferred = _DeferredBlockCalls(native)
        for step in range(3):                     # one-token decode steps through KDeepseekV3MoE.forward
            xs = [(torch.randn(1, 1, H, device="cuda") / 10).to(torch.bfloat16) for _ in range(world)]
            with monkeypatch.context() as m:
                m.setattr(experts_mod, "native", deferred)
                ys = [b(xs[r]) for r, b in enumerate(blocks)]
            assert len(deferred.calls) == world and all(a[2] == blocks[r]._ktb_mlp for r, a in enumerate(deferred.calls))
            deferred.replay()
            torch.cuda.synchronize()
            check(xs, ys)

        counts = [5, 3]                           # one multi-token step: begin_step, then the phases rank by rank
        xs = [(torch.randn(1, c, H, device="cuda") / 10).to(torch.bfloat16) for c in counts]
        for b in blocks:
            b.ep_exchange.begin_step(counts)
        for mask in (1, 2):
            for r, b in enumerate(blocks):
                assert b.ep_tokens_forward(xs[r], mask) is None
        ys = [b.ep_tokens_forward(xs[r], 4) for r, b in enumerate(blocks)]
        torch.cuda.synchronize()
        check(xs, ys)
    finally:
        torch.set_default_dtype(old)


# ------------------------------------------------------------------------------------------------ GPU: real peer memory
@pytest.mark.gpu
@pytest.mark.parametrize("types_", [(Q2K, Q2K, Q3K), (Q3K, Q3K, Q4K)], ids=_set_id)
@pytest.mark.parametrize("world", [2, 4, 8])
def test_ep_block_kquant_on_peer_memory(world, types_):
    """tests/ep_kquant_worker.py under torchrun: one process per GPU, the one-launch kernel on real peer memory"""
    import os
    import subprocess
    import sys
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(29600 + world + 10 * types_[2]), os.path.join(root, "tests", "ep_kquant_worker.py"),
           ",".join(str(t) for t in types_)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("EP block OK") == world, r.stdout[-3000:]
