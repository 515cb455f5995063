"""Causal MLA prefill: ktb200_mla_prefill (csrc/mla_prefill.cu) and the q_len > 1 path of KDeepseekV2Attention.

CPU: the float64 oracle in tests/mla_prefill_oracle.py against DeepseekV3Attention.forward and, at q_len == 1, against the
absorbed decode oracle (oracle/mla_oracle.py, pinned to the reference's attention_ref_torch); argument checks of the C-ABI.
GPU: the kernel against the oracle over lengths that are not tile multiples, causality and padding, the operator against
the plain module through prefill (one chunk and three chunks) and the decode steps after it, no device-to-host
synchronisation, and which kernels ran."""
import ctypes as C

import numpy as np
import pytest
import torch

import mla_prefill_oracle as mpo
from ktransformers_b200 import native

SCALE = (128 + 64) ** -0.5


# ------------------------------------------------------------------------------------------------ oracle pins (CPU)
@pytest.mark.parametrize("past", [0, 5])
@pytest.mark.parametrize("q_len", [1, 4, 9])
def test_oracle_equals_plain_module_attention_core(past, q_len):
    """the oracle reproduces DeepseekV3Attention.forward's attention (everything before o_proj), the module run in float64;
    it forms scores, softmax and P.V in fp32 (`.float()`), hence the fp32 tolerance"""
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Attention, DeepseekV3Config
    torch.manual_seed(past * 10 + q_len)
    cfg = DeepseekV3Config(hidden_size=64, num_attention_heads=3, q_lora_rank=32, num_hidden_layers=1)
    mod = DeepseekV3Attention(cfg).double()
    past_latents = None
    if past:
        x0 = torch.randn(2, past, 64, dtype=torch.float64)
        _, past_latents = mod(x0, torch.arange(past).expand(2, past))
    x = torch.randn(2, q_len, 64, dtype=torch.float64)
    pos = torch.arange(past, past + q_len).expand(2, q_len)
    seen = {}
    hook = mod.o_proj.register_forward_pre_hook(lambda m, a: seen.setdefault("o", a[0].detach().clone()))
    try:
        mod(x, pos, past_latents)
    finally:
        hook.remove()
    q_nope, q_pe, ckv, k_pe = mod.project(x, pos)
    ckv, k_pe = ckv.squeeze(2), k_pe.squeeze(2)
    if past_latents is not None:
        ckv, k_pe = torch.cat([past_latents[0], ckv], 1), torch.cat([past_latents[1], k_pe], 1)
    kv = mod.kv_b_proj(ckv).view(2, ckv.shape[1], 3, 256)
    want = mpo.mla_prefill(q_nope.detach().numpy(), q_pe.detach().numpy(), kv[..., :128].detach().numpy(), k_pe.detach().numpy(),
                           kv[..., 128:].detach().numpy(), mod.softmax_scale)
    got = seen["o"].view(2, q_len, 3, 128).numpy()
    np.testing.assert_allclose(got, want, rtol=0, atol=2e-6 * np.abs(want).max())


@pytest.mark.parametrize("S", [1, 37, 130])
def test_oracle_at_one_query_equals_absorbed_decode_oracle(S):
    """at q_len == 1, attention over decompressed heads == absorbed attention over the latents, then W_UV (mla_decode
    returns float32, hence the tolerance)"""
    from oracle import mla_oracle
    rng = np.random.default_rng(S)
    B, H, page = 2, 4, 64
    W = rng.standard_normal((H * 256, 512)) / 16                 # kv_b_proj weight
    W_UK, W_UV = W.reshape(H, 256, 512)[:, :128], W.reshape(H, 256, 512)[:, 128:]
    ckv, k_pe = rng.standard_normal((B, S, 512)), rng.standard_normal((B, S, 64))
    q_nope, q_pe = rng.standard_normal((B, 1, H, 128)), rng.standard_normal((B, 1, H, 64))
    kv = (ckv @ W.T).reshape(B, S, H, 256)
    want = mpo.mla_prefill(q_nope, q_pe, kv[..., :128], k_pe, kv[..., 128:], SCALE)[:, 0]
    npg = (S + page - 1) // page
    cache = np.zeros((B * npg, page, 576))
    for b in range(B):
        cache[b * npg: (b + 1) * npg].reshape(-1, 576)[:S] = np.concatenate([ckv[b], k_pe[b]], -1)
    table = np.arange(B * npg).reshape(B, npg)
    q_abs = np.einsum("bhd,hdc->bhc", q_nope[:, 0], W_UK)
    lat, _ = mla_oracle.mla_decode(q_abs, q_pe[:, 0], cache, table, np.full(B, S), SCALE, p_bf16=False)
    got = np.einsum("bhc,hdc->bhd", lat.astype(np.float64), W_UV)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-6 * np.abs(want).max())


# ------------------------------------------------------------------------------------------------ C-ABI checks (CPU)
def _valid_params():
    """a well-formed parameter set over fake 16-byte-aligned addresses: every check passes, so each test breaks one thing"""
    base = 1 << 24
    H, q_len, S = 16, 8, 20
    return native.MlaPrefillParams(1, q_len, S, H, 128, 64, 128, SCALE,
                                   base, H * 192, 192, q_len * H * 192,
                                   base + (1 << 20), H * 64, 64, q_len * H * 64,
                                   base + (2 << 20), H * 256, 256, S * H * 256,
                                   base + (2 << 20) + 256, H * 256, 256, S * H * 256,
                                   base + (3 << 20) + 1024, 576, 64 * 576,
                                   base + (4 << 20))


BAD = {
    "q_len 0": (lambda p: setattr(p, "q_len", 0), "q_len"),
    "q_len > kv_len": (lambda p: setattr(p, "q_len", 21), "q_len"),
    "batch 0": (lambda p: setattr(p, "batch", 0), "batch"),
    "heads 0": (lambda p: setattr(p, "num_heads", 0), "num_heads"),
    "nope dim": (lambda p: setattr(p, "qk_nope_head_dim", 64), "head dims"),
    "rope dim": (lambda p: setattr(p, "qk_rope_head_dim", 32), "head dims"),
    "v dim": (lambda p: setattr(p, "v_head_dim", 192), "head dims"),
    "scale 0": (lambda p: setattr(p, "sm_scale", 0.0), "sm_scale"),
    "scale nan": (lambda p: setattr(p, "sm_scale", float("nan")), "sm_scale"),
    "null q_nope": (lambda p: setattr(p, "q_nope", None), "null"),
    "null q_pe": (lambda p: setattr(p, "q_pe", None), "null"),
    "null k_nope": (lambda p: setattr(p, "k_nope", None), "null"),
    "null v": (lambda p: setattr(p, "v", None), "null"),
    "null k_pe": (lambda p: setattr(p, "k_pe", None), "null"),
    "null out": (lambda p: setattr(p, "out", None), "null"),
    "q_nope +2 B": (lambda p: setattr(p, "q_nope", p.q_nope + 2), "q_nope must be 16-byte aligned"),
    "v +8 B": (lambda p: setattr(p, "v", p.v + 8), "v must be 16-byte aligned"),
    "k_pe +2 B": (lambda p: setattr(p, "k_pe", p.k_pe + 2), "k_pe must be 16-byte aligned"),
    "out +4 B": (lambda p: setattr(p, "out", p.out + 4), "out must be 16-byte aligned"),
    "q_pe head stride 68": (lambda p: setattr(p, "q_pe_head_stride", 68), "q_pe head stride"),
    "k_pe token stride 577": (lambda p: setattr(p, "k_pe_token_stride", 577), "k_pe token stride"),
    "k_nope batch stride 0": (lambda p: setattr(p, "k_nope_batch_stride", 0), "k_nope batch stride"),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_prefill_argument_checks(case):
    """each malformed call returns KTB200_EINVAL with a message naming the problem, before any device work"""
    lib = native.lib()
    p = _valid_params()
    mutate, msg = BAD[case]
    mutate(p)
    assert lib.ktb200_mla_prefill(C.byref(p), None) == native.EINVAL
    assert msg in lib.ktb200_last_error().decode()


def test_prefill_null_params():
    lib = native.lib()
    assert lib.ktb200_mla_prefill(None, None) == native.EINVAL
    assert "null" in lib.ktb200_last_error().decode()


# ------------------------------------------------------------------------------------------------ kernel (GPU)
class _Case:
    """operands in the layouts the operator passes: q_nope inside a [B, q, H, 192] q_b output, k_nope / v the halves of a
    [B, S, H, 256] kv_b_proj output, k_pe columns 512.. of [B, rows, 576] cache rows.  Every buffer has spare rows past
    q_len / S, filled with `pad` (0 by default)."""

    def __init__(self, B, H, past, q_len, seed, pad=0.0, spare=40):
        g = torch.Generator().manual_seed(seed)
        S = past + q_len
        self.B, self.H, self.past, self.q_len, self.S = B, H, past, q_len, S
        rnd = lambda *shape: torch.randn(*shape, generator=g).to(torch.bfloat16)
        self.q = rnd(B, q_len + spare, H, 192).cuda()
        self.q_pe = rnd(B, q_len + spare, H, 64).cuda()
        self.kv = rnd(B, S + spare, H, 256).cuda()
        self.rows = rnd(B, S + spare, 576).cuda()
        for t in (self.q, self.q_pe, self.kv, self.rows):
            t[:, t.shape[1] - spare:] = pad
        if pad != 0.0 and spare >= 2:     # NaN and Inf both
            for t in (self.q, self.q_pe, self.kv, self.rows):
                t[:, t.shape[1] - spare::2] = float("inf")

    def run(self):
        q_nope, q_pe = self.q[:, : self.q_len, :, :128], self.q_pe[:, : self.q_len]
        k_nope, v, k_pe = self.kv[..., :128], self.kv[..., 128:], self.rows[..., 512:]
        out = torch.full((self.B, self.q_len, self.H, 128), float("nan"), dtype=torch.bfloat16, device="cuda")
        p = native.MlaPrefillParams(self.B, self.q_len, self.S, self.H, 128, 64, 128, SCALE,
                                    q_nope.data_ptr(), q_nope.stride(1), q_nope.stride(2), q_nope.stride(0),
                                    q_pe.data_ptr(), q_pe.stride(1), q_pe.stride(2), q_pe.stride(0),
                                    k_nope.data_ptr(), k_nope.stride(1), k_nope.stride(2), k_nope.stride(0),
                                    v.data_ptr(), v.stride(1), v.stride(2), v.stride(0),
                                    k_pe.data_ptr(), k_pe.stride(1), k_pe.stride(0), out.data_ptr())
        native.check(native.lib().ktb200_mla_prefill(C.byref(p), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        return out

    def oracle(self, p_bf16=False):
        f = lambda t: t.float().cpu().numpy()
        S, q = self.S, self.q_len
        out = np.empty((self.B, q, self.H, 128))
        for h0 in range(0, self.H, 16):     # bounded memory at long lengths
            hs = slice(h0, h0 + 16)
            out[:, :, hs] = mpo.mla_prefill(f(self.q[:, :q, hs, :128]), f(self.q_pe[:, :q, hs]), f(self.kv[:, :S, hs, :128]),
                                            f(self.rows[:, :S, 512:]), f(self.kv[:, :S, hs, 128:]), SCALE, p_bf16)
        return out


GRID = [(0, 2), (0, 64), (0, 129), (0, 1024), (63, 1), (300, 200), (1000, 37), (2100, 300)]   # longer: test_mla_lengths.py


@pytest.mark.gpu
@pytest.mark.parametrize("past,q_len", GRID)
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("H", [16, 128])
def test_prefill_kernel_vs_oracle(H, B, past, q_len):
    """against exact-softmax attention: the bf16 P and bf16 output bound of the decode kernel's test; against the bf16-P
    restatement: output rounding and accumulation order only"""
    c = _Case(B, H, past, q_len, seed=past * 7 + q_len + H + B)
    out = c.run().float().cpu().numpy()
    exact = c.oracle()
    mag = np.abs(exact).max()
    err = np.abs(out - exact)
    print(f"H={H} B={B} P={past} q={q_len}: max err {err.max() / mag:.2e} of max |out|, mean {err.mean() / np.abs(exact).mean():.2e}")
    assert np.isfinite(out).all()
    assert err.max() <= 2e-2 * mag
    assert err.mean() <= 5e-3 * np.abs(exact).mean()
    if H == 16:
        want = c.oracle(p_bf16=True)
        assert np.abs(out - want).max() <= 2.0 ** -7 * mag + 1e-3 * mag


@pytest.mark.gpu
@pytest.mark.parametrize("past,q_len,cut", [(0, 300, 130), (0, 300, 128), (300, 200, 377), (1000, 37, 1001)])
def test_prefill_is_causal(past, q_len, cut):
    """K / V rows at positions >= cut changed to other finite values: every query at a position < cut is bit-identical"""
    c = _Case(2, 16, past, q_len, seed=cut)
    before = c.run()
    g = torch.Generator().manual_seed(cut + 1)
    c.kv[:, cut:] = (torch.randn(c.kv[:, cut:].shape, generator=g) * 3).to(torch.bfloat16).cuda()
    c.rows[:, cut:] = (torch.randn(c.rows[:, cut:].shape, generator=g) * 3).to(torch.bfloat16).cuda()
    after = c.run()
    n = cut - past       # queries at positions < cut
    assert torch.equal(before[:, :n].view(torch.int16), after[:, :n].view(torch.int16))
    assert not torch.equal(before[:, n:].view(torch.int16), after[:, n:].view(torch.int16))


@pytest.mark.gpu
@pytest.mark.parametrize("past,q_len", [(0, 129), (300, 200), (63, 1)])
def test_prefill_ignores_rows_past_the_lengths(past, q_len):
    """NaN / Inf in the q rows past q_len and in the cache and kv_b_proj rows past S: finite output, equal to the clean run"""
    clean = _Case(2, 16, past, q_len, seed=5).run()
    dirty = _Case(2, 16, past, q_len, seed=5, pad=float("nan")).run()
    assert torch.isfinite(dirty.float()).all()
    assert torch.equal(clean.view(torch.int16), dirty.view(torch.int16))


# ------------------------------------------------------------------------------------------------ operator (GPU)
def _modules(heads, seed):
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Attention, DeepseekV3Config
    from ktransformers_b200.operators.attention import KDeepseekV2Attention
    from ktransformers_b200.operators.flashinfer_wrapper import MLAWrapperSingleton
    torch.manual_seed(seed)
    cfg = DeepseekV3Config(hidden_size=1024, num_attention_heads=heads, q_lora_rank=256, num_hidden_layers=1)
    plain = DeepseekV3Attention(cfg, layer_idx=0).to(device="cuda", dtype=torch.bfloat16)
    MLAWrapperSingleton.wrappers.clear()
    return cfg, plain, KDeepseekV2Attention("blk.0.self_attn", None, cfg, plain, "cuda", "cuda")


def _step(op, cache, x, start):
    n = x.shape[1]
    pos = torch.arange(start, start + n, device="cuda").expand(x.shape[0], n)
    out, _, _ = op(x, position_ids=pos, past_key_value=cache, cache_position=torch.arange(start, start + n, device="cuda"))
    return out


def _rel(got, want):
    return (got.float() - want.float()).abs().max().item() / max(want.float().abs().max().item(), 1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("chunks", [1, 3])
@pytest.mark.parametrize("prompt", [2, 65, 300])
@pytest.mark.parametrize("heads,bsz", [(16, 1), (16, 2), (128, 1), (128, 2)])
def test_operator_prefill_then_decode_matches_plain_attention(heads, bsz, prompt, chunks):
    """KDeepseekV2Attention over a prompt (one chunk, or three) and then 5 decode steps through the same cache, against
    the plain module (fp32 softmax over explicit latents); the bar of the decode operator test"""
    from ktransformers_b200.models.custom_cache import StaticCache
    cfg, plain, op = _modules(heads, prompt + heads + bsz)
    cache = StaticCache(cfg, max_batch_size=bsz, max_cache_len=512, device="cuda")
    x = (torch.randn(bsz, prompt, 1024, device="cuda") * 2).to(torch.bfloat16)
    want, past = plain(x, torch.arange(prompt, device="cuda").expand(bsz, prompt))
    cuts = [0, prompt // 3, 2 * prompt // 3, prompt] if chunks == 3 else [0, prompt]
    cuts = sorted(set(cuts))
    got = torch.cat([_step(op, cache, x[:, a:b], a) for a, b in zip(cuts[:-1], cuts[1:])], 1)
    worst = _rel(got, want)
    assert cache.get_seq_length(0) == prompt
    for t in range(prompt, prompt + 5):
        xt = (torch.randn(bsz, 1, 1024, device="cuda") * 2).to(torch.bfloat16)
        g = _step(op, cache, xt, t)
        w, past = plain(xt, torch.full((bsz, 1), t, device="cuda"), past)
        worst = max(worst, _rel(g, w))
    assert worst < 4e-2, worst
    assert cache.get_seq_length(0) == prompt + 5


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [16, 128])
def test_prefill_then_decode_equals_decode_only(heads):
    """a 100-token prompt through prefill, and the same tokens one decode step at a time: the cache rows written and the
    output of the next token agree within the decode bar"""
    from ktransformers_b200.models.custom_cache import StaticCache
    cfg, plain, op = _modules(heads, 11)
    bsz, n = 2, 100
    x = (torch.randn(bsz, n + 1, 1024, device="cuda") * 2).to(torch.bfloat16)
    a = StaticCache(cfg, max_batch_size=bsz, max_cache_len=256, device="cuda")
    b = StaticCache(cfg, max_batch_size=bsz, max_cache_len=256, device="cuda")
    _step(op, a, x[:, :n], 0)
    for t in range(n):
        _step(op, b, x[:, t: t + 1], t)
    ra, rb = a.key_cache[0].view(bsz, -1, 576)[:, :n], b.key_cache[0].view(bsz, -1, 576)[:, :n]
    assert _rel(ra, rb) < 4e-2
    assert _rel(_step(op, a, x[:, n:], n), _step(op, b, x[:, n:], n)) < 4e-2


@pytest.mark.gpu
def test_prefill_makes_no_host_synchronisation():
    from ktransformers_b200.models.custom_cache import StaticCache
    cfg, plain, op = _modules(16, 12)
    cache = StaticCache(cfg, max_batch_size=2, max_cache_len=512, device="cuda")
    x = (torch.randn(2, 200, 1024, device="cuda") * 2).to(torch.bfloat16)
    pos, cpos = torch.arange(200, device="cuda").expand(2, 200), torch.arange(200, device="cuda")
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:   # a first chunk and a second one after it
        op(x[:, :100], position_ids=pos[:, :100], past_key_value=cache, cache_position=cpos[:100])
        op(x[:, 100:], position_ids=pos[:, 100:], past_key_value=cache, cache_position=cpos[100:])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert cache.get_seq_length(0) == 200


def _kernels_of(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.key for e in prof.key_averages()]


@pytest.mark.gpu
def test_prefill_runs_the_prefill_kernel_not_the_decode_kernel():
    from ktransformers_b200.models.custom_cache import StaticCache
    cfg, plain, op = _modules(16, 13)
    cache = StaticCache(cfg, max_batch_size=1, max_cache_len=256, device="cuda")
    x = (torch.randn(1, 65, 1024, device="cuda") * 2).to(torch.bfloat16)
    names = _kernels_of(lambda: _step(op, cache, x[:, :64], 0))
    assert any("mla_prefill_kernel" in k for k in names), names
    assert not any("mla_decode_tc_kernel" in k for k in names), names
    names = _kernels_of(lambda: _step(op, cache, x[:, 64:], 64))
    assert any("mla_decode_tc_kernel" in k for k in names) and not any("mla_prefill_kernel" in k for k in names), names
