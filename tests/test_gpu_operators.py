"""GPU tests of the Python operator layer (the reference-facing injection API) on a tiny GGUF file:
`optimize_and_load_gguf` with the shipped H100 rule file -> KDeepseekV3MoE / KTransformersExperts(KExpertsB200) /
KMoEGateB200 / KTransformersLinear(KLinearB200), decode through the single-launch block call and through the
three-step path (reference control flow, experts.py:972-1012), both against a dense fp32 restatement."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

E, H, I, K = 8, 4096, 512, 4   # rows of 16 super-blocks: the persistent block kernel applies


def _write_gguf(path):
    import gguf
    from ktransformers_b200.util.synth import synth_blocks
    from oracle.bindings import Oracle
    orc = Oracle()
    rng = np.random.default_rng(7)
    w = gguf.GGUFWriter(path, "deepseek2")
    dense, seed = {}, [100]

    def add_q(name, shape, qt):
        seed[0] += 1
        n = int(np.prod(shape))
        q = synth_blocks(int(qt), n, "cpu", seed[0]).numpy()
        w.add_tensor(name, q.reshape(*shape[:-1], -1), raw_dtype=qt)
        dense[name] = orc.to_float(q, int(qt), n).reshape(shape)

    Q4, Q6 = gguf.GGMLQuantizationType.Q4_K, gguf.GGMLQuantizationType.Q6_K
    for n in ("gate", "up"):
        add_q(f"blk.0.ffn_{n}.weight", (I, H), Q4)
        add_q(f"blk.1.ffn_{n}_exps.weight", (E, I, H), Q4)
        add_q(f"blk.1.ffn_{n}_shexp.weight", (I, H), Q4)
    add_q("blk.0.ffn_down.weight", (H, I), Q6)
    add_q("blk.1.ffn_down_exps.weight", (E, H, I), Q6)
    add_q("blk.1.ffn_down_shexp.weight", (H, I), Q6)
    gi = rng.standard_normal((E, H)).astype(np.float32)
    gb = rng.standard_normal((E,)).astype(np.float32)
    w.add_tensor("blk.1.ffn_gate_inp.weight", gi)
    w.add_tensor("blk.1.exp_probs_b.bias", gb)
    dense["blk.1.ffn_gate_inp.weight"], dense["blk.1.exp_probs_b.bias"] = gi, gb
    w.write_header_to_file(); w.write_kv_data_to_file(); w.write_tensors_to_file(); w.close()
    return dense


def test_injected_v3_moe_decodes_through_one_launch_and_matches_dense(tmp_path):
    from ktransformers_b200 import native
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Config, DeepseekV3MoEOnlyForCausalLM
    from ktransformers_b200.operators.experts import KDeepseekV3MoE, KExpertsB200
    from ktransformers_b200.operators.gate import KMoEGateB200
    from ktransformers_b200.optimize.optimize import optimize_and_load_gguf
    import ktransformers_b200.optimize.optimize as opt
    dense = _write_gguf(str(tmp_path / "tiny.gguf"))
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
        assert isinstance(moe, KDeepseekV3MoE) and isinstance(moe.gate, KMoEGateB200)
        assert isinstance(moe.experts.generate_experts, KExpertsB200) and moe.experts.generate_experts.handle is not None

        W = {k: torch.from_numpy(np.array(v)).cuda() for k, v in dense.items()}
        for n_tok in (1, 3, 12, 64):     # block kernel | per-pair kernels | grouped tensor-core path (qlen >= KTB200_GROUPED_MIN)
            x = (torch.randn(1, n_tok, H, device="cuda") / 10).to(torch.bfloat16)
            n0 = native.launch_count()
            y = moe(x)
            torch.cuda.synchronize()
            launches = native.launch_count() - n0
            assert (launches == 1) if n_tok <= 8 else (launches >= 5 if n_tok < 48 else launches >= 13), launches   # block call | gate + 2 (experts) + shared-expert linears | gate + 10 + linears
            # the reference's three-step control flow gives the same bits (decode) / dense fp32 agrees (all)
            if n_tok <= 8:
                keep, KDeepseekV3MoE.BLOCK_MAX_TOKENS = KDeepseekV3MoE.BLOCK_MAX_TOKENS, 0
                try:
                    y3 = moe(x)
                finally:
                    KDeepseekV3MoE.BLOCK_MAX_TOKENS = keep
                idx, wt = moe.last_topk
                ridx, rwt = moe.gate(x)
                assert torch.equal(idx, ridx) and torch.equal(wt, rwt)
                # shared expert: one fused MLP handle vs three KLinearB200 calls with bf16 hand-offs -> close, not equal
                assert (y.float() - y3.float()).abs().max() <= 0.03 * y3.float().abs().max()
            xf = x.view(-1, H).float()
            idx, wt = moe.gate(x)
            ref = torch.zeros_like(xf)
            for t in range(xf.shape[0]):
                for j in range(K):
                    e = int(idx[t, j])
                    g, u, d = W["blk.1.ffn_gate_exps.weight"][e], W["blk.1.ffn_up_exps.weight"][e], W["blk.1.ffn_down_exps.weight"][e]
                    ref[t] += (torch.nn.functional.silu(g @ xf[t]) * (u @ xf[t])) @ d.T * wt[t, j]
            sh = (torch.nn.functional.silu(xf @ W["blk.1.ffn_gate_shexp.weight"].T) * (xf @ W["blk.1.ffn_up_shexp.weight"].T)) @ W["blk.1.ffn_down_shexp.weight"].T
            want = ref + sh
            # int8 activations (the reference CPU arithmetic) vs dense fp32: ~1-2 % of the output scale
            assert (y.view(-1, H).float() - want).abs().max() <= 0.05 * want.abs().max()
    finally:
        torch.set_default_dtype(old)


def test_kt_moe_wrapper_serves_a_layer_from_gguf(tmp_path):
    """KTMoEWrapper(method="B200_GGUF"): load_weights with an EPLB permutation, gpu_experts_mask skipping, submit/sync on a
    caller stream — against the dense fp32 restatement."""
    from ktransformers_b200.kt_moe_wrapper import KTMoEWrapper
    dense = _write_gguf(str(tmp_path / "tiny.gguf"))
    KTMoEWrapper.clear_buffer_cache()
    mask = torch.zeros(E, dtype=torch.bool); mask[2] = True                  # physical expert 2 is served elsewhere
    w = KTMoEWrapper(1, E, K, H, I, mask, cpuinfer_threads=32, threadpool_count=2, weight_path=str(tmp_path), chunked_prefill_size=16)
    p2l = torch.arange(E - 1, -1, -1)                                         # physical slot p holds logical expert E-1-p
    w.load_weights(p2l)
    g = torch.Generator(device="cpu").manual_seed(5)
    n_tok = 5
    x = (torch.randn(n_tok, H, generator=g) / 10).to(torch.bfloat16).cuda()
    ids = torch.stack([torch.randperm(E, generator=g)[:K] for _ in range(n_tok)]).cuda()
    ids[0, 0] = 2                                                             # make sure the mask is exercised
    wt = torch.rand(n_tok, K, generator=g).cuda()
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    w.submit_forward(x, ids, wt, st.cuda_stream)
    y = w.sync_forward(x, st.cuda_stream)
    st.synchronize()
    W = {k_: torch.from_numpy(np.array(v)).cuda() for k_, v in dense.items() if "exps" in k_}
    xf = x.float()
    ref = torch.zeros_like(xf)
    for t in range(n_tok):
        for j in range(K):
            p = int(ids[t, j])
            if p == 2:
                continue
            e = int(p2l[p])
            gw, uw, dw = W["blk.1.ffn_gate_exps.weight"][e], W["blk.1.ffn_up_exps.weight"][e], W["blk.1.ffn_down_exps.weight"][e]
            ref[t] += (torch.nn.functional.silu(gw @ xf[t]) * (uw @ xf[t])) @ dw.T * wt[t, j]
    assert y.dtype == torch.bfloat16 and tuple(y.shape) == (n_tok, H)
    assert (y.float() - ref).abs().max() <= 0.05 * ref.abs().max()
    assert torch.equal(w.forward(x, ids, wt, None), y)                        # forward == submit + sync


def test_pybind_extension_runs_the_reference_submit_sync_sequence(oracle):
    """The compiled pybind module driven the way kt-kernel/python/experts_base.py drives kt_kernel_ext:
    CPUInfer.submit(moe.load_weights_task()); sync(); per step submit_with_cuda_stream(stream, moe.forward_task(qlen_ptr, k,
    ids, w, in, out)); sync_with_cuda_stream(stream) — output vs the CPU oracle."""
    import importlib
    import sys as _sys
    _sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ktransformers_b200"))
    ext = importlib.import_module("kt_kernel_ext_b200")
    from ktransformers_b200.util.synth import synth_blocks
    from oracle.bindings import BF16, Q4_K, Q6_K, f32_to_bf16_bits
    E, k, H, I = 8, 4, 4096, 512
    gate, up, down = (synth_blocks(Q4_K, E * I * H, "cuda", 1), synth_blocks(Q4_K, E * I * H, "cuda", 2), synth_blocks(Q6_K, E * H * I, "cuda", 3))
    g_np, u_np, d_np = gate.cpu().numpy(), up.cpu().numpy(), down.cpu().numpy()
    cfg = ext.moe.MOEConfig(E, k, H, I)
    cfg.gate_proj, cfg.up_proj, cfg.down_proj = gate.data_ptr(), up.data_ptr(), down.data_ptr()
    cfg.gate_type, cfg.up_type, cfg.down_type, cfg.hidden_type, cfg.max_len = Q4_K, Q4_K, Q6_K, BF16, 16
    moe = ext.moe.B200_MOE(cfg)
    cpuinfer = ext.CPUInfer(1)
    with pytest.raises(RuntimeError, match="Not Loaded"):
        moe.forward(torch.tensor([1], dtype=torch.int32).data_ptr(), k, 0, 0, 0, 0, False)
    cpuinfer.submit(moe.load_weights_task())
    cpuinfer.sync()
    rng = np.random.default_rng(0)
    qlen = 3
    x = f32_to_bf16_bits((rng.standard_normal((qlen, H)) / 100).astype(np.float32))
    ids = np.stack([rng.permutation(E)[:k] for _ in range(qlen)]).astype(np.int64)
    w = rng.random((qlen, k)).astype(np.float32)
    x_d = torch.from_numpy(x.view(np.int16)).view(torch.bfloat16).cuda()
    ids_d, w_d = torch.from_numpy(ids).cuda(), torch.from_numpy(w).cuda()
    out_d = torch.zeros((qlen, H), dtype=torch.bfloat16, device="cuda")
    bsz = torch.tensor([qlen], dtype=torch.int32).pin_memory()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    cpuinfer.submit_with_cuda_stream(side.cuda_stream, moe.forward_task(bsz.data_ptr(), k, ids_d.data_ptr(), w_d.data_ptr(), x_d.data_ptr(), out_d.data_ptr()))
    cpuinfer.sync_with_cuda_stream(side.cuda_stream)
    side.synchronize()
    want = oracle.moe_forward(E, H, I, g_np, u_np, d_np, Q4_K, Q4_K, Q6_K, BF16, ids, w, x)
    got = out_d.cpu().view(torch.int16).numpy().view(np.uint16)
    from oracle.bindings import bf16_to_f32
    a, b = bf16_to_f32(got), bf16_to_f32(want)
    assert (np.abs(a - b) <= 2.0 ** -7 * np.maximum(np.abs(a), np.abs(b)) + 1e-3 * np.abs(b).max()).all()


@pytest.mark.parametrize("heads,bsz", [(16, 1), (128, 2)])
def test_kdeepseek_v2_attention_absorbed_paged_decode_matches_plain_attention(heads, bsz):
    """KDeepseekV2Attention (operators/attention.py; reference attention.py:349-478): q/kv projections, RoPE, paged latent
    cache write (ktb200_mla_kv_write), W_UK absorb, ktb200_mla_decode (wgmma), W_UV, o_proj — token by token against the
    plain non-absorbed attention of the same module (fp32 softmax over explicit latents)."""
    from ktransformers_b200.models.custom_cache import StaticCache
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Attention, DeepseekV3Config
    from ktransformers_b200.operators.attention import KDeepseekV2Attention
    from ktransformers_b200.operators.flashinfer_wrapper import MLAWrapperSingleton
    torch.manual_seed(3)
    cfg = DeepseekV3Config(hidden_size=1024, num_attention_heads=heads, q_lora_rank=256, num_hidden_layers=1)
    plain = DeepseekV3Attention(cfg, layer_idx=0).to(device="cuda", dtype=torch.bfloat16)
    MLAWrapperSingleton.wrappers.clear()
    op = KDeepseekV2Attention("blk.0.self_attn", None, cfg, plain, "cuda", "cuda")
    cache = StaticCache(cfg, max_batch_size=bsz, max_cache_len=256, device="cuda")
    steps, past, worst = 70, None, 0.0
    for t in range(steps):
        x = (torch.randn(bsz, 1, 1024, device="cuda") * 2).to(torch.bfloat16)
        pos = torch.full((bsz, 1), t, dtype=torch.int64, device="cuda")
        got, _, _ = op(x, position_ids=pos, past_key_value=cache, cache_position=torch.tensor([t], device="cuda"))
        want, past = plain(x, pos, past)
        err = (got.float() - want.float()).abs().max().item() / max(want.float().abs().max().item(), 1e-6)
        worst = max(worst, err)
    assert worst < 4e-2, worst        # bf16 projections / bf16 P and absorbed products vs the fp32-softmax restatement
    assert cache.get_seq_length(0) == steps


def test_serve_rule_file_v2_classes_carry_bsz_tensor(tmp_path):
    """balance-serve flavour (experts.py:1172-1350): KDeepseekV3MoEV2 / KTransformersExpertsV2 with a device-side batch size; rows
    below bsz equal the V1 forward bit for bit, through the block kernel (3 tokens), the per-pair kernels (12) and the grouped path (64)."""
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Config, DeepseekV3MoEOnlyForCausalLM
    from ktransformers_b200.operators.experts import KDeepseekV3MoE, KDeepseekV3MoEV2, KTransformersExpertsV2
    from ktransformers_b200.optimize.optimize import optimize_and_load_gguf
    import ktransformers_b200.optimize.optimize as opt
    _write_gguf(str(tmp_path / "tiny.gguf"))
    rule = os.path.join(os.path.dirname(opt.__file__), "optimize_rules", "DeepSeek-V3-Chat-b200-serve.yaml")
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        cfg = DeepseekV3Config(hidden_size=H, intermediate_size=I, moe_intermediate_size=I, n_routed_experts=E, n_shared_experts=1,
                               num_experts_per_tok=K, n_group=2, topk_group=1, num_hidden_layers=2, first_k_dense_replace=1)
        with torch.device("meta"):
            model = DeepseekV3MoEOnlyForCausalLM(cfg)
        optimize_and_load_gguf(model, rule, str(tmp_path), cfg, default_device="cuda")
        moe = model.model.layers[1].mlp
        assert isinstance(moe, KDeepseekV3MoEV2) and isinstance(moe.experts, KTransformersExpertsV2) and moe.experts.prefill_experts is None
        for n_tok, live in ((3, 2), (12, 7), (64, 50)):
            x = (torch.randn(1, n_tok, H, device="cuda") / 10).to(torch.bfloat16)
            bsz = torch.tensor([live], dtype=torch.int32, device="cuda")
            y2 = moe(x, bsz)
            y1 = moe(x)      # bsz_tensor None -> the V1 control flow
            torch.cuda.synchronize()
            assert torch.equal(y2[0, :live].view(torch.int16), y1[0, :live].view(torch.int16)), n_tok
    finally:
        torch.set_default_dtype(old)


def test_klinear_fp8_operator_from_safetensors(tmp_path):
    """KLinearFP8 (operators/linear.py:388-435 contract) through KTransformersLinear, weights found by the SafeTensorLoader as
    `<key>.weight` (float8_e4m3fn) + `<key>.weight_scale_inv`; output against the dequantised dense fp32 product."""
    from safetensors.torch import save_file
    from ktransformers_b200.operators.linear import KLinearFP8, KTransformersLinear, LINEAR_MAP
    from ktransformers_b200.util.custom_loader import ModelLoaderFactory, SafeTensorLoader
    from ktransformers_b200.util.utils import InferenceState
    assert LINEAR_MAP["KLinearFP8"] is KLinearFP8
    Kf, Nf = 1024, 384
    g = torch.Generator().manual_seed(5)
    w = (torch.randn(Nf, Kf, generator=g) * 0.5).to(torch.float8_e4m3fn)
    s = torch.rand(Nf // 128, Kf // 128, generator=g) * 0.02 + 0.001
    save_file({"model.layers.0.self_attn.o_proj.weight": w, "model.layers.0.self_attn.o_proj.weight_scale_inv": s}, str(tmp_path / "m.safetensors"))
    ld = ModelLoaderFactory.create_loader(str(tmp_path))
    assert isinstance(ld, SafeTensorLoader) and ld.has_tensor("model.layers.0.self_attn.o_proj.weight_scale_inv")
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        lin = KTransformersLinear("model.layers.0.self_attn.o_proj", ld, None, torch.nn.Linear(Kf, Nf, bias=False, device="meta"),
                                  generate_op="KLinearFP8", prefill_op=None)
        lin.load(mode=InferenceState.GENERATE)
        x = (torch.randn(2, 3, Kf, device="cuda") / 10).to(torch.bfloat16)
        y = lin(x)
        assert y.shape == (2, 3, Nf) and y.dtype == torch.bfloat16
        dense = w.float().view(Nf // 128, 128, Kf // 128, 128) * s.view(Nf // 128, 1, Kf // 128, 1)
        want = x.float().cpu().view(-1, Kf) @ dense.view(Nf, Kf).T
        assert (y.float().cpu().view(-1, Nf) - want).abs().max() <= 0.06 * want.abs().max()     # fp8 activations: a few %
        lin.unload()
        with pytest.raises(Exception):
            lin.generate_linear.forward(x)
    finally:
        torch.set_default_dtype(old)


def test_fp8_linear_ggml_experts_rule_file_on_a_hybrid_safetensors(tmp_path):
    """BASELINE config 3's layout end to end on the host side: the FP8 + GGUF hybrid safetensors (FP8 128x128 linears under HF
    names, raw GGUF expert blocks + `.ggml_type` under GGUF names) through `optimize_and_load_gguf` with
    DeepSeek-V3-Chat-fp8-linear-ggml-experts-b200.yaml: KLinearFP8 linears, KExpertsB200 experts, KMoEGateB200 router."""
    from safetensors.torch import save_file
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Config, DeepseekV3MoEOnlyForCausalLM
    from ktransformers_b200.operators.experts import KDeepseekV3MoE, KExpertsB200
    from ktransformers_b200.operators.linear import KLinearFP8, KTransformersLinear
    from ktransformers_b200.optimize.optimize import optimize_and_load_gguf
    from ktransformers_b200.util.synth import synth_blocks
    from oracle.bindings import Oracle
    import ktransformers_b200.optimize.optimize as opt
    orc = Oracle()
    g = torch.Generator().manual_seed(11)
    tensors, dense = {}, {}

    def add_fp8(name, out_f, in_f):
        w = (torch.randn(out_f, in_f, generator=g) * 0.3).to(torch.float8_e4m3fn)
        s = torch.rand((out_f + 127) // 128, in_f // 128, generator=g) * 0.02 + 0.005
        tensors[name + ".weight"], tensors[name + ".weight_scale_inv"] = w, s
        d = w.float().view(-1, 128, in_f // 128, 128) * s.view(-1, 1, in_f // 128, 1) if out_f % 128 == 0 else None
        dense[name] = d.reshape(out_f, in_f)

    for n, (o, i) in {"gate_proj": (I, H), "up_proj": (I, H), "down_proj": (H, I)}.items():
        add_fp8(f"model.layers.0.mlp.{n}", o, i)
        add_fp8(f"model.layers.1.mlp.shared_experts.{n}", o, i)
    for n, qt, shape in (("gate", 12, (E, I, H)), ("up", 12, (E, I, H)), ("down", 14, (E, H, I))):
        q = synth_blocks(qt, int(np.prod(shape)), "cpu", 300 + qt + len(n)).numpy()
        tensors[f"blk.1.ffn_{n}_exps.weight"] = torch.from_numpy(q.copy())
        tensors[f"blk.1.ffn_{n}_exps.ggml_type"] = torch.tensor(qt)
        dense[f"exps.{n}"] = torch.from_numpy(orc.to_float(q, qt, int(np.prod(shape))).reshape(shape))
    tensors["blk.1.ffn_gate_inp.weight"] = torch.randn(E, H, generator=g)
    tensors["blk.1.exp_probs_b.bias"] = 0.01 * torch.randn(E, generator=g)
    save_file(tensors, str(tmp_path / "hybrid.safetensors"))
    rule = os.path.join(os.path.dirname(opt.__file__), "optimize_rules", "DeepSeek-V3-Chat-fp8-linear-ggml-experts-b200.yaml")
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        cfg = DeepseekV3Config(hidden_size=H, intermediate_size=I, moe_intermediate_size=I, n_routed_experts=E, n_shared_experts=1,
                               num_experts_per_tok=K, n_group=2, topk_group=1, num_hidden_layers=2, first_k_dense_replace=1)
        with torch.device("meta"):
            model = DeepseekV3MoEOnlyForCausalLM(cfg)
        optimize_and_load_gguf(model, rule, str(tmp_path), cfg, default_device="cuda")
        moe = model.model.layers[1].mlp
        assert isinstance(moe, KDeepseekV3MoE) and isinstance(moe.experts.generate_experts, KExpertsB200) and moe.experts.generate_experts.handle is not None
        sh = moe.shared_experts.gate_proj
        assert isinstance(sh, KTransformersLinear) and isinstance(sh.generate_linear, KLinearFP8) and sh.generate_linear.handle is not None
        assert isinstance(model.model.layers[0].mlp.down_proj.generate_linear, KLinearFP8)
        x = (torch.randn(1, 3, H, device="cuda") / 10).to(torch.bfloat16)
        y = moe(x)
        xf = x.view(-1, H).float().cpu()
        idx, wt = moe.gate(x)
        idx, wt = idx.cpu(), wt.cpu()
        want = torch.zeros_like(xf)
        for t in range(xf.shape[0]):
            for j in range(K):
                e = int(idx[t, j])
                want[t] += (torch.nn.functional.silu(dense["exps.gate"][e] @ xf[t]) * (dense["exps.up"][e] @ xf[t])) @ dense["exps.down"][e].T * wt[t, j]
        p = "model.layers.1.mlp.shared_experts."
        want += (torch.nn.functional.silu(xf @ dense[p + "gate_proj"].T) * (xf @ dense[p + "up_proj"].T)) @ dense[p + "down_proj"].T
        assert (y.view(-1, H).float().cpu() - want).abs().max() <= 0.06 * want.abs().max()
        y0 = model.model.layers[0].mlp(x)                       # the dense layer: three KLinearFP8 projections
        p0 = "model.layers.0.mlp."
        want0 = (torch.nn.functional.silu(xf @ dense[p0 + "gate_proj"].T) * (xf @ dense[p0 + "up_proj"].T)) @ dense[p0 + "down_proj"].T
        assert (y0.view(-1, H).float().cpu() - want0).abs().max() <= 0.06 * want0.abs().max()
    finally:
        torch.set_default_dtype(old)
