"""CPU: host-side logic — the C-ABI library loads and exports every declared symbol (no compute calls),
GGUF loading, name translation, the YAML injection framework, error behaviour, and the rule that the product
never routes through the oracle or a CPU fallback."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    from ktransformers_b200 import native
    hdr = open(os.path.join(ROOT, "include", "ktb200.h")).read()
    declared = set(re.findall(r"\b(ktb200_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(native.SYMBOLS), declared ^ set(native.SYMBOLS)
    lib = native.lib()
    for name in declared:
        assert hasattr(lib, name), name
    # non-compute calls work without a GPU
    assert lib.ktb200_type_size(12) == 144 and lib.ktb200_blck_size(12) == 256
    assert lib.ktb200_type_size(14) == 210 and lib.ktb200_type_size(15) == 292
    assert lib.ktb200_type_size(99) == 0
    assert b"sm_90a" in lib.ktb200_version()


def test_missing_library_fails_loudly(monkeypatch):
    from ktransformers_b200 import native
    monkeypatch.setattr(native, "_lib", None)
    monkeypatch.setattr(native, "LIB_PATH", "/nonexistent/libktb200.so")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        native.lib()


def test_product_never_touches_the_oracle():
    bad = []
    for base, _, files in os.walk(os.path.join(ROOT, "ktransformers_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(base, f), errors="replace").read()
                if re.search(r"^\s*(from|import)\s+oracle\b", src, re.M) or "ktoracle" in src and not f.endswith((".cuh", ".cu")):
                    bad.append(os.path.join(base, f))
    assert not bad, bad


def test_error_codes_map_to_reference_exceptions():
    import ctypes as C

    from ktransformers_b200 import native
    lib = native.lib()
    # invalid ggml type -> ValueError (kt-kernel/ext_bindings.cpp:88-92); no GPU needed: validation precedes CUDA calls
    cfg = native.MoeConfig(4, 2, 512, 256, 64, 10, 8, 1, 1, 1, 1, 2, 12, 14, 30, 0)   # gate_type=2 (Q4_0)
    h = C.c_void_p()
    with pytest.raises(ValueError, match="unsupported ggml weight type"):
        native.check(lib.ktb200_moe_create(C.byref(cfg), 0, C.byref(h)))
    cfg = native.MoeConfig(4, 2, 500, 256, 64, 10, 8, 1, 1, 1, 1, 12, 12, 14, 30, 0)
    with pytest.raises(ValueError, match="multiples of 256"):
        native.check(lib.ktb200_moe_create(C.byref(cfg), 0, C.byref(h)))
    with pytest.raises(ValueError):
        native.check(lib.ktb200_dequantize(1, 12, 100, 1, 0, None))                    # n not a multiple of the block


# ------------------------------------------------------------------------------------------ GGUF + injection
E, H, I, K = 4, 256, 256, 2


def _write_gguf(path):
    import gguf
    rng = np.random.default_rng(0)
    w = gguf.GGUFWriter(path, "deepseek2")
    dense = {}

    from ktransformers_b200.util.synth import synth_blocks
    from oracle.bindings import Oracle
    orc = Oracle()
    seed = [0]

    def add_q(name, arr, qt):
        # well-formed random blocks of the type (gguf-py has no K-quant quantiser); dense truth from the oracle
        seed[0] += 1
        q = synth_blocks(int(qt), arr.size, "cpu", seed[0]).numpy()
        w.add_tensor(name, q.reshape(*arr.shape[:-1], -1), raw_dtype=qt)
        dense[name] = orc.to_float(q, int(qt), arr.size).reshape(arr.shape)

    # layer 0: dense MLP ; layer 1: MoE
    add_q("blk.0.ffn_gate.weight", rng.standard_normal((I, H)), gguf.GGMLQuantizationType.Q4_K)
    add_q("blk.0.ffn_up.weight", rng.standard_normal((I, H)), gguf.GGMLQuantizationType.Q4_K)
    add_q("blk.0.ffn_down.weight", rng.standard_normal((H, I)), gguf.GGMLQuantizationType.Q6_K)
    add_q("blk.1.ffn_gate_exps.weight", rng.standard_normal((E, I, H)), gguf.GGMLQuantizationType.Q4_K)
    add_q("blk.1.ffn_up_exps.weight", rng.standard_normal((E, I, H)), gguf.GGMLQuantizationType.Q4_K)
    add_q("blk.1.ffn_down_exps.weight", rng.standard_normal((E, H, I)), gguf.GGMLQuantizationType.Q6_K)
    add_q("blk.1.ffn_gate_shexp.weight", rng.standard_normal((I, H)), gguf.GGMLQuantizationType.Q4_K)
    add_q("blk.1.ffn_up_shexp.weight", rng.standard_normal((I, H)), gguf.GGMLQuantizationType.Q4_K)
    add_q("blk.1.ffn_down_shexp.weight", rng.standard_normal((H, I)), gguf.GGMLQuantizationType.Q6_K)
    gi = rng.standard_normal((E, H)).astype(np.float32)
    gb = rng.standard_normal((E,)).astype(np.float32)
    w.add_tensor("blk.1.ffn_gate_inp.weight", gi)
    w.add_tensor("blk.1.exp_probs_b.bias", gb)
    dense["blk.1.ffn_gate_inp.weight"], dense["blk.1.exp_probs_b.bias"] = gi, gb
    w.write_header_to_file(); w.write_kv_data_to_file(); w.write_tensors_to_file(); w.close()
    return dense


@pytest.fixture(scope="module")
def tiny_gguf(tmp_path_factory):
    d = tmp_path_factory.mktemp("gguf")
    dense = _write_gguf(str(d / "tiny.gguf"))
    return str(d), dense


def test_gguf_loader_raw_and_dense(tiny_gguf):
    from ktransformers_b200.util.custom_loader import GGUFLoader, ModelLoaderFactory
    path, dense = tiny_gguf
    ld = ModelLoaderFactory.create_loader(path)
    assert isinstance(ld, GGUFLoader)
    key = "model.layers.1.mlp.experts"
    assert ld.has_tensor(key + ".ffn_gate_exps.weight") and not ld.has_tensor("model.layers.9.mlp.gate.weight")
    assert ld.get_ggml_type(key + ".ffn_gate_exps.weight") == 12 and ld.get_ggml_type(key + ".ffn_down_exps.weight") == 14
    raw = ld.get_mmap_tensor(key + ".ffn_gate_exps.weight")
    assert raw.dtype == np.uint8 and raw.size == E * I * H // 256 * 144      # 144-byte Q4_K blocks, row-major [E][I][H/256]
    with pytest.raises(KeyError):
        ld.get_ggml_type("model.layers.3.mlp.gate.weight")
    # dense load on CPU == gguf's own dequantiser, shape reversed like the reference (custom_loader.py:506)
    t = ld.load_gguf_tensor("model.layers.1.mlp.shared_experts.down_proj.weight", device="cpu", target_dtype=torch.float32)
    assert tuple(t.shape) == (H, I)
    np.testing.assert_allclose(t.numpy(), dense["blk.1.ffn_down_shexp.weight"], atol=1e-6)
    t = ld.load_gguf_tensor("model.layers.1.mlp.gate.e_score_correction_bias", device="cpu", target_dtype=torch.float32)
    np.testing.assert_array_equal(t.numpy(), dense["blk.1.exp_probs_b.bias"])
    one = ld.load_expert_tensor(key + ".ffn_up_exps.weight", ld.get_mmap_tensor(key + ".ffn_up_exps.weight"), 2, I * H, device="cpu", target_dtype=torch.float32)
    np.testing.assert_allclose(one.numpy(), dense["blk.1.ffn_up_exps.weight"][2], atol=1e-6)


RULES_CPU = """
- match:
    name: "^model\\\\.layers\\\\..*$"
    class: torch.nn.Linear
  replace:
    class: ktransformers_b200.operators.linear.KTransformersLinear
    kwargs: {generate_device: "cpu", prefill_device: "cpu", generate_op: "KLinearTorch", prefill_op: "KLinearTorch"}
- match:
    name: "^model\\\\.layers\\\\..*\\\\.mlp$"
    class: ktransformers_b200.models.modeling_deepseek_v3.DeepseekV3MoE
  replace:
    class: ktransformers_b200.operators.experts.KDeepseekV3MoE
    kwargs: {generate_device: "cpu", prefill_device: "cpu"}
- match:
    class: ktransformers_b200.models.modeling_deepseek_v3.MoEGate
  replace:
    class: ktransformers_b200.operators.gate.KMoEGate
    kwargs: {generate_device: "cpu", prefill_device: "cpu"}
- match:
    name: "^model\\\\.layers\\\\..*\\\\.mlp\\\\.experts$"
  replace:
    class: ktransformers_b200.operators.experts.KTransformersExperts
    kwargs: {prefill_device: "cpu", prefill_op: "KExpertsTorch", generate_device: "cpu", generate_op: "KExpertsTorch"}
  recursive: False
"""


def test_rule_matching_injection_and_forward(tiny_gguf, tmp_path):
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Config, DeepseekV3MoEOnlyForCausalLM
    from ktransformers_b200.operators.base_operator import BaseInjectedModule
    from ktransformers_b200.operators.experts import KDeepseekV3MoE, KTransformersExperts
    from ktransformers_b200.operators.gate import KMoEGate
    from ktransformers_b200.operators.linear import KTransformersLinear
    from ktransformers_b200.optimize.optimize import gen_optimize_config, optimize_and_load_gguf
    from ktransformers_b200.util.utils import InferenceState
    path, dense = tiny_gguf
    torch.set_default_dtype(torch.float32)
    cfg = DeepseekV3Config(hidden_size=H, intermediate_size=I, moe_intermediate_size=I, n_routed_experts=E, n_shared_experts=1,
                           num_experts_per_tok=K, n_group=2, topk_group=1, num_hidden_layers=2, first_k_dense_replace=1)
    with torch.device("meta"):
        model = DeepseekV3MoEOnlyForCausalLM(cfg)
    rule = tmp_path / "rules.yaml"
    rule.write_text(RULES_CPU)
    # rule matching: first rule wins, `recursive: False` prunes the expert sub-modules
    import yaml
    oc = {}
    gen_optimize_config(model, oc, yaml.safe_load(RULES_CPU), default_device="cpu")
    assert oc["model.layers.1.mlp"]["class"].endswith("KDeepseekV3MoE")
    assert oc["model.layers.1.mlp.experts"]["class"].endswith("KTransformersExperts")
    assert oc["model.layers.1.mlp.experts"]["kwargs"]["generate_op"] == "KExpertsTorch"
    assert "model.layers.1.mlp.experts.0" not in oc and "model.layers.1.mlp.experts.0.gate_proj" not in oc
    assert oc["model.layers.0.mlp.gate_proj"]["class"].endswith("KTransformersLinear")
    assert oc["model.layers"]["class"] == "default" and oc["model.layers"]["kwargs"]["generate_device"] == "cpu"

    optimize_and_load_gguf(model, str(rule), path, cfg, default_device="cpu")
    moe = model.model.layers[1].mlp
    assert isinstance(moe, KDeepseekV3MoE) and isinstance(moe, BaseInjectedModule)
    assert isinstance(moe.experts, KTransformersExperts) and isinstance(moe.gate, KMoEGate)
    assert isinstance(model.model.layers[0].mlp.gate_proj, KTransformersLinear)
    assert moe.experts.mode == InferenceState.GENERATE and len(moe.experts.orig_module) == E
    assert model.gguf_loader.tensor_device_map["model.layers.1.mlp.experts"]["generate_op"] == "KExpertsTorch"
    # attribute forwarding of the proxy (base_operator.py:31-55)
    assert moe.gate.top_k == K and moe.gate.n_routed_experts == E

    x = torch.randn(1, 3, H) / 10
    y = model.model.layers[1].mlp(x)
    # dense fp32 restatement of the block
    W = {k: torch.from_numpy(np.array(v)) for k, v in dense.items()}
    xf = x.view(-1, H)
    idx, wt = moe.gate(x)
    ref = torch.zeros_like(xf)
    for t in range(xf.shape[0]):
        for j in range(K):
            e = int(idx[t, j])
            g, u, d = W["blk.1.ffn_gate_exps.weight"][e], W["blk.1.ffn_up_exps.weight"][e], W["blk.1.ffn_down_exps.weight"][e]
            ref[t] += (torch.nn.functional.silu(g @ xf[t]) * (u @ xf[t])) @ d.T * wt[t, j]
    sh = (torch.nn.functional.silu(xf @ W["blk.1.ffn_gate_shexp.weight"].T) * (xf @ W["blk.1.ffn_up_shexp.weight"].T)) @ W["blk.1.ffn_down_shexp.weight"].T
    torch.testing.assert_close(y.view(-1, H), ref + sh, rtol=1e-4, atol=1e-4)
    # mode switching contract
    moe.experts.set_inference_mode(InferenceState.PREFILL)
    assert moe.experts.mode == InferenceState.PREFILL
    torch.testing.assert_close(model.model.layers[1].mlp(x), y, rtol=1e-5, atol=1e-5)
    moe.experts.set_inference_mode(InferenceState.UNLOAD)
    with pytest.raises(ValueError):
        moe.experts.set_inference_mode("bogus")


def test_b200_ops_are_registered_and_refuse_cpu():
    from ktransformers_b200.operators.experts import EXPERTS_MAP, KExpertsB200
    from ktransformers_b200.operators.linear import LINEAR_MAP
    assert "KExpertsB200" in EXPERTS_MAP and "KLinearB200" in LINEAR_MAP
    with pytest.raises(AssertionError):
        KExpertsB200("k", None, None, 8, device="cpu")
    import yaml
    rules = yaml.safe_load(open(os.path.join(ROOT, "ktransformers_b200", "optimize", "optimize_rules", "DeepSeek-V3-Chat-b200.yaml")))
    ops = [r["replace"]["kwargs"].get("generate_op") for r in rules if "kwargs" in r["replace"]]
    assert "KExpertsB200" in ops and "KLinearB200" in ops


def test_kt_moe_wrapper_front_door_contract():
    """KTMoEWrapper (kt-kernel/python/experts.py:72-262) for the H100 backend: constructor checks, mask handling and the
    EPLB permutation are host logic; the compute goes through KExpertsB200 (GPU tests)."""
    from ktransformers_b200.kt_moe_wrapper import KTMoEWrapper
    with pytest.raises(NotImplementedError):
        KTMoEWrapper(0, 8, 2, 256, 256, None, 32, 2, "/x", 64, method="AMXINT4")            # CPU backends are not built here
    with pytest.raises(NotImplementedError):
        KTMoEWrapper(0, 8, 2, 256, 256, None, 32, 2, "/x", 64, method="B200_GGUF", mode="sft")
    with pytest.raises(ValueError):
        KTMoEWrapper(0, 8, 2, 256, 256, None, 32, 2, "/x", 64, max_deferred_experts_per_token=1)
    with pytest.raises(ValueError):
        KTMoEWrapper(0, 8, 2, 256, 256, torch.zeros(7, dtype=torch.bool), 32, 2, "/x", 64)
    mask = torch.zeros(8, dtype=torch.bool); mask[[0, 5]] = True
    w = KTMoEWrapper(3, 8, 2, 256, 256, mask, 32, 2, "/x", 64)
    assert w.num_gpu_experts == 2 and w.key == "model.layers.3.mlp.experts" and w.moe.hidden_dtype == torch.bfloat16
    raw = torch.arange(8 * 4, dtype=torch.uint8)                                          # 8 experts x 4 bytes
    p2l = torch.tensor([7, 6, 5, 4, 3, 2, 1, 0])
    assert KTMoEWrapper._permute(raw, 8, p2l).reshape(8, 4)[0].tolist() == [28, 29, 30, 31]   # physical slot 0 holds logical expert 7
    assert torch.equal(KTMoEWrapper._permute(raw, 8, None), raw)
    with pytest.raises(ValueError):
        KTMoEWrapper._permute(raw, 8, torch.tensor([0, 0, 1, 2, 3, 4, 5, 6]))
    with pytest.raises(NotImplementedError):
        w.load_weights_from_tensors(torch.zeros(8, 4, 4), torch.zeros(8, 4, 4), torch.zeros(8, 4, 4))   # no online K-quant quantiser
    with pytest.raises(RuntimeError):
        w.submit_forward(torch.zeros(1, 256), torch.zeros(1, 2, dtype=torch.long), torch.zeros(1, 2))
    KTMoEWrapper.set_capture_batch_sizes([8, 1, 4])
    assert KTMoEWrapper.get_capture_batch_sizes() == [1, 4, 8]


def test_ep_comm_argument_checks_need_no_gpu():
    """ktb200_ep_* validate their communicator before touching CUDA (include/ktb200.h)."""
    import ctypes as C
    from ktransformers_b200 import native
    lib = native.lib()
    ok = native.EpComm.make(0, 2, 256, 30, [16, 32], [48, 64], [80, 96])
    assert ok.world == 2 and ok.token_bufs[1] == 32 and ok.flag_bufs[0] == 80
    for bad in (native.EpComm.make(2, 2, 256, 30, [16, 32], [48, 64], [80, 96]),          # rank out of range
                native.EpComm.make(0, 2, 250, 30, [16, 32], [48, 64], [80, 96]),          # hidden not a multiple of 8
                native.EpComm.make(0, 2, 256, 12, [16, 32], [48, 64], [80, 96]),          # Q4_K is not a hidden type
                native.EpComm.make(0, 2, 256, 30, [16, 0], [48, 64], [80, 96])):          # a peer pointer is missing
        with pytest.raises(ValueError):
            native.check(lib.ktb200_ep_all_gather_tokens(C.byref(bad), 16, None, None))
        with pytest.raises(ValueError):
            native.check(lib.ktb200_ep_reduce_own_token(C.byref(bad), 16, None, None))
    with pytest.raises(ValueError):
        native.check(lib.ktb200_ep_all_gather_tokens(C.byref(ok), None, None, None))       # null token


@pytest.mark.parametrize("splits", [129, 200, 2 ** 31 - 1])
def test_mla_decode_refuses_more_than_128_kv_splits(splits):
    """the split-KV merge weighs at most 128 partials: ktb200_mla_decode refuses more before any device work (the pointers
    are aligned stand-ins that are never dereferenced; 128 itself runs on the GPU in tests/test_mla_lengths.py)"""
    import ctypes as C
    from ktransformers_b200 import native
    lib = native.lib()
    base = 1 << 24
    p = native.MlaParams(1, 128, 64, 128, splits, 0.07, base, base + (1 << 20), base + (2 << 20), base + (3 << 20), base + (4 << 20),
                         base + (5 << 20), None, base + (6 << 20), 1 << 30, 128 * 64)
    assert lib.ktb200_mla_decode(C.byref(p), None) == native.EINVAL
    assert f"num_kv_splits {splits} exceeds the maximum of 128" in lib.ktb200_last_error().decode()


def test_pybind_module_exposes_the_reference_extension_surface():
    """kt_kernel_ext_b200 (csrc/ext_bindings.cpp) — the compiled pybind boundary: names and call shapes of
    kt-kernel/ext_bindings.cpp (MOEConfig :746-831, bind_moe_module :447-471, CPUInfer :554-565)."""
    import importlib
    import sys
    sys.path.insert(0, os.path.join(ROOT, "ktransformers_b200"))
    ext = importlib.import_module("kt_kernel_ext_b200")
    assert "sm_90a" in ext.version()
    cfg = ext.moe.MOEConfig(8, 2, 512, 256)
    for f in ("expert_num", "num_experts_per_tok", "hidden_size", "intermediate_size", "layer_idx", "max_len", "group_min_len",
              "group_max_len", "gate_type", "up_type", "down_type", "hidden_type", "gate_proj", "up_proj", "down_proj",
              "physical_to_logical_map", "gpu_experts_mask", "pool"):
        assert hasattr(cfg, f), f
    cfg.gate_proj = 4096
    assert cfg.gate_proj == 4096 and cfg.expert_num == 8 and cfg.num_experts_per_tok == 2
    assert ext.moe.MOEConfig(8, 2, 512, 256, 0).gpu_experts_mask == 0
    for meth in ("warm_up_task", "load_weights_task", "forward_task", "warm_up", "load_weights", "forward"):
        assert hasattr(ext.moe.B200_MOE, meth), meth
    for meth in ("submit", "sync", "submit_with_cuda_stream", "sync_with_cuda_stream"):
        assert hasattr(ext.CPUInfer, meth), meth
    with pytest.raises(RuntimeError, match="null weight pointer"):       # C++ exception -> Python, like the reference
        ext.moe.B200_MOE(ext.moe.MOEConfig(8, 2, 512, 256))


def test_shipped_rule_files_name_importable_classes():
    """Every `class:` a shipped rule file names resolves (the serve flavour swaps in the V2 MoE / experts classes, experts.py:1172-1350)."""
    import importlib
    import yaml
    import ktransformers_b200.optimize.optimize as opt
    d = os.path.join(os.path.dirname(opt.__file__), "optimize_rules")
    seen = set()
    for fn in sorted(os.listdir(d)):
        for rule in yaml.safe_load(open(os.path.join(d, fn))):
            for part in ("match", "replace"):
                c = rule.get(part, {}).get("class")
                if c and c != "default":
                    mod, name = c.rsplit(".", 1)
                    assert hasattr(importlib.import_module(mod), name), c
                    seen.add(name)
    assert {"KDeepseekV3MoE", "KDeepseekV3MoEV2", "KTransformersExperts", "KTransformersExpertsV2"} <= seen
    from ktransformers_b200.operators.experts import KTransformersExpertsV2
    import inspect
    assert list(inspect.signature(KTransformersExpertsV2.forward).parameters)[1:] == ["input_tensor", "expert_ids", "weights", "bsz_tensor", "cuda_graph_idx"]


def test_safetensor_loader_and_klinear_fp8_contract(tmp_path):
    """util/custom_loader.py SafeTensorLoader (custom_loader.py:52-112) finds `<key>.weight` / `<key>.weight_scale_inv`; KLinearFP8
    keeps the reference's constructor / load contract (linear.py:388-435) and refuses anything but a CUDA device (no CPU fallback)."""
    import torch
    from safetensors.torch import save_file
    from ktransformers_b200.operators.linear import KLinearFP8, LINEAR_MAP
    from ktransformers_b200.util.custom_loader import GGUFLoader, ModelLoaderFactory, SafeTensorLoader
    w = torch.randn(256, 128).to(torch.float8_e4m3fn)
    s = torch.rand(2, 1)
    save_file({"blk.q_proj.weight": w, "blk.q_proj.weight_scale_inv": s}, str(tmp_path / "a.safetensors"))
    ld = ModelLoaderFactory.create_loader(str(tmp_path))
    assert isinstance(ld, SafeTensorLoader) and not isinstance(ld, GGUFLoader)
    assert ld.has_tensor("blk.q_proj.weight") and not ld.has_tensor("blk.k_proj.weight")
    assert torch.equal(ld.load_tensor("blk.q_proj.weight").view(torch.uint8), w.view(torch.uint8)) and torch.equal(ld.load_tensor("blk.q_proj.weight_scale_inv"), s)
    with pytest.raises(KeyError):
        ld.load_tensor("blk.k_proj.weight")
    with pytest.raises(FileNotFoundError):
        ModelLoaderFactory.create_loader(str(tmp_path / "nothing_here"))
    lin = LINEAR_MAP["KLinearFP8"]("blk.q_proj", ld, None, torch.nn.Linear(128, 256, bias=False, device="meta"), device="cuda")
    assert isinstance(lin, KLinearFP8) and lin.block_size == 128 and (lin.in_features, lin.out_features) == (128, 256)
    with pytest.raises(AssertionError):
        lin.load(device="cpu")
    with pytest.raises(Exception):
        lin.forward(torch.zeros(1, 128))           # Not Loaded


def test_hybrid_safetensors_serve_the_gguf_loader_surface(tmp_path):
    """The FP8 + GGUF hybrid of archive/merge_tensors (custom_loader.py:114-250): raw ggml expert blocks + scalar `.ggml_type`
    under GGUF names, router tensors under GGUF names, FP8 linears under HF names — read through the calls the operators make."""
    import torch
    from safetensors.torch import save_file
    from ktransformers_b200.util.custom_loader import SafeTensorLoader
    E, nbytes = 4, 144 * 8
    raw = {n: torch.randint(0, 255, (E, nbytes), dtype=torch.uint8) for n in ("gate", "up", "down")}
    tensors = {f"blk.1.ffn_{n}_exps.weight": raw[n] for n in raw}
    tensors.update({f"blk.1.ffn_{n}_exps.ggml_type": torch.tensor(12 if n != "down" else 14) for n in raw})
    tensors["blk.1.ffn_gate_inp.weight"] = torch.randn(E, 64)
    tensors["blk.1.exp_probs_b.bias"] = torch.randn(E)
    tensors["model.layers.1.mlp.shared_experts.up_proj.weight"] = torch.randn(128, 128).to(torch.float8_e4m3fn)
    tensors["model.layers.1.mlp.shared_experts.up_proj.weight_scale_inv"] = torch.rand(1, 1)
    save_file(tensors, str(tmp_path / "hybrid.safetensors"))
    ld = SafeTensorLoader(str(tmp_path))
    key = "model.layers.1.mlp.experts"
    assert ld.has_tensor(key + ".ffn_gate_exps.weight") and ld.has_tensor("blk.1.ffn_down_exps.weight")
    assert ld.get_ggml_type(key + ".ffn_down_exps.weight") == 14 and ld.get_ggml_type("blk.1.ffn_up_exps.weight") == 12
    assert np.array_equal(ld.get_mmap_tensor(key + ".ffn_up_exps.weight"), raw["up"].numpy().reshape(-1))
    ex = ld.load_experts(key)
    assert ex["gate_type"] == 12 and ex["down_type"] == 14 and np.array_equal(ex["down"], raw["down"].numpy().reshape(-1))
    g = ld.load_gate("model.layers.1.mlp.gate")
    assert torch.equal(g["weight"], tensors["blk.1.ffn_gate_inp.weight"]) and torch.equal(g["e_score_correction_bias"], tensors["blk.1.exp_probs_b.bias"])
    assert ld.load_gguf_tensor("model.layers.1.mlp.gate.weight", target_dtype=torch.float32).shape == (E, 64)
    with pytest.raises(KeyError):
        ld.get_ggml_type("model.layers.1.mlp.shared_experts.up_proj.weight")      # an FP8 linear, not raw ggml blocks
    with pytest.raises(NotImplementedError):
        ld.load_gguf_tensor("model.layers.1.mlp.shared_experts.up_proj.weight")
    with pytest.raises(ValueError):
        ld.load_experts("model.layers.7.mlp.experts")
