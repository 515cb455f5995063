"""Dense-linear operators.  API mirror of archive/ktransformers/operators/linear.py:

    KLinearBase          :57-155   ctor / load_weight / load / unload contract
    KLinearB200          replaces KLinearMarlin (:595-721): the raw GGUF blocks stay in HBM and are
                         consumed directly by the sm_90a integer GEMV (no dequant -> 4-bit g64
                         re-quantisation, linear.py:664-666); arithmetic equals the reference's CPU
                         Linear (operators/llamafile/linear.cpp:37-63).
    KLinearTorch         :158-216  dequantised weight + torch matmul
    LINEAR_MAP           :896-904
    KTransformersLinear  :906-983  prefill / generate switch
"""
from __future__ import annotations

import ctypes as C
from abc import ABC, abstractmethod

import numpy as np
import torch
from torch import nn

from .. import native
from ..util.custom_gguf import GGML_NAMES, TORCH_TO_GGML_HIDDEN, B200_WEIGHT_TYPES
from ..util.utils import InferenceState
from .base_operator import BaseInjectedModule

_GGML_TO_TORCH = {0: torch.float32, 1: torch.float16, 30: torch.bfloat16}


class KLinearBase(ABC):
    def __init__(self, key, gguf_loader, config, orig_module: nn.Module = None, device: str = "cuda", **kwargs):
        super().__init__()
        self.key = key
        self.gguf_loader = gguf_loader
        self.device = device
        self.config = config
        self.has_bias = False
        self.dtype = torch.get_default_dtype()
        if orig_module is not None:
            self.in_features = orig_module.in_features
            self.out_features = orig_module.out_features
        else:
            shape = self.gguf_loader.tensor_info[key + ".weight"]["shape"]
            if len(shape) == 1:
                print("Warning: orig_module is not set, but has in_features or out_features equals to 1, can't get in_features and out_features from GGUF")
            self.in_features, self.out_features = shape[0], shape[1]
        self.loaded = False

    @abstractmethod
    def forward(self, x: torch.Tensor, bsz_tensor: torch.Tensor = None) -> torch.Tensor:
        ...

    def load_weight(self, override_key=None, device: str | None = None):
        keys = override_key if override_key is not None else [self.key]
        for key in keys:
            if self.gguf_loader.has_tensor(key + ".weight"):
                w = self.gguf_loader.load_gguf_tensor(key + ".weight", device=device)
                if self.gguf_loader.has_tensor(key + ".bias"):
                    return nn.Parameter(w, requires_grad=False), nn.Parameter(self.gguf_loader.load_gguf_tensor(key + ".bias", device=device), requires_grad=False)
                return nn.Parameter(w, requires_grad=False)
            raise FileNotFoundError(f"Weight file not found for key {key}")

    @abstractmethod
    def load(self, w=None, device: str | None = "cuda"):
        ...

    @abstractmethod
    def unload(self):
        ...


class KLinearTorch(KLinearBase):
    def __init__(self, key, gguf_loader, config, orig_module=None, device: str = "cuda", **kwargs):
        super().__init__(key, gguf_loader, config, orig_module, device, **kwargs)
        self.weight = None
        self.bias = None

    def forward(self, x: torch.Tensor, bsz_tensor: torch.Tensor = None, **kwargs) -> torch.Tensor:
        dtype, out_device = x.dtype, x.device
        x = x.to(device=self.weight.device, dtype=self.dtype)
        y = torch.matmul(x, self.weight)
        if self.has_bias:
            y = y + self.bias
        return y.to(dtype=dtype, device=out_device)

    def load(self, w=None, device: str | None = None):
        if self.loaded:
            return
        device = device or self.device
        if w is None:
            w = self.load_weight(device=device)
        if isinstance(w, tuple):
            weight, bias = w
            self.bias = bias.data.to(device=device, dtype=self.dtype)
            self.has_bias = True
        else:
            weight = w
        self.weight = weight.data.to(dtype=self.dtype).view(self.out_features, self.in_features).T.to(device)
        self.loaded = True

    def unload(self):
        self.weight = None
        self.bias = None
        self.loaded = False


class KLinearB200(KLinearBase):
    """GGUF-native linear: y = x · Wᵀ with W kept as raw ggml blocks in HBM.

    Calls of `prompt_min` tokens or more (ktb200_linear_prompt_min: a threshold per weight type and shape, 0 for types the
    tiled GEMM does not take) run ktb200_linear_forward_prompt, which reads each weight once per chunk of up to 2048 tokens;
    shorter calls run the decode GEMVs.  So with Q4_K / Q6_K weights, KTransformersLinear(generate_op="KLinearB200",
    prefill_op=None) serves both phases from one resident copy.  The prompt route's activation scratch is a grow-only
    per-device arena: before capturing a prompt-sized call in a CUDA graph, run one eager prompt-sized call (any length of
    `prompt_min` tokens or more) of the largest in_features on the device."""

    def __init__(self, key, gguf_loader, config, orig_module=None, device: str = "cuda", max_tokens: int = 1024, **kwargs):
        super().__init__(key, gguf_loader, config, orig_module, device, **kwargs)
        self.handle = None
        self.weight = None       # raw block bytes on the device (modeling code may touch `.weight`)
        self.bias = None
        self.max_tokens = max_tokens
        self.prompt_min = 0

    def load(self, w=None, device: str | None = None):
        if self.loaded:
            return
        device = device or self.device
        assert "cuda" in str(device).lower(), "KLinearB200 can only be loaded on a CUDA device"
        lib = native.lib()
        ld = self.gguf_loader
        if w is None:
            raw, ggml_type = ld.get_mmap_tensor(self.key + ".weight"), int(ld.get_ggml_type(self.key + ".weight"))
            if ld.has_tensor(self.key + ".bias"):
                self.bias = ld.load_gguf_tensor(self.key + ".bias", device=device, target_dtype=torch.float32).contiguous()
                self.has_bias = True
        else:  # (raw_bytes, ggml_type[, bias])
            raw, ggml_type = w[0], int(w[1])
            if len(w) > 2 and w[2] is not None:
                self.bias = w[2].to(device=device, dtype=torch.float32).contiguous()
                self.has_bias = True
        if GGML_NAMES.get(ggml_type) not in B200_WEIGHT_TYPES:
            raise ValueError(f"KLinearB200: ggml type {GGML_NAMES.get(ggml_type, ggml_type)} is not supported by the sm_90a kernels")
        raw = raw if isinstance(raw, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(raw)).view(np.uint8).reshape(-1))
        self.weight = raw.reshape(-1).to(device).contiguous()
        self.ggml_type = ggml_type
        self.hidden_type = TORCH_TO_GGML_HIDDEN.get(self.dtype, 30)
        dev = torch.device(device)
        self.dev_index = dev.index if dev.index is not None else torch.cuda.current_device()
        h = C.c_void_p()
        native.check(lib.ktb200_linear_create(self.in_features, self.out_features, self.weight.data_ptr(), ggml_type,
                                              self.hidden_type, self.max_tokens, self.dev_index, C.byref(h)))
        self.handle = h
        native.check(lib.ktb200_linear_load_weights(self.handle, torch.cuda.current_stream(dev).cuda_stream))
        self.prompt_min = lib.ktb200_linear_prompt_min(self.handle)
        self.loaded = True

    def forward(self, x: torch.Tensor, bsz_tensor: torch.Tensor = None, **kwargs) -> torch.Tensor:
        if self.handle is None:
            raise native.KTB200Error("Not Loaded")
        orig_shape, in_dtype = x.shape, x.dtype
        x2 = x.reshape(-1, x.shape[-1]).to(_GGML_TO_TORCH[self.hidden_type]).contiguous()
        out = torch.empty((x2.shape[0], self.out_features), dtype=x2.dtype, device=x2.device)
        prompt = self.prompt_min > 0 and x2.shape[0] >= self.prompt_min
        lib = native.lib()
        native.check((lib.ktb200_linear_forward_prompt if prompt else lib.ktb200_linear_forward)(
            self.handle, x2.shape[0], x2.data_ptr(), out.data_ptr(), self.bias.data_ptr() if self.has_bias else None,
            bsz_tensor.data_ptr() if bsz_tensor is not None else None, torch.cuda.current_stream(x2.device).cuda_stream))
        return out.reshape(*orig_shape[:-1], self.out_features).to(in_dtype)

    def unload(self):
        if self.handle is not None:
            native.lib().ktb200_linear_destroy(self.handle)
            self.handle = None
        self.weight = None
        self.bias = None
        self.loaded = False

    def __del__(self):
        try:
            self.unload()
        except Exception:
            pass


class KLinearFP8(KLinearBase):
    """DeepSeek-V3's native FP8 checkpoints: e4m3 weight [out][in] + fp32 `weight_scale_inv` per 128 x 128 block, activations
    quantised per token and 128 values inside the kernel.  Same contract as the reference's KLinearFP8 (operators/linear.py:388-435:
    `load(w=(weight, weight_scale_inv))`, `forward(x, bsz_tensor)`), which runs Triton's act_quant + fp8_gemm; here
    `ktb200_fp8_linear_forward` (TMA -> e4m3 widened to fp16 in registers -> fp16 wgmma, csrc/fp8_linear.cu).  Decode batches
    stream the weights once per 16 tokens; prompts (from 32, 48 or 96 tokens by shape, DESIGN.md §4.6) run a tiled GEMM that
    reads each weight once per 2048-token chunk, so `prefill_op: None` serves both phases.  The prompt route uses a grow-only
    per-device scratch arena: before capturing a CUDA graph that contains a prompt-sized call, run one such call eagerly."""

    def __init__(self, key, gguf_loader, config, orig_module=None, device: str = "cuda", block_size: int = 128, **kwargs):
        super().__init__(key, gguf_loader, config, orig_module, device, **kwargs)
        assert block_size == 128, "the checkpoint format fixes 128 x 128 weight blocks"
        self.block_size = block_size
        self.handle = None
        self.weight = self.weight_scale_inv = None

    def load(self, w=None, device: str | None = None):
        if self.loaded:
            return
        device = device or self.device
        assert "cuda" in str(device).lower(), "KLinearFP8 can only be loaded on a CUDA device"
        lib = native.lib()
        if w is None:
            ld = self.gguf_loader       # a SafeTensorLoader (util/custom_loader.py): `<key>.weight` (float8_e4m3fn) + `<key>.weight_scale_inv`
            w = (ld.load_tensor(self.key + ".weight"), ld.load_tensor(self.key + ".weight_scale_inv"))
        if not isinstance(w, tuple) or len(w) != 2:
            raise ValueError("Invalid weight type")                       # linear.py:427
        weight, scale = (t.data if isinstance(t, nn.Parameter) else t for t in w)
        if weight.dtype != torch.float8_e4m3fn or tuple(weight.shape) != (self.out_features, self.in_features):
            raise ValueError(f"KLinearFP8: weight must be float8_e4m3fn [{self.out_features}][{self.in_features}], got {weight.dtype} {tuple(weight.shape)}")
        want = ((self.out_features + 127) // 128, self.in_features // 128)
        if tuple(scale.shape) != want:
            raise ValueError(f"KLinearFP8: weight_scale_inv must be {want}, got {tuple(scale.shape)}")
        self.weight = weight.to(device).contiguous()
        self.weight_scale_inv = scale.to(device=device, dtype=torch.float32).contiguous()
        self.hidden_type = TORCH_TO_GGML_HIDDEN.get(self.dtype, 30)
        dev = torch.device(device)
        self.dev_index = dev.index if dev.index is not None else torch.cuda.current_device()
        h = C.c_void_p()
        native.check(lib.ktb200_fp8_linear_create(self.in_features, self.out_features, self.weight.data_ptr(), self.weight_scale_inv.data_ptr(),
                                                  self.hidden_type, self.dev_index, C.byref(h)))
        self.handle = h
        self.loaded = True

    def forward(self, x: torch.Tensor, bsz_tensor: torch.Tensor = None, **kwargs) -> torch.Tensor:
        if self.handle is None:
            raise native.KTB200Error("Not Loaded")
        orig_shape, in_dtype = x.shape, x.dtype
        x2 = x.reshape(-1, x.shape[-1]).to(_GGML_TO_TORCH[self.hidden_type]).contiguous()
        out = torch.empty((x2.shape[0], self.out_features), dtype=x2.dtype, device=x2.device)
        native.check(native.lib().ktb200_fp8_linear_forward(self.handle, x2.shape[0], x2.data_ptr(), out.data_ptr(),
                                                            bsz_tensor.data_ptr() if bsz_tensor is not None else None,
                                                            torch.cuda.current_stream(x2.device).cuda_stream))
        return out.reshape(*orig_shape[:-1], self.out_features).to(in_dtype)

    def unload(self):
        if self.handle is not None:
            native.lib().ktb200_fp8_linear_destroy(self.handle)
            self.handle = None
        self.weight = self.weight_scale_inv = None
        self.loaded = False

    def __del__(self):
        try:
            self.unload()
        except Exception:
            pass


LINEAR_MAP = {
    "KLinearB200": KLinearB200,
    "KLinearFP8": KLinearFP8,
    "KLinearTorch": KLinearTorch,
}


class KTransformersLinear(BaseInjectedModule, KLinearBase):
    def __init__(self, key, gguf_loader, config, orig_module, generate_device: str = "cuda",
                 generate_op: str | None = "KLinearB200", prefill_device: str = "cuda",
                 prefill_op: str | None = "KLinearTorch", **kwargs):
        BaseInjectedModule.__init__(self, key, gguf_loader, config, orig_module, prefill_device, generate_device, **kwargs)
        KLinearBase.__init__(self, key, gguf_loader, config, orig_module, generate_device, **kwargs)
        prefill_op = None if prefill_op == "None" else prefill_op        # YAML spells it as a string
        generate_op = None if generate_op == "None" else generate_op
        for op in (prefill_op, generate_op):
            assert op is None or op in LINEAR_MAP, f"linear_type {op} not supported"
        self.prefill_linear = LINEAR_MAP[prefill_op](key, gguf_loader, config, orig_module, prefill_device, **kwargs) if prefill_op else None
        self.generate_linear = LINEAR_MAP[generate_op](key, gguf_loader, config, orig_module, generate_device, **kwargs) if generate_op else None
        self.mode = InferenceState.UNLOAD

    def forward(self, x, bsz_tensor=None):
        if self.mode == InferenceState.PREFILL and self.prefill_linear is not None:
            return self.prefill_linear.forward(x, bsz_tensor)
        assert self.generate_linear is not None, "generate linear is not initialized"
        return self.generate_linear.forward(x, bsz_tensor)

    def load(self, w=None, mode: InferenceState = InferenceState.GENERATE):
        mode = mode or InferenceState.GENERATE
        if mode == InferenceState.PREFILL and self.prefill_linear is None:
            # `prefill_op: None`: the generate linear serves both phases (GPU-resident weights, nothing to swap)
            self.generate_linear.load(w=w)
            self.device = self.generate_linear.device
            self.weight = self.generate_linear.weight
        elif mode == InferenceState.PREFILL:
            if self.generate_linear is not None:
                self.generate_linear.unload()
            self.prefill_linear.load(w=w)
            self.device = self.prefill_linear.device
            self.weight = self.prefill_linear.weight
        elif mode == InferenceState.GENERATE:
            if self.prefill_linear is not None:
                self.prefill_linear.unload()
            self.generate_linear.load(w=w)
            self.device = self.generate_linear.device
            self.weight = self.generate_linear.weight
        elif mode == InferenceState.UNLOAD:
            self.unload()
            self.device = "cpu"
        else:
            raise ValueError("mode must be either InferenceState.GENERATE, InferenceState.PREFILL or InferenceState.UNLOAD")
        self.mode = mode

    def unload(self):
        if self.prefill_linear is not None:
            self.prefill_linear.unload()
        if self.generate_linear is not None:
            self.generate_linear.unload()
            self.device = self.generate_linear.device

    def set_inference_mode(self, mode: InferenceState):
        mode = mode or InferenceState.GENERATE
        if mode in (InferenceState.GENERATE, InferenceState.PREFILL):
            self.load(mode=mode)
        elif mode == InferenceState.UNLOAD:
            self.unload()
        else:
            raise ValueError("mode must be either InferenceState.GENERATE, InferenceState.PREFILL or InferenceState.UNLOAD")
