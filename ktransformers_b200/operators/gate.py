"""MoE router operators.  API mirror of archive/ktransformers/operators/gate.py:

    KMoEGateBase  :23-89   load_weights(weight, e_score_correction_bias) contract
    KMoEGate      :91-127  the reference delegates to the torch MoEGate.forward (≈10 ATen kernels)
    KMoEGateB200  the same routing as two sm_90a kernels (ktb200_moe_gate_forward): fp32 GEMV +
                  warp-shuffle grouped top-k; ids are bit-exact vs torch up to fp32 summation-order ties.
"""
from __future__ import annotations

import ctypes as C

import torch
from torch import nn

from .. import native
from ..util.custom_gguf import TORCH_TO_GGML_HIDDEN
from .base_operator import BaseInjectedModule

_SCORING = {"sigmoid": 0, "softmax": 1}
_TOPK = {"noaux_tc": 0, "greedy": 1, "group_limited_greedy": 2}


class KMoEGateBase:
    def __init__(self, key, gguf_loader, config, orig_module, device: str = "cuda", **kwargs):
        self.key = key
        self.gguf_loader = gguf_loader
        self.config = config
        self.device = device
        self.orig_module = orig_module

    def load_weights(self, override_key=None, device: str = "cpu"):
        keys = override_key if override_key is not None else [self.key]
        for key in keys:
            if self.gguf_loader.has_tensor(key + ".weight"):
                res = {"weight": self.gguf_loader.load_gguf_tensor(key + ".weight", device=device, target_dtype=torch.float32)}
                if self.gguf_loader.has_tensor(key + ".e_score_correction_bias"):
                    res["e_score_correction_bias"] = self.gguf_loader.load_gguf_tensor(key + ".e_score_correction_bias", device=device, target_dtype=torch.float32)
                return res
        raise ValueError(f"Experts {keys} not found in gguf_loader")


class KMoEGate(BaseInjectedModule, KMoEGateBase):
    """Reference behaviour: torch MoEGate.forward on the loaded weights."""

    def __init__(self, key, gguf_loader, config, orig_module=None, generate_device: str = "cuda", prefill_device: str = "cuda", **kwargs):
        BaseInjectedModule.__init__(self, key, gguf_loader, config, orig_module, prefill_device, generate_device, **kwargs)
        KMoEGateBase.__init__(self, key, gguf_loader, config, orig_module, generate_device, **kwargs)

    def forward(self, hidden_states):
        return self.orig_module.forward(hidden_states)

    def load(self, w=None, device: str | None = None):
        device = device or self.device
        if w is None:
            w = self.load_weights(device=device)
        if not isinstance(w, dict):
            raise ValueError("Invalid weight type")
        self.orig_module.weight = nn.Parameter(w["weight"].to(device), requires_grad=False)
        if "e_score_correction_bias" in w:
            self.orig_module.e_score_correction_bias = nn.Parameter(w["e_score_correction_bias"].to(device), requires_grad=False)

    def unload(self):
        self.orig_module.weight = None
        if hasattr(self.orig_module, "e_score_correction_bias"):
            self.orig_module.e_score_correction_bias = None


class KMoEGateB200(KMoEGate):
    """Same interface, routing done by libktb200 on the GPU (no torch ops on the decode path).

    The router's partial-sum scratch is per device and grow-only, and it cannot grow inside a CUDA graph capture: before
    capturing a forward, run one eager forward of at least as many tokens (bsz * q_len) on that device, or the captured
    call raises KTB200Error (KTB200_ESTATE) naming that warm-up."""

    def load(self, w=None, device: str | None = None):
        native.lib()  # fail loudly without the CUDA library
        super().load(w, device)
        m = self.orig_module
        self._w = m.weight.data.to(torch.float32).contiguous()
        b = getattr(m, "e_score_correction_bias", None)
        self._b = b.data.to(torch.float32).contiguous() if b is not None else None

    def forward(self, hidden_states, bsz_tensor=None):
        m = self.orig_module
        x = hidden_states.reshape(-1, hidden_states.shape[-1]).contiguous()
        n = x.shape[0]
        idx = torch.empty((n, m.top_k), dtype=torch.int64, device=x.device)
        wt = torch.empty((n, m.top_k), dtype=torch.float32, device=x.device)
        cfg = native.GateConfig(m.n_routed_experts, x.shape[1], m.top_k, m.n_group or 1, m.topk_group or 1,
                                _SCORING[m.scoring_func], _TOPK[m.topk_method], int(bool(m.norm_topk_prob)),
                                float(m.routed_scaling_factor), self._w.data_ptr(),
                                self._b.data_ptr() if self._b is not None else None, TORCH_TO_GGML_HIDDEN[x.dtype])
        native.check(native.lib().ktb200_moe_gate_forward(
            C.byref(cfg), n, x.data_ptr(), idx.data_ptr(), wt.data_ptr(), None,
            bsz_tensor.data_ptr() if bsz_tensor is not None else None, torch.cuda.current_stream(x.device).cuda_stream))
        return idx, wt
