"""`KTMoEWrapper` front door for the H100 experts (SURVEY §8f rank 1).

API mirror of kt-kernel's factory (kt-kernel/python/experts.py:72-262) and its inference base class
(kt-kernel/python/experts_base.py:227-544): same constructor arguments, `load_weights(physical_to_logical_map_cpu)`,
`load_weights_from_tensors(...)`, `submit_forward / sync_forward / forward(hidden_states, topk_ids, topk_weights,
cuda_stream)`, the capture-batch-size helpers.  What changes underneath:

  * `method="B200_GGUF"`: the layer's GGUF expert tensors (`blk.L.ffn_{gate,up,down}_exps.weight`, any K-quant the
    sm_90a kernels take, or IQ1_S / IQ1_M / IQ2_XXS / IQ2_XS / IQ2_S / IQ3_XXS / IQ3_S) are uploaded as raw blocks and consumed on the GPU through the C-ABI (`ktb200_moe_*`);
    there is no CPU worker pool, so `cpuinfer_threads`, `threadpool_count`, `numa_nodes`, `cpu_save` are accepted and
    ignored, and `submit_forward` launches on `cuda_stream` while `sync_forward` only hands back the (stream-ordered)
    output buffer — the two names keep their meaning for callers such as SGLang's KTEPWrapperMethod.
  * `gpu_experts_mask[i] = True` means, as in the reference, "expert i is served by somebody else": those ids are
    skipped (the reference's should_skip_expert, operators/common.hpp:255-258).
  * `physical_to_logical_map_cpu[p]` = logical expert stored in physical slot p (EPLB): the upload permutes the experts
    accordingly, exactly like `load_weights_task(physical_to_logical_map_ptr)` (ext_bindings.cpp:447-471).
  * `method="B200_RAWINT4"`: kt-kernel's RAWINT4 — the compressed-tensors "pack-quantized" experts Kimi-K2 ships
    (symmetric INT4, group 32, bf16 scales, `<key>.{e}.{gate,up,down}_proj.{weight_packed,weight_scale,weight_shape}` in a
    safetensors directory).  The packed words and scales are uploaded and converted once on the GPU
    (`ktb200_rawint4_pack`); decode runs W4A16 on the sm_90a kernels (no activation quantisation).
  * deferred experts (`max_deferred_experts_per_token`) have no purpose without a CPU/GPU overlap: must be 0 / None.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import List, Optional

import numpy as np
import torch

from .native import RAWINT4_G32
from .operators.experts import KExpertsB200
from .util.custom_gguf import GGML_NAMES, B200_ROUTED_LOAD_TYPES
from .util.custom_loader import ModelLoaderFactory

B200_METHODS = frozenset(["B200_GGUF", "B200_RAWINT4"])


class KTMoEWrapper:
    _capture_batch_sizes: List[int] = []
    _loaders: dict = {}     # weight_path -> loader (a GGUF directory is parsed once)

    def __init__(self, layer_idx: int, num_experts: int, num_experts_per_tok: int, hidden_size: int, moe_intermediate_size: int,
                 gpu_experts_mask: Optional[torch.Tensor], cpuinfer_threads: int = 0, threadpool_count: int = 0,
                 weight_path: str = "", chunked_prefill_size: int = 1024, cpu_save: bool = False,
                 max_deferred_experts_per_token: Optional[int] = None, method: str = "B200_GGUF",
                 numa_nodes: Optional[List[int]] = None, mode: str = "inference", device: str = "cuda",
                 key_template: str = "model.layers.{layer}.mlp.experts", dtype: torch.dtype = torch.bfloat16, **kwargs):
        if mode != "inference":
            raise NotImplementedError("KTMoEWrapper (H100): only mode='inference' (SFT is out of scope, DESIGN.md §6)")
        if method not in B200_METHODS:
            raise NotImplementedError(f"Unsupported method: {method}. Supported methods: {sorted(B200_METHODS)}")
        if max_deferred_experts_per_token:
            raise ValueError("deferred experts overlap a CPU backend with the GPU; the H100 backend has nothing to defer")
        if num_experts <= 0 or num_experts_per_tok <= 0 or num_experts_per_tok > num_experts:
            raise ValueError("num_experts / num_experts_per_tok out of range")
        self.layer_idx, self.num_experts, self.num_experts_per_tok = layer_idx, num_experts, num_experts_per_tok
        self.hidden_size, self.moe_intermediate_size = hidden_size, moe_intermediate_size
        self.weight_path, self.chunked_prefill_size, self.method, self.device = weight_path, int(chunked_prefill_size), method, device
        if gpu_experts_mask is None:
            self.gpu_experts_mask = torch.zeros(num_experts, dtype=torch.bool)
        else:
            if gpu_experts_mask.numel() != num_experts:
                raise ValueError("gpu_experts_mask must have num_experts entries")
            self.gpu_experts_mask = gpu_experts_mask.to(dtype=torch.bool, device="cpu").clone()
        self.num_gpu_experts = int(self.gpu_experts_mask.sum().item())
        self.key = key_template.format(layer=layer_idx)
        self._mask_dev = None
        self._out = None
        cfg = SimpleNamespace(num_experts_per_tok=num_experts_per_tok, hidden_size=hidden_size,
                              moe_intermediate_size=moe_intermediate_size, hidden_act="silu")
        self.moe = KExpertsB200(self.key, None, cfg, num_experts, device=device, max_tokens=max(self.chunked_prefill_size, 1), hidden_dtype=dtype)

    # ------------------------------------------------------------------------------------------ weights
    @staticmethod
    def _permute(raw, num_experts: int, p2l: Optional[torch.Tensor]):
        a = raw if isinstance(raw, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(raw)).view(np.uint8).reshape(-1))
        a = a.reshape(num_experts, -1)
        if p2l is not None:
            idx = p2l.to(dtype=torch.long, device=a.device).reshape(-1)
            if idx.numel() != num_experts or sorted(idx.tolist()) != list(range(num_experts)):
                raise ValueError("physical_to_logical_map must be a permutation of range(num_experts)")
            a = a.index_select(0, idx)
        return a.reshape(-1)

    def load_weights(self, physical_to_logical_map_cpu: Optional[torch.Tensor] = None):
        ld = KTMoEWrapper._loaders.get(self.weight_path)
        if ld is None:
            ld = KTMoEWrapper._loaders[self.weight_path] = ModelLoaderFactory.create_loader(self.weight_path)
        if self.method == "B200_RAWINT4":
            if not hasattr(ld, "load_experts"):
                raise ValueError(f"B200_RAWINT4 reads compressed-tensors safetensors; {self.weight_path} is not a safetensors directory")
            w = ld.load_experts(self.key)
            if w.get("gate_type") != RAWINT4_G32:
                raise ValueError(f"B200_RAWINT4: the experts of {self.key} are not compressed-tensors INT4 tensors")
            self._load_rawint4(w, physical_to_logical_map_cpu)
            return
        names = {n: f"{self.key}.ffn_{n}_exps.weight" for n in ("gate", "up", "down")}
        types = {n: int(ld.get_ggml_type(names[n])) for n in names}
        self._load({n: ld.get_mmap_tensor(names[n]) for n in names}, types, physical_to_logical_map_cpu)

    def load_weights_from_tensors(self, gate_proj, up_proj, down_proj, physical_to_logical_map_cpu=None, ggml_types=None,
                                  gate_scale=None, up_scale=None, down_scale=None):
        """The reference quantises bf16/fp16 tensors online here; this backend takes tensors that ARE quantised already:
        B200_GGUF: ggml blocks (uint8, `[E, rows, blocks * block_bytes]`) together with `ggml_types=(gate, up, down)`;
        B200_RAWINT4: compressed-tensors `weight_packed` (int32 `[E, rows, cols/8]`) as gate/up/down_proj and
        `weight_scale` (bfloat16 `[E, rows, cols/32]`) as gate/up/down_scale."""
        if self.method == "B200_RAWINT4":
            if gate_scale is None or up_scale is None or down_scale is None:
                raise ValueError("B200_RAWINT4: gate_scale, up_scale and down_scale (bfloat16 weight_scale tensors) are required")
            if ggml_types is not None:
                raise ValueError("B200_RAWINT4: ggml_types does not apply to compressed-tensors INT4 weights")
            self._load_rawint4({"gate": gate_proj, "up": up_proj, "down": down_proj, "gate_scale": gate_scale, "up_scale": up_scale,
                                "down_scale": down_scale}, physical_to_logical_map_cpu)
            return
        if any(t is not None for t in (gate_scale, up_scale, down_scale)):
            raise ValueError("gate/up/down_scale belong to method='B200_RAWINT4'")
        if ggml_types is None or any(t.dtype != torch.uint8 for t in (gate_proj, up_proj, down_proj)):
            raise NotImplementedError("online quantisation to K-quants is not built: pass raw ggml blocks (uint8) and ggml_types=(g, u, d)")
        self._load({"gate": gate_proj, "up": up_proj, "down": down_proj},
                   dict(zip(("gate", "up", "down"), (int(t) for t in ggml_types))), physical_to_logical_map_cpu)

    def _load_rawint4(self, t, p2l):
        w = {}
        for n in ("gate", "up", "down", "gate_scale", "up_scale", "down_scale"):
            a = torch.as_tensor(t[n])
            if a.dim() != 3 or a.shape[0] != self.num_experts:
                raise ValueError(f"B200_RAWINT4: {n} must be [num_experts={self.num_experts}, rows, cols], got {tuple(a.shape)}")
            w[n] = self._permute(a, self.num_experts, p2l).reshape(a.shape)
        w.update(gate_type=RAWINT4_G32, up_type=RAWINT4_G32, down_type=RAWINT4_G32)
        self._finish_load(w)

    def _load(self, raw, types, p2l):
        for t in types.values():
            if GGML_NAMES.get(t) not in B200_ROUTED_LOAD_TYPES:
                raise ValueError(f"ggml type {GGML_NAMES.get(t, t)} is not supported by the sm_90a kernels")
        w = {n: self._permute(raw[n], self.num_experts, p2l) for n in ("gate", "up", "down")}
        w.update(gate_type=types["gate"], up_type=types["up"], down_type=types["down"])
        self._finish_load(w)

    def _finish_load(self, w):
        self.moe.load(w, device=self.device)
        dt = {0: torch.float32, 1: torch.float16, 30: torch.bfloat16}[self.moe.hidden_type]
        self._out = torch.zeros((self.moe.max_tokens, self.hidden_size), dtype=dt, device=self.device)
        self._mask_dev = self.gpu_experts_mask.to(self.device) if self.num_gpu_experts else None

    # ------------------------------------------------------------------------------------------ forward
    def submit_forward(self, hidden_states: torch.Tensor, topk_ids: torch.Tensor, topk_weights: torch.Tensor, cuda_stream=None):
        if self._out is None:
            raise RuntimeError("Not Loaded")
        x = hidden_states.view(-1, hidden_states.shape[-1])
        if x.shape[0] > self._out.shape[0]:
            raise ValueError(f"batch {x.shape[0]} exceeds chunked_prefill_size {self._out.shape[0]}")
        stream = torch.cuda.ExternalStream(int(cuda_stream)) if isinstance(cuda_stream, int) and cuda_stream else (cuda_stream or torch.cuda.current_stream(x.device))
        with torch.cuda.stream(stream):
            # the id cast and the gpu_experts_mask masking are kernels too: they run on the SAME stream as the expert kernels, so a
            # caller-supplied stream other than the current one never reads ids that are still being written
            ids = topk_ids.view(x.shape[0], -1).to(torch.int64)
            if self._mask_dev is not None:
                valid = (ids >= 0) & (ids < self.num_experts)
                masked = self._mask_dev[ids.clamp(0, self.num_experts - 1)] & valid
                ids = torch.where(masked, torch.full_like(ids, -1), ids)
            self.moe._launch(x, ids, topk_weights.view(x.shape[0], -1), self._out[: x.shape[0]])
        self._pending = x.shape[0]

    def sync_forward(self, hidden_states: torch.Tensor, cuda_stream=None) -> torch.Tensor:
        n = hidden_states.view(-1, hidden_states.shape[-1]).shape[0]
        if getattr(self, "_pending", None) is None:
            raise RuntimeError("sync_forward without a pending submit_forward")
        if n != self._pending:
            raise ValueError(f"sync_forward for {n} tokens, but {self._pending} were submitted")
        self._pending = None
        return self._out[:n]          # ordered on cuda_stream behind the launches of submit_forward

    def forward(self, hidden_states, topk_ids, topk_weights, cuda_stream=None) -> torch.Tensor:
        self.submit_forward(hidden_states, topk_ids, topk_weights, cuda_stream)
        return self.sync_forward(hidden_states, cuda_stream)

    # ------------------------------------------------------------------------------------------ helpers of the reference API
    @staticmethod
    def set_capture_batch_sizes(capture_bs: List[int]):
        KTMoEWrapper._capture_batch_sizes = sorted(int(b) for b in capture_bs)

    @staticmethod
    def get_capture_batch_sizes() -> List[int]:
        return list(KTMoEWrapper._capture_batch_sizes)

    @staticmethod
    def clear_buffer_cache():
        KTMoEWrapper._loaders.clear()
