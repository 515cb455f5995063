"""Routed-expert operators.  API mirror of archive/ktransformers/operators/experts.py:

    KExpertsBase          :68-140    ctor/load/unload/forward/load_weights contract
    KExpertsB200          replaces KExpertsCPU (:143-435) / KExpertsMarlin (:437-559): the raw GGUF expert
                          blocks live in HBM and are consumed by the sm_90a kernels through the C-ABI
                          (include/ktb200.h: ktb200_moe_*).  No CPU hand-off: submit_for_one_decode /
                          sync_for_one_decode keep their names and stream-ordered semantics (:293-318) but
                          launch the kernels directly on torch's current stream.
    KExpertsTorch         :562-678   dequantise-then-matmul torch operator (prefill_op default)
    EXPERTS_MAP           :680-684
    KTransformersExperts  :686-757   prefill/generate switch
    KDeepseekV3MoE        :972-1012  gate -> (experts || shared_experts) -> add
    KDeepseekV2MoE        :760-800
"""
from __future__ import annotations

import ctypes as C
from abc import ABC, abstractmethod

import numpy as np
import torch
from torch import nn

from .. import native
from ..util.custom_gguf import GGML_NAMES, TORCH_TO_GGML_HIDDEN, B200_WEIGHT_TYPES, B200_EXPERT_TYPES
from ..util.utils import InferenceState
from .base_operator import BaseInjectedModule


def _stream(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


class KExpertsBase(ABC):
    def __init__(self, key, gguf_loader, config, orig_module, device: str = "cuda", **kwargs):
        self.key = key
        self.gguf_loader = gguf_loader
        self.config = config
        self.device = device

    @abstractmethod
    def forward(self, input_tensor, expert_ids, weights):
        ...

    @abstractmethod
    def load(self, w: dict | nn.Parameter | tuple | None = None, device: str = "cpu", warmup: bool = False):
        ...

    @abstractmethod
    def unload(self):
        ...

    def load_weights(self, override_key=None, device: str = "cpu"):
        """{key: {gate, up, down (raw ggml bytes, numpy), gate_type, up_type, down_type}} — same shape as
        KExpertsCPU.load_weights (experts.py:370-435)."""
        res = {}
        keys = override_key if override_key is not None else [self.key]
        for key in keys:
            ld = self.gguf_loader
            if ld.has_tensor(key + ".ffn_gate_exps.weight"):
                names = [key + f".ffn_{s}_exps.weight" for s in ("gate", "up", "down")]
                gate, up, down = (ld.get_mmap_tensor(n) for n in names)
                gt, ut, dt = (ld.get_ggml_type(n) for n in names)
            elif ld.has_tensor(key + ".ffn_down.0.weight"):
                # Mixtral-style per-expert tensors: stack (experts.py:399-416)
                n = 0
                while ld.has_tensor(f"{key}.ffn_down.{n}.weight"):
                    n += 1
                gate = np.stack([ld.get_mmap_tensor(f"{key}.ffn_gate.{i}.weight") for i in range(n)])
                up = np.stack([ld.get_mmap_tensor(f"{key}.ffn_up.{i}.weight") for i in range(n)])
                down = np.stack([ld.get_mmap_tensor(f"{key}.ffn_down.{i}.weight") for i in range(n)])
                gt, ut, dt = (ld.get_ggml_type(f"{key}.ffn_{s}.0.weight") for s in ("gate", "up", "down"))
            else:
                raise ValueError(f"Experts {key} not found in gguf_loader")
            res[key] = {"gate": gate, "up": up, "down": down, "gate_type": gt, "up_type": ut, "down_type": dt}
        return res


class KExpertsB200(KExpertsBase):
    """GPU-resident GGUF experts on the hand-written sm_90a kernels."""

    # graph-safe output buffers per device, like KExpertsCPU.output_gpu_map (experts.py:147)
    output_gpu_map: dict = {}
    MAX_TOKENS = 1024  # group_max_len of the reference config (experts.py:209)

    def __init__(self, key, gguf_loader, config, n_routed_experts, orig_module=None, device: str = "cuda",
                 out_device: str | None = None, expert_parallel_rank: int = 0, expert_parallel_size: int = 1,
                 max_tokens: int | None = None, hidden_dtype: torch.dtype | None = None, **kwargs):
        super().__init__(key, gguf_loader, config, orig_module, device, **kwargs)
        assert "cuda" in str(device).lower(), "KExpertsB200 can only be loaded on a CUDA device"
        self.n_routed_experts = n_routed_experts
        self.out_device = out_device or device
        self.ep_rank, self.ep_size = int(expert_parallel_rank), int(expert_parallel_size)
        assert n_routed_experts % self.ep_size == 0, "expert count must divide evenly across the EP group"
        self.max_tokens = int(max_tokens or KExpertsB200.MAX_TOKENS)
        self.hidden_dtype = hidden_dtype      # None: torch's default dtype at load time (the reference's behaviour)
        self.handle = None
        self.gate = self.up = self.down = None
        self._pending = None

    # ------------------------------------------------------------------------------------------
    def load(self, w: dict | None = None, device: str | None = None, warmup: bool = False):
        if self.handle is not None:
            return
        device = device or self.device
        assert "cuda" in str(device).lower(), "KExpertsB200 can only be loaded on a CUDA device"
        lib = native.lib()  # raises if the CUDA library is missing: no fallback
        if w is None:
            w = self.load_weights()[self.key]
        self.gate_type, self.up_type, self.down_type = int(w["gate_type"]), int(w["up_type"]), int(w["down_type"])
        n_i4 = sum(t == native.RAWINT4_G32 for t in (self.gate_type, self.up_type, self.down_type))
        if n_i4 not in (0, 3):
            raise ValueError("KExpertsB200: RAWINT4_G32 must be the type of all three expert tensors")
        for t in (self.gate_type, self.up_type, self.down_type) if not n_i4 else ():
            if GGML_NAMES.get(t) not in B200_EXPERT_TYPES:
                raise ValueError(f"KExpertsB200: ggml type {GGML_NAMES.get(t, t)} is not supported by the sm_90a kernels")
        E = self.n_routed_experts
        per, lo = E // self.ep_size, (E // self.ep_size) * self.ep_rank
        dev = torch.device(device)
        H, I = self.config.hidden_size, self.config.moe_intermediate_size

        def pack_rawint4(name, rows, cols):
            # compressed-tensors weight_packed int32 [E][rows][cols/8] + weight_scale bf16 [E][rows][cols/32]: the shard's
            # experts go up as staging copies and are converted into a fresh buffer; the caller's tensors are not touched
            p, s = torch.as_tensor(w[name]), torch.as_tensor(w[name + "_scale"])
            if p.dtype != torch.int32 or s.dtype != torch.bfloat16:
                raise ValueError(f"KExpertsB200: RAWINT4 {name} needs int32 weight_packed and bfloat16 weight_scale, got {p.dtype} / {s.dtype}")
            if tuple(p.shape) != (E, rows, cols // 8) or tuple(s.shape) != (E, rows, cols // 32):
                raise ValueError(f"KExpertsB200: RAWINT4 {name} shapes {tuple(p.shape)} / {tuple(s.shape)}, expected "
                                 f"{(E, rows, cols // 8)} / {(E, rows, cols // 32)}")
            p_d = p[lo:lo + per].to(dev).contiguous()
            s_d = s[lo:lo + per].to(dev).contiguous()
            out = torch.empty(per * rows * cols // 256 * 144, dtype=torch.uint8, device=dev)
            with torch.cuda.device(dev):
                native.check(lib.ktb200_rawint4_pack(p_d.data_ptr(), s_d.data_ptr(), per * rows, cols, out.data_ptr(), _stream(dev)))
            return out

        def upload(a):
            a = a if isinstance(a, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(np.asarray(a)).view(np.uint8).reshape(-1))
            a = a.reshape(-1)
            nb = a.numel() // E
            sl = a[lo * nb:(lo + per) * nb]
            # load_weights re-tiles Q6_K bytes IN PLACE: never hand it memory the caller still owns
            return sl.clone() if sl.device == torch.device(device) else sl.to(device).contiguous()

        if n_i4:
            self.gate, self.up, self.down = pack_rawint4("gate", I, H), pack_rawint4("up", I, H), pack_rawint4("down", H, I)
        else:
            self.gate, self.up, self.down = upload(w["gate"]), upload(w["up"]), upload(w["down"])
        self.dev_index = dev.index if dev.index is not None else torch.cuda.current_device()
        want_dtype = self.hidden_dtype or torch.get_default_dtype()
        hidden_type = TORCH_TO_GGML_HIDDEN[want_dtype] if want_dtype in TORCH_TO_GGML_HIDDEN else 30
        self.hidden_type = hidden_type
        cfg = native.MoeConfig(per, self.config.num_experts_per_tok, self.config.hidden_size,
                               self.config.moe_intermediate_size, 64, 10, self.max_tokens,
                               int(getattr(self.config, "hidden_act", "silu") == "silu"), self.gate.data_ptr(),
                               self.up.data_ptr(), self.down.data_ptr(), self.gate_type, self.up_type, self.down_type,
                               hidden_type, lo)
        h = C.c_void_p()
        native.check(lib.ktb200_moe_create(C.byref(cfg), self.dev_index, C.byref(h)))
        self.handle = h
        native.check(lib.ktb200_moe_load_weights(self.handle, _stream(dev)))
        if warmup:
            native.check(lib.ktb200_moe_warm_up(self.handle, _stream(dev)))
        if self.out_device not in KExpertsB200.output_gpu_map:
            KExpertsB200.output_gpu_map[self.out_device] = torch.zeros(
                (self.max_tokens, self.config.hidden_size), device=self.out_device,
                dtype={0: torch.float32, 1: torch.float16, 30: torch.bfloat16}[hidden_type])

    def unload(self):
        if self.handle is not None:
            native.lib().ktb200_moe_destroy(self.handle)
            self.handle = None
        self.gate = self.up = self.down = None

    def __del__(self):
        try:
            self.unload()
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------
    def _launch(self, input_tensor, expert_ids, weights, out, bsz_tensor=None):
        if self.handle is None:
            raise native.KTB200Error("Not Loaded")
        x = input_tensor.reshape(-1, input_tensor.shape[-1])
        ids = expert_ids.reshape(x.shape[0], -1)
        if ids.dtype != torch.int64:
            ids = ids.to(torch.int64)
        w = weights.reshape(x.shape[0], -1)
        if w.dtype != torch.float32:
            w = w.to(torch.float32)
        x, ids, w = x.contiguous(), ids.contiguous(), w.contiguous()
        want = {0: torch.float32, 1: torch.float16, 30: torch.bfloat16}[self.hidden_type]
        if x.dtype != want:
            # the reference silently mis-types here (SURVEY appendix A); take the dtype from the tensor instead
            x = x.to(want)
        bsz_ptr = None
        if bsz_tensor is not None:
            assert bsz_tensor.dtype == torch.int32 and bsz_tensor.is_cuda
            bsz_ptr = bsz_tensor.data_ptr()
        native.check(native.lib().ktb200_moe_forward(self.handle, x.shape[0], ids.shape[1], ids.data_ptr(), w.data_ptr(),
                                                     x.data_ptr(), out.data_ptr(), bsz_ptr, _stream(x.device)))
        return out

    def forward(self, input_tensor, expert_ids, weights, bsz_tensor=None, cuda_graph_idx=0):
        n = input_tensor.reshape(-1, input_tensor.shape[-1]).shape[0]
        capturing = torch.cuda.is_current_stream_capturing()
        if capturing:
            out = KExpertsB200.output_gpu_map[self.out_device][:n]      # static buffer: graph-replay safe
        else:
            out = torch.empty((n, self.config.hidden_size), device=input_tensor.device,
                              dtype=KExpertsB200.output_gpu_map[self.out_device].dtype)
        self._launch(input_tensor, expert_ids, weights, out, bsz_tensor)
        return out.to(self.out_device) if str(out.device) != str(torch.device(self.out_device)) and not capturing else out

    # names and stream-ordered semantics of KExpertsCPU (experts.py:293-318); KDeepseekV3MoE's fast
    # decode branch is gated on hasattr(generate_experts, "submit_for_one_decode") (:982)
    def submit_for_one_decode(self, input_tensor, expert_ids, weights, bsz_tensor=None, cuda_graph_idx=0):
        out = KExpertsB200.output_gpu_map[self.out_device][:1]
        self._launch(input_tensor.reshape(1, -1), expert_ids.reshape(1, -1), weights.reshape(1, -1), out, bsz_tensor)
        self._pending = out

    def sync_for_one_decode(self, cuda_graph_idx=0):
        out, self._pending = self._pending, None
        return out[0]


class KExpertsTorch(KExpertsBase):
    """Dequantise-then-matmul in torch (the reference's prefill_op default, experts.py:562-678).
    Works on any device; used on CPU by the injection tests and as the long-prompt operator."""

    def __init__(self, key, gguf_loader, config, n_routed_experts, orig_module=None, device: str = "cpu", **kwargs):
        super().__init__(key, gguf_loader, config, orig_module, device, **kwargs)
        self.n_routed_experts = n_routed_experts
        self.gate = self.up = self.down = None
        self.act_fn = torch.nn.functional.silu

    def load(self, w: dict | None = None, device: str | None = None, warmup: bool = False):
        if self.gate is not None:
            return
        device = device or self.device
        ld = self.gguf_loader
        dt = torch.get_default_dtype()
        E, H, I = self.n_routed_experts, self.config.hidden_size, self.config.moe_intermediate_size
        self.gate = ld.load_gguf_tensor(self.key + ".ffn_gate_exps.weight", device=device, target_dtype=dt).view(E, I, H)
        self.up = ld.load_gguf_tensor(self.key + ".ffn_up_exps.weight", device=device, target_dtype=dt).view(E, I, H)
        self.down = ld.load_gguf_tensor(self.key + ".ffn_down_exps.weight", device=device, target_dtype=dt).view(E, H, I)

    def unload(self):
        self.gate = self.up = self.down = None

    @torch.no_grad()
    def forward(self, hidden_states_cpu, selected_experts_cpu, routing_weights_cpu, bsz_tensor=None, cuda_graph_idx=0):
        x = hidden_states_cpu.reshape(-1, hidden_states_cpu.shape[-1]).to(self.gate.device)
        ids = selected_experts_cpu.reshape(x.shape[0], -1).to(self.gate.device)
        w = routing_weights_cpu.reshape(x.shape[0], -1).to(self.gate.device)
        out = torch.zeros_like(x)
        for e in torch.unique(ids).tolist():
            if e < 0 or e >= self.n_routed_experts:
                continue
            tok, slot = torch.where(ids == e)
            cur = x[tok]
            h = self.act_fn(cur @ self.gate[e].T) * (cur @ self.up[e].T)
            y = (h @ self.down[e].T) * w[tok, slot, None].to(h.dtype)
            out.index_add_(0, tok, y.to(out.dtype))
        return out.to(hidden_states_cpu.device)


EXPERTS_MAP = {
    "KExpertsB200": KExpertsB200,
    "KExpertsTorch": KExpertsTorch,
}


class KTransformersExperts(BaseInjectedModule, KExpertsBase):
    def __init__(self, key, gguf_loader, config, orig_module, prefill_device: str = "cuda",
                 prefill_op: str | None = "KExpertsTorch", generate_device: str = "cuda",
                 generate_op: str | None = "KExpertsB200", **kwargs):
        BaseInjectedModule.__init__(self, key, gguf_loader, config, orig_module, prefill_device, generate_device, **kwargs)
        KExpertsBase.__init__(self, key, gguf_loader, config, orig_module, generate_device, **kwargs)
        n = len(orig_module)
        prefill_op = None if prefill_op == "None" else prefill_op        # YAML spells it as a string (experts.py:1287-1290)
        generate_op = None if generate_op == "None" else generate_op
        self.generate_experts = EXPERTS_MAP[generate_op](key, gguf_loader, config, n, device=generate_device, **kwargs) if generate_op else None
        self.prefill_experts = EXPERTS_MAP[prefill_op](key, gguf_loader, config, n, device=prefill_device, **kwargs) if prefill_op else None
        self.gpu_mlp_type = prefill_op
        self.cpu_mlp_type = generate_op
        self.mode = InferenceState.UNLOAD

    def load(self, w: dict = None, mode: InferenceState = None, warmup: bool = True):
        mode = mode or InferenceState.GENERATE
        if mode == InferenceState.GENERATE:
            if self.prefill_experts is not None:
                self.prefill_experts.unload()
            self.generate_experts.load(w, warmup=warmup)
            self.device = self.generate_experts.device
        elif mode == InferenceState.PREFILL:
            if self.generate_experts is not None:
                self.generate_experts.unload()
            self.prefill_experts.load(w, warmup=warmup)
            self.device = self.prefill_experts.device
        elif mode == InferenceState.UNLOAD:
            self.unload()
            self.device = self.generate_experts.device
        else:
            raise ValueError("mode must be either InferenceState.GENERATE, InferenceState.PREFILL or InferenceState.UNLOAD")
        self.mode = mode

    def unload(self):
        if self.generate_experts is not None:
            self.generate_experts.unload()
        if self.prefill_experts is not None:
            self.prefill_experts.unload()
        self.device = self.generate_experts.device

    def forward(self, input_tensor, expert_ids, weights, *args, **kwargs):
        if self.mode == InferenceState.GENERATE:
            assert self.generate_experts is not None, "generate_experts is None"
            return self.generate_experts.forward(input_tensor, expert_ids, weights, *args, **kwargs)
        if self.mode == InferenceState.PREFILL:
            assert self.prefill_experts is not None, "prefill_experts is None"
            return self.prefill_experts.forward(input_tensor, expert_ids, weights, *args, **kwargs)
        raise ValueError("load or set_inference_mode before forward")

    def set_inference_mode(self, mode: InferenceState):
        if mode == InferenceState.GENERATE:
            self.load(mode=InferenceState.GENERATE, warmup=False)
        elif mode == InferenceState.PREFILL:
            self.load(mode=InferenceState.PREFILL, warmup=False)
        elif mode == InferenceState.UNLOAD:
            self.unload()
        else:
            raise ValueError("mode must be either InferenceState.GENERATE, InferenceState.PREFILL or InferenceState.UNLOAD")


class KTransformersExpertsV2(KTransformersExperts):
    """experts.py:1273-1350: the balance-serve variant whose forward carries `bsz_tensor` (device-side live batch size) and a
    CUDA-graph slot.  With `prefill_op: None` the generate experts serve both phases (one GPU-resident KExpertsB200: per-pair
    GEMV kernels for decode batches, the grouped tensor-core path from KTB200_GROUPED_MIN tokens up)."""

    def forward(self, input_tensor, expert_ids, weights, bsz_tensor=None, cuda_graph_idx=0):
        if self.mode == InferenceState.GENERATE or (self.mode == InferenceState.PREFILL and self.prefill_experts is None):
            assert self.generate_experts is not None, "generate_experts is None"
            return self.generate_experts.forward(input_tensor, expert_ids, weights, bsz_tensor, cuda_graph_idx)
        if self.mode == InferenceState.PREFILL:
            return self.prefill_experts.forward(input_tensor, expert_ids, weights, bsz_tensor, cuda_graph_idx)
        raise ValueError("load or set_inference_mode before forward")

    def load(self, w: dict = None, mode: InferenceState = None, warmup: bool = True):
        if (mode or InferenceState.GENERATE) == InferenceState.PREFILL and self.prefill_experts is None:
            self.generate_experts.load(w, warmup=warmup)
            self.device, self.mode = self.generate_experts.device, InferenceState.PREFILL
            return
        super().load(w, mode, warmup)


class _KDeepseekMoEMixin:
    """forward shared by KDeepseekV3MoE / KDeepseekV2MoE (experts.py:760-800, 972-1012).

    Decode batches (<= 8 tokens) whose gate is a KMoEGateB200 and whose generate experts are a fully resident
    KExpertsB200 take ONE call, `ktb200_moe_block_forward`: router, routed experts and shared expert in a single
    persistent launch, bit-identical to the three-step path below (include/ktb200.h).  The shared expert for that call
    is a `ktb200_mlp` handle built once from the raw GGUF tensors `<key>.shared_experts.{gate,up,down}_proj.weight`.

    Sharded experts (expert_parallel_size > 1) need `ep_exchange` (attach_expert_parallel) and raise without it.  A step
    with one token on every rank takes the one-launch decode kernel (`ktb200_moe_ep_block_forward`); any other step
    (prompt chunks, ranks with different token counts, 0 included) takes `ktb200_moe_ep_forward_tokens` with the counts
    announced by `ep_exchange.begin_step`.
    """

    BLOCK_MAX_TOKENS = 8

    def load(self):
        """children first (base_operator.py:45-48), then the shared expert's handle for the single-launch path: handles
        are created here, never inside forward (which may be running under CUDA-graph capture)."""
        super().load()
        gen = getattr(getattr(self, "experts", None), "generate_experts", None)
        if isinstance(gen, KExpertsB200) and gen.handle is not None and self.config.n_shared_experts is not None:
            self._shared_mlp_handle(gen)

    def _block_handles(self, x, need_mlp=True):
        """(gate_cfg, moe_handle, mlp_handle_or_None) when the single-launch path applies, else None.  need_mlp=False: also
        when the block's shared expert has no ktb200_mlp handle (mlp None then; the caller runs the shared module)."""
        gate, gen = getattr(self, "gate", None), getattr(getattr(self, "experts", None), "generate_experts", None)
        if not (isinstance(gen, KExpertsB200) and gen.handle is not None and x.is_cuda):
            return None
        if gen.ep_size > 1 and getattr(self, "ep_exchange", None) is None:
            return None
        if getattr(self.experts, "mode", None) != InferenceState.GENERATE or getattr(gate, "_w", None) is None:
            return None
        m = gate.orig_module
        from .gate import _SCORING, _TOPK
        if x.dtype not in TORCH_TO_GGML_HIDDEN or TORCH_TO_GGML_HIDDEN[x.dtype] != gen.hidden_type:
            return None
        cfg = native.GateConfig(m.n_routed_experts, x.shape[-1], m.top_k, m.n_group or 1, m.topk_group or 1,
                                _SCORING[m.scoring_func], _TOPK[m.topk_method], int(bool(m.norm_topk_prob)),
                                float(m.routed_scaling_factor), gate._w.data_ptr(),
                                gate._b.data_ptr() if gate._b is not None else None, gen.hidden_type)
        mlp = None
        if self.config.n_shared_experts is not None:
            mlp = getattr(self, "_ktb_mlp", None)
            if mlp is None and need_mlp:
                return None
        return cfg, gen.handle, mlp

    def _shared_mlp_handle(self, gen):
        if getattr(self, "_ktb_mlp", None) is not None:
            return self._ktb_mlp
        ld = self.gguf_loader
        names = [f"{self.key}.shared_experts.{n}_proj.weight" for n in ("gate", "up", "down")]
        if ld is None or not all(ld.has_tensor(n) for n in names):
            return None
        try:
            types = [int(ld.get_ggml_type(n)) for n in names]
        except KeyError:      # e.g. FP8 shared experts in a hybrid safetensors file: they stay KLinearFP8 modules
            return None
        if any(GGML_NAMES.get(t) not in B200_WEIGHT_TYPES for t in types):
            return None
        dev = torch.device("cuda", gen.dev_index)
        raw = [torch.from_numpy(np.ascontiguousarray(np.asarray(ld.get_mmap_tensor(n))).view(np.uint8).reshape(-1)).to(dev) for n in names]
        inter = self.config.moe_intermediate_size * self.config.n_shared_experts
        h = C.c_void_p()
        native.check(native.lib().ktb200_mlp_create(self.config.hidden_size, inter, raw[0].data_ptr(), raw[1].data_ptr(), raw[2].data_ptr(),
                                                    types[0], types[1], types[2], gen.hidden_type, self.BLOCK_MAX_TOKENS, gen.dev_index, C.byref(h)))
        native.check(native.lib().ktb200_mlp_load_weights(h, _stream(dev)))
        self._ktb_mlp, self._ktb_mlp_raw = h, raw
        return h

    def _ep_check(self, gen):
        if getattr(gen, "ep_size", 1) > 1 and getattr(self, "ep_exchange", None) is None:
            # without the exchange the shard's experts would return only their partial sum as the layer output
            raise RuntimeError(f"{getattr(self, 'key', type(self).__name__)}: the experts are sharded (expert_parallel_size "
                               f"{gen.ep_size}) but no expert-parallel exchange is attached (attach_expert_parallel)")

    def ep_tokens_forward(self, hidden_states, phase_mask=7, counts=None):
        """The sharded layer for any number of tokens on this rank (`ktb200_moe_ep_forward_tokens`); `counts` defaults to
        this layer's take of the step's counts (`ep_exchange.take_step_counts`).  phase_mask 7 returns the output; 1, 2 and
        4 run one phase each (1 takes the counts and keeps them with the routing and output buffers for 2 and 4; 4 returns
        the output), so that one GPU can drive N ranks' blocks in loopback."""
        orig_shape = hidden_states.shape
        n_tok = hidden_states.numel() // orig_shape[-1]
        hs = self._block_handles(hidden_states, need_mlp=False)
        if hs is None:
            raise RuntimeError(f"{getattr(self, 'key', type(self).__name__)}: the expert-parallel layer needs KMoEGateB200 routing and "
                               "loaded KExpertsB200 experts of the hidden dtype in generate mode")
        cfg, moe, mlp = hs
        if phase_mask & 1 or getattr(self, "_ep_pending", None) is None:
            counts = counts if counts is not None else self.ep_exchange.take_step_counts(n_tok)
            if counts is None:
                raise RuntimeError("expert-parallel step: no token counts were announced for this step; call "
                                   "ep_exchange.begin_step(n_tokens) on every rank at the start of each forward step")
            x = hidden_states.reshape(n_tok, orig_shape[-1]).contiguous()
            self._ep_pending = (x, torch.empty_like(x), torch.empty((n_tok, cfg.top_k), dtype=torch.int64, device=x.device),
                                torch.empty((n_tok, cfg.top_k), dtype=torch.float32, device=x.device), counts)
        x, y, idx, wt, counts = self._ep_pending
        native.check(native.lib().ktb200_moe_ep_forward_tokens(C.byref(cfg), moe, mlp, C.byref(self.ep_exchange.tok_comm), counts,
                                                               x.data_ptr(), y.data_ptr(), idx.data_ptr(), wt.data_ptr(), phase_mask,
                                                               _stream(x.device)))
        if not phase_mask & 4:
            return None
        self._ep_pending = None
        self.last_topk = (idx, wt)
        y = y.view(*orig_shape)
        if mlp is None and self.config.n_shared_experts is not None:
            y = y + self.shared_experts(hidden_states).view(*orig_shape)       # two rounded terms, like the unsharded block
        return y

    def forward(self, hidden_states):
        identity = hidden_states
        orig_shape = hidden_states.shape
        sequence_length = orig_shape[1]
        n_tok = hidden_states.numel() // orig_shape[-1]
        gen0 = getattr(getattr(self, "experts", None), "generate_experts", None)
        self._ep_check(gen0)
        if getattr(gen0, "ep_size", 1) > 1:
            # one take per layer: None when no step was announced (then only the one-token decode case can run)
            counts = self.ep_exchange.take_step_counts(n_tok)
            if n_tok != 1 or (counts is not None and any(c != 1 for c in counts)):
                return self.ep_tokens_forward(hidden_states, counts=counts)
        if getattr(gen0, "ep_size", 1) > 1 and n_tok == 1:
            # expert-parallel decode, one token per GPU: router, NVLink exchange, owned experts and combine in ONE launch
            hs = self._block_handles(hidden_states)
            if hs is not None:
                cfg, moe, mlp = hs
                x = hidden_states.reshape(1, orig_shape[-1]).contiguous()
                capturing = torch.cuda.is_current_stream_capturing()
                y = KExpertsB200.output_gpu_map[gen0.out_device][:1] if capturing else torch.empty_like(x)
                idx = torch.empty((1, cfg.top_k), dtype=torch.int64, device=x.device)
                wt = torch.empty((1, cfg.top_k), dtype=torch.float32, device=x.device)
                native.check(native.lib().ktb200_moe_ep_block_forward(C.byref(cfg), moe, mlp, C.byref(self.ep_exchange.comm), x.data_ptr(),
                                                                      y.data_ptr(), idx.data_ptr(), wt.data_ptr(), 7, _stream(x.device)))
                self.last_topk = (idx, wt)
                return y.view(*orig_shape)
            return self.ep_tokens_forward(hidden_states, counts=counts)
        if n_tok <= self.BLOCK_MAX_TOKENS and getattr(gen0, "ep_size", 1) == 1:
            hs = self._block_handles(hidden_states)
            if hs is not None:
                cfg, moe, mlp = hs
                x = hidden_states.reshape(n_tok, orig_shape[-1]).contiguous()
                gen = self.experts.generate_experts
                capturing = torch.cuda.is_current_stream_capturing()
                y = KExpertsB200.output_gpu_map[gen.out_device][:n_tok] if capturing else torch.empty_like(x)
                idx = torch.empty((n_tok, cfg.top_k), dtype=torch.int64, device=x.device)
                wt = torch.empty((n_tok, cfg.top_k), dtype=torch.float32, device=x.device)
                native.check(native.lib().ktb200_moe_block_forward(C.byref(cfg), moe, mlp, n_tok, x.data_ptr(), y.data_ptr(),
                                                                   idx.data_ptr(), wt.data_ptr(), None, _stream(x.device)))
                self.last_topk = (idx, wt)
                return y.view(*orig_shape)
        topk_idx, topk_weight = self.gate(hidden_states)
        hidden_states = hidden_states.view(-1, hidden_states.shape[-1])
        gen = getattr(self.experts, "generate_experts", None)
        if (sequence_length == 1 and hasattr(gen, "submit_for_one_decode") and hidden_states.is_cuda
                and torch.cuda.is_current_stream_capturing()):
            gen.submit_for_one_decode(hidden_states[0], topk_idx[0], topk_weight[0])
            if self.config.n_shared_experts is not None:
                y_ = self.shared_experts(identity).squeeze(0)
            y = gen.sync_for_one_decode().unsqueeze(0)
            if self.config.n_shared_experts is not None:
                y += y_
            y.resize_(*orig_shape)
            return y
        if self.config.n_shared_experts is not None:
            y_ = self.shared_experts(identity).squeeze(0)
        y = self.moe_kexperts(hidden_states, topk_idx, topk_weight).view(*orig_shape).to(device=hidden_states.device)
        if self.config.n_shared_experts is not None:
            y += y_.view(*orig_shape)
        return y

    @torch.no_grad()
    def moe_kexperts(self, x, topk_ids, topk_weight):
        return self.experts(x, topk_ids, topk_weight)


def chain_moe_prefetch(model: "torch.nn.Module") -> int:
    """Link consecutive injected MoE blocks: while block i streams its down projection, its kernel pulls block i+1's router
    weight and shared-expert gate / up tensors into L2 (ktb200_moe_block_prefetch_hint).  Returns the number of links.
    Call after `optimize_and_load_gguf` / `load()`; a no-op for blocks that do not take the single-launch path."""
    blocks = [m for m in model.modules() if isinstance(m, _KDeepseekMoEMixin)]
    n = 0
    for cur, nxt in zip(blocks, blocks[1:]):
        gen = getattr(getattr(cur, "experts", None), "generate_experts", None)
        gate = getattr(nxt, "gate", None)
        if not (isinstance(gen, KExpertsB200) and gen.handle is not None and getattr(gate, "_w", None) is not None):
            continue
        bufs = [gate._w] + list(getattr(nxt, "_ktb_mlp_raw", [])[:2])
        ptrs = (C.c_void_p * len(bufs))(*[b.data_ptr() for b in bufs])
        sizes = (C.c_size_t * len(bufs))(*[b.numel() * b.element_size() for b in bufs])
        native.check(native.lib().ktb200_moe_block_prefetch_hint(gen.handle, ptrs, sizes, len(bufs)))
        n += 1
    return n


def _moe_bases():
    from ..models.modeling_deepseek_v3 import DeepseekV3MoE
    from ..models.modeling_deepseek import DeepseekV2MoE
    return DeepseekV3MoE, DeepseekV2MoE


_V3, _V2 = _moe_bases()


class KDeepseekV3MoE(_KDeepseekMoEMixin, BaseInjectedModule, _V3):
    pass


class KDeepseekV2MoE(_KDeepseekMoEMixin, BaseInjectedModule, _V2):
    pass


class KDeepseekV3MoEV2(_KDeepseekMoEMixin, BaseInjectedModule, _V3):
    """experts.py:1172-1271: `forward(hidden_states, bsz_tensor, cuda_graph_idx)`; rows at or beyond `bsz_tensor[0]` are padding
    and are left untouched by every kernel (kt-kernel/operators/common.hpp:255-258 semantics, on the device).

    Except under expert parallelism (sharded experts): the exchange works on host-known token counts, so `bsz_tensor` is
    not read, and every row of the chunk, padding included, is computed and written like a real token."""

    def forward(self, hidden_states, bsz_tensor=None, cuda_graph_idx=0):
        gen0 = getattr(getattr(self, "experts", None), "generate_experts", None)
        if bsz_tensor is None or getattr(gen0, "ep_size", 1) > 1:
            return super().forward(hidden_states)
        identity, orig_shape = hidden_states, hidden_states.shape
        n_tok = hidden_states.numel() // orig_shape[-1]
        gen = getattr(getattr(self, "experts", None), "generate_experts", None)
        if n_tok <= self.BLOCK_MAX_TOKENS and getattr(gen, "ep_size", 1) == 1:
            hs = self._block_handles(hidden_states)
            if hs is not None:
                cfg, moe, mlp = hs
                x = hidden_states.reshape(n_tok, orig_shape[-1]).contiguous()
                capturing = torch.cuda.is_current_stream_capturing()
                y = KExpertsB200.output_gpu_map[gen.out_device][:n_tok] if capturing else torch.zeros_like(x)
                idx = torch.zeros((n_tok, cfg.top_k), dtype=torch.int64, device=x.device)
                wt = torch.zeros((n_tok, cfg.top_k), dtype=torch.float32, device=x.device)
                native.check(native.lib().ktb200_moe_block_forward(C.byref(cfg), moe, mlp, n_tok, x.data_ptr(), y.data_ptr(), idx.data_ptr(),
                                                                   wt.data_ptr(), bsz_tensor.data_ptr(), _stream(x.device)))
                self.last_topk = (idx, wt)
                return y.view(*orig_shape)
        topk_idx, topk_weight = self.gate(hidden_states)
        x = hidden_states.view(-1, orig_shape[-1])
        y = self.experts(x, topk_idx, topk_weight, bsz_tensor, cuda_graph_idx).view(*orig_shape).to(device=x.device)
        if self.config.n_shared_experts is not None:
            y = y + self.shared_experts(identity).view(*orig_shape)
        return y
