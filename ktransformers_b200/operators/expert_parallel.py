"""Expert-parallel dispatch/combine for decode (SURVEY §8e; spec: the HF EP branch of DeepseekV3MoE.moe_infer,
archive/ktransformers/models/modeling_deepseek_v3.py:550-605, minus its host round trips).

GPU g owns experts [g*E/N, (g+1)*E/N).  Every rank holds one (or a few) decode tokens.  Per MoE layer:

  dispatch  all-gather of the ranks' tokens, expert ids and routing weights (N x 14 KB at bs=1 per rank:
            latency-bound, so no count exchange and no variable-size all-to-all — every rank sees all
            (token, expert) pairs and keeps the ones it owns: ids outside its shard are skipped by the kernel,
            like the reference's gpu_experts_mask / should_skip_expert, kt-kernel/operators/common.hpp:255-258)
  compute   local experts on the gathered tokens, fp32 partial sums
  combine   reduce-scatter (sum) of the [N*t, H] fp32 partials: each rank receives its own tokens' totals, which
            are rounded to the hidden dtype once — the same sum the single-GPU path forms.

All buffers are static so the whole layer is CUDA-graph capturable with NCCL.
"""
from __future__ import annotations

from typing import Callable

import torch
import torch.distributed as dist


def shard_range(n_experts: int, rank: int, world: int) -> tuple[int, int]:
    assert n_experts % world == 0, "expert count must divide evenly across the EP group"
    per = n_experts // world
    return rank * per, (rank + 1) * per


class PeerExchange:
    """Peer-mapped buffers of the ONE-launch expert-parallel MoE block (`ktb200_moe_ep_block_forward`, include/ktb200.h):
    one symmetric allocation per rank (torch.distributed._symmetric_memory) holding the message rows {x, ids, weights},
    the fp32 partial rows and the flag block.  One instance serves every MoE layer of a model: layers run one after the
    other on the same stream and the epochs live in the flag block.  `KDeepseekV3MoE.forward` takes this path when its
    experts are sharded (expert_parallel_size > 1) and `module.ep_exchange` is set (see `attach_expert_parallel`)."""

    def __init__(self, hidden_size: int, hidden_type: int, device, group=None):
        import torch.distributed._symmetric_memory as symm_mem

        from .. import native
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        lib = native.lib()
        msg_b = self.world * lib.ktb200_ep_msg_bytes(hidden_size, hidden_type)
        part_b, flag_b = self.world * hidden_size * 4, 4 * (2 * self.world + 2)
        o_part = (msg_b + 255) // 256 * 256
        o_flag = o_part + (part_b + 255) // 256 * 256
        self.buf = symm_mem.empty(o_flag + (flag_b + 255) // 256 * 256, dtype=torch.uint8, device=device)
        self.buf.zero_()
        hdl = symm_mem.rendezvous(self.buf, self.group)
        base = [int(p) for p in hdl.buffer_ptrs]
        self.comm = native.EpComm.make(self.rank, self.world, hidden_size, hidden_type, base, [b + o_part for b in base],
                                       [b + o_flag for b in base])
        self.flags = self.buf[o_flag:o_flag + flag_b].view(torch.int32)
        torch.cuda.synchronize(device)
        dist.barrier(self.group)

    def timed_out(self) -> bool:
        """True when a peer wait inside a kernel gave up (a rank did not take part in a layer)."""
        return bool(self.flags[2 * self.world + 1].item())


def attach_expert_parallel(model: torch.nn.Module, hidden_size: int, hidden_type: int, device, group=None) -> PeerExchange:
    """Give every injected MoE block of `model` whose experts are sharded the same PeerExchange."""
    from ..native import RAWINT4_G32
    from ..util.custom_gguf import GGML_NAMES, B200_EP_GATE_UP_TYPES, B200_EP_DOWN_TYPES
    for m in model.modules():
        gen = getattr(getattr(m, "experts", None), "generate_experts", None)
        if not hasattr(m, "_block_handles") or getattr(gen, "gate_type", None) is None:
            continue
        types = (gen.gate_type, gen.up_type, gen.down_type)
        names = ["RAWINT4_G32" if t == RAWINT4_G32 else GGML_NAMES.get(int(t), str(t)) for t in types]
        if names[0] not in B200_EP_GATE_UP_TYPES or names[1] not in B200_EP_GATE_UP_TYPES or names[2] not in B200_EP_DOWN_TYPES:
            # the single-launch NVLink kernel takes Q4_K gate/up and Q4_K/Q6_K down only, and without it a sharded block would
            # return its shard's partial sums as the layer output
            raise ValueError(f"attach_expert_parallel: {getattr(m, 'key', type(m).__name__)} has {'/'.join(names)} experts "
                             "(gate/up/down), which the expert-parallel kernel does not support")
    ex = PeerExchange(hidden_size, hidden_type, device, group)
    for m in model.modules():
        if hasattr(m, "_block_handles"):
            m.ep_exchange = ex
    return ex


class ExpertParallelCombine:
    """local_forward(x_all[T,H] (fp32), ids_all[T,k], w_all[T,k], out_partial[T,H] fp32) computes this rank's share."""

    def __init__(self, hidden_size: int, top_k: int, tokens_per_rank: int, device, group=None, in_dtype=torch.bfloat16):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.t = tokens_per_rank
        T = self.world * tokens_per_rank
        self.x_all = torch.zeros((T, hidden_size), dtype=in_dtype, device=device)
        self.x_all_f32 = torch.zeros((T, hidden_size), dtype=torch.float32, device=device)
        self.ids_all = torch.zeros((T, top_k), dtype=torch.int64, device=device)
        self.w_all = torch.zeros((T, top_k), dtype=torch.float32, device=device)
        self.partial = torch.zeros((T, hidden_size), dtype=torch.float32, device=device)
        self.own = torch.zeros((tokens_per_rank, hidden_size), dtype=torch.float32, device=device)
        self._nccl = dist.is_initialized() and dist.get_backend(group) == "nccl"

    def dispatch(self, x: torch.Tensor, ids: torch.Tensor, w: torch.Tensor):
        if self.world == 1:
            self.x_all.copy_(x); self.ids_all.copy_(ids); self.w_all.copy_(w)
        else:
            dist.all_gather_into_tensor(self.x_all, x.contiguous(), group=self.group)
            dist.all_gather_into_tensor(self.ids_all, ids.contiguous(), group=self.group)
            dist.all_gather_into_tensor(self.w_all, w.contiguous(), group=self.group)
        self.x_all_f32.copy_(self.x_all)
        return self.x_all_f32, self.ids_all, self.w_all

    def combine(self) -> torch.Tensor:
        if self.world == 1:
            self.own.copy_(self.partial)
        elif self._nccl:
            dist.reduce_scatter_tensor(self.own, self.partial, group=self.group)
        else:  # gloo has no reduce_scatter: all-reduce and keep the own rows (CPU tests)
            dist.all_reduce(self.partial, group=self.group)
            self.own.copy_(self.partial[self.rank * self.t:(self.rank + 1) * self.t])
        return self.own

    def forward(self, x, ids, w, local_forward: Callable) -> torch.Tensor:
        xa, ia, wa = self.dispatch(x, ids, w)
        local_forward(xa, ia, wa, self.partial)
        return self.combine()
