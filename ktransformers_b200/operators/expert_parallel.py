"""Expert-parallel dispatch/combine (SURVEY §8e; spec: the HF EP branch of DeepseekV3MoE.moe_infer,
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

import ctypes as C
from typing import Callable

import torch
import torch.distributed as dist


def shard_range(n_experts: int, rank: int, world: int) -> tuple[int, int]:
    assert n_experts % world == 0, "expert count must divide evenly across the EP group"
    per = n_experts // world
    return rank * per, (rank + 1) * per


class StepTokenCounts:
    """The token count of every rank of an expert-parallel group for the current forward step.

    `ktb200_moe_ep_forward_tokens` needs the same host array `counts[world]` on every rank.  It is exchanged ONCE per
    forward step, not per layer: every rank calls `begin_step(n_tokens)` before its first MoE layer (one host all-gather
    over `group`, which should be a CPU (gloo) group so that the exchange needs no device synchronise), and every MoE layer
    of the step takes it with `take(n_tokens)`.  A prefill step is eager anyway (the MLA cache's host counter rules out
    graph capture), so one host exchange per step costs little next to the layer stack.

    The counts belong to one step only: after `layers_per_step` takes (the number of expert-parallel MoE layers of the
    model) or `end_step()` they are gone, so a later step that announces nothing never runs on stale counts."""

    def __init__(self, group=None, layers_per_step: int | None = None):
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        self.layers_per_step = layers_per_step
        self.counts, self.left = None, None

    def begin_step(self, n_tokens: int) -> list[int]:
        mine = torch.tensor([int(n_tokens)], dtype=torch.int64)
        every = [torch.zeros_like(mine) for _ in range(self.world)]
        dist.all_gather(every, mine, group=self.group)
        self.counts = (C.c_int * self.world)(*[int(t) for t in every])
        self.left = self.layers_per_step
        return list(self.counts)

    def end_step(self):
        self.counts, self.left = None, None

    def take(self, n_tokens: int):
        """One MoE layer's use of the step's counts: the ctypes int array, or None when no step was announced.  Raises when
        this rank announced another token count than the layer got."""
        counts = self.counts
        if counts is None:
            return None
        if counts[self.rank] != n_tokens:
            raise RuntimeError(f"expert-parallel step: this rank announced {counts[self.rank]} tokens but a MoE layer got "
                               f"{n_tokens}; call begin_step(n_tokens) on every rank at the start of each forward step")
        if self.left is not None:
            self.left -= 1
            if self.left <= 0:
                self.end_step()
        return counts


def exchange_layout(world: int, hidden_size: int, hidden_type: int, top_k: int, max_tokens_per_rank: int) -> dict:
    """Byte offsets of one rank's PeerExchange allocation: the one-token block's message rows (0), partial rows and flag
    block, then the multi-token layer's region ("tokens"; its own offsets in "token_regions"); "bytes" in all."""
    from .. import native
    up = lambda n: (n + 255) // 256 * 256    # noqa: E731
    msg_b = world * native.lib().ktb200_ep_msg_bytes(hidden_size, hidden_type)
    o_part = up(msg_b)
    o_flag = o_part + up(world * hidden_size * 4)
    o_tok = o_flag + up(4 * (2 * world + 2))
    tok_b, tok_off = native.ep_tokens_layout(world, max_tokens_per_rank, hidden_size, hidden_type, top_k)
    return {"message": 0, "partial": o_part, "flags": o_flag, "tokens": o_tok, "token_regions": tok_off, "bytes": o_tok + tok_b}


class PeerExchange:
    """Peer-mapped buffers of the expert-parallel MoE layer, one symmetric allocation per rank
    (torch.distributed._symmetric_memory), zeroed once:
      - the one-launch decode block (`ktb200_moe_ep_block_forward`, one token per GPU): the message rows {x, ids, weights},
        the fp32 partial rows and the flag block, behind `comm`;
      - the multi-token layer (`ktb200_moe_ep_forward_tokens`, any number of tokens per GPU, prompt chunks): its own
        region laid out by `ktb200_ep_tokens_layout` for `max_tokens_per_rank` tokens per rank (default: the experts'
        group_max_len // world, so that the gathered rows of a full step fit one expert launch), behind `tok_comm`.
    One instance serves every MoE layer of a model: layers run one after the other on the same stream and the epochs live
    in the flag words.  `KDeepseekV3MoE.forward` uses it when its experts are sharded (expert_parallel_size > 1) and
    `module.ep_exchange` is set (see `attach_expert_parallel`).  Multi-token steps need the step's token counts: call
    `begin_step(n_tokens)` on every rank at the start of each forward step (see StepTokenCounts; `layers_per_step` is the
    number of MoE layers that use this exchange in one step, after which the counts expire).

    The counts travel over a gloo group.  `count_group` gives it; by default it is `group` itself when that is a gloo
    group, else a new gloo group over `group`'s ranks made with `dist.new_group`, which is a collective over the DEFAULT
    group: then every process of the default group must construct the exchange, so a proper subgroup with another backend
    needs `count_group`."""

    def __init__(self, hidden_size: int, hidden_type: int, device, group=None, top_k: int = 8, max_tokens_per_rank: int | None = None,
                 count_group=None, layers_per_step: int | None = None):
        import torch.distributed._symmetric_memory as symm_mem

        from .. import native
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        if max_tokens_per_rank is None:
            from .experts import KExpertsB200
            max_tokens_per_rank = max(1, KExpertsB200.MAX_TOKENS // self.world)
        lay = exchange_layout(self.world, hidden_size, hidden_type, top_k, max_tokens_per_rank)
        o_part, o_flag, o_tok, flag_b = lay["partial"], lay["flags"], lay["tokens"], 4 * (2 * self.world + 2)
        self.tok_offsets = lay["token_regions"]
        self.buf = symm_mem.empty(lay["bytes"], dtype=torch.uint8, device=device)
        self.buf.zero_()
        hdl = symm_mem.rendezvous(self.buf, self.group)
        base = [int(p) for p in hdl.buffer_ptrs]
        self.comm = native.EpComm.make(self.rank, self.world, hidden_size, hidden_type, base, [b + o_part for b in base],
                                       [b + o_flag for b in base])
        self.flags = self.buf[o_flag:o_flag + flag_b].view(torch.int32)
        self.max_tokens_per_rank, self.top_k = max_tokens_per_rank, top_k
        self.tok_comm = native.EpTokensComm.make(self.rank, self.world, max_tokens_per_rank, hidden_size, hidden_type, top_k,
                                                 [b + o_tok for b in base])
        o_tf = o_tok + self.tok_offsets["flags"]
        self.tok_flags = self.buf[o_tf:o_tf + 4 * (2 * self.world + 5)].view(torch.int32)
        if count_group is None:
            # the per-step count exchange is a host all-gather: over gloo it needs no device synchronise
            if dist.get_backend(self.group) == "gloo":
                count_group = self.group
            elif dist.get_world_size(self.group) == dist.get_world_size():
                count_group = dist.new_group(dist.get_process_group_ranks(self.group), backend="gloo")
            else:
                raise ValueError("PeerExchange: pass count_group (a gloo group over the expert-parallel ranks) when the group is a "
                                 "proper subgroup of another backend; making one here would be a collective over every process")
        self.step = StepTokenCounts(count_group, layers_per_step)
        torch.cuda.synchronize(device)
        dist.barrier(self.group)

    def timed_out(self) -> bool:
        """True when a peer wait inside a kernel gave up (a rank did not take part in a layer)."""
        return bool(self.flags[2 * self.world + 1].item()) or bool(self.tok_flags[2 * self.world + 2].item())

    def begin_step(self, n_tokens: int) -> list[int]:
        """Announce this rank's token count for the forward step that starts now (every rank, once per step)."""
        return self.step.begin_step(n_tokens)

    def take_step_counts(self, n_tokens: int):
        """One MoE layer's use of the step's counts (StepTokenCounts.take)."""
        return self.step.take(n_tokens)


def attach_expert_parallel(model: torch.nn.Module, hidden_size: int, hidden_type: int, device, group=None, count_group=None) -> PeerExchange:
    """Give every injected MoE block of `model` whose experts are sharded the same PeerExchange; its step counts expire
    after one use by each of those blocks."""
    from ..native import RAWINT4_G32
    from ..util.custom_gguf import GGML_NAMES, B200_EP_TYPE_SETS
    for m in model.modules():
        gen = getattr(getattr(m, "experts", None), "generate_experts", None)
        if not hasattr(m, "_block_handles") or getattr(gen, "gate_type", None) is None:
            continue
        types = (gen.gate_type, gen.up_type, gen.down_type)
        names = ["RAWINT4_G32" if t == RAWINT4_G32 else GGML_NAMES.get(int(t), str(t)) for t in types]
        if names[0] != names[1] or (names[0], names[2]) not in B200_EP_TYPE_SETS:
            # the single-launch NVLink kernel takes these sets only, and without it a sharded block would return its shard's
            # partial sums as the layer output
            raise ValueError(f"attach_expert_parallel: {getattr(m, 'key', type(m).__name__)} has {'/'.join(names)} experts "
                             "(gate/up/down), which the expert-parallel kernel does not support")
    gens = [m.experts.generate_experts for m in model.modules() if hasattr(m, "_block_handles")
            and getattr(getattr(getattr(m, "experts", None), "generate_experts", None), "max_tokens", None) is not None]
    sharded = [g for g in gens if getattr(g, "ep_size", 1) > 1]
    world = dist.get_world_size(group if group is not None else dist.group.WORLD)
    kw = {}
    if gens:
        kw = dict(top_k=int(gens[0].config.num_experts_per_tok), max_tokens_per_rank=max(1, min(g.max_tokens for g in gens) // world))
    ex = PeerExchange(hidden_size, hidden_type, device, group, count_group=count_group, layers_per_step=len(sharded) or None, **kw)
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
