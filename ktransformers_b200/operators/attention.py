"""KDeepseekV2Attention — absorbed multi-head latent attention for decode (V3 MLA is the same as V2).

Mirrors archive/ktransformers/operators/attention.py:49-75 (`get_absorbed`) and :349-478 (`forward_linux_flashinfer`,
decode branch): q projections -> RoPE -> paged latent-cache update -> q_nope . W_UK (batched matmul) -> MLA paged decode
over the 576-wide latents -> . W_UV^T -> o_proj.  The attention itself is `MLAWrapper.run` = ktb200_mla_decode (wgmma +
TMA, csrc/mla.cu); the cache write is ktb200_mla_kv_write; the projections are whatever modules the rules injected
(KLinearB200 on raw GGUF blocks, or nn.Linear); the two absorb products are ktb200_mla_absorb_q / _o (HBM-bound batched
GEMVs over the bf16 halves of kv_b_proj; torch.matmul for other dtypes).

Prefill (q_len > 1 without absorb_for_prefill) follows the reference's non-absorbed branch of the same function: the same
projections, RoPE and cache update, then the first S = P + q_len cached latents of each sequence go through kv_b_proj
(dense, as the reference calls it) and ktb200_mla_prefill (csrc/mla_prefill.cu, wgmma + TMA) runs causal attention over
the decompressed heads in place: q_nope from the q_b output, k_nope / v from the kv_b_proj output, k_pe from the cache
rows.  P is the cache's host-side token count, so the path makes no device-to-host synchronisation; positions are
[P, P + q_len), as StaticCache.update assumes.  bf16 only.

With absorb_for_prefill (the reference's switch, DeepSeek-V3-Chat.yaml) a chunk of q_len > 1 takes the absorbed branch
instead: the decode steps up to absorb_q, then causal latent-space attention straight from the paged cache
(MLAWrapper.run -> ktb200_mla_decode_chunk, lengths position_ids[:, -1] + 1 on the device, nothing decompressed), then
absorb_o and o_proj.  Like decode, it makes no host synchronisation and can be captured in a CUDA graph.

forward_ragged is the flat-token entry of a serving step (balance_serve's flashinfer_attn.forward): tokens of several
sequences at their own positions, decode tokens and prompt chunks mixed, through the same projections and RoPE and a
per-token cache write (StaticCache.write_tokens).  With absorb_for_prefill, or when no sequence of the step has more than one
token, every row then takes the absorbed branch: absorb_q, one ragged MLAWrapper call (ktb200_mla_decode_ragged), absorb_o.
Otherwise the step splits by forward's rule (SGLang's DeepSeek path makes the same split): the prompt sequences (q_len > 1)
gather their cached latents through the layer's page table into one packed buffer, one dense kv_b_proj decompresses it and
one ktb200_mla_prefill_varlen call (csrc/mla_prefill.cu) attends with the queries in place in the q_b output; the decode
sequences (q_len == 1) take the absorbed branch on their rows only, and their output is scattered into the same rows.
One o_proj follows either way.  The ragged wrapper is one per device, shared by every layer, with its own row and item
capacities."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import torch

from .. import native
from ..models.modeling_deepseek_v3 import DeepseekV3Attention, apply_rotary_pos_emb
from .base_operator import BaseInjectedModule
from .flashinfer_wrapper import MLAWrapper, MLAWrapperSingleton

_RAGGED_WRAPPERS: dict = {}   # device -> the MLAWrapper of forward_ragged (one plan and one split workspace for all layers)


def _ragged_wrapper(cache, dev, batch: int, max_rows: int, max_items: int) -> MLAWrapper:
    key = str(dev)
    if key not in _RAGGED_WRAPPERS:
        _RAGGED_WRAPPERS[key] = MLAWrapper(cache.max_batch_size, cache.max_pages, device=key, max_rows=max_rows, max_items=max_items)
    w = _RAGGED_WRAPPERS[key]
    assert batch <= w.max_batch_size and cache.max_pages <= w.max_pages, "the shared ragged wrapper was made for a smaller cache"
    return w


class KDeepseekV2Attention(BaseInjectedModule, DeepseekV3Attention):
    def __init__(self, key, gguf_loader, config, orig_module, prefill_device: str = "cuda", generate_device: str = "cuda",
                 chunck_size: int = 1000, absorb_for_prefill: bool = False, **kwargs):
        BaseInjectedModule.__init__(self, key, gguf_loader, config, orig_module, prefill_device, generate_device, **kwargs)
        self.chunck_size = chunck_size
        self.mla_wrapper = None
        self.absorb_for_prefill = absorb_for_prefill

    def get_absorbed(self) -> Tuple[torch.Tensor, torch.Tensor]:
        """kv_b_proj [heads * (128 + 128), 512] viewed per head: q_absorb = W_UK [h, 128, 512], out_absorb = W_UV [h, 128, 512]
        (attention.py:69-75); kv_b_proj is the one projection the rules keep dense."""
        if not (hasattr(self, "q_absorb") and hasattr(self, "out_absorb")):
            kv_b = self.kv_b_proj.weight.view(self.num_heads, -1, self.kv_lora_rank)
            object.__setattr__(self, "q_absorb", kv_b[:, : self.qk_nope_head_dim, :].contiguous())
            object.__setattr__(self, "out_absorb", kv_b[:, self.qk_nope_head_dim:, :].contiguous())
        return self.q_absorb, self.out_absorb

    def forward(self, hidden_states: torch.Tensor, attention_mask: Optional[torch.Tensor] = None,
                position_ids: Optional[torch.Tensor] = None, past_key_value=None, output_attentions: bool = False,
                use_cache: bool = False, cache_position: Optional[torch.Tensor] = None, **kwargs):
        bsz, q_len, _ = hidden_states.size()
        prefill = q_len != 1 and not self.absorb_for_prefill
        assert past_key_value is not None, "decode needs the paged latent cache (models/custom_cache.StaticCache)"
        if prefill:   # the reference's kv_seq_len: the cache's host counter before the update, plus the new tokens
            kv_seq_len = past_key_value.get_seq_length(self.layer_idx) + q_len
        q = self.q_proj(hidden_states) if self.q_lora_rank is None else self.q_b_proj(self.q_a_layernorm(self.q_a_proj(hidden_states)))
        q = q.view(bsz, q_len, self.num_heads, self.q_head_dim)
        q_nope, q_pe = torch.split(q, [self.qk_nope_head_dim, self.qk_rope_head_dim], dim=-1)
        compressed_kv = self.kv_a_proj_with_mqa(hidden_states)
        compressed_kv, k_pe = torch.split(compressed_kv, [self.kv_lora_rank, self.qk_rope_head_dim], dim=-1)
        compressed_kv = self.kv_a_layernorm(compressed_kv).view(bsz, q_len, 1, self.kv_lora_rank)
        k_pe = k_pe.view(bsz, q_len, 1, self.qk_rope_head_dim)
        cos, sin = self.rotary_emb(q_pe, position_ids)
        q_pe, k_pe = apply_rotary_pos_emb(q_pe, k_pe, cos, sin, unsqueeze_dim=2)

        cache_kwargs = {"sin": sin, "cos": cos, "cache_position": cache_position}
        kv_with_k_pe, page_table = past_key_value.update(compressed_kv, k_pe, self.layer_idx, cache_kwargs)
        if prefill:
            return self.forward_prefill(q, q_pe, kv_with_k_pe, past_key_value.max_pages, kv_seq_len), None, past_key_value
        ckv_pages = kv_with_k_pe[:, :, :, : self.kv_lora_rank].view(-1, past_key_value.page_size, self.kv_lora_rank)
        kpe_pages = kv_with_k_pe[:, :, :, self.kv_lora_rank:].view(-1, past_key_value.page_size, self.qk_rope_head_dim)

        q_absorb, out_absorb = self.get_absorbed()
        fused = (q.dtype == torch.bfloat16 and q_absorb.dtype == torch.bfloat16 and q.is_contiguous())
        stream = torch.cuda.current_stream(hidden_states.device).cuda_stream
        if fused:   # q_nope . W_UK straight from the q_b output (no slice copy): ktb200_mla_absorb_q
            q_abs = torch.empty((bsz * q_len, self.num_heads, self.kv_lora_rank), dtype=q.dtype, device=q.device)
            native.check(native.lib().ktb200_mla_absorb_q(q.data_ptr(), self.q_head_dim, self.num_heads * self.q_head_dim, q_absorb.data_ptr(), self.num_heads,
                                                          self.qk_nope_head_dim, self.kv_lora_rank, q_abs.data_ptr(), bsz * q_len, stream))
            q_nope = q_abs
        else:
            q_nope = torch.matmul(q_nope.transpose(1, 2), q_absorb).transpose(1, 2).contiguous().reshape(bsz * q_len, self.num_heads, self.kv_lora_rank)
        q_pe = q_pe.reshape(bsz * q_len, self.num_heads, self.qk_rope_head_dim)

        if self.mla_wrapper is None:
            self.mla_wrapper = MLAWrapperSingleton.get_instance(str(hidden_states.device), bsz, past_key_value.max_pages * bsz, use_cuda_graph=True)
        w = self.mla_wrapper
        if w.need_plan or w.q_len != q_len:
            # q_len queries per sequence (the chunk's causal offsets follow from kv length = last position + 1), identity
            # page table of the static cache; qo_indptr on the host, so planning makes no synchronisation
            qo_indptr = None if q_len == 1 else torch.arange(0, bsz + 1, dtype=torch.int32) * q_len
            kv_len = (position_ids.reshape(bsz, -1)[:, -1] + 1).to(torch.int32)
            pages = past_key_value.max_pages
            indptr = torch.arange(0, bsz + 1, dtype=torch.int32, device=hidden_states.device) * pages
            w.plan(qo_indptr, indptr, page_table.reshape(-1), kv_len, None, self.num_heads, self.kv_lora_rank, self.qk_rope_head_dim,
                   past_key_value.page_size, self.softmax_scale, q_nope.dtype, ckv_pages.dtype)
            w.max_pages_per_seq = pages
        else:   # the plan is static (identity page table); only the lengths move from step to step (a captured device copy)
            w.kv_len_arr_buf[:bsz].copy_((position_ids.reshape(bsz, -1)[:, -1] + 1).to(torch.int32))
        attn = w.run(q_nope, q_pe.contiguous(), ckv_pages, kpe_pages).view(bsz, q_len, self.num_heads, self.kv_lora_rank)
        if fused:
            o = torch.empty((bsz, q_len, self.num_heads, self.v_head_dim), dtype=attn.dtype, device=attn.device)
            native.check(native.lib().ktb200_mla_absorb_o(attn.data_ptr(), out_absorb.data_ptr(), self.num_heads, self.v_head_dim, self.kv_lora_rank, o.data_ptr(),
                                                          bsz * q_len, stream))
            attn = o
        else:
            attn = torch.matmul(attn.transpose(1, 2), out_absorb.mT).transpose(1, 2).contiguous()     # [b, 1, h, 128]
        attn = self.o_proj(attn.reshape(bsz, q_len, self.num_heads * self.v_head_dim))
        return attn, None, past_key_value

    def forward_ragged(self, hidden_states: torch.Tensor, position_ids: torch.Tensor, qo_indptr: torch.Tensor, kv_len: torch.Tensor,
                       cache_rows, past_key_value, max_rows: int = 1024, max_items: int = 4096) -> torch.Tensor:
        """Attention of a ragged batch of flat tokens.  hidden_states [T, hidden]; position_ids [T] (device) each token's
        position; qo_indptr [B + 1] (host) sequence b's tokens are rows [qo_indptr[b], qo_indptr[b + 1]); kv_len [B] (host)
        each sequence's length after this step; cache_rows [B] (host) the StaticCache batch row (page range) sequence b
        owns.  A sequence's tokens are its last q_len_b positions, kv_len[b] - q_len_b .. kv_len[b] - 1.  max_rows /
        max_items size the shared wrapper when this call creates it.  Returns [T, hidden].  The host data reaches the device
        through pinned, non-blocking copies, so the step makes no host synchronisation.

        Without absorb_for_prefill, a step in which some sequence has q_len_b > 1 runs those sequences on the decompressed
        path (kv_b_proj over their kv_len[b] cached latents, ktb200_mla_prefill_varlen; bf16 only, as forward's prefill) and
        the q_len_b == 1 sequences on the absorbed one; otherwise every row is absorbed.  The decompressed keys and values
        take 64 KB per cached token of the prompt sequences, as in forward."""
        T = hidden_states.shape[0]
        cache = past_key_value
        qo = torch.as_tensor(qo_indptr, dtype=torch.int32)
        rows = torch.as_tensor(cache_rows, dtype=torch.int32)
        B = rows.numel()
        assert qo.numel() == B + 1 and int(qo[-1]) == T, f"qo_indptr {qo.tolist()} does not cover {T} tokens of {B} sequences"
        dev = hidden_states.device
        # the cache row of every token, then the cache row of every sequence: one pinned copy
        host = torch.cat([torch.repeat_interleave(rows, qo[1:] - qo[:-1]), rows]).pin_memory()
        rows_dev = host.to(dev, non_blocking=True)
        token_rows, seq_rows = rows_dev[:T], rows_dev[T:]
        x = hidden_states.view(1, T, -1)
        pos = position_ids.view(1, T)
        q = self.q_proj(x) if self.q_lora_rank is None else self.q_b_proj(self.q_a_layernorm(self.q_a_proj(x)))
        q = q.view(1, T, self.num_heads, self.q_head_dim)
        q_nope, q_pe = torch.split(q, [self.qk_nope_head_dim, self.qk_rope_head_dim], dim=-1)
        compressed_kv = self.kv_a_proj_with_mqa(x)
        compressed_kv, k_pe = torch.split(compressed_kv, [self.kv_lora_rank, self.qk_rope_head_dim], dim=-1)
        compressed_kv = self.kv_a_layernorm(compressed_kv).view(1, T, 1, self.kv_lora_rank)
        k_pe = k_pe.view(1, T, 1, self.qk_rope_head_dim)
        cos, sin = self.rotary_emb(q_pe, pos)
        q_pe, k_pe = apply_rotary_pos_emb(q_pe, k_pe, cos, sin, unsqueeze_dim=2)
        kv_with_k_pe = cache.write_tokens(compressed_kv, k_pe, self.layer_idx, token_rows, position_ids)
        if not self.absorb_for_prefill and bool(((qo[1:] - qo[:-1]) > 1).any()):
            attn = self._ragged_split(q, q_pe.reshape(T, self.num_heads, self.qk_rope_head_dim).contiguous(), kv_with_k_pe, qo,
                                      torch.as_tensor(kv_len, dtype=torch.int32), rows, cache, max_rows, max_items)
            return self.o_proj(attn.reshape(1, T, self.num_heads * self.v_head_dim)).view(T, -1)
        ckv_pages = kv_with_k_pe[:, :, :, : self.kv_lora_rank].view(-1, cache.page_size, self.kv_lora_rank)
        kpe_pages = kv_with_k_pe[:, :, :, self.kv_lora_rank:].view(-1, cache.page_size, self.qk_rope_head_dim)

        q_absorb, out_absorb = self.get_absorbed()
        fused = (q.dtype == torch.bfloat16 and q_absorb.dtype == torch.bfloat16 and q.is_contiguous())
        stream = torch.cuda.current_stream(dev).cuda_stream
        if fused:
            q_abs = torch.empty((T, self.num_heads, self.kv_lora_rank), dtype=q.dtype, device=dev)
            native.check(native.lib().ktb200_mla_absorb_q(q.data_ptr(), self.q_head_dim, self.num_heads * self.q_head_dim, q_absorb.data_ptr(), self.num_heads,
                                                          self.qk_nope_head_dim, self.kv_lora_rank, q_abs.data_ptr(), T, stream))
            q_nope = q_abs
        else:
            q_nope = torch.matmul(q_nope.transpose(1, 2), q_absorb).transpose(1, 2).contiguous().reshape(T, self.num_heads, self.kv_lora_rank)
        q_pe = q_pe.reshape(T, self.num_heads, self.qk_rope_head_dim).contiguous()

        w = _ragged_wrapper(cache, dev, B, max_rows, max_items)
        # sequence b's page table is its cache row's: kv_indices = the static table's rows, cache.max_pages pages each
        kv_indptr = torch.arange(0, B + 1, dtype=torch.int32, device=dev) * cache.max_pages
        kv_indices = cache.page_table_list[self.layer_idx].index_select(0, seq_rows.long()).reshape(-1)
        w.plan(qo, kv_indptr, kv_indices, torch.as_tensor(kv_len, dtype=torch.int32), None, self.num_heads, self.kv_lora_rank,
               self.qk_rope_head_dim, cache.page_size, self.softmax_scale, q_nope.dtype, ckv_pages.dtype)
        attn = w.run(q_nope, q_pe, ckv_pages, kpe_pages)
        if fused:
            o = torch.empty((T, self.num_heads, self.v_head_dim), dtype=attn.dtype, device=dev)
            native.check(native.lib().ktb200_mla_absorb_o(attn.data_ptr(), out_absorb.data_ptr(), self.num_heads, self.v_head_dim, self.kv_lora_rank, o.data_ptr(),
                                                          T, stream))
            attn = o
        else:
            attn = torch.matmul(attn.view(T, self.num_heads, 1, -1), out_absorb.mT.unsqueeze(0)).view(T, self.num_heads, self.v_head_dim)
        return self.o_proj(attn.reshape(1, T, self.num_heads * self.v_head_dim)).view(T, -1)

    def _ragged_split(self, q: torch.Tensor, q_pe: torch.Tensor, kv_with_k_pe: torch.Tensor, qo: torch.Tensor, kv_len: torch.Tensor,
                      rows: torch.Tensor, cache, max_rows: int, max_items: int) -> torch.Tensor:
        """The attention core of a ragged step with prompt sequences, before o_proj: [T, heads, 128].  q [1, T, heads, 192] is
        the q_b output, q_pe [T, heads, 64] the roped part, kv_with_k_pe the layer's latent buffer after write_tokens; qo,
        kv_len and rows are host int32 tensors."""
        T, H, dev = q.shape[1], self.num_heads, q.device
        if q.dtype != torch.bfloat16 or q_pe.dtype != torch.bfloat16 or self.kv_b_proj.weight.dtype != torch.bfloat16:
            raise NotImplementedError(f"KDeepseekV2Attention prefill is bf16 only (q {q.dtype}, kv_b_proj {self.kv_b_proj.weight.dtype})")
        q_lens = qo[1:] - qo[:-1]
        pre, dec = torch.nonzero(q_lens > 1).flatten(), torch.nonzero(q_lens == 1).flatten()
        S, n, nd, page = kv_len[pre], int(kv_len[pre].sum()), dec.numel(), cache.page_size
        # token j of prompt sequence b is row page_table[rows[b], j // page] * page + j % page of the layer's buffer: the
        # page-table entry's index, the offset, then the decode rows and their cache rows, in one pinned copy
        j = torch.arange(n, dtype=torch.int32) - torch.repeat_interleave(torch.cumsum(S, 0, dtype=torch.int32) - S, S)
        host = torch.cat([torch.repeat_interleave(rows[pre], S) * cache.max_pages + j // page, j % page, qo[dec], rows[dec]]).pin_memory()
        idx = host.to(dev, non_blocking=True)
        table = cache.page_table_list[self.layer_idx]
        flat = table.reshape(-1).index_select(0, idx[:n]) * page + idx[n:2 * n]
        lat = kv_with_k_pe.view(-1, kv_with_k_pe.shape[-1]).index_select(0, flat)                 # [sum S, 576]
        kv = self.kv_b_proj(lat[:, : self.kv_lora_rank]).view(n, H, self.qk_nope_head_dim + self.v_head_dim)
        k_nope, v, k_pe = kv[..., : self.qk_nope_head_dim], kv[..., self.qk_nope_head_dim:], lat[:, self.kv_lora_rank:]
        q_nope = q.view(T, H, self.q_head_dim)[..., : self.qk_nope_head_dim]
        seq = torch.stack([qo[pre], q_lens[pre], torch.cumsum(S, 0, dtype=torch.int32) - S, S], 1).to(torch.int32).contiguous()
        out = torch.empty((T, H, self.v_head_dim), dtype=q.dtype, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        p = native.MlaPrefillVarlenParams(pre.numel(), T, n, H, self.qk_nope_head_dim, self.qk_rope_head_dim, self.v_head_dim, self.softmax_scale,
                                          seq.data_ptr(), q_nope.data_ptr(), q_nope.stride(0), q_nope.stride(1), q_pe.data_ptr(), q_pe.stride(0),
                                          q_pe.stride(1), k_nope.data_ptr(), k_nope.stride(0), k_nope.stride(1), v.data_ptr(), v.stride(0),
                                          v.stride(1), k_pe.data_ptr(), k_pe.stride(0), out.data_ptr())
        native.check(native.lib().ktb200_mla_prefill_varlen(C.byref(p), stream))
        if nd:   # the decode rows: absorb_q, one MLAWrapper call over those sequences only, absorb_o, scattered into their rows
            d_rows, d_cache = idx[2 * n:2 * n + nd].long(), idx[2 * n + nd:]
            q_absorb, out_absorb = self.get_absorbed()
            q_dec = q.view(T, -1).index_select(0, d_rows)
            q_abs = torch.empty((nd, H, self.kv_lora_rank), dtype=q.dtype, device=dev)
            native.check(native.lib().ktb200_mla_absorb_q(q_dec.data_ptr(), self.q_head_dim, H * self.q_head_dim,
                                                          q_absorb.data_ptr(), H, self.qk_nope_head_dim, self.kv_lora_rank, q_abs.data_ptr(), nd, stream))
            w = _ragged_wrapper(cache, dev, nd, max_rows, max_items)
            kv_indptr = torch.arange(0, nd + 1, dtype=torch.int32, device=dev) * cache.max_pages
            w.plan(torch.arange(nd + 1, dtype=torch.int32), kv_indptr, table.index_select(0, d_cache).reshape(-1), kv_len[dec], None, H,
                   self.kv_lora_rank, self.qk_rope_head_dim, page, self.softmax_scale, q_abs.dtype, kv_with_k_pe.dtype)
            ckv_pages = kv_with_k_pe[:, :, :, : self.kv_lora_rank].view(-1, page, self.kv_lora_rank)
            kpe_pages = kv_with_k_pe[:, :, :, self.kv_lora_rank:].view(-1, page, self.qk_rope_head_dim)
            attn = w.run(q_abs, q_pe.index_select(0, d_rows), ckv_pages, kpe_pages)
            o = torch.empty((nd, H, self.v_head_dim), dtype=attn.dtype, device=dev)
            native.check(native.lib().ktb200_mla_absorb_o(attn.data_ptr(), out_absorb.data_ptr(), H, self.v_head_dim, self.kv_lora_rank, o.data_ptr(),
                                                          nd, stream))
            out.index_copy_(0, d_rows, o)
        return out

    def forward_prefill(self, q: torch.Tensor, q_pe: torch.Tensor, cache: torch.Tensor, max_pages: int, kv_seq_len: int) -> torch.Tensor:
        """Causal attention of a prompt chunk over the first kv_seq_len cached tokens of each sequence (attention.py:349-478,
        q_len > 1), then o_proj.  q [b, q_len, heads, 192] is the q_b output, q_pe [b, q_len, heads, 64] the roped part,
        cache the layer's latent buffer [max_batch * max_pages, page_size, 1, 576] after the update; with the identity page
        table the rows of sequence b are the contiguous rows [b * max_pages * page_size, ...)."""
        bsz, q_len = q.shape[0], q.shape[1]
        if q.dtype != torch.bfloat16 or q_pe.dtype != torch.bfloat16 or self.kv_b_proj.weight.dtype != torch.bfloat16:
            raise NotImplementedError(f"KDeepseekV2Attention prefill is bf16 only (q {q.dtype}, kv_b_proj {self.kv_b_proj.weight.dtype})")
        rows = cache.view(-1, max_pages * cache.shape[1], cache.shape[-1])[:bsz, :kv_seq_len]      # [b, S, 576]
        kv = self.kv_b_proj(rows[..., : self.kv_lora_rank])                                          # [b, S, heads * 256]
        kv = kv.view(bsz, kv_seq_len, self.num_heads, self.qk_nope_head_dim + self.v_head_dim)
        k_nope, v = kv[..., : self.qk_nope_head_dim], kv[..., self.qk_nope_head_dim:]
        q_nope, k_pe = q[..., : self.qk_nope_head_dim], rows[..., self.kv_lora_rank:]
        out = torch.empty((bsz, q_len, self.num_heads, self.v_head_dim), dtype=q.dtype, device=q.device)
        p = native.MlaPrefillParams(bsz, q_len, kv_seq_len, self.num_heads, self.qk_nope_head_dim, self.qk_rope_head_dim, self.v_head_dim,
                                    self.softmax_scale,
                                    q_nope.data_ptr(), q_nope.stride(1), q_nope.stride(2), q_nope.stride(0),
                                    q_pe.data_ptr(), q_pe.stride(1), q_pe.stride(2), q_pe.stride(0),
                                    k_nope.data_ptr(), k_nope.stride(1), k_nope.stride(2), k_nope.stride(0),
                                    v.data_ptr(), v.stride(1), v.stride(2), v.stride(0),
                                    k_pe.data_ptr(), k_pe.stride(1), k_pe.stride(0), out.data_ptr())
        native.check(native.lib().ktb200_mla_prefill(C.byref(p), torch.cuda.current_stream(q.device).cuda_stream))
        return self.o_proj(out.view(bsz, q_len, self.num_heads * self.v_head_dim))
