"""StaticCache — the paged latent KV cache of absorbed MLA (archive/ktransformers/models/custom_cache.py:26-200).

Same contract as the reference's DeepSeek branch: per layer one buffer `[max_pages, page_size, 1, kv_lora_rank + rope]`
(page_size 64), a static identity page table per batch row, `update(ckv, k_pe, layer_idx, {"cache_position": ...})`
writes the new rows at `(pos // page, pos % page)` and returns `(buffer, page_table)`.  The write is one
`ktb200_mla_kv_write` launch (csrc/mla.cu) instead of two advanced-indexing copies; buffers never move, so the cache
is CUDA-graph safe."""
from __future__ import annotations

from typing import Any, Dict, Optional, Tuple

import torch

from .. import native


class StaticCache:
    def __init__(self, config, max_batch_size: int, max_cache_len: int, device, dtype=torch.bfloat16, page_size: int = 64):
        assert dtype == torch.bfloat16, "the latent cache is bf16"
        self.config = config
        self._max_batch_size, self._max_cache_len = max_batch_size, max_cache_len
        self.page_size = page_size
        self.max_pages = (max_cache_len + page_size - 1) // page_size
        self.kv_lora_rank, self.qk_rope_head_dim = config.kv_lora_rank, config.qk_rope_head_dim
        self.device = torch.device(device)
        latent = (self.max_pages * max_batch_size, page_size, 1, self.kv_lora_rank + self.qk_rope_head_dim)
        self.key_cache = [torch.zeros(latent, dtype=dtype, device=device) for _ in range(config.num_hidden_layers)]
        self.value_cache = [None] * config.num_hidden_layers
        table = torch.arange(self.max_pages * max_batch_size, dtype=torch.int32, device=device).reshape(max_batch_size, self.max_pages)
        self.page_table_list = [table] * config.num_hidden_layers
        self.past_tokens = [0] * config.num_hidden_layers
        self.is_MLA = self.is_page = True

    @property
    def max_batch_size(self):
        return self._max_batch_size

    @property
    def max_cache_len(self):
        return self._max_cache_len

    def get_seq_length(self, layer_idx: int = 0) -> int:
        return self.past_tokens[layer_idx]

    def get_usable_length(self, kv_seq_len: int, layer_idx: int = 0) -> int:
        return self.past_tokens[layer_idx]

    def update(self, key_states: torch.Tensor, value_states: torch.Tensor, layer_idx: int,
               cache_kwargs: Optional[Dict[str, Any]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """key_states = compressed_kv [bsz, q_len, 1, 512], value_states = k_pe [bsz, q_len, 1, 64] (the reference's argument
        order, custom_cache.py:147-193); batch row b writes into its own page range."""
        cache_position = cache_kwargs.get("cache_position")
        k_out = self.key_cache[layer_idx]
        bsz, q_len = key_states.shape[0], key_states.shape[1]
        pos = cache_position.to(torch.int32).reshape(1, -1).expand(bsz, q_len)
        page_idx = (pos // self.page_size + torch.arange(bsz, device=pos.device, dtype=torch.int32).reshape(bsz, 1) * self.max_pages).reshape(-1).contiguous()
        page_off = (pos % self.page_size).reshape(-1).contiguous()
        ckv = key_states.reshape(-1, self.kv_lora_rank).contiguous()
        kpe = value_states.reshape(-1, self.qk_rope_head_dim).contiguous()
        native.check(native.lib().ktb200_mla_kv_write(k_out.data_ptr(), self.page_size, ckv.data_ptr(), kpe.data_ptr(), page_idx.data_ptr(),
                                                      page_off.data_ptr(), ckv.shape[0], torch.cuda.current_stream(k_out.device).cuda_stream))
        if not torch.cuda.is_current_stream_capturing():
            self.past_tokens[layer_idx] += q_len
        return k_out, self.page_table_list[layer_idx]

    def write_tokens(self, ckv: torch.Tensor, k_pe: torch.Tensor, layer_idx: int, cache_rows: torch.Tensor, positions: torch.Tensor) -> torch.Tensor:
        """Flat tokens at their own positions: token t (ckv [T, 512], k_pe [T, 64]) goes to position positions[t] of batch row
        cache_rows[t] (device int tensors [T]), page cache_rows[t] * max_pages + pos // page_size, offset pos % page_size.
        One ktb200_mla_kv_write launch, no host synchronisation; the host counter past_tokens is left alone (a batch at several
        positions has no single length).  Returns the layer's buffer."""
        k_out = self.key_cache[layer_idx]
        pos = positions.to(torch.int32)
        page_idx = (cache_rows.to(torch.int32) * self.max_pages + pos // self.page_size).contiguous()
        page_off = (pos % self.page_size).contiguous()
        ckv = ckv.reshape(-1, self.kv_lora_rank).contiguous()
        kpe = k_pe.reshape(-1, self.qk_rope_head_dim).contiguous()
        native.check(native.lib().ktb200_mla_kv_write(k_out.data_ptr(), self.page_size, ckv.data_ptr(), kpe.data_ptr(), page_idx.data_ptr(),
                                                      page_off.data_ptr(), ckv.shape[0], torch.cuda.current_stream(k_out.device).cuda_stream))
        return k_out

    def reset(self):
        for t in self.key_cache:
            t.zero_()
        self.past_tokens = [0] * len(self.past_tokens)
