"""MLAWrapper — same plan()/run() surface as the reference's flashinfer wrapper
(archive/ktransformers/operators/flashinfer_wrapper.py:78-161, MLAWrapperSingleton :163-199), backed by
ktb200_mla_decode instead of flashinfer.mla.BatchMLAPagedAttentionWrapper(backend="fa2").

plan() takes the CSR page description flashinfer uses (kv_indptr / kv_indices / kv_len_arr) and turns it into
the dense int32 page table the kernel reads; run() takes q_nope [B,H,512], q_pe [B,H,64] and the paged latent
cache as the two VIEWS the reference passes (ckv = cache[..., :512], k_pe = cache[..., 512:] of one
[pages, page_size, 576] buffer, archive/ktransformers/models/custom_cache.py:81-96).

plan() records q_len from the reference's qo_indptr (None: one query per sequence).  With q_len > 1, run() takes the
[B * q_len, H, 512] / [B * q_len, H, 64] queries of a prompt chunk and attends causally, query i of sequence b to the
first kv_len[b] - q_len + i + 1 cached tokens (ktb200_mla_decode_chunk); kv_len is the length after the chunk was
written.  Every sequence has the same q_len."""
from __future__ import annotations

import ctypes as C

import torch

from .. import native


class MLAWrapper:
    def __init__(self, max_batch_size, max_pages, use_cuda_graph=True, device="cuda"):
        native.lib()
        self.max_batch_size, self.max_pages, self.device = max_batch_size, max_pages, device
        self.page_table = torch.zeros((max_batch_size, max_pages), dtype=torch.int32, device=device)
        self.kv_len_arr_buf = torch.zeros(max_batch_size, dtype=torch.int32, device=device)
        self.batch_size_tensor_buf = torch.tensor([max_batch_size], dtype=torch.int32, device=device)
        self.qo_indptr_buf = torch.arange(0, max_batch_size + 1, dtype=torch.int32, device=device)
        self.kv_indptr_buf = torch.arange(0, max_batch_size + 1, dtype=torch.int32, device=device) * max(1, max_pages // max_batch_size)
        self.kv_indices_buf = torch.arange(0, max_pages, dtype=torch.int32, device=device)
        self.workspace = None
        self.need_plan = True
        self.num_heads = self.page_size = None
        self.sm_scale = None
        self.batch = max_batch_size
        self.q_len = 1

    def plan(self, qo_indptr, kv_indptr, kv_indices, kv_len_arr, bsz_tensor, num_heads, head_dim_ckv, head_dim_kpe,
             page_size, sm_scale, q_data_type, kv_data_type):
        assert head_dim_ckv == 512 and head_dim_kpe == 64, "MLA latent layout is 512 + 64"
        assert q_data_type == torch.bfloat16 and kv_data_type == torch.bfloat16, "bf16 only"
        kv_indptr = self.kv_indptr_buf if kv_indptr is None else kv_indptr
        kv_indices = self.kv_indices_buf if kv_indices is None else kv_indices
        self.batch = int(kv_indptr.numel() - 1)
        q_len = 1
        if qo_indptr is not None:   # a device qo_indptr costs one host synchronisation here; the operator passes a host one
            q_lens = (qo_indptr[1:] - qo_indptr[:-1]).tolist()
            assert len(q_lens) == self.batch and len(set(q_lens)) == 1 and q_lens[0] >= 1, \
                f"every sequence must have the same q_len >= 1, got {q_lens}"
            q_len = int(q_lens[0])
        # CSR -> dense page table (device-side torch ops; no host sync)
        counts = (kv_indptr[1:] - kv_indptr[:-1]).to(torch.int64)
        col = torch.arange(self.max_pages, device=self.device).unsqueeze(0)
        src = (kv_indptr[:-1].to(torch.int64).unsqueeze(1) + col).clamp_(max=max(int(kv_indices.numel()) - 1, 0))
        table = kv_indices.to(torch.int32)[src]
        self.page_table[: self.batch].copy_(torch.where(col < counts.unsqueeze(1), table, torch.zeros_like(table)))
        self.kv_len_arr_buf[: self.batch].copy_(kv_len_arr[: self.batch].to(torch.int32))
        self.num_heads, self.page_size, self.sm_scale = num_heads, page_size, float(sm_scale)
        need = native.lib().ktb200_mla_workspace_bytes(self.max_batch_size, num_heads, 0)
        if q_len > 1:   # the most splits the chunk entry picks by itself: ceil(SMs / (batch * q_len * head groups)), <= 128
            sms = torch.cuda.get_device_properties(torch.device(self.device)).multi_processor_count
            splits = min(128, -(-sms // (self.batch * q_len * -(-num_heads // 64))))
            need = max(need, native.lib().ktb200_mla_chunk_workspace_bytes(self.batch, q_len, num_heads, splits))
        self.q_len = q_len
        if self.workspace is None or self.workspace.numel() < need:
            self.workspace = torch.empty(need, dtype=torch.uint8, device=self.device)
        self.need_plan = False

    def run(self, q_nope, q_pe, ckv, k_pe, return_lse=False):
        assert not self.need_plan, "plan() before run()"
        if self.q_len > 1:
            return self._run_chunk(q_nope, q_pe, ckv, k_pe, return_lse)
        B = q_nope.shape[0]
        # the two views must alias one [pages, page, 576] buffer
        cache_ptr = ckv.data_ptr()
        assert ckv.stride(-1) == 1 and k_pe.data_ptr() == cache_ptr + 512 * ckv.element_size() and \
            ckv.stride(-2) in (576, 576 * ckv.shape[-2] if ckv.dim() > 3 else 576), \
            "ckv / k_pe must be the [..., :512] / [..., 512:] views of one 576-wide latent cache"
        q_nope, q_pe = q_nope.contiguous(), q_pe.contiguous()
        out = torch.empty_like(q_nope)
        lse = torch.empty((B, self.num_heads), dtype=torch.float32, device=q_nope.device) if return_lse else None
        p = native.MlaParams(B, self.num_heads, self.page_size, self.max_pages, 0, self.sm_scale, q_nope.data_ptr(), q_pe.data_ptr(),
                             cache_ptr, self.page_table.data_ptr(), self.kv_len_arr_buf.data_ptr(), out.data_ptr(),
                             lse.data_ptr() if lse is not None else None, self.workspace.data_ptr(), self.workspace.numel())
        native.check(native.lib().ktb200_mla_decode(C.byref(p), torch.cuda.current_stream(q_nope.device).cuda_stream))
        return (out, lse) if return_lse else out

    def _run_chunk(self, q_nope, q_pe, ckv, k_pe, return_lse):
        rows = self.batch * self.q_len
        assert q_nope.shape[0] == rows and q_pe.shape[0] == rows, f"a chunk of q_len {self.q_len} for {self.batch} sequences has {rows} query rows"
        cache_ptr = ckv.data_ptr()
        assert ckv.stride(-1) == 1 and k_pe.data_ptr() == cache_ptr + 512 * ckv.element_size(), \
            "ckv / k_pe must be the [..., :512] / [..., 512:] views of one 576-wide latent cache"
        q_nope, q_pe = q_nope.contiguous(), q_pe.contiguous()
        out = torch.empty_like(q_nope)
        lse = torch.empty((rows, self.num_heads), dtype=torch.float32, device=q_nope.device) if return_lse else None
        p = native.MlaChunkParams(self.batch, self.q_len, self.num_heads, self.page_size, self.max_pages, 0, self.sm_scale,
                                  q_nope.data_ptr(), q_pe.data_ptr(), cache_ptr, self.page_table.data_ptr(), self.kv_len_arr_buf.data_ptr(),
                                  out.data_ptr(), lse.data_ptr() if lse is not None else None, self.workspace.data_ptr(), self.workspace.numel(), 0)
        native.check(native.lib().ktb200_mla_decode_chunk(C.byref(p), torch.cuda.current_stream(q_nope.device).cuda_stream))
        return (out, lse) if return_lse else out


class MLAWrapperSingleton:
    wrappers: dict = {}

    @classmethod
    def get_instance(cls, device, *args, **kwargs) -> MLAWrapper:
        if device not in cls.wrappers:
            cls.wrappers[device] = MLAWrapper(*args, **kwargs, device=device)
        return cls.wrappers[device]

    @classmethod
    def plan_all(cls, *args, **kwargs):
        for w in cls.wrappers.values():
            w.plan(*args, **kwargs)

    @classmethod
    def need_plan_all(cls):
        for w in cls.wrappers.values():
            w.need_plan = True

    @classmethod
    def reset_buffer(cls):
        for w in cls.wrappers.values():
            w.page_table.zero_()
