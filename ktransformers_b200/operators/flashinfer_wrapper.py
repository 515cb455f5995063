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
written.

A qo_indptr whose sequences have different lengths (decode tokens and prompt chunks, a q_len of 0 included) plans the
ragged path: ktb200_mla_ragged_plan fills a pinned host buffer with a work list, which is copied on the current stream into
a device buffer of fixed size; run() takes the [rows, H, 512] / [rows, H, 64] queries in qo_indptr order and calls
ktb200_mla_decode_ragged, one launch over the item capacity that a CUDA graph can capture and replay after later plans.
Host qo_indptr / kv_len_arr cost no synchronisation; device ones cost one each.  The row and item capacities are the
constructor's max_rows / max_items, fixed for the wrapper's life."""
from __future__ import annotations

import ctypes as C

import torch

from .. import native


class MLAWrapper:
    def __init__(self, max_batch_size, max_pages, use_cuda_graph=True, device="cuda", max_rows=1024, max_items=4096):
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
        self.max_rows, self.max_items = max_rows, max_items
        self.ragged = False
        self.rows = 0               # query rows of the current ragged plan
        self.plan_host = self.plan_dev = self.plan_copied = None   # created by the first ragged plan

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
            assert len(q_lens) == self.batch, f"qo_indptr has {len(q_lens)} sequences, kv_indptr {self.batch}"
            if len(set(q_lens)) > 1:
                self._plan_ragged(qo_indptr, kv_indptr, kv_indices, kv_len_arr, num_heads, page_size, sm_scale)
                return
            assert q_lens[0] >= 1, f"every sequence must have the same q_len >= 1, got {q_lens}"
            q_len = int(q_lens[0])
        self._dense_page_table(kv_indptr, kv_indices)
        self.kv_len_arr_buf[: self.batch].copy_(kv_len_arr[: self.batch].to(torch.int32), non_blocking=True)   # a host kv_len: no stream sync
        self.num_heads, self.page_size, self.sm_scale = num_heads, page_size, float(sm_scale)
        need = native.lib().ktb200_mla_workspace_bytes(self.max_batch_size, num_heads, 0)
        if q_len > 1:   # the most splits the chunk entry picks by itself: ceil(SMs / (batch * q_len * head groups)), <= 128
            sms = torch.cuda.get_device_properties(torch.device(self.device)).multi_processor_count
            splits = min(128, -(-sms // (self.batch * q_len * -(-num_heads // 64))))
            need = max(need, native.lib().ktb200_mla_chunk_workspace_bytes(self.batch, q_len, num_heads, splits))
        self.q_len, self.ragged = q_len, False
        if self.workspace is None or self.workspace.numel() < need:
            self.workspace = torch.empty(need, dtype=torch.uint8, device=self.device)
        self.need_plan = False

    def _dense_page_table(self, kv_indptr, kv_indices):
        """CSR -> dense page table (device-side torch ops; no host sync)"""
        counts = (kv_indptr[1:] - kv_indptr[:-1]).to(torch.int64)
        col = torch.arange(self.max_pages, device=self.device).unsqueeze(0)
        src = (kv_indptr[:-1].to(torch.int64).unsqueeze(1) + col).clamp_(max=max(int(kv_indices.numel()) - 1, 0))
        table = kv_indices.to(torch.int32)[src]
        self.page_table[: self.batch].copy_(torch.where(col < counts.unsqueeze(1), table, torch.zeros_like(table)))

    def _plan_ragged(self, qo_indptr, kv_indptr, kv_indices, kv_len_arr, num_heads, page_size, sm_scale):
        lib = native.lib()
        cuda = torch.device(self.device).type == "cuda"
        if self.plan_host is None:
            n = lib.ktb200_mla_ragged_plan_ints(self.max_items, self.max_rows)
            self.plan_host = torch.zeros(n, dtype=torch.int32, pin_memory=cuda)
            self.plan_dev = torch.zeros(n, dtype=torch.int32, device=self.device)
            self.plan_copied = torch.cuda.Event() if cuda else None
        elif self.plan_copied is not None:
            self.plan_copied.synchronize()   # the previous plan's copy may still read the pinned buffer
        qo = qo_indptr.to("cpu", torch.int32).contiguous()
        kv_len = kv_len_arr[: self.batch].to("cpu", torch.int32).contiguous()   # a device kv_len_arr costs one synchronisation
        # a wrapper on the CPU only plans (the planner is host code): it balances for the H100's 132 SMs
        sms = torch.cuda.get_device_properties(torch.device(self.device)).multi_processor_count if cuda else 132
        slots, ws = C.c_int(), C.c_size_t()
        native.check(lib.ktb200_mla_ragged_plan(qo.data_ptr(), kv_len.data_ptr(), self.batch, num_heads, page_size, self.max_pages, sms,
                                                0, self.max_items, self.max_rows, self.plan_host.data_ptr(),
                                                self.plan_host.numel(), C.byref(slots), C.byref(ws)))
        # the header and the items in use, then the row offsets (they sit after the item capacity)
        items, self.rows = int(self.plan_host[0]), int(self.plan_host[1])
        head, off = 8 + 8 * items, 8 + 8 * self.max_items
        self.plan_dev[:head].copy_(self.plan_host[:head], non_blocking=True)
        self.plan_dev[off:off + self.rows + 1].copy_(self.plan_host[off:off + self.rows + 1], non_blocking=True)
        if self.plan_copied is not None:
            self.plan_copied.record()
        self._dense_page_table(kv_indptr, kv_indices)
        self.num_heads, self.page_size, self.sm_scale = num_heads, page_size, float(sm_scale)
        need = lib.ktb200_mla_ragged_workspace_bytes(self.max_items, num_heads)
        if self.workspace is None or self.workspace.numel() < need:
            self.workspace = torch.empty(need, dtype=torch.uint8, device=self.device)
        self.q_len, self.ragged = 0, True   # q_len 0: no uniform q_len, so KDeepseekV2Attention.forward re-plans
        self.need_plan = False

    def run(self, q_nope, q_pe, ckv, k_pe, return_lse=False):
        assert not self.need_plan, "plan() before run()"
        if self.ragged:
            return self._run_ragged(q_nope, q_pe, ckv, k_pe, return_lse)
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

    def _run_ragged(self, q_nope, q_pe, ckv, k_pe, return_lse):
        """no host synchronisation and nothing that depends on the plan's contents: a CUDA graph can capture it and replay
        it after later plans of at most q_nope.shape[0] rows"""
        rows = q_nope.shape[0]
        assert q_pe.shape[0] == rows and rows >= self.rows, f"the plan has {self.rows} query rows, q_nope {rows}"
        cache_ptr = ckv.data_ptr()
        assert ckv.stride(-1) == 1 and k_pe.data_ptr() == cache_ptr + 512 * ckv.element_size(), \
            "ckv / k_pe must be the [..., :512] / [..., 512:] views of one 576-wide latent cache"
        q_nope, q_pe = q_nope.contiguous(), q_pe.contiguous()
        out = torch.empty_like(q_nope)
        lse = torch.empty((rows, self.num_heads), dtype=torch.float32, device=q_nope.device) if return_lse else None
        p = native.MlaRaggedParams(rows, self.max_items, self.num_heads, self.page_size, self.max_pages, self.sm_scale,
                                   q_nope.data_ptr(), q_pe.data_ptr(), cache_ptr, self.page_table.data_ptr(), self.plan_dev.data_ptr(),
                                   out.data_ptr(), lse.data_ptr() if lse is not None else None, self.workspace.data_ptr(),
                                   self.workspace.numel(), 0)
        native.check(native.lib().ktb200_mla_decode_ragged(C.byref(p), torch.cuda.current_stream(q_nope.device).cuda_stream))
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
