"""ctypes face of libktb200.so — the C-ABI declared in include/ktb200.h.

This is the only door between Python and the CUDA kernels (the role pybind's ``cpuinfer_ext`` /
``kt_kernel_ext`` plays in the reference, archive/csrc/ktransformers_ext/ext_bindings.cpp,
kt-kernel/ext_bindings.cpp).  No fallback: if the library is absent, importing ``lib()`` raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libktb200.so")
CSRC = os.path.join(_HERE, "csrc")

OK, EINVAL, ECUDA, ESTATE, ENOMEM = 0, -1, -2, -3, -4

# ggml type ids (third_party/llama.cpp/ggml.h:349-380)
GGML_F32, GGML_F16, GGML_Q8_0, GGML_Q2_K, GGML_Q3_K, GGML_Q4_K, GGML_Q5_K, GGML_Q6_K, GGML_Q8_K = 0, 1, 8, 10, 11, 12, 13, 14, 15
GGML_IQ4_XS, GGML_BF16 = 23, 30
GGML_IQ2_XXS, GGML_IQ1_S, GGML_IQ1_M = 16, 19, 29   # codebook i-quants: routed experts only
GGML_IQ3_XXS, GGML_IQ3_S = 18, 21
GGML_IQ2_XS, GGML_IQ2_S = 17, 22
# not a ggml id (include/ktb200.h): symmetric INT4, group 32, bf16 scales, in the layout ktb200_rawint4_pack writes
RAWINT4_G32 = 256


class MoeConfig(C.Structure):
    """struct ktb200_moe_config (mirrors cpuinfer_ext.moe.MOEConfig, archive ext_bindings.cpp:683-695)."""
    _fields_ = [("expert_num", C.c_int), ("routed_expert_num", C.c_int), ("hidden_size", C.c_int),
                ("intermediate_size", C.c_int), ("stride", C.c_int), ("group_min_len", C.c_int),
                ("group_max_len", C.c_int), ("use_silu", C.c_int), ("gate_proj", C.c_void_p), ("up_proj", C.c_void_p),
                ("down_proj", C.c_void_p), ("gate_type", C.c_int), ("up_type", C.c_int), ("down_type", C.c_int),
                ("hidden_type", C.c_int), ("expert_id_offset", C.c_int)]


class GateConfig(C.Structure):
    _fields_ = [("n_experts", C.c_int), ("hidden_size", C.c_int), ("top_k", C.c_int), ("n_group", C.c_int),
                ("topk_group", C.c_int), ("scoring", C.c_int), ("topk_method", C.c_int), ("norm_topk_prob", C.c_int),
                ("routed_scaling_factor", C.c_float), ("weight", C.c_void_p), ("bias", C.c_void_p),
                ("hidden_type", C.c_int)]


class MlaParams(C.Structure):
    _fields_ = [("batch", C.c_int), ("num_heads", C.c_int), ("page_size", C.c_int), ("max_pages_per_seq", C.c_int),
                ("num_kv_splits", C.c_int), ("sm_scale", C.c_float), ("q_nope", C.c_void_p), ("q_pe", C.c_void_p),
                ("kv_cache", C.c_void_p), ("page_table", C.c_void_p), ("kv_len", C.c_void_p), ("out", C.c_void_p),
                ("lse_out", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("kv_cache_rows", C.c_long)]


class MlaChunkParams(C.Structure):
    """struct ktb200_mla_chunk_params (include/ktb200.h)."""
    _fields_ = [("batch", C.c_int), ("q_len", C.c_int), ("num_heads", C.c_int), ("page_size", C.c_int), ("max_pages_per_seq", C.c_int),
                ("num_kv_splits", C.c_int), ("sm_scale", C.c_float), ("q_nope", C.c_void_p), ("q_pe", C.c_void_p),
                ("kv_cache", C.c_void_p), ("page_table", C.c_void_p), ("kv_len", C.c_void_p), ("out", C.c_void_p),
                ("lse_out", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("kv_cache_rows", C.c_long)]


class MlaRaggedParams(C.Structure):
    """struct ktb200_mla_ragged_params (include/ktb200.h)."""
    _fields_ = [("rows", C.c_int), ("max_items", C.c_int), ("num_heads", C.c_int), ("page_size", C.c_int), ("max_pages_per_seq", C.c_int),
                ("sm_scale", C.c_float), ("q_nope", C.c_void_p), ("q_pe", C.c_void_p), ("kv_cache", C.c_void_p),
                ("page_table", C.c_void_p), ("plan", C.c_void_p), ("out", C.c_void_p), ("lse_out", C.c_void_p),
                ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t), ("kv_cache_rows", C.c_long)]


class MlaPrefillParams(C.Structure):
    """struct ktb200_mla_prefill_params (include/ktb200.h); strides in elements, token / head / batch."""
    _fields_ = [("batch", C.c_int), ("q_len", C.c_int), ("kv_len", C.c_int), ("num_heads", C.c_int),
                ("qk_nope_head_dim", C.c_int), ("qk_rope_head_dim", C.c_int), ("v_head_dim", C.c_int), ("sm_scale", C.c_float),
                ("q_nope", C.c_void_p), ("q_nope_token_stride", C.c_long), ("q_nope_head_stride", C.c_long), ("q_nope_batch_stride", C.c_long),
                ("q_pe", C.c_void_p), ("q_pe_token_stride", C.c_long), ("q_pe_head_stride", C.c_long), ("q_pe_batch_stride", C.c_long),
                ("k_nope", C.c_void_p), ("k_nope_token_stride", C.c_long), ("k_nope_head_stride", C.c_long), ("k_nope_batch_stride", C.c_long),
                ("v", C.c_void_p), ("v_token_stride", C.c_long), ("v_head_stride", C.c_long), ("v_batch_stride", C.c_long),
                ("k_pe", C.c_void_p), ("k_pe_token_stride", C.c_long), ("k_pe_batch_stride", C.c_long),
                ("out", C.c_void_p)]


MLA_PREFILL_VARLEN_MAX_BATCH = 1024


class MlaPrefillVarlenParams(C.Structure):
    """struct ktb200_mla_prefill_varlen_params (include/ktb200.h); seq is a HOST int32 [batch][4] {q_row, q_len, k_row,
    kv_len}; strides in elements, token / head."""
    _fields_ = [("batch", C.c_int), ("q_rows", C.c_int), ("k_rows", C.c_int), ("num_heads", C.c_int),
                ("qk_nope_head_dim", C.c_int), ("qk_rope_head_dim", C.c_int), ("v_head_dim", C.c_int), ("sm_scale", C.c_float),
                ("seq", C.c_void_p),
                ("q_nope", C.c_void_p), ("q_nope_token_stride", C.c_long), ("q_nope_head_stride", C.c_long),
                ("q_pe", C.c_void_p), ("q_pe_token_stride", C.c_long), ("q_pe_head_stride", C.c_long),
                ("k_nope", C.c_void_p), ("k_nope_token_stride", C.c_long), ("k_nope_head_stride", C.c_long),
                ("v", C.c_void_p), ("v_token_stride", C.c_long), ("v_head_stride", C.c_long),
                ("k_pe", C.c_void_p), ("k_pe_token_stride", C.c_long),
                ("out", C.c_void_p)]


_lib = None
_lock = threading.Lock()

# every symbol include/ktb200.h declares: (name, restype, argtypes)
_VP, _I, _L = C.c_void_p, C.c_int, C.c_long
SYMBOLS = {
    "ktb200_last_error": (C.c_char_p, []),
    "ktb200_version": (C.c_char_p, []),
    "ktb200_type_size": (_L, [_I]),
    "ktb200_blck_size": (_L, [_I]),
    "ktb200_launch_count": (C.c_ulonglong, []),
    "ktb200_moe_create": (_I, [C.POINTER(MoeConfig), _I, C.POINTER(_VP)]),
    "ktb200_moe_destroy": (None, [_VP]),
    "ktb200_moe_load_weights": (_I, [_VP, _VP]),
    "ktb200_moe_warm_up": (_I, [_VP, _VP]),
    "ktb200_moe_forward": (_I, [_VP, _I, _I, _VP, _VP, _VP, _VP, _VP, _VP]),
    "ktb200_moe_forward_host": (_I, [_VP, _I, _I, _VP, _VP, _VP, _VP, _VP]),
    "ktb200_moe_forward_timed": (_I, [_VP, _I, _I, _VP, _VP, _VP, _VP, _VP, C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "ktb200_moe_intermediate": (_VP, [_VP]),
    "ktb200_fp8_linear_create": (_I, [_I, _I, _VP, _VP, _I, _I, C.POINTER(_VP)]),
    "ktb200_fp8_linear_destroy": (None, [_VP]),
    "ktb200_fp8_linear_forward": (_I, [_VP, _I, _VP, _VP, _VP, _VP]),
    "ktb200_linear_create": (_I, [_I, _I, _VP, _I, _I, _I, _I, C.POINTER(_VP)]),
    "ktb200_linear_destroy": (None, [_VP]),
    "ktb200_linear_load_weights": (_I, [_VP, _VP]),
    "ktb200_linear_forward": (_I, [_VP, _I, _VP, _VP, _VP, _VP, _VP]),
    "ktb200_linear_forward_prompt": (_I, [_VP, _I, _VP, _VP, _VP, _VP, _VP]),
    "ktb200_linear_prompt_min": (_I, [_VP]),
    "ktb200_mlp_create": (_I, [_I, _I, _VP, _VP, _VP, _I, _I, _I, _I, _I, _I, C.POINTER(_VP)]),
    "ktb200_mlp_destroy": (None, [_VP]),
    "ktb200_mlp_load_weights": (_I, [_VP, _VP]),
    "ktb200_mlp_forward": (_I, [_VP, _I, _VP, _VP, _I, _VP, _VP]),
    "ktb200_moe_forward_shared": (_I, [_VP, _VP, _I, _I, _VP, _VP, _VP, _VP, _VP, _VP]),
    "ktb200_quantize_activations": (_I, [_VP, _I, _L, _L, _I, _VP, _VP]),
    "ktb200_dequantize": (_I, [_VP, _I, _L, _VP, _I, _VP]),
    "ktb200_rawint4_pack": (_I, [_VP, _VP, _L, _L, _VP, _VP]),
    "ktb200_moe_gate_forward": (_I, [C.POINTER(GateConfig), _I, _VP, _VP, _VP, _VP, _VP, _VP]),
    "ktb200_moe_block_forward": (_I, [C.POINTER(GateConfig), _VP, _VP, _I, _VP, _VP, _VP, _VP, _VP, _VP]),
    "ktb200_moe_block_forward_host": (_I, [C.POINTER(GateConfig), _VP, _VP, _I, _VP, _VP, _VP, _VP, _VP]),
    "ktb200_moe_forward_ep": (_I, [_VP, _VP, _I, _I, _VP, _VP, _VP, _VP, _I, _VP, _VP, _VP]),
    "ktb200_ep_all_gather_tokens": (_I, [_VP, _VP, _VP, _VP]),
    "ktb200_ep_reduce_own_token": (_I, [_VP, _VP, _VP, _VP]),
    "ktb200_moe_block_prefetch_hint": (_I, [_VP, _VP, _VP, _I]),
    "ktb200_ep_msg_bytes": (_L, [_I, _I]),
    "ktb200_moe_ep_block_forward": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _I, _VP]),
    "ktb200_ep_tokens_layout": (_L, [_I, _I, _I, _I, _I, _VP]),
    "ktb200_moe_ep_forward_tokens": (_I, [_VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _VP, _I, _VP]),
    "ktb200_debug_block_trace": (None, [_VP]),
    "ktb200_debug_block_sync_words": (_L, [_VP, _VP, _L]),
    "ktb200_debug_gate_ticket": (_I, [_I, _VP]),
    "ktb200_debug_stream_read": (_I, [_VP, _L, _I, _I, _I, _I, _VP, C.POINTER(C.c_float)]),
    "ktb200_mla_workspace_bytes": (C.c_size_t, [_I, _I, _I]),
    "ktb200_mla_decode": (_I, [C.POINTER(MlaParams), _VP]),
    "ktb200_debug_mla": (None, [_VP]),
    "ktb200_mla_chunk_workspace_bytes": (C.c_size_t, [_I, _I, _I, _I]),
    "ktb200_mla_decode_chunk": (_I, [C.POINTER(MlaChunkParams), _VP]),
    "ktb200_mla_ragged_plan_ints": (C.c_size_t, [_I, _I]),
    "ktb200_mla_ragged_workspace_bytes": (C.c_size_t, [_I, _I]),
    "ktb200_mla_ragged_plan": (_I, [_VP, _VP, _I, _I, _I, _I, _I, _I, _I, _I, _VP, C.c_size_t, C.POINTER(_I), C.POINTER(C.c_size_t)]),
    "ktb200_mla_decode_ragged": (_I, [C.POINTER(MlaRaggedParams), _VP]),
    "ktb200_mla_prefill": (_I, [C.POINTER(MlaPrefillParams), _VP]),
    "ktb200_mla_prefill_varlen": (_I, [C.POINTER(MlaPrefillVarlenParams), _VP]),
    "ktb200_debug_grouped": (None, [_VP]),
    "ktb200_mla_absorb_q": (_I, [_VP, _L, _L, _VP, _I, _I, _I, _VP, _I, _VP]),
    "ktb200_mla_absorb_o": (_I, [_VP, _VP, _I, _I, _I, _VP, _I, _VP]),
    "ktb200_add_rmsnorm": (_I, [_VP, _VP, _VP, C.c_float, _VP, _I, _I, _VP]),
    "ktb200_mla_prep": (_I, [_VP, _I, _I, _VP, _VP, C.c_float, _VP, _VP, _VP, _I, _VP, _VP, _VP, _I, _VP]),
    "ktb200_mla_kv_write": (_I, [_VP, _I, _VP, _VP, _VP, _VP, _I, _VP]),
}


class EpComm(C.Structure):
    """ktb200_ep_comm (include/ktb200.h): peer-mapped token / partial / flag buffers of an expert-parallel group."""
    _fields_ = [("rank", C.c_int), ("world", C.c_int), ("hidden_size", C.c_int), ("hidden_type", C.c_int),
                ("token_bufs", C.POINTER(C.c_void_p)), ("partial_bufs", C.POINTER(C.c_void_p)), ("flag_bufs", C.POINTER(C.c_void_p))]

    @classmethod
    def make(cls, rank, world, hidden_size, hidden_type, tok_ptrs, part_ptrs, flag_ptrs):
        arr = lambda ps: (C.c_void_p * world)(*[int(x) for x in ps])
        c = cls(rank, world, hidden_size, hidden_type)
        c._keep = (arr(tok_ptrs), arr(part_ptrs), arr(flag_ptrs))      # the host arrays must outlive the struct
        c.token_bufs, c.partial_bufs, c.flag_bufs = (C.cast(a, C.POINTER(C.c_void_p)) for a in c._keep)
        return c


class EpTokensComm(C.Structure):
    """ktb200_ep_tokens_comm (include/ktb200.h): every rank's region of the multi-token expert-parallel layer."""
    _fields_ = [("rank", C.c_int), ("world", C.c_int), ("max_tokens_per_rank", C.c_int), ("hidden_size", C.c_int),
                ("hidden_type", C.c_int), ("top_k", C.c_int), ("bufs", C.POINTER(C.c_void_p))]

    @classmethod
    def make(cls, rank, world, max_tokens_per_rank, hidden_size, hidden_type, top_k, buf_ptrs):
        c = cls(rank, world, max_tokens_per_rank, hidden_size, hidden_type, top_k)
        c._keep = (C.c_void_p * world)(*[int(x) for x in buf_ptrs])      # the host array must outlive the struct
        c.bufs = C.cast(c._keep, C.POINTER(C.c_void_p))
        return c


EP_TOKENS_REGIONS = ("x", "ids", "weights", "partial", "scratch", "flags")


def ep_tokens_layout(world: int, max_tokens_per_rank: int, hidden_size: int, hidden_type: int, top_k: int) -> tuple[int, dict]:
    """(bytes, {region: byte offset}) of one rank's region of ktb200_moe_ep_forward_tokens."""
    off = (C.c_long * 6)()
    n = lib().ktb200_ep_tokens_layout(world, max_tokens_per_rank, hidden_size, hidden_type, top_k, off)
    if n < 0:
        check(EINVAL)
    return int(n), dict(zip(EP_TOKENS_REGIONS, (int(o) for o in off)))


def build(verbose: bool = False) -> str:
    """Compile libktb200.so for sm_90a with nvcc (cross-compiles without a GPU)."""
    out = None if verbose else subprocess.DEVNULL
    subprocess.check_call(["make", "-C", CSRC, "-j", "4"], stdout=out)
    return LIB_PATH


def lib() -> C.CDLL:
    """Load the CUDA library; raise (never fall back) when it is missing."""
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise RuntimeError(
                        f"{LIB_PATH} is missing: the H100 path has no CPU fallback. Build it with "
                        "`python -c 'import __graft_entry__ as g; g.build()'` or `make -C ktransformers_b200/csrc`.")
                l = C.CDLL(LIB_PATH)
                for name, (res, args) in SYMBOLS.items():
                    fn = getattr(l, name)  # AttributeError if the .so does not export a declared symbol
                    fn.restype = res
                    fn.argtypes = args
                _lib = l
    return _lib


class KTB200Error(RuntimeError):
    pass


def check(rc: int) -> None:
    """Map C-ABI return codes onto the reference's Python-visible errors (SURVEY §8b error convention)."""
    if rc == OK:
        return
    msg = lib().ktb200_last_error().decode(errors="replace")
    if rc == EINVAL:
        raise ValueError(msg)          # e.g. invalid ggml_type -> ValueError (kt-kernel/ext_bindings.cpp:88-92)
    if rc == ENOMEM:
        raise MemoryError(msg)
    raise KTB200Error(msg)             # "Not Loaded" (moe-tp.hpp:203-205), CUDA errors


def launch_count() -> int:
    return int(lib().ktb200_launch_count())


def type_size(ggml_type: int) -> int:
    """Bytes per block of a weight type (ktb200_type_size; 144 for RAWINT4_G32), 0 when unsupported."""
    return int(lib().ktb200_type_size(int(ggml_type)))
