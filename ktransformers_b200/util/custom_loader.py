"""GGUF weight loader.  Behavioural mirror of GGUFLoader / ModelLoaderFactory
(archive/ktransformers/util/custom_loader.py:278-526, 531-598) for the GGUF container:

* every ``*.gguf`` under a directory is indexed (header parse, 32-byte aligned data offsets) and
  memory-mapped; tensors are addressed by HF module path through ``translate_name_to_gguf``;
* ``get_mmap_tensor`` hands out the raw ggml block bytes (what KExperts*/KLinear* upload to HBM);
* ``load_gguf_tensor`` returns a dense tensor; on a CUDA device the blocks are uploaded in chunks and
  dequantised by libktb200 (``ktb200_dequantize``) — the reference calls
  ``KTransformersOps.dequantize_*`` there (custom_loader.py:474-493);
* ``tensor_device_map`` is filled by ``inject`` and read by ``get_device``.
"""
from __future__ import annotations

import json
import math
import os
import struct
import warnings
from typing import BinaryIO, Dict

import numpy as np
import torch

from .custom_gguf import (DATA_TYPES, GGML_BLOCK_SIZES, GGML_ELEMENTS_PER_BLOCK, GGML_NAMES, GGML_QUANT_SIZES,
                          B200_DEQUANT_TYPES, GGMLQuantizationType, dequantize_cpu, quant_shape_to_byte_shape,
                          translate_name_to_gguf)

_SCALAR_FMT = {0: "<B", 1: "<b", 2: "<H", 3: "<h", 4: "<I", 5: "<i", 6: "<f", 7: "<?", 10: "<Q", 11: "<q", 12: "<d"}
_PLAIN_NP = {GGMLQuantizationType.F16: np.float16, GGMLQuantizationType.F32: np.float32,
             GGMLQuantizationType.F64: np.float64, GGMLQuantizationType.I8: np.int8, GGMLQuantizationType.I16: np.int16,
             GGMLQuantizationType.I32: np.int32, GGMLQuantizationType.I64: np.int64}
_TORCH_TO_GGML_OUT = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 30}


def read_value(f: BinaryIO, data_type: int):
    if data_type == DATA_TYPES["string"]:
        (length,) = struct.unpack("<Q", f.read(8))
        return f.read(length).decode("utf-8", errors="replace")
    if data_type == DATA_TYPES["array"]:
        elem_type, count = struct.unpack("<IQ", f.read(12))
        return [read_value(f, elem_type) for _ in range(count)]
    fmt = _SCALAR_FMT.get(data_type)
    if fmt is None:
        raise NotImplementedError(f"GGUF metadata type {data_type} not implemented")
    return struct.unpack(fmt, f.read(struct.calcsize(fmt)))[0]


class ModelLoader:
    tensor_file_map: Dict[str, str]
    tensor_device_map: Dict[str, dict]

    def has_tensor(self, name: str) -> bool:  # pragma: no cover - interface
        raise NotImplementedError


class GGUFLoader(ModelLoader):
    def __init__(self, gguf_path: str, quantize: str = None):
        if not os.path.exists(gguf_path):
            raise FileNotFoundError(f"GGUF dir not found: {gguf_path}")
        if os.path.isfile(gguf_path):
            gguf_path = os.path.dirname(gguf_path)
        self.safetensor_loader = None
        self.tensor_info: Dict[str, dict] = {}
        self.gguf_path = gguf_path
        self.tensor_file_map: Dict[str, str] = {}
        self.file_data_map: Dict[str, np.memmap] = {}
        self.gguf_file_meta: Dict[str, object] = {}
        self.tensor_device_map: Dict[str, dict] = {}
        found = False
        for root, _, files in os.walk(gguf_path):
            for fn in sorted(files):
                if fn.endswith(".gguf"):
                    found = True
                    path = os.path.join(root, fn)
                    with open(path, "rb") as f:
                        self.load_gguf(f)
                    self.file_data_map.setdefault(path, np.memmap(path, mode="r"))
        if not found:
            raise FileNotFoundError(f"Cannot find any .gguf files in: {gguf_path}")

    # -- header ------------------------------------------------------------------------------------
    def load_gguf(self, f: BinaryIO) -> None:
        f.seek(0)
        if f.read(4) != b"GGUF":
            raise ValueError(f"{f.name}: not a GGUF file")
        version, n_tensors, n_kv = struct.unpack("<IQQ", f.read(20))
        if version != 3:
            warnings.warn(f"Version {version} has never been tested, might not work")
        info = {}
        for _ in range(n_kv):
            key = read_value(f, DATA_TYPES["string"])
            (vt,) = struct.unpack("<I", f.read(4))
            info[key] = read_value(f, vt)
        tensor_info = {}
        for _ in range(n_tensors):
            name = read_value(f, DATA_TYPES["string"])
            ndim = read_value(f, DATA_TYPES["uint32"])
            shape = [read_value(f, DATA_TYPES["uint64"]) for _ in range(ndim)]
            ggml_type = read_value(f, DATA_TYPES["uint32"])
            rel_offset = read_value(f, DATA_TYPES["uint64"])
            n_elems = int(math.prod(shape))
            epb, bpb = GGML_QUANT_SIZES[GGMLQuantizationType(ggml_type)]
            np_dims = tuple(reversed(shape))
            qt = GGMLQuantizationType(ggml_type)
            if qt in _PLAIN_NP:
                item_type, item_count = _PLAIN_NP[qt], n_elems
            else:
                item_type, item_count = np.uint8, n_elems * bpb // epb
                np_dims = quant_shape_to_byte_shape(np_dims, ggml_type)
            tensor_info[name] = {"ggml_type": ggml_type, "shape": shape, "bad_offset": rel_offset, "item_type": item_type,
                                 "item_count": item_count, "np_dims": np_dims}
        data_start = f.tell()
        alignment = info.get("general.alignment", 32)
        for t in tensor_info.values():
            off = data_start + t["bad_offset"]
            t["offset"] = off + (alignment - off % alignment) % alignment
        for name in tensor_info:
            self.tensor_file_map[name] = f.name
        self.tensor_info.update(tensor_info)
        self.gguf_file_meta.update(info)

    # -- raw access --------------------------------------------------------------------------------
    def has_tensor(self, name: str) -> bool:
        return translate_name_to_gguf(name) in self.tensor_info

    def get_ggml_type(self, name: str) -> int:
        name = translate_name_to_gguf(name)
        if name not in self.tensor_info:
            raise KeyError(f"Key {name} not found in GGUF files")
        return self.tensor_info[name]["ggml_type"]

    def get_mmap_tensor(self, name: str) -> np.ndarray:
        name = translate_name_to_gguf(name)
        t = self.tensor_info[name]
        data = self.file_data_map[self.tensor_file_map[name]]
        itemsize = int(np.dtype(t["item_type"]).itemsize)
        return data[t["offset"]: t["offset"] + itemsize * t["item_count"]]

    def get_undequanted_tensor_and_ggml_type(self, name: str):
        name = translate_name_to_gguf(name)
        return torch.from_numpy(np.asarray(self.get_mmap_tensor(name))), self.tensor_info[name]["ggml_type"]

    def load_raw_to_device(self, name: str, device: str) -> torch.Tensor:
        """Upload the raw ggml blocks of a tensor to HBM as a flat uint8 tensor (no dequantisation)."""
        raw = np.asarray(self.get_mmap_tensor(name))
        return torch.from_numpy(raw.view(np.uint8) if raw.dtype != np.uint8 else raw).to(device)

    # -- dense tensors -----------------------------------------------------------------------------
    def _dequant(self, data: np.ndarray, ggml_type: int, n_elements: int, device: str, target_dtype) -> torch.Tensor:
        ggml_name = GGML_NAMES[ggml_type]
        if "cuda" in str(device).lower():
            if ggml_name not in B200_DEQUANT_TYPES:
                raise NotImplementedError(f"ggml_type {ggml_name} has no sm_90a dequantiser")
            from .. import native
            out_dtype = target_dtype if target_dtype in _TORCH_TO_GGML_OUT else torch.float32
            raw = torch.from_numpy(np.ascontiguousarray(data).view(np.uint8)).to(device)
            out = torch.empty(n_elements, dtype=out_dtype, device=device)
            stream = torch.cuda.current_stream(out.device).cuda_stream
            with torch.cuda.device(out.device):
                native.check(native.lib().ktb200_dequantize(raw.data_ptr(), int(ggml_type), n_elements, out.data_ptr(),
                                                            _TORCH_TO_GGML_OUT[out_dtype], stream))
            return out if out_dtype == target_dtype else out.to(target_dtype)
        vals = dequantize_cpu(np.asarray(data), ggml_type)
        t = torch.from_numpy(np.array(vals, copy=True))
        if ggml_name == "BF16":
            t = t.view(torch.bfloat16)
        return t.to(target_dtype) if target_dtype is not None and t.dtype != target_dtype else t

    def load_gguf_tensor(self, name: str, device: str = "cpu", target_dtype=None) -> torch.Tensor:
        name = translate_name_to_gguf(name)
        t = self.tensor_info[name]
        if target_dtype is None:
            target_dtype = torch.get_default_dtype()
        ggml_type = t["ggml_type"]
        if ggml_type not in GGML_NAMES:
            raise NotImplementedError(f"ggml_type {ggml_type} not implemented")
        ggml_name = GGML_NAMES[ggml_type]
        data = self.get_mmap_tensor(name)
        bpb, epb = GGML_BLOCK_SIZES[ggml_name], GGML_ELEMENTS_PER_BLOCK[ggml_name]
        n_elems = int(np.prod(t["shape"]))
        n_blocks = n_elems // epb
        raw = np.asarray(data).view(np.uint8)
        chunk = 1 << 20  # blocks per upload
        if n_blocks > chunk:
            values = torch.empty(n_elems, dtype=target_dtype, device=device)
            for b0 in range(0, n_blocks, chunk):
                b1 = min(b0 + chunk, n_blocks)
                values[b0 * epb: b1 * epb] = self._dequant(raw[b0 * bpb: b1 * bpb], ggml_type, (b1 - b0) * epb, device, target_dtype)
        else:
            values = self._dequant(raw, ggml_type, n_elems, device, target_dtype).to(device)
        values = values.view(t["shape"][::-1])
        arch = self.gguf_file_meta.get("general.architecture")
        if arch == "llama" and ("attn_q" in name or "attn_k" in name):
            # llama.cpp permutes q/k rows for its rope layout; undo it (custom_loader.py:508-517)
            n_head = self.gguf_file_meta["llama.attention.head_count" if "attn_q" in name else "llama.attention.head_count_kv"]
            values = (values.reshape(n_head, values.shape[0] // n_head // 2, 2, *values.shape[1:]).swapaxes(1, 2).reshape(values.shape))
        return values

    def load_expert_tensor(self, name, data, expert_id, elements_per_expert, device="cuda", target_dtype=None) -> torch.Tensor:
        name = translate_name_to_gguf(name)
        t = self.tensor_info[name]
        ggml_type = t["ggml_type"]
        if ggml_type not in GGML_NAMES:
            raise NotImplementedError(f"ggml_type {ggml_type} not implemented")
        ggml_name = GGML_NAMES[ggml_type]
        epb, bpb = GGML_ELEMENTS_PER_BLOCK[ggml_name], GGML_BLOCK_SIZES[ggml_name]
        assert elements_per_expert % epb == 0, "experts may fused in quant block, please use CPU dequant"
        nb = elements_per_expert // epb
        raw = np.asarray(data).view(np.uint8)[expert_id * bpb * nb: (expert_id + 1) * bpb * nb]
        if target_dtype is None:
            target_dtype = torch.get_default_dtype()
        values = self._dequant(raw, ggml_type, elements_per_expert, device, target_dtype)
        return values.view(t["shape"][-2::-1])


class SafeTensorLoader(ModelLoader):
    """custom_loader.py:52-112: key -> file map over a directory of *.safetensors, `load_tensor(key, device)`; what KLinearFP8 needs
    to find `<key>.weight` (float8_e4m3fn) and `<key>.weight_scale_inv`.  (The FP8 + GGUF hybrid produced by
    archive/merge_tensors is a separate on-disk contract and not read here.)"""

    def __init__(self, file_path: str):
        from safetensors import safe_open
        self._open = safe_open
        self.tensor_file_map: dict = {}
        self.tensor_device_map: dict = {}        # filled by optimize.inject, like GGUFLoader's
        self.tensor_info: dict = {}
        root = os.path.dirname(file_path) if os.path.isfile(file_path) else file_path
        self.root = root
        found = False
        for cur, _, files in os.walk(root):
            for fn in sorted(files):
                if fn.endswith(".safetensors"):
                    found = True
                    full = os.path.join(cur, fn)
                    with safe_open(full, framework="pt") as f:
                        for k in f.keys():
                            self.tensor_file_map[k] = full
                            self.tensor_info[k] = {"shape": list(f.get_slice(k).get_shape())}
        if not found:
            raise FileNotFoundError(f"No Safetensor files found in {root}")

    # The FP8 + GGUF hybrid written by archive/merge_tensors (BASELINE configs 3 / 5): FP8 linears under their HF names
    # (`*.weight` float8_e4m3fn + `*.weight_scale_inv`), routed experts as RAW ggml blocks under their GGUF names
    # (`blk.N.ffn_{gate,up,down}_exps.weight` uint8 + a scalar `*.ggml_type`), router / norms as plain tensors under GGUF names.
    # The methods below give that file the GGUFLoader surface the operators use (custom_loader.py:114-262).
    def _resolve(self, name: str):
        if name in self.tensor_file_map:
            return name
        g = translate_name_to_gguf(name)
        return g if g in self.tensor_file_map else None

    def has_tensor(self, name: str) -> bool:
        return self._resolve(name) is not None

    def load_tensor(self, key: str, device: str = "cpu"):
        k = self._resolve(key)
        if k is None:
            raise KeyError(f"Key {key} not found in Safetensor files")
        with self._open(self.tensor_file_map[k], framework="pt") as f:
            return f.get_tensor(k).to(device)

    def get_ggml_type(self, name: str) -> int:
        k = self._resolve(name)
        tk = (k[:-len(".weight")] if k and k.endswith(".weight") else str(k)) + ".ggml_type"
        if k is None or tk not in self.tensor_file_map:
            raise KeyError(f"{name} is not stored as raw ggml blocks (no {tk})")
        return int(self.load_tensor(tk).item())

    def get_mmap_tensor(self, name: str) -> np.ndarray:
        self.get_ggml_type(name)                         # raw blocks only
        return self.load_tensor(name).contiguous().view(torch.uint8).reshape(-1).numpy()

    def load_gguf_tensor(self, name: str, device: str = "cpu", target_dtype=None) -> torch.Tensor:
        """plain (unquantised) tensors of the hybrid file: router weight, e_score_correction_bias, norms"""
        t = self.load_tensor(name, device)
        if t.dtype in (torch.uint8, torch.float8_e4m3fn):
            raise NotImplementedError(f"{name}: quantised tensors of a safetensors file are consumed raw (get_mmap_tensor / KLinearFP8), not dequantised")
        return t.to(target_dtype) if target_dtype is not None else t

    def _check_int4_quantization_config(self):
        """config.json's compressed-tensors `quantization_config`, when present, must describe the INT4 format the
        RAWINT4 kernels compute: every config group's weights are num_bits 4, group_size 32, symmetric, type int, strategy group."""
        path = os.path.join(self.root, "config.json")
        if not os.path.isfile(path):
            return
        with open(path) as f:
            qc = json.load(f).get("quantization_config")
        if qc is None:
            return
        groups = qc.get("config_groups")
        if not isinstance(groups, dict) or not groups:
            raise ValueError("quantization_config: config_groups is missing; expected compressed-tensors INT4 weights")
        want = {"num_bits": 4, "group_size": 32, "symmetric": True, "type": "int", "strategy": "group"}
        for gname, g in groups.items():
            wq = (g or {}).get("weights") or {}
            for field, val in want.items():
                if wq.get(field) != val:
                    raise ValueError(f"quantization_config: config_groups.{gname}.weights.{field} = {wq.get(field)!r}, "
                                     f"the RAWINT4 kernels need {val!r}")

    def load_experts(self, key: str, device: str = "cpu") -> dict:
        """custom_loader.py:114-148 (hybrid branch): {gate, up, down: raw ggml bytes, *_type: ggml type}.
        Per-expert compressed-tensors INT4 tensors (`{key}.{e}.{gate,up,down}_proj.{weight_packed,weight_scale,weight_shape}`,
        Kimi-K2) are stacked instead: {gate, up, down: int32 [E, rows, cols/8], *_scale: bf16 [E, rows, cols/32],
        *_type: RAWINT4_G32}."""
        if f"{key}.0.gate_proj.weight_packed" in self.tensor_file_map:
            return self._load_int4_experts(key)
        base = translate_name_to_gguf(key)
        if not self.has_tensor(base + ".ffn_gate_exps.weight"):
            raise ValueError(f"No experts found for key {key}")
        out = {}
        for n in ("gate", "up", "down"):
            out[n] = self.get_mmap_tensor(f"{base}.ffn_{n}_exps.weight")
            out[n + "_type"] = self.get_ggml_type(f"{base}.ffn_{n}_exps.weight")
        return out

    def _load_int4_experts(self, key: str) -> dict:
        from ..native import RAWINT4_G32
        self._check_int4_quantization_config()
        E = 0
        while f"{key}.{E}.gate_proj.weight_packed" in self.tensor_file_map:
            E += 1
        out = {}
        for n in ("gate", "up", "down"):
            packed, scales, shape = [], [], None
            for e in range(E):
                p = f"{key}.{e}.{n}_proj"
                for suffix in ("weight_packed", "weight_scale", "weight_shape"):
                    if f"{p}.{suffix}" not in self.tensor_file_map:
                        raise ValueError(f"{p}.{suffix} is missing")
                w, s = self.load_tensor(f"{p}.weight_packed"), self.load_tensor(f"{p}.weight_scale")
                ws = tuple(int(v) for v in self.load_tensor(f"{p}.weight_shape").reshape(-1).tolist())
                if w.dtype != torch.int32 or s.dtype != torch.bfloat16:
                    raise ValueError(f"{p}: weight_packed must be int32 and weight_scale bfloat16, got {w.dtype} / {s.dtype}")
                if len(ws) != 2 or ws[1] % 256:
                    raise ValueError(f"{p}.weight_shape {ws}: expected [rows, cols] with cols a multiple of 256")
                if tuple(w.shape) != (ws[0], ws[1] // 8) or tuple(s.shape) != (ws[0], ws[1] // 32):
                    raise ValueError(f"{p}: weight_packed {tuple(w.shape)} / weight_scale {tuple(s.shape)} do not match weight_shape {ws}")
                if shape is not None and ws != shape:
                    raise ValueError(f"{p}.weight_shape {ws} differs from expert 0's {shape}")
                shape = ws
                packed.append(w)
                scales.append(s)
            out[n], out[n + "_scale"], out[n + "_type"] = torch.stack(packed), torch.stack(scales), RAWINT4_G32
        return out

    def load_gate(self, key: str, device: str = "cpu") -> dict:
        """custom_loader.py:225-250: {'weight', 'e_score_correction_bias'} (None when absent)"""
        res = {"weight": None, "e_score_correction_bias": None}
        for k in res:
            if self.has_tensor(f"{key}.{k}"):
                res[k] = self.load_tensor(f"{key}.{k}", device)
        return res


class ModelLoaderFactory:
    """create_loader(path): GGUF directories/files -> GGUFLoader, directories of *.safetensors -> SafeTensorLoader
    (custom_loader.py:531-598)."""

    @staticmethod
    def create_loader(path: str) -> ModelLoader:
        if not os.path.exists(path):
            raise FileNotFoundError(f"Path not found: {path}")
        root = os.path.dirname(path) if os.path.isfile(path) else path
        for _, _, files in os.walk(root):
            if any(f.endswith(".gguf") for f in files):
                return GGUFLoader(path)
        for _, _, files in os.walk(root):
            if any(f.endswith(".safetensors") for f in files):
                return SafeTensorLoader(path)
        raise FileNotFoundError(f"No .gguf or .safetensors files found in: {path}")
