"""TEST INFRASTRUCTURE ONLY — ctypes faces of the two CPU checkers.

``Oracle``  -> oracle/libktoracle.so      (this repo's plain-C restatement, oracle/ktoracle.c)
``Ref``     -> oracle/_ref/libktref_*.so  (the unmodified reference sources, oracle/Makefile)

Both expose the same numpy-level helpers so a test can run one against the other.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Optional

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# ggml type ids (third_party/llama.cpp/ggml.h:349-380)
F32, F16, Q8_0, Q2_K, Q3_K, Q4_K, Q5_K, Q6_K, Q8_K, IQ4_XS, BF16 = 0, 1, 8, 10, 11, 12, 13, 14, 15, 23, 30
TYPE_NAMES = {F32: "F32", F16: "F16", Q8_0: "Q8_0", Q2_K: "Q2_K", Q3_K: "Q3_K", Q4_K: "Q4_K", Q5_K: "Q5_K",
              Q6_K: "Q6_K", Q8_K: "Q8_K", IQ4_XS: "IQ4_XS", BF16: "BF16"}
# (block bytes, block elements) — archive/ktransformers/util/custom_gguf.py:72-102
BLOCK = {F32: (4, 1), F16: (2, 1), BF16: (2, 1), Q8_0: (34, 32), Q2_K: (84, 256), Q3_K: (110, 256),
         Q4_K: (144, 256), Q5_K: (176, 256), Q6_K: (210, 256), Q8_K: (292, 256), IQ4_XS: (136, 256)}


def nbytes(n_elems: int, t: int) -> int:
    b, e = BLOCK[t]
    assert n_elems % e == 0
    return n_elems // e * b


def _p(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _hidden_np(t: int):
    return {F32: np.float32, F16: np.float16, BF16: np.uint16}[t]


def build_oracle(force: bool = False) -> str:
    so = os.path.join(HERE, "libktoracle.so")
    src = os.path.join(HERE, "ktoracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", HERE, "oracle"], stdout=subprocess.DEVNULL)
    return so


class _Common:
    """numpy helpers shared by both checkers; subclasses bind the symbol prefix."""

    lib: C.CDLL
    pfx: str

    def _f(self, name):
        return getattr(self.lib, self.pfx + name)

    def from_float(self, x: np.ndarray, t: int) -> np.ndarray:
        x = np.ascontiguousarray(x, dtype=np.float32)
        out = np.zeros(nbytes(x.size, t), np.uint8)
        self._f("from_float")(_p(x), _p(out), C.c_long(x.size), C.c_int(t))
        return out

    def to_float(self, q: np.ndarray, t: int, n: int) -> np.ndarray:
        q = np.ascontiguousarray(q)
        out = np.zeros(n, np.float32)
        self._f("to_float")(_p(q), _p(out), C.c_long(n), C.c_int(t))
        return out

    def vec_dot(self, wtype: int, n: int, w: np.ndarray, act: np.ndarray) -> float:
        fn = self._f("vec_dot")
        fn.restype = C.c_float
        if self.pfx == "ktref_":
            return float(fn(C.c_int(wtype), C.c_long(n), _p(w), _p(act)))
        return float(fn(C.c_int(wtype), C.c_long(n), _p(w), _p(act)))


class Oracle(_Common):
    """This repo's C restatement (libktoracle.so)."""

    pfx = "kto_"

    def __init__(self):
        self.lib = C.CDLL(build_oracle())
        for n in ("type_size", "blck_size"):
            self._f(n).restype = C.c_long

    def moe_forward(self, E, H, I, gate, up, down, gate_type, up_type, down_type, hidden_type, ids, weights, x,
                    use_silu=True):
        qlen, k = ids.shape
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        weights = np.ascontiguousarray(weights, dtype=np.float32)
        x = np.ascontiguousarray(x)
        out = np.zeros((qlen, H), _hidden_np(hidden_type))
        self.lib.kto_moe_forward(E, H, I, int(use_silu), _p(gate), _p(up), _p(down), gate_type, up_type, down_type,
                                 hidden_type, qlen, k, _p(ids), _p(weights), _p(x), _p(out))
        return out

    def linear_forward(self, in_size, out_size, proj, proj_type, hidden_type, x):
        x = np.ascontiguousarray(x)
        qlen = x.shape[0]
        out = np.zeros((qlen, out_size), _hidden_np(hidden_type))
        self.lib.kto_linear_forward(in_size, out_size, _p(proj), proj_type, hidden_type, qlen, _p(x), _p(out))
        return out

    def mlp_forward(self, H, I, gate, up, down, gate_type, up_type, down_type, hidden_type, x):
        x = np.ascontiguousarray(x)
        qlen = x.shape[0]
        out = np.zeros((qlen, H), _hidden_np(hidden_type))
        self.lib.kto_mlp_forward(H, I, _p(gate), _p(up), _p(down), gate_type, up_type, down_type, hidden_type, qlen,
                                 _p(x), _p(out))
        return out


def _cpu_flags() -> set:
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("flags"):
                    return set(line.split(":", 1)[1].split())
    except OSError:
        pass
    return set()


def ref_library_path() -> Optional[str]:
    """Pick the prebuilt reference library whose ISA this host can execute (None if absent)."""
    flags = _cpu_flags()
    need512 = {"avx512f", "avx512bw", "avx512dq", "avx512vl", "avx512_vnni", "avx512_bf16"}
    order = ["avx512", "avx2"] if need512 <= flags else (["avx2"] if {"avx2", "fma", "f16c"} <= flags else [])
    for isa in order:
        p = os.path.join(HERE, "_ref", f"libktref_{isa}.so")
        if os.path.exists(p):
            return p
    return None


class Ref(_Common):
    """The unmodified reference CPU path (oracle/_ref/libktref_<isa>.so via oracle/ref_shim.cpp)."""

    pfx = "ktref_"
    _inst = None

    @classmethod
    def available(cls) -> bool:
        return ref_library_path() is not None

    @classmethod
    def get(cls, threads: Optional[int] = None) -> "Ref":
        if cls._inst is None:
            cls._inst = cls()
        cls._inst.init(threads or min(os.cpu_count() or 1, 64))
        return cls._inst

    def __init__(self):
        path = ref_library_path()
        if path is None:
            raise RuntimeError("oracle/_ref is not built (run `make -C oracle ref` with REF pointing at the reference sources, see oracle/Makefile)")
        self.path = path
        self.lib = C.CDLL(path)
        for n in ("type_size", "blck_size"):
            self._f(n).restype = C.c_long
        self.lib.ktref_isa.restype = C.c_char_p
        for n in ("moe_create", "linear_create", "mlp_create"):
            self._f(n).restype = C.c_void_p
        self.threads = 0

    def init(self, threads: int) -> int:
        self.threads = int(self.lib.ktref_init(int(threads)))
        return self.threads

    def isa(self) -> str:
        return self.lib.ktref_isa().decode()

    def moe_create(self, E, k, H, I, gate, up, down, gate_type, up_type, down_type, hidden_type, stride=64,
                   group_min_len=10, group_max_len=1024, use_silu=True):
        # stride / group_* defaults are the archive's (operators/experts.py:205-209)
        h = self.lib.ktref_moe_create(E, k, H, I, stride, group_min_len, group_max_len, int(use_silu), _p(gate),
                                      _p(up), _p(down), gate_type, up_type, down_type, hidden_type)
        return C.c_void_p(h)

    def moe_forward_handle(self, h, H, hidden_type, ids, weights, x, out=None):
        qlen, k = ids.shape
        ids = np.ascontiguousarray(ids, dtype=np.uint64)
        weights = np.ascontiguousarray(weights, dtype=np.float32)
        x = np.ascontiguousarray(x)
        if out is None:
            out = np.zeros((qlen, H), _hidden_np(hidden_type))
        self.lib.ktref_moe_forward(h, qlen, k, _p(ids), _p(weights), _p(x), _p(out))
        return out

    def moe_destroy(self, h):
        self.lib.ktref_moe_destroy(h)

    def moe_forward(self, E, H, I, gate, up, down, gate_type, up_type, down_type, hidden_type, ids, weights, x,
                    use_silu=True, **kw):
        h = self.moe_create(E, ids.shape[1], H, I, gate, up, down, gate_type, up_type, down_type, hidden_type,
                            use_silu=use_silu, **kw)
        try:
            return self.moe_forward_handle(h, H, hidden_type, ids, weights, x)
        finally:
            self.moe_destroy(h)

    def linear_forward(self, in_size, out_size, proj, proj_type, hidden_type, x, stride=64, group_max_len=1024):
        x = np.ascontiguousarray(x)
        qlen = x.shape[0]
        out = np.zeros((qlen, out_size), _hidden_np(hidden_type))
        h = C.c_void_p(self.lib.ktref_linear_create(in_size, out_size, stride, group_max_len, _p(proj), proj_type,
                                                    hidden_type))
        self.lib.ktref_linear_forward(h, qlen, _p(x), _p(out))
        self.lib.ktref_linear_destroy(h)
        return out

    def mlp_forward(self, H, I, gate, up, down, gate_type, up_type, down_type, hidden_type, x, stride=64,
                    group_max_len=1024):
        x = np.ascontiguousarray(x)
        qlen = x.shape[0]
        out = np.zeros((qlen, H), _hidden_np(hidden_type))
        h = C.c_void_p(self.lib.ktref_mlp_create(H, I, stride, group_max_len, _p(gate), _p(up), _p(down), gate_type,
                                                 up_type, down_type, hidden_type))
        self.lib.ktref_mlp_forward(h, qlen, _p(x), _p(out))
        self.lib.ktref_mlp_destroy(h)
        return out


def bf16_to_f32(u16: np.ndarray) -> np.ndarray:
    return (u16.astype(np.uint32) << 16).view(np.float32)


def f32_to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """ggml_compute_fp32_to_bf16 (ggml-impl.h:87-104) vectorised: RNE, flush subnormals, quiet NaN."""
    i = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    r = ((i + (0x7FFF + ((i >> 16) & 1))) >> 16).astype(np.uint16)
    sub = (i & 0x7F800000) == 0
    r = np.where(sub, ((i & 0x80000000) >> 16).astype(np.uint16), r)
    nan = (i & 0x7FFFFFFF) > 0x7F800000
    r = np.where(nan, ((i >> 16) | 64).astype(np.uint16), r)
    return r.astype(np.uint16)


class AmxRef:
    """The reference's AMX MoE backend (kt_kernel_ext.moe.AMXInt4_MOE) compiled UNMODIFIED from the reference sources (REF in oracle/Makefile) through the
    single-node numa/hwloc shim (oracle/amx_shim.cpp, oracle/amx_shim/*.h): the "CPU-AMX" baseline of BASELINE.json.
    A SHIMMED build; runs only on hosts whose /proc/cpuinfo shows amx_tile + amx_int8."""

    _inst = None

    @staticmethod
    def path() -> str:
        return os.path.join(HERE, "_ref", "libktamx.so")

    @classmethod
    def available(cls) -> bool:
        return os.path.exists(cls.path()) and {"amx_tile", "amx_int8", "amx_bf16"} <= _cpu_flags()

    @classmethod
    def why_unavailable(cls) -> str:
        if not os.path.exists(cls.path()):
            return "oracle/_ref/libktamx.so not built (needs the reference sources, see REF in oracle/Makefile)"
        return "host CPU has no AMX (amx_tile / amx_int8 / amx_bf16 absent from /proc/cpuinfo)"

    @classmethod
    def get(cls, threads: int) -> "AmxRef":
        if cls._inst is None:
            cls._inst = cls()
        cls._inst.threads = cls._inst.lib.ktamx_init(int(threads))
        return cls._inst

    def __init__(self):
        self.lib = C.CDLL(self.path())
        self.lib.ktamx_moe_create.restype = C.c_void_p
        self.lib.ktamx_moe_create.argtypes = [C.c_int] * 5 + [C.c_void_p] * 3
        self.lib.ktamx_moe_forward.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        self.lib.ktamx_moe_destroy.argtypes = [C.c_void_p]
        self.threads = 0

    def moe_create(self, E, k, H, I, gate_bf16: np.ndarray, up_bf16: np.ndarray, down_bf16: np.ndarray, max_len: int = 64):
        """gate/up [E][I][H], down [E][H][I] as bf16 bit patterns (uint16); the backend quantises them to INT4 at load."""
        self._keep = (np.ascontiguousarray(gate_bf16), np.ascontiguousarray(up_bf16), np.ascontiguousarray(down_bf16))
        return self.lib.ktamx_moe_create(E, k, H, I, max_len, _p(self._keep[0]), _p(self._keep[1]), _p(self._keep[2]))

    def moe_forward(self, h, ids: np.ndarray, weights: np.ndarray, x_bf16: np.ndarray, out: Optional[np.ndarray] = None) -> np.ndarray:
        qlen, k = ids.shape
        ids = np.ascontiguousarray(ids, np.int64)
        weights = np.ascontiguousarray(weights, np.float32)
        x_bf16 = np.ascontiguousarray(x_bf16, np.uint16)
        if out is None:
            out = np.zeros_like(x_bf16)
        self.lib.ktamx_moe_forward(h, qlen, k, _p(ids), _p(weights), _p(x_bf16), _p(out))
        return out

    def moe_destroy(self, h):
        self.lib.ktamx_moe_destroy(h)
