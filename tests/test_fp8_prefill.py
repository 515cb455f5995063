"""The prompt route of ktb200_fp8_linear_forward (csrc/fp8_linear.cu fp8_gemm_kernel, DESIGN.md §4.6): from a threshold
that depends on the shape (32, 48 or 96 tokens) a call quantises its tokens once per chunk of at most 2048 and runs a tiled wgmma GEMM that reads each weight once per chunk,
with the decode route's arithmetic (e4m3 widened to fp16, one fp32 dot per 128 of K, acc + (dot * a_s) * b_s in kb order).
Below it the decode route runs unchanged.  Held to oracle/fp8_oracle.py with test_fp8_linear_vs_oracle's bound, to itself
(determinism, narrow outputs = the rounded F32 output), to the 16-token slices of the decode route, to the device batch-size
contract of tests/test_batch_size_contract.py, and through KLinearFP8 and the FP8 + GGUF hybrid rule file."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from ktransformers_b200 import native
from oracle.bindings import BF16, F16, F32, bf16_to_f32, f32_to_bf16_bits
from test_batch_size_contract import REPLAY_BS, Case, _tokens, contract_eager, contract_graph
from test_gpu_parity import assert_bf16_close
import gpu_util as G

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CHUNK = 2048    # tokens per GEMM launch at most (kPChunk); longer calls are cut into balanced chunks of whole 128-token tiles
TILE = 128      # tokens per CTA
TORCH = {BF16: torch.bfloat16, F16: torch.float16, F32: torch.float32}


def tmin(N, K):
    """fp8_prompt_min (csrc/fp8_linear.cu): the smallest qlen on the prompt route, measured per shape (DESIGN.md §4.6)"""
    return 96 if N <= 2048 else 48 if K >= 16384 else 32


def chunk_tokens(qlen):
    """fp8_forward_prompt's chunk: qlen cut into ceil(qlen / CHUNK) balanced parts, rounded up to whole token tiles"""
    n = (qlen + CHUNK - 1) // CHUNK
    return ((qlen + n - 1) // n + TILE - 1) // TILE * TILE


def chunks(qlen):
    return (qlen + chunk_tokens(qlen) - 1) // chunk_tokens(qlen)


def decode_launches(qlen):
    return sum(2 if min(16, qlen - t0) > 2 else 1 for t0 in range(0, qlen, 16))


def launches(qlen, N, K):
    return 2 * chunks(qlen) if qlen >= tmin(N, K) else decode_launches(qlen)


def _weights(rng, K, N):
    from oracle import fp8_oracle as F
    w = F.to_e4m3_bytes((rng.standard_normal((N, K)) * 0.7).astype(np.float32))
    ws = (rng.random(((N + 127) // 128, K // 128)) * 0.02 + 0.001).astype(np.float32)
    return w, ws


class Lin:
    """one ktb200_fp8_linear handle over device copies of (w, ws)"""

    def __init__(self, w, ws, hid=BF16):
        self.lib = native.lib()
        self.N, self.K = w.shape
        self.hid = hid
        self.w_d, self.ws_d = torch.from_numpy(w).cuda(), torch.from_numpy(ws).cuda()
        self.h = C.c_void_p()
        native.check(self.lib.ktb200_fp8_linear_create(self.K, self.N, self.w_d.data_ptr(), self.ws_d.data_ptr(), hid, 0, C.byref(self.h)))

    def __call__(self, x_d, out=None, bsz=None, qlen=None, stream=None):
        T = x_d.shape[0] if qlen is None else qlen
        y = torch.zeros((x_d.shape[0], self.N), dtype=TORCH[self.hid], device="cuda") if out is None else out
        native.check(self.lib.ktb200_fp8_linear_forward(self.h, T, x_d.data_ptr(), y.data_ptr(), None if bsz is None else bsz.data_ptr(),
                                                        G.stream() if stream is None else stream))
        return y

    def close(self):
        if self.h:
            self.lib.ktb200_fp8_linear_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()]).cpu().numpy()


def _x_bf16(rng, T, K):
    return f32_to_bf16_bits((rng.standard_normal((T, K)) / 10).astype(np.float32))


def _dev_bf16(xb):
    return torch.from_numpy(xb.view(np.int16)).view(torch.bfloat16).cuda()


# ------------------------------------------------------------------------------------------------ against the oracle
SMALL = [(128, 128), (1024, 200), (7168, 576)]
LARGE = [(7168, 1536), (1536, 24576), (16384, 7168)]
ORACLE_CASES = ([(K, N, T) for K, N in SMALL for T in sorted({tmin(N, K) - 1, tmin(N, K), tmin(N, K) + 1, 100, 300})]
                + [(K, N, CHUNK + 37) for K, N in SMALL[:2]]
                + [(K, N, T) for K, N in LARGE for T in (tmin(N, K), 100)] + [(7168, 1536, 300)])


@pytest.mark.parametrize("K,N,T", ORACLE_CASES)
def test_prompt_route_vs_oracle(K, N, T):
    """bf16 outputs within 1 ulp of the oracle and > 97 % identical, on both sides of the threshold and across a chunk edge"""
    from oracle import fp8_oracle as F
    rng = np.random.default_rng(K * 7 + N * 3 + T)
    w, ws = _weights(rng, K, N)
    x = _x_bf16(rng, T, K)
    lin = Lin(w, ws)
    got = _bits(lin(_dev_bf16(x))).view(np.uint16)
    lin.close()
    assert_bf16_close(got, f32_to_bf16_bits(F.linear_forward(bf16_to_f32(x), w, ws)))


@pytest.mark.parametrize("K,N,T", [(1024, 200, 300), (7168, 576, 100), (128, 128, CHUNK + 37)])
def test_prompt_route_f32_vs_oracle_accumulator(K, N, T):
    from oracle import fp8_oracle as F
    rng = np.random.default_rng(K + N + T)
    w, ws = _weights(rng, K, N)
    x = (rng.standard_normal((T, K)) / 10).astype(np.float32)
    lin = Lin(w, ws, F32)
    got = lin(torch.from_numpy(x).cuda()).cpu().numpy()
    lin.close()
    want = F.linear_forward(x, w, ws)
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()


# ------------------------------------------------------------------------------------------------ determinism and hidden types
@pytest.mark.parametrize("K,N,T", [(1024, 200, 300), (7168, 576, 96)])
def test_prompt_route_deterministic_and_narrow_is_rounded_f32(K, N, T):
    """two calls give the same bits; with BF16 and F16 hidden types the output is the F32 handle's output (on the same values,
    widened) rounded, bit for bit; F16 and F32 inputs go through the same quantiser"""
    rng = np.random.default_rng(K + 2 * N + T)
    w, ws = _weights(rng, K, N)
    x32 = torch.from_numpy((rng.standard_normal((T, K)) / 10).astype(np.float32)).cuda()
    l32 = Lin(w, ws, F32)
    for hid in (BF16, F16):
        xh = x32.to(TORCH[hid])
        lh = Lin(w, ws, hid)
        a, b = lh(xh), lh(xh)
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "two calls differ"
        y32 = l32(xh.float())
        assert torch.equal(a.view(torch.int16), y32.to(TORCH[hid]).view(torch.int16)), f"hidden type {hid}: not the rounded F32 output"
        lh.close()
    y1, y2 = l32(x32), l32(x32)
    assert torch.equal(y1.view(torch.int32), y2.view(torch.int32))
    l32.close()


# ------------------------------------------------------------------------------------------------ crossing the threshold
@pytest.mark.parametrize("K,N,T", [(1024, 200, 96), (7168, 576, 300), (16384, 7168, 48), (7168, 7168, 32)])
def test_prompt_route_vs_16_token_slices(K, N, T):
    """one call at T >= tmin (GEMM) against the same tokens sent in 16-token slices (the decode route): within the oracle bound"""
    rng = np.random.default_rng(K + N + 3 * T)
    w, ws = _weights(rng, K, N)
    x = _dev_bf16(_x_bf16(rng, T, K))
    lin = Lin(w, ws)
    one = lin(x)
    sliced = torch.zeros_like(one)
    for t0 in range(0, T, 16):
        lin(x[t0:t0 + 16], out=sliced[t0:t0 + 16])
    lin.close()
    assert_bf16_close(_bits(one).view(np.uint16), _bits(sliced).view(np.uint16))


# ------------------------------------------------------------------------------------------------ census
def _prompt_census():
    from test_linear_routes import _census
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    w, ws = _weights(rng, 1024, 200)
    lin = Lin(w, ws)
    w2, ws2 = _weights(rng, 512, 4096)
    big = Lin(w2, ws2)
    calls = []
    for m, K, N, Ts in ((lin, 1024, 200, (1, 2, 20, 95, 96, 97, 300, CHUNK + 37)), (big, 512, 4096, (31, 32, 33))):
        for T in Ts:
            x = _dev_bf16(_x_bf16(rng, T, K))
            calls.append(((T, N, K), None, (lambda m=m, x=x: m(x))))
    for (T, N, K), _, n, names in _census(calls):
        assert n == launches(T, N, K), f"T={T}: {n} launches, want {launches(T, N, K)}"
        gemm = sum("ktb::fp8_gemm_kernel(" in s for s in names)
        dec = sum("ktb::fp8_linear_kernel(" in s for s in names)
        if T < tmin(N, K):
            assert gemm == 0 and dec == (T + 15) // 16, (T, names)
        else:
            assert dec == 0 and gemm == chunks(T), (T, names)
            assert sum("ktb::fp8_gemm_quant_kernel(" in s for s in names) == chunks(T), (T, names)
    lin.close(); big.close()


def test_route_census():
    """below tmin the decode route's launches and no fp8_gemm_kernel; from tmin on fp8_gemm_kernel (one per chunk) and no
    fp8_linear_kernel, on both sides of the 96-token (N <= 2048) and 32-token thresholds.  In an interpreter of its own: after other profiler sessions in one process, torch.profiler can miss kernels"""
    root = os.path.dirname(HERE)
    code = ("import sys; sys.path[:0] = sys.argv[1:]; import test_fp8_prefill as t\n"
            "try:\n    t._prompt_census(); print('OK')\nexcept AssertionError as e:\n    print(e); sys.exit(1)")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, root, HERE]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-3000:] + r.stderr[-3000:]


def test_chunk_rule():
    assert [chunks(q) for q in (32, 2048, 2049, 2085, 4096, 4097, 6144)] == [1, 1, 2, 2, 2, 3, 3]


# ------------------------------------------------------------------------------------------------ device batch size
def prompt_case(T, K, N):
    rng = np.random.default_rng(T * 1000 + K + N)
    w, ws = _weights(rng, K, N)
    lin = Lin(w, ws)
    x, y = torch.empty((T, K), dtype=torch.bfloat16, device="cuda"), torch.empty((T, N), dtype=torch.bfloat16, device="cuda")

    def call(p, s):
        native.check(lin.lib.ktb200_fp8_linear_forward(lin.h, T, x.data_ptr(), y.data_ptr(), p, s))
    case = Case(T, call, [(x, "x")], [(y, "out")], None, launches(T, N, K), exact=True, keep=(lin,))
    case.fresh = lambda: x.copy_(_tokens(case.gen, T, K, torch.bfloat16) * 5)
    case.fresh()
    return case


@pytest.mark.parametrize("T,K,N", [(300, 1024, 200), (CHUNK + 37, 512, 384)])
def test_bsz_contract_eager(T, K, N):
    """rows >= min(b, qlen) untouched (NaN / Inf in the padded input rows), live rows bit-identical to the call without bsz"""
    case = prompt_case(T, K, N)
    bs = (0, 0, 1, TILE - 1, TILE, TILE + 1, T, T + 5)
    if T > CHUNK:
        c = chunk_tokens(T)                # the second chunk's first token
        bs += (c - 1, c, c + 1)
    contract_eager(case, bs)


@pytest.mark.parametrize("T,K,N", [(300, 1024, 200), (CHUNK + 37, 512, 384)])
def test_bsz_contract_graph_replay(T, K, N):
    case = prompt_case(T, K, N)
    contract_graph(case, REPLAY_BS + (TILE - 1, TILE + 1, T // 2 + 1, T))


# ------------------------------------------------------------------------------------------------ capture, NaN blocks, interleaving
def test_capture_without_warmup_fails_and_leaves_the_stream_usable():
    """a capture whose call would have to grow the prompt arena fails with the warm-up it needs; the stream stays usable, and
    after one eager call the same capture succeeds and replays the eager result"""
    from oracle import fp8_oracle as F
    # 640 tokens at in_features 65536 need 84 MB of arena: more than the whole chunk (2048 tokens) at any other test's K holds
    K, N, T = 65536, 256, 640
    rng = np.random.default_rng(1)
    w, ws = _weights(rng, K, N)
    xb = _x_bf16(rng, T, K)
    x = _dev_bf16(xb)
    lin = Lin(w, ws)
    y = torch.zeros((T, N), dtype=torch.bfloat16, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(native.KTB200Error, match="before capture"):
        with torch.cuda.graph(g, stream=s):
            lin(x, out=y, stream=s.cuda_stream)
    torch.cuda.synchronize()
    assert (y == 0).all()
    eager = _bits(lin(x)).view(np.uint16)
    assert_bf16_close(eager[:48], f32_to_bf16_bits(F.linear_forward(bf16_to_f32(xb[:48]), w, ws)))   # rows are independent
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2, stream=s):
        lin(x, out=y, stream=s.cuda_stream)
    g2.replay()
    torch.cuda.synchronize()
    assert np.array_equal(_bits(y).view(np.uint16), eager)
    del g, g2
    lin.close()


def test_all_zero_block_gives_the_oracles_nan_row():
    from oracle import fp8_oracle as F
    K, N, T = 1024, 200, 100
    rng = np.random.default_rng(2)
    w, ws = _weights(rng, K, N)
    x = (rng.standard_normal((T, K)) / 10).astype(np.float32)
    x[37, 256:384] = 0.0
    xb = f32_to_bf16_bits(x)
    lin = Lin(w, ws)
    got = _bits(lin(_dev_bf16(xb))).view(np.uint16)
    lin.close()
    want = f32_to_bf16_bits(F.linear_forward(bf16_to_f32(xb), w, ws))
    assert np.isnan(bf16_to_f32(want[37])).all() and np.isnan(bf16_to_f32(got[37])).all()
    keep = np.ones(T, bool)
    keep[37] = False
    assert_bf16_close(got[keep], want[keep])


def test_decode_call_after_a_prompt_call_on_the_same_handle():
    """the prompt route leaves the handle's decode buffers as they were: a decode call after it is bit-identical to a fresh handle's"""
    K, N = 1536, 256   # three K splits: the decode call uses the workspace and tickets
    rng = np.random.default_rng(4)
    w, ws = _weights(rng, K, N)
    xp, xd = _dev_bf16(_x_bf16(rng, 300, K)), _dev_bf16(_x_bf16(rng, 5, K))
    lin, fresh = Lin(w, ws), Lin(w, ws)
    lin(xp)
    a, b = lin(xd), fresh(xd)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    lin.close(); fresh.close()


# ------------------------------------------------------------------------------------------------ operators
def test_klinear_fp8_prefill_prompt():
    """KTransformersLinear(generate_op="KLinearFP8", prefill_op=None) in PREFILL mode on a prompt above tmin, against the
    dequantised fp32 product with test_klinear_fp8_operator_from_safetensors' bound"""
    from ktransformers_b200.operators.linear import KTransformersLinear
    from ktransformers_b200.util.utils import InferenceState
    Kf, Nf = 2048, 640
    g = torch.Generator().manual_seed(6)
    w = (torch.randn(Nf, Kf, generator=g) * 0.5).to(torch.float8_e4m3fn)
    s = torch.rand(Nf // 128, Kf // 128, generator=g) * 0.02 + 0.001
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        lin = KTransformersLinear("model.layers.0.self_attn.o_proj", None, None, torch.nn.Linear(Kf, Nf, bias=False, device="meta"),
                                  generate_op="KLinearFP8", prefill_op=None)
        lin.load(w=(w, s), mode=InferenceState.PREFILL)
        x = (torch.randn(1, tmin(Nf, Kf) + 5, Kf, device="cuda") / 10).to(torch.bfloat16)
        n0 = native.launch_count()
        y = lin(x)
        torch.cuda.synchronize()
        assert native.launch_count() - n0 == 2, "the prompt route: one quantiser and one GEMM launch"
        dense = w.float().view(Nf // 128, 128, Kf // 128, 128) * s.view(Nf // 128, 1, Kf // 128, 1)
        want = x.float().cpu().view(-1, Kf) @ dense.view(Nf, Kf).T
        assert (y.float().cpu().view(-1, Nf) - want).abs().max() <= 0.06 * want.abs().max()
        lin.unload()
    finally:
        torch.set_default_dtype(old)


def test_hybrid_rule_file_dense_layer_and_shared_expert_on_a_prompt(tmp_path):
    """DeepSeek-V3-Chat-fp8-linear-ggml-experts-b200.yaml on an FP8 + GGUF hybrid file: the dense layer's MLP and the MoE
    layer's shared expert (KLinearFP8 gate, up, down) on a 100-token prompt against the dequantised fp32 MLPs"""
    from safetensors.torch import save_file
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Config, DeepseekV3MoEOnlyForCausalLM
    from ktransformers_b200.operators.linear import KLinearFP8
    from ktransformers_b200.optimize.optimize import optimize_and_load_gguf
    from ktransformers_b200.util.synth import synth_blocks
    import ktransformers_b200.optimize.optimize as opt
    E, H, I, K = 8, 4096, 512, 4
    g = torch.Generator().manual_seed(12)
    tensors, dense = {}, {}

    def add_fp8(name, out_f, in_f):
        w = (torch.randn(out_f, in_f, generator=g) * 0.3).to(torch.float8_e4m3fn)
        s = torch.rand((out_f + 127) // 128, in_f // 128, generator=g) * 0.02 + 0.005
        tensors[name + ".weight"], tensors[name + ".weight_scale_inv"] = w, s
        dense[name] = (w.float().view(-1, 128, in_f // 128, 128) * s.view(-1, 1, in_f // 128, 1)).reshape(out_f, in_f)

    for n, (o, i) in {"gate_proj": (I, H), "up_proj": (I, H), "down_proj": (H, I)}.items():
        add_fp8(f"model.layers.0.mlp.{n}", o, i)
        add_fp8(f"model.layers.1.mlp.shared_experts.{n}", o, i)
    for n, qt, shape in (("gate", 12, (E, I, H)), ("up", 12, (E, I, H)), ("down", 14, (E, H, I))):
        tensors[f"blk.1.ffn_{n}_exps.weight"] = synth_blocks(qt, int(np.prod(shape)), "cpu", 400 + qt + len(n)).clone()
        tensors[f"blk.1.ffn_{n}_exps.ggml_type"] = torch.tensor(qt)
    tensors["blk.1.ffn_gate_inp.weight"] = torch.randn(E, H, generator=g)
    tensors["blk.1.exp_probs_b.bias"] = 0.01 * torch.randn(E, generator=g)
    save_file(tensors, str(tmp_path / "hybrid.safetensors"))
    rule = os.path.join(os.path.dirname(opt.__file__), "optimize_rules", "DeepSeek-V3-Chat-fp8-linear-ggml-experts-b200.yaml")
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        cfg = DeepseekV3Config(hidden_size=H, intermediate_size=I, moe_intermediate_size=I, n_routed_experts=E, n_shared_experts=1,
                               num_experts_per_tok=K, n_group=2, topk_group=1, num_hidden_layers=2, first_k_dense_replace=1)
        with torch.device("meta"):
            model = DeepseekV3MoEOnlyForCausalLM(cfg)
        optimize_and_load_gguf(model, rule, str(tmp_path), cfg, default_device="cuda")
        x = (torch.randn(1, 100, H, device="cuda") / 10).to(torch.bfloat16)
        xf = x.view(-1, H).float().cpu()
        for p, mlp in (("model.layers.0.mlp.", model.model.layers[0].mlp), ("model.layers.1.mlp.shared_experts.", model.model.layers[1].mlp.shared_experts)):
            assert isinstance(mlp.down_proj.generate_linear, KLinearFP8)
            n0 = native.launch_count()
            y = mlp(x)
            torch.cuda.synchronize()
            assert native.launch_count() - n0 >= 6, "three projections on the prompt route (two launches each)"
            want = (torch.nn.functional.silu(xf @ dense[p + "gate_proj"].T) * (xf @ dense[p + "up_proj"].T)) @ dense[p + "down_proj"].T
            assert (y.view(-1, H).float().cpu() - want).abs().max() <= 0.06 * want.abs().max(), p
    finally:
        torch.set_default_dtype(old)
