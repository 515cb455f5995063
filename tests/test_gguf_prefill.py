"""The prompt route of the GGUF dense linear (ktb200_linear_forward_prompt, csrc/gguf_gemm.cu gguf_gemm_kernel, DESIGN.md §4.17):
Q4_K weights and Q6_K weights in the 8-row SoA layout, a chunk of at most 2048 tokens quantised once to Q8_K and multiplied on
the integer tensor cores in tiles of 128 weight rows x 64 tokens, with the decode kernels' arithmetic (exact integer sub-block
dots, int32 scale-and-add per super-block, the decode kernels' fp32 term, fp32 sum in kb order).

Held to test_linear_routes' references and bounds, unchanged (the C oracle on sampled rows, the float64 restatement on every
element), to ktb200_linear_forward on the same inputs, to itself (determinism, a token's row independent of its tile offset,
chunk and qlen), to the device batch-size contract of tests/test_batch_size_contract.py, and through KLinearB200 and the serve
rule file with `prefill_op: None`."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from ktransformers_b200 import native
from oracle.bindings import BF16, F16, F32, IQ4_XS, Q2_K, Q3_K, Q4_K, Q5_K, Q6_K, TYPE_NAMES, bf16_to_f32, f32_to_bf16_bits
from test_linear_routes import F32_REL, Linear, linear_route, oracle_rows, q8k_values, restated, tokens

HERE = os.path.dirname(os.path.abspath(__file__))
QK = 256
CHUNK = 2048    # tokens per GEMM launch at most (kGgChunk); longer calls are cut into balanced chunks of whole token tiles
TILE = 64       # tokens per CTA (kGgT)


def soa(t, n_in, n_out):
    """ktb200_linear_load_weights re-lays Q6_K into the 8-row SoA layout"""
    return t == Q6_K and n_out % 8 == 0 and 8 * 210 * (n_in // QK) <= 200 * 1024


def prompt_min(t, n_in, n_out):
    """gguf_prompt_min (csrc/gguf_gemm.cu): measured crossovers (DESIGN.md §4.17), 0 where the GEMM does not take the handle"""
    if t == Q4_K or soa(t, n_in, n_out):
        return 24 if n_out <= 1024 else 16
    return 0


def chunk_tokens(qlen):
    n = (qlen + CHUNK - 1) // CHUNK
    return ((qlen + n - 1) // n + TILE - 1) // TILE * TILE


def chunks(qlen):
    return (qlen + chunk_tokens(qlen) - 1) // chunk_tokens(qlen)


# ------------------------------------------------------------------------------------------------ CPU
def test_chunk_rule():
    assert [chunks(q) for q in (1, 64, 2048, 2049, 4096, 4097, 6144)] == [1, 1, 1, 2, 2, 3, 3]
    assert [chunk_tokens(q) for q in (1, 65, 2048, 2049, 4096)] == [64, 128, 2048, 1088, 2048]


@pytest.mark.parametrize("t,n_in,n_out", [(Q4_K, 7168, 1536), (Q4_K, 16384, 7168), (Q4_K, 256, 576), (Q6_K, 18432, 7168),
                                          (Q6_K, 2048, 7168), (Q6_K, 7168, 129280), (Q6_K, 1536, 2051), (Q6_K, 256, 777),
                                          (Q5_K, 7168, 1536), (Q2_K, 7168, 1536), (Q3_K, 7168, 576), (IQ4_XS, 7168, 1536)])
def test_prompt_min_is_the_restated_table(t, n_in, n_out):
    """ktb200_linear_prompt_min is a pure function of (type, layout, in, out): a loaded Q6_K handle of out_features % 8 == 0
    has the SoA layout; one that keeps the raw layout, and every type the GEMM does not take, gives 0"""
    lib = native.lib()
    h = C.c_void_p()
    fake = C.c_void_p(1 << 20)    # never dereferenced: creating a handle reads no weight
    native.check(lib.ktb200_linear_create(n_in, n_out, fake, t, BF16, 1024, 0, C.byref(h)))
    try:
        got = lib.ktb200_linear_prompt_min(h)
    finally:
        lib.ktb200_linear_destroy(h)
    # an unloaded handle has no SoA layout yet: the Q6_K value applies once ktb200_linear_load_weights has re-laid it
    assert got == (prompt_min(t, n_in, n_out) if t != Q6_K else 0), TYPE_NAMES[t]


# ------------------------------------------------------------------------------------------------ GPU helpers
def _stream():
    return torch.cuda.current_stream().cuda_stream


def prompt(lin, x, bias=None, bsz=None, out=None, qlen=None, stream=None):
    """ktb200_linear_forward_prompt on a test_linear_routes.Linear handle; rows it does not write stay NaN"""
    from test_linear_routes import TORCH_HID
    y = torch.full((x.shape[0], lin.n_out), float("nan"), dtype=TORCH_HID[lin.hid], device="cuda") if out is None else out
    native.check(lin.lib.ktb200_linear_forward_prompt(lin.h, x.shape[0] if qlen is None else qlen, x.data_ptr(), y.data_ptr(),
                                                      None if bias is None else bias.data_ptr(), None if bsz is None else bsz.data_ptr(),
                                                      _stream() if stream is None else stream))
    return y


def _weights(t, n, seed):
    from ktransformers_b200.util.synth import synth_blocks
    return synth_blocks(t, n, device="cuda", seed=seed)


def _bf16_bits(t):
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


# ------------------------------------------------------------------------------------------------ GPU: against the oracle
SHAPES = {
    # name: (type, in, out).  The probe's DeepSeek-V3 shapes except lm_head, then edge shapes
    "q4k-q_a-7168x1536": (Q4_K, 7168, 1536),
    "q4k-kv_a-7168x576": (Q4_K, 7168, 576),
    "q4k-q_b-1536x24576": (Q4_K, 1536, 24576),
    "q4k-o_proj-16384x7168": (Q4_K, 16384, 7168),
    "q4k-dense_gate_up-7168x18432": (Q4_K, 7168, 18432),
    "q4k-shared_gate_up-7168x2048": (Q4_K, 7168, 2048),
    "q6k-dense_down-18432x7168": (Q6_K, 18432, 7168),
    "q6k-shared_down-2048x7168": (Q6_K, 2048, 7168),
    "q4k-one_block-256x200": (Q4_K, 256, 200),
    "q4k-2048x777": (Q4_K, 2048, 777),
    "q6k-one_block-256x576": (Q6_K, 256, 576),
    "q6k-3072x840": (Q6_K, 3072, 840),
}
BIG_TS = (129, 2047, 2048, 2049, 4096)


def _cases():
    out = []
    for name, (t, n_in, n_out) in SHAPES.items():
        pm = prompt_min(t, n_in, n_out)
        ts = {pm - 1, pm, 129}
        if n_in * n_out <= 2048 * 7168 or name == "q4k-q_a-7168x1536":
            ts |= set(BIG_TS)
        out += [(name, T) for T in sorted(ts)]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,T", _cases())
def test_prompt_route_vs_oracle_and_float64(oracle, name, T):
    """test_linear_vs_oracle_and_float64's bounds: F32 within F32_REL x |W|.|x_q| of the float64 restatement on every element and
    within F32_REL of the row max against the C oracle; BF16 one ulp of the oracle (+ the F32 bound), >= 99 % identical; F16
    the rounded F32 output on the widened input.  With and without bias.  Also the two routes on the same input agree within
    the F32 bound."""
    t, n_in, n_out = SHAPES[name]
    w = _weights(t, n_out * n_in, n_in + n_out)
    w_np = w.cpu().numpy()
    w64 = torch.from_numpy(oracle.to_float(w_np, t, n_out * n_in).reshape(n_out, n_in)).cuda().double()
    lin = {h: Linear(t, n_in, n_out, w, h) for h in (F32, BF16, F16)}
    bias = torch.from_numpy(np.random.default_rng(n_out).standard_normal(n_out).astype(np.float32)).cuda()
    x = tokens(T, n_in, T * 7 + n_in)
    x_d = torch.from_numpy(x).cuda()
    ref, mag = restated(w64, torch.from_numpy(q8k_values(oracle, x)).cuda())
    del w64
    rows = oracle_rows(T, T)
    want = oracle.linear_forward(n_in, n_out, w_np, t, F32, x[rows])
    for b in (None, bias):
        what = f"{name} T={T} bias={b is not None}"
        v = ref + b.double() if b is not None else ref
        y = prompt(lin[F32], x_d, b)
        e64 = ((y.double() - v).abs() - 2.0 ** -24 * v.abs()) / mag.clamp_min(1e-300)
        assert float(e64.max()) <= F32_REL, f"{what}: F32 vs float64 {float(e64.max()):.3g} x |W|.|x_q| at {divmod(int(e64.argmax()), n_out)}"
        got = y[torch.from_numpy(rows).cuda()].cpu().numpy()
        wb = want + b.cpu().numpy() if b is not None else want
        eo = np.abs(got - wb).max(1) / np.maximum(np.abs(wb).max(1), 1e-30)
        assert eo.max() <= F32_REL, f"{what}: F32 vs oracle {eo.max():.3g} of the row's max at token {rows[eo.argmax()]}"
        # the decode route on the same input: both within the F32 bound of the float64 value, so of each other
        yg = lin[F32](x_d, b)
        eg = ((y.double() - yg.double()).abs() - 2.0 ** -23 * v.abs()) / mag.clamp_min(1e-300)
        assert float(eg.max()) <= 2 * F32_REL, f"{what}: prompt vs decode route {float(eg.max()):.3g}"
        del yg, eg, e64
        yb = prompt(lin[BF16], x_d.to(torch.bfloat16), b)
        eb = ((yb.double() - v).abs() - 2.0 ** -8 * v.abs()) / mag.clamp_min(1e-300)
        assert float(eb.max()) <= F32_REL, f"{what}: BF16 vs float64 beyond rounding at {divmod(int(eb.argmax()), n_out)}"
        gb, wbb = _bf16_bits(yb[torch.from_numpy(rows).cuda()]), f32_to_bf16_bits(wb)
        a, c = bf16_to_f32(gb), bf16_to_f32(wbb)
        tol = 2.0 ** -7 * np.maximum(np.abs(a), np.abs(c)) + F32_REL * np.abs(c).max(1, keepdims=True)
        assert (np.abs(a - c) <= tol).all(), f"{what}: BF16 more than one ulp (+ the F32 bound) from the oracle"
        assert float((gb == wbb).mean()) >= 0.99, f"{what}: BF16 {float((gb == wbb).mean()):.4f} bit-identical to the oracle"
        del eb
        xh = x_d.to(torch.float16)
        yh, y32 = prompt(lin[F16], xh, b), prompt(lin[F32], xh.float(), b)
        assert torch.equal(yh.view(torch.int16), y32.to(torch.float16).view(torch.int16)), f"{what}: F16 != rounded F32"
    for h in lin.values():
        h.close()


# ------------------------------------------------------------------------------------------------ GPU: bit-exact invariants
@pytest.mark.gpu
@pytest.mark.parametrize("t,n_in,n_out", [(Q4_K, 2048, 777), (Q6_K, 3072, 840)])
def test_rows_independent_of_position_chunk_and_qlen(t, n_in, n_out):
    """two calls give the same bits; a token's row is the same at another tile offset, in the second chunk and in a call of
    another qlen (no K splits, no atomics, no dependence on the tile)"""
    lin = Linear(t, n_in, n_out, _weights(t, n_out * n_in, 11), F32)
    x = torch.from_numpy(tokens(2100, n_in, 5)).cuda()
    a, b = prompt(lin, x[:300]), prompt(lin, x[:300])
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "two calls differ"
    shifted = prompt(lin, x[1:300])                       # every token one place earlier in its tile
    assert torch.equal(shifted.view(torch.int32), a[1:].view(torch.int32))
    long = prompt(lin, x)                                 # 2100 tokens: two chunks of 1088; tokens 1088.. sit in the second
    c0 = chunk_tokens(2100)
    assert chunks(2100) == 2 and c0 == 1088
    tail = prompt(lin, x[c0 - 5:c0 + 300])
    assert torch.equal(long[c0 - 5:c0 + 300].view(torch.int32), tail.view(torch.int32))
    assert torch.equal(long[:300].view(torch.int32), a.view(torch.int32))
    one = prompt(lin, x[7:8])                            # qlen 1
    assert torch.equal(one.view(torch.int32), a[7:8].view(torch.int32))
    lin.close()


# ------------------------------------------------------------------------------------------------ GPU: census
def _prompt_census():
    from test_linear_routes import _census
    torch.cuda.set_device(0)
    calls, keep = [], []
    for t, n_in, n_out, ts in ((Q4_K, 7168, 1536, (15, 16, 17, 300, CHUNK + 37)), (Q4_K, 7168, 576, (23, 24)), (Q6_K, 2048, 7168, (16, 129)),
                             (Q4_K, 256, 200, (1, 64))):
        lin = Linear(t, n_in, n_out, _weights(t, n_out * n_in, 3), BF16)
        keep.append(lin)
        for T in ts:
            x = torch.randn((T, n_in), device="cuda").to(torch.bfloat16) / 10
            calls.append((("prompt", t, n_in, n_out, T), None, (lambda lin=lin, x=x: prompt(lin, x))))
            calls.append((("decode", t, n_in, n_out, T), None, (lambda lin=lin, x=x: lin(x))))
    for (route, t, n_in, n_out, T), _, n, names in _census(calls):
        if route == "prompt":
            assert n == 2 * chunks(T), (T, n, names)
            gemm = f"ktb::gguf_gemm_kernel<{0 if t == Q4_K else 1}>("
            assert all(("ktb::grp_quant_x_kernel(" in k) if i % 2 == 0 else (gemm in k) for i, k in enumerate(names)), (T, names)
        else:
            want = linear_route(t, n_in, n_out, T)
            assert names and all(want in k for k in names) and not any("gguf_gemm" in k for k in names), (T, want, names)
    for h in keep:
        h.close()


@pytest.mark.gpu
def test_route_census():
    """the prompt entry launches the quantiser and the GEMM per chunk and nothing else; ktb200_linear_forward at the same token
    counts launches exactly its old kernels (test_linear_routes' route table).  In an interpreter of its own: after other
    profiler sessions in one process, torch.profiler can miss kernels"""
    root = os.path.dirname(HERE)
    code = ("import sys; sys.path[:0] = sys.argv[1:]; import test_gguf_prefill as t\n"
            "try:\n    t._prompt_census(); print('OK')\nexcept AssertionError as e:\n    print(e); sys.exit(1)")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, root, HERE]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-3000:] + r.stderr[-3000:]


# ------------------------------------------------------------------------------------------------ GPU: refusals
@pytest.mark.gpu
@pytest.mark.parametrize("t,n_in,n_out", [(Q5_K, 1536, 512), (Q2_K, 1536, 512), (Q3_K, 1536, 512), (IQ4_XS, 1536, 512), (Q6_K, 1536, 2051),
                                          (Q4_K, 1536, 512), (Q6_K, 1536, 512)])
def test_types_the_gemm_does_not_take_are_refused(t, n_in, n_out):
    lin = Linear(t, n_in, n_out, _weights(t, n_out * n_in, 2), BF16)
    x = torch.randn((40, n_in), device="cuda").to(torch.bfloat16)
    pm = lin.lib.ktb200_linear_prompt_min(lin.h)
    assert pm == prompt_min(t, n_in, n_out)
    if pm == 0:
        y = torch.full((40, n_out), float("nan"), dtype=torch.bfloat16, device="cuda")
        rc = lin.lib.ktb200_linear_forward_prompt(lin.h, 40, x.data_ptr(), y.data_ptr(), None, None, _stream())
        assert rc == native.EINVAL, rc
        msg = lin.lib.ktb200_last_error().decode()
        assert ("raw block layout" in msg) if t == Q6_K else (TYPE_NAMES[t] in msg), msg
        torch.cuda.synchronize()
        assert torch.isnan(y.float()).all()
    else:
        assert pm > 0
        prompt(lin, x)
    lin.close()


# ------------------------------------------------------------------------------------------------ GPU: device batch size
def prompt_case(T, t, n_in, n_out):
    from test_batch_size_contract import Case, _tokens
    lin = Linear(t, n_in, n_out, _weights(t, n_out * n_in, T + n_in), BF16)
    x, y = torch.empty((T, n_in), dtype=torch.bfloat16, device="cuda"), torch.empty((T, n_out), dtype=torch.bfloat16, device="cuda")

    def call(p, s):
        native.check(lin.lib.ktb200_linear_forward_prompt(lin.h, T, x.data_ptr(), y.data_ptr(), None, p, s))
    case = Case(T, call, [(x, "x")], [(y, "out")], None, 2 * chunks(T), exact=True, keep=(lin,))
    case.fresh = lambda: x.copy_(_tokens(case.gen, T, n_in, torch.bfloat16) * 5)
    case.fresh()
    return case


@pytest.mark.gpu
@pytest.mark.parametrize("T,t,n_in,n_out", [(300, Q4_K, 1024, 200), (CHUNK + 37, Q6_K, 512, 384)])
def test_bsz_contract_eager(T, t, n_in, n_out):
    """rows >= min(b, qlen) untouched (NaN / Inf in the padded input rows), live rows bit-identical to the call without bsz"""
    from test_batch_size_contract import contract_eager
    case = prompt_case(T, t, n_in, n_out)
    bs = (0, 0, 1, TILE - 1, TILE, TILE + 1, T, T + 5)
    if T > CHUNK:
        c = chunk_tokens(T)
        bs += (c - 1, c, c + 1)
    contract_eager(case, bs)


@pytest.mark.gpu
@pytest.mark.parametrize("T,t,n_in,n_out", [(300, Q4_K, 1024, 200), (CHUNK + 37, Q6_K, 512, 384)])
def test_bsz_contract_graph_replay(T, t, n_in, n_out):
    from test_batch_size_contract import REPLAY_BS, contract_graph
    case = prompt_case(T, t, n_in, n_out)
    contract_graph(case, REPLAY_BS + (TILE - 1, TILE + 1, T // 2 + 1, T))


@pytest.mark.gpu
def test_capture_without_warmup_fails_and_leaves_the_stream_usable():
    """a capture whose call would have to grow the Q8_K arena fails with the warm-up it needs and writes nothing; after one
    eager call the same capture succeeds and replays the eager result"""
    # 640 tokens at in_features 65536 need 42 M activation bytes: more than a whole chunk (2048 tokens) at any other test's K
    t, n_in, n_out, T = Q4_K, 65536, 256, 640
    lin = Linear(t, n_in, n_out, _weights(t, n_out * n_in, 1), BF16)
    x = torch.from_numpy(tokens(T, n_in, 3)).cuda().to(torch.bfloat16)
    y = torch.zeros((T, n_out), dtype=torch.bfloat16, device="cuda")
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(native.KTB200Error, match="before capture"):
        with torch.cuda.graph(g, stream=s):
            prompt(lin, x, out=y, stream=s.cuda_stream)
    torch.cuda.synchronize()
    assert (y == 0).all()
    eager = prompt(lin, x)
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2, stream=s):
        prompt(lin, x, out=y, stream=s.cuda_stream)
    g2.replay()
    torch.cuda.synchronize()
    assert torch.equal(y.view(torch.int16), eager.view(torch.int16))
    del g, g2
    lin.close()


# ------------------------------------------------------------------------------------------------ GPU: operators
def _serve_model(tmp_path, rule):
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Config, DeepseekV3MoEOnlyForCausalLM
    from ktransformers_b200.operators.linear import KTransformersLinear
    from ktransformers_b200.optimize.optimize import optimize_and_load_gguf
    from ktransformers_b200.util.utils import InferenceState
    from test_gpu_operators import E, H, I, K
    cfg = DeepseekV3Config(hidden_size=H, intermediate_size=I, moe_intermediate_size=I, n_routed_experts=E, n_shared_experts=1,
                           num_experts_per_tok=K, n_group=2, topk_group=1, num_hidden_layers=2, first_k_dense_replace=1)
    with torch.device("meta"):
        model = DeepseekV3MoEOnlyForCausalLM(cfg)
    optimize_and_load_gguf(model, rule, str(tmp_path), cfg, default_device="cuda")
    for m in model.modules():
        if isinstance(m, KTransformersLinear):
            m.set_inference_mode(InferenceState.PREFILL)
    return model


@pytest.mark.gpu
def test_serve_rule_file_with_prefill_op_none_matches_the_shipped_file(tmp_path):
    """a tmp copy of DeepSeek-V3-Chat-b200-serve.yaml whose linears say `prefill_op: None`: in PREFILL mode the GGUF linears of
    the dense layer and the MoE layer's shared expert stay KLinearB200 (nothing reloaded) and take the prompt route; a prompt
    through both layers gives the shipped file's (KLinearTorch, dequantised bf16) output within the suite's tolerance, and a
    linear's output is within the int8 bound of the dequantised float64 product"""
    from ktransformers_b200.operators.linear import KLinearB200, KTransformersLinear
    import ktransformers_b200.optimize.optimize as opt
    from test_gpu_operators import H, _write_gguf
    dense = _write_gguf(str(tmp_path / "tiny.gguf"))
    shipped = os.path.join(os.path.dirname(opt.__file__), "optimize_rules", "DeepSeek-V3-Chat-b200-serve.yaml")
    text = open(shipped).read()
    assert 'prefill_op: "KLinearTorch"' in text
    mine = tmp_path / "serve-prefill-none.yaml"
    mine.write_text(text.replace('prefill_op: "KLinearTorch"', "prefill_op: None"))
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.bfloat16)
    try:
        new, ref = _serve_model(tmp_path, str(mine)), _serve_model(tmp_path, shipped)
        gate = new.model.layers[0].mlp.gate_proj
        assert isinstance(gate, KTransformersLinear) and gate.prefill_linear is None and isinstance(gate.generate_linear, KLinearB200)
        pm = gate.generate_linear.prompt_min
        assert pm > 0
        T = max(pm, 100) + 3
        x = (torch.randn(1, T, H, device="cuda") / 10).to(torch.bfloat16)
        handle = gate.generate_linear.handle.value
        n0 = native.launch_count()
        yg = gate(x)
        torch.cuda.synchronize()
        assert native.launch_count() - n0 == 2, "the prompt route: one quantiser and one GEMM launch"
        assert gate.generate_linear.handle.value == handle
        w64 = torch.from_numpy(np.array(dense["blk.0.ffn_gate.weight"])).cuda().double()
        want = x.view(-1, H).double() @ w64.T
        assert (yg.view(-1, w64.shape[0]).double() - want).abs().max() <= 0.02 * want.abs().max()
        for layer in (0, 1):
            a, b = new.model.layers[layer].mlp, ref.model.layers[layer].mlp
            ya, yb = a(x), b(x)
            torch.cuda.synchronize()
            ya, yb = (y[0] if isinstance(y, tuple) else y for y in (ya, yb))
            assert (ya.float() - yb.float()).abs().max() <= 0.05 * yb.float().abs().max(), layer
    finally:
        torch.set_default_dtype(old)
