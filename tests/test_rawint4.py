"""RAWINT4_G32 routed experts (compressed-tensors INT4, group 32, bf16 scales): format pin, loader, wrapper, C-ABI checks
and the sm_90a kernels against the float64 oracle in tests/int4_oracle.py."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import int4_oracle as o4
from ktransformers_b200 import native

I4 = native.RAWINT4_G32
F32, BF16 = native.GGML_F32, native.GGML_BF16


def _golden(golden_dir):
    return np.load(os.path.join(golden_dir, "rawint4_pack.npz"))


# ------------------------------------------------------------------------------------------------ format (CPU)
def test_oracle_unpack_matches_golden(golden_dir):
    g = _golden(golden_dir)
    assert np.array_equal(o4.unpack(g["weight_packed"]), g["values"])
    assert np.array_equal(o4.pack(g["values"]), g["weight_packed"])
    assert tuple(g["weight_shape"]) == g["values"].shape


def test_oracle_unpack_matches_compressed_tensors(golden_dir):
    helpers = pytest.importorskip("compressed_tensors.compressors.pack_quantized.helpers")
    g = _golden(golden_dir)
    packed = torch.from_numpy(g["weight_packed"])
    ref = helpers.unpack_from_int32(packed, 4, torch.Size(g["values"].shape)).numpy()
    assert np.array_equal(o4.unpack(g["weight_packed"]), ref)
    assert np.array_equal(helpers.pack_to_int32(torch.from_numpy(g["values"]), 4).numpy(), g["weight_packed"])


def test_device_layout_of_golden(golden_dir):
    g = _golden(golden_dir)
    lay = o4.device_layout(g["weight_packed"], g["weight_scale_bits"]).reshape(4, 2, 144)
    # block 1 of row 2: scales 8..15 of the row, then the packed words 32..63 unchanged
    assert np.array_equal(lay[2, 1, :16].view(np.uint16), g["weight_scale_bits"][2, 8:16])
    assert np.array_equal(lay[2, 1, 16:].view(np.int32), g["weight_packed"][2, 32:64])


def test_type_size_and_block():
    lib = native.lib()
    assert lib.ktb200_type_size(I4) == 144 and lib.ktb200_blck_size(I4) == 256
    assert native.type_size(I4) == 144 == native.type_size(native.GGML_Q4_K)


# ------------------------------------------------------------------------------------------------ C-ABI checks (CPU)
def _cfg(H, I, gt=I4, ut=I4, dt=I4):
    fake = 1 << 20       # never dereferenced: create rejects before it touches the device
    return native.MoeConfig(8, 2, H, I, 64, 10, 16, 1, fake, fake, fake, gt, ut, dt, BF16, 0)


@pytest.mark.parametrize("H,I,types", [(7168, 2000, (I4, I4, I4)), (7000, 2048, (I4, I4, I4)),
                                       (512, 256, (I4, I4, native.GGML_Q6_K)), (512, 256, (native.GGML_Q4_K, I4, I4))])
def test_moe_create_rejects(H, I, types):
    lib = native.lib()
    h = C.c_void_p()
    cfg = _cfg(H, I, *types)
    assert lib.ktb200_moe_create(C.byref(cfg), 0, C.byref(h)) == native.EINVAL
    assert not h.value


def test_linear_and_mlp_reject_rawint4():
    lib = native.lib()
    h = C.c_void_p()
    assert lib.ktb200_linear_create(512, 256, 1 << 20, I4, BF16, 16, 0, C.byref(h)) == native.EINVAL
    assert lib.ktb200_mlp_create(512, 256, 1 << 20, 1 << 20, 1 << 20, I4, I4, I4, BF16, 16, 0, C.byref(h)) == native.EINVAL


def test_pack_rejects_cols():
    lib = native.lib()
    rc = lib.ktb200_rawint4_pack(1 << 20, 1 << 20, 4, 288, 1 << 20, None)
    assert rc == native.EINVAL and "256" in lib.ktb200_last_error().decode()


# ------------------------------------------------------------------------------------------------ loader (CPU)
def _write_ct_dir(path, E, H, I, seed=0, qc=True, override=None):
    """a tiny compressed-tensors checkpoint: per-expert weight_packed / weight_scale / weight_shape of layer 0"""
    from safetensors.torch import save_file
    rng = np.random.default_rng(seed)
    tensors, ref = {}, {}
    for n, (rows, cols) in (("gate", (I, H)), ("up", (I, H)), ("down", (H, I))):
        q = rng.integers(-8, 8, size=(E, rows, cols), dtype=np.int8)
        s = torch.from_numpy((rng.random((E, rows, cols // 32)) * 0.02 + 0.005).astype(np.float32)).to(torch.bfloat16)
        ref[n] = (o4.pack(q), s)
        for e in range(E):
            p = f"model.layers.0.mlp.experts.{e}.{n}_proj"
            tensors[p + ".weight_packed"] = torch.from_numpy(ref[n][0][e].copy())
            tensors[p + ".weight_scale"] = s[e].clone()
            tensors[p + ".weight_shape"] = torch.tensor([rows, cols], dtype=torch.int64)
    if override:
        tensors.update(override)
    os.makedirs(path, exist_ok=True)
    save_file(tensors, os.path.join(path, "model.safetensors"))
    if qc:
        w = {"num_bits": 4, "group_size": 32, "symmetric": True, "type": "int", "strategy": "group", "dynamic": False}
        if isinstance(qc, dict):
            w.update(qc)
        cfg = {"quantization_config": {"quant_method": "compressed-tensors", "format": "pack-quantized",
                                       "config_groups": {"group_0": {"targets": ["Linear"], "weights": w}}}}
        with open(os.path.join(path, "config.json"), "w") as f:
            json.dump(cfg, f)
    return ref


def test_loader_stacks_experts(tmp_path):
    from ktransformers_b200.util.custom_loader import ModelLoaderFactory
    E, H, I = 3, 256, 512
    ref = _write_ct_dir(str(tmp_path), E, H, I)
    w = ModelLoaderFactory.create_loader(str(tmp_path)).load_experts("model.layers.0.mlp.experts")
    for n, (rows, cols) in (("gate", (I, H)), ("up", (I, H)), ("down", (H, I))):
        assert w[n + "_type"] == I4
        assert w[n].dtype == torch.int32 and tuple(w[n].shape) == (E, rows, cols // 8)
        assert w[n + "_scale"].dtype == torch.bfloat16 and tuple(w[n + "_scale"].shape) == (E, rows, cols // 32)
        assert np.array_equal(w[n].numpy(), ref[n][0])
        assert torch.equal(w[n + "_scale"], ref[n][1])


@pytest.mark.parametrize("field,value", [("num_bits", 8), ("group_size", 128), ("symmetric", False), ("type", "float"),
                                         ("strategy", "channel")])
def test_loader_rejects_quantization_config(tmp_path, field, value):
    from ktransformers_b200.util.custom_loader import SafeTensorLoader
    _write_ct_dir(str(tmp_path), 2, 256, 256, qc={field: value})
    with pytest.raises(ValueError, match=field):
        SafeTensorLoader(str(tmp_path)).load_experts("model.layers.0.mlp.experts")


def test_loader_checks_shape_and_dtype(tmp_path):
    from ktransformers_b200.util.custom_loader import SafeTensorLoader
    p = "model.layers.0.mlp.experts.1.up_proj"
    _write_ct_dir(str(tmp_path / "a"), 2, 256, 256, override={p + ".weight_shape": torch.tensor([256, 512])})
    with pytest.raises(ValueError, match="weight_shape"):
        SafeTensorLoader(str(tmp_path / "a")).load_experts("model.layers.0.mlp.experts")
    _write_ct_dir(str(tmp_path / "b"), 2, 256, 256, override={p + ".weight_scale": torch.zeros((256, 8), dtype=torch.float32)})
    with pytest.raises(ValueError, match="bfloat16"):
        SafeTensorLoader(str(tmp_path / "b")).load_experts("model.layers.0.mlp.experts")


# ------------------------------------------------------------------------------------------------ wrapper (CPU)
def _wrapper(**kw):
    from ktransformers_b200.kt_moe_wrapper import KTMoEWrapper
    args = dict(layer_idx=0, num_experts=4, num_experts_per_tok=2, hidden_size=256, moe_intermediate_size=256,
                gpu_experts_mask=None, method="B200_RAWINT4")
    args.update(kw)
    return KTMoEWrapper(**args)


def test_wrapper_argument_checks():
    with pytest.raises(NotImplementedError):
        _wrapper(method="B200_INT4")
    w = _wrapper()
    p = torch.zeros((4, 256, 32), dtype=torch.int32)
    s = torch.zeros((4, 256, 8), dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="scale"):
        w.load_weights_from_tensors(p, p, p)
    with pytest.raises(ValueError, match="ggml_types"):
        w.load_weights_from_tensors(p, p, p, ggml_types=(12, 12, 14), gate_scale=s, up_scale=s, down_scale=s)
    with pytest.raises(ValueError, match="num_experts"):
        w.load_weights_from_tensors(p[:3], p, p, gate_scale=s, up_scale=s, down_scale=s)
    with pytest.raises(ValueError, match="permutation"):
        w.load_weights_from_tensors(p, p, p, torch.tensor([0, 0, 1, 2]), gate_scale=s, up_scale=s, down_scale=s)


# ------------------------------------------------------------------------------------------------ GPU
def _rand_experts(E, rows, cols, seed, device="cuda"):
    """random weight_packed (any int32 is a valid word) and bf16 scales on `device`"""
    g = torch.Generator(device=device).manual_seed(seed)
    packed = torch.randint(0, 256, (E * rows * cols // 2,), dtype=torch.uint8, generator=g, device=device).view(torch.int32)
    scale = torch.rand((E, rows, cols // 32), generator=g, device=device) * (1.0 / cols ** 0.5) + 0.25 / cols ** 0.5
    return packed.view(E, rows, cols // 8), scale.to(torch.bfloat16)


def _pack(packed, scale):
    rows, cols = packed.numel() // packed.shape[-1], packed.shape[-1] * 8
    out = torch.empty(rows * cols // 256 * 144, dtype=torch.uint8, device=packed.device)
    native.check(native.lib().ktb200_rawint4_pack(packed.data_ptr(), scale.data_ptr(), rows, cols, out.data_ptr(),
                                                  torch.cuda.current_stream().cuda_stream))
    return out


class _Experts:
    """gate/up/down as packed + scales (device) and as device blocks; expert(e) for the oracle"""

    def __init__(self, E, H, I, seed):
        self.E, self.H, self.I = E, H, I
        self.src = {n: _rand_experts(E, r, c, seed + i) for i, (n, r, c) in enumerate((("gate", I, H), ("up", I, H), ("down", H, I)))}
        self.blocks = {n: _pack(*self.src[n]) for n in self.src}

    def expert(self, e):
        return tuple(o4.dequant(self.src[n][0][e].cpu().numpy(), self.src[n][1][e].cpu().view(torch.int16).numpy().view(np.uint16))
                     for n in ("gate", "up", "down"))

    def moe(self, k, hidden_type, max_tokens=64, offset=0, E=None, lo=0):
        """a handle over experts lo..lo+E-1 (default: all) that owns global ids offset..offset+E-1"""
        from gpu_util import Moe
        E = E or self.E
        sl = [self.blocks[n].view(self.E, -1)[lo:lo + E].reshape(-1) for n in ("gate", "up", "down")]
        return Moe(E, k, self.H, self.I, *sl, I4, I4, I4, hidden_type, max_tokens=max_tokens, offset=offset)


def _x(T, H, seed, hidden_type):
    x = np.random.default_rng(seed).standard_normal((T, H)).astype(np.float32)
    if hidden_type == BF16:
        bits = o4.f32_to_bf16_bits(x)
        return bits, o4.bf16_bits_to_f64(bits)
    return x, x.astype(np.float64)


def _check(got, ref, hidden_type):
    if hidden_type == F32:
        err = np.abs(got.astype(np.float64) - ref).max()
        assert err <= 1e-5 * np.abs(ref).max(), (err, np.abs(ref).max())
    else:
        # bf16 bit patterns -> integers that count representable values in order: |difference| = distance in ulps
        order = lambda b: np.where(b & 0x8000, -(b.astype(np.int64) & 0x7FFF), b.astype(np.int64) & 0x7FFF)
        r_bits = o4.f32_to_bf16_bits(ref.astype(np.float32))
        steps = np.abs(order(got) - order(r_bits))
        # The fp32 re-association error of a dot product scales with its terms, not with its result: where the experts'
        # contributions cancel to far below the layer's output scale, that absolute error (the F32 bound above, measured
        # ~2e-7 * max|out| on an H100) exceeds a bf16 ulp of the small result.  Those elements are held to the F32 bound.
        far = (steps > 1) & (np.abs(o4.bf16_bits_to_f64(got) - ref) > 1e-5 * np.abs(ref).max())
        assert not far.any(), (steps.max(), np.argwhere(far)[:8].tolist())
        assert (steps != 0).mean() <= 1e-3, (steps != 0).mean()


@pytest.mark.gpu
def test_pack_and_dequantize_bit_exact():
    packed, scale = _rand_experts(3, 64, 512, 7)
    blocks = _pack(packed, scale)
    torch.cuda.synchronize()
    p_np, s_np = packed.cpu().numpy(), scale.cpu().view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(blocks.cpu().numpy(), o4.device_layout(p_np, s_np))
    from gpu_util import dequantize
    ref = o4.dequant(p_np, s_np).reshape(-1)
    assert np.array_equal(dequantize(blocks, I4, ref.size, F32).numpy(), ref.astype(np.float32))
    assert torch.equal(dequantize(blocks, I4, ref.size, BF16), torch.from_numpy(ref.astype(np.float32)).to(torch.bfloat16))
    assert torch.equal(dequantize(blocks, I4, ref.size, native.GGML_F16), torch.from_numpy(ref.astype(np.float32)).to(torch.float16))


@pytest.mark.gpu
@pytest.mark.parametrize("hidden_type", [F32, BF16])
@pytest.mark.parametrize("E,k,H,I", [(8, 4, 512, 256), (4, 2, 9216, 512)])
@pytest.mark.parametrize("qlen", [1, 8, 64])
def test_moe_forward_small(hidden_type, E, k, H, I, qlen):
    ex = _Experts(E, H, I, 100 + H)
    m = ex.moe(k, hidden_type)
    rng = np.random.default_rng(qlen)
    ids = np.stack([rng.permutation(E)[:k] for _ in range(qlen)]).astype(np.int64)
    w = rng.random((qlen, k)).astype(np.float32)
    x, x64 = _x(qlen, H, qlen, hidden_type)
    got = m.forward(ids, w, x)
    _check(got, o4.moe_forward(x64, ids, w, ex.expert, E), hidden_type)


# torch.profiler in an interpreter of its own, as test_rawint4_grouped's census at the grouped threshold
_CENSUS = r"""
import json, sys
import numpy as np, torch
sys.path[:0] = sys.argv[1:]
from torch.profiler import ProfilerActivity, profile
from test_rawint4 import F32, _Experts, _x
res = {}
m = _Experts(8, 1024, 512, 5).moe(4, F32)
for T in (1, 8):
    rng = np.random.default_rng(T)
    ids = np.stack([rng.permutation(8)[:4] for _ in range(T)]).astype(np.int64)
    w = rng.random((T, 4)).astype(np.float32)
    x = _x(T, 1024, T, F32)[0]
    m.forward(ids, w, x)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.forward(ids, w, x)
        torch.cuda.synchronize()
    res[T] = [e.key for e in prof.key_averages() if "ktb::" in e.key for _ in range(e.count)]
m.close()
print("CENSUS " + json.dumps(res))
"""


@pytest.mark.gpu
def test_kernels_that_ran_below_the_grouped_threshold():
    """1 and 8 tokens: gate/up on rows_bulk_i4_kernel, down on reduce_bulk_kernel<BulkI4>, and nothing else"""
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CENSUS, here, root]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads(next(l for l in r.stdout.splitlines() if l.startswith("CENSUS "))[7:])
    for T, names in res.items():
        assert len(names) == 2, (T, names)
        gate_up = [n for n in names if "rows_" in n]
        down = [n for n in names if "reduce_" in n]
        assert len(gate_up) == 1 and len(down) == 1, (T, names)
        assert "rows_bulk_i4_kernel<" in gate_up[0], (T, names)
        assert "reduce_bulk_kernel<ktb::BulkI4," in down[0], (T, names)


@pytest.mark.gpu
def test_moe_forward_skips_ids_and_rows_beyond_bsz():
    E, k, H, I, T = 8, 4, 512, 256, 8
    ex = _Experts(E, H, I, 5)
    m = ex.moe(k, F32)
    rng = np.random.default_rng(1)
    ids = np.stack([rng.permutation(E)[:k] for _ in range(T)]).astype(np.int64)
    ids[0, 1], ids[2, 0], ids[3, 3] = -1, E, E + 7
    w = rng.random((T, k)).astype(np.float32)
    x, x64 = _x(T, H, 2, F32)
    out = torch.full((T, H), 1234.5, dtype=torch.float32, device="cuda")
    got = m.forward(ids, w, x, bsz=5, out=out)
    _check(got[:5], o4.moe_forward(x64[:5], ids[:5], w[:5], ex.expert, E), F32)
    assert (got[5:] == 1234.5).all()


@pytest.mark.gpu
def test_expert_id_offset_shards_sum_to_full():
    E, k, H, I, T = 8, 4, 512, 256, 4
    ex = _Experts(E, H, I, 9)
    rng = np.random.default_rng(3)
    ids = np.stack([rng.permutation(E)[:k] for _ in range(T)]).astype(np.int64)
    w = rng.random((T, k)).astype(np.float32)
    x, x64 = _x(T, H, 4, F32)
    full = ex.moe(k, F32).forward(ids, w, x)
    parts = [ex.moe(k, F32, E=4, lo=lo, offset=lo).forward(ids, w, x) for lo in (0, 4)]
    ref = o4.moe_forward(x64, ids, w, ex.expert, E)
    _check(parts[0] + parts[1], ref, F32)
    assert np.abs((parts[0] + parts[1]).astype(np.float64) - full).max() <= 1e-6 * np.abs(ref).max()


@pytest.mark.gpu
def test_moe_block_forward_takes_the_separate_launches():
    from gpu_util import Gate, Mlp, moe_block_forward, gate_forward, moe_forward_shared
    from ktransformers_b200.util.synth import synth_blocks
    E, k, H, I, T = 16, 4, 4096, 512, 3
    ex = _Experts(E, H, I, 11)
    m = ex.moe(k, BF16)
    Q4K = native.GGML_Q4_K
    mlp = Mlp(H, 256, synth_blocks(Q4K, 256 * H, "cuda", 1), synth_blocks(Q4K, 256 * H, "cuda", 2),
              synth_blocks(Q4K, H * 256, "cuda", 3), Q4K, Q4K, Q4K, BF16)
    rng = np.random.default_rng(5)
    W, b = rng.standard_normal((E, H)).astype(np.float32), rng.standard_normal(E).astype(np.float32)
    gate = Gate(W, b, k, 1, 1, hidden_type=BF16)
    x, _ = _x(T, H, 6, BF16)
    out, idx, wt = moe_block_forward(gate, m, mlp, x)
    idx2, wt2, _ = gate_forward(x, W, b, k, 1, 1, hidden_type=BF16)
    assert np.array_equal(idx, idx2) and np.array_equal(wt, wt2)
    assert np.array_equal(out, moe_forward_shared(m, mlp, idx2, wt2, x))
    mlp.close()


@pytest.mark.gpu
def test_forward_ep_refuses_rawint4():
    from gpu_util import Mlp
    from ktransformers_b200.util.synth import synth_blocks
    E, k, H, I = 8, 2, 4096, 512
    m = _Experts(E, H, I, 13).moe(k, BF16)
    Q4K = native.GGML_Q4_K
    mlp = Mlp(H, I, synth_blocks(Q4K, I * H, "cuda", 1), synth_blocks(Q4K, I * H, "cuda", 2), synth_blocks(Q4K, H * I, "cuda", 3),
              Q4K, Q4K, Q4K, BF16)
    ids = torch.zeros((1, k), dtype=torch.int64, device="cuda")
    wt = torch.ones((1, k), device="cuda")
    x = torch.zeros((1, H), dtype=torch.bfloat16, device="cuda")
    part, sh = torch.zeros((1, H), device="cuda"), torch.zeros((H,), dtype=torch.bfloat16, device="cuda")
    rc = native.lib().ktb200_moe_forward_ep(m.h, mlp.h, 1, k, ids.data_ptr(), wt.data_ptr(), x.data_ptr(), part.data_ptr(), 0,
                                            sh.data_ptr(), None, torch.cuda.current_stream().cuda_stream)
    assert rc == native.EINVAL and "RAWINT4" in native.lib().ktb200_last_error().decode()
    mlp.close()


@pytest.mark.gpu
def test_moe_forward_k2_shapes():
    """Kimi-K2 routed experts: E=384, H=7168, I=2048, k=8; qlen 8 over 16 experts and qlen 1; F32 and BF16 hidden."""
    E, k, H, I = 384, 8, 7168, 2048
    ex = _Experts(E, H, I, 2026)    # the oracle pulls only the hit experts to the host
    rng = np.random.default_rng(8)
    hit = rng.permutation(E)[:16]
    ids = np.stack([rng.permutation(hit)[:k] for _ in range(8)]).astype(np.int64)
    w = rng.random((8, k)).astype(np.float32)
    xf, xf64 = _x(8, H, 9, F32)
    xb, xb64 = _x(8, H, 10, BF16)
    ref = o4.moe_forward(np.concatenate([xf64, xb64]), np.concatenate([ids, ids]), np.concatenate([w, w]), ex.expert, E)
    for ht, x, r in ((F32, xf, ref[:8]), (BF16, xb, ref[8:])):
        m = ex.moe(k, ht, max_tokens=8)
        _check(m.forward(ids, w, x), r, ht)
        _check(m.forward(ids[:1], w[:1], x[:1]), r[:1], ht)
        m.close()


@pytest.mark.gpu
def test_ktmoe_wrapper_rawint4_end_to_end(tmp_path):
    E, k, H, I, T = 8, 3, 512, 256, 5
    ref = _write_ct_dir(str(tmp_path), E, H, I, seed=21)
    p2l = torch.tensor([3, 0, 7, 1, 6, 2, 5, 4])
    mask = torch.zeros(E, dtype=torch.bool)
    mask[[2, 5]] = True
    wr = _wrapper(num_experts=E, num_experts_per_tok=k, hidden_size=H, moe_intermediate_size=I, gpu_experts_mask=mask,
                  weight_path=str(tmp_path), chunked_prefill_size=16)
    wr.load_weights(p2l)
    rng = np.random.default_rng(22)
    ids = np.stack([rng.permutation(E)[:k] for _ in range(T)]).astype(np.int64)
    w = rng.random((T, k)).astype(np.float32)
    xb, x64 = _x(T, H, 23, BF16)
    x = torch.from_numpy(xb.view(np.int16)).view(torch.bfloat16).cuda()
    out = wr.forward(x, torch.from_numpy(ids).cuda(), torch.from_numpy(w).cuda())
    torch.cuda.synchronize()
    got = out.cpu().view(torch.int16).numpy().view(np.uint16)

    def expert(pslot):
        le = int(p2l[pslot])
        return tuple(o4.dequant(ref[n][0][le], ref[n][1][le].view(torch.int16).numpy().view(np.uint16)) for n in ("gate", "up", "down"))
    ids_m = np.where(mask.numpy()[ids], -1, ids)
    _check(got, o4.moe_forward(x64, ids_m, w, expert, E), BF16)
