"""The hidden-type and activation contract of every compute entry point (include/ktb200.h).

Every entry point takes its activations and writes its outputs in one of three hidden types (F32, F16, BF16), and the
routed experts take `use_silu` (1: silu(g) * u, 0: relu(g) * u).  Each kernel family has its own hand-written F16 and
BF16 loads and stores, and its own use_silu switch.

  1. CPU: the oracle's own F16 conversion is pinned to numpy's IEEE rounding, its F16 MoE / linear / MLP to its F32 ones,
     and its ReLU experts to a dense float64 restatement.
  2. GPU: for h in {F16, BF16}, x_h in type h and x32 = widen(x_h), every call gives exactly round_h(the F32 call on x32)
     with the same number of launches (round_h: numpy's float16 cast / ggml's bf16 rounding).  The F32 calls are held to
     the oracle elsewhere, so this anchors the narrow types bit for bit; a few direct F16-vs-oracle checks stand beside it.
  3. GPU: use_silu = 0 against the oracle on every path, and the routes that must not take a fused shared-expert slot.
  4. GPU: KTMoEWrapper(dtype=torch.float16) against the same wrapper at torch.float32.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from ktransformers_b200 import native
from ktransformers_b200.util.synth import synth_blocks
from oracle.bindings import BF16, F16, F32, Q4_K, Q5_K, Q6_K, TYPE_NAMES, bf16_to_f32, f32_to_bf16_bits
import gpu_util as G
import int4_oracle as o4
from test_batch_size_contract import fp8_ksplit
from test_gpu_parity import COMBOS, FP_TOL, assert_bf16_close, relmax

gpu = pytest.mark.gpu
NARROW = (F16, BF16)
I4 = native.RAWINT4_G32


# ------------------------------------------------------------------------------------------------ helpers
def to_h(x32, h):
    """float32 -> the numpy carrier of hidden type h: IEEE RNE float16 (overflow to inf) / ggml's bf16 bits / float32"""
    x32 = np.ascontiguousarray(x32, dtype=np.float32)
    if h == F16:
        with np.errstate(over="ignore"):
            return x32.astype(np.float16)
    return f32_to_bf16_bits(x32) if h == BF16 else x32


def widen(xh, h):
    return xh.astype(np.float32) if h == F16 else (bf16_to_f32(xh) if h == BF16 else xh)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def assert_same_bits(got, want, what=""):
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = _bits(got) != _bits(want)
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements differ, first at {i}: got {got[i]!r}, want {want[i]!r}")


def assert_f16_close(got, want, min_exact=0.97, ulps=1):
    """1 fp16 ulp (2^-10 relative) + 1e-3 of the largest value, and more than `min_exact` bit-identical"""
    a, b = got.astype(np.float32), want.astype(np.float32)
    assert np.isfinite(a).all() and np.isfinite(b).all()
    err = np.abs(a - b) - ulps * 2.0 ** -10 * np.maximum(np.abs(a), np.abs(b)) - FP_TOL * np.abs(b).max()
    assert (err <= 0).all(), f"{int((err > 0).sum())} elements outside the bound, worst at {np.unravel_index(err.argmax(), err.shape)}"
    assert (_bits(got) == _bits(want)).mean() > min_exact, (_bits(got) == _bits(want)).mean()


def assert_close_h(got, want, h, **kw):
    if h == F16:
        assert_f16_close(got, want, **kw)
    elif h == BF16:
        assert_bf16_close(got, want, **kw)
    else:
        assert relmax(got, want) < FP_TOL


def two_terms(r, s, h):
    """y = round_h(round_h(R) + round_h(S)), R and S given as fp32 or in the carrier of h"""
    r32, s32 = (v if v.dtype == np.float32 else widen(v, h) for v in (r, s))
    return to_h(widen(to_h(r32, h), h) + widen(to_h(s32, h), h), h)


def assert_two_terms_close(got, r, s, h):
    """y vs oracle R + S, each term rounded to h on its own: one ulp of EACH term (the two may cancel), as
    test_moe_block_full_shape_vs_oracle bounds it; fp32: test_gpu_parity's relative bound"""
    want = two_terms(r, s, h)
    if h == F32:
        assert relmax(got, want) < FP_TOL
        return
    ulp = 2.0 ** -10 if h == F16 else 2.0 ** -7
    a, b = widen(got, h), widen(want, h)
    tol = ulp * (np.abs(widen(r, h)) + np.abs(widen(s, h)) + np.abs(b)) + FP_TOL * np.abs(b).max()
    assert (np.abs(a - b) <= tol).all(), float((np.abs(a - b) / tol).max())
    assert (_bits(got) == _bits(want)).mean() > 0.9


def counted(fn, *args, **kw):
    n0 = native.launch_count()
    r = fn(*args, **kw)
    return r, native.launch_count() - n0


def _synth(t, n, seed):
    return synth_blocks(t, n, device="cuda", seed=seed)


def _x32(rng, rows, cols, scale=0.01):
    return (rng.standard_normal((rows, cols)) * scale).astype(np.float32)


def _routing(rng, qlen, E, k):
    return np.stack([rng.permutation(E)[:k] for _ in range(qlen)]).astype(np.int64), rng.random((qlen, k)).astype(np.float32)


class Experts:
    """routed-expert blocks on the device; every handle gets its own copy (load_weights re-lays Q6_K out in place), and
    the numpy copies for the oracle are taken before the first handle exists"""

    def __init__(self, types, E, H, I, seed, cpu=False):
        self.types, self.E, self.H, self.I = types, E, H, I
        gen = (lambda t, n, s: synth_blocks(t, n, device="cpu", seed=s).cuda()) if cpu else _synth
        self.w = [gen(types[0], E * I * H, seed), gen(types[1], E * I * H, seed + 1), gen(types[2], E * H * I, seed + 2)]
        self.np = [t.cpu().numpy() for t in self.w]

    def moe(self, k, hid, **kw):
        return G.Moe(self.E, k, self.H, self.I, *(t.clone() for t in self.w), *self.types, hid, **kw)

    def mlp(self, hid):
        assert self.E == 1
        return G.Mlp(self.H, self.I, *(t.clone() for t in self.w), *self.types, hid)

    def mlp_forward(self, hid, x, accumulate_into=None):
        assert self.E == 1
        return G.mlp_forward(self.H, self.I, *(t.clone() for t in self.w), *self.types, hid, x, accumulate_into=accumulate_into)

    def oracle_moe(self, oracle, hid, ids, w, x, use_silu=True):
        return oracle.moe_forward(self.E, self.H, self.I, *self.np, *self.types, hid, ids, w, x, use_silu=use_silu)

    def oracle_mlp(self, oracle, hid, x):
        return oracle.mlp_forward(self.H, self.I, *self.np, *self.types, hid, x)


def _mlp_call(mlp, x, hid):
    """ktb200_mlp_forward on an existing handle (an MLP maps H columns to H columns)"""
    x_d = G.dev(x, torch.bfloat16 if hid == BF16 else None)
    out = torch.zeros(x.shape, dtype=G.TORCH_HID[hid], device="cuda")
    native.check(native.lib().ktb200_mlp_forward(mlp.h, x.shape[0], x_d.data_ptr(), out.data_ptr(), 0, None, G.stream()))
    torch.cuda.synchronize()
    return _np(out, hid)


def _np(t, hid):
    t = t.cpu()
    return t.view(torch.int16).numpy().view(np.uint16) if hid == BF16 else t.numpy()


# ================================================================================================ 1. the oracle (CPU)
def _f16_probe_values():
    """float32 inputs at every place an fp32 -> fp16 conversion can go wrong"""
    rng = np.random.default_rng(2024)
    parts = [rng.integers(0, 1 << 32, 1 << 18, dtype=np.uint64).astype(np.uint32).view(np.float32)]   # any bit pattern
    # random bit patterns whose exponent lies in or next to fp16's range
    b = rng.integers(0, 1 << 32, 1 << 18, dtype=np.uint64).astype(np.uint32)
    b = (b & 0x807FFFFF) | (rng.integers(100, 145, b.size).astype(np.uint32) << 23)
    parts.append(b.view(np.float32))
    # every rounding tie between two adjacent finite fp16 values (subnormals included), the values one fp32 ulp either
    # side of it, and their negatives
    h = np.arange(0, 0x7BFF, dtype=np.uint16)
    lo, hi = h.view(np.float16).astype(np.float32), (h + 1).view(np.float16).astype(np.float32)
    mid = (lo + hi) / 2                                   # exact: an fp16 pair has 11 significant bits
    parts += [mid, np.nextafter(mid, np.float32(np.inf)), np.nextafter(mid, np.float32(0))]
    t25, t14 = np.float32(2.0 ** -25), np.float32(2.0 ** -14)
    special = [t25, np.nextafter(t25, np.float32(1)), np.nextafter(t25, np.float32(0)), np.float32(2.0 ** -24), np.float32(2.0 ** -26),
               t14, np.nextafter(t14, np.float32(1)), np.nextafter(t14, np.float32(0)), np.float32(1023 * 2.0 ** -24),
               np.float32(1023.5 * 2.0 ** -24), np.float32(65504), np.float32(65519.99), np.float32(65520),
               np.nextafter(np.float32(65520), np.float32(0)), np.nextafter(np.float32(65520), np.float32(np.inf)), np.float32(65536), np.float32(1e10), np.float32(np.inf),
               np.float32(0.0), np.float32(1.0), np.float32(np.finfo(np.float32).tiny), np.float32(np.finfo(np.float32).max)]
    parts.append(np.array(special, np.float32))
    x = np.concatenate(parts)
    return np.concatenate([x, -x])


def test_oracle_fp32_to_fp16_is_ieee_round_to_nearest_even(oracle):
    x = _f16_probe_values()
    got = oracle.from_float(x, F16).view(np.uint16)
    want = to_h(x, F16).view(np.uint16)
    nan = np.isnan(x)
    assert np.isnan(got[nan].view(np.float16)).all()
    bad = (got != want) & ~nan
    assert not bad.any(), f"{int(bad.sum())} differ, e.g. {x[bad][:4]} -> {got[bad][:4]} (want {want[bad][:4]})"
    # the edges, spelled out
    probe = np.array([2.0 ** -25, np.nextafter(np.float32(2.0 ** -25), np.float32(1)), 65504, 65519.99, np.nextafter(np.float32(65520), np.float32(0)),
                      65520, -65520, np.inf, -np.inf, -0.0], np.float32)
    assert oracle.from_float(probe, F16).view(np.uint16).tolist() == [0x0000, 0x0001, 0x7BFF, 0x7BFF, 0x7BFF, 0x7C00, 0xFC00, 0x7C00, 0xFC00, 0x8000]


def test_oracle_fp16_to_fp32_is_exact_for_every_bit_pattern(oracle):
    h = np.arange(1 << 16, dtype=np.uint32).astype(np.uint16)
    got = oracle.to_float(h.view(np.uint8), F16, h.size)
    want = h.view(np.float16).astype(np.float32)
    nan = np.isnan(want)
    assert np.isnan(got[nan]).all()
    assert np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))


SMALL_COMBOS = [c for c in COMBOS if c[5] <= 1024]


@pytest.mark.parametrize("gt,ut,dt,E,k,H,I", SMALL_COMBOS)
def test_oracle_f16_moe_is_the_rounded_f32_moe(oracle, gt, ut, dt, E, k, H, I):
    ws = [synth_blocks(t, n, "cpu", s).numpy() for t, n, s in ((gt, E * I * H, 1), (ut, E * I * H, 2), (dt, E * H * I, 3))]
    rng = np.random.default_rng(E * 1000 + H)
    ids, w = _routing(rng, 3, E, k)
    x16 = to_h(_x32(rng, 3, H), F16)
    got = oracle.moe_forward(E, H, I, *ws, gt, ut, dt, F16, ids, w, x16)
    want = to_h(oracle.moe_forward(E, H, I, *ws, gt, ut, dt, F32, ids, w, widen(x16, F16)), F16)
    assert_same_bits(got, want, "oracle moe F16")


@pytest.mark.parametrize("t,in_f,out_f", [(Q4_K, 1536, 512), (Q6_K, 512, 100), (Q5_K, 256, 64)])
def test_oracle_f16_linear_and_mlp_are_the_rounded_f32_ones(oracle, t, in_f, out_f):
    rng = np.random.default_rng(in_f + out_f)
    wl = synth_blocks(t, in_f * out_f, "cpu", 5).numpy()
    x16 = to_h(_x32(rng, 3, in_f, 0.1), F16)
    assert_same_bits(oracle.linear_forward(in_f, out_f, wl, t, F16, x16),
                     to_h(oracle.linear_forward(in_f, out_f, wl, t, F32, widen(x16, F16)), F16), "oracle linear F16")
    H, I = in_f, 256
    g, u, d = (synth_blocks(tt, H * I, "cpu", s).numpy() for tt, s in ((Q4_K, 6), (Q4_K, 7), (t, 8)))
    assert_same_bits(oracle.mlp_forward(H, I, g, u, d, Q4_K, Q4_K, t, F16, x16),
                     to_h(oracle.mlp_forward(H, I, g, u, d, Q4_K, Q4_K, t, F32, widen(x16, F16)), F16), "oracle mlp F16")


def _dense_moe(oracle, ex_np, types, E, H, I, ids, w, x, act):
    gd, ud, dd = (oracle.to_float(a, t, E * I * H).astype(np.float64).reshape(shape)
                  for a, t, shape in zip(ex_np, types, ((E, I, H), (E, I, H), (E, H, I))))
    out = np.zeros((x.shape[0], H))
    for t in range(x.shape[0]):
        xt = x[t].astype(np.float64)
        for j in range(ids.shape[1]):
            e = ids[t, j]
            out[t] += w[t, j] * (dd[e] @ (act(gd[e] @ xt) * (ud[e] @ xt)))
    return out


def test_oracle_relu_experts_match_a_dense_restatement(oracle):
    """use_silu=False is relu(g) * u: within test_gpu_operators' 5 % of the output scale of the dense float64 product (int8
    activations), and far from the silu one, so an oracle with the switch inverted fails here"""
    types, E, k, H, I = (Q4_K, Q4_K, Q6_K), 8, 4, 1024, 512
    ws = [synth_blocks(t, n, "cpu", s).numpy() for t, n, s in zip(types, (E * I * H, E * I * H, E * H * I), (11, 12, 13))]
    rng = np.random.default_rng(4)
    ids, w = _routing(rng, 4, E, k)
    x = _x32(rng, 4, H)
    got = oracle.moe_forward(E, H, I, *ws, *types, F32, ids, w, x, use_silu=False)
    relu = _dense_moe(oracle, ws, types, E, H, I, ids, w, x, lambda v: np.maximum(v, 0.0))
    silu = _dense_moe(oracle, ws, types, E, H, I, ids, w, x, lambda v: v / (1.0 + np.exp(-v)))
    assert np.abs(got - relu).max() <= 0.05 * np.abs(relu).max()
    assert np.abs(got - silu).max() > 0.2 * np.abs(silu).max()


# ================================================================================================ 2. F16 / BF16 == round(F32)
@gpu
@pytest.mark.parametrize("gt,ut,dt,E,k,H,I", COMBOS)
def test_moe_forward_narrow_is_rounded_f32(gt, ut, dt, E, k, H, I):
    """register-staged, pipelined and bulk-copy kernels; F16 and BF16 against the F32 handle on the widened input"""
    ex = Experts((gt, ut, dt), E, H, I, 1)
    m32 = ex.moe(k, F32)
    rng = np.random.default_rng(E * 1000 + H)
    for h in NARROW:
        mh = ex.moe(k, h)
        for qlen in (1, 9, 33):
            ids, w = _routing(rng, qlen, E, k)
            xh = to_h(_x32(rng, qlen, H), h)
            got, nh = counted(mh.forward, ids, w, xh)
            want, n32 = counted(m32.forward, ids, w, widen(xh, h))
            assert nh == n32 == 2
            assert_same_bits(got, to_h(want, h), f"{TYPE_NAMES[gt]}/{TYPE_NAMES[ut]}/{TYPE_NAMES[dt]} {TYPE_NAMES[h]} qlen={qlen}")
            if h == F16 and qlen == 9:
                assert_same_bits(mh.forward_host(ids, w, xh), got, "ktb200_moe_forward_host")
        mh.close()
    m32.close()


@gpu
@pytest.mark.parametrize("dt,qlen", [(Q6_K, 131), (Q4_K, 131), (Q6_K, 1084)])
def test_grouped_narrow_is_rounded_f32(dt, qlen):
    """the grouped tensor-core path (10 launches per 1024-token chunk); 1084 tokens put the second chunk at a byte offset of
    1024 * H * sizeof(hidden)"""
    E, k, H, I = 8, 4, 1024, 512
    ex = Experts((Q4_K, Q4_K, dt), E, H, I, 21)
    rng = np.random.default_rng(qlen + dt)
    ids, w = _routing(rng, qlen, E, k)
    ids[5:90, 0] = 1                      # a crowded expert
    ids[7, :] = [-1, E, 1 << 40, -7]      # invalid ids are skipped
    x32 = _x32(rng, qlen, H)
    m32 = ex.moe(k, F32, max_tokens=qlen)
    for h in NARROW:
        xh = to_h(x32, h)
        mh = ex.moe(k, h, max_tokens=qlen)
        got, nh = counted(mh.forward, ids, w, xh)
        want, n32 = counted(m32.forward, ids, w, widen(xh, h))
        assert nh == n32 == 10 * ((qlen + 1023) // 1024)
        assert_same_bits(got, to_h(want, h), f"grouped {TYPE_NAMES[h]} qlen={qlen}")
        mh.close()
    m32.close()


def _rawint4(E, H, I, seed):
    from test_rawint4 import _Experts
    return _Experts(E, H, I, seed)


def _rawint4_moe(ex, k, hid, use_silu=1):
    sl = [ex.blocks[n] for n in ("gate", "up", "down")]
    return G.Moe(ex.E, k, ex.H, ex.I, *sl, I4, I4, I4, hid, max_tokens=64, use_silu=use_silu)


@gpu
@pytest.mark.parametrize("qlen", [1, 64])
def test_rawint4_narrow_is_rounded_f32(qlen):
    E, k, H, I = 8, 4, 512, 256
    ex = _rawint4(E, H, I, 31)
    rng = np.random.default_rng(qlen)
    ids, w = _routing(rng, qlen, E, k)
    x32 = rng.standard_normal((qlen, H)).astype(np.float32)
    m32 = _rawint4_moe(ex, k, F32)
    for h in NARROW:
        xh = to_h(x32, h)
        got, nh = counted(_rawint4_moe(ex, k, h).forward, ids, w, xh)
        want, n32 = counted(m32.forward, ids, w, widen(xh, h))
        assert nh == n32
        assert_same_bits(got, to_h(want, h), f"RAWINT4 {TYPE_NAMES[h]} qlen={qlen}")


@gpu
@pytest.mark.parametrize("t,in_f,out_f", [(Q6_K, 2048, 512), (Q5_K, 1536, 512), (Q4_K, 7168, 2112), (Q4_K, 256, 777)])
def test_linear_narrow_is_rounded_f32(t, in_f, out_f):
    """register-staged rows (Q6_K, Q5_K) and the dense segment-ring kernel (Q4_K), with and without bias"""
    wt = _synth(t, out_f * in_f, 31)
    rng = np.random.default_rng(in_f)
    x32 = _x32(rng, 5, in_f, 0.1)
    bias = rng.standard_normal(out_f).astype(np.float32)
    for h in NARROW:
        xh = to_h(x32, h)
        for b in (None, bias):
            got, nh = counted(G.linear_forward, in_f, out_f, wt.clone(), t, h, xh, bias=b)
            want, n32 = counted(G.linear_forward, in_f, out_f, wt.clone(), t, F32, widen(xh, h), bias=b)
            assert nh == n32
            assert_same_bits(got, to_h(want, h), f"linear {TYPE_NAMES[t]} {TYPE_NAMES[h]} bias={b is not None}")


@gpu
@pytest.mark.parametrize("H,I,dt", [(512, 256, Q6_K), (4096, 512, Q6_K), (1024, 512, Q4_K)])
def test_mlp_narrow_is_rounded_f32(H, I, dt):
    """accumulate 0: round_h(mlp(x32)); accumulate 1: round_h(widen(y_h) + round_h(mlp(x32))) (gemv.cuh's epilogue)"""
    ex = Experts((Q4_K, Q4_K, dt), 1, H, I, 41)
    rng = np.random.default_rng(H)
    x32 = _x32(rng, 4, H, 0.1)
    y32 = rng.standard_normal((4, H)).astype(np.float32)
    for h in NARROW:
        xh, yh = to_h(x32, h), to_h(y32, h)
        got, nh = counted(ex.mlp_forward, h, xh)
        s32, n32 = counted(ex.mlp_forward, F32, widen(xh, h))
        assert nh == n32
        assert_same_bits(got, to_h(s32, h), f"mlp {TYPE_NAMES[h]}")
        got_acc = ex.mlp_forward(h, xh, accumulate_into=yh)
        assert_same_bits(got_acc, to_h(widen(yh, h) + widen(to_h(s32, h), h), h), f"mlp accumulate {TYPE_NAMES[h]}")


@gpu
@pytest.mark.parametrize("H,sgt,sdt,fused,qlens", [(1024, Q4_K, Q6_K, True, (1, 5)), (4096, Q4_K, Q6_K, True, (1, 5)),
                                                  (1024, Q5_K, Q4_K, False, (1, 5)), (4096, Q5_K, Q4_K, False, (1, 5)),
                                                  (1024, Q4_K, Q6_K, False, (60,))])
def test_moe_forward_shared_narrow_is_two_rounded_f32_terms(H, sgt, sdt, fused, qlens):
    """the shared expert as slot k of the routed launches, as a separate MLP, and after the grouped path (60 tokens):
    round_h(round_h(R) + round_h(S)) with R, S the F32 routed and F32 MLP calls on x32"""
    E, k, I = 8, 4, 512
    ex = Experts((Q4_K, Q4_K, Q6_K), E, H, I, 71)
    sh = Experts((sgt, sgt, sdt), 1, H, I, 74)
    m32 = ex.moe(k, F32)
    rng = np.random.default_rng(H + sgt)
    for h in NARROW:
        mh, mlph = ex.moe(k, h), sh.mlp(h)
        for qlen in qlens:
            ids, w = _routing(rng, qlen, E, k)
            xh = to_h(_x32(rng, qlen, H), h)
            x32 = widen(xh, h)
            got, n = counted(G.moe_forward_shared, mh, mlph, ids, w, xh)
            assert n == (12 if qlen >= 48 else 2 if fused else 4), n
            r32, s32 = m32.forward(ids, w, x32), sh.mlp_forward(F32, x32)
            assert_same_bits(got, two_terms(r32, s32, h), f"shared {TYPE_NAMES[h]} H={H} qlen={qlen}")
        mh.close(); mlph.close()
    m32.close()


@gpu
@pytest.mark.parametrize("dt,H,I,shared", [(Q6_K, 4096, 512, True), (Q4_K, 4096, 2048, False), (Q6_K, 1024, 512, True)])
def test_moe_block_narrow_is_rounded_f32(dt, H, I, shared):
    """the single persistent launch (qlen <= 8, H = 4096) and the separate launches behind the same call (qlen 9, and
    H = 1024 at every qlen): ids and weights bit-equal to the F32 block call, output = the two rounded F32 terms"""
    Eg, k, ng, tg = 16, 4, 4, 2
    ex = Experts((Q4_K, Q4_K, dt), Eg, H, I, 81)
    sh = Experts((Q4_K, Q4_K, dt), 1, H, I, 84) if shared else None
    rng = np.random.default_rng(H + I)
    W, bias = rng.standard_normal((Eg, H)).astype(np.float32), rng.standard_normal(Eg).astype(np.float32)
    m32, g32 = ex.moe(k, F32, max_tokens=16), G.Gate(W, bias, k, ng, tg, hidden_type=F32)
    mlp32 = sh.mlp(F32) if shared else None
    for h in NARROW:
        mh, gh = ex.moe(k, h, max_tokens=16), G.Gate(W, bias, k, ng, tg, hidden_type=h)
        mlph = sh.mlp(h) if shared else None
        for qlen in (1, 3, 8, 9):
            xh = to_h(_x32(rng, qlen, H, 0.1), h)
            x32 = widen(xh, h)
            (out, idx, w), nh = counted(G.moe_block_forward, gh, mh, mlph, xh)
            (out32, idx32, w32), n32 = counted(G.moe_block_forward, g32, m32, mlp32, x32)
            assert nh == n32 and (nh == 1) == (H >= 4096 and qlen <= 8), nh
            assert_same_bits(idx, idx32, "block ids")
            assert_same_bits(w, w32, "block weights")
            r32 = m32.forward(idx, w, x32)
            want = two_terms(r32, _mlp_call(mlp32, x32, F32), h) if shared else to_h(r32, h)
            assert_same_bits(out, want, f"block {TYPE_NAMES[h]} H={H} qlen={qlen}")
        mh.close()
        if mlph is not None:
            mlph.close()


@gpu
@pytest.mark.parametrize("E,H,k,ng,tg,scoring,method,norm,scale", [
    (256, 7168, 8, 8, 4, 0, 0, 1, 2.5), (384, 7168, 8, 1, 1, 0, 0, 1, 2.827), (64, 2048, 6, 1, 1, 1, 1, 0, 1.0),
    (160, 5120, 6, 8, 3, 1, 2, 0, 16.0)])
def test_gate_narrow_is_the_f32_router_on_the_widened_input(E, H, k, ng, tg, scoring, method, norm, scale):
    """the router widens x to fp32 as it loads it: ids, weights and logits are the F32 call's bits"""
    rng = np.random.default_rng(42)
    W = rng.standard_normal((E, H)).astype(np.float32)
    bias = rng.standard_normal(E).astype(np.float32) if method == 0 else None
    x32 = _x32(rng, 64, H, 0.1)
    for h in NARROW:
        xh = to_h(x32, h)
        (idx, w, lg), nh = counted(G.gate_forward, xh, W, bias, k, ng, tg, scoring, method, norm, scale, hidden_type=h, want_logits=True)
        (idx32, w32, lg32), n32 = counted(G.gate_forward, widen(xh, h), W, bias, k, ng, tg, scoring, method, norm, scale, want_logits=True)
        assert nh == n32
        for a, b, n in ((idx, idx32, "ids"), (w, w32, "weights"), (lg, lg32, "logits")):
            assert_same_bits(a, b, f"router {TYPE_NAMES[h]} {n}")


def _fp8_case(rng, T, K, N):
    from oracle import fp8_oracle as F
    x32 = _x32(rng, T, K, 0.1)
    w = F.to_e4m3_bytes((rng.standard_normal((N, K)) * 0.7).astype(np.float32))
    ws = (rng.random(((N + 127) // 128, K // 128)) * 0.02 + 0.001).astype(np.float32)
    return x32, w, ws


def _fp8_run(xh, w, ws, hid):
    lib = native.lib()
    T, K = xh.shape
    N = w.shape[0]
    w_d, ws_d = torch.from_numpy(w).cuda(), torch.from_numpy(ws).cuda()
    x_d = G.dev(xh, torch.bfloat16 if hid == BF16 else None)
    y_d = torch.zeros((T, N), dtype=G.TORCH_HID[hid], device="cuda")
    h = C.c_void_p()
    native.check(lib.ktb200_fp8_linear_create(K, N, w_d.data_ptr(), ws_d.data_ptr(), hid, 0, C.byref(h)))
    n0 = native.launch_count()
    native.check(lib.ktb200_fp8_linear_forward(h, T, x_d.data_ptr(), y_d.data_ptr(), None, G.stream()))
    torch.cuda.synchronize()
    n = native.launch_count() - n0
    lib.ktb200_fp8_linear_destroy(h)
    return _np(y_d, hid), n


@gpu
@pytest.mark.parametrize("T,K,N", [(1, 256, 256), (2, 1024, 256), (3, 1536, 24576), (5, 128, 128), (8, 7168, 2112), (20, 512, 384),
                                   (20, 1024, 200), (20, 1536, 256)])
def test_fp8_linear_narrow_is_rounded_f32(T, K, N):
    """in-kernel act quant (T <= 2), the separate quant kernel, two 16-token chunks, K splits; the F32 and F16 inputs have
    never run before.  Up to two K splits the sum is exact; from three on fp32 atomics reorder it, and the bound is
    test_fp8_linear_vs_oracle's one ulp"""
    from oracle import fp8_oracle as F
    rng = np.random.default_rng(T * 100003 + K + N)
    x32, w, ws = _fp8_case(rng, T, K, N)
    exact = fp8_ksplit(K, N) <= 2
    for h in NARROW:
        xh = to_h(x32, h)
        got, nh = _fp8_run(xh, w, ws, h)
        y32, n32 = _fp8_run(widen(xh, h), w, ws, F32)
        assert nh == n32
        if exact:
            assert_same_bits(got, to_h(y32, h), f"fp8 linear {TYPE_NAMES[h]}")
        else:
            assert_close_h(got, to_h(y32, h), h)
        if h == F16:
            assert_f16_close(got, to_h(F.linear_forward(widen(xh, h), w, ws), F16))   # and directly against the oracle


@gpu
@pytest.mark.parametrize("name", ["Q2_K", "Q3_K", "Q4_K", "Q5_K", "Q6_K", "IQ4_XS", "Q8_0"])
def test_dequantize_f16_is_rounded_f32(golden_dir, name):
    g = np.load(os.path.join(golden_dir, "dequant.npz"))
    t = {n: i for i, n in TYPE_NAMES.items()}[name]
    n = g[f"val_{name}"].size
    f32 = G.dequantize(g[f"raw_{name}"], t, n, F32).numpy()
    for h in NARROW:
        got = _np(G.dequantize(g[f"raw_{name}"], t, n, h), h)
        assert_same_bits(got, to_h(f32, h), f"dequantize {name} -> {TYPE_NAMES[h]}")


@gpu
@pytest.mark.parametrize("H,I", [(512, 256), (4096, 512)])
def test_f16_output_overflows_to_inf_exactly_where_fp32_passes_65504(H, I):
    """routing weights that push one token's fp32 output past the fp16 range: +-inf exactly where numpy's cast puts it"""
    E, k = 8, 4
    ex = Experts((Q4_K, Q4_K, Q6_K), E, H, I, 91)
    m32, m16 = ex.moe(k, F32), ex.moe(k, F16)
    rng = np.random.default_rng(H)
    ids, w = _routing(rng, 2, E, k)
    x16 = to_h(_x32(rng, 2, H), F16)
    w[1] *= 2.0e5 / np.abs(m32.forward(ids, w, widen(x16, F16))[1]).max()
    want32 = m32.forward(ids, w, widen(x16, F16))
    got = m16.forward(ids, w, x16)
    assert_same_bits(got, to_h(want32, F16), "F16 output at the overflow edge")
    assert np.isinf(got[1]).any() and np.isfinite(got[1]).any() and np.isfinite(got[0]).all()
    assert (np.isinf(got[1]) == (np.abs(want32[1]) >= 65520)).all()


@gpu
def test_moe_ep_block_loopback_f16_matches_the_single_gpu_f16_block():
    """ktb200_moe_ep_block_forward at world 2 with F16 token messages, emulated on one GPU as
    test_moe_ep_block_loopback_matches_single_gpu does: the same routing bits as the single-GPU F16 block, the output within
    fp32 re-association of the partial sums (2 fp16 ulps, > 90 % identical)"""
    _ep_loopback(F16, shared=True, use_silu=1)


def _ep_loopback(hid, shared, use_silu, world=2):
    lib = native.lib()
    E, k, H, I, ng, tg = 32, 4, 4096, 512, 4, 2
    El = E // world
    gate_w, up_w, down_w = _synth(Q4_K, E * I * H, 401), _synth(Q4_K, E * I * H, 402), _synth(Q6_K, E * H * I, 403)
    sgs = (_synth(Q4_K, I * H, 404), _synth(Q4_K, I * H, 405), _synth(Q6_K, H * I, 406))
    gb, db = gate_w.numel() // E, down_w.numel() // E
    rng = np.random.default_rng(world + hid)
    Wr, bias = rng.standard_normal((E, H)).astype(np.float32), rng.standard_normal(E).astype(np.float32)
    gate = G.Gate(Wr, bias, k, ng, tg, hidden_type=hid)
    full = G.Moe(E, k, H, I, gate_w.clone(), up_w.clone(), down_w.clone(), Q4_K, Q4_K, Q6_K, hid, max_tokens=8, use_silu=use_silu)
    full_mlp = G.Mlp(H, I, *(t.clone() for t in sgs), Q4_K, Q4_K, Q6_K, hid) if shared else None
    shards, mlps = [], []
    for r in range(world):
        sl = slice(r * El, (r + 1) * El)
        shards.append(G.Moe(El, k, H, I, gate_w[sl.start * gb: sl.stop * gb].clone(), up_w[sl.start * gb: sl.stop * gb].clone(),
                            down_w[sl.start * db: sl.stop * db].clone(), Q4_K, Q4_K, Q6_K, hid, max_tokens=8, offset=sl.start,
                            use_silu=use_silu))
        mlps.append(G.Mlp(H, I, *(t.clone() for t in sgs), Q4_K, Q4_K, Q6_K, hid) if shared else None)
    msgb = lib.ktb200_ep_msg_bytes(H, hid)
    msg = [torch.zeros(world * msgb, dtype=torch.uint8, device="cuda") for _ in range(world)]
    part = [torch.zeros((world, H), dtype=torch.float32, device="cuda") for _ in range(world)]
    flags = [torch.zeros(2 * world + 2, dtype=torch.int32, device="cuda") for _ in range(world)]
    comms = [native.EpComm.make(r, world, H, hid, [t.data_ptr() for t in msg], [t.data_ptr() for t in part], [t.data_ptr() for t in flags])
             for r in range(world)]
    dtype = G.TORCH_HID[hid]
    for layer in range(2):
        xs = [to_h(_x32(rng, 1, H, 0.1), hid) for _ in range(world)]
        x_d = [G.dev(x, torch.bfloat16 if hid == BF16 else None) for x in xs]
        y = [torch.zeros((1, H), dtype=dtype, device="cuda") for _ in range(world)]
        idx = [torch.zeros((1, k), dtype=torch.int64, device="cuda") for _ in range(world)]
        w = [torch.zeros((1, k), dtype=torch.float32, device="cuda") for _ in range(world)]
        for mask in (1, 2, 4):
            for r in range(world):
                native.check(lib.ktb200_moe_ep_block_forward(C.byref(gate.cfg), shards[r].h, mlps[r].h if shared else None, C.byref(comms[r]),
                                                             x_d[r].data_ptr(), y[r].data_ptr(), idx[r].data_ptr(), w[r].data_ptr(), mask, G.stream()))
        torch.cuda.synchronize()
        for r in range(world):
            assert int(flags[r][2 * world + 1]) == 0, "a peer wait timed out"
            (want, widx, ww), n = counted(G.moe_block_forward, gate, full, full_mlp, xs[r])
            assert n == 1, "the single-GPU block must be the one persistent launch"
            assert np.array_equal(idx[r].cpu().numpy(), widx) and np.array_equal(w[r].cpu().numpy(), ww)
            assert_close_h(_np(y[r], hid), want, hid, min_exact=0.9, ulps=2)
    for m_ in shards + mlps + [full, full_mlp]:
        if m_ is not None:
            m_.close()


@gpu
def test_f16_direct_vs_oracle(oracle):
    """one check per path that does not go through the F32 relation: 1 fp16 ulp + 1e-3 of the largest value, > 97 % identical"""
    rng = np.random.default_rng(77)
    for types, E, k, H, I, qlen, mt in (((Q4_K, Q4_K, Q6_K), 8, 4, 1024, 512, 9, 64),      # register-staged
                                        ((Q4_K, Q4_K, Q6_K), 4, 3, 4096, 512, 5, 64),      # bulk-copy
                                        ((Q4_K, Q4_K, Q6_K), 8, 4, 1024, 512, 131, 256)):  # grouped
        ex = Experts(types, E, H, I, 5)
        ids, w = _routing(rng, qlen, E, k)
        x16 = to_h(_x32(rng, qlen, H), F16)
        got = ex.moe(k, F16, max_tokens=mt).forward(ids, w, x16)
        assert_f16_close(got, ex.oracle_moe(oracle, F16, ids, w, x16))
    ex = Experts((Q4_K, Q4_K, Q6_K), 1, 1024, 512, 6)
    x16 = to_h(_x32(rng, 4, 1024, 0.1), F16)
    assert_f16_close(ex.mlp_forward(F16, x16), ex.oracle_mlp(oracle, F16, x16))
    wl = _synth(Q4_K, 7168 * 2112, 7)
    x16 = to_h(_x32(rng, 3, 7168, 0.1), F16)
    assert_f16_close(G.linear_forward(7168, 2112, wl.clone(), Q4_K, F16, x16), oracle.linear_forward(7168, 2112, wl.cpu().numpy(), Q4_K, F16, x16))
    # RAWINT4 against its float64 oracle
    ex4 = _rawint4(8, 512, 256, 33)
    ids, w = _routing(rng, 8, 8, 4)
    x16 = to_h(rng.standard_normal((8, 512)).astype(np.float32), F16)
    got = _rawint4_moe(ex4, 4, F16).forward(ids, w, x16)
    assert_f16_close(got, to_h(o4.moe_forward(widen(x16, F16).astype(np.float64), ids, w, ex4.expert, 8).astype(np.float32), F16))


# ================================================================================================ 3. ReLU experts vs the oracle
@gpu
@pytest.mark.parametrize("gt,ut,dt,E,k,H,I", COMBOS)
def test_relu_moe_forward_vs_oracle(oracle, gt, ut, dt, E, k, H, I):
    ex = Experts((gt, ut, dt), E, H, I, 1)
    rng = np.random.default_rng(E * 1000 + H + 1)
    for hid in (F32, BF16):
        m = ex.moe(k, hid, use_silu=0)
        for qlen in (1, 2, 9, 33):
            ids, w = _routing(rng, qlen, E, k)
            x = to_h(_x32(rng, qlen, H), hid)
            got, n = counted(m.forward, ids, w, x)
            assert n == 2
            assert_close_h(got, ex.oracle_moe(oracle, hid, ids, w, x, use_silu=False), hid)
        m.close()


@gpu
@pytest.mark.parametrize("dt", [Q6_K, Q4_K])
def test_relu_grouped_vs_oracle(oracle, dt):
    E, k, H, I, qlen = 8, 4, 1024, 512, 131
    ex = Experts((Q4_K, Q4_K, dt), E, H, I, 21)
    rng = np.random.default_rng(dt)
    for hid in (F32, BF16):
        ids, w = _routing(rng, qlen, E, k)
        ids[5:90, 0] = 1
        x = to_h(_x32(rng, qlen, H), hid)
        got, n = counted(ex.moe(k, hid, max_tokens=256, use_silu=0).forward, ids, w, x)
        assert n == 10, "the grouped path did not run"
        assert_close_h(got, ex.oracle_moe(oracle, hid, ids, w, x, use_silu=False), hid)


@gpu
@pytest.mark.parametrize("E,k,H,I", [(8, 4, 512, 256), (4, 2, 9216, 512)])
def test_relu_rawint4_vs_oracle(E, k, H, I):
    from test_rawint4 import _check, _x
    ex = _rawint4(E, H, I, 100 + H)
    for hid in (F32, BF16):
        m = _rawint4_moe(ex, k, hid, use_silu=0)
        for qlen in (1, 8, 64):
            rng = np.random.default_rng(qlen)
            ids, w = _routing(rng, qlen, E, k)
            x, x64 = _x(qlen, H, qlen, hid)
            _check(m.forward(ids, w, x), o4.moe_forward(x64, ids, w, ex.expert, E, use_silu=False), hid)


def _block_setup(dt, H, I, hid, use_silu, shared, Eg=16, k=4, ng=4, tg=2, seed=81):
    ex = Experts((Q4_K, Q4_K, dt), Eg, H, I, seed)
    sh = Experts((Q4_K, Q4_K, dt), 1, H, I, seed + 3) if shared else None
    rng = np.random.default_rng(H + I + hid)
    W, bias = rng.standard_normal((Eg, H)).astype(np.float32), rng.standard_normal(Eg).astype(np.float32)
    return ex, sh, ex.moe(k, hid, max_tokens=16, use_silu=use_silu), (sh.mlp(hid) if shared else None), G.Gate(W, bias, k, ng, tg, hidden_type=hid), W, bias, rng


@gpu
@pytest.mark.parametrize("dt,I", [(Q6_K, 512), (Q4_K, 2048)])
@pytest.mark.parametrize("hid", [F32, BF16])
def test_relu_moe_block_single_launch_vs_oracle(oracle, dt, I, hid):
    """no shared expert: ReLU experts stay in the one persistent launch"""
    H, k = 4096, 4
    ex, _, m, _, gate, W, bias, rng = _block_setup(dt, H, I, hid, 0, False)
    for qlen in (1, 3, 8):
        x = to_h(_x32(rng, qlen, H, 0.1), hid)
        (out, idx, w), n = counted(G.moe_block_forward, gate, m, None, x)
        assert n == 1
        ridx, rw, _ = G.gate_forward(x, W, bias, k, 4, 2, hidden_type=hid)
        assert np.array_equal(idx, ridx) and np.array_equal(w, rw)
        assert_close_h(out, ex.oracle_moe(oracle, hid, idx, w, x, use_silu=False), hid)


@gpu
@pytest.mark.parametrize("hid", [F32, BF16])
def test_relu_moe_block_with_shared_expert_takes_the_separate_launches(oracle, hid):
    """the MLP handle always applies silu: a ReLU layer with a shared expert cannot use the single launch; the result is
    the ReLU routed term + the silu shared term, rounded apart"""
    H, I, k = 4096, 512, 4
    ex, sh, m, mlp, gate, W, bias, rng = _block_setup(Q6_K, H, I, hid, 0, True)
    for qlen in (1, 3, 8):
        x = to_h(_x32(rng, qlen, H, 0.1), hid)
        (out, idx, w), n = counted(G.moe_block_forward, gate, m, mlp, x)
        assert n > 1, "a ReLU layer with a shared expert took the single launch"
        assert_same_bits(out, G.moe_forward_shared(m, mlp, idx, w, x), "block == router + forward_shared")
        assert_two_terms_close(out, ex.oracle_moe(oracle, hid, idx, w, x, use_silu=False), sh.oracle_mlp(oracle, hid, x), hid)


@gpu
@pytest.mark.parametrize("H,qlen", [(1024, 1), (1024, 5), (4096, 1), (4096, 5), (1024, 60)])
@pytest.mark.parametrize("hid", [F32, BF16])
def test_relu_moe_forward_shared_takes_the_separate_mlp(oracle, H, qlen, hid):
    """shared expert of the routed experts' types (it would ride as slot k under silu): with ReLU routed experts it runs as
    the separate silu MLP (2 + 2 launches; 10 + 2 after the grouped path)"""
    E, k, I = 8, 4, 512
    ex = Experts((Q4_K, Q4_K, Q6_K), E, H, I, 71, cpu=True)
    sh = Experts((Q4_K, Q4_K, Q6_K), 1, H, I, 74, cpu=True)
    m, mlp = ex.moe(k, hid, use_silu=0), sh.mlp(hid)
    rng = np.random.default_rng(H + qlen)
    ids, w = _routing(rng, qlen, E, k)
    x = to_h(_x32(rng, qlen, H), hid)
    got, n = counted(G.moe_forward_shared, m, mlp, ids, w, x)
    assert n == (4 if qlen < 48 else 12)
    assert_two_terms_close(got, ex.oracle_moe(oracle, hid, ids, w, x, use_silu=False), sh.oracle_mlp(oracle, hid, x), hid)
    m.close(); mlp.close()


@gpu
def test_relu_moe_ep_block_loopback_matches_the_single_gpu_block():
    """the expert-parallel kernel's own gate/up epilogue with use_silu = 0 (no shared expert: the single-GPU block is one
    launch, and test_relu_moe_block_single_launch_vs_oracle holds it to the oracle)"""
    _ep_loopback(BF16, shared=False, use_silu=0)


# ================================================================================================ 4. operator level
@gpu
def test_kt_moe_wrapper_f16_is_the_rounded_f32_wrapper(tmp_path):
    from ktransformers_b200.kt_moe_wrapper import KTMoEWrapper
    from test_gpu_operators import E, H, I, K, _write_gguf
    _write_gguf(str(tmp_path / "tiny.gguf"))
    KTMoEWrapper.clear_buffer_cache()
    wr = {dt: KTMoEWrapper(1, E, K, H, I, None, weight_path=str(tmp_path), chunked_prefill_size=16, dtype=dt)
          for dt in (torch.float16, torch.float32)}
    for w_ in wr.values():
        w_.load_weights()
    assert wr[torch.float16].moe.hidden_type == F16 and wr[torch.float32].moe.hidden_type == F32
    g = torch.Generator(device="cpu").manual_seed(5)
    n_tok = 5
    x16 = (torch.randn(n_tok, H, generator=g) / 10).to(torch.float16).cuda()
    ids = torch.stack([torch.randperm(E, generator=g)[:K] for _ in range(n_tok)]).cuda()
    wt = torch.rand(n_tok, K, generator=g).cuda()
    y16 = wr[torch.float16].forward(x16, ids, wt).clone()
    y32 = wr[torch.float32].forward(x16.float(), ids, wt)
    torch.cuda.synchronize()
    assert y16.dtype == torch.float16 and y32.dtype == torch.float32
    assert torch.equal(y16.view(torch.int16), y32.to(torch.float16).view(torch.int16))
