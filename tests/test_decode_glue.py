"""The small kernels between the projections of a DeepSeek decode layer (csrc/elementwise.cu: ktb200_add_rmsnorm,
ktb200_mla_prep, ktb200_mla_absorb_q / _o; csrc/mla.cu: ktb200_mla_kv_write) against the float64 oracle of
tests/decode_glue_oracle.py, and their programmatic-dependent chain as bench.py's whole-decode leg runs it.

Shapes cover DeepSeek-V3/R1 and V2 (128 heads), Kimi-K2 (64 heads) and V2-Lite (16 heads).  Bounds:
  * norms (add_rmsnorm, the latent columns of mla_prep): every element within 2 bf16 ulps of the oracle and at least
    99.5 % bit-identical.  The kernel's fp32 variance sum and rsqrtf move 1/rms by about 1e-6 relative, so a bf16 rounding
    flips only where r / rms lies that close to a rounding midpoint.  Measured on an H100 80GB HBM3 (700 W):
    add_rmsnorm at least 99.994 % identical in every case (2 ulps worst), the latent columns at least 99.998 % (1 ulp).
  * RoPE: with bf16-valued tables (the module's tables after .to(bf16), passed as fp32) the kernel's arithmetic is the
    module's (bf16 products, one fp32 sum, one rounding): bit-identical.  With raw fp32 tables the kernel rounds each
    product to fp32 before bf16; a product that lands on a bf16 midpoint that way is one product ulp off, and where the
    two products nearly cancel that is many ulps of the result (up to 15232 ulps of a near-zero output measured), so no
    ulp bound against exact products holds.  Those cases are bit-identical to the oracle with fp32 products, and at
    least 99.9 % identical to exact products (measured at least 99.988 %).
  * absorb GEMVs: |got - want| <= 2^-8 |want| + 2 L 2^-24 sum|q W| (bf16 output rounding plus fp32 accumulation over L
    terms) and at least 99 % bit-identical to bf16(want).  Measured: worst 0.994 of the bound (the bf16 rounding term
    itself), at least 99.98 % identical.
The worst error of each case as a fraction of its bound, and the bit-identical fraction, are printed (pytest -s)."""
import ctypes as C

import numpy as np
import pytest
import torch

import decode_glue_oracle as dgo
from ktransformers_b200 import native
from oracle import mla_oracle

EPS = float(np.float32(1e-6))     # what the kernels receive as a C float
gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ helpers
def to_bits(x64):
    """bf16-valued float array -> uint16 bit patterns"""
    return (np.ascontiguousarray(x64, np.float32).view(np.uint32) >> 16).astype(np.uint16)


def dev_bits(t):
    return t.contiguous().cpu().view(torch.int16).numpy().view(np.uint16)


def f64(t):
    return t.float().cpu().numpy().astype(np.float64)


def ulps(a, b):
    """distance in bf16 steps between two arrays of bit patterns (+0 and -0 are 0 apart)"""
    o = [np.where(x.astype(np.int32) & 0x8000, -(x.astype(np.int32) & 0x7FFF), x.astype(np.int32)) for x in (a, b)]
    return np.abs(o[0] - o[1])


def _report(family, case, **vals):
    print(f"[{family}] {case}: " + ", ".join(f"{k} {v:.6f}" for k, v in vals.items()))


def check_norm(family, case, got_bits, want64, min_identical=0.995):
    d = ulps(got_bits, to_bits(want64))
    ident = float((d == 0).mean())
    _report(family, case, identical=ident, worst_ulps=float(d.max()))
    assert d.max() <= 2, (case, int(d.max()))
    assert ident >= min_identical, (case, ident)
    return ident


def check_rope(family, case, got_bits, want64, want_fp32_products):
    """bit-identical to the oracle with the kernel's fp32 products, and at least 99.9 % identical to exact products (the
    same thing with bf16 tables)"""
    assert np.array_equal(got_bits, to_bits(want_fp32_products)), (case, int(ulps(got_bits, to_bits(want_fp32_products)).max()))
    d = ulps(got_bits, to_bits(want64))
    ident = float((d == 0).mean())
    _report(family, case, identical=ident, worst_ulps=float(d.max()))
    assert ident >= 0.999, (case, ident)


def gemv_bound(want, mag, L):
    return 2.0 ** -8 * np.abs(want) + 2.0 * L * 2.0 ** -24 * mag


def check_gemv(family, case, got, want, mag, L):
    """got: float64 of the kernel's bf16 output"""
    bound = gemv_bound(want, mag, L)
    err = np.abs(got - want)
    ident = float((to_bits(got) == to_bits(dgo.bf16(want))).mean())
    with np.errstate(invalid="ignore", divide="ignore"):
        frac = float(np.nanmax(np.where(bound > 0, err / bound, np.where(err > 0, np.inf, 0.0))))
    _report(family, case, worst_of_bound=frac, identical=ident)
    assert np.isfinite(got).all(), case
    assert (err <= bound).all(), (case, frac)
    assert ident >= 0.99, (case, ident)


def rnd(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def normw(g, n):
    return (1.0 + 0.1 * torch.randn(n, generator=g, device="cuda")).to(torch.bfloat16)


def stream():
    return torch.cuda.current_stream().cuda_stream


def scattered_slots(rng, T, page, n_pages):
    """T distinct (page, offset) targets spread over n_pages pages, one of them at offset page - 1"""
    last = rng.integers(0, n_pages) * page + page - 1
    rest = rng.permutation(np.setdiff1d(np.arange(n_pages * page), [last]))[: T - 1]
    slots = rng.permutation(np.concatenate([[last], rest]))
    return (slots // page).astype(np.int32), (slots % page).astype(np.int32)


def rope_tables(kind, pos, rng):
    """cos / sin float32 [T, 64]: 'bf16' = DeepseekV3RotaryEmbedding's tables for a bf16 model (bf16 values), 'fp32' =
    the same tables unrounded, 'yarn' = random values of magnitude up to 1.4 (yarn's mscale multiplies the tables)"""
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3RotaryEmbedding
    if kind == "yarn":
        return (rng.uniform(-1.4, 1.4, (len(pos), 64)).astype(np.float32), rng.uniform(-1.4, 1.4, (len(pos), 64)).astype(np.float32))
    dt = torch.bfloat16 if kind == "bf16" else torch.float32
    cos, sin = DeepseekV3RotaryEmbedding(64)(torch.zeros(1, dtype=dt), torch.as_tensor(pos, dtype=torch.int64)[None])
    return cos[0].float().numpy(), sin[0].float().numpy()


# ------------------------------------------------------------------------------------------------ oracle pins (CPU)
def test_bf16_rounding_of_the_oracle_matches_torch():
    """on float32 values (torch rounds from float32) including ties, bf16 subnormals and overflow"""
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(100000) * 10.0 ** rng.integers(-30, 30, 100000),
                        [0.0, -0.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8), 2.0 ** -130, 3 * 2.0 ** -134, 3.0e38, -3.4e38]])
    x = x.astype(np.float32)
    want = torch.from_numpy(x).to(torch.bfloat16).float().numpy()
    assert np.array_equal(dgo.bf16(x.astype(np.float64)), want.astype(np.float64))


def test_rope_oracle_is_apply_rotary_pos_emb_bit_for_bit():
    """bf16 tensors on the CPU, tables from DeepseekV3RotaryEmbedding (bf16) and random yarn-scaled bf16 tables"""
    from ktransformers_b200.models.modeling_deepseek_v3 import apply_rotary_pos_emb
    torch.manual_seed(1)
    rng = np.random.default_rng(1)
    T, H = 37, 16
    pos = np.concatenate([[0, 1, 63, 64, 4095, 163839], rng.integers(0, 163840, T - 6)])
    q = torch.randn(1, T, H, 64).to(torch.bfloat16)
    k = torch.randn(1, T, 1, 64).to(torch.bfloat16)
    for kind in ("bf16", "yarn"):
        cos, sin = rope_tables(kind, pos, rng)
        cb, sb = torch.from_numpy(cos).to(torch.bfloat16)[None], torch.from_numpy(sin).to(torch.bfloat16)[None]
        qw, kw = apply_rotary_pos_emb(q, k, cb, sb, unsqueeze_dim=2)
        c64, s64 = cb[0].double().numpy(), sb[0].double().numpy()
        assert np.array_equal(to_bits(dgo.rope(q[0].double().numpy(), c64[:, None], s64[:, None])), dev_bits(qw[0]))
        assert np.array_equal(to_bits(dgo.rope(k[0, :, 0].double().numpy(), c64, s64)), dev_bits(kw[0, :, 0]))


@pytest.mark.parametrize("hidden", [512, 1536, 7168])
def test_add_rmsnorm_oracle_is_the_module_up_to_its_fp32_variance(hidden):
    """DeepseekV3RMSNorm(x + d) on CPU bf16 tensors: >= 99.9 % identical, every element within 2 ulps"""
    from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3RMSNorm
    torch.manual_seed(hidden)
    norm = DeepseekV3RMSNorm(hidden).to(torch.bfloat16)
    with torch.no_grad():
        norm.weight.copy_((1 + 0.1 * torch.randn(hidden)).to(torch.bfloat16))
    x, d = torch.randn(64, hidden).to(torch.bfloat16), torch.randn(64, hidden).to(torch.bfloat16)
    with torch.no_grad():
        want = norm(x + d)
    r, out = dgo.add_rmsnorm(x.double().numpy(), d.double().numpy(), norm.weight.detach().double().numpy(), 1e-6)
    assert np.array_equal(to_bits(r), dev_bits(x + d))
    dist = ulps(to_bits(out), dev_bits(want))
    assert dist.max() <= 2 and (dist == 0).mean() >= 0.999, (int(dist.max()), float((dist == 0).mean()))


def test_absorb_oracles_are_einsums():
    rng = np.random.default_rng(2)
    q, w = rng.standard_normal((3, 5, 7)), rng.standard_normal((5, 7, 16))
    want, mag = dgo.absorb_q(q, w)
    np.testing.assert_allclose(want, np.einsum("thd,hdc->thc", q, w), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(mag, np.einsum("thd,hdc->thc", np.abs(q), np.abs(w)), rtol=1e-12)
    lat, wv = rng.standard_normal((3, 5, 16)), rng.standard_normal((5, 9, 16))
    want, mag = dgo.absorb_o(lat, wv)
    np.testing.assert_allclose(want, np.einsum("thc,hvc->thv", lat, wv), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(mag, np.einsum("thc,hvc->thv", np.abs(lat), np.abs(wv)), rtol=1e-12)


# ------------------------------------------------------------------------------------------------ argument checks (CPU)
BASE = 1 << 24     # aligned stand-in pointers; n_tokens = 0, so nothing is ever dereferenced


def _refused(rc, lib, msg):
    assert rc == native.EINVAL, rc
    assert msg in lib.ktb200_last_error().decode(), lib.ktb200_last_error().decode()


def test_add_rmsnorm_refuses_bad_hidden_and_misalignment_before_any_work():
    lib = native.lib()
    p = [BASE, BASE + (1 << 20), BASE + (2 << 20), BASE + (3 << 20)]        # residual, delta, weight, out
    call = lambda r, d, w, o, hidden: lib.ktb200_add_rmsnorm(r, d, w, 1e-6, o, 0, hidden, None)
    assert call(*p, 7168) == native.OK and call(p[0], None, p[2], p[3], 8192) == native.OK
    for hidden in (7167, 8194, 16384, 0):
        _refused(call(*p, hidden), lib, f"hidden {hidden} must be even and <= 8192")
    for i, name in enumerate(("residual", "delta", "weight", "out")):
        for off in (1, 2):
            bad = list(p)
            bad[i] += off
            _refused(call(*bad, 7168), lib, f"add_rmsnorm: {name} must be 4-byte aligned")


def test_absorb_gemvs_refuse_bad_shapes_and_misalignment_before_any_work():
    lib = native.lib()
    q, w, out = BASE, BASE + (1 << 20), BASE + (2 << 20)
    absorb_q = lambda q, w, out, nope=128, c=512: lib.ktb200_mla_absorb_q(q, 192, 128 * 192, w, 128, nope, c, out, 0, None)
    absorb_o = lambda lat, w, out, c=512: lib.ktb200_mla_absorb_o(lat, w, 128, 128, c, out, 0, None)
    assert absorb_q(q + 2, w, out) == native.OK and absorb_q(q, w, out, nope=512) == native.OK   # q is read element-wise
    assert absorb_o(q, w, out + 2) == native.OK                                                  # out is written element-wise
    _refused(absorb_q(q, w, out, nope=513), lib, "qk_nope_head_dim 513 must be in 1..512")
    for c in (516, 4, 0):
        _refused(absorb_q(q, w, out, c=c), lib, f"mla_absorb_q: kv_lora_rank {c} must be a positive multiple of 8")
        _refused(absorb_o(q, w, out, c=c), lib, f"mla_absorb_o: kv_lora_rank {c} must be a positive multiple of 8")
    for off in (2, 8):
        _refused(absorb_q(q, w + off, out), lib, "mla_absorb_q: w_uk must be 16-byte aligned")
        _refused(absorb_o(q + off, w, out), lib, "mla_absorb_o: attn_latent must be 16-byte aligned")
        _refused(absorb_o(q, w + off, out), lib, "mla_absorb_o: w_uv must be 16-byte aligned")
    _refused(absorb_q(q, w, out + 2), lib, "mla_absorb_q: q_abs_out must be 4-byte aligned")


def test_kv_write_refuses_misalignment():
    lib = native.lib()
    p = [BASE, BASE + (1 << 20), BASE + (2 << 20)]       # kv_cache, ckv, k_pe
    call = lambda kv, ckv, kpe: lib.ktb200_mla_kv_write(kv, 64, ckv, kpe, BASE + (3 << 20), BASE + (4 << 20), 0, None)
    assert call(*p) == native.OK
    for i, name in enumerate(("kv_cache", "ckv", "k_pe")):
        for off in (2, 8):
            bad = list(p)
            bad[i] += off
            _refused(call(*bad), lib, f"mla_kv_write: {name} must be 16-byte aligned")


# ------------------------------------------------------------------------------------------------ add_rmsnorm (GPU)
def add_rmsnorm(res, delta, w, out, T, hidden, eps=EPS):
    native.check(native.lib().ktb200_add_rmsnorm(res.data_ptr(), delta.data_ptr() if delta is not None else None, w.data_ptr(), eps,
                                                 out.data_ptr(), T, hidden, stream()))


@gpu
@pytest.mark.parametrize("with_delta", [True, False])
@pytest.mark.parametrize("hidden", [512, 1536, 2048, 5120, 6146, 7168, 8192])
def test_add_rmsnorm_vs_oracle(hidden, with_delta):
    """1, 3, 130 and 4096 tokens; the residual is the bf16 add (untouched without a delta), the output within the norm
    bounds"""
    g = torch.Generator(device="cuda").manual_seed(hidden * 2 + with_delta)
    w = normw(g, hidden)
    for T in (1, 3, 130, 4096):
        x = rnd(g, T, hidden)
        d = rnd(g, T, hidden) if with_delta else None
        res, out = x.clone(), torch.full_like(x, float("nan"))
        add_rmsnorm(res, d, w, out, T, hidden)
        torch.cuda.synchronize()
        r, want = dgo.add_rmsnorm(f64(x), f64(d) if with_delta else None, f64(w), EPS)
        assert np.array_equal(dev_bits(res), to_bits(r))
        check_norm("add_rmsnorm", f"H={hidden} T={T} delta={with_delta}", dev_bits(out), want)


@gpu
@pytest.mark.parametrize("with_delta", [True, False])
def test_add_rmsnorm_rows_where_eps_and_range_matter(with_delta):
    """hidden 7168: an all-zero row gives exact zeros, a row of scale 1e-4 (mean square 1e-8, next to eps = 1e-6), a row
    of scale 2^40 (squares near 2^88) stays finite and within the bounds, an ordinary row"""
    H = 7168
    g = torch.Generator(device="cuda").manual_seed(71 + with_delta)
    w = normw(g, H)
    x = torch.stack([torch.zeros(H, device="cuda").to(torch.bfloat16), rnd(g, H, scale=1e-4), rnd(g, H, scale=2.0 ** 40), rnd(g, H)])
    d = None
    if with_delta:
        d = torch.stack([torch.zeros(H, device="cuda").to(torch.bfloat16), rnd(g, H, scale=1e-4), rnd(g, H, scale=2.0 ** 40), rnd(g, H)])
    res, out = x.clone(), torch.full_like(x, float("nan"))
    add_rmsnorm(res, d, w, out, 4, H)
    torch.cuda.synchronize()
    r, want = dgo.add_rmsnorm(f64(x), f64(d) if with_delta else None, f64(w), EPS)
    assert np.array_equal(dev_bits(res), to_bits(r))
    got = f64(out)
    assert (got[0] == 0).all()
    assert np.isfinite(got).all()
    for i, name in enumerate(("zero", "1e-4", "2^40", "unit")):
        check_norm("add_rmsnorm edge rows", f"{name} delta={with_delta}", dev_bits(out[i]), want[i])


# ------------------------------------------------------------------------------------------------ mla_prep (GPU)
def mla_prep(q, heads, nope, kva, kvn, cos, sin, cache, page, pidx, poff, q_pe_out, T):
    native.check(native.lib().ktb200_mla_prep(q.data_ptr(), heads, nope, kva.data_ptr(), kvn.data_ptr(), EPS, cos.data_ptr(), sin.data_ptr(),
                                              cache.data_ptr(), page, pidx.data_ptr(), poff.data_ptr(), q_pe_out.data_ptr(), T, stream()))


def check_cache(family, case, before, after, want_rows, want_rows32, page):
    """target rows: latent columns within the norm bounds, k_pe columns as RoPE; every other row unchanged bit for bit"""
    a, b = dev_bits(after).reshape(-1, 576), dev_bits(before).reshape(-1, 576)
    slots = np.array([p * page + o for p, o in want_rows])
    rows, rows32 = np.stack(list(want_rows.values())), np.stack(list(want_rows32.values()))
    keep = np.ones(len(a), bool)
    keep[slots] = False
    assert np.array_equal(a[keep], b[keep]), f"{case}: rows outside the targets changed"
    check_norm(family + " latent", case, a[slots, :512], rows[:, :512])
    check_rope(family + " k_pe", case, a[slots, 512:], rows[:, 512:], rows32[:, 512:])


@gpu
@pytest.mark.parametrize("page", [16, 64, 256])
@pytest.mark.parametrize("T", [1, 4, 130])
@pytest.mark.parametrize("heads", [16, 64, 128])
def test_mla_prep_vs_oracle(heads, T, page):
    """each token to a scattered (page, offset), one at offset page - 1, in a cache filled with random rows first; tables
    'bf16' (bit-identical RoPE), 'fp32' and 'yarn' (within 1 ulp); token 0 at position 0 returns the de-interleaved input"""
    rng = np.random.default_rng(heads * 1000 + T * 10 + page)
    g = torch.Generator(device="cuda").manual_seed(heads * 1000 + T * 10 + page)
    nope = 128
    n_pages = 2 * -(-T // page) + 3
    q, kva, kvn = rnd(g, T, heads, nope + 64), rnd(g, T, 576), normw(g, 512)
    pidx, poff = scattered_slots(rng, T, page, n_pages)
    pos = np.concatenate([[0], rng.integers(1, 163840, T - 1)])
    pidx_d, poff_d = torch.from_numpy(pidx).cuda(), torch.from_numpy(poff).cuda()
    for kind in ("bf16", "fp32", "yarn"):
        cos, sin = rope_tables(kind, pos, rng)
        cache = rnd(g, n_pages, page, 576)
        before = cache.clone()
        q_pe = torch.full((T, heads, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
        mla_prep(q, heads, nope, kva, kvn, torch.from_numpy(cos).cuda(), torch.from_numpy(sin).cuda(), cache, page, pidx_d, poff_d, q_pe, T)
        torch.cuda.synchronize()
        want_qpe, want_rows = dgo.mla_prep(f64(q), nope, f64(kva), f64(kvn), EPS, cos, sin, pidx, poff)
        want_qpe32, want_rows32 = dgo.mla_prep(f64(q), nope, f64(kva), f64(kvn), EPS, cos, sin, pidx, poff, fp32_products=True)
        if kind == "bf16":
            assert np.array_equal(want_qpe32, want_qpe)
        case = f"heads={heads} T={T} page={page} tables={kind}"
        check_rope("mla_prep q_pe", case, dev_bits(q_pe), want_qpe, want_qpe32)
        check_cache("mla_prep", case, before, cache, want_rows, want_rows32, page)
        if kind != "yarn":      # position 0: cos = 1, sin = 0
            assert np.array_equal(dev_bits(q_pe[0]), to_bits(dgo.deinterleave(f64(q[0, :, nope:]))))
            assert np.array_equal(dev_bits(cache[pidx[0], poff[0], 512:]), to_bits(dgo.deinterleave(f64(kva[0, 512:]))))


# ------------------------------------------------------------------------------------------------ absorb GEMVs (GPU)
def absorb_q(q, head_stride, tok_stride, w, heads, D, C_, out, T):
    native.check(native.lib().ktb200_mla_absorb_q(q.data_ptr(), head_stride, tok_stride, w.data_ptr(), heads, D, C_, out.data_ptr(), T, stream()))


def absorb_o(lat, w, heads, V, C_, out, T):
    native.check(native.lib().ktb200_mla_absorb_o(lat.data_ptr(), w.data_ptr(), heads, V, C_, out.data_ptr(), T, stream()))


# (heads, D, C, tokens, token-stride padding): the V3 / V2 decode and batch shapes, Kimi-K2, V2-Lite, partial 512-column
# slabs (520, 8), a d range that does not split into four equal quarters (126, 5: the last quarter of 5 is empty), D = 512
ABSORB_Q = [(128, 128, 512, 1, 0), (128, 128, 512, 130, 0), (64, 128, 512, 64, 0), (16, 128, 512, 2, 0), (16, 128, 512, 3, 40),
            (128, 126, 520, 2, 0), (1, 5, 8, 130, 0), (16, 512, 256, 64, 0), (1, 512, 520, 1, 0), (64, 5, 256, 2, 8),
            (16, 126, 8, 64, 0)]
# (heads, V, C, tokens): V = 100 and 1 leave warps of the last CTA without an output
ABSORB_O = [(128, 128, 512, 1), (128, 128, 512, 130), (64, 128, 512, 64), (16, 128, 512, 2), (1, 1, 8, 130), (16, 100, 520, 64),
            (128, 100, 256, 2), (64, 1, 520, 1), (1, 128, 512, 2)]


@gpu
@pytest.mark.parametrize("heads,D,C_,T,pad", ABSORB_Q)
def test_absorb_q_vs_oracle(heads, D, C_, T, pad):
    """q addressed as the q_b output: head stride D + 64, token stride heads (D + 64) (+ pad); the rope columns and the
    padding hold other data"""
    g = torch.Generator(device="cuda").manual_seed(heads * 7 + D * 3 + C_ + T + pad)
    hs, ts = D + 64, heads * (D + 64) + pad
    q = rnd(g, T, ts)
    w = rnd(g, heads, D, C_, scale=0.05)
    out = torch.full((T, heads, C_), float("nan"), dtype=torch.bfloat16, device="cuda")
    absorb_q(q, hs, ts, w, heads, D, C_, out, T)
    torch.cuda.synchronize()
    qn = f64(q)[:, : heads * hs].reshape(T, heads, hs)[..., :D]
    want, mag = dgo.absorb_q(qn, f64(w))
    check_gemv("absorb_q", f"heads={heads} D={D} C={C_} T={T} pad={pad}", f64(out), want, mag, D)


@gpu
@pytest.mark.parametrize("heads,V,C_,T", ABSORB_O)
def test_absorb_o_vs_oracle(heads, V, C_, T):
    g = torch.Generator(device="cuda").manual_seed(heads * 5 + V * 3 + C_ + T)
    lat = rnd(g, T, heads, C_)
    w = rnd(g, heads, V, C_, scale=0.05)
    out = torch.full((T, heads, V), float("nan"), dtype=torch.bfloat16, device="cuda")
    absorb_o(lat, w, heads, V, C_, out, T)
    torch.cuda.synchronize()
    want, mag = dgo.absorb_o(f64(lat), f64(w))
    check_gemv("absorb_o", f"heads={heads} V={V} C={C_} T={T}", f64(out), want, mag, C_)


@gpu
def test_absorb_gemvs_past_65535_tokens():
    """65537 tokens of one head: two launches (65535 + 2 tokens); tokens on both sides of the split against the oracle"""
    T, D, C_, V = 65537, 128, 512, 128
    g = torch.Generator(device="cuda").manual_seed(65537)
    q = rnd(g, T, D + 64)
    wk, wv = rnd(g, 1, D, C_, scale=0.05), rnd(g, 1, V, C_, scale=0.05)
    qa = torch.full((T, 1, C_), float("nan"), dtype=torch.bfloat16, device="cuda")
    absorb_q(q, D + 64, D + 64, wk, 1, D, C_, qa, T)
    o = torch.full((T, 1, V), float("nan"), dtype=torch.bfloat16, device="cuda")
    absorb_o(qa, wv, 1, V, C_, o, T)
    torch.cuda.synchronize()
    assert not torch.isnan(qa).any() and not torch.isnan(o).any()
    rng = np.random.default_rng(5)
    ts = torch.as_tensor(np.unique(np.concatenate([[0, 1, 65533, 65534, 65535, 65536], rng.integers(0, T, 10)])), device="cuda")
    want, mag = dgo.absorb_q(f64(q[ts])[:, None, :D], f64(wk))
    check_gemv("absorb_q", "T=65537 sampled", f64(qa[ts]), want, mag, D)
    want, mag = dgo.absorb_o(f64(qa[ts]), f64(wv))
    check_gemv("absorb_o", "T=65537 sampled", f64(o[ts]), want, mag, C_)


# ------------------------------------------------------------------------------------------------ kv write (GPU)
@gpu
@pytest.mark.parametrize("T", [1, 7, 64, 300])
@pytest.mark.parametrize("page", [16, 64, 256])
def test_kv_write_scattered_rows(page, T):
    rng = np.random.default_rng(page + T)
    g = torch.Generator(device="cuda").manual_seed(page + T)
    n_pages = 2 * -(-T // page) + 3
    cache = rnd(g, n_pages, page, 576)
    before = cache.clone()
    ckv, kpe = rnd(g, T, 512), rnd(g, T, 64)
    pidx, poff = scattered_slots(rng, T, page, n_pages)
    pidx_d, poff_d = torch.from_numpy(pidx).cuda(), torch.from_numpy(poff).cuda()
    native.check(native.lib().ktb200_mla_kv_write(cache.data_ptr(), page, ckv.data_ptr(), kpe.data_ptr(), pidx_d.data_ptr(), poff_d.data_ptr(),
                                                  T, stream()))
    torch.cuda.synchronize()
    a, b = dev_bits(cache).reshape(-1, 576), dev_bits(before).reshape(-1, 576)
    slots = pidx.astype(np.int64) * page + poff
    assert np.array_equal(a[slots], np.concatenate([dev_bits(ckv), dev_bits(kpe)], axis=1))
    keep = np.ones(len(a), bool)
    keep[slots] = False
    assert np.array_equal(a[keep], b[keep])


# ------------------------------------------------------------------------------------------------ the chain (GPU)
class _Block:
    """One DeepSeek-V3 attention sub-block as bench.py's full_decode_leg runs it: hidden 7168, 128 heads, q_lora 1536,
    kv_lora 512, pages of 64; Q4_K ktb200_linear projections from synth_blocks, random bf16 W_UK / W_UV.  `stacked`:
    q_a and kv_a as one projection into [1][1536 + 576] (bench.py's qkva view, valid at one token)."""
    H, NH, QL, KVL, ROPE, NOPE, VD, PAGE, WIDTH = 7168, 128, 1536, 512, 64, 128, 128, 64, 2
    SCALE = (128 + 64) ** -0.5

    def __init__(self, B, stacked, seed):
        from ktransformers_b200.util.synth import synth_blocks
        from oracle.bindings import BF16, Q4_K
        self.lib, self.B, self.stacked = native.lib(), B, stacked
        H, NH, QL, KVL, ROPE, NOPE, VD = self.H, self.NH, self.QL, self.KVL, self.ROPE, self.NOPE, self.VD
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.keep = []

        def linear(inf, outf, s):
            w = synth_blocks(Q4_K, outf * inf, "cuda", s)
            h = C.c_void_p()
            native.check(self.lib.ktb200_linear_create(inf, outf, w.data_ptr(), Q4_K, BF16, 8, torch.cuda.current_device(), C.byref(h)))
            native.check(self.lib.ktb200_linear_load_weights(h, stream()))
            self.keep.append((h, w))
            return h
        if stacked:
            self.qkv_a = linear(H, QL + KVL + ROPE, seed + 1)
        else:
            self.q_a, self.kv_a = linear(H, QL, seed + 1), linear(H, KVL + ROPE, seed + 2)
        self.q_b, self.o = linear(QL, NH * (NOPE + ROPE), seed + 3), linear(NH * VD, H, seed + 4)
        self.w_uk, self.w_uv = rnd(g, NH, NOPE, KVL, scale=0.05), rnd(g, NH, VD, KVL, scale=0.05)
        self.ln_in, self.ln_qa, self.ln_kv, self.ln_post = normw(g, H), normw(g, QL), normw(g, KVL), normw(g, H)
        rng = np.random.default_rng(seed)
        self.n_pages = self.WIDTH * B + 3
        self.ptab_h = rng.permutation(self.n_pages)[: self.WIDTH * B].reshape(B, self.WIDTH).astype(np.int32)
        self.cache0 = rnd(g, self.n_pages, self.PAGE, KVL + ROPE)   # every position below 60 (and the rest) pre-filled
        z = lambda *s: torch.zeros(*s, dtype=torch.bfloat16, device="cuda")
        self.x, self.delta, self.hbuf = z(B, H), z(B, H), z(B, H)
        if stacked:
            self.qkva = z(B, QL + KVL + ROPE)
            self.qa, self.kva = self.qkva[:, :QL], self.qkva[:, QL:]
        else:
            self.qa, self.kva = z(B, QL), z(B, KVL + ROPE)
        self.qan, self.q = z(B, QL), z(B, NH * (NOPE + ROPE))
        self.q_pe, self.q_abs, self.lat = z(B, NH, ROPE), z(B, NH, KVL), z(B, NH, KVL)
        self.o_in, self.attn_out = z(B, NH, VD), z(B, H)
        self.lse = torch.zeros(B, NH, device="cuda")
        self.cache = self.cache0.clone()
        self.cos, self.sin = torch.zeros(B, ROPE, device="cuda"), torch.zeros(B, ROPE, device="cuda")
        self.pidx, self.poff = torch.zeros(B, dtype=torch.int32, device="cuda"), torch.zeros(B, dtype=torch.int32, device="cuda")
        self.klen = torch.zeros(B, dtype=torch.int32, device="cuda")
        self.ptab = torch.from_numpy(self.ptab_h).cuda()
        wsb = self.lib.ktb200_mla_workspace_bytes(B, NH, 0)
        self.ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
        # the synthetic Q4_K projections give outputs of rms ~1e5 on unit inputs, so every softmax would be one-hot (LSE
        # ~3e5, where one fp32 ulp is 0.03): scale the input and q_a norm weights so that kv_a and q_b give unit rms, as
        # in a trained model
        lin = lambda h, src, dst: native.check(self.lib.ktb200_linear_forward(h, B, src.data_ptr(), dst.data_ptr(), None, None, stream()))
        rms = lambda t: float(t.float().pow(2).mean().sqrt())
        self.hbuf.copy_(rnd(g, B, H))
        if stacked:
            lin(self.qkv_a, self.hbuf, self.qkva)
        else:
            lin(self.kv_a, self.hbuf, self.kva)
        self.qan.copy_(rnd(g, B, QL))
        lin(self.q_b, self.qan, self.q)
        torch.cuda.synchronize()
        self.ln_in = (self.ln_in.float() / rms(self.kva)).to(torch.bfloat16)
        self.ln_qa = (self.ln_qa.float() / rms(self.q)).to(torch.bfloat16)
        self.mla = native.MlaParams(B, NH, self.PAGE, self.WIDTH, 0, float(self.SCALE), self.q_abs.data_ptr(), self.q_pe.data_ptr(),
                                    self.cache.data_ptr(), self.ptab.data_ptr(), self.klen.data_ptr(), self.lat.data_ptr(),
                                    self.lse.data_ptr(), self.ws.data_ptr(), wsb, self.n_pages * self.PAGE)
        # per step: residual and delta inputs, RoPE tables (fp32, computed as bench.py does), targets and lengths
        inv = 1.0 / (10000.0 ** (np.arange(0, ROPE, 2) / ROPE))
        self.steps = []
        for s, p in enumerate(range(60, 68)):
            ang = np.concatenate([inv * p, inv * p]).astype(np.float32)
            tab = lambda f: torch.from_numpy(np.tile(f(ang), (B, 1)).astype(np.float32)).cuda()
            self.steps.append(dict(pos=p, x=rnd(g, B, H), delta=rnd(g, B, H), cos=tab(np.cos), sin=tab(np.sin),
                                   pidx=torch.from_numpy(self.ptab_h[:, p // self.PAGE].copy()).cuda(),
                                   poff=torch.full((B,), p % self.PAGE, dtype=torch.int32, device="cuda"),
                                   klen=torch.full((B,), p + 1, dtype=torch.int32, device="cuda")))

    def close(self):
        for h, _ in self.keep:
            self.lib.ktb200_linear_destroy(h)

    def reset(self):
        self.cache.copy_(self.cache0)
        for t in (self.x, self.delta, self.hbuf, self.qa, self.kva, self.qan, self.q, self.q_pe, self.q_abs, self.lat, self.o_in, self.attn_out):
            t.zero_()
        self.lse.zero_()

    def load(self, s):
        """the step's inputs, by device copies on the current stream"""
        st = self.steps[s]
        for dst, k in ((self.x, "x"), (self.delta, "delta"), (self.cos, "cos"), (self.sin, "sin"), (self.pidx, "pidx"), (self.poff, "poff"),
                       (self.klen, "klen")):
            dst.copy_(st[k])

    def calls(self):
        """full_decode_leg's sequence: (name, launch) pairs"""
        lib, B, S = self.lib, self.B, stream
        H, NH, QL, KVL, ROPE, NOPE, VD = self.H, self.NH, self.QL, self.KVL, self.ROPE, self.NOPE, self.VD
        lin = lambda h, src, dst: native.check(lib.ktb200_linear_forward(h, B, src.data_ptr(), dst.data_ptr(), None, None, S()))

        def proj():
            if self.stacked:
                lin(self.qkv_a, self.hbuf, self.qkva)
            else:
                lin(self.q_a, self.hbuf, self.qa)
                lin(self.kv_a, self.hbuf, self.kva)
        return [
            ("norm", lambda: add_rmsnorm(self.x, self.delta, self.ln_in, self.hbuf, B, H)),
            ("q_a / kv_a", proj),
            ("q_a norm", lambda: add_rmsnorm(self.qa, None, self.ln_qa, self.qan, B, QL)),
            ("q_b", lambda: lin(self.q_b, self.qan, self.q)),
            ("mla_prep", lambda: mla_prep(self.q, NH, NOPE, self.kva, self.ln_kv, self.cos, self.sin, self.cache, self.PAGE, self.pidx,
                                          self.poff, self.q_pe, B)),
            ("absorb_q", lambda: absorb_q(self.q, NOPE + ROPE, NH * (NOPE + ROPE), self.w_uk, NH, NOPE, KVL, self.q_abs, B)),
            ("mla_decode", lambda: native.check(lib.ktb200_mla_decode(C.byref(self.mla), S()))),
            ("absorb_o", lambda: absorb_o(self.lat, self.w_uv, NH, VD, KVL, self.o_in, B)),
            ("o_proj", lambda: lin(self.o, self.o_in.view(B, NH * VD), self.attn_out)),
            ("post norm", lambda: add_rmsnorm(self.x, self.attn_out, self.ln_post, self.hbuf, B, H)),
        ]

    def state(self):
        return [t.clone() for t in (self.x, self.hbuf, self.q_pe, self.q_abs, self.lat, self.o_in, self.attn_out, self.cache, self.lse)]

    def snap(self):
        return {k: t.clone() for k, t in dict(x=self.x, delta=self.delta, hbuf=self.hbuf, qa=self.qa, kva=self.kva, qan=self.qan, q=self.q, q_pe=self.q_pe,
                                               q_abs=self.q_abs, lat=self.lat, lse=self.lse, o_in=self.o_in, attn_out=self.attn_out,
                                               cache=self.cache).items()}

    def run(self, mode):
        """8 decode steps at positions 60..67 from the initial state -> (per-step end states, per-step snapshots after every
        call for mode 'sync')"""
        self.reset()
        torch.cuda.synchronize()
        calls = self.calls()
        graph = None
        if mode == "graph":
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _, f in calls:
                    f()
            torch.cuda.synchronize()
            self.reset()
        ends, snaps = [], []
        for s in range(len(self.steps)):
            torch.cuda.synchronize()
            per = {} if mode == "sync" else None
            self.load(s)
            if mode == "sync":
                torch.cuda.synchronize()
                per["in"] = self.snap()
            if mode == "graph":
                graph.replay()
            else:
                for name, f in calls:
                    f()
                    if mode == "sync":
                        torch.cuda.synchronize()
                        per[name] = self.snap()
            torch.cuda.synchronize()
            ends.append(self.state())
            snaps.append(per)
        return ends, snaps


def _check_chain_step(blk, s, per):
    """each glue kernel of step s against the oracle on the inputs it received; mla_decode against oracle/mla_oracle"""
    from test_mla_lengths import boundary_rows, check_decode
    B, NH, NOPE = blk.B, blk.NH, blk.NOPE
    st, case = blk.steps[s], f"B={blk.B} stacked={blk.stacked} pos={blk.steps[s]['pos']}"
    inp = per["in"]
    # input norm: residual += delta, then the norm
    r, want = dgo.add_rmsnorm(f64(inp["x"]), f64(inp["delta"]), f64(blk.ln_in), EPS)
    assert np.array_equal(dev_bits(per["norm"]["x"]), to_bits(r))
    check_norm("chain norm", case, dev_bits(per["norm"]["hbuf"]), want)
    # q_a norm: no delta, the projection output untouched
    pr = per["q_a / kv_a"]
    _, want = dgo.add_rmsnorm(f64(pr["qa"]), None, f64(blk.ln_qa), EPS)
    assert torch.equal(per["q_a norm"]["qa"].view(torch.int16), pr["qa"].view(torch.int16))
    check_norm("chain q_a norm", case, dev_bits(per["q_a norm"]["qan"]), want)
    # mla_prep on the q_b output and kv_a
    q = f64(per["q_b"]["q"]).reshape(B, NH, NOPE + 64)
    pidx, poff = st["pidx"].cpu().numpy(), st["poff"].cpu().numpy()
    args = (q, NOPE, f64(pr["kva"]), f64(blk.ln_kv), EPS, st["cos"].cpu().numpy(), st["sin"].cpu().numpy(), pidx, poff)
    (want_qpe, want_rows), (want_qpe32, want_rows32) = dgo.mla_prep(*args), dgo.mla_prep(*args, fp32_products=True)
    prep = per["mla_prep"]
    check_rope("chain q_pe", case, dev_bits(prep["q_pe"]), want_qpe, want_qpe32)
    check_cache("chain mla_prep", case, per["q_b"]["cache"], prep["cache"], want_rows, want_rows32, blk.PAGE)
    # absorb_q on the q_b output
    want, mag = dgo.absorb_q(q[..., :NOPE], f64(blk.w_uk))
    check_gemv("chain absorb_q", case, f64(per["absorb_q"]["q_abs"]), want, mag, NOPE)
    # mla_decode on sampled heads
    dec = per["mla_decode"]
    rng = np.random.default_rng(s)
    heads = boundary_rows(NH, rng, extra=2)
    q_abs, q_pe = f64(dec["q_abs"]).astype(np.float32), f64(dec["q_pe"]).astype(np.float32)
    kv = dec["cache"].float().cpu().numpy()
    kl = st["klen"].cpu().numpy()
    want_o, want_lse = mla_oracle.mla_decode(q_abs[:, heads], q_pe[:, heads], kv, blk.ptab_h, kl, blk.SCALE, p_bf16=True)
    exact, _ = mla_oracle.mla_decode(q_abs[:, heads], q_pe[:, heads], kv, blk.ptab_h, kl, blk.SCALE, p_bf16=False)
    check_decode("chain mla_decode", case, f64(dec["lat"])[:, heads], dec["lse"].cpu().numpy()[:, heads], want_o, want_lse, exact)
    # absorb_o on the latents
    want, mag = dgo.absorb_o(f64(per["absorb_o"]["lat"]), f64(blk.w_uv))
    check_gemv("chain absorb_o", case, f64(per["absorb_o"]["o_in"]), want, mag, blk.KVL)
    # post norm: residual += attn_out, then the norm
    r, want = dgo.add_rmsnorm(f64(per["o_proj"]["x"]), f64(per["o_proj"]["attn_out"]), f64(blk.ln_post), EPS)
    assert np.array_equal(dev_bits(per["post norm"]["x"]), to_bits(r))
    check_norm("chain post norm", case, dev_bits(per["post norm"]["hbuf"]), want)


@gpu
@pytest.mark.parametrize("B,stacked", [(1, True), (4, False)])
def test_decode_chain_as_bench_runs_it(B, stacked):
    """norm -> q_a / kv_a -> q_a norm -> q_b -> mla_prep -> absorb_q -> mla_decode -> absorb_o -> o_proj -> post norm, all
    programmatic dependent launches, at positions 60..67 (a new page at 64) after 60 cached positions: synchronised after
    every call, back to back on one stream, and one CUDA graph replayed per step give the same bits after every step;
    every kernel of the synchronised run matches its oracle on the inputs it received.  Measured on an H100: the norms,
    q_pe and the cache rows bit-identical to the oracle, absorb_q / _o at most 0.98 / 0.91 of their bound (at least
    99.98 % identical), mla_decode at most 0.58 of test_mla_decode_vs_oracle's bounds."""
    blk = _Block(B, stacked, seed=600 + B)
    try:
        sync, snaps = blk.run("sync")
        back, _ = blk.run("stream")
        graph, _ = blk.run("graph")
    finally:
        blk.close()
    names = ("residual", "normed", "q_pe", "q_abs", "latents", "o_in", "attn_out", "cache", "lse")
    for s in range(len(sync)):
        for name, a, b, c in zip(names, sync[s], back[s], graph[s]):
            va, vb, vc = (t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int16) for t in (a, b, c))
            assert torch.equal(va, vb), f"step {s}: {name} differs between synchronised and back-to-back launches"
            assert torch.equal(va, vc), f"step {s}: {name} differs between synchronised launches and the graph replay"
    for s, per in enumerate(snaps):
        _check_chain_step(blk, s, per)
