"""The MoE router (`ktb200_moe_gate_forward`, csrc/gate.cu + gate.cuh) at prompt lengths, on every configuration
`gate_config_ok` accepts, against float64 logits and routing.

A prefill sends the whole prompt of every MoE layer through one router call (KMoEGateB200.forward), and every expert kernel
takes the router's ids and weights as given: a wrong routing decision shows nowhere downstream.  The kernel computes
  phase 1  logits[t][e].  Column split s of S (`gate_splits`) covers the float4 columns [n4*s/S, n4*(s+1)/S) of n4 = H/4.  Lane
           l of expert e's warp runs ONE fmaf chain over its float4 columns l, l+32, ...: 4 terms each, 4*ceil(nc4/32) in
           all.  The 32 lane sums go through the 5-step xor-butterfly `warp_sum`, the split's partial is stored, and the
           selector adds the S partials to 0 in split order.  Tokens go in tiles of 8 (gate_dot<1|2|4|8>).
  phase 2  at most 16 selector CTAs, token t on CTA t % nsel: sigmoid (__fdiv_rn(1, 1 + expf(-l))) or softmax; + bias
           (noaux_tc); group scores; top-k by iterative arg-max, ties to the lowest index; the weights are gathered, summed
           in pick order, normalised with __fdiv_rn and scaled.

(a) Logit bound.  Each product x_h * W_eh of the float32 inputs (BF16 / F16 widened exactly) goes through one chain of
    N = 4*ceil(nc4_max/32) fmaf roundings + 5 warp_sum additions + (S - 1) split additions (the first add to 0 is exact).
    A sum evaluated with N rounded operations is within gamma_N * sum|terms| of the exact sum (Higham, Accuracy and Stability
    of Numerical Algorithms, 2nd ed., section 3.1), so per element
        |logit - logit64| <= gamma_N * (|x| . |W|),   gamma_N = N u / (1 - N u),   u = 2^-24,
    with logit64 = x64 @ W64.T on the same (widened) inputs.  V3 on 132 SMs: S = 6, nc4_max = 299, N = 40 + 5 + 5 = 50,
    gamma = 3.0e-6.  One float4 of one split dropped or counted twice moves a logit by about 4/7168 = 5.6e-4 of |x|.|W|.
    S is restated here from the SM count (`gate_splits`); the capture test pins it through the scratch size.
(b) Selection.  oracle.gate_oracle.route_from_logits in float32 on the kernel's own logits, with the device's expf
    (torch.exp on the GPU calls the same libdevice expf as the kernel): ids equal IN ORDER on every token, no exclusion.
    Exact float32 ties are settled by the lowest index in both; the oracle reports them (`tie`), and the selection-rule test
    asserts that it saw them.  Weights: sigmoid applies the kernel's operations to the same float32 values except the sum of
    the picked weights (numpy adds 8 or more values pairwise, the kernel in pick order: <= 10 u relative on positive terms)
    and its division, so W_ULP_SIG = 16 ulps.  Softmax also sums exp over the experts in another order (kernel: depth
    3 + 5 + 3 = 11; numpy's pairwise blocks: <= 24) before every division, so W_ULP_SOFT = 64 ulps.
(c) Routing against float64.  The float64 route of the float64 logits.  Every logit lies within the bound of (a), so each
    expert's selection score lies in an interval (sigmoid [sig(l-d), sig(l+d)], softmax s * exp(+-2 d_max), plus 2^-21 of the
    score and 2^-23 of the biased score for the float32 rounding of expf, the divisions and the bias add; group scores in
    the sums / maxima of the interval ends).  A token is decided when every decision (the groups kept, the top-k boundary,
    each pair of consecutive picks) separates the intervals.  Decided tokens must give the float64 ids in order and weights
    within 2e-5 relative, and must be >= 99 % of every case.  The prompts are built from router rows plus noise (`prompt`), so
    that most tokens route decisively as they do in a trained model; the share depends only on seeded inputs.
"""
import copy
import ctypes as C
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from ktransformers_b200 import native
from oracle import gate_oracle
from oracle.bindings import BF16, F16, F32, Q6_K
import gpu_util as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

U = 2.0 ** -24
W_ULP_SIG, W_ULP_SOFT = 16, 64
W64_REL = 2e-5
HID = {"f32": F32, "bf16": BF16, "f16": F16}
SCORING, METHOD = ("sigmoid", "softmax"), ("noaux_tc", "greedy", "group_limited_greedy")

# name: (E, H, top_k, n_group, topk_group, scoring, topk_method, norm_topk_prob, routed_scaling_factor)
CONFIGS = {
    "v3": (256, 7168, 8, 8, 4, 0, 0, 1, 2.5),                 # DeepSeek-V3 / R1
    "kimi-k2": (384, 7168, 8, 1, 1, 0, 0, 1, 2.827),
    "v2": (160, 5120, 6, 8, 3, 1, 2, 0, 16.0),                # softmax, group_limited_greedy, no norm
    "v2-lite": (64, 2048, 6, 1, 1, 1, 1, 0, 1.0),             # softmax, greedy
    "e512": (512, 2048, 8, 1, 1, 0, 0, 1, 1.0),               # every thread of the selector owns 4 experts
    "e72-softmax-norm": (72, 1024, 6, 1, 1, 1, 1, 1, 1.0),    # E not a multiple of 32
    "top32-all-groups": (256, 4096, 32, 8, 8, 0, 0, 1, 1.0),  # top_k = 32, topk_group = n_group
    "ng32": (64, 1024, 8, 32, 8, 0, 0, 1, 2.5),               # 32 groups of 2 experts
    "s1": (256, 256, 8, 8, 4, 0, 0, 1, 2.5),                  # H/4 = 64: one column split
    "uneven": (128, 3076, 8, 4, 2, 0, 0, 1, 1.0),             # 769 float4 over 8 splits: ranges of 96 and 97
}

T_ALL = (1, 2, 3, 4, 5, 6, 7, 8, 9, 15, 16, 17, 63, 64, 65, 255, 1000, 1024)
CASES = [("v3", T, "f32") for T in T_ALL]
CASES += [(c, T, "f32") for c in CONFIGS if c != "v3" for T in (1, 2, 3, 7, 9, 17, 65)]
CASES += [(c, 255, h) for c in CONFIGS for h in ("bf16", "f16")]
CASES += [("v3", 2048, "bf16"), ("v3", 4097, "f32"), ("v3", 8192, "bf16"), ("kimi-k2", 8192, "f16"), ("v2", 4097, "bf16"),
          ("v2-lite", 8192, "f32"), ("e512", 2048, "f32"), ("top32-all-groups", 1000, "f32"), ("uneven", 2048, "f32")]


H100_SMS = 132   # H100 SXM


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def gate_splits(E, H, nsms):
    """csrc/gate.cuh gate_splits"""
    S = min(8, max(1, nsms * 12 // E))
    while S > 1 and H // 4 // S < 64:
        S -= 1
    return S


def gamma(E, H, nsms):
    S = gate_splits(E, H, nsms)
    nc4_max = -(-(H // 4) // S)
    N = 4 * -(-nc4_max // 32) + 5 + (S - 1)
    return N * U / (1 - N * U)


def kw(name):
    E, H, k, ng, tg, sc, me, norm, scale = CONFIGS[name]
    return dict(top_k=k, n_group=ng, topk_group=tg, scoring=SCORING[sc], topk_method=METHOD[me], norm_topk_prob=bool(norm),
                routed_scaling_factor=scale)


def router(name, rng, bias_scale=2.0):
    E, H = CONFIGS[name][:2]
    W = rng.standard_normal((E, H)).astype(np.float32)
    bias = (rng.standard_normal(E) * bias_scale).astype(np.float32) if CONFIGS[name][6] == 0 else None
    return W, bias


def prompt(rng, T, W, k, noise=0.1):
    """tokens that route decisively, as a trained router's do: each is a sum of k + 8 random router rows with logit
    contributions spread evenly over [0, 6], plus noise of std `noise` per logit"""
    E, H = W.shape
    m = min(E, k + 8)
    A = np.zeros((T, E), np.float32)
    rows = np.argsort(rng.random((T, E)), axis=1)[:, :m]
    np.put_along_axis(A, rows, (np.linspace(0, 6, m) + rng.uniform(-0.02, 0.02, (T, m))).astype(np.float32), axis=1)
    return (A @ W / H + rng.standard_normal((T, H)).astype(np.float32) * (noise / np.sqrt(H))).astype(np.float32)


def to_hidden(x32, hid):
    """(x in the hidden type on the device, its exact float32 widening on the device)"""
    xh = torch.from_numpy(np.ascontiguousarray(x32)).cuda().to(G.TORCH_HID[hid])
    return xh, xh.float()


class Router:
    def __init__(self, name, W, bias, hid):
        E, H, k, ng, tg, sc, me, norm, scale = CONFIGS[name]
        self.gate = G.Gate(W, bias, k, ng, tg, sc, me, norm, scale, hidden_type=hid)
        self.E, self.k = E, k

    def __call__(self, x, bsz=None, stream=None):
        T = x.shape[0]
        idx = torch.full((T, self.k), -7, dtype=torch.int64, device="cuda")
        w = torch.full((T, self.k), float("nan"), dtype=torch.float32, device="cuda")
        logits = torch.full((T, self.E), float("nan"), dtype=torch.float32, device="cuda")
        native.check(native.lib().ktb200_moe_gate_forward(C.byref(self.gate.cfg), T, x.data_ptr(), idx.data_ptr(), w.data_ptr(),
                                                          logits.data_ptr(), bsz, G.stream() if stream is None else stream))
        torch.cuda.synchronize()
        return idx, w, logits


def bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def device_exp(a):
    return torch.exp(torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()).cpu().numpy()


def logits64(xw, W):
    """(x64 @ W64.T, |x|64 @ |W|64.T) on the device, as numpy"""
    Wd = torch.from_numpy(W).cuda().double()
    x64 = xw.double()
    return (x64 @ Wd.T).cpu().numpy(), (x64.abs() @ Wd.abs().T).cpu().numpy()


def check_logits(name, logits, l64, absdot):
    """(a): every element within gamma_N |x|.|W|; returns the worst error as a fraction of |x|.|W|"""
    E, H = CONFIGS[name][:2]
    g = gamma(E, H, num_sms())
    err = np.abs(logits.astype(np.float64) - l64)
    bad = np.argwhere(err > g * absdot)
    assert bad.size == 0, f"{name}: {len(bad)} logits outside gamma_N |x|.|W| (gamma {g:.3g}), first (t, e) {bad[:4].tolist()}"
    return float((err / np.maximum(absdot, 1e-300)).max())


def ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.abs(a.astype(np.float64) - b.astype(np.float64)) / np.spacing(np.maximum(np.abs(a), np.abs(b)))


def check_selection(name, bias, logits, idx, w):
    """(b): the oracle on the kernel's logits, float32, device expf; every token; returns (worst weight ulps, tie mask)"""
    oidx, ow, _, tie = gate_oracle.route_from_logits(logits, bias, dtype=np.float32, exp=device_exp, **kw(name))
    bad = np.nonzero((oidx != idx).any(1))[0]
    assert bad.size == 0, f"{name}: ids differ from the oracle on the kernel's logits at tokens {bad[:8].tolist()}: " \
                          f"{idx[bad[0]].tolist()} vs {oidx[bad[0]].tolist()}"
    u = ulps(w, ow)
    lim = W_ULP_SIG if CONFIGS[name][5] == 0 else W_ULP_SOFT
    assert u.max() <= lim, f"{name}: weights {u.max():.0f} ulps from the oracle (bound {lim}) at token {np.argmax(u.max(1))}"
    return float(u.max()), tie


def decided(name, l64, bound, bias, idx64):
    """(c): tokens whose every decision is separated by more than the logit bound (and float32 rounding) can move it"""
    E, H, k, ng, tg, sc, me, norm, scale = CONFIGS[name]
    T = l64.shape[0]
    if sc == 0:
        sig = lambda z: 1.0 / (1.0 + np.exp(-z))
        s, lo, hi = sig(l64), sig(l64 - bound), sig(l64 + bound)
    else:
        z = np.exp(l64 - l64.max(-1, keepdims=True))
        s = z / z.sum(-1, keepdims=True)
        dm = bound.max(-1, keepdims=True)
        lo, hi = s * np.exp(-2 * dm), s * np.exp(2 * dm)
    b = bias[None, :].astype(np.float64) if (me == 0 and bias is not None) else 0.0
    r = 2.0 ** -21 * np.abs(s) + 2.0 ** -23 * np.abs(s + b)
    clo, chi = lo + b - r, hi + b + r
    ok = np.ones(T, bool)
    if ng > 1 and me != 1:
        gs = E // ng
        gsc = (lambda a: np.sort(a.reshape(T, ng, gs), -1)[..., -2:].sum(-1)) if me == 0 else (lambda a: a.reshape(T, ng, gs).max(-1))
        g, glo, ghi = gsc(s + b), gsc(clo), gsc(chi)
        glo, ghi = glo - 2.0 ** -23 * np.abs(glo), ghi + 2.0 ** -23 * np.abs(ghi)
        sel = np.zeros((T, ng), bool)
        np.put_along_axis(sel, np.argsort(-g, -1, kind="stable")[:, :tg], True, -1)
        if tg < ng:
            ok &= np.where(sel, glo, np.inf).min(-1) > np.where(sel, -np.inf, ghi).max(-1)
        keep = np.repeat(sel, gs, 1)
        fill = -np.inf if me == 0 else 0.0
        clo, chi = np.where(keep, clo, fill), np.where(keep, chi, fill)
    plo, phi = np.take_along_axis(clo, idx64, -1), np.take_along_axis(chi, idx64, -1)
    ok &= (plo[:, :-1] > phi[:, 1:]).all(-1)
    if k < E:
        rest = chi.copy()
        np.put_along_axis(rest, idx64, -np.inf, -1)
        ok &= plo[:, -1] > rest.max(-1)
    return ok


def check_float64(name, bias, l64, absdot, idx, w):
    """(c): returns the share of decided tokens"""
    E, H = CONFIGS[name][:2]
    idx64, w64, _, _ = gate_oracle.route_from_logits(l64, bias, dtype=np.float64, **kw(name))
    ok = decided(name, l64, gamma(E, H, num_sms()) * absdot, bias, idx64)
    assert ok.mean() >= 0.99, f"{name}: only {ok.mean():.4f} of {ok.size} tokens are decided in float64"
    bad = np.nonzero(ok & (idx != idx64).any(1))[0]
    assert bad.size == 0, f"{name}: decided tokens route differently from float64 at {bad[:8].tolist()}"
    rel = np.abs(w[ok] - w64[ok]) / np.maximum(np.abs(w64[ok]), 1e-30)
    assert rel.max(initial=0) <= W64_REL, f"{name}: weights {rel.max():.3g} from float64"
    return float(ok.mean())


# ------------------------------------------------------------------------------------------------ (a)-(c), (e), (f)
@pytest.mark.gpu
@pytest.mark.parametrize("name,T,hid", CASES, ids=[f"{c}-T{T}-{h}" for c, T, h in CASES])
def test_router_vs_float64(name, T, hid):
    """(a) logits against float64, (b) selection against the oracle on the kernel's logits, (c) routing against float64"""
    t0 = time.perf_counter()
    rng = np.random.default_rng([T, HID[hid], list(CONFIGS).index(name)])
    W, bias = router(name, rng)
    E, H, k = CONFIGS[name][:3]
    x32 = prompt(rng, T, W, k)
    xh, xw = to_hidden(x32, HID[hid])
    idx, w, logits = (t.cpu().numpy() for t in Router(name, W, bias, HID[hid])(xh))
    l64, absdot = logits64(xw, W)
    la = check_logits(name, logits, l64, absdot)
    wu, _ = check_selection(name, bias, logits, idx, w)
    share = check_float64(name, bias, l64, absdot, idx, w)
    print(f"{name} T={T} {hid}: S={gate_splits(E, H, num_sms())} logit err <= {la:.3g} |x|.|W|, weights {wu:.0f} ulps from the "
          f"oracle, {share:.4f} decided in float64, {time.perf_counter() - t0:.2f} s")


def test_cases_reach_every_kernel_path():
    """CPU: the parametrisation covers, on an H100, every gate_dot specialisation and tail tile, the selector counts below
    and at 16, scratch past its 1 MB floor, every gate_config_ok limit, and H / 4 not divisible by S"""
    Ts = {T for c, T, h in CASES}
    assert {1, 2, 3, 4}.issubset(Ts) and any(T % 8 in (5, 6, 7) and T > 8 for T in Ts) and any(T % 8 == 1 and T > 8 for T in Ts)
    assert {T for T in Ts if T < 16} and 16 in Ts and max(Ts) == 8192
    nsms = H100_SMS
    assert max(T * CONFIGS[c][0] * gate_splits(*CONFIGS[c][:2], nsms) * 4 for c, T, h in CASES) > 8 << 20
    assert gate_splits(*CONFIGS["s1"][:2], nsms) == 1
    E, H = CONFIGS["uneven"][:2]
    assert (H // 4) % gate_splits(E, H, nsms) != 0
    assert CONFIGS["e512"][0] == 512 and CONFIGS["e72-softmax-norm"][0] % 32 and CONFIGS["top32-all-groups"][2] == 32
    assert {h for c, T, h in CASES} == set(HID) and {c for c, T, h in CASES} == set(CONFIGS)


def test_route_from_logits_is_route_and_reports_ties():
    """CPU: route() is the logits followed by route_from_logits(); exact ties go to the lowest index and are reported
    (also where float32 rounding makes them: exp(-1e-45) == 1), distinct scores are not"""
    rng = np.random.default_rng(0)
    x, W, bias = rng.standard_normal((6, 64)), rng.standard_normal((32, 64)), rng.standard_normal(32)
    a = gate_oracle.route(x, W, bias, top_k=4, n_group=4, topk_group=2, routed_scaling_factor=2.5)
    b = gate_oracle.route_from_logits(a[3], bias, top_k=4, n_group=4, topk_group=2, routed_scaling_factor=2.5)
    for u, v in zip(a[:3], b[:3]):
        assert np.array_equal(u, v)
    logits = np.zeros((2, 8), np.float32)
    logits[1, 5] = np.nextafter(np.float32(0), np.float32(1))
    idx, w, _, tie = gate_oracle.route_from_logits(logits, None, top_k=3, scoring="softmax", topk_method="greedy",
                                                   norm_topk_prob=False)
    assert idx.tolist() == [[0, 1, 2], [0, 1, 2]] and tie.tolist() == [True, True]
    logits[1] = np.arange(8, dtype=np.float32)
    idx, _, _, tie = gate_oracle.route_from_logits(logits, None, top_k=3)
    assert idx[1].tolist() == [7, 6, 5] and not tie[1]


# ------------------------------------------------------------------------------------------------ (d) bit-exact invariants
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v3", "v2"])
def test_rows_independent_of_position_tile_offset_and_qlen(name):
    """a token's logits, ids and weights are the same bits at any position, one token later (another tile offset), alone,
    and inside an 8192-token call; two calls give the same bits"""
    rng = np.random.default_rng(7)
    W, bias = router(name, rng)
    k = CONFIGS[name][2]
    T = 4096
    x = torch.from_numpy(prompt(rng, 8192, W, k)).cuda()
    r = Router(name, W, bias, F32)
    base = r(x[:T].contiguous())
    again = r(x[:T].contiguous())
    shifted = r(torch.cat([x[T:T + 1], x[:T - 1]]).contiguous())
    whole = r(x)
    for a, b in zip(base, again):
        assert torch.equal(bits(a), bits(b)), "two calls differ"
    for a, b in zip(base, shifted):
        assert torch.equal(bits(a[:T - 1]), bits(b[1:])), "a token's row depends on its tile offset"
    for a, b in zip(base, whole):
        assert torch.equal(bits(a), bits(b[:T])), "a token's row depends on the call's length"
    for t in (0, 1, 7, 8, 13, 2047, 4095):
        one = r(x[t:t + 1].contiguous())
        for a, b in zip(base, one):
            assert torch.equal(bits(a[t:t + 1]), bits(b)), f"token {t} alone differs from token {t} of a {T}-token call"


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v3", "v2", "e72-softmax-norm"])
@pytest.mark.parametrize("hid", [BF16, F16])
def test_half_inputs_equal_f32_router_on_widened_values(name, hid):
    rng = np.random.default_rng(hid)
    W, bias = router(name, rng)
    xh, xw = to_hidden(prompt(rng, 2048, W, CONFIGS[name][2]), hid)
    a, b = Router(name, W, bias, hid)(xh), Router(name, W, bias, F32)(xw)
    for u, v in zip(a, b):
        assert torch.equal(bits(u), bits(v))


# ------------------------------------------------------------------------------------------------ (g) where the rules decide
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["v3", "kimi-k2", "v2", "v2-lite", "ng32"])
def test_selection_rules_on_ties_saturation_and_underflow(name):
    """a 1000-token prompt with all-zero tokens (exact ties: lowest index, weights exact), duplicated tokens (identical rows),
    tokens so large that sigmoid gives exactly 1.0f (only the bias, quantised to produce ties, and the index separate them),
    and tokens with one dominant logit (the other softmax scores underflow to 0.0, V2's mask value)"""
    E, H, k, ng, tg, sc, me, norm, scale = CONFIGS[name]
    rng = np.random.default_rng(11)
    W, _ = router(name, rng)
    bias = (np.round(rng.standard_normal(E) * 2) / 8).astype(np.float32) if me == 0 else None
    T = 1000
    x = prompt(rng, T, W, k)
    zero, dup, big, dom = [0, 9, 500, 999], [300, 777], list(range(100, 108)), list(range(200, 206))
    x[zero] = 0
    x[dup] = x[17]
    x[big] = x[big] * 1e4
    for j, t in enumerate(dom):
        x[t] = W[(37 * j) % E] * (120.0 / H)
    xd = torch.from_numpy(x).cuda()
    idx, w, logits = (t.cpu().numpy() for t in Router(name, W, bias, F32)(xd))
    l64, absdot = logits64(xd, W)
    check_logits(name, logits, l64, absdot)
    assert (logits[zero] == 0).all()
    _, tie = check_selection(name, bias, logits, idx, w)
    oidx, ow, _, _ = gate_oracle.route_from_logits(logits, bias, dtype=np.float32, exp=device_exp, **kw(name))
    assert np.array_equal(w[zero].view(np.int32), ow[zero].view(np.int32)), "all-zero tokens: weights not exact"
    for t in dup:
        assert np.array_equal(idx[t], idx[17]) and np.array_equal(w[t].view(np.int32), w[17].view(np.int32))
        assert np.array_equal(logits[t].view(np.int32), logits[17].view(np.int32))
    if sc == 0:
        scores = 1.0 / (1.0 + device_exp(-logits[big]))
        assert (scores == 1.0).sum() >= 8 * k, "the large tokens do not saturate sigmoid"
        assert tie[big].any() and tie[zero].any()
    else:
        e = device_exp(logits[dom] - logits[dom].max(-1, keepdims=True))
        assert ((e / e.sum(-1, keepdims=True)) == 0).sum(-1).min() >= E - 8, "the dominant tokens do not underflow the others"
        assert tie[dom].all() and tie[zero].all()
    print(f"{name}: {int(tie.sum())} tokens with exact float32 ties, all routed by the index rule")


@pytest.mark.gpu
def test_f16_inputs_near_the_largest_half():
    """F16 tokens with entries at +-65504 and +-60000 against float64 and the oracle, softmax and sigmoid"""
    for name in ("v2-lite", "v3"):
        E, H, k = CONFIGS[name][:3]
        rng = np.random.default_rng(5)
        W, bias = router(name, rng)
        T = 300
        x = prompt(rng, T, W, k)
        sel = rng.random((T, H)) < 0.02
        x[sel] = np.where(rng.random(sel.sum()) < 0.5, -1, 1) * np.where(rng.random(sel.sum()) < 0.5, 65504.0, 60000.0)
        xh, xw = to_hidden(x, F16)
        assert (xw.abs() == 65504).any()
        idx, w, logits = (t.cpu().numpy() for t in Router(name, W, bias, F16)(xh))
        l64, absdot = logits64(xw, W)
        check_logits(name, logits, l64, absdot)
        check_selection(name, bias, logits, idx, w)


# ------------------------------------------------------------------------------------------------ (h) device batch size
@pytest.mark.gpu
@pytest.mark.parametrize("name,hid", [("v3", F32), ("v2", BF16)])
def test_device_bsz_at_prompt_length(name, hid):
    """rows >= min(bsz, T) untouched, live rows the bits of the call without bsz, the ticket clean after each (the following
    ordinary call is exact).  A negative bsz has a test of its own, in a process of its own."""
    from test_batch_size_contract import contract_eager, contract_graph, gate_case
    E, H, k, ng, tg, sc, me, norm, scale = CONFIGS[name]
    T = 4096
    bs = (0, 1, 7, 8, 9, 16, 17, T - 1, T, T + 5, 0)
    contract_eager(gate_case(T, E, H, k, ng, tg, sc, me, norm, scale, hid), bs)
    contract_graph(gate_case(T, E, H, k, ng, tg, sc, me, norm, scale, hid), bs)


def _ticket():
    words = (C.c_uint * 2)()
    native.check(native.lib().ktb200_debug_gate_ticket(0, words))
    return list(words)


def _negative_bsz():
    """In a fresh process: bsz = -1 writes nothing and leaves the router's ticket at zero, eagerly and in a graph replay.  The
    ticket is read back after each such launch and BEFORE any further router launch: a ticket left set lets the next
    launches select before the partial sums exist, or wait for CTAs that never arrive, so nothing runs after one that is
    not clean and the ticket ends with the process.  Returns what went wrong, or None."""
    from test_batch_size_contract import gate_case
    torch.cuda.set_device(0)
    try:
        E, H, k, ng, tg, sc, me, norm, scale = CONFIGS["v3"]
        T = 4096
        case = gate_case(T, E, H, k, ng, tg, sc, me, norm, scale)
        outs = [t for t, _ in case.outs]
        init = case.initial()
        case.run(init, None)
        want = [t.clone() for t in outs]
        assert _ticket() == [0, 0], f"the ticket is {_ticket()} after an ordinary call"
        bsz = torch.full((1,), -1, dtype=torch.int32, device="cuda")

        def untouched(what):
            for t, v in zip(outs, init):
                assert torch.equal(t.view(torch.uint8), v.view(torch.uint8)), f"{what}: an output was written"
            words = _ticket()
            assert words == [0, 0], f"{what}: the ticket is left at {words}"

        def exact(what):
            for t, v in zip(outs, want):
                assert torch.equal(t.view(torch.uint8), v.view(torch.uint8)), f"{what}: differs from the first call"

        case.run(init, bsz.data_ptr())
        untouched("eager bsz = -1")
        case.run(init, None)
        exact("the ordinary call after bsz = -1")
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=torch.cuda.Stream()):
            case.call(bsz.data_ptr(), torch.cuda.current_stream().cuda_stream)
        for t, v in zip(outs, init):
            t.copy_(v)
        g.replay()
        torch.cuda.synchronize()
        untouched("graph replay with bsz = -1")
        bsz.fill_(T)
        g.replay()
        torch.cuda.synchronize()
        exact("graph replay with bsz = T after bsz = -1")
        del g
    except AssertionError as e:
        return str(e) or "assertion failed"
    return None


def _in_fresh_process(fn):
    code = (f"import sys; sys.path[:0] = sys.argv[1:]; import test_router_prompt as t; e = t.{fn}(); "
            "print(e or 'OK'); sys.exit(1 if e else 0)")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, ROOT, os.path.join(ROOT, "tests")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-2000:] + r.stderr[-2000:]


@pytest.mark.gpu
def test_negative_device_bsz_selects_nothing_and_leaves_the_ticket_clean():
    """a negative value in the device bsz tensor behaves as 0 (max(0, min(T, *bsz)))"""
    _in_fresh_process("_negative_bsz")


# ------------------------------------------------------------------------------------------------ (i) capture
def _refused(call, outs):
    """capture `call` on a side stream: it must raise KTB200_ESTATE before any device work; returns the message"""
    before = [t.clone() for t in outs]
    g = torch.cuda.CUDAGraph()
    try:
        with torch.cuda.graph(g, stream=torch.cuda.Stream()):
            call(torch.cuda.current_stream().cuda_stream)
    except native.KTB200Error as e:
        msg = str(e)
    else:
        raise AssertionError("the capture succeeded")
    torch.cuda.synchronize()
    for a, b in zip(outs, before):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "a refused capture wrote an output"
    return msg


def _replayed(call, outs, want):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=torch.cuda.Stream()):
        call(torch.cuda.current_stream().cuda_stream)
    for t in outs:
        t.view(torch.uint8).fill_(0xAB)
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(outs, want):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), "the replay differs from the eager call"
    del g


def _capture_rule():
    """In a fresh process (the router scratch is per process and device, and grows only).  Returns what went wrong, or None."""
    from test_batch_size_contract import block_case, gate_case
    torch.cuda.set_device(0)
    try:
        # 1. the MoE block at qlen 12 runs the separate launches: its router call is the first of the process (ticket + 1 MB)
        case = block_case(12, Q6_K, True)
        outs = [t for t, _ in case.outs]
        call = lambda s: case.call(None, s)
        msg = _refused(call, outs)
        assert "first call" in msg and "12 or more tokens" in msg and "device 0" in msg and "eager" in msg, msg
        call(G.stream())                                       # the stream is usable, and this is the warm-up
        torch.cuda.synchronize()
        want = [t.clone() for t in outs]
        _replayed(call, outs, want)
        # 2. the router alone: the scratch holds 1 MB = q_fit tokens of E * S partial sums; one more token must grow it
        E, H, k, ng, tg, sc, me, norm, scale = CONFIGS["v3"]
        per_token = E * gate_splits(E, H, num_sms()) * 4
        q_fit = (1 << 20) // per_token
        for q, grows in ((q_fit, False), (q_fit + 1, True)):
            gc = gate_case(q, E, H, k, ng, tg, sc, me, norm, scale)
            outs = [t for t, _ in gc.outs]
            call = lambda s: gc.call(None, s)
            if grows:
                msg = _refused(call, outs)
                assert f"{q} or more tokens" in msg and "n_experts 256" in msg and "device 0" in msg and "eager" in msg, msg
            call(G.stream())
            torch.cuda.synchronize()
            want = [t.clone() for t in outs]
            _replayed(call, outs, want)
    except AssertionError as e:
        return str(e) or "assertion failed"
    return None


@pytest.mark.gpu
def test_capture_that_would_grow_the_router_scratch_is_refused():
    """a capture that would allocate or grow the router scratch returns KTB200_ESTATE naming the warm-up and writes nothing;
    after one eager call at that size the same capture replays the eager bits — through ktb200_moe_gate_forward, and through
    ktb200_moe_block_forward at qlen 12 (the separate launches).  The 1 MB boundary sits where the restated gate_splits puts it."""
    _in_fresh_process("_capture_rule")


# ------------------------------------------------------------------------------------------------ (j) the operator
def _reference_gate(kind):
    if kind == "v3":
        from ktransformers_b200.models.modeling_deepseek_v3 import DeepseekV3Config, MoEGate
        return "v3", DeepseekV3Config(hidden_size=7168, n_routed_experts=256, num_experts_per_tok=8, n_group=8, topk_group=4), MoEGate
    from ktransformers_b200.models.modeling_deepseek import DeepseekV2Config, MoEGate
    if kind == "v2":
        return "v2", DeepseekV2Config(hidden_size=5120, n_routed_experts=160, num_experts_per_tok=6, n_group=8, topk_group=3,
                                      topk_method="group_limited_greedy", routed_scaling_factor=16.0), MoEGate
    return "v2-lite", DeepseekV2Config(), MoEGate


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["v3", "v2", "v2-lite"])
def test_operator_on_reference_modules(kind):
    """KMoEGateB200 over the reference MoEGate, a [2, 2100, H] BF16 prompt, with and without bsz_tensor, against
    module.double().forward(x.double()): ids as sets (the reference's topk is unsorted), weights by id, on (c)'s decided tokens"""
    from ktransformers_b200.operators.gate import KMoEGateB200
    name, cfg, MoEGate = _reference_gate(kind)
    E, H, k = CONFIGS[name][:3]
    assert (cfg.n_routed_experts, cfg.hidden_size, cfg.num_experts_per_tok) == (E, H, k)
    rng = np.random.default_rng(3)
    W, bias = router(name, rng)
    op = KMoEGateB200("blk.3.ffn_gate_inp", None, cfg, MoEGate(cfg))
    op.load(w={"weight": torch.from_numpy(W), **({"e_score_correction_bias": torch.from_numpy(bias)} if bias is not None else {})},
            device="cuda")
    x = torch.from_numpy(prompt(rng, 4200, W, k)).cuda().to(torch.bfloat16).view(2, 2100, H)
    idx, wt = op(x)
    live = 3001
    idx_b, wt_b = op.forward(x, bsz_tensor=torch.tensor([live], dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    assert torch.equal(idx_b[:live], idx[:live]) and torch.equal(wt_b[:live].view(torch.int32), wt[:live].view(torch.int32))
    ref = copy.deepcopy(op.orig_module).double()
    with torch.no_grad():
        ridx, rw = ref(x.double())
    idx, wt, ridx, rw = idx.cpu().numpy(), wt.cpu().numpy(), ridx.cpu().numpy(), rw.double().cpu().numpy()
    l64, absdot = logits64(x.reshape(-1, H).float(), W)
    idx64 = gate_oracle.route_from_logits(l64, bias, dtype=np.float64, **kw(name))[0]
    ok = decided(name, l64, gamma(E, H, num_sms()) * absdot, bias, idx64)
    assert ok.mean() >= 0.99, ok.mean()
    o = np.nonzero(ok)[0]
    assert np.array_equal(np.sort(idx[o], 1), np.sort(ridx[o], 1)), "ids differ from the reference module"
    mine = np.take_along_axis(wt[o], np.argsort(idx[o], 1), 1)
    theirs = np.take_along_axis(rw[o], np.argsort(ridx[o], 1), 1)
    assert (np.abs(mine - theirs) <= W64_REL * np.abs(theirs)).all(), np.abs(mine - theirs).max()
