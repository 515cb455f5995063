"""The device batch-size contract of every compute entry point (include/ktb200.h): with a device `bsz` the effective batch
is min(qlen, *bsz), read on the device, so one captured CUDA graph serves a variable batch.

For every call and live count b:
  * rows >= min(b, qlen) of every output keep what the caller put there, bit for bit (a NaN with a payload, -7 for ids,
    or the previous values where the call accumulates);
  * rows < b equal, bit for bit, the same call without `bsz` on the same inputs (which the parity tests hold to the
    oracle); the FP8 linear with three or more K splits adds its partials with fp32 atomics and is held to the
    tolerance of its oracle test instead;
  * the padded input rows hold what serving padding can hold (NaN / Inf activations, ids 1 << 40 and -3, NaN weights)
    and the live rows do not see them;
  * the call without `bsz` that follows a short batch is still exact: workspaces, tickets and readiness words clean up
    after themselves.
The same holds for one captured graph replayed while the value in the bsz tensor changes between replays."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from ktransformers_b200 import native
from ktransformers_b200.util.synth import synth_blocks
from oracle.bindings import BF16, F32, Q4_K, Q5_K, Q6_K, bf16_to_f32, f32_to_bf16_bits
import gpu_util as G

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

NAN32 = 0x7FC0DEAD   # NaNs with a payload: arithmetic on a NaN returns the canonical one, so any write shows in the bits
NAN16 = 0x7FDE
INTS = {1: torch.int8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def _ints(t):
    return t.view(INTS[t.element_size()])


def _synth(t, n, seed):
    return synth_blocks(t, n, device="cuda", seed=seed)


def _lib():
    return native.lib()


# ------------------------------------------------------------------------------------------------ the harness
class Case:
    """One entry point over caller-owned device buffers.
    ins  [(tensor, kind)]: token-major inputs, kind "x" (activations), "ids" (expert ids) or "w" (routing weights)
    outs [(tensor, kind)]: token-major outputs, kind "out" / "w" (NaN sentinel), "idx" (-7) or "prev" (accumulated into)
    call(bsz_ptr or None, stream) issues the call; fresh() writes new valid inputs into every row of `ins`;
    launches: the kernel count that proves the intended path ran (int, or a predicate)."""

    def __init__(self, qlen, call, ins, outs, fresh, launches, exact=True, after=None, keep=()):
        self.qlen, self.call, self.ins, self.outs, self.fresh = qlen, call, ins, outs, fresh
        self.launches, self.exact, self.after, self.keep = launches, exact, after, keep
        self.gen = torch.Generator().manual_seed(qlen)

    def initial(self):
        """the caller's output contents before each call: sentinels, or previous values where the call accumulates"""
        init = []
        for t, kind in self.outs:
            if kind == "prev":
                v = (torch.randn(t.shape, generator=self.gen) / 4).to(t.dtype).cuda()
            else:
                v = torch.empty_like(t)
                _ints(v).fill_(-7 if kind == "idx" else (NAN16 if t.element_size() == 2 else NAN32))
            init.append(v)
        return init

    def run(self, init, bsz_ptr, stream=None):
        for (t, _), v in zip(self.outs, init):
            t.copy_(v)
        n0 = native.launch_count()
        self.call(bsz_ptr, G.stream() if stream is None else stream)
        torch.cuda.synchronize()
        n = native.launch_count() - n0
        assert (self.launches(n) if callable(self.launches) else n == self.launches), f"{n} launches: not the intended path"


def _garbage(t, kind):
    """what padded rows of a serving batch can hold"""
    if t.shape[0] == 0:
        return
    if kind == "x":
        pat = torch.tensor([float("nan"), float("inf"), -float("inf"), 3.0e38], dtype=torch.float32)
        t.copy_(pat.repeat(t.numel() // 4 + 1)[: t.numel()].view(t.shape).to(t.dtype))
    elif kind == "ids":
        pat = torch.tensor([1 << 40, -3], dtype=torch.int64)
        t.copy_(pat.repeat(t.numel() // 2 + 1)[: t.numel()].view(t.shape))
    else:
        t.fill_(float("nan"))


def _close(a, b):
    """test_fp8_linear_vs_oracle's bound: bf16 within 1 ulp (+ 1e-3 of the largest value), > 97 % identical"""
    x, y = a.float(), b.float()
    ok = (x - y).abs() <= 2.0 ** -7 * torch.maximum(x.abs(), y.abs()) + 1e-3 * y.abs().max()
    return bool(ok.all()) and (x.numel() == 0 or float((_ints(a) == _ints(b)).float().mean()) > 0.97)


def _check_rows(case, init, base, live, what):
    for i, ((t, kind), v, r) in enumerate(zip(case.outs, init, base)):
        assert torch.equal(_ints(t[live:]), _ints(v[live:])), f"{what}: output {i} ({kind}) written at rows >= {live}"
        if live == 0:
            continue
        if case.exact or kind == "idx":
            bad = (_ints(t[:live]) != _ints(r[:live])).reshape(live, -1).any(1).nonzero().flatten().tolist()
            assert not bad, f"{what}: output {i} ({kind}) differs from the call without bsz at rows {bad[:8]}"
        else:
            assert _close(t[:live], r[:live]), f"{what}: output {i} ({kind}) outside the tolerance of the call without bsz"


def contract_eager(case, bs):
    """every b of `bs` eagerly, each followed by a call without bsz that must reproduce the first one exactly"""
    bsz = torch.zeros(1, dtype=torch.int32, device="cuda")
    init = case.initial()
    case.run(init, None)
    base = [t.clone() for t, _ in case.outs]
    clean = [t.clone() for t, _ in case.ins]
    for b in bs:
        live = max(0, min(b, case.qlen))
        for t, kind in case.ins:
            _garbage(t[live:], kind)
        bsz.fill_(b)
        case.run(init, bsz.data_ptr())
        _check_rows(case, init, base, live, f"bsz={b} of qlen={case.qlen}")
        for (t, _), c in zip(case.ins, clean):
            t.copy_(c)
        case.run(init, None)
        _check_rows(case, init, base, case.qlen, f"the call without bsz after bsz={b}")
    if case.after:
        case.after()


def contract_graph(case, bs):
    """ONE captured call, replayed with a new bsz value and new inputs each time; then an eager call"""
    bsz = torch.full((1,), case.qlen, dtype=torch.int32, device="cuda")
    init = case.initial()
    case.run(init, bsz.data_ptr())          # warm-up: grow-only scratch is allocated here, never during capture
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=torch.cuda.Stream()):
        case.call(bsz.data_ptr(), torch.cuda.current_stream().cuda_stream)
    for b in bs:
        live = max(0, min(b, case.qlen))
        case.fresh()
        init = case.initial()
        case.run(init, None)
        base = [t.clone() for t, _ in case.outs]
        clean = [t.clone() for t, _ in case.ins]
        for t, kind in case.ins:
            _garbage(t[live:], kind)
        for (t, _), v in zip(case.outs, init):
            t.copy_(v)
        bsz.fill_(b)
        g.replay()
        torch.cuda.synchronize()
        _check_rows(case, init, base, live, f"graph replay with bsz={b} of qlen={case.qlen}")
        for (t, _), c in zip(case.ins, clean):
            t.copy_(c)
    case.run(init, None)                     # same inputs as the last replay: the eager call after the replays is exact
    _check_rows(case, init, base, case.qlen, "the eager call after the replays")
    if case.after:
        case.after()
    del g


def _bs(qlen):
    """0 twice in a row, 1, an interior value, qlen, and qlen + 5 (clamped by the call)"""
    return (0, 0, 1) + tuple(dict.fromkeys(b for b in (qlen // 2, qlen, qlen + 5) if b > 1))


REPLAY_BS = (3, 1, 0, 8, 2)


# ------------------------------------------------------------------------------------------------ cases
def _tokens(case_gen, qlen, H, dtype):
    return (torch.randn((qlen, H), generator=case_gen) / 50).to(dtype).cuda()


def _routing(gen, qlen, E, k):
    ids = torch.argsort(torch.rand((qlen, E), generator=gen), dim=1)[:, :k].contiguous()
    if qlen > 2:
        ids[1, 0] = -1                       # an invalid id inside the live batch is skipped as well
    return ids.cuda(), torch.rand((qlen, k), generator=gen).cuda()


def moe_case(qlen, H, I, dt, hid=BF16, E=8, k=4, shared=None, launches=2, m=None, seed=0):
    """ktb200_moe_forward (shared=None) / ktb200_moe_forward_shared (shared = (gate/up type, down type) of the shared expert)"""
    lib = _lib()
    if m is None:
        m = G.Moe(E, k, H, I, _synth(Q4_K, E * I * H, seed + 1), _synth(Q4_K, E * I * H, seed + 2), _synth(dt, E * H * I, seed + 3),
                  Q4_K, Q4_K, dt, hid, max_tokens=max(qlen, 16))
    mlp = None
    if shared is not None:
        sgt, sdt = shared
        mlp = G.Mlp(H, I, _synth(sgt, I * H, seed + 4), _synth(sgt, I * H, seed + 5), _synth(sdt, H * I, seed + 6), sgt, sgt, sdt, hid)
    dtype = G.TORCH_HID[hid]
    x, ids, w = torch.empty((qlen, H), dtype=dtype, device="cuda"), torch.empty((qlen, k), dtype=torch.int64, device="cuda"), \
        torch.empty((qlen, k), dtype=torch.float32, device="cuda")
    out = torch.empty((qlen, H), dtype=dtype, device="cuda")

    def call(p, s):
        if mlp is None:
            native.check(lib.ktb200_moe_forward(m.h, qlen, k, ids.data_ptr(), w.data_ptr(), x.data_ptr(), out.data_ptr(), p, s))
        else:
            native.check(lib.ktb200_moe_forward_shared(m.h, mlp.h, qlen, k, ids.data_ptr(), w.data_ptr(), x.data_ptr(), out.data_ptr(), p, s))

    case = Case(qlen, call, [(x, "x"), (ids, "ids"), (w, "w")], [(out, "out")], None, launches, keep=(m, mlp))

    def fresh():
        x.copy_(_tokens(case.gen, qlen, H, dtype))
        i, ww = _routing(case.gen, qlen, E, k)
        ids.copy_(i); w.copy_(ww)
    case.fresh = fresh
    fresh()
    return case


def rawint4_case(qlen, H=512, I=256, E=8, k=4):
    """RAWINT4_G32 routed experts (rows_bulk_i4_kernel + reduce_bulk_kernel<BulkI4>)"""
    lib = _lib()
    gen = torch.Generator(device="cuda").manual_seed(5)
    blocks = []
    for rows, cols in ((I, H), (I, H), (H, I)):
        packed = torch.randint(0, 256, (E * rows * cols // 2,), dtype=torch.uint8, generator=gen, device="cuda").view(torch.int32)
        scale = ((torch.rand((E * rows, cols // 32), generator=gen, device="cuda") + 0.25) / cols ** 0.5).to(torch.bfloat16)
        out = torch.empty(E * rows * cols // 256 * 144, dtype=torch.uint8, device="cuda")
        native.check(lib.ktb200_rawint4_pack(packed.data_ptr(), scale.data_ptr(), E * rows, cols, out.data_ptr(), G.stream()))
        blocks.append(out)
    I4 = native.RAWINT4_G32
    m = G.Moe(E, k, H, I, *blocks, I4, I4, I4, BF16, max_tokens=max(qlen, 16))
    return moe_case(qlen, H, I, None, BF16, E, k, m=m)


def gate_case(qlen, E, H, k, ng, tg, scoring, method, norm, scale, hid=F32):
    lib = _lib()
    rng = np.random.default_rng(E + H)
    gate = G.Gate(rng.standard_normal((E, H)).astype(np.float32), rng.standard_normal(E).astype(np.float32) if method == 0 else None,
                  k, ng, tg, scoring, method, norm, scale, hidden_type=hid)
    dtype = G.TORCH_HID[hid]
    x = torch.empty((qlen, H), dtype=dtype, device="cuda")
    idx, w = torch.empty((qlen, k), dtype=torch.int64, device="cuda"), torch.empty((qlen, k), dtype=torch.float32, device="cuda")
    logits = torch.empty((qlen, E), dtype=torch.float32, device="cuda")

    def call(p, s):
        native.check(lib.ktb200_moe_gate_forward(C.byref(gate.cfg), qlen, x.data_ptr(), idx.data_ptr(), w.data_ptr(), logits.data_ptr(), p, s))

    case = Case(qlen, call, [(x, "x")], [(idx, "idx"), (w, "w"), (logits, "w")], None, 1, keep=(gate,))
    case.fresh = lambda: x.copy_(_tokens(case.gen, qlen, H, dtype) * 5)
    case.fresh()
    return case


def _sync_words_zero(m):
    lib = _lib()
    n = lib.ktb200_debug_block_sync_words(m.h, None, 0)
    assert n > 8
    buf = (C.c_uint * n)()
    assert lib.ktb200_debug_block_sync_words(m.h, buf, n) == n
    words = np.frombuffer(buf, dtype=np.uint32)
    assert words[4] == 0, "a readiness wait timed out"
    assert not words.any(), f"synchronisation words left non-zero at {np.nonzero(words)[0][:8].tolist()}"


def block_case(qlen, dt, shared, H=4096, I=512, Eg=16, k=4, ng=4, tg=2, seed=0):
    lib = _lib()
    m = G.Moe(Eg, k, H, I, _synth(Q4_K, Eg * I * H, seed + 1), _synth(Q4_K, Eg * I * H, seed + 2), _synth(dt, Eg * H * I, seed + 3),
              Q4_K, Q4_K, dt, BF16, max_tokens=16)
    mlp = G.Mlp(H, I, _synth(Q4_K, I * H, seed + 4), _synth(Q4_K, I * H, seed + 5), _synth(dt, H * I, seed + 6), Q4_K, Q4_K, dt, BF16) if shared else None
    rng = np.random.default_rng(H + I)
    gate = G.Gate(rng.standard_normal((Eg, H)).astype(np.float32), rng.standard_normal(Eg).astype(np.float32), k, ng, tg, hidden_type=BF16)
    x = torch.empty((qlen, H), dtype=torch.bfloat16, device="cuda")
    out = torch.empty((qlen, H), dtype=torch.bfloat16, device="cuda")
    idx, w = torch.empty((qlen, k), dtype=torch.int64, device="cuda"), torch.empty((qlen, k), dtype=torch.float32, device="cuda")

    def call(p, s):
        native.check(lib.ktb200_moe_block_forward(C.byref(gate.cfg), m.h, mlp.h if mlp is not None else None, qlen, x.data_ptr(), out.data_ptr(),
                                                  idx.data_ptr(), w.data_ptr(), p, s))

    single = qlen <= 8
    case = Case(qlen, call, [(x, "x")], [(out, "out"), (idx, "idx"), (w, "w")], None, 1 if single else (lambda n: n > 1),
                after=(lambda: _sync_words_zero(m)) if single else None, keep=(m, mlp, gate))
    case.fresh = lambda: x.copy_(_tokens(case.gen, qlen, H, torch.bfloat16) * 5)
    case.fresh()
    return case


def linear_case(qlen, t, in_f, out_f, bias, launches=1, hid=BF16):
    lib = _lib()
    wt = _synth(t, out_f * in_f, in_f + out_f)
    h = C.c_void_p()
    native.check(lib.ktb200_linear_create(in_f, out_f, wt.data_ptr(), t, hid, 64, torch.cuda.current_device(), C.byref(h)))
    native.check(lib.ktb200_linear_load_weights(h, G.stream()))
    dtype = G.TORCH_HID[hid]
    x, y = torch.empty((qlen, in_f), dtype=dtype, device="cuda"), torch.empty((qlen, out_f), dtype=dtype, device="cuda")
    b = torch.randn(out_f, device="cuda") if bias else None

    def call(p, s):
        native.check(lib.ktb200_linear_forward(h, qlen, x.data_ptr(), y.data_ptr(), b.data_ptr() if b is not None else None, p, s))

    class Handle:                               # destroys the handle with the case
        def __del__(self):
            lib.ktb200_linear_destroy(h)
    case = Case(qlen, call, [(x, "x")], [(y, "out")], None, launches, keep=(wt, b, Handle()))
    case.fresh = lambda: x.copy_(_tokens(case.gen, qlen, in_f, dtype) * 5)
    case.fresh()
    return case


def mlp_case(qlen, accumulate, H=512, I=256, hid=BF16):
    lib = _lib()
    mlp = G.Mlp(H, I, _synth(Q4_K, I * H, 41), _synth(Q4_K, I * H, 42), _synth(Q6_K, H * I, 43), Q4_K, Q4_K, Q6_K, hid)
    dtype = G.TORCH_HID[hid]
    x, y = torch.empty((qlen, H), dtype=dtype, device="cuda"), torch.empty((qlen, H), dtype=dtype, device="cuda")

    def call(p, s):
        native.check(lib.ktb200_mlp_forward(mlp.h, qlen, x.data_ptr(), y.data_ptr(), accumulate, p, s))

    case = Case(qlen, call, [(x, "x")], [(y, "prev" if accumulate else "out")], None, 2, keep=(mlp,))
    case.fresh = lambda: x.copy_(_tokens(case.gen, qlen, H, dtype) * 5)
    case.fresh()
    return case


def fp8_ksplit(K, N):
    """ktb200_fp8_linear_create's K-split rule"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    nkb, row_tiles = K // 128, (N + 127) // 128
    ks = min(max((4 * sms + row_tiles - 1) // row_tiles, (nkb + 7) // 8), nkb)
    kb = (nkb + ks - 1) // ks
    if kb < 4 and nkb >= 4:
        kb = 4
    return (nkb + kb - 1) // kb


def fp8_case(T, K, N):
    from oracle import fp8_oracle as F
    lib = _lib()
    rng = np.random.default_rng(T * 1000 + K + N)
    w_d = torch.from_numpy(F.to_e4m3_bytes((rng.standard_normal((N, K)) * 0.7).astype(np.float32))).cuda()
    ws_d = torch.from_numpy((rng.random(((N + 127) // 128, K // 128)) * 0.02 + 0.001).astype(np.float32)).cuda()
    h = C.c_void_p()
    native.check(lib.ktb200_fp8_linear_create(K, N, w_d.data_ptr(), ws_d.data_ptr(), BF16, 0, C.byref(h)))
    x, y = torch.empty((T, K), dtype=torch.bfloat16, device="cuda"), torch.empty((T, N), dtype=torch.bfloat16, device="cuda")

    def call(p, s):
        native.check(lib.ktb200_fp8_linear_forward(h, T, x.data_ptr(), y.data_ptr(), p, s))

    class Handle:
        def __del__(self):
            lib.ktb200_fp8_linear_destroy(h)
    chunks = (T + 15) // 16
    case = Case(T, call, [(x, "x")], [(y, "out")], None, sum(2 if min(16, T - c * 16) > 2 else 1 for c in range(chunks)),
                exact=fp8_ksplit(K, N) < 3, keep=(w_d, ws_d, Handle()))
    case.fresh = lambda: x.copy_(_tokens(case.gen, T, K, torch.bfloat16) * 5)
    case.fresh()
    return case


# every entry point and the path its shape picks (the grouped path has tests of its own below)
CASES = {
    # ktb200_moe_forward: register-staged per-pair kernels (gemv.cuh), bulk-copy kernels (gemv_bulk.cuh), RAWINT4 (rawint4.cuh)
    "moe-H512-register": lambda: moe_case(6, 512, 256, Q6_K),
    "moe-H4096-bulk": lambda: moe_case(6, 4096, 512, Q6_K),
    "moe-H4096-bulk-q4k-down-f32": lambda: moe_case(6, 4096, 512, Q4_K, hid=F32),
    "moe-rawint4": lambda: rawint4_case(8),
    # ktb200_moe_forward_shared: the shared expert as an extra slot of the two routed launches / as a separate MLP
    "shared-fused": lambda: moe_case(6, 4096, 512, Q6_K, shared=(Q4_K, Q6_K), launches=2),
    "shared-separate": lambda: moe_case(6, 1024, 512, Q6_K, shared=(Q5_K, Q4_K), launches=4),
    # ktb200_moe_gate_forward with logits: V3 sigmoid / noaux_tc, V2 softmax / group_limited_greedy
    "gate-sigmoid-noaux": lambda: gate_case(12, 64, 2048, 6, 8, 4, 0, 0, 1, 2.5),
    "gate-softmax-grouped": lambda: gate_case(12, 32, 1024, 6, 4, 2, 1, 2, 0, 16.0, hid=BF16),
    # ktb200_moe_block_forward: the single persistent launch (qlen <= 8) and the separate launches behind it (qlen 12)
    "block-q6k-shared-1": lambda: block_case(1, Q6_K, True),
    "block-q6k-shared-3": lambda: block_case(3, Q6_K, True),
    "block-q6k-shared-8": lambda: block_case(8, Q6_K, True),
    "block-q4k-noshared-3": lambda: block_case(3, Q4_K, False, I=2048),
    "block-q4k-noshared-8": lambda: block_case(8, Q4_K, False, I=2048),
    "block-q6k-shared-12-fallback": lambda: block_case(12, Q6_K, True),
    # ktb200_linear_forward: register-staged rows (Q6_K, Q5_K) and dense_q4k_kernel segments (dense_bulk.cuh), +- bias
    "linear-q6k": lambda: linear_case(6, Q6_K, 2048, 512, False),
    "linear-q5k-bias": lambda: linear_case(6, Q5_K, 1536, 512, True),
    "linear-q4k-7168x2112": lambda: linear_case(6, Q4_K, 7168, 2112, False),
    "linear-q4k-7168x2112-bias": lambda: linear_case(8, Q4_K, 7168, 2112, True),
    "linear-q4k-256x777-bias": lambda: linear_case(5, Q4_K, 256, 777, True),
    # prompt-sized batches: rows_bulk_q4k_kernel in token chunks of 8, rows_kernel (rows under 16 blocks), the Q5_K pipe kernel
    "linear-q4k-bulk-T40-bias": lambda: linear_case(40, Q4_K, 7168, 1536, True),
    "linear-q4k-rows-T20-bias": lambda: linear_case(20, Q4_K, 1536, 2048, True),
    "linear-q5k-pipe-T12-bias": lambda: linear_case(12, Q5_K, 7168, 1536, True),
    # ktb200_mlp_forward
    "mlp": lambda: mlp_case(6, 0),
    "mlp-accumulate": lambda: mlp_case(6, 1),
    # ktb200_fp8_linear_forward: in-kernel act quant (T <= 2), separate quant kernel, two 16-token chunks, K splits
    "fp8-T2-ksplit2": lambda: fp8_case(2, 1024, 256),
    "fp8-T7-ksplit2": lambda: fp8_case(7, 1024, 256),
    "fp8-T20-two-chunks": lambda: fp8_case(20, 512, 384),
    "fp8-T20-ksplit3": lambda: fp8_case(20, 1536, 256),
}


@pytest.mark.parametrize("name", list(CASES))
def test_bsz_contract_eager(name):
    case = CASES[name]()
    if name.startswith("fp8-T20"):
        bs = (0, 0, 1, 15, 16, 17, 18, 20, 25)    # inside the first chunk, at its edge, inside the second (t0 = 16)
    else:
        bs = _bs(case.qlen)
    contract_eager(case, bs)


@pytest.mark.parametrize("name", list(CASES))
def test_bsz_contract_graph_replay(name):
    """batches of more than 16 tokens also replay with a live count inside a later token chunk"""
    case = CASES[name]()
    contract_graph(case, REPLAY_BS + ((case.qlen // 2 + 1,) if case.qlen > 16 else ()) + (case.qlen,))


def test_fp8_case_shapes_pick_the_k_splits():
    assert fp8_ksplit(512, 384) == 1 and fp8_ksplit(1024, 256) == 2 and fp8_ksplit(1536, 256) >= 3


def test_gate_bsz_zero_then_normal_call_keeps_the_ticket_clean():
    """bsz = 0 launches select nothing: the last CTA must still reset the ticket, or the next call selects early"""
    case = gate_case(5, 64, 2048, 6, 8, 4, 0, 0, 1, 2.5)
    bsz = torch.zeros(1, dtype=torch.int32, device="cuda")
    init = case.initial()
    case.run(init, None)
    base = [t.clone() for t, _ in case.outs]
    for _ in range(3):
        case.run(init, bsz.data_ptr())
        _check_rows(case, init, base, 0, "bsz=0")
    bsz.fill_(5)
    case.run(init, bsz.data_ptr())
    _check_rows(case, init, base, 5, "bsz=5 after three bsz=0 calls")


# ------------------------------------------------------------------------------------------------ grouped (prefill) path
def _grouped_launches(qlen, chunk=1024, extra=0):
    return 10 * ((qlen + chunk - 1) // chunk) + extra


@pytest.mark.parametrize("dt", [Q6_K, Q4_K])
def test_bsz_contract_grouped_eager(dt):
    case = moe_case(100, 1024, 512, dt, launches=_grouped_launches(100))
    contract_eager(case, (0, 0, 1, 31, 32, 33, 60, 100, 105))


def test_bsz_contract_grouped_shared_mlp_accumulate():
    """grouped routed experts, then the shared expert as a separate MLP accumulating into the same rows"""
    case = moe_case(60, 1024, 512, Q6_K, shared=(Q4_K, Q6_K), launches=_grouped_launches(60, extra=2))
    contract_eager(case, _bs(60))


@pytest.mark.parametrize("dt", [Q6_K, Q4_K])
def test_bsz_contract_grouped_graph_replay(dt):
    """grouped scratch is grow-only and per device: warm up at the captured qlen, and nothing larger runs after the capture"""
    case = moe_case(100, 1024, 512, dt, launches=_grouped_launches(100))
    contract_graph(case, (60, 20, 0, 100))


@pytest.mark.parametrize("qlen", [1024 + 60, 1024 + 5])
@pytest.mark.parametrize("hid", [F32, BF16])
def test_grouped_second_chunk_vs_oracle(oracle, qlen, hid):
    """qlen just above one 1024-token chunk: a second chunk ending partway through a 32-token tile (60), and one of 5 tokens
    that still runs on the grouped kernels because the path is chosen by the total qlen; tolerances of
    test_moe_grouped_tensor_core_path_vs_oracle."""
    E, k, H, I = 8, 4, 1024, 512
    gate, up, down = _synth(Q4_K, E * I * H, 21), _synth(Q4_K, E * I * H, 22), _synth(Q6_K, E * H * I, 23)
    g_np, u_np, d_np = gate.cpu().numpy(), up.cpu().numpy(), down.cpu().numpy()
    m = G.Moe(E, k, H, I, gate, up, down, Q4_K, Q4_K, Q6_K, hid, max_tokens=qlen)
    rng = np.random.default_rng(qlen + hid)
    x = (rng.standard_normal((qlen, H)) / 100).astype(np.float32)
    ids = np.stack([rng.permutation(E)[:k] for _ in range(qlen)]).astype(np.int64)
    ids[1030:, 0] = 1                        # the second chunk crowds one expert
    w = rng.random((qlen, k)).astype(np.float32)
    xin = x if hid == F32 else f32_to_bf16_bits(x)
    n0 = native.launch_count()
    got = m.forward(ids, w, xin)
    assert native.launch_count() - n0 == 20, "two chunks of the grouped path"
    want = oracle.moe_forward(E, H, I, g_np, u_np, d_np, Q4_K, Q4_K, Q6_K, hid, ids, w, xin)
    for sl in (slice(None), slice(1024, None)):            # the whole batch, and the second chunk on its own
        if hid == F32:
            assert np.abs(got[sl] - want[sl]).max() < 1e-3 * np.abs(want[sl]).max()
        else:
            a, b = bf16_to_f32(got[sl]), bf16_to_f32(want[sl])
            assert (np.abs(a - b) <= 2.0 ** -7 * np.maximum(np.abs(a), np.abs(b)) + 1e-3 * np.abs(b).max()).all()
            assert (got[sl] == want[sl]).mean() > 0.97
    m.close()


def test_bsz_contract_grouped_across_the_chunk_edge():
    """qlen 1084 = a 1024-token chunk + 60: b = 1000 leaves the second chunk empty, 1024 ends exactly on the edge, 1030 ends
    inside the second chunk"""
    case = moe_case(1084, 1024, 512, Q6_K, launches=_grouped_launches(1084))
    contract_eager(case, (1000, 1024, 1030, 0, 1, 1084, 1089))


def _small_chunks():
    """KTB200_GROUPED_CHUNK=64 (read once per process): qlen 200 crosses four chunks; b inside and exactly on chunk edges,
    and the call without bsz against the oracle.  Returns what went wrong, or None."""
    from oracle.bindings import Oracle
    torch.cuda.set_device(0)
    E, k, H, I, qlen = 8, 4, 1024, 512, 200
    gate, up, down = _synth(Q4_K, E * I * H, 61), _synth(Q4_K, E * I * H, 62), _synth(Q6_K, E * H * I, 63)
    g_np, u_np, d_np = gate.cpu().numpy(), up.cpu().numpy(), down.cpu().numpy()
    m = G.Moe(E, k, H, I, gate, up, down, Q4_K, Q4_K, Q6_K, F32, max_tokens=qlen)
    case = moe_case(qlen, H, I, Q6_K, hid=F32, m=m, launches=_grouped_launches(qlen, chunk=64))
    try:
        contract_eager(case, (0, 1, 63, 64, 65, 100, 128, 150, 192, 193, 200, 205))
    except AssertionError as e:
        return str(e)
    ids, w, x = (t.cpu().numpy() for t in (case.ins[1][0], case.ins[2][0], case.ins[0][0]))
    got = m.forward(ids, w, x)
    want = Oracle().moe_forward(E, H, I, g_np, u_np, d_np, Q4_K, Q4_K, Q6_K, F32, ids, w, x)
    err = float(np.abs(got - want).max() / np.abs(want).max())
    return None if err < 1e-3 else f"64-token chunks vs the oracle: relative error {err}"


# the chunk size is read once per process: the small chunks run in their own interpreter
def test_bsz_contract_grouped_small_chunks():
    code = ("import sys; sys.path[:0] = sys.argv[1:]; import test_batch_size_contract as t; e = t._small_chunks(); "
            "print(e or 'OK'); sys.exit(1 if e else 0)")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, ROOT, os.path.join(ROOT, "tests")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT, env={**os.environ, "KTB200_GROUPED_CHUNK": "64"})
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-2000:] + r.stderr[-2000:]
