"""Varlen causal MLA prefill: ktb200_mla_prefill_varlen (csrc/mla_prefill.cu, mla_prefill_varlen_kernel) and the split path
of KDeepseekV2Attention.forward_ragged (prompt sequences decompressed, decode rows absorbed).

CPU: every refusal with its message; the binding's struct layout against the header.  GPU: the kernel against the float64
oracle per sequence (test_mla_prefill's bounds) on mixed batches in shuffled order with gaps between their rows; bit for bit
each sequence equals ktb200_mla_prefill on it alone, and permuting or moving the sequences changes nothing; isolation from
every row the call does not name; causality; empty sequences.  The operator against each sequence run alone through forward
and against the float64 module; decode-only steps equal the absorbed path; the launch census; no host synchronisation."""
import copy
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import mla_prefill_oracle as mpo
from ktransformers_b200 import native
from test_mla_lengths import boundary_rows
from test_mla_prefill import SCALE, _modules, _rel

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
MAX_BATCH = native.MLA_PREFILL_VARLEN_MAX_BATCH


# ------------------------------------------------------------------------------------------------ C-ABI (CPU)
def _params(rows, q_rows=4096, k_rows=8192, H=16, **over):
    """a well-formed call over fake 16-byte-aligned addresses; `rows` the host int32 seq array [batch][4], kept alive by the
    caller"""
    base = 1 << 24
    a = dict(batch=len(rows), q_rows=q_rows, k_rows=k_rows, num_heads=H, qk_nope_head_dim=128, qk_rope_head_dim=64, v_head_dim=128,
             sm_scale=SCALE, seq=rows.ctypes.data,
             q_nope=base, q_nope_token_stride=H * 192, q_nope_head_stride=192,
             q_pe=base + (1 << 28), q_pe_token_stride=H * 64, q_pe_head_stride=64,
             k_nope=base + (2 << 28), k_nope_token_stride=H * 256, k_nope_head_stride=256,
             v=base + (2 << 28) + 256, v_token_stride=H * 256, v_head_stride=256,
             k_pe=base + (3 << 28), k_pe_token_stride=576, out=base + (4 << 28))
    a.update(over)
    return native.MlaPrefillVarlenParams(**a)


def _seq(rows):
    return np.ascontiguousarray(np.array(rows, np.int32).reshape(-1, 4))


GOOD = [[0, 100, 0, 300], [200, 1, 300, 50], [100, 0, 0, 0], [150, 50, 400, 50]]

BAD = {
    "nope dim": (dict(qk_nope_head_dim=64), None, "head dims"),
    "rope dim": (dict(qk_rope_head_dim=32), None, "head dims"),
    "v dim": (dict(v_head_dim=192), None, "head dims"),
    "heads 0": (dict(num_heads=0), None, "num_heads"),
    "scale 0": (dict(sm_scale=0.0), None, "sm_scale"),
    "scale nan": (dict(sm_scale=float("nan")), None, "sm_scale"),
    "scale inf": (dict(sm_scale=float("inf")), None, "sm_scale"),
    "null q_nope": (dict(q_nope=None), None, "null pointer (q_nope)"),
    "null q_pe": (dict(q_pe=None), None, "null pointer (q_pe)"),
    "null k_nope": (dict(k_nope=None), None, "null pointer (k_nope)"),
    "null v": (dict(v=None), None, "null pointer (v)"),
    "null k_pe": (dict(k_pe=None), None, "null pointer (k_pe)"),
    "null out": (dict(out=None), None, "null pointer (out)"),
    "null seq": (dict(seq=None), None, "null pointer (seq)"),
    "q_nope +2 B": (dict(q_nope=(1 << 24) + 2), None, "q_nope must be 16-byte aligned"),
    "v +8 B": (dict(v=(1 << 24) + (2 << 28) + 264), None, "v must be 16-byte aligned"),
    "k_pe +2 B": (dict(k_pe=(1 << 24) + (3 << 28) + 2), None, "k_pe must be 16-byte aligned"),
    "out +4 B": (dict(out=(1 << 24) + (4 << 28) + 4), None, "out must be 16-byte aligned"),
    "q_pe head stride 68": (dict(q_pe_head_stride=68), None, "q_pe head stride"),
    "k_pe token stride 577": (dict(k_pe_token_stride=577), None, "k_pe token stride"),
    "k_nope token stride 0": (dict(k_nope_token_stride=0), None, "k_nope token stride"),
    "v head stride -8": (dict(v_head_stride=-8), None, "v head stride"),
    "batch 0": (dict(batch=0), None, "batch 0 must be in 1 .. 1024"),
    "batch over the cap": (dict(batch=MAX_BATCH + 1), [[0, 0, 0, 0]] * (MAX_BATCH + 1), "batch 1025 must be in 1 .. 1024"),
    "q_rows negative": (dict(q_rows=-1), None, "q_rows -1"),
    "k_rows negative": (dict(k_rows=-1), None, "k_rows"),
    "negative q_row": (None, [[-1, 2, 0, 2]], "negative value"),
    "negative q_len": (None, [[0, -2, 0, 2]], "negative value"),
    "negative k_row": (None, [[0, 2, -64, 2]], "negative value"),
    "negative kv_len": (None, [[0, 0, 0, -1]], "negative value"),
    "q_len > kv_len": (None, [[0, 101, 0, 100]], "needs q_len (101) <= kv_len (100)"),
    "q_len over the grid": (dict(q_rows=1 << 24), [[0, 65535 * 128 + 1, 0, 65535 * 128 + 1]], "exceeds 8388480 tokens"),
    "queries past q_rows": (None, [[4000, 97, 0, 100]], "query rows 4000 .. 4097 are outside q_rows 4096"),
    "keys past k_rows": (None, [[0, 10, 8190, 10]], "key rows 8190 .. 8200 are outside k_rows 8192"),
    "empty queries past q_rows": (None, [[4097, 0, 0, 0]], "outside q_rows"),
    "output rows overlap": (None, GOOD + [[250, 10, 0, 10], [255, 3, 0, 3]], "sequences 4 and 5 overlap"),
    "output rows overlap by one": (None, [[10, 5, 0, 5], [0, 11, 0, 11]], "sequences 1 and 0 overlap"),
    "same output rows": (None, [[0, 4, 0, 4], [0, 4, 100, 4]], "overlap"),
}


@pytest.mark.parametrize("case", sorted(BAD))
def test_refusals(case):
    """each malformed call returns KTB200_EINVAL with a message naming the problem, before any device work (the addresses
    are fake: a launch would fault)"""
    lib = native.lib()
    over, rows, msg = BAD[case]
    seq = _seq(rows if rows is not None else GOOD)
    p = _params(seq, **(over or {}))
    assert lib.ktb200_mla_prefill_varlen(C.byref(p), None) == native.EINVAL
    assert msg in lib.ktb200_last_error().decode(), lib.ktb200_last_error().decode()


def test_null_params_and_no_work():
    lib = native.lib()
    assert lib.ktb200_mla_prefill_varlen(None, None) == native.EINVAL
    assert "null" in lib.ktb200_last_error().decode()
    # sequences without queries: valid, nothing to launch (no device is touched, so this runs without one)
    seq = _seq([[0, 0, 0, 0], [0, 0, 3, 7]])
    assert lib.ktb200_mla_prefill_varlen(C.byref(_params(seq, q_rows=0)), None) == native.OK
    # adjacent output rows do not overlap; key ranges may
    seq = _seq([[10, 5, 0, 5], [0, 10, 0, 10], [15, 1, 0, 9]])
    p = _params(seq, num_heads=0)     # refused after the sequence checks would have passed: the rows themselves are fine
    assert lib.ktb200_mla_prefill_varlen(C.byref(p), None) == native.EINVAL and "num_heads" in lib.ktb200_last_error().decode()


FIELDS = [f for f, _ in native.MlaPrefillVarlenParams._fields_]


def test_struct_layout_matches_the_header(tmp_path):
    """offsetof / sizeof of ktb200_mla_prefill_varlen_params from the header, compiled, against the ctypes structure"""
    cxx = shutil.which("c++") or shutil.which("g++") or shutil.which("gcc")
    assert cxx, "a C++ compiler is needed to read the header's layout"
    src = tmp_path / "layout.cpp"
    body = "".join(f'    printf("{f} %zu\\n", offsetof(ktb200_mla_prefill_varlen_params, {f}));\n' for f in FIELDS)
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "ktb200.h"\nint main() {\n' + body +
                   '    printf("size %zu\\n", sizeof(ktb200_mla_prefill_varlen_params));\n'
                   '    printf("cap %d\\n", KTB200_MLA_PREFILL_VARLEN_MAX_BATCH);\n    return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call([cxx, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    for f in FIELDS:
        assert int(got[f]) == getattr(native.MlaPrefillVarlenParams, f).offset, f
    assert int(got["size"]) == C.sizeof(native.MlaPrefillVarlenParams)
    assert int(got["cap"]) == MAX_BATCH


# ------------------------------------------------------------------------------------------------ GPU helpers
class Batch:
    """operands in the operator's layouts, rows placed by the caller: q [q_rows, H, 192] (q_nope = columns :128, as in the q_b
    output), q_pe [q_rows, H, 64], kv [k_rows, H, 256] (k_nope | v, as kv_b_proj's output), lat [k_rows, 576] (k_pe = columns
    512:).  Rows the sequences do not name hold `fill` (NaN and Inf by default)."""

    def __init__(self, H, seq, q_rows, k_rows, seed, fill=float("nan")):
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.H, self.seq = H, np.ascontiguousarray(np.array(seq, np.int32).reshape(-1, 4))
        rnd = lambda *s: torch.randn(*s, generator=g, device="cuda", dtype=torch.bfloat16)
        self.q, self.q_pe, self.kv, self.lat = rnd(q_rows, H, 192), rnd(q_rows, H, 64), rnd(k_rows, H, 256), rnd(k_rows, 576)
        self.fill_unnamed(fill)

    def named(self):
        qm = torch.zeros(self.q.shape[0], dtype=torch.bool)
        km = torch.zeros(self.kv.shape[0], dtype=torch.bool)
        for qr, ql, kr, kl in self.seq.tolist():
            qm[qr:qr + ql] = True
            km[kr:kr + kl] = True
        return qm.cuda(), km.cuda()

    def fill_unnamed(self, fill):
        if fill is None:
            return
        qm, km = self.named()
        for t, m in ((self.q, qm), (self.q_pe, qm), (self.kv, km), (self.lat, km)):
            idx = torch.nonzero(~m).flatten()
            t[idx[0::2]] = fill
            t[idx[1::2]] = float("inf") if fill != fill else fill

    def run(self, seq=None, out=None):
        seq = self.seq if seq is None else np.ascontiguousarray(seq, np.int32)
        H = self.H
        qn, kn, v, kp = self.q[..., :128], self.kv[..., :128], self.kv[..., 128:], self.lat[:, 512:]
        if out is None:
            out = torch.full((self.q.shape[0], H, 128), float("nan"), dtype=torch.bfloat16, device="cuda")
        p = native.MlaPrefillVarlenParams(len(seq), self.q.shape[0], self.kv.shape[0], H, 128, 64, 128, SCALE, seq.ctypes.data,
                                          qn.data_ptr(), qn.stride(0), qn.stride(1), self.q_pe.data_ptr(), self.q_pe.stride(0),
                                          self.q_pe.stride(1), kn.data_ptr(), kn.stride(0), kn.stride(1), v.data_ptr(), v.stride(0),
                                          v.stride(1), kp.data_ptr(), kp.stride(0), out.data_ptr())
        native.check(native.lib().ktb200_mla_prefill_varlen(C.byref(p), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        return out

    def dense(self, b):
        """ktb200_mla_prefill (batch 1) on sequence b alone -> [q_len, H, 128]"""
        qr, ql, kr, kl = self.seq[b].tolist()
        q, qp, kv, lat = self.q[qr:qr + ql], self.q_pe[qr:qr + ql], self.kv[kr:kr + kl], self.lat[kr:kr + kl]
        qn, kn, v, kp = q[..., :128], kv[..., :128], kv[..., 128:], lat[:, 512:]
        out = torch.full((ql, self.H, 128), float("nan"), dtype=torch.bfloat16, device="cuda")
        big = 1 << 30
        p = native.MlaPrefillParams(1, ql, kl, self.H, 128, 64, 128, SCALE, qn.data_ptr(), qn.stride(0), qn.stride(1), big,
                                    qp.data_ptr(), qp.stride(0), qp.stride(1), big, kn.data_ptr(), kn.stride(0), kn.stride(1), big,
                                    v.data_ptr(), v.stride(0), v.stride(1), big, kp.data_ptr(), kp.stride(0), big, out.data_ptr())
        native.check(native.lib().ktb200_mla_prefill(C.byref(p), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        return out

    def oracle(self, b, rows, heads, p_bf16=False):
        """float64 oracle of sequence b's query rows `rows` at heads `heads` -> [rows, heads, 128]; query i sees the first
        P + i + 1 keys"""
        qr, ql, kr, kl = self.seq[b].tolist()
        P = kl - ql
        hs = torch.as_tensor(heads, device="cuda")
        f = lambda t: t.double().cpu().numpy()
        kv, kp = f(self.kv[kr:kr + kl].index_select(1, hs)), f(self.lat[kr:kr + kl, 512:])
        q, qp = f(self.q[qr:qr + ql].index_select(1, hs)), f(self.q_pe[qr:qr + ql].index_select(1, hs))
        out = []
        for i in rows:
            S = P + i + 1
            out.append(mpo.mla_prefill(q[None, i:i + 1, :, :128], qp[None, i:i + 1], kv[None, :S, :, :128], kp[None, :S], kv[None, :S, :, 128:],
                                       SCALE, p_bf16)[0, 0])
        return np.stack(out)


def place(rng, qk, gap=37, share_keys=False):
    """(q_len, kv_len) pairs -> seq rows in a shuffled order with gaps between them; (seq, q_rows, k_rows)"""
    order = rng.permutation(len(qk))
    seq = np.zeros((len(qk), 4), np.int32)
    qr = kr = int(rng.integers(1, gap))
    for b in order:
        ql, kl = qk[b]
        seq[b] = (qr, ql, kr if not share_keys else 5, kl)
        qr += ql + int(rng.integers(0, gap))
        if not share_keys:
            kr += kl + int(rng.integers(0, gap))
    k_rows = kr + gap if not share_keys else 5 + max(kl for _, kl in qk) + gap
    return seq, qr + gap, k_rows


def check_vs_oracle(bt, b, rng, got, family):
    """test_mla_prefill's bounds on sampled rows and heads of sequence b"""
    qr, ql, kr, kl = bt.seq[b].tolist()
    rows = boundary_rows(ql, rng, extra=2) if ql <= 300 else np.unique(np.r_[0, 1, 63, 64, 127, 128, 129, ql - 1, rng.integers(0, ql, 4)])
    heads = np.arange(bt.H) if bt.H <= 16 else np.unique(np.r_[0, 63, 64, bt.H - 1, rng.integers(0, bt.H, 2)])
    out = got[qr + rows][:, heads].float().cpu().numpy()
    exact = bt.oracle(b, rows, heads)
    mag = np.abs(exact).max()
    err = np.abs(out - exact)
    print(f"{family} q_len={ql} P={kl - ql}: max err {err.max() / mag:.2e} of max |out|")
    assert np.isfinite(out).all()
    assert err.max() <= 2e-2 * mag and err.mean() <= 5e-3 * np.abs(exact).mean(), (family, ql, kl - ql)
    if bt.H == 16:
        want = bt.oracle(b, rows, heads, p_bf16=True)
        assert np.abs(out - want).max() <= 2.0 ** -7 * mag + 1e-3 * mag


def bits(t):
    return t.view(torch.int16)


Q_LENS = [1, 2, 127, 128, 129, 1000]


# ------------------------------------------------------------------------------------------------ kernel (GPU)
@pytest.mark.gpu
@pytest.mark.parametrize("past", [0, 1, 63, 4095, 32768])
@pytest.mark.parametrize("H", [128, 16])
def test_varlen_vs_oracle_and_each_sequence_alone(H, past):
    """the six q_lens at `past`, plus a 200-token chunk after 300 and a decode row after 5000 (mixed P), shuffled, gaps
    between their rows (NaN / Inf there): every sequence within the oracle bounds, and equal to ktb200_mla_prefill on it
    alone bit for bit.  At P = 32768 and 128 heads the sequences share one key range (13 GB otherwise)."""
    rng = np.random.default_rng(past * 3 + H)
    qk = [(q, past + q) for q in Q_LENS] + [(200, 500), (1, 5001)]
    seq, q_rows, k_rows = place(rng, qk, share_keys=past == 32768 and H == 128)
    bt = Batch(H, seq, q_rows, k_rows, seed=past + H)
    got = bt.run()
    for b in range(len(seq)):
        qr, ql = int(seq[b, 0]), int(seq[b, 1])
        assert torch.equal(bits(got[qr:qr + ql]), bits(bt.dense(b))), f"sequence {b} {qk[b]} differs from its run alone"
        check_vs_oracle(bt, b, rng, got, f"varlen H={H}")


@pytest.mark.gpu
def test_permuting_and_moving_sequences_changes_no_bit():
    """the same sequences listed in another order, and with their rows moved to other offsets (other gaps, other order in
    memory): every sequence's output bit-identical"""
    rng = np.random.default_rng(11)
    qk = [(129, 129), (1, 300), (1000, 1100), (2, 4097), (127, 127), (128, 700)]
    seq, q_rows, k_rows = place(rng, qk)
    a = Batch(128, seq, q_rows, k_rows, seed=11)
    base = a.run()
    perm = rng.permutation(len(qk))
    again = a.run(seq=seq[perm])
    assert torch.equal(bits(base), bits(again))
    seq2, q_rows2, k_rows2 = place(np.random.default_rng(12), qk, gap=300)
    b = Batch(128, seq2, q_rows2, k_rows2, seed=99)
    for i in range(len(qk)):   # copy sequence i's rows to their new places
        (qr, ql, kr, kl), (qr2, _, kr2, _) = seq[i].tolist(), seq2[i].tolist()
        b.q[qr2:qr2 + ql], b.q_pe[qr2:qr2 + ql] = a.q[qr:qr + ql], a.q_pe[qr:qr + ql]
        b.kv[kr2:kr2 + kl], b.lat[kr2:kr2 + kl] = a.kv[kr:kr + kl], a.lat[kr:kr + kl]
    moved = b.run(seq=seq2[perm[::-1]])
    for i in range(len(qk)):
        qr, ql, qr2 = int(seq[i, 0]), int(seq[i, 1]), int(seq2[i, 0])
        assert torch.equal(bits(base[qr:qr + ql]), bits(moved[qr2:qr2 + ql])), i


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 16])
def test_isolation_from_rows_not_named(H):
    """sequences back to back and with gaps, the last one's keys ending at k_rows (the TMA zero-fill edge), one followed
    directly by the next sequence's keys: unnamed output rows keep their NaN; NaN / Inf in every unnamed query row and in
    every key row outside the named ranges (gaps, after the last) change no bit against finite random values there; every
    sequence equals its run alone"""
    # q rows: [3, 203) [203, 204) gap [260, 389) gap [400, 401); k rows: [0, 330) [330, 631) gap [700, 1000) [1100, 1229]
    seq = np.array([[3, 200, 0, 330], [203, 1, 330, 301], [260, 129, 1100, 129], [400, 1, 700, 300]], np.int32)
    q_rows, k_rows = 430, 1229
    dirty = Batch(H, seq, q_rows, k_rows, seed=H)
    clean = copy.copy(dirty)
    clean.q, clean.q_pe, clean.kv, clean.lat = dirty.q.clone(), dirty.q_pe.clone(), dirty.kv.clone(), dirty.lat.clone()
    g = torch.Generator(device="cuda").manual_seed(3)
    qm, km = clean.named()
    for t, m in ((clean.q, qm), (clean.q_pe, qm), (clean.kv, km), (clean.lat, km)):
        t[~m] = torch.randn(t[~m].shape, generator=g, device="cuda").to(torch.bfloat16) * 4
    out_d, out_c = dirty.run(), clean.run()
    assert torch.isnan(out_d[~qm].float()).all() and torch.isnan(out_c[~qm].float()).all(), "a row no sequence names was written"
    assert torch.isfinite(out_d[qm].float()).all()
    assert torch.equal(bits(out_d), bits(out_c))
    for b in range(len(seq)):
        qr, ql = int(seq[b, 0]), int(seq[b, 1])
        assert torch.equal(bits(out_d[qr:qr + ql]), bits(dirty.dense(b))), b


@pytest.mark.gpu
@pytest.mark.parametrize("P,q_len,k", [(0, 300, 130), (0, 300, 128), (300, 200, 77), (1000, 37, 1)])
def test_varlen_is_causal(P, q_len, k):
    """keys of the middle sequence at positions >= P + k overwritten with other finite values leave its queries i < k and the
    other sequences bit-identical, and change its queries >= k (within a sequence, as in the dense kernel and
    flash_attn_func, a key above a row's diagonal meets P = 0 in P.V, and 0 * NaN would be NaN: only keys past kv_len, which
    belong to no row of the sequence, are zeroed)"""
    seq = np.array([[0, 50, 0, 60], [60, q_len, 70, P + q_len], [70 + q_len, 3, 80 + P + q_len, 10]], np.int32)
    bt = Batch(16, seq, 80 + q_len, 100 + P + q_len, seed=k)
    base = bt.run()
    kr = 70 + P + k
    bt.kv[kr:70 + P + q_len:2], bt.lat[kr:70 + P + q_len:2] = 300.0, 300.0
    bt.kv[kr + 1:70 + P + q_len:2], bt.lat[kr + 1:70 + P + q_len:2] = -300.0, -300.0
    after = bt.run()
    keep = torch.cat([torch.arange(0, 60 + k), torch.arange(60 + q_len, 73 + q_len)])
    assert torch.equal(bits(base[keep]), bits(after[keep]))
    assert not torch.equal(bits(base[60 + k:60 + q_len]), bits(after[60 + k:60 + q_len]))


@pytest.mark.gpu
def test_empty_sequences_write_nothing():
    """q_len 0 sequences (with and without keys) between others: their rows, and every unnamed row, stay NaN; the others
    equal the batch without the empty ones bit for bit"""
    seq = np.array([[0, 0, 0, 500], [0, 130, 0, 200], [130, 0, 200, 0], [140, 1, 200, 40], [141, 0, 0, 0]], np.int32)
    bt = Batch(128, seq, 200, 600, seed=4)
    out = bt.run()
    qm, _ = bt.named()
    assert torch.isnan(out[~qm].float()).all()
    assert torch.equal(bits(out), bits(bt.run(seq=seq[[1, 3]])))
    only_empty = bt.run(seq=seq[[0, 2, 4]])
    assert torch.isnan(only_empty.float()).all()


# ------------------------------------------------------------------------------------------------ operator (GPU)
def _mixed_operator(absorb):
    from ktransformers_b200.operators import attention as attn_mod
    from ktransformers_b200.operators.attention import KDeepseekV2Attention
    cfg, plain, _ = _modules(128, 77)
    attn_mod._RAGGED_WRAPPERS.clear()
    return cfg, plain, KDeepseekV2Attention("blk.0.self_attn", None, cfg, plain, "cuda", "cuda", absorb_for_prefill=absorb)


# the five steps of test_mla_ragged's operator test over its four sequences, then three new prompts (700 / 128 / 2 tokens)
# beside four long-history decode rows
STEPS = [[126, 1000, 500, 0, 0, 0, 0], [1, 1, 200, 150, 0, 0, 0], [1, 1, 1, 7, 0, 0, 0], [1, 1, 3, 1, 0, 0, 0], [1, 1, 1, 1, 0, 0, 0],
         [1, 1, 1, 1, 700, 128, 2]]
CACHE_ROWS = [2, 0, 5, 3, 1, 6, 4]


def _drive(op, cfg, xs, steps, on_step=None):
    from ktransformers_b200.models.custom_cache import StaticCache
    n = len(xs)
    cache = StaticCache(cfg, max_batch_size=n, max_cache_len=1536, device="cuda")
    got = [[] for _ in range(n)]
    done = np.zeros(n, np.int64)
    for k, q in enumerate(steps):
        q = np.array(q)
        x = torch.cat([xs[b][done[b]:done[b] + q[b]] for b in range(n)])
        pos = torch.cat([torch.arange(done[b], done[b] + q[b], device="cuda") for b in range(n)])
        qo = torch.from_numpy(np.r_[0, np.cumsum(q)].astype(np.int32))
        kv_len = torch.from_numpy((done + q).astype(np.int32))
        rows = torch.from_numpy(np.argsort(CACHE_ROWS[:n]).astype(np.int32))   # a permutation of the cache's rows
        call = lambda: op.forward_ragged(x, pos, qo, kv_len, rows, cache, max_rows=2048, max_items=8192)
        out = on_step(k, call) if on_step else call()
        for b in range(n):
            got[b].append(out[qo[b]:qo[b + 1]])
        done += q
    return got, cache


@pytest.mark.gpu
def test_operator_split_steps_match_each_sequence_alone():
    """absorb_for_prefill=False: the mixed steps through forward_ragged, each sequence against it run alone through forward
    (decompressed chunks, absorbed decode) and against the float64 module, within the operator bar; one whole mixed step
    under torch.cuda.set_sync_debug_mode("error")"""
    cfg, plain, op = _mixed_operator(False)
    plain64 = copy.deepcopy(plain).double()
    total = np.sum(STEPS, 0)
    xs = [(torch.randn(int(n), 1024, device="cuda") * 2).to(torch.bfloat16) for n in total]

    def on_step(k, call):
        if k != 5:
            return call()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            return call()
        finally:
            torch.cuda.set_sync_debug_mode("default")

    got, cache = _drive(op, cfg, xs, STEPS, on_step)
    assert cache.get_seq_length(0) == 0, "forward_ragged leaves the host counter alone"
    from ktransformers_b200.models.custom_cache import StaticCache
    worst_alone = worst64 = 0.0
    for b in range(len(xs)):
        g = torch.cat(got[b])
        alone_cache = StaticCache(cfg, max_batch_size=1, max_cache_len=1536, device="cuda")
        alone, start = [], 0
        for q in np.array(STEPS)[:, b]:
            if q:
                o, _, _ = op(xs[b][None, start:start + q], position_ids=torch.arange(start, start + q, device="cuda")[None],
                             past_key_value=alone_cache, cache_position=torch.arange(start, start + q, device="cuda"))
                alone.append(o[0])
            start += q
        alone = torch.cat(alone)
        want, _ = plain64(xs[b][None].double(), torch.arange(int(total[b]), device="cuda")[None])
        worst_alone, worst64 = max(worst_alone, _rel(g, alone)), max(worst64, _rel(g, want[0]))
    print(f"[operator split] {worst_alone / 4e-2:.3f} of the bound vs alone, {worst64 / 4e-2:.3f} vs float64")
    assert worst_alone < 4e-2 and worst64 < 4e-2, (worst_alone, worst64)


@pytest.mark.gpu
def test_decode_only_steps_equal_the_absorbed_path():
    """after a prompt step, decode-only steps give the same bits with absorb_for_prefill False and True (the same calls)"""
    cfg, plain, op = _mixed_operator(False)
    steps = [[300, 5, 64, 0], [1, 1, 1, 0], [1, 0, 1, 1]]
    xs = [(torch.randn(int(n), 1024, device="cuda") * 2).to(torch.bfloat16) for n in np.sum(steps, 0)]
    outs = []

    def on_step(k, call):
        out = call()
        if k:   # the same step again through the absorbed layer: it rewrites the same latents at the same positions
            op_k, op.absorb_for_prefill = op.absorb_for_prefill, True
            try:
                outs.append((out.clone(), call()))
            finally:
                op.absorb_for_prefill = op_k
        return out

    _drive(op, cfg, xs, steps, on_step)
    assert len(outs) == 2
    for a, b in outs:
        assert torch.equal(bits(a), bits(b))


def _launch_census():
    from test_linear_routes import _census
    torch.cuda.set_device(0)
    cfg, plain, op = _mixed_operator(False)
    from ktransformers_b200.models.custom_cache import StaticCache
    cache = StaticCache(cfg, max_batch_size=4, max_cache_len=1024, device="cuda")
    xs = (torch.randn(900, 1024, device="cuda") * 2).to(torch.bfloat16)
    state = {"done": np.zeros(4, np.int64)}

    def step(q, absorb):
        def fn():
            q_ = np.array(q)
            done = state["done"]
            x = xs[:int(q_.sum())]
            pos = torch.cat([torch.arange(done[b], done[b] + q_[b], device="cuda") for b in range(4)])
            op.absorb_for_prefill = absorb
            op.forward_ragged(x, pos, torch.from_numpy(np.r_[0, np.cumsum(q_)].astype(np.int32)),
                              torch.from_numpy((done + q_).astype(np.int32)), torch.tensor([1, 3, 0, 2], dtype=torch.int32), cache,
                              max_rows=1024, max_items=4096)
            state["done"] = done + q_
        return fn

    plan = [("prompts only", [100, 30, 0, 0], False), ("mixed", [1, 1, 200, 0], False), ("mixed absorbed", [1, 1, 1, 40], True),
            ("decode only", [1, 1, 1, 1], False), ("prompt beside decode", [1, 2, 1, 1], False)]
    calls = [(label, (q, absorb), step(q, absorb)) for label, q, absorb in plan]
    for label, (q, absorb), n, names in _census(calls):
        varlen = sum("mla_prefill_varlen_kernel" in k for k in names)
        decode = sum(("mla_decode_tc_kernel" in k) or ("mla_ragged_tc_kernel" in k) for k in names)
        has_prompt, has_decode = any(v > 1 for v in q), any(v == 1 for v in q)
        assert not any("mla_prefill_kernel" in k for k in names), (label, names)
        if absorb or not has_prompt:
            assert varlen == 0 and decode >= 1, (label, names)
        else:
            assert varlen == 1, (label, names)
            assert (decode >= 1) == has_decode, (label, names)


@pytest.mark.gpu
def test_launch_census():
    """one varlen launch per step with a prompt chunk (without absorb_for_prefill), the absorbed MLA kernels only when decode
    rows exist, no varlen launch with absorb_for_prefill or in a decode-only step.  In an interpreter of its own: after other
    profiler sessions in one process, torch.profiler can miss kernels"""
    code = ("import sys; sys.path[:0] = sys.argv[1:]; import test_mla_prefill_varlen as t\n"
            "try:\n    t._launch_census(); print('OK')\nexcept AssertionError as e:\n    print(e); sys.exit(1)")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code, ROOT, HERE]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and r.stdout.strip().endswith("OK"), r.stdout[-3000:] + r.stderr[-3000:]
