"""Ragged batches through absorbed MLA: ktb200_mla_ragged_plan (host), ktb200_mla_decode_ragged (csrc/mla.cu,
mla_ragged_tc_kernel + mla_ragged_merge_kernel), the ragged path of MLAWrapper and KDeepseekV2Attention.forward_ragged.

Token i of sequence b attends to the first kv_len[b] - q_len_b + i + 1 cached latents, so every row must equal the absorbed
decode oracle (oracle/mla_oracle.mla_decode) at that length; rows and heads are sampled as in test_mla_chunk.

CPU: the planner's coverage, limits, explicit-split ranges and refusals, the run entry's refusals, the wrapper's choice of
path.  GPU: mixed batches against the oracle; bit-exact pins against ktb200_mla_decode_chunk and ktb200_mla_decode,
causality, sentinels, CUDA-graph replays across re-plans; the operator against each sequence run alone and in float64."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from ktransformers_b200 import native
from oracle import mla_oracle
from test_mla_chunk import _decode, chunk, queries, random_pages
from test_mla_lengths import MAX_SPLITS, POOL_ROWS, boundary_rows, check_decode, sms
from test_mla_prefill import SCALE, _modules, _rel

PAGE = 64
H100_SMS = 132


# ------------------------------------------------------------------------------------------------ helpers
def plan(qo, kv_len, H, page, max_pages, num_sms=H100_SMS, splits=0, max_items=1 << 16, max_rows=1 << 15, plan_ints=None):
    """ktb200_mla_ragged_plan on host arrays -> (rc, plan int32 array, slots, workspace bytes)"""
    lib = native.lib()
    qo, kv = np.ascontiguousarray(qo, np.int32), np.ascontiguousarray(kv_len, np.int32)
    n = lib.ktb200_mla_ragged_plan_ints(max_items, max_rows) if plan_ints is None else plan_ints
    buf = np.zeros(max(n, 1), np.int32)
    slots, ws = C.c_int(), C.c_size_t()
    rc = lib.ktb200_mla_ragged_plan(qo.ctypes.data, kv.ctypes.data, len(kv), H, page, max_pages, num_sms, splits, max_items, max_rows,
                                    buf.ctypes.data, n, C.byref(slots), C.byref(ws))
    return rc, buf, slots.value, ws.value


def items_of(buf):
    """-> (items [n, 7]: row, seq, head group, tile0, tile1, limit, slot ; row_off [rows + 1])"""
    n, rows, _, cap = buf[:4]
    it = buf[8:8 + 8 * n].reshape(n, 8)[:, :7]
    off = 8 + 8 * cap
    return it, buf[off:off + rows + 1]


def tiles(x):
    return -(-np.asarray(x, np.int64) // 32)


def row_limits(qo, kv_len):
    """per query row: (sequence, key limit)"""
    seq, lim = [], []
    for b in range(len(kv_len)):
        q = qo[b + 1] - qo[b]
        seq += [b] * q
        lim += [kv_len[b] - q + i + 1 for i in range(q)]
    return np.array(seq, np.int64), np.array(lim, np.int64)


def check_plan(qo, kv_len, H, buf, slots, num_sms=H100_SMS, max_items=None):
    """every (row, head group) tile below the row's limit covered exactly once, nothing at or past it; slots, row offsets,
    launch order; -> (largest item in tiles, the balance bound, whether some sequence has 128 ranges)"""
    it, row_off = items_of(buf)
    hgs = -(-H // 64)
    seq, lim = row_limits(qo, kv_len)
    rows = len(lim)
    assert buf[1] == rows and buf[2] == slots and row_off[-1] == slots and len(row_off) == rows + 1
    if max_items is not None:
        assert buf[0] <= max_items
    if rows == 0:
        assert buf[0] == 0
        return 0, 0, False
    r, s, g, t0, t1, L, sl = (it[:, k].astype(np.int64) for k in range(7))
    assert (s == seq[r]).all() and (L == lim[r]).all() and (g >= 0).all() and (g < hgs).all()
    assert (t0 < t1).all() and (t1 <= tiles(L)).all()
    # exact cover: per (row, head group) the tile counts add up, and ranges are disjoint (sorted, each starts at the last end)
    key = (r * hgs + g)
    order = np.lexsort((t0, key))
    k2, a, e = key[order], t0[order], t1[order]
    first = np.r_[True, k2[1:] != k2[:-1]]
    assert (a[first] == 0).all()
    prev_end = np.r_[0, e[:-1]]
    assert (a[~first] == prev_end[~first]).all()
    last = np.r_[k2[1:] != k2[:-1], True]
    ends = np.zeros(rows * hgs, np.int64)
    ends[k2[last]] = e[last]
    assert (ends == np.repeat(tiles(lim), hgs)).all(), "a (row, head group) is not covered up to its limit"
    assert len(np.unique(k2)) == rows * hgs
    # slots: inside the row's range, at most 128 per row, each used by exactly one item per head group
    assert (sl >= row_off[r]).all() and (sl < row_off[r + 1]).all()
    assert (np.diff(row_off) <= MAX_SPLITS).all() and (np.diff(row_off) >= 1).all()
    assert (np.bincount(sl, minlength=slots) == hgs).all()
    # launch order: the items of one (sequence, range) are adjacent
    rng_start = np.r_[True, (s[1:] != s[:-1]) | (t0[1:] != t0[:-1])]
    starts = list(zip(s[rng_start].tolist(), t0[rng_start].tolist()))
    assert len(starts) == len(set(starts)), "a (sequence, range) is split across the list"
    work = int(tiles(lim).sum()) * hgs
    bound = max(4, -(-work // num_sms))
    capped = any(len(np.unique(t0[s == b])) == MAX_SPLITS for b in np.unique(s))
    return int((t1 - t0).max()), bound, capped


def random_batch(rng, B, cap=131072):
    """B sequences: mostly decode rows, some prompt chunks (up to 1000), some empty; lengths up to cap"""
    kind = rng.choice(3, B, p=[0.6, 0.3, 0.1])
    q = np.where(kind == 0, 1, np.where(kind == 1, rng.integers(2, 1001, B), 0))
    past = np.where(rng.random(B) < 0.3, rng.integers(0, 4096, B), rng.integers(0, cap, B))
    kv = np.minimum(past + q, cap)
    q = np.minimum(q, kv)
    return np.r_[0, np.cumsum(q)].astype(np.int32), kv.astype(np.int32)


# ------------------------------------------------------------------------------------------------ planner (CPU)
@pytest.mark.parametrize("seed", range(24))
def test_planner_covers_every_tile_once(seed):
    rng = np.random.default_rng(seed)
    B = int(rng.choice([1, 2, 7, 66, 130]))
    H = int(rng.choice([16, 40, 128]))
    page = int(rng.choice([64, 256]))
    qo, kv = random_batch(rng, B)
    rc, buf, slots, ws = plan(qo, kv, H, page, -(-131072 // page))
    assert rc == native.OK, native.lib().ktb200_last_error()
    biggest, bound, capped = check_plan(qo, kv, H, buf, slots)
    assert capped or biggest <= bound, (biggest, bound)
    assert ws == slots * H * 513 * 4


def test_planner_balances_the_skewed_batch():
    """one sequence at 131072 and 65 at 1024: the long one is cut to the balance bound, the short ones stay whole"""
    kv = np.array([131072] + [1024] * 65, np.int32)
    qo = np.arange(67, dtype=np.int32)
    rc, buf, slots, _ = plan(qo, kv, 128, PAGE, 2048)
    assert rc == native.OK
    biggest, bound, capped = check_plan(qo, kv, 128, buf, slots)
    assert not capped and biggest <= bound
    it, _ = items_of(buf)
    assert len(np.unique(it[it[:, 1] == 0, 3])) == -(-4096 // bound)
    assert (it[it[:, 1] > 0, 4] - it[it[:, 1] > 0, 3] == 32).all()


@pytest.mark.parametrize("max_items", [268, 300, 1000, 4000])
def test_planner_respects_the_item_capacity(max_items):
    """the bound doubles until the items fit; at the minimum (one range per sequence) it still fits, below it refuses"""
    kv = np.array([131072, 100000, 5000, 70] + [2048] * 128, np.int32)
    qo = np.r_[0, np.cumsum([1, 1, 1, 3] + [1] * 128)].astype(np.int32)
    rc, buf, slots, _ = plan(qo, kv, 128, PAGE, 2048, max_items=max_items)
    assert rc == native.OK, native.lib().ktb200_last_error()
    check_plan(qo, kv, 128, buf, slots, max_items=max_items)
    rc, *_ = plan(qo, kv, 128, PAGE, 2048, max_items=267)
    assert rc == native.EINVAL and "item capacity" in native.lib().ktb200_last_error().decode()


@pytest.mark.parametrize("B,q_len,splits", [(1, 16, 7), (3, 40, 2), (4, 1, 5), (2, 100, 128), (1, 1, 1)])
def test_explicit_splits_give_the_chunk_entry_ranges(B, q_len, splits):
    """tiles_per = ceil(tiles(P + q_len) / splits); token i has the splits that start below its limit, in split order"""
    rng = np.random.default_rng(B * q_len + splits)
    kv = (rng.integers(0, 9000, B) + q_len).astype(np.int32)
    qo = (np.arange(B + 1) * q_len).astype(np.int32)
    max_pages = 150
    rc, buf, slots, _ = plan(qo, kv, 128, PAGE, max_pages, splits=splits)
    assert rc == native.OK
    check_plan(qo, kv, 128, buf, slots)
    it, row_off = items_of(buf)
    s = min(splits, max_pages * PAGE // 32)
    want = set()
    for b in range(B):
        tp = -(-int(tiles(kv[b])) // s)
        for i in range(q_len):
            lim = kv[b] - q_len + i + 1
            for k in range(s):
                if k * tp < tiles(lim):
                    for g in range(2):
                        want.add((b * q_len + i, b, g, k * tp, min(int(tiles(lim)), (k + 1) * tp), lim, row_off[b * q_len + i] + k))
    assert set(map(tuple, it.tolist())) == want


def test_planner_sequences_without_queries():
    qo = np.array([0, 0, 3, 3, 4, 4], np.int32)
    kv = np.array([500, 3, 0, 900, 77], np.int32)
    rc, buf, slots, _ = plan(qo, kv, 16, PAGE, 20)
    assert rc == native.OK
    check_plan(qo, kv, 16, buf, slots)
    it, _ = items_of(buf)
    assert set(it[:, 1].tolist()) == {1, 3}
    rc, buf, slots, _ = plan(np.zeros(1, np.int32), np.zeros(0, np.int32), 16, PAGE, 20)
    assert rc == native.OK and buf[0] == buf[1] == slots == 0


@pytest.mark.parametrize("case,msg", [
    (dict(qo=[0, 2, 1]), "monotone"), (dict(qo=[1, 2, 3]), "qo_indptr[0]"), (dict(kv=[1, 5]), "shorter than its q_len"),
    (dict(kv=[-1, 5]), "shorter"), (dict(kv=[3, 64 * 10 + 1]), "exceeds max_pages_per_seq"), (dict(max_rows=2), "row capacity"),
    (dict(max_items=3), "item capacity"), (dict(plan_ints=10), "too small"), (dict(splits=129), "num_kv_splits"),
    (dict(page=48), "page_size"), (dict(H=0), "num_heads"), (dict(max_pages=0), "max_pages"), (dict(num_sms=0), "num_sms"),
    (dict(max_items=0), "capacity"),
])
def test_planner_refusals(case, msg):
    a = dict(qo=[0, 2, 3], kv=[100, 5], H=128, page=64, max_pages=10, num_sms=132, splits=0, max_items=1000, max_rows=64, plan_ints=None)
    a.update(case)
    rc, buf, *_ = plan(a.pop("qo"), a.pop("kv"), a.pop("H"), a.pop("page"), a.pop("max_pages"), **a)
    assert rc == native.EINVAL and msg in native.lib().ktb200_last_error().decode()
    assert not buf.any(), "a refused plan writes nothing"


def test_planner_refuses_null_pointers():
    lib = native.lib()
    kv = np.array([3], np.int32)
    buf = np.zeros(100, np.int32)
    assert lib.ktb200_mla_ragged_plan(None, kv.ctypes.data, 1, 16, 64, 1, 132, 0, 4, 4, buf.ctypes.data, 100, None, None) == native.EINVAL
    assert "null" in lib.ktb200_last_error().decode()


def _ragged_params(**over):
    a = dict(rows=4, max_items=64, H=128, page=64, max_pages=4, q_nope=1 << 20, q_pe=2 << 20, kv=3 << 20, pt=4 << 20, plan=5 << 20,
             out=6 << 20, lse=None, ws=7 << 20, ws_bytes=1 << 40, kv_rows=0)
    a.update(over)
    v = list(a.values())
    return native.MlaRaggedParams(v[0], v[1], v[2], v[3], v[4], SCALE, *v[5:])


@pytest.mark.parametrize("over,msg", [
    (dict(q_nope=None), "null"), (dict(q_pe=None), "null"), (dict(kv=None), "null"), (dict(pt=None), "null"), (dict(plan=None), "null"),
    (dict(out=None), "null"), (dict(ws=None), "null"), (dict(max_items=0), "capacity"), (dict(rows=-1), "rows"),
    (dict(page=48), "page_size"), (dict(H=0), "num_heads"), (dict(max_pages=0), "max_pages"),
    (dict(q_nope=(1 << 20) + 8), "aligned"), (dict(kv=(3 << 20) + 4), "aligned"), (dict(plan=(5 << 20) + 4), "aligned"),
    (dict(ws_bytes=32 * 128 * 513 * 4 - 4), "workspace"), (dict(rows=1 << 25), "too large"),
])
def test_run_refusals(over, msg):
    lib = native.lib()
    p = _ragged_params(**over)
    assert lib.ktb200_mla_decode_ragged(C.byref(p), None) == native.EINVAL
    assert msg in lib.ktb200_last_error().decode()
    assert lib.ktb200_mla_decode_ragged(None, None) == native.EINVAL


def test_workspace_and_plan_sizes():
    lib = native.lib()
    assert lib.ktb200_mla_ragged_workspace_bytes(64, 128) == 32 * 128 * 513 * 4
    assert lib.ktb200_mla_ragged_workspace_bytes(64, 16) == 64 * 16 * 513 * 4
    assert lib.ktb200_mla_ragged_workspace_bytes(0, 16) == lib.ktb200_mla_ragged_workspace_bytes(4, 0) == 0
    assert lib.ktb200_mla_ragged_plan_ints(10, 3) == 8 + 80 + 4 and lib.ktb200_mla_ragged_plan_ints(0, 3) == 0


def test_wrapper_plans_uniform_q_len_on_the_old_path():
    from ktransformers_b200.operators.flashinfer_wrapper import MLAWrapper
    w = MLAWrapper(3, 30, device="cpu", max_rows=16, max_items=64)
    args = (torch.arange(4, dtype=torch.int32) * 10, torch.arange(30, dtype=torch.int32), torch.tensor([5, 70, 300], dtype=torch.int32), None,
            128, 512, 64, PAGE, SCALE, torch.bfloat16, torch.bfloat16)
    for qo in (None, torch.arange(4, dtype=torch.int32)):
        w.plan(qo, *args)
        assert not w.ragged and w.q_len == 1 and w.plan_host is None
    w.plan(torch.tensor([0, 1, 4, 5], dtype=torch.int32), *args)
    assert w.ragged and w.rows == 5 and w.q_len == 0
    rc, buf, _, _ = plan([0, 1, 4, 5], [5, 70, 300], 128, PAGE, 30, max_items=64, max_rows=16)
    n = 8 + 8 * int(buf[0])
    assert np.array_equal(w.plan_dev[:n].numpy(), buf[:n]) and np.array_equal(w.plan_dev[8 + 8 * 64:].numpy()[:6], buf[8 + 8 * 64:][:6])
    w.plan(torch.arange(4, dtype=torch.int32), *args)
    assert not w.ragged and w.q_len == 1


# ------------------------------------------------------------------------------------------------ GPU helpers
@pytest.fixture(scope="module")
def pool():
    g = torch.Generator(device="cuda").manual_seed(1)
    kv = torch.randn((POOL_ROWS, 576), generator=g, device="cuda").to(torch.bfloat16)
    return kv.view(-1, PAGE, 576), kv.float().cpu().numpy().reshape(-1, PAGE, 576)


def ragged(q_nope, q_pe, kv, pt, qo, kv_len, splits=0, max_items=1 << 14, rows=None, lse_fill=None):
    """plan on the host, copy, ktb200_mla_decode_ragged -> (out [R, H, 512], lse [R, H], host plan)"""
    lib = native.lib()
    R, H = q_nope.shape[:2]
    rows = R if rows is None else rows
    rc, buf, slots, _ = plan(qo, kv_len, H, kv.shape[1], pt.shape[1], sms(), splits, max_items, max(rows, 1))
    assert rc == native.OK, lib.ktb200_last_error()
    plan_d = torch.from_numpy(buf).cuda()
    pt_d = torch.from_numpy(np.ascontiguousarray(pt, np.int32)).cuda()
    out = torch.full((rows, H, 512), float("nan"), dtype=torch.bfloat16, device="cuda")
    lse = torch.full((rows, H), float("nan"), device="cuda")
    ws_bytes = lib.ktb200_mla_ragged_workspace_bytes(max_items, H)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    p = native.MlaRaggedParams(rows, max_items, H, kv.shape[1], pt.shape[1], SCALE, q_nope.data_ptr(), q_pe.data_ptr(), kv.data_ptr(),
                               pt_d.data_ptr(), plan_d.data_ptr(), out.data_ptr(), lse.data_ptr(), ws.data_ptr(), ws_bytes, 0)
    native.check(lib.ktb200_mla_decode_ragged(C.byref(p), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out, lse, buf


def flat_queries(R, H, seed):
    qn, qp = queries(1, R, H, seed)
    return qn[0].contiguous(), qp[0].contiguous()


def check_flat(family, case, out, lse, qn, qp, host, pt, qo, kv_len, rows, heads):
    """sampled flat rows against mla_decode at each row's own length"""
    seq, lim = row_limits(qo, kv_len)
    rows = np.asarray(rows)
    hs = torch.as_tensor(heads, device="cuda")
    pick = lambda t: t[torch.as_tensor(rows, device="cuda")].index_select(1, hs).float().cpu().numpy()
    a, b = pick(qn), pick(qp)
    want, want_lse = mla_oracle.mla_decode(a, b, host, pt[seq[rows]], lim[rows].astype(np.int32), SCALE, p_bf16=True)
    exact, _ = mla_oracle.mla_decode(a, b, host, pt[seq[rows]], lim[rows].astype(np.int32), SCALE, p_bf16=False)
    check_decode(family, case, pick(out), pick(lse), want, want_lse, exact)


def sample_flat(rng, qo):
    rows = []
    for b in range(len(qo) - 1):
        q = qo[b + 1] - qo[b]
        if q:
            ii = boundary_rows(q, rng, extra=2) if q <= 300 else np.unique(np.r_[0, 1, 63, 64, q - 1, rng.integers(0, q, 6)])
            rows += (qo[b] + ii).tolist()
    return rows


# ------------------------------------------------------------------------------------------------ against the oracle (GPU)
@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 16])
@pytest.mark.parametrize("past", [0, 1, 63, 4095, 32768, 131072])
def test_mixed_batch_vs_oracle(pool, past, H):
    """7 decode rows at 33..30000 tokens and a prompt chunk after `past` cached tokens (placed third), permuted pages"""
    kv, host = pool
    rng = np.random.default_rng(past + H)
    chunk_q = 8 if past == 131072 else 40
    q = [1, 1, chunk_q, 1, 1, 1, 1, 1]
    kv_len = np.array([33, 4096, past + chunk_q, 1, 30000, 64, 65, 12345], np.int32)
    qo = np.r_[0, np.cumsum(q)].astype(np.int32)
    width = -(-int(kv_len.max()) // PAGE)
    pt = random_pages(rng, kv.shape[0], len(q), width)
    qn, qp = flat_queries(int(qo[-1]), H, past + H)
    out, lse, _ = ragged(qn, qp, kv, pt, qo, kv_len)
    check_flat("ragged mixed", f"P={past} H={H}", out, lse, qn, qp, host, pt, qo, kv_len, sample_flat(rng, qo),
               boundary_rows(H, rng, extra=2) if H > 16 else np.arange(H))


@pytest.mark.gpu
def test_empty_sequences(pool):
    """q_len 0 sequences between others produce no rows; the rows past the plan's rows are zeros with lse -inf"""
    kv, host = pool
    rng = np.random.default_rng(5)
    qo = np.array([0, 0, 3, 3, 4, 4], np.int32)
    kv_len = np.array([500, 700, 0, 900, 77], np.int32)
    pt = random_pages(rng, kv.shape[0], 5, 16)
    qn, qp = flat_queries(6, 128, 5)
    out, lse, _ = ragged(qn, qp, kv, pt, qo, kv_len)
    check_flat("ragged empty", "q_len 0 sequences", out[:4], lse[:4], qn[:4], qp[:4], host, pt, qo, kv_len, [0, 1, 2, 3], np.arange(0, 128, 9))
    assert not out[4:].float().any() and torch.isneginf(lse[4:]).all()


@pytest.mark.gpu
def test_skewed_decode_batch(pool):
    """one sequence at 131072 tokens and 65 at 1024, automatic plan"""
    kv, host = pool
    rng = np.random.default_rng(66)
    kv_len = np.array([131072] + [1024] * 65, np.int32)
    qo = np.arange(67, dtype=np.int32)
    pt = np.concatenate([random_pages(rng, kv.shape[0], 1, 2048), random_pages(rng, kv.shape[0], 65, 2048)[:, :2048]])
    qn, qp = flat_queries(66, 128, 66)
    out, lse, buf = ragged(qn, qp, kv, pt, qo, kv_len)
    check_flat("ragged skewed", f"items={buf[0]}", out, lse, qn, qp, host, pt, qo, kv_len, [0, 1, 2, 33, 64, 65], np.array([0, 63, 64, 127]))


# ------------------------------------------------------------------------------------------------ exact properties (GPU)
@pytest.mark.gpu
@pytest.mark.parametrize("B,q_len,H,splits", [(1, 16, 128, 7), (3, 40, 128, 2), (2, 5, 16, 128), (4, 24, 40, 5)])
def test_uniform_batch_equals_the_chunk_entry(pool, B, q_len, H, splits):
    kv, _ = pool
    rng = np.random.default_rng(B + q_len + H)
    kl = (rng.integers(0, 9000, B) + q_len).astype(np.int32)
    pt = random_pages(rng, kv.shape[0], B, 150)
    q_nope, q_pe = queries(B, q_len, H, B + H)
    c_out, c_lse, _ = chunk(q_nope, q_pe, kv, pt, kl, splits=splits, ws_splits=MAX_SPLITS)
    qo = (np.arange(B + 1) * q_len).astype(np.int32)
    out, lse, _ = ragged(q_nope.reshape(B * q_len, H, 512), q_pe.reshape(B * q_len, H, 64), kv, pt, qo, kl, splits=splits)
    assert torch.equal(out.view(torch.int16), c_out.reshape(B * q_len, H, 512).view(torch.int16))
    assert torch.equal(lse, c_lse.reshape(B * q_len, H))


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,splits", [(1, 128, 9), (5, 16, 3), (3, 128, 1), (2, 40, 128)])
def test_decode_batch_equals_decode(pool, B, H, splits):
    kv, _ = pool
    rng = np.random.default_rng(B * H + splits)
    kl = rng.integers(1, 30000, B).astype(np.int32)
    kl[0] = 33
    pt = random_pages(rng, kv.shape[0], B, 480)
    qn, qp = flat_queries(B, H, B + H)
    d_out, d_lse = _decode(qn, qp, kv, pt, kl, splits)
    out, lse, _ = ragged(qn, qp, kv, pt, np.arange(B + 1, dtype=np.int32), kl, splits=splits)
    assert torch.equal(out.view(torch.int16), d_out.view(torch.int16)) and torch.equal(lse, d_lse)


def _private_cache(pool, n_pages):
    kv, _ = pool
    return kv[:n_pages].clone()


@pytest.mark.gpu
def test_ragged_is_causal(pool):
    """a chunk of 64 after 100 tokens between two decode rows: rows of its cache at positions >= P + k overwritten (NaN and
    large values) leave its queries i < k and the other sequences bit-identical"""
    rng = np.random.default_rng(7)
    cache = _private_cache(pool, 40)
    pt = rng.permutation(40)[:30].reshape(3, 10).astype(np.int32)
    qo = np.array([0, 1, 65, 66], np.int32)
    kl = np.array([300, 164, 500], np.int32)
    qn, qp = flat_queries(66, 128, 7)
    base, base_lse, _ = ragged(qn, qp, cache, pt, qo, kl)
    for k in (1, 28, 63):
        rows = [(int(pt[1, t // PAGE]), t % PAGE) for t in range(100 + k, 164)]
        saved = [cache[a, b].clone() for a, b in rows]
        for t, (a, b) in zip(range(100 + k, 164), rows):
            cache[a, b] = float("nan") if t % 2 else 300.0
        out, lse, _ = ragged(qn, qp, cache, pt, qo, kl)
        for (a, b), s in zip(rows, saved):
            cache[a, b] = s
        keep = list(range(0, 1 + k)) + [65]
        assert torch.equal(out[keep].view(torch.int16), base[keep].view(torch.int16)) and torch.equal(lse[keep], base_lse[keep]), k
        assert not torch.equal(out[1 + k:65].view(torch.int16), base[1 + k:65].view(torch.int16)), k


@pytest.mark.gpu
def test_ragged_reads_nothing_past_the_limits(pool):
    """NaN / Inf past every sequence's kv_len and in every page no table names: bit-identical output"""
    rng = np.random.default_rng(8)
    cache = _private_cache(pool, 120)
    pt = rng.permutation(120)[:100].reshape(4, 25).astype(np.int32)
    qo = np.array([0, 1, 38, 39, 139], np.int32)
    kl = np.array([1000, 37, 1537, 100], np.int32)
    qn, qp = flat_queries(139, 128, 8)
    base, base_lse, _ = ragged(qn, qp, cache, pt, qo, kl)
    named = set()
    for b in range(4):
        named |= set(pt[b, : -(-kl[b] // PAGE)].tolist())
        last = cache[int(pt[b, (kl[b] - 1) // PAGE])]
        last[kl[b] % PAGE or PAGE:: 2] = float("nan")
        last[(kl[b] % PAGE or PAGE) + 1:: 2] = -float("inf")
    for i in range(cache.shape[0]):
        if i not in named:
            cache[i] = float("nan") if i % 2 else float("inf")
    out, lse, _ = ragged(qn, qp, cache, pt, qo, kl)
    assert torch.equal(out.view(torch.int16), base.view(torch.int16)) and torch.equal(lse, base_lse)
    assert torch.isfinite(out.float()).all()


@pytest.mark.gpu
def test_graph_replays_after_re_plans(pool):
    """MLAWrapper: one run captured at 200 rows, then three plans of other batch compositions; each replay equals the eager
    run of the same plan bit for bit, and its padded rows are zeros"""
    from ktransformers_b200.operators.flashinfer_wrapper import MLAWrapper
    kv, host = pool
    rng = np.random.default_rng(9)
    B, pages, R = 6, 200, 200
    w = MLAWrapper(B, pages, max_rows=R, max_items=2048)
    pt = random_pages(rng, kv.shape[0], B, pages)
    indptr = torch.arange(0, B + 1, dtype=torch.int32, device="cuda") * pages
    indices = torch.from_numpy(pt.reshape(-1)).cuda()
    ckv, kpe = kv[..., :512], kv[..., 512:]
    qn, qp = flat_queries(R, 128, 9)

    def do_plan(q, kl):
        w.plan(torch.from_numpy(np.r_[0, np.cumsum(q)].astype(np.int32)), indptr, indices, torch.tensor(kl, dtype=torch.int32), None,
               128, 512, 64, PAGE, SCALE, torch.bfloat16, torch.bfloat16)

    do_plan([1, 2, 3, 4, 5, 6], [10, 20, 30, 40, 50, 60])
    w.run(qn, qp, ckv, kpe, return_lse=True)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_out, g_lse = w.run(qn, qp, ckv, kpe, return_lse=True)
    for q, kl in (([1, 1, 150, 1, 0, 1], [12800, 3, 150, 9000, 0, 1]), ([40, 1, 1, 1, 1, 1], [4000, 5000, 6000, 7000, 8000, 12000]),
                  ([0, 0, 200, 0, 0, 0], [0, 0, 12000, 0, 0, 0])):
        do_plan(q, kl)
        graph.replay()
        torch.cuda.synchronize()
        r_out, r_lse = g_out.clone(), g_lse.clone()
        e_out, e_lse = w.run(qn, qp, ckv, kpe, return_lse=True)
        torch.cuda.synchronize()
        assert torch.equal(r_out.view(torch.int16), e_out.view(torch.int16)) and torch.equal(r_lse, e_lse), q
        n = sum(q)
        assert not r_out[n:].float().any() and torch.isneginf(r_lse[n:]).all()
        qo = np.r_[0, np.cumsum(q)].astype(np.int32)
        check_flat("ragged graph", f"q={q}", r_out[:n], r_lse[:n], qn[:n], qp[:n], host, pt, qo, np.array(kl, np.int32),
                   sample_flat(rng, qo)[:12], np.array([0, 63, 64, 127]))


# ------------------------------------------------------------------------------------------------ operator (GPU)
@pytest.mark.gpu
def test_operator_mixed_steps_match_each_sequence_alone():
    """four sequences through forward_ragged on one cache (rows permuted): history of 126 / 1000 / 500 / 0 tokens, then a
    step with two decoding sequences, a 200-token chunk of the third and a new 150-token prompt, then three mixed steps (the
    first sequence crosses the page boundary at 128).  Each sequence's outputs against it run alone through forward
    (absorbed, bsz 1) and against the float64 module, within the operator bar; run makes no host synchronisation."""
    from ktransformers_b200.models.custom_cache import StaticCache
    from ktransformers_b200.operators import attention as attn_mod
    from ktransformers_b200.operators.attention import KDeepseekV2Attention
    cfg, plain, _ = _modules(128, 77)
    op = KDeepseekV2Attention("blk.0.self_attn", None, cfg, plain, "cuda", "cuda", absorb_for_prefill=True)
    attn_mod._RAGGED_WRAPPERS.clear()
    plain64 = copy.deepcopy(plain).double()
    cache = StaticCache(cfg, max_batch_size=4, max_cache_len=1536, device="cuda")
    cache_rows = [2, 0, 3, 1]
    steps = [[126, 1000, 500, 0], [1, 1, 200, 150], [1, 1, 1, 7], [1, 1, 3, 1], [1, 1, 1, 1]]
    total = np.sum(steps, 0)
    xs = [(torch.randn(int(n), 1024, device="cuda") * 2).to(torch.bfloat16) for n in total]
    got = [[] for _ in range(4)]
    done = np.zeros(4, np.int64)
    for k, q in enumerate(steps):
        q = np.array(q)
        x = torch.cat([xs[b][done[b]:done[b] + q[b]] for b in range(4)])
        pos = torch.cat([torch.arange(done[b], done[b] + q[b], device="cuda") for b in range(4)])
        qo = torch.from_numpy(np.r_[0, np.cumsum(q)].astype(np.int32))
        kv_len = torch.from_numpy((done + q).astype(np.int32))
        out = op.forward_ragged(x, pos, qo, kv_len, torch.tensor(cache_rows, dtype=torch.int32), cache, max_rows=2048, max_items=8192)
        for b in range(4):
            got[b].append(out[qo[b]:qo[b + 1]])
        done += q
        if k == 1:   # run alone makes no host synchronisation
            w = next(iter(attn_mod._RAGGED_WRAPPERS.values()))
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                w.run(torch.zeros(int(q.sum()), 128, 512, dtype=torch.bfloat16, device="cuda"),
                      torch.zeros(int(q.sum()), 128, 64, dtype=torch.bfloat16, device="cuda"),
                      cache.key_cache[0][..., :512].view(-1, PAGE, 512), cache.key_cache[0][..., 512:].view(-1, PAGE, 64))
            finally:
                torch.cuda.set_sync_debug_mode("default")
    assert cache.get_seq_length(0) == 0, "forward_ragged leaves the host counter alone"
    worst_alone = worst64 = 0.0
    for b in range(4):
        g = torch.cat(got[b])
        alone_cache = StaticCache(cfg, max_batch_size=1, max_cache_len=1536, device="cuda")
        alone, start = [], 0
        for q in np.array(steps)[:, b]:
            if q:
                o, _, _ = op(xs[b][None, start:start + q], position_ids=torch.arange(start, start + q, device="cuda")[None],
                             past_key_value=alone_cache, cache_position=torch.arange(start, start + q, device="cuda"))
                alone.append(o[0])
            start += q
        alone = torch.cat(alone)
        want, _ = plain64(xs[b][None].double(), torch.arange(int(total[b]), device="cuda")[None])
        worst_alone, worst64 = max(worst_alone, _rel(g, alone)), max(worst64, _rel(g, want[0]))
    print(f"[operator ragged] {worst_alone / 4e-2:.3f} of the bound vs alone, {worst64 / 4e-2:.3f} vs float64")
    assert worst_alone < 4e-2 and worst64 < 4e-2, (worst_alone, worst64)
