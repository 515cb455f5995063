"""MLA decode (csrc/mla.cu) and causal MLA prefill (csrc/mla_prefill.cu) at the lengths and batches DeepSeek-V3/R1 serves.

Decode: single sequences up to 131072 tokens (64 to 66 auto splits on a 132-SM H100, up to 63 tiles of 32 tokens per CTA, so
the 4-stage ring wraps many times), explicit split counts 1..128 (1024 tiles through one CTA at 1 split), batches up to 130
with lengths 0..16384 (one split per sequence from 66 sequences of 128 heads), 16 and 40 heads; bit-exact properties: the
physical page placement, batch independence, nothing past kv_len is read, CUDA-graph replays at a 128K-token capacity.
Prefill: prompts up to 8192 tokens and chunks after up to 32767 cached tokens, causality, and KDeepseekV2Attention through a
2108-token prompt in chunks of 700 / 700 / 708 and decode steps across a page boundary.

The float64 oracles (oracle/mla_oracle.py, tests/mla_prefill_oracle.py) run on sampled heads and query rows: every output
row depends only on its own query, so the restriction is the same computation on fewer rows (pinned on the CPU below).
Tolerances are those of test_mla_decode_vs_oracle and test_prefill_kernel_vs_oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

import mla_prefill_oracle as mpo
from ktransformers_b200 import native
from oracle import mla_oracle
from test_mla_prefill import SCALE, _Case, _modules, _rel, _step
H100_SMS = 132
MAX_SPLITS = 128                 # kMaxSplits in csrc/mla.cu
POOL_ROWS = 131072 + 512         # the shared decode cache: 2056 pages of 64 (514 of 256, 4112 of 32)


# ------------------------------------------------------------------------------------------------ helpers
def pick_splits(batch, num_heads, max_kv_tiles, sms):
    """csrc/mla.cu pick_splits: one CTA per SM over (sequence, 64-head group), at least 4 tiles of 32 tokens per split,
    at most 128 splits"""
    groups = batch * -(-num_heads // 64)
    s = -(-sms // groups)
    s = min(s, -(-max_kv_tiles // 4), MAX_SPLITS)
    return max(s, 1)


def boundary_rows(n, rng, extra=6):
    """the first and last row, both sides of every 64-row boundary (every 128-row boundary is one of them), random rows"""
    rows = {0, n - 1}
    for b in range(64, n, 64):
        rows |= {b - 1, b}
    rows |= set(rng.integers(0, n, extra).tolist())
    return np.array(sorted(rows))


def decode_oracle(q_nope, q_pe, kv, page_table, kv_len, heads, seqs=None, p_bf16=True):
    """oracle/mla_oracle.mla_decode on the chosen sequences and heads only -> (out [seqs, heads, 512], lse [seqs, heads])"""
    seqs = np.arange(len(kv_len)) if seqs is None else np.asarray(seqs)
    ix = np.ix_(seqs, heads)
    return mla_oracle.mla_decode(q_nope[ix], q_pe[ix], kv, page_table[seqs], kv_len[seqs], SCALE, p_bf16=p_bf16)


def _runs(rows):
    """sorted rows -> lists of consecutive rows"""
    runs, cur = [], [rows[0]]
    for r in rows[1:]:
        if r == cur[-1] + 1:
            cur.append(r)
        else:
            runs.append(cur)
            cur = [r]
    return runs + [cur]


def prefill_oracle(q_nope, q_pe, k_nope, k_pe, v, past, rows, p_bf16=False):
    """tests/mla_prefill_oracle.mla_prefill on the chosen query rows (the arrays may already be restricted to some heads):
    a run of consecutive rows i0..i1-1 with the keys cut at past + i1 is the same bottom-right causal problem, query i at
    position past + i -> out [B, rows, H, 128]"""
    rows = np.asarray(rows)
    out = np.empty((q_nope.shape[0], len(rows), q_nope.shape[2], 128))
    k = 0
    for run in _runs(rows.tolist()):
        i0, i1 = run[0], run[-1] + 1
        S = past + i1
        out[:, k:k + len(run)] = mpo.mla_prefill(q_nope[:, i0:i1], q_pe[:, i0:i1], k_nope[:, :S], k_pe[:, :S], v[:, :S], SCALE, p_bf16)
        k += len(run)
    return out


def _report(family, case, frac):
    print(f"[{family}] {case}: worst error {frac:.3f} of its bound")


def check_decode(family, case, out, lse, want, want_lse, exact):
    """the bounds of test_mla_decode_vs_oracle (out / lse as float32 numpy on the sampled rows)"""
    mag = np.abs(exact).max()
    err_w, err_e = np.abs(out - want), np.abs(out - exact)
    fracs = [err_w.max() / ((2.0 ** -7 + 1e-3) * mag), err_e.max() / (2e-2 * mag),
             err_e.mean() / (5e-3 * np.abs(exact).mean() + 1e-6), np.abs(lse - want_lse).max() / 2e-3]
    _report(family, case, max(fracs))
    assert np.isfinite(out).all()
    assert err_w.max() <= 2.0 ** -7 * mag + 1e-3 * mag
    assert err_e.max() <= 2e-2 * mag
    assert err_e.mean() <= 5e-3 * np.abs(exact).mean() + 1e-6
    np.testing.assert_allclose(lse, want_lse, rtol=0, atol=2e-3)


def bf16_dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(torch.bfloat16).cuda()


def queries(rng, B, H):
    """bf16-valued float32 q_nope [B, H, 512], q_pe [B, H, 64], the scale of tests/test_gpu_parity._mla_case"""
    return (mla_oracle.bf16_round((rng.standard_normal((B, H, 512)) * 0.5).astype(np.float32)),
            mla_oracle.bf16_round((rng.standard_normal((B, H, 64)) * 0.5).astype(np.float32)))


def decode(q_nope, q_pe, kv, page_table, kv_len, splits=0, kv_cache_rows=0, ws_splits=MAX_SPLITS):
    """ktb200_mla_decode with host q (float32 bf16 values), page table and lengths, and the device cache kv [pages, page, 576]
    -> (out float32 [B, H, 512], lse [B, H], the number of KV splits the call used).  The workspace starts as NaN: the
    call fills o_part [B][splits][H][512] and then lse_part [B][splits][H], so the count of written floats gives the
    split count."""
    lib = native.lib()
    B, H = q_nope.shape[:2]
    qn, qp = bf16_dev(q_nope), bf16_dev(q_pe)
    pt = torch.from_numpy(np.ascontiguousarray(page_table, np.int32)).cuda()
    kl = torch.from_numpy(np.ascontiguousarray(kv_len, np.int32)).cuda()
    out = torch.empty((B, H, 512), dtype=torch.bfloat16, device="cuda")
    lse = torch.empty((B, H), dtype=torch.float32, device="cuda")
    ws_bytes = lib.ktb200_mla_workspace_bytes(B, H, ws_splits)
    ws = torch.full((ws_bytes // 4,), float("nan"), dtype=torch.float32, device="cuda")
    p = native.MlaParams(B, H, kv.shape[1], page_table.shape[1], splits, SCALE, qn.data_ptr(), qp.data_ptr(), kv.data_ptr(),
                         pt.data_ptr(), kl.data_ptr(), out.data_ptr(), lse.data_ptr(), ws.data_ptr(), ws_bytes, kv_cache_rows)
    native.check(lib.ktb200_mla_decode(C.byref(p), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    written = int((~torch.isnan(ws)).sum())
    per_split = B * H * 513
    assert written % per_split == 0 and not torch.isnan(ws[:written]).any(), written
    return out.float().cpu().numpy(), lse.cpu().numpy(), written // per_split


def sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.fixture(scope="module")
def pool():
    """one bf16 latent cache of POOL_ROWS token rows on the device and its float32 copy on the host, viewed at any page size"""
    g = torch.Generator(device="cuda").manual_seed(0)
    kv = torch.randn((POOL_ROWS, 576), generator=g, device="cuda").to(torch.bfloat16)
    return kv, kv.float().cpu().numpy()


def paged(pool, page):
    kv, host = pool
    return kv.view(-1, page, 576), host.reshape(-1, page, 576)


# ------------------------------------------------------------------------------------------------ CPU
LONG = [(8191, 64), (8192, 64), (8193, 65), (32768 + 17, 66), (131072, 66)]


@pytest.mark.parametrize("L,want", LONG)
def test_pick_splits_at_serving_lengths_on_132_sms(L, want):
    """the split counts the long-sequence cases below run with on an H100 (H = 128, pages of 64, capacity = L rounded up)"""
    assert pick_splits(1, 128, -(-L // 64) * 2, H100_SMS) == want


@pytest.mark.parametrize("B,want", [(8, 9), (64, 2), (66, 1), (130, 1)])
def test_pick_splits_for_large_batches_on_132_sms(B, want):
    assert pick_splits(B, 128, 16384 // 32, H100_SMS) == want


def test_sampled_decode_oracle_equals_full_oracle():
    rng = np.random.default_rng(1)
    B, H, page, L = 3, 128, 32, 200
    kv = mla_oracle.bf16_round(rng.standard_normal((3 * 7, page, 576)).astype(np.float32))
    pt = rng.permutation(3 * 7).reshape(3, 7).astype(np.int32)
    kl = np.array([L, 1, 150], np.int32)
    q_nope, q_pe = queries(rng, B, H)
    heads, seqs = boundary_rows(H, rng), np.array([0, 2])
    for p_bf16 in (True, False):
        full, full_lse = mla_oracle.mla_decode(q_nope, q_pe, kv, pt, kl, SCALE, p_bf16=p_bf16)
        got, got_lse = decode_oracle(q_nope, q_pe, kv, pt, kl, heads, seqs, p_bf16=p_bf16)
        np.testing.assert_allclose(got, full[np.ix_(seqs, heads)], rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(got_lse, full_lse[np.ix_(seqs, heads)], rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("past,q_len", [(0, 300), (70, 200)])
def test_sampled_prefill_oracle_equals_full_oracle(past, q_len):
    rng = np.random.default_rng(q_len)
    B, H, S = 2, 3, past + q_len
    q_nope, q_pe = rng.standard_normal((B, q_len, H, 128)), rng.standard_normal((B, q_len, H, 64))
    k_nope, k_pe, v = rng.standard_normal((B, S, H, 128)), rng.standard_normal((B, S, 64)), rng.standard_normal((B, S, H, 128))
    rows = boundary_rows(q_len, rng)
    assert {0, 63, 64, 127, 128, q_len - 1} <= set(rows.tolist())
    for p_bf16 in (False, True):
        full = mpo.mla_prefill(q_nope, q_pe, k_nope, k_pe, v, SCALE, p_bf16)
        got = prefill_oracle(q_nope, q_pe, k_nope, k_pe, v, past, rows, p_bf16)
        np.testing.assert_allclose(got, full[:, rows], rtol=0, atol=1e-12 * np.abs(full).max())


# ------------------------------------------------------------------------------------------------ decode (GPU)
@pytest.mark.gpu
@pytest.mark.parametrize("L,want", LONG)
def test_decode_long_sequence_vs_oracle(pool, L, want):
    """one sequence of 128 heads at a serving length, auto splits, its pages scattered over the pool"""
    kv, host = paged(pool, 64)
    rng = np.random.default_rng(L)
    pages = -(-L // 64)
    pt = rng.permutation(kv.shape[0])[:pages].reshape(1, pages)
    kl = np.array([L], np.int32)
    q_nope, q_pe = queries(rng, 1, 128)
    out, lse, used = decode(q_nope, q_pe, kv, pt, kl)
    assert used == pick_splits(1, 128, pages * 2, sms())
    if sms() == H100_SMS:
        assert used == want
    heads = boundary_rows(128, rng)
    want_o, want_lse = decode_oracle(q_nope, q_pe, host, pt, kl, heads)
    exact, _ = decode_oracle(q_nope, q_pe, host, pt, kl, heads, p_bf16=False)
    check_decode("decode long", f"L={L} splits={used}", out[:, heads], lse[:, heads], want_o, want_lse, exact)


@pytest.fixture(scope="module")
def seq32k(pool):
    kv, host = paged(pool, 64)
    rng = np.random.default_rng(32768)
    pt = rng.permutation(kv.shape[0])[:512].reshape(1, 512)
    kl = np.array([32768], np.int32)
    q_nope, q_pe = queries(rng, 1, 128)
    heads = boundary_rows(128, rng)
    want = decode_oracle(q_nope, q_pe, host, pt, kl, heads)
    exact, _ = decode_oracle(q_nope, q_pe, host, pt, kl, heads, p_bf16=False)
    return kv, q_nope, q_pe, pt, kl, heads, want, exact


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [1, 2, 65, 127, 128])
def test_decode_explicit_splits_at_32k(seq32k, splits):
    """1 split: 1024 tiles through one CTA; 128: the most the merge takes"""
    kv, q_nope, q_pe, pt, kl, heads, (want, want_lse), exact = seq32k
    out, lse, used = decode(q_nope, q_pe, kv, pt, kl, splits=splits)
    assert used == splits
    check_decode("decode explicit splits", f"L=32768 splits={splits}", out[:, heads], lse[:, heads], want, want_lse, exact)


def _batch(rng, B, capacity, n_pool_pages, page=64):
    """B sequences with lengths mixed from 0 to the capacity (the edges 0, 1, 31, 32, 33, page - 1, page + 1 and the
    capacity itself among them), each with its own random pages of the pool (sequences may share pages: the cache is
    only read)"""
    edges = [0, 1, 31, 32, 33, page - 1, page + 1, capacity]
    lens = np.array((edges + rng.integers(0, capacity + 1, max(B - len(edges), 0)).tolist())[:B], np.int32)
    lens = rng.permutation(lens).astype(np.int32)
    width = capacity // page
    pt = np.stack([rng.choice(n_pool_pages, width, replace=False) for _ in range(B)]).astype(np.int32)
    return pt, lens


@pytest.mark.gpu
@pytest.mark.parametrize("B", [8, 64, 66, 130])
def test_decode_large_batch_vs_oracle(pool, B):
    """128 heads, lengths 0..16384: from 66 sequences on, one split (one CTA streams a whole sequence)"""
    kv, host = paged(pool, 64)
    rng = np.random.default_rng(B)
    pt, kl = _batch(rng, B, 16384, kv.shape[0])
    q_nope, q_pe = queries(rng, B, 128)
    out, lse, used = decode(q_nope, q_pe, kv, pt, kl, ws_splits=16)
    assert used == pick_splits(B, 128, 16384 // 32, sms())
    if sms() == H100_SMS and B >= 66:
        assert used == 1
    empty = kl == 0
    assert empty.any() and not out[empty].any() and np.isneginf(lse[empty]).all()
    seqs = np.flatnonzero(~empty)
    heads = boundary_rows(128, rng, extra=2)
    want, want_lse = decode_oracle(q_nope, q_pe, host, pt, kl, heads, seqs)
    exact, _ = decode_oracle(q_nope, q_pe, host, pt, kl, heads, seqs, p_bf16=False)
    ix = np.ix_(seqs, heads)
    check_decode("decode large batch", f"B={B} splits={used}", out[ix], lse[ix], want, want_lse, exact)


@pytest.mark.gpu
@pytest.mark.parametrize("H,page,L", [(16, 32, 24577), (40, 256, 30001)])
def test_decode_heads_not_a_multiple_of_64(pool, H, page, L):
    """one partial head group at a long length (auto splits reach the 128 cap)"""
    kv, host = paged(pool, page)
    rng = np.random.default_rng(H + L)
    pages = -(-L // page)
    pt = rng.permutation(kv.shape[0])[:pages].reshape(1, pages)
    kl = np.array([L], np.int32)
    q_nope, q_pe = queries(rng, 1, H)
    out, lse, used = decode(q_nope, q_pe, kv, pt, kl)
    assert used == pick_splits(1, H, pages * (page // 32), sms())
    heads = np.arange(H)
    want, want_lse = decode_oracle(q_nope, q_pe, host, pt, kl, heads)
    exact, _ = decode_oracle(q_nope, q_pe, host, pt, kl, heads, p_bf16=False)
    check_decode("decode partial head group", f"H={H} page={page} L={L} splits={used}", out, lse, want, want_lse, exact)


# ------------------------------------------------------------------------------------------------ decode properties (GPU)
@pytest.mark.gpu
def test_decode_page_placement_is_invisible():
    """the same 20000-token sequence on pages 0..312 in order and on a permutation of the 313 highest page ids of a
    4096-page cache (NaN everywhere else), kv_cache_rows the exact allocation: bit-identical"""
    L, page, n_pages = 20000, 64, 4096
    pages = -(-L // page)
    rng = np.random.default_rng(3)
    g = torch.Generator(device="cuda").manual_seed(3)
    content = torch.randn((pages, page, 576), generator=g, device="cuda").to(torch.bfloat16)
    q_nope, q_pe = queries(rng, 1, 128)
    kl = np.array([L], np.int32)
    results = []
    for ids in (np.arange(pages), rng.permutation(np.arange(n_pages - pages, n_pages))):
        assert ids.max() <= n_pages - 1
        cache = torch.full((n_pages, page, 576), float("nan"), dtype=torch.bfloat16, device="cuda")
        cache[torch.from_numpy(ids).long().cuda()] = content
        for rows in (n_pages * page, 0):
            results.append(decode(q_nope, q_pe, cache, ids.reshape(1, -1), kl, kv_cache_rows=rows))
        del cache
    assert (n_pages - 1) in ids
    for out, lse, used in results[1:]:
        assert used == results[0][2]
        assert np.array_equal(out, results[0][0]) and np.array_equal(lse, results[0][1])
    assert np.isfinite(results[0][0]).all()


@pytest.mark.gpu
def test_decode_batch_independence(pool):
    """num_kv_splits fixed and the same page-table width: sequence b of a batch of 64 equals it decoded alone"""
    kv, _ = paged(pool, 64)
    rng = np.random.default_rng(64)
    pt, kl = _batch(rng, 64, 16384, kv.shape[0])
    q_nope, q_pe = queries(rng, 64, 128)
    out, lse, _ = decode(q_nope, q_pe, kv, pt, kl, splits=8, ws_splits=8)
    picks = sorted({0, 1, 31, 63, int(np.argmax(kl)), int(np.argmin(kl)), int(np.flatnonzero(kl == 33)[0])})
    for b in picks:
        o1, l1, _ = decode(q_nope[b:b + 1], q_pe[b:b + 1], kv, pt[b:b + 1], kl[b:b + 1], splits=8, ws_splits=8)
        assert np.array_equal(o1[0], out[b]) and np.array_equal(l1[0], lse[b]), (b, int(kl[b]))


class _Needle:
    """one 5000-token sequence of 128 heads on 100 pages of 64 (capacity 6400; pages 79..99 unused), auto splits.  Every
    head's q_pe[0] is 2, so a key whose k_pe[0] is 512 scores about 74 against at most ~5 for the others: where it is
    read it takes the whole softmax."""
    L, page, width = 5000, 64, 100

    def __init__(self):
        rng = np.random.default_rng(17)
        g = torch.Generator(device="cuda").manual_seed(17)
        self.cache = torch.randn((self.width + 4, self.page, 576), generator=g, device="cuda").to(torch.bfloat16)
        self.pt = rng.permutation(self.width + 4)[: self.width].reshape(1, -1).astype(np.int32)
        self.q_nope, self.q_pe = queries(rng, 1, 128)
        self.q_pe[:, :, 0] = 2.0
        self.kl = np.array([self.L], np.int32)
        self.needle = torch.randn((576,), generator=g, device="cuda").to(torch.bfloat16)
        self.needle[512:] = 0
        self.needle[512] = 512.0

    def row(self, t):
        return self.cache[int(self.pt[0, t // self.page]), t % self.page]

    def run(self):
        return decode(self.q_nope, self.q_pe, self.cache, self.pt, self.kl)


@pytest.mark.gpu
def test_decode_reads_nothing_past_kv_len():
    """a needle key at position kv_len, then NaN / Inf in every row past kv_len and in every unused page: the output and
    LSE stay bit-identical"""
    n = _Needle()
    base_out, base_lse, _ = n.run()
    n.row(n.L).copy_(n.needle)
    out, lse, _ = n.run()
    assert np.array_equal(out, base_out) and np.array_equal(lse, base_lse)
    used_pages = set(n.pt[0, : -(-n.L // n.page)].tolist())
    for i in range(n.cache.shape[0]):
        if i not in used_pages:
            n.cache[i] = float("nan") if i % 2 else float("inf")
    last = n.cache[int(n.pt[0, (n.L - 1) // n.page])]
    last[n.L % n.page:: 2] = float("nan")
    last[n.L % n.page + 1:: 2] = -float("inf")
    out, lse, _ = n.run()
    assert np.array_equal(out, base_out) and np.array_equal(lse, base_lse)


@pytest.mark.gpu
def test_decode_needle_inside_the_length_dominates():
    """the needle at kv_len - 1, at position 0, and at the first token of the last non-empty split: every head's output is
    the needle's latent within bf16"""
    n = _Needle()
    tiles = -(-n.L // 32)
    splits = pick_splits(1, 128, n.width * 2, sms())
    per = -(-tiles // splits)
    first_of_last = ((tiles - 1) // per) * per * 32
    assert 0 < first_of_last < n.L - 1
    want = n.needle[:512].float().cpu().numpy()
    for t in (n.L - 1, 0, first_of_last):
        saved = n.row(t).clone()
        n.row(t).copy_(n.needle)
        out, _, _ = n.run()
        n.row(t).copy_(saved)
        err = np.abs(out[0] - want[None, :])
        _report("decode needle", f"t={t}", float((err / (2.0 ** -7 * np.abs(want) + 1e-6)).max()))
        assert (err <= 2.0 ** -7 * np.abs(want)[None, :] + 1e-6).all(), (t, err.max())


@pytest.mark.gpu
def test_decode_graph_replays_at_128k_capacity(pool):
    """MLAWrapper.run captured once at a 131072-token capacity (66 splits whatever the length), replayed after writing new
    lengths into kv_len_arr_buf: bit-identical to the eager call and within the oracle bounds"""
    from ktransformers_b200.operators.flashinfer_wrapper import MLAWrapper
    kv, host = paged(pool, 64)
    rng = np.random.default_rng(128)
    pages = 2048
    perm = rng.permutation(kv.shape[0])[:pages].astype(np.int32)
    w = MLAWrapper(1, pages)
    w.plan(None, torch.tensor([0, pages], dtype=torch.int32, device="cuda"), torch.from_numpy(perm).cuda(),
           torch.tensor([1], dtype=torch.int32, device="cuda"), None, 128, 512, 64, 64, SCALE, torch.bfloat16, torch.bfloat16)
    ckv, kpe = kv[..., :512], kv[..., 512:]
    q_nope, q_pe = queries(rng, 1, 128)
    qn, qp = bf16_dev(q_nope), bf16_dev(q_pe)
    w.run(qn, qp, ckv, kpe, return_lse=True)     # warm-up outside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_out, g_lse = w.run(qn, qp, ckv, kpe, return_lse=True)
    heads = boundary_rows(128, rng, extra=2)
    pt = perm.reshape(1, -1)
    for L in (1, 33, 4096, 100000):
        w.kv_len_arr_buf[:1].fill_(L)
        graph.replay()
        torch.cuda.synchronize()
        r_out, r_lse = g_out.clone(), g_lse.clone()
        e_out, e_lse = w.run(qn, qp, ckv, kpe, return_lse=True)
        torch.cuda.synchronize()
        assert torch.equal(r_out.view(torch.int16), e_out.view(torch.int16)) and torch.equal(r_lse, e_lse), L
        kl = np.array([L], np.int32)
        want, want_lse = decode_oracle(q_nope, q_pe, host, pt, kl, heads)
        exact, _ = decode_oracle(q_nope, q_pe, host, pt, kl, heads, p_bf16=False)
        check_decode("decode graph replay", f"L={L}", r_out.float().cpu().numpy()[:, heads], r_lse.cpu().numpy()[:, heads],
                     want, want_lse, exact)


# ------------------------------------------------------------------------------------------------ prefill (GPU)
class _Prefill(_Case):
    """test_mla_prefill._Case (the layouts KDeepseekV2Attention passes, its run()) with the operands drawn on the device
    and the oracle on sampled rows and heads"""

    def __init__(self, B, H, past, q_len, seed, spare=8):
        g = torch.Generator(device="cuda").manual_seed(seed)
        rnd = lambda *shape: torch.randn(*shape, generator=g, device="cuda").to(torch.bfloat16)
        S = past + q_len
        self.B, self.H, self.past, self.q_len, self.S = B, H, past, q_len, S
        self.q, self.q_pe = rnd(B, q_len + spare, H, 192), rnd(B, q_len + spare, H, 64)
        self.kv, self.rows = rnd(B, S + spare, H, 256), rnd(B, S + spare, 576)

    def oracle(self, rows, heads, p_bf16=False):
        f = lambda t: t.float().cpu().numpy()
        hs = torch.as_tensor(heads, device="cuda")
        q, q_pe = self.q[:, : self.q_len].index_select(2, hs), self.q_pe[:, : self.q_len].index_select(2, hs)
        kv = self.kv[:, : self.S].index_select(2, hs)
        return prefill_oracle(f(q[..., :128]), f(q_pe), f(kv[..., :128]), f(self.rows[:, : self.S, 512:]), f(kv[..., 128:]),
                              self.past, rows, p_bf16)


@pytest.mark.gpu
@pytest.mark.parametrize("B,past,q_len", [(1, 0, 4096), (1, 0, 8192), (1, 4096, 4096), (1, 16384, 1000), (2, 12345, 777),
                                          (1, 32767, 2)])
def test_prefill_long_vs_oracle(B, past, q_len):
    """128 heads; the bounds of test_prefill_kernel_vs_oracle on sampled rows and heads"""
    c = _Prefill(B, 128, past, q_len, seed=past + q_len + B)
    rng = np.random.default_rng(past + q_len)
    rows, heads = boundary_rows(q_len, rng), boundary_rows(128, rng, extra=2)
    out = c.run().index_select(1, torch.as_tensor(rows, device="cuda")).index_select(2, torch.as_tensor(heads, device="cuda"))
    out = out.float().cpu().numpy()
    exact, want = c.oracle(rows, heads), c.oracle(rows, heads, p_bf16=True)
    mag = np.abs(exact).max()
    err, err_w = np.abs(out - exact), np.abs(out - want)
    _report("prefill long", f"B={B} past={past} q={q_len}",
            max(err.max() / (2e-2 * mag), err.mean() / (5e-3 * np.abs(exact).mean()), err_w.max() / ((2.0 ** -7 + 1e-3) * mag)))
    assert np.isfinite(out).all()
    assert err.max() <= 2e-2 * mag
    assert err.mean() <= 5e-3 * np.abs(exact).mean()
    assert err_w.max() <= 2.0 ** -7 * mag + 1e-3 * mag


@pytest.mark.gpu
def test_prefill_is_causal_at_length():
    """past 4096, 4096 queries: K / V rows at positions >= 6601 (mid key tile; query row 2505 is mid query tile) changed to
    other finite values: every query at a position < 6601 is bit-identical, the others change"""
    past, q_len, cut = 4096, 4096, 6601
    c = _Prefill(2, 16, past, q_len, seed=cut)
    before = c.run()
    g = torch.Generator(device="cuda").manual_seed(cut + 1)
    c.kv[:, cut:] = (torch.randn(c.kv[:, cut:].shape, generator=g, device="cuda") * 3).to(torch.bfloat16)
    c.rows[:, cut:] = (torch.randn(c.rows[:, cut:].shape, generator=g, device="cuda") * 3).to(torch.bfloat16)
    after = c.run()
    n = cut - past
    assert torch.equal(before[:, :n].view(torch.int16), after[:, :n].view(torch.int16))
    assert not torch.equal(before[:, n:n + 1].view(torch.int16), after[:, n:n + 1].view(torch.int16))
    assert not torch.equal(before[:, -1:].view(torch.int16), after[:, -1:].view(torch.int16))


@pytest.mark.gpu
def test_operator_long_prompt_in_chunks_then_decode_across_a_page():
    """KDeepseekV2Attention with 128 heads: a 2108-token prompt in chunks of 700, 700 and 708 (none a multiple of 128),
    then decode steps at positions 2108..2113 (a new page at 2112), against the plain module; the bar of
    test_operator_prefill_then_decode_matches_plain_attention"""
    from ktransformers_b200.models.custom_cache import StaticCache
    cfg, plain, op = _modules(128, 2108)
    prompt, cuts = 2108, [0, 700, 1400, 2108]
    cache = StaticCache(cfg, max_batch_size=1, max_cache_len=2176, device="cuda")
    x = (torch.randn(1, prompt, 1024, device="cuda") * 2).to(torch.bfloat16)
    want, past = plain(x, torch.arange(prompt, device="cuda").expand(1, prompt))
    got = torch.cat([_step(op, cache, x[:, a:b], a) for a, b in zip(cuts[:-1], cuts[1:])], 1)
    worst = _rel(got, want)
    assert cache.get_seq_length(0) == prompt
    for t in range(prompt, prompt + 6):
        xt = (torch.randn(1, 1, 1024, device="cuda") * 2).to(torch.bfloat16)
        g = _step(op, cache, xt, t)
        w, past = plain(xt, torch.full((1, 1), t, device="cuda"), past)
        worst = max(worst, _rel(g, w))
    _report("operator", "prompt 2108 + 6 decode steps", worst / 4e-2)
    assert worst < 4e-2, worst
    assert cache.get_seq_length(0) == prompt + 6
