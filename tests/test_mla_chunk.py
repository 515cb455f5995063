"""Absorbed MLA for prompt chunks: ktb200_mla_decode_chunk (csrc/mla.cu, mla_chunk_tc_kernel) and the absorb_for_prefill
path of KDeepseekV2Attention.

Query i of sequence b in a chunk of q_len attends to the first P + i + 1 cached latents, P = kv_len[b] - q_len, so it must
equal the absorbed decode oracle (oracle/mla_oracle.mla_decode) at length P + i + 1.  The oracle runs on sampled query rows
and heads (every output row depends only on its own query and length); the bounds are those of test_mla_lengths'
decode checks.

CPU: the argument checks and the workspace size.  GPU: the kernel against the oracle over chunk lengths and prefixes up to
131072 tokens, batches, head counts, page placement and split counts; bit-exact properties (q_len 1 is decode, causality,
nothing read past kv_len, empty sequences, CUDA-graph replays, batch independence); the operator through a chunked prompt
and decode steps, and a captured 4-token step."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from ktransformers_b200 import native
from oracle import mla_oracle
from test_mla_lengths import MAX_SPLITS, POOL_ROWS, boundary_rows, check_decode, pick_splits, sms
from test_mla_prefill import SCALE, _modules, _rel, _step

PAGE = 64


# ------------------------------------------------------------------------------------------------ helpers
def chunk_params(B, q_len, H, page, max_pages, splits, q_nope, q_pe, kv, pt, kl, out, lse, ws, ws_bytes, rows=0):
    return native.MlaChunkParams(B, q_len, H, page, max_pages, splits, SCALE, q_nope, q_pe, kv, pt, kl, out, lse, ws, ws_bytes, rows)


def chunk(q_nope, q_pe, kv, page_table, kv_len, splits=0, ws_splits=None, count=True):
    """ktb200_mla_decode_chunk with device q_nope [B, q, H, 512] / q_pe [B, q, H, 64] (bf16), the device cache kv
    [pages, page, 576] and host page table / lengths -> (out [B, q, H, 512] bf16, lse [B, q, H], splits used).  The
    workspace starts as NaN; the count of floats the call wrote gives the split count (count=False: not counted, for
    calls whose partials hold NaN because the cache rows a query reads are NaN)."""
    lib = native.lib()
    B, q_len, H = q_nope.shape[:3]
    if ws_splits is None:
        ws_splits = splits if splits > 0 else min(MAX_SPLITS, -(-sms() // (B * q_len * -(-H // 64))))
    pt = torch.from_numpy(np.ascontiguousarray(page_table, np.int32)).cuda()
    kl = torch.from_numpy(np.ascontiguousarray(kv_len, np.int32)).cuda()
    out = torch.empty((B, q_len, H, 512), dtype=torch.bfloat16, device="cuda")
    lse = torch.empty((B, q_len, H), dtype=torch.float32, device="cuda")
    ws_bytes = lib.ktb200_mla_chunk_workspace_bytes(B, q_len, H, ws_splits)
    ws = torch.full((ws_bytes // 4,), float("nan"), dtype=torch.float32, device="cuda")
    p = chunk_params(B, q_len, H, kv.shape[1], page_table.shape[1], splits, q_nope.data_ptr(), q_pe.data_ptr(), kv.data_ptr(),
                     pt.data_ptr(), kl.data_ptr(), out.data_ptr(), lse.data_ptr(), ws.data_ptr(), ws_bytes)
    native.check(lib.ktb200_mla_decode_chunk(C.byref(p), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    if not count:
        return out, lse, None
    written = int((~torch.isnan(ws)).sum())
    per_split = B * q_len * H * 513
    assert written % per_split == 0, written
    return out, lse, written // per_split


def queries(B, q_len, H, seed):
    """bf16 q_nope / q_pe on the device at the scale of test_mla_lengths.queries"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    return ((torch.randn((B, q_len, H, 512), generator=g, device="cuda") * 0.5).to(torch.bfloat16),
            (torch.randn((B, q_len, H, 64), generator=g, device="cuda") * 0.5).to(torch.bfloat16))


def check_rows(family, case, out, lse, q_nope, q_pe, host, pt, kl, rows, heads):
    """query rows `rows` (pairs (b, i)) and heads `heads` against mla_decode at length P + i + 1"""
    q_len = q_nope.shape[1]
    bs, iis = np.array([r[0] for r in rows]), np.array([r[1] for r in rows])
    hs = torch.as_tensor(heads, device="cuda")
    pick = lambda t: t[torch.as_tensor(bs, device="cuda"), torch.as_tensor(iis, device="cuda")].index_select(1, hs).float().cpu().numpy()
    qn, qp = pick(q_nope), pick(q_pe)
    lens = (kl[bs] - q_len + iis + 1).astype(np.int32)
    want, want_lse = mla_oracle.mla_decode(qn, qp, host, pt[bs], lens, SCALE, p_bf16=True)
    exact, _ = mla_oracle.mla_decode(qn, qp, host, pt[bs], lens, SCALE, p_bf16=False)
    check_decode(family, case, pick(out), pick(lse), want, want_lse, exact)


def sample_rows(rng, B, q_len, per_seq=6):
    rows = []
    for b in range(B):
        ii = boundary_rows(q_len, rng, extra=2) if q_len <= 300 else np.unique(np.r_[0, 1, 63, 64, q_len - 1, rng.integers(0, q_len, per_seq)])
        rows += [(b, int(i)) for i in ii]
    return rows


@pytest.fixture(scope="module")
def pool():
    """one bf16 latent cache of POOL_ROWS token rows on the device (pages of 64) and its float32 copy on the host"""
    g = torch.Generator(device="cuda").manual_seed(1)
    kv = torch.randn((POOL_ROWS, 576), generator=g, device="cuda").to(torch.bfloat16)
    return kv.view(-1, PAGE, 576), kv.float().cpu().numpy().reshape(-1, PAGE, 576)


def random_pages(rng, n_pool_pages, B, width):
    return np.stack([rng.choice(n_pool_pages, width, replace=False) for _ in range(B)]).astype(np.int32)


# ------------------------------------------------------------------------------------------------ CPU
def _valid(**over):
    """a parameter set every check passes (fake device addresses: nothing is dereferenced before the checks)"""
    a = dict(B=1, q_len=4, H=128, page=64, max_pages=4, splits=2, q_nope=1 << 20, q_pe=2 << 20, kv=3 << 20, pt=4 << 20, kl=5 << 20,
             out=6 << 20, lse=None, ws=7 << 20, ws_bytes=1 << 40)
    a.update(over)
    return chunk_params(*a.values())


@pytest.mark.parametrize("over,msg", [
    (dict(q_len=0), "q_len"), (dict(q_len=-3), "q_len"),
    (dict(q_nope=None), "null"), (dict(q_pe=None), "null"), (dict(kv=None), "null"), (dict(pt=None), "null"),
    (dict(kl=None), "null"), (dict(out=None), "null"), (dict(ws=None), "null"),
    (dict(page=48), "page_size"), (dict(page=0), "page_size"), (dict(H=0), "num_heads"), (dict(max_pages=0), "max_pages"),
    (dict(q_nope=(1 << 20) + 8), "aligned"), (dict(q_pe=(2 << 20) + 2), "aligned"), (dict(kv=(3 << 20) + 4), "aligned"),
    (dict(splits=129), "num_kv_splits"),
    (dict(ws_bytes=1 * 4 * 2 * 128 * 513 * 4 - 4), "workspace"),
    (dict(B=65536, q_len=1, H=16), "too large"), (dict(B=1, q_len=1 << 25, H=128), "too large"),
])
def test_chunk_refuses_bad_arguments(over, msg):
    lib = native.lib()
    p = _valid(**over)
    assert lib.ktb200_mla_decode_chunk(C.byref(p), None) == native.EINVAL
    assert msg in lib.ktb200_last_error().decode()


def test_chunk_refuses_null_params():
    lib = native.lib()
    assert lib.ktb200_mla_decode_chunk(None, None) == native.EINVAL
    assert "null" in lib.ktb200_last_error().decode()


def test_chunk_workspace_bytes_is_monotone():
    lib = native.lib()
    f = lib.ktb200_mla_chunk_workspace_bytes
    grid = [1, 2, 3, 7, 64, 128, 1000]
    for a in grid:
        for b in grid:
            for c in grid:
                vals = [f(x, a, b, c) for x in grid] + [f(a, x, b, c) for x in grid] + [f(a, b, x, c) for x in grid] + [f(a, b, c, x) for x in grid[:6]]
                for run in (vals[0:7], vals[7:14], vals[14:21], vals[21:27]):
                    assert all(x < y for x, y in zip(run, run[1:])), (a, b, c, run)
    assert f(2, 3, 128, 0) == f(2, 3, 128, MAX_SPLITS)
    assert f(0, 3, 128, 4) == f(2, 0, 128, 4) == f(2, 3, 0, 4) == 0
    assert f(1, 1, 128, 0) == lib.ktb200_mla_workspace_bytes(1, 128, 0)


# ------------------------------------------------------------------------------------------------ against the oracle (GPU)
@pytest.mark.gpu
@pytest.mark.parametrize("past", [0, 1, 63, 4095, 32768])
@pytest.mark.parametrize("q_len", [2, 3, 16, 64, 170, 1000])
def test_chunk_vs_oracle(pool, q_len, past):
    """one sequence of 128 heads, its pages a random permutation of pool pages, automatic splits"""
    kv, host = pool
    rng = np.random.default_rng(q_len * 100003 + past)
    L = past + q_len
    width = -(-L // PAGE) + 1
    pt = random_pages(rng, kv.shape[0], 1, width)
    kl = np.array([L], np.int32)
    q_nope, q_pe = queries(1, q_len, 128, q_len + past)
    out, lse, used = chunk(q_nope, q_pe, kv, pt, kl)
    assert used == min(pick_splits(q_len, 128, width * 2, sms()), width * 2)
    check_rows("chunk", f"q={q_len} P={past} splits={used}", out, lse, q_nope, q_pe, host, pt, kl, sample_rows(rng, 1, q_len),
               boundary_rows(128, rng, extra=2) if past < 32768 else np.array([0, 1, 63, 64, 127]))


@pytest.mark.gpu
def test_chunk_after_a_131072_token_prefix(pool):
    kv, host = pool
    rng = np.random.default_rng(131072)
    q_len, L = 8, 131072 + 8
    width = -(-L // PAGE)
    pt = random_pages(rng, kv.shape[0], 1, width)
    kl = np.array([L], np.int32)
    q_nope, q_pe = queries(1, q_len, 128, 131072)
    out, lse, used = chunk(q_nope, q_pe, kv, pt, kl)
    assert used == pick_splits(q_len, 128, width * 2, sms())
    check_rows("chunk long prefix", f"q=8 P=131072 splits={used}", out, lse, q_nope, q_pe, host, pt, kl,
               [(0, i) for i in range(q_len)], np.array([0, 37, 64, 127]))


@pytest.mark.gpu
@pytest.mark.parametrize("H", [128, 16])
@pytest.mark.parametrize("B", [1, 4, 8])
def test_chunk_batches_vs_oracle(pool, B, H):
    """B sequences with different prefixes (0, 1, 31, 33, 64 and random up to 20000), q_len 40, automatic splits"""
    kv, host = pool
    rng = np.random.default_rng(B * 1000 + H)
    q_len = 40
    past = np.array(([0, 1, 31, 33, 64] + rng.integers(0, 20000, 8).tolist())[:B])
    past = rng.permutation(past)
    kl = (past + q_len).astype(np.int32)
    width = -(-int(kl.max()) // PAGE) + 2
    pt = random_pages(rng, kv.shape[0], B, width)
    q_nope, q_pe = queries(B, q_len, H, B + H)
    out, lse, used = chunk(q_nope, q_pe, kv, pt, kl)
    assert used == min(pick_splits(B * q_len, H, width * 2, sms()), width * 2)
    check_rows("chunk batch", f"B={B} H={H} splits={used}", out, lse, q_nope, q_pe, host, pt, kl, sample_rows(rng, B, q_len),
               boundary_rows(H, rng, extra=2) if H > 16 else np.arange(H))


@pytest.mark.gpu
@pytest.mark.parametrize("splits", [1, 2, 7, 128])
def test_chunk_explicit_splits_vs_oracle(pool, splits):
    """q_len 16 after 8191 cached tokens, 16 heads: 1 split streams 256 tiles per CTA, 128 splits leave 2 tiles each"""
    kv, host = pool
    rng = np.random.default_rng(splits)
    q_len, L = 16, 8191 + 16
    width = -(-L // PAGE)
    pt = random_pages(rng, kv.shape[0], 1, width)
    kl = np.array([L], np.int32)
    q_nope, q_pe = queries(1, q_len, 16, splits)
    out, lse, used = chunk(q_nope, q_pe, kv, pt, kl, splits=splits)
    assert used == splits
    check_rows("chunk explicit splits", f"splits={splits}", out, lse, q_nope, q_pe, host, pt, kl, [(0, i) for i in range(q_len)], np.arange(16))


# ------------------------------------------------------------------------------------------------ exact properties (GPU)
def _decode(q_nope, q_pe, kv, pt, kl, splits):
    """ktb200_mla_decode with device queries [B, H, *] -> (out, lse) on the device"""
    lib = native.lib()
    B, H = q_nope.shape[:2]
    pt_d = torch.from_numpy(np.ascontiguousarray(pt, np.int32)).cuda()
    kl_d = torch.from_numpy(np.ascontiguousarray(kl, np.int32)).cuda()
    out = torch.empty((B, H, 512), dtype=torch.bfloat16, device="cuda")
    lse = torch.empty((B, H), dtype=torch.float32, device="cuda")
    ws_bytes = lib.ktb200_mla_workspace_bytes(B, H, 0)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    p = native.MlaParams(B, H, kv.shape[1], pt.shape[1], splits, SCALE, q_nope.data_ptr(), q_pe.data_ptr(), kv.data_ptr(), pt_d.data_ptr(),
                         kl_d.data_ptr(), out.data_ptr(), lse.data_ptr(), ws.data_ptr(), ws_bytes, 0)
    native.check(lib.ktb200_mla_decode(C.byref(p), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out, lse


@pytest.mark.gpu
@pytest.mark.parametrize("B,H,splits", [(1, 128, 0), (3, 128, 0), (5, 16, 9), (2, 40, 1)])
def test_chunk_of_one_query_is_decode(pool, B, H, splits):
    kv, _ = pool
    rng = np.random.default_rng(B * H + splits)
    kl = rng.integers(1, 30000, B).astype(np.int32)
    kl[0] = 33
    pt = random_pages(rng, kv.shape[0], B, 480)
    q_nope, q_pe = queries(B, 1, H, B + H)
    out, lse, _ = chunk(q_nope, q_pe, kv, pt, kl, splits=splits, ws_splits=MAX_SPLITS)
    d_out, d_lse = _decode(q_nope[:, 0], q_pe[:, 0], kv, pt, kl, splits)
    assert torch.equal(out[:, 0].view(torch.int16), d_out.view(torch.int16)) and torch.equal(lse[:, 0], d_lse)


def _private_cache(pool, width, seed):
    """a cache of its own (the tests below write into it): `width` pages of pool content in a random order"""
    kv, _ = pool
    rng = np.random.default_rng(seed)
    cache = kv[: width + 8].clone()
    pt = rng.permutation(width + 8)[:width].reshape(1, -1).astype(np.int32)
    return cache, pt


def _row(cache, pt, t):
    return cache[int(pt[0, t // PAGE]), t % PAGE]


@pytest.mark.gpu
@pytest.mark.parametrize("past,q_len,splits", [(100, 64, 0), (4095, 16, 3), (0, 170, 0)])
def test_chunk_is_causal(pool, past, q_len, splits):
    """rows at positions >= P + k overwritten (NaN in every other row, large finite values between): queries i < k are
    bit-identical, for k at a tile edge, mid tile and the last query"""
    L = past + q_len
    width = -(-L // PAGE) + 1
    cache, pt = _private_cache(pool, width, past + q_len)
    q_nope, q_pe = queries(1, q_len, 128, past)
    kl = np.array([L], np.int32)
    base, base_lse, _ = chunk(q_nope, q_pe, cache, pt, kl, splits=splits, ws_splits=MAX_SPLITS)
    for k in sorted({1, q_len // 2, (32 - past % 32) % 32 or 32, q_len - 1}):
        if not 0 < k < q_len:
            continue
        saved = [_row(cache, pt, t).clone() for t in range(past + k, L)]
        for t in range(past + k, L):
            _row(cache, pt, t).fill_(float("nan") if t % 2 else 300.0)
        out, lse, _ = chunk(q_nope, q_pe, cache, pt, kl, splits=splits, ws_splits=MAX_SPLITS, count=False)
        for t, s in zip(range(past + k, L), saved):
            _row(cache, pt, t).copy_(s)
        assert torch.equal(out[:, :k].view(torch.int16), base[:, :k].view(torch.int16)), k
        assert torch.equal(lse[:, :k], base_lse[:, :k]), k
        assert not torch.equal(out[:, k:].view(torch.int16), base[:, k:].view(torch.int16)), k


@pytest.mark.gpu
def test_chunk_reads_nothing_past_kv_len(pool):
    """NaN / Inf in every row past kv_len and in every page the table does not name: bit-identical output"""
    past, q_len = 5000, 37
    L = past + q_len
    width = -(-L // PAGE) + 3
    cache, pt = _private_cache(pool, width, 5)
    q_nope, q_pe = queries(1, q_len, 128, 5)
    kl = np.array([L], np.int32)
    base, base_lse, _ = chunk(q_nope, q_pe, cache, pt, kl)
    named = set(pt[0, : -(-L // PAGE)].tolist())
    for i in range(cache.shape[0]):
        if i not in named:
            cache[i] = float("nan") if i % 2 else float("inf")
    last = cache[int(pt[0, (L - 1) // PAGE])]
    last[L % PAGE:: 2] = float("nan")
    last[L % PAGE + 1:: 2] = -float("inf")
    out, lse, _ = chunk(q_nope, q_pe, cache, pt, kl)
    assert torch.equal(out.view(torch.int16), base.view(torch.int16)) and torch.equal(lse, base_lse)
    assert torch.isfinite(out.float()).all()


@pytest.mark.gpu
def test_chunk_shorter_than_q_len_is_empty(pool):
    """kv_len < q_len (device data, so not refused): that sequence's rows are zeros with lse -inf, the others unaffected"""
    kv, _ = pool
    rng = np.random.default_rng(9)
    q_len = 16
    kl = np.array([700, 15, 0, 16], np.int32)
    pt = random_pages(rng, kv.shape[0], 4, 16)
    q_nope, q_pe = queries(4, q_len, 128, 9)
    out, lse, _ = chunk(q_nope, q_pe, kv, pt, kl, splits=4)
    assert not out[1:3].float().any() and torch.isneginf(lse[1:3]).all()
    assert torch.isfinite(out.float()).all() and torch.isfinite(lse[[0, 3]]).all()
    alone, alone_lse, _ = chunk(q_nope[:1], q_pe[:1], kv, pt[:1], kl[:1], splits=4)
    assert torch.equal(alone.view(torch.int16), out[:1].view(torch.int16)) and torch.equal(alone_lse, lse[:1])


@pytest.mark.gpu
def test_chunk_batch_independence(pool):
    """fixed splits and page-table width: each sequence of a batch of 8 equals it run alone"""
    kv, _ = pool
    rng = np.random.default_rng(8)
    q_len = 24
    kl = (rng.integers(0, 9000, 8) + q_len).astype(np.int32)
    pt = random_pages(rng, kv.shape[0], 8, 150)
    q_nope, q_pe = queries(8, q_len, 128, 8)
    out, lse, _ = chunk(q_nope, q_pe, kv, pt, kl, splits=5)
    for b in range(8):
        o1, l1, _ = chunk(q_nope[b:b + 1], q_pe[b:b + 1], kv, pt[b:b + 1], kl[b:b + 1], splits=5)
        assert torch.equal(o1[0].view(torch.int16), out[b].view(torch.int16)) and torch.equal(l1[0], lse[b]), b


@pytest.mark.gpu
def test_chunk_graph_replays_with_positions_advancing_on_the_device(pool):
    """MLAWrapper planned for q_len 4 over 2 sequences; the captured step computes kv_len from a device position tensor,
    which advances by 4 between replays: every replay equals the eager call bit for bit and is within the oracle bounds"""
    from ktransformers_b200.operators.flashinfer_wrapper import MLAWrapper
    kv, host = pool
    rng = np.random.default_rng(44)
    B, q_len, pages = 2, 4, 160
    pt = random_pages(rng, kv.shape[0], B, pages)
    w = MLAWrapper(B, B * pages)
    pos = torch.tensor([[60, 61, 62, 63], [3000, 3001, 3002, 3003]], dtype=torch.int64, device="cuda")
    w.plan(torch.arange(0, B + 1, dtype=torch.int32) * q_len, torch.arange(0, B + 1, dtype=torch.int32, device="cuda") * pages,
           torch.from_numpy(pt.reshape(-1)).cuda(), (pos[:, -1] + 1).to(torch.int32), None, 128, 512, 64, PAGE, SCALE,
           torch.bfloat16, torch.bfloat16)
    assert w.q_len == q_len
    q_nope, q_pe = queries(B, q_len, 128, 44)
    qn, qp = q_nope.reshape(B * q_len, 128, 512), q_pe.reshape(B * q_len, 128, 64)
    ckv, kpe = kv[..., :512], kv[..., 512:]

    def step():
        w.kv_len_arr_buf[:B].copy_((pos[:, -1] + 1).to(torch.int32))
        return w.run(qn, qp, ckv, kpe, return_lse=True)

    step()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_out, g_lse = step()
    heads = np.array([0, 63, 64, 127])
    for r in range(4):
        graph.replay()
        torch.cuda.synchronize()
        r_out, r_lse = g_out.clone(), g_lse.clone()
        e_out, e_lse = step()
        torch.cuda.synchronize()
        assert torch.equal(r_out.view(torch.int16), e_out.view(torch.int16)) and torch.equal(r_lse, e_lse), r
        kl = (pos[:, -1] + 1).int().cpu().numpy()
        check_rows("chunk graph replay", f"replay {r} kv_len={kl.tolist()}", r_out.view(B, q_len, 128, 512), r_lse.view(B, q_len, 128),
                   q_nope, q_pe, host, pt, kl, [(b, i) for b in range(B) for i in range(q_len)], heads)
        pos += q_len


# ------------------------------------------------------------------------------------------------ operator (GPU)
def _absorbed(cfg, plain):
    from ktransformers_b200.operators.attention import KDeepseekV2Attention
    return KDeepseekV2Attention("blk.0.self_attn", None, cfg, plain, "cuda", "cuda", absorb_for_prefill=True)


@pytest.mark.gpu
def test_operator_absorbed_prompt_in_chunks_then_decode():
    """128 heads: a 2108-token prompt in chunks of 700 / 700 / 708 with absorb_for_prefill, then decode steps at positions
    2108..2113 (a new page at 2112).  Against the module in float64 and against the non-absorbed layer on the same prompt,
    both within the operator decode bar; the chunks run the chunk kernel, not the prefill kernel."""
    from test_mla_prefill import _kernels_of
    from ktransformers_b200.models.custom_cache import StaticCache
    cfg, plain, op_plain = _modules(128, 2108)
    op = _absorbed(cfg, plain)
    plain64 = copy.deepcopy(plain).double()
    prompt, cuts = 2108, [0, 700, 1400, 2108]
    cache = StaticCache(cfg, max_batch_size=1, max_cache_len=2176, device="cuda")
    cache_plain = StaticCache(cfg, max_batch_size=1, max_cache_len=2176, device="cuda")
    x = (torch.randn(1, prompt, 1024, device="cuda") * 2).to(torch.bfloat16)
    want, past = plain64(x.double(), torch.arange(prompt, device="cuda").expand(1, prompt))
    got, other = [], []
    for a, b in zip(cuts[:-1], cuts[1:]):
        if a == 0:
            names = _kernels_of(lambda: got.append(_step(op, cache, x[:, a:b], a)))
            assert any("mla_chunk_tc_kernel" in n for n in names) and not any("mla_prefill" in n or "mla_decode_tc" in n for n in names), names
        else:
            got.append(_step(op, cache, x[:, a:b], a))
        other.append(_step(op_plain, cache_plain, x[:, a:b], a))
    got, other = torch.cat(got, 1), torch.cat(other, 1)
    worst, vs_plain = _rel(got, want), _rel(got, other)
    assert cache.get_seq_length(0) == prompt
    for t in range(prompt, prompt + 6):
        xt = (torch.randn(1, 1, 1024, device="cuda") * 2).to(torch.bfloat16)
        g = _step(op, cache, xt, t)
        o = _step(op_plain, cache_plain, xt, t)
        w, past = plain64(xt.double(), torch.full((1, 1), t, device="cuda"), past)
        worst, vs_plain = max(worst, _rel(g, w)), max(vs_plain, _rel(g, o))
    print(f"[operator absorbed] prompt 2108 + 6 decode steps: {worst / 4e-2:.3f} of the bound vs float64, {vs_plain / 4e-2:.3f} vs non-absorbed")
    assert worst < 4e-2, worst
    assert vs_plain < 4e-2, vs_plain
    assert cache.get_seq_length(0) == prompt + 6


@pytest.mark.gpu
def test_operator_absorbed_chunk_makes_no_host_synchronisation():
    from ktransformers_b200.models.custom_cache import StaticCache
    """after a first call has built the MLA wrapper (its constructor copies to the device), chunks of other lengths re-plan
    and run without synchronising"""
    cfg, plain, _ = _modules(16, 21)
    op = _absorbed(cfg, plain)
    cache = StaticCache(cfg, max_batch_size=2, max_cache_len=512, device="cuda")
    x = (torch.randn(2, 200, 1024, device="cuda") * 2).to(torch.bfloat16)
    pos, cpos = torch.arange(200, device="cuda").expand(2, 200), torch.arange(200, device="cuda")
    warm = StaticCache(cfg, max_batch_size=2, max_cache_len=512, device="cuda")
    op(x[:, :50], position_ids=pos[:, :50], past_key_value=warm, cache_position=cpos[:50])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        op(x[:, :100], position_ids=pos[:, :100], past_key_value=cache, cache_position=cpos[:100])
        op(x[:, 100:], position_ids=pos[:, 100:], past_key_value=cache, cache_position=cpos[100:])
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_operator_absorbed_4_token_step_in_a_cuda_graph():
    """bsz 2, 16 heads: a 90-token prompt, then a 4-token step captured once and replayed at positions 90, 94, 98 with
    positions and cache positions written into the captured inputs on the device; each replay equals the eager step on a
    twin cache bit for bit"""
    from ktransformers_b200.models.custom_cache import StaticCache
    cfg, plain, _ = _modules(16, 31)
    op = _absorbed(cfg, plain)
    bsz, n, q = 2, 90, 4
    caches = [StaticCache(cfg, max_batch_size=bsz, max_cache_len=256, device="cuda") for _ in range(2)]
    x = (torch.randn(bsz, n + 3 * q, 1024, device="cuda") * 2).to(torch.bfloat16)
    for c in caches:
        _step(op, c, x[:, :n], 0)
    xs = torch.empty(bsz, q, 1024, dtype=torch.bfloat16, device="cuda")
    pos = torch.empty(bsz, q, dtype=torch.int64, device="cuda")
    cpos = torch.empty(q, dtype=torch.int64, device="cuda")

    def set_inputs(t):
        xs.copy_(x[:, t:t + q])
        cpos.copy_(torch.arange(t, t + q, device="cuda"))
        pos.copy_(cpos.expand(bsz, q))

    set_inputs(n)      # warm-up on a third cache: plans q_len 4 and allocates before the capture
    warm = StaticCache(cfg, max_batch_size=bsz, max_cache_len=256, device="cuda")
    op(xs, position_ids=pos, past_key_value=warm, cache_position=cpos)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        g_out, _, _ = op(xs, position_ids=pos, past_key_value=caches[0], cache_position=cpos)
    # the capture ran nothing: caches[0] still ends at n
    for t in (n, n + q, n + 2 * q):
        set_inputs(t)
        graph.replay()
        torch.cuda.synchronize()
        e_out = _step(op, caches[1], x[:, t:t + q], t)
        torch.cuda.synchronize()
        assert torch.equal(g_out.view(torch.int16), e_out.view(torch.int16)), t
    assert torch.equal(caches[0].key_cache[0].view(torch.int16), caches[1].key_cache[0].view(torch.int16))
