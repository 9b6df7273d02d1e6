"""The bf16 scan family on the GPU, bit for bit against tests/scan_reference.py.

crag_search_scores (score-all) is held to float64 under the derived bound SCORE_BOUND -- the only bounded comparison
here.  Every other variant shares its main loop, so its outputs must equal, bit for bit, what the reference derives
from the score-all matrix of the same rows and queries: flat top-k (every selector and pooled-floor tier, rank
continuation pages, ids beyond 2^32, corpora dense in exact and one-ulp ties), a query's results wherever it sits in
its batch, and crag_ivf_assign.  Each score-all test records its worst err/bound as `worst_err_over_bound`."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import scan_reference as sr  # noqa: E402
from util_search import make_unit_rows  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SENTINEL = 0x7FA5A5A5            # a NaN payload no kernel writes: the canary of every output gap
BIG_OFFSET = (1 << 33) + 7


@pytest.fixture(scope="module", autouse=True)
def lib():
    assert torch.cuda.is_available()
    from comorag_b200 import _native
    return _native.load()


def _lib():
    from comorag_b200 import _native
    return _native.load()


def _check(rc, what):
    from comorag_b200 import _native
    _native.check(rc, what)


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ----------------------------------------------------------------------------------------------------- native calls
def strided(rows, pad):
    """rows bf16 [n, dim] inside a buffer of row stride dim + pad whose extra columns are NaN: (view, stride)."""
    n, dim = rows.shape
    buf = torch.full((max(n, 1), dim + pad), float("nan"), dtype=torch.bfloat16, device=rows.device)
    buf[:n, :dim] = rows
    return buf[:n, :dim], dim + pad


def score_all(rows, queries, out_ld=None):
    """crag_search_scores of rows (bf16 [n, dim], any row stride) against queries (bf16 [nq, dim], dense):
    (S fp32 [nq, n], minmax fp32 [nq, 2]).  The output has out_ld columns and one spare row, all sentinels, which must
    be intact afterwards."""
    lib = _lib()
    n, dim = rows.shape
    q = queries.contiguous()
    nq = q.shape[0]
    ld = max(n, 1) if out_ld is None else out_ld
    out = torch.full((nq + 1, ld), SENTINEL, dtype=torch.int32, device=DEV)
    mm = torch.full((nq, 2), SENTINEL, dtype=torch.int32, device=DEV)
    ws_bytes = lib.crag_search_workspace_bytes(nq, 1)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    _check(lib.crag_search_scores(rows.data_ptr(), n, dim, rows.stride(0), q.data_ptr(), nq, out.data_ptr(), ld,
                                  mm.data_ptr(), ws.data_ptr(), ws_bytes, _stream()), "crag_search_scores")
    torch.cuda.synchronize()
    assert bool((out[:nq, n:] == SENTINEL).all()) and bool((out[nq] == SENTINEL).all()), "wrote outside [nq, n_rows]"
    return out[:nq, :n].view(torch.float32), mm.view(torch.float32)


def topk_after(rows, queries, k, row_offset=0, after=None):
    """crag_search_topk_after: (ids [nq, k], scores [nq, k], minmax [nq, 2], last_keys int64 [nq])."""
    lib = _lib()
    n, dim = rows.shape
    q = queries.contiguous()
    nq = q.shape[0]
    ids = torch.full((nq, k), -7, dtype=torch.int64, device=DEV)
    sc = torch.full((nq, k), SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)
    mm = torch.full((nq, 2), SENTINEL, dtype=torch.int32, device=DEV).view(torch.float32)
    last = torch.full((nq,), -7, dtype=torch.int64, device=DEV)
    ws_bytes = lib.crag_search_workspace_bytes(nq, k)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    _check(lib.crag_search_topk_after(rows.data_ptr(), n, dim, rows.stride(0), row_offset, q.data_ptr(), nq, k,
                                      0 if after is None else after.data_ptr(), ids.data_ptr(), sc.data_ptr(),
                                      mm.data_ptr(), last.data_ptr(), ws.data_ptr(), ws_bytes, _stream()),
           "crag_search_topk_after")
    torch.cuda.synchronize()
    return ids, sc, mm, last


def scaled(rows):
    """Row r times 2^(r mod 17 - 8): exact in bf16, so the bound is tested at each row's own magnitude."""
    e = (torch.arange(rows.shape[0], device=rows.device) % 17 - 8).float()
    return (rows.float() * torch.exp2(e)[:, None]).bfloat16()


def corpus(kind, n, dim, seed):
    """unit: random unit rows.  dyadic: entries in {-3/8 .. 3/8}, so every dot product is exact in fp32 and exact
    ties are everywhere.  near_dup: 97 base rows repeated, each copy with one entry moved by one bf16 step, so scores
    sit one or a few fp32 ulps apart."""
    if kind == "unit":
        return make_unit_rows(n, dim, seed, device=DEV)
    g = torch.Generator(device=DEV).manual_seed(seed)
    if kind == "dyadic":
        return (torch.randint(-3, 4, (n, dim), generator=g, device=DEV).float() / 8).bfloat16()
    base = make_unit_rows(97, dim, seed, device=DEV)
    rows = base[torch.arange(n, device=DEV) % 97].clone()
    col = torch.randint(0, dim, (n,), generator=g, device=DEV)
    r = torch.arange(n, device=DEV)
    bits = rows.view(torch.int16)
    step = torch.where(torch.rand(n, generator=g, device=DEV) < 0.5, 1, -1).to(torch.int16)
    bits[r, col] = torch.where(r >= 97, bits[r, col] + step, bits[r, col])
    return rows


def queries_for(kind, nq, dim, seed):
    if kind == "dyadic":
        g = torch.Generator(device=DEV).manual_seed(seed)
        return (torch.randint(-3, 4, (nq, dim), generator=g, device=DEV).float() / 8).bfloat16()
    return make_unit_rows(nq, dim, seed, device=DEV)


def assert_minmax_of_rows(mm, S):
    sr.assert_bits(mm, sr.ordered_minmax(S, torch.ones_like(S, dtype=torch.bool)), "minmax")


# ------------------------------------------------------------------------------------------------------- score-all
DIMS = list(range(64, 1025, 64))
N_ROWS = [1, 127, 128, 129, 132 * 128 - 1, 132 * 128 + 1]
N_Q = [1, 31, 32, 33, 65]
PADS = [0, 8, 64]


@pytest.mark.parametrize("dim", DIMS)
def test_score_all_within_bound(record_property, dim):
    """Every K-block count 1 .. 16, with n_rows and nq rotated through the tile and query-pass edges, a row stride
    above dim (NaN in the gap) on two of three dims, an output leading dimension above n_rows (sentinels in the gap),
    unit and scaled rows."""
    i = dim // 64 - 1
    n, nq = N_ROWS[i % len(N_ROWS)], N_Q[i % len(N_Q)]
    worst = 0.0
    for kind in ("unit", "scaled"):
        x = make_unit_rows(n, dim, 10 + i, device=DEV)
        q = make_unit_rows(nq, dim, 50 + i, device=DEV)
        if kind == "scaled":
            x, q = scaled(x), scaled(q)
        xs, _ = strided(x, PADS[i % 3])
        S, mm = score_all(xs, q, out_ld=n + 3 + 32 * (i % 4))
        ref, mag = sr.score_reference(q, x)
        r = sr.err_over_bound(S, ref, mag)
        assert r <= 1.0, f"{kind}: worst err/bound {r:.3f}"
        worst = max(worst, r)
        assert_minmax_of_rows(mm, S)
    record_property("worst_err_over_bound", worst)


def test_score_all_two_million_rows(record_property):
    """2.2M rows: about 130 tiles per CTA, past the 128th-tile point of the scan's refresh schedule."""
    n, dim = 2_200_001, 64
    x = scaled(make_unit_rows(n, dim, 3, device=DEV))
    q = make_unit_rows(3, dim, 4, device=DEV)
    S, mm = score_all(x, q, out_ld=n + 5)
    ref, mag = sr.score_reference(q, x)
    r = sr.err_over_bound(S, ref, mag)
    assert r <= 1.0, r
    assert_minmax_of_rows(mm, S)
    record_property("worst_err_over_bound", r)


def test_score_all_unaligned_dim_through_dense_index(record_property):
    """dim 100: DenseIndex pads rows and queries with zero columns to 128; the bound holds against the 100 columns."""
    from comorag_b200.index import DenseIndex
    x, q = make_unit_rows(5000, 100, 5, device=DEV), make_unit_rows(33, 100, 6, device=DEV)
    idx = DenseIndex(100, device=DEV)
    idx.add(x)
    S, mm = idx.scores_device(idx.prepare_queries(q.float().cpu().numpy()))
    ref, mag = sr.score_reference(q, x)
    r = sr.err_over_bound(S, ref, mag)
    assert r <= 1.0, r
    assert_minmax_of_rows(mm, S)
    record_property("worst_err_over_bound", r)


def test_score_all_is_exact_on_dyadic_rows():
    """Where every partial sum is exact in fp32, score-all equals the float64 product bit for bit."""
    x, q = corpus("dyadic", 20_000, 1024, 7), queries_for("dyadic", 40, 1024, 8)
    S, _ = score_all(x, q)
    ref, _ = sr.score_reference(q, x)
    sr.assert_bits(S, ref.float())


# -------------------------------------------------------------------------------------------------------- flat top-k
TOPK_K = [1, 16, 17, 64, 65, 105, 106, 107, 128]


@pytest.mark.parametrize("kind", ["unit", "dyadic", "near_dup"])
@pytest.mark.parametrize("k", TOPK_K)
def test_flat_topk_equals_reference_of_score_all(k, kind):
    """Ids, scores and (min, max) bit for bit against topk_from_scores(score-all of the same rows and queries), for
    the 64- and 128-key selectors, the three pooled-floor variants (k <= 16, 5k <= 4 CTAs, above; the pool is on
    from 4 tiles per CTA), a shard smaller than k (a -1 / -inf tail), and 33 queries (two passes)."""
    dim = 128
    q = queries_for(kind, 33, dim, 100 + k)
    offset = BIG_OFFSET if kind == "unit" else 0
    for n in (max(1, k - 1), 1000, 80_000, 300_000):
        x = corpus(kind, n, dim, 200 + k)
        ids, sc, mm, _ = topk_after(x, q, k, row_offset=offset)
        S, _ = score_all(x, q)
        w_ids, w_sc, w_mm, _ = sr.topk_from_scores(S, k, row_offset=offset)
        sr.assert_bits(ids, w_ids, f"ids n={n}")
        sr.assert_bits(sc, w_sc, f"scores n={n}")
        sr.assert_bits(mm, w_mm, f"minmax n={n}")


@pytest.mark.parametrize("kind", ["unit", "dyadic"])
@pytest.mark.parametrize("n,k", [(5000, 300), (3000, 2047), (200, 500)])
def test_rank_continuation_pages(n, k, kind):
    """k > 128 as pages of crag_search_topk_after, each continuing after the previous page's last key: every page
    and every last key bit for bit against the reference's, and the pages together equal the reference's top-k."""
    dim = 256
    x, q = corpus(kind, n, dim, 300 + n), queries_for(kind, 33, dim, 400 + n)
    S, _ = score_all(x, q)
    after, w_after, got, want = None, None, [], []
    for p0 in range(0, k, 128):
        kk = min(128, k - p0)
        ids, sc, mm, after = topk_after(x, q, kk, row_offset=BIG_OFFSET, after=after)
        w_ids, w_sc, w_mm, w_after = sr.topk_from_scores(S, kk, row_offset=BIG_OFFSET, after_keys=w_after)
        sr.assert_bits(after, w_after, f"last keys of page {p0}")
        sr.assert_bits(mm, w_mm, "minmax")
        got.append((ids, sc)), want.append((w_ids, w_sc))
    for j in range(2):
        sr.assert_bits(torch.cat([g[j] for g in got], 1), torch.cat([w[j] for w in want], 1), ("ids", "scores")[j])
    one_ids, one_sc, _, _ = sr.topk_from_scores(S, k, row_offset=BIG_OFFSET)
    sr.assert_bits(torch.cat([g[0] for g in got], 1), one_ids, "pages vs one-shot")


# ------------------------------------------------------------------------------------------------- batch invariance
def test_query_results_do_not_depend_on_batch_slot():
    """A query's scores, top-k and (min, max) are bit-identical alone and at slots 0, 5, 31, 32, 63 of a 64-query
    block (the retrieval wave batches unrelated queries)."""
    dim = 256
    x = corpus("near_dup", 100_000, dim, 11)
    q0 = make_unit_rows(1, dim, 12, device=DEV)
    others = make_unit_rows(64, dim, 13, device=DEV)
    S1, mm1 = score_all(x, q0)
    alone = {k: topk_after(x, q0, k) for k in (10, 100)}
    for slot in (0, 5, 31, 32, 63):
        blk = others.clone()
        blk[slot] = q0[0]
        S, mm = score_all(x, blk)
        sr.assert_bits(S[slot], S1[0], f"scores at slot {slot}")
        sr.assert_bits(mm[slot], mm1[0], f"minmax at slot {slot}")
        for k, (a_ids, a_sc, a_mm, _) in alone.items():
            ids, sc, mm_k, _ = topk_after(x, blk, k)
            sr.assert_bits(ids[slot], a_ids[0], f"ids at slot {slot}, k={k}")
            sr.assert_bits(sc[slot], a_sc[0], f"scores at slot {slot}, k={k}")
            sr.assert_bits(mm_k[slot], a_mm[0], f"minmax at slot {slot}, k={k}")


# --------------------------------------------------------------------------------------------------- ivf assignment
@pytest.mark.parametrize("nlist", [1, 31, 32, 33, 100, 4096])
def test_ivf_assign_equals_reference_of_score_all(nlist):
    """crag_ivf_assign (through ivf.assign_device) against assign_from_scores(score-all with the rows as corpus and
    the centroid table as queries): list ids and best scores bit for bit.  Half the rows score negative against
    every centroid (a zero padding centroid of the last block must not win); centroids l + 1, l + 32 and l + 64
    repeat centroid l (the smallest id must win); the rows have a row stride above dim; dyadic rows add exact ties
    between different centroids."""
    from comorag_b200.ivf import assign_device
    dim, n = 128, 6000
    g = torch.Generator(device=DEV).manual_seed(nlist)
    e0 = torch.zeros(dim, device=DEV)
    e0[0] = 1.0
    # every centroid has an e0 component of about +0.58; the first half of the rows about -0.97 and little else
    cent = torch.nn.functional.normalize(8 * e0 + torch.randn(nlist, dim, generator=g, device=DEV), dim=1)
    dups = [3 + l for l in (1, 32, 64) if 3 + l < nlist]
    if dups:
        cent[dups] = cent[3].clone()
    cent = cent.bfloat16()
    x = torch.nn.functional.normalize(torch.randn(n, dim, generator=g, device=DEV), dim=1)
    x[: n // 2] = torch.nn.functional.normalize(-e0 + 0.02 * torch.randn(n // 2, dim, generator=g, device=DEV), dim=1)
    x[n // 2: n // 2 + 500] = cent[torch.arange(500, device=DEV) % min(nlist, 4)].float() + 0.01 * torch.randn(500, dim, generator=g, device=DEV)
    x = x.bfloat16()
    x[-300:] = (torch.randint(-3, 4, (300, dim), generator=g, device=DEV).float() / 8).bfloat16()
    xs, _ = strided(x, 64)
    ids, best = assign_device(xs, cent)
    torch.cuda.synchronize()
    S, _ = score_all(x, cent)
    w_ids, w_best = sr.assign_from_scores(S)
    sr.assert_bits(ids, w_ids, "list ids")
    sr.assert_bits(best, w_best, "best scores")
    assert bool((best[: n // 2] < 0).all())
    if dups:                                   # a repeat of centroid 3 never wins: 3 does, on every row near it
        assert not bool(torch.isin(ids, torch.tensor(dups, device=DEV, dtype=torch.int32)).any())
        assert bool((ids[n // 2: n // 2 + 500][3::4] == 3).all())
