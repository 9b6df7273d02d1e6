"""crag_knn_topk on the GPU: the fp32 score block of the wgmma GEMM against float64 dot products at tile edges, the
exact top-k (k <= 2048) against the numpy oracle, ids against the scan path (crag_search_topk / a crag_search_topk_after
chain called directly), the routing of DenseIndex, argument errors, and the retrieve_knn self-join at k = 2047."""
import numpy as np
import pytest
import torch

from oracle import search_oracle as so
from util_search import make_unit_rows, torch_reference_topk

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from comorag_b200 import _native
    _native.load()
    return torch.device("cuda:0")


def _knn(corpus, queries, k, row_offset=0, ws_queries=None, stride=None):
    """crag_knn_topk through the C ABI; ws_queries caps the workspace at that many score rows (forces chunking)."""
    from comorag_b200 import _native
    lib = _native.load()
    n, dim = corpus.shape[0], queries.shape[1]
    nq = queries.shape[0]
    dev = queries.device
    ids = torch.full((nq, k), -7, dtype=torch.int64, device=dev)
    scores = torch.full((nq, k), -7.0, dtype=torch.float32, device=dev)
    minmax = torch.full((nq, 2), -7.0, dtype=torch.float32, device=dev)
    ws_bytes = lib.crag_knn_workspace_bytes(n, ws_queries or nq)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    rc = lib.crag_knn_topk(corpus.data_ptr() if n else 0, n, dim, stride or (corpus.stride(0) if n else dim), row_offset,
                           queries.data_ptr(), nq, k, ids.data_ptr(), scores.data_ptr(), minmax.data_ptr(), ws.data_ptr(),
                           ws_bytes, torch.cuda.current_stream(dev).cuda_stream)
    _native.check(rc, "crag_knn_topk")
    torch.cuda.synchronize(dev)
    return ids, scores, minmax


def _search_after_chain(corpus, queries, k):
    """The scan path for k > 128: ceil(k/128) crag_search_topk_after calls, each continuing after the last one."""
    from comorag_b200 import _native
    lib = _native.load()
    n, dim = corpus.shape
    nq = queries.shape[0]
    dev = queries.device
    ids = torch.empty((nq, k), dtype=torch.int64, device=dev)
    scores = torch.empty((nq, k), dtype=torch.float32, device=dev)
    minmax = torch.empty((nq, 2), dtype=torch.float32, device=dev)
    ws_bytes = lib.crag_search_workspace_bytes(nq, 128)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    after = None
    for p0 in range(0, k, 128):
        kk = min(128, k - p0)
        p_ids = torch.empty((nq, kk), dtype=torch.int64, device=dev)
        p_sc = torch.empty((nq, kk), dtype=torch.float32, device=dev)
        last = torch.empty((nq,), dtype=torch.int64, device=dev)
        rc = lib.crag_search_topk_after(corpus.data_ptr(), n, dim, corpus.stride(0), 0, queries.data_ptr(), nq, kk,
                                        _native.ptr(after), p_ids.data_ptr(), p_sc.data_ptr(), minmax.data_ptr(),
                                        last.data_ptr(), ws.data_ptr(), ws_bytes, torch.cuda.current_stream(dev).cuda_stream)
        _native.check(rc, "crag_search_topk_after")
        ids[:, p0:p0 + kk], scores[:, p0:p0 + kk] = p_ids, p_sc
        after = last
    torch.cuda.synchronize(dev)
    return ids, scores, minmax


def _assert_ids_equal_outside_near_ties(got, want, want_scores, tie_tol=2e-6):
    """Vectorised: every rank whose score is more than tie_tol away from both neighbours holds the same id."""
    got, want, s = np.asarray(got), np.asarray(want), np.asarray(want_scores, dtype=np.float64)
    gap = np.full(s.shape, np.inf)
    gap[:, :-1] = s[:, :-1] - s[:, 1:]
    near = gap < tie_tol
    near[:, 1:] |= gap[:, :-1] < tie_tol
    near[:, -1] = True                    # the (k+1)-th row may tie the last one
    bad = (got != want) & ~near
    assert not bad.any(), f"{bad.sum()} ranks differ outside near-tie runs, first at {np.argwhere(bad)[0]}"


# ------------------------------------------------------------------------------------------------ score block
EDGES = [1, 127, 128, 129, 255]
DIMS = [64, 384, 768, 1024]


@pytest.mark.parametrize("m", EDGES)
@pytest.mark.parametrize("n", EDGES)
def test_score_block_equals_the_dot_products(dev, m, n):
    """k = n_rows returns every score of the block: each must equal the float64 dot product within 2e-6 (the bound
    test_score_all_pass_equals_the_dot_products holds the scan's wgmma tile to), at M and N tails of the 128 tile; odd
    cases read the corpus through a row stride wider than dim."""
    dim = DIMS[(EDGES.index(m) + EDGES.index(n)) % len(DIMS)]
    strided = (m + n) % 2 == 1
    rows = make_unit_rows(n, dim, 10 * m + n, device=dev)
    if strided:
        wide = torch.full((n, dim + 72), float("nan"), dtype=torch.bfloat16, device=dev)
        wide[:, :dim] = rows
        corpus = wide[:, :dim]
    else:
        corpus = rows
    queries = make_unit_rows(m, dim, 7 * m + n + 1, device=dev)
    ids, scores, minmax = _knn(corpus, queries, n, stride=corpus.stride(0))
    want = queries.double() @ rows.double().T
    assert sorted(ids[0].tolist()) == list(range(n))
    got_at = torch.gather(want, 1, ids)
    assert (scores.double() - got_at).abs().max().item() < 2e-6
    assert (scores[:, :-1] >= scores[:, 1:]).all()
    assert torch.equal(minmax[:, 0], scores[:, -1]) and torch.equal(minmax[:, 1], scores[:, 0])


# ------------------------------------------------------------------------------------------------------ top-k
KS = [1, 10, 128, 129, 1000, 2047, 2048]


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("rel", ["less", "equal", "more"])
def test_topk_matches_the_oracle(dev, k, rel):
    n = {"less": max(1, k - 3) if k > 1 else 1, "equal": k, "more": 3 * k + 517}[rel]
    if rel == "less" and k == 1:
        pytest.skip("no shard smaller than k = 1 except the empty one (tested on its own)")
    dim = 128 if k > 500 else 384
    corpus, queries = make_unit_rows(n, dim, 1000 + k + n), make_unit_rows(37, dim, 2000 + k)
    want_i, want_s, want_mm, gaps = so.topk_exact(corpus.float().numpy(), queries.float().numpy(), k, row_offset=5_000_000_000)
    ids, scores, minmax = _knn(corpus.to(dev), queries.to(dev), k, row_offset=5_000_000_000)
    so.assert_topk_matches(ids.cpu().numpy(), scores.double().cpu().numpy(), want_i, want_s, gaps, score_tol=2e-6)
    np.testing.assert_allclose(minmax.cpu().numpy(), want_mm, atol=2e-6)


def test_empty_shard(dev):
    from comorag_b200 import _native
    lib = _native.load()
    q = make_unit_rows(3, 64, 1, device=dev)
    corpus = torch.empty((0, 64), dtype=torch.bfloat16, device=dev)
    ids, scores, minmax = _knn(corpus, q, 300)
    assert (ids == -1).all() and torch.isneginf(scores).all()
    assert torch.isposinf(minmax[:, 0]).all() and torch.isneginf(minmax[:, 1]).all()
    assert lib.crag_knn_workspace_bytes(0, 3) > 0


@pytest.mark.parametrize("ws_queries", [1, 100, 129, 300])
def test_chunks_of_queries(dev, ws_queries):
    """nq = 700 over a workspace of 1 / 100 / 129 / 300 score rows: chunk edges that are not multiples of 128."""
    corpus, queries = make_unit_rows(3000, 256, 41, device=dev), make_unit_rows(700, 256, 42, device=dev)
    k = 300
    ids, scores, minmax = _knn(corpus, queries, k, ws_queries=ws_queries)
    whole = _knn(corpus, queries, k)
    assert torch.equal(ids, whole[0]) and torch.equal(scores, whole[1]) and torch.equal(minmax, whole[2])
    want_i, want_s, want_mm, gaps = torch_reference_topk(corpus, queries, k)
    so.assert_topk_matches(ids.cpu().numpy(), scores.double().cpu().numpy(), want_i, want_s, gaps, score_tol=2e-6)


@pytest.mark.parametrize("k", [10, 129, 2047])
def test_duplicated_corpus_ties_resolve_to_ascending_rows(dev, k):
    base = make_unit_rows(1500, 128, 7, device=dev)
    corpus = torch.cat([base, base])            # every score appears twice: row r and row r + 1500
    queries = make_unit_rows(9, 128, 8, device=dev)
    ids, scores, _ = _knn(corpus, queries, k)
    assert (ids[:, 0:k - 1:2] + 1500 == ids[:, 1:k:2]).all() and (scores[:, 0:k - 1:2] == scores[:, 1:k:2]).all()
    want_i, want_s, _, gaps = torch_reference_topk(corpus, queries, k)
    np.testing.assert_array_equal(ids.cpu().numpy(), want_i)


def test_constant_corpus(dev):
    corpus = make_unit_rows(1, 64, 3, device=dev).repeat(5000, 1)
    q = make_unit_rows(2, 64, 4, device=dev)
    for k in (1, 129, 2048):
        ids, scores, minmax = _knn(corpus, q, k)
        assert torch.equal(ids.cpu(), torch.arange(k).repeat(2, 1))
        assert (scores == scores[:, :1]).all() and torch.equal(minmax[:, 0], minmax[:, 1])


# ------------------------------------------------------------------------------------------------ cross-check
@pytest.mark.parametrize("k", [1, 10, 100, 128])
def test_ids_equal_the_scan_path_up_to_128(dev, k):
    corpus, queries = make_unit_rows(60_000, 1024, 51, device=dev), make_unit_rows(300, 1024, 52, device=dev)
    ids, scores, minmax = _knn(corpus, queries, k)
    s_ids, s_scores, s_mm = _scan(corpus, queries, k)
    _assert_ids_equal_outside_near_ties(ids.cpu().numpy(), s_ids.cpu().numpy(), s_scores.cpu().numpy())
    assert (scores - s_scores).abs().max().item() < 2e-6 and torch.equal(minmax, s_mm)


@pytest.mark.parametrize("k", [129, 1000, 2048])
def test_ids_equal_a_search_after_chain(dev, k):
    """The continuation ABI keeps its own GPU coverage: crag_search_topk_after, chained directly, against crag_knn_topk."""
    corpus, queries = make_unit_rows(40_000, 768, 61, device=dev), make_unit_rows(70, 768, 62, device=dev)
    ids, scores, minmax = _knn(corpus, queries, k)
    c_ids, c_scores, c_mm = _search_after_chain(corpus, queries, k)
    _assert_ids_equal_outside_near_ties(ids.cpu().numpy(), c_ids.cpu().numpy(), c_scores.cpu().numpy())
    assert (scores - c_scores).abs().max().item() < 2e-6 and torch.equal(minmax, c_mm)


def _scan(corpus, queries, k):
    from comorag_b200 import _native
    lib = _native.load()
    nq = queries.shape[0]
    dev = queries.device
    ids = torch.empty((nq, k), dtype=torch.int64, device=dev)
    scores = torch.empty((nq, k), dtype=torch.float32, device=dev)
    minmax = torch.empty((nq, 2), dtype=torch.float32, device=dev)
    ws_bytes = lib.crag_search_workspace_bytes(nq, k)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    rc = lib.crag_search_topk(corpus.data_ptr(), corpus.shape[0], corpus.shape[1], corpus.stride(0), 0, queries.data_ptr(),
                              nq, k, ids.data_ptr(), scores.data_ptr(), minmax.data_ptr(), ws.data_ptr(), ws_bytes,
                              torch.cuda.current_stream(dev).cuda_stream)
    _native.check(rc, "crag_search_topk")
    torch.cuda.synchronize(dev)
    return ids, scores, minmax


# ----------------------------------------------------------------------------------------------------- routing
def test_index_routes_many_queries_to_the_gemm_path(dev):
    from comorag_b200 import index as ix
    corpus, queries = make_unit_rows(20_000, 256, 71, device=dev), make_unit_rows(600, 256, 72, device=dev)
    idx = ix.DenseIndex.from_tensor(corpus, row_offset=123)
    assert ix.use_knn(600, 20_000, 1000) and ix.use_knn(20_000, 20_000, 10)
    assert not ix.use_knn(600, 20_000, 300) and not ix.use_knn(600, 10_000_000, 10)
    ids, scores, minmax = idx.search_device(queries, 1000)
    d_ids, d_scores, d_mm = _knn(corpus, queries, 1000, row_offset=123)
    assert torch.equal(ids, d_ids) and torch.equal(scores, d_scores) and torch.equal(minmax, d_mm)


@pytest.mark.parametrize("k", [2500, 4100])
def test_k_beyond_2048_keeps_the_paged_scan(dev, k):
    from comorag_b200 import index as ix
    corpus, queries = make_unit_rows(6000, 128, 81), make_unit_rows(5, 128, 82)
    assert not ix.use_knn(5, 6000, k) and not ix.use_knn(5000, 6000, k)
    idx = ix.DenseIndex.from_tensor(corpus.to(dev))
    ids, scores, minmax = idx.search(queries.float().numpy(), k)
    want_i, want_s, want_mm, gaps = so.topk_exact(corpus.float().numpy(), queries.float().numpy(), k)
    so.assert_topk_matches(ids, scores.astype(np.float64), want_i, want_s, gaps, score_tol=2e-6)


# ------------------------------------------------------------------------------------------------------ errors
def test_argument_errors(dev):
    from comorag_b200 import _native
    lib = _native.load()
    corpus, q = make_unit_rows(100, 64, 1, device=dev), make_unit_rows(2, 64, 2, device=dev)
    out_i = torch.empty((2, 2049), dtype=torch.int64, device=dev)
    out_s = torch.empty((2, 2049), dtype=torch.float32, device=dev)
    ws = torch.empty((1 << 20,), dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream

    def call(k, dim=64, cptr=corpus.data_ptr(), ws_bytes=1 << 20):
        return lib.crag_knn_topk(cptr, 100, dim, dim, 0, q.data_ptr(), 2, k, out_i.data_ptr(), out_s.data_ptr(), 0,
                                 ws.data_ptr(), ws_bytes, st)

    for k in (0, 2049):
        assert call(k) < 0 and b"k <= 2048" in lib.crag_last_error()
    assert call(10, dim=1088) < 0 and b"dim" in lib.crag_last_error()
    assert call(10, cptr=corpus.data_ptr() + 2) < 0 and b"aligned" in lib.crag_last_error()
    assert call(10, ws_bytes=100 * 4 - 1) == -3 and b"workspace" in lib.crag_last_error()
    assert call(10, ws_bytes=100 * 4) == 0


# ---------------------------------------------------------------------------------------------------- self-join
def test_retrieve_knn_self_join_at_k_2047(dev):
    """retrieve_knn (embed_utils.py:8-97) with every entity as a query against every entity, at the reference's
    synonymy_edge_topk = 2047 (ComoRAG.py:670-684): the exact answer on the stored bf16 rows."""
    from comorag_b200.retrieval import retrieve_knn
    n, dim, k = 5000, 256, 2047
    g = torch.Generator().manual_seed(91)
    vecs = torch.randn(n, dim, generator=g).numpy()
    names = [f"e{i}" for i in range(n)]
    res = retrieve_knn(names, names, vecs, vecs, k=k, device=dev)
    got_ids = np.array([[int(x[1:]) for x in res[f"e{i}"][0]] for i in range(n)])
    got_sc = np.array([res[f"e{i}"][1] for i in range(n)], dtype=np.float64)
    assert got_ids.shape == (n, k)
    assert all(len(set(r.tolist())) == k for r in got_ids) and np.all(np.diff(got_sc, axis=1) <= 0)
    rows = torch.nn.functional.normalize(torch.from_numpy(vecs), dim=1).bfloat16().to(dev)
    want_i, want_s, _, gaps = torch_reference_topk(rows, rows, k)
    _assert_ids_equal_outside_near_ties(got_ids, want_i, want_s)
    assert np.abs(got_sc - want_s).max() < 2e-6
    for qi in range(0, n, 97):
        so.assert_topk_matches(got_ids[qi:qi + 1], got_sc[qi:qi + 1], want_i[qi:qi + 1], want_s[qi:qi + 1], gaps[qi:qi + 1],
                               score_tol=2e-6)
