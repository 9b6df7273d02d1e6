"""crag_knn_topk on the GPU, bit for bit.

The score block of crag_knn_topk's wgmma GEMM (queries on the A side, m64n128k16) is compared with crag_search_scores
(score-all: corpus on the A side, m64n32k16): both start from zero fp32 accumulators and run the same K-block order,
so every score must be bit-identical, and the score-all bound SCORE_BOUND against float64 then holds for both.  With
the block pinned, everything else is exact: the top-k of crag_knn_topk must equal, in ids, scores and (min, max),
tests/scan_reference.py's topk_from_scores of the score-all matrix -- at k, n_rows and query-chunk edges, on integer
corpora whose exact scores need no kernel and which reach each regime of the radix select (tests/knn_cases.py), past
65 535 column tiles and over many query blocks.  DenseIndex then has to answer a query the same whether its batch
routes to crag_knn_topk or to the scan, and repeated calls and concurrent streams must agree bit for bit.
test_score_block_equals_score_all records its worst err/bound as `worst_err_over_bound`."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import knn_cases as kc  # noqa: E402
import scan_reference as sr  # noqa: E402
from test_scan_exact_gpu import score_all  # noqa: E402
from util_search import make_unit_rows  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SENTINEL = 0x7FA5A5A5            # a NaN payload no kernel writes: the canary around every output
ID_SENTINEL = -7
PAD = 8                          # canary elements before and after every output
BIG_OFFSET = (1 << 33) + 7
INF_BITS, NAN_BITS = 0x7F800000, 0x7FC00000


@pytest.fixture(scope="module", autouse=True)
def lib():
    assert torch.cuda.is_available()
    from comorag_b200 import _native
    return _native.load()


def _lib():
    from comorag_b200 import _native
    return _native.load()


# ----------------------------------------------------------------------------------------------------- native call
def launch_knn(rows, queries, k, row_offset=0, ws_queries=None, stream=None):
    """Enqueue crag_knn_topk of rows (bf16 [n, dim], any row stride) against queries (bf16 [nq, dim]).  Outputs sit
    between canaries, and the workspace is filled with +inf / NaN words, so a select that read the unwritten columns
    [n, ld) of the score block would rank them first.  ws_queries sizes the workspace for that many score rows."""
    from comorag_b200 import _native
    lib = _lib()
    n, dim = rows.shape
    q = queries.contiguous()
    nq = q.shape[0]
    ids = torch.full((nq * k + 2 * PAD,), ID_SENTINEL, dtype=torch.int64, device=DEV)
    sc = torch.full((nq * k + 2 * PAD,), SENTINEL, dtype=torch.int32, device=DEV)
    mm = torch.full((nq * 2 + 2 * PAD,), SENTINEL, dtype=torch.int32, device=DEV)
    ws_bytes = lib.crag_knn_workspace_bytes(n, ws_queries or nq)
    ws = torch.empty(ws_bytes // 4, dtype=torch.int32, device=DEV)
    ws[0::2], ws[1::2] = INF_BITS, NAN_BITS
    st = (stream or torch.cuda.current_stream()).cuda_stream
    if stream is not None:
        stream.wait_stream(torch.cuda.current_stream())
    rc = lib.crag_knn_topk(rows.data_ptr() if n else 0, n, dim, rows.stride(0) if n else dim, row_offset, q.data_ptr(),
                           nq, k, ids[PAD:].data_ptr(), sc[PAD:].data_ptr(), mm[PAD:].data_ptr(), ws.data_ptr(), ws_bytes,
                           st)
    _native.check(rc, "crag_knn_topk")
    return nq, k, ids, sc, mm, ws, q


def finish_knn(launched):
    """(ids int64 [nq, k], scores fp32 [nq, k], minmax fp32 [nq, 2]) after checking every canary."""
    nq, k, ids, sc, mm, _, _ = launched
    torch.cuda.synchronize()
    for buf, fill, what in ((ids, ID_SENTINEL, "ids"), (sc, SENTINEL, "scores"), (mm, SENTINEL, "minmax")):
        assert bool((buf[:PAD] == fill).all()) and bool((buf[buf.numel() - PAD:] == fill).all()), f"wrote outside {what}"
    return (ids[PAD:PAD + nq * k].view(nq, k), sc[PAD:PAD + nq * k].view(torch.float32).view(nq, k),
            mm[PAD:PAD + 2 * nq].view(torch.float32).view(nq, 2))


def knn(rows, queries, k, row_offset=0, ws_queries=None):
    return finish_knn(launch_knn(rows, queries, k, row_offset, ws_queries))


def assert_topk(got, want, what=""):
    for j, name in enumerate(("ids", "scores", "minmax")):
        sr.assert_bits(got[j], want[j], f"{name} {what}")


# ------------------------------------------------------------------------------------------ 1. score block = score-all
DIMS = list(range(64, 1025, 64))
EDGES = [1, 127, 128, 129, 255, 2048]
PADS = [0, 8, 64]


@pytest.mark.parametrize("dim", DIMS)
def test_score_block_equals_score_all(record_property, dim):
    """k = n_rows <= 2048 takes the sort-only path and returns every score of the block: scattered back by id it
    must be a permutation of the rows, bit-identical to crag_search_scores and within SCORE_BOUND of float64.  Every
    K-block count 1 .. 16; n_rows and nq rotate through the M and N tile tails (odd n_rows splits the float2 store);
    a row stride above dim with NaN in the gap on two of three dims; unit and scaled rows."""
    i = dim // 64 - 1
    n, nq = EDGES[i % len(EDGES)], EDGES[(i + 3 + i // len(EDGES)) % len(EDGES)]
    worst = 0.0
    for kind in ("unit", "scaled"):
        x = make_unit_rows(n, dim, 20 + i, device=DEV)
        q = make_unit_rows(nq, dim, 60 + i, device=DEV)
        if kind == "scaled":
            x, q = kc.scaled(x), kc.scaled(q)
        xs, _ = kc.strided(x, PADS[i % 3])
        ids, sc, mm = knn(xs, q, n)
        assert torch.equal(ids.sort(dim=1).values, torch.arange(n, device=DEV).expand(nq, n)), "not a permutation"
        block = torch.empty((nq, n), dtype=torch.float32, device=DEV).scatter_(1, ids, sc)
        S, _ = score_all(xs, q)
        sr.assert_bits(block, S, f"{kind}: knn score block vs score-all")
        ref, mag = sr.score_reference(q, x)
        r = sr.err_over_bound(block, ref, mag)
        assert r <= 1.0, f"{kind}: worst err/bound {r:.3f}"
        worst = max(worst, r)
        assert_topk((ids, sc, mm), sr.topk_from_scores(S, n)[:3], kind)
    record_property("worst_err_over_bound", worst)


# ------------------------------------------------------------------------------------------------- 2. top-k exact
TOPK_K = [1, 2, 127, 128, 129, 641, 1000, 2047, 2048]
N_Q = [1, 129, 700]
WS_Q = [1, 100, 129, 300]
KINDS = ["unit", "dyadic", "near_dup"]


@pytest.mark.parametrize("k", TOPK_K)
def test_topk_equals_reference_of_score_all(k):
    """Ids, scores and (min, max) bit for bit against topk_from_scores(score-all) for n_rows in {0, 1, k - 1, k,
    k + 1, 4 097, 100 003}, with nq, the workspace's queries per chunk (1 / 100 / 129 / 300), the corpus kind, dim and
    row stride rotating across the shapes; ids offset beyond 2^33."""
    ki = TOPK_K.index(k)
    shapes = sorted({0, 1, max(k - 1, 1), k, k + 1, 4097, 100_003})
    for j, n in enumerate(shapes):
        nq = N_Q[(ki + j) % len(N_Q)]
        ws_q = WS_Q[(ki + j) % len(WS_Q)]
        kind = KINDS[(ki + j) % len(KINDS)]
        dim = 64 * (1 + (ki + j) % 4)
        q = kc.queries_for(kind, nq, dim, 500 + 10 * ki + j)
        what = f"n={n} nq={nq} chunk={ws_q} {kind} dim={dim}"
        if n == 0:
            ids, sc, mm = knn(torch.empty((0, dim), dtype=torch.bfloat16, device=DEV), q, k, BIG_OFFSET, ws_q)
            assert bool((ids == -1).all()) and bool(torch.isneginf(sc).all()), what
            assert bool(torch.isposinf(mm[:, 0]).all()) and bool(torch.isneginf(mm[:, 1]).all()), what
            continue
        x = kc.corpus(kind, n, dim, 600 + 10 * ki + j)
        xs, _ = kc.strided(x, 8 * (j % 2))
        got = knn(xs, q, k, BIG_OFFSET, ws_q)
        S, _ = score_all(xs, q)
        assert_topk(got, sr.topk_from_scores(S, k, row_offset=BIG_OFFSET)[:3], what)


# ---------------------------------------------------------------------------------------------- 3. regime cases
@pytest.mark.parametrize("name", sorted(kc.INT_CASES))
def test_regime_case_equals_its_exact_scores(name):
    """The integer corpora of knn_cases.py against their planned scores, which need no kernel: each radix pass
    deciding, tie runs of thousands at k = 129 / 1 000 / 2 048 cut mid-iteration, ties from row 0 and to the last
    row, all-negative scores, a constant corpus and copies 2 048 rows apart.  Query scales 1, 2^-12 and -2^6; rows
    read through a row stride above dim on every other case."""
    rows, q, S, k, _ = kc.int_case(name, device=DEV)
    want = sr.topk_from_scores(S.float(), k, row_offset=BIG_OFFSET)[:3]
    xs, _ = kc.strided(rows, 64 * (sorted(kc.INT_CASES).index(name) % 2))
    sr.assert_bits(score_all(xs, q)[0], S.float(), "score-all of an exact corpus")
    assert_topk(knn(xs, q, k, BIG_OFFSET), want, name)
    assert_topk(knn(xs, q, k, BIG_OFFSET, ws_queries=1), want, f"{name}, one query per chunk")


# ------------------------------------------------------------------------------------------------- 4. grid limits
def test_more_than_65535_column_tiles():
    """65 535 * 128 + 200 rows at dim 64 (about 1.1 GB): the 1-D grid's column tiles run past 65 535.  The best rows
    for each query are planted in the last tiles, so a grid that stopped short would change every answer."""
    n, dim = 65_535 * 128 + 200, 64
    q = make_unit_rows(3, dim, 31, device=DEV)
    x = make_unit_rows(n, dim, 32, device=DEV)
    tail = n - 150 + torch.arange(0, 150, 50, device=DEV)            # rows in tiles 65 535 and 65 536
    x[tail] = q
    assert (n + 127) // 128 > 65_535 and int(tail[0]) >= 65_535 * 128
    from comorag_b200 import index as ix
    S, _ = score_all(x, q)
    for k in (641, 2048):
        assert ix.use_knn(3, n, k)
        got = knn(x, q, k, BIG_OFFSET)
        want = sr.topk_from_scores(S, k, row_offset=BIG_OFFSET)[:3]
        assert_topk(got, want, f"k={k}")
        assert torch.equal(got[0][:, 0].cpu(), tail.cpu() + BIG_OFFSET)


@pytest.mark.parametrize("k", [129, 2048])
def test_many_query_blocks(k):
    """nq = 20 000 against 3 000 rows: 157 query blocks times 24 column tiles on the 1-D grid, one chunk."""
    x = kc.corpus("near_dup", 3000, 128, 41)
    q = make_unit_rows(20_000, 128, 42, device=DEV)
    S, _ = score_all(x, q)
    assert_topk(knn(x, q, k), sr.topk_from_scores(S, k)[:3], f"k={k}")


# ---------------------------------------------------------------------------------------- 5. routing independence
def _index(dim, n, seed):
    from comorag_b200.index import DenseIndex
    x = kc.corpus("near_dup", n, dim, seed)
    idx = DenseIndex(dim, device=DEV, row_offset=BIG_OFFSET)
    idx.add(x)
    return idx


@pytest.mark.parametrize("dim", [128, 100])
def test_dense_index_answers_do_not_depend_on_routing(dim):
    """The same 10 000 queries as one batch (crag_knn_topk) and as three slices (the scan): bit-identical for
    k = 10 and 128, and equal to the reference of score-all; k = 640 on 50 queries (the paged scan) equals the first
    640 of k = 641 (crag_knn_topk).  At dim 100 the index pads rows and queries with zero columns to 128."""
    from comorag_b200 import index as ix
    n = 50_000
    idx = _index(dim, n, 51)
    q = idx.prepare_queries(make_unit_rows(10_000, dim, 52).float())
    S, _ = idx.scores_device(q)
    for k in (10, 128):
        assert ix.use_knn(10_000, n, k) and not ix.use_knn(3_500, n, k)
        whole = idx.search_device(q, k)
        parts = [idx.search_device(q[a:b], k) for a, b in ((0, 3_000), (3_000, 6_500), (6_500, 10_000))]
        torch.cuda.synchronize()
        assert_topk(whole, [torch.cat([p[j] for p in parts]) for j in range(3)], f"k={k}: knn batch vs scan slices")
        assert_topk(whole, sr.topk_from_scores(S, k, row_offset=BIG_OFFSET)[:3], f"k={k} vs score-all")
    few = q[:50]
    assert not ix.use_knn(50, n, 640) and ix.use_knn(50, n, 641)
    scan = idx.search_device(few, 640)
    gemm = idx.search_device(few, 641)
    torch.cuda.synchronize()
    assert_topk(scan, (gemm[0][:, :640], gemm[1][:, :640], gemm[2]), "k=640 paged scan vs k=641 knn")
    assert_topk(gemm, sr.topk_from_scores(S[:50], 641, row_offset=BIG_OFFSET)[:3], "k=641 vs score-all")


def test_retrieve_knn_self_join_is_exact():
    """retrieve_knn's self-join sends groups of 1 024 queries: k = 2047 takes crag_knn_topk and must equal the
    reference built from the index's own bf16 rows; k = 640 takes the paged scan and must equal its first 640."""
    from comorag_b200 import index as ix
    from comorag_b200.retrieval import retrieve_knn
    n, dim = 3000, 256
    vecs = torch.randn(n, dim, generator=torch.Generator().manual_seed(91)).numpy()
    names = [f"e{i}" for i in range(n)]
    kv = torch.nn.functional.normalize(torch.as_tensor(vecs, dtype=torch.float32), dim=1)
    idx = ix.DenseIndex(dim, device=DEV, capacity=n)
    idx.add(kv)
    m = idx.matrix()
    S, _ = score_all(m, m.contiguous())

    def run(k):
        assert ix.use_knn(1024, n, k) == (k > 640)
        res = retrieve_knn(names, names, vecs, vecs, k=k, device=DEV)
        ids = torch.tensor([[int(x[1:]) for x in res[f"e{i}"][0]] for i in range(n)])
        sc = torch.tensor(np.array([res[f"e{i}"][1] for i in range(n)], dtype=np.float64)).float()
        return ids, sc

    ids, sc = run(2047)
    w_ids, w_sc, _, _ = sr.topk_from_scores(S, 2047)
    sr.assert_bits(ids, w_ids, "ids k=2047")
    sr.assert_bits(sc, w_sc, "scores k=2047")
    ids640, sc640 = run(640)
    sr.assert_bits(ids640, ids[:, :640], "ids k=640 vs k=2047")
    sr.assert_bits(sc640, sc[:, :640], "scores k=640 vs k=2047")


# ----------------------------------------------------------------------------------------------- 6. determinism
def test_repeats_and_streams_are_bit_identical():
    """The long-tie corpus at k = 2048 and unit rows at k = 1000: three repeats on the current stream, then two side
    streams at once, each with its own workspace and outputs, all bit-identical."""
    rows, q, _, k, _ = kc.int_case("long_tie_2048", device=DEV)
    x = make_unit_rows(30_000, 256, 71, device=DEV)
    qu = make_unit_rows(300, 256, 72, device=DEV)
    for r, qq, kk in ((rows, q, k), (x, qu, 1000)):
        first = knn(r, qq, kk, BIG_OFFSET)
        for _ in range(2):
            assert_topk(knn(r, qq, kk, BIG_OFFSET), first, "repeat")
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        launched = [launch_knn(r, qq, kk, BIG_OFFSET, ws_queries=100, stream=s) for s in streams]
        for lt in launched:
            assert_topk(finish_knn(lt), first, "side stream")
