"""crag_knn_threshold on the GPU, bit for bit.

Its score block is crag_knn_topk's (the same GEMM call), so with the block pinned by tests/test_knn_exact_gpu.py the
threshold join is exact: counts, ids and scores must equal the numpy walk of tests/synonymy_oracle.py over
scan_reference.topk_from_scores of the score-all matrix -- on the integer corpora of tests/knn_cases.py, whose scores
are exact, and on unit rows against crag_knn_topk(k = limit) followed by the same walk.  Query-chunk edges with a small
workspace, an overflow of more than 2 048 duplicate rows, canaries around every output, two streams, every argument
error, and add_synonymy_edges end to end on a planted self-join against the reference loop over retrieve_knn."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import knn_cases as kc  # noqa: E402
import scan_reference as sr  # noqa: E402
import synonymy_oracle as so  # noqa: E402
from test_knn_exact_gpu import knn  # noqa: E402
from test_scan_exact_gpu import score_all  # noqa: E402
from util_search import make_unit_rows  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SENTINEL = 0x7FA5A5A5
ID_SENTINEL = -7
PAD = 8


def _lib():
    from comorag_b200 import _native
    return _native.load()


def launch(rows, queries, threshold, limit, cap, self_rows=None, exclude=(), ws_queries=None, stream=None):
    """Enqueue crag_knn_threshold; outputs between canaries, the workspace filled with +inf / NaN words."""
    lib = _lib()
    n, dim = rows.shape
    q = queries.contiguous()
    nq = q.shape[0]
    cnt = torch.full((nq + 2 * PAD,), SENTINEL, dtype=torch.int32, device=DEV)
    ids = torch.full((nq * cap + 2 * PAD,), ID_SENTINEL, dtype=torch.int64, device=DEV)
    sc = torch.full((nq * cap + 2 * PAD,), SENTINEL, dtype=torch.int32, device=DEV)
    ws_bytes = lib.crag_knn_workspace_bytes(n, ws_queries or nq)
    ws = torch.empty(ws_bytes // 4, dtype=torch.int32, device=DEV)
    ws[0::2], ws[1::2] = 0x7F800000, 0x7FC00000
    selfr = None if self_rows is None else torch.as_tensor(self_rows, dtype=torch.int64, device=DEV)
    excl = torch.as_tensor(list(exclude), dtype=torch.int64, device=DEV)
    if stream is not None:
        stream.wait_stream(torch.cuda.current_stream())
    st = (stream or torch.cuda.current_stream()).cuda_stream
    rc = lib.crag_knn_threshold(rows.data_ptr() if n else 0, n, dim, rows.stride(0) if n else dim, q.data_ptr(), nq,
                                float(threshold), limit, cap, 0 if selfr is None else selfr.data_ptr(),
                                excl.data_ptr() if excl.numel() else 0, excl.numel(), cnt[PAD:].data_ptr(),
                                ids[PAD:].data_ptr(), sc[PAD:].data_ptr(), ws.data_ptr(), ws_bytes, st)
    from comorag_b200 import _native
    _native.check(rc, "crag_knn_threshold")
    return nq, cap, cnt, ids, sc, (ws, selfr, excl, q)


def finish(launched):
    nq, cap, cnt, ids, sc, _ = launched
    torch.cuda.synchronize()
    for buf, fill, what in ((cnt, SENTINEL, "counts"), (ids, ID_SENTINEL, "ids"), (sc, SENTINEL, "scores")):
        assert bool((buf[:PAD] == fill).all()) and bool((buf[buf.numel() - PAD:] == fill).all()), f"wrote outside {what}"
    return (cnt[PAD:PAD + nq].cpu().numpy(), ids[PAD:PAD + nq * cap].view(nq, cap).cpu().numpy(),
            sc[PAD:PAD + nq * cap].view(torch.float32).view(nq, cap).cpu().numpy())


def threshold_join(*a, **kw):
    return finish(launch(*a, **kw))


def assert_same(got, want, what=""):
    for j, name in enumerate(("counts", "ids", "scores")):
        g, w = np.asarray(got[j]), np.asarray(want[j])
        assert g.shape == w.shape and g.tobytes() == w.tobytes(), f"{name} {what}"


def want_from_scores(S, threshold, limit, cap, self_rows=None, exclude=()):
    """The walk over the exact top-min(limit, n) list of topk_from_scores (crag_knn_topk's contract)."""
    S = S.float()
    n = S.shape[1]
    k = min(limit, n, 2048)
    ids, sc, _, _ = sr.topk_from_scores(S, k)
    return walk_lists(ids.cpu().numpy(), sc.cpu().numpy(), threshold, cap, self_rows, exclude, limit <= 2048 or n <= 2048)


def walk_lists(ids, sc, threshold, cap, self_rows=None, exclude=(), complete=True):
    nq = ids.shape[0]
    counts = np.zeros(nq, dtype=np.int32)
    out_i = np.full((nq, cap), -1, dtype=np.int64)
    out_s = np.full((nq, cap), -np.inf, dtype=np.float32)
    skip = set(int(r) for r in exclude)
    t = np.float32(threshold)
    for q in range(nq):
        me = -1 if self_rows is None else int(self_rows[q])
        for r, s in zip(ids[q].tolist(), sc[q].tolist()):
            if counts[q] == cap or r < 0 or not (np.float32(s) >= t):
                break
            if r == me or r in skip:
                continue
            out_i[q, counts[q]], out_s[q, counts[q]] = r, s
            counts[q] += 1
        else:
            assert complete or counts[q] == cap, "the reference list ended before the walk did"
    return counts, out_i, out_s


# ------------------------------------------------------------------------------------------------ exact corpora
@pytest.mark.parametrize("name", sorted(kc.INT_CASES))
def test_integer_corpora_equal_the_walk_over_score_all(name):
    """Thresholds on the planned integer scores: at, just above and below a tie level; the list limit at the case's k
    and at 2047; self rows and excluded rows taken from the top of each list."""
    rows, q, S, k, _ = kc.int_case(name, device=DEV)
    Sf = score_all(rows, q)[0]
    sr.assert_bits(Sf, S.float(), "score-all of an exact corpus")
    ids, _, _, _ = sr.topk_from_scores(Sf, min(k, rows.shape[0]))
    top = ids[:, 0].cpu().numpy()
    excl = [int(ids[0, min(3, ids.shape[1] - 1)]), int(ids[1, 0])]
    for qi in range(q.shape[0]):
        for t in (float(Sf[qi, ids[qi, min(k, ids.shape[1]) - 1]]), float(Sf[qi, ids[qi, 0]]), -1e9):
            for limit, cap in ((k, 101), (2047, 1983), (5, 2000)):
                for self_rows in (None, top[qi:qi + 1]):
                    got = threshold_join(rows, q[qi:qi + 1], t, limit, cap, self_rows, excl[: (2047 - cap) // 2 + 1])
                    want = want_from_scores(Sf[qi:qi + 1], t, limit, cap, self_rows, excl[: (2047 - cap) // 2 + 1])
                    assert_same(got, want, f"{name} q={qi} t={t} limit={limit} cap={cap}")


def test_overflow_of_more_than_2048_duplicate_rows():
    """5 000 copies of each query among 20 000 rows: every query has > 2 048 rows at its top score."""
    dim = 256
    q = make_unit_rows(4, dim, 11, device=DEV)
    x = make_unit_rows(20_000, dim, 12, device=DEV)
    x[:5000], x[5000:10000], x[10000:12500], x[17500:] = q[0], q[1], q[2], q[3]
    S = score_all(x, q)[0]
    for limit, cap, excl in ((2047, 101, [0, 5001, 3]), (4000, 1983, list(range(7, 7 + 64))), (10, 101, [])):
        got = threshold_join(x, q, 0.5, limit, cap, [0, 5000, 10000, 19999], excl)
        assert (got[0] == min(cap, limit - 1)).sum() >= 2, got[0]
        assert_same(got, want_from_scores(S, 0.5, limit, cap, [0, 5000, 10000, 19999], excl), f"limit={limit}")


@pytest.mark.parametrize("ws_q", [1, 100, 129])
def test_unit_rows_equal_knn_topk_then_the_walk(ws_q):
    """Unit rows with planted near-duplicates, query chunks forced small: against crag_knn_topk(k = limit) + walk."""
    n, dim, nq = 7001, 384, 300
    x = make_unit_rows(n, dim, 21, device=DEV)
    src = torch.randint(0, n, (n // 3,), generator=torch.Generator().manual_seed(3)).to(DEV)
    x[torch.arange(1, n, 3, device=DEV)[: src.numel()]] = torch.nn.functional.normalize(
        x[src].float() + 0.05 * make_unit_rows(src.numel(), dim, 22, device=DEV).float(), dim=1).bfloat16()
    rows = torch.arange(0, nq * 7, 7, device=DEV)
    q = x[rows]
    from comorag_b200.index import fp32_threshold
    for t, limit, cap in ((0.8, 2047, 101), (0.7, 2047, 101), (0.0, 300, 101), (0.9, 3, 2)):
        ft = fp32_threshold(t)
        ids, sc, _ = knn(x, q, limit, 0, ws_q)
        want = walk_lists(ids.cpu().numpy(), sc.cpu().numpy(), ft, cap, rows.cpu().numpy(), [5])
        got = threshold_join(x, q, ft, limit, cap, rows, [5], ws_queries=ws_q)
        assert_same(got, want, f"t={t} limit={limit} chunk={ws_q}")


def test_two_streams_and_repeats_are_bit_identical():
    x = make_unit_rows(30_000, 256, 31, device=DEV)
    q = x[:500]
    first = threshold_join(x, q, 0.1, 2047, 101, torch.arange(500))
    assert_same(threshold_join(x, q, 0.1, 2047, 101, torch.arange(500)), first, "repeat")
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    launched = [launch(x, q, 0.1, 2047, 101, torch.arange(500), ws_queries=77, stream=s) for s in streams]
    for lt in launched:
        assert_same(finish(lt), first, "side stream")


CRAG_ERR_INVALID, CRAG_ERR_WORKSPACE = -1, -3


def test_argument_errors():
    lib = _lib()
    x = make_unit_rows(100, 64, 1, device=DEV)
    q = x[:2].contiguous()
    cnt = torch.zeros(2, dtype=torch.int32, device=DEV)
    ids = torch.zeros(2 * 2048, dtype=torch.int64, device=DEV)
    sc = torch.zeros(2 * 2048, dtype=torch.float32, device=DEV)
    excl = torch.zeros(65, dtype=torch.int64, device=DEV)
    wsb = lib.crag_knn_workspace_bytes(100, 2)
    ws = torch.empty(wsb, dtype=torch.uint8, device=DEV)

    def call(t=0.5, limit=10, cap=5, n_ex=0, c=cnt.data_ptr(), i=ids.data_ptr(), s=sc.data_ptr(), ex=excl.data_ptr(),
             wb=wsb, nq=2):
        return lib.crag_knn_threshold(x.data_ptr(), 100, 64, 64, q.data_ptr(), nq, t, limit, cap, 0, ex, n_ex, c, i, s,
                                      ws.data_ptr(), wb, torch.cuda.current_stream().cuda_stream)
    assert call() == 0
    torch.cuda.synchronize()
    invalid = [dict(t=float("nan")), dict(t=float("inf")), dict(t=float("-inf")), dict(limit=0), dict(cap=0),
               dict(n_ex=-1), dict(n_ex=65), dict(cap=2048 - 64, n_ex=64), dict(cap=2048), dict(c=0), dict(i=0),
               dict(s=0), dict(n_ex=3, ex=0), dict(nq=0)]
    for kw in invalid:
        assert call(**kw) == CRAG_ERR_INVALID, kw
    assert call(cap=2048 - 64 - 1, n_ex=64) == 0
    assert call(wb=100 * 4 - 1) == CRAG_ERR_WORKSPACE                         # less than one score row
    assert call(wb=256 * 2) == 0                                             # one row per chunk
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ the method
def test_add_synonymy_edges_on_a_planted_self_join():
    """20 000 entities at dim 1 024 in synonym groups of 1 to 3 000 rows: node_to_node_stats of the device method
    equals, as list(items()), the reference loop over retrieval.retrieve_knn(k = 2047)'s lists."""
    from types import SimpleNamespace
    from comorag_b200 import comorag_methods as cm
    from comorag_b200.retrieval import retrieve_knn
    n, dim = 20_000, 1024
    rng = np.random.default_rng(7)
    sizes = [3000, 1500, 700, 200, 50, 10, 3, 2] + [1] * 100
    groups = []
    for g, size in enumerate(sizes):
        groups += [g] * size
    groups += list(range(len(sizes), len(sizes) + n - len(groups)))
    centers = rng.standard_normal((max(groups) + 1, dim)).astype(np.float32)
    emb = centers[np.asarray(groups)] + 0.3 * rng.standard_normal((n, dim)).astype(np.float32)
    texts = [f"entity {i}" for i in range(n)]
    texts[17], texts[3001] = "", "ab"
    hash_ids = [f"entity-{i:05d}" for i in range(n)]
    store = SimpleNamespace(get_text_for_all_rows=lambda: {h: {"hash_id": h, "content": t} for h, t in zip(hash_ids, texts)},
                            get_embeddings=lambda keys: emb[[int(k[7:]) for k in keys]])
    cfg = SimpleNamespace(synonymy_edge_topk=2047, synonymy_edge_sim_threshold=0.8, synonymy_edge_query_batch_size=1000,
                          synonymy_edge_key_batch_size=10000)
    pre = {(hash_ids[0], hash_ids[1]): 1.0, (hash_ids[5], hash_ids[9]): 2.0}
    rag = SimpleNamespace(entity_embedding_store=store, global_config=cfg, node_to_node_stats=dict(pre))
    cm.add_synonymy_edges(rag)
    knn_lists = retrieve_knn(hash_ids, hash_ids, emb, emb, k=2047, device=DEV)
    want = dict(pre)
    for edge, score in so.edges_from_knn(knn_lists, dict(zip(hash_ids, texts)), 0.8, cm.SYNONYMY_CAP):
        want[edge] = score
    got = list(rag.node_to_node_stats.items())
    assert got == list(want.items())
    assert len(got) > 3000 * 101
