"""End to end: the reference's UNMODIFIED ComoRAG.index() + try_answer() on its bundled cinderella sample (BASELINE
config 1; entry point main_openai.py:23-25), driven offline by tests/e2e_harness.py (LLM stub, igraph/umap/tiktoken
stand-ins), once on the reference's own classes (CPU, fp32 HF encoder + numpy search) and once on the comorag_b200 shim
(cuda:0) -- then the retrieved ids / scores of every question and probe are compared.

The reference tree is not in this repository: the tests use the unmodified copy build() stages under oracle/_ref
(oracle/stage_reference.py) or the checkout $COMORAG_REFERENCE names, and skip when neither exists.
"""
import json
import os
import sys
import tempfile

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import e2e_harness as H  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "e2e_cinderella_reference.json")
REF_ROOT = H.find_reference_root()
needs_ref = pytest.mark.skipif(REF_ROOT is None, reason="reference tree not present (build() stages it under oracle/_ref)")

_cache = {}


def reference_arm():
    if "ref" not in _cache:
        with tempfile.TemporaryDirectory() as tmp:
            _cache["ref"] = H.run_cinderella("reference", tmp, REF_ROOT)
    return _cache["ref"]


def test_llm_stub_covers_every_prompt_family():
    sysm = lambda s: [{"role": "system", "content": s}]
    ner = json.loads(H.llm_reply(sysm("Your task is to extract named entities from the given paragraph.") +
                                 [{"role": "user", "content": "Cinderella went to the Palace with the Prince."}]))
    assert ner["named_entities"][:3] == ["Cinderella", "Palace", "Prince"]
    tri = json.loads(H.llm_reply(sysm("Your task is to construct an RDF graph") + [{"role": "user", "content":
                     "Paragraph:\n```\nx\n```\n\n" + json.dumps({"named_entities": ["A", "B"]})}]))
    assert ["A", "appears with", "B"] in tri["triples"]
    qa = H.llm_reply(sysm("qa") + [{"role": "user", "content": "### Detail Chunks\nabc\n\nQuestion: q\nThought: "}])
    assert qa.split("### Final Answer")[1].strip() == "*"
    qa2 = H.llm_reply(sysm("qa") + [{"role": "user", "content": "### Historical Information\nx\n\nQuestion: q\nThought: "}])
    assert qa2.split("### Final Answer")[1].strip() == "Cinderella"
    probes = json.loads(H.llm_reply(sysm("You are an expert in multi-turn retrieval-oriented probe generation.") +
                                    [{"role": "user", "content": "Original Query:\nHow did the prince find her?\n\nContext:\n"}]))
    assert sorted(probes) == ["probe_1", "probe_2"]


def test_igraph_stand_in_pagerank_is_a_distribution():
    g = H._Graph()
    g.add_vertices(4, attributes={"name": list("abcd")})
    g.add_edges([("a", "b"), ("b", "c"), ("c", "d")], attributes={"weight": [1.0, 2.0, 1.0]})
    p = g.personalized_pagerank(vertices=range(4), damping=0.5, reset=[1, 0, 0, 0])
    assert abs(sum(p) - 1.0) < 1e-9 and p[0] > p[1] > p[2] > p[3]


@needs_ref
def test_reference_arm_reproduces_the_committed_trace():
    """The reference's own classes, run here, give the trace that was committed from the build container: the loop is
    deterministic under the harness, so the fixture pins the reference side of the comparison."""
    out = reference_arm()
    gold = json.load(open(GOLDEN))
    assert {k: sorted(v) for k, v in out["stores"].items()} == {k: sorted(v) for k, v in gold["stores"].items()}
    assert out["answers"] == gold["answers"]
    assert set(out["trace"]) == set(gold["trace"])
    # run-to-run the reference moves by ~3e-5 in normalised score (fp32 padding-batch effects: a text's batch
    # companions depend on thread completion order), nothing more
    summary = H.compare_traces(gold, out, raw_tol=0.0, floor_tol=5e-4)
    assert not summary["problems"], summary["problems"]
    assert summary["queries"] == len(gold["trace"]) == 12
    # the char-iteration bug (ComoRAG.py:470, 909-935): each tri_retrieve encodes len(query) single characters twice
    assert out["query_encodes"]["encoded_texts"] > 20 * len(out["trace"])


def _count_device_calls():
    from comorag_b200 import index as crag_index
    calls = {"scores": 0, "rank": 0, "topk": 0}
    real = (crag_index.DenseIndex.scores_device, crag_index.DenseIndex.rank_device, crag_index.DenseIndex.search_device)

    def counting(name, fn):
        def inner(self, *a, **kw):
            calls[name] += 1
            return fn(self, *a, **kw)
        return inner
    crag_index.DenseIndex.scores_device = counting("scores", real[0])
    crag_index.DenseIndex.rank_device = counting("rank", real[1])
    crag_index.DenseIndex.search_device = counting("topk", real[2])

    def restore():
        (crag_index.DenseIndex.scores_device, crag_index.DenseIndex.rank_device, crag_index.DenseIndex.search_device) = real
    return calls, restore


def _report(name, payload):
    out = os.path.join(os.path.dirname(HERE), "gpurun_out")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, name), "w") as f:
        json.dump(payload, f, indent=1)


@needs_ref
@pytest.mark.gpu
def test_unmodified_comorag_search_half_on_the_device_matches_the_reference_rankings():
    """install(encoder=False): the reference's own fp32 encoder feeds OUR stores, and unmodified ComoRAG.py runs its
    fact / passage / summary / timeline searches and the synonymy kNN on the device kernels.  Only the bf16 storage
    of rows and queries separates the two arms: raw inner products may move by <= 4e-3, i.e. normalised scores by
    that over the result's raw range, and rankings must be consistent within the measured deviation."""
    ref = reference_arm()
    calls, restore = _count_device_calls()
    try:
        with tempfile.TemporaryDirectory() as tmp:
            got = H.run_cinderella("shim_search", tmp, REF_ROOT)
    finally:
        restore()
        import comorag_b200.install as crag
        crag.uninstall_search("src.comorag")
    summary = H.compare_traces(ref, got, raw_tol=4e-3)
    _report("e2e_search_half.json", {"summary": summary, "device_calls": calls, "wave_stats": got["wave_stats"]})
    assert not summary["problems"], summary["problems"]
    n = len(ref["trace"])
    assert summary["queries"] == n >= 9
    # every tri_retrieve went through a retrieval wave: per wave one score-all pass over each of the fact / passage /
    # summary shards and one fused top-k pass over the timeline shard; per query two device rankings
    # (a probe string that repeats across questions is served from the wave's parked results: queries <= n)
    waves, served = got["wave_stats"]["waves"], got["wave_stats"]["queries"]
    assert 1 <= waves <= served <= n and served >= n - 3
    assert calls["scores"] >= 3 * waves and calls["rank"] >= 2 * served and calls["topk"] >= waves


@needs_ref
@pytest.mark.gpu
def test_unmodified_comorag_runs_on_the_shim_and_retrieves_what_the_reference_retrieves():
    import torch
    ref = reference_arm()
    calls, restore = _count_device_calls()
    try:
        with tempfile.TemporaryDirectory() as tmp:
            got = H.run_cinderella("shim", tmp, REF_ROOT)
    finally:
        restore()
    main = sys.modules["src.comorag.ComoRAG"]
    assert main.ComoRAG.get_fact_scores.__module__ == "comorag_b200.comorag_methods"
    assert main.EmbeddingStore.__module__ == "comorag_b200.embedding_store"
    # the GPU encoder is bf16 against the reference's fp32 HF model (parity bar: embedding max-abs error <= 1e-2, i.e.
    # raw inner products of unit vectors within ~3e-2); this synthetic 2-layer checkpoint packs all texts into a
    # narrow cone, so the raw ranges that normalise the scores are small and the normalised deviations large.
    summary = H.compare_traces(ref, got, raw_tol=3e-2)
    n = len(ref["trace"])
    _report("e2e_full_shim.json", {"summary": summary, "device_calls": calls, "wave_stats": got["wave_stats"], "query_encodes": got["query_encodes"],
                                   "reference_query_encodes": ref["query_encodes"]})
    assert not summary["problems"], summary["problems"]
    assert summary["queries"] == n >= 9
    # every tri_retrieve ran on the device kernels, shared by the concurrent questions (one wave = one encode + one
    # pass per shard); retrieve_knn added fused top-k passes at index time
    # (a probe string that repeats across questions is served from the wave's parked results: queries <= n)
    waves, served = got["wave_stats"]["waves"], got["wave_stats"]["queries"]
    assert 1 <= waves <= served <= n and served >= n - 3
    assert calls["scores"] >= 3 * waves and calls["rank"] >= 2 * served and calls["topk"] >= waves
    # and the per-character encode waste is gone: one encoded text per tri_retrieve instead of 2 * len(query) + 4
    assert got["query_encodes"]["encoded_texts"] <= n + 16 * 3
    assert ref["query_encodes"]["encoded_texts"] > 5 * got["query_encodes"]["encoded_texts"]
    # the golden trace committed from the build container agrees with the shim as well
    gold = json.load(open(GOLDEN))
    assert not H.compare_traces(gold, got, raw_tol=3e-2)["problems"]
    torch.cuda.synchronize()
