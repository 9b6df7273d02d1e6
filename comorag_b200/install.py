"""Drop the engine under an unmodified ComoRAG checkout by import-time substitution (SURVEY.md section 8b).

    import comorag_b200.install as crag
    crag.install("src.comorag")          # before or after `from src.comorag import ComoRAG`
    rag = ComoRAG(global_config=BaseConfig(embedding_model_name=".../bge-large-en-v1.5", ...))

`ComoRAG.py` binds `_get_embedding_model_class`, `EmbeddingStore`, `DSPyFilter`, `get_similar_summaries`,
`retrieve_knn` by `from ... import` (ComoRAG.py:21-35), so the substitution rewrites those names in every
already-imported module of the package as well as in their defining modules; class bodies resolve them from module
globals at call time.  The search half of the path lives in METHODS of the `ComoRAG` class itself
(`prepare_retrieval_objects`, `get_query_embeddings`, `get_fact_scores`, `dense_passage_retrieval`,
ComoRAG.py:876-967): those are replaced on the class object (comorag_b200/comorag_methods.py), the file stays
untouched.
"""
from __future__ import annotations

import importlib
import sys
from typing import Dict


def install(package: str = "src.comorag", rerank: bool = False, summaries: bool = True, search: bool = True,
            knn: bool = True, encoder: bool = True, graph: bool = False) -> Dict[str, int]:
    """Returns {name: number of module attributes (or class methods) rebound}.  `rerank=True` also swaps the LLM
    filter for the dense reranker (new arithmetic, off by default so answers stay reference-identical); `search`
    rebinds the four ComoRAG retrieval methods, `knn` the synonymy-edge retrieve_knn; `encoder=False` keeps the
    reference's own embedding model class (HF, fp32) and swaps only the store / search half -- the parity tests use
    that to compare rankings without the bf16 encoder's error in the way.  `graph=True` also rebinds
    graph_search_with_fact_entities and run_ppr (comorag_methods.GRAPH_METHODS: PPR on the device, crag_ppr); it
    needs a real igraph.Graph (get_edgelist, es["weight"]) and is off by default."""
    from . import embedding_model as em
    from . import embedding_store as es
    from . import rerank as rr
    from . import retrieval as rt

    ref_em = importlib.import_module(package + ".embedding_model")
    ref_es = importlib.import_module(package + ".embedding_store")
    swaps = {"EmbeddingStore": (ref_es.EmbeddingStore, es.EmbeddingStore)}
    if encoder:
        swaps["_get_embedding_model_class"] = (ref_em._get_embedding_model_class, em._get_embedding_model_class)
        swaps["BGEEmbeddingModel"] = (ref_em.BGEEmbeddingModel, em.BGEEmbeddingModel)
    if summaries:
        ref_eu = importlib.import_module(package + ".utils.embed_utils")
        swaps["get_similar_summaries"] = (ref_eu.get_similar_summaries, rt.get_similar_summaries)
    if knn:
        ref_eu = importlib.import_module(package + ".utils.embed_utils")
        swaps["retrieve_knn"] = (ref_eu.retrieve_knn, rt.retrieve_knn)
    if rerank:
        ref_rr = importlib.import_module(package + ".rerank")
        swaps["DSPyFilter"] = (ref_rr.DSPyFilter, rr.DSPyFilter)
    counts = {k: 0 for k in swaps}
    for name, mod in list(sys.modules.items()):
        if mod is None or not (name == package or name.startswith(package + ".")):
            continue
        for attr, (old, new) in swaps.items():
            if getattr(mod, attr, None) is old:
                setattr(mod, attr, new)
                counts[attr] += 1
    if search or graph:
        from . import comorag_methods as cm
        main = sys.modules.get(package + ".ComoRAG") or importlib.import_module(package + ".ComoRAG")
        cls = main.ComoRAG
        methods = {**(cm.METHODS if search else {}), **(cm.GRAPH_METHODS if graph else {})}
        originals = cls.__dict__.get("_comorag_b200_originals")
        if originals is None:
            originals = {}
            cls._comorag_b200_originals = originals       # uninstall() / the parity tests can reach the reference methods
        for name, fn in methods.items():
            if name not in originals:
                originals[name] = cls.__dict__[name]
            setattr(cls, name, fn)
            counts["ComoRAG." + name] = 1
    return counts


def uninstall_search(package: str = "src.comorag") -> None:
    """Put the reference's own retrieval methods back on the ComoRAG class (used by the parity tests to run the
    reference arm in the same process)."""
    main = sys.modules.get(package + ".ComoRAG")
    if main is None:
        return
    originals = main.ComoRAG.__dict__.get("_comorag_b200_originals")
    if originals:
        for name, fn in originals.items():
            setattr(main.ComoRAG, name, fn)
