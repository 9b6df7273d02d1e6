"""comorag_b200 -- H100 (sm_90a) embedding + dense-retrieval engine behind
ComoRAG's embedding_model / EmbeddingStore / rerank call surfaces."""

__version__ = "0.1.0"
