"""Factory + classes, same names as the reference package (embedding_model/__init__.py:1-17)."""
import logging

from .base import BaseEmbeddingModel, EmbeddingCache, EmbeddingConfig
from .BGEEmbedding import BGEEmbeddingModel

logger = logging.getLogger(__name__)


class OpenAIEmbeddingModel(BaseEmbeddingModel):
    """The reference's OpenAI-API variant (embedding_model/OpenAI.py) is a network client, outside the
    hot path this engine replaces; the name is kept so the factory's dispatch table is complete."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("OpenAIEmbeddingModel is an HTTP client in the reference and is out of scope "
                                  "for the H100 engine; use a local 'bge-' checkpoint")


def _get_embedding_model_class(embedding_model_name: str = "None"):
    """embedding_model/__init__.py:10-17.  The reference's fall-through branch logs "using BGEEmbeddingModel as
    default" but returns None (and then crashes at ComoRAG.py:92-94); here the logged intent is honoured."""
    if "bge-" in embedding_model_name.lower():
        return BGEEmbeddingModel
    if "text-embedding-3-small" in embedding_model_name:
        return OpenAIEmbeddingModel
    logger.info(f"Unknown embedding model name: {embedding_model_name}, using BGEEmbeddingModel as default")
    return BGEEmbeddingModel
