"""BGEEmbeddingModel call surface on the H100 engine (reference: embedding_model/BGEEmbedding.py).

What is kept bit-for-bit from the reference's behaviour (SURVEY.md section 7 "reference quirks"):
  * `batch_encode` ALWAYS prefixes the passage instruction, whatever `instruction=` / `is_query=` say, and
    concatenates it with NO separator (BGEEmbedding.py:108-109, 150-155);
  * pooling is the attention-masked MEAN over all tokens, not BGE's CLS (BGEEmbedding.py:15-28, 123);
  * embeddings are L2-normalised unless `normalize=False` is passed (BGEEmbedding.py:126-127, 181-183);
  * a bare `str` is treated as one text -> [1, D]; `norm=`, `num_workers=` ... kwargs are accepted and ignored;
  * `.encode(prompts, **kw)` is positional-friendly and returns a torch.Tensor [n, D] (BGEEmbedding.py:57-61),
    with NO instruction unless one is passed; `batch_encode` returns np.float32 [n, D] (C-contiguous).
What differs: the forward runs on hand-written sm_90a kernels over an unpadded token stream with bf16
weights (see comorag_b200/encoder.py); batches are cut by a packed-token budget rather than only by
`batch_size`, which changes nothing arithmetically because rows are independent.
"""
from __future__ import annotations

import logging
import threading
from copy import deepcopy
from typing import Any, List, Optional, Union

import numpy as np
import torch

from ..config import cfg_get
from ..encoder import BertEncoderB200
from .base import BaseEmbeddingModel, EmbeddingConfig, make_cache_embed

logger = logging.getLogger(__name__)

_INSTRUCTION = "Generate a representation for this sentence to retrieve relevant articles:"


def mean_pooling(token_embeddings: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """Same contract as the reference helper (BGEEmbedding.py:15-28) for callers that import it; the engine
    itself pools inside crag_encoder_forward."""
    token_embeddings = token_embeddings.masked_fill(~mask[..., None].bool(), 0.0)
    return token_embeddings.sum(dim=1) / mask.sum(dim=1)[..., None]


class BGEEmbeddingModel(BaseEmbeddingModel):
    # batch_encode overwrites any caller instruction with the passage instruction (BGEEmbedding.py:150-155), so the
    # reference's "query_to_fact" and "query_to_passage" encodes of one text are the same row; callers may rely on it
    instruction_is_forced = True
    _MEMO_ROWS = 512      # single-text batch_encode results kept (one tri_retrieve asks for the same query 4 times)

    def __init__(self, global_config: Optional[Any] = None, embedding_model_name: Optional[str] = None,
                 encoder: Optional[BertEncoderB200] = None, tokenizer: Optional[Any] = None) -> None:
        super().__init__(global_config=global_config)
        if embedding_model_name is not None:
            self.embedding_model_name = embedding_model_name
        self._init_embedding_config()
        if tokenizer is None:
            from transformers import AutoTokenizer
            tokenizer = AutoTokenizer.from_pretrained(self.embedding_model_name)
        self.tokenizer = tokenizer
        device = torch.device(cfg_get(self.global_config, "embedding_device", "cuda"))
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        self.embedding_model = encoder if encoder is not None else BertEncoderB200.from_pretrained(
            self.embedding_model_name, device)
        self.device = self.embedding_model.device
        self.embedding_dim = self.embedding_model.config.hidden_size
        self._token_budget = int(cfg_get(self.global_config, "embedding_token_budget", 16384))
        self._tok_lock = threading.Lock()  # HF fast tokenizers are not re-entrant across threads
        self._memo = {}                    # (text, max_length, normalize) -> np.float32 [1, D]
        self._memo_lock = threading.Lock()
        # optional dynamic batching of concurrent callers (ComoRAG.py:436-441 runs <=16 threads); off by default
        self._coalescer = None
        if cfg_get(self.global_config, "embedding_coalesce", False):
            from ..coalescer import CoalescedEncode
            self._coalescer = CoalescedEncode(
                self._encode_direct, max_texts=int(cfg_get(self.global_config, "embedding_coalesce_max_texts", 64)),
                max_wait_s=float(cfg_get(self.global_config, "embedding_coalesce_wait_ms", 0.3)) * 1e-3)
        if cfg_get(self.global_config, "embedding_cache_enabled", False):
            cache_path = cfg_get(self.global_config, "embedding_cache_path", "bge_embeddings_cache.db")
            self.encode = make_cache_embed(self._encode, cache_path, self.device)
        else:
            self.encode = self._encode

    def _init_embedding_config(self) -> None:
        """BGEEmbedding.py:63-90 (without HF `model_init_params`' device_map: the engine owns placement)."""
        self.embedding_config = EmbeddingConfig.from_dict({
            "embedding_model_name": self.embedding_model_name,
            "norm": cfg_get(self.global_config, "embedding_return_as_normalized", True),
            "model_init_params": {"pretrained_model_name_or_path": self.embedding_model_name},
            "encode_params": {
                "max_length": cfg_get(self.global_config, "embedding_max_seq_len", 2048),
                "query_instruction": _INSTRUCTION,
                "passage_instruction": _INSTRUCTION,
                "batch_size": cfg_get(self.global_config, "embedding_batch_size", 32),
                "num_workers": 32,
            },
        })

    # ------------------------------------------------------------------ encode
    def _tokenize(self, prompts: List[str], max_length: int) -> List[List[int]]:
        # the position table bounds what the model can embed; the reference would index past it and crash for
        # BERT checkpoints when max_length (default 2048) > 512 -- clamp instead (documented in DESIGN.md)
        cfg = self.embedding_model.config
        max_length = min(int(max_length), cfg.max_position_embeddings - cfg.position_offset)
        with self._tok_lock:
            enc = self.tokenizer(prompts, padding=False, truncation=True, max_length=max_length)
        return enc["input_ids"]

    def _encode(self, prompts: Union[str, List[str]], **kwargs) -> torch.Tensor:
        """BGEEmbedding.py:92-129: [instruction +] text -> tokenizer -> encoder -> mean pool -> (normalise)."""
        if self._coalescer is None:
            return self._encode_direct(prompts, **kwargs)
        return self._coalescer.encode(
            prompts, instruction=kwargs.get("instruction", ""),
            max_length=kwargs.get("max_length", self.embedding_config.encode_params.get("max_length", 512)),
            normalize=bool(kwargs.get("normalize", True)))

    def _encode_direct(self, prompts: Union[str, List[str]], **kwargs) -> torch.Tensor:
        if isinstance(prompts, str):
            prompts = [prompts]
        instruction = kwargs.get("instruction", "")
        if instruction:
            prompts = [instruction + text for text in prompts]
        if len(prompts) == 0:
            return torch.empty((0, self.embedding_dim), dtype=torch.float32, device=self.device)
        max_length = kwargs.get("max_length", self.embedding_config.encode_params.get("max_length", 512))
        ids = self._tokenize(list(prompts), max_length)
        normalize = bool(kwargs.get("normalize", True))
        outs = []
        # cut by packed-token budget (rows are independent, so batching never changes a row's value)
        start, tokens = 0, 0
        for i, seq in enumerate(ids):
            if i > start and tokens + len(seq) > self._token_budget:
                outs.append(self.embedding_model.encode_token_lists(ids[start:i], normalize))
                start, tokens = i, 0
            tokens += len(seq)
        outs.append(self.embedding_model.encode_token_lists(ids[start:], normalize))
        return outs[0] if len(outs) == 1 else torch.cat(outs, 0)

    def batch_encode(self, texts: Union[str, List[str]], **kwargs) -> np.ndarray:
        """BGEEmbedding.py:131-185."""
        if isinstance(texts, str):
            texts = [texts]
        params = deepcopy(self.embedding_config.encode_params)
        if kwargs:
            params.update(kwargs)
        # the reference overwrites whatever instruction the caller passed (BGEEmbedding.py:150-155)
        if "is_query" in kwargs and kwargs["is_query"]:
            params["instruction"] = params.get("query_instruction", _INSTRUCTION)
        else:
            params["instruction"] = params.get("passage_instruction", _INSTRUCTION)
        batch_size = params.pop("batch_size", 16)
        # One tri_retrieve encodes the same query string up to four times (ComoRAG.py:941,953 twice, and
        # embed_utils.py:143); the forward is deterministic, so a repeated single text is served from a small memo.
        memo_key = None
        if len(texts) == 1 and isinstance(texts[0], str):
            memo_key = (texts[0], params.get("max_length"), bool(kwargs.get("normalize", True)))
            with self._memo_lock:
                hit = self._memo.get(memo_key)
            if hit is not None:
                return hit.copy()
        if len(texts) <= batch_size:
            params["prompts"] = texts
            results = self.encode(**params)
        else:
            chunks = []
            for i in range(0, len(texts), batch_size):
                params["prompts"] = texts[i:i + batch_size]
                chunks.append(self.encode(**params))
            results = torch.cat(chunks, dim=0)
        if isinstance(results, torch.Tensor):
            results = results.detach().float().cpu().numpy()
        if self.embedding_config.norm and not kwargs.get("normalize", True):
            results = (results.T / np.linalg.norm(results, axis=1)).T
        results = np.ascontiguousarray(results, dtype=np.float32)
        if memo_key is not None:
            with self._memo_lock:
                if len(self._memo) >= self._MEMO_ROWS:
                    self._memo.pop(next(iter(self._memo)))
                self._memo[memo_key] = results.copy()
        return results

    def encode_queries(self, queries: Union[str, List[str]], **kwargs) -> np.ndarray:
        kwargs["is_query"] = True
        return self.batch_encode(queries, **kwargs)

    def encode_passages(self, passages: Union[str, List[str]], **kwargs) -> np.ndarray:
        kwargs["is_query"] = False
        return self.batch_encode(passages, **kwargs)

    # ---------------------------------------------------------- engine extras
    def encode_to_device(self, texts: List[str], out_bf16: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Index-build fast path: same arithmetic as batch_encode(texts) but the rows stay on the device
        (fp32 [n, D]); used by EmbeddingStore to fill the bf16 corpus shard without a host round trip."""
        return self._encode(texts, instruction=_INSTRUCTION,
                            max_length=self.embedding_config.encode_params.get("max_length", 512))
