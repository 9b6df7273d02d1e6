"""EmbeddingStore call surface on the H100 engine (reference: src/comorag/embedding_store.py).

Same constructor, methods, attributes, return values, id scheme (namespace + "-" + md5(text),
misc_utils.py:152-163) and parquet file (`vdb_<namespace>.parquet`, columns hash_id / content / embedding =
large_string / large_string / list<float>) as the reference, so ComoRAG.py and its helpers use it unchanged.

What is different underneath:
  * rows live in one growing fp32 host matrix (not a Python list of N arrays) AND as bf16 rows of a
    device-resident DenseIndex, filled straight from the encoder's device output;
  * `search(queries, k)` runs the fused sm_90a top-k kernel over the shard instead of callers pulling the
    whole matrix with get_embeddings() and doing np.dot + argsort per query (ComoRAG.py:937-967);
  * parquet I/O goes through pyarrow arrays built from the matrix (no per-row Python objects).
"""
from __future__ import annotations

import logging
import os
import threading
from copy import deepcopy
from hashlib import md5
from typing import Dict, List, Optional, Tuple

import numpy as np

logger = logging.getLogger(__name__)


def compute_mdhash_id(content: str, prefix: str = "") -> str:
    """misc_utils.py:152-163."""
    return prefix + md5(content.encode()).hexdigest()


class _RowList:
    """List-like, read-only view of the embedding matrix rows (`store.embeddings` in the reference is a
    List[np.ndarray]; embedding_store.py:96,119)."""

    def __init__(self, store: "EmbeddingStore"):
        self._s = store

    def __len__(self) -> int:
        return self._s._n

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self._s._host[j] for j in range(*i.indices(self._s._n))]
        if i < 0:
            i += self._s._n
        if not 0 <= i < self._s._n:
            raise IndexError("embedding index out of range")
        return self._s._host[i]

    def __iter__(self):
        return (self._s._host[j] for j in range(self._s._n))


class EmbeddingStore:
    def __init__(self, embedding_model, db_filename, batch_size, namespace):
        self.embedding_model = embedding_model
        self.batch_size = batch_size
        self.namespace = namespace
        if not os.path.exists(db_filename):
            logger.info(f"Creating working directory: {db_filename}")
            os.makedirs(db_filename, exist_ok=True)
        self.filename = os.path.join(db_filename, f"vdb_{self.namespace}.parquet")
        self._lock = threading.RLock()
        self._dim: Optional[int] = getattr(embedding_model, "embedding_dim", None)
        self._host = np.zeros((0, self._dim or 0), dtype=np.float32)
        self._n = 0
        self._index = None  # DenseIndex, created on first use (needs a CUDA device)
        self._index_rows = 0
        # persistence: "parquet" (reference behaviour: whole-file rewrite per upsert) or "append" (O(new rows) raw
        # shards + jsonl; vdb_<ns>.parquet is produced on demand by export_parquet())
        cfg = getattr(embedding_model, "global_config", None)
        self._persist = "append" if getattr(cfg, "embedding_store_append_only", False) else "parquet"
        self._base = os.path.join(db_filename, f"vdb_{self.namespace}")
        self._search_coalescer = None
        if getattr(getattr(embedding_model, "global_config", None), "embedding_coalesce", False):
            from .coalescer import CoalescedSearch
            self._search_coalescer = CoalescedSearch(lambda: self.index)
        self._load_data()

    # ------------------------------------------------------------- bookkeeping
    @property
    def embeddings(self):
        return _RowList(self)

    def _rebuild_maps(self) -> None:
        self.hash_id_to_idx = {h: i for i, h in enumerate(self.hash_ids)}
        self.hash_id_to_row = {h: {"hash_id": h, "content": t} for h, t in zip(self.hash_ids, self.texts)}
        self.hash_id_to_text = dict(zip(self.hash_ids, self.texts))
        self.text_to_hash_id = {t: h for h, t in zip(self.hash_ids, self.texts)}

    def _append_host(self, rows: np.ndarray) -> None:
        rows = np.asarray(rows, dtype=np.float32)
        if rows.ndim == 1:
            rows = rows[None, :]
        if self._dim is None or self._host.shape[1] == 0:
            self._dim = rows.shape[1]
            self._host = np.zeros((0, self._dim), dtype=np.float32)
        n1 = self._n + rows.shape[0]
        if n1 > self._host.shape[0]:
            grown = np.empty((max(n1, int(self._host.shape[0] * 1.5) + 64), self._dim), dtype=np.float32)
            grown[: self._n] = self._host[: self._n]
            self._host = grown
        self._host[self._n:n1] = rows
        self._n = n1

    # ------------------------------------------------------------------ inserts
    def _nodes(self, texts: List[str]) -> Dict[str, Dict[str, str]]:
        return {compute_mdhash_id(text, prefix=self.namespace + "-"): {"content": text} for text in texts}

    def get_missing_string_hash_ids(self, texts: List[str]):
        """embedding_store.py:44-61."""
        nodes = self._nodes(texts)
        if not nodes:
            return {}
        missing = [h for h in nodes if h not in self.hash_id_to_row]
        return {h: {"hash_id": h, "content": nodes[h]["content"]} for h in missing}

    def insert_strings(self, texts: List[str]):
        """embedding_store.py:63-90: dedup by md5 id, encode what is missing, append, persist."""
        with self._lock:
            nodes = self._nodes(texts)
            if not nodes:
                return
            missing_ids = [h for h in nodes if h not in self.hash_id_to_row]
            logger.info(f"Inserting {len(missing_ids)} new records, {len(nodes) - len(missing_ids)} records already exist.")
            if not missing_ids:
                return {}
            texts_to_encode = [nodes[h]["content"] for h in missing_ids]
            device_rows = None
            encode_dev = getattr(self.embedding_model, "encode_to_device", None)
            if encode_dev is not None and self._index is not None and self._index_rows == self._n:
                # index-build fast path: the encoder's device output goes straight into the bf16 shard (no host
                # round trip); the host fp32 copy kept for get_embeddings()/parquet is the same rows read back.
                device_rows = encode_dev(texts_to_encode)
                missing_embeddings = device_rows.detach().float().cpu().numpy()
            else:
                missing_embeddings = self.embedding_model.batch_encode(texts_to_encode)
            self._upsert(missing_ids, texts_to_encode, missing_embeddings, device_rows)

    def _upsert(self, hash_ids, texts, embeddings, device_rows=None):
        n0 = self._n
        self._append_host(embeddings)
        if device_rows is not None and self._index is not None and self._index_rows == n0:
            self._index.add(device_rows)
            self._index_rows = self._n
        self.hash_ids.extend(hash_ids)
        self.texts.extend(texts)
        logger.info("Saving new records.")
        if self._persist == "append":
            self._append_raw(n0)
            self._rebuild_maps_incremental(n0)
        else:
            self._save_data()

    # ---- append-only persistence (SURVEY.md section 8f item 2): raw row shards + a jsonl row table
    def _append_raw(self, n0: int) -> None:
        import json
        import torch
        mode = "a"
        if n0 > 0 and not os.path.exists(self._base + ".meta.json"):
            # first append over rows that came from somewhere else (a vdb_<ns>.parquet written in parquet mode): the
            # raw shards must hold EVERY row the meta file is about to vouch for, so write the whole matrix once
            n0, mode = 0, "w"
        rows = self._host[n0:self._n]
        with open(self._base + ".rows.jsonl", mode) as f:
            for h, t in zip(self.hash_ids[n0:], self.texts[n0:]):
                f.write(json.dumps({"hash_id": h, "content": t}) + "\n")
        with open(self._base + ".f32", mode + "b") as f:
            f.write(np.ascontiguousarray(rows, dtype=np.float32).tobytes())
        dim_pad = (self._dim + 63) // 64 * 64
        padded = torch.zeros((rows.shape[0], dim_pad), dtype=torch.bfloat16)
        padded[:, : self._dim] = torch.from_numpy(np.ascontiguousarray(rows)).to(torch.bfloat16)
        with open(self._base + ".bf16", mode + "b") as f:
            f.write(padded.view(torch.int16).numpy().tobytes())
        # the meta file is the commit record: written last, atomically; a crash before it leaves longer data files,
        # which _load_raw() cuts back to what the meta file vouches for
        tmp = self._base + ".meta.json.tmp"
        with open(tmp, "w") as f:
            json.dump({"dim": self._dim, "dim_pad": dim_pad, "rows": self._n, "format": "comorag_b200.raw.v1",
                       "jsonl_bytes": os.path.getsize(self._base + ".rows.jsonl")}, f)
        os.replace(tmp, self._base + ".meta.json")

    def _rebuild_maps_incremental(self, n0: int) -> None:
        for i in range(n0, self._n):
            h, t = self.hash_ids[i], self.texts[i]
            self.hash_id_to_idx[h] = i
            self.hash_id_to_row[h] = {"hash_id": h, "content": t}
            self.hash_id_to_text[h] = t
            self.text_to_hash_id[t] = h

    def _load_raw(self) -> bool:
        import json
        meta_p = self._base + ".meta.json"
        if not os.path.exists(meta_p):
            return False
        meta = json.load(open(meta_p))
        n, d = meta["rows"], meta["dim"]
        # roll back an append that was interrupted before its meta commit
        want = {".f32": n * d * 4, ".bf16": n * meta.get("dim_pad", (d + 63) // 64 * 64) * 2}
        if "jsonl_bytes" in meta:
            want[".rows.jsonl"] = meta["jsonl_bytes"]
        for ext, size in want.items():
            have = os.path.getsize(self._base + ext) if os.path.exists(self._base + ext) else -1
            if have < size:
                raise ValueError(f"{self._base}{ext}: {have} bytes, shorter than the {size} the meta file records for {n} rows")
            if have > size:
                logger.warning(f"{self._base}{ext}: dropping {have - size} bytes of an uncommitted append")
                with open(self._base + ext, "r+b") as f:
                    f.truncate(size)
        rows = [json.loads(l) for l in open(self._base + ".rows.jsonl") if l.strip()]
        if len(rows) < n:
            raise ValueError(f"{self._base}.rows.jsonl: {len(rows)} rows, the meta file records {n}")
        self.hash_ids = [r["hash_id"] for r in rows[:n]]
        self.texts = [r["content"] for r in rows[:n]]
        self._dim = d
        self._host = np.zeros((0, d), dtype=np.float32)
        self._n = 0
        if n:
            self._append_host(np.fromfile(self._base + ".f32", dtype=np.float32, count=n * d).reshape(n, d))
        self._rebuild_maps()
        return True

    def raw_shard_path(self) -> Optional[str]:
        """Path of the bf16 [rows, dim_pad] shard file if it is in sync with the store (direct GPU upload)."""
        p = self._base + ".bf16"
        if self._persist == "append" and os.path.exists(p) and self._dim:
            dim_pad = (self._dim + 63) // 64 * 64
            if os.path.getsize(p) == self._n * dim_pad * 2:
                return p
        return None

    def export_parquet(self) -> str:
        """Write the reference-compatible vdb_<ns>.parquet (embedding_store.py:109-115) from the current rows."""
        self._save_data()
        return self.filename

    # -------------------------------------------------------------- persistence
    def _load_data(self):
        """embedding_store.py:92-107."""
        if self._persist == "append" and os.path.exists(self._base + ".meta.json") and os.path.exists(self.filename):
            # both formats present: a parquet file with MORE rows was written later in parquet mode; the raw shards
            # are stale, so drop their commit record (the next append rewrites them in full) and load the parquet
            import json
            import pyarrow.parquet as pq
            if pq.ParquetFile(self.filename).metadata.num_rows > json.load(open(self._base + ".meta.json")).get("rows", 0):
                logger.warning(f"{self._base}.*: raw shards are older than {self.filename}; rebuilding them on the next insert")
                os.remove(self._base + ".meta.json")
        if self._persist == "append" and self._load_raw():
            logger.info(f"Loaded {len(self.hash_ids)} records from {self._base}.* (raw shards)")
            return
        if self._persist == "parquet" and os.path.exists(self._base + ".meta.json"):
            # the directory was last written in append-only mode: its raw shards are the truth (a vdb_<ns>.parquet
            # beside them may be older, or absent); load them and bring the parquet file up to date
            import json
            raw_rows = json.load(open(self._base + ".meta.json")).get("rows", 0)
            pq_rows = -1
            if os.path.exists(self.filename):
                import pyarrow.parquet as pq
                pq_rows = pq.ParquetFile(self.filename).metadata.num_rows
            if raw_rows > pq_rows and self._load_raw():
                logger.info(f"Loaded {len(self.hash_ids)} records from {self._base}.* (raw shards newer than the parquet file)")
                self._save_data()
                return
        if os.path.exists(self.filename):
            import pyarrow.parquet as pq
            table = pq.read_table(self.filename)
            self.hash_ids = table.column("hash_id").to_pylist()
            self.texts = table.column("content").to_pylist()
            emb = table.column("embedding").combine_chunks()
            n = len(self.hash_ids)
            flat = emb.flatten().to_numpy(zero_copy_only=False).astype(np.float32, copy=False)
            if n and flat.size % n != 0:
                raise ValueError(f"{self.filename}: ragged embedding column")
            self._host = np.zeros((0, 0), dtype=np.float32)
            self._n = 0
            if n:
                self._dim = flat.size // n
                self._append_host(flat.reshape(n, self._dim))
            self._rebuild_maps()
            assert len(self.hash_ids) == len(self.texts) == self._n
            logger.info(f"Loaded {len(self.hash_ids)} records from {self.filename}")
        else:
            self.hash_ids, self.texts = [], []
            self._rebuild_maps()  # the reference leaves hash_id_to_text / text_to_hash_id undefined here (:106-107)

    _PARQUET_MAX_VALUES = (1 << 31) - 1024   # list<float> carries int32 offsets: keep each written batch below 2^31 floats

    def _save_data(self):
        """embedding_store.py:109-120: whole-file rewrite, same schema (large_string, large_string, list<float>).
        Written in row batches so stores past 2^31 floats (2.1M rows x 1024) do not overflow the list offsets."""
        import pyarrow as pa
        import pyarrow.parquet as pq
        n, d = self._n, (self._dim or 0)
        schema = pa.schema([("hash_id", pa.large_string()), ("content", pa.large_string()),
                            ("embedding", pa.list_(pa.float32()))])
        step = max(1, self._PARQUET_MAX_VALUES // max(d, 1))
        tmp = self.filename + ".tmp"
        with pq.ParquetWriter(tmp, schema) as writer:
            for s0 in range(0, max(n, 1), step):
                s1 = min(n, s0 + step)
                values = pa.array(self._host[s0:s1].reshape(-1), type=pa.float32())
                offsets = pa.array(np.arange(s1 - s0 + 1, dtype=np.int64) * d, type=pa.int32())
                writer.write_table(pa.table({
                    "hash_id": pa.array(self.hash_ids[s0:s1], type=pa.large_string()),
                    "content": pa.array(self.texts[s0:s1], type=pa.large_string()),
                    "embedding": pa.ListArray.from_arrays(offsets, values),
                }, schema=schema))
        os.replace(tmp, self.filename)
        self._rebuild_maps()
        logger.info(f"Saved {len(self.hash_ids)} records to {self.filename}")

    # ------------------------------------------------------------------ lookups
    def get_row(self, hash_id):
        return self.hash_id_to_row[hash_id]

    def get_rows(self, hash_ids, dtype=np.float32):
        if not hash_ids:
            return {}
        return {id: self.hash_id_to_row[id] for id in hash_ids}

    def get_all_ids(self):
        return deepcopy(self.hash_ids)

    def get_text_for_all_rows(self):
        return deepcopy(self.hash_id_to_row)

    def get_embedding(self, hash_id, dtype=np.float32) -> np.ndarray:
        return self._host[self.hash_id_to_idx[hash_id]].astype(dtype)

    def get_embeddings(self, hash_ids, dtype=np.float32):
        if not hash_ids:
            return []
        indices = np.array([self.hash_id_to_idx[h] for h in hash_ids], dtype=np.intp)
        return self._host[: self._n][indices].astype(dtype, copy=False)

    def get_hash_id_to_order(self) -> Dict[str, int]:
        return {h: idx for idx, h in enumerate(self.hash_ids)}

    # ------------------------------------------------------------ engine extras
    @property
    def index(self):
        """Device-resident bf16 shard holding every stored row (built / extended lazily)."""
        from .index import DenseIndex
        with self._lock:
            if self._index is None:
                if self._dim is None:
                    raise ValueError("empty store: embedding width unknown")
                device = getattr(self.embedding_model, "device", None)
                self._index = DenseIndex(self._dim, device=device, capacity=max(self._n, 1024))
                self._index_rows = 0
                shard = self.raw_shard_path()
                if shard is not None and self._n:
                    self._index.add_bf16_file(shard, self._n)   # bf16 rows straight from disk, no fp32 round trip
                    self._index_rows = self._n
            if self._index_rows < self._n:
                self._index.add(self._host[self._index_rows: self._n])
                self._index_rows = self._n
            return self._index

    def search(self, query_embeddings, k: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
        """Top-k rows for a block of query embeddings [nq, D] (host or device): (row indices int64 [nq, k]
        into hash_ids/texts, raw inner products [nq, k], (min, max) over all rows [nq, 2])."""
        if self._search_coalescer is not None:
            return self._search_coalescer.search(query_embeddings, k)
        return self.index.search(query_embeddings, k)
