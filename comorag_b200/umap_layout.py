"""UMAP on the device for ChunkSoftClustering._reduce_dimensions (cluster_utils.py:191-211).

    umap_reduce(X, n_neighbors, n_components)  umap-learn 0.5's UMAP(n_neighbors, n_components, metric="cosine",
                                               random_state) with its default parameters, on the device: exact
                                               cosine k-NN (DenseIndex), fuzzy simplicial set (crag_umap_fuzzy_graph),
                                               the symmetric graph (torch sorts on the device), spectral start
                                               (crag_umap_spectral_init) and layout epochs (crag_umap_optimize)
    reduce_dimensions(self, embeddings)        _reduce_dimensions with the same n_neighbors and dimension formulas, log
                                               lines and fallback; install(umap=True) binds it

Parity with umap-learn is not pinned (it cannot run where the tests run): the contract is DESIGN.md section 2c and
its restatement in tests/umap_oracle.py.  The named departures: a subspace-iteration spectral start instead of
ARPACK, no meta-layout for a graph of several components, and layout epochs in which each vertex moves from its own
current position against a snapshot of the others (umap-learn moves one edge at a time on one thread).
"""
from __future__ import annotations

import functools
import logging
import sys
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import _native

MAX_D = 16                      # the GMM sweep's limit (cluster.MAX_D)
MAX_NEIGHBORS = 256
MAX_DIM = 1024
RANDOM_SEED = 224
MIN_DIST, SPREAD = 0.1, 1.0
# Subspace-iteration steps of the spectral start.  Calibrated on connected planted-cluster graphs (N = 400 and 2000,
# d + 1 clusters): the largest principal angle to eigsh's subspace is below 1e-5 after 100 steps where the gap after
# the (d+1)th eigenvalue is 0.87 / 0.88 and 1.6e-2 after 200 where it is 0.79 / 0.80; 300 leaves a margin.
SPECTRAL_ITERS = 300


@functools.lru_cache(maxsize=None)
def find_ab_params(spread: float = SPREAD, min_dist: float = MIN_DIST):
    """umap-learn's find_ab_params: scipy's curve_fit of 1 / (1 + a x^2b) on 300 points of [0, 3 spread]."""
    from scipy.optimize import curve_fit

    def curve(x, a, b):
        return 1.0 / (1.0 + a * x ** (2 * b))
    xv = np.linspace(0, spread * 3, 300)
    yv = np.zeros(xv.shape)
    yv[xv < min_dist] = 1.0
    yv[xv >= min_dist] = np.exp(-(xv[xv >= min_dist] - min_dist) / spread)
    params, _ = curve_fit(curve, xv, yv)
    return float(params[0]), float(params[1])


def default_epochs(n: int) -> int:
    return 500 if n <= 10000 else 200


@dataclass
class Stages:
    """Every stage's output, on the device (the tests compare them one by one)."""
    knn_ids: torch.Tensor        # int64 [N, k]: the search's lists
    knn_scores: torch.Tensor     # fp32 [N, k]
    nbr: torch.Tensor            # int32 [N, k]: the lists after the self rule
    dist: torch.Tensor           # fp32 [N, k]
    rho: torch.Tensor            # fp32 [N]
    sigma: torch.Tensor          # fp32 [N]
    memb: torch.Tensor           # fp32 [N, k]: directed memberships
    indptr: torch.Tensor         # int64 [N + 1]: the symmetric graph G, columns ascending
    indices: torch.Tensor        # int32 [nnz]
    weights: torch.Tensor        # fp32 [nnz]
    eps: torch.Tensor            # fp64 [nnz]: epochs_per_sample
    y0: torch.Tensor             # fp32 [N, d]: the start layout
    a: float
    b: float
    n_epochs: int


def _stream(dev, stream):
    return stream if stream is not None else torch.cuda.current_stream(dev)


def fuzzy_graph(ids: torch.Tensor, scores: torch.Tensor, stream=None):
    """crag_umap_fuzzy_graph on a self-join's lists: (nbr, dist, rho, sigma, memb)."""
    n, k = ids.shape
    dev = ids.device
    lib = _native.load()
    nbr = torch.empty(n, k, dtype=torch.int32, device=dev)
    dist = torch.empty(n, k, dtype=torch.float32, device=dev)
    rho = torch.empty(n, dtype=torch.float32, device=dev)
    sigma = torch.empty(n, dtype=torch.float32, device=dev)
    memb = torch.empty(n, k, dtype=torch.float32, device=dev)
    ws_bytes = lib.crag_umap_fuzzy_graph_workspace_bytes(n, k)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    s = _stream(dev, stream)
    _native.check(lib.crag_umap_fuzzy_graph(ids.contiguous().data_ptr(), scores.contiguous().data_ptr(), n, k,
                                            nbr.data_ptr(), dist.data_ptr(), rho.data_ptr(), sigma.data_ptr(),
                                            memb.data_ptr(), ws.data_ptr(), ws_bytes, s.cuda_stream),
                  "crag_umap_fuzzy_graph")
    return nbr, dist, rho, sigma, memb


def symmetric_graph(nbr: torch.Tensor, memb: torch.Tensor, n_epochs: int):
    """The fuzzy union G = P + P^T - P o P^T (fp32, zeros dropped), then the entries below max(G) / n_epochs dropped;
    CSR with ascending columns, built with torch sort / unique on the device.  Every directed pair occurs once in P, so
    no entry is a sum and G is exactly symmetric.  Returns (indptr, indices, weights, epochs_per_sample fp64)."""
    n, k = nbr.shape
    dev = nbr.device
    rows = torch.arange(n, device=dev, dtype=torch.int64).repeat_interleave(k)
    cols = nbr.reshape(-1).to(torch.int64)
    val = memb.reshape(-1)
    keep = val > 0
    rows, cols, val = rows[keep], cols[keep], val[keep]
    e = rows.numel()
    key, inv = torch.unique(torch.cat([rows * n + cols, cols * n + rows]), sorted=True, return_inverse=True)
    pa = torch.zeros(key.numel(), dtype=torch.float32, device=dev)
    pb = torch.zeros_like(pa)
    pa[inv[:e]] = val
    pb[inv[e:]] = val
    g = pa + pb - pa * pb
    keep = g > 0
    key, g = key[keep], g[keep]
    if g.numel() == 0:
        raise ValueError("umap: the fuzzy graph has no edges")
    gmax = g.max()
    keep = g >= gmax / float(n_epochs)
    key, g = key[keep], g[keep]
    row = key // n
    indptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    indptr[1:] = torch.cumsum(torch.bincount(row, minlength=n), 0)
    eps = gmax.double() / g.double()
    return indptr, (key % n).to(torch.int32), g.contiguous(), eps


def spectral_init(indptr, indices, weights, d: int, iters: int = SPECTRAL_ITERS, seed: int = RANDOM_SEED,
                  stream=None, vectors: bool = False):
    """crag_umap_spectral_init: the start layout fp32 [N, d]; with vectors=True also (signed Ritz vectors fp64
    [N, d], Ritz values fp64 [p])."""
    n = indptr.numel() - 1
    dev = indptr.device
    lib = _native.load()
    y = torch.empty(n, d, dtype=torch.float32, device=dev)
    vec = torch.empty(n, d, dtype=torch.float64, device=dev) if vectors else None
    p = min(max(16, d + 1), n)
    vals = torch.empty(p, dtype=torch.float64, device=dev) if vectors else None
    ws_bytes = lib.crag_umap_spectral_init_workspace_bytes(n, d)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    s = _stream(dev, stream)
    _native.check(lib.crag_umap_spectral_init(indptr.data_ptr(), indices.data_ptr(), weights.data_ptr(), n, d, iters,
                                              seed, y.data_ptr(), _native.ptr(vec), _native.ptr(vals), ws.data_ptr(),
                                              ws_bytes, s.cuda_stream), "crag_umap_spectral_init")
    return (y, vec, vals) if vectors else y


def optimize(indptr, indices, eps, y0, a: float, b: float, n_epochs: int, epoch_begin: int = 0,
             epoch_end: Optional[int] = None, seed: int = RANDOM_SEED, schedule=None, stream=None):
    """crag_umap_optimize: epochs [epoch_begin, epoch_end) from y0.  `schedule` (next_sample, next_neg) fp64 [nnz]
    are advanced in place; None starts them at (eps, eps / 5), the state before epoch 0."""
    n, d = y0.shape
    dev = y0.device
    lib = _native.load()
    epoch_end = n_epochs if epoch_end is None else epoch_end
    if schedule is None:
        schedule = (eps.clone(), eps / 5.0)
    next_sample, next_neg = schedule
    y = torch.empty_like(y0)
    ws_bytes = lib.crag_umap_optimize_workspace_bytes(n, d)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    s = _stream(dev, stream)
    _native.check(lib.crag_umap_optimize(indptr.data_ptr(), indices.data_ptr(), eps.data_ptr(), n, indices.numel(), d,
                                         a, b, n_epochs, epoch_begin, epoch_end, seed, next_sample.data_ptr(),
                                         next_neg.data_ptr(), y0.contiguous().data_ptr(), y.data_ptr(), ws.data_ptr(),
                                         ws_bytes, s.cuda_stream), "crag_umap_optimize")
    return y


def knn_self_join(X, k: int, device=None, stream=None):
    """Rows normalised in fp32 (a zero row stays zero) and rounded to bf16, then crag_knn_topk's (or the scan's:
    they are bit-identical) k best of every row among all rows: (ids int64 [N, k], scores fp32 [N, k])."""
    from .index import DenseIndex
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    x = torch.as_tensor(X).to(dev, torch.float32)
    nrm = torch.linalg.vector_norm(x, dim=1, keepdim=True)
    xn = torch.where(nrm > 0, x / torch.where(nrm > 0, nrm, torch.ones_like(nrm)), torch.zeros_like(x))
    index = DenseIndex(x.shape[1], device=dev)
    index.add(xn)
    ids, scores, _ = index.search_device(index.prepare_queries(xn), k, stream=stream)
    return ids, scores


def umap_reduce(X, n_neighbors: int, n_components: int, random_state: int = RANDOM_SEED,
                n_epochs: Optional[int] = None, device=None, stream=None, return_stages: bool = False,
                spectral_iters: int = SPECTRAL_ITERS):
    """UMAP(n_neighbors, n_components, metric="cosine", random_state).fit_transform(X) on the device (DESIGN.md
    section 2c): fp32 [N, n_components] as a numpy array, and the per-stage outputs with return_stages=True.
    Limits: N >= 2, 1 <= n_components <= min(16, N - 1), n_neighbors in [2, 256], at most 1024 columns."""
    X = np.asarray(X, dtype=np.float32) if not torch.is_tensor(X) else X
    if X.ndim != 2:
        raise ValueError(f"umap_reduce: X must be [N, D], got shape {tuple(X.shape)}")
    n, dim = X.shape
    d = int(n_components)
    if d < 1:
        raise ValueError("n_components must be greater than 0")       # as umap-learn says it
    if int(n_neighbors) < 2:
        raise ValueError("n_neighbors must be greater than 1")
    if n < 2 or d > MAX_D or d + 1 > n:
        raise ValueError(f"umap_reduce: n_components = {d} needs 1 <= n_components <= min({MAX_D}, N - 1) (N = {n})")
    if n_neighbors > MAX_NEIGHBORS:
        raise ValueError(f"umap_reduce: n_neighbors = {n_neighbors} > {MAX_NEIGHBORS}")
    if not 1 <= dim <= MAX_DIM:
        raise ValueError(f"umap_reduce: {dim} columns is outside [1, {MAX_DIM}]")
    k = int(n_neighbors) if n > n_neighbors else n - 1                 # umap-learn: n_neighbors >= N -> N - 1
    n_epochs = int(n_epochs) if n_epochs is not None else default_epochs(n)
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev):
        s = _stream(dev, stream)
        with torch.cuda.stream(s):
            ids, scores = knn_self_join(X, k, dev, s)
            nbr, dist, rho, sigma, memb = fuzzy_graph(ids, scores, s)
            indptr, indices, weights, eps = symmetric_graph(nbr, memb, n_epochs)
            a, b = find_ab_params()
            y0 = spectral_init(indptr, indices, weights, d, spectral_iters, random_state, s)
            y = optimize(indptr, indices, eps, y0, a, b, n_epochs, seed=random_state, stream=s)
        s.synchronize()
    out = y.cpu().numpy()
    if return_stages:
        return out, Stages(ids, scores, nbr, dist, rho, sigma, memb, indptr, indices, weights, eps, y0, a, b, n_epochs)
    return out


def reduce_dimensions(self, embeddings: np.ndarray) -> np.ndarray:
    """ChunkSoftClustering._reduce_dimensions (cluster_utils.py:191-211) on the device: the same n_neighbors and
    dimension formulas, log lines and fallback to the original rows when the reduction raises."""
    ref = sys.modules[type(self).__module__]
    logger = getattr(ref, "logger", logging.getLogger(__name__))
    n_neighbors = min(30, max(5, int(len(embeddings) * 0.2)))
    dim = min(self.reduction_dimension, len(embeddings) - 2)
    try:
        reduced_embeddings = umap_reduce(embeddings, n_neighbors, dim, getattr(ref, "RANDOM_SEED", RANDOM_SEED))
        if self.verbose:
            logger.info(f"Reduced dimensions from {embeddings.shape[1]} to {dim}")
        return reduced_embeddings
    except Exception as e:
        logger.warning(f"Error during dimension reduction: {e}. Using original embeddings.")
        return embeddings
