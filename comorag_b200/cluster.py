"""Soft clustering on the device: the BIC sweep of ChunkSoftClustering (cluster_utils.py:175-357) through
crag_gmm_sweep.

    gmm_sweep(X, max_components)   scikit-learn's GaussianMixture(m, random_state=224) for m = 1..M in float64, all
                                   M models in one call: chosen n, BIC, EM iterations, converged flags, the winner's
                                   weights, means and memberships (predict_proba)
    perform_clustering(self, ...)  ChunkSoftClustering.perform_clustering with the same control flow and outputs,
                                   each sweep + refit + predict_proba replaced by one gmm_sweep; install(cluster=True)
                                   binds it

The one deliberate deviation: the arithmetic is always float64, where scikit-learn fits UMAP's float32 output in
float32 (DESIGN.md section 1).
"""
from __future__ import annotations

import logging
import sys
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import torch

from . import _native

MAX_D = 16
MAX_COMPONENTS = 64
RANDOM_SEED = 224


def _trials(m: int) -> int:
    return 2 + int(np.log(m))


def seed_draws(n: int, max_components: int, random_state: int = RANDOM_SEED):
    """The random draws of every model's k-means++ seeding, which do not depend on the data: a fresh
    RandomState(random_state) per model, consumed as scikit-learn's _kmeans_plusplus consumes it (unit sample
    weights).  Returns (first_centre int64 [M], draws fp64 [sum_m (m - 1)(2 + int(log m))])."""
    first = np.empty(max_components, dtype=np.int64)
    rest = []
    p = np.ones(n, dtype=np.float64)
    p /= p.sum()
    for m in range(1, max_components + 1):
        rs = np.random.RandomState(random_state)
        first[m - 1] = rs.choice(n, p=p)
        rest.extend(rs.uniform(size=_trials(m)) for _ in range(1, m))
    return first, (np.concatenate(rest) if rest else np.zeros(0)).astype(np.float64)


@dataclass
class SweepResult:
    n_components: int            # the first BIC argmin
    bic: np.ndarray              # [M]
    iterations: np.ndarray       # [M] EM iterations
    converged: np.ndarray        # [M] bool
    weights: np.ndarray          # [n_components]
    means: np.ndarray            # [n_components, d]
    memberships: np.ndarray      # [N, n_components]
    seeds: Optional[np.ndarray] = None    # [M(M+1)/2] k-means++ rows, model m at [m(m-1)/2, m(m+1)/2)
    labels: Optional[np.ndarray] = None   # [M, N] final k-means labels


def gmm_sweep(X, max_components: int, random_state: int = RANDOM_SEED, device=None, stream=None,
              keep_kmeans: bool = False) -> SweepResult:
    """Fit GaussianMixture(m, covariance_type="full", random_state=random_state) for m = 1..max_components on the
    rows of X ([N, d], 1 <= d <= 16, 1 <= max_components <= min(64, N - 1)) on the device, and return the model with
    the smallest BIC.  `keep_kmeans` also returns every model's k-means++ rows and final k-means labels."""
    X = np.ascontiguousarray(np.asarray(X, dtype=np.float64))
    if X.ndim != 2:
        raise ValueError(f"gmm_sweep: X must be [N, d], got shape {X.shape}")
    n, d = X.shape
    M = int(max_components)
    if not 1 <= d <= MAX_D:
        raise ValueError(f"gmm_sweep: d = {d} is outside [1, {MAX_D}]")
    if n < 2 or not 1 <= M <= min(MAX_COMPONENTS, n - 1):
        raise ValueError(f"gmm_sweep: max_components = {M} is outside [1, min({MAX_COMPONENTS}, N - 1)] (N = {n})")
    if not np.isfinite(X).all():
        raise ValueError("gmm_sweep: X holds a NaN or an infinity")
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    lib = _native.load()
    first, draws = seed_draws(n, M, random_state)
    x = torch.from_numpy(X).to(dev)
    t_first = torch.from_numpy(first).to(dev)
    t_draws = torch.from_numpy(draws).to(dev) if draws.size else None
    f64 = dict(dtype=torch.float64, device=dev)
    i32 = dict(dtype=torch.int32, device=dev)
    bic, iters, conv = torch.empty(M, **f64), torch.empty(M, **i32), torch.empty(M, **i32)
    best = torch.empty(1, **i32)
    weights, means = torch.empty(M, **f64), torch.empty(M, d, **f64)
    memb = torch.empty(n * M, **f64)
    seeds = torch.empty(M * (M + 1) // 2, **i32) if keep_kmeans else None
    labels = torch.empty(M, n, **i32) if keep_kmeans else None
    ws_bytes = lib.crag_gmm_sweep_workspace_bytes(n, d, M)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    s = stream if stream is not None else torch.cuda.current_stream(dev)
    _native.check(lib.crag_gmm_sweep(x.data_ptr(), n, d, M, t_first.data_ptr(), _native.ptr(t_draws), bic.data_ptr(),
                                     iters.data_ptr(), conv.data_ptr(), best.data_ptr(), weights.data_ptr(),
                                     means.data_ptr(), memb.data_ptr(), _native.ptr(seeds), _native.ptr(labels),
                                     ws.data_ptr(), ws_bytes, s.cuda_stream), "crag_gmm_sweep")
    s.synchronize()
    k = int(best.item())
    conv_h = conv.cpu().numpy()
    if (conv_h < 0).any():
        bad = (np.where(conv_h < 0)[0] + 1).tolist()
        raise ValueError(f"gmm_sweep: a covariance of the {bad}-component model(s) is not positive definite")
    return SweepResult(k, bic.cpu().numpy(), iters.cpu().numpy(), conv_h > 0, weights[:k].cpu().numpy(),
                       means[:k].cpu().numpy(), memb[:n * k].view(n, k).cpu().numpy(),
                       seeds.cpu().numpy() if keep_kmeans else None, labels.cpu().numpy() if keep_kmeans else None)


def fit_best(X, max_components: int, random_state: int = RANDOM_SEED):
    """(n_components, means, memberships) of the sweep ChunkSoftClustering runs on X: with one component every
    membership is 1.0, and the device is not needed; otherwise X must have at most 16 columns."""
    X = np.asarray(X)
    if max_components == 1:
        Xd = X.astype(np.float64)
        mean = Xd.sum(axis=0) / (len(Xd) + 10 * np.finfo(np.float64).eps)
        return 1, mean[None, :], np.ones((len(Xd), 1))
    if X.shape[1] > MAX_D:
        raise ValueError(f"soft clustering on the device supports d <= {MAX_D} dimensions, got d = {X.shape[1]} "
                         f"(the reduction to reduction_dimension failed?)")
    r = gmm_sweep(X, max_components, random_state)
    return r.n_components, r.means, r.memberships


def perform_clustering(self, hash_ids: Optional[List[str]] = None):
    """ChunkSoftClustering.perform_clustering (cluster_utils.py:213-357) with each GMM sweep on the device: the
    same reductions (the instance's own _reduce_dimensions), thresholds, small-cluster shortcut, empty-cluster
    skipping and cluster numbering, and SoftCluster objects of the reference's own class."""
    ref = sys.modules[type(self).__module__]
    SoftCluster = ref.SoftCluster
    logger = getattr(ref, "logger", logging.getLogger(__name__))
    if hash_ids is None or len(hash_ids) == 0:
        hash_ids = self.embedding_store.get_all_ids()
    if len(hash_ids) <= 1:
        logger.warning("Insufficient data to perform clustering")
        if len(hash_ids) == 1:
            cluster = SoftCluster(0)
            cluster.add_member(hash_ids[0], 1.0)
            self.clusters = [cluster]
            self.hash_id_to_cluster_memberships = {hash_ids[0]: {0: 1.0}}
        return self.clusters

    embeddings = np.array(self.embedding_store.get_embeddings(hash_ids))
    if embeddings.shape[1] > self.reduction_dimension:
        try:
            reduced_global = self._reduce_dimensions(embeddings)
        except Exception as e:
            logger.warning(f"Global dimension reduction error: {e}")
            reduced_global = embeddings
    else:
        reduced_global = embeddings
    n_global, _, global_scores = fit_best(reduced_global, min(self.max_clusters, len(reduced_global) - 1))
    global_clusters = [np.where(global_scores[i] >= self.threshold)[0] for i in range(len(hash_ids))]
    if self.verbose:
        logger.info(f"Global cluster count: {n_global}")

    self.clusters = []
    self.hash_id_to_cluster_memberships = {}
    total_clusters = 0
    for i in range(n_global):
        idx = np.array([j for j, gc in enumerate(global_clusters) if i in gc])
        if len(idx) == 0:
            continue
        local_embeddings = embeddings[idx]
        local_hash_ids = [hash_ids[j] for j in idx]
        if len(local_embeddings) <= self.reduction_dimension + 1:
            cluster = SoftCluster(total_clusters)
            for hash_id in local_hash_ids:
                cluster.add_member(hash_id, 1.0)
                self.hash_id_to_cluster_memberships.setdefault(hash_id, {})[total_clusters] = 1.0
            self.clusters.append(cluster)
            total_clusters += 1
            continue
        try:
            reduced_local = self._reduce_dimensions(local_embeddings)
        except Exception as e:
            logger.warning(f"Local dimension reduction error: {e}")
            reduced_local = local_embeddings
        n_local, means, scores = fit_best(reduced_local, min(self.max_clusters, len(reduced_local) - 1))
        if self.verbose:
            logger.info(f"Local cluster count in global cluster {i}: {n_local}")
        for j in range(n_local):
            cluster = SoftCluster(total_clusters, means[j])
            for k, hash_id in enumerate(local_hash_ids):
                if scores[k, j] >= self.threshold:
                    cluster.add_member(hash_id, scores[k, j])
                    self.hash_id_to_cluster_memberships.setdefault(hash_id, {})[total_clusters] = scores[k, j]
            if len(cluster.members) > 0:
                self.clusters.append(cluster)
            total_clusters += 1
    if self.verbose:
        logger.info(f"Total cluster count: {total_clusters}")
    return self.clusters
