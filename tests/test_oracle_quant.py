"""oracle/quant_oracle.py on the CPU: its quantiser against an independent torch formulation, the bound that makes the
int8 scan's fp32 conversion exact, and the recall of the whole int8-scan + bf16-rescore pipeline."""
import numpy as np
import torch

from oracle import quant_oracle as qo


def _bf16_values(x):
    return torch.from_numpy(np.ascontiguousarray(x, np.float32)).bfloat16().float().numpy()


def _torch_quantize(x: np.ndarray, dim8: int):
    """The quantiser restated with torch ops: scale by true division, round half to even, clamp."""
    t = torch.from_numpy(x)
    amax = t.abs().amax(dim=1)
    s = torch.div(amax, torch.tensor(127.0, dtype=torch.float32))
    safe = torch.where(s == 0, torch.ones_like(s), s)
    q = torch.round(t / safe[:, None]).clamp(-127, 127)
    q = torch.where(s[:, None] == 0, torch.zeros_like(q), q).to(torch.int8)
    out = torch.zeros((x.shape[0], dim8), dtype=torch.int8)
    out[:, : x.shape[1]] = q
    return out.numpy(), s.numpy()


def test_quantiser_matches_torch_formulation():
    rng = np.random.default_rng(0)
    for dim in (64, 384, 1000, 1024):
        x = rng.standard_normal((500, dim)).astype(np.float32) * rng.uniform(1e-3, 10, (500, 1)).astype(np.float32)
        x[0] = 0
        x[1, :3] = [127 / 128, 0.5 / 128, -2.5 / 128]          # exact .5 ties of x / s (s = 2^-7)
        x[1, 3:] = 0
        x[2] = rng.integers(-127, 128, dim) * np.float32(2.0 ** -133)   # bf16 denormals
        x = _bf16_values(x)
        q, s = qo.quantize(x)
        tq, ts = _torch_quantize(x, qo.dim8_of(dim))
        assert np.array_equal(s.view(np.uint32), ts.view(np.uint32))
        assert np.array_equal(q, tq)
        assert list(q[1, :3]) == [127, 0, -2]                   # half to even
        assert q.shape[1] % 128 == 0 and not q[:, dim:].any()


def test_integer_dot_bound_at_dim_1024():
    """All-+-127 rows at dim 1024 reach |acc| = 127^2 * 1024 < 2^24: the s32 -> fp32 conversion and every float32
    partial sum of the oracle are exact."""
    a = np.full((2, 1024), 127, np.int8)
    a[1] = -127
    acc = qo.s1_scores(a, np.ones(2, np.float32), a, np.ones(2, np.float32))
    assert abs(int(acc[0, 1])) == 127 * 127 * 1024 < 2 ** 24
    assert np.array_equal(acc, np.array([[1, -1], [-1, 1]], np.float32) * 127 * 127 * 1024)
    assert float(np.float32(127 * 127 * 1024)) == 127 * 127 * 1024


def test_oracle_recall_k10_40_candidates_200k():
    """Seeded 200k x 1024 random unit rows (bf16), 32 queries: the pipeline's top 10 from 40 candidates against the
    exact bf16 top 10.  Rows are processed in chunks to keep memory modest."""
    rng = np.random.default_rng(2026)
    n, dim, nq, k, cand = 200_000, 1024, 32, 10, 40
    q = rng.standard_normal((nq, dim), dtype=np.float32)
    q = _bf16_values(q / np.linalg.norm(q, axis=1, keepdims=True))
    q8, qs = qo.quantize(q)
    exact_s = np.full((nq, 0), -np.inf)
    exact_i = np.zeros((nq, 0), np.int64)
    s1_s = np.full((nq, 0), -np.inf, np.float32)
    s1_i = np.zeros((nq, 0), np.int64)
    rows = []
    for r0 in range(0, n, 25_000):
        x = rng.standard_normal((25_000, dim), dtype=np.float32)
        x = _bf16_values(x / np.linalg.norm(x, axis=1, keepdims=True))
        rows.append(torch.from_numpy(x).bfloat16())
        ex = q.astype(np.float64) @ x.astype(np.float64).T
        x8, xs = qo.quantize(x)
        s1 = qo.s1_scores(x8, xs, q8, qs)
        ids = np.arange(r0, r0 + x.shape[0])
        exact_s, exact_i = np.concatenate([exact_s, ex], 1), np.concatenate([exact_i, np.tile(ids, (nq, 1))], 1)
        s1_s, s1_i = np.concatenate([s1_s, s1], 1), np.concatenate([s1_i, np.tile(ids, (nq, 1))], 1)
        keep = np.argsort(-exact_s, axis=1, kind="stable")[:, :k]
        exact_s, exact_i = np.take_along_axis(exact_s, keep, 1), np.take_along_axis(exact_i, keep, 1)
        keep = np.argsort(-s1_s, axis=1, kind="stable")[:, :cand]
        s1_s, s1_i = np.take_along_axis(s1_s, keep, 1), np.take_along_axis(s1_i, keep, 1)
    allrows = torch.cat(rows).float().numpy()
    ids, _ = qo.rescore(allrows, n, 0, q, s1_i, k)
    recall = np.mean([len(set(ids[j]) & set(exact_i[j])) / k for j in range(nq)])
    assert recall >= 0.99, recall
