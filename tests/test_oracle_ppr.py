"""oracle/ppr_oracle.py against the end-to-end harness's igraph stand-in (tests/e2e_harness._Graph), which produced
the committed golden trace: random small graphs with parallel edges, both orientations, isolated vertices and
reset mass on them agree within 1e-12.  The stand-in does not sanitise the reset, so resets with NaN or negative
entries go to it after run_ppr's rule (ComoRAG.py:1091)."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import e2e_harness as H  # noqa: E402
from oracle import ppr_oracle as O  # noqa: E402


def _random_graph(rng, n):
    m = int(rng.integers(n, 4 * n))
    a, b = rng.integers(0, n - n // 4, m), rng.integers(0, n - n // 4, m)    # the last quarter stays isolated
    keep = a != b
    e = np.stack([a[keep], b[keep]], 1)
    e = np.concatenate([e, e[: len(e) // 3, ::-1], e[: len(e) // 5]])       # both orientations, parallel edges
    return e, rng.uniform(0.05, 3.0, len(e))


def _stand_in(n, edges, weights):
    g = H._Graph()
    g.add_vertices(n, attributes={"name": [f"v{i}" for i in range(n)]})
    g.add_edges([tuple(map(int, x)) for x in edges], attributes={"weight": list(map(float, weights))})
    return g


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("damping", [0.5, 0.85])
def test_oracle_equals_the_harness_stand_in(seed, damping):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(8, 60))
    edges, weights = _random_graph(rng, n)
    reset = rng.uniform(0, 1, n) * (rng.uniform(size=n) < 0.5)
    reset[n - 1] = 0.8                                                       # mass on an isolated vertex
    got = O.ppr(n, edges, weights, reset, damping)
    want = np.array(_stand_in(n, edges, weights).personalized_pagerank(vertices=range(n), damping=damping,
                                                                       directed=False, weights="weight", reset=reset))
    assert abs(got.sum() - 1) < 1e-12
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)


def test_oracle_sanitises_the_reset_as_run_ppr_does():
    rng = np.random.default_rng(7)
    n = 30
    edges, weights = _random_graph(rng, n)
    reset = rng.uniform(-1, 1, n)
    reset[[2, 5, 11]] = np.nan
    clean = np.where(np.isnan(reset) | (reset < 0), 0, reset)               # ComoRAG.py:1091
    want = np.array(_stand_in(n, edges, weights).personalized_pagerank(vertices=range(n), damping=0.5, reset=clean))
    np.testing.assert_allclose(O.ppr(n, edges, weights, reset, 0.5), want, rtol=0, atol=1e-12)
    with pytest.raises(ValueError):
        O.ppr(n, edges, weights, -np.ones(n), 0.5)


def test_t_step_iterate_converges_to_the_solve_within_the_truncation_bound():
    rng = np.random.default_rng(3)
    n = 40
    edges, weights = _random_graph(rng, n)
    reset = rng.uniform(0, 1, n)
    exact = O.ppr(n, edges, weights, reset, 0.5)
    for T in (0, 1, 5, 35):
        x_T = O.ppr(n, edges, weights, reset, 0.5, iterations=T)
        assert np.abs(x_T - exact).sum() <= 2 * 0.5 ** (T + 1) / 0.5 + 1e-15
