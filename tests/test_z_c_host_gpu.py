"""crag_search_topk driven by a host with no Python / torch in it (examples/c_host_search.cu), on the GPU.
Kept in its own, alphabetically last file: it shells out to a separate binary, so under `pytest -x` nothing it does can
hide the result of an in-process parity test."""
import json
import subprocess

import pytest


@pytest.mark.gpu
def test_c_host_search_ids_exact_through_the_c_abi():
    """crag_search_topk called from a plain CUDA-runtime host: planted-neighbour shards whose exact top-k is known in
    closed form (ids exact, scores / max within 1e-3).  Shapes = one rank's shard of the 8-GPU split."""
    from comorag_b200 import build
    exe = build.build_examples()
    for rows, dim, nq, k in ((1_250_000, 1024, 32, 10), (1_250_000, 1024, 32, 100), (1_250_000, 1024, 32, 128)):
        r = subprocess.run([str(exe), str(rows), str(dim), str(nq), str(k), "5"], capture_output=True, text=True, timeout=300)
        assert r.returncode == 0, r.stderr + r.stdout
        line = json.loads(r.stdout.strip().splitlines()[-1])
        assert line["ok"] and line["id_mismatches"] == 0 and line["max_score_err"] < 1e-3
