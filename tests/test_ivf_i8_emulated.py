"""The IVF rescore of crag_ivf_search_i8 and its id map on the CPU, against tests/ivf_i8_oracle.py bit for bit (ids and
scores).  tests/warp_emu/ivf_i8_emu_test.cpp runs ivf_rescore_topk_kernel and ivf_map_ids_kernel on emulated
thread blocks.

The layout has empty lists (first, inner and last), lists of exactly 128 and 129 rows and small lists; candidates sit
on list boundaries (the first and last row of a list, the first row of a list's second tile), -1 candidates leave
fewer valid candidates than k, two identical rows in two lists with equal coarse terms tie across lists, and the
original ids lie beyond 2^32.  Two mutants must fail: a list lookup that takes the neighbouring list's coarse term,
and ties kept in descending position order."""
import os
import shutil
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ivf_i8_oracle as io  # noqa: E402

ROOT = os.path.dirname(HERE)
EMU = os.path.join(ROOT, "tests", "warp_emu")
CSRC = os.path.join(ROOT, "comorag_b200", "csrc")
ROW_OFFSET = (1 << 33) + 5


def _build(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-pthread",
                        "-I", os.path.join(EMU, "stub"), "-I", str(csrc_dir), os.path.join(EMU, "ivf_i8_emu_test.cpp"),
                        "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return str(exe)


@pytest.fixture(autouse=True)
def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")


@pytest.fixture(scope="module")
def emulator(tmp_path_factory):
    return _build(CSRC, tmp_path_factory.mktemp("ivf_i8_emu") / "ivf_i8_emu_test")


def _bf16(x):
    """float32 -> (bf16 bits uint16, the bf16 values as float32), rounded to nearest even."""
    b = torch.from_numpy(np.ascontiguousarray(x, np.float32)).bfloat16()
    return b.view(torch.int16).numpy().view(np.uint16), b.float().numpy()


LIST_ROWS = [0, 5, 128, 0, 129, 1, 40, 0]


def _case(rng, dim, nq, n_cand, k):
    """-> (payload, residual values, list_tile_start, coarse [nlist, 32], query values, candidates, row_ids)."""
    nlist = len(LIST_ROWS)
    tiles = [(r + 127) // 128 for r in LIST_ROWS]
    starts = np.concatenate([[0], np.cumsum(tiles)]).astype(np.int32)
    n_rows = int(starts[-1]) * 128
    x = np.zeros((n_rows, dim), np.float32)
    row_ids = np.full(n_rows, -1, np.int64)
    real = []
    nid = 0
    for l, m in enumerate(LIST_ROWS):
        p = starts[l] * 128 + np.arange(m)
        x[p] = rng.standard_normal((m, dim)).astype(np.float32) * 0.1
        row_ids[p] = ROW_OFFSET + nid + np.arange(m) * 3   # ascending, spread out, beyond 2^32
        nid += 3 * m
        real.append(p)
    # ties across two lists: the first row of list 4 repeats row 2 of list 2, and both lists get the same coarse terms
    a, b = starts[2] * 128 + 2, starts[4] * 128
    x[b] = x[a]
    bits, vals = _bf16(x)
    stride = dim + 8
    rows = np.zeros((n_rows, stride), np.uint16)
    rows[:, :dim] = bits
    rows[:, dim:] = 0x7FC0                                   # NaN past dim: never read
    qbits, qvals = _bf16(rng.standard_normal((nq, dim)).astype(np.float32))
    coarse = (rng.standard_normal((nlist, 32)) * 0.5).astype(np.float32)
    coarse[4] = coarse[2]
    # candidates: list boundaries first, then random real rows, then -1
    bounds = [int(starts[l] * 128) for l, m in enumerate(LIST_ROWS) if m] + \
             [int(starts[l] * 128 + m - 1) for l, m in enumerate(LIST_ROWS) if m] + [int(starts[4] * 128 + 128), int(a)]
    pool = np.concatenate(real)
    cand = np.full((nq, n_cand), -1, np.int64)
    for j in range(nq):
        extra = rng.permutation(np.setdiff1d(pool, bounds))
        c = np.concatenate([bounds, extra])[:n_cand]
        cand[j, :len(c)] = rng.permutation(c)
    cand[:, -1] = -1
    if nq > 1:
        cand[1, 3:] = -1                                     # fewer valid candidates than k
    payload = struct.pack("<q6i", n_rows, dim, stride, nq, n_cand, k, nlist) + rows.tobytes() + qbits.tobytes() + \
        cand.tobytes() + starts.tobytes() + coarse.tobytes() + row_ids.tobytes()
    return payload, vals, starts, coarse, qvals, cand, row_ids


def _run(exe, payload, tmp_path):
    fi, fo = tmp_path / "ivf_i8.in", tmp_path / "ivf_i8.out"
    fi.write_bytes(payload)
    r = subprocess.run([exe, str(fi), str(fo)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return fo.read_bytes()


def _check(exe, tmp_path, dim, nq, n_cand, k, seed):
    rng = np.random.default_rng(seed)
    payload, vals, starts, coarse, qvals, cand, row_ids = _case(rng, dim, nq, n_cand, k)
    out = _run(exe, payload, tmp_path)
    got_ids = np.frombuffer(out[: nq * k * 8], np.int64).reshape(nq, k)
    got_sc = np.frombuffer(out[nq * k * 8:], np.float32).reshape(nq, k)
    pos, want_sc = io.rescore(vals, starts, lambda j, l: coarse[l, j], qvals, cand, k)
    want_ids = np.where(pos >= 0, row_ids[np.maximum(pos, 0)], -1)
    assert np.array_equal(got_ids, want_ids), np.argwhere(got_ids != want_ids)[:5]
    assert np.array_equal(got_sc.view(np.uint32), want_sc.view(np.uint32))
    if nq > 1:                                               # 3 candidates, so a -1 / -inf tail
        assert (got_ids[1, 3:] == -1).all() and np.isneginf(got_sc[1, 3:]).all() and (got_ids[1, :3] >= 1 << 32).all()
    return got_ids, got_sc


@pytest.mark.parametrize("dim,nq,n_cand,k", [(64, 3, 128, 128), (128, 5, 40, 10), (768, 32, 100, 64), (1024, 2, 16, 1)])
def test_ivf_rescore_matches_oracle(emulator, tmp_path, dim, nq, n_cand, k):
    _check(emulator, tmp_path, dim, nq, n_cand, k, seed=dim + k)


def test_list_lookup_skips_empty_lists():
    starts = np.array([0, 0, 1, 1, 3, 3, 4], np.int32)       # lists 0, 2, 4 empty; list 3 holds two tiles
    p = np.array([0, 127, 128, 255, 256, 383, 384, 511])
    assert io.list_of_positions(starts, p).tolist() == [1, 1, 3, 3, 3, 3, 5, 5]


def test_ties_across_lists_in_ascending_position(emulator, tmp_path):
    rng = np.random.default_rng(11)
    nq, n_cand, k = 2, 128, 128
    payload, vals, starts, coarse, qvals, cand, row_ids = _case(rng, 128, nq, n_cand, k)
    got_ids, got_sc = _check(emulator, tmp_path, 128, nq, n_cand, k, seed=11)
    a, b = starts[2] * 128 + 2, starts[4] * 128
    ia, ib = list(got_ids[0]).index(row_ids[a]), list(got_ids[0]).index(row_ids[b])
    assert got_sc[0, ia] == got_sc[0, ib] and ib == ia + 1  # the tie: adjacent, the smaller position first


# ------------------------------------------------------------------------------------------------ mutants
MUTANTS = {
    "coarse term of the neighbouring list": ("if (__ldg(&list_tile_start[mid]) <= tile) lo = mid;",
                                             "if (__ldg(&list_tile_start[mid]) < tile) lo = mid;"),
    "ties in descending position order": ("key = make_key(partial, uint32_t(local));",
                                          "key = make_key(partial, 0x7FFFFFFFu - uint32_t(local));"),
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutant_fails(tmp_path, name):
    old, new = MUTANTS[name]
    mdir = tmp_path / "csrc"
    shutil.copytree(CSRC, mdir)
    src = (mdir / "quant_kernels.cuh").read_text()
    assert src.count(old) == 1
    src = src.replace(old, new)
    if name.startswith("ties"):   # the positions come back through key_id, so undo the mutation's map on the way out
        src = src.replace("int64_t(key_id(v[j]))", "int64_t(0x7FFFFFFFu - key_id(v[j]))")
    (mdir / "quant_kernels.cuh").write_text(src)
    exe = _build(mdir, tmp_path / "mutant")
    tests = [lambda: test_ties_across_lists_in_ascending_position(exe, tmp_path),
             lambda: test_ivf_rescore_matches_oracle(exe, tmp_path, 128, 5, 40, 10)]
    failed = 0
    for t in tests:
        try:
            t()
        except (AssertionError, ValueError):
            failed += 1
    assert failed > 0, f"mutant '{name}' passed every check"
