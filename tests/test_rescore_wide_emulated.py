"""crag_rescore_topk above 128 candidates (rescore_wide_kernel, csrc/quant_kernels.cuh) on the CPU, against
oracle/quant_oracle.py bit for bit (ids and scores).  tests/warp_emu/rescore_wide_emu_test.cpp runs the kernel on
emulated 512-thread blocks.

Cases: n_cand from 129 to 2048, k = 1 and k = n_cand, duplicate rows whose tied S2 must come out in ascending row order
(their candidate slots are in descending row order), an all-zero query (every S2 ties at 0), ids -1 and out of range on
both sides, and a nonzero row_offset.  The row buffer holds rows past n_rows with large values, so reading a row
outside the shard changes the answer.  Three mutants must fail: ties broken by candidate slot instead of row, a changed
dot order, and reading a row past the shard."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest
import torch

from oracle import quant_oracle as qo

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EMU = os.path.join(ROOT, "tests", "warp_emu")
CSRC = os.path.join(ROOT, "comorag_b200", "csrc")
EXTRA = 8                                                    # rows allocated past the shard


def _build(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-pthread",
                        "-I", os.path.join(EMU, "stub"), "-I", str(csrc_dir), os.path.join(EMU, "rescore_wide_emu_test.cpp"),
                        "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return str(exe)


@pytest.fixture(autouse=True)
def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")


@pytest.fixture(scope="module")
def emulator(tmp_path_factory):
    return _build(CSRC, tmp_path_factory.mktemp("rescore_wide_emu") / "rescore_wide_emu_test")


def _bf16(x):
    """float32 -> (bf16 bits uint16, the bf16 values as float32), rounded to nearest even."""
    b = torch.from_numpy(np.ascontiguousarray(x, np.float32)).bfloat16()
    return b.view(torch.int16).numpy().view(np.uint16), b.float().numpy()


def _case(rng, n_rows, dim, nq, n_cand, k, row_offset):
    stride = dim + 8
    x = rng.standard_normal((n_rows + EXTRA, dim)).astype(np.float32)
    x[5] = x[3]                                              # duplicate rows: tied S2, ascending row order
    x[9] = x[3]
    x[n_rows:] = 64.0                                        # past the shard: would win every query it is read for
    bits, vals = _bf16(x)
    qbits, qvals = _bf16(rng.standard_normal((nq, dim)).astype(np.float32))
    qbits[nq - 1] = 0                                        # an all-zero query: every S2 ties at 0
    qvals[nq - 1] = 0
    cand = np.stack([rng.permutation(n_rows)[:n_cand] for _ in range(nq)]).astype(np.int64)
    for j in range(nq):                                      # the duplicates in descending row order of their slots
        rest = cand[j][~np.isin(cand[j], [3, 5, 9])]
        cand[j] = np.concatenate([[9, 5, 3], rest[:n_cand - 3]])
    cand += row_offset
    cand[:, -1] = -1                                         # -1 and out-of-range ids are no candidates
    cand[:, -2] = row_offset + n_rows                        # the first row past the shard
    cand[:, -3] = row_offset + n_rows + EXTRA - 1
    cand[1 % nq, 3] = row_offset - 1
    rows = np.zeros((n_rows + EXTRA, stride), np.uint16)
    rows[:, :dim] = bits
    rows[:, dim:] = 0x7FC0                                   # NaN past dim: must never be read
    payload = struct.pack("<3q5i", n_rows, n_rows + EXTRA, row_offset, dim, stride, nq, n_cand, k) + rows.tobytes() + \
        qbits.tobytes() + cand.tobytes()
    return payload, vals[:n_rows], qvals, cand


def _run(exe, payload, tmp_path):
    fi, fo = tmp_path / "wide.in", tmp_path / "wide.out"
    fi.write_bytes(payload)
    r = subprocess.run([exe, str(fi), str(fo)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return fo.read_bytes()


CASES = [(64, 129, 1, 0), (384, 129, 129, 1 << 33), (1000, 300, 10, 0), (128, 1000, 1000, 7),
         (1024, 2048, 1, 1 << 33), (256, 2048, 2048, 0), (1024, 2048, 100, 0)]


@pytest.mark.parametrize("dim,n_cand,k,row_offset", CASES)
def test_rescore_wide_matches_oracle(emulator, tmp_path, dim, n_cand, k, row_offset):
    rng = np.random.default_rng(dim * 10_000 + n_cand + k)
    n_rows, nq = n_cand + 50, 4
    payload, vals, qvals, cand = _case(rng, n_rows, dim, nq, n_cand, k, row_offset)
    out = _run(emulator, payload, tmp_path)
    got_ids = np.frombuffer(out[: nq * k * 8], np.int64).reshape(nq, k)
    got_sc = np.frombuffer(out[nq * k * 8:], np.float32).reshape(nq, k)
    want_ids, want_sc = qo.rescore(vals, n_rows, row_offset, qvals, cand, k)
    assert np.array_equal(got_ids, want_ids)
    assert np.array_equal(got_sc.view(np.uint32), want_sc.view(np.uint32))
    assert ((got_ids == -1) | ((got_ids >= row_offset) & (got_ids < row_offset + n_rows))).all()
    if k == n_cand:                                          # the invalid candidates leave -1 / -inf at the tail
        assert (got_ids[:, -3:] == -1).all() and np.isneginf(got_sc[:, -3:]).all()
    z = got_ids[nq - 1][got_ids[nq - 1] >= 0]                # the zero query: all tied, ascending rows
    assert (np.diff(z) > 0).all()


def test_rescore_wide_ties_in_ascending_row_order(emulator, tmp_path):
    """Rows 3, 5 and 9 are equal and sit in candidate slots 0, 1, 2 in descending row order; the query equal to row 3
    ranks them first, in ascending row order."""
    rng = np.random.default_rng(11)
    n_rows, dim, nq, n_cand, k = 400, 128, 2, 200, 3
    payload, vals, qvals, cand = _case(rng, n_rows, dim, nq, n_cand, k, 0)
    q = vals[3].copy()
    qbits, _ = _bf16(q[None])
    head = struct.calcsize("<3q5i") + (n_rows + EXTRA) * (dim + 8) * 2
    payload = payload[:head] + qbits.tobytes() + payload[head + dim * 2:]
    qvals = qvals.copy()
    qvals[0] = q
    out = _run(emulator, payload, tmp_path)
    ids = np.frombuffer(out[: nq * k * 8], np.int64).reshape(nq, k)
    want, _ = qo.rescore(vals, n_rows, 0, qvals, cand, k)
    assert np.array_equal(ids, want)
    assert list(ids[0]) == [3, 5, 9]


# ------------------------------------------------------------------------------------------------ mutants
MUTANTS = {
    "ties broken by candidate slot": [
        ("if (lane == 0) s_keys[c] = key;", "if (lane == 0) s_keys[c] = key ? (key >> 32 << 32) | (0xFFFFFFFFu - uint32_t(c)) : 0;"),
        ("key ? int64_t(key_id(key)) + row_offset : -1", "key ? cand[key_id(key)] : -1")],
    "changed dot order": [("for (int o = 16; o > 0; o >>= 1) partial = __fadd_rn(partial, __shfl_xor_sync",
                           "for (int o = 1; o < 32; o <<= 1) partial = __fadd_rn(partial, __shfl_xor_sync")],
    "a row past the shard": [("if (local >= 0 && local < n_rows) {", "if (local >= 0 && local < n_rows + 8) {")],
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutant_fails(tmp_path, name):
    mdir = tmp_path / "csrc"
    shutil.copytree(CSRC, mdir)
    src = (mdir / "quant_kernels.cuh").read_text()
    for old, new in MUTANTS[name]:
        assert src.count(old) == 1, old
        src = src.replace(old, new)
    (mdir / "quant_kernels.cuh").write_text(src)
    exe = _build(mdir, tmp_path / "mutant")
    tests = [lambda: test_rescore_wide_ties_in_ascending_row_order(exe, tmp_path)]
    tests += [lambda c=c: test_rescore_wide_matches_oracle(exe, tmp_path, *c) for c in (CASES[2], CASES[4])]
    failed = 0
    for t in tests:
        try:
            t()
        except AssertionError:
            failed += 1
    assert failed > 0, f"mutant '{name}' passed every check"
