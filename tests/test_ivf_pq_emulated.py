"""The PQ kernels of crag_ivf_search_pq on the CPU, against tests/ivf_pq_oracle.py bit for bit.
tests/warp_emu/ivf_pq_emu_test.cpp runs pq_encode_kernel, pq_table_kernel, the IVF plan, pq_scan_kernel and the merge
of its per-CTA lists on emulated thread blocks; the scan's blocks also run interleaved (all resident together).

The layout has empty lists (first, inner and last), lists of 1, 127, 128 and 129 rows, two identical rows in two lists
with equal coarse terms (the tie goes to the smaller position), duplicate codewords (equal distances go to the smaller
codeword), and probes of -1, out-of-range ids and a list probed twice.  Two mutants must fail: an encode that sends
equal distances to the larger codeword, and a scan that scores rows of lists the query does not probe."""
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
import ivf_pq_oracle as po  # noqa: E402

ROOT = os.path.dirname(HERE)
EMU = os.path.join(ROOT, "tests", "warp_emu")
CSRC = os.path.join(ROOT, "comorag_b200", "csrc")


def _build(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-pthread",
                        "-I", os.path.join(EMU, "stub"), "-I", EMU, "-I", str(csrc_dir),
                        os.path.join(EMU, "ivf_pq_emu_test.cpp"), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return str(exe)


@pytest.fixture(autouse=True)
def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")


@pytest.fixture(scope="module")
def emulator(tmp_path_factory):
    return _build(CSRC, tmp_path_factory.mktemp("ivf_pq_emu") / "ivf_pq_emu_test")


def _bf16(x):
    """float32 -> (bf16 bits uint16, the bf16 values as float32), rounded to nearest even."""
    b = torch.from_numpy(np.ascontiguousarray(x, np.float32)).bfloat16()
    return b.view(torch.int16).numpy().view(np.uint16), b.float().numpy()


LIST_ROWS = [0, 1, 127, 0, 128, 129, 40, 0]


def _case(rng, dim, m, nq, nprobe):
    nlist = len(LIST_ROWS)
    dsub = dim // m
    tiles = [(r + 127) // 128 for r in LIST_ROWS]
    starts = np.concatenate([[0], np.cumsum(tiles)]).astype(np.int32)
    n_rows = int(starts[-1]) * 128
    x = np.zeros((n_rows, dim), np.float32)
    for l, r in enumerate(LIST_ROWS):
        x[starts[l] * 128 + np.arange(r)] = rng.standard_normal((r, dim)).astype(np.float32) * 0.1
    q = rng.standard_normal((nq, dim)).astype(np.float32)
    a, b = starts[2] * 128 + 3, starts[5] * 128 + 128          # identical rows in lists 2 and 5, close to query 1
    x[a] = x[b] = 0.05 * q[min(1, nq - 1)]
    bits, vals = _bf16(x)
    cb = rng.standard_normal((m, 256, dsub)).astype(np.float32) * 0.1
    cb[:, 9] = cb[:, 4]                                         # duplicate codewords
    real = np.concatenate([starts[l] * 128 + np.arange(r) for l, r in enumerate(LIST_ROWS)])
    cb[:, 4] = vals[real[:1]].reshape(m, dsub)                  # one row sits exactly on codewords 4 and 9
    cb[:, 9] = cb[:, 4]
    qbits, qvals = _bf16(q)
    coarse = (rng.standard_normal((nq, nlist)) * 0.5).astype(np.float32)
    coarse[:, 5] = coarse[:, 2]
    probed = np.stack([rng.permutation(nlist)[:nprobe] for _ in range(nq)]).astype(np.int64)
    probed[:, 0] = 2
    probed[:, 1] = 5
    if nprobe >= 5:
        probed[0, 2], probed[0, 3], probed[0, 4] = -1, nlist + 3, 2     # absent, out of range, probed twice
    scores = np.take_along_axis(coarse, np.clip(probed, 0, nlist - 1), axis=1)
    return dict(n_rows=n_rows, starts=starts, bits=bits, vals=vals, cb=cb, qbits=qbits, qvals=qvals,
                probed=(probed, scores), ab=(a, b))


def _run(exe, tmp_path, c, dim, m, nq, n_cand, slices, seed):
    probed, scores = c["probed"]
    cs = (m + 15) // 16 * 16
    payload = struct.pack("<q9i", c["n_rows"], dim, m, cs, nq, probed.shape[1], len(LIST_ROWS), n_cand, slices, seed) + \
        c["bits"].tobytes() + c["cb"].tobytes() + c["qbits"].tobytes() + probed.tobytes() + scores.tobytes() + \
        c["starts"].tobytes() + np.array(LIST_ROWS, np.int32).tobytes()
    fi, fo = tmp_path / "ivf_pq.in", tmp_path / "ivf_pq.out"
    fi.write_bytes(payload)
    r = subprocess.run([exe, str(fi), str(fo)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = fo.read_bytes()
    sizes = [c["n_rows"] * cs, nq * m * 256 * 4, nq * n_cand * 8, nq * n_cand * 4, nq * 2 * 4]
    parts, at = [], 0
    for s in sizes:
        parts.append(out[at:at + s])
        at += s
    codes = np.frombuffer(parts[0], np.uint8).reshape(c["n_rows"], cs)
    lut = np.frombuffer(parts[1], np.float32).reshape(nq, m, 256)
    pos = np.frombuffer(parts[2], np.int64).reshape(nq, n_cand)
    s1 = np.frombuffer(parts[3], np.float32).reshape(nq, n_cand)
    mm = np.frombuffer(parts[4], np.float32).reshape(nq, 2)
    return codes, lut, pos, s1, mm


def _check(exe, tmp_path, dim, m, nq, nprobe, n_cand, slices, seed, case_seed):
    c = _case(np.random.default_rng(case_seed), dim, m, nq, nprobe)
    codes, lut, pos, s1, mm = _run(exe, tmp_path, c, dim, m, nq, n_cand, slices, seed)
    want_codes = po.encode(c["vals"], c["cb"])
    assert np.array_equal(codes[:, :m], want_codes), np.argwhere(codes[:, :m] != want_codes)[:5]
    assert not codes[:, m:].any()                                    # the padding bytes are not written
    assert np.array_equal(lut.view(np.uint32), po.table(c["qvals"], c["cb"]).view(np.uint32))
    row_ids = np.arange(c["n_rows"], dtype=np.int64)
    _, _, want_mm, (want_pos, want_s1) = po.search_pq(c["vals"], want_codes, c["cb"], row_ids, c["starts"],
                                                      np.array(LIST_ROWS, np.int32), c["qvals"], c["probed"],
                                                      1, n_cand)
    assert np.array_equal(pos, want_pos), np.argwhere(pos != want_pos)[:5]
    assert np.array_equal(s1.view(np.uint32), want_s1.view(np.uint32))
    assert np.array_equal(mm.view(np.uint32), want_mm.view(np.uint32))
    return c, codes, pos


@pytest.mark.parametrize("dim,m,nq,nprobe,n_cand,slices,seed", [
    (64, 8, 3, 5, 128, 2, 0),
    (192, 96, 5, 8, 40, 3, 0),
    (192, 192, 2, 6, 10, 1, 0),
    (128, 16, 32, 8, 64, 2, 0),
    (64, 8, 4, 5, 128, 3, 7),         # interleaved CTAs
    (192, 96, 3, 8, 33, 2, 11),       # interleaved CTAs
])
def test_pq_kernels_match_oracle(emulator, tmp_path, dim, m, nq, nprobe, n_cand, slices, seed):
    _check(emulator, tmp_path, dim, m, nq, nprobe, n_cand, slices, seed, case_seed=dim + m + nq)


def test_equal_distances_and_tied_rows_go_to_the_smaller_index(emulator, tmp_path):
    c, codes, pos = _check(emulator, tmp_path, 64, 8, 2, 5, 128, 2, 0, case_seed=5)
    assert np.array_equal(codes[c["ab"][0]], codes[c["ab"][1]])
    first = c["starts"][1] * 128                               # list 1's only row sits on codewords 4 and 9
    assert (codes[first, :8] == 4).all()
    a, b = c["ab"]
    p = list(pos[1])
    assert a in p and b in p and p.index(a) < p.index(b)         # equal S1 (same codes, same coarse term)


# ------------------------------------------------------------------------------------------------ mutants
MUTANTS = {
    "equal distances to the larger codeword": ("if (d < best) { best = d; best_c = c; }",
                                               "if (d <= best) { best = d; best_c = c; }"),
    "rows of unprobed lists scored": ("if (r >= item.y || !((__ldg(&plan.list_mask[item.z]) >> q) & 1u)) return 0ull;",
                                      "if (r >= item.y) return 0ull;"),
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutant_fails(tmp_path, name):
    old, new = MUTANTS[name]
    mdir = tmp_path / "csrc"
    shutil.copytree(CSRC, mdir)
    src = (mdir / "pq_kernels.cuh").read_text()
    assert src.count(old) == 1
    (mdir / "pq_kernels.cuh").write_text(src.replace(old, new))
    exe = _build(mdir, tmp_path / "mutant")
    tests = [lambda: test_equal_distances_and_tied_rows_go_to_the_smaller_index(exe, tmp_path),
             lambda: _check(exe, tmp_path, 192, 96, 5, 8, 40, 3, 0, case_seed=9)]
    failed = 0
    for t in tests:
        try:
            t()
        except AssertionError:
            failed += 1
    assert failed > 0, f"mutant '{name}' passed every check"
