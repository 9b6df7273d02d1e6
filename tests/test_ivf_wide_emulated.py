"""The wide IVF stage 1 and rescore (crag_ivf_search_i8_wide / _pq_wide) on the CPU, bit for bit against
tests/ivf_wide_oracle.py with tests/ivf_i8_oracle.py and tests/ivf_pq_oracle.py.  tests/warp_emu/ivf_wide_emu_test.cpp
runs the IVF plan, the wide plan, the int8 or PQ fill, the ragged select, the slot map and the wide IVF rescore of one
32-query pass on emulated thread blocks.

The layout has empty lists (first, inner and last), one-row lists and lists spanning many tiles; probes hold -1,
out-of-range ids and lists probed twice; two lists share a coarse term and hold an identical row, and one list holds
a duplicate row, so S1 and S2 tie inside and across lists.  Cases cover n_q < n_cand, a query with no probed rows and
a max_probe_rows below a query's probed rows, whose slots past it stay unwritten.  Four mutants must fail: probes
sorted descending, a repeated probe counted twice, the coarse term added before the PQ sum, and rescore ties broken
by candidate slot."""
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
import ivf_pq_oracle as po  # noqa: E402
import ivf_wide_oracle as wo  # noqa: E402
from oracle import quant_oracle as qo  # noqa: E402

ROOT = os.path.dirname(HERE)
EMU = os.path.join(ROOT, "tests", "warp_emu")
CSRC = os.path.join(ROOT, "comorag_b200", "csrc")
SENTINEL = 0x7FBADBAD

LIST_ROWS = [0, 1, 300, 0, 128, 129, 700, 1, 40, 0]


def _build(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-pthread",
                        "-I", os.path.join(EMU, "stub"), "-I", EMU, "-I", str(csrc_dir),
                        os.path.join(EMU, "ivf_wide_emu_test.cpp"), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return str(exe)


@pytest.fixture(autouse=True)
def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")


@pytest.fixture(scope="module")
def emulator(tmp_path_factory):
    return _build(CSRC, tmp_path_factory.mktemp("ivf_wide_emu") / "ivf_wide_emu_test")


def _bf16(x):
    """float32 -> (bf16 bits uint16, the bf16 values as float32), rounded to nearest even."""
    b = torch.from_numpy(np.ascontiguousarray(x, np.float32)).bfloat16()
    return b.view(torch.int16).numpy().view(np.uint16), b.float().numpy()


def _case(seed, dim, nq, nprobe):
    rng = np.random.default_rng(seed)
    nlist = len(LIST_ROWS)
    tiles = [(r + 127) // 128 for r in LIST_ROWS]
    starts = np.concatenate([[0], np.cumsum(tiles)]).astype(np.int32)
    n_rows = int(starts[-1]) * 128
    x = np.zeros((n_rows, dim), np.float32)
    for l, r in enumerate(LIST_ROWS):
        x[starts[l] * 128 + np.arange(r)] = rng.standard_normal((r, dim)).astype(np.float32) * 0.1
    a, b = starts[2] * 128 + 5, starts[5] * 128 + 128               # identical rows in lists 2 and 5
    x[b] = x[a]
    x[starts[6] * 128 + 600] = x[starts[6] * 128 + 3]               # a duplicate inside list 6
    bits, vals = _bf16(x)
    qbits, qvals = _bf16(rng.standard_normal((nq, dim)).astype(np.float32))
    coarse = (rng.standard_normal((nq, nlist)) * 0.5).astype(np.float32)
    coarse[:, 5] = coarse[:, 2]
    probed = np.stack([rng.permutation(nlist)[:nprobe] for _ in range(nq)]).astype(np.int64)
    probed[:, 0], probed[:, 1] = 5, 2
    probed[0, 2], probed[0, 3], probed[0, 4] = -1, nlist + 3, 5          # absent, out of range, probed twice
    probed[1 % nq, 2] = 2
    probed[nq - 1] = [0, 3, -1, nlist, 9] + [-1] * (nprobe - 5)          # only empty lists: no probed rows
    scores = np.take_along_axis(coarse, np.clip(probed, 0, nlist - 1), axis=1)
    return dict(n_rows=n_rows, starts=starts, bits=bits, vals=vals, qbits=qbits, qvals=qvals, probed=(probed, scores),
                rng=rng)


def _run(exe, tmp_path, c, mode, nq, n_cand, k, cap, slices, width, tail):
    probed, scores = c["probed"]
    dim = c["vals"].shape[1]
    payload = struct.pack("<11i", mode, c["n_rows"], dim, nq, probed.shape[1], len(LIST_ROWS), n_cand, k, cap, slices,
                          width) + c["bits"].tobytes() + c["qbits"].tobytes() + probed.tobytes() + scores.tobytes() + \
        c["starts"].tobytes() + np.array(LIST_ROWS, np.int32).tobytes() + tail
    fi, fo = tmp_path / "wide.in", tmp_path / "wide.out"
    fi.write_bytes(payload)
    r = subprocess.run([exe, str(fi), str(fo)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = fo.read_bytes()
    ld = (cap + 3) // 4 * 4
    spec = [("n_q", np.int32, (nq,)), ("block", np.float32, (nq, ld)), ("slots", np.int64, (nq, n_cand)),
            ("cand", np.int64, (nq, n_cand)), ("cand_s1", np.float32, (nq, n_cand)), ("mm", np.float32, (nq, 2)),
            ("pos", np.int64, (nq, k)), ("s2", np.float32, (nq, k))]
    got, at = {}, 0
    for name, dt, shape in spec:
        n = int(np.prod(shape)) * np.dtype(dt).itemsize
        got[name] = np.frombuffer(out[at:at + n], dt).reshape(shape)
        at += n
    assert at == len(out)
    return got


def _check(exe, tmp_path, mode, nq, nprobe, n_cand, k, cap, slices, seed, width):
    dim = 128 if mode == 0 else 64
    c = _case(seed, dim, nq, nprobe)
    vals, starts = c["vals"], c["starts"]
    probed, _ = c["probed"]
    per_q = io._probed_of(c["probed"], nq, len(LIST_ROWS))
    if mode == 0:
        r8, rs = qo.quantize(vals, width)
        q8, qs = qo.quantize(c["qvals"], width)
        tail = r8.tobytes() + rs.tobytes() + q8.tobytes() + qs.tobytes()
        s1_of = lambda i, p: qo.s1_scores(r8[p], rs[p], q8[i:i + 1], qs[i:i + 1])[0]
    else:
        m = width
        cb = (c["rng"].standard_normal((m, 256, dim // m)) * 0.1).astype(np.float32)
        codes = po.encode(vals, cb)
        codes[[starts[6] * 128 + 7, starts[6] * 128 + 8]] = codes[starts[2] * 128 + 5]   # equal S1, different S2
        stored = np.zeros((c["n_rows"], (m + 15) // 16 * 16), np.uint8)
        stored[:, :m] = codes
        tail = stored.tobytes() + cb.tobytes()
        lut = po.table(c["qvals"], cb)
        s1_of = lambda i, p: po.pq_sums(lut[i], codes[p])
    got = _run(exe, tmp_path, c, mode, nq, n_cand, k, cap, slices, width, tail)
    want_cand = np.full((nq, n_cand), -1, np.int64)
    for i in range(nq):
        p = wo.slot_positions(probed[i], starts, LIST_ROWS, len(LIST_ROWS), cap)
        assert got["n_q"][i] == p.size, (i, got["n_q"][i], p.size)
        lists = io.list_of_positions(starts, p)
        s1 = (s1_of(i, p) + np.array([per_q[i][int(l)] for l in lists], np.float32)).astype(np.float32) if p.size \
            else np.zeros(0, np.float32)
        blk = got["block"][i].view(np.uint32)
        assert np.array_equal(blk[:p.size], s1.view(np.uint32)), f"query {i}: S1 block"
        assert (blk[p.size:] == SENTINEL).all(), f"query {i}: a slot past n_q was written"
        slots, pos, sc, mm = wo.stage1(s1, p, n_cand)
        assert np.array_equal(got["slots"][i], slots), f"query {i}: slots {np.argwhere(got['slots'][i] != slots)[:5]}"
        assert np.array_equal(got["cand"][i], pos), f"query {i}: positions"
        assert np.array_equal(got["cand_s1"][i].view(np.uint32), sc.view(np.uint32)), f"query {i}: candidate S1"
        assert np.array_equal(got["mm"][i].view(np.uint32), mm.view(np.uint32)), f"query {i}: minmax"
        want_cand[i] = pos
    want_pos, want_s2 = io.rescore(vals, starts, lambda j, l: per_q[j][int(l)], c["qvals"], want_cand, k)
    assert np.array_equal(got["pos"], want_pos), np.argwhere(got["pos"] != want_pos)[:5]
    assert np.array_equal(got["s2"].view(np.uint32), want_s2.view(np.uint32))
    return got


FULL = sum(LIST_ROWS)
CASES = [  # mode, nq, nprobe, n_cand, k, cap, slices, seed, width (int8 dim8 / PQ m)
    (0, 3, 6, 200, 50, FULL, 2, 1, 128),
    (0, 5, 8, 1500, 1500, FULL, 3, 2, 128),      # n_q < n_cand for every query
    (0, 4, 7, 129, 129, 150, 1, 3, 128),         # max_probe_rows below the probed rows
    (1, 3, 6, 300, 20, FULL, 2, 4, 8),
    (1, 32, 8, 64, 64, 1001, 3, 5, 16),
    (1, 6, 9, 2048, 100, 333, 2, 6, 32),
]


@pytest.mark.parametrize("mode,nq,nprobe,n_cand,k,cap,slices,seed,width", CASES)
def test_wide_stage1_and_rescore_match_oracle(emulator, tmp_path, mode, nq, nprobe, n_cand, k, cap, slices, seed, width):
    got = _check(emulator, tmp_path, mode, nq, nprobe, n_cand, k, cap, slices, seed, width)
    assert got["n_q"][nq - 1] == 0 and (got["slots"][nq - 1] == -1).all() and np.isneginf(got["s2"][nq - 1]).all()


# ------------------------------------------------------------------------------------------------ mutants
MUTANTS = {
    "probes sorted descending": [("ivf_kernels.cuh", "rank += s_probe[u] < l ? 1 : 0;", "rank += s_probe[u] > l ? 1 : 0;")],
    "a repeated probe counted twice": [("ivf_kernels.cuh", "for (int u = 0; u < t; ++u) keep = keep && s_probe[u] != l;", "")],
    "coarse term added before the PQ sum": [
        ("pq_kernels.cuh", "pq_row_sum(const uint8_t* __restrict__ row_codes, int m, const float* table) {\n  float acc = 0.f;",
         "pq_row_sum(const uint8_t* __restrict__ row_codes, int m, const float* table, float acc0 = -0.f) {\n  float acc = acc0;"),
        ("pq_kernels.cuh", "acc = j == 0 ? x : __fadd_rn(acc, x);", "acc = j == 0 && acc0 == -0.f ? x : __fadd_rn(acc, x);"),
        ("ivf_wide_kernels.cuh", "__fadd_rn(pq_row_sum(codes + pos * code_stride, m, table), coarse)",
         "pq_row_sum(codes + pos * code_stride, m, table, coarse)")],
    "rescore ties by candidate slot": [
        ("quant_kernels.cuh", "if (lane == 0) s_keys[c] = key;", "if (lane == 0) s_keys[c] = key ? (key >> 32 << 32) | uint32_t(c) : 0;"),
        ("quant_kernels.cuh", "key ? int64_t(key_id(key)) + row_offset : -1", "key ? cand[key_id(key)] : -1")],
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutant_fails(tmp_path, name):
    mdir = tmp_path / "csrc"
    shutil.copytree(CSRC, mdir)
    for fname, old, new in MUTANTS[name]:
        src = (mdir / fname).read_text()
        assert src.count(old) == 1, old
        (mdir / fname).write_text(src.replace(old, new))
    exe = _build(mdir, tmp_path / "mutant")
    failed = 0
    for case in (CASES[0], CASES[3], CASES[5]):
        try:
            _check(exe, tmp_path, *case)
        except AssertionError:
            failed += 1
    assert failed > 0, f"mutant '{name}' passed every check"
