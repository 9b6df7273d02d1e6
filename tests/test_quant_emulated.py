"""The int8 shard's quantiser and rescore kernels (csrc/quant_kernels.cuh) on the CPU, against oracle/quant_oracle.py
bit for bit.  tests/warp_emu/quant_emu_test.cpp runs the kernels on emulated thread blocks.

Quantiser: dims 64, 384, 1000 and 1024, strided input, zero rows, exact .5 ties of x / s, bf16 denormals and rows of
+-amax; the element rule clamp(rint(x / s), -127, 127) is also run on ratios outside the int8 range, where the clamp
is what decides.  Rescore: -1 and out-of-range candidates, rows with tied S2 (which must come out in ascending row
order), k = 1 and k = n_cand.  Three mutants of the header must fail: rounding half away from zero, a clamp at +-128
and ties kept in descending row order."""
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


def _build(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-pthread",
                        "-I", os.path.join(EMU, "stub"), "-I", str(csrc_dir), os.path.join(EMU, "quant_emu_test.cpp"),
                        "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return str(exe)


@pytest.fixture(autouse=True)
def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")


@pytest.fixture(scope="module")
def emulator(tmp_path_factory):
    return _build(CSRC, tmp_path_factory.mktemp("quant_emu") / "quant_emu_test")


def _run(exe, mode, payload: bytes, tmp_path):
    fi, fo = tmp_path / f"{mode}.in", tmp_path / f"{mode}.out"
    fi.write_bytes(payload)
    r = subprocess.run([exe, mode, str(fi), str(fo)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return fo.read_bytes()


def _bf16(x):
    """float32 -> (bf16 bits uint16, the bf16 values as float32), rounded to nearest even."""
    b = torch.from_numpy(np.ascontiguousarray(x, np.float32)).bfloat16()
    return b.view(torch.int16).numpy().view(np.uint16), b.float().numpy()


# ------------------------------------------------------------------------------------------------ quantiser
def _rows(n, dim, rng):
    x = rng.standard_normal((n, dim)).astype(np.float32) * 0.05
    x[0] = 0.0                                               # zero row: s = 0
    if n > 1:                                                # .5 ties: amax = 127 * 2^-7 -> s = 2^-7, x = (m + .5) s
        x[1] = 0.0
        x[1, :: 3] = np.float32(127 / 128)
        x[1, 1:: 3] = (np.arange(len(x[1, 1:: 3])) % 100 + 0.5).astype(np.float32) / 128 * np.where(
            np.arange(len(x[1, 1:: 3])) % 2, 1, -1)
    if n > 2:                                                # bf16 denormals only
        x[2] = rng.integers(-127, 128, dim).astype(np.float32) * np.float32(2.0 ** -133)
    if n > 3:                                                # +-amax in one row, and many equal magnitudes
        x[3] = np.where(rng.random(dim) < 0.5, -1.0, 1.0).astype(np.float32) * np.float32(0.3)
    if n > 4:                                                # a denormal next to a normal amax
        x[4, 0], x[4, 1] = np.float32(1e-39), np.float32(-2.5)
    return x


@pytest.mark.parametrize("dim", [64, 384, 1000, 1024])
def test_quantiser_matches_oracle(emulator, tmp_path, dim):
    rng = np.random.default_rng(dim)
    n = 37
    stride = dim + 24                                        # strided input
    bits, vals = _bf16(_rows(n, dim, rng))
    buf = np.zeros((n, stride), np.uint16)
    buf[:, :dim] = bits
    buf[:, dim:] = 0x7F80                                    # +inf past dim: must never be read
    dim8 = qo.dim8_of(dim)
    out = _run(emulator, "quant", struct.pack("<4i", n, dim, stride, dim8) + buf.tobytes(), tmp_path)
    got_q = np.frombuffer(out[: n * dim8], np.int8).reshape(n, dim8)
    got_s = np.frombuffer(out[n * dim8:], np.float32)
    want_q, want_s = qo.quantize(vals, dim8)
    assert np.array_equal(got_s.view(np.uint32), want_s.view(np.uint32))
    assert np.array_equal(got_q, want_q)
    assert not got_q[0].any() and got_s[0] == 0
    if dim >= 64:   # the tie row really has ties, resolved to even
        r = vals[1, :dim] / want_s[1]
        assert (np.abs(r - np.trunc(r)) == 0.5).sum() > 10


def test_element_rule_matches_oracle_out_of_range(emulator, tmp_path):
    """quant_value on ratios the quantiser itself cannot produce: +-127.5, +-128, 200, ties at .5 of both parities."""
    x = np.array([127.5, -127.5, 128.0, -128.0, 200.0, -1e6, 126.5, -126.5, 0.5, -0.5, 1.5, -2.5, 126.49, 0.0],
                 np.float32)
    s = np.ones_like(x)
    s[-1] = np.float32(3.0)
    m = len(x)
    out = _run(emulator, "values", struct.pack("<i", m) + x.tobytes() + s.tobytes(), tmp_path)
    got = np.frombuffer(out, np.int32)
    assert np.array_equal(got, qo.quant_value(x, s).astype(np.int32))
    assert list(got[:6]) == [127, -127, 127, -127, 127, -127] and list(got[6:12]) == [126, -126, 0, 0, 2, -2]


# ------------------------------------------------------------------------------------------------ rescore
def _rescore_case(rng, n_rows, dim, nq, n_cand, k, row_offset):
    stride = dim + 8
    x = rng.standard_normal((n_rows, dim)).astype(np.float32)
    x[5] = x[3]                                              # duplicate rows: tied S2, ascending row order
    x[9] = x[3]
    bits, vals = _bf16(x)
    qbits, qvals = _bf16(rng.standard_normal((nq, dim)).astype(np.float32))
    qbits[nq - 1] = 0                                        # an all-zero query: every S2 ties at 0
    qvals[nq - 1] = 0
    cand = np.stack([rng.permutation(n_rows)[:n_cand] for _ in range(nq)]).astype(np.int64) + row_offset
    cand[0, :3] = [3 + row_offset, 9 + row_offset, 5 + row_offset]
    cand[:, -1] = -1                                         # -1 and out-of-range ids are no candidates
    if n_cand > 2:
        cand[:, -2] = row_offset + n_rows + 7
        cand[1 % nq, 1] = row_offset - 1
    rows = np.zeros((n_rows, stride), np.uint16)
    rows[:, :dim] = bits
    rows[:, dim:] = 0x7FC0                                   # NaN past dim: must never be read
    payload = struct.pack("<2q5i", n_rows, row_offset, dim, stride, nq, n_cand, k) + rows.tobytes() + \
        qbits.tobytes() + cand.tobytes()
    return payload, vals, qvals, cand


@pytest.mark.parametrize("dim,n_cand,k", [(64, 128, 1), (384, 40, 10), (1000, 128, 128), (1024, 17, 17), (1024, 100, 64)])
def test_rescore_matches_oracle(emulator, tmp_path, dim, n_cand, k):
    rng = np.random.default_rng(dim * 1000 + k)
    n_rows, nq, row_offset = 300, 5, (1 << 33) if dim == 1024 else 0
    payload, vals, qvals, cand = _rescore_case(rng, n_rows, dim, nq, n_cand, k, row_offset)
    out = _run(emulator, "rescore", payload, tmp_path)
    got_ids = np.frombuffer(out[: nq * k * 8], np.int64).reshape(nq, k)
    got_sc = np.frombuffer(out[nq * k * 8:], np.float32).reshape(nq, k)
    want_ids, want_sc = qo.rescore(vals, n_rows, row_offset, qvals, cand, k)
    assert np.array_equal(got_ids, want_ids)
    assert np.array_equal(got_sc.view(np.uint32), want_sc.view(np.uint32))
    if k == n_cand:                                          # the invalid candidates leave -1 / -inf at the tail
        assert (got_ids[:, -1] == -1).all() and np.isneginf(got_sc[:, -1]).all()
    z = got_ids[nq - 1][got_ids[nq - 1] >= 0]                # the zero query: all tied, ascending rows
    assert (np.diff(z) > 0).all()


def test_rescore_ties_in_ascending_row_order(emulator, tmp_path):
    rng = np.random.default_rng(7)
    payload, vals, qvals, cand = _rescore_case(rng, 64, 128, 2, 8, 3, 0)
    out = _run(emulator, "rescore", payload, tmp_path)
    ids = np.frombuffer(out[: 2 * 3 * 8], np.int64).reshape(2, 3)
    want, _ = qo.rescore(vals, 64, 0, qvals, cand, 3)
    assert np.array_equal(ids, want)
    s2 = qo.s2_scores(vals[[3, 5, 9]], qvals[0])
    assert s2[0] == s2[1] == s2[2]


# ------------------------------------------------------------------------------------------------ mutants
MUTANTS = {
    "round half away from zero": ("__float2int_rn(__fdiv_rn(x, s))", "int(roundf(__fdiv_rn(x, s)))"),
    "clamp at +-128": ("kQuantClamp = 127", "kQuantClamp = 128"),
    "ties in descending row order": ("key = make_key(partial, uint32_t(local));",
                                     "key = make_key(partial, 0x7FFFFFFFu - uint32_t(local));"),
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutant_fails(tmp_path, name):
    old, new = MUTANTS[name]
    mdir = tmp_path / "csrc"
    shutil.copytree(CSRC, mdir)
    src = (mdir / "quant_kernels.cuh").read_text()
    assert src.count(old) == 1
    (mdir / "quant_kernels.cuh").write_text(src.replace(old, new))
    if name.startswith("ties"):   # the ids come back through key_id, so undo the mutation's id map on the way out
        src = (mdir / "quant_kernels.cuh").read_text()
        src = src.replace("int64_t(key_id(v[j]))", "int64_t(0x7FFFFFFFu - key_id(v[j]))")
        (mdir / "quant_kernels.cuh").write_text(src)
    exe = _build(mdir, tmp_path / "mutant")
    tests = [lambda: test_element_rule_matches_oracle_out_of_range(exe, tmp_path)]
    tests += [lambda d=d: test_quantiser_matches_oracle(exe, tmp_path, d) for d in (64, 1000)]
    tests += [lambda: test_rescore_ties_in_ascending_row_order(exe, tmp_path),
              lambda: test_rescore_matches_oracle(exe, tmp_path, 384, 40, 10)]
    failed = 0
    for t in tests:
        try:
            t()
        except AssertionError:
            failed += 1
    assert failed > 0, f"mutant '{name}' passed every check"
