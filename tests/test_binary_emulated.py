"""The one-bit shard's binarize kernel (csrc/quant_kernels.cuh) and its bit -> wgmma A-fragment map (csrc/binary.cuh)
on the CPU.  tests/warp_emu/binary_emu_test.cpp runs the kernel on emulated thread blocks; its codes and alpha must
equal tests/binary_oracle.py bit for bit at dims 64, 320, 1000 and 1024 (64 and 320 are not multiples of 128, so
padding bits appear), with zero rows, -0, bf16 denormals and rows of one magnitude.  The fragment of every lane must
equal a model of the PTX ISA's register layout for an s8 A operand at k32.  Three mutants must fail: the bit order in a
byte, the order of alpha's sum, and a swap of the fragment's column halves."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest
import torch

import binary_oracle as bo

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EMU = os.path.join(ROOT, "tests", "warp_emu")
CSRC = os.path.join(ROOT, "comorag_b200", "csrc")


def _build(csrc_dir, exe):
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas", "-pthread",
                        "-I", os.path.join(EMU, "stub"), "-I", str(csrc_dir), os.path.join(EMU, "binary_emu_test.cpp"),
                        "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return str(exe)


@pytest.fixture(autouse=True)
def _need_gxx():
    if shutil.which("g++") is None:
        pytest.skip("g++ not installed")


@pytest.fixture(scope="module")
def emulator(tmp_path_factory):
    return _build(CSRC, tmp_path_factory.mktemp("binary_emu") / "binary_emu_test")


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


# ------------------------------------------------------------------------------------------------ binarize
def _rows(n, dim, rng):
    x = rng.standard_normal((n, dim)).astype(np.float32) * np.float32(0.05)
    x[0] = 0.0                                               # zero row: alpha = 0, every bit clear
    x[1] = -0.0                                              # -0 is not positive
    x[2] = rng.integers(-127, 128, dim).astype(np.float32) * np.float32(2.0 ** -133)   # bf16 denormals only
    x[3] = np.where(rng.random(dim) < 0.5, -1.0, 1.0).astype(np.float32) * np.float32(0.375)   # one magnitude
    x[4, ::5] = 0.0                                          # zeros among the values
    x[5] *= np.float32(1e4)                                  # a wide range of magnitudes
    x[5, ::7] *= np.float32(1e-6)
    return x


def _binarize(exe, tmp_path, n, dim, stride, rng):
    bits, vals = _bf16(_rows(n, dim, rng))
    buf = np.zeros((n, stride), np.uint16)
    buf[:, :dim] = bits
    buf[:, dim:] = 0x7F80                                    # +inf past dim: must never be read
    buf[1, :dim] = 0x8000                                    # the -0 row as bits
    vals[1] = -0.0
    dim8 = bo.dim8_of(dim)
    out = _run(exe, "binarize", struct.pack("<4i", n, dim, stride, dim8) + buf.tobytes(), tmp_path)
    got_c = np.frombuffer(out[: n * dim8 // 8], np.uint8).reshape(n, dim8 // 8)
    got_a = np.frombuffer(out[n * dim8 // 8:], np.float32)
    return got_c, got_a, vals, dim8


@pytest.mark.parametrize("dim", [64, 320, 1000, 1024])
def test_binarize_matches_oracle(emulator, tmp_path, dim):
    rng = np.random.default_rng(dim)
    n = 37
    got_c, got_a, vals, dim8 = _binarize(emulator, tmp_path, n, dim, dim + 24, rng)
    want_c, want_a = bo.binarize(vals, dim8)
    assert np.array_equal(got_a.view(np.uint32), want_a.view(np.uint32))
    assert np.array_equal(got_c, want_c)
    assert not got_c[:2].any() and got_a[0] == 0 and got_a[1] == 0
    assert got_a[3] == np.float32(0.375)                     # one magnitude: alpha is that magnitude exactly
    signs = bo.signs(got_c)
    assert (signs[:, dim:] == -1).all()                      # padding columns read as -1


def test_binarize_bit_layout(emulator, tmp_path):
    """Column 8 b + j is bit j of byte b: a single positive column per row lands where the layout says."""
    dim = 320
    cols = [0, 1, 7, 8, 31, 32, 100, 255, 256, 319]
    x = np.full((len(cols), dim), -1.0, np.float32)
    for r, c in enumerate(cols):
        x[r, c] = 1.0
    bits, _ = _bf16(x)
    dim8 = bo.dim8_of(dim)
    out = _run(emulator, "binarize", struct.pack("<4i", len(cols), dim, dim, dim8) + bits.tobytes(), tmp_path)
    codes = np.frombuffer(out[: len(cols) * dim8 // 8], np.uint8).reshape(len(cols), dim8 // 8)
    for r, c in enumerate(cols):
        want = np.zeros(dim8 // 8, np.uint8)
        want[c // 8] = 1 << (c % 8)
        assert np.array_equal(codes[r], want), (c, codes[r])


# ------------------------------------------------------------------------------------------------ A fragment
def fragment_model(words: np.ndarray) -> np.ndarray:
    """The PTX ISA layout of an s8 A fragment at k32, per warp: lane (g, t) holds in register r, byte e, the element of
    row g + 8 (r % 2), column 4 t + e + 16 (r // 2).  words [16] (row r's 32 columns, bit j = column j) -> [32, 4]."""
    a = np.where((words[:, None] >> np.arange(32, dtype=np.uint32)[None, :]) & 1, 1, -1).astype(np.int8)   # [16, 32]
    out = np.zeros((32, 4), np.uint32)
    for lane in range(32):
        g, t = lane // 4, lane % 4
        for r in range(4):
            b = [a[g + 8 * (r % 2), 4 * t + e + 16 * (r // 2)] for e in range(4)]
            out[lane, r] = np.frombuffer(np.array(b, np.int8).tobytes(), np.uint32)[0]
    return out


def _fragment_words(rng):
    w = rng.integers(0, 1 << 32, (40, 16), dtype=np.uint64).astype(np.uint32)
    w[0] = 0
    w[1] = 0xFFFFFFFF
    w[2] = np.array([1 << i for i in range(16)], np.uint32)          # one column per row
    w[3] = np.array([1 << (16 + i) for i in range(16)], np.uint32)
    w[4] = 0x0000FFFF
    return w


def test_fragment_matches_ptx_layout(emulator, tmp_path):
    w = _fragment_words(np.random.default_rng(5))
    out = _run(emulator, "fragment", struct.pack("<i", len(w)) + w.tobytes(), tmp_path)
    got = np.frombuffer(out, np.uint32).reshape(len(w), 32, 4)
    for i in range(len(w)):
        assert np.array_equal(got[i], fragment_model(w[i])), i


def test_fragment_dot_is_the_signed_dot():
    """The int8 bytes of the fragment, multiplied by a query block laid out as the rows' columns, give sum q_i b_i."""
    rng = np.random.default_rng(9)
    w = rng.integers(0, 1 << 32, 16, dtype=np.uint64).astype(np.uint32)
    q = rng.integers(-127, 128, 32).astype(np.int64)
    frag = fragment_model(w)
    acc = np.zeros(16, np.int64)
    for lane in range(32):
        g, t = lane // 4, lane % 4
        for r in range(4):
            b = np.frombuffer(np.uint32(frag[lane, r]).tobytes(), np.int8).astype(np.int64)
            cols = 4 * t + 16 * (r // 2) + np.arange(4)
            acc[g + 8 * (r % 2)] += (b * q[cols]).sum()
    signs = np.where((w[:, None] >> np.arange(32, dtype=np.uint32)[None, :]) & 1, 1, -1)
    assert np.array_equal(acc, signs @ q)


# ------------------------------------------------------------------------------------------------ mutants
MUTANTS = {
    "bit order in a byte": ("quant_kernels.cuh", [("const int c = 32 * w + lane;", "const int c = 32 * w + (lane ^ 7);")]),
    "alpha summation order": ("quant_kernels.cuh", [("for (int o = 16; o > 0; o >>= 1) abs_sum",
                                                      "for (int o = 1; o < 32; o <<= 1) abs_sum")]),
    "fragment column swap": ("binary.cuh", [("a[0] = b1_widen4((lo >> (4 * t)) & 0xFu);", "a[0] = @LO16;"),
                                            ("a[2] = b1_widen4((lo >> (16 + 4 * t)) & 0xFu);",
                                             "a[2] = b1_widen4((lo >> (4 * t)) & 0xFu);"),
                                            ("@LO16", "b1_widen4((lo >> (16 + 4 * t)) & 0xFu)")]),
}


@pytest.mark.parametrize("name", list(MUTANTS))
def test_mutant_fails(tmp_path, name):
    header, edits = MUTANTS[name]
    mdir = tmp_path / "csrc"
    shutil.copytree(CSRC, mdir)
    src = (mdir / header).read_text()
    for old, new in edits:
        assert src.count(old) == 1, old
        src = src.replace(old, new)
    (mdir / header).write_text(src)
    exe = _build(mdir, tmp_path / "mutant")
    tests = [lambda d=d: test_binarize_matches_oracle(exe, tmp_path, d) for d in (64, 320, 1000)]
    tests += [lambda: test_binarize_bit_layout(exe, tmp_path), lambda: test_fragment_matches_ptx_layout(exe, tmp_path)]
    failed = 0
    for t in tests:
        try:
            t()
        except AssertionError:
            failed += 1
    assert failed > 0, f"mutant '{name}' passed every check"
