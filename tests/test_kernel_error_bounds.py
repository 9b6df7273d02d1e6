"""Error bounds for the tensor-core kernels that the warp emulator cannot run: the wgmma GEMM (crag_gemm_bf16), the
wgmma attention for head dim 64 (crag_attention_varlen_tc) and the mma.sync attention for head dims 32 and 64
(crag_attention_varlen).

Each kernel is compared with a float64 reference of the same operation on the same bf16 inputs and fp32 biases, under
a bound derived from the kernel's arithmetic rather than a tolerance chosen by hand:

GEMM, BIAS and RESIDUAL epilogues:   |out - ref| <= 2^-7 |ref| + 2^-16 S,   S = sum_k |a_ik w_jk| + |bias_j| (+ |res_ij|)
    2^-7 |ref| is one bf16 step relative: the output is rounded to bf16 once (at most half a step).
    2^-16 S covers fp32 accumulation, with 8x headroom over the 2e-6 (about 2^-19 S) that
    test_search_gpu.py::test_score_all_pass_equals_the_dot_products measures for the scan's wgmma on unit rows.
GEMM, GELU epilogue:   2^-7 |ref| + 1.13 * 2^-16 S + 1e-6
    GELU's slope is at most 1.129, so an accumulation error d moves the output by at most 1.13 d.  1e-6 covers the
    Abramowitz-Stegun erf of gelu_erf (gemm.cu), which emulated in fp32 is within 4.6e-7 of the exact GELU on
    [-10, 10] (test_gelu_erf_formula_error).  Below x = -4 that is a large RELATIVE error, up to the whole value
    (|gelu(x)| < 1.3e-4 there, around 1e-8 at the far end): the bound accepts this on purpose, because next to the
    O(1) activations it is summed with it is far below what bf16 resolves.
Attention:   |ctx - ref| <= 2^-7 (|ref| + sum_j p_j |v_j|) + 1e-6,   p = the float64 softmax
    P is rounded to bf16 before P.V (each p_j off by at most 2^-8 relative) while l is summed from the unrounded p:
    that is the sum_j p_j |v_j| term; the bf16 output is the |ref| term; 1e-6 absorbs fp32 noise where ctx ~ 0.

The CPU tests (not gpu-marked) check that the bounds are neither vacuous nor too tight: a torch model of each kernel's
arithmetic stays well under its bound, and the same model with one specific bug exceeds it many times over.

Every GPU test records its worst err/bound as the pytest property `worst_err_over_bound` (see --junitxml).
"""
import math

import numpy as np
import pytest
import torch

GEMM_EPI_BIAS, GEMM_EPI_BIAS_GELU, GEMM_EPI_BIAS_RESIDUAL = 0, 1, 2
LOG2E = 1.4426950408889634
SENTINEL = 0x7FA5                     # a bf16 NaN payload no kernel produces: the canary of every output buffer


# ------------------------------------------------------------------------------------------------ references, bounds
def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gemm_reference(a, w, bias, epi, res=None):
    """float64 epi(a . w^T + bias) and the magnitude sum S of the bound, from the kernel's bf16 / fp32 inputs."""
    a64, w64, b64 = a.double(), w.double(), bias.double()
    ref = a64 @ w64.T + b64
    mag = a64.abs() @ w64.abs().T + b64.abs()
    if epi == GEMM_EPI_BIAS_GELU:
        ref = gelu64(ref)
    elif epi == GEMM_EPI_BIAS_RESIDUAL:
        ref = ref + res.double()
        mag = mag + res.double().abs()
    return ref, mag


def gemm_bound(ref, mag, epi):
    if epi == GEMM_EPI_BIAS_GELU:
        return 2.0 ** -7 * ref.abs() + 1.13 * 2.0 ** -16 * mag + 1e-6
    return 2.0 ** -7 * ref.abs() + 2.0 ** -16 * mag


def attention_reference(qkv, lens, H, heads, budget=1 << 25):
    """float64 softmax(q k^T / sqrt(dh)) v per (sequence, head) of the packed [T, 3H] activation, and the bound.
    Sequences are padded in groups of at most `budget` score elements."""
    dh, T = H // heads, qkv.shape[0]
    x = qkv.double()
    ref = torch.empty(T, H, dtype=torch.float64, device=qkv.device)
    bnd = torch.empty_like(ref)
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    i = 0
    while i < len(lens):
        j, lmax = i + 1, lens[i]
        while j < len(lens) and (j - i + 1) * heads * max(lmax, lens[j]) ** 2 <= budget:
            lmax = max(lmax, lens[j])
            j += 1
        b = j - i
        ar = torch.arange(lmax, device=qkv.device)
        st = torch.as_tensor(starts[i:j], device=qkv.device)
        ln = torch.as_tensor(np.asarray(lens[i:j], dtype=np.int64), device=qkv.device)
        valid = ar[None, :] < ln[:, None]                                               # [b, lmax]
        rows = (st[:, None] + ar[None, :]).clamp(max=T - 1)
        xp = x[rows]                                                                    # [b, lmax, 3H]
        q, k, v = (xp[..., c * H:(c + 1) * H].reshape(b, lmax, heads, dh).transpose(1, 2) for c in range(3))
        s = (q @ k.transpose(-1, -2)) / math.sqrt(dh)
        s = s.masked_fill(~valid[:, None, None, :], float("-inf"))
        p = torch.softmax(s, dim=-1)
        o = (p @ v).transpose(1, 2).reshape(b, lmax, H)
        ov = (p @ v.abs()).transpose(1, 2).reshape(b, lmax, H)
        ref[rows[valid]] = o[valid]
        bnd[rows[valid]] = 2.0 ** -7 * (o[valid].abs() + ov[valid]) + 1e-6
        i = j
    return ref, bnd


def worst_ratio(out, ref, bound):
    r = (out.double() - ref).abs() / bound
    return float(torch.nan_to_num(r, nan=float("inf")).max())


# ------------------------------------------------------------------------------------- CPU models of the kernels
def gelu_erf_fp32(x):
    """gelu_erf (gemm.cu) in fp32: Abramowitz-Stegun 7.1.26 erf, rcp / ex2 taken as exact fp32 operations."""
    x = x.float()
    z = x * 0.70710678118654752
    az = z.abs()
    t = 1.0 / (0.3275911 * az + 1.0)
    p = ((((1.061405429 * t - 1.453152027) * t + 1.421413741) * t - 0.284496736) * t + 0.254829592) * t
    e = torch.exp2(az * az * -1.4426950408889634)
    erf_abs = 1.0 - p * e
    half_x = 0.5 * x
    return half_x * torch.copysign(erf_abs, z) + half_x


def gemm_model(a, w, bias, epi, res=None, bug=None):
    """The kernel's arithmetic: fp32 accumulation over 64-wide k-blocks, fp32 epilogue, one bf16 rounding.
    bug="bf16_acc": the accumulator is rounded to bf16 after every k-block.
    bug="drop_tail": a partial last k-block after a full one is skipped."""
    K = a.shape[1]
    af, wf = a.float(), w.float()
    if bug is None:
        acc = af @ wf.T
    elif bug == "bf16_acc":
        acc = torch.zeros(a.shape[0], w.shape[0])
        for k0 in range(0, K, 64):
            acc = (acc + af[:, k0:k0 + 64] @ wf[:, k0:k0 + 64].T).bfloat16().float()
    elif bug == "drop_tail":
        kk = K // 64 * 64 if K > 64 else K
        acc = af[:, :kk] @ wf[:, :kk].T
    x = acc + bias.float()
    if epi == GEMM_EPI_BIAS_GELU:
        x = gelu_erf_fp32(x)
    elif epi == GEMM_EPI_BIAS_RESIDUAL:
        x = x + res.float()
    return x.bfloat16()


def attention_model(q, k, v):
    """The kernels' arithmetic for one (sequence, head): fp32 scores, online softmax over 64-key blocks in the base-2
    domain, P rounded to bf16 for P.V, l summed from the unrounded p, bf16 output.  Every key given is attended."""
    q, k, v = q.float(), k.float(), v.float()
    s = (q @ k.T) * (LOG2E / math.sqrt(q.shape[1]))
    m = torch.full((q.shape[0], 1), float("-inf"))
    l = torch.zeros(q.shape[0], 1)
    o = torch.zeros(q.shape[0], v.shape[1])
    for j in range(0, k.shape[0], 64):
        sj = s[:, j:j + 64]
        m_new = torch.maximum(m, sj.max(dim=1, keepdim=True).values)
        alpha = torch.exp2(m - m_new)
        p = torch.exp2(sj - m_new)
        l = l * alpha + p.sum(dim=1, keepdim=True)
        o = o * alpha + p.bfloat16().float() @ v[j:j + 64]
        m = m_new
    return (o / l).bfloat16()


def gemm_inputs(M, N, K, kind, seed, device="cpu"):
    """bf16 A [M, K], bf16 W [N, K], fp32 bias [N], bf16 residual [M, N].
    random: O(1) rows and outputs.  scaled: row r of A and of the residual scaled by 2^(r % 17 - 8) and a small bias,
    so the bound is tested relative to each row's own magnitude.  zero: A = 0, so out = epi(bias (+ residual))."""
    g = torch.Generator(device=device).manual_seed(seed)
    a = torch.randn(M, K, generator=g, device=device)
    w = torch.randn(N, K, generator=g, device=device) / math.sqrt(K)
    bias = torch.randn(N, generator=g, device=device)
    res = torch.randn(M, N, generator=g, device=device)
    if kind == "scaled":
        s = 2.0 ** ((torch.arange(M, device=device) % 17) - 8).float()
        a, res, bias = a * s[:, None], res * s[:, None], bias * 2.0 ** -12
    elif kind == "zero":
        a = torch.zeros_like(a)
    return a.bfloat16(), w.bfloat16(), bias, res.bfloat16()


# ------------------------------------------------------------------------------------ CPU: the bounds are calibrated
def test_gelu_erf_formula_error():
    """The 1e-6 term of the GELU bound: the kernel's erf formula against the exact GELU, densely on [-10, 10]."""
    x = torch.linspace(-10, 10, 200001, dtype=torch.float32)
    err = (gelu_erf_fp32(x).double() - gelu64(x.double())).abs()
    assert float(err.max()) < 6e-7, float(err.max())
    assert float(gelu_erf_fp32(torch.zeros(1))[0]) == 0.0


@pytest.mark.parametrize("M,N,K", [(300, 384, 384), (129, 136, 1000), (64, 264, 4096), (65, 120, 200)])
@pytest.mark.parametrize("kind", ["random", "scaled"])
def test_gemm_bound_is_calibrated(M, N, K, kind):
    """fp32 accumulation + one bf16 rounding stays well under the bound; rounding the accumulator to bf16 after every
    k-block, or skipping the partial last k-block, exceeds it many times over."""
    a, w, bias, res = gemm_inputs(M, N, K, kind, seed=M * 7 + N + K)
    for epi in (GEMM_EPI_BIAS, GEMM_EPI_BIAS_GELU, GEMM_EPI_BIAS_RESIDUAL):
        ref, mag = gemm_reference(a, w, bias, epi, res)
        bnd = gemm_bound(ref, mag, epi)
        good = worst_ratio(gemm_model(a, w, bias, epi, res), ref, bnd)
        acc = worst_ratio(gemm_model(a, w, bias, epi, res, bug="bf16_acc"), ref, bnd)
        assert good < 0.75, (epi, good)
        assert acc > 8, (epi, acc)
        if K % 64:
            tail = worst_ratio(gemm_model(a, w, bias, epi, res, bug="drop_tail"), ref, bnd)
            assert tail > 8, (epi, tail)


@pytest.mark.parametrize("L", [65, 130, 200, 512])
@pytest.mark.parametrize("dh", [32, 64])
def test_attention_bound_is_calibrated(L, dh):
    """The online-softmax model stays well under the bound; admitting one neighbour key, or masking the last key,
    exceeds it several times over.  On random inputs the weights are nearly uniform, so one key of 512 moves ctx by
    only ~1/512 of V's spread: 3.7x at L = 512, dh = 32 is the smallest margin here.  The structured GPU tests below
    make a mis-masked key dominate instead."""
    g = torch.Generator().manual_seed(L * 3 + dh)
    worst_good, worst_leak, worst_drop = 0.0, float("inf"), float("inf")
    for _ in range(3):
        x = torch.randn(L + 1, 3 * dh, generator=g).bfloat16()      # row L belongs to the next sequence
        q, k, v = x[:L, :dh], x[:, dh:2 * dh], x[:, 2 * dh:]
        ref, bnd = attention_reference(x[:L], [L], dh, 1)
        worst_good = max(worst_good, worst_ratio(attention_model(q, k[:L], v[:L]), ref, bnd))
        worst_leak = min(worst_leak, worst_ratio(attention_model(q, k, v), ref, bnd))
        worst_drop = min(worst_drop, worst_ratio(attention_model(q, k[:L - 1], v[:L - 1]), ref, bnd))
    assert worst_good < 0.5, worst_good
    assert worst_leak > 3, worst_leak
    assert worst_drop > 3, worst_drop


def test_attention_reference_masks_and_groups():
    """The grouped, padded reference equals a per-sequence softmax, and its bound is what the docstring states."""
    g = torch.Generator().manual_seed(5)
    lens, H, heads = [3, 70, 1, 20], 64, 2
    qkv = torch.randn(sum(lens), 3 * H, generator=g).bfloat16()
    ref, bnd = attention_reference(qkv, lens, H, heads, budget=2 * 70 * 70)      # forces several groups
    s0 = 0
    for L in lens:
        x = qkv[s0:s0 + L].double()
        q, k, v = (x[:, c * H:(c + 1) * H].view(L, heads, 32).transpose(0, 1) for c in range(3))
        p = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(32), -1)
        want = (p @ v).transpose(0, 1).reshape(L, H)
        torch.testing.assert_close(ref[s0:s0 + L], want, rtol=1e-12, atol=1e-12)
        wb = 2.0 ** -7 * (want.abs() + (p @ v.abs()).transpose(0, 1).reshape(L, H)) + 1e-6
        torch.testing.assert_close(bnd[s0:s0 + L], wb, rtol=1e-12, atol=1e-12)
        s0 += L


# -------------------------------------------------------------------------------------------------- GPU plumbing
@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available()
    from comorag_b200 import _native
    return _native.load()


def _check(rc, what):
    from comorag_b200 import _native
    _native.check(rc, what)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def run_gemm(lib, a, w, bias, epi, res=None, pads=(8, 24, 16, 40)):
    """crag_gemm_bf16 with every operand a window of a wider buffer: A and W with NaN columns past K (lda, ldw > K),
    the residual with NaN columns past N and ldr != ldo, and out at row 3, column 8 of a buffer of sentinel bits
    (ldo > N) with sentinel rows above and below.  Asserts every sentinel is intact; returns the [M, N] window."""
    M, K = a.shape
    N = w.shape[0]
    dev = a.device
    lda, ldw, ldr, ldo = K + pads[0], K + pads[1], N + pads[3], N + 8 + pads[2]
    top, bottom, left = 3, 5, 8
    nan = float("nan")
    abuf = torch.full((M, lda), nan, dtype=torch.bfloat16, device=dev)
    abuf[:, :K] = a
    wbuf = torch.full((N, ldw), nan, dtype=torch.bfloat16, device=dev)
    wbuf[:, :K] = w
    rbuf = None
    if epi == GEMM_EPI_BIAS_RESIDUAL:
        rbuf = torch.full((M, ldr), nan, dtype=torch.bfloat16, device=dev)
        rbuf[:, :N] = res
    obuf = torch.full((top + M + bottom, ldo), SENTINEL, dtype=torch.int16, device=dev)
    rc = lib.crag_gemm_bf16(abuf.data_ptr(), lda, wbuf.data_ptr(), ldw, bias.data_ptr(),
                            0 if rbuf is None else rbuf.data_ptr(), ldr, obuf[top, left:].data_ptr(), ldo, M, N, K, epi,
                            _stream())
    _check(rc, "crag_gemm_bf16")
    torch.cuda.synchronize()
    canary = obuf.clone()
    canary[top:top + M, left:left + N] = SENTINEL
    assert bool((canary == SENTINEL).all()), "crag_gemm_bf16 wrote outside its [M, N] output window"
    return obuf[top:top + M, left:left + N].view(torch.bfloat16)


# --------------------------------------------------------------------------------------------------------- GEMM
GEMM_M = [1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1000, 4097]
GEMM_N = [8, 16, 120, 136, 248, 264, 1000, 1032, 3072]
GEMM_K = [8, 16, 56, 72, 120, 200, 1000, 1032, 4096]
# every (M, N) pair once, K rotated so that each K meets every M and every N class, the epilogue rotated as well
GEMM_COVER = [(m, n, GEMM_K[(3 * i + 7 * j) % 9], (i + j) % 3) for i, m in enumerate(GEMM_M) for j, n in enumerate(GEMM_N)]
GEMM_CARRIED = [(128, 128, 64, 0), (300, 384, 384, 0), (1000, 1152, 384, 0), (777, 1536, 384, 1), (512, 384, 1536, 2),
                (2048, 3072, 1024, 0), (2048, 1024, 4096, 2), (2048, 4096, 1024, 1), (1, 768, 768, 0), (129, 8, 8, 0)]
# the encoder's projections for bge-small / base / large (H, I): QKV, attention output (+residual), FFN up (+GELU),
# FFN down (+residual), on a 777-token packed batch
GEMM_ENCODER = [(777, n, k, e) for H, I in ((384, 1536), (768, 3072), (1024, 4096))
                for n, k, e in ((3 * H, H, 0), (H, H, 2), (I, H, 1), (H, I, 2))]


@pytest.mark.gpu
@pytest.mark.parametrize("M,N,K,epi", GEMM_COVER + GEMM_CARRIED + GEMM_ENCODER)
def test_gemm_within_bound(lib, record_property, M, N, K, epi):
    dev = torch.device("cuda:0")
    worst = 0.0
    for kind in ("random", "scaled", "zero"):
        a, w, bias, res = gemm_inputs(M, N, K, kind, seed=M * 131 + N * 7 + K + epi, device=dev)
        pads = ((8, 24, 16, 40), (72, 8, 64, 8), (16, 136, 8, 24))[(M + N + K) % 3]
        out = run_gemm(lib, a, w, bias, epi, res, pads)
        ref, mag = gemm_reference(a, w, bias, epi, res)
        r = worst_ratio(out, ref, gemm_bound(ref, mag, epi))
        assert r <= 1.0, f"{kind}: worst err/bound {r:.3f}"
        worst = max(worst, r)
        if kind == "zero" and epi == GEMM_EPI_BIAS:          # 0 + bias in fp32, one rounding: exact
            assert torch.equal(out, bias.bfloat16()[None].expand(M, N))
        if kind == "zero" and epi == GEMM_EPI_BIAS_RESIDUAL:
            assert torch.equal(out, (bias[None] + res.float()).bfloat16())
    record_property("worst_err_over_bound", worst)


@pytest.mark.gpu
def test_gemm_gelu_curve(lib, record_property):
    """A = 0 and a bias sweeping [-10, 10] densely: out = gelu(bias) against the float64 exact-erf GELU."""
    dev = torch.device("cuda:0")
    N = 40960
    bias = torch.linspace(-10, 10, N, device=dev)
    bias[N // 2] = 0.0
    a = torch.zeros(2, 64, dtype=torch.bfloat16, device=dev)
    w = torch.randn(N, 64, generator=torch.Generator(device=dev).manual_seed(1), device=dev).bfloat16()
    out = run_gemm(lib, a, w, bias, GEMM_EPI_BIAS_GELU)
    ref, mag = gemm_reference(a, w, bias, GEMM_EPI_BIAS_GELU)
    r = worst_ratio(out, ref, gemm_bound(ref, mag, GEMM_EPI_BIAS_GELU))
    assert r <= 1.0, r
    assert bool((out[:, N // 2] == 0).all())
    record_property("worst_err_over_bound", r)


@pytest.mark.gpu
@pytest.mark.parametrize("epi", [0, 1, 2])
def test_gemm_is_deterministic_and_row_position_invariant(lib, epi):
    """Two identical calls agree bit for bit, and a row's output does not depend on where in the batch (which tile,
    which warpgroup, which lane) it is computed: the request coalescer relies on this when it moves queries within a
    batch (test_encoder_gpu.py::test_sixteen_threads_share_the_engine)."""
    dev = torch.device("cuda:0")
    M, N, K = 4097, 1032, 1000
    a, w, bias, res = gemm_inputs(M, N, K, "random", seed=epi + 17, device=dev)
    first = run_gemm(lib, a, w, bias, epi, res).clone()
    assert torch.equal(first.view(torch.int16), run_gemm(lib, a, w, bias, epi, res).view(torch.int16))
    row, row_res = a[5:6].clone(), res[5:6].clone()
    alone = run_gemm(lib, row, w, bias, epi, row_res).clone()
    for pos in (0, 63, 64, 127, 128, 4096):
        a2, r2 = a.clone(), res.clone()
        a2[pos], r2[pos] = row[0], row_res[0]
        out = run_gemm(lib, a2, w, bias, epi, r2)
        assert torch.equal(out[pos].view(torch.int16), alone[0].view(torch.int16)), f"row at position {pos} differs"


# ---------------------------------------------------------------------------------------------------- attention
ATT_KERNELS = [("tc", 64), ("mma", 32), ("mma", 64)]
ATT_LENGTHS = [1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 511, 512]
ATT_PACK = [5] + ATT_LENGTHS          # the 5-token head puts every sequence of interest at an offset % 64 != 0


def run_attention(lib, qkv, lens, H, heads, kernel, max_len=None):
    """One varlen attention call into a ctx buffer of NaN with sentinel rows past T, which must stay intact."""
    T = sum(lens)
    dev = qkv.device
    max_len = max(lens) if max_len is None else max_len
    cu = torch.tensor([0] + np.cumsum(lens).tolist(), dtype=torch.int32, device=dev)
    buf = torch.full((T + 64, H), SENTINEL, dtype=torch.int16, device=dev)
    buf[:T] = torch.full((T, H), float("nan"), dtype=torch.bfloat16, device=dev).view(torch.int16)
    ctx = buf.view(torch.bfloat16)
    if kernel == "tc":
        rc = lib.crag_attention_varlen_tc(qkv.data_ptr(), cu.data_ptr(), len(lens), T, max_len, H, heads, ctx.data_ptr(), _stream())
    else:
        rc = lib.crag_attention_varlen(qkv.data_ptr(), cu.data_ptr(), len(lens), max_len, H, heads, ctx.data_ptr(), _stream())
    _check(rc, f"attention ({kernel})")
    torch.cuda.synchronize()
    assert bool((buf[T:] == SENTINEL).all()), "attention wrote past the last token"
    return ctx[:T]


def check_attention(lib, qkv, lens, H, heads, kernel, max_len=None):
    out = run_attention(lib, qkv, lens, H, heads, kernel, max_len)
    ref, bnd = attention_reference(qkv, lens, H, heads)
    r = worst_ratio(out, ref, bnd)
    assert r <= 1.0, f"worst err/bound {r:.3f}"
    return out, ref, r


def pack_heads(qs, ks, vs):
    """Per-sequence [heads, L, dh] q, k, v (fp32) -> packed bf16 qkv [T, 3H]."""
    rows = []
    for q, k, v in zip(qs, ks, vs):
        heads, L, dh = q.shape
        rows.append(torch.cat([t.transpose(0, 1).reshape(L, heads * dh) for t in (q, k, v)], dim=1))
    return torch.cat(rows).bfloat16()


@pytest.mark.gpu
@pytest.mark.parametrize("heads", [1, 2, 12, 16])
@pytest.mark.parametrize("kernel,dh", ATT_KERNELS)
def test_attention_random_within_bound(lib, record_property, kernel, dh, heads):
    starts = np.cumsum(ATT_PACK)[:-1]
    assert (starts % 64 != 0).all()
    dev = torch.device("cuda:0")
    H = heads * dh
    g = torch.Generator(device=dev).manual_seed(heads * 100 + dh)
    qkv = torch.randn(sum(ATT_PACK), 3 * H, generator=g, device=dev).bfloat16()
    _, _, r = check_attention(lib, qkv, ATT_PACK, H, heads, kernel)
    record_property("worst_err_over_bound", r)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,dh", ATT_KERNELS)
def test_attention_query_wave(lib, record_property, kernel, dh):
    """ComoRAG's query encode: 2,000 sequences of 3-40 tokens in one call (grid.z = 2,000), 12 heads."""
    dev = torch.device("cuda:0")
    lens = torch.randint(3, 41, (2000,), generator=torch.Generator().manual_seed(dh)).tolist()
    H = 12 * dh
    qkv = torch.randn(sum(lens), 3 * H, generator=torch.Generator(device=dev).manual_seed(3), device=dev).bfloat16()
    _, _, r = check_attention(lib, qkv, lens, H, 12, kernel)
    record_property("worst_err_over_bound", r)


@pytest.mark.gpu
@pytest.mark.parametrize("H,heads,lens,kernel", [(128, 4, [5, 64, 65, 1, 130], "mma"), (1024, 16, [512, 33, 200], "mma"),
                                                 (384, 12, [77, 512], "mma"), (768, 12, [128] * 3, "mma"),
                                                 (128, 2, [5, 64, 65, 1, 130, 128, 129, 300, 512], "tc"),
                                                 (1024, 16, [512, 33, 200, 511], "tc"), (768, 12, [128, 63, 64], "tc")])
def test_attention_encoder_shapes(lib, record_property, H, heads, lens, kernel):
    dev = torch.device("cuda:0")
    qkv = torch.randn(sum(lens), 3 * H, generator=torch.Generator(device=dev).manual_seed(H), device=dev).bfloat16()
    _, _, r = check_attention(lib, qkv, lens, H, heads, kernel)
    record_property("worst_err_over_bound", r)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,dh", ATT_KERNELS)
def test_attention_masks_neighbours_and_padding(lib, record_property, kernel, dh):
    """Leakage sentinels.  Even sequences have queries along +u and keys along -u, odd ones the reverse, u a unit
    vector: every real score is about -20 nats, every key of a neighbouring sequence scores about +20 against these
    queries, and a zero key (a padding row) scores 0.  V is about +1 in even sequences and -8 in odd ones.  So one
    admitted neighbour key pulls ctx to the neighbour's V, and one admitted zero row pulls it to 0.  Every length
    here leaves a partial last key block; the last sequence's runs past the end of the activation, where the wgmma
    kernel's TMA loads read zero rows."""
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(dh)
    lens, heads = [37, 1, 65, 129, 200, 257, 511, 63], 2
    amp = math.sqrt(20.0 * math.sqrt(dh))                  # |q| |k| / sqrt(dh) = 20
    u = torch.ones(dh, device=dev) / math.sqrt(dh)
    qs, ks, vs = [], [], []
    for i, L in enumerate(lens):
        sg = 1.0 if i % 2 == 0 else -1.0
        qs.append(sg * amp * u + 0.2 * torch.randn(heads, L, dh, generator=g, device=dev))
        ks.append(-sg * amp * u + 0.3 * torch.randn(heads, L, dh, generator=g, device=dev))
        vs.append((1.0 + 0.5 * torch.randn(heads, L, dh, generator=g, device=dev)) if i % 2 == 0
                  else torch.full((heads, L, dh), -8.0, device=dev))
    qkv = pack_heads(qs, ks, vs)
    out, ref, r = check_attention(lib, qkv, lens, heads * dh, heads, kernel)
    assert bool(torch.isfinite(out.float()).all())
    record_property("worst_err_over_bound", r)


def _targets(L):
    return sorted({t for t in (0, 1, 63, 64, 65, 127, 128, 191, 192, 255, 256, 64 * ((L - 1) // 64), L - 2, L - 1)
                   if 0 <= t < L})


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,dh", ATT_KERNELS)
def test_attention_reaches_every_key_and_query_row(lib, record_property, kernel, dh):
    """Query row i is aimed at target key t(i) = targets[i % n] (keys 0, 63, 64, the first and last key of the last
    block, L - 1, ...): the target's key is b e_slot, the query a e_slot, with a b / sqrt(dh) = 24 nats against
    about 0.1 for every other key.  So ctx row i must equal v_t(i), for every query row of every 128-query tile and
    both warpgroups."""
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(7 + dh)
    lens, heads = [37, 200, 257, 512, 129], 2
    amp = math.sqrt(24.0 * math.sqrt(dh))
    qs, ks, vs, want = [], [], [], []
    for L in lens:
        tg = _targets(L)
        assert len(tg) <= dh
        k = 0.05 * torch.randn(heads, L, dh, generator=g, device=dev)
        q = torch.zeros(heads, L, dh, device=dev)
        for slot, t in enumerate(tg):
            k[:, t] = 0.0
            k[:, t, slot] = amp
        rows = torch.arange(L, device=dev)
        slots = rows % len(tg)
        q[:, rows, slots] = amp
        v = torch.randn(heads, L, dh, generator=g, device=dev)
        qs.append(q), ks.append(k), vs.append(v)
        tgt = torch.as_tensor(tg, device=dev)[slots]
        want.append(v[:, tgt].transpose(0, 1).reshape(L, heads * dh))
    qkv = pack_heads(qs, ks, vs)
    out, ref, r = check_attention(lib, qkv, lens, heads * dh, heads, kernel)
    want = torch.cat(want).bfloat16().double()
    assert float((ref - want).abs().max()) < 1e-5           # the construction: each query row sees one key
    record_property("worst_err_over_bound", r)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,dh", ATT_KERNELS)
def test_attention_uniform_is_the_mean_over_exactly_L_keys(lib, record_property, kernel, dh):
    dev = torch.device("cuda:0")
    H, heads = 2 * dh, 2
    qkv = torch.randn(sum(ATT_PACK), 3 * H, generator=torch.Generator(device=dev).manual_seed(11), device=dev).bfloat16()
    qkv[:, :H] = 0
    out, ref, r = check_attention(lib, qkv, ATT_PACK, H, heads, kernel)
    s0 = 0
    for L in ATT_PACK:
        mean = qkv[s0:s0 + L, 2 * H:].double().mean(dim=0)
        assert float((ref[s0:s0 + L] - mean).abs().max()) < 1e-12
        s0 += L
    record_property("worst_err_over_bound", r)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,dh", ATT_KERNELS)
def test_attention_running_max_stress(lib, record_property, kernel, dh):
    """Logits up to +-60 nats after scaling.  Key j of a sequence has k_0 = beta_j on a ramp; query rows alternate
    q_0 = +a_i and -a_i, so for half the rows the block maximum rises block after block (alpha is tiny at every
    step) and for the other half it falls (every later block is negligible)."""
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(13 + dh)
    lens, heads, A = [37, 512, 300, 129, 64], 2, 8.0
    bmax = 60.0 * math.sqrt(dh) / A                        # A * bmax / sqrt(dh) = 60 nats
    qs, ks, vs = [], [], []
    for L in lens:
        ramp = torch.linspace(-1.0, 1.0, L, device=dev)
        k = 0.5 * torch.randn(heads, L, dh, generator=g, device=dev)
        k[..., 0] = (bmax * ramp + 0.5 * torch.randn(heads, L, generator=g, device=dev)).clamp(-bmax, bmax)
        sign = torch.where(torch.arange(L, device=dev) % 2 == 0, 1.0, -1.0)
        q = torch.zeros(heads, L, dh, device=dev)
        q[..., 0] = sign * A * (0.5 + 0.5 * torch.rand(heads, L, generator=g, device=dev))
        q[:, 0, 0] = A
        qs.append(q), ks.append(k), vs.append(torch.randn(heads, L, dh, generator=g, device=dev))
    qkv = pack_heads(qs, ks, vs)
    out, ref, r = check_attention(lib, qkv, lens, heads * dh, heads, kernel)
    assert bool(torch.isfinite(out.float()).all())
    record_property("worst_err_over_bound", r)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,dh", ATT_KERNELS)
@pytest.mark.parametrize("L", [1, 63, 65, 200, 512])
def test_attention_rows_do_not_depend_on_packing(lib, kernel, dh, L):
    """A sequence's rows are bit-identical alone or packed at offset 37 between two other sequences."""
    dev = torch.device("cuda:0")
    H, heads = 2 * dh, 2
    lens = [37, L, 100]
    max_len = max(lens)
    qkv = torch.randn(sum(lens), 3 * H, generator=torch.Generator(device=dev).manual_seed(L), device=dev).bfloat16()
    packed = run_attention(lib, qkv, lens, H, heads, kernel, max_len)[37:37 + L]
    alone = run_attention(lib, qkv[37:37 + L].contiguous(), [L], H, heads, kernel, max_len)
    assert torch.equal(packed.view(torch.int16), alone.view(torch.int16))


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,dh", ATT_KERNELS)
@pytest.mark.parametrize("lens,max_lens", [([5, 64, 1, 33, 64, 17], (64, 65, 300)), ([37, 200, 129], (200, 257, 512))])
def test_attention_max_seqlen_larger_than_needed(lib, kernel, dh, lens, max_lens):
    """A max_seqlen above the longest sequence only adds CTAs that exit; for the mma.sync kernel 64 -> 65 switches
    the 64-query tile variant to the 128-query one.  The output is bit-identical."""
    dev = torch.device("cuda:0")
    H, heads = 2 * dh, 2
    qkv = torch.randn(sum(lens), 3 * H, generator=torch.Generator(device=dev).manual_seed(19), device=dev).bfloat16()
    base = run_attention(lib, qkv, lens, H, heads, kernel, max_lens[0]).clone()
    for m in max_lens[1:]:
        assert torch.equal(run_attention(lib, qkv, lens, H, heads, kernel, m).view(torch.int16), base.view(torch.int16)), m
