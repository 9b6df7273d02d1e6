"""Every crag_*_workspace_bytes against its layout restated here: the ordered list of region sizes in bytes, each region
starting on a 256-byte boundary.  Sizing needs no device, so this runs anywhere the library loads; the scan layouts
take their grid from crag_sm_count(), 132 without a device, as the library does."""
import ctypes as C
import itertools

import pytest

from comorag_b200 import _native

ALIGN = 256
NQ = 32                                  # queries per scan pass
POOL_SLOTS, POOL_MAX_CTAS = 5, 160       # pooled-floor keys per (query, CTA); no table above this grid
GMM_STATE = 32                           # sizeof(GmmState)


def total(regions):
    return sum((r + ALIGN - 1) // ALIGN * ALIGN for r in regions)


def cdiv(a, b):
    return -(-a // b)


@pytest.fixture(scope="module")
def lib():
    return _native.load()


@pytest.fixture(scope="module")
def grid(lib):
    g = lib.crag_sm_count()
    return g if g > 0 else 132


def scan_regions(grid, k):               # per-CTA keys, per-CTA (min, max), pooled-floor table
    return [grid * NQ * k * 8, grid * NQ * 2 * 4, NQ * grid * POOL_SLOTS * 8 if grid <= POOL_MAX_CTAS else 0]


def ivf_regions(grid, k, nlist, total_tiles):   # + list mask, coarse terms, work list (int4), work count
    return scan_regions(grid, k) + [nlist * 4, nlist * NQ * 4, total_tiles * 16, 4]


KS = [1, 2, 32, 33, 64, 65, 100, 128]


def test_search(lib, grid):
    for k, nq in itertools.product(KS, [1, 32, 1000]):
        assert lib.crag_search_workspace_bytes(nq, k) == total(scan_regions(grid, k)), (k, nq)


def test_ivf(lib, grid):
    for k, nlist, tiles in itertools.product(KS, [1, 2, 63, 64, 65, 1000, 1 << 20], [0, 1, 2, 3, 17, 1000, 1 << 20]):
        assert lib.crag_ivf_workspace_bytes(nlist, tiles, k) == total(ivf_regions(grid, k, nlist, tiles)), (k, nlist, tiles)


def test_ivf_i8(lib, grid):
    for n_cand, nlist, tiles in itertools.product(KS, [1, 2, 65, 4096], [0, 1, 3, 1000]):
        want = total(ivf_regions(grid, n_cand, nlist, tiles) + [NQ * n_cand * 8, NQ * n_cand * 4])
        assert lib.crag_ivf_i8_workspace_bytes(nlist, tiles, n_cand) == want, (n_cand, nlist, tiles)


def test_knn(lib):
    for n, q_chunk in itertools.product([0, 1, 2, 3, 4, 5, 63, 64, 65, 1000, 1 << 20], [1, 2, 7, 32, 1024]):
        ld = (max(n, 1) + 3) // 4 * 4
        assert lib.crag_knn_workspace_bytes(n, q_chunk) == total([q_chunk * ld * 4]), (n, q_chunk)


def test_rank(lib):
    for n in [0, 1, 2, 63, 64, 65, 2048, 2049, 8192 * 2048, 8192 * 2048 + 1, 100_000_000, (1 << 31) - 1]:
        run = 2048
        while cdiv(n, run) > 8192:
            run *= 2
        warps = max(1, cdiv(n, run))
        want = total([n * 4, n * 4, n * 4, n * 4, (256 * warps + 256) * 4])
        assert lib.crag_rank_workspace_bytes(n) == want, n


def ppr_shape(n, nnz):
    return cdiv(n + nnz, 512), min(max(cdiv(n, 256), 1), 1024)    # segments, sum blocks


PPR_SHAPES = list(itertools.product([1, 2, 63, 64, 65, 511, 512, 513, 100_000], [0, 1, 2, 511, 512, 10**6]))


def test_ppr(lib):
    for n, nnz in PPR_SHAPES:
        seg, sb = ppr_shape(n, nnz)
        want = total([n * 4, n * 4, (seg + 1) * 4, seg * 4, seg * 4, seg * 4, sb * 4])
        assert lib.crag_ppr_workspace_bytes(n, nnz) == want, (n, nnz)


def test_ppr_batch(lib):
    for (n, nnz), batch in itertools.product(PPR_SHAPES, range(1, 33)):
        seg, sb = ppr_shape(n, nnz)
        w = 2
        while w < batch:
            w *= 2
        want = total([n * w * 4] * 3 + [(seg + 1) * 4, seg * 4, seg * w * 4, seg * w * 4, sb * w * 4, w * 4])
        assert lib.crag_ppr_batch_workspace_bytes(n, nnz, batch) == want, (n, nnz, batch)


def test_gmm(lib):
    for n, d, m in itertools.product([2, 3, 51, 255, 256, 257, 8192, 8193, 100_000], [1, 2, 16], [1, 2, 50]):
        if m > n - 1:
            continue
        r = min(max(cdiv(n, 256), 1), 32)
        c = m * (m + 1) // 2
        tri = d * (d + 1) // 2
        s = 1 + d + tri
        want = total([8 * 17, GMM_STATE * m, 4 * c, 8 * n * d, 4 * n * m, 8 * n * m, 8 * c * d, 8 * r * c * (d + 1),
                      4 * r * m, 8 * c * d, 8 * c * tri, 8 * c, 8 * c, 8 * r * c * s, 8 * r * m])
        assert lib.crag_gmm_sweep_workspace_bytes(n, d, m) == want, (n, d, m)


UMAP_NS = [2, 3, 15, 16, 17, 18, 1023, 1024, 1025, 70_000]


def test_umap(lib):
    for n in UMAP_NS:
        assert lib.crag_umap_fuzzy_graph_workspace_bytes(n, 2) == total([8 * n, 8]), n
        for d in [1, 2, 15, 16]:
            assert lib.crag_umap_optimize_workspace_bytes(n, d) == total([4 * n * d]), (n, d)
            if d + 1 > n:
                continue
            p = min(n, max(16, d + 1))
            chunks = min(max(cdiv(n, 1024), 1), 64)
            want = total([8 * n, 8 * n, 8 * n * p, 8 * n * p, 8 * chunks * p * p, 8 * p * p, 8 * (p * p + p), 8 * n * d])
            assert lib.crag_umap_spectral_init_workspace_bytes(n, d) == want, (n, d)


def test_encoder(lib):
    from comorag_b200.encoder import _Model, _bind_encoder_abi
    _bind_encoder_abi(lib)
    m = _Model()
    for (h, i), tokens in itertools.product([(64, 256), (384, 1536), (768, 3072), (1024, 4096)], [0, 1, 7, 512, 10_000]):
        m.hidden, m.intermediate = h, i
        want = total([tokens * h * 2, tokens * 3 * h * 2, tokens * h * 2, tokens * h * 2, tokens * i * 2])
        assert lib.crag_encoder_workspace_bytes(C.byref(m), tokens) == want, (h, i, tokens)
