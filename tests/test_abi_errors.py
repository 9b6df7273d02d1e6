"""Error behaviour of the C ABI that does not need a device: every entry point validates its arguments before
touching CUDA, returns a negative status (include/comorag_b200.h) and leaves a message in crag_last_error();
nothing crashes, nothing falls back to a CPU path."""
import ctypes as C

import pytest

from comorag_b200 import _native

INVALID, CUDA, WORKSPACE, UNSUPPORTED = -1, -2, -3, -4


@pytest.fixture(scope="module")
def lib():
    return _native.load()


@pytest.fixture(scope="module")
def p():
    """A 256-byte aligned host address: good enough for pointer/alignment checks, never dereferenced (every call
    below is rejected before a launch)."""
    buf = (C.c_char * 8192)()
    addr = (C.addressof(buf) + 255) & ~255
    p.keepalive = buf
    return addr


def err(lib):
    return lib.crag_last_error().decode()


def test_search_argument_validation(lib, p):
    ws = lib.crag_search_workspace_bytes(32, 10)
    assert ws > 0 and ws % 256 == 0
    assert lib.crag_search_workspace_bytes(32, 128) > ws
    call = lambda **kw: lib.crag_search_topk(*[kw.get(n, d) for n, d in (
        ("corpus", p), ("n_rows", 100), ("dim", 1024), ("stride", 1024), ("row_offset", 0), ("queries", p), ("nq", 4),
        ("k", 10), ("ids", p), ("scores", p), ("minmax", p), ("ws", p), ("ws_bytes", 1 << 24), ("stream", None))])
    assert call(nq=0) == INVALID and "nq" in err(lib)
    assert call(k=0) == INVALID and call(k=129) == INVALID
    assert call(dim=1000) == INVALID and "dim" in err(lib)
    assert call(dim=2048) == INVALID
    assert call(stride=512) == INVALID and "stride" in err(lib)
    assert call(n_rows=-1) == INVALID and call(n_rows=1 << 31) == INVALID
    assert call(queries=None) == INVALID and "null" in err(lib)
    assert call(corpus=p + 8) == INVALID and "aligned" in err(lib)
    assert call(ws=p + 64) == INVALID and "workspace" in err(lib)
    assert call(ws_bytes=16) == WORKSPACE and "workspace" in err(lib)
    assert call(ids=None) == INVALID


def test_finalize_workspace_validation(lib, p):
    """The finalize entries read 8-byte keys from the scan's workspace: a misaligned one is refused before a launch."""
    fin = lambda ws=p, wsb=1 << 24: lib.crag_search_finalize(ws, wsb, 100, 4, 10, 0, p, p, p, None)
    xchg = lambda ws=p, wsb=1 << 24: lib.crag_search_finalize_exchange(ws, wsb, 100, 4, 10, 0, p, 0, 2, p, p, p, p, p,
                                                                       None)
    for call in (fin, xchg):
        assert call(ws=None) == INVALID and "null" in err(lib)
        assert call(ws=p + 8) == INVALID and "256-byte aligned" in err(lib)
        assert call(wsb=16) == WORKSPACE and "workspace 16 <" in err(lib)


def test_merge_gemm_and_encoder_piece_validation(lib, p):
    assert lib.crag_merge_topk(p, p, None, 2, 0, 10, p, p, None, None) == INVALID
    assert lib.crag_merge_topk(p, p, None, 2, 4, 200, p, p, None, None) == INVALID
    assert lib.crag_merge_topk(None, p, None, 2, 4, 10, p, p, None, None) == INVALID and "null" in err(lib)
    assert lib.crag_merge_topk_packed(p, 8, 2, 4, 10, p, p, p, None) == INVALID and "record_bytes" in err(lib)
    assert lib.crag_gemm_bf16(p, 64, p, 64, None, None, 0, p, 64, 128, 64, 60, 0, None) == INVALID and "K" in err(lib)
    assert lib.crag_layernorm(p, 4, 100, p, p, 1e-5, p, None) == INVALID
    assert lib.crag_pool_normalize(None, p, 1, 64, 1, p, None, 0, None) == INVALID
    assert lib.crag_attention_varlen(p, p, 1, 8, 100, 3, p, None) == INVALID
    assert lib.crag_attention_varlen_tc(p, p, 1, 8, 8, 128, 4, p, None) == UNSUPPORTED and "64" in err(lib)


def test_encoder_model_validation(lib, p):
    from comorag_b200.encoder import _Head, _Layer, _Model, _bind_encoder_abi
    _bind_encoder_abi(lib)
    layers = (_Layer * 1)()
    m = _Model()
    m.hidden, m.n_layers, m.heads, m.intermediate, m.vocab, m.max_pos, m.pos_offset, m.ln_eps = 128, 1, 2, 256, 100, 64, 0, 1e-12
    m.word_emb = m.pos_emb = m.type_emb = m.emb_ln_g = m.emb_ln_b = p
    m.layers = C.cast(layers, C.POINTER(_Layer))
    fwd = lambda model, n=2, T=10, L=8, out=p, ws=p, wsb=1 << 30: lib.crag_encoder_forward(
        C.byref(model), p, p, n, T, L, 1, out, None, 0, ws, wsb, None)
    assert lib.crag_encoder_workspace_bytes(C.byref(m), 1000) == 1000 * (3 * 128 * 2 + 3 * 128 * 2 + 256 * 2)   # x, ctx, tmp | qkv | ff (bf16)
    assert fwd(m, n=0) == 0                                             # empty batch: nothing to do, no launch
    assert fwd(m, L=100) == INVALID and "position table" in err(lib)   # longer than the checkpoint can embed
    assert fwd(m, out=None) == INVALID
    assert fwd(m, wsb=64) == WORKSPACE
    assert fwd(m, ws=p + 16) == INVALID and "aligned" in err(lib)
    m.hidden = 2048
    assert fwd(m) == UNSUPPORTED and "hidden" in err(lib)
    m.hidden, m.heads = 128, 3
    assert fwd(m) == INVALID
    m.heads = 8                                                          # head dim 16
    assert fwd(m) == UNSUPPORTED and "head dim" in err(lib)
    m.heads, m.word_emb = 2, None
    assert fwd(m) == INVALID and "embedding" in err(lib)
    m.word_emb = p
    h = _Head()
    cls = lambda head: lib.crag_encoder_classify(C.byref(m), C.byref(head), p, p, 2, 10, 8, p, p, 1 << 30, None)
    assert cls(h) == INVALID and "head" in err(lib)
    h.w_dense = h.b_dense = h.w_out = h.b_out = p
    h.n_labels = 0
    assert cls(h) == INVALID and "n_labels" in err(lib)


def test_host_classes_refuse_to_run_without_a_device():
    """No CPU fallback: constructing the engine's device objects without CUDA raises instead of degrading."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("this check is for the CPU-only container")
    from comorag_b200.encoder import BertEncoderB200, EncoderConfig
    from comorag_b200.index import DenseIndex
    with pytest.raises(_native.NativeError):
        DenseIndex(64)
    with pytest.raises(_native.NativeError):
        BertEncoderB200(EncoderConfig(64, 1, 1, 128, 100), {})
