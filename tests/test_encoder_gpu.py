"""GPU parity of the encoder path: each kernel against a plain torch fp32 statement of the same op, the whole forward
against the torch oracle, and the drop-in BGEEmbeddingModel / EmbeddingStore against embeddings the REFERENCE produced
for the synthetic checkpoint (tests/golden/encoder_golden.npz)."""
import os

import numpy as np
import pytest
import torch

from oracle import encoder_oracle as eo

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(__file__)
CKPT = os.path.join(HERE, "golden", "bge-tiny-synth")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    from comorag_b200 import _native
    _native.load()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(HERE, "golden", "encoder_golden.npz"), allow_pickle=True)


@pytest.mark.parametrize("H", [128, 384, 768, 1024])
def test_layernorm(dev, H):
    """Within one bf16 step of a float64 LayerNorm, the bound encoder_emu_test.cpp holds the same kernel to."""
    from comorag_b200 import _native
    lib = _native.load()
    g = torch.Generator(device=dev).manual_seed(H)
    x = (torch.randn(1001, H, generator=g, device=dev) * 3 + 1).bfloat16()
    gam, bet = torch.randn(H, generator=g, device=dev), torch.randn(H, generator=g, device=dev)
    out = torch.zeros_like(x)
    _native.check(lib.crag_layernorm(x.data_ptr(), 1001, H, gam.data_ptr(), bet.data_ptr(), 1e-12, out.data_ptr(),
                                     torch.cuda.current_stream().cuda_stream), "crag_layernorm")
    ref = torch.nn.functional.layer_norm(x.double(), (H,), gam.double(), bet.double(), 1e-12)
    step = ref.abs().clamp(min=1e-3) * 2.0 ** -7
    assert bool(((out.double() - ref).abs() <= step).all()), float(((out.double() - ref).abs() / step).max())


def test_pool_normalize_matches_reference_pooling(dev):
    from comorag_b200 import _native
    lib = _native.load()
    H, lens = 384, [3, 512, 77, 1]
    g = torch.Generator(device=dev).manual_seed(1)
    hid = torch.randn(sum(lens), H, generator=g, device=dev).bfloat16()
    cu = torch.tensor([0] + np.cumsum(lens).tolist(), dtype=torch.int32, device=dev)
    out = torch.zeros(len(lens), H, device=dev)
    shard = torch.zeros(len(lens), 512, dtype=torch.bfloat16, device=dev)      # bf16 rows with a wider stride
    _native.check(lib.crag_pool_normalize(hid.data_ptr(), cu.data_ptr(), len(lens), H, 1, out.data_ptr(), shard.data_ptr(), 512,
                                          torch.cuda.current_stream().cuda_stream), "crag_pool_normalize")
    L = max(lens)
    padded, mask, s = torch.zeros(len(lens), L, H, device=dev), torch.zeros(len(lens), L, device=dev), 0
    for i, n in enumerate(lens):
        padded[i, :n], mask[i, :n] = hid[s:s + n].float(), 1
        s += n
    ref = torch.nn.functional.normalize(eo.mean_pooling(padded, mask), p=2, dim=1)
    assert float((out - ref).abs().max()) < 1e-5
    assert float((shard[:, :H].float() - ref).abs().max()) < 4e-3 and float(shard[:, H:].abs().max()) == 0.0


@pytest.mark.parametrize("cargs,lens,std", [((128, 2, 4, 256, 1000), [5, 64, 65, 1, 130, 17], 0.08),
                                            ((384, 4, 12, 1536, 30522), [512, 100, 37], 0.02),
                                            ((1024, 24, 16, 4096, 30522), [512, 128, 45], 0.02)])
def test_forward_vs_torch_oracle(dev, cargs, lens, std):
    """cosine >= 0.999 and max-abs <= 1e-2 per embedding vs the fp32 oracle on the same bf16-rounded weights
    (SURVEY.md section 8d); the bge-large shape is BASELINE config 2/3's encoder."""
    from comorag_b200.encoder import BertEncoderB200, EncoderConfig, random_state_dict
    cfg = EncoderConfig(*cargs)
    sd = random_state_dict(cfg, seed=1, std=std, device=dev)
    enc = BertEncoderB200(cfg, sd, dev)
    g = torch.Generator().manual_seed(7)
    seqs = [([101] + torch.randint(5, cfg.vocab_size, (L - 2,), generator=g).tolist() + [102]) if L >= 2 else [101] for L in lens]
    out = enc.encode_token_lists(seqs)
    sd_q = {k: (v.bfloat16().float() if v.dim() == 2 else v) for k, v in sd.items()}
    ref = eo.encode_token_lists(sd_q, cfg, seqs)
    assert float(torch.nn.functional.cosine_similarity(out, ref, dim=1).min()) > 0.999
    assert float((out - ref).abs().max()) < 1e-2
    # rows do not depend on what they are batched with (unpadded packing == padding + mask)
    alone = enc.encode_token_lists(seqs[:1])
    assert float((alone[0] - out[0]).abs().max()) < 1e-6


def test_bge_large_256_mixed_length_chunks_centred_cosine(dev):
    """SURVEY.md 8d at its stated size: >= 256 chunks, lengths U[32, 512], the bge-large shape (24 layers).  With HF's
    default init every embedding collapses onto one direction and a plain cosine is vacuous, so the word embeddings
    get unit scale (texts then differ) and the cosine is ALSO taken after removing the mean embedding of the batch:
    that centred cosine only stays high if the per-text part of the embedding is right."""
    from comorag_b200.encoder import BertEncoderB200, EncoderConfig, random_state_dict
    cfg = EncoderConfig(1024, 24, 16, 4096, 30522)
    # layer weights N(0, 0.01), word embeddings N(0, 1): measured on the fp32 oracle, 24 layers of N(0, 0.02) weights
    # collapse any two texts to cosine 0.92+ whatever the embeddings are; at 0.01 the pair cosine stays near 0.5
    sd = random_state_dict(cfg, seed=3, std=0.01, device=dev)
    sd["embeddings.word_embeddings.weight"] = sd["embeddings.word_embeddings.weight"] * 100.0    # std 1.0
    enc = BertEncoderB200(cfg, sd, dev)
    g = torch.Generator().manual_seed(11)
    lens = torch.randint(32, 513, (256,), generator=g).tolist()
    seqs = [[101] + torch.randint(1000, cfg.vocab_size, (L - 2,), generator=g).tolist() + [102] for L in lens]
    outs = []
    for s0 in range(0, 256, 64):                      # 64 chunks (~17k tokens) per packed forward
        outs.append(enc.encode_token_lists(seqs[s0:s0 + 64]))
    out = torch.cat(outs, 0)
    sd_q = {k: (v.bfloat16().float() if v.dim() == 2 else v) for k, v in sd.items()}
    ref = eo.encode_token_lists(sd_q, cfg, seqs)
    cos = torch.nn.functional.cosine_similarity(out, ref, dim=1)
    mean = ref.mean(dim=0, keepdim=True)
    ccos = torch.nn.functional.cosine_similarity(out - mean, ref - mean, dim=1)
    spread = float(torch.nn.functional.cosine_similarity(ref[:128], ref[128:], dim=1).mean())
    err = float((out - ref).abs().max())
    assert spread < 0.9, f"the synthetic embeddings collapsed (mean pair cosine {spread:.4f}): the test would be vacuous"
    assert float(cos.min()) > 0.999 and err < 1e-2, (float(cos.min()), err)
    assert float(ccos.min()) > 0.99, f"centred cosine {float(ccos.min()):.5f} (plain {float(cos.min()):.6f}, max-abs {err:.2e})"


def test_dropin_model_matches_reference_embeddings(dev, gold):
    """BGEEmbeddingModel (ours) on the synthetic checkpoint vs what the REFERENCE's BGEEmbeddingModel returned."""
    from comorag_b200.config import EngineConfig
    from comorag_b200.embedding_model import BGEEmbeddingModel, _get_embedding_model_class
    assert _get_embedding_model_class(CKPT) is BGEEmbeddingModel
    cfg = EngineConfig(embedding_model_name=CKPT, embedding_batch_size=4, embedding_max_seq_len=512)
    model = BGEEmbeddingModel(global_config=cfg, embedding_model_name=CKPT)
    texts = gold["texts"].tolist()
    assert model.embedding_dim == 128
    ids = model._tokenize(["Generate a representation for this sentence to retrieve relevant articles:" + t for t in texts], 512)
    assert [list(x) for x in ids] == [t.tolist() for t in gold["token_ids"]]      # same tokenizer call as the reference
    emb = model.batch_encode(texts)
    assert emb.dtype == np.float32 and emb.shape == gold["emb_batch"].shape and emb.flags["C_CONTIGUOUS"]
    ref = gold["emb_batch"]
    cos = (emb * ref).sum(1) / (np.linalg.norm(emb, axis=1) * np.linalg.norm(ref, axis=1))
    assert cos.min() > 0.999 and np.abs(emb - ref).max() < 1e-2
    # centred comparison: random-weight encoders put every text near one direction; remove it so the check bites
    c_emb, c_ref = emb - ref.mean(0), ref - ref.mean(0)
    ccos = (c_emb * c_ref).sum(1) / (np.linalg.norm(c_emb, axis=1) * np.linalg.norm(c_ref, axis=1))
    assert ccos.min() > 0.99, ccos
    n_c, n_q = int(gold["n_chunks"]), int(gold["n_questions"])
    one = model.batch_encode(texts[n_c], instruction="ignored", norm=True)      # str input -> [1, D]; kwargs ignored
    assert one.shape == (1, 128) and np.abs(one[0] - emb[n_c]).max() < 1e-5
    np.testing.assert_allclose(model.encode_queries(texts[n_c:n_c + n_q]), emb[n_c:n_c + n_q], atol=1e-5)
    t = model.encode(texts[:3])                                                  # positional surface, torch.Tensor, no prefix
    assert isinstance(t, torch.Tensor) and np.abs(t.cpu().numpy() - gold["emb_encode"]).max() < 1e-2
    np.testing.assert_allclose(model.get_query_doc_scores(emb[:1], emb), emb[:1] @ emb.T)


def test_cinderella_plumbing_top10_matches_reference_math(dev, gold, tmp_path):
    """BASELINE config 1: chunks -> EmbeddingStore.insert_strings -> device index -> top-k; ids equal the reference's
    np.dot + argsort on the reference's own embeddings wherever its score gaps exceed the bf16 storage noise."""
    from comorag_b200.config import EngineConfig
    from comorag_b200.embedding_model import BGEEmbeddingModel
    from comorag_b200.embedding_store import EmbeddingStore
    from oracle import search_oracle as so
    cfg = EngineConfig(embedding_model_name=CKPT, embedding_batch_size=4, embedding_max_seq_len=512)
    model = BGEEmbeddingModel(global_config=cfg, embedding_model_name=CKPT)
    texts = gold["texts"].tolist()
    n_c, n_q = int(gold["n_chunks"]), int(gold["n_questions"])
    store = EmbeddingStore(model, str(tmp_path / "chunk_embeddings"), 4, "chunk")
    store.insert_strings(texts[:n_c] + texts[n_c + n_q:])
    assert store.insert_strings(texts[:2]) == {}
    ref_rows = np.concatenate([gold["emb_batch"][:n_c], gold["emb_batch"][n_c + n_q:]])
    got_rows = store.get_embeddings(store.get_all_ids())
    assert np.abs(got_rows - ref_rows).max() < 1e-2
    q_emb = model.batch_encode(texts[n_c:n_c + n_q])
    ids, scores, minmax = store.search(q_emb, min(10, len(store.hash_ids)))
    k = ids.shape[1]
    for qi in range(n_q):
        ref_ids, ref_sc = so.dense_passage_retrieval(ref_rows, gold["emb_batch"][n_c + qi][None])
        raw = np.dot(ref_rows, gold["emb_batch"][n_c + qi])
        order = np.argsort(-raw)
        gaps = -np.diff(raw[order])
        # ranks separated by more than the bf16/encoder noise (1e-2 abs on unit vectors -> ~2e-2 on a dot) must agree
        j = 0
        while j < k - 1 and gaps[j] > 4e-2:
            assert ids[qi, j] == order[j]
            j += 1
        assert set(ids[qi].tolist()) <= set(range(len(store.hash_ids)))
        assert np.abs(np.sort(scores[qi]) - np.sort(raw[ids[qi]])).max() < 3e-2


def test_xlm_roberta_variant_position_offset(dev):
    """XLM-R style checkpoints (position offset 2, eps 1e-5, one token type) through the same kernels."""
    from comorag_b200.encoder import BertEncoderB200, EncoderConfig, random_state_dict
    cfg = EncoderConfig(128, 2, 2, 256, 1000, max_position_embeddings=514, type_vocab_size=1, layer_norm_eps=1e-5, position_offset=2)
    sd = random_state_dict(cfg, seed=5, std=0.06, device=dev)
    enc = BertEncoderB200(cfg, sd, dev)
    g = torch.Generator().manual_seed(2)
    seqs = [[0] + torch.randint(5, 1000, (n,), generator=g).tolist() + [2] for n in (3, 100, 510)]
    out = enc.encode_token_lists(seqs)
    sd_q = {k: (v.bfloat16().float() if v.dim() == 2 else v) for k, v in sd.items()}
    ref = eo.encode_token_lists(sd_q, cfg, seqs, pad_id=1)
    assert float(torch.nn.functional.cosine_similarity(out, ref, dim=1).min()) > 0.999 and float((out - ref).abs().max()) < 1e-2
    with pytest.raises(Exception):
        enc.encode_token_lists([[0] * 600])          # longer than the position table: reported, not truncated silently


def test_sixteen_threads_share_the_engine(dev, gold, tmp_path):
    """ComoRAG answers questions from a 16-thread pool (ComoRAG.py:436-441): concurrent batch_encode / store.search
    calls (with and without the request coalescer) return exactly what serial calls return."""
    from concurrent.futures import ThreadPoolExecutor
    from comorag_b200.config import EngineConfig
    from comorag_b200.embedding_model import BGEEmbeddingModel
    from comorag_b200.embedding_store import EmbeddingStore
    texts = gold["texts"].tolist()
    queries = [f"{t[:40]} {i}" for i, t in enumerate(texts * 3)]
    for coalesce in (False, True):
        cfg = EngineConfig(embedding_model_name=CKPT, embedding_batch_size=8, embedding_max_seq_len=512, embedding_coalesce=coalesce)
        model = BGEEmbeddingModel(global_config=cfg, embedding_model_name=CKPT)
        store = EmbeddingStore(model, str(tmp_path / f"s{int(coalesce)}"), 8, "chunk")
        store.insert_strings(texts)
        serial_e = [model.batch_encode(q) for q in queries]
        serial_s = [store.search(e, 5) for e in serial_e]

        before = model._coalescer.stats["forwards"] if coalesce else 0

        def work(i):
            e = model.batch_encode(queries[i])
            return e, store.search(e, 5)

        with ThreadPoolExecutor(16) as ex:
            par = list(ex.map(work, range(len(queries))))
        for i, (e, (ids, sc, mm)) in enumerate(par):
            np.testing.assert_allclose(e, serial_e[i], atol=1e-6)
            np.testing.assert_allclose(sc, serial_s[i][1], atol=1e-5)
            ref_ids, ref_sc = serial_s[i][0][0], serial_s[i][1][0]
            for j in range(5):  # ranks whose neighbours are further than the batching noise must agree exactly
                lo = ref_sc[j] - ref_sc[j + 1] if j + 1 < 5 else 1.0
                hi = ref_sc[j - 1] - ref_sc[j] if j > 0 else 1.0
                if min(lo, hi) > 1e-4:
                    assert ids[0][j] == ref_ids[j]
        if coalesce:
            assert model._coalescer.stats["forwards"] - before < len(queries)      # requests really shared launches


def test_incremental_insert_uses_device_rows(dev, gold, tmp_path):
    """After the device index exists, insert_strings feeds it from the encoder's device output; the result equals a
    store built in one go (same ids, same rows, same search)."""
    from comorag_b200.config import EngineConfig
    from comorag_b200.embedding_model import BGEEmbeddingModel
    from comorag_b200.embedding_store import EmbeddingStore
    cfg = EngineConfig(embedding_model_name=CKPT, embedding_batch_size=4, embedding_max_seq_len=512)
    model = BGEEmbeddingModel(global_config=cfg, embedding_model_name=CKPT)
    texts = gold["texts"].tolist()
    a = EmbeddingStore(model, str(tmp_path / "a"), 4, "chunk")
    a.insert_strings(texts[:5])
    q = model.batch_encode(texts[6:9])
    a.search(q, 3)                                   # builds the device shard
    a.insert_strings(texts[3:])                      # 7 new rows through the device fast path
    assert a.index.n_rows == len(texts) == len(a.hash_ids)
    b = EmbeddingStore(model, str(tmp_path / "b"), 4, "chunk")
    b.insert_strings(texts)
    assert a.get_all_ids() == b.get_all_ids()
    np.testing.assert_allclose(a.get_embeddings(a.hash_ids), b.get_embeddings(b.hash_ids), atol=1e-6)
    ia, sa, _ = a.search(q, 5)
    ib, sb, _ = b.search(q, 5)
    np.testing.assert_allclose(sa, sb, atol=1e-5)
    assert torch.equal(a.index.matrix().float().cpu(), b.index.matrix().float().cpu()) or \
        float((a.index.matrix().float() - b.index.matrix().float()).abs().max()) < 1e-2


@pytest.mark.parametrize("cargs,lens,std,tol", [((128, 2, 2, 256, 1000), [4, 100, 257, 510], 0.06, 3e-2),
                                                ((1024, 24, 16, 4096, 3000), [512, 77], 0.02, 6e-2)])
def test_cross_encoder_logits_match_oracle(dev, cargs, lens, std, tol):
    """bge-reranker-* architecture (XLM-R encoder + classification head on <s>): crag_encoder_classify against the
    fp32 oracle on the same bf16-rounded weights; the large case is bge-reranker-large's shape (BASELINE config 5)
    with a cut-down vocabulary.  Pre-tanh activations are O(1) (head std 0.1 at H=128, scaled 1/sqrt(H)); absolute
    tolerance 3e-2 (2 layers) / 6e-2 (24 layers of bf16 activations feeding a 1024-term dot)."""
    from comorag_b200.encoder import BertEncoderB200, EncoderConfig, random_head_state_dict, random_state_dict
    cfg = EncoderConfig(*cargs, max_position_embeddings=514, type_vocab_size=1, layer_norm_eps=1e-5, position_offset=2)
    sd = random_state_dict(cfg, seed=9, std=std, device=dev)
    head = random_head_state_dict(cfg, n_labels=1, seed=9, std=0.1 * (128 / cfg.hidden_size) ** 0.5, device=dev)
    enc = BertEncoderB200(cfg, {**{"roberta." + k: v for k, v in sd.items()}, **head}, dev)
    assert enc.n_labels == 1
    g = torch.Generator().manual_seed(4)
    seqs = [[0] + torch.randint(5, cfg.vocab_size, (n - 2,), generator=g).tolist() + [2] for n in lens]
    got = enc.classify_token_lists(seqs)
    q = lambda d: {k: (v.bfloat16().float() if v.dim() == 2 else v) for k, v in d.items()}
    want = eo.classifier_logits(q(sd), q(head), cfg, seqs, pad_id=1)
    assert got.shape == want.shape == (len(lens), 1)
    assert float(want.abs().max()) > 0.05                         # the comparison is not vacuous
    assert float((got - want).abs().max()) < tol
    # pooled embeddings of the same checkpoint are untouched by the head
    emb = enc.encode_token_lists(seqs[:2])
    ref = eo.encode_token_lists(q(sd), cfg, seqs[:2], pad_id=1)
    assert float(torch.nn.functional.cosine_similarity(emb, ref, dim=1).min()) > 0.999
    # a checkpoint without classifier weights refuses instead of scoring with garbage
    plain = BertEncoderB200(cfg, sd, dev) if cfg.hidden_size == 128 else None
    if plain is not None:
        with pytest.raises(Exception):
            plain.classify_token_lists(seqs[:1])
