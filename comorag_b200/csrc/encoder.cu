// Encoder forward driver: the whole of BGEEmbeddingModel._encode's device work
// (BGEEmbedding.py:119-127: BertModel forward -> mean_pooling -> F.normalize)
// as one stream-ordered launch sequence over a packed (unpadded) token batch.
// Post-LN BERT layer, exactly HF's BertLayer:
//   qkv  = x Wqkv^T + b                      (wgmma GEMM, fused q/k/v weights)
//   ctx  = softmax(q k^T / sqrt(dh)) v       (varlen attention)
//   x    = LN(ctx Wo^T + bo + x)             (GEMM + residual epilogue, LN kernel)
//   x    = LN(gelu(x W1^T + b1) W2^T + b2 + x)
#include "common.cuh"
#include "encoder.cuh"
#include "gemm.cuh"
#include "workspace.cuh"

namespace crag {
namespace {

struct EncoderBuffers {
  uint8_t *x, *qkv, *ctx, *tmp, *ff;
  size_t total;
};

EncoderBuffers carve(void* ws, int T, int H, int I) {
  WsCursor c(ws);
  EncoderBuffers b;
  b.x = c.take<uint8_t>(size_t(T) * H * 2);
  b.qkv = c.take<uint8_t>(size_t(T) * 3 * H * 2);
  b.ctx = c.take<uint8_t>(size_t(T) * H * 2);
  b.tmp = c.take<uint8_t>(size_t(T) * H * 2);
  b.ff = c.take<uint8_t>(size_t(T) * I * 2);
  b.total = c.bytes;
  return b;
}

int check_model(const crag_encoder* m) {
  if (!m) return fail(CRAG_ERR_INVALID, "encoder: null model");
  if (m->hidden < 64 || m->hidden > 1024 || m->hidden % 8) return fail(CRAG_ERR_UNSUPPORTED, "encoder: hidden size %d unsupported (64..1024, multiple of 8)", m->hidden);
  if (m->heads < 1 || m->hidden % m->heads) return fail(CRAG_ERR_INVALID, "encoder: hidden %d not divisible by heads %d", m->hidden, m->heads);
  const int dh = m->hidden / m->heads;
  if (dh != 32 && dh != 64) return fail(CRAG_ERR_UNSUPPORTED, "encoder: head dim %d unsupported (32 or 64)", dh);
  if (m->intermediate < 8 || m->intermediate % 8) return fail(CRAG_ERR_INVALID, "encoder: intermediate size %d must be a multiple of 8", m->intermediate);
  if (m->n_layers < 0 || (m->n_layers > 0 && !m->layers)) return fail(CRAG_ERR_INVALID, "encoder: bad layer table");
  if (!m->word_emb || !m->pos_emb || !m->type_emb || !m->emb_ln_g || !m->emb_ln_b) return fail(CRAG_ERR_INVALID, "encoder: null embedding weights");
  return CRAG_OK;
}

}  // namespace
}  // namespace crag

using namespace crag;

extern "C" size_t crag_encoder_workspace_bytes(const crag_encoder* model, int total_tokens) {
  if (!model || total_tokens < 0) return 0;
  return carve(nullptr, total_tokens, model->hidden, model->intermediate).total;
}

namespace crag {
namespace {

// Validates the batch, carves the workspace and runs embeddings + all layers; on success b.x holds last_hidden_state
// (bf16 [total_tokens, H]).
int run_layers(const crag_encoder* model, const int32_t* token_ids, const int32_t* cu_seqlens, int n_seqs,
               int total_tokens, int max_seqlen, void* workspace, size_t workspace_bytes, cudaStream_t stream,
               EncoderBuffers& b) {
  if (!token_ids || !cu_seqlens || !workspace) return fail(CRAG_ERR_INVALID, "encoder: null pointer");
  if (max_seqlen > model->max_pos - model->pos_offset) return fail(CRAG_ERR_INVALID, "encoder: max_seqlen %d exceeds the position table (%d - %d)", max_seqlen, model->max_pos, model->pos_offset);
  const int T = total_tokens, H = model->hidden, I = model->intermediate;
  b = carve(workspace, T, H, I);
  int rc = check_workspace("encoder", workspace, workspace_bytes, b.total);
  if (rc != CRAG_OK) return rc;

  rc = launch_embed_layernorm(token_ids, cu_seqlens, n_seqs, T, H, model->vocab, model->max_pos, model->pos_offset,
                                  model->word_emb, model->pos_emb, model->type_emb, model->emb_ln_g, model->emb_ln_b,
                                  model->ln_eps, b.x, stream);
  if (rc != CRAG_OK) return rc;
  for (int l = 0; l < model->n_layers; ++l) {
    const crag_encoder_layer& w = model->layers[l];
    rc = gemm_bf16(b.x, H, w.w_qkv, H, w.b_qkv, nullptr, 0, b.qkv, 3 * H, T, 3 * H, H, GEMM_EPI_BIAS, stream);
    if (rc != CRAG_OK) return rc;
    // head dim 64 (bge-base / bge-large): wgmma kernel; head dim 32 (bge-small): mma.sync kernel
    rc = (H / model->heads == 64)
             ? launch_attention_tc(b.qkv, cu_seqlens, n_seqs, T, max_seqlen, H, model->heads, b.ctx, stream)
             : launch_attention(b.qkv, cu_seqlens, n_seqs, max_seqlen, H, model->heads, b.ctx, stream);
    if (rc != CRAG_OK) return rc;
    rc = gemm_bf16(b.ctx, H, w.w_o, H, w.b_o, b.x, H, b.tmp, H, T, H, H, GEMM_EPI_BIAS_RESIDUAL, stream);
    if (rc != CRAG_OK) return rc;
    rc = launch_layernorm(b.tmp, T, H, w.ln1_g, w.ln1_b, model->ln_eps, b.x, stream);
    if (rc != CRAG_OK) return rc;
    rc = gemm_bf16(b.x, H, w.w_ff1, H, w.b_ff1, nullptr, 0, b.ff, I, T, I, H, GEMM_EPI_BIAS_GELU, stream);
    if (rc != CRAG_OK) return rc;
    rc = gemm_bf16(b.ff, I, w.w_ff2, I, w.b_ff2, b.x, H, b.tmp, H, T, H, I, GEMM_EPI_BIAS_RESIDUAL, stream);
    if (rc != CRAG_OK) return rc;
    rc = launch_layernorm(b.tmp, T, H, w.ln2_g, w.ln2_b, model->ln_eps, b.x, stream);
    if (rc != CRAG_OK) return rc;
  }
  return CRAG_OK;
}

}  // namespace
}  // namespace crag

extern "C" int crag_encoder_forward(const crag_encoder* model, const int32_t* token_ids, const int32_t* cu_seqlens,
                                    int n_seqs, int total_tokens, int max_seqlen, int normalize, float* out_f32,
                                    void* out_bf16, int64_t out_bf16_stride, void* workspace,
                                    size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_model(model);
  if (rc != CRAG_OK) return rc;
  if (n_seqs < 0 || total_tokens < 0 || max_seqlen < 0) return fail(CRAG_ERR_INVALID, "encoder: negative sizes");
  if (n_seqs == 0) return CRAG_OK;
  if (!out_f32 && !out_bf16) return fail(CRAG_ERR_INVALID, "encoder: null pointer");
  if (out_bf16 && (out_bf16_stride < model->hidden || out_bf16_stride % 8 || (reinterpret_cast<uintptr_t>(out_bf16) & 15)))
    return fail(CRAG_ERR_INVALID, "encoder: out_bf16 stride/alignment");
  EncoderBuffers b;
  rc = run_layers(model, token_ids, cu_seqlens, n_seqs, total_tokens, max_seqlen, workspace, workspace_bytes, stream, b);
  if (rc != CRAG_OK) return rc;
  return launch_pool_normalize(b.x, cu_seqlens, n_seqs, model->hidden, normalize, out_f32, out_bf16, out_bf16_stride, stream);
}

// Cross-encoder scoring: the same layers, then the classification head on every sequence's first token.
extern "C" int crag_encoder_classify(const crag_encoder* model, const crag_classifier_head* head,
                                     const int32_t* token_ids, const int32_t* cu_seqlens, int n_seqs,
                                     int total_tokens, int max_seqlen, float* logits, void* workspace,
                                     size_t workspace_bytes, crag_stream_t stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  int rc = check_model(model);
  if (rc != CRAG_OK) return rc;
  if (!head || !head->w_dense || !head->b_dense || !head->w_out || !head->b_out) return fail(CRAG_ERR_INVALID, "classify: null head weights");
  if (head->n_labels < 1) return fail(CRAG_ERR_INVALID, "classify: n_labels %d", head->n_labels);
  if (n_seqs < 0 || total_tokens < 0 || max_seqlen < 0) return fail(CRAG_ERR_INVALID, "encoder: negative sizes");
  if (n_seqs == 0) return CRAG_OK;
  if (!logits) return fail(CRAG_ERR_INVALID, "classify: null logits");
  EncoderBuffers b;
  rc = run_layers(model, token_ids, cu_seqlens, n_seqs, total_tokens, max_seqlen, workspace, workspace_bytes, stream, b);
  if (rc != CRAG_OK) return rc;
  return launch_cls_head(b.x, cu_seqlens, n_seqs, model->hidden, head->w_dense, head->b_dense, head->w_out, head->b_out,
                         head->n_labels, logits, stream);
}

// Stand-alone pooling entry (K3), for callers that already hold last_hidden_state.
extern "C" int crag_pool_normalize(const void* hidden, const int32_t* cu_seqlens, int n_seqs, int hidden_size,
                                   int normalize, float* out_f32, void* out_bf16, int64_t out_bf16_stride,
                                   crag_stream_t stream) {
  if (!hidden || !cu_seqlens || (!out_f32 && !out_bf16)) return fail(CRAG_ERR_INVALID, "pool_normalize: null pointer");
  if (hidden_size % 8) return fail(CRAG_ERR_INVALID, "pool_normalize: hidden size must be a multiple of 8");
  return launch_pool_normalize(hidden, cu_seqlens, n_seqs, hidden_size, normalize, out_f32, out_bf16, out_bf16_stride,
                               static_cast<cudaStream_t>(stream));
}

// Stand-alone varlen attention (K2) and LayerNorm entries, exported so each kernel can be parity-tested alone.
extern "C" int crag_attention_varlen(const void* qkv, const int32_t* cu_seqlens, int n_seqs, int max_seqlen,
                                     int hidden_size, int heads, void* ctx, crag_stream_t stream) {
  if (!qkv || !cu_seqlens || !ctx) return fail(CRAG_ERR_INVALID, "attention: null pointer");
  if (heads < 1 || hidden_size % heads || hidden_size % 8) return fail(CRAG_ERR_INVALID, "attention: bad hidden/heads");
  return launch_attention(qkv, cu_seqlens, n_seqs, max_seqlen, hidden_size, heads, ctx, static_cast<cudaStream_t>(stream));
}

extern "C" int crag_attention_varlen_tc(const void* qkv, const int32_t* cu_seqlens, int n_seqs, int total_tokens,
                                        int max_seqlen, int hidden_size, int heads, void* ctx, crag_stream_t stream) {
  if (!qkv || !cu_seqlens || !ctx) return fail(CRAG_ERR_INVALID, "attention: null pointer");
  if (heads > 255) return fail(CRAG_ERR_INVALID, "attention_tc: heads must be <= 255 (heads=%d)", heads);
  if (heads < 1 || hidden_size % heads || hidden_size / heads != 64) return fail(CRAG_ERR_UNSUPPORTED, "attention_tc: head dim must be 64");
  return launch_attention_tc(qkv, cu_seqlens, n_seqs, total_tokens, max_seqlen, hidden_size, heads, ctx,
                             static_cast<cudaStream_t>(stream));
}

extern "C" int crag_layernorm(const void* in, int rows, int hidden_size, const float* gamma, const float* beta,
                              float eps, void* out, crag_stream_t stream) {
  if (!in || !gamma || !beta || !out) return fail(CRAG_ERR_INVALID, "layernorm: null pointer");
  if (hidden_size % 8) return fail(CRAG_ERR_INVALID, "layernorm: hidden size must be a multiple of 8");
  return launch_layernorm(in, rows, hidden_size, gamma, beta, eps, out, static_cast<cudaStream_t>(stream));
}
