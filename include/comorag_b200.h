/*
 * libcomorag_b200 -- C ABI of the H100 (sm_90a) embedding + dense-retrieval
 * engine that sits behind ComoRAG's embedding_model / EmbeddingStore call
 * surfaces.
 *
 * The reference (EternityJune25/ComoRAG) is pure Python and has no FFI of its
 * own; every entry point below names the reference arithmetic it replaces
 * (file:line relative to the reference tree).  The Python host layer in
 * comorag_b200/ binds these with ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - plain C types only; every pointer marked "device" is a CUDA device
 *     pointer owned by the caller (PyTorch's allocator in the Python host);
 *   - nothing here allocates, frees or synchronises: all work is enqueued on
 *     the given stream; scratch space is a caller-provided workspace whose size
 *     comes from the matching *_workspace_bytes();
 *   - return value 0 = CRAG_OK, negative = error; crag_last_error() returns the
 *     calling thread's message.  No C++ exception crosses the boundary;
 *   - re-entrant: concurrent calls from different host threads on different
 *     streams are safe (the reference calls in from up to 16 threads,
 *     ComoRAG.py:436-441).
 */
#ifndef COMORAG_B200_H_
#define COMORAG_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define CRAG_API __attribute__((visibility("default")))
#else
#define CRAG_API
#endif

#define CRAG_OK 0
#define CRAG_ERR_INVALID (-1)   /* bad argument (shape, alignment, null) */
#define CRAG_ERR_CUDA (-2)      /* a CUDA runtime/driver call failed */
#define CRAG_ERR_WORKSPACE (-3) /* workspace too small */
#define CRAG_ERR_UNSUPPORTED (-4)

/* Opaque CUDA stream handle (cudaStream_t). */
typedef void* crag_stream_t;

/* Library ABI version (major*1000 + minor). */
CRAG_API int crag_version(void);
/* Message for the last failing call made by the calling thread ("" if none). */
CRAG_API const char* crag_last_error(void);
/* Number of SMs of the current device (132 on H100 SXM); <0 on error. */
CRAG_API int crag_sm_count(void);

/* Growable device buffer for a corpus shard that is appended to (EmbeddingStore.insert_strings, embedding_store.py:63-90):
 * virtual address space is reserved once, physical memory is mapped behind it as rows arrive, so growth neither copies
 * the shard nor moves it (tensor maps and captured graphs stay valid).  Sizes are multiples of *granularity_out.
 *   crag_vmem_reserve  reserve >= max_bytes of address space on the current device -> base address, granularity
 *   crag_vmem_grow     back [mapped_bytes, new_mapped_bytes) of that range with device memory (read/write)
 *   crag_vmem_release  unmap [0, mapped_bytes) and free the reservation (caller has synchronised the device) */
CRAG_API int crag_vmem_reserve(size_t max_bytes, uint64_t* base_out, size_t* granularity_out);
CRAG_API int crag_vmem_grow(uint64_t base, size_t mapped_bytes, size_t new_mapped_bytes);
CRAG_API int crag_vmem_release(uint64_t base, size_t mapped_bytes, size_t reserved_bytes);

/* ------------------------------------------------------------------ search
 * Fused brute-force inner-product top-k over one corpus shard.
 *
 * Replaces, for a batch of nq queries at once, the reference's per-query
 *     scores = np.dot(E, q.T); scores = min_max_normalize(scores);
 *     order  = np.argsort(scores)[::-1]            (ComoRAG.py:950-967,
 *                                                   ComoRAG.py:937-948 + :475,
 *                                                   embed_utils.py:153-158)
 * without materialising the [nq, n_rows] score matrix: each query gets its k
 * best rows (raw inner products, descending; equal scores ordered by ascending
 * row id) plus the global (min, max) over ALL n_rows scores, from which the
 * reference's min-max-normalised score of any survivor is
 * (s - min) / (max - min)  (misc_utils.py:141-150).
 *
 *   corpus      device, bf16 [n_rows, dim] row-major, row stride
 *               corpus_row_stride elements (>= dim, multiple of 8), 16-B aligned
 *   n_rows      rows in this shard, 0 <= n_rows < 2^31
 *   dim         embedding width, multiple of 64, 64 <= dim <= 1024
 *   row_offset  added to local row indices to form the ids written out
 *               (the shard's first global row; 0 for an unsharded index)
 *   queries     device, bf16 [nq, dim] row-major contiguous, 16-B aligned
 *   nq          number of queries, >= 1 (processed 32 per corpus pass)
 *   k           1 <= k <= 128
 *   out_ids     device, int64 [nq, k]; -1 where fewer than k rows exist
 *   out_scores  device, fp32  [nq, k]; -inf where fewer than k rows exist
 *   out_minmax  device, fp32  [nq, 2] = (min, max) over the shard's scores;
 *               (+inf, -inf) for an empty shard.  May be NULL.
 *   workspace   device scratch of >= crag_search_workspace_bytes(nq, k) bytes,
 *               256-B aligned
 */
CRAG_API size_t crag_search_workspace_bytes(int nq, int k);
CRAG_API int crag_search_topk(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride, int64_t row_offset,
                     const void* queries, int nq, int k, int64_t* out_ids, float* out_scores, float* out_minmax,
                     void* workspace, size_t workspace_bytes, crag_stream_t stream);

/* Rank continuation ("search after") for k > 128 -- e.g. the reference's retrieve_knn with k = 2047
 * (embed_utils.py:8-97, ComoRAG.py:670-684).  after_keys[q] (device u64 [nq], or NULL for "from the top") is the
 * opaque position returned in last_keys by the previous call for the same queries over the same shard; only rows
 * ranking strictly after it are admitted, so ceil(K/128) calls return ranks [0,128), [128,256), ... exactly.
 * last_keys[q] is 0 once the shard is exhausted (further calls return ids -1).  Positions are shard-local. */
CRAG_API int crag_search_topk_after(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride,
                                    int64_t row_offset, const void* queries, int nq, int k, const uint64_t* after_keys,
                                    int64_t* out_ids, float* out_scores, float* out_minmax, uint64_t* last_keys,
                                    void* workspace, size_t workspace_bytes, crag_stream_t stream);

/* Exact top-k for large k and/or many queries: per chunk of queries one wgmma GEMM writes the fp32 score block
 * [q_chunk, round_up(n_rows, 4)] into the workspace, then one CTA per query radix-selects its k best.
 * Same argument rules and the same output contract as crag_search_topk (score desc, ties by ascending row, -1/-inf
 * past n_rows, minmax over all rows), except 1 <= k <= 2048.  q_chunk = workspace_bytes / per-query bytes (>= 1,
 * else CRAG_ERR_WORKSPACE); the call loops over chunks.  The self-join of the reference's add_synonymy_edges
 * (ComoRAG.py:670-684 -> retrieve_knn, embed_utils.py:8-97, k = 2047) is one GEMM per chunk instead of
 * ceil(nq/32) * ceil(k/128) passes over the shard.  Workspace 256-B aligned; crag_knn_workspace_bytes(n_rows, q)
 * is the size that holds q queries' score rows. */
CRAG_API size_t crag_knn_workspace_bytes(int64_t n_rows, int q_chunk);
CRAG_API int crag_knn_topk(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride, int64_t row_offset,
                           const void* queries, int nq, int k, int64_t* out_ids, float* out_scores, float* out_minmax,
                           void* workspace, size_t workspace_bytes, crag_stream_t stream);

/* The two halves of crag_search_topk for ONE pass (nq <= 32), exported so a caller can time or overlap them:
 * crag_search_scan streams the shard once and leaves per-CTA partial lists in the workspace;
 * crag_search_finalize merges them into (ids, scores, minmax).  Same argument rules as crag_search_topk. */
CRAG_API int crag_search_scan(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride,
                              const void* queries, int nq, int k, void* workspace, size_t workspace_bytes,
                              crag_stream_t stream);
CRAG_API int crag_search_finalize(const void* workspace, size_t workspace_bytes, int64_t n_rows, int nq, int k,
                                  int64_t row_offset, int64_t* out_ids, float* out_scores, float* out_minmax,
                                  crag_stream_t stream);

/* Merge `parts` per-shard results (the all-gathered output of
 * crag_search_topk on every rank, rank-major) into the global top-k.
 *
 * This is the exchange step the row-sharded index adds on top of the
 * reference (SURVEY.md section 8e); on one shard it is the identity.
 *
 *   scores  device fp32  [parts, nq, k]   ids  device int64 [parts, nq, k]
 *   minmax  device fp32  [parts, nq, 2]   (may be NULL together with out_minmax)
 * Invalid candidates are marked by id < 0.  Equal scores are ordered by
 * (part, position), which equals ascending global id when parts own ascending
 * contiguous row ranges.  k <= 128, parts * k <= 2^20.
 */
CRAG_API int crag_merge_topk(const float* scores, const int64_t* ids, const float* minmax, int parts, int nq, int k,
                    int64_t* out_ids, float* out_scores, float* out_minmax, crag_stream_t stream);

/* Same merge over PACKED per-shard records, the layout a single all-gather produces: record r (record_bytes apart,
 * multiple of 8) = [ids int64 nq*k][scores fp32 nq*k][minmax fp32 nq*2].  Lets every rank write its
 * crag_search_topk outputs as three views of one send buffer and merge the gathered buffer in place. */
CRAG_API int crag_merge_topk_packed(const void* records, int64_t record_bytes, int parts, int nq, int k,
                                    int64_t* out_ids, float* out_scores, float* out_minmax, crag_stream_t stream);

/* Row-sharded index, exchange step WITHOUT a collective-library launch (SURVEY.md section 8e): the per-shard
 * finalize, the cross-rank exchange and the global merge as ONE kernel over NVLink peer memory.  After
 * crag_search_scan on every rank (same query block, nq <= 32), every rank calls this with
 *   peer_bufs  device array [world] of pointers to each rank's exchange buffer as mapped in THIS process (symmetric
 *              memory: entry `rank` is the local buffer); each buffer is crag_exchange_buffer_bytes(world) bytes and
 *              zero-filled once before its first use
 *   epochs     device u64 [32], zero-filled once; counts calls per query slot (owned by the library afterwards)
 *   status     device int, set to 1 if a peer's record did not arrive within 4 s (outputs are then id -1 / -inf)
 * One CTA per query merges the shard's per-CTA partials, stores its k (id, score) pairs + (min, max) into every
 * rank's buffer, release-signals, waits for all ranks' records and merges them: every rank ends with the same
 * global (ids, scores, minmax) as crag_search_topk + all-gather + crag_merge_topk_packed would give.  A collective:
 * all ranks of the group must call it, in the same order, one call at a time per buffer. */
CRAG_API size_t crag_exchange_buffer_bytes(int world);
CRAG_API int crag_search_finalize_exchange(const void* workspace, size_t workspace_bytes, int64_t n_rows, int nq, int k,
                                           int64_t row_offset, const uint64_t* peer_bufs, int rank, int world,
                                           uint64_t* epochs, int* status, int64_t* out_ids, float* out_scores,
                                           float* out_minmax, crag_stream_t stream);

/* Score-all pass: raw inner products of EVERY shard row, for the reference's full-array contracts --
 *     query_fact_scores = np.dot(self.fact_embeddings, q.T)            (ComoRAG.py:944; get_fact_scores returns all
 *                                                                      N_f scores and callers index them, :475,:1054)
 *     query_doc_scores  = np.dot(self.passage_embeddings, q.T)         (ComoRAG.py:958-960)
 * The same TMA -> wgmma stream as crag_search_topk, but the select warps store the fp32 scores instead of
 * running the top-k selector.  out_scores device fp32, query q's row r at out_scores[q * out_ld + r]
 * (out_ld >= n_rows); out_minmax device fp32 [nq, 2] or NULL.  Other arguments and the workspace as
 * crag_search_topk (crag_search_workspace_bytes(nq, 1) bytes suffice). */
CRAG_API int crag_search_scores(const void* corpus, int64_t n_rows, int dim, int64_t corpus_row_stride,
                                const void* queries, int nq, float* out_scores, int64_t out_ld, float* out_minmax,
                                void* workspace, size_t workspace_bytes, crag_stream_t stream);

/* Full descending ranking of one score array on the device:
 *     sorted_doc_ids = np.argsort(query_doc_scores)[::-1]; sorted_doc_scores = query_doc_scores[sorted_doc_ids]
 * (ComoRAG.py:965-966; the whole permutation feeds the PPR reset weights, :1034-1042).  Stable LSD radix sort of
 * (score, row): equal scores keep ascending row order.  scores device fp32 [n] (typically one row of
 * crag_search_scores); out_ids device int64 [n]; out_scores device fp32 [n]; workspace >=
 * crag_rank_workspace_bytes(n) bytes, 256-B aligned; n < 2^31. */
CRAG_API size_t crag_rank_workspace_bytes(int64_t n);
CRAG_API int crag_rank_scores(const float* scores, int64_t n, int64_t* out_ids, float* out_scores, void* workspace,
                              size_t workspace_bytes, crag_stream_t stream);

/* Personalized PageRank, the solve of the reference's run_ppr (ComoRAG.py:1086-1105):
 *     graph.personalized_pagerank(directed=False, weights='weight', damping=d, reset=reset_prob)
 * on an undirected graph given in CSR "pull" form: row i lists every neighbour j once, ascending, with
 * coef = W_ij / s_j (W_ij = summed weight of the edges joining i and j, s_j = sum_i W_ij; no self-loops), and a
 * dangling vertex (s_j = 0, empty row) restarts by the reset.  The result is y_T / sum(y_T) of
 *     y_0 = (1 - d) v,   y_{t+1} = (1 - d) v + d A y_t          (t < T = iterations)
 * which is within 2 d^(T+1) / (1 - d) in L1 of the exact PPR (DESIGN.md section 2a).  fp32 arithmetic, merge-path
 * load balance over rows + nonzeros, no floating-point atomics: the same inputs give bit-identical output on every
 * run and stream.
 *   row_ptr device int64 [n_vertices + 1]; col device int32 [nnz]; coef device fp32 [nnz]; 1 <= n_vertices < 2^31
 *   reset device fp32 [n_vertices], >= 0, sum 1; damping in [0, 1); iterations T >= 0
 *   out_vertices device int32 [n_out], each in [0, n_vertices), or NULL with n_out = n_vertices (all vertices)
 *   out device fp32 [n_out]: out[p] = x[out_vertices[p]]
 *   workspace >= crag_ppr_workspace_bytes(n_vertices, nnz) bytes, 256-B aligned.
 * Enqueues 2T + 4 kernels. */
CRAG_API size_t crag_ppr_workspace_bytes(int64_t n_vertices, int64_t nnz);
CRAG_API int crag_ppr(const int64_t* row_ptr, const int32_t* col, const float* coef, int64_t n_vertices, int64_t nnz,
                      const float* reset, float damping, int iterations, const int32_t* out_vertices, int64_t n_out,
                      float* out, void* workspace, size_t workspace_bytes, crag_stream_t stream);

/* ------------------------------------------------------------------ encoder
 * Dense projection of the encoder forward (BGEEmbedding.py:120 runs it through
 * HF's BertModel: attention.self.{query,key,value}, attention.output.dense,
 * intermediate.dense (+ exact-erf GELU), output.dense), torch.nn.Linear layout:
 *
 *     out[m, n] = epilogue( sum_k a[m, k] * w[n, k] + bias[n] )
 *
 *   a         device bf16 [m, k], leading dimension lda (elements)
 *   w         device bf16 [n, k], leading dimension ldw
 *   bias      device fp32 [n]
 *   residual  device bf16 [m, n] (ldr), only for CRAG_GEMM_BIAS_RESIDUAL
 *   out       device bf16 [m, n] (ldo)
 * n, k, and all leading dimensions must be multiples of 8; pointers 16-B aligned.
 * Accumulation is fp32 on the wgmma tensor cores.
 */
#define CRAG_GEMM_BIAS 0          /* out = acc + bias */
#define CRAG_GEMM_BIAS_GELU 1     /* out = gelu_erf(acc + bias) */
#define CRAG_GEMM_BIAS_RESIDUAL 2 /* out = acc + bias + residual */
CRAG_API int crag_gemm_bf16(const void* a, int64_t lda, const void* w, int64_t ldw, const float* bias,
                            const void* residual, int64_t ldr, void* out, int64_t ldo, int m, int n, int k,
                            int epilogue, crag_stream_t stream);

/* IVF residual inner-product search (BASELINE config 4: "IVF-4096 coarse quantizer + fused residual-IP top-100").
 * The reference has no IVF / ANN code (faiss-cpu is pinned at requirements.txt:34 and never imported), so this
 * entry point replaces nothing of the reference's; its semantic is fixed by oracle/ivf_oracle.py.
 *
 * Shard layout (device): `residuals` bf16 [n_rows_padded, dim] = x - c_list grouped by coarse list, every list
 * padded with zero rows to whole 128-row tiles; list l owns tiles [list_tile_start[l], list_tile_start[l+1]) and
 * its first list_rows[l] rows are real; row_ids[stored row] = the row's original id (padding: -1).
 * The caller runs the coarse pass itself (crag_search_topk over the bf16 centroid table with k = nprobe) and
 * passes its output: probed_ids int64 [nq, nprobe] (-1 = absent), probed_scores fp32 [nq, nprobe] = q . c_list.
 * Per block of 32 queries: a plan kernel marks which queries probe which list and compacts the probed lists'
 * tiles into a work-list; the scan kernel (the flat kernel's TMA/wgmma/selector pipeline walking that work-list)
 * scores  q . c_list + q . residual  for the probing queries only; the per-CTA lists are merged and stored-row ids
 * mapped to original ids.  Outputs as crag_search_topk (min/max range over the probed rows).
 * workspace >= crag_ivf_workspace_bytes(nlist, total_tiles, k), 256-byte aligned. */
CRAG_API size_t crag_ivf_workspace_bytes(int nlist, int64_t total_tiles, int k);
CRAG_API int crag_ivf_search(const void* residuals, int64_t n_rows_padded, int dim, int64_t row_stride,
                             const int32_t* list_tile_start, const int32_t* list_rows, int nlist,
                             int64_t total_tiles, const int64_t* row_ids, const void* queries, int nq,
                             const int64_t* probed_ids, const float* probed_scores, int nprobe, int k,
                             int64_t* out_ids, float* out_scores, float* out_minmax, void* workspace,
                             size_t workspace_bytes, crag_stream_t stream);

/* IVF build, assignment step: best_id[r] = argmax_l bf16(row r) . bf16(centroid l) (fp32 accumulation on the tensor
 * cores, ties to the smaller l), best_score[r] = that inner product.  rows device bf16 [n_rows, dim] (row_stride
 * elements), centroids device bf16 [nlist, dim] contiguous; outputs device fp32 / int32 [n_rows].  nlist / 32 passes of
 * the scan kernel over the rows (centroids are its query blocks).  Workspace as crag_search_topk(nq = 32, k = 1). */
CRAG_API int crag_ivf_assign(const void* rows, int64_t n_rows, int dim, int64_t row_stride, const void* centroids,
                             int nlist, float* best_score, int32_t* best_id, void* workspace, size_t workspace_bytes,
                             crag_stream_t stream);

/* Encoder weights (BERT-family, post-LN; HF BertModel parameter names in
 * comments).  Matrices are device bf16 in torch.nn.Linear layout [out, in];
 * biases and LayerNorm parameters are device fp32.  The struct itself and the
 * layer table are HOST memory. */
typedef struct crag_encoder_layer {
  const void* w_qkv;   /* [3H, H]: attention.self.{query,key,value}.weight stacked */
  const float* b_qkv;  /* [3H] */
  const void* w_o;     /* [H, H]: attention.output.dense.weight */
  const float* b_o;    /* [H] */
  const float* ln1_g;  /* attention.output.LayerNorm.weight */
  const float* ln1_b;
  const void* w_ff1;   /* [I, H]: intermediate.dense.weight */
  const float* b_ff1;  /* [I] */
  const void* w_ff2;   /* [H, I]: output.dense.weight */
  const float* b_ff2;  /* [H] */
  const float* ln2_g;  /* output.LayerNorm.weight */
  const float* ln2_b;
} crag_encoder_layer;

typedef struct crag_encoder {
  int32_t hidden;        /* H: 64..1024, multiple of 8; H / heads in {32, 64} */
  int32_t n_layers;
  int32_t heads;
  int32_t intermediate;  /* I */
  int32_t vocab;
  int32_t max_pos;       /* rows of the position table */
  int32_t pos_offset;    /* 0 for BERT, padding_idx + 1 (= 2) for XLM-R */
  float ln_eps;          /* 1e-12 for BERT */
  const void* word_emb;  /* bf16 [vocab, H] */
  const void* pos_emb;   /* bf16 [max_pos, H] */
  const void* type_emb;  /* bf16 [>=1, H]; row 0 is used (token_type_ids == 0) */
  const float* emb_ln_g;
  const float* emb_ln_b;
  const crag_encoder_layer* layers; /* host array [n_layers] */
} crag_encoder;

/* Encoder forward + masked mean pool + L2 normalise for a packed batch.
 *
 * Replaces BGEEmbeddingModel._encode's device work (BGEEmbedding.py:119-127):
 * outputs = model(**inputs); mean_pooling(last_hidden_state, attention_mask)
 * (BGEEmbedding.py:15-28); F.normalize(p=2, dim=1).  Sequences are packed
 * without padding: token_ids[total_tokens], sequence i owns
 * [cu_seqlens[i], cu_seqlens[i+1]).
 *
 *   token_ids    device int32 [total_tokens]
 *   cu_seqlens   device int32 [n_seqs + 1], cu_seqlens[0] = 0
 *   max_seqlen   longest sequence in the batch (host value, sizes the grid)
 *   normalize    1 = L2-normalise rows (the reference default), 0 = raw mean
 *   out_f32      device fp32 [n_seqs, H] or NULL
 *   out_bf16     device bf16 rows with stride out_bf16_stride elements, or NULL
 *                (lets index build write straight into the corpus shard)
 *   workspace    >= crag_encoder_workspace_bytes(model, total_tokens), 256-B aligned
 */
CRAG_API size_t crag_encoder_workspace_bytes(const crag_encoder* model, int total_tokens);
CRAG_API int crag_encoder_forward(const crag_encoder* model, const int32_t* token_ids, const int32_t* cu_seqlens,
                                  int n_seqs, int total_tokens, int max_seqlen, int normalize, float* out_f32,
                                  void* out_bf16, int64_t out_bf16_stride, void* workspace, size_t workspace_bytes,
                                  crag_stream_t stream);

/* Cross-encoder rerank score (BASELINE config 5: bge-reranker-large behind the DSPyFilter call surface,
 * rerank.py:97-123 -- the reference's filter is an LLM prompt, so the arithmetic here follows the published
 * XLMRobertaForSequenceClassification forward instead: encoder layers, then on each sequence's FIRST token
 * logits = out_proj(tanh(dense(h))) ).  Weights: device bf16 [out, in]; biases device fp32. */
typedef struct crag_classifier_head {
  const void* w_dense;   /* [H, H]: classifier.dense.weight */
  const float* b_dense;  /* [H] */
  const void* w_out;     /* [n_labels, H]: classifier.out_proj.weight */
  const float* b_out;    /* [n_labels] */
  int32_t n_labels;      /* 1 for bge-reranker-* */
} crag_classifier_head;

/* Packed (query, passage) token sequences -> logits fp32 [n_seqs, n_labels] on the device.  Batch arguments and
 * workspace as crag_encoder_forward. */
CRAG_API int crag_encoder_classify(const crag_encoder* model, const crag_classifier_head* head,
                                   const int32_t* token_ids, const int32_t* cu_seqlens, int n_seqs, int total_tokens,
                                   int max_seqlen, float* logits, void* workspace, size_t workspace_bytes,
                                   crag_stream_t stream);

/* K3 on its own: masked mean pool + optional L2 normalise of a packed
 * last_hidden_state (bf16 [total_tokens, hidden_size]); mean_pooling
 * (BGEEmbedding.py:15-28) + F.normalize (:127). */
CRAG_API int crag_pool_normalize(const void* hidden, const int32_t* cu_seqlens, int n_seqs, int hidden_size,
                                 int normalize, float* out_f32, void* out_bf16, int64_t out_bf16_stride,
                                 crag_stream_t stream);

/* K2 on its own: varlen multi-head self-attention over a packed batch, as HF's
 * BertSelfAttention computes it (softmax(q k^T / sqrt(dh)) v, keys restricted
 * to the token's own sequence == the reference's key-padding mask).
 *   qkv  device bf16 [total_tokens, 3*hidden] = [q | k | v], heads contiguous
 *   ctx  device bf16 [total_tokens, hidden]
 * hidden/heads must be 32 or 64. */
CRAG_API int crag_attention_varlen(const void* qkv, const int32_t* cu_seqlens, int n_seqs, int max_seqlen,
                                   int hidden_size, int heads, void* ctx, crag_stream_t stream);

/* The same attention on the wgmma tensor cores (head dim 64 only): S = Q K^T and O += P V as wgmma tiles with
 * register accumulators, Q/K/V staged by TMA.  total_tokens = rows of qkv (sizes the TMA tensor map). */
CRAG_API int crag_attention_varlen_tc(const void* qkv, const int32_t* cu_seqlens, int n_seqs, int total_tokens,
                                      int max_seqlen, int hidden_size, int heads, void* ctx, crag_stream_t stream);

/* torch.nn.LayerNorm over the last dimension, bf16 in/out, fp32 statistics
 * (BertSelfOutput / BertOutput LayerNorm). hidden_size <= 1024, multiple of 8. */
CRAG_API int crag_layernorm(const void* in, int rows, int hidden_size, const float* gamma, const float* beta,
                            float eps, void* out, crag_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* COMORAG_B200_H_ */
