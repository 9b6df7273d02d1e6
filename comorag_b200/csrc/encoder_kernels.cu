// Non-GEMM kernels of the encoder forward (BGEEmbedding.py:92-129 =
// HF BertModel forward -> mean_pooling (BGEEmbedding.py:15-28) ->
// F.normalize (:127)), operating on the UNPADDED token stream: sequences are
// packed back to back ([T, H], T = sum of lengths, cu_seqlens[n+1]), which is
// arithmetically identical to the reference's pad-to-longest + attention-mask
// because padded keys get -inf logits and padded rows are dropped by the
// masked mean.
//
//   embed_layernorm   word+position+token_type(0) embedding gather + LayerNorm
//   layernorm         LayerNorm as its OWN pass over the [T, H] activation the
//                     residual GEMM wrote (bias + residual are fused in that
//                     GEMM's epilogue, the normalisation is not: a row spans
//                     four 256-column GEMM tiles); fp32 statistics, bf16 in/out
//   attention         varlen multi-head self-attention, flash-style online
//                     softmax, mma.sync m16n8k16 bf16 tiles: head dim 32
//                     (bge-small) only -- head dim 64 runs attention_tc.cu on
//                     wgmma
//   pool_normalize    K3: masked mean over tokens + L2 normalise, writes fp32
//                     [n, H] for the host API and (optionally) the bf16 row
//                     straight into the corpus shard
#include <cuda_bf16.h>

#include "common.cuh"
#include "encoder.cuh"
#include "encoder_simt.cuh"

namespace crag {

// --------------------------------------------------------------- attention
__device__ __forceinline__ void cp_async_16(void* smem_dst, const void* gmem_src, bool valid) {
  const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
  const int sz = valid ? 16 : 0;  // src-size 0 => zero fill
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gmem_src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* p) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* p) {
  const uint32_t a = static_cast<uint32_t>(__cvta_generic_to_shared(p));
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(a));
}
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// smem tile: ROWS x DH bf16, row = DH*2 bytes split into 16-byte chunks, chunk index XOR-swizzled with
// the row so that ldmatrix (8 rows x 16 B) is bank-conflict free.
template <int DH>
__device__ __forceinline__ __nv_bfloat16* tile_ptr(__nv_bfloat16* base, int row, int chunk) {
  constexpr int CPR = DH / 8;  // 16-byte chunks per row
  return base + row * DH + ((chunk ^ (row & (CPR - 1) & 7)) * 8);
}

template <int DH>
__device__ __forceinline__ void load_tile_async(__nv_bfloat16* smem_tile, const __nv_bfloat16* __restrict__ gbase,
                                                int64_t row_stride, int row0, int rows_valid, int tid) {
  constexpr int CPR = DH / 8;
  constexpr int CHUNKS = 64 * CPR;
#pragma unroll
  for (int i = 0; i < CHUNKS / 128; ++i) {
    const int c = tid + i * 128;
    const int row = c / CPR, chunk = c % CPR;
    const bool valid = row0 + row < rows_valid;
    const __nv_bfloat16* src = gbase + int64_t(valid ? row0 + row : 0) * row_stride + chunk * 8;
    cp_async_16(tile_ptr<DH>(smem_tile, row, chunk), src, valid);
  }
}

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// grid = (ceil(max_len / (64*MT)), heads, n_seqs), block = 128: 4 warps x MT m-tiles of 16 query rows.
// MT = 2 halves the K/V fragment (ldmatrix) traffic per flop, which co-limits the kernel with the legacy HMMA pipe.
template <int DH, int MT>
__global__ void __launch_bounds__(128) attention_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                        const int32_t* __restrict__ cu_seqlens, int H,
                                                        float scale_log2e, __nv_bfloat16* __restrict__ ctx) {
  constexpr int BM = 64 * MT;
  __shared__ __align__(128) __nv_bfloat16 sQ[BM * DH];
  __shared__ __align__(128) __nv_bfloat16 sK[2][64 * DH];
  __shared__ __align__(128) __nv_bfloat16 sV[2][64 * DH];

  const int seq = blockIdx.z, head = blockIdx.y;
  const int start = __ldg(cu_seqlens + seq);
  const int L = __ldg(cu_seqlens + seq + 1) - start;
  const int q0 = blockIdx.x * BM;
  if (q0 >= L) return;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int64_t ld = 3 * int64_t(H);
  const __nv_bfloat16* qbase = qkv + int64_t(start) * ld + head * DH;
  const __nv_bfloat16* kbase = qbase + H;
  const __nv_bfloat16* vbase = qbase + 2 * H;
  const int n_kv = (L + 63) / 64;

#pragma unroll
  for (int mt = 0; mt < MT; ++mt) load_tile_async<DH>(sQ + mt * 64 * DH, qbase, ld, q0 + mt * 64, L, tid);
  load_tile_async<DH>(sK[0], kbase, ld, 0, L, tid);
  load_tile_async<DH>(sV[0], vbase, ld, 0, L, tid);
  cp_async_commit();

  constexpr int KS = DH / 16;  // k-steps over the head dim
  constexpr int NT = DH / 8;   // output n-tiles over the head dim
  uint32_t qf[MT][KS][4];
  float o[MT][NT][4];
  float m_run[MT][2], l_run[MT][2];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
    for (int n = 0; n < NT; ++n) o[mt][n][0] = o[mt][n][1] = o[mt][n][2] = o[mt][n][3] = 0.f;
    m_run[mt][0] = m_run[mt][1] = -INFINITY;
    l_run[mt][0] = l_run[mt][1] = 0.f;
  }

  for (int j = 0; j < n_kv; ++j) {
    const int buf = j & 1;
    if (j + 1 < n_kv) {
      load_tile_async<DH>(sK[buf ^ 1], kbase, ld, (j + 1) * 64, L, tid);
      load_tile_async<DH>(sV[buf ^ 1], vbase, ld, (j + 1) * 64, L, tid);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (j == 0) {
      // warp w owns query rows [w*16*MT, (w+1)*16*MT) of the CTA tile
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int ks = 0; ks < KS; ++ks)
          ldmatrix_x4(qf[mt][ks], tile_ptr<DH>(sQ, (warp * MT + mt) * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, ks * 2 + (lane >> 4)));
    }
    // S = Q K^T : (16*MT) x 64 per warp
    float s[MT][8][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
      for (int n = 0; n < 8; ++n) s[mt][n][0] = s[mt][n][1] = s[mt][n][2] = s[mt][n][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {  // pairs of key n-tiles
        uint32_t kf[4];
        // matrices: (keys np*16+0..7, d ks*16+0..7), (same keys, d +8), (keys +8, d 0..7), (keys +8, d +8)
        ldmatrix_x4(kf, tile_ptr<DH>(sK[buf], np * 16 + (lane & 7) + (lane >> 4) * 8, ks * 2 + ((lane >> 3) & 1)));
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          mma_bf16_16816(s[mt][np * 2], qf[mt][ks], kf[0], kf[1]);
          mma_bf16_16816(s[mt][np * 2 + 1], qf[mt][ks], kf[2], kf[3]);
        }
      }
    }
    // mask keys beyond the sequence, online softmax (base-2 domain)
    const int kbase_idx = j * 64;
    const bool ragged = kbase_idx + 64 > L;
    uint32_t pf[MT][4][4];  // P as A fragments: 4 k-steps of 16 keys
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
      float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
      for (int n = 0; n < 8; ++n) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float v = s[mt][n][e] * scale_log2e;
          if (ragged && kbase_idx + n * 8 + t4 * 2 + (e & 1) >= L) v = -INFINITY;
          s[mt][n][e] = v;
        }
        mx0 = fmaxf(mx0, fmaxf(s[mt][n][0], s[mt][n][1]));
        mx1 = fmaxf(mx1, fmaxf(s[mt][n][2], s[mt][n][3]));
      }
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
      const float nm0 = fmaxf(m_run[mt][0], mx0), nm1 = fmaxf(m_run[mt][1], mx1);  // finite: >= 1 valid key per tile
      const float c0 = fast_exp2(m_run[mt][0] - nm0), c1 = fast_exp2(m_run[mt][1] - nm1);
      m_run[mt][0] = nm0;
      m_run[mt][1] = nm1;
      float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const float p0 = fast_exp2(s[mt][n][0] - nm0), p1 = fast_exp2(s[mt][n][1] - nm0);
        const float p2 = fast_exp2(s[mt][n][2] - nm1), p3 = fast_exp2(s[mt][n][3] - nm1);
        rs0 += p0 + p1;
        rs1 += p2 + p3;
        __nv_bfloat162 lo = __floats2bfloat162_rn(p0, p1), hi = __floats2bfloat162_rn(p2, p3);
        pf[mt][n >> 1][(n & 1) * 2 + 0] = *reinterpret_cast<uint32_t*>(&lo);
        pf[mt][n >> 1][(n & 1) * 2 + 1] = *reinterpret_cast<uint32_t*>(&hi);
      }
      l_run[mt][0] = l_run[mt][0] * c0 + rs0;
      l_run[mt][1] = l_run[mt][1] * c1 + rs1;
#pragma unroll
      for (int n = 0; n < NT; ++n) {
        o[mt][n][0] *= c0; o[mt][n][1] *= c0; o[mt][n][2] *= c1; o[mt][n][3] *= c1;
      }
    }
    // O += P V
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {  // 16 keys per step
#pragma unroll
      for (int dp = 0; dp < NT / 2; ++dp) {  // pairs of d n-tiles
        uint32_t vf[4];
        // .trans matrices: (keys kk*16+0..7, d dp*16+0..7), (keys +8, same d), (keys 0..7, d +8), (keys +8, d +8)
        ldmatrix_x4_trans(vf, tile_ptr<DH>(sV[buf], kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, dp * 2 + (lane >> 4)));
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
          mma_bf16_16816(o[mt][dp * 2], pf[mt][kk], vf[0], vf[1]);
          mma_bf16_16816(o[mt][dp * 2 + 1], pf[mt][kk], vf[2], vf[3]);
        }
      }
    }
    __syncthreads();  // all warps done with buf before it is refilled
  }
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
    float l0 = l_run[mt][0], l1 = l_run[mt][1];  // row sums live distributed over the 4 lanes of a quad
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
    l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float inv0 = 1.f / l0, inv1 = 1.f / l1;
    const int r0 = q0 + (warp * MT + mt) * 16 + g, r1 = r0 + 8;
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      const int col = head * DH + n * 8 + t4 * 2;
      if (r0 < L)
        *reinterpret_cast<__nv_bfloat162*>(ctx + int64_t(start + r0) * H + col) = __floats2bfloat162_rn(o[mt][n][0] * inv0, o[mt][n][1] * inv0);
      if (r1 < L)
        *reinterpret_cast<__nv_bfloat162*>(ctx + int64_t(start + r1) * H + col) = __floats2bfloat162_rn(o[mt][n][2] * inv1, o[mt][n][3] * inv1);
    }
  }
}

// -------------------------------------------------------------- launchers
int launch_embed_layernorm(const int32_t* token_ids, const int32_t* cu_seqlens, int n_seqs, int T, int H, int vocab,
                           int max_pos, int pos_offset, const void* word_emb, const void* pos_emb,
                           const void* type_emb, const float* gamma, const float* beta, float eps, void* out,
                           cudaStream_t stream) {
  if (T <= 0) return CRAG_OK;
  const int grid = (T + 3) / 4;
  const auto* we = static_cast<const __nv_bfloat16*>(word_emb);
  const auto* pe = static_cast<const __nv_bfloat16*>(pos_emb);
  const auto* te = static_cast<const __nv_bfloat16*>(type_emb);
  auto* o = static_cast<__nv_bfloat16*>(out);
  const int vpl = (H / 8 + 31) / 32;
  if (vpl <= 1) embed_layernorm_kernel<1><<<grid, 128, 0, stream>>>(token_ids, cu_seqlens, n_seqs, T, H, vocab, max_pos, pos_offset, we, pe, te, gamma, beta, eps, o);
  else if (vpl <= 2) embed_layernorm_kernel<2><<<grid, 128, 0, stream>>>(token_ids, cu_seqlens, n_seqs, T, H, vocab, max_pos, pos_offset, we, pe, te, gamma, beta, eps, o);
  else if (vpl <= 4) embed_layernorm_kernel<4><<<grid, 128, 0, stream>>>(token_ids, cu_seqlens, n_seqs, T, H, vocab, max_pos, pos_offset, we, pe, te, gamma, beta, eps, o);
  else return fail(CRAG_ERR_UNSUPPORTED, "hidden size %d > 1024 not supported", H);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

int launch_layernorm(const void* in, int T, int H, const float* gamma, const float* beta, float eps, void* out,
                     cudaStream_t stream) {
  if (T <= 0) return CRAG_OK;
  const int grid = (T + 3) / 4;
  const auto* i = static_cast<const __nv_bfloat16*>(in);
  auto* o = static_cast<__nv_bfloat16*>(out);
  const int vpl = (H / 8 + 31) / 32;
  if (vpl <= 1) layernorm_kernel<1><<<grid, 128, 0, stream>>>(i, T, H, gamma, beta, eps, o);
  else if (vpl <= 2) layernorm_kernel<2><<<grid, 128, 0, stream>>>(i, T, H, gamma, beta, eps, o);
  else if (vpl <= 4) layernorm_kernel<4><<<grid, 128, 0, stream>>>(i, T, H, gamma, beta, eps, o);
  else return fail(CRAG_ERR_UNSUPPORTED, "hidden size %d > 1024 not supported", H);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

int launch_attention(const void* qkv, const int32_t* cu_seqlens, int n_seqs, int max_len, int H, int heads, void* ctx,
                     cudaStream_t stream) {
  if (n_seqs <= 0 || max_len <= 0) return CRAG_OK;
  const int dh = H / heads;
  const float scale_log2e = 1.4426950408889634f / sqrtf(float(dh));
  const auto* q = static_cast<const __nv_bfloat16*>(qkv);
  auto* c = static_cast<__nv_bfloat16*>(ctx);
  if (dh != 64 && dh != 32) return fail(CRAG_ERR_UNSUPPORTED, "head dim %d not supported (32 or 64)", dh);
  if (max_len > 64) {  // 128-query tiles: 2 m-tiles per warp
    const dim3 grid((max_len + 127) / 128, heads, n_seqs);
    if (dh == 64) attention_kernel<64, 2><<<grid, 128, 0, stream>>>(q, cu_seqlens, H, scale_log2e, c);
    else attention_kernel<32, 2><<<grid, 128, 0, stream>>>(q, cu_seqlens, H, scale_log2e, c);
  } else {
    const dim3 grid(1, heads, n_seqs);
    if (dh == 64) attention_kernel<64, 1><<<grid, 128, 0, stream>>>(q, cu_seqlens, H, scale_log2e, c);
    else attention_kernel<32, 1><<<grid, 128, 0, stream>>>(q, cu_seqlens, H, scale_log2e, c);
  }
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

int launch_pool_normalize(const void* hidden, const int32_t* cu_seqlens, int n_seqs, int H, int normalize,
                          float* out_f32, void* out_bf16, int64_t out_bf16_stride, cudaStream_t stream) {
  if (n_seqs <= 0) return CRAG_OK;
  if (H > 2048) return fail(CRAG_ERR_UNSUPPORTED, "hidden size %d > 2048 not supported", H);
  const auto smem_bytes = [](int h) { return (size_t(kPoolGroups) * h + 4) * sizeof(float); };
  const int rc = allow_dynamic_smem<pool_normalize_kernel>(smem_bytes(2048));
  if (rc != CRAG_OK) return rc;
  const size_t smem = smem_bytes(H);
  pool_normalize_kernel<<<n_seqs, 128 * kPoolGroups, smem, stream>>>(static_cast<const __nv_bfloat16*>(hidden), cu_seqlens, H,
                                                                     normalize, out_f32, static_cast<__nv_bfloat16*>(out_bf16),
                                                                     out_bf16_stride);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

int launch_cls_head(const void* hidden, const int32_t* cu_seqlens, int n_seqs, int H, const void* w_dense,
                    const float* b_dense, const void* w_out, const float* b_out, int n_labels, float* logits,
                    cudaStream_t stream) {
  if (n_seqs <= 0) return CRAG_OK;
  if (H > 1024 || H % 8) return fail(CRAG_ERR_UNSUPPORTED, "classifier head: hidden size %d unsupported (<= 1024, multiple of 8)", H);
  if (n_labels < 1) return fail(CRAG_ERR_INVALID, "classifier head: n_labels %d", n_labels);
  cls_head_kernel<<<n_seqs, 32 * kClsWarps, 0, stream>>>(static_cast<const __nv_bfloat16*>(hidden), cu_seqlens, H,
                                                         static_cast<const __nv_bfloat16*>(w_dense), b_dense,
                                                         static_cast<const __nv_bfloat16*>(w_out), b_out, n_labels, logits);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

}  // namespace crag
