// K1: bf16 x bf16 -> fp32 GEMM on Hopper wgmma tensor cores with fused epilogues,
// the dense contractions of the encoder forward the reference runs through
// `self.embedding_model(**inputs)` (BGEEmbedding.py:120): QKV, attention-output,
// FFN-up (+GELU) and FFN-down projections of every BERT layer.
//
//   out[M, N] = epilogue( A[M, K] . W[N, K]^T + bias[N] )      (torch Linear layout)
//
// One CTA per 128 x 128 output tile, two CTAs per SM (288 threads each):
//   warps 0-7  two consumer warpgroups, 64 rows each: wgmma m64n128k16 from the
//              swizzled smem stages into fp32 register accumulators, then the
//              epilogue (+bias, optional exact GELU or residual add, bf16 stores)
//   warp 8     TMA producer: A box 128x64, W box 128x64 (128-byte swizzle)
//              through a STAGES-deep mbarrier ring
// With two CTAs resident, one CTA's epilogue overlaps the other's main loop.
// A fourth, internal epilogue (GEMM_EPI_SCORES_F32, gemm_scores_f32) stores the raw fp32 accumulators: the score
// block Q . X^T of crag_knn_topk (search.cu), on a 1-D grid with the query blocks fastest.
#include <cstdlib>

#include "common.cuh"
#include "gemm.cuh"
#include "ptx.cuh"

namespace crag {

constexpr int kGemmBM = 128;
constexpr int kGemmBN = 128;
constexpr int kGemmBK = 64;
constexpr int kGemmConsumerWarps = 8;
constexpr int kGemmThreads = 32 * kGemmConsumerWarps + 32;
// 3 stages of 32 KB: two CTAs (2 x 97 KB) fit in an SM's 228 KB of shared memory
constexpr int kGemmStages = 3;

struct GemmLayout {
  static constexpr int kABytes = kGemmBM * kGemmBK * 2;  // 16 KB
  static constexpr int kBBytes = kGemmBN * kGemmBK * 2;  // 16 KB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr size_t smem_bytes() { return 1024 + size_t(kGemmStages) * kStageBytes + 2 * kGemmStages * 8; }
};

// Exact-erf GELU (HF "gelu"), erf by Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, far below the bf16 output's
// resolution): ~16 instructions with two MUFU ops instead of erff()'s ~30, which keeps the FFN-up epilogue under the
// tile's MMA time (the epilogue is issue-slot bound: 32 thread-instructions per output element per tile at K=1024).
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = x * 0.70710678118654752f;
  const float az = fabsf(z);
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, az, 1.0f)));
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  p *= t;
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(az * az * -1.4426950408889634f));
  const float erf_abs = fmaf(-p, e, 1.0f);          // erf(|z|)
  const float half_x = 0.5f * x;
  return fmaf(half_x, copysignf(erf_abs, z), half_x);  // 0.5 x (1 + erf(z))
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

template <int EPI>
__global__ void __launch_bounds__(kGemmThreads, 2)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b, int M, int N,
                 int K, const float* __restrict__ bias, const __nv_bfloat16* __restrict__ residual, int64_t ldr,
                 __nv_bfloat16* __restrict__ out, int64_t ldo) {
  using L = GemmLayout;
  constexpr int STAGES = kGemmStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(smem + STAGES * L::kStageBytes);
  uint64_t* bar_empty = bar_full + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  int n_blk = blockIdx.x, m_blk = blockIdx.y;
  if constexpr (EPI == GEMM_EPI_SCORES_F32) {
    // 1-D grid with the query blocks fastest: the CTAs in flight share a few corpus tiles and the chunk's queries
    // stay in L2, so the corpus is read from HBM once per chunk (and N may exceed gridDim.y's 65535 tiles)
    const int m_blocks = (M + kGemmBM - 1) / kGemmBM;
    m_blk = int(blockIdx.x % unsigned(m_blocks));
    n_blk = int(blockIdx.x / unsigned(m_blocks));
  }
  const int num_kb = (K + kGemmBK - 1) / kGemmBK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&bar_full[s], 1);
      mbar_init(&bar_empty[s], kGemmConsumerWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kGemmConsumerWarps) {
    // ================================================================ producer
    if (lane == 0) {
      tma_prefetch_desc(&tm_a);
      tma_prefetch_desc(&tm_b);
      const uint64_t pol_w = policy_evict_last();
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&bar_empty[stage], phase ^ 1);
        uint8_t* sa = smem + stage * L::kStageBytes;
        mbar_arrive_expect_tx(&bar_full[stage], L::kStageBytes);
        tma_load_2d(&tm_a, &bar_full[stage], sa, kb * kGemmBK, m_blk * kGemmBM);
        tma_load_2d_hint(&tm_b, &bar_full[stage], sa + L::kABytes, kb * kGemmBK, n_blk * kGemmBN, pol_w);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ================================================ consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile
  const int wg = warp >> 2;
  float acc[kGemmBN / 2];
#pragma unroll
  for (int i = 0; i < kGemmBN / 2; ++i) acc[i] = 0.f;
  int stage = 0, prev = 0;
  uint32_t phase = 0;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait(&bar_full[stage], phase);
    const uint32_t a_addr = smem_u32(smem + stage * L::kStageBytes) + wg * 64 * 128;
    const uint32_t b_addr = smem_u32(smem + stage * L::kStageBytes + L::kABytes);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kGemmBK / 16; ++ks)
      wgmma_m64n128k16_ss(acc, wgmma_desc_sw128(a_addr + ks * 32), wgmma_desc_sw128(b_addr + ks * 32), 1u);
    wgmma_commit();
    wgmma_wait<1>();  // k-block kb - 1 has retired: its stage goes back to the producer
    if (kb > 0 && lane == 0) mbar_arrive(&bar_empty[prev]);
    prev = stage;
    if (++stage == STAGES) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);

  if constexpr (EPI == GEMM_EPI_SCORES_F32) {
    // fp32 scores straight from the accumulator fragment, no bias; `out` carries the fp32 block.  N may be odd, so
    // each element of a pair is guarded on its own
    float* outf = reinterpret_cast<float*>(out);
    const int srow0 = m_blk * kGemmBM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int scol0 = n_blk * kGemmBN + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < kGemmBN / 8; ++j) {
      const int col = scol0 + 8 * j;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = srow0 + 8 * h;
        if (row >= M) continue;
        float* p = outf + int64_t(row) * ldo + col;
        if (col + 1 < N) *reinterpret_cast<float2*>(p) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        else if (col < N) p[0] = acc[4 * j + 2 * h];
      }
    }
    return;
  }

  // epilogue: bias (+GELU | +residual), bf16 pairs straight from the accumulator fragment
  const int row0 = m_blk * kGemmBM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const int col0 = n_blk * kGemmBN + 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < kGemmBN / 8; ++j) {
    const int col = col0 + 8 * j;
    if (col >= N) continue;
    const float2 b = __ldg(reinterpret_cast<const float2*>(bias + col));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 8 * h;
      if (row >= M) continue;
      float x0 = acc[4 * j + 2 * h] + b.x, x1 = acc[4 * j + 2 * h + 1] + b.y;
      if (EPI == GEMM_EPI_BIAS_GELU) {
        x0 = gelu_erf(x0);
        x1 = gelu_erf(x1);
      }
      if (EPI == GEMM_EPI_BIAS_RESIDUAL) {
        const __nv_bfloat162 r = *reinterpret_cast<const __nv_bfloat162*>(residual + int64_t(row) * ldr + col);
        x0 += __bfloat162float(r.x);
        x1 += __bfloat162float(r.y);
      }
      *reinterpret_cast<uint32_t*>(out + int64_t(row) * ldo + col) = pack_bf16x2(x0, x1);
    }
  }
}

template <int EPI>
static int launch_gemm_t(const CUtensorMap& tm_a, const CUtensorMap& tm_b, int M, int N, int K, const float* bias,
                         const __nv_bfloat16* residual, int64_t ldr, __nv_bfloat16* out, int64_t ldo,
                         cudaStream_t stream) {
  const int rc = allow_dynamic_smem<gemm_bf16_kernel<EPI>>(GemmLayout::smem_bytes());
  if (rc != CRAG_OK) return rc;
  const unsigned n_blocks = (N + kGemmBN - 1) / kGemmBN, m_blocks = (M + kGemmBM - 1) / kGemmBM;
  const dim3 grid = EPI == GEMM_EPI_SCORES_F32 ? dim3(m_blocks * n_blocks) : dim3(n_blocks, m_blocks);
  gemm_bf16_kernel<EPI><<<grid, kGemmThreads, GemmLayout::smem_bytes(), stream>>>(tm_a, tm_b, M, N, K, bias, residual, ldr, out, ldo);
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

int gemm_bf16(const void* a, int64_t lda, const void* w, int64_t ldw, const float* bias, const void* residual,
              int64_t ldr, void* out, int64_t ldo, int M, int N, int K, int epi, cudaStream_t stream) {
  if (M <= 0) return CRAG_OK;
  if (N < 8 || K < 8 || N % 8 != 0 || K % 8 != 0) return fail(CRAG_ERR_INVALID, "gemm: N and K must be positive multiples of 8 (N=%d K=%d)", N, K);
  if (lda % 8 || ldw % 8 || ldo % 8 || (epi == GEMM_EPI_BIAS_RESIDUAL && ldr % 8)) return fail(CRAG_ERR_INVALID, "gemm: leading dimensions must be multiples of 8 elements");
  if (!a || !w || !bias || !out || (epi == GEMM_EPI_BIAS_RESIDUAL && !residual)) return fail(CRAG_ERR_INVALID, "gemm: null pointer");
  if ((uintptr_t(a) | uintptr_t(w) | uintptr_t(out) | uintptr_t(bias) | uintptr_t(residual)) & 15) return fail(CRAG_ERR_INVALID, "gemm: pointers must be 16-byte aligned");
  if ((M + kGemmBM - 1) / kGemmBM > 65535) return fail(CRAG_ERR_INVALID, "gemm: M too large (%d)", M);
  const __nv_bfloat16* res = static_cast<const __nv_bfloat16*>(residual);
  __nv_bfloat16* o = static_cast<__nv_bfloat16*>(out);
  CUtensorMap tm_a, tm_b;
  int rc = make_tmap_bf16_2d(&tm_a, a, uint64_t(M), uint64_t(K), uint64_t(lda) * 2, kGemmBM);
  if (rc != CRAG_OK) return rc;
  rc = make_tmap_bf16_2d(&tm_b, w, uint64_t(N), uint64_t(K), uint64_t(ldw) * 2, kGemmBN);
  if (rc != CRAG_OK) return rc;
  switch (epi) {
    case GEMM_EPI_BIAS: return launch_gemm_t<GEMM_EPI_BIAS>(tm_a, tm_b, M, N, K, bias, res, ldr, o, ldo, stream);
    case GEMM_EPI_BIAS_GELU: return launch_gemm_t<GEMM_EPI_BIAS_GELU>(tm_a, tm_b, M, N, K, bias, res, ldr, o, ldo, stream);
    case GEMM_EPI_BIAS_RESIDUAL: return launch_gemm_t<GEMM_EPI_BIAS_RESIDUAL>(tm_a, tm_b, M, N, K, bias, res, ldr, o, ldo, stream);
  }
  return fail(CRAG_ERR_INVALID, "gemm: unknown epilogue %d", epi);
}

int gemm_scores_f32(const void* a, int64_t lda, const void* w, int64_t ldw, float* out, int64_t ldo, int M, int N,
                    int K, cudaStream_t stream) {
  if (M <= 0 || N <= 0) return CRAG_OK;
  if (K < 64 || K % 64 != 0 || lda % 8 || ldw % 8 || ldo % 2) return fail(CRAG_ERR_INVALID, "gemm scores: K must be a multiple of 64, lda/ldw multiples of 8 and ldo even");
  if ((uintptr_t(a) | uintptr_t(w)) & 15 || uintptr_t(out) & 7) return fail(CRAG_ERR_INVALID, "gemm scores: misaligned pointer");
  if (int64_t((M + kGemmBM - 1) / kGemmBM) * ((N + kGemmBN - 1) / kGemmBN) > int64_t(0x7FFFFFFF)) return fail(CRAG_ERR_INVALID, "gemm scores: too many tiles (M=%d N=%d)", M, N);
  CUtensorMap tm_a, tm_b;
  int rc = make_tmap_bf16_2d(&tm_a, a, uint64_t(M), uint64_t(K), uint64_t(lda) * 2, kGemmBM);
  if (rc != CRAG_OK) return rc;
  rc = make_tmap_bf16_2d(&tm_b, w, uint64_t(N), uint64_t(K), uint64_t(ldw) * 2, kGemmBN);
  if (rc != CRAG_OK) return rc;
  return launch_gemm_t<GEMM_EPI_SCORES_F32>(tm_a, tm_b, M, N, K, nullptr, nullptr, 0, reinterpret_cast<__nv_bfloat16*>(out),
                                            ldo, stream);
}

}  // namespace crag

extern "C" int crag_gemm_bf16(const void* a, int64_t lda, const void* w, int64_t ldw, const float* bias,
                              const void* residual, int64_t ldr, void* out, int64_t ldo, int m, int n, int k,
                              int epilogue, crag_stream_t stream) {
  return crag::gemm_bf16(a, lda, w, ldw, bias, residual, ldr, out, ldo, m, n, k, epilogue,
                         static_cast<cudaStream_t>(stream));
}
