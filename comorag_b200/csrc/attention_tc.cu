// K2 on wgmma: varlen multi-head self-attention for head dim 64 (BERT/BGE base & large).
//
//   ctx = softmax(Q K^T / sqrt(dh)) V      per (sequence, head), keys restricted to the sequence
//
// One CTA per (sequence, head, 128-query tile).  288 threads:
//   warps 0-7  two warpgroups, 64 query rows each: S_j = Q K_j^T (wgmma m64n64k16, Q and K_j from smem) into fp32
//            registers, online softmax in registers (a row lives in the 4 lanes of a quad), P_j converted in place
//            to the bf16 A fragment of O += P_j V_j (wgmma m64n64k16 with A from registers; V consumed MN-major,
//            i.e. as stored), final O / l -> bf16 -> ctx
//   warp 8   TMA: Q tile once, then K_j / V_j blocks of 64 keys through 2-stage rings (128-byte swizzle, straight
//            out of the packed [T, 3H] qkv activation)
#include <cstdlib>

#include "common.cuh"
#include "encoder.cuh"
#include "ptx.cuh"

namespace crag {

constexpr int kAttBM = 128;   // queries per CTA
constexpr int kAttBN = 64;    // keys per block
constexpr int kAttDH = 64;
constexpr int kAttThreads = 288;
constexpr int kAttTileBytes = 128 * 64 * 2;   // 16 KB: Q tile
constexpr int kAttKVBytes = kAttBN * 64 * 2;  // 8 KB: one K or V block
// smem: Q 16K | K 2x8K | V 2x8K | barriers  (~49 KB: several CTAs per SM)
constexpr size_t kAttSmemBytes = 1024 + kAttTileBytes + 4 * kAttKVBytes + 256;

__device__ __forceinline__ float att_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ uint32_t att_pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}

__global__ void __launch_bounds__(kAttThreads, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_kv,
                    const int32_t* __restrict__ cu_seqlens, int H, float scale_log2e, __nv_bfloat16* __restrict__ ctx) {
  const int seq = blockIdx.z, head = blockIdx.y;
  const int start = __ldg(cu_seqlens + seq);
  const int L = __ldg(cu_seqlens + seq + 1) - start;
  const int q0 = blockIdx.x * kAttBM;
  if (q0 >= L) return;
  const int n_blk = (L + kAttBN - 1) / kAttBN;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kAttTileBytes;        // [2]
  uint8_t* sV = sK + 2 * kAttKVBytes;      // [2]
  uint64_t* bar_q = reinterpret_cast<uint64_t*>(sV + 2 * kAttKVBytes);
  uint64_t* bar_k_full = bar_q + 1;        // [2]
  uint64_t* bar_v_full = bar_k_full + 2;   // [2]
  uint64_t* bar_kv_empty = bar_v_full + 2; // [2] both warpgroups are done with K_j and V_j (8 warps)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(bar_q, 1);
    for (int s = 0; s < 2; ++s) {
      mbar_init(&bar_k_full[s], 1);
      mbar_init(&bar_v_full[s], 1);
      mbar_init(&bar_kv_empty[s], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      tma_prefetch_desc(&tm_q);
      tma_prefetch_desc(&tm_kv);
      mbar_arrive_expect_tx(bar_q, kAttTileBytes);
      tma_load_2d(&tm_q, bar_q, sQ, head * kAttDH, start + q0);
      for (int j = 0; j < n_blk; ++j) {
        const int st = j & 1;
        const uint32_t ph = (j >> 1) & 1;
        mbar_wait(&bar_kv_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&bar_k_full[st], kAttKVBytes);
        tma_load_2d(&tm_kv, &bar_k_full[st], sK + st * kAttKVBytes, H + head * kAttDH, start + j * kAttBN);
        mbar_arrive_expect_tx(&bar_v_full[st], kAttKVBytes);
        tma_load_2d(&tm_kv, &bar_v_full[st], sV + st * kAttKVBytes, 2 * H + head * kAttDH, start + j * kAttBN);
      }
    }
    return;
  }

  // warpgroup wg: query rows [64 wg, 64 wg + 64) of the tile; this thread holds rows r_lo = 16 (warp % 4) + lane / 4
  // and r_lo + 8, key / feature columns 8 c + 2 (lane % 4) + {0, 1}
  const int wg = warp >> 2;
  const uint32_t q_addr = smem_u32(sQ) + wg * 64 * 128;
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait(bar_q, 0);
  for (int j = 0; j < n_blk; ++j) {
    const int st = j & 1;
    const uint32_t ph = (j >> 1) & 1;
    mbar_wait(&bar_k_full[st], ph);
    float s[32];
    const uint32_t k_addr = smem_u32(sK + st * kAttKVBytes);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kAttDH / 16; ++ks)
      wgmma_m64n64k16_ss(s, wgmma_desc_sw128(q_addr + ks * 32), wgmma_desc_sw128(k_addr + ks * 32), ks > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(s);

    const int kbase = j * kAttBN + 2 * (lane & 3);
    if (j * kAttBN + kAttBN > L) {  // only the last block of a sequence whose length is not a multiple of 64
#pragma unroll
      for (int c = 0; c < 8; ++c)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (kbase + 8 * c + e >= L) s[4 * c + e] = s[4 * c + 2 + e] = -INFINITY;  // exp2 -> 0, never the max
    }
    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int c = 0; c < 8; ++c) mx = fmaxf(mx, fmaxf(s[4 * c + 2 * h], s[4 * c + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx * scale_log2e);  // finite: >= 1 valid key per block
      alpha[h] = att_exp2(m_run[h] - m_new);                 // first block: exp2(-inf) = 0
      m_run[h] = m_new;
    }
    // p = exp2(s * scale - m), packed straight into the A fragment of P V (k-slice kk = keys 16 kk .. 16 kk + 15)
    uint32_t pa[4][4];
    float rs[2] = {0.f, 0.f};
#pragma unroll
    for (int c = 0; c < 8; ++c) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float p0 = att_exp2(fmaf(s[4 * c + 2 * h], scale_log2e, -m_run[h]));
        const float p1 = att_exp2(fmaf(s[4 * c + 2 * h + 1], scale_log2e, -m_run[h]));
        rs[h] += p0 + p1;
        pa[c >> 1][(c & 1) * 2 + h] = att_pack_bf16x2(p0, p1);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * alpha[h] + rs[h];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      o[4 * c + 0] *= alpha[0];
      o[4 * c + 1] *= alpha[0];
      o[4 * c + 2] *= alpha[1];
      o[4 * c + 3] *= alpha[1];
    }
    mbar_wait(&bar_v_full[st], ph);
    const uint32_t v_addr = smem_u32(sV + st * kAttKVBytes);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kAttBN / 16; ++kk)
      wgmma_m64n64k16_rs_bmn(o, pa[kk], wgmma_desc_sw128(v_addr + kk * 16 * 128), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bar_kv_empty[st]);
  }

  // epilogue: O / l -> bf16 -> ctx[start + row, head*64 .. +64)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.f / l;
    const int row = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    if (row < L) {
      __nv_bfloat16* dst = ctx + int64_t(start + row) * H + head * kAttDH + 2 * (lane & 3);
#pragma unroll
      for (int c = 0; c < 8; ++c)
        *reinterpret_cast<uint32_t*>(dst + 8 * c) = att_pack_bf16x2(o[4 * c + 2 * h] * inv, o[4 * c + 2 * h + 1] * inv);
    }
  }
}

int launch_attention_tc(const void* qkv, const int32_t* cu_seqlens, int n_seqs, int total_tokens, int max_len, int H,
                        int heads, void* ctx, cudaStream_t stream) {
  if (n_seqs <= 0 || max_len <= 0 || total_tokens <= 0) return CRAG_OK;
  if (H / heads != kAttDH) return fail(CRAG_ERR_UNSUPPORTED, "attention_tc: head dim must be 64");
  CUtensorMap tm_q, tm_kv;
  int rc = make_tmap_bf16_2d(&tm_q, qkv, uint64_t(total_tokens), uint64_t(3) * H, uint64_t(3) * H * 2, kAttBM);
  if (rc != CRAG_OK) return rc;
  rc = make_tmap_bf16_2d(&tm_kv, qkv, uint64_t(total_tokens), uint64_t(3) * H, uint64_t(3) * H * 2, kAttBN);
  if (rc != CRAG_OK) return rc;
  const dim3 grid((max_len + kAttBM - 1) / kAttBM, heads, n_seqs);
  const float scale_log2e = 1.4426950408889634f / sqrtf(float(kAttDH));
  rc = allow_dynamic_smem<attention_tc_kernel>(kAttSmemBytes);
  if (rc != CRAG_OK) return rc;
  attention_tc_kernel<<<grid, kAttThreads, kAttSmemBytes, stream>>>(tm_q, tm_kv, cu_seqlens, H, scale_log2e,
                                                                    static_cast<__nv_bfloat16*>(ctx));
  CRAG_CUDA_OK(cudaGetLastError());
  return CRAG_OK;
}

}  // namespace crag
