// Fused causal multi-query cosine-sim attention, forward (flash-style, online softmax, no [N,N] tensor).
//
//   sim = 8 * qn . kn + table[hh, i-j];  key-padding mask; causal mask; softmax (fp32); out = P v
//
// Replaces transformer.py:304-331 (einsum / masked_fill / softmax / einsum) for the self-attention
// instance (transformer.py:377).  q/k arrive already l2-normalised and scaled (transformer.py:269-271).
// Masked logits are treated as -inf, which is identical to the reference's -finfo.max fill whenever a
// row has at least one visible key (always true: key 0 is the first start token, never masked).
//
// v1 tensor path: mma.sync m16n8k16 bf16 (legacy HMMA); see attn_common.cuh for the folded-row layout.
#include "attn_common.cuh"
#include "../../include/omlm_b200.h"

namespace omlm {

constexpr int kAttnBR = 128;  // folded query rows per CTA (8 warps x 16)
constexpr int kAttnBC = 64;   // keys per tile
constexpr int kAttnThreads = 256;
constexpr int kBiasMax = 2048;

struct AttnFwdSmem {
  uint8_t q[kAttnBR * 128];          // also reused to stage O
  uint8_t k[2][kAttnBC * 128];
  uint8_t v[2][kAttnBC * 128];
  float bias[kBiasMax];
  float kneg[2][kAttnBC];
};

__global__ void __launch_bounds__(kAttnThreads, 2)
attn_fwd_kernel(const __nv_bfloat16* __restrict__ qn, const __nv_bfloat16* __restrict__ kvn,
                const float* __restrict__ table, int table_ld, const unsigned char* __restrict__ key_mask,
                __nv_bfloat16* __restrict__ out, float* __restrict__ lse2, int N, int h, float scale) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  AttnFwdSmem& sm = *reinterpret_cast<AttnFwdSmem*>(smem_raw);
  const int b = blockIdx.y;
  const int R = N * h;
  const int nblk = (R + kAttnBR - 1) / kAttnBR;
  const int rb = nblk - 1 - blockIdx.x;  // heavy (late) row blocks first
  const int r0 = rb * kAttnBR;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int i_min = r0 / h;
  const int i_max = min(N - 1, (r0 + kAttnBR - 1) / h);
  const int W = (i_max - i_min) + kAttnBC;  // bias slice width per head
  const int n_tiles = i_max / kAttnBC + 1;

  const __nv_bfloat16* qb = qn + (static_cast<long long>(b) * R) * 64;
  const __nv_bfloat16* kvb = kvn + (static_cast<long long>(b) * N) * 128;
  const uint32_t sq = smem_u32(sm.q);

  // ---- async loads: Q tile + first K/V tile
  for (int idx = threadIdx.x; idx < kAttnBR * 8; idx += kAttnThreads) {
    const int row = idx >> 3, c = idx & 7;
    const bool ok = (r0 + row) < R;
    cp_async16(sq + tile_off(row, c), qb + static_cast<long long>(ok ? r0 + row : 0) * 64 + c * 8, ok);
  }
  auto load_kv = [&](int tile, int buf) {
    const int j0 = tile * kAttnBC;
    const uint32_t sk = smem_u32(sm.k[buf]), sv = smem_u32(sm.v[buf]);
    for (int idx = threadIdx.x; idx < kAttnBC * 16; idx += kAttnThreads) {
      const int row = idx >> 4, c = idx & 15;
      const bool ok = (j0 + row) < N;
      const __nv_bfloat16* src = kvb + static_cast<long long>(ok ? j0 + row : 0) * 128 + c * 8;
      cp_async16((c < 8 ? sk : sv) + tile_off(row, c & 7), src, ok);
    }
    if (threadIdx.x < kAttnBC) {
      const int j = j0 + threadIdx.x;
      const bool vis = (j < N) && (key_mask == nullptr || key_mask[static_cast<long long>(b) * N + j] != 0);
      sm.kneg[buf][threadIdx.x] = vis ? 0.f : -INFINITY;
    }
  };
  load_kv(0, 0);
  cp_async_commit();

  // rows owned by this thread
  const int rA = r0 + warp * 16 + g, rB = rA + 8;
  const int iA = min(rA, R - 1) / h, iB = min(rB, R - 1) / h;
  const int hA = min(rA, R - 1) - iA * h, hB = min(rB, R - 1) - iB * h;

  float o[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) { o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f; }
  float mA = -INFINITY, mB = -INFINITY, lA = 0.f, lB = 0.f;
  uint32_t qf[4][4];
  const float sc2 = scale * kLog2e;

  for (int tile = 0; tile < n_tiles; ++tile) {
    const int buf = tile & 1;
    const int j0 = tile * kAttnBC;
    __syncthreads();  // everyone done with buffer buf^1 and with the bias slice of the previous tile
    if (tile + 1 < n_tiles) load_kv(tile + 1, buf ^ 1);
    cp_async_commit();
    // bias slice for this tile: delta = delta_min + w, delta_min = i_min - j0 - 63; delta < 0 -> causal -inf
    {
      const int delta_min = i_min - j0 - (kAttnBC - 1);
      for (int idx = threadIdx.x; idx < h * W; idx += kAttnThreads) {
        const int hh = idx / W, w = idx - hh * W;
        const int delta = delta_min + w;
        sm.bias[idx] = (delta < 0) ? -INFINITY : table[hh * table_ld + delta] * kLog2e;
      }
    }
    cp_async_wait<1>();
    __syncthreads();
    if (tile == 0) {
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) load_a_frag(sq, warp * 16, ks, lane, qf[ks]);
    }
    const uint32_t sk = smem_u32(sm.k[buf]), sv = smem_u32(sm.v[buf]);
    // ---- S = Q K^T
    float s[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) { s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bf[4];
        load_b_frag_nk(sk, np * 16, ks, lane, bf);
        mma_bf16(s[2 * np], qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], bf[0], bf[1]);
        mma_bf16(s[2 * np + 1], qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3], bf[2], bf[3]);
      }
    }
    // ---- scale, bias (+causal), key mask; online softmax in the log2 domain
    const float* bA = sm.bias + hA * W + (iA - i_min) + (kAttnBC - 1);
    const float* bB = sm.bias + hB * W + (iB - i_min) + (kAttnBC - 1);
    float mxA = -INFINITY, mxB = -INFINITY;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const int c0 = n * 8 + 2 * t;
      const float k0 = sm.kneg[buf][c0], k1 = sm.kneg[buf][c0 + 1];
      s[n][0] = fmaf(s[n][0], sc2, bA[-c0] + k0);
      s[n][1] = fmaf(s[n][1], sc2, bA[-c0 - 1] + k1);
      s[n][2] = fmaf(s[n][2], sc2, bB[-c0] + k0);
      s[n][3] = fmaf(s[n][3], sc2, bB[-c0 - 1] + k1);
      mxA = fmaxf(mxA, fmaxf(s[n][0], s[n][1]));
      mxB = fmaxf(mxB, fmaxf(s[n][2], s[n][3]));
    }
    mxA = fmaxf(mxA, __shfl_xor_sync(0xffffffffu, mxA, 1));
    mxA = fmaxf(mxA, __shfl_xor_sync(0xffffffffu, mxA, 2));
    mxB = fmaxf(mxB, __shfl_xor_sync(0xffffffffu, mxB, 1));
    mxB = fmaxf(mxB, __shfl_xor_sync(0xffffffffu, mxB, 2));
    const float mnA = fmaxf(mA, mxA), mnB = fmaxf(mB, mxB);
    const float refA = (mnA == -INFINITY) ? 0.f : mnA, refB = (mnB == -INFINITY) ? 0.f : mnB;
    const float alA = exp2f(mA - refA), alB = exp2f(mB - refB);
    mA = mnA; mB = mnB;
    float sumA = 0.f, sumB = 0.f;
    uint32_t pf[8][2];
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const float p0 = exp2f(s[n][0] - refA), p1 = exp2f(s[n][1] - refA);
      const float p2 = exp2f(s[n][2] - refB), p3 = exp2f(s[n][3] - refB);
      sumA += p0 + p1; sumB += p2 + p3;
      pf[n][0] = pack_bf16x2(p0, p1);
      pf[n][1] = pack_bf16x2(p2, p3);
    }
    lA = lA * alA + sumA; lB = lB * alB + sumB;
#pragma unroll
    for (int n = 0; n < 8; ++n) { o[n][0] *= alA; o[n][1] *= alA; o[n][2] *= alB; o[n][3] *= alB; }
    // ---- O += P V
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bf[4];
        load_b_frag_kn(sv, kk * 16, np * 16, lane, bf);
        mma_bf16(o[2 * np], pf[2 * kk][0], pf[2 * kk][1], pf[2 * kk + 1][0], pf[2 * kk + 1][1], bf[0], bf[1]);
        mma_bf16(o[2 * np + 1], pf[2 * kk][0], pf[2 * kk][1], pf[2 * kk + 1][0], pf[2 * kk + 1][1], bf[2], bf[3]);
      }
    }
  }
  cp_async_wait<0>();
  // ---- finalise: row sums across the quad, normalise, stage through smem, 16B stores
  lA += __shfl_xor_sync(0xffffffffu, lA, 1); lA += __shfl_xor_sync(0xffffffffu, lA, 2);
  lB += __shfl_xor_sync(0xffffffffu, lB, 1); lB += __shfl_xor_sync(0xffffffffu, lB, 2);
  const float invA = lA > 0.f ? 1.f / lA : 0.f, invB = lB > 0.f ? 1.f / lB : 0.f;
  __syncthreads();  // Q fragments are in registers; the Q tile can be overwritten
  {
    const int rowA = warp * 16 + g, rowB = rowA + 8;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const uint32_t vA = pack_bf16x2(o[n][0] * invA, o[n][1] * invA);
      const uint32_t vB = pack_bf16x2(o[n][2] * invB, o[n][3] * invB);
      *reinterpret_cast<uint32_t*>(sm.q + tile_off(rowA, n) + t * 4) = vA;
      *reinterpret_cast<uint32_t*>(sm.q + tile_off(rowB, n) + t * 4) = vB;
    }
    if (t == 0) {
      if (rA < R) lse2[static_cast<long long>(b) * R + rA] = mA + log2f(lA);
      if (rB < R) lse2[static_cast<long long>(b) * R + rB] = mB + log2f(lB);
    }
  }
  __syncthreads();
  __nv_bfloat16* ob = out + (static_cast<long long>(b) * R) * 64;
  for (int idx = threadIdx.x; idx < kAttnBR * 8; idx += kAttnThreads) {
    const int row = idx >> 3, c = idx & 7;
    if (r0 + row < R)
      *reinterpret_cast<uint4*>(ob + static_cast<long long>(r0 + row) * 64 + c * 8) =
          *reinterpret_cast<const uint4*>(sm.q + tile_off(row, c));
  }
}

}  // namespace omlm

extern "C" int omlm_attn_fwd(const void* qn, const void* kvn, const float* table, int table_ld,
                             const unsigned char* key_mask, void* out, float* lse2, int B, int N,
                             int heads, float scale, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attn_fwd: bad shape");
  OMLM_CHECK_ARG(heads * (kAttnBR / heads + 1 + kAttnBC) <= kBiasMax, "attn_fwd: too many heads (%d)", heads);
  OMLM_CHECK_ARG(table_ld >= N, "attn_fwd: bias table shorter than the sequence");
  static bool configured = false;
  const int smem = static_cast<int>(sizeof(AttnFwdSmem));
  if (!configured) {
    OMLM_CUDA(cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  const int R = N * heads;
  dim3 grid((R + kAttnBR - 1) / kAttnBR, B);
  OMLM_KLAUNCH((attn_fwd_kernel), grid, kAttnThreads, smem, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __nv_bfloat16*>(qn), reinterpret_cast<const __nv_bfloat16*>(kvn), table, table_ld,
      key_mask, reinterpret_cast<__nv_bfloat16*>(out), lse2, N, heads, scale);
  OMLM_LAUNCH_CHECK();
  return 0;
}
