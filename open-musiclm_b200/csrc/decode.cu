// Incremental (KV-cache) decoding of the TokenConditionedTransformer: one new position per sequence and step.
//
// Replaces the full-prefix recomputation of TokenConditionedTransformerWrapper.generate (open_musiclm.py:300-319: one
// complete forward per sampled token) by a step that touches every weight once (HBM-bound: ~120 MB of 16-bit weights
// per step for the small model, whatever the batch) and the per-layer caches:
//     K / V        [B, Nmax, 128] bf16   (k l2-normalised * k_scale | v; MQA: one head, transformer.py:262-271)
//     conv state   [B, 2, 2 Fp]          the last two pre-conv FFN rows of CausalDSConv (transformer.py:122-131)
// The bias table [h, Nmax] depends on i - j only (transformer.py:55-67), so one table serves every step.
//
// Kernels (M = B <= 16 rows, SIMT: a 128-row tensor-core tile would idle 90 % of its rows and most SMs):
//   skinny_gemm     out[b, n] = A[b, :] . W[n, :] (+ residual), every warp streams two W rows with 16-byte loads; the
//                   prologue builds A in shared memory: plain 16-bit rows, fp32 rows rounded to bf16 (K/V input),
//                   LayerNorm of fp32 rows (transformer.py:24-31), or the inner FFN LayerNorm from the fused row sums
//   attn_decode     l2norm * scale of the new q / k, cache append, scores against the whole cache + bias, softmax, P V
//   conv_geglu      causal depthwise conv over (state, new row), GEGLU with exact-erf GELU, LayerNorm row sums
//   sample          eos rule, top-k, Gumbel-argmax (utils.py:71-84), next embedding row
// Rounding points mirror the training-path forward (16-bit GEMM operands, bf16 P, fp32 accumulation) so that an
// incremental step reproduces the full forward's logits to accumulation-order noise.
#include "common.cuh"
#include "../../include/omlm_b200.h"

namespace omlm {

constexpr int kDecMaxB = 16;

__device__ __forceinline__ float2 dec_unpack(uint32_t v, int f16) { return f16 ? unpack_f16x2(v) : unpack_bf16x2(v); }
__device__ __forceinline__ uint32_t dec_pack(float a, float b, int f16) { return f16 ? pack_f16x2(a, b) : pack_bf16x2(a, b); }
__device__ __forceinline__ float dec_round(float a, int f16) {
  return f16 ? __half2float(__float2half_rn(fminf(fmaxf(a, -65504.f), 65504.f))) : __bfloat162float(__float2bfloat16_rn(a));
}

// ------------------------------------------------------------------------------------------------ skinny GEMM
// prologue: 0 = A is 16-bit [B, K] in the operand format;  1 = A is fp32 [B, K], rounded to the operand format;
//           2 = LayerNorm(A fp32) * gamma;  3 = inner FFN LayerNorm: A is 16-bit h [B, K], rowsum [B, K/128, 2], gamma
//               (zero in the padding), n_real = F.
struct SkinnyArgs {
  const void* A; const uint16_t* W; const float* gamma; const float* rowsum; const float* addend; void* out;
  long lda, ldw, ldadd, ldo;
  int B, N, K, prologue, f16, out_fmt, n_real;
};

constexpr int kSkWarps = 8, kSkRowsPerWarp = 2;

__global__ void __launch_bounds__(kSkWarps * 32)
skinny_gemm_kernel(const SkinnyArgs a) {
  pdl_prologue();
  extern __shared__ __align__(16) uint8_t sk_smem[];
  uint16_t* sA = reinterpret_cast<uint16_t*>(sk_smem);              // [B][K] in the operand format
  __shared__ float s_mean[kDecMaxB], s_rstd[kDecMaxB];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int K = a.K, B = a.B;
  // ---- prologue: the activation rows, in the 16-bit operand format, into shared memory
  if (a.prologue == 2 || a.prologue == 3) {
    for (int b = warp; b < B; b += kSkWarps) {
      float mean, rstd;
      if (a.prologue == 2) {
        const float* x = reinterpret_cast<const float*>(a.A) + b * a.lda;
        float s = 0.f;
        for (int k = lane; k < K; k += 32) s += x[k];
        mean = warp_sum(s) / K;
        float q = 0.f;
        for (int k = lane; k < K; k += 32) { const float d = x[k] - mean; q += d * d; }
        rstd = rsqrtf(warp_sum(q) / K + 1e-5f);
      } else {
        const float2* rs = reinterpret_cast<const float2*>(a.rowsum) + static_cast<long>(b) * (K >> 7);
        float s1 = 0.f, s2 = 0.f;
        for (int t = lane; t < (K >> 7); t += 32) { s1 += rs[t].x; s2 += rs[t].y; }
        s1 = warp_sum(s1); s2 = warp_sum(s2);
        mean = s1 / a.n_real;
        rstd = rsqrtf(fmaxf(s2 / a.n_real - mean * mean, 0.f) + 1e-5f);
      }
      if (lane == 0) { s_mean[b] = mean; s_rstd[b] = rstd; }
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < B * (K >> 1); i += blockDim.x) {
    const int b = i / (K >> 1), k = (i - b * (K >> 1)) << 1;
    uint32_t v;
    if (a.prologue == 0) {
      v = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint16_t*>(a.A) + b * a.lda + k);
    } else if (a.prologue == 1) {
      const float* x = reinterpret_cast<const float*>(a.A) + b * a.lda + k;
      v = dec_pack(x[0], x[1], a.f16);
    } else if (a.prologue == 2) {
      const float* x = reinterpret_cast<const float*>(a.A) + b * a.lda + k;
      v = dec_pack((x[0] - s_mean[b]) * s_rstd[b] * a.gamma[k], (x[1] - s_mean[b]) * s_rstd[b] * a.gamma[k + 1], a.f16);
    } else {
      const float2 hv = dec_unpack(*reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint16_t*>(a.A) + b * a.lda + k), a.f16);
      v = dec_pack((hv.x - s_mean[b]) * s_rstd[b] * a.gamma[k], (hv.y - s_mean[b]) * s_rstd[b] * a.gamma[k + 1], a.f16);
    }
    *reinterpret_cast<uint32_t*>(sA + b * K + k) = v;
  }
  __syncthreads();
  // ---- each warp: kSkRowsPerWarp weight rows, lanes across K in 16-byte chunks
  const int row0 = (blockIdx.x * kSkWarps + warp) * kSkRowsPerWarp;
  if (row0 >= a.N) return;
  float acc[kSkRowsPerWarp][kDecMaxB];
#pragma unroll
  for (int r = 0; r < kSkRowsPerWarp; ++r)
#pragma unroll
    for (int b = 0; b < kDecMaxB; ++b) acc[r][b] = 0.f;
  const int chunks = K >> 3;
  for (int c = lane; c < chunks; c += 32) {
    float w[kSkRowsPerWarp][8];
#pragma unroll
    for (int r = 0; r < kSkRowsPerWarp; ++r) {
      uint4 raw = make_uint4(0, 0, 0, 0);
      if (row0 + r < a.N) raw = __ldg(reinterpret_cast<const uint4*>(a.W + (row0 + r) * a.ldw + c * 8));
      const uint32_t rw[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) { const float2 t = dec_unpack(rw[q], a.f16); w[r][2 * q] = t.x; w[r][2 * q + 1] = t.y; }
    }
#pragma unroll
    for (int b = 0; b < kDecMaxB; ++b) {
      if (b < B) {
        const uint4 av = *reinterpret_cast<const uint4*>(sA + b * K + c * 8);
        const uint32_t aw[4] = {av.x, av.y, av.z, av.w};
        float x[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) { const float2 t = dec_unpack(aw[q], a.f16); x[2 * q] = t.x; x[2 * q + 1] = t.y; }
#pragma unroll
        for (int r = 0; r < kSkRowsPerWarp; ++r)
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[r][b] = fmaf(x[e], w[r][e], acc[r][b]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < kSkRowsPerWarp; ++r) {
    const int n = row0 + r;
#pragma unroll
    for (int b = 0; b < kDecMaxB; ++b) {
      if (b < B) {
        float v = warp_sum(acc[r][b]);
        if (lane == 0 && n < a.N) {
          if (a.addend != nullptr) v += a.addend[b * a.ldadd + n];
          if (a.out_fmt == kFmtF32) reinterpret_cast<float*>(a.out)[b * a.ldo + n] = v;
          else if (a.out_fmt == kFmtF16) reinterpret_cast<__half*>(a.out)[b * a.ldo + n] = __float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f));
          else reinterpret_cast<__nv_bfloat16*>(a.out)[b * a.ldo + n] = __float2bfloat16_rn(v);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ attention, one new position
// grid (B, h), 128 threads.  q_raw [B, h*64] bf16, kv_raw [B, 128] bf16 (this step's projections, un-normalised),
// cache [B, Nmax, 128] bf16, table [h, table_ld] fp32, *pos_ptr = n = index of the new position (keys 0..n).
constexpr int kAdThreads = 128;

__global__ void __launch_bounds__(kAdThreads)
attn_decode_kernel(const __nv_bfloat16* __restrict__ q_raw, const __nv_bfloat16* __restrict__ kv_raw,
                   const float* __restrict__ q_scale, const float* __restrict__ k_scale,
                   __nv_bfloat16* __restrict__ cache, long cache_ld_b, const float* __restrict__ table, int table_ld,
                   const int* __restrict__ pos_ptr, __nv_bfloat16* __restrict__ out, int h, float scale) {
  pdl_prologue();
  extern __shared__ __align__(16) float ad_smem[];
  float* sc = ad_smem;                       // [n + 1] scores, then probabilities
  __shared__ float sq[64], sk[64], sv[64];
  __shared__ float red[kAdThreads / 32];
  __shared__ float so[16][64];
  const int b = blockIdx.x, head = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = *pos_ptr;
  // ---- l2norm * scale of the new query / key (utils.py:68-69, transformer.py:269-271), rounded to bf16 like the
  //      training path's qn / kvn tensors; head 0 appends [k | v] to the cache for the steps to come
  if (warp < 2) {
    const __nv_bfloat16* src = warp == 0 ? q_raw + static_cast<long>(b) * h * 64 + head * 64 : kv_raw + static_cast<long>(b) * 128;
    const float x0 = __bfloat162float(src[lane]), x1 = __bfloat162float(src[lane + 32]);
    const float inv = 1.f / fmaxf(sqrtf(warp_sum(x0 * x0 + x1 * x1)), 1e-12f);
    const float* s = warp == 0 ? q_scale : k_scale;
    float* dst = warp == 0 ? sq : sk;
    dst[lane] = bf16_round(x0 * inv * s[lane]);
    dst[lane + 32] = bf16_round(x1 * inv * s[lane + 32]);
  } else if (warp == 2) {
    sv[lane] = __bfloat162float(kv_raw[static_cast<long>(b) * 128 + 64 + lane]);
    sv[lane + 32] = __bfloat162float(kv_raw[static_cast<long>(b) * 128 + 96 + lane]);
  }
  __syncthreads();
  __nv_bfloat16* crow = cache + static_cast<long>(b) * cache_ld_b;
  if (head == 0 && tid < 128) {
    crow[static_cast<long>(n) * 128 + tid] = __float2bfloat16_rn(tid < 64 ? sk[tid] : sv[tid - 64]);
  }
  // ---- scores (log2 domain): 8 q.k_j + bias[head, n - j]
  const float l2e = 1.4426950408889634f;
  float mx = -INFINITY;
  for (int j = tid; j <= n; j += kAdThreads) {
    float dot = 0.f;
    if (j < n) {
      const uint4* kp = reinterpret_cast<const uint4*>(crow + static_cast<long>(j) * 128);
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint4 raw = __ldg(kp + c);
        const uint32_t rw[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 t = unpack_bf16x2(rw[q]);
          dot = fmaf(sq[c * 8 + 2 * q], t.x, dot);
          dot = fmaf(sq[c * 8 + 2 * q + 1], t.y, dot);
        }
      }
    } else {
#pragma unroll 8
      for (int d = 0; d < 64; ++d) dot = fmaf(sq[d], sk[d], dot);
    }
    const float s = (dot * scale + table[head * table_ld + (n - j)]) * l2e;
    sc[j] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  float sum = 0.f;
  for (int j = tid; j <= n; j += kAdThreads) {
    const float p = exp2f(sc[j] - mx);
    sum += p;
    sc[j] = bf16_round(p);                 // P enters the PV product as bf16, the normaliser stays fp32
  }
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  const float l = red[0] + red[1] + red[2] + red[3];
  // ---- o = P V: thread = (key group g of 16, 8-dim chunk)
  const int g = tid >> 3, ch = tid & 7;
  float o[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) o[e] = 0.f;
  for (int j = g; j <= n; j += 16) {
    const float p = sc[j];
    if (j < n) {
      const uint4 raw = __ldg(reinterpret_cast<const uint4*>(crow + static_cast<long>(j) * 128 + 64) + ch);
      const uint32_t rw[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 t = unpack_bf16x2(rw[q]);
        o[2 * q] = fmaf(p, t.x, o[2 * q]);
        o[2 * q + 1] = fmaf(p, t.y, o[2 * q + 1]);
      }
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = fmaf(p, bf16_round(sv[ch * 8 + e]), o[e]);
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) so[g][ch * 8 + e] = o[e];
  __syncthreads();
  if (tid < 64) {
    float acc = 0.f;
#pragma unroll
    for (int gg = 0; gg < 16; ++gg) acc += so[gg][tid];
    out[static_cast<long>(b) * h * 64 + head * 64 + tid] = __float2bfloat16_rn(acc / l);
  }
}

// ------------------------------------------------------------------------------------------------ attention, large batches
// The same step with every cached row read once per sequence: attn_decode runs one CTA per (sequence, head), so with
// multi-query attention each row is read `heads` times.  Here grid (splits, B): the CTA of split s serves ALL heads of
// sequence b over keys [128 s, 128 s + 128) ∩ [0, n] (flash decoding).  It stages those K | V rows in shared memory once,
// takes row n from this step's projections (and appends it to the cache: exactly one CTA covers n), and leaves per head
// the split's (max, sum) and unnormalised P V in a workspace.  The last split of a sequence to finish (per-sequence
// counter) combines the splits in order 0, 1, ... -- fixed order, deterministic -- and writes out.
// Rounding points of attn_decode: bf16 q / k after l2norm * scale, scores in the exp2 domain, P rounded to bf16 (here
// relative to the split's own maximum), fp32 normaliser.
constexpr int kMqThreads = 256, kMqKeys = 128;
constexpr int kMqRow = 272;                          // bytes per staged K | V row: 256 + 16 of padding (bank spread)
constexpr int kMqScLd = kMqKeys + 1;                 // score row pitch (floats)

template <int HM>                                    // HM >= heads: 4, 8 or 16
__global__ void __launch_bounds__(kMqThreads)
attn_decode_mqa_kernel(const __nv_bfloat16* __restrict__ q_raw, const __nv_bfloat16* __restrict__ kv_raw,
                       const float* __restrict__ q_scale, const float* __restrict__ k_scale,
                       __nv_bfloat16* __restrict__ cache, long cache_ld_b, const float* __restrict__ table, int table_ld,
                       const int* __restrict__ pos_ptr, __nv_bfloat16* __restrict__ out, int h, float scale,
                       float* __restrict__ part_o, float2* __restrict__ part_ml, int* __restrict__ counters, int max_splits) {
  pdl_prologue();
  extern __shared__ __align__(16) uint8_t mq_smem[];
  uint8_t* skv = mq_smem;                                                      // [kMqKeys][kMqRow]
  float* sc = reinterpret_cast<float*>(mq_smem + kMqKeys * kMqRow);            // [HM][kMqScLd] scores, then P
  constexpr int G = kMqThreads / (HM * 8);                                     // key groups of the P V product
  __shared__ float sq[HM][64], sk[64];
  __shared__ float so[G][HM * 64];
  __shared__ float s_m[HM], s_l[HM];
  __shared__ int s_last;
  const int split = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int n = *pos_ptr;
  const int j0 = split * kMqKeys;
  if (j0 > n) return;                                // beyond this step's keys (the grid covers max_pos)
  const int nk = min(kMqKeys, n + 1 - j0), active = n / kMqKeys + 1;
  // ---- l2norm * scale of every head's query and of the new key, rounded to bf16 (warp w: heads w, w + 8, then k)
  for (int t = warp; t <= h; t += kMqThreads / 32) {
    const __nv_bfloat16* src = t < h ? q_raw + static_cast<long>(b) * h * 64 + t * 64 : kv_raw + static_cast<long>(b) * 128;
    const float x0 = __bfloat162float(src[lane]), x1 = __bfloat162float(src[lane + 32]);
    const float inv = 1.f / fmaxf(sqrtf(warp_sum(x0 * x0 + x1 * x1)), 1e-12f);
    const float* s = t < h ? q_scale : k_scale;
    float* dst = t < h ? sq[t] : sk;
    dst[lane] = bf16_round(x0 * inv * s[lane]);
    dst[lane + 32] = bf16_round(x1 * inv * s[lane + 32]);
  }
  __nv_bfloat16* crow = cache + static_cast<long>(b) * cache_ld_b;
  for (int i = tid; i < nk * 16; i += kMqThreads) {  // cached rows j < n, 16 bytes per thread
    const int r = i >> 4, c = i & 15, j = j0 + r;
    if (j < n) *reinterpret_cast<uint4*>(skv + r * kMqRow + c * 16) = __ldg(reinterpret_cast<const uint4*>(crow + static_cast<long>(j) * 128) + c);
  }
  __syncthreads();
  if (n - j0 < kMqKeys && tid < 128) {               // row n: this step's [k | v], staged and appended to the cache
    const __nv_bfloat16 v = tid < 64 ? __float2bfloat16_rn(sk[tid]) : kv_raw[static_cast<long>(b) * 128 + tid];
    reinterpret_cast<__nv_bfloat16*>(skv + (n - j0) * kMqRow)[tid] = v;
    crow[static_cast<long>(n) * 128 + tid] = v;
  }
  __syncthreads();
  // ---- scores (log2 domain): 8 q.k_j + bias[head, n - j]; thread = key r, heads of parity tid / 128
  const float l2e = 1.4426950408889634f;
  {
    const int r = tid & (kMqKeys - 1), hp = tid >> 7;
    float dot[HM / 2];
#pragma unroll
    for (int u = 0; u < HM / 2; ++u) dot[u] = 0.f;
    if (r < nk) {
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const uint4 raw = *reinterpret_cast<const uint4*>(skv + r * kMqRow + c * 16);
        const uint32_t rw[4] = {raw.x, raw.y, raw.z, raw.w};
        float kf[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) { const float2 t = unpack_bf16x2(rw[q]); kf[2 * q] = t.x; kf[2 * q + 1] = t.y; }
#pragma unroll
        for (int u = 0; u < HM / 2; ++u) {
          if (hp + 2 * u < h) {
#pragma unroll
            for (int e = 0; e < 8; ++e) dot[u] = fmaf(sq[hp + 2 * u][c * 8 + e], kf[e], dot[u]);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < HM / 2; ++u) {
        const int hh = hp + 2 * u;
        if (hh < h) sc[hh * kMqScLd + r] = (dot[u] * scale + table[hh * table_ld + (n - j0 - r)]) * l2e;
      }
    }
  }
  __syncthreads();
  // ---- per head: the split's max and sum; P rounded to bf16 (warp w: heads w, w + 8)
  for (int hh = warp; hh < h; hh += kMqThreads / 32) {
    float* s = sc + hh * kMqScLd;
    float mx = -INFINITY;
    for (int r = lane; r < nk; r += 32) mx = fmaxf(mx, s[r]);
    mx = warp_max(mx);
    float sum = 0.f;
    for (int r = lane; r < nk; r += 32) {
      const float p = exp2f(s[r] - mx);
      sum += p;
      s[r] = bf16_round(p);
    }
    sum = warp_sum(sum);
    if (lane == 0) { s_m[hh] = mx; s_l[hh] = sum; }
  }
  __syncthreads();
  // ---- P V: thread = (key group g, head, 8-dim chunk)
  {
    const int g = tid / (HM * 8), hh = (tid >> 3) % HM, ch = tid & 7;
    float o[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = 0.f;
    if (hh < h) {
      for (int r = g; r < nk; r += G) {
        const float p = sc[hh * kMqScLd + r];
        const uint4 raw = *reinterpret_cast<const uint4*>(skv + r * kMqRow + 128 + ch * 16);
        const uint32_t rw[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float2 t = unpack_bf16x2(rw[q]);
          o[2 * q] = fmaf(p, t.x, o[2 * q]);
          o[2 * q + 1] = fmaf(p, t.y, o[2 * q + 1]);
        }
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) so[g][hh * 64 + ch * 8 + e] = o[e];
  }
  __syncthreads();
  if (active == 1) {                                 // a single split: normalise and write out directly
    for (int i = tid; i < h * 64; i += kMqThreads) {
      float acc = 0.f;
#pragma unroll
      for (int g = 0; g < G; ++g) acc += so[g][i];
      out[static_cast<long>(b) * h * 64 + i] = __float2bfloat16_rn(acc / s_l[i >> 6]);
    }
    return;
  }
  const long base = static_cast<long>(b) * max_splits;
  for (int i = tid; i < h * 64; i += kMqThreads) {
    float acc = 0.f;
#pragma unroll
    for (int g = 0; g < G; ++g) acc += so[g][i];
    __stcg(part_o + (base + split) * h * 64 + i, acc);
  }
  if (tid < h) __stcg(part_ml + (base + split) * h + tid, make_float2(s_m[tid], s_l[tid]));
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(counters + b, 1) == active - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // ---- last split of this sequence: combine the splits in order (rescaled to the common maximum)
  for (int i = tid; i < h * 64; i += kMqThreads) {
    const int hh = i >> 6;
    float mx = -INFINITY;
    for (int s = 0; s < active; ++s) mx = fmaxf(mx, __ldcg(part_ml + (base + s) * h + hh).x);
    float l = 0.f, acc = 0.f;
    for (int s = 0; s < active; ++s) {
      const float2 ml = __ldcg(part_ml + (base + s) * h + hh);
      const float f = exp2f(ml.x - mx);
      l = fmaf(f, ml.y, l);
      acc = fmaf(f, __ldcg(part_o + (base + s) * h * 64 + i), acc);
    }
    out[static_cast<long>(b) * h * 64 + i] = __float2bfloat16_rn(acc / l);
  }
  if (tid == 0) counters[b] = 0;                     // ready for the next step (or graph replay)
}

template <int HM>
static int launch_attn_decode_mqa(dim3 grid, cudaStream_t st, const void* q_raw, const void* kv_raw, const float* q_scale,
                                  const float* k_scale, void* cache, long cache_ld_b, const float* table, int table_ld,
                                  const int* pos_ptr, void* out, int heads, float scale, float* part_o, float2* part_ml,
                                  int* counters, int max_splits) {
  constexpr int smem = kMqKeys * kMqRow + HM * kMqScLd * 4;
  static bool configured = false;
  if (!configured) {
    OMLM_CUDA(cudaFuncSetAttribute(attn_decode_mqa_kernel<HM>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  OMLM_KLAUNCH((attn_decode_mqa_kernel<HM>), grid, kMqThreads, smem, st,
      reinterpret_cast<const __nv_bfloat16*>(q_raw), reinterpret_cast<const __nv_bfloat16*>(kv_raw), q_scale, k_scale,
      reinterpret_cast<__nv_bfloat16*>(cache), cache_ld_b, table, table_ld, pos_ptr, reinterpret_cast<__nv_bfloat16*>(out), heads,
      scale, part_o, part_ml, counters, max_splits);
  OMLM_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------ conv + GEGLU, one new row
// u_new [B, 2Fp] (interleaved GEGLU layout), state [B, 2, 2Fp] = rows t-2, t-1 -> h [B, Fp], rowsum [B, Fp/128, 2];
// the state is shifted in place.  grid (Fp/128, B), 128 threads (one per channel of the group).
__global__ void __launch_bounds__(128)
decode_conv_geglu_kernel(const uint16_t* __restrict__ u_new, uint16_t* __restrict__ state, const float* __restrict__ conv_w,
                         uint16_t* __restrict__ h_out, float* __restrict__ rowsum, int Fp, int f16) {
  pdl_prologue();
  const int grp = blockIdx.x, b = blockIdx.y, c = threadIdx.x;
  const long col_v = static_cast<long>(grp) * 256 + c, col_g = col_v + 128;
  const long ld = 2L * Fp;
  uint16_t* st0 = state + static_cast<long>(b) * 2 * ld;
  uint16_t* st1 = st0 + ld;
  auto val = [&](const uint16_t* p) -> float {
    return f16 ? __half2float(*reinterpret_cast<const __half*>(p)) : __uint_as_float(static_cast<uint32_t>(*p) << 16);
  };
  const float v2 = val(st0 + col_v), v1 = val(st1 + col_v), v0 = val(u_new + b * ld + col_v);
  const float g2 = val(st0 + col_g), g1 = val(st1 + col_g), g0 = val(u_new + b * ld + col_g);
  const float* wv = conv_w + col_v * 3;
  const float* wg = conv_w + col_g * 3;
  const float yv = fmaf(wv[0], v2, fmaf(wv[1], v1, wv[2] * v0));
  const float yg = fmaf(wg[0], g2, fmaf(wg[1], g1, wg[2] * g0));
  const float hval = gelu_erf(yg) * yv;
  // shift the history: (t-1, t) become (t-2, t-1) of the next step
  st0[col_v] = st1[col_v]; st0[col_g] = st1[col_g];
  st1[col_v] = u_new[b * ld + col_v]; st1[col_g] = u_new[b * ld + col_g];
  if (f16) reinterpret_cast<__half*>(h_out)[static_cast<long>(b) * Fp + grp * 128 + c] = __float2half_rn(fminf(fmaxf(hval, -65504.f), 65504.f));
  else reinterpret_cast<__nv_bfloat16*>(h_out)[static_cast<long>(b) * Fp + grp * 128 + c] = __float2bfloat16_rn(hval);
  __shared__ float r1[4], r2[4];
  const float s1 = warp_sum(hval), s2 = warp_sum(hval * hval);
  if ((c & 31) == 0) { r1[c >> 5] = s1; r2[c >> 5] = s2; }
  __syncthreads();
  if (c == 0) {
    float* dst = rowsum + (static_cast<long>(b) * (Fp >> 7) + grp) * 2;
    dst[0] = r1[0] + r1[1] + r1[2] + r1[3];
    dst[1] = r2[0] + r2[1] + r2[2] + r2[3];
  }
}

// ------------------------------------------------------------------------------------------------ sampling
// logits [B, ld] fp32, C classes.  eos (= class C-1) is forbidden unless allow_eos (open_musiclm.py:311-313); top-k with
// k = max(int((1 - thres) C), 1) (utils.py:78-84); Gumbel-argmax at temperature T (utils.py:71-76) with the uniform
// draw either supplied (uniform [steps, B, C], slice *step_ptr: parity runs reproduce torch's stream) or generated
// (Philox keyed by seed, step).
// Writes tokens[b, t] (t = *step_ptr), the embedding-table row of the sampled token for the next step, and advances
// the device-side counters (*step_ptr, *pos_ptr) once per launch.  grid B, 256 threads.
__global__ void __launch_bounds__(256)
sample_kernel(const float* __restrict__ logits, long ld, int C, int k, float temperature, int allow_eos,
              const float* __restrict__ uniform, const unsigned long long* __restrict__ seed_ptr,
              long long* __restrict__ tokens, long tokens_ld, int* __restrict__ next_row, int row_offset,
              int* __restrict__ step_ptr, int* __restrict__ pos_ptr, int B) {
  pdl_prologue();
  extern __shared__ float sm_l[];          // [C] logits, then [C] sort keys
  float* lg = sm_l;
  uint32_t* key = reinterpret_cast<uint32_t*>(sm_l + C);
  __shared__ float rv[8];
  __shared__ int ri[8];
  __shared__ uint32_t s_thr;
  const int b = blockIdx.x, tid = threadIdx.x;
  const int step = *step_ptr;
  for (int c = tid; c < C; c += 256) {
    float v = logits[b * ld + c];
    if (c == C - 1 && !allow_eos) v = -INFINITY;
    lg[c] = v;
    const uint32_t u = __float_as_uint(v);
    key[c] = (u & 0x80000000u) ? ~u : (u | 0x80000000u);       // order-preserving map float -> uint
  }
  __syncthreads();
  // ---- k-th largest key by bitwise bisection (32 counting passes over C <= a few thousand values)
  if (tid < 32) {
    uint32_t thr = 0;
    for (int bit = 31; bit >= 0; --bit) {
      const uint32_t cand = thr | (1u << bit);
      int cnt = 0;
      for (int c = tid; c < C; c += 32) cnt += key[c] >= cand;
      cnt = __reduce_add_sync(0xffffffffu, cnt);
      if (cnt >= k) thr = cand;
    }
    if (tid == 0) s_thr = thr;
  }
  __syncthreads();
  const uint32_t thr = s_thr;
  // torch.topk keeps exactly k entries: among equal values at the threshold the lower indices win
  __shared__ int s_tie_budget;
  if (tid == 0) {
    int above = 0;
    for (int c = 0; c < C; ++c) above += key[c] > thr;
    s_tie_budget = k - above;
  }
  __syncthreads();
  float best = -INFINITY;
  int best_i = 0x7fffffff;
  const unsigned long long seed = seed_ptr != nullptr ? *seed_ptr : 0ull;
  for (int c = tid; c < C; c += 256) {
    bool keep = key[c] > thr;
    if (!keep && key[c] == thr) {
      int rank = 0;
      for (int j = 0; j < c; ++j) rank += key[j] == thr;
      keep = rank < s_tie_budget;
    }
    if (!keep) continue;
    float u;
    if (uniform != nullptr) {
      u = uniform[(static_cast<long>(step) * B + b) * C + c];
    } else {
      const uint4 r = philox4x32(static_cast<uint32_t>(c), static_cast<uint32_t>(b), static_cast<uint32_t>(step), 0x5a17u,
                                 static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
      u = (r.x >> 8) * (1.0f / 16777216.0f);                    // [0, 1) with 24 bits, like torch's float uniform_
    }
    const float noise = -logf(-logf(u + 1e-20f) + 1e-20f);
    const float v = lg[c] / temperature + noise;
    if (v > best || (v == best && c < best_i)) { best = v; best_i = c; }
  }
  // block arg-max (first index wins ties, like torch.argmax)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
    if (ov > best || (ov == best && oi < best_i)) { best = ov; best_i = oi; }
  }
  if ((tid & 31) == 0) { rv[tid >> 5] = best; ri[tid >> 5] = best_i; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < 8; ++w)
      if (rv[w] > best || (rv[w] == best && ri[w] < best_i)) { best = rv[w]; best_i = ri[w]; }
    tokens[b * tokens_ld + step] = best_i;
    next_row[b] = row_offset + best_i;
  }
  // the counters advance once per launch, after every block has read them: last block to finish does it
  __shared__ bool last;
  __threadfence();
  if (tid == 0) {
    const int done = atomicAdd(step_ptr + 1, 1);               // step_ptr[1]: arrival counter
    last = done == B - 1;
  }
  __syncthreads();
  if (last && tid == 0) {
    step_ptr[1] = 0;
    step_ptr[0] = step + 1;
    if (pos_ptr != nullptr) pos_ptr[0] = pos_ptr[0] + 1;
    __threadfence();
  }
}

}  // namespace omlm

extern "C" {

int omlm_skinny_gemm(const void* A, long lda, int prologue, const void* W, long ldw, int w_f16, const float* gamma,
                     const float* rowsum, int n_real, const float* addend, long ldadd, void* out, int out_fmt, long ldo,
                     int B, int N, int K, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(B >= 1 && B <= kDecMaxB, "skinny_gemm: batch %d out of range (1..%d)", B, kDecMaxB);
  OMLM_CHECK_ARG(N > 0 && K > 0 && K % 8 == 0 && ldw % 8 == 0, "skinny_gemm: K and ldw must be multiples of 8 (K=%d ldw=%ld)", K, ldw);
  OMLM_CHECK_ARG(prologue >= 0 && prologue <= 3, "skinny_gemm: prologue %d", prologue);
  OMLM_CHECK_ARG((prologue < 2) || gamma != nullptr, "skinny_gemm: LayerNorm prologue needs gamma");
  OMLM_CHECK_ARG(prologue != 3 || (rowsum != nullptr && K % 128 == 0 && n_real > 0), "skinny_gemm: inner-norm prologue needs rowsum and K % 128 == 0");
  OMLM_CHECK_ARG(out_fmt == kFmtBF16 || out_fmt == kFmtF32 || out_fmt == kFmtF16, "skinny_gemm: out_fmt");
  OMLM_CHECK_ARG((reinterpret_cast<uintptr_t>(W) & 15) == 0, "skinny_gemm: W must be 16-byte aligned");
  SkinnyArgs a;
  a.A = A; a.W = reinterpret_cast<const uint16_t*>(W); a.gamma = gamma; a.rowsum = rowsum; a.addend = addend; a.out = out;
  a.lda = lda; a.ldw = ldw; a.ldadd = ldadd; a.ldo = ldo; a.B = B; a.N = N; a.K = K; a.prologue = prologue; a.f16 = w_f16;
  a.out_fmt = out_fmt; a.n_real = n_real;
  const int smem = B * K * 2;
  static int configured = 0;
  if (smem > configured) {
    OMLM_CUDA(cudaFuncSetAttribute(skinny_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = smem;
  }
  const int rows_per_cta = kSkWarps * kSkRowsPerWarp;
  OMLM_KLAUNCH((skinny_gemm_kernel), (N + rows_per_cta - 1) / rows_per_cta, kSkWarps * 32, smem, reinterpret_cast<cudaStream_t>(stream), a);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_attn_decode(const void* q_raw, const void* kv_raw, const float* q_scale, const float* k_scale, void* cache,
                     long cache_ld_b, const float* table, int table_ld, const int* pos_ptr, int max_pos, void* out, int B,
                     int heads, float scale, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(B >= 1 && heads >= 1 && max_pos >= 1 && table_ld >= max_pos, "attn_decode: bad shape");
  const int smem = max_pos * 4;
  OMLM_CHECK_ARG(smem <= 200 * 1024, "attn_decode: context %d too long", max_pos);
  static int configured = 0;
  if (smem > configured) {
    OMLM_CUDA(cudaFuncSetAttribute(attn_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = smem;
  }
  OMLM_KLAUNCH((attn_decode_kernel), dim3(B, heads), kAdThreads, smem, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __nv_bfloat16*>(q_raw), reinterpret_cast<const __nv_bfloat16*>(kv_raw), q_scale, k_scale,
      reinterpret_cast<__nv_bfloat16*>(cache), cache_ld_b, table, table_ld, pos_ptr, reinterpret_cast<__nv_bfloat16*>(out), heads, scale);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_attn_decode_mqa(const void* q_raw, const void* kv_raw, const float* q_scale, const float* k_scale, void* cache,
                         long cache_ld_b, const float* table, int table_ld, const int* pos_ptr, int max_pos, void* out, int B,
                         int heads, float scale, float* ws, long ws_bytes, int* counters, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(B >= 1 && heads >= 1 && heads <= 16 && max_pos >= 1 && table_ld >= max_pos, "attn_decode_mqa: bad shape");
  const int max_splits = (max_pos + kMqKeys - 1) / kMqKeys;
  const long need = static_cast<long>(B) * max_splits * heads * (64 + 2) * 4;
  OMLM_CHECK_ARG(ws != nullptr && counters != nullptr && ws_bytes >= need, "attn_decode_mqa: workspace of %ld bytes, %ld needed", ws_bytes, need);
  float* part_o = ws;
  float2* part_ml = reinterpret_cast<float2*>(ws + static_cast<long>(B) * max_splits * heads * 64);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const dim3 grid(max_splits, B);
  if (heads <= 4) return launch_attn_decode_mqa<4>(grid, st, q_raw, kv_raw, q_scale, k_scale, cache, cache_ld_b, table, table_ld,
                                                   pos_ptr, out, heads, scale, part_o, part_ml, counters, max_splits);
  if (heads <= 8) return launch_attn_decode_mqa<8>(grid, st, q_raw, kv_raw, q_scale, k_scale, cache, cache_ld_b, table, table_ld,
                                                   pos_ptr, out, heads, scale, part_o, part_ml, counters, max_splits);
  return launch_attn_decode_mqa<16>(grid, st, q_raw, kv_raw, q_scale, k_scale, cache, cache_ld_b, table, table_ld,
                                    pos_ptr, out, heads, scale, part_o, part_ml, counters, max_splits);
}

int omlm_decode_conv_geglu(const void* u_new, void* state, const float* conv_w, void* h_out, float* rowsum, int B, int Fp,
                           int act_f16, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(B >= 1 && Fp > 0 && Fp % 128 == 0, "decode_conv_geglu: bad shape");
  OMLM_KLAUNCH((decode_conv_geglu_kernel), dim3(Fp / 128, B), 128, 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const uint16_t*>(u_new), reinterpret_cast<uint16_t*>(state), conv_w, reinterpret_cast<uint16_t*>(h_out), rowsum, Fp, act_f16);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_sample(const float* logits, long ld, int C, int top_k, float temperature, int allow_eos, const float* uniform,
                const unsigned long long* seed, long long* tokens, long tokens_ld, int* next_row, int row_offset, int* step_ptr,
                int* pos_ptr, int B, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(B >= 1 && C >= 2 && C <= 16384 && temperature > 0.f && top_k >= 1 && top_k <= C, "sample: bad arguments");
  OMLM_KLAUNCH((sample_kernel), B, 256, 2 * C * 4, reinterpret_cast<cudaStream_t>(stream), logits, ld, C, top_k, temperature, allow_eos, uniform, seed, tokens,
                                                                            tokens_ld, next_row, row_offset, step_ptr, pos_ptr, B);
  OMLM_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
