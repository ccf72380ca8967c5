// One incremental decoding step of the TokenConditionedTransformer as ONE persistent kernel.
//
// The per-op decode path (decode.cu) spends a token in 45 launches of a few microseconds of work each: the step is
// launch/latency bound (120 MB of weights per token).  Here the whole step --
// embedding row, L x (q/kv projection, cached attention, out-projection + residual, FFN-up + causal conv + GEGLU,
// inner LayerNorm + FFN-down + residual), final LayerNorm + logit head -- runs in one launch of one CTA per SM; the
// stages are separated by a grid-wide barrier (a global arrive counter; every CTA is resident: 1 CTA per SM, launched
// with at most as many CTAs as SMs), and inside a stage the output features are spread over all warps of the grid,
// each warp streaming two weight rows with 16-byte loads exactly like skinny_gemm_kernel.
//
// Every arithmetic step repeats the per-op kernels' formulas and summation orders (LayerNorm statistics, lane-strided dot
// products + butterfly, conv / GEGLU, the 4 x 32 tree of the inner-LayerNorm row sums, the attention of
// attn_decode_kernel), so both paths produce bit-identical logits (tests/test_decode_gpu.py compares them).
//
// Status: opt-in (OMLM_DECODE_FUSED=1); the CUDA-graph replay of the per-op kernels is the default.  The step's
// stages are each behind single-warp sections (LayerNorm statistics, the row-sum tree, lane-0 epilogues) and a grid
// barrier, so the launches it saves are not its bound.  Kept as the base for a batched-decode version.
//
// Replaces the loop body of TokenConditionedTransformerWrapper.generate (open_musiclm.py:300-319).
#include "common.cuh"
#include "../../include/omlm_b200.h"

namespace omlm {

constexpr int kDfMaxB = 16;
constexpr int kDfThreads = 512, kDfWarps = kDfThreads / 32;

__device__ __forceinline__ float2 df_unpack(uint32_t v, int f16) { return f16 ? unpack_f16x2(v) : unpack_bf16x2(v); }
__device__ __forceinline__ uint32_t df_pack(float a, float b, int f16) { return f16 ? pack_f16x2(a, b) : pack_bf16x2(a, b); }
__device__ __forceinline__ float df_round(float a, int f16) {
  return f16 ? __half2float(__float2half_rn(fminf(fmaxf(a, -65504.f), 65504.f))) : __bfloat162float(__float2bfloat16_rn(a));
}
__device__ __forceinline__ float df_load16(const uint16_t* p, int f16) {
  return f16 ? __half2float(*reinterpret_cast<const __half*>(p)) : __uint_as_float(static_cast<uint32_t>(*p) << 16);
}
// Buffers written by other CTAs earlier in the same launch (residual stream, projections, attention output, GEGLU output)
// are read with .cg loads: L1 is not coherent across SMs within a kernel.
__device__ __forceinline__ float df_ldcg_bf16(const __nv_bfloat16* p) {
  return __uint_as_float(static_cast<uint32_t>(__ldcg(reinterpret_cast<const unsigned short*>(p))) << 16);
}
__device__ __forceinline__ void df_store16(uint16_t* p, float v, int f16) {
  if (f16) *reinterpret_cast<__half*>(p) = __float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f));
  else *reinterpret_cast<__nv_bfloat16*>(p) = __float2bfloat16_rn(v);
}

// ---- grid-wide barrier: monotonic arrive counter (zeroed by the host before the launch) --------------------------------
__device__ __forceinline__ void df_grid_sync(unsigned int* bar, unsigned int& epoch, int* err) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    ++epoch;
    const unsigned int target = epoch * gridDim.x;
    atomicAdd(bar, 1u);
    const long long t0 = clock64();
    for (;;) {
      unsigned int v;
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
      if (v >= target) break;
      if (clock64() - t0 > (1LL << 33)) { atomicExch(err, 1); break; }     // ~4 s: never hang the device
    }
    __threadfence();
  }
  __syncthreads();
}

// ---- activation rows into shared memory (the prologues of skinny_gemm_kernel) ---------------------------------------------
// plain rounding of fp32 rows
__device__ __forceinline__ void df_rows_round(const float* __restrict__ x, long ldx, int B, int K, int f16, uint16_t* sA) {
  for (int i = threadIdx.x; i < B * (K >> 1); i += blockDim.x) {
    const int b = i / (K >> 1), k = (i - b * (K >> 1)) << 1;
    const float2 xv = __ldcg(reinterpret_cast<const float2*>(x + b * ldx + k));
    *reinterpret_cast<uint32_t*>(sA + b * K + k) = df_pack(xv.x, xv.y, f16);
  }
}
// LayerNorm(x) * gamma (transformer.py:24-31).  The rows are staged once in shared memory (sX, fp32 [B][K]); the
// statistics are then formed from there in the per-op kernel's summation order (lane-strided sums, butterfly).
__device__ __forceinline__ void df_rows_layernorm(const float* __restrict__ x, long ldx, const float* __restrict__ gamma, int B, int K,
                                                  int f16, uint16_t* sA, float* sX, float* s_mean, float* s_rstd) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < B * (K >> 2); i += blockDim.x) {
    const int b = i / (K >> 2), k = (i - b * (K >> 2)) << 2;
    *reinterpret_cast<float4*>(sX + b * K + k) = __ldcg(reinterpret_cast<const float4*>(x + b * ldx + k));
  }
  __syncthreads();
  for (int b = warp; b < B; b += kDfWarps) {
    const float* xr = sX + b * K;
    float s = 0.f;
    for (int k = lane; k < K; k += 32) s += xr[k];
    const float mean = warp_sum(s) / K;
    float q = 0.f;
    for (int k = lane; k < K; k += 32) { const float d = xr[k] - mean; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) / K + 1e-5f);
    if (lane == 0) { s_mean[b] = mean; s_rstd[b] = rstd; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < B * (K >> 1); i += blockDim.x) {
    const int b = i / (K >> 1), k = (i - b * (K >> 1)) << 1;
    const float2 xv = *reinterpret_cast<const float2*>(sX + b * K + k);
    *reinterpret_cast<uint32_t*>(sA + b * K + k) =
        df_pack((xv.x - s_mean[b]) * s_rstd[b] * gamma[k], (xv.y - s_mean[b]) * s_rstd[b] * gamma[k + 1], f16);
  }
}

// L2 prefetch of the two weight rows a warp will stream first in the NEXT stage, issued before the grid barrier: the rows do
// not depend on the activations, so their DRAM latency hides behind the barrier and the next prologue.
__device__ __forceinline__ void df_prefetch_rows(const uint16_t* W, long ldw, int row0, int row1, int K) {
  const int lane = threadIdx.x & 31;
  const int lines = (K * 2 + 127) >> 7;
  for (int i = lane; i < 2 * lines; i += 32) {
    const int r = i >= lines ? row1 : row0, ln = i >= lines ? i - lines : i;
    asm volatile("prefetch.global.L2 [%0];" ::"l"(reinterpret_cast<const char*>(W + static_cast<long>(r) * ldw) + ln * 128));
  }
}

// ---- two weight rows against all activation rows: the inner loop of skinny_gemm_kernel --------------------------------------
// returns acc[r][b] = warp_sum over the lane-strided partial dot products (identical order to the per-op kernel)
__device__ __forceinline__ void df_dot2(const uint16_t* __restrict__ W, long ldw, int row0, int row1, bool ok0, bool ok1, const uint16_t* sA,
                                        int K, int B, int f16, float (&acc)[2][kDfMaxB]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int b = 0; b < kDfMaxB; ++b) acc[r][b] = 0.f;
  const int chunks = K >> 3;
  // four 16-byte chunks per row are requested before any of them is used (same accumulation order as one at a time):
  // a step is a chain of ~30 such streaming loops, so every exposed DRAM round trip counts
  for (int c0 = lane; c0 < chunks; c0 += 128) {
    uint4 raw[4][2];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int c = c0 + 32 * u;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        raw[u][r] = make_uint4(0, 0, 0, 0);
        const bool ok = (r == 0 ? ok0 : ok1) && c < chunks;
        const int row = r == 0 ? row0 : row1;
        if (ok) raw[u][r] = __ldg(reinterpret_cast<const uint4*>(W + static_cast<long>(row) * ldw + c * 8));
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int c = c0 + 32 * u;
      if (c < chunks) {
        float w[2][8];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const uint32_t rw[4] = {raw[u][r].x, raw[u][r].y, raw[u][r].z, raw[u][r].w};
#pragma unroll
          for (int q = 0; q < 4; ++q) { const float2 t = df_unpack(rw[q], f16); w[r][2 * q] = t.x; w[r][2 * q + 1] = t.y; }
        }
#pragma unroll
        for (int b = 0; b < kDfMaxB; ++b) {
          if (b < B) {
            const uint4 av = *reinterpret_cast<const uint4*>(sA + b * K + c * 8);
            const uint32_t aw[4] = {av.x, av.y, av.z, av.w};
            float x[8];
#pragma unroll
            for (int q = 0; q < 4; ++q) { const float2 t = df_unpack(aw[q], f16); x[2 * q] = t.x; x[2 * q + 1] = t.y; }
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
              for (int e = 0; e < 8; ++e) acc[r][b] = fmaf(x[e], w[r][e], acc[r][b]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int b = 0; b < kDfMaxB; ++b)
      if (b < B) acc[r][b] = warp_sum(acc[r][b]);
}

struct DfLayer {
  const uint16_t *wq, *wkv, *wo, *w1, *w2;       // packed 16-bit weights (wq, w1, w2 in the activation format; wkv, wo bf16)
  const float *conv, *gin, *g_attn, *g_ff, *q_scale, *k_scale;
  __nv_bfloat16* cache;                          // [B, n_max, 128]
  uint16_t* conv_state;                          // [B, 2, 2 Fp]
};
struct DfArgs {
  const DfLayer* layers;
  int L, B, d, HD, h, F, Fp, n_max, f16, C_pad;
  const float* emb_table; const int* next_row;   // embedding row of the token processed by this step
  const float* table; int table_ld; const int* pos;
  float *x0, *x1;                                // residual stream [B, d] fp32 (two buffers)
  __nv_bfloat16 *q_raw, *kv_raw, *o;             // [B, HD], [B, 128], [B, HD]
  uint16_t* hbuf; float* hf32;                   // GEGLU output [B, Fp] (activation format) and its unrounded fp32 copy
  const uint16_t* w_logit; const float* g_final; float* logits; long ld_logits;
  unsigned int* bar; int* err;
  float scale;
};

// The attention of one (sequence, head) for the new position: body of attn_decode_kernel (decode.cu), run by the first 128
// threads of the CTA (all threads take part in the barriers).
__device__ __forceinline__ void df_attention(const DfArgs& a, const DfLayer& ly, int b, int head, float* sc, float* sq, float* sk, float* sv,
                                             float* red, float (*so)[64]) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int h = a.h;
  const int n = *a.pos;
  const bool act = tid < 128;
  if (act) {
    if (warp < 2) {
      const __nv_bfloat16* src = warp == 0 ? a.q_raw + static_cast<long>(b) * h * 64 + head * 64 : a.kv_raw + static_cast<long>(b) * 128;
      const float x0 = df_ldcg_bf16(src + lane), x1 = df_ldcg_bf16(src + lane + 32);
      const float inv = 1.f / fmaxf(sqrtf(warp_sum(x0 * x0 + x1 * x1)), 1e-12f);
      const float* s = warp == 0 ? ly.q_scale : ly.k_scale;
      float* dst = warp == 0 ? sq : sk;
      dst[lane] = bf16_round(x0 * inv * s[lane]);
      dst[lane + 32] = bf16_round(x1 * inv * s[lane + 32]);
    } else if (warp == 2) {
      sv[lane] = df_ldcg_bf16(a.kv_raw + static_cast<long>(b) * 128 + 64 + lane);
      sv[lane + 32] = df_ldcg_bf16(a.kv_raw + static_cast<long>(b) * 128 + 96 + lane);
    }
  }
  __syncthreads();
  __nv_bfloat16* crow = ly.cache + static_cast<long>(b) * a.n_max * 128;
  if (act && head == 0) crow[static_cast<long>(n) * 128 + tid] = __float2bfloat16_rn(tid < 64 ? sk[tid] : sv[tid - 64]);
  const float l2e = 1.4426950408889634f;
  float mx = -INFINITY;
  if (act) {
    for (int j = tid; j <= n; j += 128) {
      float dot = 0.f;
      if (j < n) {
        const uint4* kp = reinterpret_cast<const uint4*>(crow + static_cast<long>(j) * 128);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const uint4 raw = __ldcg(kp + c);       // (cache rows of this launch's earlier layers never alias; .cg: other SMs wrote them in earlier steps)
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
        for (int dd = 0; dd < 64; ++dd) dot = fmaf(sq[dd], sk[dd], dot);
      }
      const float s = (dot * a.scale + a.table[head * a.table_ld + (n - j)]) * l2e;
      sc[j] = s;
      mx = fmaxf(mx, s);
    }
    mx = warp_max(mx);
    if (lane == 0) red[warp] = mx;
  }
  __syncthreads();
  mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  float sum = 0.f;
  if (act) {
    for (int j = tid; j <= n; j += 128) {
      const float p = exp2f(sc[j] - mx);
      sum += p;
      sc[j] = bf16_round(p);
    }
    sum = warp_sum(sum);
    if (lane == 0) red[warp] = sum;
  }
  __syncthreads();
  const float l = red[0] + red[1] + red[2] + red[3];
  if (act) {
    const int g = tid >> 3, ch = tid & 7;
    float o[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = 0.f;
    for (int j = g; j <= n; j += 16) {
      const float p = sc[j];
      if (j < n) {
        const uint4 raw = __ldcg(reinterpret_cast<const uint4*>(crow + static_cast<long>(j) * 128 + 64) + ch);
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
  }
  __syncthreads();
  if (tid < 64) {
    float acc = 0.f;
#pragma unroll
    for (int gg = 0; gg < 16; ++gg) acc += so[gg][tid];
    a.o[static_cast<long>(b) * h * 64 + head * 64 + tid] = __float2bfloat16_rn(acc / l);
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kDfThreads, 1) decode_step_kernel(const DfArgs a) {
  extern __shared__ __align__(16) uint8_t df_smem[];
  uint16_t* sA = reinterpret_cast<uint16_t*>(df_smem);                 // [B][Kmax] activation rows (Kmax = max(d, Fp, HD))
  const int Kmax = max(max(a.d, a.Fp), a.HD);
  float* sc = reinterpret_cast<float*>(df_smem + static_cast<size_t>(a.B) * Kmax * 2);      // [n_max] attention scores
  float* sX = sc + ((a.n_max + 3) & ~3);                                                                 // [B][d] fp32 rows for the LayerNorm prologues
  __shared__ float s_mean[kDfMaxB], s_rstd[kDfMaxB];
  __shared__ float sq[64], sk[64], sv[64], red[4];
  __shared__ float so[16][64];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int gwarp = blockIdx.x * kDfWarps + warp, nwarps = gridDim.x * kDfWarps;
  const int B = a.B, d = a.d, HD = a.HD, Fp = a.Fp, f16 = a.f16;
  unsigned int epoch = 0;
  float* xa = a.x0;
  float* xm = a.x1;

  // ---- stage 0: embedding row of the token to process (embed_gather)
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B * d; i += gridDim.x * blockDim.x) {
    const int b = i / d, k = i - b * d;
    const int r = a.next_row[b];
    xa[i] = r >= 0 ? a.emb_table[static_cast<long>(r) * d + k] : 0.f;
  }
  if (gwarp < HD / 2) df_prefetch_rows(a.layers[0].wq, d, 2 * gwarp, 2 * gwarp + 1, d);
  df_grid_sync(a.bar, epoch, a.err);

  for (int l = 0; l < a.L; ++l) {
    const DfLayer ly = a.layers[l];
    // ---- stage A: q = LayerNorm(x) Wq^T (fp16/bf16 operand format), [k | v] = x Wkv^T (bf16)
    {
      df_rows_layernorm(xa, d, ly.g_attn, B, d, f16, sA, sX, s_mean, s_rstd);
      __syncthreads();
      for (int it = gwarp; it < HD / 2; it += nwarps) {
        float acc[2][kDfMaxB];
        df_dot2(ly.wq, d, 2 * it, 2 * it + 1, true, true, sA, d, B, f16, acc);
        if (lane == 0)
#pragma unroll
          for (int b = 0; b < kDfMaxB; ++b) if (b < B) {
            a.q_raw[static_cast<long>(b) * HD + 2 * it] = __float2bfloat16_rn(acc[0][b]);
            a.q_raw[static_cast<long>(b) * HD + 2 * it + 1] = __float2bfloat16_rn(acc[1][b]);
          }
      }
      __syncthreads();
      df_rows_round(xa, d, B, d, 0, sA);      // the K/V projection reads the raw residual stream, rounded to bf16
      __syncthreads();
      for (int it = gwarp; it < 64; it += nwarps) {
        float acc[2][kDfMaxB];
        df_dot2(ly.wkv, d, 2 * it, 2 * it + 1, true, true, sA, d, B, 0, acc);
        if (lane == 0)
#pragma unroll
          for (int b = 0; b < kDfMaxB; ++b) if (b < B) {
            a.kv_raw[static_cast<long>(b) * 128 + 2 * it] = __float2bfloat16_rn(acc[0][b]);
            a.kv_raw[static_cast<long>(b) * 128 + 2 * it + 1] = __float2bfloat16_rn(acc[1][b]);
          }
      }
    }
    if (gwarp < d / 2) df_prefetch_rows(ly.wo, HD, 2 * gwarp, 2 * gwarp + 1, HD);      // stage C's rows (stage B streams no weights)
    df_grid_sync(a.bar, epoch, a.err);
    // ---- stage B: attention of the new position against the cache (one CTA per (sequence, head))
    for (int item = blockIdx.x; item < B * a.h; item += gridDim.x) df_attention(a, ly, item / a.h, item % a.h, sc, sq, sk, sv, red, so);
    df_grid_sync(a.bar, epoch, a.err);
    // ---- stage C: xm = xa + o Wo^T
    {
      for (int i = threadIdx.x; i < B * (HD >> 1); i += blockDim.x) {
        const int b = i / (HD >> 1), k = (i - b * (HD >> 1)) << 1;
        *reinterpret_cast<uint32_t*>(sA + b * HD + k) = __ldcg(reinterpret_cast<const unsigned int*>(a.o + static_cast<long>(b) * HD + k));
      }
      __syncthreads();
      for (int it = gwarp; it < d / 2; it += nwarps) {
        float acc[2][kDfMaxB];
        df_dot2(ly.wo, HD, 2 * it, 2 * it + 1, true, true, sA, HD, B, 0, acc);
        if (lane == 0)
#pragma unroll
          for (int b = 0; b < kDfMaxB; ++b) if (b < B) {
            xm[static_cast<long>(b) * d + 2 * it] = acc[0][b] + __ldcg(xa + static_cast<long>(b) * d + 2 * it);
            xm[static_cast<long>(b) * d + 2 * it + 1] = acc[1][b] + __ldcg(xa + static_cast<long>(b) * d + 2 * it + 1);
          }
      }
    }
    if (gwarp < Fp) df_prefetch_rows(ly.w1, d, (gwarp >> 7) * 256 + (gwarp & 127), (gwarp >> 7) * 256 + 128 + (gwarp & 127), d);
    df_grid_sync(a.bar, epoch, a.err);
    // ---- stage D: u = LayerNorm(xm) W1^T; causal depthwise conv over (state, u); GEGLU (transformer.py:122-137)
    {
      df_rows_layernorm(xm, d, ly.g_ff, B, d, f16, sA, sX, s_mean, s_rstd);
      __syncthreads();
      const long ld = 2L * Fp;
      for (int it = gwarp; it < Fp; it += nwarps) {          // it = natural channel; rows: value g*256 + c, gate g*256 + 128 + c
        const int g = it >> 7, c = it & 127;
        const int rv = g * 256 + c, rg = rv + 128;
        float acc[2][kDfMaxB];
        df_dot2(ly.w1, d, rv, rg, true, true, sA, d, B, f16, acc);
        if (lane == 0) {
          const float* wv = ly.conv + static_cast<long>(rv) * 3;
          const float* wg = ly.conv + static_cast<long>(rg) * 3;
#pragma unroll
          for (int b = 0; b < kDfMaxB; ++b) if (b < B) {
            uint16_t* st0 = ly.conv_state + static_cast<long>(b) * 2 * ld;
            uint16_t* st1 = st0 + ld;
            const float v0 = df_round(acc[0][b], f16), g0 = df_round(acc[1][b], f16);      // u as the per-op path stores it
            const float v2 = df_load16(st0 + rv, f16), v1 = df_load16(st1 + rv, f16);
            const float g2 = df_load16(st0 + rg, f16), g1 = df_load16(st1 + rg, f16);
            const float yv = fmaf(wv[0], v2, fmaf(wv[1], v1, wv[2] * v0));
            const float yg = fmaf(wg[0], g2, fmaf(wg[1], g1, wg[2] * g0));
            const float hval = gelu_erf(yg) * yv;
            st0[rv] = st1[rv]; st0[rg] = st1[rg];
            df_store16(st1 + rv, acc[0][b], f16); df_store16(st1 + rg, acc[1][b], f16);
            df_store16(a.hbuf + static_cast<long>(b) * Fp + it, hval, f16);
            a.hf32[static_cast<long>(b) * Fp + it] = hval;
          }
        }
      }
    }
    if (gwarp < d / 2) df_prefetch_rows(ly.w2, Fp, 2 * gwarp, 2 * gwarp + 1, Fp);
    df_grid_sync(a.bar, epoch, a.err);
    // ---- stage E: xa = xm + LayerNorm_F(h) W2^T  (inner LayerNorm from the per-128-channel sums, summed as the per-op path does)
    {
      for (int b = warp; b < B; b += kDfWarps) {
        const float* hr = a.hf32 + static_cast<long>(b) * Fp;
        float my1 = 0.f, my2 = 0.f;          // lane t keeps the sums of channel group t (+ 32, + 64, ...)
        for (int g = 0; g < (Fp >> 7); ++g) {
          float t1 = 0.f, t2 = 0.f;
#pragma unroll
          for (int k4 = 0; k4 < 4; ++k4) {
            const float v = __ldcg(hr + g * 128 + k4 * 32 + lane);
            const float p1 = warp_sum(v), p2 = warp_sum(v * v);
            t1 = k4 == 0 ? p1 : t1 + p1;
            t2 = k4 == 0 ? p2 : t2 + p2;
          }
          if ((g & 31) == lane) { my1 += t1; my2 += t2; }
        }
        const float s1 = warp_sum(my1), s2 = warp_sum(my2);
        const float mean = s1 / a.F;
        const float rstd = rsqrtf(fmaxf(s2 / a.F - mean * mean, 0.f) + 1e-5f);
        if (lane == 0) { s_mean[b] = mean; s_rstd[b] = rstd; }
      }
      __syncthreads();
      for (int i = threadIdx.x; i < B * (Fp >> 1); i += blockDim.x) {
        const int b = i / (Fp >> 1), k = (i - b * (Fp >> 1)) << 1;
        const uint32_t raw = __ldcg(reinterpret_cast<const unsigned int*>(a.hbuf + static_cast<long>(b) * Fp + k));
        const float2 hv = df_unpack(raw, f16);
        *reinterpret_cast<uint32_t*>(sA + b * Fp + k) =
            df_pack((hv.x - s_mean[b]) * s_rstd[b] * ly.gin[k], (hv.y - s_mean[b]) * s_rstd[b] * ly.gin[k + 1], f16);
      }
      __syncthreads();
      for (int it = gwarp; it < d / 2; it += nwarps) {
        float acc[2][kDfMaxB];
        df_dot2(ly.w2, Fp, 2 * it, 2 * it + 1, true, true, sA, Fp, B, f16, acc);
        if (lane == 0)
#pragma unroll
          for (int b = 0; b < kDfMaxB; ++b) if (b < B) {
            xa[static_cast<long>(b) * d + 2 * it] = acc[0][b] + __ldcg(xm + static_cast<long>(b) * d + 2 * it);
            xa[static_cast<long>(b) * d + 2 * it + 1] = acc[1][b] + __ldcg(xm + static_cast<long>(b) * d + 2 * it + 1);
          }
      }
    }
    if (l + 1 < a.L) { if (gwarp < HD / 2) df_prefetch_rows(a.layers[l + 1].wq, d, 2 * gwarp, 2 * gwarp + 1, d); }
    else if (gwarp < a.C_pad / 2) df_prefetch_rows(a.w_logit, d, 2 * gwarp, 2 * gwarp + 1, d);
    df_grid_sync(a.bar, epoch, a.err);
  }
  // ---- logits of the requested head: LayerNorm(x) * gamma, then the head's rows
  df_rows_layernorm(xa, d, a.g_final, B, d, f16, sA, sX, s_mean, s_rstd);
  __syncthreads();
  for (int it = gwarp; it < (a.C_pad + 1) / 2; it += nwarps) {
    float acc[2][kDfMaxB];
    const bool ok1 = 2 * it + 1 < a.C_pad;
    df_dot2(a.w_logit, d, 2 * it, 2 * it + 1, true, ok1, sA, d, B, f16, acc);
    if (lane == 0)
#pragma unroll
      for (int b = 0; b < kDfMaxB; ++b) if (b < B) {
        a.logits[static_cast<long>(b) * a.ld_logits + 2 * it] = acc[0][b];
        if (ok1) a.logits[static_cast<long>(b) * a.ld_logits + 2 * it + 1] = acc[1][b];
      }
  }
}

}  // namespace omlm

extern "C" int omlm_decode_step(const omlm_decode_layer* layers_device, int L, int B, int d, int heads, int F, int Fp, int n_max, int act_f16,
                                const float* emb_table, const int* next_row, const float* table, int table_ld, const int* pos_ptr,
                                float* x0, float* x1, void* q_raw, void* kv_raw, void* o, void* hbuf, float* hf32, const void* w_logit,
                                int C_pad, const float* g_final, float* logits, long ld_logits, unsigned int* barrier, int* err_flag,
                                float scale, void* stream) {
  using namespace omlm;
  static_assert(sizeof(omlm_decode_layer) == sizeof(DfLayer), "omlm_decode_layer must mirror DfLayer");
  OMLM_CHECK_ARG(B >= 1 && B <= kDfMaxB, "decode_step: batch %d out of range (1..%d)", B, kDfMaxB);
  OMLM_CHECK_ARG(L >= 1 && d % 8 == 0 && Fp % 128 == 0 && heads >= 1 && n_max >= 1 && table_ld >= n_max, "decode_step: bad shape");
  OMLM_CHECK_ARG(layers_device != nullptr && barrier != nullptr && err_flag != nullptr, "decode_step: null table / barrier");
  DfArgs a;
  a.layers = reinterpret_cast<const DfLayer*>(layers_device);
  a.L = L; a.B = B; a.d = d; a.HD = heads * 64; a.h = heads; a.F = F; a.Fp = Fp; a.n_max = n_max; a.f16 = act_f16; a.C_pad = C_pad;
  a.emb_table = emb_table; a.next_row = next_row; a.table = table; a.table_ld = table_ld; a.pos = pos_ptr;
  a.x0 = x0; a.x1 = x1;
  a.q_raw = reinterpret_cast<__nv_bfloat16*>(q_raw); a.kv_raw = reinterpret_cast<__nv_bfloat16*>(kv_raw); a.o = reinterpret_cast<__nv_bfloat16*>(o);
  a.hbuf = reinterpret_cast<uint16_t*>(hbuf); a.hf32 = hf32;
  a.w_logit = reinterpret_cast<const uint16_t*>(w_logit); a.g_final = g_final; a.logits = logits; a.ld_logits = ld_logits;
  a.bar = barrier; a.err = err_flag; a.scale = scale;
  const int Kmax = std::max(std::max(d, Fp), heads * 64);
  const int smem = B * Kmax * 2 + ((n_max + 3) & ~3) * 4 + B * d * 4;
  OMLM_CHECK_ARG(smem <= 200 * 1024, "decode_step: batch x width / context too large for shared memory (%d bytes)", smem);
  static int configured = 0;
  if (smem > configured) {
    OMLM_CUDA(cudaFuncSetAttribute(decode_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = smem;
  }
  auto st = reinterpret_cast<cudaStream_t>(stream);
  OMLM_CUDA(cudaMemsetAsync(barrier, 0, sizeof(unsigned int), st));
  // every CTA must be resident for the grid-wide barriers: one CTA per SM, never more CTAs than SMs
  int per_sm = 0;
  OMLM_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, decode_step_kernel, kDfThreads, smem));
  OMLM_CHECK_ARG(per_sm >= 1, "decode_step: kernel does not fit on an SM");
  OMLM_KLAUNCH((decode_step_kernel), num_sms(), kDfThreads, smem, st, a);
  OMLM_LAUNCH_CHECK();
  return 0;
}
