// Bias-less LayerNorm (forward / backward) and the cosine-attention l2norm * scale (forward / backward).
// HBM-bound kernels: one warp per row, 128-bit vectorised accesses, row cached in registers.
//
// Replaces  LayerNorm.forward        open_musiclm/transformer.py:24-31  (F.layer_norm, eps 1e-5, beta == 0)
//           l2norm + q/k scale        open_musiclm/transformer.py:269-271, utils.py:68-69
#include "common.cuh"
#include <algorithm>
#include "../../include/omlm_b200.h"

namespace omlm {

constexpr int kNormThreads = 256;  // 8 rows per block

// ------------------------------------------------------------------------------------------------
// LayerNorm forward: y = (x - mean) * rstd * gamma  -> fp16 (y_f16) or bf16;  optional bf16 copy of y (the
// backward GEMMs pair it with bf16 gradients: one wgmma takes one format for both operands); optional raw bf16 copy
// of x;  stats[m] = (mean, rstd).  NCHUNK * 128 >= D.  (|y| <= sqrt(D) * |gamma|: bounded, hence fp16-safe.)
template <int NCHUNK>
__global__ void __launch_bounds__(kNormThreads)
layernorm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                     __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ ycopy, __nv_bfloat16* __restrict__ xraw,
                     float2* __restrict__ stats, const int* __restrict__ dest_row, int M, int D, int y_f16) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * (kNormThreads / 32) + warp;
  if (row >= M) return;
  const float* xr = x + static_cast<long long>(row) * D;
  float4 v[NCHUNK];
  float sum = 0.f;
#pragma unroll
  for (int c = 0; c < NCHUNK; ++c) {
    const int col = (c * 32 + lane) * 4;
    v[c] = (col < D) ? *reinterpret_cast<const float4*>(xr + col) : make_float4(0.f, 0.f, 0.f, 0.f);
    sum += v[c].x + v[c].y + v[c].z + v[c].w;
  }
  const float mean = warp_sum(sum) / D;
  float sq = 0.f;
#pragma unroll
  for (int c = 0; c < NCHUNK; ++c) {
    const int col = (c * 32 + lane) * 4;
    if (col < D) {
      const float a = v[c].x - mean, b = v[c].y - mean, cc = v[c].z - mean, d = v[c].w - mean;
      sq += a * a + b * b + cc * cc + d * d;
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / D + 1e-5f);
  if (lane == 0 && stats != nullptr) stats[row] = make_float2(mean, rstd);
  long long orow = row;
  if (dest_row != nullptr) orow = dest_row[row];
#pragma unroll
  for (int c = 0; c < NCHUNK; ++c) {
    const int col = (c * 32 + lane) * 4;
    if (col < D) {
      if (orow >= 0) {
        const float4 g = *reinterpret_cast<const float4*>(gamma + col);
        const float y0 = (v[c].x - mean) * rstd * g.x, y1 = (v[c].y - mean) * rstd * g.y;
        const float y2 = (v[c].z - mean) * rstd * g.z, y3 = (v[c].w - mean) * rstd * g.w;
        uint2 o;
        if (y_f16) { o.x = pack_f16x2(y0, y1); o.y = pack_f16x2(y2, y3); }
        else       { o.x = pack_bf16x2(y0, y1); o.y = pack_bf16x2(y2, y3); }
        *reinterpret_cast<uint2*>(y + orow * D + col) = o;
        if (ycopy != nullptr) {
          o.x = pack_bf16x2(y0, y1); o.y = pack_bf16x2(y2, y3);
          *reinterpret_cast<uint2*>(ycopy + orow * D + col) = o;
        }
      }
      if (xraw != nullptr) {
        uint2 o;
        o.x = pack_bf16x2(v[c].x, v[c].y);
        o.y = pack_bf16x2(v[c].z, v[c].w);
        *reinterpret_cast<uint2*>(xraw + static_cast<long long>(row) * D + col) = o;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm backward.  dx = [dres] + [draw] + rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat))
// dgamma[col] += sum_rows dy * xhat  (fp32; per-block partials in smem, one global atomic per column per block).
// dgamma == NULL (gamma frozen): no dgamma reduction, no partial rows.
// dy rows may be permuted (src_row: row of dy for this x row, -1 = no gradient).
// One warp per row.  The row's operands (x, dy, dres, draw: up to 12 bytes per element) are brought to a per-warp,
// double-buffered shared-memory stage with cp.async, so a warp always has the whole NEXT row in flight while it
// reduces the current one: bytes in flight per SM (~100 KB) are set by shared memory, not by registers.  Every lane
// reads back only the bytes it copied itself, so no barrier is needed beyond cp.async.wait_group.
__device__ __forceinline__ void ln_cp16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(dst))), "l"(src) : "memory");
}
__device__ __forceinline__ void ln_cp8(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(static_cast<uint32_t>(__cvta_generic_to_shared(dst))), "l"(src) : "memory");
}

// DET: no atomics -- the warps' dgamma sums are combined in warp order and written as this block's row of part
// [gridDim.x, D]; omlm_colsum then adds the rows to dgamma in block order.
template <int NCHUNK, int WARPS, bool DET>
__global__ void __launch_bounds__(WARPS * 32)
layernorm_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const float* __restrict__ x,
                     const float2* __restrict__ stats, const float* __restrict__ gamma,
                     const float* __restrict__ dres, const __nv_bfloat16* __restrict__ draw,
                     const int* __restrict__ src_row, float* __restrict__ dx,
                     __nv_bfloat16* __restrict__ dx_bf16, float* __restrict__ dgamma, int M, int D,
                     int rows_per_block, float* __restrict__ part) {
  constexpr int kRow = NCHUNK * 128;                 // padded row length in elements
  constexpr int kStage = kRow * 12;                  // x fp32 | dres fp32 | dy bf16 | draw bf16
  extern __shared__ __align__(16) uint8_t lsm[];
  float* sdg = reinterpret_cast<float*>(lsm + WARPS * 2 * kStage);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < kRow; i += WARPS * 32) sdg[i] = 0.f;
  __syncthreads();
  uint8_t* wbuf = lsm + warp * 2 * kStage;
  float4 dg[NCHUNK], gm[NCHUNK];
#pragma unroll
  for (int c = 0; c < NCHUNK; ++c) {
    dg[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    const int col = (c * 32 + lane) * 4;
    gm[c] = col < D ? *reinterpret_cast<const float4*>(gamma + col) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const int row0 = blockIdx.x * rows_per_block;
  const int row1 = min(M, row0 + rows_per_block);
  auto src_of = [&](int r) -> long long { return (r < row1) ? (src_row != nullptr ? static_cast<long long>(src_row[r]) : r) : -1; };
  auto issue = [&](int r, long long drow, int stage) {
    uint8_t* sb = wbuf + stage * kStage;
    const float* xr = x + static_cast<long long>(r) * D;
#pragma unroll
    for (int c = 0; c < NCHUNK; ++c) {
      const int col = (c * 32 + lane) * 4;
      if (col < D) {
        ln_cp16(sb + col * 4, xr + col);
        if (dres != nullptr) ln_cp16(sb + kRow * 4 + col * 4, dres + static_cast<long long>(r) * D + col);
        if (drow >= 0) ln_cp8(sb + kRow * 8 + col * 2, dy + drow * D + col);
        if (draw != nullptr) ln_cp8(sb + kRow * 10 + col * 2, draw + static_cast<long long>(r) * D + col);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  int row = row0 + warp;
  long long d_cur = src_of(row), d_nxt = src_of(row + WARPS);
  float2 st_nxt = make_float2(0.f, 0.f);
  if (row < row1) { issue(row, d_cur, 0); st_nxt = stats[row]; }
  int stage = 0;
  for (; row < row1; row += WARPS, stage ^= 1) {
    const float2 st = st_nxt;
    const long long d_nn = src_of(row + 2 * WARPS);     // two rows ahead: ready when its copies are issued
    if (row + WARPS < row1) {
      issue(row + WARPS, d_nxt, stage ^ 1);
      st_nxt = stats[row + WARPS];
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    const uint8_t* sb = wbuf + stage * kStage;
    // element-wise math on fp32x2 pairs (common.cuh), two channels per call
    float2 hA[NCHUNK], hB[NCHUNK], gA[NCHUNK], gB[NCHUNK];
    float2 s1v = make_float2(0.f, 0.f), s2v = s1v;
    const float2 rs2 = splat2(st.y), nmr = splat2(-st.x * st.y);          // xhat = x * rstd - mean * rstd
#pragma unroll
    for (int c = 0; c < NCHUNK; ++c) {
      const int col = (c * 32 + lane) * 4;
      hA[c] = hB[c] = gA[c] = gB[c] = make_float2(0.f, 0.f);
      if (col < D && d_cur >= 0) {
        const float4 xv = *reinterpret_cast<const float4*>(sb + col * 4);
        const uint2 dv = *reinterpret_cast<const uint2*>(sb + kRow * 8 + col * 2);
        const float2 dA = unpack_bf16x2(dv.x), dB = unpack_bf16x2(dv.y);
        hA[c] = fma2(make_float2(xv.x, xv.y), rs2, nmr);
        hB[c] = fma2(make_float2(xv.z, xv.w), rs2, nmr);
        const float2 a = fma2(dA, hA[c], make_float2(dg[c].x, dg[c].y)), b2 = fma2(dB, hB[c], make_float2(dg[c].z, dg[c].w));
        dg[c] = make_float4(a.x, a.y, b2.x, b2.y);
        gA[c] = mul2(dA, make_float2(gm[c].x, gm[c].y));
        gB[c] = mul2(dB, make_float2(gm[c].z, gm[c].w));
        s1v = add2(s1v, add2(gA[c], gB[c]));
        s2v = fma2(gA[c], hA[c], fma2(gB[c], hB[c], s2v));
      }
    }
    const float s1 = warp_sum(s1v.x + s1v.y) / D;
    const float s2 = warp_sum(s2v.x + s2v.y) / D;
    const float2 ns1r = splat2(-s1 * st.y), ns2r = splat2(-s2 * st.y);   // dx = g*rstd - s1*rstd - xhat*s2*rstd
#pragma unroll
    for (int c = 0; c < NCHUNK; ++c) {
      const int col = (c * 32 + lane) * 4;
      if (col < D) {
        float2 oA = make_float2(0.f, 0.f), oB = oA;
        if (d_cur >= 0) {
          oA = fma2(hA[c], ns2r, fma2(gA[c], rs2, ns1r));
          oB = fma2(hB[c], ns2r, fma2(gB[c], rs2, ns1r));
        }
        if (dres != nullptr) {
          const float4 r = *reinterpret_cast<const float4*>(sb + kRow * 4 + col * 4);
          oA = add2(oA, make_float2(r.x, r.y)); oB = add2(oB, make_float2(r.z, r.w));
        }
        if (draw != nullptr) {
          const uint2 rv = *reinterpret_cast<const uint2*>(sb + kRow * 10 + col * 2);
          oA = add2(oA, unpack_bf16x2(rv.x)); oB = add2(oB, unpack_bf16x2(rv.y));
        }
        *reinterpret_cast<float4*>(dx + static_cast<long long>(row) * D + col) = make_float4(oA.x, oA.y, oB.x, oB.y);
        if (dx_bf16 != nullptr) {
          uint2 ob;
          ob.x = pack_bf16x2(oA.x, oA.y);
          ob.y = pack_bf16x2(oB.x, oB.y);
          *reinterpret_cast<uint2*>(dx_bf16 + static_cast<long long>(row) * D + col) = ob;
        }
      }
    }
    d_cur = d_nxt; d_nxt = d_nn;
  }
  if (dgamma == nullptr) return;
  if constexpr (DET) {
    __syncthreads();                                  // every warp is done with its stage buffers: reuse them
    float* wdg = reinterpret_cast<float*>(lsm);       // [WARPS][kRow]
#pragma unroll
    for (int c = 0; c < NCHUNK; ++c) *reinterpret_cast<float4*>(wdg + warp * kRow + (c * 32 + lane) * 4) = dg[c];
    __syncthreads();
    for (int i = threadIdx.x; i < D; i += WARPS * 32) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < WARPS; ++w) v += wdg[w * kRow + i];
      part[static_cast<long>(blockIdx.x) * D + i] = v;
    }
  } else {
#pragma unroll
    for (int c = 0; c < NCHUNK; ++c) {
      const int col = (c * 32 + lane) * 4;
      atomicAdd(&sdg[col + 0], dg[c].x);
      atomicAdd(&sdg[col + 1], dg[c].y);
      atomicAdd(&sdg[col + 2], dg[c].z);
      atomicAdd(&sdg[col + 3], dg[c].w);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < D; i += WARPS * 32) atomicAdd(&dgamma[i], sdg[i]);
  }
}

// ------------------------------------------------------------------------------------------------
// l2norm * scale forward.  Vectors of 64 bf16; 8 lanes per vector (16 bytes each).
// per row: h query heads (from q_raw), 1 key (kv_raw[:, :64]) normalised; value (kv_raw[:, 64:]) copied.
__global__ void __launch_bounds__(256)
qk_l2norm_fwd_kernel(const __nv_bfloat16* __restrict__ q_raw, const __nv_bfloat16* __restrict__ kv_raw,
                     const float* __restrict__ q_scale, const float* __restrict__ k_scale,
                     __nv_bfloat16* __restrict__ qn, __nv_bfloat16* __restrict__ kvn, int M, int h) {
  const long long gvec = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 3;
  const int sub = threadIdx.x & 7;
  const int per_row = h + 2;
  const long long total = static_cast<long long>(M) * per_row;
  const bool active = gvec < total;
  const long long row = !active ? 0 : (total <= 0x7fffffffLL ? static_cast<long long>(static_cast<unsigned int>(gvec) / static_cast<unsigned int>(per_row))
                                                                : gvec / per_row);
  const int j = active ? static_cast<int>(gvec - row * per_row) : 0;
  const __nv_bfloat16* src;
  __nv_bfloat16* dst;
  const float* sc = nullptr;
  if (j < h) { src = q_raw + row * (h * 64) + j * 64; dst = qn + row * (h * 64) + j * 64; sc = q_scale; }
  else if (j == h) { src = kv_raw + row * 128; dst = kvn + row * 128; sc = k_scale; }
  else { src = kv_raw + row * 128 + 64; dst = kvn + row * 128 + 64; }
  uint4 raw = make_uint4(0, 0, 0, 0);
  if (active) raw = *reinterpret_cast<const uint4*>(src + sub * 8);
  float f[8];
  { float2 t;
    t = unpack_bf16x2(raw.x); f[0] = t.x; f[1] = t.y;
    t = unpack_bf16x2(raw.y); f[2] = t.x; f[3] = t.y;
    t = unpack_bf16x2(raw.z); f[4] = t.x; f[5] = t.y;
    t = unpack_bf16x2(raw.w); f[6] = t.x; f[7] = t.y; }
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ss += f[i] * f[i];
  ss += __shfl_xor_sync(0xffffffffu, ss, 1);
  ss += __shfl_xor_sync(0xffffffffu, ss, 2);
  ss += __shfl_xor_sync(0xffffffffu, ss, 4);
  if (!active) return;
  if (sc != nullptr) {
    const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);  // F.normalize eps
    const float4 s0 = *reinterpret_cast<const float4*>(sc + sub * 8);
    const float4 s1 = *reinterpret_cast<const float4*>(sc + sub * 8 + 4);
    uint4 o;
    o.x = pack_bf16x2(f[0] * inv * s0.x, f[1] * inv * s0.y);
    o.y = pack_bf16x2(f[2] * inv * s0.z, f[3] * inv * s0.w);
    o.z = pack_bf16x2(f[4] * inv * s1.x, f[5] * inv * s1.y);
    o.w = pack_bf16x2(f[6] * inv * s1.z, f[7] * inv * s1.w);
    *reinterpret_cast<uint4*>(dst + sub * 8) = o;
  } else {
    *reinterpret_cast<uint4*>(dst + sub * 8) = raw;
  }
}

// l2norm * scale backward.  y = s * x/|x|.  dx = (s*dy - xh * (xh . s*dy)) / |x| ;  ds += dy * xh.
// |x| < 1e-12 (F.normalize's clamp, e.g. the zero q / k of a pad row): y = s * x / 1e-12, dx = s*dy / 1e-12.
// dqn: fp32 [M, h*64] (atomically accumulated by the attention backward); dkvn: fp32 [M, 128].
// Outputs bf16 dq_raw [M, h*64], dkv_raw [M, 128] (value gradient passes through).
// DET: the 32 vector slots of a block are combined in slot order and written as this block's row of part [gridDim.x,
// 128] (q scale | k scale); omlm_colsum adds the rows in block order.
// dq_scale / dk_scale may each be NULL (that scale frozen): its sum is not reduced; both NULL: no partial rows.
template <bool DET>
__global__ void __launch_bounds__(256)
qk_l2norm_bwd_kernel(const float* __restrict__ dqn, const float* __restrict__ dkvn,
                     const __nv_bfloat16* __restrict__ q_raw, const __nv_bfloat16* __restrict__ kv_raw,
                     const float* __restrict__ q_scale, const float* __restrict__ k_scale,
                     __nv_bfloat16* __restrict__ dq_raw, __nv_bfloat16* __restrict__ dkv_raw,
                     float* __restrict__ dq_scale, float* __restrict__ dk_scale, int M, int h, float* __restrict__ part) {
  __shared__ float sds[2][64];
  __shared__ float sslot[DET ? 2 * 32 * 64 : 1];
  if (threadIdx.x < 128) sds[threadIdx.x >> 6][threadIdx.x & 63] = 0.f;
  __syncthreads();
  const int sub = threadIdx.x & 7;
  const int per_row = h + 2;
  const long long total = static_cast<long long>(M) * per_row;
  float dsq[8], dsk[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { dsq[i] = 0.f; dsk[i] = 0.f; }
  for (long long base = static_cast<long long>(blockIdx.x) * (blockDim.x >> 3); base < total;
       base += static_cast<long long>(gridDim.x) * (blockDim.x >> 3)) {
    const long long gvec = base + (threadIdx.x >> 3);
    const bool active = gvec < total;
    // (32-bit division whenever the vector count allows it: the 64-bit form is a ~100-instruction routine per thread)
    const long long row = !active ? 0 : (total <= 0x7fffffffLL ? static_cast<long long>(static_cast<unsigned int>(gvec) / static_cast<unsigned int>(per_row))
                                                                  : gvec / per_row);
    const int j = active ? static_cast<int>(gvec - row * per_row) : 0;
    const __nv_bfloat16* src;
    const float* dsrc;
    __nv_bfloat16* dst;
    const float* sc = nullptr;
    if (j < h) { src = q_raw + row * (h * 64) + j * 64; dsrc = dqn + row * (h * 64) + j * 64; dst = dq_raw + row * (h * 64) + j * 64; sc = q_scale; }
    else if (j == h) { src = kv_raw + row * 128; dsrc = dkvn + row * 128; dst = dkv_raw + row * 128; sc = k_scale; }
    else { src = kv_raw + row * 128 + 64; dsrc = dkvn + row * 128 + 64; dst = dkv_raw + row * 128 + 64; }
    float f[8], g[8];
    if (active) {
      const uint4 raw = *reinterpret_cast<const uint4*>(src + sub * 8);
      float2 t;
      t = unpack_bf16x2(raw.x); f[0] = t.x; f[1] = t.y;
      t = unpack_bf16x2(raw.y); f[2] = t.x; f[3] = t.y;
      t = unpack_bf16x2(raw.z); f[4] = t.x; f[5] = t.y;
      t = unpack_bf16x2(raw.w); f[6] = t.x; f[7] = t.y;
      const float4 g0 = *reinterpret_cast<const float4*>(dsrc + sub * 8);
      const float4 g1 = *reinterpret_cast<const float4*>(dsrc + sub * 8 + 4);
      g[0] = g0.x; g[1] = g0.y; g[2] = g0.z; g[3] = g0.w; g[4] = g1.x; g[5] = g1.y; g[6] = g1.z; g[7] = g1.w;
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) { f[i] = 0.f; g[i] = 0.f; }
    }
    float o[8];
    {
      // all 32 lanes run the same shuffles; the value vectors (sc == nullptr) just discard the result
      const bool norm = (sc != nullptr);
      float ss = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) ss += f[i] * f[i];
      ss += __shfl_xor_sync(0xffffffffu, ss, 1);
      ss += __shfl_xor_sync(0xffffffffu, ss, 2);
      ss += __shfl_xor_sync(0xffffffffu, ss, 4);
      const float nrm = sqrtf(ss);
      const float inv = 1.f / fmaxf(nrm, 1e-12f);
      float s[8];
      if (norm) {
        const float4 s0 = *reinterpret_cast<const float4*>(sc + sub * 8);
        const float4 s1 = *reinterpret_cast<const float4*>(sc + sub * 8 + 4);
        s[0] = s0.x; s[1] = s0.y; s[2] = s0.z; s[3] = s0.w; s[4] = s1.x; s[5] = s1.y; s[6] = s1.z; s[7] = s1.w;
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) s[i] = 1.f;
      }
      float dot = 0.f, xh[8], sg[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        xh[i] = f[i] * inv;
        if (norm) { if (j < h) dsq[i] += g[i] * xh[i]; else dsk[i] += g[i] * xh[i]; }
        sg[i] = g[i] * s[i];
        dot += xh[i] * sg[i];
      }
      dot += __shfl_xor_sync(0xffffffffu, dot, 1);
      dot += __shfl_xor_sync(0xffffffffu, dot, 2);
      dot += __shfl_xor_sync(0xffffffffu, dot, 4);
      // below the clamp F.normalize divides by the constant eps, whose gradient has no projection term: dx = s dy / eps
      if (nrm < 1e-12f) dot = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) o[i] = norm ? (sg[i] - xh[i] * dot) * inv : g[i];
    }
    if (active) {
      uint4 ov;
      ov.x = pack_bf16x2(o[0], o[1]); ov.y = pack_bf16x2(o[2], o[3]);
      ov.z = pack_bf16x2(o[4], o[5]); ov.w = pack_bf16x2(o[6], o[7]);
      *reinterpret_cast<uint4*>(dst + sub * 8) = ov;
    }
  }
  if (dq_scale == nullptr && dk_scale == nullptr) return;
  if constexpr (DET) {
    const int slot = threadIdx.x >> 3;
#pragma unroll
    for (int i = 0; i < 8; ++i) { sslot[slot * 64 + sub * 8 + i] = dsq[i]; sslot[(32 + slot) * 64 + sub * 8 + i] = dsk[i]; }
    __syncthreads();
    if (threadIdx.x < 128) {
      const int k = threadIdx.x >> 6, c = threadIdx.x & 63;
      float v = 0.f;
      for (int sl = 0; sl < 32; ++sl) v += sslot[(k * 32 + sl) * 64 + c];
      part[static_cast<long>(blockIdx.x) * 128 + threadIdx.x] = v;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      atomicAdd(&sds[0][sub * 8 + i], dsq[i]);
      atomicAdd(&sds[1][sub * 8 + i], dsk[i]);
    }
    __syncthreads();
    if (threadIdx.x < 64) { if (dq_scale != nullptr) atomicAdd(&dq_scale[threadIdx.x], sds[0][threadIdx.x]); }
    else if (threadIdx.x < 128) { if (dk_scale != nullptr) atomicAdd(&dk_scale[threadIdx.x - 64], sds[1][threadIdx.x - 64]); }
  }
}

template <int NCHUNK>
static int launch_ln_fwd(const float* x, const float* gamma, __nv_bfloat16* y, __nv_bfloat16* ycopy, __nv_bfloat16* xraw,
                         float2* stats, const int* dest_row, int M, int D, int y_f16, cudaStream_t st) {
  const int rows_per_block = kNormThreads / 32;
  OMLM_KLAUNCH((layernorm_fwd_kernel<NCHUNK>), (M + rows_per_block - 1) / rows_per_block, kNormThreads, 0, st, 
      x, gamma, y, ycopy, xraw, stats, dest_row, M, D, y_f16);
  OMLM_LAUNCH_CHECK();
  return 0;
}

template <int NCHUNK, bool DET = false>
static int launch_ln_bwd(const __nv_bfloat16* dy, const float* x, const float2* stats, const float* gamma,
                         const float* dres, const __nv_bfloat16* draw, const int* src_row, float* dx,
                         __nv_bfloat16* dx_bf16, float* dgamma, int M, int D, cudaStream_t st, float* part = nullptr,
                         long part_bytes = 0) {
  // shared memory (2 stages of 12 B/element per warp) decides residency: 8 warps up to D = 1024, 4 above
  constexpr int WARPS = NCHUNK <= 8 ? 8 : 4;
  constexpr int smem = WARPS * 2 * NCHUNK * 128 * 12 + NCHUNK * 128 * 4;
  static bool configured = false;
  if (!configured) {
    OMLM_CUDA(cudaFuncSetAttribute(layernorm_bwd_kernel<NCHUNK, WARPS, DET>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  const int per_sm = std::max(1, std::min(4, (220 * 1024) / smem));
  int blocks = num_sms() * per_sm;
  int rows_per_block = (M + blocks - 1) / blocks;
  if (rows_per_block < WARPS) rows_per_block = WARPS;
  blocks = (M + rows_per_block - 1) / rows_per_block;
  if (DET) OMLM_CHECK_ARG(part != nullptr && part_bytes >= static_cast<long>(blocks) * D * 4,
                          "layernorm_bwd_det: partials need %ld bytes", static_cast<long>(blocks) * D * 4);
  OMLM_KLAUNCH((layernorm_bwd_kernel<NCHUNK, WARPS, DET>), blocks, WARPS * 32, smem, st, dy, x, stats, gamma, dres, draw, src_row, dx,
                                                                       dx_bf16, dgamma, M, D, rows_per_block, part);
  OMLM_LAUNCH_CHECK();
  if (DET && dgamma != nullptr) return omlm_colsum(part, D, 1, dgamma, blocks, D, 1, st);
  return 0;
}

}  // namespace omlm

extern "C" {

int omlm_layernorm_fwd(const float* x, const float* gamma, void* y_bf16, int y_f16, void* ycopy_bf16, void* xraw_bf16,
                       float* stats, const int* dest_row, int M, int D, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && D > 0 && D % 4 == 0 && D <= 2048, "layernorm_fwd: unsupported shape %d x %d", M, D);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  auto y = reinterpret_cast<__nv_bfloat16*>(y_bf16);
  auto xr = reinterpret_cast<__nv_bfloat16*>(xraw_bf16);
  auto yc = reinterpret_cast<__nv_bfloat16*>(ycopy_bf16);
  auto s2 = reinterpret_cast<float2*>(stats);
  const int nchunk = (D + 127) / 128;
  if (nchunk <= 1) return launch_ln_fwd<1>(x, gamma, y, yc, xr, s2, dest_row, M, D, y_f16, st);
  if (nchunk <= 2) return launch_ln_fwd<2>(x, gamma, y, yc, xr, s2, dest_row, M, D, y_f16, st);
  if (nchunk <= 4) return launch_ln_fwd<4>(x, gamma, y, yc, xr, s2, dest_row, M, D, y_f16, st);
  if (nchunk <= 8) return launch_ln_fwd<8>(x, gamma, y, yc, xr, s2, dest_row, M, D, y_f16, st);
  return launch_ln_fwd<16>(x, gamma, y, yc, xr, s2, dest_row, M, D, y_f16, st);
}

int omlm_layernorm_bwd(const void* dy_bf16, const float* x, const float* stats, const float* gamma,
                       const float* dres, const void* draw_bf16, const int* src_row, float* dx,
                       void* dx_bf16, float* dgamma, int M, int D, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && D > 0 && D % 4 == 0 && D <= 2048, "layernorm_bwd: unsupported shape %d x %d", M, D);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  auto dy = reinterpret_cast<const __nv_bfloat16*>(dy_bf16);
  auto dr = reinterpret_cast<const __nv_bfloat16*>(draw_bf16);
  auto s2 = reinterpret_cast<const float2*>(stats);
  auto dxb = reinterpret_cast<__nv_bfloat16*>(dx_bf16);
  const int nchunk = (D + 127) / 128;
  if (nchunk <= 1) return launch_ln_bwd<1>(dy, x, s2, gamma, dres, dr, src_row, dx, dxb, dgamma, M, D, st);
  if (nchunk <= 2) return launch_ln_bwd<2>(dy, x, s2, gamma, dres, dr, src_row, dx, dxb, dgamma, M, D, st);
  if (nchunk <= 4) return launch_ln_bwd<4>(dy, x, s2, gamma, dres, dr, src_row, dx, dxb, dgamma, M, D, st);
  if (nchunk <= 8) return launch_ln_bwd<8>(dy, x, s2, gamma, dres, dr, src_row, dx, dxb, dgamma, M, D, st);
  return launch_ln_bwd<16>(dy, x, s2, gamma, dres, dr, src_row, dx, dxb, dgamma, M, D, st);
}

int omlm_layernorm_bwd_det(const void* dy_bf16, const float* x, const float* stats, const float* gamma,
                           const float* dres, const void* draw_bf16, const int* src_row, float* dx,
                           void* dx_bf16, float* dgamma, int M, int D, float* part_ws, long part_ws_bytes, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && D > 0 && D % 4 == 0 && D <= 2048, "layernorm_bwd_det: unsupported shape %d x %d", M, D);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  auto dy = reinterpret_cast<const __nv_bfloat16*>(dy_bf16);
  auto dr = reinterpret_cast<const __nv_bfloat16*>(draw_bf16);
  auto s2 = reinterpret_cast<const float2*>(stats);
  auto dxb = reinterpret_cast<__nv_bfloat16*>(dx_bf16);
  const int nchunk = (D + 127) / 128;
  if (nchunk <= 1) return launch_ln_bwd<1, true>(dy, x, s2, gamma, dres, dr, src_row, dx, dxb, dgamma, M, D, st, part_ws, part_ws_bytes);
  if (nchunk <= 2) return launch_ln_bwd<2, true>(dy, x, s2, gamma, dres, dr, src_row, dx, dxb, dgamma, M, D, st, part_ws, part_ws_bytes);
  if (nchunk <= 4) return launch_ln_bwd<4, true>(dy, x, s2, gamma, dres, dr, src_row, dx, dxb, dgamma, M, D, st, part_ws, part_ws_bytes);
  if (nchunk <= 8) return launch_ln_bwd<8, true>(dy, x, s2, gamma, dres, dr, src_row, dx, dxb, dgamma, M, D, st, part_ws, part_ws_bytes);
  return launch_ln_bwd<16, true>(dy, x, s2, gamma, dres, dr, src_row, dx, dxb, dgamma, M, D, st, part_ws, part_ws_bytes);
}

int omlm_qk_l2norm_fwd(const void* q_raw, const void* kv_raw, const float* q_scale, const float* k_scale,
                       void* qn, void* kvn, int M, int heads, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && heads > 0, "qk_l2norm_fwd: bad shape");
  const long long total = static_cast<long long>(M) * (heads + 2);
  const int blocks = static_cast<int>((total * 8 + 255) / 256);
  OMLM_KLAUNCH((qk_l2norm_fwd_kernel), blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __nv_bfloat16*>(q_raw), reinterpret_cast<const __nv_bfloat16*>(kv_raw), q_scale,
      k_scale, reinterpret_cast<__nv_bfloat16*>(qn), reinterpret_cast<__nv_bfloat16*>(kvn), M, heads);
  OMLM_LAUNCH_CHECK();
  return 0;
}

static int qk_l2norm_bwd_impl(const float* dqn, const float* dkvn, const void* q_raw, const void* kv_raw,
                              const float* q_scale, const float* k_scale, void* dq_raw, void* dkv_raw,
                              float* dq_scale, float* dk_scale, int M, int heads, float* part, long part_bytes, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && heads > 0, "qk_l2norm_bwd: bad shape");
  const long long total = static_cast<long long>(M) * (heads + 2);
  long long blocks = (total + 31) / 32;
  const long long cap = static_cast<long long>(num_sms()) * 8;
  if (blocks > cap) blocks = cap;
  const bool det = part != nullptr;
  if (det) OMLM_CHECK_ARG(part_bytes >= blocks * 128 * 4, "qk_l2norm_bwd_det: partials need %lld bytes", blocks * 128 * 4);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  OMLM_KLAUNCH((det ? qk_l2norm_bwd_kernel<true> : qk_l2norm_bwd_kernel<false>), static_cast<int>(blocks), 256, 0, st,
      dqn, dkvn, reinterpret_cast<const __nv_bfloat16*>(q_raw), reinterpret_cast<const __nv_bfloat16*>(kv_raw),
      q_scale, k_scale, reinterpret_cast<__nv_bfloat16*>(dq_raw), reinterpret_cast<__nv_bfloat16*>(dkv_raw),
      dq_scale, dk_scale, M, heads, part);
  OMLM_LAUNCH_CHECK();
  if (det) {
    if (dq_scale != nullptr) {
      const int rc = omlm_colsum(part, 128, 1, dq_scale, static_cast<int>(blocks), 64, 1, stream);
      if (rc) return rc;
    }
    if (dk_scale != nullptr) return omlm_colsum(part + 64, 128, 1, dk_scale, static_cast<int>(blocks), 64, 1, stream);
  }
  return 0;
}

int omlm_qk_l2norm_bwd(const float* dqn, const float* dkvn, const void* q_raw, const void* kv_raw,
                       const float* q_scale, const float* k_scale, void* dq_raw, void* dkv_raw,
                       float* dq_scale, float* dk_scale, int M, int heads, void* stream) {
  return qk_l2norm_bwd_impl(dqn, dkvn, q_raw, kv_raw, q_scale, k_scale, dq_raw, dkv_raw, dq_scale, dk_scale, M, heads,
                            nullptr, 0, stream);
}

int omlm_qk_l2norm_bwd_det(const float* dqn, const float* dkvn, const void* q_raw, const void* kv_raw,
                           const float* q_scale, const float* k_scale, void* dq_raw, void* dkv_raw,
                           float* dq_scale, float* dk_scale, int M, int heads, float* part_ws, long part_ws_bytes, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(part_ws != nullptr, "qk_l2norm_bwd_det: no partials buffer");
  return qk_l2norm_bwd_impl(dqn, dkvn, q_raw, kv_raw, q_scale, k_scale, dq_raw, dkv_raw, dq_scale, dk_scale, M, heads,
                            part_ws, part_ws_bytes, stream);
}

}  // extern "C"
