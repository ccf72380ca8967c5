// The SIMT parts of ConvFeedForward that are NOT fused into a GEMM epilogue (transformer.py:140-150):
//   forward : LayerNorm(F) + dropout on the h tile that the FFN-up GEMM epilogue produced (gemm_ffn_up.cu does the
//             causal depthwise conv k=3 (122-131) and GEGLU with exact-erf GELU (134-137) under the MMA);
//   backward: dropout/LN backward, GEGLU backward, transposed causal conv and the conv / gamma weight gradients.
//
// Layout: u / du are [M, 2*Fp] bf16 in the INTERLEAVED GEGLU order: channels in groups of 128, each group stored as
// [128 value columns | 128 gate columns] (Fp = F padded to a multiple of 128; padded weights are zero so padded
// channels are exactly 0 everywhere).  h / hn / dhn are [M, Fp] in natural channel order.
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/omlm_b200.h"

namespace omlm {

// Column of channel c's VALUE half in the interleaved u / W1 / conv layout: 128-channel groups stored as
// [128 value columns | 128 gate columns] so that one 256-wide GEMM tile holds both halves of its channels.
__device__ __forceinline__ int ileave(int c) { return ((c >> 7) << 8) + (c & 127); }

// F16 selects the storage format of the forward activations u / h / hn (fp16 or bf16); gradients are always bf16.
template <bool F16 = false>
__device__ __forceinline__ void load8(const __nv_bfloat16* p, bool ok, float (&f)[8]) {
  uint4 raw = make_uint4(0, 0, 0, 0);
  if (ok) raw = *reinterpret_cast<const uint4*>(p);
  float2 t;
  t = unpack16x2<F16>(raw.x); f[0] = t.x; f[1] = t.y;
  t = unpack16x2<F16>(raw.y); f[2] = t.x; f[3] = t.y;
  t = unpack16x2<F16>(raw.z); f[4] = t.x; f[5] = t.y;
  t = unpack16x2<F16>(raw.w); f[6] = t.x; f[7] = t.y;
}
template <bool F16 = false>
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&f)[8]) {
  uint4 o;
  o.x = pack16x2<F16>(f[0], f[1]); o.y = pack16x2<F16>(f[2], f[3]);
  o.z = pack16x2<F16>(f[4], f[5]); o.w = pack16x2<F16>(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = o;
}

// keep flags for 8 channels of (row, chunk): 16 random bits per channel.
__device__ __forceinline__ void dropout_keep8(unsigned long long seed, uint32_t layer, long long row, int chunk,
                                              uint32_t thresh16, bool (&keep)[8]) {
  const uint4 r = philox4x32(static_cast<uint32_t>(row), static_cast<uint32_t>(row >> 32), static_cast<uint32_t>(chunk), layer,
                             static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32));
  keep[0] = (r.x & 0xffffu) >= thresh16; keep[1] = (r.x >> 16) >= thresh16;
  keep[2] = (r.y & 0xffffu) >= thresh16; keep[3] = (r.y >> 16) >= thresh16;
  keep[4] = (r.z & 0xffffu) >= thresh16; keep[5] = (r.z >> 16) >= thresh16;
  keep[6] = (r.w & 0xffffu) >= thresh16; keep[7] = (r.w >> 16) >= thresh16;
}

struct MidArgs {
  const __nv_bfloat16* u;     // [M, 2Fp]
  const float* conv_w;        // [2Fp, 3] packed
  const float* gamma;         // [Fp] packed (zeros in the padding)
  int N, F, Fp;
  float drop_p;               // 0 -> no dropout
  const uint8_t* keep_bits;   // [M, Fp/8] dropout keep mask written by ffn_norm_fwd (bit i of byte j: channel 8 j + i)
};

// ------------------------------------------------------------------------------------------------
// forward, second half: the FFN-up GEMM epilogue (gemm_ffn_up.cu) already produced h = gelu(conv(u)_gate) * conv(u)_value
// as bf16 and the per-row sums (sum h, sum h^2) in fp32.  This kernel finishes LayerNorm(F) + dropout:
//   hn = dropout((h - mean) * rstd * gamma),   stats[row] = (mean, rstd)  (kept for the backward pass).
// One warp per row, 16-byte accesses; HBM-bound (2 * M * Fp * 2 bytes).
__device__ __forceinline__ void load4(const __nv_bfloat16* p, bool ok, float (&f)[4]) {
  uint2 raw = make_uint2(0, 0);
  if (ok) raw = *reinterpret_cast<const uint2*>(p);
  const float2 a = unpack_bf16x2(raw.x), b = unpack_bf16x2(raw.y);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
}

template <bool F16>
__global__ void __launch_bounds__(256)
ffn_norm_fwd_kernel(const __nv_bfloat16* __restrict__ h, const float2* __restrict__ rowsum,
                    const float* __restrict__ gamma, __nv_bfloat16* __restrict__ hn, __nv_bfloat16* __restrict__ hn_copy, float2* __restrict__ stats,
                    uint8_t* __restrict__ keep_bits, long M, int F, int Fp, float drop_p,
                    const unsigned long long* __restrict__ seed_ptr, uint32_t layer) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long row = static_cast<long>(blockIdx.x) * 8 + warp;
  if (row >= M) return;
  // per-tile partial sums from the FFN-up epilogue, [row][Fp/128] float2: fixed-order (butterfly) reduction
  const int n_tiles = Fp >> 7;
  float2 rsum = make_float2(0.f, 0.f);
  for (int t = lane; t < n_tiles; t += 32) { const float2 p = rowsum[row * n_tiles + t]; rsum.x += p.x; rsum.y += p.y; }
  rsum.x = warp_sum(rsum.x); rsum.y = warp_sum(rsum.y);
  const float mean = rsum.x / F;
  const float var = fmaxf(rsum.y / F - mean * mean, 0.f);
  const float rstd = rsqrtf(var + 1e-5f);
  if (lane == 0) stats[row] = make_float2(mean, rstd);
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const uint32_t thresh = static_cast<uint32_t>(drop_p * 65536.f);
  const unsigned long long seed = (drop_p > 0.f) ? *seed_ptr : 0ull;
  for (int chunk = lane; chunk * 8 < Fp; chunk += 32) {
    float v[8];
    load8<F16>(h + row * Fp + chunk * 8, true, v);
    const float4 g0 = *reinterpret_cast<const float4*>(gamma + chunk * 8);
    const float4 g1 = *reinterpret_cast<const float4*>(gamma + chunk * 8 + 4);
    const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
    bool keep[8];
    if (drop_p > 0.f) dropout_keep8(seed, layer, row, chunk, thresh, keep);
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      o[i] = (v[i] - mean) * rstd * gm[i];          // gamma is zero in the padding -> padded channels stay 0
      if (drop_p > 0.f) o[i] = keep[i] ? o[i] * keep_scale : 0.f;
    }
    store8<F16>(hn + row * Fp + chunk * 8, o);
    if (hn_copy != nullptr) store8<false>(hn_copy + row * Fp + chunk * 8, o);   // bf16 copy for the backward GEMMs
    if (drop_p > 0.f) {   // the backward pass reads the mask back (1 bit per element) instead of replaying Philox
      uint32_t bits = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) bits |= (keep[i] ? 1u : 0u) << i;
      keep_bits[row * (Fp >> 3) + chunk] = static_cast<uint8_t>(bits);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// backward.
//
// LayerNorm backward needs two row sums before any element can be finished:
//   m1 = mean_c(gamma * g),  m2 = mean_c(gamma * g * hhat),   g = dropout-backward(dhn).
// Since hn = hhat * gamma * mask/(1-p) was saved by the forward pass, gamma*g*hhat == dhn * hn, so both
// sums come from one cheap pass over (dhn, hn)  [kernel 1, one warp per row].
// With m1/m2 known the rest is element-local in the channel dimension, so kernel 2 lets every thread own
// 4 channels (of both GEGLU halves) and WALK DOWN a slab of time steps with sliding windows: it recomputes
// conv/GEGLU/LN from u, forms dy (never written to memory), applies the transposed causal conv
// du[t] = w2 dy[t] + w1 dy[t+1] + w0 dy[t+2] and accumulates dconv_w / dgamma in registers.
__global__ void __launch_bounds__(256)
ffn_mid_bwd_stats_kernel(const __nv_bfloat16* __restrict__ dhn, const __nv_bfloat16* __restrict__ hn,
                         const float* __restrict__ gamma, float2* __restrict__ rowstat, long M, int F, int Fp,
                         float drop_p, const uint8_t* __restrict__ keep_bits) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long row = static_cast<long>(blockIdx.x) * 8 + warp;
  if (row >= M) return;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  float s1 = 0.f, s2 = 0.f;
  for (int chunk = lane; chunk * 8 < Fp; chunk += 32) {
    float d[8], hv[8];
    load8(dhn + row * Fp + chunk * 8, true, d);
    load8(hn + row * Fp + chunk * 8, true, hv);
    const uint32_t kb = drop_p > 0.f ? keep_bits[row * (Fp >> 3) + chunk] : 0xffu;
    const float4 g0 = *reinterpret_cast<const float4*>(gamma + chunk * 8);
    const float4 g1 = *reinterpret_cast<const float4*>(gamma + chunk * 8 + 4);
    const float gm[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float g = ((kb >> i) & 1u) ? d[i] * keep_scale : 0.f;
      s1 += gm[i] * g;
      s2 += d[i] * hv[i];
    }
  }
  s1 = warp_sum(s1); s2 = warp_sum(s2);
  if (lane == 0) rowstat[row] = make_float2(s1, s2);     // raw sums (one "partial"); the tile kernel divides by F
}

// Tile geometry of the walk: a CTA owns 128 time steps x one 128-channel group (= 256 contiguous u columns in the
// interleaved layout).  All operands of the tile (u with a 2-row history + 2-row look-ahead, dhn, the per-row LN
// constants and the keep bits) are brought to shared memory with 16-byte cp.async in one burst -- every byte of the
// tile is in flight at once, which is what the HBM latency needs -- and two CTAs per SM overlap one tile's load with
// the other's arithmetic.  Each of the 8 warps then walks a 16-row slab with lanes across channels (4 value + 4 gate
// per lane): shared-memory reads and global stores are contiguous across the warp, the conv windows slide through
// registers.
constexpr int kTileRows = 128, kTileWarps = 8, kTileSlab = 16, kTileThreads = kTileWarps * 32;
constexpr int kTuRows = kTileRows + 4, kTdRows = kTileRows + 2;
constexpr int kTOffU = 0;                               // [132][512 B]  u rows tb-2 .. tb+129
constexpr int kTOffD = kTOffU + kTuRows * 512;          // [130][256 B]  dhn rows tb .. tb+129
constexpr int kTOffS = kTOffD + kTdRows * 256;          // [130] float4 (mean, rstd, m1, m2)
constexpr int kTOffK = kTOffS + kTdRows * 16;           // [130][16 B] keep bits of the group's 128 channels
constexpr int kTOffAcc = kTOffK + kTdRows * 16;         // [7][128] fp32: dgamma, dconv value taps, dconv gate taps
constexpr int kTileSmem = kTOffAcc + 7 * 128 * 4;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool ok) {
  const int n = ok ? 16 : 0;   // src-size 0 -> the 16 destination bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gsrc, bool ok) {
  const int n = ok ? 8 : 0;
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(n) : "memory");
}

// DET: no atomics -- the warps' sums are combined in warp order and written to this CTA's row blockIdx.x of part
// [gridDim.x, 7F] in the parameters' layouts (dgamma [F] | dconv_w [2F, 3]); omlm_colsum adds the rows in order.
// dgamma / dconv_w may each be NULL (frozen, or no conv): that part is neither reduced nor written to part.
template <bool F16, bool DET>
__global__ void __launch_bounds__(kTileThreads, 2)
ffn_mid_bwd_walk_kernel(const MidArgs a, const __nv_bfloat16* __restrict__ dhn, const float2* __restrict__ stats,
                        const float2* __restrict__ rowstat, const int parts, __nv_bfloat16* __restrict__ du,
                        float* __restrict__ dgamma, float* __restrict__ dconv_w, float* __restrict__ part) {
  extern __shared__ __align__(16) uint8_t tsm[];
  uint8_t* su = tsm + kTOffU;
  uint8_t* sd = tsm + kTOffD;
  float4* sst = reinterpret_cast<float4*>(tsm + kTOffS);
  uint8_t* skb = tsm + kTOffK;
  float* sacc = reinterpret_cast<float*>(tsm + kTOffAcc);

  const int blocks_per_seq = (a.N + kTileRows - 1) / kTileRows;
  const int b = blockIdx.x / blocks_per_seq, tb = (blockIdx.x - b * blocks_per_seq) * kTileRows;
  const int g = blockIdx.y;                            // 128-channel group
  const long long row_base = static_cast<long long>(b) * a.N;
  const long ld = 2L * a.Fp;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  // ---- one burst of async copies for the whole tile
  for (int idx = tid; idx < kTuRows * 32; idx += kTileThreads) {
    const int j = idx >> 5, c = idx & 31, t = tb - 2 + j;
    const bool ok = t >= 0 && t < a.N;
    cp_async16(su + j * 512 + c * 16, a.u + (row_base + (ok ? t : 0)) * ld + g * 256 + c * 8, ok);
  }
  for (int idx = tid; idx < kTdRows * 16; idx += kTileThreads) {
    const int j = idx >> 4, c = idx & 15, t = tb + j;
    const bool ok = t < a.N;
    cp_async16(sd + j * 256 + c * 16, dhn + (row_base + (ok ? t : 0)) * a.Fp + g * 128 + c * 8, ok);
  }
  if (tid < kTdRows) {
    const int t = tb + tid;
    const bool ok = t < a.N;
    const long long row = row_base + (ok ? t : 0);
    cp_async8(reinterpret_cast<uint8_t*>(sst + tid), stats + row, ok);
    if (a.drop_p > 0.f) cp_async16(skb + tid * 16, a.keep_bits + row * (a.Fp >> 3) + g * 16, ok);
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  for (int i = tid; i < 7 * 128; i += kTileThreads) sacc[i] = 0.f;
  // LayerNorm-backward row means m1, m2: `parts` partial sums per row (from the d_hn GEMM's epilogue, or one from the
  // statistics kernel), added in a fixed order.  Plain loads into the .zw half of the row constants (the cp.async above
  // writes only .xy of the same float4)
  if (tid < kTdRows) {       // one thread per row; the (<= 32) partial sums are loaded back to back, then added in order
    const int t = tb + tid;
    float2 v[32];
    const float2* pr = rowstat + (row_base + min(t, a.N - 1)) * parts;
#pragma unroll
    for (int k = 0; k < 32; ++k) v[k] = (k < parts) ? __ldg(pr + k) : make_float2(0.f, 0.f);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) { s1 += v[k].x; s2 += v[k].y; }
    for (int k = 32; k < parts; ++k) { const float2 w = __ldg(pr + k); s1 += w.x; s2 += w.y; }
    const float invF = 1.f / a.F;
    reinterpret_cast<float2*>(sst + tid)[1] = (t < a.N) ? make_float2(s1 * invF, s2 * invF) : make_float2(0.f, 0.f);
  }

  // ---- per-lane constants: 4 value + 4 gate channels, held as two fp32x2 pairs (channels 2q, 2q+1)
  const int c0 = g * 128 + lane * 4;                   // natural channel index of this lane's first channel
  float2 wa[3][2], wg[3][2], gm[2], pm[2];             // taps [k][pair], gamma, 1/0 mask of real (c < F) channels
  {
    const float4* wp = reinterpret_cast<const float4*>(a.conv_w + static_cast<long>(g * 256 + lane * 4) * 3);
    const float4* gp = reinterpret_cast<const float4*>(a.conv_w + static_cast<long>(g * 256 + 128 + lane * 4) * 3);
    const float4 a0 = __ldg(wp), a1 = __ldg(wp + 1), a2 = __ldg(wp + 2);
    const float4 b0 = __ldg(gp), b1 = __ldg(gp + 1), b2 = __ldg(gp + 2);
    const float fa[12] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w};
    const float fb[12] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w, b2.x, b2.y, b2.z, b2.w};
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        wa[k][q] = make_float2(fa[(2 * q) * 3 + k], fa[(2 * q + 1) * 3 + k]);
        wg[k][q] = make_float2(fb[(2 * q) * 3 + k], fb[(2 * q + 1) * 3 + k]);
      }
    const float4 gg = __ldg(reinterpret_cast<const float4*>(a.gamma + c0));   // zero in the padding
    gm[0] = make_float2(gg.x, gg.y); gm[1] = make_float2(gg.z, gg.w);
    // padded channels are c >= F.  Not gamma == 0: a real channel whose gamma is exactly zero (zero-initialised, pruned)
    // still has dh = rstd (-m1 - hhat m2) != 0, and with it a gradient in u and in its conv taps
    pm[0] = make_float2(c0 < a.F ? 1.f : 0.f, c0 + 1 < a.F ? 1.f : 0.f);
    pm[1] = make_float2(c0 + 2 < a.F ? 1.f : 0.f, c0 + 3 < a.F ? 1.f : 0.f);
  }
  const float keep_scale = a.drop_p > 0.f ? 1.f / (1.f - a.drop_p) : 1.f;
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();

  // ---- walk this warp's slab: rows tb + 16 warp .. +15, plus two look-ahead rows for the transposed conv
  const int ts = warp * kTileSlab;
  float2 ua2[2], ua1[2], ug2[2], ug1[2];
  {
    const uint2 p2 = *reinterpret_cast<const uint2*>(su + ts * 512 + lane * 8);
    const uint2 q2 = *reinterpret_cast<const uint2*>(su + ts * 512 + 256 + lane * 8);
    const uint2 p1 = *reinterpret_cast<const uint2*>(su + (ts + 1) * 512 + lane * 8);
    const uint2 q1 = *reinterpret_cast<const uint2*>(su + (ts + 1) * 512 + 256 + lane * 8);
    ua2[0] = unpack16x2<F16>(p2.x); ua2[1] = unpack16x2<F16>(p2.y); ug2[0] = unpack16x2<F16>(q2.x); ug2[1] = unpack16x2<F16>(q2.y);
    ua1[0] = unpack16x2<F16>(p1.x); ua1[1] = unpack16x2<F16>(p1.y); ug1[0] = unpack16x2<F16>(q1.x); ug1[1] = unpack16x2<F16>(q1.y);
  }
  const float2 z2 = make_float2(0.f, 0.f);
  float2 da2[2] = {z2, z2}, da1[2] = {z2, z2}, dg2[2] = {z2, z2}, dg1[2] = {z2, z2};
  float2 dwa[3][2], dwg[3][2], dgam[2] = {z2, z2};
#pragma unroll
  for (int k = 0; k < 3; ++k) { dwa[k][0] = dwa[k][1] = z2; dwg[k][0] = dwg[k][1] = z2; }
  const int kshift = (lane & 1) * 4;
  __nv_bfloat16* du_lane = du + (row_base + tb + ts) * ld + g * 256 + lane * 4;
#pragma unroll 3
  for (int i = 0; i < kTileSlab + 2; ++i) {
    const int tl = ts + i;                              // row tb + tl
    const bool valid = tb + tl < a.N;
    const bool own = i < kTileSlab;                      // later rows are recomputed only for the conv look-ahead
    float2 ua0[2], ug0[2], da0[2], dg0[2];
    {
      const uint2 p = *reinterpret_cast<const uint2*>(su + (tl + 2) * 512 + lane * 8);
      const uint2 q = *reinterpret_cast<const uint2*>(su + (tl + 2) * 512 + 256 + lane * 8);
      ua0[0] = unpack16x2<F16>(p.x); ua0[1] = unpack16x2<F16>(p.y); ug0[0] = unpack16x2<F16>(q.x); ug0[1] = unpack16x2<F16>(q.y);
    }
    if (valid) {
      const uint2 dr = *reinterpret_cast<const uint2*>(sd + tl * 256 + lane * 8);
      const float4 st = sst[tl];
      float2 d[2] = {unpack_bf16x2(dr.x), unpack_bf16x2(dr.y)};
      if (a.drop_p > 0.f) {
        const uint32_t kb = static_cast<uint32_t>(skb[tl * 16 + (lane >> 1)]) >> kshift;
        const float2 k0 = make_float2((kb & 1u) ? keep_scale : 0.f, (kb & 2u) ? keep_scale : 0.f);
        const float2 k1 = make_float2((kb & 4u) ? keep_scale : 0.f, (kb & 8u) ? keep_scale : 0.f);
        d[0] = mul2(d[0], k0); d[1] = mul2(d[1], k1);
      }
      const float2 nmean = splat2(-st.x), rstd = splat2(st.y), nm1 = splat2(-st.z), nm2 = splat2(-st.w);
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float2 ya = fma2(wa[0][q], ua2[q], fma2(wa[1][q], ua1[q], mul2(wa[2][q], ua0[q])));
        const float2 yg = fma2(wg[0][q], ug2[q], fma2(wg[1][q], ug1[q], mul2(wg[2][q], ug0[q])));
        float2 phi, pdf;
        normal_cdf_pdf2(yg, phi, pdf);
        const float2 ge = mul2(yg, phi);
        const float2 hhat = mul2(fma2(ge, ya, nmean), rstd);
        // dh = rstd * (gamma d - m1 - hhat m2), forced to 0 on padded channels (c >= F)
        const float2 dh = mul2(mul2(rstd, pm[q]), fma2(hhat, nm2, fma2(gm[q], d[q], nm1)));
        da0[q] = mul2(dh, ge);
        dg0[q] = mul2(mul2(dh, ya), fma2(yg, pdf, phi));
        if (own) {
          dgam[q] = fma2(d[q], hhat, dgam[q]);
          dwa[0][q] = fma2(da0[q], ua2[q], dwa[0][q]); dwa[1][q] = fma2(da0[q], ua1[q], dwa[1][q]); dwa[2][q] = fma2(da0[q], ua0[q], dwa[2][q]);
          dwg[0][q] = fma2(dg0[q], ug2[q], dwg[0][q]); dwg[1][q] = fma2(dg0[q], ug1[q], dwg[1][q]); dwg[2][q] = fma2(dg0[q], ug0[q], dwg[2][q]);
        }
      }
    } else {
      da0[0] = da0[1] = z2; dg0[0] = dg0[1] = z2;
    }
    if (i >= 2 && tb + tl - 2 < a.N) {   // du[t-2] = w2 dy[t-2] + w1 dy[t-1] + w0 dy[t]
      float2 oa[2], og[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        oa[q] = fma2(wa[2][q], da2[q], fma2(wa[1][q], da1[q], mul2(wa[0][q], da0[q])));
        og[q] = fma2(wg[2][q], dg2[q], fma2(wg[1][q], dg1[q], mul2(wg[0][q], dg0[q])));
      }
      __nv_bfloat16* o = du_lane + static_cast<long>(i - 2) * ld;
      *reinterpret_cast<uint2*>(o) = make_uint2(pack_bf16x2(oa[0].x, oa[0].y), pack_bf16x2(oa[1].x, oa[1].y));
      *reinterpret_cast<uint2*>(o + 128) = make_uint2(pack_bf16x2(og[0].x, og[0].y), pack_bf16x2(og[1].x, og[1].y));
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      ua2[q] = ua1[q]; ua1[q] = ua0[q]; ug2[q] = ug1[q]; ug1[q] = ug0[q];
      da2[q] = da1[q]; da1[q] = da0[q]; dg2[q] = dg1[q]; dg1[q] = dg0[q];
    }
  }
  if (dgamma == nullptr && dconv_w == nullptr) return;
  if constexpr (DET) {
    __syncthreads();                                      // every warp is done with the u tile: reuse it
    float* wsum = reinterpret_cast<float*>(su);           // [warps][7][128]
    float* ws = wsum + warp * 7 * 128;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      ws[lane * 4 + 2 * q] = dgam[q].x;
      ws[lane * 4 + 2 * q + 1] = dgam[q].y;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        ws[(1 + k) * 128 + lane * 4 + 2 * q] = dwa[k][q].x;
        ws[(1 + k) * 128 + lane * 4 + 2 * q + 1] = dwa[k][q].y;
        ws[(4 + k) * 128 + lane * 4 + 2 * q] = dwg[k][q].x;
        ws[(4 + k) * 128 + lane * 4 + 2 * q + 1] = dwg[k][q].y;
      }
    }
    __syncthreads();
    float* prow = part + static_cast<long>(blockIdx.x) * 7 * a.F;
    for (int i = tid; i < 7 * 128; i += kTileThreads) {
      const int q = i >> 7, ch = g * 128 + (i & 127);
      if (ch >= a.F || (q == 0 ? dgamma : dconv_w) == nullptr) continue;
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < kTileWarps; ++w) v += wsum[w * 7 * 128 + i];
      if (q == 0) prow[ch] = v;
      else if (q < 4) prow[a.F + static_cast<long>(ch) * 3 + (q - 1)] = v;
      else prow[a.F + (static_cast<long>(a.F) + ch) * 3 + (q - 4)] = v;
    }
  } else {
    // ---- weight gradients: warps combine in shared memory, one global atomic per (channel, tap) and CTA
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      atomicAdd(&sacc[lane * 4 + 2 * q], dgam[q].x);
      atomicAdd(&sacc[lane * 4 + 2 * q + 1], dgam[q].y);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        atomicAdd(&sacc[(1 + k) * 128 + lane * 4 + 2 * q], dwa[k][q].x);
        atomicAdd(&sacc[(1 + k) * 128 + lane * 4 + 2 * q + 1], dwa[k][q].y);
        atomicAdd(&sacc[(4 + k) * 128 + lane * 4 + 2 * q], dwg[k][q].x);
        atomicAdd(&sacc[(4 + k) * 128 + lane * 4 + 2 * q + 1], dwg[k][q].y);
      }
    }
    __syncthreads();
    // parameter gradients in the parameters' own layout: inner gamma [F]; conv taps [2F, 3] with the value half in rows
    // [0, F) and the gate half in rows [F, 2F) (transformer.py:122-137) -- accumulated (+=), padded channels dropped
    for (int i = tid; i < 7 * 128; i += kTileThreads) {
      const int q = i >> 7, ch = g * 128 + (i & 127);
      if (ch >= a.F) continue;
      const float v = sacc[i];
      if (q == 0) { if (dgamma != nullptr) atomicAdd(&dgamma[ch], v); }
      else if (dconv_w != nullptr) {
        if (q < 4) atomicAdd(&dconv_w[static_cast<long>(ch) * 3 + (q - 1)], v);
        else atomicAdd(&dconv_w[(static_cast<long>(a.F) + ch) * 3 + (q - 4)], v);
      }
    }
  }
}

}  // namespace omlm

extern "C" {

int omlm_ffn_norm_fwd(const void* h, const float* rowsum, const float* gamma, void* hn, void* hn_copy_bf16, float* stats,
                      void* keep_bits, long M, int F, int Fp, float drop_p, const unsigned long long* seed, int layer,
                      int act_f16, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && F > 0 && Fp >= F && Fp % 128 == 0, "ffn_norm_fwd: bad shape F=%d Fp=%d", F, Fp);
  OMLM_CHECK_ARG(drop_p >= 0.f && drop_p < 1.f && (drop_p == 0.f || (seed != nullptr && keep_bits != nullptr)),
                 "ffn_norm_fwd: dropout needs a seed and a keep_bits buffer");
  auto kern = act_f16 ? ffn_norm_fwd_kernel<true> : ffn_norm_fwd_kernel<false>;
  OMLM_KLAUNCH((kern), static_cast<int>((M + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream), 
      reinterpret_cast<const __nv_bfloat16*>(h), reinterpret_cast<const float2*>(rowsum), gamma,
      reinterpret_cast<__nv_bfloat16*>(hn), reinterpret_cast<__nv_bfloat16*>(hn_copy_bf16), reinterpret_cast<float2*>(stats),
      reinterpret_cast<uint8_t*>(keep_bits), M, F, Fp,
      drop_p, seed, static_cast<uint32_t>(layer));
  OMLM_LAUNCH_CHECK();
  return 0;
}

static int ffn_mid_bwd_impl(const void* dhn, const void* hn, const void* u, const float* stats, const float* conv_w,
                            const float* gamma, const void* keep_bits, float* rowstat, int rowstat_parts, void* du, float* dgamma,
                            float* dconv_w, int B, int N, int F, int Fp, float drop_p, int act_f16, float* part, long part_bytes,
                            void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(B > 0 && N > 0 && F > 0 && Fp >= F && Fp % 128 == 0, "ffn_mid_bwd: bad shape F=%d Fp=%d", F, Fp);
  OMLM_CHECK_ARG(drop_p >= 0.f && drop_p < 1.f && (drop_p == 0.f || keep_bits != nullptr), "ffn_mid_bwd: dropout needs keep_bits");
  auto st = reinterpret_cast<cudaStream_t>(stream);
  MidArgs a{reinterpret_cast<const __nv_bfloat16*>(u), conv_w, gamma, N, F, Fp, drop_p, reinterpret_cast<const uint8_t*>(keep_bits)};
  const long M = static_cast<long>(B) * N;
  auto stats_kern = ffn_mid_bwd_stats_kernel;
  const bool det = part != nullptr;
  auto walk_kern = act_f16 ? (det ? ffn_mid_bwd_walk_kernel<true, true> : ffn_mid_bwd_walk_kernel<true, false>)
                           : (det ? ffn_mid_bwd_walk_kernel<false, true> : ffn_mid_bwd_walk_kernel<false, false>);
  const int row_blocks = B * ((N + kTileRows - 1) / kTileRows);
  if (det) OMLM_CHECK_ARG(part_bytes >= static_cast<long>(row_blocks) * 7 * F * 4, "ffn_mid_bwd_det: partials need %ld bytes",
                          static_cast<long>(row_blocks) * 7 * F * 4);
  OMLM_CHECK_ARG(rowstat_parts >= 0 && rowstat != nullptr, "ffn_mid_bwd: rowstat buffer / parts");
  if (rowstat_parts == 0) {      // no partial sums from the d_hn GEMM: one pass over (dhn, hn) here
    OMLM_KLAUNCH((stats_kern), static_cast<int>((M + 7) / 8), 256, 0, st,
        reinterpret_cast<const __nv_bfloat16*>(dhn), reinterpret_cast<const __nv_bfloat16*>(hn), gamma,
        reinterpret_cast<float2*>(rowstat), M, F, Fp, drop_p, a.keep_bits);
    OMLM_LAUNCH_CHECK();
    rowstat_parts = 1;
  }
  static bool configured = false;
  if (!configured) {
    OMLM_CUDA(cudaFuncSetAttribute(ffn_mid_bwd_walk_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileSmem));
    OMLM_CUDA(cudaFuncSetAttribute(ffn_mid_bwd_walk_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileSmem));
    OMLM_CUDA(cudaFuncSetAttribute(ffn_mid_bwd_walk_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileSmem));
    OMLM_CUDA(cudaFuncSetAttribute(ffn_mid_bwd_walk_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileSmem));
    configured = true;
  }
  dim3 grid(row_blocks, Fp / 128);
  OMLM_KLAUNCH((walk_kern), grid, kTileThreads, kTileSmem, st, a, reinterpret_cast<const __nv_bfloat16*>(dhn),
                                                                reinterpret_cast<const float2*>(stats),
                                                                reinterpret_cast<const float2*>(rowstat), rowstat_parts,
                                                                reinterpret_cast<__nv_bfloat16*>(du), dgamma, dconv_w, part);
  OMLM_LAUNCH_CHECK();
  if (det) {
    if (dgamma != nullptr) {
      const int rc = omlm_colsum(part, 7L * F, 1, dgamma, row_blocks, F, 1, stream);
      if (rc) return rc;
    }
    if (dconv_w != nullptr) return omlm_colsum(part + F, 7L * F, 1, dconv_w, row_blocks, 6 * F, 1, stream);
  }
  return 0;
}

int omlm_ffn_mid_bwd(const void* dhn, const void* hn, const void* u, const float* stats, const float* conv_w,
                     const float* gamma, const void* keep_bits, float* rowstat, int rowstat_parts, void* du, float* dgamma,
                     float* dconv_w, int B, int N, int F, int Fp, float drop_p, int act_f16, void* stream) {
  return ffn_mid_bwd_impl(dhn, hn, u, stats, conv_w, gamma, keep_bits, rowstat, rowstat_parts, du, dgamma, dconv_w, B, N, F, Fp,
                          drop_p, act_f16, nullptr, 0, stream);
}

int omlm_ffn_mid_bwd_det(const void* dhn, const void* hn, const void* u, const float* stats, const float* conv_w,
                         const float* gamma, const void* keep_bits, float* rowstat, int rowstat_parts, void* du, float* dgamma,
                         float* dconv_w, int B, int N, int F, int Fp, float drop_p, int act_f16, float* part_ws, long part_ws_bytes,
                         void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(part_ws != nullptr, "ffn_mid_bwd_det: no partials buffer");
  return ffn_mid_bwd_impl(dhn, hn, u, stats, conv_w, gamma, keep_bits, rowstat, rowstat_parts, du, dgamma, dconv_w, B, N, F, Fp,
                          drop_p, act_f16, part_ws, part_ws_bytes, stream);
}

}  // extern "C"
