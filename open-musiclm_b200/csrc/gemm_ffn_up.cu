// FFN up-projection as a persistent wgmma GEMM whose epilogue does the causal depthwise conv (k=3), GEGLU with
// exact-erf GELU and the LayerNorm row statistics.  Warpgroup 0 is the TMA producer (it keeps loading the next tile's
// operands during the epilogue); warpgroups 1 and 2 each own 64 rows of the tile for the wgmma and then share the
// conv / GEGLU phase.
//
//   u = xn @ W1^T                  [M, 2Fp]  (bf16, kept for the backward pass)      transformer.py:144
//   y[t] = w0 u[t-2] + w1 u[t-1] + w2 u[t]   per channel, zero history at sequence start   transformer.py:122-131
//   h = gelu_erf(y_gate) * y_value  [M, Fp]  (bf16)                                         transformer.py:134-137
//   rowsum[m][n tile] = (sum_c h, sum_c h^2) over the tile's 128 channels -> LN(F) statistics  transformer.py:147
//
// Tiling: 128 x 256 x 64, W1 rows interleaved so that one 256-column tile = [128 value | 128 gate] columns of the same
// 128 channels.  The conv needs rows t-1, t-2, so M tiles overlap by two rows (tile i covers rows 126 i - 2 ..
// 126 i + 125 and emits rows 126 i .. 126 i + 125; +1.6 % MMA work, no inter-CTA exchange).  The epilogue first parks
// the bf16 u tile in shared memory (row pitch 528 B), then every thread reads its own row and the two rows above it.
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/omlm_b200.h"

namespace omlm {

constexpr int kFuBM = 128, kFuBN = 256, kFuBK = 64, kFuStages = 3, kFuRowsOut = 126;
constexpr int kFuA = kFuBM * kFuBK * 2, kFuB = kFuBN * kFuBK * 2, kFuStage = kFuA + kFuB;   // 16K + 32K
constexpr int kFuUPitch = 528;                                   // bytes per row of the parked u tile
constexpr int kFuOffU = kFuStages * kFuStage;                    // 147456
constexpr int kFuOffBar = kFuOffU + kFuBM * kFuUPitch;
constexpr int kFuSmem = kFuOffBar + 256 + 1024;
constexpr int kFuThreads = 384;   // TMA warpgroup, two wgmma / epilogue warpgroups

// F16: xn, W1 arrive as fp16 and u, h leave as fp16 (all bounded by construction: LayerNorm output x weights);
// otherwise everything is bf16.
// kVarlen: sequences of their own lengths packed back to back; row m's position within its sequence is row_pos[m]
// (0 at each sequence start) instead of m % Nseq.  With hist_idx: a row m with c = hist_idx[m] >= 0 is the first row
// of a chunk that continues a sequence (position p0 > 0): its t-2 and t-1 conv inputs are rows 2c and 2c + 1 of hist
// (pre-conv u rows in the activation format, [*, 2 Fp]), and the next row's t-2 input is row 2c + 1.
template <bool F16, bool kVarlen = false>
__global__ void __launch_bounds__(kFuThreads, 1)
gemm_ffn_up_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   __nv_bfloat16* __restrict__ u_out, __nv_bfloat16* __restrict__ h_out, float* __restrict__ rowsum,
                   const float* __restrict__ conv_w, int M, int Nseq, int K, int Fp, const int* __restrict__ row_pos,
                   const __nv_bfloat16* __restrict__ hist, const int* __restrict__ hist_idx) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kFuOffBar);
  uint64_t* empty_bar = full_bar + kFuStages;
  uint8_t* usm = smem + kFuOffU;

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int m_tiles = (M + kFuRowsOut - 1) / kFuRowsOut;
  const int n_tiles = (2 * Fp) / kFuBN;
  const int kb_total = (K + kFuBK - 1) / kFuBK;
  const int work_total = m_tiles * n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB);
    for (int i = 0; i < kFuStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {   // ---------------------------------------------------------------- TMA producer
      int stage = 0; uint32_t phase = 0;
      for (int w = blockIdx.x; w < work_total; w += gridDim.x) {
        const int n_blk = w % n_tiles, m_blk = w / n_tiles;
        for (int kb = 0; kb < kb_total; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * kFuStage;
          mbar_expect_tx(&full_bar[stage], kFuStage);
          tma_load_2d(sa, &tmA, &full_bar[stage], kb * kFuBK, m_blk * kFuRowsOut - 2);   // rows < 0 / >= M are zero-filled
          tma_load_2d(sa + kFuA, &tmB, &full_bar[stage], kb * kFuBK, n_blk * kFuBN);
          if (++stage == kFuStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // -------------------------------------------------------------------------------------- consumers (256 threads)
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;                         // 64-row half of the tile for the wgmma
    const int wq = (threadIdx.x >> 5) & 3, qr = lane >> 2, qc = lane & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    const int et = threadIdx.x - 128;            // 0..255 within the consumer group
    int stage = 0; uint32_t phase = 0;
    bool first = true;
    for (int w = blockIdx.x; w < work_total; w += gridDim.x) {
      const int n_blk = w % n_tiles, m_blk = w / n_tiles;
      // varlen: lane r holds the position of row r of this warp's epilogue run (phase 2), loaded under the main loop
      // and hist_idx of that row; lane 16 holds hist_idx of the row before the run
      int lane_pos = 0, lane_hist = -1;
      if constexpr (kVarlen) {
        const long g0 = static_cast<long>(m_blk) * kFuRowsOut + (et >> 5) * 16;
        if (lane < min(16, kFuRowsOut - (et >> 5) * 16) && g0 + lane < M) {
          lane_pos = row_pos[g0 + lane];
          if (hist_idx != nullptr) lane_hist = hist_idx[g0 + lane];
        } else if (lane == 16 && hist_idx != nullptr && g0 >= 1 && g0 <= M) {
          lane_hist = hist_idx[g0 - 1];
        }
      }
      float acc[kFuBN / 2];
#pragma unroll
      for (int i = 0; i < kFuBN / 2; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < kb_total; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * kFuStage) + cw * 8192, sb = smem_u32(smem + stage * kFuStage + kFuA);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kFuBK / 16; ++k)
          Wgmma<kFuBN, F16>::template ss<0, 0>(acc, make_smem_desc(sa + k * 32, 16, 1024), make_smem_desc(sb + k * 32, 16, 1024),
                                               (kb > 0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == kFuStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_reg_fence(acc);
      if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
      // conv taps of this lane's 4 value + 4 gate channels (phase 2 mapping)
      float2 wv[3][2], wg2[3][2];                    // taps [k][channel pair]
      {
        const float4* wp = reinterpret_cast<const float4*>(conv_w + static_cast<long>(n_blk * kFuBN + lane * 4) * 3);
        const float4* gp = reinterpret_cast<const float4*>(conv_w + static_cast<long>(n_blk * kFuBN + 128 + lane * 4) * 3);
        const float4 a0 = __ldg(wp), a1 = __ldg(wp + 1), a2 = __ldg(wp + 2);
        const float4 b0 = __ldg(gp), b1 = __ldg(gp + 1), b2 = __ldg(gp + 2);
        const float fa[12] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w, a2.x, a2.y, a2.z, a2.w};
        const float fb[12] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w, b2.x, b2.y, b2.z, b2.w};
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            wv[k][q] = make_float2(fa[(2 * q) * 3 + k], fa[(2 * q + 1) * 3 + k]);
            wg2[k][q] = make_float2(fb[(2 * q) * 3 + k], fb[(2 * q + 1) * 3 + k]);
          }
      }
      if (!first) asm volatile("bar.sync 2, 256;" ::: "memory");   // everyone is done reading the previous u tile
      first = false;
      // ---- phase 1: accumulator fragment -> 16-bit -> parked u tile
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        uint8_t* urow = usm + (cw * 64 + wq * 16 + qr + hr * 8) * kFuUPitch + qc * 4;
#pragma unroll
        for (int i = 0; i < kFuBN / 8; ++i)
          *reinterpret_cast<uint32_t*>(urow + i * 16) = pack16x2<F16>(acc[4 * i + 2 * hr], acc[4 * i + 2 * hr + 1]);
      }
      asm volatile("bar.sync 2, 256;" ::: "memory");  // u tile complete
      // ---- phase 2: conv + GEGLU + row statistics.  Warp ew owns tile rows 2+16 ew .. (16 rows), lanes span the 128
      // channels (4 value + 4 gate columns each): every smem read and global store is contiguous across the warp, the
      // two history rows slide through registers, and the row sums are reduced with one transposing butterfly.
      {
        const int ew = et >> 5;
        const int t0 = 2 + ew * 16;
        const long grow0 = static_cast<long>(m_blk) * kFuRowsOut - 2 + t0;
        const int nrows = min(min(16, kFuBM - t0), static_cast<int>(min(static_cast<long>(16), M - grow0)));
        int pos = kVarlen ? __shfl_sync(0xffffffffu, lane_pos, 0) : static_cast<int>(grow0 % Nseq);
        // varlen: bit r set when row r starts a sequence (one ballot per run instead of a shuffle per row)
        const unsigned starts = kVarlen ? __ballot_sync(0xffffffffu, lane < nrows && lane_pos == 0) : 0u;
        const uint8_t* rp = usm + t0 * kFuUPitch;
        float2 xv1[2], xg1[2], xv2[2], xg2[2];        // fp32x2 pairs: channels (0,1) and (2,3) of this lane
        {
          const uint2 a = *reinterpret_cast<const uint2*>(rp - kFuUPitch + lane * 8);
          const uint2 g = *reinterpret_cast<const uint2*>(rp - kFuUPitch + 256 + lane * 8);
          xv1[0] = unpack16x2<F16>(a.x); xv1[1] = unpack16x2<F16>(a.y); xg1[0] = unpack16x2<F16>(g.x); xg1[1] = unpack16x2<F16>(g.y);
        }
        {
          const uint2 a = *reinterpret_cast<const uint2*>(rp - 2 * kFuUPitch + lane * 8);
          const uint2 g = *reinterpret_cast<const uint2*>(rp - 2 * kFuUPitch + 256 + lane * 8);
          xv2[0] = unpack16x2<F16>(a.x); xv2[1] = unpack16x2<F16>(a.y); xg2[0] = unpack16x2<F16>(g.x); xg2[1] = unpack16x2<F16>(g.y);
        }
        if (pos == 1) { xv2[0] = xv2[1] = xg2[0] = xg2[1] = make_float2(0.f, 0.f); }   // row t-2 belongs to the previous sequence
        // varlen with history: bit r set when row r starts a chunk with history rows
        const unsigned hstarts = kVarlen ? __ballot_sync(0xffffffffu, lane < nrows && lane_hist >= 0) : 0u;
        if constexpr (kVarlen) {
          const int prev_c = __shfl_sync(0xffffffffu, lane_hist, 16);
          if (prev_c >= 0) {   // the run's first row is the second row of a chunk: its t-2 input is that chunk's t-1 history row
            const uint8_t* hp = reinterpret_cast<const uint8_t*>(hist) + (2L * prev_c + 1) * (4L * Fp) + n_blk * 512 + lane * 8;
            const uint2 a = *reinterpret_cast<const uint2*>(hp), g = *reinterpret_cast<const uint2*>(hp + 256);
            xv2[0] = unpack16x2<F16>(a.x); xv2[1] = unpack16x2<F16>(a.y); xg2[0] = unpack16x2<F16>(g.x); xg2[1] = unpack16x2<F16>(g.y);
          }
        }
        float st[32];
        __nv_bfloat16* ug = u_out + grow0 * (2L * Fp) + n_blk * kFuBN + lane * 8;
        __nv_bfloat16* hg = h_out + grow0 * static_cast<long>(Fp) + n_blk * 128 + lane * 4;
#pragma unroll
        for (int r = 0; r < 16; ++r) {
          float s1 = 0.f, s2 = 0.f;
          if (r < nrows) {
            const uint8_t* rr = rp + r * kFuUPitch;
            *reinterpret_cast<uint4*>(ug + static_cast<long>(r) * (2L * Fp)) = *reinterpret_cast<const uint4*>(rr + lane * 16);
            const uint2 a = *reinterpret_cast<const uint2*>(rr + lane * 8);
            const uint2 g = *reinterpret_cast<const uint2*>(rr + 256 + lane * 8);
            const float2 xv0[2] = {unpack16x2<F16>(a.x), unpack16x2<F16>(a.y)}, xg0[2] = {unpack16x2<F16>(g.x), unpack16x2<F16>(g.y)};
            // one test per row on the common path: a sequence start or (varlen) a chunk start with history
            if (kVarlen ? (((starts | hstarts) >> r) & 1u) != 0 : pos == 0) {
              if (!kVarlen || ((starts >> r) & 1u) != 0) {   // sequence start: no history (the zeros then slide into the t-2 slot for the next row)
                const float2 z = make_float2(0.f, 0.f);
                xv1[0] = xv1[1] = xg1[0] = xg1[1] = z;
                xv2[0] = xv2[1] = xg2[0] = xg2[1] = z;
              } else {                                       // chunk start: history rows 2c (t-2), 2c + 1 (t-1)
                const uint8_t* hp = reinterpret_cast<const uint8_t*>(hist) + 2L * hist_idx[grow0 + r] * (4L * Fp) + n_blk * 512 + lane * 8;
                const uint2 a2 = *reinterpret_cast<const uint2*>(hp), g2 = *reinterpret_cast<const uint2*>(hp + 256);
                const uint2 a1 = *reinterpret_cast<const uint2*>(hp + 4L * Fp), g1 = *reinterpret_cast<const uint2*>(hp + 4L * Fp + 256);
                xv2[0] = unpack16x2<F16>(a2.x); xv2[1] = unpack16x2<F16>(a2.y); xg2[0] = unpack16x2<F16>(g2.x); xg2[1] = unpack16x2<F16>(g2.y);
                xv1[0] = unpack16x2<F16>(a1.x); xv1[1] = unpack16x2<F16>(a1.y); xg1[0] = unpack16x2<F16>(g1.x); xg1[1] = unpack16x2<F16>(g1.y);
              }
            }
            float2 h[2], sq = make_float2(0.f, 0.f), sm = sq;
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              const float2 yv = fma2(wv[0][q], xv2[q], fma2(wv[1][q], xv1[q], mul2(wv[2][q], xv0[q])));
              const float2 yg = fma2(wg2[0][q], xg2[q], fma2(wg2[1][q], xg1[q], mul2(wg2[2][q], xg0[q])));
              h[q] = mul2(gelu_erf2(yg), yv);
              sm = add2(sm, h[q]);
              sq = fma2(h[q], h[q], sq);
              xv2[q] = xv1[q]; xv1[q] = xv0[q];
              xg2[q] = xg1[q]; xg1[q] = xg0[q];
            }
            s1 = sm.x + sm.y; s2 = sq.x + sq.y;
            *reinterpret_cast<uint2*>(hg + static_cast<long>(r) * Fp) = make_uint2(pack16x2<F16>(h[0].x, h[0].y), pack16x2<F16>(h[1].x, h[1].y));
            if (!kVarlen && ++pos == Nseq) pos = 0;
          }
          st[2 * r] = s1;
          st[2 * r + 1] = s2;
        }
        // transposing butterfly: lane l ends up with the warp-wide sum of st[l]
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1) {
          const bool hi = (lane & off) != 0;
#pragma unroll
          for (int i = 0; i < off; ++i) {
            const float send = hi ? st[i] : st[i + off];
            const float keep = hi ? st[i + off] : st[i];
            st[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
          }
        }
        // per-tile partial sums, one slot per (row, n tile): omlm_ffn_norm_fwd adds the n_tiles partials in a fixed
        // order, so the forward pass stays bit-reproducible (fp32 atomics would make the LayerNorm statistics, and
        // after six layers of bf16 rounding every logit, depend on CTA timing)
        if ((lane >> 1) < nrows) rowsum[(grow0 + (lane >> 1)) * (2L * n_tiles) + 2 * n_blk + (lane & 1)] = st[0];
      }
    }
  }
}

}  // namespace omlm

#ifndef OMLM_GEMM_FFN_UP_VARLEN
extern "C" int omlm_gemm_ffn_up(const void* xn, const void* w1_packed, const float* conv_w_packed, void* u_out, void* h_out,
                                float* rowsum, int M, int Nseq, int K, int Fp, int act_f16, int max_ctas, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && Nseq > 0 && K > 0 && K % 8 == 0 && Fp > 0 && Fp % 128 == 0, "gemm_ffn_up: bad shape M=%d K=%d Fp=%d", M, K, Fp);
  CUtensorMap tmA, tmB;
  int rc = make_tmap_bf16_2d(&tmA, xn, static_cast<uint64_t>(K), static_cast<uint64_t>(M), static_cast<uint64_t>(K) * 2, 64, kFuBM);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmB, w1_packed, static_cast<uint64_t>(K), static_cast<uint64_t>(2 * Fp), static_cast<uint64_t>(K) * 2, 64, kFuBN);
  if (rc) return rc;
  static bool configured = false;
  if (!configured) {
    OMLM_CUDA(cudaFuncSetAttribute(gemm_ffn_up_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFuSmem));
    OMLM_CUDA(cudaFuncSetAttribute(gemm_ffn_up_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFuSmem));
    configured = true;
  }
  const int m_tiles = (M + kFuRowsOut - 1) / kFuRowsOut, n_tiles = (2 * Fp) / kFuBN;
  int grid = num_sms();
  if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
  if (m_tiles * n_tiles < grid) grid = m_tiles * n_tiles;
  auto kern = act_f16 ? gemm_ffn_up_kernel<true> : gemm_ffn_up_kernel<false>;
  OMLM_KLAUNCH((kern), grid, kFuThreads, kFuSmem, reinterpret_cast<cudaStream_t>(stream), 
      tmA, tmB, reinterpret_cast<__nv_bfloat16*>(u_out), reinterpret_cast<__nv_bfloat16*>(h_out), rowsum, conv_w_packed, M,
      Nseq, K, Fp, nullptr, nullptr, nullptr);
  OMLM_LAUNCH_CHECK();
  return 0;
}
#else
static int gemm_ffn_up_varlen_launch(const void* xn, const void* w1_packed, const float* conv_w_packed, void* u_out, void* h_out,
                                     float* rowsum, const int* row_pos, const void* hist, const int* hist_idx, int M, int K, int Fp,
                                     int act_f16, int max_ctas, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && K > 0 && K % 8 == 0 && Fp > 0 && Fp % 128 == 0 && row_pos != nullptr,
                 "gemm_ffn_up_varlen: bad shape M=%d K=%d Fp=%d", M, K, Fp);
  CUtensorMap tmA, tmB;
  int rc = make_tmap_bf16_2d(&tmA, xn, static_cast<uint64_t>(K), static_cast<uint64_t>(M), static_cast<uint64_t>(K) * 2, 64, kFuBM);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmB, w1_packed, static_cast<uint64_t>(K), static_cast<uint64_t>(2 * Fp), static_cast<uint64_t>(K) * 2, 64, kFuBN);
  if (rc) return rc;
  static bool configured = false;
  if (!configured) {
    OMLM_CUDA(cudaFuncSetAttribute(gemm_ffn_up_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFuSmem));
    OMLM_CUDA(cudaFuncSetAttribute(gemm_ffn_up_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kFuSmem));
    configured = true;
  }
  const int m_tiles = (M + kFuRowsOut - 1) / kFuRowsOut, n_tiles = (2 * Fp) / kFuBN;
  int grid = num_sms();
  if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
  if (m_tiles * n_tiles < grid) grid = m_tiles * n_tiles;
  auto kern = act_f16 ? gemm_ffn_up_kernel<true, true> : gemm_ffn_up_kernel<false, true>;
  OMLM_KLAUNCH((kern), grid, kFuThreads, kFuSmem, reinterpret_cast<cudaStream_t>(stream),
      tmA, tmB, reinterpret_cast<__nv_bfloat16*>(u_out), reinterpret_cast<__nv_bfloat16*>(h_out), rowsum, conv_w_packed, M,
      1, K, Fp, row_pos, reinterpret_cast<const __nv_bfloat16*>(hist), hist_idx);
  OMLM_LAUNCH_CHECK();
  return 0;
}

extern "C" int omlm_gemm_ffn_up_varlen(const void* xn, const void* w1_packed, const float* conv_w_packed, void* u_out,
                                       void* h_out, float* rowsum, const int* row_pos, int M, int K, int Fp, int act_f16,
                                       int max_ctas, void* stream) {
  return gemm_ffn_up_varlen_launch(xn, w1_packed, conv_w_packed, u_out, h_out, rowsum, row_pos, nullptr, nullptr, M, K, Fp,
                                   act_f16, max_ctas, stream);
}

extern "C" int omlm_gemm_ffn_up_chunk(const void* xn, const void* w1_packed, const float* conv_w_packed, void* u_out,
                                      void* h_out, float* rowsum, const int* row_pos, const void* hist, const int* hist_idx, int M,
                                      int K, int Fp, int act_f16, int max_ctas, void* stream) {
  OMLM_CHECK_ARG(hist != nullptr && hist_idx != nullptr, "gemm_ffn_up_chunk: hist and hist_idx are required");
  return gemm_ffn_up_varlen_launch(xn, w1_packed, conv_w_packed, u_out, h_out, rowsum, row_pos, hist, hist_idx, M, K, Fp,
                                   act_f16, max_ctas, stream);
}
#endif
