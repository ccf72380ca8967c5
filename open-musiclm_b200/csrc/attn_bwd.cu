// Fused causal multi-query cosine-sim attention, backward (flash-style recompute; see attn_common.cuh
// for the folded-row layout that turns the MQA head reductions into ordinary row reductions).
//
// Autograd of transformer.py:304-331 for the self-attention instance:
//   P = softmax(8 qn.kn + table[hh, i-j] + masks);  O = P v
//   dV = P^T dO;  dS = P * (dO v^T - D), D = rowsum(dO * O);  dQn = 8 dS kn;  dKn = 8 dS^T qn;
//   dTable[hh, i-j] += dS   (Toeplitz: summed over batch, positions and layers)
//
// Work unit = (batch b, key tile of 128 keys, chunk of query-row tiles).  Each of the 8 warps owns 16
// keys and keeps S^T / dP^T tiles (keys x rows) in registers so that P^T and dS^T are directly the
// A operands of dV += P^T dO and dK += dS^T Q; dS goes through smem once for dQ += dS K.
// dQn is accumulated with vector red.global.add (fp32); dKn/dVn likewise across row chunks.
#include "attn_common.cuh"
#include "../../include/omlm_b200.h"

namespace omlm {

constexpr int kBQ = 64;     // folded query rows per tile
constexpr int kBKV = 128;   // keys per CTA
constexpr int kBwdThreads = 256;
constexpr int kDbW = 256;   // circular dbias window per head
constexpr int kBwdMaxHeads = 16;
constexpr int kDsPad = 64;  // zero key-rows in front of the dS^T tile (>= positions per 64-row tile - 1)

struct AttnBwdSmem {
  uint8_t k[kBKV * 128];
  uint8_t v[kBKV * 128];
  uint8_t q[2][kBQ * 128];
  uint8_t d_o[2][kBQ * 128];
  uint8_t ds[(kDsPad + kBKV + 80) * 128];   // [64 zero rows | dS^T as [key][row] bf16 | 80 zero rows]: guard bands for the diagonal MMA
  float lse[2][kBQ];
  float dsum[2][kBQ];
  int rowinfo[kBQ];
  float kneg[kBKV];
  float bias[kBwdMaxHeads * (kBQ + 1 + kBKV)];
  float dbias[kBwdMaxHeads * kDbW];
};

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// D[r] = sum_d dO[r, d] * O[r, d]   (one 8-lane group per row of 64)
__global__ void __launch_bounds__(256)
attn_bwd_dsum_kernel(const __nv_bfloat16* __restrict__ d_o, const __nv_bfloat16* __restrict__ o,
                     float* __restrict__ dsum, long rows) {
  const long r = (static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 3;
  const int sub = threadIdx.x & 7;
  float s = 0.f;
  if (r < rows) {
    const uint4 a = *reinterpret_cast<const uint4*>(d_o + r * 64 + sub * 8);
    const uint4 b = *reinterpret_cast<const uint4*>(o + r * 64 + sub * 8);
    const uint32_t aa[4] = {a.x, a.y, a.z, a.w}, bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 x = unpack_bf16x2(aa[i]), y = unpack_bf16x2(bb[i]);
      s += x.x * y.x + x.y * y.y;
    }
  }
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  if (r < rows && sub == 0) dsum[r] = s;
}

__global__ void __launch_bounds__(kBwdThreads, 1)
attn_bwd_kernel(const __nv_bfloat16* __restrict__ qn, const __nv_bfloat16* __restrict__ kvn,
                const __nv_bfloat16* __restrict__ d_o, const float* __restrict__ lse2,
                const float* __restrict__ dsum, const float* __restrict__ table, int table_ld,
                const unsigned char* __restrict__ key_mask, float* __restrict__ dqn,
                float* __restrict__ dkvn, float* __restrict__ dtable, int N, int h, float scale,
                int tiles_per_chunk, int units_per_batch) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  AttnBwdSmem& sm = *reinterpret_cast<AttnBwdSmem*>(smem_raw);
  const int R = N * h;
  const int n_row_tiles = (R + kBQ - 1) / kBQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;

  // ---- decode the work unit: (b, key tile, row-tile chunk); units are enumerated key tile by key tile
  const int b = blockIdx.x / units_per_batch;
  int u = blockIdx.x - b * units_per_batch;
  int kt = 0, rt_begin = 0, rt_end = 0;
  for (;; ++kt) {
    const int first = (kt * kBKV * h) / kBQ;  // first row tile that can see key tile kt
    const int chunks = (n_row_tiles - first + tiles_per_chunk - 1) / tiles_per_chunk;
    if (u < chunks) { rt_begin = first + u * tiles_per_chunk; rt_end = min(n_row_tiles, rt_begin + tiles_per_chunk); break; }
    u -= chunks;
  }
  const int j0 = kt * kBKV;

  const __nv_bfloat16* qb = qn + (static_cast<long long>(b) * R) * 64;
  const __nv_bfloat16* dob = d_o + (static_cast<long long>(b) * R) * 64;
  const __nv_bfloat16* kvb = kvn + (static_cast<long long>(b) * N) * 128;
  const float* lseb = lse2 + static_cast<long long>(b) * R;
  const float* dsb = dsum + static_cast<long long>(b) * R;
  const uint32_t sk = smem_u32(sm.k), sv = smem_u32(sm.v), sds = smem_u32(sm.ds);

  // ---- K/V tile (once) + first Q/dO tile
  for (int idx = threadIdx.x; idx < kBKV * 16; idx += kBwdThreads) {
    const int row = idx >> 4, c = idx & 15;
    const bool ok = (j0 + row) < N;
    cp_async16((c < 8 ? sk : sv) + tile_off(row, c & 7), kvb + static_cast<long long>(ok ? j0 + row : 0) * 128 + c * 8, ok);
  }
  if (threadIdx.x < kBKV) {
    const int j = j0 + threadIdx.x;
    const bool vis = (j < N) && (key_mask == nullptr || key_mask[static_cast<long long>(b) * N + j] != 0);
    sm.kneg[threadIdx.x] = vis ? 0.f : -INFINITY;
  }
  for (int i = threadIdx.x; i < kBwdMaxHeads * kDbW; i += kBwdThreads) sm.dbias[i] = 0.f;
  for (int i = threadIdx.x; i < kDsPad * 32; i += kBwdThreads) reinterpret_cast<uint32_t*>(sm.ds)[i] = 0u;
  for (int i = threadIdx.x; i < 80 * 32; i += kBwdThreads) reinterpret_cast<uint32_t*>(sm.ds + (kDsPad + kBKV) * 128)[i] = 0u;
  auto load_q = [&](int rt, int buf) {
    const int r0 = rt * kBQ;
    const uint32_t sq = smem_u32(sm.q[buf]), sdo = smem_u32(sm.d_o[buf]);
    for (int idx = threadIdx.x; idx < kBQ * 16; idx += kBwdThreads) {
      const int row = idx >> 4, c = idx & 15;
      const bool ok = (r0 + row) < R;
      const long long off = static_cast<long long>(ok ? r0 + row : 0) * 64 + (c & 7) * 8;
      cp_async16((c < 8 ? sq : sdo) + tile_off(row, c & 7), (c < 8 ? qb : dob) + off, ok);
    }
    if (threadIdx.x < kBQ) {
      const int r = r0 + threadIdx.x;
      sm.lse[buf][threadIdx.x] = r < R ? lseb[r] : INFINITY;
      sm.dsum[buf][threadIdx.x] = r < R ? dsb[r] : 0.f;
    }
  };
  load_q(rt_begin, 0);
  cp_async_commit();

  float dk[8][4], dv[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) { dk[n][0] = dk[n][1] = dk[n][2] = dk[n][3] = 0.f; dv[n][0] = dv[n][1] = dv[n][2] = dv[n][3] = 0.f; }
  uint32_t kf[4][4], vf[4][4];
  const float sc2 = scale * kLog2e;
  const int key_a = warp * 16 + g, key_b = key_a + 8;  // local key rows owned by this thread
  int flushed_lo = 0;                                   // dbias bins below this delta are already in global memory

  for (int rt = rt_begin; rt < rt_end; ++rt) {
    const int buf = (rt - rt_begin) & 1;
    const int r0 = rt * kBQ;
    const int i_min = r0 / h, i_max = min(N - 1, (r0 + kBQ - 1) / h);
    const int W = (i_max - i_min) + kBKV;
    const int delta_min = i_min - (j0 + kBKV - 1);
    __syncthreads();  // previous tile fully consumed (q/dO buffer buf^1, ds, bias, rowinfo, dbias adds)
    if (rt + 1 < rt_end) load_q(rt + 1, buf ^ 1);
    cp_async_commit();
    // flush dbias bins that slid out of the window, then build this tile's bias slice and row info
    {
      const int new_lo = max(delta_min, 0);
      const int span = new_lo - flushed_lo;
      for (int idx = threadIdx.x; idx < h * max(span, 0); idx += kBwdThreads) {
        const int hh = idx / span, d = flushed_lo + (idx - hh * span);
        float* slot = &sm.dbias[hh * kDbW + (d & (kDbW - 1))];
        const float val = *slot;
        if (val != 0.f) atomicAdd(&dtable[hh * table_ld + d], val);
        *slot = 0.f;
      }
      if (span > 0) flushed_lo = new_lo;
      for (int idx = threadIdx.x; idx < h * W; idx += kBwdThreads) {
        const int hh = idx / W, w = idx - hh * W;
        const int delta = delta_min + w;
        sm.bias[idx] = (delta < 0) ? -INFINITY : table[hh * table_ld + delta] * kLog2e;
      }
      if (threadIdx.x < kBQ) {
        const int r = min(r0 + threadIdx.x, R - 1);
        const int i = r / h, hh = r - i * h;
        sm.rowinfo[threadIdx.x] = (hh << 16) | (i - i_min);  // head, position offset
      }
    }
    cp_async_wait<1>();
    __syncthreads();
    if (rt == rt_begin) {
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) { load_a_frag(sk, warp * 16, ks, lane, kf[ks]); load_a_frag(sv, warp * 16, ks, lane, vf[ks]); }
    }
    const uint32_t sq = smem_u32(sm.q[buf]), sdo = smem_u32(sm.d_o[buf]);
    // ---- S^T = K Q^T and dP^T = V dO^T   (16 keys x 64 rows per warp)
    float s[8][4], dp[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) { s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f; dp[n][0] = dp[n][1] = dp[n][2] = dp[n][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bq[4], bd[4];
        load_b_frag_nk(sq, np * 16, ks, lane, bq);
        load_b_frag_nk(sdo, np * 16, ks, lane, bd);
        mma_bf16(s[2 * np], kf[ks][0], kf[ks][1], kf[ks][2], kf[ks][3], bq[0], bq[1]);
        mma_bf16(s[2 * np + 1], kf[ks][0], kf[ks][1], kf[ks][2], kf[ks][3], bq[2], bq[3]);
        mma_bf16(dp[2 * np], vf[ks][0], vf[ks][1], vf[ks][2], vf[ks][3], bd[0], bd[1]);
        mma_bf16(dp[2 * np + 1], vf[ks][0], vf[ks][1], vf[ks][2], vf[ks][3], bd[2], bd[3]);
      }
    }
    // ---- P^T, dS^T
    const float knA = sm.kneg[key_a], knB = sm.kneg[key_b];
    uint32_t pf[8][2], dsf[8][2];
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = n * 8 + 2 * t + e;  // local row index of the query tile
        const int info = sm.rowinfo[col];
        const int hh = info >> 16, di = info & 0xffff;
        const float l2 = sm.lse[buf][col], dsm = sm.dsum[buf][col];
        const int base = hh * W + di + (kBKV - 1);
        const float pa = exp2f(fmaf(s[n][e], sc2, sm.bias[base - key_a] + knA) - l2);
        const float pb = exp2f(fmaf(s[n][2 + e], sc2, sm.bias[base - key_b] + knB) - l2);
        const float da = pa * (dp[n][e] - dsm), db = pb * (dp[n][2 + e] - dsm);
        s[n][e] = pa; s[n][2 + e] = pb;
        dp[n][e] = da; dp[n][2 + e] = db;
      }
      pf[n][0] = pack_bf16x2(s[n][0], s[n][1]);   pf[n][1] = pack_bf16x2(s[n][2], s[n][3]);
      dsf[n][0] = pack_bf16x2(dp[n][0], dp[n][1]); dsf[n][1] = pack_bf16x2(dp[n][2], dp[n][3]);
      // dS^T to smem as [key][row]: rows 2t,2t+1 of chunk n
      *reinterpret_cast<uint32_t*>(sm.ds + tile_off(key_a + kDsPad, n) + t * 4) = dsf[n][0];
      *reinterpret_cast<uint32_t*>(sm.ds + tile_off(key_b + kDsPad, n) + t * 4) = dsf[n][1];
    }
    // ---- dV += P^T dO ;  dK += dS^T Q    (k = 64 rows of the tile)
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bd[4], bq[4];
        load_b_frag_kn(sdo, kk * 16, np * 16, lane, bd);
        load_b_frag_kn(sq, kk * 16, np * 16, lane, bq);
        mma_bf16(dv[2 * np], pf[2 * kk][0], pf[2 * kk][1], pf[2 * kk + 1][0], pf[2 * kk + 1][1], bd[0], bd[1]);
        mma_bf16(dv[2 * np + 1], pf[2 * kk][0], pf[2 * kk][1], pf[2 * kk + 1][0], pf[2 * kk + 1][1], bd[2], bd[3]);
        mma_bf16(dk[2 * np], dsf[2 * kk][0], dsf[2 * kk][1], dsf[2 * kk + 1][0], dsf[2 * kk + 1][1], bq[0], bq[1]);
        mma_bf16(dk[2 * np + 1], dsf[2 * kk][0], dsf[2 * kk][1], dsf[2 * kk + 1][0], dsf[2 * kk + 1][1], bq[2], bq[3]);
      }
    }
    __syncthreads();  // dS tile complete
    // ---- dTable[hh, i-j] += dS on the tensor cores.  For position p of this tile the rows r = (p, hh) of dS^T
    // [key][row] contribute dS^T[key][r] to bin delta = i_min + p - key.  Shifting the tile DOWN by p key-rows
    // (free: ldmatrix takes per-row addresses) aligns every position on delta = i_min - j0 - k', so
    //     out[k'][hh] = sum_p  dS^T[k' + p][:] . E_p[:, hh],   E_p[r][hh] = [row r is (position p, head hh)]
    // is a sum of small MMAs with 0/1 B fragments built from rowinfo.  Each (k', hh) bin then has one owner thread.
    {
      const int P = i_max - i_min + 1;
      const int n_heads_tiles = (h + 7) >> 3;
      for (int mt = warp; mt < (kDsPad + kBKV) / 16; mt += 8) {      // output rows k' = kb0 .. kb0+15, k' in [-64, 127]
        const int kb0 = mt * 16 - kDsPad;
        if (kb0 + 15 < -(P - 1)) continue;                             // no position can reach these rows
        for (int nt = 0; nt < n_heads_tiles; ++nt) {
          float acc[4] = {0.f, 0.f, 0.f, 0.f};
          for (int p = 0; p < P; ++p) {
            const int rbase = (i_min + p) * h - r0;                    // local row of (position p, head 0)
            const int lo = max(0, rbase), hi = min(kBQ, rbase + h);
            if (lo >= hi) continue;
            for (int ks = lo >> 4; ks <= (hi - 1) >> 4; ++ks) {
              // B fragment (k = tile row, n = head), built arithmetically: 1.0 where row is (position p, head g + 8 nt)
              const int want = rbase + g + 8 * nt;                     // the one local row that carries this head at position p
              const int ra = ks * 16 + 2 * t;
              const bool okh = (g + 8 * nt) < h;
              const uint32_t b0 = (okh && ra == want ? 0x3F80u : 0u) | (okh && ra + 1 == want ? 0x3F800000u : 0u);
              const uint32_t b1 = (okh && ra + 8 == want ? 0x3F80u : 0u) | (okh && ra + 9 == want ? 0x3F800000u : 0u);
              uint32_t af[4];
              load_a_frag(sds, kb0 + kDsPad + p, ks, lane, af);      // rows (k' + p) of dS^T, shifted by the position
              mma_bf16(acc, af[0], af[1], af[2], af[3], b0, b1);
            }
          }
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int kp = kb0 + g + (e >> 1) * 8;
            const int hh = nt * 8 + 2 * t + (e & 1);
            const int delta = i_min - j0 - kp;
            if (hh < h && delta >= 0 && acc[e] != 0.f) sm.dbias[hh * kDbW + (delta & (kDbW - 1))] += acc[e];
          }
        }
      }
    }
    // ---- dQ[64 rows x 64 d] += dS K : warp w -> rows 16*(w&3).., d half (w>>2)*32, k over the 128 keys
    {
      const int m0 = (warp & 3) * 16, n0 = (warp >> 2) * 32;
      float dq[4][4];
#pragma unroll
      for (int n = 0; n < 4; ++n) { dq[n][0] = dq[n][1] = dq[n][2] = dq[n][3] = 0.f; }
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) {
        uint32_t af[4];
        load_a_frag_t(sds, kk * 16 + kDsPad, m0, lane, af);
#pragma unroll
        for (int np = 0; np < 2; ++np) {
          uint32_t bk[4];
          load_b_frag_kn(sk, kk * 16, n0 + np * 16, lane, bk);
          mma_bf16(dq[2 * np], af[0], af[1], af[2], af[3], bk[0], bk[1]);
          mma_bf16(dq[2 * np + 1], af[0], af[1], af[2], af[3], bk[2], bk[3]);
        }
      }
      const int rowA = r0 + m0 + g, rowB = rowA + 8;
      float* dqb = dqn + (static_cast<long long>(b) * R) * 64;
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        const int d0 = n0 + n * 8 + 2 * t;
        if (rowA < R) red_add_v2(dqb + static_cast<long long>(rowA) * 64 + d0, dq[n][0] * scale, dq[n][1] * scale);
        if (rowB < R) red_add_v2(dqb + static_cast<long long>(rowB) * 64 + d0, dq[n][2] * scale, dq[n][3] * scale);
      }
    }
  }
  cp_async_wait<0>();
  __syncthreads();
  // ---- flush the remaining dbias window
  {
    const int last_r0 = (rt_end - 1) * kBQ;
    const int d_hi = min(N - 1, (last_r0 + kBQ - 1) / h) - j0;  // largest delta touched
    const int span = d_hi - flushed_lo + 1;
    for (int idx = threadIdx.x; idx < h * max(span, 0); idx += kBwdThreads) {
      const int hh = idx / span, d = flushed_lo + (idx - hh * span);
      const float val = sm.dbias[hh * kDbW + (d & (kDbW - 1))];
      if (val != 0.f) atomicAdd(&dtable[hh * table_ld + d], val);
    }
  }
  // ---- dK (x scale), dV -> global fp32 (accumulated across row chunks)
  {
    float* dkb = dkvn + (static_cast<long long>(b) * N) * 128;
    const int jA = j0 + key_a, jB = j0 + key_b;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      const int d0 = n * 8 + 2 * t;
      if (jA < N) {
        red_add_v2(dkb + static_cast<long long>(jA) * 128 + d0, dk[n][0] * scale, dk[n][1] * scale);
        red_add_v2(dkb + static_cast<long long>(jA) * 128 + 64 + d0, dv[n][0], dv[n][1]);
      }
      if (jB < N) {
        red_add_v2(dkb + static_cast<long long>(jB) * 128 + d0, dk[n][2] * scale, dk[n][3] * scale);
        red_add_v2(dkb + static_cast<long long>(jB) * 128 + 64 + d0, dv[n][2], dv[n][3]);
      }
    }
  }
}

}  // namespace omlm

extern "C" int omlm_attn_bwd(const void* qn, const void* kvn, const void* d_o, const void* o, const float* lse2,
                             const float* table, int table_ld, const unsigned char* key_mask, float* dsum_scratch,
                             float* dqn, float* dkvn, float* dtable, int B, int N, int heads, float scale,
                             void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(B > 0 && N > 0 && heads > 0 && heads <= kBwdMaxHeads, "attn_bwd: unsupported shape (heads=%d)", heads);
  OMLM_CHECK_ARG(table_ld >= N, "attn_bwd: bias table shorter than the sequence");
  auto st = reinterpret_cast<cudaStream_t>(stream);
  const long rows = static_cast<long>(B) * N * heads;
  OMLM_KLAUNCH((attn_bwd_dsum_kernel), static_cast<int>((rows * 8 + 255) / 256), 256, 0, st, 
      reinterpret_cast<const __nv_bfloat16*>(d_o), reinterpret_cast<const __nv_bfloat16*>(o), dsum_scratch, rows);
  OMLM_LAUNCH_CHECK();
  static bool configured = false;
  const int smem = static_cast<int>(sizeof(AttnBwdSmem));
  if (!configured) {
    OMLM_CUDA(cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  const int R = N * heads;
  const int n_row_tiles = (R + kBQ - 1) / kBQ;
  const int n_key_tiles = (N + kBKV - 1) / kBKV;
  // chunk the row range so that the grid has a few waves of roughly equal units
  int tiles_per_chunk = n_row_tiles;
  for (int cand = 8; cand <= n_row_tiles; cand *= 2) {
    long units = 0;
    for (int kt = 0; kt < n_key_tiles; ++kt) {
      const int first = (kt * kBKV * heads) / kBQ;
      units += (n_row_tiles - first + cand - 1) / cand;
    }
    if (units * B <= 4L * num_sms()) { tiles_per_chunk = cand; break; }
  }
  int units_per_batch = 0;
  for (int kt = 0; kt < n_key_tiles; ++kt) {
    const int first = (kt * kBKV * heads) / kBQ;
    units_per_batch += (n_row_tiles - first + tiles_per_chunk - 1) / tiles_per_chunk;
  }
  OMLM_KLAUNCH((attn_bwd_kernel), B * units_per_batch, kBwdThreads, smem, st, 
      reinterpret_cast<const __nv_bfloat16*>(qn), reinterpret_cast<const __nv_bfloat16*>(kvn),
      reinterpret_cast<const __nv_bfloat16*>(d_o), lse2, dsum_scratch, table, table_ld, key_mask, dqn, dkvn, dtable,
      N, heads, scale, tiles_per_chunk, units_per_batch);
  OMLM_LAUNCH_CHECK();
  return 0;
}
