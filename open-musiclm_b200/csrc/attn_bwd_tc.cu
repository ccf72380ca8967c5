// Fused causal multi-query cosine-sim attention, backward, on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
// Autograd of transformer.py:304-331.  Folded-row layout: R = N*h query rows per batch element share one K/V head
// (row r = i*h + head).  Work unit = (batch, 128-key tile, chunk of 64-row query tiles).  384 threads:
//
//   warpgroup 0     TMA producer: the K/V tile once, Q/dO row tiles through a 2-stage ring
//   warpgroups 1,2  64 keys each, per row tile (all wgmma M = 64, operands in 128B-swizzled smem):
//                      S  = Q K^T,  dP = dO V^T          (registers)
//                      P = exp2(s - lse), dS = P (dP - D) in fp32 registers; P, dS -> bf16 [row][key] smem tiles
//                      dV += P^T dO,  dK += dS^T Q        (A read MN-major; accumulated in registers over the chunk)
//                      dQ  = dS K                         (per tile, red.global.add.v2.f32 into dqn)
//                   the bias enters from a per-tile Toeplitz window in shared memory (per head), copied by cp.async
//                   one tile ahead, while the previous tile's dV, dK and dQ run; lse2 and D are loaded as far ahead.
//                   The bias gradient dTable[hh, i-j] += dS: the fp32 dS tile is staged in shared memory and, while dV,
//                   dK and dQ run, each thread owns (head, diagonal) pairs and sums them in row order into its
//                   warpgroup's table (no shared-memory float atomics); the two tables are flushed once per unit.
//
// Deterministic variant (DET, omlm_attn_bwd_tc_det): the same work units and arithmetic, with every float reduction in a
// fixed order.  dQ of a row tile and dK|dV of a key tile are still added with red.global.add, but in turns enforced by
// per-tile counters (the deterministic backward of FlashAttention-3): row tile rt takes the (key tile, warpgroup) pairs
// in the order (0,0), (0,1), (1,0), ...; key tile kt takes its row chunks in chunk order.  A turn only ever waits for
// a CTA with a lower block index, which the hardware dispatched first, so the waits cannot deadlock; a wait that does not
// end within seconds sets an error word and gives up instead of hanging.  The two diagonal tables of a unit are added
// into a partial table in global memory (the default adds them to dtable with one atomic per entry), and a second
// kernel adds the partial tables to dtable in unit order.  After a time-out the error word stays set and later calls
// skip their waits, until the caller clears it: their sums are then added in arrival order (correct up to rounding, not
// reproducible).
//
// Without the bias gradient (DTAB = false, dtable == NULL: nothing trains the bias table) the kernel skips the fp32 dS
// staging, the diagonal sums, the two per-warpgroup tables and their flush, and in DET mode the partial tables and the
// reduce kernel.  Everything else, and with it the order of every dQ, dK and dV sum, is unchanged: dQ and dK|dV are
// bit-identical to the variant with the table.
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/omlm_b200.h"
#include <stdlib.h>
#include <algorithm>
#include <array>
#include <functional>
#include <map>
#include <mutex>
#include <vector>

namespace omlm {

constexpr int kBtThreads = 384;
constexpr int kBtBQ = 64, kBtBK = 128;
constexpr float kBtL2e = 1.4426950408889634f;

constexpr int kBoK = 0, kBoV = 16384, kBoQ = 32768 /*2 stages x 8K*/, kBoDO = 49152 /*2 x 8K*/;
constexpr int kBoP = 65536 /*2 wg x 8K*/, kBoDS = 81920 /*2 wg x 8K*/, kBoBar = 98304 /*64 B*/;
constexpr int kBoSds = 98368;     // fp32 dS tiles [2 wg][64 rows][kBtSdsLd]
constexpr int kBtMaxSmem = 232448;
constexpr int kBtSdsLd = 72;      // padded row: the fragment stores of the 8 rows of a quad land in different banks
// then the bias windows [2 wg][h][win_ld] floats, then one diagonal-sum table per warpgroup [2][h][Wacc] floats
constexpr int kBoWin = kBoSds + 2 * 64 * kBtSdsLd * 4;

// Row stride of a bias window: a row tile spans at most ceil(63 / h) + 1 positions, so a warpgroup's window (64 keys)
// holds at most ceil(63 / h) + 64 deltas; 8 mod 32 floats, so the eight rows of a quad column hit at most two per bank.
static int bt_win_ld(int h) { return ((62 + h) / h + 64 + 23) / 32 * 32 + 8; }

__device__ __forceinline__ float bt_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ void bt_red2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void bt_cp_async4(float* dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}

// ---- DET turn counters.  One thread of a warpgroup waits for the turn, the warpgroup adds, fences and signals.
__device__ __forceinline__ int bt_ld_acquire(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long bt_globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __noinline__ void bt_wait_turn(const int* ctr, int turn, int* err) {
  const unsigned long long t0 = bt_globaltimer();
  while (bt_ld_acquire(ctr) != turn) {
    if (*reinterpret_cast<volatile int*>(err) != 0) return;
    if (bt_globaltimer() - t0 > 4000000000ull) { atomicExch(err, 1); return; }   // 4 s: report, never hang
    __nanosleep(64);
  }
}
__device__ __forceinline__ void bt_pass_turn(int* ctr) {
  asm volatile("red.release.gpu.global.add.s32 [%0], 1;" ::"l"(ctr) : "memory");
}

struct BtDet {
  int* turn_dq;     // [B, row tiles]
  int* turn_kv;     // [B, key tiles, 2]
  int* meta;        // [units, 2]: (dmin, used width) of each unit's partial table
  int* err;
  float* dpart;     // [units, h, Wacc]
};

template <bool DET, bool DTAB>
__global__ void __launch_bounds__(kBtThreads, 1)
attn_bwd_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmDO,
                   const __grid_constant__ CUtensorMap tmKV, const float* __restrict__ lse2, const float* __restrict__ dsum,
                   const float* __restrict__ table, int table_ld, const unsigned char* __restrict__ key_mask,
                   float* __restrict__ dqn, float* __restrict__ dkvn, float* __restrict__ dtable, int N, int h, float scale,
                   int Wacc, int win_ld, int tiles_per_chunk, int nbatch, const BtDet det) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kBoBar);
  uint64_t* kv_full = bars + 0;
  uint64_t* qd_full = bars + 1;    // [2]
  uint64_t* qd_empty = bars + 3;   // [2]
  float* dacc = reinterpret_cast<float*>(smem + kBoWin) + 2 * h * win_ld;

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int R = N * h;
  const int n_rt = (R + kBtBQ - 1) / kBtBQ;
  const int n_kt = (N + kBtBK - 1) / kBtBK;
  // unit -> (batch, key tile, chunk): key tile 0 (the most row tiles) first
  const int b = blockIdx.x % nbatch;
  int u = blockIdx.x / nbatch, kt = 0;
  for (; kt < n_kt; ++kt) {
    const int cnt = (n_rt - (kt * kBtBK * h) / kBtBQ + tiles_per_chunk - 1) / tiles_per_chunk;
    if (u < cnt) break;
    u -= cnt;
  }
  const int j0 = kt * kBtBK;
  const int rt0 = (j0 * h) / kBtBQ + u * tiles_per_chunk;
  const int rt1 = min(n_rt, rt0 + tiles_per_chunk);
  const int T = rt1 - rt0;
  const int i_lo = (rt0 * kBtBQ) / h, i_hi = min(N - 1, (rt1 * kBtBQ - 1) / h);
  const int dmin = max(0, i_lo - j0 - (kBtBK - 1));
  const int wacc_used = i_hi - j0 - dmin + 1;       // <= Wacc (host bound)

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmDO); tma_prefetch_desc(&tmKV);
    mbar_init(kv_full, 1);
    for (int i = 0; i < 2; ++i) { mbar_init(&qd_full[i], 1); mbar_init(&qd_empty[i], 2); }
    fence_barrier_init();
  }
  if constexpr (DTAB)
    for (int x = threadIdx.x; x < 2 * h * Wacc; x += blockDim.x) dacc[x] = 0.f;
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      mbar_expect_tx(kv_full, 2 * 16384);
      tma_load_2d(smem + kBoK, &tmKV, kv_full, 0, b * N + j0);
      tma_load_2d(smem + kBoV, &tmKV, kv_full, 64, b * N + j0);
      for (int t = 0; t < T; ++t) {
        const int st = t & 1;
        mbar_wait(&qd_empty[st], ((t >> 1) & 1) ^ 1);
        mbar_expect_tx(&qd_full[st], 2 * 8192);
        tma_load_2d(smem + kBoQ + st * 8192, &tmQ, &qd_full[st], 0, b * R + (rt0 + t) * kBtBQ);
        tma_load_2d(smem + kBoDO + st * 8192, &tmDO, &qd_full[st], 0, b * R + (rt0 + t) * kBtBQ);
      }
    }
  } else {
    // ------------------------------------------------------------------ consumers: 64 keys per warpgroup
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;
    const int wq = (threadIdx.x >> 5) & 3, qr = lane >> 2, qc = lane & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    const int kbase = j0 + cw * 64;
    const uint32_t sk = smem_u32(smem + kBoK) + cw * 8192, sv = smem_u32(smem + kBoV) + cw * 8192;
    uint8_t* p_tile = smem + kBoP + cw * 8192;
    uint8_t* ds_tile = smem + kBoDS + cw * 8192;
    float* sdsf = reinterpret_cast<float*>(smem + kBoSds) + cw * 64 * kBtSdsLd;    // this warpgroup's fp32 dS tile
    float* win = reinterpret_cast<float*>(smem + kBoWin) + cw * h * win_ld;        // this warpgroup's bias window
    float* wacc = dacc + cw * h * Wacc;                                             // this warpgroup's diagonal table
    const int tid128 = threadIdx.x & 127;
    const uint32_t sp = smem_u32(p_tile), sds = smem_u32(ds_tile);
    const float sc2 = scale * kBtL2e;
    // key visibility of this thread's 16 columns (8 c + 2 qc + e)
    uint32_t vis = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int j = kbase + 8 * c + 2 * qc + e;
        if (j < N && (key_mask == nullptr || key_mask[static_cast<long long>(b) * N + j] != 0)) vis |= 1u << (2 * c + e);
      }
    // A row tile's operands from global memory are fetched one tile ahead, while the previous tile's GEMMs run:
    //  - its bias window (per head, deltas it_lo - kbase - 63 .. it_hi - kbase) by cp.async; the raw table values are
    //    scaled by log2 e where they are read.  Entries for delta < 0 are never read and are not copied.
    //  - lse2 and D of this thread's two rows, into registers.
    auto fetch_tile = [&](int rb, float (&lse)[2], float (&D)[2]) {
      const int it_lo = min(rb, R - 1) / h, it_hi = min(rb + kBtBQ - 1, R - 1) / h;
      const int win_w = it_hi - it_lo + 64, dlo = it_lo - kbase - 63;
      for (int hh = tid128 / win_w, w = tid128 - hh * win_w; hh < h;) {      // entry (hh, w); win_w >= 64
        if (dlo + w >= 0) bt_cp_async4(win + hh * win_ld + w, table + hh * static_cast<long>(table_ld) + dlo + w);
        for (w += 128; w >= win_w; ++hh) w -= win_w;
      }
      asm volatile("cp.async.commit_group;" ::: "memory");
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int rc = min(rb + wq * 16 + qr + hr * 8, R - 1);
        lse[hr] = lse2[static_cast<long long>(b) * R + rc];
        D[hr] = dsum[static_cast<long long>(b) * R + rc];
      }
    };
    float lse_t[2], D_t[2];
    fetch_tile(rt0 * kBtBQ, lse_t, D_t);
    float dv[32], dk[32];
#pragma unroll
    for (int x = 0; x < 32; ++x) { dv[x] = 0.f; dk[x] = 0.f; }
    mbar_wait(kv_full, 0);
    for (int t = 0; t < T; ++t) {
      const int st = t & 1;
      const int rbase = (rt0 + t) * kBtBQ;
      const uint32_t sq = smem_u32(smem + kBoQ + st * 8192), sdo = smem_u32(smem + kBoDO + st * 8192);
      mbar_wait(&qd_full[st], (t >> 1) & 1);
      float s[32], dp[32];
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        Wgmma<64, false>::ss<0, 0>(s, make_smem_desc(sq + ks * 32, 16, 1024), make_smem_desc(sk + ks * 32, 16, 1024), ks > 0 ? 1u : 0u);
        Wgmma<64, false>::ss<0, 0>(dp, make_smem_desc(sdo + ks * 32, 16, 1024), make_smem_desc(sv + ks * 32, 16, 1024), ks > 0 ? 1u : 0u);
      }
      wgmma_commit();
      const int it_lo = min(rbase, R - 1) / h, it_hi = min(rbase + kBtBQ - 1, R - 1) / h;
      asm volatile("cp.async.wait_all;" ::: "memory");                // this thread's part of the tile's bias window
      asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
      wgmma_wait<0>();
      wgmma_reg_fence(s);
      wgmma_reg_fence(dp);
      // ---- P, dS (fp32 staged for the diagonal sums), bf16 tiles
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int lr = wq * 16 + qr + hr * 8;
        const int r = rbase + lr;
        const bool row_ok = r < R;
        const int rc = min(r, R - 1);
        const int i = rc / h, hh = rc - i * h;
        const float lse = lse_t[hr], D = D_t[hr];
        const float* wrow = win + hh * win_ld + i - it_lo + 63 - 2 * qc;   // column 8 c + e at wrow[-8 c - e]
        const int dcol = i - kbase - 2 * qc;                                 // delta of column 8 c + e is dcol - 8 c - e
        uint8_t* prow = p_tile + lr * 128;
        uint8_t* drow = ds_tile + lr * 128;
        // the row's 16 window entries, loaded together (always inside the window; those of masked columns may be
        // stale and are discarded below)
        float wv[16];
#pragma unroll
        for (int x = 0; x < 16; ++x) wv[x] = wrow[-8 * (x >> 1) - (x & 1)];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          float pp[2], dd[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            // the causal compare stays: a row whose visible keys all lie in the future has lse2 = -inf, and
            // exp2(-inf - -inf) would turn its P into NaN instead of 0
            const bool live = row_ok && ((vis >> (2 * c + e)) & 1u) && dcol >= 8 * c + e;
            const float x = s[4 * c + 2 * hr + e];
            pp[e] = live ? bt_ex2(fmaf(x, sc2, wv[2 * c + e] * kBtL2e) - lse) : 0.f;
            dd[e] = pp[e] * (dp[4 * c + 2 * hr + e] - D);
          }
          if constexpr (DTAB) *reinterpret_cast<float2*>(sdsf + lr * kBtSdsLd + 8 * c + 2 * qc) = make_float2(dd[0], dd[1]);
          const uint32_t off = static_cast<uint32_t>(((c ^ (lr & 7)) << 4) + 4 * qc);
          *reinterpret_cast<uint32_t*>(prow + off) = pack_bf16x2(pp[0], pp[1]);
          *reinterpret_cast<uint32_t*>(drow + off) = pack_bf16x2(dd[0], dd[1]);
        }
      }
      fence_proxy_async();                                   // P / dS (generic stores) -> visible to wgmma
      asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");   // also: every thread is done with the window
      if (t + 1 < T) fetch_tile(rbase + kBtBQ, lse_t, D_t);
      float dq[32];
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        // rows are the contraction dimension: P^T / dS^T (A) and dO / Q (B) are read MN-major, 16 rows = 2048 bytes
        Wgmma<64, false>::ss<1, 1>(dv, make_smem_desc(sp + ks * 2048, 8192, 1024), make_smem_desc(sdo + ks * 2048, 8192, 1024), 1u);
        Wgmma<64, false>::ss<1, 1>(dk, make_smem_desc(sds + ks * 2048, 8192, 1024), make_smem_desc(sq + ks * 2048, 8192, 1024), 1u);
        // dQ = dS K: keys are the contraction dimension; K [key][dim] is read MN-major
        Wgmma<64, false>::ss<0, 1>(dq, make_smem_desc(sds + ks * 32, 16, 1024), make_smem_desc(sk + ks * 2048, 8192, 1024), ks > 0 ? 1u : 0u);
      }
      wgmma_commit();
      if constexpr (DTAB) {
        // diagonal sums of the fp32 dS tile while the tensor cores run: thread-owned (head, diagonal) pairs, rows in order
        const int dlo = max(0, it_lo - kbase - 63), dhi = it_hi - kbase;
        const int W = dhi - dlo + 1;
        // head hh has the tile's rows at positions ceil((rbase - hh) / h) .. floor((rbase + 63 - hh) / h)
        const int q0 = rbase / h, r0 = rbase - q0 * h;
        const int q1 = (rbase + kBtBQ - 1) / h, r1 = rbase + kBtBQ - 1 - q1 * h;
        // W <= 0: this warpgroup's keys all lie after the tile's last position, no pairs
        for (int hh = W > 0 ? tid128 / W : h, w = W > 0 ? tid128 - hh * W : 0; hh < h;) {   // pair (hh, dlo + w)
          const int dl = dlo + w;
          const int i0 = max(q0 + (hh < r0 ? 1 : 0), kbase + dl);
          const int i1 = min(min(q1 - (hh > r1 ? 1 : 0), N - 1), kbase + dl + 63);
          // eight rows' loads in flight at once; the adds stay in row order
          const float* src = sdsf + (i0 * h + hh - rbase) * kBtSdsLd + (i0 - dl - kbase);
          const int stride = h * kBtSdsLd + 1;
          float sum = 0.f;
          for (int i = i0; i <= i1; i += 8, src += 8 * stride) {
            float x[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) x[k] = i + k <= i1 ? src[k * stride] : 0.f;
#pragma unroll
            for (int k = 0; k < 8; ++k)
              if (i + k <= i1) sum += x[k];
          }
          wacc[hh * Wacc + dl - dmin] += sum;
          for (w += 128; w >= W && hh < h; ++hh) w -= W;
        }
      }
      wgmma_wait<0>();
      wgmma_reg_fence(dq);
      wgmma_reg_fence(dv);
      wgmma_reg_fence(dk);
      asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");   // every thread's wgmma have read the P / dS tiles
      if (leader) mbar_arrive(&qd_empty[st]);
      int* turn = DET ? det.turn_dq + static_cast<long>(b) * n_rt + rt0 + t : nullptr;
      if constexpr (DET) {
        if (leader) bt_wait_turn(turn, 2 * kt + cw, det.err);
        asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
      }
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int r = rbase + wq * 16 + qr + hr * 8;
        if (r < R) {
          float* dst = dqn + (static_cast<long long>(b) * R + r) * 64 + 2 * qc;
#pragma unroll
          for (int c = 0; c < 8; ++c) bt_red2(dst + 8 * c, dq[4 * c + 2 * hr] * scale, dq[4 * c + 2 * hr + 1] * scale);
        }
      }
      if constexpr (DET) {
        __threadfence();
        asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
        if (leader) bt_pass_turn(turn);
      }
    }
    // ---- dK (scaled), dV into dkvn [key][dK 0..63 | dV 64..127]
    int* kv_turn = DET ? det.turn_kv + (static_cast<long>(b) * n_kt + kt) * 2 + cw : nullptr;
    if constexpr (DET) {
      if (leader) bt_wait_turn(kv_turn, u, det.err);
      asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int j = kbase + wq * 16 + qr + hr * 8;
      if (j < N) {
        float* dst = dkvn + (static_cast<long long>(b) * N + j) * 128 + 2 * qc;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          bt_red2(dst + 8 * c, dk[4 * c + 2 * hr] * scale, dk[4 * c + 2 * hr + 1] * scale);
          bt_red2(dst + 64 + 8 * c, dv[4 * c + 2 * hr], dv[4 * c + 2 * hr + 1]);
        }
      }
    }
    if constexpr (DET) {
      __threadfence();
      asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
      if (leader) bt_pass_turn(kv_turn);
    }
    // ---- flush the diagonal sums of this unit
    if constexpr (!DTAB) return;
    asm volatile("bar.sync 3, 256;" ::: "memory");
    if constexpr (DET) {       // (warpgroup 1 + warpgroup 2) -> this unit's partial table; summed in unit order later
      float* up = det.dpart + static_cast<long>(blockIdx.x) * h * Wacc;
      for (int x = threadIdx.x - 128; x < h * wacc_used; x += 256) {
        const int hh = x / wacc_used, w = x - hh * wacc_used;
        up[hh * Wacc + w] = dacc[hh * Wacc + w] + dacc[(h + hh) * Wacc + w];
      }
      if (threadIdx.x == 128) { det.meta[2 * blockIdx.x] = dmin; det.meta[2 * blockIdx.x + 1] = wacc_used; }
    } else {
      for (int x = threadIdx.x - 128; x < h * wacc_used; x += 256) {
        const int hh = x / wacc_used, w = x - hh * wacc_used;
        const float v = dacc[hh * Wacc + w] + dacc[(h + hh) * Wacc + w];
        if (v != 0.f) atomicAdd(dtable + hh * static_cast<long>(table_ld) + dmin + w, v);
      }
    }
  }
}

// DET: dtable[hh, d] += the partial tables of all units, in unit order
__global__ void __launch_bounds__(256)
attn_bwd_dtable_reduce_kernel(const float* __restrict__ dpart, const int* __restrict__ meta, int units, int h, int Wacc,
                              float* __restrict__ dtable, int table_ld, int N) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= h * N) return;
  const int hh = x / N, d = x - hh * N;
  float* dst = dtable + hh * static_cast<long>(table_ld) + d;
  float acc = *dst;
  for (int u = 0; u < units; ++u) {
    const int w = d - __ldg(meta + 2 * u);
    if (w >= 0 && w < __ldg(meta + 2 * u + 1)) acc += dpart[(static_cast<long>(u) * h + hh) * Wacc + w];
  }
  *dst = acc;
}

// D[r] = sum_d dO[r, d] * O[r, d];  also clears the dQ / dK|dV accumulators the main kernel reduces into
// (dqn [rows, 64] fp32: this thread's 8 columns; dkvn: kv_vec4 float4s spread over the grid)
__global__ void __launch_bounds__(256)
attn_bwd_tc_dsum_kernel(const __nv_bfloat16* __restrict__ d_o, const __nv_bfloat16* __restrict__ o,
                        float* __restrict__ dsum, long rows, float* __restrict__ dqn, float* __restrict__ dkvn, long kv_vec4) {
  const long tid = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long r = tid >> 3;
  const int sub = threadIdx.x & 7;
  float s = 0.f;
  for (long i = tid; i < kv_vec4; i += static_cast<long>(gridDim.x) * blockDim.x)     // (fewer threads than float4s when heads < 4)
    reinterpret_cast<float4*>(dkvn)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (r < rows) {
    float4* zq = reinterpret_cast<float4*>(dqn + r * 64 + sub * 8);
    zq[0] = make_float4(0.f, 0.f, 0.f, 0.f);
    zq[1] = make_float4(0.f, 0.f, 0.f, 0.f);
    const uint4 a = *reinterpret_cast<const uint4*>(d_o + r * 64 + sub * 8);
    const uint4 bq = *reinterpret_cast<const uint4*>(o + r * 64 + sub * 8);
    const uint32_t aa[4] = {a.x, a.y, a.z, a.w}, bb[4] = {bq.x, bq.y, bq.z, bq.w};
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

}  // namespace omlm

namespace omlm {

// Launch geometry shared by the launch and the workspace query.
struct BtConfig {
  int tiles_per_chunk, wacc, win_ld, smem_bytes, units_per_batch, n_row_tiles, n_key_tiles;
};

// Chunk length T (row tiles per unit).  One CTA runs per SM and the units differ in length (the row tiles of key tile
// kt start at 2 kt h, and a unit's last chunk may be short), so T is picked by replaying the hardware's dispatch: units
// in block order, each to the SM that frees first, a unit costing its row tiles plus about one tile for its K/V load
// and dK/dV flush.  T is at most 16: longer chunks leave few units to fill the last wave, and in the deterministic mode
// a row tile's later key tiles wait for the earlier ones, so long chunks serialise the turns.  Among equal makespans
// the longer chunk wins (fewer K/V loads and dK/dV flushes).  Memoised: the replay costs up to a millisecond.
template <class Fits>
static int bt_pick_chunk(int B, int n_row_tiles, int n_key_tiles, int heads, Fits fits) {
  static std::mutex mu;
  static std::map<std::array<int, 5>, int> memo;
  const int sms = num_sms();
  const std::array<int, 5> key{B, n_row_tiles, n_key_tiles, heads, sms};
  std::lock_guard<std::mutex> lock(mu);
  const auto hit = memo.find(key);
  if (hit != memo.end()) return hit->second;
  int best_T = 1;
  long best = -1;
  std::vector<long> busy(sms);
  for (int T = 1; T <= std::min(16, n_row_tiles); ++T) {
    if (!fits(T)) break;
    std::fill(busy.begin(), busy.end(), 0L);      // a min-heap of the SMs' busy-until times
    for (int kt = 0; kt < n_key_tiles; ++kt) {
      const int first = (kt * kBtBK * heads) / kBtBQ;
      for (int rt = first; rt < n_row_tiles; rt += T) {
        const long cost = std::min(T, n_row_tiles - rt) + 1;
        for (int b = 0; b < B; ++b) {
          std::pop_heap(busy.begin(), busy.end(), std::greater<long>());
          busy.back() += cost;
          std::push_heap(busy.begin(), busy.end(), std::greater<long>());
        }
      }
    }
    const long makespan = *std::max_element(busy.begin(), busy.end());
    if (best < 0 || makespan <= best) { best = makespan; best_T = T; }
  }
  memo[key] = best_T;
  return best_T;
}

static int bt_config(int B, int N, int heads, BtConfig* cfg) {
  const long R = static_cast<long>(N) * heads;
  const int n_row_tiles = static_cast<int>((R + kBtBQ - 1) / kBtBQ);
  const int n_key_tiles = (N + kBtBK - 1) / kBtBK;
  // chunk length T: bt_pick_chunk, among the lengths whose per-CTA diagonal tables (2 x heads x (64 T / heads + 130)
  // floats) fit in shared memory
  const int win_ld = bt_win_ld(heads);
  auto wacc_of = [&](int T) { return (T * kBtBQ + heads - 1) / heads + kBtBK + 2; };
  auto smem_of = [&](int T) { return kBoWin + 2 * heads * (win_ld + wacc_of(T)) * 4 + 1024; };
  auto units_of = [&](int T) {
    long units = 0;
    for (int kt = 0; kt < n_key_tiles; ++kt) {
      const int first = (kt * kBtBK * heads) / kBtBQ;
      units += (n_row_tiles - first + T - 1) / T;
    }
    return units;
  };
  OMLM_CHECK_ARG(smem_of(1) <= kBtMaxSmem, "attn_bwd_tc: too many heads (%d) for the shared-memory bias tables", heads);
  int tiles_per_chunk = bt_pick_chunk(B, n_row_tiles, n_key_tiles, heads, [&](int T) { return smem_of(T) <= kBtMaxSmem; });
  if (const char* e = getenv("OMLM_ATTN_BWD_T")) {      // diagnostics: force the chunk length
    const int T = atoi(e);
    if (T >= 1 && T <= n_row_tiles && smem_of(T) <= kBtMaxSmem) tiles_per_chunk = T;
  }
  cfg->tiles_per_chunk = tiles_per_chunk;
  cfg->wacc = wacc_of(tiles_per_chunk);
  cfg->win_ld = win_ld;
  cfg->smem_bytes = smem_of(tiles_per_chunk);
  cfg->units_per_batch = static_cast<int>(units_of(tiles_per_chunk));
  cfg->n_row_tiles = n_row_tiles;
  cfg->n_key_tiles = n_key_tiles;
  return 0;
}

static int bt_ints(int B, const BtConfig& c) {     // turn counters, then the units' (dmin, width), then the error word
  return B * c.n_row_tiles + 2 * B * c.n_key_tiles + 2 * B * c.units_per_batch + 1;
}

static int attn_bwd_tc_impl(const void* qn, const void* kvn, const void* d_o, const void* o, const float* lse2,
                            const float* table, int table_ld, const unsigned char* key_mask, float* dsum_scratch,
                            float* dqn, float* dkvn, float* dtable, int B, int N, int heads, float scale, bool det,
                            float* ws, long ws_bytes, int* iws, long iws_count, void* stream) {
  OMLM_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attn_bwd_tc: bad shape");
  OMLM_CHECK_ARG(table_ld >= N, "attn_bwd_tc: bias table shorter than the sequence");
  auto st = reinterpret_cast<cudaStream_t>(stream);
  const long R = static_cast<long>(N) * heads;
  const long rows = static_cast<long>(B) * R;
  BtConfig cfg;
  int rc = bt_config(B, N, heads, &cfg);
  if (rc) return rc;
  const int units = B * cfg.units_per_batch;
  BtDet dp{nullptr, nullptr, nullptr, nullptr, nullptr};
  const bool dtab = dtable != nullptr;
  if (det) {
    // without the bias gradient the partial tables (ws) are not used
    OMLM_CHECK_ARG((!dtab || (ws != nullptr && ws_bytes >= static_cast<long>(units) * heads * cfg.wacc * 4)) && iws != nullptr &&
                   iws_count >= bt_ints(B, cfg), "attn_bwd_tc_det: workspace too small (see omlm_attn_bwd_tc_det_workspace)");
    dp.turn_dq = iws;
    dp.turn_kv = iws + static_cast<long>(B) * cfg.n_row_tiles;
    dp.meta = dp.turn_kv + 2L * B * cfg.n_key_tiles;
    dp.err = iws + iws_count - 1;      // the caller's last int, whatever the buffer's size
    dp.dpart = ws;
    OMLM_CUDA(cudaMemsetAsync(iws, 0, (static_cast<long>(B) * cfg.n_row_tiles + 2L * B * cfg.n_key_tiles) * sizeof(int), st));
  }
  OMLM_KLAUNCH((attn_bwd_tc_dsum_kernel), static_cast<int>((rows * 8 + 255) / 256), 256, 0, st,
      reinterpret_cast<const __nv_bfloat16*>(d_o), reinterpret_cast<const __nv_bfloat16*>(o), dsum_scratch, rows,
      dqn, dkvn, static_cast<long>(B) * N * 128 / 4);
  OMLM_LAUNCH_CHECK();
  CUtensorMap tmQ, tmDO, tmKV;
  rc = make_tmap_bf16_2d(&tmQ, qn, 64, static_cast<uint64_t>(rows), 128, 64, kBtBQ);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmDO, d_o, 64, static_cast<uint64_t>(rows), 128, 64, kBtBQ);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmKV, kvn, 128, static_cast<uint64_t>(B) * N, 256, 64, kBtBK);
  if (rc) return rc;
  // the variant without the table keeps the same chunk length and shared-memory layout (the chunk length decides the
  // order of the dK|dV sums, so dQ, dK and dV stay bit-identical to the variant with the table)
  auto kern = det ? (dtab ? attn_bwd_tc_kernel<true, true> : attn_bwd_tc_kernel<true, false>)
                  : (dtab ? attn_bwd_tc_kernel<false, true> : attn_bwd_tc_kernel<false, false>);
  const int variant = 2 * det + dtab;
  static int configured[4] = {0, 0, 0, 0};
  if (configured[variant] < cfg.smem_bytes) {
    OMLM_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, cfg.smem_bytes));
    configured[variant] = cfg.smem_bytes;
  }
  OMLM_KLAUNCH((kern), units, kBtThreads, cfg.smem_bytes, st,
      tmQ, tmDO, tmKV, lse2, dsum_scratch, table, table_ld, key_mask, dqn, dkvn, dtable, N, heads, scale,
      cfg.wacc, cfg.win_ld, cfg.tiles_per_chunk, B, dp);
  OMLM_LAUNCH_CHECK();
  if (det && dtab) {
    OMLM_KLAUNCH((attn_bwd_dtable_reduce_kernel), (heads * N + 255) / 256, 256, 0, st,
        static_cast<const float*>(dp.dpart), static_cast<const int*>(dp.meta), units, heads, cfg.wacc, dtable, table_ld, N);
    OMLM_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace omlm

extern "C" int omlm_attn_bwd_tc(const void* qn, const void* kvn, const void* d_o, const void* o, const float* lse2,
                                const float* table, int table_ld, const unsigned char* key_mask, float* dsum_scratch,
                                float* dqn, float* dkvn, float* dtable, int B, int N, int heads,
                                float scale, void* stream) {
  return omlm::attn_bwd_tc_impl(qn, kvn, d_o, o, lse2, table, table_ld, key_mask, dsum_scratch, dqn, dkvn, dtable, B, N, heads,
                                scale, false, nullptr, 0, nullptr, 0, stream);
}

extern "C" int omlm_attn_bwd_tc_det(const void* qn, const void* kvn, const void* d_o, const void* o, const float* lse2,
                                    const float* table, int table_ld, const unsigned char* key_mask, float* dsum_scratch,
                                    float* dqn, float* dkvn, float* dtable, int B, int N, int heads, float scale,
                                    float* ws, long ws_bytes, int* iws, long iws_count, void* stream) {
  return omlm::attn_bwd_tc_impl(qn, kvn, d_o, o, lse2, table, table_ld, key_mask, dsum_scratch, dqn, dkvn, dtable, B, N, heads,
                                scale, true, ws, ws_bytes, iws, iws_count, stream);
}

extern "C" int omlm_attn_bwd_tc_det_workspace(int B, int N, int heads, long* ws_bytes, long* iws_count) {
  using namespace omlm;
  OMLM_CHECK_ARG(B > 0 && N > 0 && heads > 0 && ws_bytes != nullptr && iws_count != nullptr, "attn_bwd_tc_det_workspace: bad arguments");
  BtConfig cfg;
  const int rc = bt_config(B, N, heads, &cfg);
  if (rc) return rc;
  *ws_bytes = static_cast<long>(B) * cfg.units_per_batch * heads * cfg.wacc * 4;
  *iws_count = bt_ints(B, cfg);
  return 0;
}
