// Persistent warp-specialised bf16 / fp16 GEMM for sm_90a:  C[m,n] = alpha * sum_k A(m,k) * B(n,k) (+ addend)
//
//   warpgroup 0     : TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier complete_tx)
//   warpgroups 1, 2 : consumers.  Each owns 64 rows of the 128-row tile, issues wgmma (m64 x BN x k16, fp32 accumulators
//                     in registers) straight from the swizzled ring, keeps one k-block of wgmma in flight and frees the
//                     previous slot, then runs the fused epilogue from its accumulator fragment (alpha, residual addend,
//                     row remapping, split-K reductions, bf16 / fp32 stores, LayerNorm-backward row statistics).
//
// Staged epilogue (every launch whose output rows are the tile's rows, without atomics, with 16-byte-aligned rows):
// each consumer warpgroup owns a ring of kEpiBoxes 64-row x 128-byte boxes in shared memory.  It writes its fragment
// into a box, and one thread stores the box by TMA and goes on; the warpgroup only waits until a box has been read
// out before it writes that box again, never for the global write, so the next tile's wgmma run under the stores.
// The fp32 addend (and hn for the row statistics) comes into the same boxes by TMA: the first boxes of a tile are
// requested before the tile's k-loop, the later ones as soon as an earlier box has been stored.
//
// Operand majors are template parameters so that one kernel serves the forward projections
// (A K-major, B K-major: nn.Linear weights are [out,in]), the data-gradient GEMMs (B MN-major: the
// same weight read "transposed" without a transposed copy) and the weight-gradient GEMMs
// (A and B MN-major: activations [tokens, features] contracted over tokens).
//
// This replaces the cuBLAS calls behind nn.Linear / einsum in the reference
// (open_musiclm/transformer.py:144,149,254,333; open_musiclm/open_musiclm.py:173,181).
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/omlm_b200.h"
#include <stdlib.h>
#include <string.h>
#include <algorithm>

namespace omlm {

constexpr int BM = 128;
constexpr int BK = 64;  // 64 16-bit elements = 128 bytes = one swizzle row
constexpr int kGemmThreads = 384;

struct EpiParams {
  void* out;            // bf16 or fp32
  const float* addend;  // optional fp32 [M, ldadd]
  long ldo;
  long ldadd;
  float alpha;
  int out_f32;    // 0: bf16, 1: fp32
  int atomic;     // 1: red.add into fp32 out (split-K)
  long split_stride;   // > 0 (deterministic split-K): split s stores its fp32 partial at out + s * split_stride, no atomics
  int vec_ok;     // out / addend rows 16-byte aligned: column pairs move as one vector
  int staged;     // the tile goes out through the shared-memory boxes and TMA stores (see the top of this file)
  int row_split;  // >0: rows are two halves of row_split, each with row_valid live rows; <0: interleaved GEGLU groups of 128
  int row_valid;
  int n_valid;    // columns >= n_valid are dropped
  // row statistics (the d_hn data-gradient GEMM of the conv feed-forward): with d = this GEMM's fp32 output row and hn
  // the saved forward output, part[row, 2 n_blk + half] = (sum_c gamma[c] drop(d[c]), sum_c d[c] hn[c]) over each
  // 128-column half tile -- the two row sums LayerNorm-backward needs (ffn_mid.cu), without a separate pass.
  // hn comes in by TMA through the epilogue's second tensor map.
  const float* rs_gamma;      // [N] fp32 (zero in padded columns)
  const uint8_t* rs_keep;      // dropout keep bits [M, N/8] or nullptr
  float2* rs_part;             // [M, rs_parts]
  float rs_keep_scale;         // 1 / (1 - p)
  int rs_parts;
};

__device__ __forceinline__ float bf16lo(uint32_t v) { return __uint_as_float(v << 16); }
__device__ __forceinline__ float bf16hi(uint32_t v) { return __uint_as_float(v & 0xffff0000u); }

template <int BN>
struct GemmSmem {
  static constexpr int kABytes = BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kMaxStages = 8;
};

// Staging boxes per consumer warpgroup.  Four leave room for 3 operand stages at 256-wide tiles (two boxes: 4 stages);
// four measured faster in sum over the cfg2 GEMM shapes (DESIGN.md section 6).
constexpr int kEpiBoxes = 4;
constexpr int kBoxBytes = 64 * 128;         // 64 rows x 128 bytes: 32 fp32 or 64 bf16 columns (the 128B-swizzle limit)
constexpr int kStagingBytes = 2 * kEpiBoxes * kBoxBytes;

__device__ __forceinline__ void wg_bar_sync(int cw) { asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory"); }

// Byte offset of the column pair (8 g + 2 qc, +1) of row r in a 128B-swizzled box: 16-byte chunk c of row r sits at c ^ (r & 7).
template <bool F32>
__device__ __forceinline__ uint32_t box_offset(int r, int g, int qc) {
  const int chunk = F32 ? 2 * g + (qc >> 1) : g;
  return r * 128 + ((chunk ^ (r & 7)) << 4) + (F32 ? 8 * (qc & 1) : 4 * qc);
}

__device__ __forceinline__ void load_box(const CUtensorMap* tm, uint8_t* box, uint64_t* bar, int col, int row) {
  mbar_expect_tx(bar, kBoxBytes);   // a box reaching past the tensor counts in full (zero-filled)
  tma_load_2d(box, tm, bar, col, row);
}

// The staged epilogue of one tile for one consumer warpgroup (rows row0 .. row0 + 63, the first `live` boxes of
// columns).  The arithmetic and, for the row statistics, the order of every sum are those of the direct epilogue.
// seq counts the boxes this warpgroup has staged (slot = seq % kEpiBoxes); ephase holds one parity bit per slot.
template <int BN, bool RS, bool F32>
__device__ __forceinline__ void epilogue_staged(float (&acc)[BN / 2], const EpiParams& ep, const CUtensorMap* tmO,
                                                const CUtensorMap* tmE, uint8_t* ring, uint64_t* ebar, uint32_t& seq,
                                                uint32_t& ephase, int live, int n_blk, int row0, int M, int N, int cw,
                                                bool leader) {
  constexpr int kCols = F32 ? 32 : 64, kGroups = kCols / 8, kBoxesPerTile = BN / kCols;
  constexpr int kBatch = RS ? 4 : kGroups;   // the row statistics load gamma and keep bits 4 column groups ahead
  const bool with_e = RS || ep.addend != nullptr;
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3, qr = lane >> 2, qc = lane & 3;
  float rs1[2][2] = {{0.f, 0.f}, {0.f, 0.f}}, rs2[2][2] = {{0.f, 0.f}, {0.f, 0.f}};   // [row][half]
#pragma unroll
  for (int b = 0; b < kBoxesPerTile; ++b) {
    if (b >= live) break;
    const uint32_t slot = seq % kEpiBoxes;
    uint8_t* box = ring + slot * kBoxBytes;
    if (with_e) {
      mbar_wait(&ebar[slot], (ephase >> slot) & 1u);
      ephase ^= 1u << slot;
    } else {
      if (leader) tma_store_wait_read<kEpiBoxes - 1>();   // the store that last used this slot has read it
      wg_bar_sync(cw);
    }
#pragma unroll
    for (int g0 = 0; g0 < kGroups; g0 += kBatch) {
      float2 gam[kBatch];
      uint32_t keep[2][kBatch];
      if constexpr (RS) {
#pragma unroll
        for (int j = 0; j < kBatch; ++j) {
          const int col = n_blk * BN + b * kCols + 8 * (g0 + j) + 2 * qc;
          gam[j] = __ldg(reinterpret_cast<const float2*>(ep.rs_gamma + col));
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const int row = row0 + wq * 16 + qr + hr * 8;
            keep[hr][j] = (row < M && ep.rs_keep != nullptr) ? ep.rs_keep[static_cast<long>(row) * (N >> 3) + (col >> 3)] : 0xffu;
          }
        }
      }
#pragma unroll
      for (int j = 0; j < kBatch; ++j) {
        const int i = b * kGroups + g0 + j;   // column group of the fragment
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int r = wq * 16 + qr + hr * 8;
          uint8_t* p = box + box_offset<F32>(r, g0 + j, qc);
          // rounded product, then the addend, as in the direct epilogue (a contracted fma would round once)
          float v0 = __fmul_rn(acc[4 * i + 2 * hr], ep.alpha), v1 = __fmul_rn(acc[4 * i + 2 * hr + 1], ep.alpha);
          if constexpr (RS) {
            const uint32_t kb = keep[hr][j], hv = *reinterpret_cast<const uint32_t*>(p);
            const int col = n_blk * BN + 8 * i + 2 * qc;
            const int hf = (8 * i) / (BN / 2);
            rs1[hr][hf] = fmaf(gam[j].x, ((kb >> (col & 7)) & 1u) ? v0 : 0.f, rs1[hr][hf]);
            rs1[hr][hf] = fmaf(gam[j].y, ((kb >> ((col + 1) & 7)) & 1u) ? v1 : 0.f, rs1[hr][hf]);
            rs2[hr][hf] = fmaf(v0, bf16lo(hv), rs2[hr][hf]);
            rs2[hr][hf] = fmaf(v1, bf16hi(hv), rs2[hr][hf]);
          }
          if constexpr (F32) {
            if (ep.addend != nullptr) { const float2 a = *reinterpret_cast<const float2*>(p); v0 += a.x; v1 += a.y; }
            *reinterpret_cast<float2*>(p) = make_float2(v0, v1);
          } else {
            *reinterpret_cast<uint32_t*>(p) = pack_bf16x2(v0, v1);
          }
        }
      }
    }
    fence_proxy_async();   // the generic-proxy writes of every thread become visible to the TMA store
    wg_bar_sync(cw);
    if (leader) {
      tma_store_2d(tmO, box, n_blk * BN + b * kCols, row0);
      tma_store_commit();
      if (with_e && b >= 1 && b - 1 + kEpiBoxes < live) {   // refill the previous box's slot once its store has read it
        const uint32_t s = (seq - 1) % kEpiBoxes;
        tma_store_wait_read<1>();
        load_box(tmE, ring + s * kBoxBytes, &ebar[s], n_blk * BN + (b - 1 + kEpiBoxes) * kCols, row0);
      }
    }
    ++seq;
  }
  if constexpr (RS) {       // quad reduction: the four lanes of a fragment row hold disjoint column pairs
#pragma unroll
    for (int hr = 0; hr < 2; ++hr)
#pragma unroll
      for (int hf = 0; hf < 2; ++hf) {
        float a1 = rs1[hr][hf], a2 = rs2[hr][hf];
        a1 += __shfl_xor_sync(0xffffffffu, a1, 1); a1 += __shfl_xor_sync(0xffffffffu, a1, 2);
        a2 += __shfl_xor_sync(0xffffffffu, a2, 1); a2 += __shfl_xor_sync(0xffffffffu, a2, 2);
        const int row = row0 + wq * 16 + qr + hr * 8;
        if (qc == 0 && row < M) ep.rs_part[static_cast<long>(row) * ep.rs_parts + 2 * n_blk + hf] = make_float2(a1 * ep.rs_keep_scale, a2);
      }
  }
}

template <int BN, int A_MN, int B_MN, bool F16, bool RS = false>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmE,
                 const EpiParams ep, const int M, const int N, const int K, const int splits, const int kStages) {
  using S = GemmSmem<BN>;
  extern __shared__ uint8_t smem_raw[];
  // 1024B alignment is required by the 128B swizzle atoms.
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* staging = smem + kStages * S::kStageBytes;                 // [2 warpgroups][kEpiBoxes] boxes when ep.staged
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + (ep.staged ? kStagingBytes : 0));
  uint64_t* empty_bar = full_bar + S::kMaxStages;
  uint64_t* epi_bar = empty_bar + S::kMaxStages;                      // [2 warpgroups][kEpiBoxes]: addend / hn box loaded

  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;

  const int m_tiles = (M + BM - 1) / BM;
  const int n_tiles = (N + BN - 1) / BN;
  const int kb_total = (K + BK - 1) / BK;
  const int kb_per_split = (kb_total + splits - 1) / splits;
  const int tiles_total = m_tiles * n_tiles;
  const int work_total = tiles_total * splits;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);        // one arrival per consumer warpgroup
    }
    if (ep.staged) {
      tma_prefetch_desc(&tmO);
      for (int i = 0; i < 2 * kEpiBoxes; ++i) mbar_init(&epi_bar[i], 1);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int w = blockIdx.x; w < work_total; w += gridDim.x) {
        const int split = w / tiles_total;      // split-major order: the CTAs of a wave share one K range, so the
        const int tile = w - split * tiles_total;   // operand slices of that range stay in L2 (tile-major thrashed it)
        const int n_blk = tile % n_tiles, m_blk = tile / n_tiles;
        const int kb0 = split * kb_per_split;
        const int kb1 = min(kb_total, kb0 + kb_per_split);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          uint8_t* sa = smem + stage * S::kStageBytes;
          uint8_t* sb = sa + S::kABytes;
          mbar_expect_tx(&full_bar[stage], S::kStageBytes);
          if (A_MN == 0) {
            tma_load_2d(sa, &tmA, &full_bar[stage], kb * BK, m_blk * BM);
          } else {
#pragma unroll
            for (int c = 0; c < BM / 64; ++c)
              tma_load_2d(sa + c * 8192, &tmA, &full_bar[stage], m_blk * BM + c * 64, kb * BK);
          }
          if (B_MN == 0) {
            tma_load_2d(sb, &tmB, &full_bar[stage], kb * BK, n_blk * BN);
          } else {
#pragma unroll
            for (int c = 0; c < BN / 64; ++c)
              tma_load_2d(sb + c * 8192, &tmB, &full_bar[stage], n_blk * BN + c * 64, kb * BK);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int cw = wg - 1;                                   // 64-row half of the tile
  const int wq = (threadIdx.x >> 5) & 3;                   // warp within the warpgroup: 16 rows each
  const int qr = lane >> 2, qc = lane & 3;                 // fragment row / column pair within the warp's rows
  const bool leader = (threadIdx.x & 127) == 0;
  uint8_t* ring = staging + cw * kEpiBoxes * kBoxBytes;
  uint64_t* ebar = epi_bar + cw * kEpiBoxes;
  const bool with_e = ep.staged && (RS || ep.addend != nullptr);
  const int box_cols = (RS || !ep.out_f32) ? 64 : 32;
  uint32_t seq = 0, ephase = 0;
  int stage = 0;
  uint32_t phase = 0;
  for (int w = blockIdx.x; w < work_total; w += gridDim.x) {
    const int split = w / tiles_total;
    const int tile = w - split * tiles_total;
    const int n_blk = tile % n_tiles, m_blk = tile / n_tiles;
    const int kb0 = split * kb_per_split;
    const int kb1 = min(kb_total, kb0 + kb_per_split);
    const int row0 = m_blk * BM + cw * 64;
    // boxes of this warpgroup's 64 rows that hold any output (none when the rows lie past M)
    const int live = row0 < M ? max(0, min(BN / box_cols, (ep.n_valid - n_blk * BN + box_cols - 1) / box_cols)) : 0;
    if (with_e && leader) {   // the tile's first addend / hn boxes load under its k-loop, once the last stores have read their slots
      tma_store_wait_read<0>();
      for (int j = 0; j < min(kEpiBoxes, live); ++j) {
        const uint32_t s = (seq + j) % kEpiBoxes;
        load_box(&tmE, ring + s * kBoxBytes, &ebar[s], n_blk * BN + j * box_cols, row0);
      }
    }
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * S::kStageBytes) + cw * 8192;   // this warpgroup's 64 rows of A
      const uint32_t sb = smem_u32(smem + stage * S::kStageBytes + S::kABytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        // K-major: 16 elements = 32 bytes inside the swizzle row; 8-row groups 1024B apart.
        // MN-major: 16 k-rows = 2048 bytes; 64-element MN chunks 8192B apart (LBO), 8-row groups 1024B (SBO).
        const uint64_t ad = A_MN ? make_smem_desc(sa + k * 2048, 8192, 1024) : make_smem_desc(sa + k * 32, 16, 1024);
        const uint64_t bd = B_MN ? make_smem_desc(sb + k * 2048, 8192, 1024) : make_smem_desc(sb + k * 32, 16, 1024);
        const uint32_t accum = (kb > kb0 || k > 0) ? 1u : 0u;
        Wgmma<BN, F16>::template ss<A_MN, B_MN>(acc, ad, bd, accum);
      }
      wgmma_commit();
      wgmma_wait<1>();                                      // the previous k-block's wgmma have read their slot
      if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_reg_fence(acc);
    if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);

    if constexpr (RS) {   // the row statistics are always staged (checked on the host)
      epilogue_staged<BN, true, false>(acc, ep, &tmO, &tmE, ring, ebar, seq, ephase, live, n_blk, row0, M, N, cw, leader);
    } else if (ep.staged) {
      if (ep.out_f32) epilogue_staged<BN, false, true>(acc, ep, &tmO, &tmE, ring, ebar, seq, ephase, live, n_blk, row0, M, N, cw, leader);
      else epilogue_staged<BN, false, false>(acc, ep, &tmO, &tmE, ring, ebar, seq, ephase, live, n_blk, row0, M, N, cw, leader);
    } else {
      // ------------------------------------------------------------------ direct epilogue: rows r_lo, r_lo + 8 of the fragment
      // (atomic split-K, the row remaps, split-K partial slices, rows that are not 16-byte aligned)
      long orow[2], arow[2];
      bool row_ok[2];
  #pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        int row = m_blk * BM + cw * 64 + wq * 16 + qr + hr * 8;
        row_ok[hr] = row < M;
        if (ep.row_split > 0) {
          const int half = row / ep.row_split, r = row - half * ep.row_split;
          row_ok[hr] = row_ok[hr] && r < ep.row_valid;
          row = half * ep.row_valid + r;
        } else if (ep.row_split < 0) {   // interleaved GEGLU rows: [128 value | 128 gate] per group of 128 channels
          const int w256 = row & 255, ch = ((row >> 8) << 7) + (w256 & 127);
          row_ok[hr] = row_ok[hr] && ch < ep.row_valid;
          row = (w256 >> 7) * ep.row_valid + ch;
        }
        orow[hr] = static_cast<long>(row) * ep.ldo;
        arow[hr] = static_cast<long>(row) * ep.ldadd;
      }
      // The columns go in batches of kEpiBatch 8-column groups, and every addend load of a batch is issued before the
      // batch's first store.  The stores may alias the loads (a weight gradient without split-K adds into its own
      // output), so the compiler keeps each load behind every earlier store: loads interleaved with stores each waited a
      // full memory latency.
      constexpr int kEpiBatch = 8;
  #pragma unroll
      for (int i0 = 0; i0 < BN / 8; i0 += kEpiBatch) {
        float2 add[2][kEpiBatch];
  #pragma unroll
        for (int j = 0; j < kEpiBatch; ++j) {
          const int col = n_blk * BN + 8 * (i0 + j) + 2 * qc;
          const bool c0_ok = col < ep.n_valid, c1_ok = col + 1 < ep.n_valid;
  #pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            add[hr][j] = make_float2(0.f, 0.f);
            if (!row_ok[hr] || !c0_ok) continue;
            if (ep.addend != nullptr) {
              const float* ap = ep.addend + arow[hr] + col;
              if (c1_ok && ep.vec_ok) add[hr][j] = *reinterpret_cast<const float2*>(ap);
              else { add[hr][j].x = ap[0]; if (c1_ok) add[hr][j].y = ap[1]; }
            }
          }
        }
  #pragma unroll
        for (int j = 0; j < kEpiBatch; ++j) {
          const int i = i0 + j;
          const int col = n_blk * BN + 8 * i + 2 * qc;
          if (col >= ep.n_valid) continue;
          const bool pair = col + 1 < ep.n_valid && ep.vec_ok;
  #pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            if (!row_ok[hr]) continue;
            // rounded product, then the addend (a contracted fma would round once and differ from the staged epilogue)
            float v0 = __fmul_rn(acc[4 * i + 2 * hr], ep.alpha), v1 = __fmul_rn(acc[4 * i + 2 * hr + 1], ep.alpha);
            if (ep.addend != nullptr) { v0 += add[hr][j].x; v1 += add[hr][j].y; }
            if (ep.atomic) {
              float* op = reinterpret_cast<float*>(ep.out) + orow[hr] + col;
              if (pair) asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(op), "f"(v0), "f"(v1) : "memory");
              else { atomicAdd(op, v0); if (col + 1 < ep.n_valid) atomicAdd(op + 1, v1); }
            } else if (ep.out_f32) {
              float* op = reinterpret_cast<float*>(ep.out) + split * ep.split_stride + orow[hr] + col;
              if (pair) *reinterpret_cast<float2*>(op) = make_float2(v0, v1);
              else { op[0] = v0; if (col + 1 < ep.n_valid) op[1] = v1; }
            } else {
              __nv_bfloat16* op = reinterpret_cast<__nv_bfloat16*>(ep.out) + orow[hr] + col;
              if (pair) *reinterpret_cast<uint32_t*>(op) = pack_bf16x2(v0, v1);
              else { op[0] = __float2bfloat16_rn(v0); if (col + 1 < ep.n_valid) op[1] = __float2bfloat16_rn(v1); }
            }
          }
        }
      }
    }
  }
  if (ep.staged && leader) tma_store_wait_all();   // the boxes stay allocated until the last stores have completed
}

constexpr int kMaxDynSmem = 232448;      // 227 KB per CTA on sm_90
constexpr int kBarrierBytes = 256;

template <int BN, int A_MN, int B_MN, bool RS = false>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmO, const CUtensorMap& tmE,
                       const EpiParams& ep, int M, int N, int K, int splits, int max_ctas, int f16, cudaStream_t stream) {
  using S = GemmSmem<BN>;
  auto kern = f16 ? gemm_bf16_kernel<BN, A_MN, B_MN, true, RS> : gemm_bf16_kernel<BN, A_MN, B_MN, false, RS>;
  const int staging = ep.staged ? kStagingBytes : 0;
  int stages = (kMaxDynSmem - 1024 - kBarrierBytes - staging) / S::kStageBytes;
  if (stages > 6) stages = 6;
  const int smem_bytes = stages * S::kStageBytes + staging + kBarrierBytes + 1024;
  static bool configured[2] = {false, false};
  if (!configured[f16]) {
    OMLM_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxDynSmem));
    configured[f16] = true;
  }
  const int m_tiles = (M + BM - 1) / BM, n_tiles = (N + BN - 1) / BN;
  const int work = m_tiles * n_tiles * splits;
  int grid = num_sms();
  if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
  if (work < grid) grid = work;
  OMLM_KLAUNCH((kern), grid, kGemmThreads, smem_bytes, stream, tmA, tmB, tmO, tmE, ep, M, N, K, splits, stages);
  OMLM_LAUNCH_CHECK();
  return 0;
}

}  // namespace omlm

namespace omlm {
struct RowStatArgs { const void* hn; long ldhn; const void* keep_bits; const float* gamma; float keep_scale; float* part; int parts; };
}

static int gemm16_impl(const void* A, int a_f16, int a_mn_major, long lda, const void* B, int b_f16, int b_mn_major,
                       long ldb, int M, int N, int K, void* out, int out_f32, long ldo,
                       const float* addend, long ldadd, float alpha, int splits,
                       int row_split, int row_valid, int n_valid, int block_n, int max_ctas,
                       void* stream_, const omlm::RowStatArgs* rs, long split_stride = 0) {
  using namespace omlm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  OMLM_CHECK_ARG(M > 0 && N > 0 && K > 0, "gemm: empty problem %d x %d x %d", M, N, K);
  OMLM_CHECK_ARG(block_n == 128 || block_n == 256, "gemm: block_n must be 128 or 256");
  OMLM_CHECK_ARG(splits >= 1, "gemm: splits must be >= 1");
  OMLM_CHECK_ARG((a_f16 != 0) == (b_f16 != 0), "gemm: both operands must have the same 16-bit format (one wgmma takes one operand format)");
  OMLM_CHECK_ARG(splits == 1 || (out_f32 && addend == nullptr), "gemm: split-K needs fp32 atomic output and no addend");
  OMLM_CHECK_ARG(split_stride == 0 || (out_f32 && addend == nullptr && rs == nullptr), "gemm: partial slices need fp32 output");
  if (n_valid <= 0 || n_valid > N) n_valid = N;
  // split-K adds onto the output's contents; that stays so when the clamp below leaves a single split
  const bool accumulate = splits > 1 && split_stride == 0;
  {  // every split must own at least one k-block (an empty split would publish an unwritten accumulator)
    const int kb_total = (K + BK - 1) / BK;
    if (splits > kb_total) splits = kb_total;
    const int per = (kb_total + splits - 1) / splits;
    splits = (kb_total + per - 1) / per;
  }
  CUtensorMap tmA, tmB;
  int rc;
  if (a_mn_major == 0) rc = make_tmap_bf16_2d(&tmA, A, (uint64_t)K, (uint64_t)M, (uint64_t)lda * 2, 64, BM);
  else                 rc = make_tmap_bf16_2d(&tmA, A, (uint64_t)M, (uint64_t)K, (uint64_t)lda * 2, 64, 64);
  if (rc) return rc;
  if (b_mn_major == 0) rc = make_tmap_bf16_2d(&tmB, B, (uint64_t)K, (uint64_t)N, (uint64_t)ldb * 2, 64, block_n);
  else                 rc = make_tmap_bf16_2d(&tmB, B, (uint64_t)N, (uint64_t)K, (uint64_t)ldb * 2, 64, 64);
  if (rc) return rc;
  EpiParams ep;
  ep.out = out; ep.addend = addend; ep.ldo = ldo; ep.ldadd = ldadd; ep.alpha = alpha;
  ep.out_f32 = out_f32; ep.atomic = accumulate ? 1 : 0; ep.split_stride = split_stride;
  const long esz = out_f32 ? 4 : 2;
  ep.vec_ok = ((ldo * esz) % 16 == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0) &&
              (addend == nullptr || ((ldadd * 4) % 16 == 0 && (reinterpret_cast<uintptr_t>(addend) & 15) == 0));
  ep.row_split = row_split; ep.row_valid = row_valid; ep.n_valid = n_valid;
  ep.rs_gamma = nullptr; ep.rs_keep = nullptr; ep.rs_part = nullptr; ep.rs_keep_scale = 1.f; ep.rs_parts = 0;
  // The staged epilogue stores whole boxes of tile rows by TMA: the output rows must be the tile's rows, without
  // atomics, and TMA needs 16-byte-aligned bases and pitches.  The boxes hold one element type, so an addend goes
  // with an fp32 output.  Stores are clipped to M x n_valid by the map, but only at 16-byte granularity in a row,
  // so n_valid must end on a 16-byte boundary.
  ep.staged = !ep.atomic && split_stride == 0 && row_split == 0 && ep.vec_ok && (addend == nullptr || out_f32) &&
              (n_valid * esz) % 16 == 0;
  CUtensorMap tmO, tmE;
  memset(&tmO, 0, sizeof(tmO));
  memset(&tmE, 0, sizeof(tmE));
  if (ep.staged) {
    rc = make_tmap_2d(&tmO, static_cast<int>(esz), out, (uint64_t)n_valid, (uint64_t)M, (uint64_t)(ldo * esz), out_f32 ? 32 : 64, 64);
    if (rc == 0 && addend != nullptr) rc = make_tmap_2d(&tmE, 4, addend, (uint64_t)n_valid, (uint64_t)M, (uint64_t)(ldadd * 4), 32, 64);
    if (rc) return rc;
  }
  const int f16 = a_f16 ? 1 : 0;
  const int key = (block_n == 256 ? 4 : 0) | (a_mn_major ? 2 : 0) | (b_mn_major ? 1 : 0);
  if (rs != nullptr) {
    OMLM_CHECK_ARG(block_n == 256 && N % 256 == 0 && n_valid == N && !out_f32 && addend == nullptr && splits == 1 && row_split == 0 &&
                   ep.vec_ok && rs->parts == 2 * (N / 256) && rs->ldhn % 8 == 0 && (reinterpret_cast<uintptr_t>(rs->hn) & 15) == 0,
                   "gemm row statistics: needs 256-wide tiles, N %% 256 == 0, a dense bf16 output, 16-byte-aligned hn rows "
                   "and parts == N / 128");
    OMLM_CHECK_ARG(key == 5, "gemm row statistics: only the A K-major / B MN-major 256-wide instantiation exists");
    rc = make_tmap_2d(&tmE, 2, rs->hn, (uint64_t)N, (uint64_t)M, (uint64_t)rs->ldhn * 2, 64, 64);
    if (rc) return rc;
    ep.rs_gamma = rs->gamma; ep.rs_keep = reinterpret_cast<const uint8_t*>(rs->keep_bits);
    ep.rs_part = reinterpret_cast<float2*>(rs->part); ep.rs_keep_scale = rs->keep_scale; ep.rs_parts = rs->parts;
    return launch_gemm<256, 0, 1, true>(tmA, tmB, tmO, tmE, ep, M, N, K, splits, max_ctas, f16, stream);
  }
  switch (key) {
    case 0: return launch_gemm<128, 0, 0>(tmA, tmB, tmO, tmE, ep, M, N, K, splits, max_ctas, f16, stream);
    case 1: return launch_gemm<128, 0, 1>(tmA, tmB, tmO, tmE, ep, M, N, K, splits, max_ctas, f16, stream);
    case 3: return launch_gemm<128, 1, 1>(tmA, tmB, tmO, tmE, ep, M, N, K, splits, max_ctas, f16, stream);
    case 4: return launch_gemm<256, 0, 0>(tmA, tmB, tmO, tmE, ep, M, N, K, splits, max_ctas, f16, stream);
    case 5: return launch_gemm<256, 0, 1>(tmA, tmB, tmO, tmE, ep, M, N, K, splits, max_ctas, f16, stream);
    case 7: return launch_gemm<256, 1, 1>(tmA, tmB, tmO, tmE, ep, M, N, K, splits, max_ctas, f16, stream);
    default:
      set_last_error("gemm: operand majors (a_mn=%d, b_mn=%d) not instantiated", a_mn_major, b_mn_major);
      return 1;
  }
}

extern "C" int omlm_gemm16(const void* A, int a_f16, int a_mn_major, long lda, const void* B, int b_f16, int b_mn_major,
                           long ldb, int M, int N, int K, void* out, int out_f32, long ldo,
                           const float* addend, long ldadd, float alpha, int splits,
                           int row_split, int row_valid, int n_valid, int block_n, int max_ctas,
                           void* stream_) {
  return gemm16_impl(A, a_f16, a_mn_major, lda, B, b_f16, b_mn_major, ldb, M, N, K, out, out_f32, ldo, addend, ldadd, alpha, splits,
                     row_split, row_valid, n_valid, block_n, max_ctas, stream_, nullptr);
}

namespace omlm {
// out[r, c] = out[r, c] + part[0][r, c] + part[1][r, c] + ... (split order) over rows_out x n_valid
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(float* __restrict__ out, long ldo, const float* __restrict__ part, long slice, long ldp, int splits,
                     int rows_out, int n_valid) {
  const long total = static_cast<long>(rows_out) * n_valid;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const long r = i / n_valid, c = i - r * n_valid;
    float v = out[r * ldo + c];
    for (int s = 0; s < splits; ++s) v += part[s * slice + r * ldp + c];
    out[r * ldo + c] = v;
  }
}

// rows of the output a GEMM with this row remap writes (row_split > 0: whole halves of row_split rows, row_valid live
// rows each; < 0: value and gate halves of row_valid channels; 0: M)
static int gemm_rows_out(int M, int row_split, int row_valid) {
  if (row_split > 0) return (M + row_split - 1) / row_split * row_valid;
  if (row_split < 0) return 2 * row_valid;
  return M;
}

static int gemm_splits_effective(int K, int splits) {   // the clamp of gemm16_impl: every split owns >= 1 k-block
  const int kb_total = (K + BK - 1) / BK;
  if (splits > kb_total) splits = kb_total;
  if (splits < 1) splits = 1;
  const int per = (kb_total + splits - 1) / splits;
  return (kb_total + per - 1) / per;
}
}  // namespace omlm

extern "C" int omlm_gemm16_splitk_det_workspace(int M, int N, int K, int splits, int row_split, int row_valid, int n_valid,
                                                long* part_bytes) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && N > 0 && K > 0 && splits >= 1 && part_bytes != nullptr, "gemm16_splitk_det_workspace: bad arguments");
  if (n_valid <= 0 || n_valid > N) n_valid = N;
  OMLM_CHECK_ARG(row_split <= 0 || M % row_split == 0, "gemm16_splitk_det: M (%d) must be whole halves of row_split (%d)", M, row_split);
  const int s = gemm_splits_effective(K, splits);
  *part_bytes = s > 1 ? static_cast<long>(s) * gemm_rows_out(M, row_split, row_valid) * ((n_valid + 3) / 4 * 4) * 4 : 0;
  return 0;
}

extern "C" int omlm_gemm16_splitk_det(const void* A, int a_f16, int a_mn_major, long lda, const void* B, int b_f16, int b_mn_major,
                                      long ldb, int M, int N, int K, float* out, long ldo, int splits, int row_split, int row_valid,
                                      int n_valid, int block_n, int max_ctas, float* part_ws, long part_ws_bytes, void* stream_) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && N > 0 && K > 0 && splits >= 1, "gemm16_splitk_det: empty problem %d x %d x %d", M, N, K);
  if (n_valid <= 0 || n_valid > N) n_valid = N;
  const int s = gemm_splits_effective(K, splits);
  // every partial row the reduction reads must be written by some split: a remap of row_split > 0 needs whole halves
  OMLM_CHECK_ARG(row_split <= 0 || M % row_split == 0, "gemm16_splitk_det: M (%d) must be whole halves of row_split (%d)", M, row_split);
  if (s == 1)         // one split: the plain in-place accumulation (out += A B through the addend)
    return gemm16_impl(A, a_f16, a_mn_major, lda, B, b_f16, b_mn_major, ldb, M, N, K, out, 1, ldo, out, ldo, 1.f, 1,
                       row_split, row_valid, n_valid, block_n, max_ctas, stream_, nullptr);
  const int rows_out = gemm_rows_out(M, row_split, row_valid);
  const long ldp = (n_valid + 3) / 4 * 4;
  const long slice = static_cast<long>(rows_out) * ldp;
  OMLM_CHECK_ARG(part_ws != nullptr && part_ws_bytes >= s * slice * 4 && (reinterpret_cast<uintptr_t>(part_ws) & 15) == 0,
                 "gemm16_splitk_det: partials need %ld bytes (16-byte aligned), got %ld", s * slice * 4, part_ws_bytes);
  int rc = gemm16_impl(A, a_f16, a_mn_major, lda, B, b_f16, b_mn_major, ldb, M, N, K, part_ws, 1, ldp, nullptr, 0, 1.f, s,
                       row_split, row_valid, n_valid, block_n, max_ctas, stream_, nullptr, slice);
  if (rc) return rc;
  const long total = static_cast<long>(rows_out) * n_valid;
  const int grid = static_cast<int>(std::min<long>((total + 255) / 256, static_cast<long>(num_sms()) * 8));
  OMLM_KLAUNCH((splitk_reduce_kernel), grid, 256, 0, reinterpret_cast<cudaStream_t>(stream_), out, ldo,
               static_cast<const float*>(part_ws), slice, ldp, s, rows_out, n_valid);
  OMLM_LAUNCH_CHECK();
  return 0;
}

extern "C" int omlm_gemm16_rowstat(const void* A, int a_f16, int a_mn_major, long lda, const void* B, int b_f16, int b_mn_major,
                                   long ldb, int M, int N, int K, void* out_bf16, long ldo, const void* hn_bf16, long ldhn,
                                   const void* keep_bits, const float* gamma, float keep_scale, float* part, int parts,
                                   int max_ctas, void* stream_) {
  omlm::RowStatArgs rs{hn_bf16, ldhn, keep_bits, gamma, keep_scale, part, parts};
  return gemm16_impl(A, a_f16, a_mn_major, lda, B, b_f16, b_mn_major, ldb, M, N, K, out_bf16, 0, ldo, nullptr, 0, 1.f, 1,
                     0, 0, N, 256, max_ctas, stream_, &rs);
}

extern "C" int omlm_gemm_bf16(const void* A, int a_mn_major, long lda, const void* B, int b_mn_major,
                              long ldb, int M, int N, int K, void* out, int out_f32, long ldo,
                              const float* addend, long ldadd, float alpha, int splits,
                              int row_split, int row_valid, int n_valid, int block_n, int max_ctas,
                              void* stream_) {
  return omlm_gemm16(A, 0, a_mn_major, lda, B, 0, b_mn_major, ldb, M, N, K, out, out_f32, ldo, addend, ldadd, alpha, splits,
                     row_split, row_valid, n_valid, block_n, max_ctas, stream_);
}
