// Weight-streaming GEMM of the incremental decode step for 1..256 rows, on the wgmma tensor cores.
//
// The SIMT skinny_gemm (csrc/decode.cu) does 2 B N K fp32 FMAs per step; above ~16 rows that arithmetic, not the weight
// stream, bounds it.  Here the operands are swapped so that the tensor cores take the work:
//   M = 64 weight rows per consumer warpgroup (one or two warpgroups: 64- or 128-row tiles),
//   N = the batch, padded to Bp = 64, 128 or 256 (TMA fills the rows >= B with zeros),
//   K in 64-element blocks.
// Both operands are TMA-loaded K-major with the 128B swizzle into a multi-stage mbarrier ring fed by one producer thread.
// The activation operand is built once per call by a small prologue kernel into a packed 16-bit [B, K] buffer, with
// the rounding points of skinny_gemm (the LayerNorm statistics are computed once per row, not in every CTA); 16-bit
// rows that TMA can read in place skip it.
//
// A step's matrices have few 64-row tiles (musiclm_small: 2 .. 88), so the K range is split over CTAs until the grid
// covers the SMs -- but only as far as the fp32 partials stay small against the weights (their bytes grow with the
// batch).  The partials go to a workspace and a reduction kernel sums them in split order 0, 1, ... -- a fixed order,
// no floating-point atomics: bit-identical results from call to call and between eager launches and CUDA-graph
// replays -- then applies the addend and stores.
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/omlm_b200.h"

namespace omlm {

constexpr int kDgMaxB = 256;
constexpr int kDgBK = 64;                 // 64 16-bit elements = 128 bytes = one swizzle row
constexpr int kDgSmemBudget = 200 * 1024;

// ------------------------------------------------------------------------------------------------ activation prologue
// Row b of the 16-bit operand, exactly as skinny_gemm builds it in shared memory (same statistics, same expressions).
// grid B, 128 threads; a16 [B, K] packed.
template <bool F16>
__global__ void __launch_bounds__(128)
decode_gemm_prologue_kernel(const void* __restrict__ A, long lda, int prologue, const float* __restrict__ gamma,
                            const float* __restrict__ rowsum, int n_real, uint16_t* __restrict__ a16, int K) {
  pdl_prologue();
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  __shared__ float s_mean, s_rstd;
  if (prologue >= 2) {
    if (tid < 32) {
      float mean, rstd;
      if (prologue == 2) {
        const float* x = reinterpret_cast<const float*>(A) + b * lda;
        float s = 0.f;
        for (int k = lane; k < K; k += 32) s += x[k];
        mean = warp_sum(s) / K;
        float q = 0.f;
        for (int k = lane; k < K; k += 32) { const float d = x[k] - mean; q += d * d; }
        rstd = rsqrtf(warp_sum(q) / K + 1e-5f);
      } else {
        const float2* rs = reinterpret_cast<const float2*>(rowsum) + static_cast<long>(b) * (K >> 7);
        float s1 = 0.f, s2 = 0.f;
        for (int t = lane; t < (K >> 7); t += 32) { s1 += rs[t].x; s2 += rs[t].y; }
        s1 = warp_sum(s1); s2 = warp_sum(s2);
        mean = s1 / n_real;
        rstd = rsqrtf(fmaxf(s2 / n_real - mean * mean, 0.f) + 1e-5f);
      }
      if (lane == 0) { s_mean = mean; s_rstd = rstd; }
    }
    __syncthreads();
  }
  uint32_t* dst = reinterpret_cast<uint32_t*>(a16 + static_cast<long>(b) * K);
  for (int k = tid * 2; k < K; k += 256) {
    uint32_t v;
    if (prologue == 0) {
      v = *reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint16_t*>(A) + b * lda + k);
    } else if (prologue == 1) {
      const float* x = reinterpret_cast<const float*>(A) + b * lda + k;
      v = pack16x2<F16>(x[0], x[1]);
    } else if (prologue == 2) {
      const float* x = reinterpret_cast<const float*>(A) + b * lda + k;
      v = pack16x2<F16>((x[0] - s_mean) * s_rstd * gamma[k], (x[1] - s_mean) * s_rstd * gamma[k + 1]);
    } else {
      const float2 hv = unpack16x2<F16>(*reinterpret_cast<const uint32_t*>(reinterpret_cast<const uint16_t*>(A) + b * lda + k));
      v = pack16x2<F16>((hv.x - s_mean) * s_rstd * gamma[k], (hv.y - s_mean) * s_rstd * gamma[k + 1]);
    }
    dst[k >> 1] = v;
  }
}

// ------------------------------------------------------------------------------------------------ GEMM
template <int BN, int WGS>
struct DgSmem {
  static constexpr int kWBytes = WGS * 64 * kDgBK * 2;       // WGS x 64 weight rows
  static constexpr int kABytes = BN * kDgBK * 2;             // Bp activation rows
  static constexpr int kStageBytes = kWBytes + kABytes;
  static constexpr int kMaxStages = kDgSmemBudget / kStageBytes > 8 ? 8 : kDgSmemBudget / kStageBytes;
  static constexpr int kBytes = kMaxStages * kStageBytes + 1024 + 2 * kMaxStages * 8;   // + alignment slack, barriers
};

struct DgEpi {
  void* out; const float* addend; float* part;
  long ldo, ldadd;
  int out_fmt;
};

// Accumulator element i of a thread with fragment row `row` (weight row, before the +8 of the upper half) and column
// pair qc: acc[4 j + 2 hr + e] = out[b = 8 j + 2 qc + e, n = row + 8 hr].
__device__ __forceinline__ void dg_store(const DgEpi& ep, int B, int N, int row, int i, int qc, float v) {
  const int n = row + ((i >> 1) & 1) * 8, b = (i >> 2) * 8 + qc * 2 + (i & 1);
  if (n >= N || b >= B) return;
  if (ep.addend != nullptr) v += ep.addend[b * ep.ldadd + n];
  if (ep.out_fmt == kFmtF32) reinterpret_cast<float*>(ep.out)[b * ep.ldo + n] = v;
  else if (ep.out_fmt == kFmtF16) reinterpret_cast<__half*>(ep.out)[b * ep.ldo + n] = __float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f));
  else reinterpret_cast<__nv_bfloat16*>(ep.out)[b * ep.ldo + n] = __float2bfloat16_rn(v);
}

// grid (tiles, splits); WGS consumer warpgroups + one producer warp.
template <int BN, int WGS, bool F16>
__global__ void __launch_bounds__(WGS * 128 + 32, 1)
decode_gemm_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmA, const DgEpi ep,
                   const int B, const int N, const int K, const int kb_per_split, const int stages) {
  pdl_launch_dependents();
  using S = DgSmem<BN, WGS>;
  constexpr int kConsumers = WGS * 128;
  extern __shared__ uint8_t dg_smem_raw[];
  uint8_t* smem = dg_smem_raw + ((1024u - (smem_u32(dg_smem_raw) & 1023u)) & 1023u);   // 128B-swizzle atoms: 1024B aligned
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + stages * S::kStageBytes);
  uint64_t* empty_bar = full_bar + S::kMaxStages;

  const int tile = blockIdx.x, split = blockIdx.y;
  const int kb_total = (K + kDgBK - 1) / kDgBK;
  const int kb0 = split * kb_per_split, kb1 = min(kb_total, kb0 + kb_per_split);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmA);
    for (int i = 0; i < stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], WGS);      // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();

  if (threadIdx.x >= kConsumers) {
    // ------------------------------------------------------------------ TMA producer (one thread)
    if (threadIdx.x == kConsumers) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sw = smem + stage * S::kStageBytes;
        mbar_expect_tx(&full_bar[stage], S::kStageBytes);     // out-of-range rows / columns arrive as zeros, counted in full
        tma_load_2d(sw, &tmW, &full_bar[stage], kb * kDgBK, tile * 64 * WGS);
        tma_load_2d(sw + S::kWBytes, &tmA, &full_bar[stage], kb * kDgBK, 0);
        if (++stage == stages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: 64 weight rows x Bp batch rows each
  const int cw = threadIdx.x >> 7;
  const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, qr = lane >> 2, qc = lane & 3;
  const bool leader = (threadIdx.x & 127) == 0;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  int stage = 0, prev = -1;
  uint32_t phase = 0;
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sw = smem_u32(smem + stage * S::kStageBytes) + cw * 8192;
    const uint32_t sa = smem_u32(smem + stage * S::kStageBytes + S::kWBytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kDgBK / 16; ++k) {
      const uint32_t accum = (kb > kb0 || k > 0) ? 1u : 0u;
      Wgmma<BN, F16>::template ss<0, 0>(acc, make_smem_desc(sw + k * 32, 16, 1024), make_smem_desc(sa + k * 32, 16, 1024), accum);
    }
    wgmma_commit();
    wgmma_wait<1>();                                      // the previous k-block's wgmma have read their slot
    if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == stages) { stage = 0; phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_reg_fence(acc);

  if (gridDim.y > 1) {                                    // split-K: partials, summed in order by decode_gemm_reduce_kernel
    float* mine = ep.part + (static_cast<long>(split) * gridDim.x + tile) * (BN / 2) * kConsumers + threadIdx.x;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) __stcg(mine + i * kConsumers, acc[i]);
    return;
  }
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) dg_store(ep, B, N, tile * 64 * WGS + cw * 64 + wq * 16 + qr, i, qc, acc[i]);
}

// Split-K: out = sum of the partials in split order 0, 1, ... (+ addend).  One thread per accumulator element, laid out
// like the partials (consecutive threads = consecutive consumer threads: coalesced loads).
template <int BN, int WGS>
__global__ void __launch_bounds__(256)
decode_gemm_reduce_kernel(const DgEpi ep, const int B, const int N, const int tiles, const int splits) {
  pdl_prologue();
  constexpr int kConsumers = WGS * 128;
  const long per_split = static_cast<long>(tiles) * (BN / 2) * kConsumers;
  const long idx = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= per_split) return;
  const int t = static_cast<int>(idx % kConsumers);
  const long ti = idx / kConsumers;
  const int i = static_cast<int>(ti % (BN / 2)), tile = static_cast<int>(ti / (BN / 2));
  float v = __ldcg(ep.part + idx);
  for (int s = 1; s < splits; ++s) v += __ldcg(ep.part + s * per_split + idx);
  const int cw = t >> 7, wq = (t >> 5) & 3, lane = t & 31;
  dg_store(ep, B, N, tile * 64 * WGS + cw * 64 + wq * 16 + (lane >> 2), i, lane & 3, v);
}

// ------------------------------------------------------------------------------------------------ host side
struct DgPlan {
  int bn, wgs, tiles, splits, kb_per_split;
  long part_floats;
};

// Batch padding, tile height and K split of one call: enough CTAs to cover the SMs, every split non-empty, and at most
// K / Bp splits, so that the partials (written and read: 8 Bp bytes per output row and split) stay within 4x the
// weight bytes (2 K per row) -- they live in L2, the weights come from HBM.
static DgPlan dg_plan(int B, int N, int K) {
  DgPlan p;
  p.bn = B <= 64 ? 64 : (B <= 128 ? 128 : 256);
  p.wgs = p.bn >= 128 ? 2 : 1;                    // wider batches: 128-row tiles halve the re-reads of the activations
  p.tiles = (N + 64 * p.wgs - 1) / (64 * p.wgs);
  const int kb = (K + kDgBK - 1) / kDgBK;
  int splits = (num_sms() + p.tiles - 1) / p.tiles;
  const int cap = K / p.bn;
  splits = splits > cap ? cap : splits;
  splits = splits < 1 ? 1 : (splits > kb ? kb : splits);
  p.kb_per_split = (kb + splits - 1) / splits;
  p.splits = (kb + p.kb_per_split - 1) / p.kb_per_split;
  p.part_floats = p.splits > 1 ? static_cast<long>(p.splits) * p.tiles * 64 * p.wgs * p.bn : 0;
  return p;
}

template <int BN, int WGS, bool F16>
static int dg_launch(const CUtensorMap& tmW, const CUtensorMap& tmA, const DgEpi& ep, const DgPlan& p, int B, int N, int K,
                     cudaStream_t stream) {
  using S = DgSmem<BN, WGS>;
  static bool configured = false;                 // the largest ring, once: later calls (graph capture) set nothing
  if (!configured) {
    OMLM_CUDA(cudaFuncSetAttribute(decode_gemm_kernel<BN, WGS, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize, S::kBytes));
    configured = true;
  }
  const int stages = p.kb_per_split < S::kMaxStages ? p.kb_per_split : S::kMaxStages;
  const int smem = stages * S::kStageBytes + 1024 + 2 * S::kMaxStages * 8;
  OMLM_KLAUNCH((decode_gemm_kernel<BN, WGS, F16>), dim3(p.tiles, p.splits), WGS * 128 + 32, smem, stream, tmW, tmA, ep, B, N, K,
               p.kb_per_split, stages);
  OMLM_LAUNCH_CHECK();
  if (p.splits > 1) {
    const long elems = static_cast<long>(p.tiles) * (BN / 2) * WGS * 128;
    OMLM_KLAUNCH((decode_gemm_reduce_kernel<BN, WGS>), static_cast<unsigned>((elems + 255) / 256), 256, 0, stream, ep, B, N, p.tiles, p.splits);
    OMLM_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace omlm

extern "C" {

int omlm_decode_gemm_workspace(int B, int N, int K, long* part_bytes) {
  using namespace omlm;
  OMLM_CHECK_ARG(B >= 1 && B <= kDgMaxB && N > 0 && K > 0, "decode_gemm_workspace: bad shape B=%d N=%d K=%d", B, N, K);
  const DgPlan p = dg_plan(B, N, K);
  if (part_bytes != nullptr) *part_bytes = p.part_floats * 4;
  return 0;
}

int omlm_decode_gemm(const void* A, long lda, int prologue, const void* W, long ldw, int w_f16, const float* gamma,
                     const float* rowsum, int n_real, const float* addend, long ldadd, void* out, int out_fmt, long ldo,
                     int B, int N, int K, void* a16_ws, float* part_ws, long part_ws_bytes, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(B >= 1 && B <= kDgMaxB, "decode_gemm: batch %d out of range (1..%d)", B, kDgMaxB);
  OMLM_CHECK_ARG(N > 0 && K > 0 && K % 8 == 0 && ldw % 8 == 0, "decode_gemm: K and ldw must be multiples of 8 (K=%d ldw=%ld)", K, ldw);
  OMLM_CHECK_ARG(prologue >= 0 && prologue <= 3, "decode_gemm: prologue %d", prologue);
  OMLM_CHECK_ARG((prologue < 2) || gamma != nullptr, "decode_gemm: LayerNorm prologue needs gamma");
  OMLM_CHECK_ARG(prologue != 3 || (rowsum != nullptr && K % 128 == 0 && n_real > 0), "decode_gemm: inner-norm prologue needs rowsum and K % 128 == 0");
  OMLM_CHECK_ARG(out_fmt == kFmtBF16 || out_fmt == kFmtF32 || out_fmt == kFmtF16, "decode_gemm: out_fmt");
  OMLM_CHECK_ARG((reinterpret_cast<uintptr_t>(W) & 15) == 0, "decode_gemm: W must be 16-byte aligned");
  const DgPlan p = dg_plan(B, N, K);
  OMLM_CHECK_ARG(part_ws_bytes >= p.part_floats * 4 && (p.part_floats == 0 || part_ws != nullptr),
                 "decode_gemm: split-K workspace of %ld bytes, %ld needed", part_ws_bytes, p.part_floats * 4);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // the activation operand: 16-bit rows TMA can read in place, else built once into a16_ws [B, K]
  const void* a_op = A;
  long a_ld = lda;
  const bool in_place = prologue == 0 && (reinterpret_cast<uintptr_t>(A) & 15) == 0 && lda % 8 == 0;
  if (!in_place) {
    OMLM_CHECK_ARG(a16_ws != nullptr && (reinterpret_cast<uintptr_t>(a16_ws) & 15) == 0, "decode_gemm: needs a 16-byte aligned [B, K] 16-bit workspace");
    if (w_f16) OMLM_KLAUNCH((decode_gemm_prologue_kernel<true>), B, 128, 0, st, A, lda, prologue, gamma, rowsum, n_real, reinterpret_cast<uint16_t*>(a16_ws), K);
    else       OMLM_KLAUNCH((decode_gemm_prologue_kernel<false>), B, 128, 0, st, A, lda, prologue, gamma, rowsum, n_real, reinterpret_cast<uint16_t*>(a16_ws), K);
    OMLM_LAUNCH_CHECK();
    a_op = a16_ws;
    a_ld = K;
  }
  CUtensorMap tmW, tmA;
  int rc = make_tmap_bf16_2d(&tmW, W, static_cast<uint64_t>(K), static_cast<uint64_t>(N), static_cast<uint64_t>(ldw) * 2, 64, 64 * p.wgs);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmA, a_op, static_cast<uint64_t>(K), static_cast<uint64_t>(B), static_cast<uint64_t>(a_ld) * 2, 64, p.bn);
  if (rc) return rc;
  DgEpi ep;
  ep.out = out; ep.addend = addend; ep.part = part_ws; ep.ldo = ldo; ep.ldadd = ldadd; ep.out_fmt = out_fmt;
  if (p.bn == 64)  return w_f16 ? dg_launch<64, 1, true>(tmW, tmA, ep, p, B, N, K, st) : dg_launch<64, 1, false>(tmW, tmA, ep, p, B, N, K, st);
  if (p.bn == 128) return w_f16 ? dg_launch<128, 2, true>(tmW, tmA, ep, p, B, N, K, st) : dg_launch<128, 2, false>(tmW, tmA, ep, p, B, N, K, st);
  return w_f16 ? dg_launch<256, 2, true>(tmW, tmA, ep, p, B, N, K, st) : dg_launch<256, 2, false>(tmW, tmA, ep, p, B, N, K, st);
}

}  // extern "C"
