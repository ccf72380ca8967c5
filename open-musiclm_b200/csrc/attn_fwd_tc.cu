// Fused causal multi-query cosine-sim attention, forward, on the Hopper tensor cores (wgmma + TMA + mbarrier).
//
//   sim = 8 * qn . kn + table[hh, i-j];  key-padding mask; causal mask; softmax (fp32); out = P v
//   (transformer.py:304-331; q/k arrive l2-normalised and scaled, transformer.py:269-271)
//
// Folded-row layout (attn_common.cuh): per batch element the h heads of MQA are R = N*h query rows,
// row r = i*h + head, sharing one K/V head.  A CTA owns one 128-row query tile and streams 128-key K/V tiles
// through a 2-stage TMA ring:
//
//   warpgroup 0     TMA producer (Q tile once, K/V ring)
//   warpgroups 1,2  64 query rows each: S = Q K^T (wgmma m64n128k16, operands in 128B-swizzled smem, S in registers),
//                   online softmax in the log2 domain on the accumulator fragment (a row lives in the four lanes of a
//                   quad), P -> bf16 in registers, O += P V (wgmma m64n64k16 with A from registers, V read MN-major).
//                   While S is in flight each warpgroup stages the Toeplitz bias window of its 64 rows and the key tile
//                   (per head, deltas i_lo - j0 - 127 .. i_hi - j0, pre-scaled by log2 e, -inf for delta < 0 so the
//                   causal mask costs nothing) in shared memory and ballots the tile's key mask into four words; the
//                   softmax then reads the bias with LDS instead of one gathered global load per score.
#include "common.cuh"
#include "ptx.cuh"
#include "../../include/omlm_b200.h"

namespace omlm {

constexpr int kTcThreads = 384;
constexpr int kTcBQ = 128;      // query rows per CTA (64 per consumer warpgroup)
constexpr int kTcBK = 128;      // keys per tile
constexpr float kL2e = 1.4426950408889634f;

// smem carve-up (offsets from a 1024-aligned base)
constexpr int kOffQ = 0;                        // 16 KB
constexpr int kOffK = 16384;                    // 2 x 16 KB
constexpr int kOffV = 49152;                    // 2 x 16 KB
constexpr int kOffBar = 81920;                  // barriers
constexpr int kOffWin = kOffBar + 64;           // bias windows: [2 warpgroups][2 buffers][h][win_ld] floats
constexpr int kTcMaxSmem = 232448;

// Row stride of a bias window: a warpgroup's 64 rows span at most ceil(63 / h) + 1 positions, so a window holds at most
// ceil(63 / h) + 128 deltas.  The stride is 8 mod 32 floats so the eight rows of a quad column (eight heads at h = 8)
// read from at most two rows per bank.
static int fwd_win_ld(int h) { return ((62 + h) / h + 128 + 23) / 32 * 32 + 8; }
static int fwd_smem(int h) { return kOffWin + 4 * h * fwd_win_ld(h) * 4 + 1024; }

__device__ __forceinline__ float ex2_fast(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// kVarlen: sequences of their own lengths packed back to back.  CTA x takes the unit (sequence work[2x], row block
// work[2x + 1]) of a host-built list (heaviest first); sequence b is rows seq_start[b] .. seq_start[b] + seq_len[b] - 1
// of the packed Q and K/V buffers.  N, nbatch and key_mask are then unused (no key mask: visibility is j < seq_len[b]).
// With q_off and kv_start (a chunk of a longer prompt): sequence b's query rows are positions p0 = q_off[b] ..
// p0 + seq_len[b] - 1 (p0 * h a multiple of 128, so its row blocks are row blocks of the whole prompt), and its keys are
// rows kv_start[b] + j of the K/V buffer, visible for j < p0 + seq_len[b].  Key rows past the visible end may hold
// anything; their V rows are zeroed in shared memory, so P = 0 gives exact zero products as TMA zero fill does.
template <bool kVarlen>
__global__ void __launch_bounds__(kTcThreads, 1)
attn_fwd_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmKV,
                   const float* __restrict__ table, int table_ld, const unsigned char* __restrict__ key_mask,
                   __nv_bfloat16* __restrict__ out, float* __restrict__ lse2, int N_fixed, int h, float scale, int nbatch,
                   int win_ld, const int* __restrict__ work, const int* __restrict__ seq_start, const int* __restrict__ seq_len,
                   const int* __restrict__ q_off, const int* __restrict__ kv_start) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // pointer arithmetic (not an integer round trip) keeps the shared address space visible to the compiler: LDS/STS, not generic LD/ST
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* q_full = bars + 0;
  uint64_t* kv_full = bars + 1;    // [2]
  uint64_t* kv_empty = bars + 3;   // [2]

  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
  const int p0 = kVarlen && q_off != nullptr ? q_off[work[2 * blockIdx.x]] : 0;   // varlen: first query row's position
  const int N = kVarlen ? p0 + seq_len[work[2 * blockIdx.x]] : N_fixed;
  const int R = N * h;
  const int nblk = (R + kTcBQ - 1) / kTcBQ;
  // longest-processing-time-first: all batch elements of the heaviest (latest) row block are scheduled first
  const int b = kVarlen ? work[2 * blockIdx.x] : blockIdx.x % nbatch;
  const int rb = kVarlen ? p0 * h / kTcBQ + work[2 * blockIdx.x + 1] : nblk - 1 - blockIdx.x / nbatch;
  const int s0 = kVarlen ? seq_start[b] : 0;    // varlen: first packed row of the sequence
  const int kv0 = kVarlen && kv_start != nullptr ? kv_start[b] : s0;   // varlen: K/V row of key 0
  const int r0 = rb * kTcBQ;
  const int i_max_cta = min(N - 1, (r0 + kTcBQ - 1) / h);
  const int T = i_max_cta / kTcBK + 1;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmKV);
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 2); }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------------------------------------------ TMA producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      mbar_expect_tx(q_full, 16384);
      tma_load_2d(smem + kOffQ, &tmQ, q_full, 0, kVarlen ? (s0 - p0) * h + r0 : b * R + r0);
      for (int t = 0; t < T; ++t) {
        const int st = t & 1;
        mbar_wait(&kv_empty[st], ((t >> 1) & 1) ^ 1);
        mbar_expect_tx(&kv_full[st], 2 * 16384);
        tma_load_2d(smem + kOffK + st * 16384, &tmKV, &kv_full[st], 0, (kVarlen ? kv0 : b * N) + t * kTcBK);
        tma_load_2d(smem + kOffV + st * 16384, &tmKV, &kv_full[st], 64, (kVarlen ? kv0 : b * N) + t * kTcBK);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumer warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int cw = wg - 1;
  const int wq = (threadIdx.x >> 5) & 3, qr = lane >> 2, qc = lane & 3;
  const int tid128 = threadIdx.x & 127;
  const bool leader = tid128 == 0;
  // this warpgroup's rows span positions i_lo .. i_hi; a tile's window starts at delta i_lo - j0 - 127
  const int i_lo = min(r0 + cw * 64, R - 1) / h, i_hi = min(r0 + cw * 64 + 63, R - 1) / h;
  const int win_w = i_hi - i_lo + kTcBK;
  float* win = reinterpret_cast<float*>(smem + kOffWin) + cw * 2 * h * win_ld;   // [2 buffers][h][win_ld]
  int rr[2], woff[2];    // woff: window offset of (row, column 2 qc) in a buffer; column 8 c + e is woff - 8 c - e
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    rr[hr] = r0 + cw * 64 + wq * 16 + qr + hr * 8;
    const int rc = min(rr[hr], R - 1);
    const int i = rc / h;
    woff[hr] = (rc - i * h) * win_ld + i - i_lo + kTcBK - 1 - 2 * qc;
  }
  const unsigned char* km = key_mask != nullptr ? key_mask + static_cast<long long>(b) * N : nullptr;
  const float sc2 = scale * kL2e;
  const uint32_t sq = smem_u32(smem + kOffQ) + cw * 8192, sk = smem_u32(smem + kOffK), sv = smem_u32(smem + kOffV);
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) o[c] = 0.f;

  mbar_wait(q_full, 0);
  for (int t = 0; t < T; ++t) {
    const int st = t & 1;
    mbar_wait(&kv_full[st], (t >> 1) & 1);
    float s[64];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
      Wgmma<128, false>::ss<0, 0>(s, make_smem_desc(sq + ks * 32, 16, 1024), make_smem_desc(sk + st * 16384 + ks * 32, 16, 1024),
                                  ks > 0 ? 1u : 0u);
    wgmma_commit();
    // ---- while S runs: the tile's bias window (buffer t & 1) and key-visibility words (bit l of word k = column 32 k + l)
    const int j0 = t * kTcBK;
    float* wt = win + (t & 1) * h * win_ld;
    {
      const int dlo = i_lo - j0 - (kTcBK - 1);
      for (int x = tid128; x < h * win_w; x += 128) {
        const int hh = x / win_w, w = x - hh * win_w, d = dlo + w;
        wt[hh * win_ld + w] = d >= 0 ? __ldg(table + hh * static_cast<long>(table_ld) + d) * kL2e : -INFINITY;
      }
    }
    uint32_t visw[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int j = j0 + 32 * k + lane;
      visw[k] = __ballot_sync(0xffffffffu, j < N && (km == nullptr || km[j] != 0));
    }
    if constexpr (kVarlen) {
      const int nz = j0 + kTcBK - N;    // key rows past the visible end in this tile: zero V (128 B per row)
      if (nz > 0) {
        uint4* vz = reinterpret_cast<uint4*>(smem + kOffV + st * 16384 + (kTcBK - nz) * 128);
        for (int x = tid128; x < nz * 8; x += 128) vz[x] = make_uint4(0u, 0u, 0u, 0u);
        fence_proxy_async();            // generic-proxy stores before the wgmma reads them (after the barrier below)
      }
    }
    // the buffer written here was last read in tile t - 2, before every thread's barrier of tile t - 1
    asm volatile("bar.sync %0, 128;" ::"r"(1 + cw) : "memory");
    wgmma_wait<0>();
    wgmma_reg_fence(s);
    // ---- bias, masks, row maxima (columns j = j0 + 8 c + 2 qc + {0,1} of this thread's two rows)
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int c = 0; c < 16; ++c) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool vis = (visw[c >> 2] >> (8 * (c & 3) + 2 * qc + e)) & 1u;
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          float& x = s[4 * c + 2 * hr + e];
          x = vis ? fmaf(x, sc2, wt[woff[hr] - 8 * c - e]) : -INFINITY;   // delta < 0: the window holds -inf
          mx[hr] = fmaxf(mx[hr], x);
        }
      }
    }
    float alpha[2], ref[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 1));
      mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 2));
      const float m_new = fmaxf(m[hr], mx[hr]);
      ref[hr] = (m_new == -INFINITY) ? 0.f : m_new;
      alpha[hr] = ex2_fast(m[hr] - ref[hr]);
      m[hr] = m_new;
    }
    // ---- P = exp2(s - ref) -> bf16 A fragments (k16 chunk kk = columns 16 kk .. 16 kk + 15)
    uint32_t pa[8][4];
    float sum[2] = {0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      float p[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) p[e] = ex2_fast(s[8 * kk + e] - ref[(e >> 1) & 1]);
      sum[0] += (p[0] + p[1]) + (p[4] + p[5]);
      sum[1] += (p[2] + p[3]) + (p[6] + p[7]);
      pa[kk][0] = pack_bf16x2(p[0], p[1]);
      pa[kk][1] = pack_bf16x2(p[2], p[3]);
      pa[kk][2] = pack_bf16x2(p[4], p[5]);
      pa[kk][3] = pack_bf16x2(p[6], p[7]);
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) l[hr] = l[hr] * alpha[hr] + sum[hr];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      o[4 * c + 0] *= alpha[0]; o[4 * c + 1] *= alpha[0];
      o[4 * c + 2] *= alpha[1]; o[4 * c + 3] *= alpha[1];
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      Wgmma<64, false>::rs<1>(o, pa[kk], make_smem_desc(sv + st * 16384 + kk * 2048, 8192, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence(o);
    if (leader) mbar_arrive(&kv_empty[st]);
  }
  // ---- finalise: row sums over the quad, normalise, store
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    l[hr] += __shfl_xor_sync(0xffffffffu, l[hr], 1);
    l[hr] += __shfl_xor_sync(0xffffffffu, l[hr], 2);
    if (rr[hr] < R) {
      const float inv = l[hr] > 0.f ? 1.f / l[hr] : 0.f;
      __nv_bfloat16* op = out + ((kVarlen ? static_cast<long long>(s0 - p0) * h : static_cast<long long>(b) * R) + rr[hr]) * 64 + 2 * qc;
#pragma unroll
      for (int c = 0; c < 8; ++c)
        *reinterpret_cast<uint32_t*>(op + 8 * c) = pack_bf16x2(o[4 * c + 2 * hr] * inv, o[4 * c + 2 * hr + 1] * inv);
      if (qc == 0) lse2[(kVarlen ? static_cast<long long>(s0 - p0) * h : static_cast<long long>(b) * R) + rr[hr]] = m[hr] + log2f(l[hr]);
    }
  }
}

}  // namespace omlm

#ifndef OMLM_ATTN_FWD_TC_VARLEN
extern "C" int omlm_attn_fwd_tc(const void* qn, const void* kvn, const float* table, int table_ld,
                                const unsigned char* key_mask, void* out, float* lse2, int B, int N, int heads,
                                float scale, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(B > 0 && N > 0 && heads > 0, "attn_fwd_tc: bad shape");
  OMLM_CHECK_ARG(table_ld >= N, "attn_fwd_tc: bias table shorter than the sequence");
  const int smem = fwd_smem(heads);
  OMLM_CHECK_ARG(smem <= kTcMaxSmem, "attn_fwd_tc: too many heads (%d) for the shared-memory bias windows", heads);
  const long R = static_cast<long>(N) * heads;
  CUtensorMap tmQ, tmKV;
  int rc = make_tmap_bf16_2d(&tmQ, qn, 64, static_cast<uint64_t>(B) * R, 128, 64, kTcBQ);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmKV, kvn, 128, static_cast<uint64_t>(B) * N, 256, 64, kTcBK);
  if (rc) return rc;
  static int configured = 0;
  if (configured < smem) {
    OMLM_CUDA(cudaFuncSetAttribute(attn_fwd_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = smem;
  }
  const unsigned grid = static_cast<unsigned>((R + kTcBQ - 1) / kTcBQ) * B;   // (row block, batch) in LPT order
  OMLM_KLAUNCH((attn_fwd_tc_kernel<false>), grid, kTcThreads, smem, reinterpret_cast<cudaStream_t>(stream),
      tmQ, tmKV, table, table_ld, key_mask, reinterpret_cast<__nv_bfloat16*>(out), lse2, N, heads, scale, B,
      fwd_win_ld(heads), nullptr, nullptr, nullptr, nullptr, nullptr);
  OMLM_LAUNCH_CHECK();
  return 0;
}

#else
// Both varlen entry points: Q from the packed qn, K/V from kv (kv_rows rows of 128), sequence b's keys at kv_start[b]
// (seq_start[b] when kv_start is null), its queries at positions q_off[b] ... (0 when q_off is null).
static int attn_fwd_tc_varlen_launch(const void* qn, const void* kv, long kv_rows, const float* table, int table_ld,
                                     const int* work, int n_work, const int* seq_start, const int* seq_len, const int* q_off,
                                     const int* kv_start, int M, int max_end, void* out, float* lse2, int heads, float scale,
                                     void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && n_work > 0 && max_end > 0 && heads > 0 && kv_rows > 0, "attn_fwd_tc_varlen: bad shape");
  OMLM_CHECK_ARG(table_ld >= max_end, "attn_fwd_tc_varlen: bias table shorter than the longest sequence");
  const int smem = fwd_smem(heads);
  OMLM_CHECK_ARG(smem <= kTcMaxSmem, "attn_fwd_tc_varlen: too many heads (%d) for the shared-memory bias windows", heads);
  CUtensorMap tmQ, tmKV;
  int rc = make_tmap_bf16_2d(&tmQ, qn, 64, static_cast<uint64_t>(M) * heads, 128, 64, kTcBQ);
  if (rc) return rc;
  rc = make_tmap_bf16_2d(&tmKV, kv, 128, static_cast<uint64_t>(kv_rows), 256, 64, kTcBK);
  if (rc) return rc;
  static int configured = 0;
  if (configured < smem) {
    OMLM_CUDA(cudaFuncSetAttribute(attn_fwd_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = smem;
  }
  OMLM_KLAUNCH((attn_fwd_tc_kernel<true>), static_cast<unsigned>(n_work), kTcThreads, smem, reinterpret_cast<cudaStream_t>(stream),
      tmQ, tmKV, table, table_ld, nullptr, reinterpret_cast<__nv_bfloat16*>(out), lse2, 0, heads, scale, 0, fwd_win_ld(heads),
      work, seq_start, seq_len, q_off, kv_start);
  OMLM_LAUNCH_CHECK();
  return 0;
}

extern "C" int omlm_attn_fwd_tc_varlen(const void* qn, const void* kvn, const float* table, int table_ld, const int* work,
                                       int n_work, const int* seq_start, const int* seq_len, int M, int max_len, void* out,
                                       float* lse2, int heads, float scale, void* stream) {
  return attn_fwd_tc_varlen_launch(qn, kvn, M, table, table_ld, work, n_work, seq_start, seq_len, nullptr, nullptr, M, max_len,
                                   out, lse2, heads, scale, stream);
}

extern "C" int omlm_attn_fwd_tc_chunk(const void* qn, const void* kv, long kv_rows, const float* table, int table_ld,
                                      const int* work, int n_work, const int* seq_start, const int* seq_len, const int* q_off,
                                      const int* kv_start, int M, int max_end, void* out, float* lse2, int heads, float scale,
                                      void* stream) {
  OMLM_CHECK_ARG(q_off != nullptr && kv_start != nullptr, "attn_fwd_tc_chunk: q_off and kv_start are required");
  return attn_fwd_tc_varlen_launch(qn, kv, kv_rows, table, table_ld, work, n_work, seq_start, seq_len, q_off, kv_start, M,
                                   max_end, out, lse2, heads, scale, stream);
}
#endif
