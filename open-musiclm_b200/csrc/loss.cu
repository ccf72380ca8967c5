// Cross-entropy over the per-quantizer logit heads, forward + gradient in one pass.
// Replaces F.cross_entropy in TokenConditionedTransformerWrapper.forward (open_musiclm.py:401) and
// its autograd backward.  One warp per row, eight rows per CTA.  Rows of C <= 1280 fp32 logits (and Cp <= 1280) are
// cached in registers (ce_fwd_bwd_kernel); longer rows are streamed twice (ce_stream_kernel): once for the row's
// online (max, sum of exp), once for the gradient.
#include "common.cuh"
#include "../../include/omlm_b200.h"

namespace omlm {

constexpr int kCeMaxPerLane = 40;

// loss_acc[0] += loss_scale * sum_rows (lse - logit[label]);  loss_acc[1] += number of non-ignored rows.
// dlogits[row, c] = (softmax(row)[c] - [c == label]) * grad_scale  (bf16, zero for c >= C and ignored rows)
// The label of row r is labels[(r / rows_per_batch) * batch_stride + (r % rows_per_batch) * label_stride]: the rows of a
// logit-head group are ordered (sequence b, step t) while its labels sit at positions qi + q t of sequence b's label
// row -- a strided view, read in place.
// DET (part != nullptr): instead of the two atomics, the block writes (loss_scale * its loss sum, its row count) to
// part[blockIdx.x]; omlm_colsum adds the blocks' pairs to loss_acc in block order.
template <bool kRowOut>
__global__ void __launch_bounds__(256)
ce_fwd_bwd_kernel(const float* __restrict__ logits, long ld, const int* __restrict__ labels, int label_stride,
                  int rows_per_batch, long batch_stride,
                  int rows, int C, int ignore_index, float grad_scale, float loss_scale, __nv_bfloat16* __restrict__ dlogits,
                  long ldd, int Cp, float* __restrict__ loss_acc, float2* __restrict__ part,
                  float* __restrict__ row_out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + warp;
  float my_loss = 0.f, my_cnt = 0.f;
  if (row < rows) {
    const float* lr = logits + static_cast<long>(row) * ld;
    const int rb = row / rows_per_batch;
    const int label = labels[rb * batch_stride + static_cast<long>(row - rb * rows_per_batch) * label_stride];
    float v[kCeMaxPerLane];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < kCeMaxPerLane; ++i) {
      const int c = i * 32 + lane;
      v[i] = (c < C) ? lr[c] : -INFINITY;
      mx = fmaxf(mx, v[i]);
    }
    mx = warp_max(mx);
    float se = 0.f;
#pragma unroll
    for (int i = 0; i < kCeMaxPerLane; ++i) {
      v[i] = __expf(v[i] - mx);  // exp(-inf) = 0 for the padding
      se += v[i];
    }
    se = warp_sum(se);
    const bool ignored = (label == ignore_index) || (kRowOut && (label < 0 || label >= C));
    if (!ignored && lane == 0) {
      my_loss = (mx + logf(se)) - lr[label];
      my_cnt = 1.f;
    }
    if constexpr (kRowOut) {
      if (lane == 0) row_out[row] = ignored ? 0.f : -my_loss;
    }
    if (dlogits != nullptr) {
      const float inv = ignored ? 0.f : grad_scale / se;
      __nv_bfloat16* dr = dlogits + static_cast<long>(row) * ldd;
#pragma unroll
      for (int i = 0; i < kCeMaxPerLane; ++i) {
        const int c = i * 32 + lane;
        if (c < Cp) {
          float g = (c < C) ? v[i] * inv : 0.f;
          if (c == label && !ignored) g -= grad_scale;
          dr[c] = __float2bfloat16_rn(g);
        }
      }
    }
  }
  if constexpr (kRowOut) return;                       // the same on every thread: no loss sum, no barrier
  __shared__ float sl[8], sc[8];
  if (lane == 0) { sl[warp] = my_loss; sc[warp] = my_cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a += sl[i]; b += sc[i]; }
    if (part != nullptr) part[blockIdx.x] = make_float2(a * loss_scale, b);
    else if (b > 0.f) { atomicAdd(&loss_acc[0], a * loss_scale); atomicAdd(&loss_acc[1], b); }
  }
}

// Online softmax statistics: fold four logits into the lane's running (max m, sum s of exp(x - m)).
__device__ __forceinline__ void ce_online4(float4 v, float& m, float& s) {
  const float nm = fmaxf(m, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
  s = s * __expf(m - nm) + (__expf(v.x - nm) + __expf(v.y - nm)) + (__expf(v.z - nm) + __expf(v.w - nm));
  m = nm;
}

// Eight gradient columns c0 .. c0+7 as bf16: (exp(x - mx) * inv  -  [c == label] * gs), zero for c >= C.
__device__ __forceinline__ uint4 ce_grad8(float4 a, float4 b, int c0, int C, float mx, float inv, int label, float gs) {
  const float x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  float g[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    g[k] = (c0 + k < C) ? __expf(x[k] - mx) * inv : 0.f;
    if (c0 + k == label) g[k] -= gs;
  }
  return make_uint4(pack_bf16x2(g[0], g[1]), pack_bf16x2(g[2], g[3]), pack_bf16x2(g[4], g[5]), pack_bf16x2(g[6], g[7]));
}

// ce_fwd_bwd_kernel's contract for any C.  Host-checked layout: logits 16-byte aligned with ld % 4 == 0 and ld >= C;
// dlogits 16-byte aligned with ldd % 8 == 0, Cp % 8 == 0, C <= Cp <= ldd.
// Pass 1 reads the row as float4 (lane l takes chunks l, l + 32, ...: four loads in flight per lane) into a per-lane
// online (max, sum of exp); the lanes are combined by the warp_max / warp_sum butterflies, so a row's logsumexp is the
// same on every run.  Pass 2 reads the row again (mostly from L2: the warp has just read it) and writes eight bf16
// gradients per 16-byte store.  Columns beyond C are never read.  Ignored rows are written as zeros
// without reading the row again.
template <bool kRowOut>
__global__ void __launch_bounds__(256)
ce_stream_kernel(const float* __restrict__ logits, long ld, const int* __restrict__ labels, int label_stride,
                 int rows_per_batch, long batch_stride,
                 int rows, int C, int ignore_index, float grad_scale, float loss_scale, __nv_bfloat16* __restrict__ dlogits,
                 long ldd, int Cp, float* __restrict__ loss_acc, float2* __restrict__ part,
                  float* __restrict__ row_out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + warp;
  float my_loss = 0.f, my_cnt = 0.f;
  if (row < rows) {
    const float* lr = logits + static_cast<long>(row) * ld;
    const float4* l4 = reinterpret_cast<const float4*>(lr);
    const int rb = row / rows_per_batch;
    const int label = labels[rb * batch_stride + static_cast<long>(row - rb * rows_per_batch) * label_stride];
    const bool ignored = (label == ignore_index) || (kRowOut && (label < 0 || label >= C));
    // ---- pass 1: online max / sum of exp
    const int n4 = C >> 2;
    float m = -INFINITY, s = 0.f;
    int j = lane;
    for (; j + 96 < n4; j += 128) {
      float4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) v[u] = __ldg(l4 + j + 32 * u);
#pragma unroll
      for (int u = 0; u < 4; ++u) ce_online4(v[u], m, s);
    }
    for (; j < n4; j += 32) ce_online4(__ldg(l4 + j), m, s);
    {  // the last C % 4 columns, one per lane
      const int c = 4 * n4 + lane;
      const float x = (c < C) ? __ldg(lr + c) : -INFINITY;
      const float nm = fmaxf(m, x);
      if (nm != -INFINITY) { s = s * __expf(m - nm) + __expf(x - nm); m = nm; }
    }
    const float mx = warp_max(m);
    const float se = warp_sum(m == -INFINITY ? 0.f : s * __expf(m - mx));
    if (!ignored && lane == 0) {
      my_loss = (mx + logf(se)) - lr[label];
      my_cnt = 1.f;
    }
    if constexpr (kRowOut) {
      if (lane == 0) row_out[row] = ignored ? 0.f : -my_loss;
    }
    // ---- pass 2: dlogits, eight columns per 16-byte store
    if (dlogits != nullptr) {
      uint4* d8 = reinterpret_cast<uint4*>(dlogits + static_cast<long>(row) * ldd);
      const int n8 = Cp >> 3;
      if (ignored) {
        for (int k = lane; k < n8; k += 32) d8[k] = make_uint4(0u, 0u, 0u, 0u);
      } else {
        const float inv = grad_scale / se;
        const int full8 = C >> 3;                  // chunks whose eight columns are all < C
        int k = lane;
        for (; k + 32 < full8; k += 64) {
          const float4 a0 = __ldg(l4 + 2 * k), b0 = __ldg(l4 + 2 * k + 1);
          const float4 a1 = __ldg(l4 + 2 * (k + 32)), b1 = __ldg(l4 + 2 * (k + 32) + 1);
          d8[k] = ce_grad8(a0, b0, 8 * k, C, mx, inv, label, grad_scale);
          d8[k + 32] = ce_grad8(a1, b1, 8 * (k + 32), C, mx, inv, label, grad_scale);
        }
        for (; k < full8; k += 32) d8[k] = ce_grad8(__ldg(l4 + 2 * k), __ldg(l4 + 2 * k + 1), 8 * k, C, mx, inv, label, grad_scale);
        for (; k < n8; k += 32) {                  // the chunk holding column C - 1 (if partial) and the zero padding
          float x[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) x[e] = (8 * k + e < C) ? __ldg(lr + 8 * k + e) : 0.f;
          d8[k] = ce_grad8(make_float4(x[0], x[1], x[2], x[3]), make_float4(x[4], x[5], x[6], x[7]), 8 * k, C, mx, inv,
                           label, grad_scale);
        }
      }
    }
  }
  if constexpr (kRowOut) return;                       // the same on every thread: no loss sum, no barrier
  __shared__ float sl[8], sc[8];
  if (lane == 0) { sl[warp] = my_loss; sc[warp] = my_cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a += sl[i]; b += sc[i]; }
    if (part != nullptr) part[blockIdx.x] = make_float2(a * loss_scale, b);
    else if (b > 0.f) { atomicAdd(&loss_acc[0], a * loss_scale); atomicAdd(&loss_acc[1], b); }
  }
}

}  // namespace omlm

static int cross_entropy_impl(const float* logits, long ld, const int* labels, int label_stride, int rows_per_batch,
                              long batch_stride, int rows, int C, int ignore_index, float grad_scale, float loss_scale,
                              void* dlogits_bf16, long ldd, int Cp, float* loss_acc, float* part, long part_bytes, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(rows > 0 && C > 0, "cross_entropy: unsupported C=%d", C);
  if (rows_per_batch <= 0) { rows_per_batch = rows; batch_stride = 0; }      // one flat label vector
  const int blocks = (rows + 7) / 8;
  if (part != nullptr) OMLM_CHECK_ARG(part_bytes >= blocks * 8L, "cross_entropy_det: partials need %ld bytes", blocks * 8L);
  // both kernels write every column below Cp of a gradient row: a row narrower than C would lose part of its gradient
  if (dlogits_bf16 != nullptr)
    OMLM_CHECK_ARG(Cp >= C && ldd >= Cp, "cross_entropy: dlogits needs C <= Cp <= ldd (C=%d, Cp=%d, ldd=%ld)", C, Cp, ldd);
  if (C > 32 * kCeMaxPerLane || Cp > 32 * kCeMaxPerLane) {
    // rows too long for registers: the streaming kernel (128-bit loads and 16-byte stores)
    OMLM_CHECK_ARG(reinterpret_cast<uintptr_t>(logits) % 16 == 0 && ld % 4 == 0 && ld >= C,
                   "cross_entropy: C=%d needs 16-byte aligned logits with ld %% 4 == 0 and ld >= C (ld=%ld)", C, ld);
    if (dlogits_bf16 != nullptr)
      OMLM_CHECK_ARG(reinterpret_cast<uintptr_t>(dlogits_bf16) % 16 == 0 && ldd % 8 == 0 && Cp % 8 == 0 && Cp >= C && ldd >= Cp,
                     "cross_entropy: C=%d needs 16-byte aligned dlogits with ldd %% 8 == 0, Cp %% 8 == 0 and C <= Cp <= ldd "
                     "(Cp=%d, ldd=%ld)", C, Cp, ldd);
    OMLM_KLAUNCH((ce_stream_kernel<false>), blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream),
        logits, ld, labels, label_stride, rows_per_batch, batch_stride, rows, C, ignore_index, grad_scale, loss_scale,
        reinterpret_cast<__nv_bfloat16*>(dlogits_bf16), ldd, Cp, loss_acc, reinterpret_cast<float2*>(part), nullptr);
    OMLM_LAUNCH_CHECK();
    if (part != nullptr) return omlm_colsum(part, 2, 1, loss_acc, blocks, 2, 1, stream);
    return 0;
  }
  OMLM_KLAUNCH((ce_fwd_bwd_kernel<false>), blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream),
      logits, ld, labels, label_stride, rows_per_batch, batch_stride, rows, C, ignore_index, grad_scale, loss_scale,
      reinterpret_cast<__nv_bfloat16*>(dlogits_bf16), ldd, Cp, loss_acc, reinterpret_cast<float2*>(part), nullptr);
  OMLM_LAUNCH_CHECK();
  if (part != nullptr) return omlm_colsum(part, 2, 1, loss_acc, blocks, 2, 1, stream);
  return 0;
}

extern "C" int omlm_cross_entropy(const float* logits, long ld, const int* labels, int label_stride, int rows_per_batch,
                                  long batch_stride, int rows, int C, int ignore_index, float grad_scale, float loss_scale,
                                  void* dlogits_bf16, long ldd, int Cp, float* loss_acc, void* stream) {
  return cross_entropy_impl(logits, ld, labels, label_stride, rows_per_batch, batch_stride, rows, C, ignore_index, grad_scale,
                            loss_scale, dlogits_bf16, ldd, Cp, loss_acc, nullptr, 0, stream);
}

extern "C" int omlm_cross_entropy_det(const float* logits, long ld, const int* labels, int label_stride, int rows_per_batch,
                                      long batch_stride, int rows, int C, int ignore_index, float grad_scale, float loss_scale,
                                      void* dlogits_bf16, long ldd, int Cp, float* loss_acc, float* part_ws, long part_ws_bytes,
                                      void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(part_ws != nullptr, "cross_entropy_det: no partials buffer");
  return cross_entropy_impl(logits, ld, labels, label_stride, rows_per_batch, batch_stride, rows, C, ignore_index, grad_scale,
                            loss_scale, dlogits_bf16, ldd, Cp, loss_acc, part_ws, part_ws_bytes, stream);
}

// The per-row value of the kernels above, written out instead of summed: out[r] = log softmax(row r)[label_r] =
// l[label] - (mx + log se), bit for bit the negated row loss of omlm_cross_entropy.  The same kernel bodies (kRowOut);
// no gradient, no loss sum.  A label outside [0, C) (ignore_index included) gives 0.
extern "C" int omlm_token_logprob(const float* logits, long ld, const int* labels, int label_stride, int rows_per_batch,
                                  long batch_stride, int rows, int C, float* out, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(rows > 0 && C > 0 && out != nullptr, "token_logprob: bad arguments (rows=%d, C=%d)", rows, C);
  if (rows_per_batch <= 0) { rows_per_batch = rows; batch_stride = 0; }
  const int blocks = (rows + 7) / 8;
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (C > 32 * kCeMaxPerLane) {
    OMLM_CHECK_ARG(reinterpret_cast<uintptr_t>(logits) % 16 == 0 && ld % 4 == 0 && ld >= C,
                   "token_logprob: C=%d needs 16-byte aligned logits with ld %% 4 == 0 and ld >= C (ld=%ld)", C, ld);
    OMLM_KLAUNCH((ce_stream_kernel<true>), blocks, 256, 0, st, logits, ld, labels, label_stride, rows_per_batch, batch_stride,
                 rows, C, -100, 0.f, 0.f, nullptr, 0L, 0, nullptr, nullptr, out);
  } else {
    OMLM_KLAUNCH((ce_fwd_bwd_kernel<true>), blocks, 256, 0, st, logits, ld, labels, label_stride, rows_per_batch, batch_stride,
                 rows, C, -100, 0.f, 0.f, nullptr, 0L, 0, nullptr, nullptr, out);
  }
  OMLM_LAUNCH_CHECK();
  return 0;
}
