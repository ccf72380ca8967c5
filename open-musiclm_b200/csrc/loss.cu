// Cross-entropy over the per-quantizer logit heads, forward + gradient in one pass.
// Replaces F.cross_entropy in TokenConditionedTransformerWrapper.forward (open_musiclm.py:401) and
// its autograd backward.  One warp per row; the row (C <= 1280 fp32 logits) is cached in registers.
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
__global__ void __launch_bounds__(256)
ce_fwd_bwd_kernel(const float* __restrict__ logits, long ld, const int* __restrict__ labels, int label_stride,
                  int rows_per_batch, long batch_stride,
                  int rows, int C, int ignore_index, float grad_scale, float loss_scale, __nv_bfloat16* __restrict__ dlogits,
                  long ldd, int Cp, float* __restrict__ loss_acc, float2* __restrict__ part) {
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
    const bool ignored = (label == ignore_index);
    if (!ignored && lane == 0) {
      my_loss = (mx + logf(se)) - lr[label];
      my_cnt = 1.f;
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
  OMLM_CHECK_ARG(rows > 0 && C > 0 && C <= 32 * kCeMaxPerLane && Cp <= 32 * kCeMaxPerLane, "cross_entropy: unsupported C=%d", C);
  if (rows_per_batch <= 0) { rows_per_batch = rows; batch_stride = 0; }      // one flat label vector
  const int blocks = (rows + 7) / 8;
  if (part != nullptr) OMLM_CHECK_ARG(part_bytes >= blocks * 8L, "cross_entropy_det: partials need %ld bytes", blocks * 8L);
  OMLM_KLAUNCH((ce_fwd_bwd_kernel), blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream),
      logits, ld, labels, label_stride, rows_per_batch, batch_stride, rows, C, ignore_index, grad_scale, loss_scale,
      reinterpret_cast<__nv_bfloat16*>(dlogits_bf16), ldd, Cp, loss_acc, reinterpret_cast<float2*>(part));
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
