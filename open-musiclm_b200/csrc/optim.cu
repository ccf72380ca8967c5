// Optimiser step on the flat fp32 parameter/gradient arena + (un)packing between the canonical
// (state_dict) parameter layout and the padded bf16 compute layout.
//
// Replaces  clip_grad_norm_(0.5) + AdamW.step (trainer.py:443-449, optimizer.py:3-34: weight decay only
// on ndim >= 2 parameters, betas (0.9, 0.99), eps 1e-8).  The arena is ordered [decayed | non-decayed],
// so the decay rule is a single index compare.  Clip coefficient and hyper-parameters are read from
// device memory: the step never synchronises with the host.
#include "common.cuh"
#include <type_traits>
#include "../../include/omlm_b200.h"

namespace omlm {

// acc[0] (double) += sum (g * prescale)^2.  part != nullptr (deterministic): the block's sum goes to part[blockIdx.x]
// instead, and sumsq_finish_kernel adds the blocks' sums to acc in block order.
__global__ void __launch_bounds__(512)
sumsq_kernel(const float* __restrict__ g, long n, float prescale, double* __restrict__ acc, double* __restrict__ part) {
  float s = 0.f;
  const long n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n4; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const float4 v = g4[i];
    s += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) { const float v = g[(n4 << 2) + threadIdx.x]; s += v * v; }
  __shared__ float red[16];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < 16 ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) {
      if (part != nullptr) part[blockIdx.x] = static_cast<double>(v) * prescale * prescale;
      else atomicAdd(acc, static_cast<double>(v) * prescale * prescale);
    }
  }
}

__global__ void __launch_bounds__(32) sumsq_finish_kernel(const double* __restrict__ part, int n, double* __restrict__ acc) {
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += 32) s += part[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (threadIdx.x == 0) acc[0] += s;
}

// hyper: [0] lr  [1] beta1  [2] beta2  [3] eps  [4] weight_decay  [5] 1-beta1^t  [6] 1-beta2^t
//        [7] max_grad_norm (<=0: no clipping)  [8] grad prescale (1/world for DDP-mean)
__global__ void __launch_bounds__(512)
adamw_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
             long n, long n_decay, const float* __restrict__ hyper, const double* __restrict__ sumsq) {
  const float lr = hyper[0], b1 = hyper[1], b2 = hyper[2], eps = hyper[3], wd = hyper[4];
  const float bc1 = hyper[5], bc2 = hyper[6], max_norm = hyper[7], prescale = hyper[8];
  float coef = prescale;
  if (max_norm > 0.f) {
    const float norm = static_cast<float>(sqrt(*sumsq));
    coef *= fminf(1.f, max_norm / (norm + 1e-6f));  // torch.nn.utils.clip_grad_norm_
  }
  const float step_size = lr / bc1;
  const float inv_sqrt_bc2 = rsqrtf(bc2);
  const float decay = 1.f - lr * wd;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const float gi = g[i] * coef;
    float pi = p[i];
    if (i < n_decay) pi *= decay;
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi; v[i] = vi;
    const float denom = sqrtf(vi) * inv_sqrt_bc2 + eps;
    p[i] = pi - step_size * (mi / denom);
  }
}

// one fp16 with the vector path's conversion (cvt.rn.satfinite): finite overflow saturates to +-65504, NaN stays NaN
__device__ __forceinline__ __half f16_satfinite(float x) { return __ushort_as_half(static_cast<unsigned short>(pack_f16x2(x, 0.f) & 0xffffu)); }

// dst[r, c] = src[map(r), c] for c < cols_valid and live r, else 0.
// map: split_dst > 0: half = r / split_dst, rr = r % split_dst, live iff rr < split_src, src row = half*split_src + rr
//      split_dst < 0: interleaved GEGLU order, groups of 128 channels stored as [128 value rows | 128 gate rows]:
//                     w = r % 256, c = (r / 256) * 128 + w % 128, src row = (w / 128) * split_src + c, live iff c < split_src
//      split_dst = 0: live iff r < rows_valid.
template <typename OutT>
__device__ __forceinline__ void store_quad(OutT* __restrict__ dst, long dst_ld, int r, int c, int cols_p, const float (&v)[4]) {
  const bool vec_dst = ((dst_ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) && ((cols_p & 3) == 0);
  OutT* d = dst + r * dst_ld + c;
  if (vec_dst) {
    if constexpr (sizeof(OutT) == 2) {
      constexpr bool kHalf = std::is_same<OutT, __half>::value;
      uint2 o; o.x = pack16x2<kHalf>(v[0], v[1]); o.y = pack16x2<kHalf>(v[2], v[3]);
      *reinterpret_cast<uint2*>(d) = o;
    } else {
      *reinterpret_cast<float4*>(d) = make_float4(v[0], v[1], v[2], v[3]);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (c + j < cols_p) {
        if constexpr (std::is_same<OutT, __half>::value) d[j] = f16_satfinite(v[j]);
        else if constexpr (sizeof(OutT) == 2) d[j] = __float2bfloat16_rn(v[j]);
        else d[j] = v[j];
      }
    }
  }
}
__device__ __forceinline__ void store_quad_fmt(void* dst, int fmt, long dst_ld, int r, int c, int cols_p, const float (&v)[4]) {
  if (fmt == kFmtF32) store_quad<float>(reinterpret_cast<float*>(dst), dst_ld, r, c, cols_p, v);
  else if (fmt == kFmtF16) store_quad<__half>(reinterpret_cast<__half*>(dst), dst_ld, r, c, cols_p, v);
  else store_quad<__nv_bfloat16>(reinterpret_cast<__nv_bfloat16*>(dst), dst_ld, r, c, cols_p, v);
}

// loads the 4 source values of quad i (zeros where the destination is padding); returns its destination (row, column)
__device__ __forceinline__ void load_quad(long i, const float* __restrict__ src, long src_ld, int rows_valid, int cols_valid,
                                          int cols_p, int split_dst, int split_src, int& r, int& c, float (&v)[4]) {
  const int c4n = (cols_p + 3) >> 2;
  const bool vec_src = ((src_ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
  r = static_cast<int>(i / c4n); c = static_cast<int>(i - static_cast<long>(r) * c4n) << 2;
  int sr = r; bool live = r < rows_valid;
  if (split_dst > 0) { const int half = r / split_dst, rr = r - half * split_dst; sr = half * split_src + rr; live = rr < split_src && sr < rows_valid; }
  else if (split_dst < 0) { const int w = r & 255, ch = ((r >> 8) << 7) + (w & 127); sr = (w >> 7) * split_src + ch; live = ch < split_src && sr < rows_valid; }
  v[0] = v[1] = v[2] = v[3] = 0.f;
  if (live) {
    if (vec_src && c + 3 < cols_valid) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(src + sr * src_ld + c));
      v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) if (c + j < cols_valid) v[j] = src[sr * src_ld + c + j];
    }
  }
}

template <typename OutT>
__device__ __forceinline__ void pack_quad(long i, const float* __restrict__ src, long src_ld, int rows_valid, int cols_valid,
                                          OutT* __restrict__ dst, long dst_ld, int cols_p, int split_dst, int split_src) {
  // one call per 4 consecutive columns of a destination row
  const int c4n = (cols_p + 3) >> 2;
  const bool vec_src = ((src_ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(src) & 15) == 0);
  const bool vec_dst = ((dst_ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) && ((cols_p & 3) == 0);
  const int r = static_cast<int>(i / c4n), c = static_cast<int>(i - static_cast<long>(r) * c4n) << 2;
  int sr = r; bool live = r < rows_valid;
  if (split_dst > 0) { const int half = r / split_dst, rr = r - half * split_dst; sr = half * split_src + rr; live = rr < split_src && sr < rows_valid; }
  else if (split_dst < 0) { const int w = r & 255, ch = ((r >> 8) << 7) + (w & 127); sr = (w >> 7) * split_src + ch; live = ch < split_src && sr < rows_valid; }
  float v[4] = {0.f, 0.f, 0.f, 0.f};
  if (live) {
    if (vec_src && c + 3 < cols_valid) {
      const float4 t = *reinterpret_cast<const float4*>(src + sr * src_ld + c);
      v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) if (c + j < cols_valid) v[j] = src[sr * src_ld + c + j];
    }
  }
  OutT* d = dst + r * dst_ld + c;
  if (vec_dst) {
    if constexpr (sizeof(OutT) == 2) {
      constexpr bool kHalf = std::is_same<OutT, __half>::value;
      uint2 o; o.x = pack16x2<kHalf>(v[0], v[1]); o.y = pack16x2<kHalf>(v[2], v[3]);
      *reinterpret_cast<uint2*>(d) = o;
    } else {
      *reinterpret_cast<float4*>(d) = make_float4(v[0], v[1], v[2], v[3]);
    }
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (c + j < cols_p) {
        if constexpr (std::is_same<OutT, __half>::value) d[j] = f16_satfinite(v[j]);
        else if constexpr (sizeof(OutT) == 2) d[j] = __float2bfloat16_rn(v[j]);
        else d[j] = v[j];
      }
    }
  }
}

template <typename OutT>
__global__ void pack_kernel(const float* __restrict__ src, long src_ld, int rows_valid, int cols_valid,
                            OutT* __restrict__ dst, long dst_ld, int rows_p, int cols_p, int split_dst, int split_src) {
  const long total = static_cast<long>(rows_p) * ((cols_p + 3) >> 2);
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x)
    pack_quad<OutT>(i, src, src_ld, rows_valid, cols_valid, dst, dst_ld, cols_p, split_dst, split_src);
}

// All repacks of one optimiser step in ONE launch: the job table lives in device memory, work is cut into units of
// 256 quads and blocks stride over the concatenated unit list (45 small launches -> 1 bandwidth-bound pass).
constexpr int kPackMaxJobs = 512;
constexpr int kPackUnit = 1024;      // quads per unit: 4 per thread, 256 apart (coalesced), all four loads in flight together
__global__ void __launch_bounds__(256) pack_multi_kernel(const omlm_pack_job* __restrict__ jobs, int njobs, long total_units) {
  __shared__ long starts[kPackMaxJobs + 1];
  __shared__ omlm_pack_job s_job;
  for (int j = threadIdx.x; j < njobs; j += blockDim.x) starts[j] = jobs[j].unit_start;
  if (threadIdx.x == 0) starts[njobs] = total_units;
  __syncthreads();
  int cur = -1;
  for (long u = blockIdx.x; u < total_units; u += gridDim.x) {
    int lo = 0, hi = njobs - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (starts[mid] <= u) lo = mid; else hi = mid - 1; }
    if (lo != cur) {                  // (uniform across the block) fetch the job record once per job, not per thread
      __syncthreads();
      if (threadIdx.x == 0) s_job = jobs[lo];
      __syncthreads();
      cur = lo;
    }
    const omlm_pack_job& jb = s_job;
    const long total = static_cast<long>(jb.rows_p) * ((jb.cols_p + 3) >> 2);
    const long i0 = (u - jb.unit_start) * kPackUnit + threadIdx.x;
    float v[4][4];
    int r[4], c[4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (i0 + k * 256 < total) load_quad(i0 + k * 256, jb.src, jb.src_ld, jb.rows_valid, jb.cols_valid, jb.cols_p, jb.split_dst, jb.split_src, r[k], c[k], v[k]);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (i0 + k * 256 < total) {
        store_quad_fmt(jb.dst, jb.dst_fmt, jb.dst_ld, r[k], c[k], jb.cols_p, v[k]);
        if (jb.dst2 != nullptr) store_quad_fmt(jb.dst2, jb.dst2_fmt, jb.dst_ld, r[k], c[k], jb.cols_p, v[k]);
      }
    }
  }
}

// canonical[map(r), c] += packed[r, c]  (inverse of pack for fp32 gradients)
__global__ void unpack_add_kernel(const float* __restrict__ packed, long p_ld, int rows_p, int cols_p,
                                  float* __restrict__ dst, long dst_ld, int rows_valid, int cols_valid,
                                  int split_dst, int split_src) {
  const long total = static_cast<long>(rows_p) * cols_p;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / cols_p), c = static_cast<int>(i - static_cast<long>(r) * cols_p);
    int sr = r; bool live = r < rows_valid;
    if (split_dst > 0) { const int half = r / split_dst, rr = r - half * split_dst; live = rr < split_src; sr = half * split_src + rr; live = live && sr < rows_valid; }
    else if (split_dst < 0) { const int w = r & 255, c = ((r >> 8) << 7) + (w & 127); sr = (w >> 7) * split_src + c; live = c < split_src && sr < rows_valid; }
    if (live && c < cols_valid) dst[sr * dst_ld + c] += packed[r * p_ld + c];
  }
}

}  // namespace omlm

extern "C" {

int omlm_grad_sumsq(const float* g, long n, float prescale, double* acc, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(n > 0, "grad_sumsq: empty");
  OMLM_CHECK_ARG((reinterpret_cast<uintptr_t>(g) & 15) == 0, "grad_sumsq: arena must be 16B aligned");
  const int blocks = static_cast<int>(std::min<long>((n / 4 + 511) / 512 + 1, static_cast<long>(num_sms()) * 4));
  OMLM_KLAUNCH((sumsq_kernel), blocks, 512, 0, reinterpret_cast<cudaStream_t>(stream), g, n, prescale, acc, nullptr);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_grad_sumsq_det(const float* g, long n, float prescale, double* acc, double* part_ws, long part_ws_bytes, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(n > 0, "grad_sumsq_det: empty");
  OMLM_CHECK_ARG((reinterpret_cast<uintptr_t>(g) & 15) == 0, "grad_sumsq_det: arena must be 16B aligned");
  const int blocks = static_cast<int>(std::min<long>((n / 4 + 511) / 512 + 1, static_cast<long>(num_sms()) * 4));
  OMLM_CHECK_ARG(part_ws != nullptr && part_ws_bytes >= blocks * 8L, "grad_sumsq_det: partials need %ld bytes", blocks * 8L);
  auto st = reinterpret_cast<cudaStream_t>(stream);
  OMLM_KLAUNCH((sumsq_kernel), blocks, 512, 0, st, g, n, prescale, acc, part_ws);
  OMLM_LAUNCH_CHECK();
  OMLM_KLAUNCH((sumsq_finish_kernel), 1, 32, 0, st, static_cast<const double*>(part_ws), blocks, acc);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_adamw_step(float* p, const float* g, float* m, float* v, long n, long n_decay, const float* hyper,
                    const double* sumsq, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(n > 0 && n_decay >= 0 && n_decay <= n, "adamw_step: bad sizes");
  const int blocks = static_cast<int>(std::min<long>((n + 511) / 512, static_cast<long>(num_sms()) * 8));
  OMLM_KLAUNCH((adamw_kernel), blocks, 512, 0, reinterpret_cast<cudaStream_t>(stream), p, g, m, v, n, n_decay, hyper, sumsq);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_pack(const float* src, long src_ld, int rows_valid, int cols_valid, void* dst, int dst_fmt, long dst_ld,
              int rows_p, int cols_p, int split_dst, int split_src, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(rows_p > 0 && cols_p > 0, "pack: empty");
  const long total = static_cast<long>(rows_p) * ((cols_p + 3) / 4);
  const int blocks = static_cast<int>(std::min<long>((total + 255) / 256, static_cast<long>(num_sms()) * 16));
  auto st = reinterpret_cast<cudaStream_t>(stream);
  OMLM_CHECK_ARG(dst_fmt == kFmtBF16 || dst_fmt == kFmtF32 || dst_fmt == kFmtF16, "pack: dst_fmt must be 0 (bf16), 1 (fp32) or 2 (fp16)");
  if (dst_fmt == kFmtF32)
    OMLM_KLAUNCH((pack_kernel<float>), blocks, 256, 0, st, src, src_ld, rows_valid, cols_valid, reinterpret_cast<float*>(dst), dst_ld, rows_p, cols_p, split_dst, split_src);
  else if (dst_fmt == kFmtF16)
    OMLM_KLAUNCH((pack_kernel<__half>), blocks, 256, 0, st, src, src_ld, rows_valid, cols_valid, reinterpret_cast<__half*>(dst), dst_ld, rows_p, cols_p, split_dst, split_src);
  else
    OMLM_KLAUNCH((pack_kernel<__nv_bfloat16>), blocks, 256, 0, st, src, src_ld, rows_valid, cols_valid, reinterpret_cast<__nv_bfloat16*>(dst), dst_ld, rows_p, cols_p, split_dst, split_src);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_pack_multi(const omlm_pack_job* jobs_device, int njobs, long total_units, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(jobs_device != nullptr && njobs > 0 && njobs <= kPackMaxJobs && total_units > 0, "pack_multi: need 1..%d jobs per table (got %d)", kPackMaxJobs, njobs);
  const int blocks = static_cast<int>(std::min<long>(total_units, static_cast<long>(num_sms()) * 16));
  OMLM_KLAUNCH((pack_multi_kernel), blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream), jobs_device, njobs, total_units);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_unpack_add(const float* packed, long p_ld, int rows_p, int cols_p, float* dst, long dst_ld, int rows_valid,
                    int cols_valid, int split_dst, int split_src, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(rows_p > 0 && cols_p > 0, "unpack_add: empty");
  const long total = static_cast<long>(rows_p) * cols_p;
  const int blocks = static_cast<int>(std::min<long>((total + 255) / 256, static_cast<long>(num_sms()) * 8));
  OMLM_KLAUNCH((unpack_add_kernel), blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream), packed, p_ld, rows_p, cols_p, dst, dst_ld, rows_valid, cols_valid, split_dst, split_src);
  OMLM_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
