// fp32 SIMT kernels for the relative-position-bias MLP (RelativePositionBias, transformer.py:36-67).
// The MLP is evaluated on the N causal distances 0..N-1 only (negative distances are overwritten by
// the causal mask, transformer.py:315-322) and yields the Toeplitz table[h, delta] that the
// attention kernels index by i-j.  fp32 throughout: table values reach |b| ~ 100 and dominate the
// logits (SURVEY B.1), so bf16 tensor-core inputs are not acceptable here; the work is ~1 GFLOP.
#include "common.cuh"
#include <algorithm>
#include "../../include/omlm_b200.h"

namespace omlm {

// C[m,n] (+)= sum_k A[m*sa_m + k*sa_k] * B[k*sb_k + n*sb_n] (+ bias[n]);  act: 0 none, 1 SiLU
// (pre-activation optionally saved to Z with C's strides).  64x64 tile, 256 threads, 4x4 per thread.
__global__ void __launch_bounds__(256)
sgemm_small_kernel(const float* __restrict__ A, long sa_m, long sa_k, const float* __restrict__ B,
                   long sb_k, long sb_n, float* __restrict__ C, long sc_m, long sc_n,
                   float* __restrict__ Z, const float* __restrict__ bias, int M, int N, int K, int act,
                   int accumulate) {
  __shared__ float As[16][64 + 4];
  __shared__ float Bs[16][64 + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  // split-K (gridDim.z > 1): this CTA reduces k in [k_lo, k_hi) and adds its partial product into C atomically
  const int k_per = ((K + gridDim.z - 1) / gridDim.z + 15) & ~15;
  const int k_lo = blockIdx.z * k_per, k_hi = min(K, k_lo + k_per);
  for (int k0 = k_lo; k0 < k_hi; k0 += 16) {
    for (int i = threadIdx.x; i < 16 * 64; i += 256) {
      const int kk = i & 15, mm = i >> 4;
      const int m = m0 + mm, k = k0 + kk;
      As[kk][mm] = (m < M && k < k_hi) ? A[m * sa_m + k * sa_k] : 0.f;
      const int n = n0 + mm;
      Bs[kk][mm] = (n < N && k < k_hi) ? B[k * sb_k + n * sb_n] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j];
      const long off = m * sc_m + n * sc_n;
      if (gridDim.z > 1) {   // accumulate-only mode (checked by the launcher)
        if (bias != nullptr && blockIdx.z == 0) v += bias[n];
        atomicAdd(&C[off], v);
        continue;
      }
      if (bias != nullptr) v += bias[n];
      if (Z != nullptr) Z[off] = v;
      if (act == 1) v = v / (1.f + expf(-v));
      if (accumulate) v += C[off];
      C[off] = v;
    }
  }
}

// dZ = dA * silu'(z),  silu'(z) = s + z*s*(1-s), s = sigmoid(z)
__global__ void silu_bwd_kernel(const float* __restrict__ dA, const float* __restrict__ Zp,
                                float* __restrict__ dZ, __nv_bfloat16* __restrict__ dZ_bf16, long n) {
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long>(gridDim.x) * blockDim.x) {
    const float z = Zp[i];
    const float s = 1.f / (1.f + expf(-z));
    const float g = dA[i] * (s + z * s * (1.f - s));
    dZ[i] = g;
    if (dZ_bf16 != nullptr) dZ_bf16[i] = __float2bfloat16_rn(g);
  }
}

// out[n] (+)= sum_m X[m*s_m + n*s_n]
__global__ void colsum_kernel(const float* __restrict__ X, long s_m, long s_n, float* __restrict__ out,
                              int M, int N, int accumulate) {
  const int n = blockIdx.x;
  float s = 0.f;
  for (int m = threadIdx.x; m < M; m += blockDim.x) s += X[m * s_m + n * s_n];
  __shared__ float red[32];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0) out[n] = accumulate ? out[n] + v : v;
  }
}

// bf16x3 split for near-fp32 tensor-core products:  x = hi + lo (both bf16).  With
//   A3 = [a_hi | a_hi | a_lo]  and  W3 = [w_hi | w_lo | w_hi]   (K concatenated),
// A3 . W3^T = a_hi w_hi + a_hi w_lo + a_lo w_hi  ~  a . w  to ~2^-16 relative, accumulated in fp32 by wgmma.
// Each third is Cpad >= C columns wide, columns [C, Cpad) zero: with Cpad a multiple of 8 every third starts on a
// 16-byte boundary, as a TMA view of one third needs, and the zero columns add nothing to the product.
__global__ void split3_kernel(const float* __restrict__ src, long src_ld, __nv_bfloat16* __restrict__ dst, int R,
                              int C, int Cpad, int weight_mode) {
  const long total = static_cast<long>(R) * Cpad;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / Cpad), c = static_cast<int>(i - static_cast<long>(r) * Cpad);
    __nv_bfloat16* d = dst + static_cast<long>(r) * 3 * Cpad + c;
    if (c >= C) {
      d[0] = d[Cpad] = d[2 * Cpad] = __float2bfloat16_rn(0.f);
      continue;
    }
    const float v = src[r * src_ld + c];
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    const __nv_bfloat16 lo = __float2bfloat16_rn(v - __bfloat162float(hi));
    d[0] = hi;
    d[Cpad] = weight_mode ? lo : hi;
    d[2 * Cpad] = weight_mode ? hi : lo;
  }
}

// z += bias (in place);  a = silu(z)
__global__ void bias_silu_kernel(float* __restrict__ z, const float* __restrict__ bias, float* __restrict__ a, int R, int C) {
  const long total = static_cast<long>(R) * C;
  for (long i = blockIdx.x * static_cast<long>(blockDim.x) + threadIdx.x; i < total; i += static_cast<long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % C);
    const float v = z[i] + bias[c];
    z[i] = v;
    a[i] = v / (1.f + expf(-v));
  }
}

__global__ void arange_kernel(float* out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = static_cast<float>(i);
}

}  // namespace omlm

extern "C" {

static int sgemm_small_impl(const float* A, long sa_m, long sa_k, const float* B, long sb_k, long sb_n, float* C,
                            long sc_m, long sc_n, float* Z, const float* bias, int M, int N, int K, int act,
                            int accumulate, bool allow_split, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && N > 0 && K > 0, "sgemm_small: empty problem");
  dim3 grid((N + 63) / 64, (M + 63) / 64);
  // skinny problems with a long reduction (dW of the rel-pos MLP, the h-column table): split K over up to ~256 CTAs
  if (allow_split && accumulate && act == 0 && Z == nullptr && K >= 128) {
    const int ctas = static_cast<int>(grid.x * grid.y);
    if (ctas < 64) grid.z = static_cast<unsigned>(std::max(1, std::min((K + 31) / 32, 256 / ctas)));
  }
  OMLM_KLAUNCH((sgemm_small_kernel), grid, 256, 0, reinterpret_cast<cudaStream_t>(stream), 
      A, sa_m, sa_k, B, sb_k, sb_n, C, sc_m, sc_n, Z, bias, M, N, K, act, accumulate);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_sgemm_small(const float* A, long sa_m, long sa_k, const float* B, long sb_k, long sb_n, float* C,
                     long sc_m, long sc_n, float* Z, const float* bias, int M, int N, int K, int act,
                     int accumulate, void* stream) {
  return sgemm_small_impl(A, sa_m, sa_k, B, sb_k, sb_n, C, sc_m, sc_n, Z, bias, M, N, K, act, accumulate, true, stream);
}

int omlm_sgemm_small_det(const float* A, long sa_m, long sa_k, const float* B, long sb_k, long sb_n, float* C,
                         long sc_m, long sc_n, float* Z, const float* bias, int M, int N, int K, int act,
                         int accumulate, void* stream) {
  return sgemm_small_impl(A, sa_m, sa_k, B, sb_k, sb_n, C, sc_m, sc_n, Z, bias, M, N, K, act, accumulate, false, stream);
}

int omlm_silu_bwd(const float* dA, const float* Z, float* dZ, void* dZ_bf16, long n, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(n > 0, "silu_bwd: empty");
  const int blocks = static_cast<int>(std::min<long>((n + 255) / 256, 4096));
  OMLM_KLAUNCH((silu_bwd_kernel), blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream), dA, Z, dZ, reinterpret_cast<__nv_bfloat16*>(dZ_bf16), n);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_colsum(const float* X, long s_m, long s_n, float* out, int M, int N, int accumulate, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(M > 0 && N > 0, "colsum: empty");
  OMLM_KLAUNCH((colsum_kernel), N, 256, 0, reinterpret_cast<cudaStream_t>(stream), X, s_m, s_n, out, M, N, accumulate);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_split3_bf16(const float* src, long src_ld, void* dst, int R, int C, int Cpad, int weight_mode, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(R > 0 && C > 0, "split3: empty");
  OMLM_CHECK_ARG(Cpad >= C && src_ld >= C, "split3: third width %d and source pitch %ld must be >= C = %d", Cpad, src_ld, C);
  const long total = static_cast<long>(R) * Cpad;
  const int blocks = static_cast<int>(std::min<long>((total + 255) / 256, 2048));
  OMLM_KLAUNCH((split3_kernel), blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream), src, src_ld, reinterpret_cast<__nv_bfloat16*>(dst), R, C, Cpad, weight_mode);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_bias_silu(float* z, const float* bias, float* a, int R, int C, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(R > 0 && C > 0, "bias_silu: empty");
  const long total = static_cast<long>(R) * C;
  const int blocks = static_cast<int>(std::min<long>((total + 255) / 256, 2048));
  OMLM_KLAUNCH((bias_silu_kernel), blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream), z, bias, a, R, C);
  OMLM_LAUNCH_CHECK();
  return 0;
}

int omlm_arange_f32(float* out, int n, void* stream) {
  using namespace omlm;
  OMLM_CHECK_ARG(n > 0, "arange: empty");
  OMLM_KLAUNCH((arange_kernel), (n + 255) / 256, 256, 0, reinterpret_cast<cudaStream_t>(stream), out, n);
  OMLM_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
