// Shared host/device helpers for libomlm_b200 (sm_90a): error plumbing, TMA descriptor cache, small math.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda.h>
#include <stdint.h>
#include <stdio.h>

namespace omlm {

// ---- error reporting across the C ABI (no exceptions cross the boundary) -----------------
void set_last_error(const char* fmt, ...);
#define OMLM_CHECK_ARG(cond, ...)          \
  do {                                     \
    if (!(cond)) {                         \
      ::omlm::set_last_error(__VA_ARGS__); \
      return 1;                            \
    }                                      \
  } while (0)
#define OMLM_CUDA(expr)                                                                       \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      ::omlm::set_last_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return 1000 + static_cast<int>(_e);                                                     \
    }                                                                                         \
  } while (0)
#define OMLM_LAUNCH_CHECK() OMLM_CUDA(cudaGetLastError())

// ---- TMA descriptors ----------------------------------------------------------------------
// 2-D bf16 tensor map: inner (contiguous) extent dim0, outer extent dim1, row pitch in bytes,
// box {box0, box1}, SWIZZLE_128B (box0 * 2 bytes must be 128).
int make_tmap_bf16_2d(CUtensorMap* out, const void* gptr, uint64_t dim0, uint64_t dim1,
                      uint64_t pitch_bytes, uint32_t box0, uint32_t box1);

// 2-D tensor map of 2-byte (elem_bytes = 2) or fp32 (elem_bytes = 4) elements, SWIZZLE_128B, box0 * elem_bytes = 128:
// the staging layout of the GEMM epilogue's TMA stores / residual loads (32-row boxes).
int make_tmap_2d(CUtensorMap* out, int elem_bytes, const void* gptr, uint64_t dim0, uint64_t dim1, uint64_t pitch_bytes,
                 uint32_t box0, uint32_t box1);

// 3-D bf16 tensor map (dim0 contiguous), SWIZZLE_128B, box {box0, box1, 1}: out-of-range rows/planes are clipped.
int make_tmap_bf16_3d(CUtensorMap* out, const void* gptr, uint64_t dim0, uint64_t dim1, uint64_t dim2,
                      uint64_t pitch1_bytes, uint64_t pitch2_bytes, uint32_t box0, uint32_t box1);

int num_sms();

// ---- kernel launches ----------------------------------------------------------------------------------------------------
// cudaLaunchKernelEx returns the launch's own error, so a failure is reported at the launch that caused it.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
#define OMLM_KLAUNCH(kern, grid, block, smem, stream, ...)                                                   \
  do {                                                                                                       \
    cudaError_t _le = ::omlm::launch_k(kern, dim3(grid), dim3(block), smem, stream, __VA_ARGS__);            \
    if (_le != cudaSuccess) {                                                                                \
      ::omlm::set_last_error("%s:%d launch of %s -> %s", __FILE__, __LINE__, #kern, cudaGetErrorString(_le)); \
      return 1000 + static_cast<int>(_le);                                                                   \
    }                                                                                                        \
  } while (0)

// ---- device math --------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t v) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&v);
  return __bfloat1622float2(t);
}
__device__ __forceinline__ float bf16_round(float x) {
  return __bfloat162float(__float2bfloat16_rn(x));
}
// ---- 16-bit operand formats -------------------------------------------------------------------
// The tensor-core operands are 16-bit in two flavours (wgmma takes either at the same rate; both operands of one wgmma share the format):
//   fp16 (11-bit significand) for tensors that are bounded by construction -- LayerNorm outputs, weights, and the
//        FFN activations derived from them -- where it cuts the operand rounding error 8x against bf16;
//   bf16 (8-bit significand, fp32 range) for everything whose range is not bounded: gradients, the raw residual
//        stream feeding K/V, attention operands.
// fp16 conversions saturate (F2FP.SATFINITE) instead of producing inf.
enum : int { kFmtBF16 = 0, kFmtF32 = 1, kFmtF16 = 2 };
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t v) {
  __half2 t = *reinterpret_cast<__half2*>(&v);
  return __half22float2(t);
}
template <bool F16>
__device__ __forceinline__ uint32_t pack16x2(float lo, float hi) {
  if constexpr (F16) return pack_f16x2(lo, hi); else return pack_bf16x2(lo, hi);
}
template <bool F16>
__device__ __forceinline__ float2 unpack16x2(uint32_t v) {
  if constexpr (F16) return unpack_f16x2(v); else return unpack_bf16x2(v);
}

// ---- fp32x2 helpers: two neighbouring channels per call, written as two scalar IEEE round-to-nearest operations
// (sm_90 has no packed fp32 arithmetic; the pairing keeps the element-wise code compact).
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 splat2(float v) { return make_float2(v, v); }
__device__ __forceinline__ float rcp_approx(float x) {   // MUFU.RCP, <= 1 ulp, no slow path
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ float ex2_approx(float x) {
  float r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}

// ---- GELU (exact erf) ------------------------------------------------------------------------
// Abramowitz-Stegun 7.1.26 rational form (|error| <= 1.5e-7, below fp32 resolution of the products here),
// erf(x/sqrt(2)).  cdf = Phi(x), pdf = phi(x);  gelu(x) = x*cdf, gelu'(x) = cdf + x*pdf.
__device__ __forceinline__ void normal_cdf_pdf(float x, float& cdf, float& pdf) {
  const float e = ex2_approx(-0.72134752044448170f * x * x);          // exp(-x^2/2)
  const float t = rcp_approx(fmaf(0.23164189f, fabsf(x), 1.f));        // 0.3275911 / sqrt(2)
  float p = fmaf(0.5f * 1.061405429f, t, 0.5f * -1.453152027f);        // the 1/2 of erfc/2 folded into the coefficients
  p = fmaf(p, t, 0.5f * 1.421413741f);
  p = fmaf(p, t, 0.5f * -0.284496736f);
  p = fmaf(p, t, 0.5f * 0.254829592f);
  const float half_erfc = p * t * e;                    // 0.5 * erfc(|x|/sqrt2)
  cdf = x >= 0.f ? 1.f - half_erfc : half_erfc;
  pdf = 0.3989422804014327f * e;
}
// the same on two channels at once
__device__ __forceinline__ void normal_cdf_pdf2(float2 x, float2& cdf, float2& pdf) {
  const float2 q = mul2(mul2(x, x), splat2(-0.72134752044448170f));
  const float2 e = make_float2(ex2_approx(q.x), ex2_approx(q.y));
  const float2 t = make_float2(rcp_approx(fmaf(0.23164189f, fabsf(x.x), 1.f)), rcp_approx(fmaf(0.23164189f, fabsf(x.y), 1.f)));
  float2 p = fma2(splat2(0.5f * 1.061405429f), t, splat2(0.5f * -1.453152027f));
  p = fma2(p, t, splat2(0.5f * 1.421413741f));
  p = fma2(p, t, splat2(0.5f * -0.284496736f));
  p = fma2(p, t, splat2(0.5f * 0.254829592f));
  const float2 h = mul2(mul2(p, t), e);
  cdf = make_float2(x.x >= 0.f ? 1.f - h.x : h.x, x.y >= 0.f ? 1.f - h.y : h.y);
  pdf = mul2(e, splat2(0.3989422804014327f));
}
__device__ __forceinline__ float gelu_erf(float x) {
  float c, p;
  normal_cdf_pdf(x, c, p);
  return x * c;
}
__device__ __forceinline__ float2 gelu_erf2(float2 x) {
  float2 c, p;
  normal_cdf_pdf2(x, c, p);
  return mul2(x, c);
}

// Philox-4x32 counter RNG, 7 rounds (the shortest variant that passes BigCrush): dropout / forgetful-mask
// randomness, replayable in the backward pass from (seed, layer, row, chunk).
__device__ __forceinline__ uint4 philox4x32(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                            uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

}  // namespace omlm
