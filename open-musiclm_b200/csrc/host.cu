// Host-side plumbing of libomlm_b200: last-error string, driver entry point for TMA descriptor
// encoding (resolved at run time so the library links without libcuda), device queries.
#include "common.cuh"
#include "../../include/omlm_b200.h"
#include <cudaTypedefs.h>
#include <stdarg.h>
#include <string.h>
#include <mutex>

namespace omlm {

static thread_local char g_err[1024] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
static std::once_flag g_encode_once;

static void resolve_encode() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) {
    g_encode = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(fn);
  }
}

int make_tmap_bf16_2d(CUtensorMap* out, const void* gptr, uint64_t dim0, uint64_t dim1,
                      uint64_t pitch_bytes, uint32_t box0, uint32_t box1) {
  std::call_once(g_encode_once, resolve_encode);
  OMLM_CHECK_ARG(g_encode != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  OMLM_CHECK_ARG((reinterpret_cast<uintptr_t>(gptr) & 15) == 0, "TMA base pointer must be 16B aligned");
  OMLM_CHECK_ARG((pitch_bytes & 15) == 0, "TMA row pitch must be a multiple of 16B (got %llu)",
                 (unsigned long long)pitch_bytes);
  OMLM_CHECK_ARG(box0 * 2 == 128 && box1 >= 1 && box1 <= 256, "bad TMA box %u x %u", box0, box1);
  cuuint64_t dims[2] = {dim0, dim1};
  cuuint64_t strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {box0, box1};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(gptr), dims,
                        strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  OMLM_CHECK_ARG(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return 0;
}

int make_tmap_2d(CUtensorMap* out, int elem_bytes, const void* gptr, uint64_t dim0, uint64_t dim1, uint64_t pitch_bytes,
                 uint32_t box0, uint32_t box1) {
  std::call_once(g_encode_once, resolve_encode);
  OMLM_CHECK_ARG(g_encode != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  OMLM_CHECK_ARG(elem_bytes == 2 || elem_bytes == 4, "make_tmap_2d: element size %d", elem_bytes);
  OMLM_CHECK_ARG((reinterpret_cast<uintptr_t>(gptr) & 15) == 0 && (pitch_bytes & 15) == 0, "TMA base / pitch must be 16B aligned");
  OMLM_CHECK_ARG(box0 * elem_bytes == 128 && box1 >= 1 && box1 <= 256, "bad TMA box %u x %u", box0, box1);
  cuuint64_t dims[2] = {dim0, dim1};
  cuuint64_t strides[1] = {pitch_bytes};
  cuuint32_t box[2] = {box0, box1};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(out, elem_bytes == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                        const_cast<void*>(gptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  OMLM_CHECK_ARG(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return 0;
}

int make_tmap_bf16_3d(CUtensorMap* out, const void* gptr, uint64_t dim0, uint64_t dim1, uint64_t dim2,
                      uint64_t pitch1_bytes, uint64_t pitch2_bytes, uint32_t box0, uint32_t box1) {
  std::call_once(g_encode_once, resolve_encode);
  OMLM_CHECK_ARG(g_encode != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  OMLM_CHECK_ARG((reinterpret_cast<uintptr_t>(gptr) & 15) == 0 && (pitch1_bytes & 15) == 0 && (pitch2_bytes & 15) == 0,
                 "TMA 3-D map: base and pitches must be 16B aligned");
  OMLM_CHECK_ARG(box0 * 2 == 128 && box1 >= 1 && box1 <= 256, "bad TMA box %u x %u", box0, box1);
  cuuint64_t dims[3] = {dim0, dim1, dim2};
  cuuint64_t strides[2] = {pitch1_bytes, pitch2_bytes};
  cuuint32_t box[3] = {box0, box1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(gptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  OMLM_CHECK_ARG(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled (3-D) failed with CUresult %d", (int)r);
  return 0;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

}  // namespace omlm

extern "C" {

const char* omlm_last_error(void) { return omlm::g_err; }

int omlm_abi_version(void) { return OMLM_B200_ABI_VERSION; }

int omlm_num_sms(void) { return omlm::num_sms(); }

int omlm_device_check(void) {
  int dev = 0;
  OMLM_CUDA(cudaGetDevice(&dev));
  int major = 0, minor = 0;
  OMLM_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  OMLM_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  OMLM_CHECK_ARG(major == 9 && minor == 0, "libomlm_b200 is built for sm_90a only; device is sm_%d%d", major, minor);
  return 0;
}

}  // extern "C"
