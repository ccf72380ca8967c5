// omlm_gemm_ffn_up_varlen: gemm_ffn_up_kernel<F16, true>, compiled in a translation unit of its own, so that the
// fixed-length instantiations of gemm_ffn_up.cu keep their SASS.
#define OMLM_GEMM_FFN_UP_VARLEN
#include "gemm_ffn_up.cu"
