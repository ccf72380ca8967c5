// omlm_attn_fwd_tc_varlen: attn_fwd_tc_kernel<true>, compiled in a translation unit of its own.  With both
// instantiations in one unit ptxas schedules the fixed-length kernel differently; apart, that kernel keeps its SASS.
#define OMLM_ATTN_FWD_TC_VARLEN
#include "attn_fwd_tc.cu"
