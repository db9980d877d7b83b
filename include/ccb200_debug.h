/* ccb200_debug.h - bring-up and diagnostic entry points of libccb200.so.  NOT part of the drop-in boundary
 * (include/ccb200.h): bench.py's per-kernel timing and the unit tests use them; a reference-side binding never needs them. */
#ifndef CCB200_DEBUG_H
#define CCB200_DEBUG_H
#include "ccb200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* which kernel the last convolution call of this thread launched ("conv_tc", "conv_tc_wgrad",
 * "conv2d_fprop" ... for the CUDA-core GEMM): bench.py buckets its per-call timings by it */
const char* ccb_debug_last_conv_kernel(void);
/* host-side geometry of the wgmma convolution kernels for N output channels (no launch; unit tests):
 * out4 = {wgmma N, bytes of one B operand copy, pipeline stages, dynamic shared memory bytes} */
int ccb_debug_tc_plan(int N, int* out4);

#ifdef __cplusplus
}
#endif
#endif
