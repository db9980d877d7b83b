/* ccb200_debug.h - bring-up and diagnostic entry points of libccb200.so.  NOT part of the drop-in boundary
 * (include/ccb200.h): bench.py's per-kernel timing and the unit tests use them; a reference-side binding never needs them. */
#ifndef CCB200_DEBUG_H
#define CCB200_DEBUG_H
#include "ccb200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* which kernel the last convolution call of this thread launched ("conv_tc", "conv_tc_wgrad", or
 * "conv2d_fprop" / "conv2d_dgrad" / "conv2d_wgrad" for the CUDA-core GEMM): bench.py buckets its per-call timings by it */
const char* ccb_debug_last_conv_kernel(void);
/* host-side geometry of the wgmma convolution kernels for N output channels (no launch; unit tests):
 * out4 = {wgmma N, bytes of one B operand copy, pipeline stages, dynamic shared memory bytes} */
int ccb_debug_tc_plan(int N, int* out4);
/* the plan a convolution call with this descriptor runs (no launch; the layer audit records it per call):
 * out2 = {path: 0 CUDA-core GEMM, 1 tensor cores, 2 tensor-core weight gradient through rows padded to a multiple of 4;
 *         split-K count} */
int ccb_debug_conv_plan(const ccb_conv_desc* d, int op, int* out2);

#ifdef __cplusplus
}
#endif
#endif
