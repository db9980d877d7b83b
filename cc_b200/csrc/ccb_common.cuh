// ccb_common.cuh - shared host/device helpers for libccb200 (sm_90a).
#pragma once
#include "../../include/ccb200.h"
#include "../../include/ccb200_debug.h"

#ifdef CCB_CPU_SIM
#include "cusim.h"   // tests/sim: CPU execution-model simulator, TEST BUILDS ONLY
#else
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <cmath>
// Every kernel is launched with programmatic stream serialisation (PDL) and starts with CCB_PDL_WAIT(): a kernel's
// launch + block scheduling then overlaps the tail of its predecessor (inside the step's CUDA graph: programmatic edges),
// and griddepcontrol.wait holds it before its first global-memory access until the predecessor has completed and flushed -
// same results, ~1900 launch gaps per step shorter.  CCB_PDL=0 in the environment turns the attribute off.
#define CCB_LAUNCH(kern_, grid_, block_, smem_, stream_, ...)                                     \
    do {                                                                                           \
        ++ccb::g_launches;                                                                         \
        cudaLaunchConfig_t cfg_ = {};                                                              \
        cfg_.gridDim = (grid_);                                                                    \
        cfg_.blockDim = (block_);                                                                  \
        cfg_.dynamicSmemBytes = (size_t)(smem_);                                                   \
        cfg_.stream = (cudaStream_t)(stream_);                                                     \
        cudaLaunchAttribute at_[1];                                                                \
        at_[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                            \
        at_[0].val.programmaticStreamSerializationAllowed = ccb::pdl_enabled();                    \
        cfg_.attrs = at_;                                                                          \
        cfg_.numAttrs = 1;                                                                         \
        cudaLaunchKernelEx(&cfg_, kern_, __VA_ARGS__);                                             \
    } while (0)
// CCB_PDL_TRIGGER: let the SUCCESSOR's blocks be scheduled as soon as every block of this grid has started (they park at their
// own CCB_PDL_SYNC; no block of this grid is left unscheduled by then, so nothing can starve).  CCB_PDL_SYNC: wait for the
// predecessor's completion + memory flush; must precede the first access to global data.  CCB_PDL_WAIT: both, at the top of
// a kernel.  The tensor-core kernels trigger at the top and sync AFTER their prologue (barrier init), which
// therefore overlaps the predecessor's tail.
#define CCB_PDL_TRIGGER() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")
#define CCB_PDL_SYNC() asm volatile("griddepcontrol.wait;" ::: "memory")
#define CCB_PDL_WAIT()      \
    do {                    \
        CCB_PDL_SYNC();     \
        CCB_PDL_TRIGGER();  \
    } while (0)
#define CCB_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#endif

namespace ccb {
extern long long g_launches;   // kernels launched through the library by this process (bench.py gpu_launches)
int pdl_enabled();             // common.cu: 1 unless CCB_PDL=0
}

namespace ccb {

// ---- error plumbing (C ABI never throws; reference raises AssertionError in Python instead) ----
void set_error(const char* fmt, ...);
int check_launch(const char* what);

#define CCB_REQUIRE(cond, code, ...)            \
    do {                                        \
        if (!(cond)) {                          \
            ccb::set_error(__VA_ARGS__);        \
            return (code);                      \
        }                                       \
    } while (0)

// ---- weight preparation for the tensor-core conv kernels (wprep.cu) ----
enum { WPREP_TC = 0 };
struct WPrepDesc {
    const float* w;
    float* wp;
    int N, Cc, KK, Ci, mode, Kp, ntaps;
    int layout, p0, p1, p2;      // TC: p0 = cpad
    signed char tap_index[64];
};
#ifndef CCB_CPU_SIM
int launch_wprep(const WPrepDesc& d, cudaStream_t st);
// prepared copy of d.w in d's layout: from the active weight cache (ccb_conv_desc.wcache) or produced now in d.wp
int wprep_get(const WPrepDesc& d, cudaStream_t st, const float** out);
struct WCache;
extern thread_local WCache* g_cur_wcache;
#endif

// ---- small device helpers ----
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Block-wide sum of NV values per thread; result valid in thread 0.  `scratch` holds >= NV*32 floats.
template <int NV>
__device__ __forceinline__ void block_sum(float (&v)[NV], float* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int i = 0; i < NV; ++i) v[i] = warp_sum(v[i]);
    __syncthreads();
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < NV; ++i) scratch[i * 32 + warp] = v[i];
    }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            float x = (lane < nwarps) ? scratch[i * 32 + lane] : 0.f;
            v[i] = warp_sum(x);
        }
    }
}

__host__ __device__ __forceinline__ int cdiv(int a, int b) { return (a + b - 1) / b; }

// streaming multiprocessors of the H100 SXM: grid and split-K plans aim at whole waves of this many CTAs
constexpr int NUM_SMS = 132;

}  // namespace ccb
