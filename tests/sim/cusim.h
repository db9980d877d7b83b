// cusim.h - a tiny single-threaded CUDA *execution-model* simulator for CPU-side unit tests.
//
// TEST TOOL ONLY.  The product library (libccb200.so) is compiled by nvcc for sm_90a and never
// includes this file.  tests/sim/build_sim.py compiles the very same kernel sources with
// g++ -DCCB_CPU_SIM so that the kernels' indexing / tiling / reduction logic can be checked against
// the oracle in the GPU-less build container before GPU minutes are spent.
//
// Model: one block at a time; every CUDA thread of the block is a ucontext fiber; __syncthreads(),
// __syncwarp() and the warp shuffles are cooperative barriers between fibers.  No timing model,
// no tensor cores, no TMA (kernels using those are compiled out under CCB_CPU_SIM).
#pragma once
#include <ucontext.h>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>
#include <algorithm>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__ __attribute__((noinline))
#define __restrict__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))
#define __constant__ static

struct dim3 {
    unsigned x, y, z;
    dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct uint3_ { unsigned x, y, z; };
struct float2 { float x, y; };
struct float4 { float x, y, z, w; };
struct int2 { int x, y; };
static inline float4 make_float4(float a, float b, float c, float d) { return float4{a, b, c, d}; }
static inline float2 make_float2(float a, float b) { return float2{a, b}; }
typedef int cudaError_t;
typedef void* cudaStream_t;
#define cudaSuccess 0
static inline cudaError_t cudaGetLastError() { return 0; }
static inline cudaError_t cudaPeekAtLastError() { return 0; }
static inline const char* cudaGetErrorString(cudaError_t) { return "sim"; }
static inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { memset(p, v, n); return 0; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, int, cudaStream_t) { memcpy(d, s, n); return 0; }
#define cudaMemcpyDeviceToDevice 3
template <class T> static inline cudaError_t cudaFuncSetAttribute(T, int, int) { return 0; }
#define cudaFuncAttributeMaxDynamicSharedMemorySize 8

namespace cusim {

struct Fiber {
    ucontext_t ctx;
    uint3_ tid;
    int lin;        // linear thread id
    bool done;
    char* stack;
};

struct Block {
    std::vector<Fiber> fibers;
    ucontext_t sched;
    int cur = -1;
    int nthreads = 0;
    // block barrier
    int bar_count = 0;
    unsigned bar_gen = 0;
    // warp barriers / exchange slots
    std::vector<int> wbar_count;
    std::vector<unsigned> wbar_gen;
    std::vector<uint64_t> wslot;  // [nwarps*32]
    std::function<void()> body;
    unsigned char* dyn_smem = nullptr;
};

extern Block* g_blk;
extern unsigned long g_progress;
extern uint3_ g_blockIdx;
extern dim3 g_blockDim, g_gridDim;

inline Fiber& cur() { return g_blk->fibers[g_blk->cur]; }
inline void yield() { swapcontext(&cur().ctx, &g_blk->sched); }

inline void block_barrier() {
    Block* b = g_blk;
    unsigned gen = b->bar_gen;
    if (++b->bar_count == b->nthreads) {
        b->bar_count = 0;
        b->bar_gen++;
        g_progress++;
        return;
    }
    while (b->bar_gen == gen) yield();
}

inline void warp_barrier() {
    Block* b = g_blk;
    int w = cur().lin >> 5;
    int wsize = std::min(32, b->nthreads - (w << 5));
    unsigned gen = b->wbar_gen[w];
    if (++b->wbar_count[w] == wsize) {
        b->wbar_count[w] = 0;
        b->wbar_gen[w]++;
        g_progress++;
        return;
    }
    while (b->wbar_gen[w] == gen) yield();
}

template <class T>
inline T exchange(T v, int src_lane) {
    static_assert(sizeof(T) <= 8, "shuffle payload");
    Block* b = g_blk;
    int lin = cur().lin, w = lin >> 5;
    uint64_t raw = 0;
    memcpy(&raw, &v, sizeof(T));
    b->wslot[lin] = raw;
    warp_barrier();
    int wsize = std::min(32, b->nthreads - (w << 5));
    T out = v;
    if (src_lane >= 0 && src_lane < wsize) {
        uint64_t r = b->wslot[(w << 5) + src_lane];
        memcpy(&out, &r, sizeof(T));
    }
    warp_barrier();
    return out;
}

void launch(dim3 grid, dim3 block, size_t smem, std::function<void()> body);
unsigned char* dyn_smem();

}  // namespace cusim

#define threadIdx (cusim::cur().tid)
#define blockIdx (cusim::g_blockIdx)
#define blockDim (cusim::g_blockDim)
#define gridDim (cusim::g_gridDim)
#define warpSize 32

static inline void __syncthreads() { cusim::block_barrier(); }
static inline void __syncwarp(unsigned = 0xffffffffu) { cusim::warp_barrier(); }
static inline void __threadfence() {}
static inline void __threadfence_block() {}
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int m, int = 32) { return cusim::exchange(v, (cusim::cur().lin & 31) ^ m); }
template <class T> static inline T __shfl_down_sync(unsigned, T v, unsigned d, int = 32) { return cusim::exchange(v, (cusim::cur().lin & 31) + (int)d); }
template <class T> static inline T __shfl_up_sync(unsigned, T v, unsigned d, int = 32) { return cusim::exchange(v, (cusim::cur().lin & 31) - (int)d); }
template <class T> static inline T __shfl_sync(unsigned, T v, int l, int = 32) { return cusim::exchange(v, l); }
static inline unsigned __ballot_sync(unsigned, int pred) {
    unsigned r = 0;
    for (int l = 0; l < 32; ++l) r |= (cusim::exchange<int>(pred != 0, l) ? 1u : 0u) << l;
    return r;
}
static inline unsigned __activemask() { return 0xffffffffu; }

template <class T> static inline T __ldg(const T* p) { return *p; }
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
static inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
static inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
static inline float __fsqrt_rn(float a) { return sqrtf(a); }
static inline float __frcp_rn(float a) { return 1.0f / a; }
static inline float __fdividef(float a, float b) { return a / b; }
// (__expf/__logf/__powf exist in glibc as internal symbols with the right meaning)
static inline float rsqrtf(float a) { return 1.0f / sqrtf(a); }
static inline float __saturatef(float a) { return a < 0 ? 0.f : (a > 1 ? 1.f : a); }
static inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline unsigned __float_as_uint(float f) { unsigned i; memcpy(&i, &f, 4); return i; }
static inline float __uint_as_float(unsigned i) { float f; memcpy(&f, &i, 4); return f; }
static inline int __float2int_rd(float f) { return (int)floorf(f); }
static inline float atomicAdd(float* p, float v) { float o = *p; *p = o + v; return o; }
static inline int atomicAdd(int* p, int v) { int o = *p; *p = o + v; return o; }
static inline unsigned atomicAdd(unsigned* p, unsigned v) { unsigned o = *p; *p = o + v; return o; }
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; *p = o + v; return o; }
static inline unsigned long long atomicMax(unsigned long long* p, unsigned long long v) { unsigned long long o = *p; if (v > o) *p = v; return o; }
static inline long long __double2ll_rn(double x) { return llrint(x); }
using std::isfinite;
static inline int __clzll(long long x) { return x == 0 ? 64 : __builtin_clzll((unsigned long long)x); }
static inline unsigned atomicInc(unsigned* p, unsigned lim) { unsigned o = *p; *p = (o >= lim) ? 0 : o + 1; return o; }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }

#define CCB_LAUNCH(kern, grid, block, smem, stream, ...)                     \
    do {                                                                      \
        ++ccb::g_launches;                                                    \
        cusim::launch(grid, block, smem, [&]() { kern(__VA_ARGS__); });       \
    } while (0)
namespace ccb { extern long long g_launches; }
#define CCB_DYN_SMEM(name) unsigned char* name = cusim::dyn_smem()
#define CCB_PDL_WAIT() ((void)0)      /* programmatic dependent launch: GPU builds only */
#define CCB_PDL_TRIGGER() ((void)0)
#define CCB_PDL_SYNC() ((void)0)
