// conv_tc.cu - implicit-GEMM convolution on the Hopper tensor cores (wgmma), sm_90a.
//
//   D[128 pixels x N<=128 channels] (fp32, registers) += A[128 x 32] (im2col tile) * B[N x 32]^T (weights)
//
// * one CTA works on one 128-row x N-channel output tile at a time (one persistent CTA per SM walks the tiles and
//   splits through one stage ring); one producer warpgroup + two consumer warpgroups, each
//   consumer owning 64 of the 128 rows (wgmma m64nNk8, N = the launch's channel tile rounded up to 16/32/64/128);
// * A is gathered straight from the NCHW activations (no im2col buffer in HBM): a K-chunk (wgrad: a group of 4 rows)
//   is 4 consecutive input channels of one filter tap, so the 4 loads of a chunk share the tap's bounds check; they
//   are coalesced across the 128 pixels of the tile (wgrad: the 32 pixels of the k-tile);
// * operands are staged in shared memory K-major with the 128-byte swizzle ([row][128 B], 16 B chunk ^= row & 7,
//   8-row atoms 1 KB apart): the layout wgmma reads for tf32, which it accepts only K-major.  In fprop / dgrad the
//   weight tiles arrive by TMA, which writes that swizzle itself: no producer thread waits for them.  In wgrad, B is the
//   output gradient: the producers copy it raw by 16-byte cp.async, the consumers split it into that layout;
// * fp32 parity: every fp32 operand is split hi = tf32(x), lo = x - hi and each k-step issues three
//   tf32 MMAs (hi*hi + lo*hi + hi*lo) ("3xTF32", error ~2^-21).  The tensor core only sums one 32-deep stage (small
//   cross terms first, then hi*hi) into a scratch register set; the stage's sum is added to the real accumulator with
//   fp32 adds, so no long accumulation chain runs through the tensor core's own rounding;
// * the producers gather the A tile once, unsplit, with zero-filling 4-byte cp.async straight from global into shared
//   memory (fprop / dgrad: k-major, see tc_a_idx; wgrad: row-major, see TcAWgrad), several stages of loads in flight;
//   each copy is one wide multiply-add from a pointer and stride worked out once per tap, since below N = 128 the
//   producers' instruction issue, not memory, is what paces the ring.
//   Each consumer thread loads its 16 values with 16 conflict-free LDS.32, splits them and issues wgmma with A from
//   registers (B by descriptor), so A crosses shared memory twice per stage instead of being stored twice and read
//   three times;
// * mbarrier pipeline of up to 4 stages: producers -> full[s] -> consumers (wgmma, commit group, wait, fp32 add)
//   -> empty[s].  Below N = 128 the consumers double-buffer the stage sums: while one stage's MMAs run they add the
//   previous stage's sum, release it and load and split the next stage, so the wgmma pipe is not drained between
//   stages; they take registers from the producers (setmaxnreg) to hold two sums and two A fragments.  At N = 128,
//   where one of each fills the registers, the two consumer warpgroups of fprop / dgrad issue their MMAs in turn
//   (named-barrier token), so one warpgroup's wait, add and next load overlap the other's MMAs (tc_consume_rs);
//   the epilogue adds bias / residual, applies the activation and stores NCHW straight from the accumulators.
//
// The same kernel serves FPROP, stride-1 DGRAD and the stride-parity classes of strided DGRAD /
// ConvTranspose2d forward through a per-tap offset table ("generalised fprop").
#include "conv.cuh"

#ifndef CCB_CPU_SIM

#include <cuda.h>            // CUtensorMap (the driver entry point is looked up at run time: no libcuda link)
#include <cudaTypedefs.h>    // PFN_cuTensorMapEncodeTiled
#include <type_traits>       // std::integral_constant: compile-time register-set index of tc_consume_rs

namespace ccb {

constexpr int TC_M = 128;          // pixels per tile (two wgmma M = 64 halves)
constexpr int TC_NMAX = 128;       // channels per tile
constexpr int TC_KC = 8;           // 16-byte k-chunks per stage (K = 32 fp32 per stage)
constexpr int TC_MAX_STAGES = 4;
constexpr int TC_PRODUCERS = 128;
constexpr int TC_CONSUMER_WARPS = 8;
constexpr int TC_THREADS = TC_PRODUCERS + 32 * TC_CONSUMER_WARPS;
constexpr int TC_MAX_TAPS = 49;
// Registers per thread of the fprop kernel: 168 at launch (384 threads at 1 CTA/SM hold 64512); from there the producers
// hand registers to the consumers, whose A fragments stay in registers: below wgmma N = 128 a consumer thread holds acc
// + two stage sums + the split A of the stage in flight and of the next (2 x 32): 160 at N = 64, as acc + part + one
// fragment at N = 128.  128 x 72 + 256 x 216 = 64512.  With nvcc 12.9, -Xptxas -v shows no spill, no stack and no
// serialized wgmma for any N at these counts (tests/test_conv_tc_resources.py); 64 / 224 spills the producers.
constexpr int TC_PRODUCER_REGS = 72, TC_CONSUMER_REGS = 216;

struct TcArgs {
    // prepared weights wp: tf32 hi copy [N][Kp] followed by the lo copy [N][Kp] (k = tap*cpad + c), as a 3-D TMA map
    // {Kp, N, 2} whose {32, NT, 1} box is one stage's B operand copy in the 128-byte-swizzled K-major layout; rows >= N
    // read as zeros
    CUtensorMap wmap;
    const float* x;        // input activations [B, Cin, Hin, Win]
    const float* bias;
    const float* res;
    float* out;            // [B, N_total, Hout, Wout]
    int B, Cin, Hin, Win;  // gathered tensor
    int Ntot;              // output channels
    int Hout, Wout;        // full output tensor size
    int Hc, Wc;            // output pixel grid of this launch (== Hout, Wout unless a parity class)
    int out_stride, out_oy, out_ox;   // y_out = oy * out_stride + out_oy
    int in_stride;         // iy = oy * in_stride + off_y[tap]
    int ntaps, cpad, Kp;   // taps in this launch, channels padded to 4, Kp = roundup(ntaps*cpad, 32)
    int M;                 // B * Hc * Wc
    int act;
    float slope;
    int ktiles, kt_per_split, splits;  // k-tiles of 32 (Kp / 32), split-K over them; partials go to `partial`
    float* partial;                    // [splits][numel(out)] raw accumulators (bias/res/act applied by the reduce kernel)
    int tiles_m, tiles_n, units;       // work units: 128-pixel tile (fastest) x channel tile x split, units = product
    long long out_numel;
    int depth, b_tile_bytes;           // stage ring (tc_geometry)
    signed char off_y[TC_MAX_TAPS], off_x[TC_MAX_TAPS];
};

// ---- PTX helpers ---------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded spin: a protocol bug traps (the launch fails) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try(bar, parity)) {
        if (++spins > (1u << 26)) asm volatile("trap;");
    }
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// one arrival on `bar` that also makes its current phase wait for `bytes` more of asynchronous (TMA) transfer
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// TMA: the box of `map` at coordinates (c0, c1, c2) into shared memory at `dst`, counted in as transfer bytes on `bar`
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_prefetch_map(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
// 4-byte asynchronous copy global -> shared (through L1, not through registers).  With `valid` false no byte is read
// and the destination is zero-filled; `src` must still be a valid global address.
__device__ __forceinline__ void cp_async_4(uint32_t dst, const float* src, bool valid) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(valid ? 4 : 0) : "memory");
}
// one arrival on `bar`, made once every cp.async this thread issued before it has landed; .noinc: the arrival counts
// against the barrier's expected count
__device__ __forceinline__ void cp_async_arrive(uint64_t* bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// 16-byte asynchronous copy global -> shared (L2 only); `src` 16-byte aligned, zero-fill as in cp_async_4
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ float tf32_hi(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

// wgmma shared-memory matrix descriptor of a K-major SWIZZLE_128B tile: 8-row atoms 1024 B apart (stride byte
// offset); the leading byte offset is unused by this layout; layout type 1 = 128-byte swizzle.  A k-step of 8 tf32
// advances the start address by 32 B inside the 128-byte row (the swizzle is a function of the absolute address,
// so every tile starts on a 1 KB boundary).
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }
template <int R>
__device__ __forceinline__ void wg_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int K, int R>
__device__ __forceinline__ void wg_fence_regs(uint32_t (&d)[K][R]) {
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
        for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[k][i])::"memory");
}

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, tf32 in, fp32 accumulators in registers (N / 2 per thread), A from registers:
// the m64k8 tf32 fragment, a[i] = A[wq * 16 + lane / 4 + 8 * (i & 1)][lane % 4 + 4 * (i >> 1)]
// for thread `lane` of warp wq of the warpgroup.  The registers must hold until the wgmma's group has been waited on.
__device__ __forceinline__ void wgmma_tf32_rs_n16(float (&d)[8], const uint32_t (&a)[4], uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "{%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}
__device__ __forceinline__ void wgmma_tf32_rs_n32(float (&d)[16], const uint32_t (&a)[4], uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "{%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}
__device__ __forceinline__ void wgmma_tf32_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}
__device__ __forceinline__ void wgmma_tf32_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
        " %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "{%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}
template <int NT>
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[NT / 2], const uint32_t (&a)[4], uint64_t db) {
    if constexpr (NT == 16) wgmma_tf32_rs_n16(d, a, db);
    else if constexpr (NT == 32) wgmma_tf32_rs_n32(d, a, db);
    else if constexpr (NT == 64) wgmma_tf32_rs_n64(d, a, db);
    else wgmma_tf32_rs_n128(d, a, db);
}

// setmaxnreg: a warpgroup hands registers back to the CTA's pool or takes them from it (counts: multiples of 8)
template <int R> __device__ __forceinline__ void wg_regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void wg_regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

constexpr int TC_TILE_BYTES = TC_KC * TC_M * 16;                   // one A operand copy of one stage: 16 KB
constexpr int TC_SMEM_MAX = 227 * 1024;

// float4 index of (row, 16-byte chunk) inside one swizzled operand tile
__device__ __forceinline__ int tile_idx(int row, int chunk) { return row * TC_KC + (chunk ^ (row & 7)); }

// x split into hi = tf32(x) and lo = tf32(x - hi), stored as float4 `idx` of the hi and the lo tile
__device__ __forceinline__ void tc_split_store(unsigned char* hi, unsigned char* lo, int idx, float4 x) {
    float4 h, l;
    h.x = tf32_hi(x.x); h.y = tf32_hi(x.y); h.z = tf32_hi(x.z); h.w = tf32_hi(x.w);
    ((float4*)hi)[idx] = h;
    l.x = tf32_hi(x.x - h.x); l.y = tf32_hi(x.y - h.y); l.z = tf32_hi(x.z - h.z); l.w = tf32_hi(x.w - h.w);
    ((float4*)lo)[idx] = l;
}

// The four operand tiles of one stage as byte addresses of type T: unsigned char* for the producers' stores, the
// uint32_t shared-space address for the consumers' wgmma descriptors.
template <typename T> struct TcTiles { T a_hi, a_lo, b_hi, b_lo; };

// The stage ring of both kernels in dynamic shared memory: `depth` stages of [A hi | A lo | B hi | B lo] (A: the 128
// rows of the tile, B: the wgmma N rows), then a full (producers -> consumers) and an empty (consumers -> producers)
// mbarrier per stage.  The it-th k-tile of a CTA passes through stage it % depth in round it / depth.
struct TcRing {
    unsigned char* smem;        // stage 0, on a 1 KB boundary: SWIZZLE_128B atoms are 1 KB
    int depth, stage_bytes, b_tile_bytes;
    uint64_t *full, *empty;

    template <typename T>
    __device__ __forceinline__ TcTiles<T> tiles(T base, int s) const {
        const T st = base + s * stage_bytes;
        return {st, st + TC_TILE_BYTES, st + 2 * TC_TILE_BYTES, st + 2 * TC_TILE_BYTES + b_tile_bytes};
    }
    // producers: wait until the consumers have released stage s = it % depth (the first round finds every stage free),
    // then write its tiles
    __device__ __forceinline__ TcTiles<unsigned char*> acquire(int it, int s) const {
        if (it >= depth) mbar_wait(&empty[s], ((it / depth) - 1) & 1);
        return tiles(smem, s);
    }
    // producers: make this thread's stores into stage s visible to wgmma (the async proxy) and count them in
    __device__ __forceinline__ void publish(int s) const { fence_proxy_async(); mbar_arrive(&full[s]); }
};

// Set-up at the top of both kernels: it touches no global data, so it overlaps the predecessor's tail (PDL), and
// returns once the predecessor's results are visible.  A full[s] phase completes after `full_arrivals` arrivals (and
// the transfer bytes any of them announced).
__device__ __forceinline__ TcRing tc_ring(int depth, int b_tile_bytes, int full_arrivals) {
    CCB_PDL_TRIGGER();
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int stage_bytes = 2 * TC_TILE_BYTES + 2 * b_tile_bytes;
    uint64_t* full = (uint64_t*)(smem + depth * stage_bytes);
    const TcRing r = {smem, depth, stage_bytes, b_tile_bytes, full, full + TC_MAX_STAGES};
    if (threadIdx.x == 0) {
        for (int s = 0; s < depth; ++s) { mbar_init(&r.full[s], full_arrivals); mbar_init(&r.empty[s], TC_CONSUMER_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();
    CCB_PDL_SYNC();
    return r;
}

// wgmma m64nN accumulator layout: register tc_acc_reg(i, half, e) of consumer warp wq of warpgroup wg holds row
// tc_acc_row(wg, wq, lane, half) of the CTA's 128 rows and column tc_acc_col(lane, i, e), i < N / 8, half, e < 2.
__device__ __forceinline__ int tc_acc_row(int wg, int wq, int lane, int half) { return wg * 64 + wq * 16 + (lane >> 2) + half * 8; }
__device__ __forceinline__ int tc_acc_col(int lane, int i, int e) { return 8 * i + 2 * (lane & 3) + e; }
__device__ __forceinline__ int tc_acc_reg(int i, int half, int e) { return 4 * i + 2 * half + e; }

// The A tile: one fp32 copy of the stage's 128 x 32 im2col values, unsplit, in the first A slot of the stage.  Each
// consumer thread (rows r0 = wg * 64 + wq * 16 + lane / 4 and r0 + 8, column t = lane % 4) reads its 16 values with 16
// LDS.32 at k = t + 4 j.  The two kernels gather along different axes, so each has its own swizzled layout, both
// bank-conflict free on both sides.  A layout L gives the byte offset L::off(r0, t) of A[r0][t] and, from it, the byte
// offset L::at(off, h, j) of A[r0 + 8 h][t + 4 j].
//
// TcAFprop (fprop / dgrad), k-major with the row index swizzled by k:  A[r][k] is float tc_a_idx(r, k) = 128 k + (r ^ 8 (k % 4)).
// The producers write it with 4-byte cp.async, a warp's 32 lanes being the 32 consecutive rows 32 w + lane at one k:
// r ^ 8 (k % 4) permutes those 32 rows among themselves (8 (k % 4) < 32), so the 32 words land on the 32 banks.  The
// consumers read all 16 values with k % 4 = t: lane l of a warp reads bank (r0 + 8 h) ^ 8 t mod 32, whose low 3 bits
// are lane / 4 and whose bits 3-4 are those of wq * 16 + 8 h flipped by t, so the 8 row offsets times the 4 columns
// of the warp cover the 32 banks once.  r0 & 8 = 0, so row r0 + 8 flips bit 3 of the row, byte bit 5, and k + 4 j is
// 2 KB further on.
//
// TcAWgrad (wgrad: rows (tap, ci), k = 32 pixels), row-major with k swizzled by the row:  A[r][k] is float
// TcAWgrad::idx(r, k) = 32 r + (k ^ 4 (r % 8)).  The producers write one row per warp instruction, lane = k:
// k ^ 4 (r % 8) permutes the 32 lanes, so the 32 words land on the 32 banks.  Consumer lane l reads word
// 32 (r0 + 8 h) + (t + 4 j) ^ 4 (lane / 4) = ... + t + 4 (j ^ lane / 4) (r0 % 8 = lane / 4, t < 4): bank
// t + 4 (j ^ lane / 4), which for one j covers the 32 banks once over the 4 t and 8 lane / 4.  In bytes that is
// (off(r0, t) + 1024 h) ^ 16 j: bits 4-6 of off hold lane / 4, and no other term reaches them.
struct TcAFrag { uint32_t hi[TC_KC / 2][4], lo[TC_KC / 2][4]; };   // [k-step][wgmma A register]

__device__ __forceinline__ int tc_a_idx(int r, int k) { return k * TC_M + (r ^ (8 * (k & 3))); }
struct TcAFprop {
    __device__ __forceinline__ static int off(int r0, int t) { return tc_a_idx(r0, t) * 4; }
    __device__ __forceinline__ static int at(int off, int h, int j) { return (off ^ (32 * h)) + 2048 * j; }
};
struct TcAWgrad {
    __device__ __forceinline__ static int idx(int r, int k) { return 32 * r + (k ^ (4 * (r & 7))); }
    __device__ __forceinline__ static int off(int r0, int t) { return idx(r0, t) * 4; }
    __device__ __forceinline__ static int at(int off, int h, int j) { return (off + 1024 * h) ^ (16 * j); }
};
// this thread's 16 raw values of the A tile at `tile` in layout L: v[h][j] = A[r0 + 8 h][t + 4 j], off = L::off(r0, t)
template <typename L>
__device__ __forceinline__ void tc_load_a(const unsigned char* tile, int off, float (&v)[2][8]) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j) v[h][j] = *(const float*)(tile + L::at(off, h, j));
}
// the split of tc_split_store, hi = tf32(x), lo = tf32(x - hi), into the fragment: k-step ks, register i holds
// row r0 + 8 (i & 1), k = 8 ks + t + 4 (i >> 1)
__device__ __forceinline__ void tc_split_a(const float (&v)[2][8], TcAFrag& f) {
#pragma unroll
    for (int ks = 0; ks < TC_KC / 2; ++ks)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float x = v[i & 1][2 * ks + (i >> 1)], h = tf32_hi(x);
            f.hi[ks][i] = __float_as_uint(h);
            f.lo[ks][i] = __float_as_uint(tf32_hi(x - h));
        }
}

// The consumers' named barrier (barrier 0 is __syncthreads): the 256 threads of both consumer warpgroups
__device__ __forceinline__ void tc_consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(32 * TC_CONSUMER_WARPS) : "memory"); }

// What the consumers do to a full stage's B operand before its MMAs (tc_consume_rs): nothing in fprop / dgrad, whose B
// tiles arrive by TMA already split.
struct TcFpropFeed {
    static constexpr bool split_b = false;
    __device__ __forceinline__ void prep_b(const TcTiles<unsigned char*>&) const {}
};

// The token the two consumer warpgroups pass so that their MMAs reach the tensor cores in turn (tc_consume_rs, N = 128
// fprop / dgrad): warpgroup 0 arrives on TC_BAR_WG0_ISSUED once it has issued a stage, warpgroup 1 on
// TC_BAR_WG1_ISSUED.  Named barriers 2 and 3 (0 is __syncthreads, 1 tc_consumer_sync), each completed by the 128
// arrivals of one warpgroup and the 128 waiting threads of the other.
constexpr int TC_BAR_WG0_ISSUED = 2, TC_BAR_WG1_ISSUED = 3;
template <int ID> __device__ __forceinline__ void tc_token_arrive() {
    asm volatile("bar.arrive %0, %1;" ::"n"(ID), "n"(32 * TC_CONSUMER_WARPS) : "memory");
}
template <int ID> __device__ __forceinline__ void tc_token_wait() {
    asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(32 * TC_CONSUMER_WARPS) : "memory");
}

// One stage's MMAs on this warpgroup's 64 rows into `part`, zeroed first: 4 k-steps of (lo*hi) + (hi*lo), then the 4
// (hi*hi), as one commit group.  The registers of `part` and `f` belong to the MMAs until that group is waited on.
template <int NT>
__device__ __forceinline__ void tc_issue_stage(const TcTiles<uint32_t>& tl, const TcAFrag& f, float (&part)[NT / 2]) {
#pragma unroll
    for (int j = 0; j < NT / 2; ++j) part[j] = 0.f;
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < TC_KC / 2; ++ks) {
        const uint32_t koff = (uint32_t)ks * 32u;
        wgmma_tf32_rs<NT>(part, f.lo[ks], wg_desc(tl.b_hi + koff));
        wgmma_tf32_rs<NT>(part, f.hi[ks], wg_desc(tl.b_lo + koff));
    }
#pragma unroll
    for (int ks = 0; ks < TC_KC / 2; ++ks)
        wgmma_tf32_rs<NT>(part, f.hi[ks], wg_desc(tl.b_hi + (uint32_t)ks * 32u));
    wg_commit();
}

// Consumer side of both kernels, A (in layout L) from registers: acc = 0 (an empty split contributes zeros), then for
// each of the unit's `nkt` stages its MMAs into a scratch register set `part` (tc_issue_stage), then acc += part in
// fp32, in stage order, and the stage goes back to the producers.  Taking a full stage means loading and splitting this
// thread's A fragment and, where Feed::split_b, its share of the B operand (prep_b, by all 256 consumer threads, then
// made visible to wgmma: proxy fence, consumer barrier).  B of a stage is read by its MMAs until their group is waited
// on, so the stage is released after that wait.  The unit's k-tiles are the CTA's g-th onwards: they start in stage
// g % depth.
//
// Below N = 128 the stage sums are double-buffered, part[2] with a fragment each, so the wgmma pipe is never drained
// inside a unit: stage it goes into part[it & 1], then wg_wait<1> retires stage it - 1 alone, which is released and
// added while stage it's MMAs run, and stage it + 1 is taken into the fragment stage it - 1 has freed.  The consumers
// hold two stages, the one in flight and the one just taken.  The loop is unrolled by two so that it & 1 is a
// compile-time index and both sets stay in registers, and each step is take, issue, wait, retire: the only branches
// are the exits, so a set in flight never meets a retired one at a join, which ptxas answers by serializing every
// wgmma (tests/test_conv_tc_resources.py).
//
// At N = 128 acc + part already take 128 registers and a second fragment does not fit without spilling, so each stage
// is taken after the previous one's wait.  In fprop / dgrad the two warpgroups then issue in turn (`ordered`): warpgroup
// 1 issues stage it once warpgroup 0 has, and warpgroup 0 issues stage it + 1 once warpgroup 1 has issued stage it, so
// one warpgroup's wait, add and take overlap the other's MMAs instead of both draining the tensor cores together.  Each
// unit ends with warpgroup 0 waiting for warpgroup 1's last token, so every arrival is matched within the unit.  In
// wgrad prep_b's barrier keeps the two warpgroups in step at every stage, and they issue together.
template <int NT, typename L, typename Feed>
__device__ __forceinline__ void tc_consume_rs(const TcRing& ring, int g, int nkt, int wg, int wq, int lane, const Feed& feed,
                                              float (&acc)[NT / 2]) {
#pragma unroll
    for (int j = 0; j < NT / 2; ++j) acc[j] = 0.f;
    const uint32_t base = smem_u32(ring.smem);
    const int a_off = L::off(wg * 64 + wq * 16 + (lane >> 2), lane & 3);
    auto take = [&](int st, uint32_t ph, TcAFrag& f) {
        mbar_wait(&ring.full[st], ph);
        const TcTiles<unsigned char*> t = ring.tiles(ring.smem, st);
        float v[2][8];
        tc_load_a<L>(t.a_hi, a_off, v);
        tc_split_a(v, f);
        if constexpr (Feed::split_b) {
            feed.prep_b(t);
            fence_proxy_async();
            tc_consumer_sync();
        }
    };
    // after the wait that retired a stage's group: hand its sum to acc and its registers back to the compiler (the MMAs
    // read f and wrote part until then: the fences keep the compiler from reusing or reading them before the wait)
    auto retire = [&](int st, float (&part)[NT / 2], TcAFrag& f) {
        wg_fence_regs(part);
        wg_fence_regs(f.hi);
        wg_fence_regs(f.lo);
        if (lane == 0) mbar_arrive(&ring.empty[st]);
#pragma unroll
        for (int j = 0; j < NT / 2; ++j) acc[j] += part[j];
    };
    int s = g % ring.depth;                     // stage of k-tile it
    uint32_t phase = (g / ring.depth) & 1;      // parity of k-tile it's round
    if constexpr (NT < 128) {
        TcAFrag f[2];
        float part[2][NT / 2];
        int sp = s;                             // stage of k-tile it - 1
        // k-tile it, B = it & 1: taken into f[B] and issued into part[B]; then k-tile it - 1, in flight in the other set,
        // is retired.  The group of k-tile it is in flight at the end.
        auto step = [&](auto B, bool first) {
            constexpr int b = decltype(B)::value;
            take(s, phase, f[b]);
            tc_issue_stage<NT>(ring.tiles(base, s), f[b], part[b]);
            if (!first) {
                wg_wait<1>();
                retire(sp, part[b ^ 1], f[b ^ 1]);
            }
            sp = s;
            s = s + 1 == ring.depth ? 0 : s + 1;
            phase ^= (s == 0);
        };
        // after the unit's last k-tile, in flight in set B
        auto finish = [&](auto B) {
            wg_wait<0>();
            retire(sp, part[decltype(B)::value], f[decltype(B)::value]);
        };
        using Set0 = std::integral_constant<int, 0>;
        using Set1 = std::integral_constant<int, 1>;
        if (nkt > 0) {
            step(Set0(), true);
            for (int it = 1;; it += 2) {
                if (it == nkt) { finish(Set0()); break; }
                step(Set1(), false);
                if (it + 1 == nkt) { finish(Set1()); break; }
                step(Set0(), false);
            }
        }
    } else {
        constexpr bool ordered = !Feed::split_b;
        TcAFrag f;
        float part[NT / 2];
        for (int it = 0; it < nkt; ++it) {
            take(s, phase, f);
            if constexpr (ordered) {
                if (wg == 1) tc_token_wait<TC_BAR_WG0_ISSUED>();
                else if (it > 0) tc_token_wait<TC_BAR_WG1_ISSUED>();
            }
            tc_issue_stage<NT>(ring.tiles(base, s), f, part);
            if constexpr (ordered) {
                if (wg == 0) tc_token_arrive<TC_BAR_WG0_ISSUED>();
                else tc_token_arrive<TC_BAR_WG1_ISSUED>();
            }
            wg_wait<0>();
            retire(s, part, f);
            s = s + 1 == ring.depth ? 0 : s + 1;
            phase ^= (s == 0);
        }
        if constexpr (ordered) {
            if (wg == 0 && nkt > 0) tc_token_wait<TC_BAR_WG1_ISSUED>();
        }
    }
}

// One work unit: the 128-row x 128-channel output tile and the k-tiles of one split (Args: TcArgs or TcWgradArgs).
struct TcUnit { int m0, n0, z, kt_beg, nkt; };
template <typename Args>
__device__ __forceinline__ TcUnit tc_unit(const Args& a, int u) {
    TcUnit w;
    w.m0 = (u % a.tiles_m) * TC_M;
    u /= a.tiles_m;
    w.n0 = (u % a.tiles_n) * TC_NMAX;
    w.z = u / a.tiles_n;
    w.kt_beg = w.z * a.kt_per_split;
    w.nkt = max(0, min(a.ktiles, w.kt_beg + a.kt_per_split) - w.kt_beg);   // k-tiles of this split
    return w;
}

// Persistent: a CTA runs units blockIdx.x, blockIdx.x + gridDim.x, ... through one stage ring, its g-th k-tile in stage
// g % depth, so the producers gather the next unit's first stages while the consumers finish the current one and
// store it, and the set-up and the ring's first fill are paid once per CTA instead of once per tile.
template <int NT>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const __grid_constant__ TcArgs a) {
    // full[s]: the 128 producers' arrivals, each made when that thread's A copies have landed, + producer 0's arrival
    // that announces the B tiles' TMA bytes
    const TcRing ring = tc_ring(a.depth, a.b_tile_bytes, TC_PRODUCERS + 1);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const long long HWin = (long long)a.Hin * a.Win;

    if (warp < TC_PRODUCERS / 32) {
        // ===================== producers: thread == tile row =====================
        wg_regs_dec<TC_PRODUCER_REGS>();
        const int r = tid;
        const int cpt = a.cpad >> 2;                 // chunks per tap; chunks of taps >= ntaps are Kp's zero padding
        const int hwin = a.Hin * a.Win;              // channel-plane stride (a plane has < 2^31 pixels)
        if (r == 0) tma_prefetch_map(&a.wmap);
        int g = 0;                                   // k-tiles this CTA has gathered
        for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
            const TcUnit w = tc_unit(a, u);
            const int m = w.m0 + r;
            const bool mvalid = m < a.M;
            int b = 0, oy = 0, ox = 0;
            if (mvalid) {
                int hw = a.Hc * a.Wc;
                b = m / hw;
                int rem = m - b * hw;
                oy = rem / a.Wc;
                ox = rem - oy * a.Wc;
            }
            const float* xb = a.x + (long long)b * a.Cin * HWin;
            const int iy0 = oy * a.in_stride, ix0 = ox * a.in_stride;
            for (int it = 0; it < w.nkt; ++it, ++g) {
                const int s = g % ring.depth;
                const int kt = w.kt_beg + it;                 // global k-tile
                const TcTiles<unsigned char*> t = ring.acquire(g, s);
                // ---- B: the weights were split into tf32 hi / lo by the prep kernel: one TMA box per copy; rows in
                //      [ntile, NT) past the last channel are zero-filled, and the epilogue ignores those columns
                if (r == 0) {
                    mbar_arrive_expect_tx(&ring.full[s], 2 * ring.b_tile_bytes);
                    tma_load_3d(t.b_hi, &a.wmap, &ring.full[s], kt * (TC_KC * 4), w.n0, 0);
                    tma_load_3d(t.b_lo, &a.wmap, &ring.full[s], kt * (TC_KC * 4), w.n0, 1);
                }
                const uint32_t at = smem_u32(t.a_hi);
                // ---- A: the 8 chunks (32 floats) of this thread's pixel row, k = 4c + j of the stage, copied by cp.async
                //      straight into the tile (tc_a_idx) with zeros where the im2col matrix has none.  The thread never
                //      waits for its copies: its arrival on full[s] is made when they land, so up to `depth` stages of
                //      loads are in flight.  The consumers read A with ld.shared, so no proxy fence is needed.
                //      The producers issue one instruction stream per scheduler, and below N = 128 that stream is what
                //      paces the stage ring, so each copy is one wide multiply-add from a base pointer and a
                //      channel-plane step worked out once per tap.  A pixel without a value copies from its image's
                //      base with step 0, and a channel past C_in from the last channel's address: every copy names a
                //      valid address, and those copies read nothing (zero fill).
                const int q0 = kt * TC_KC;
                const int tap0 = q0 / cpt, c40 = q0 - tap0 * cpt;
                // this thread's pixel under tap `tap` (Kp's zero padding past the last tap has none): the address of
                // channel 4 c4 and the channel-plane step, 0 when there is no value
                auto tap_src = [&](int tap, int c4, const float*& p, int& step) {
                    const bool real = tap < a.ntaps;
                    const int t = real ? tap : 0;
                    const int iy = iy0 + a.off_y[t], ix = ix0 + a.off_x[t];
                    const bool ok = mvalid && real && (unsigned)iy < (unsigned)a.Hin && (unsigned)ix < (unsigned)a.Win;
                    p = xb + (ok ? c4 * 4 * hwin + iy * a.Win + ix : 0);
                    step = ok ? hwin : 0;
                };
                if (c40 + TC_KC <= cpt) {
                    // the whole stage reads one filter tap (C_in % 32 == 0 layers): one bounds check, one base
                    // pointer, 32 copies one channel plane apart
                    const float* p;
                    int step;
                    tap_src(tap0, c40, p, step);
                    const int nv = a.Cin - c40 * 4;           // channels from the stage's first: >= 1
                    if (nv >= TC_KC * 4) {
#pragma unroll
                        for (int k = 0; k < TC_KC * 4; ++k) cp_async_4(at + 4 * tc_a_idx(r, k), p + k * step, step != 0);
                    } else {
#pragma unroll
                        for (int k = 0; k < TC_KC * 4; ++k)
                            cp_async_4(at + 4 * tc_a_idx(r, k), p + min(k, nv - 1) * step, step != 0 && k < nv);
                    }
                } else {
                    // one tap per chunk of 4 channels; with C_in % 4 == 0 every chunk has its 4 channels
                    auto chunks = [&](auto whole4) {
                        int tap = tap0, c4 = c40;
#pragma unroll
                        for (int c = 0; c < TC_KC; ++c) {
                            const float* p;
                            int step;
                            tap_src(tap, c4, p, step);
                            const int nv = a.Cin - c4 * 4;    // >= 1: c4 < cpad / 4
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                if constexpr (decltype(whole4)::value)
                                    cp_async_4(at + 4 * tc_a_idx(r, 4 * c + j), p + j * step, step != 0);
                                else
                                    cp_async_4(at + 4 * tc_a_idx(r, 4 * c + j), p + min(j, nv - 1) * step, step != 0 && j < nv);
                            }
                            if (++c4 == cpt) { c4 = 0; ++tap; }
                        }
                    };
                    if ((a.Cin & 3) == 0) chunks(std::true_type());
                    else chunks(std::false_type());
                }
                cp_async_arrive(&ring.full[s]);
            }
        }
        cp_async_wait_all();      // no thread leaves copies in flight behind it
    } else {
        // ===================== consumers: MMA + epilogue =====================
        wg_regs_inc<TC_CONSUMER_REGS>();
        const int wg = (warp - TC_PRODUCERS / 32) >> 2, wq = warp & 3;
        const long long HWout = (long long)a.Hout * a.Wout;
        int g = 0;                                   // k-tiles this CTA has consumed
        for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
            const TcUnit w = tc_unit(a, u);
            const int ntile = min(TC_NMAX, a.Ntot - w.n0);
            float acc[NT / 2];
            tc_consume_rs<NT, TcAFprop>(ring, g, w.nkt, wg, wq, lane, TcFpropFeed(), acc);
            g += w.nkt;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int em = w.m0 + tc_acc_row(wg, wq, lane, half);
                if (em >= a.M) continue;
                int hw = a.Hc * a.Wc;
                int eb = em / hw;
                int rem = em - eb * hw;
                int eoy = rem / a.Wc, eox = rem - eoy * a.Wc;
                const long long obase = (long long)eb * a.Ntot * HWout + (long long)(eoy * a.out_stride + a.out_oy) * a.Wout +
                                        (eox * a.out_stride + a.out_ox);
#pragma unroll
                for (int i = 0; i < NT / 8; ++i)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int nl = tc_acc_col(lane, i, e);
                        if (nl < ntile) {
                            float o = acc[tc_acc_reg(i, half, e)];
                            const int n = w.n0 + nl;
                            const long long off = obase + (long long)n * HWout;
                            if (a.splits > 1) {
                                a.partial[(long long)w.z * a.out_numel + off] = o;
                            } else {
                                if (a.bias) o += __ldg(a.bias + n);
                                if (a.res) o += __ldg(a.res + off);
                                a.out[off] = apply_act(o, a.act, a.slope);
                            }
                        }
                    }
            }
        }
    }
}

// Weight re-layout: wp[n][t*cpad + c] = w[(co,ci) by mode][tap(t)], zero padded to Kp.
//   mode 0 (fprop): n = co, c = ci : w[n][c][tap]        mode 1 (dgrad): n = ci, c = co : w[c][n][tap]
static int roundup(int v, int m) { return (v + m - 1) / m * m; }
// Kp of `ntaps` taps of Cc channels: whole k-tiles; a parity class without taps still runs one all-zero k-tile
static int tc_kp(int ntaps, int Cc) { return ntaps > 0 ? roundup(ntaps * roundup(Cc, 4), TC_KC * 4) : TC_KC * 4; }

// Operand tile geometry of one launch: the B tile holds the wgmma N (16/32/64/128) rows, and as many stages as fit
// in shared memory as the ring's depth (up to 4: 3 at N = 128 in 3xTF32 layout, 4 below).
static void tc_geometry(int N, int& nt, int& b_tile_bytes, int& depth, int& smem) {
    const int ntile_max = N < TC_NMAX ? N : TC_NMAX;
    nt = 16;
    while (nt < ntile_max) nt <<= 1;
    b_tile_bytes = nt * 128;
    const int stage = 2 * TC_TILE_BYTES + 2 * b_tile_bytes;
    depth = (TC_SMEM_MAX - 2048) / stage;
    if (depth > TC_MAX_STAGES) depth = TC_MAX_STAGES;
    smem = depth * stage + 2048;                      // + barriers / alignment slack
}

template <typename Args>
static int tc_launch_kernel(void (*const (&kfns)[4])(const Args), const Args& a, int nt, dim3 grid, int smem, cudaStream_t st,
                            const char* what) {
    auto kfn = kfns[nt == 16 ? 0 : nt == 32 ? 1 : nt == 64 ? 2 : 3];
    cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_MAX);
    CCB_LAUNCH(kfn, grid, dim3(TC_THREADS), smem, st, a);
    return check_launch(what);
}

static void (*const TC_FPROP_KERNELS[4])(const TcArgs) = {conv_tc_kernel<16>, conv_tc_kernel<32>, conv_tc_kernel<64>,
                                                          conv_tc_kernel<128>};

// The TMA map of a prepared weight panel wp [2][N][Kp] (see TcArgs::wmap) with boxes of `nt` rows.  The encode is a host
// call: under graph capture its result is baked into the launch, which holds because the panel (weight cache or
// workspace) stays at the same address in replay.
static int tc_weight_map(CUtensorMap* map, const float* wp, int N, int Kp, int nt) {
    static PFN_cuTensorMapEncodeTiled_v12000 encode = [] {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &fn, 12000, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            fn = nullptr;
        return (PFN_cuTensorMapEncodeTiled_v12000)fn;
    }();
    CCB_REQUIRE(encode, CCB_ERR_LAUNCH, "conv_tc: the driver has no cuTensorMapEncodeTiled");
    const cuuint64_t dims[3] = {(cuuint64_t)Kp, (cuuint64_t)N, 2};
    const cuuint64_t strides[2] = {(cuuint64_t)Kp * sizeof(float), (cuuint64_t)N * Kp * sizeof(float)};
    const cuuint32_t box[3] = {TC_KC * 4, (cuuint32_t)nt, 1};
    const cuuint32_t estrides[3] = {1, 1, 1};
    const CUresult rc = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)wp, dims, strides, box, estrides,
                               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CCB_REQUIRE(rc == CUDA_SUCCESS, CCB_ERR_LAUNCH, "conv_tc: cuTensorMapEncodeTiled failed (%d) for N %d Kp %d", (int)rc, N, Kp);
    return CCB_OK;
}

// The grid of a persistent launch: one CTA per SM (launch bounds, registers) runs units until none are left
static dim3 tc_persistent_grid(int units) {
    static int sms = [] {
        int dev = 0, n = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        return n > 0 ? n : NUM_SMS;
    }();
    return dim3(units < sms ? units : sms);
}

// One generalised-fprop launch (+ its weight preparation into `wp`, tf32 hi copy + lo copy).
static int launch_tc(TcArgs& a, const float* w, int mode, int N, int Cc, int KK, int Ci, const signed char* tap_index,
                     float* wp, float* partial, int splits, cudaStream_t st) {
    a.cpad = roundup(Cc, 4);
    a.Kp = tc_kp(a.ntaps, Cc);
    WPrepDesc p;
    memset(&p, 0, sizeof(p));
    p.w = w; p.wp = wp; p.N = N; p.Cc = Cc; p.KK = KK; p.ntaps = a.ntaps; p.Kp = a.Kp; p.mode = mode; p.Ci = Ci;
    p.layout = WPREP_TC; p.p0 = a.cpad;
    for (int t = 0; t < a.ntaps; ++t) p.tap_index[t] = tap_index[t];
    const float* wpp = nullptr;
    int rc = wprep_get(p, st, &wpp);
    if (rc) return rc;
    a.Ntot = N;
    a.splits = splits;
    a.ktiles = a.Kp / (TC_KC * 4);
    a.kt_per_split = cdiv(a.ktiles, splits);
    a.partial = partial;
    int nt, smem;
    tc_geometry(N, nt, a.b_tile_bytes, a.depth, smem);
    rc = tc_weight_map(&a.wmap, wpp, N, a.Kp, nt);
    if (rc) return rc;
    a.tiles_m = cdiv(a.M, TC_M);
    a.tiles_n = cdiv(N, TC_NMAX);
    a.units = a.tiles_m * a.tiles_n * splits;
    return tc_launch_kernel(TC_FPROP_KERNELS, a, nt, tc_persistent_grid(a.units), smem, st, "conv_tc");
}

// ================================================================================================
// WGRAD on the tensor cores:  D[m=(tap,ci)][n=co] = sum_{k=pixel} X_im2col[m][k] * dY[n][k]
// Rows m are (tap, ci) with ci padded to cpad (rows ci >= Ci are zero), k runs over the B*Ho*Wo output pixels in
// k-tiles of 32.  Both operands are K(=pixel)-contiguous in NCHW, so the producers copy along K: 32 consecutive pixels
// of one row per warp instruction.  Split-K over pixel ranges with a deterministic two-stage reduce.
struct TcWgradArgs {
    const float* x;      // [B,Ci,Hi,Wi]
    const float* dy;     // [B,Co,Ho,Wo]
    float* out;          // dw [Co,Ci,kh,kw]  or  work[splits][Co*Ci*kh*kw]
    int B, Ci, Hi, Wi, Co, Ho, Wo, kh, kw, stride, pad;
    int cpad, Mtot;      // channels padded to 4; Mtot = kh*kw*cpad rows
    int P;               // B*Ho*Wo pixels (Wo % 4 == 0)
    int ktiles, kt_per_split, splits;  // k-tiles of 32 pixels (P / 32 rounded up), split-K over them
    int tiles_m, tiles_n, units;       // work units: 128-row tile (fastest) x channel tile x split, units = product
    int depth, b_tile_bytes;           // stage ring (tc_geometry)
};

// What the wgrad kernel's consumers do to a full stage's B operand (tc_consume_rs): dy, copied raw into the stage's
// second A slot, is split into tf32 hi / lo in the B slots, float4 q at float4 q (the raw copy is already in the
// swizzled K-major layout); consumer thread ct splits float4s ct, ct + 256, ...: a warp's 32 consecutive float4s are
// conflict free.
template <int NT>
struct TcWgradFeed {
    static constexpr bool split_b = true;
    int ct;                                                  // consumer thread, 0 .. 255
    __device__ __forceinline__ void prep_b(const TcTiles<unsigned char*>& t) const {
        constexpr int n4 = NT * TC_KC, nthr = 32 * TC_CONSUMER_WARPS;      // float4s of one B copy: 128 .. 1024
#pragma unroll
        for (int i = 0; i < (n4 + nthr - 1) / nthr; ++i) {
            const int q = ct + nthr * i;
            if (n4 % nthr == 0 || q < n4) tc_split_store(t.b_hi, t.b_lo, q, ((const float4*)t.a_lo)[q]);
        }
    }
};

// Persistent, as conv_tc_kernel: a CTA runs units blockIdx.x, blockIdx.x + gridDim.x, ..., its g-th k-tile in stage
// g % depth, and its producers gather the way that kernel's do: zero-filling cp.async straight into the stage, full[s]
// counting each thread's arrival once its copies have landed, never a wait for its own copies, so up to `depth`
// stages of loads are in flight.  A stage holds the raw im2col tile in its first A slot (layout TcAWgrad, read by
// tc_consume_rs as in fprop), the raw dy tile [NT rows][32 pixels] in its second A slot (float4 tile_idx(n, chunk),
// NT x 128 B <= 16 KB), and dy split into tf32 hi / lo in its B slots, in the swizzled K-major layout wgmma reads B
// in.  The consumers split dy (TcWgradFeed) when they take a stage: below N = 128 while the previous stage's MMAs run.
// A producer that had to split dy itself could publish a stage only between its waits for free stages, which would
// put a consumer -> producer -> consumer round trip into the path of every stage.
template <int NT>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_wgrad_kernel(const TcWgradArgs a) {
    const TcRing ring = tc_ring(a.depth, a.b_tile_bytes, TC_PRODUCERS);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int HWo = a.Ho * a.Wo, HWi = a.Hi * a.Wi;

    if (warp < TC_PRODUCERS / 32) {
        // ===================== producers =====================
        wg_regs_dec<TC_PRODUCER_REGS>();
        // A: warp w copies rows 32 w + i (i < 32) of the tile, lane = pixel of the k-tile.  dy: the thread copies 16-byte
        // chunk c = tid % 8 (pixels 4 c .. 4 c + 3 of the k-tile) of rows n = tid / 8 + 16 j, j < NT / 16; n % 8 does not
        // depend on j, so chunk j is float4 tile_idx(tid / 8, c) + 128 j of the raw tile.
        const int c = tid & 7, n_lo = tid >> 3, dy_idx = tile_idx(n_lo, c);
        // the warp's row-group table for the current unit, in the shared memory past the stage barriers: tc_geometry
        // keeps 2 KB there for the barriers and the 1 KB alignment, and the table fits beside both
        static_assert(1023 + 2 * TC_MAX_STAGES * 8 + TC_PRODUCERS / 32 * 8 * 8 <= 2048, "row-group table past the ring");
        int2* const gtab = (int2*)(ring.empty + TC_MAX_STAGES) + 8 * warp;
        int g = 0;                                   // k-tiles this CTA has copied
        for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
            const TcUnit w = tc_unit(a, u);
            const int ntile = min(TC_NMAX, a.Co - w.n0);
            // the warp's 8 row groups q, rows 32 w + 4 q .. + 3: one tap (ky, kx), channels ci .. ci + 3 (cpad % 4 == 0).
            // gtab[q] = {ci * HWi + ky * Wi + kx: the x offset of the group's first row from its pixel's window corner,
            // ky | kx << 8 | nv << 16: nv = the rows of the group that exist (ci + e < Ci and m < Mtot)}, by lane q
            __syncwarp();                            // the previous unit's entries have been read
            if (lane < 8) {
                const int m = w.m0 + 32 * warp + 4 * lane;
                const int tap = m / a.cpad, ci = m - tap * a.cpad, ky = tap / a.kw, kx = tap - ky * a.kw;
                const int nv = m < a.Mtot ? max(0, min(4, a.Ci - ci)) : 0;
                gtab[lane] = make_int2(ci * HWi + ky * a.Wi + kx, ky | kx << 8 | nv << 16);
            }
            __syncwarp();
            // this lane's pixel p = (b, oy, ox), the k-tile's first pixel + lane, advanced by 32 pixels per k-tile
            int p = w.kt_beg * (TC_KC * 4) + lane;
            int b = p / HWo, oy = (p - b * HWo) / a.Wo, ox = p - b * HWo - oy * a.Wo;
            const float* dyn = a.dy + (long long)(w.n0 + n_lo) * HWo;     // row n0 + tid / 8 of image 0
            for (int it = 0; it < w.nkt; ++it, ++g) {
                const int s = g % ring.depth;
                const TcTiles<unsigned char*> t = ring.acquire(g, s);
                // ---- A: the group's rows share the pixel's bounds check; a copy without a value is zero-filled from xb
                const bool pvalid = p < a.P;
                const int iy0 = oy * a.stride - a.pad, ix0 = ox * a.stride - a.pad, pix = iy0 * a.Wi + ix0;
                const float* xb = a.x + (pvalid ? (long long)b * a.Ci * HWi : 0ll);
                asm("" : "+l"(xb));      // one 64-bit base: each copy's address is then one wide multiply-add
                // row i of the warp is byte TcAWgrad::idx(32 w + i, lane) * 4 = ab[i % 8] + 128 i of the tile: the swizzle
                // flips bits 4-6 of the row's lane offset, and 128 i reaches only bits 7 and up
                uint32_t ab[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) ab[k] = (smem_u32(t.a_hi) + 4096 * warp + 4 * lane) ^ (16 * k);
                int2 gh[4];                          // the table, 4 groups at a time: each copy is a compiler barrier
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    if (q % 4 == 0) {
#pragma unroll
                        for (int i = 0; i < 4; ++i) gh[i] = gtab[q + i];
                    }
                    const int2 gq = gh[q % 4];
                    const int ky = gq.y & 0xff, kx = (gq.y >> 8) & 0xff, nv = gq.y >> 16;
                    const bool ok = pvalid && (unsigned)(iy0 + ky) < (unsigned)a.Hi && (unsigned)(ix0 + kx) < (unsigned)a.Wi;
                    const int o = pix + gq.x;
                    if (nv == 4) {                   // the warp's usual case (uniform): the 4 rows are channel planes apart
                        const float* src = xb + (ok ? o : 0);
                        const int step = ok ? HWi : 0;
#pragma unroll
                        for (int e = 0; e < 4; ++e)
                            cp_async_4(ab[(4 * q + e) % 8] + 128 * (4 * q + e), src + e * step, ok);
                    } else {
                        const int n = ok ? nv : 0;
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const bool v = e < n;
                            cp_async_4(ab[(4 * q + e) % 8] + 128 * (4 * q + e), xb + (v ? o + e * HWi : 0), v);
                        }
                    }
                }
                // ---- dy: chunk c's 4 pixels lie in one output row (Wo % 4 == 0); lane 4 c holds the first of them
                const int p0 = p - lane;                                   // the k-tile's first pixel
                const int bc = __shfl_sync(0xffffffffu, b, 4 * c), remc = __shfl_sync(0xffffffffu, oy * a.Wo + ox, 4 * c);
                const bool cvalid = p0 + 4 * c < a.P;
                const float* dyc = dyn + (long long)bc * a.Co * HWo + remc;
                const uint32_t bt = smem_u32(t.a_lo) + 16 * dy_idx;
#pragma unroll
                for (int j = 0; j < NT / 16; ++j) {
                    const bool v = cvalid && n_lo + 16 * j < ntile;
                    cp_async_16(bt + 2048 * j, v ? dyc + (long long)(16 * j) * HWo : a.dy, v);
                }
                p += TC_KC * 4;
                for (ox += TC_KC * 4; ox >= a.Wo; ox -= a.Wo)
                    if (++oy == a.Ho) { oy = 0; ++b; }
                cp_async_arrive(&ring.full[s]);
            }
        }
        cp_async_wait_all();      // no thread leaves copies in flight behind it
    } else {
        // ===================== consumers: MMA + epilogue; row m = (tap, ci), column = co =====================
        wg_regs_inc<TC_CONSUMER_REGS>();
        const int wg = (warp - TC_PRODUCERS / 32) >> 2, wq = warp & 3;
        const int KK = a.kh * a.kw;
        const TcWgradFeed<NT> feed = {tid - TC_PRODUCERS};
        int g = 0;                                   // k-tiles this CTA has consumed
        for (int u = blockIdx.x; u < a.units; u += gridDim.x) {
            const TcUnit w = tc_unit(a, u);
            const int ntile = min(TC_NMAX, a.Co - w.n0);
            float acc[NT / 2];
            tc_consume_rs<NT, TcAWgrad>(ring, g, w.nkt, wg, wq, lane, feed, acc);
            g += w.nkt;
            float* outp = a.out + (long long)w.z * a.Co * a.Ci * KK;
#pragma unroll
            for (int half = 0; half < 2; ++half) {
                const int em = w.m0 + tc_acc_row(wg, wq, lane, half);
                if (em >= a.Mtot) continue;
                const int etap = em / a.cpad;
                const int eci = em - etap * a.cpad;
                if (eci >= a.Ci) continue;
#pragma unroll
                for (int i = 0; i < NT / 8; ++i)
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int nl = tc_acc_col(lane, i, e);
                        if (nl < ntile) outp[((long long)(w.n0 + nl) * a.Ci + eci) * KK + etap] = acc[tc_acc_reg(i, half, e)];
                    }
            }
        }
    }
}

static void (*const TC_WGRAD_KERNELS[4])(const TcWgradArgs) = {conv_tc_wgrad_kernel<16>, conv_tc_wgrad_kernel<32>,
                                                                conv_tc_wgrad_kernel<64>, conv_tc_wgrad_kernel<128>};

// Shapes the kernels can express, and those where they pay off (CCB_CONV_IMPL_AUTO)
bool tc_supported(const ccb_conv_desc* d, int op) {
    if (d->kh != d->kw || d->kh * d->kw > TC_MAX_TAPS) return false;
    if (op == CCB_CONV_WGRAD) return (d->Wo % 4 == 0);      // 16-byte pixel chunks must not straddle rows
    return true;
}
bool tc_profitable(const ccb_conv_desc* d, int op) {
    if (!tc_supported(d, op)) return false;
    const long long M = (op == CCB_CONV_FPROP) ? (long long)d->B * d->Ho * d->Wo : (long long)d->B * d->Hi * d->Wi;
    const long long wsize = (long long)d->Ci * d->Co * d->kh * d->kw;
    // tiny feature maps (2x7, 4x13 ...) under a large weight matrix are split-K problems: one M tile, many k-tiles
    return (M >= 128 && wsize >= 64) || (M >= 8 && wsize >= 65536);
}

// Split-K count of a tensor-core call, and the prepared weights (tf32 hi + lo copies) a fprop / dgrad keeps at the start of
// its workspace, in floats.  fprop / dgrad: enough CTAs for ~2 waves, >= 2 k-tiles per split, <= 32 splits; the data
// gradient plans once for all its parity classes (they share the partials, each writes its own pixels), sized by the
// class with the most taps.  wgrad: ~2 waves of (tap, channel) x Co tiles, >= 4 k-tiles of 32 pixels per split.
int tc_plan(const ccb_conv_desc* d, int op, long long& panel_floats) {
    panel_floats = 0;
    if (op == CCB_CONV_WGRAD) {
        const int ktiles = cdiv(d->B * d->Ho * d->Wo, 32);
        const int tiles = cdiv(d->kh * d->kw * roundup(d->Ci, 4), TC_M) * cdiv(d->Co, TC_NMAX);
        int splits = cdiv(2 * NUM_SMS, tiles);
        if (splits > ktiles / 4) splits = ktiles / 4;
        if (splits > 2 * NUM_SMS) splits = 2 * NUM_SMS;
        if (splits < 1) splits = 1;
        return cdiv(ktiles, cdiv(ktiles, splits));          // no empty split
    }
    const bool fp = op == CCB_CONV_FPROP;
    const int s = fp ? 1 : d->stride, N = fp ? d->Co : d->Ci;
    const int Kp = tc_kp(cdiv(d->kh, s) * cdiv(d->kw, s), fp ? d->Ci : d->Co);
    panel_floats = 2ll * N * Kp;
    const long long M = fp ? (long long)d->B * d->Ho * d->Wo : (long long)d->B * cdiv(d->Hi, s) * cdiv(d->Wi, s);
    const long long tiles = (long long)cdiv((int)M, TC_M) * cdiv(N, TC_NMAX);
    const int ktiles = Kp / (TC_KC * 4);
    if (tiles >= NUM_SMS || ktiles < 4) return 1;
    long long splits = (2 * NUM_SMS + tiles - 1) / tiles;
    if (splits > ktiles / 2) splits = ktiles / 2;
    if (splits > 32) splits = 32;
    return splits < 2 ? 1 : (int)splits;
}

// y = act(conv(x, w) + bias + res): weights prepared into `wp`, split-K partials in `partial`
int tc_fprop(const ccb_conv_desc* d, const float* x, const float* w, const float* bias, const float* res, float* y,
             float* wp, float* partial, int splits, cudaStream_t st) {
    TcArgs a;
    memset(&a, 0, sizeof(a));
    a.x = x; a.bias = bias; a.res = res; a.out = y;
    a.B = d->B; a.Cin = d->Ci; a.Hin = d->Hi; a.Win = d->Wi;
    a.Hout = d->Ho; a.Wout = d->Wo; a.Hc = d->Ho; a.Wc = d->Wo;
    a.out_stride = 1; a.out_oy = 0; a.out_ox = 0; a.in_stride = d->stride;
    a.ntaps = d->kh * d->kw;
    a.M = d->B * d->Ho * d->Wo;
    a.act = d->act; a.slope = d->slope;
    signed char tix[TC_MAX_TAPS];
    for (int ky = 0; ky < d->kh; ++ky)
        for (int kx = 0; kx < d->kw; ++kx) {
            int t = ky * d->kw + kx;
            a.off_y[t] = (signed char)(ky - d->pad);
            a.off_x[t] = (signed char)(kx - d->pad);
            tix[t] = (signed char)t;
        }
    a.out_numel = (long long)d->B * d->Co * d->Ho * d->Wo;
    int rc = launch_tc(a, w, 0, d->Co, d->Ci, d->kh * d->kw, d->Ci, tix, wp, partial, splits, st);
    if (rc || splits == 1) return rc;
    launch_splitk_reduce(partial, y, bias, res, a.out_numel, splits, d->Ho * d->Wo, d->Co, d->act, d->slope, st);
    return check_launch("conv_tc splitk reduce");
}

// dx[b,ci,iy,ix] = sum_{co,ky,kx} dy[b,co,(iy+p-ky)/s,(ix+p-kx)/s] w[co,ci,ky,kx]   (one launch per parity class; every
// class prepares its own weights into `wp`, all share the split-K partials in `partial`)
int tc_dgrad(const ccb_conv_desc* d, const float* dy, const float* w, const float* bias, const float* res, float* dx,
             float* wp, float* partial, int splits, cudaStream_t st) {
    const int s = d->stride;
    const long long out_numel = (long long)d->B * d->Ci * d->Hi * d->Wi;
    for (int py = 0; py < s && py < d->Hi; ++py)
        for (int px = 0; px < s && px < d->Wi; ++px) {
            const DgradClass k = dgrad_class(d, py, px);
            TcArgs a;
            memset(&a, 0, sizeof(a));
            a.out_numel = out_numel;
            a.x = dy; a.bias = bias; a.res = res; a.out = dx;
            a.B = d->B; a.Cin = d->Co; a.Hin = d->Ho; a.Win = d->Wo;
            a.Hout = d->Hi; a.Wout = d->Wi;
            a.Hc = k.Hc; a.Wc = k.Wc;
            a.out_stride = s; a.out_oy = py; a.out_ox = px; a.in_stride = 1;
            a.M = d->B * a.Hc * a.Wc;
            a.act = d->act; a.slope = d->slope;
            a.ntaps = k.nky * k.nkx;
            signed char tix[TC_MAX_TAPS];
            for (int ty = 0; ty < k.nky; ++ty)
                for (int tx = 0; tx < k.nkx; ++tx) {
                    const int ky = k.ky0 + ty * s, kx = k.kx0 + tx * s, t = ty * k.nkx + tx;
                    // oy = (iy + p - ky)/s = jy + (py + p - ky)/s   (exact division, may be negative)
                    a.off_y[t] = (signed char)((py + d->pad - ky) / s);
                    a.off_x[t] = (signed char)((px + d->pad - kx) / s);
                    tix[t] = (signed char)(ky * d->kw + kx);
                }
            int rc = launch_tc(a, w, 1, d->Ci, d->Co, d->kh * d->kw, d->Ci, tix, wp, partial, splits, st);
            if (rc) return rc;
        }
    if (splits > 1) {
        launch_splitk_reduce(partial, dx, bias, res, out_numel, splits, d->Hi * d->Wi, d->Ci, d->act, d->slope, st);
        return check_launch("conv_tc dgrad splitk reduce");
    }
    return CCB_OK;
}

// dw; split-K partials in `partial`
int tc_wgrad(const ccb_conv_desc* d, const float* x, const float* dy, float* dw, float* partial, int splits, cudaStream_t st) {
    TcWgradArgs a;
    memset(&a, 0, sizeof(a));
    a.x = x; a.dy = dy;
    a.B = d->B; a.Ci = d->Ci; a.Hi = d->Hi; a.Wi = d->Wi; a.Co = d->Co; a.Ho = d->Ho; a.Wo = d->Wo;
    a.kh = d->kh; a.kw = d->kw; a.stride = d->stride; a.pad = d->pad;
    a.cpad = roundup(d->Ci, 4);
    a.Mtot = d->kh * d->kw * a.cpad;
    a.P = d->B * d->Ho * d->Wo;
    a.ktiles = cdiv(a.P, 32);
    a.kt_per_split = cdiv(a.ktiles, splits);
    a.splits = splits;
    a.out = splits > 1 ? partial : dw;
    const long long numel = (long long)d->Co * d->Ci * d->kh * d->kw;
    int nt, wsmem;
    tc_geometry(d->Co, nt, a.b_tile_bytes, a.depth, wsmem);
    a.tiles_m = cdiv(a.Mtot, TC_M);
    a.tiles_n = cdiv(d->Co, TC_NMAX);
    a.units = a.tiles_m * a.tiles_n * splits;
    int rc = tc_launch_kernel(TC_WGRAD_KERNELS, a, nt, tc_persistent_grid(a.units), wsmem, st, "conv_tc_wgrad");
    if (rc || a.splits == 1) return rc;
    launch_splitk_reduce(partial, dw, nullptr, nullptr, numel, splits, 1, 1, CCB_ACT_NONE, 0.f, st);
    return check_launch("conv_tc_wgrad_reduce");
}

}  // namespace ccb

// host-side tile geometry of a launch with N output channels (no launch, no GPU needed):
// out4 = {wgmma N, bytes of one B operand copy, pipeline stages, dynamic shared memory bytes}
extern "C" int ccb_debug_tc_plan(int N, int* out4) {
    if (N < 1 || !out4) return CCB_ERR_ARG;
    ccb::tc_geometry(N, out4[0], out4[1], out4[2], out4[3]);
    return CCB_OK;
}

#else   // CCB_CPU_SIM: no tensor cores in the CPU execution-model simulator

namespace ccb {
bool tc_supported(const ccb_conv_desc*, int) { return false; }
bool tc_profitable(const ccb_conv_desc*, int) { return false; }
int tc_plan(const ccb_conv_desc*, int, long long& panel_floats) { panel_floats = 0; return 1; }
int tc_fprop(const ccb_conv_desc*, const float*, const float*, const float*, const float*, float*, float*, float*, int,
             cudaStream_t) { return CCB_ERR_UNSUPPORTED; }
int tc_dgrad(const ccb_conv_desc*, const float*, const float*, const float*, const float*, float*, float*, float*, int,
             cudaStream_t) { return CCB_ERR_UNSUPPORTED; }
int tc_wgrad(const ccb_conv_desc*, const float*, const float*, float*, float*, int, cudaStream_t) { return CCB_ERR_UNSUPPORTED; }
}  // namespace ccb

extern "C" int ccb_debug_tc_plan(int, int*) { return CCB_ERR_UNSUPPORTED; }

#endif
