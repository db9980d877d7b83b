// conv_tc.cu - implicit-GEMM convolution on the Hopper tensor cores (wgmma), sm_90a.
//
//   D[128 pixels x N<=128 channels] (fp32, registers) += A[128 x 32] (im2col tile) * B[N x 32]^T (weights)
//
// * one CTA = one 128-pixel x N-channel output tile; one producer warpgroup + two consumer warpgroups, each
//   consumer owning 64 of the 128 rows (wgmma m64nNk8, N = the launch's channel tile rounded up to 16/32/64/128);
// * A is gathered straight from the NCHW activations (no im2col buffer in HBM): a K-chunk is 4
//   consecutive input channels of one filter tap, so the 4 loads of a chunk share the tap's bounds
//   check and are coalesced across the 128 pixels of the tile;
// * operands are staged in shared memory K-major with the 128-byte swizzle ([row][128 B], 16 B chunk ^= row & 7,
//   8-row atoms 1 KB apart): the layout wgmma reads for tf32, which it accepts only K-major;
// * fp32 parity: every fp32 operand is split hi = tf32(x), lo = x - hi and each k-step issues three
//   tf32 MMAs (hi*hi + lo*hi + hi*lo) ("3xTF32", error ~2^-21).  The tensor core only sums one 32-deep stage (small
//   cross terms first, then hi*hi) into a scratch register set; the stage's sum is added to the real accumulator with
//   fp32 adds, so no long accumulation chain runs through the tensor core's own rounding;
//   CCB_CONV_IMPL_TC_TF32 issues hi*hi only (what cuDNN does by default for the reference on Ampere+);
// * mbarrier pipeline of up to 4 stages: producers -> full[s] -> consumers (wgmma, commit group, wait, fp32 add)
//   -> empty[s];
//   the epilogue adds bias / residual, applies the activation and stores NCHW straight from the accumulators.
//
// The same kernel serves FPROP, stride-1 DGRAD and the stride-parity classes of strided DGRAD /
// ConvTranspose2d forward through a per-tap offset table ("generalised fprop").
#include "ccb_common.cuh"

#ifndef CCB_CPU_SIM

namespace ccb {

constexpr int TC_M = 128;          // pixels per tile (two wgmma M = 64 halves)
constexpr int TC_NMAX = 128;       // channels per tile
constexpr int TC_KC = 8;           // 16-byte k-chunks per stage (K = 32 fp32 per stage)
constexpr int TC_MAX_STAGES = 4;
constexpr int TC_PRODUCERS = 128;
constexpr int TC_CONSUMER_WARPS = 8;
constexpr int TC_THREADS = TC_PRODUCERS + 32 * TC_CONSUMER_WARPS;
constexpr int TC_MAX_TAPS = 49;

struct TcArgs {
    const float* x;        // input activations [B, Cin, Hin, Win]
    const float* wp;       // prepared weights: tf32 hi copy [N][Kp] followed by the lo copy [N][Kp] (k = tap*cpad + c)
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
    int splits, kt_per_split;          // split-K over k-tiles (grid.z); partials go to `partial`
    float* partial;                    // [splits][numel(out)] raw accumulators (bias/res/act applied by the reduce kernel)
    long long out_numel;
    int stages, b_tile_bytes;          // pipeline depth and bytes of one B operand copy (N-tile dependent)
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
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
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

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, tf32 in, fp32 accumulators in registers (N / 2 per thread)
__device__ __forceinline__ void wgmma_tf32_n16(float (&d)[8], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, "
        "%8, %9, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db));
}
__device__ __forceinline__ void wgmma_tf32_n32(float (&d)[16], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db));
}
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db));
}
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t da, uint64_t db) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        " %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
        " %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db));
}
template <int NT>
__device__ __forceinline__ void wgmma_tf32(float (&d)[NT / 2], uint64_t da, uint64_t db) {
    if constexpr (NT == 16) wgmma_tf32_n16(d, da, db);
    else if constexpr (NT == 32) wgmma_tf32_n32(d, da, db);
    else if constexpr (NT == 64) wgmma_tf32_n64(d, da, db);
    else wgmma_tf32_n128(d, da, db);
}

// float4 index of (row, 16-byte chunk) inside one swizzled operand tile
__device__ __forceinline__ int tile_idx(int row, int chunk) { return row * TC_KC + (chunk ^ (row & 7)); }

__device__ __forceinline__ float tc_act(float v, int act, float slope) {
    switch (act) {
        case CCB_ACT_RELU: return fmaxf(v, 0.f);
        case CCB_ACT_LEAKY: return v > 0.f ? v : v * slope;
        case CCB_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
        default: return v;
    }
}

constexpr int TC_TILE_BYTES = TC_KC * TC_M * 16;                   // one A operand copy of one stage: 16 KB
constexpr int TC_SMEM_MAX = 227 * 1024;

// Consumer side shared by both kernels: for each full stage, 4 k-steps of [(lo*hi) + (hi*lo) +] (hi*hi) on this
// warpgroup's 64 rows into the scratch registers `part`, then acc += part in fp32 and the stage goes back to the producers.
template <bool THREE, int NT>
__device__ __forceinline__ void tc_consume(unsigned char* smem, int stage_bytes, int b_tile_bytes, int NST, int nst,
                                           uint64_t* full_bar, uint64_t* empty_bar, int wg, int lane,
                                           float (&acc)[NT / 2], float (&part)[NT / 2]) {
    for (int it = 0; it < nst; ++it) {
        const int s = it % NST;
        mbar_wait(&full_bar[s], (it / NST) & 1);
        const uint32_t base = smem_u32(smem + s * stage_bytes);
        const uint32_t a_hi = base + wg * (TC_TILE_BYTES / 2), a_lo = a_hi + TC_TILE_BYTES;
        const uint32_t b_hi = base + 2 * TC_TILE_BYTES, b_lo = b_hi + b_tile_bytes;
#pragma unroll
        for (int j = 0; j < NT / 2; ++j) part[j] = 0.f;
        wg_fence();
        if (THREE) {
#pragma unroll
            for (int ks = 0; ks < TC_KC / 2; ++ks) {
                const uint32_t koff = (uint32_t)ks * 32u;
                wgmma_tf32<NT>(part, wg_desc(a_lo + koff), wg_desc(b_hi + koff));
                wgmma_tf32<NT>(part, wg_desc(a_hi + koff), wg_desc(b_lo + koff));
            }
        }
#pragma unroll
        for (int ks = 0; ks < TC_KC / 2; ++ks) {
            const uint32_t koff = (uint32_t)ks * 32u;
            wgmma_tf32<NT>(part, wg_desc(a_hi + koff), wg_desc(b_hi + koff));
        }
        wg_commit();
        wg_wait<0>();
        wg_fence_regs(part);
        if (lane == 0) mbar_arrive(&empty_bar[s]);
#pragma unroll
        for (int j = 0; j < NT / 2; ++j) acc[j] += part[j];
    }
}

template <bool THREE, int NT>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const TcArgs a) {
    CCB_PDL_TRIGGER();
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // SWIZZLE_128B atoms are 1 KB
    const int NST = a.stages;
    const int stage_bytes = 2 * TC_TILE_BYTES + 2 * a.b_tile_bytes;     // A hi, A lo, B hi, B lo
    uint64_t* full_bar = (uint64_t*)(smem + NST * stage_bytes);
    uint64_t* empty_bar = full_bar + TC_MAX_STAGES;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.x * TC_M, n0 = blockIdx.y * TC_NMAX;
    const int ntile = min(TC_NMAX, a.Ntot - n0);
    const int ktiles_all = a.Kp / (TC_KC * 4);
    const int kt_beg = blockIdx.z * a.kt_per_split;
    const int ktiles = max(0, min(ktiles_all, kt_beg + a.kt_per_split) - kt_beg);   // k-tiles of this split
    const long long HWin = (long long)a.Hin * a.Win;

    if (tid == 0) {
        for (int s = 0; s < NST; ++s) { mbar_init(&full_bar[s], TC_PRODUCERS); mbar_init(&empty_bar[s], TC_CONSUMER_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();
    CCB_PDL_SYNC();                                               // everything above touched no global data

    if (warp < TC_PRODUCERS / 32) {
        // ===================== producers: thread == tile row =====================
        const int r = tid;
        const int m = m0 + r;
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
        const int cpt = a.cpad >> 2;                 // chunks per tap
        const int nchunks = a.ntaps * cpt;           // real chunks; the rest of Kp is zero padding
        for (int it = 0; it < ktiles; ++it) {
            const int s = it % NST;
            const int kt = kt_beg + it;                   // global k-tile
            // ---- A: the 8 chunks (32 floats) of this thread's pixel row
            float av[TC_KC][4];
            const int q0 = kt * TC_KC;
            const int tap0 = q0 / cpt, c40 = q0 - tap0 * cpt;
            if (c40 + TC_KC <= cpt) {
                // fast path (C_in % 32 == 0 layers): the whole stage reads one filter tap -> one bounds check,
                // one base pointer, 32 loads that differ only by the channel-plane stride
                bool ok = mvalid && tap0 < a.ntaps;
                int pix = 0;
                if (ok) {
                    const int iy = iy0 + a.off_y[tap0], ix = ix0 + a.off_x[tap0];
                    ok = (iy >= 0) && (iy < a.Hin) && (ix >= 0) && (ix < a.Win);
                    pix = iy * a.Win + ix;
                }
                const float* p = xb + (long long)(c40 * 4) * HWin + pix;
                const int nv = ok ? (a.Cin - c40 * 4) : 0;
#pragma unroll
                for (int c = 0; c < TC_KC; ++c)
#pragma unroll
                    for (int j = 0; j < 4; ++j) av[c][j] = (c * 4 + j < nv) ? __ldg(p + (c * 4 + j) * HWin) : 0.f;
            } else {
                int q = q0, tap = tap0, c4 = c40;
#pragma unroll
                for (int c = 0; c < TC_KC; ++c) {
                    av[c][0] = av[c][1] = av[c][2] = av[c][3] = 0.f;
                    if (mvalid && q < nchunks) {
                        const int iy = iy0 + a.off_y[tap], ix = ix0 + a.off_x[tap];
                        if (iy >= 0 && iy < a.Hin && ix >= 0 && ix < a.Win) {
                            const float* p = xb + (long long)(c4 * 4) * HWin + (iy * a.Win + ix);
                            const int nv = a.Cin - c4 * 4;
#pragma unroll
                            for (int j = 0; j < 4; ++j)
                                if (j < nv) av[c][j] = __ldg(p + j * HWin);
                        }
                    }
                    ++q;
                    if (++c4 == cpt) { c4 = 0; ++tap; }
                }
            }
            if (it >= NST) mbar_wait(&empty_bar[s], ((it / NST) - 1) & 1);
            unsigned char* st = smem + s * stage_bytes;
            float4* a_hi = (float4*)st;
            float4* a_lo = (float4*)(st + TC_TILE_BYTES);
            float4* b_hi = (float4*)(st + 2 * TC_TILE_BYTES);
            float4* b_lo = (float4*)(st + 2 * TC_TILE_BYTES + a.b_tile_bytes);
            // ---- B: the weights were split into tf32 hi / lo by the prep kernel: plain 16-byte async copies
            //      (pairs of threads cover one 32-byte sector of a weight row)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int idx = r + j * 128;                      // 0 .. 1023
                const int c = ((idx >> 8) << 1) | (idx & 1);
                const int n = (idx >> 1) & 127;
                if (n < NT) {
                    // rows in [ntile, NT) are clamped to row 0: the epilogue ignores those columns
                    const int nn = (n < ntile) ? n : 0;
                    const float* src = a.wp + (long long)(n0 + nn) * a.Kp + kt * (TC_KC * 4) + c * 4;
                    cp_async16(&b_hi[tile_idx(n, c)], src);
                    if (THREE) cp_async16(&b_lo[tile_idx(n, c)], src + (long long)a.Ntot * a.Kp);
                }
            }
            // ---- A: split + store
#pragma unroll
            for (int c = 0; c < TC_KC; ++c) {
                float4 h, l;
                h.x = tf32_hi(av[c][0]); h.y = tf32_hi(av[c][1]); h.z = tf32_hi(av[c][2]); h.w = tf32_hi(av[c][3]);
                a_hi[tile_idx(r, c)] = h;
                if (THREE) {
                    l.x = tf32_hi(av[c][0] - h.x); l.y = tf32_hi(av[c][1] - h.y); l.z = tf32_hi(av[c][2] - h.z); l.w = tf32_hi(av[c][3] - h.w);
                    a_lo[tile_idx(r, c)] = l;
                }
            }
            cp_async_wait_all();
            fence_proxy_async();
            mbar_arrive(&full_bar[s]);
        }
    } else {
        // ===================== consumers: MMA + epilogue =====================
        const int wg = (warp - TC_PRODUCERS / 32) >> 2, wq = warp & 3;
        float acc[NT / 2], part[NT / 2];
#pragma unroll
        for (int j = 0; j < NT / 2; ++j) acc[j] = 0.f;                  // an empty split contributes zeros
        tc_consume<THREE, NT>(smem, stage_bytes, a.b_tile_bytes, NST, ktiles, full_bar, empty_bar, wg, lane, acc, part);
        const long long HWout = (long long)a.Hout * a.Wout;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            // accumulator layout of wgmma m64nN: row 16 * warp + lane / 4 (+ 8), columns 8 i + 2 (lane % 4) (+ 1)
            const int em = m0 + wg * 64 + wq * 16 + (lane >> 2) + half * 8;
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
                    const int nl = 8 * i + 2 * (lane & 3) + e;
                    if (nl < ntile) {
                        const int j = 4 * i + 2 * half + e;
                        float o = acc[j];
                        const int n = n0 + nl;
                        const long long off = obase + (long long)n * HWout;
                        if (a.splits > 1) {
                            a.partial[(long long)blockIdx.z * a.out_numel + off] = o;
                        } else {
                            if (a.bias) o += __ldg(a.bias + n);
                            if (a.res) o += __ldg(a.res + off);
                            a.out[off] = tc_act(o, a.act, a.slope);
                        }
                    }
                }
        }
    }
}

// Weight re-layout: wp[n][t*cpad + c] = w[(co,ci) by mode][tap(t)], zero padded to Kp.
//   mode 0 (fprop): n = co, c = ci : w[n][c][tap]        mode 1 (dgrad): n = ci, c = co : w[c][n][tap]
static int roundup(int v, int m) { return (v + m - 1) / m * m; }

void launch_splitk_reduce(const float* work, float* out, const float* bias, const float* res, long long numel, int splits,
                          int plane, int C, int act, float slope, cudaStream_t st);   // conv_ffma.cu

// Operand tile geometry of one launch: the B tile holds the wgmma N (16/32/64/128) rows, and as many stages as fit
// in shared memory (up to 4: 3 at N = 128 in 3xTF32 layout, 4 below).
static void tc_geometry(int N, int& nt, int& b_tile_bytes, int& stages, int& smem) {
    const int ntile_max = N < TC_NMAX ? N : TC_NMAX;
    nt = 16;
    while (nt < ntile_max) nt <<= 1;
    b_tile_bytes = nt * 128;
    const int stage = 2 * TC_TILE_BYTES + 2 * b_tile_bytes;
    stages = (TC_SMEM_MAX - 2048) / stage;
    if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
    smem = stages * stage + 2048;                     // + barriers / alignment slack
}

template <typename Args>
static int tc_launch_kernel(void (*const (&kfns)[2][4])(const Args), const Args& a, int three, int nt, dim3 grid, int smem,
                            cudaStream_t st, const char* what) {
    const int ni = nt == 16 ? 0 : nt == 32 ? 1 : nt == 64 ? 2 : 3;
    auto kfn = kfns[three ? 1 : 0][ni];
    cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_MAX);
    CCB_LAUNCH(kfn, grid, dim3(TC_THREADS), smem, st, a);
    return check_launch(what);
}

static void (*const TC_FPROP_KERNELS[2][4])(const TcArgs) = {
    {conv_tc_kernel<false, 16>, conv_tc_kernel<false, 32>, conv_tc_kernel<false, 64>, conv_tc_kernel<false, 128>},
    {conv_tc_kernel<true, 16>, conv_tc_kernel<true, 32>, conv_tc_kernel<true, 64>, conv_tc_kernel<true, 128>}};

// Split-K plan shared by all parity classes of one call: enough CTAs for ~2 waves, >= 2 k-tiles per split.
static int plan_splits(long long M, int N, int max_ktiles, long long out_numel, long long part_floats) {
    const long long tiles = (long long)cdiv((int)M, TC_M) * cdiv(N, TC_NMAX);
    if (tiles >= NUM_SMS || max_ktiles < 4) return 1;
    long long s = (2 * NUM_SMS + tiles - 1) / tiles;
    if (s > max_ktiles / 2) s = max_ktiles / 2;
    if (s > 32) s = 32;
    if (out_numel > 0 && s * out_numel > part_floats) s = part_floats / out_numel;
    return s < 2 ? 1 : (int)s;
}

// One generalised-fprop launch (+ its weight preparation).  `work` = [prepared weights | split-K partials].
static int launch_tc(TcArgs& a, const float* w, int mode, int N, int Cc, int KK, int Ci, const signed char* tap_index,
                     float* work, long long work_floats, int splits, float* partial, int three, cudaStream_t st) {
    a.cpad = roundup(Cc, 4);
    a.Kp = roundup(a.ntaps * a.cpad, TC_KC * 4);
    if (a.Kp == 0) a.Kp = TC_KC * 4;      // a parity class without taps still runs one all-zero k-tile
    const long long wp_floats = 2ll * N * a.Kp;                  // tf32 hi copy + lo copy
    CCB_REQUIRE(wp_floats + (splits > 1 ? (long long)splits * a.out_numel : 0) <= work_floats, CCB_ERR_ARG,
                "conv_tc: workspace too small (%lld floats)", work_floats);
    WPrepDesc p;
    memset(&p, 0, sizeof(p));
    p.w = w; p.wp = work; p.N = N; p.Cc = Cc; p.KK = KK; p.ntaps = a.ntaps; p.Kp = a.Kp; p.mode = mode; p.Ci = Ci;
    p.layout = WPREP_TC; p.p0 = a.cpad;
    for (int t = 0; t < a.ntaps; ++t) p.tap_index[t] = tap_index[t];
    const float* wpp = nullptr;
    int rc = wprep_get(p, st, &wpp);
    if (rc) return rc;
    a.wp = wpp;
    a.Ntot = N;
    a.splits = splits;
    a.kt_per_split = cdiv(a.Kp / (TC_KC * 4), splits);
    a.partial = partial ? partial : work + wp_floats;
    int nt, smem;
    tc_geometry(N, nt, a.b_tile_bytes, a.stages, smem);
    dim3 grid(cdiv(a.M, TC_M), cdiv(N, TC_NMAX), splits);
    return tc_launch_kernel(TC_FPROP_KERNELS, a, three, nt, grid, smem, st, "conv_tc");
}

// ================================================================================================
// WGRAD on the tensor cores:  D[m=(tap,ci)][n=co] = sum_{k=pixel} X_im2col[m][k] * dY[n][k]
// Both operands are K(=pixel)-contiguous in NCHW, so producers walk along K: 8 consecutive threads
// load the 8 16-byte chunks (32 consecutive output pixels) of one row -> coalesced global loads, and
// with the SWIZZLE_128B operand layout their shared-memory stores are conflict-free.
// Split-K over pixel ranges (grid.z) with a deterministic two-stage reduce.
struct TcWgradArgs {
    const float* x;      // [B,Ci,Hi,Wi]
    const float* dy;     // [B,Co,Ho,Wo]
    float* out;          // dw [Co,Ci,kh,kw]  or  work[splits][Co*Ci*kh*kw]
    int B, Ci, Hi, Wi, Co, Ho, Wo, kh, kw, stride, pad;
    int cpad, Mtot;      // channels padded to 4; Mtot = kh*kw*cpad rows
    int P;               // B*Ho*Wo pixels (Wo % 4 == 0)
    int stages, per_split, splits;
    int nstages, b_tile_bytes;   // pipeline depth / bytes of one dY operand copy (Co-tile dependent)
};

template <bool THREE, int NT>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_wgrad_kernel(const TcWgradArgs a) {
    CCB_PDL_TRIGGER();
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int NST = a.nstages;
    const int stage_bytes = 2 * TC_TILE_BYTES + 2 * a.b_tile_bytes;
    uint64_t* full_bar = (uint64_t*)(smem + NST * stage_bytes);
    uint64_t* empty_bar = full_bar + TC_MAX_STAGES;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m0 = blockIdx.x * TC_M, n0 = blockIdx.y * TC_NMAX;
    const int ntile = min(TC_NMAX, a.Co - n0);
    const int st_beg = blockIdx.z * a.per_split, st_end = min(a.stages, st_beg + a.per_split);
    const int nst = st_end - st_beg;          // >= 1 by construction
    const int KK = a.kh * a.kw;
    const int HWo = a.Ho * a.Wo, HWi = a.Hi * a.Wi;

    if (tid == 0) {
        for (int s = 0; s < NST; ++s) { mbar_init(&full_bar[s], TC_PRODUCERS); mbar_init(&empty_bar[s], TC_CONSUMER_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();
    CCB_PDL_SYNC();                                               // everything above touched no global data

    if (warp < TC_PRODUCERS / 32) {
        // 8 consecutive threads walk the 8 K-chunks (32 consecutive pixels) of one row, rows rbase + 16 j
        const int c = tid & 7, rbase = tid >> 3;
        // per-row constants: x offset of the row's (ci, ky, kx) relative to the pixel base, and its tap shift
        int rowoff[8], dky[8], dkx[8];
        unsigned rvalid = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            int m = m0 + rbase + 16 * j;
            rowoff[j] = 0; dky[j] = dkx[j] = 0;
            if (m < a.Mtot) {
                int tap = m / a.cpad, ci = m - tap * a.cpad;
                if (ci < a.Ci) {
                    int ky = tap / a.kw, kx = tap - ky * a.kw;
                    dky[j] = ky - a.pad; dkx[j] = kx - a.pad;
                    rowoff[j] = ci * HWi + dky[j] * a.Wi + dkx[j];       // may be negative: only used where the tap is in bounds
                    rvalid |= 1u << j;
                }
            }
        }
        for (int it = 0; it < nst; ++it) {
            const int s = it % NST;
            const int p0 = ((st_beg + it) * TC_KC + c) * 4;       // first of this chunk's 4 pixels
            const bool pvalid = p0 < a.P;
            int b = 0, oy = 0, ox0 = 0;
            if (pvalid) {
                b = p0 / HWo;
                int rem = p0 - b * HWo;
                oy = rem / a.Wo;
                ox0 = rem - oy * a.Wo;
            }
            const float* xpix = a.x + (long long)b * a.Ci * HWi + (oy * a.stride) * a.Wi + ox0 * a.stride;
            const int iyb = oy * a.stride, ixb = ox0 * a.stride;
            float av[8][4];
            float4 bv[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                av[j][0] = av[j][1] = av[j][2] = av[j][3] = 0.f;
                const int iy = iyb + dky[j], ix0 = ixb + dkx[j];
                if (pvalid && ((rvalid >> j) & 1u) && iy >= 0 && iy < a.Hi) {
                    const float* px = xpix + rowoff[j];
                    if (ix0 >= 0 && ix0 + 3 * a.stride < a.Wi) {          // interior: no per-element checks
#pragma unroll
                        for (int e = 0; e < 4; ++e) av[j][e] = __ldg(px + e * a.stride);
                    } else {
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const int ix = ix0 + e * a.stride;
                            if (ix >= 0 && ix < a.Wi) av[j][e] = __ldg(px + e * a.stride);
                        }
                    }
                }
                bv[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                const int n = rbase + 16 * j;
                if (pvalid && n < ntile)
                    bv[j] = __ldg((const float4*)(a.dy + ((long long)b * a.Co + n0 + n) * HWo + oy * a.Wo + ox0));
            }
            if (it >= NST) mbar_wait(&empty_bar[s], ((it / NST) - 1) & 1);
            unsigned char* st = smem + s * stage_bytes;
            float4* a_hi = (float4*)st;
            float4* a_lo = (float4*)(st + TC_TILE_BYTES);
            float4* b_hi = (float4*)(st + 2 * TC_TILE_BYTES);
            float4* b_lo = (float4*)(st + 2 * TC_TILE_BYTES + a.b_tile_bytes);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int r = rbase + 16 * j;
                float4 h, l;
                h.x = tf32_hi(av[j][0]); h.y = tf32_hi(av[j][1]); h.z = tf32_hi(av[j][2]); h.w = tf32_hi(av[j][3]);
                a_hi[tile_idx(r, c)] = h;
                if (THREE) {
                    l.x = tf32_hi(av[j][0] - h.x); l.y = tf32_hi(av[j][1] - h.y); l.z = tf32_hi(av[j][2] - h.z); l.w = tf32_hi(av[j][3] - h.w);
                    a_lo[tile_idx(r, c)] = l;
                }
                if (r < NT) {
                    h.x = tf32_hi(bv[j].x); h.y = tf32_hi(bv[j].y); h.z = tf32_hi(bv[j].z); h.w = tf32_hi(bv[j].w);
                    b_hi[tile_idx(r, c)] = h;
                    if (THREE) {
                        l.x = tf32_hi(bv[j].x - h.x); l.y = tf32_hi(bv[j].y - h.y); l.z = tf32_hi(bv[j].z - h.z); l.w = tf32_hi(bv[j].w - h.w);
                        b_lo[tile_idx(r, c)] = l;
                    }
                }
            }
            fence_proxy_async();
            mbar_arrive(&full_bar[s]);
        }
    } else {
        // ---- consumers; epilogue: row m = (tap, ci); columns == co
        const int wg = (warp - TC_PRODUCERS / 32) >> 2, wq = warp & 3;
        float acc[NT / 2], part[NT / 2];
#pragma unroll
        for (int j = 0; j < NT / 2; ++j) acc[j] = 0.f;
        tc_consume<THREE, NT>(smem, stage_bytes, a.b_tile_bytes, NST, nst, full_bar, empty_bar, wg, lane, acc, part);
        float* outp = a.out + (long long)blockIdx.z * a.Co * a.Ci * KK;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int em = m0 + wg * 64 + wq * 16 + (lane >> 2) + half * 8;
            if (em >= a.Mtot) continue;
            const int etap = em / a.cpad;
            const int eci = em - etap * a.cpad;
            if (eci >= a.Ci) continue;
#pragma unroll
            for (int i = 0; i < NT / 8; ++i)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int nl = 8 * i + 2 * (lane & 3) + e;
                    const int j = 4 * i + 2 * half + e;
                    if (nl < ntile) outp[((long long)(n0 + nl) * a.Ci + eci) * KK + etap] = acc[j];
                }
        }
    }
}

static void (*const TC_WGRAD_KERNELS[2][4])(const TcWgradArgs) = {
    {conv_tc_wgrad_kernel<false, 16>, conv_tc_wgrad_kernel<false, 32>, conv_tc_wgrad_kernel<false, 64>, conv_tc_wgrad_kernel<false, 128>},
    {conv_tc_wgrad_kernel<true, 16>, conv_tc_wgrad_kernel<true, 32>, conv_tc_wgrad_kernel<true, 64>, conv_tc_wgrad_kernel<true, 128>}};

// out[i] = sum_s work[s][i]
__global__ void __launch_bounds__(256) tc_splitk_sum_kernel(const float* __restrict__ work, float* __restrict__ out,
                                                            long long numel, int splits) {
    CCB_PDL_WAIT();
    long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= numel) return;
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += __ldg(work + (long long)s * numel + i);
    out[i] = v;
}

// Shape gate: which problems take the tensor-core path under CCB_CONV_IMPL_AUTO
bool tc_supported(const ccb_conv_desc* d, int op) {
    if (d->kh != d->kw || d->kh * d->kw > TC_MAX_TAPS) return false;
    if (op == CCB_CONV_WGRAD) return (d->Wo % 4 == 0);      // 16-byte pixel chunks must not straddle rows
    return true;
}
bool tc_profitable(const ccb_conv_desc* d, int op) {
    if (!tc_supported(d, op)) return false;
    long long M = (op == CCB_CONV_FPROP) ? (long long)d->B * d->Ho * d->Wo : (long long)d->B * d->Hi * d->Wi;
    int N = (op == CCB_CONV_FPROP) ? d->Co : d->Ci;
    int Cc = (op == CCB_CONV_FPROP) ? d->Ci : d->Co;
    (void)N; (void)Cc;
    const long long wsize = (long long)d->Ci * d->Co * d->kh * d->kw;
    // tiny feature maps (2x7, 4x13 ...) under a large weight matrix are split-K problems: one M tile, many k-tiles
    return (M >= 128 && wsize >= 64) || (M >= 8 && wsize >= 65536);
}

static int wgrad_splits(const ccb_conv_desc* d, int& stages, int& per_split) {
    const int cpad = roundup(d->Ci, 4);
    const long long P = (long long)d->B * d->Ho * d->Wo;
    stages = (int)((P + 31) / 32);
    const int tiles = cdiv(d->kh * d->kw * cpad, TC_M) * cdiv(d->Co, TC_NMAX);
    int splits = cdiv(2 * NUM_SMS, tiles);
    if (splits > stages / 4) splits = stages / 4;
    if (splits > 2 * NUM_SMS) splits = 2 * NUM_SMS;
    if (splits < 1) splits = 1;
    per_split = cdiv(stages, splits);
    splits = cdiv(stages, per_split);          // no empty split
    return splits;
}

long long tc_workspace_floats(const ccb_conv_desc* d, int op) {
    if (op == CCB_CONV_WGRAD) {
        int stages, per;
        int splits = wgrad_splits(d, stages, per);
        return splits > 1 ? (long long)splits * d->Co * d->Ci * d->kh * d->kw : 0;
    }
    int N = (op == CCB_CONV_FPROP) ? d->Co : d->Ci;
    int Cc = (op == CCB_CONV_FPROP) ? d->Ci : d->Co;
    long long wpf = 2ll * N * roundup(d->kh * d->kw * roundup(Cc, 4), 32);
    long long out_numel = (op == CCB_CONV_FPROP) ? (long long)d->B * d->Co * d->Ho * d->Wo : (long long)d->B * d->Ci * d->Hi * d->Wi;
    long long M = (op == CCB_CONV_FPROP) ? (long long)d->B * d->Ho * d->Wo : (long long)d->B * d->Hi * d->Wi / (d->stride * d->stride);
    long long tiles = (long long)cdiv((int)M, TC_M) * cdiv(N, TC_NMAX);
    long long part = (tiles < NUM_SMS) ? 32 * out_numel : 0;       // room for up to 32 splits when the grid is small
    return wpf + part;
}

int tc_fprop(const ccb_conv_desc* d, const float* x, const float* w, const float* bias, const float* res, float* y,
             float* work, long long work_floats, int three, cudaStream_t st) {
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
    const int Kp = roundup(a.ntaps * roundup(d->Ci, 4), 32);
    const long long wpf = 2ll * d->Co * Kp;
    const int splits = plan_splits(a.M, d->Co, Kp / 32, a.out_numel, work_floats - wpf);
    int rc = launch_tc(a, w, 0, d->Co, d->Ci, d->kh * d->kw, d->Ci, tix, work, work_floats, splits, nullptr, three, st);
    if (rc || splits == 1) return rc;
    launch_splitk_reduce(a.partial, y, bias, res, a.out_numel, splits, d->Ho * d->Wo, d->Co, d->act, d->slope, st);
    return check_launch("conv_tc splitk reduce");
}

// dx[b,ci,iy,ix] = sum_{co,ky,kx} dy[b,co,(iy+p-ky)/s,(ix+p-kx)/s] w[co,ci,ky,kx]   (one launch per parity class)
int tc_dgrad(const ccb_conv_desc* d, const float* dy, const float* w, const float* bias, const float* res, float* dx,
             float* work, long long work_floats, int three, cudaStream_t st) {
    const int s = d->stride;
    // one split-K plan for every parity class (they share the partial buffers; each writes its own pixels)
    const long long out_numel = (long long)d->B * d->Ci * d->Hi * d->Wi;
    const int max_taps = cdiv(d->kh, s) * cdiv(d->kw, s);
    const int Kp_max = roundup(max_taps * roundup(d->Co, 4), 32);
    const long long wpf_max = 2ll * d->Ci * Kp_max;
    const long long Mclass = (long long)d->B * cdiv(d->Hi, s) * cdiv(d->Wi, s);
    const int splits = plan_splits(Mclass, d->Ci, Kp_max / 32, out_numel, work_floats - wpf_max);
    for (int py = 0; py < s && py < d->Hi; ++py)
        for (int px = 0; px < s && px < d->Wi; ++px) {
            TcArgs a;
            memset(&a, 0, sizeof(a));
            a.out_numel = out_numel;
            a.x = dy; a.bias = bias; a.res = res; a.out = dx;
            a.B = d->B; a.Cin = d->Co; a.Hin = d->Ho; a.Win = d->Wo;
            a.Hout = d->Hi; a.Wout = d->Wi;
            a.Hc = (d->Hi - py + s - 1) / s; a.Wc = (d->Wi - px + s - 1) / s;
            a.out_stride = s; a.out_oy = py; a.out_ox = px; a.in_stride = 1;
            a.M = d->B * a.Hc * a.Wc;
            a.act = d->act; a.slope = d->slope;
            signed char tix[TC_MAX_TAPS];
            int nt = 0;
            for (int ky = 0; ky < d->kh; ++ky) {
                if ((py + d->pad - ky) % s != 0) continue;
                for (int kx = 0; kx < d->kw; ++kx) {
                    if ((px + d->pad - kx) % s != 0) continue;
                    // oy = (iy + p - ky)/s = jy + (py + p - ky)/s   (exact division, may be negative)
                    a.off_y[nt] = (signed char)((py + d->pad - ky) / s);
                    a.off_x[nt] = (signed char)((px + d->pad - kx) / s);
                    tix[nt] = (signed char)(ky * d->kw + kx);
                    ++nt;
                }
            }
            a.ntaps = nt;
            // every class prepares its own weights at the start of `work`; partials live after the largest prep
            int rc = launch_tc(a, w, 1, d->Ci, d->Co, d->kh * d->kw, d->Ci, tix, work, wpf_max + (splits > 1 ? splits * out_numel : 0),
                               splits, work + wpf_max, three, st);
            if (rc) return rc;
        }
    if (splits > 1) {
        launch_splitk_reduce(work + wpf_max, dx, bias, res, out_numel, splits, d->Hi * d->Wi, d->Ci, d->act, d->slope, st);
        return check_launch("conv_tc dgrad splitk reduce");
    }
    return CCB_OK;
}

int tc_wgrad(const ccb_conv_desc* d, const float* x, const float* dy, float* dw, float* work, long long work_floats,
             int three, cudaStream_t st) {
    TcWgradArgs a;
    memset(&a, 0, sizeof(a));
    a.x = x; a.dy = dy;
    a.B = d->B; a.Ci = d->Ci; a.Hi = d->Hi; a.Wi = d->Wi; a.Co = d->Co; a.Ho = d->Ho; a.Wo = d->Wo;
    a.kh = d->kh; a.kw = d->kw; a.stride = d->stride; a.pad = d->pad;
    a.cpad = roundup(d->Ci, 4);
    a.Mtot = d->kh * d->kw * a.cpad;
    a.P = d->B * d->Ho * d->Wo;
    a.splits = wgrad_splits(d, a.stages, a.per_split);
    const long long numel = (long long)d->Co * d->Ci * d->kh * d->kw;
    if (a.splits > 1) {
        CCB_REQUIRE(work && (long long)a.splits * numel <= work_floats, CCB_ERR_ARG, "conv_tc wgrad: workspace too small");
        a.out = work;
    } else {
        a.out = dw;
    }
    int nt, wsmem;
    tc_geometry(d->Co, nt, a.b_tile_bytes, a.nstages, wsmem);
    dim3 grid(cdiv(a.Mtot, TC_M), cdiv(d->Co, TC_NMAX), a.splits);
    int rc = tc_launch_kernel(TC_WGRAD_KERNELS, a, three, nt, grid, wsmem, st, "conv_tc_wgrad");
    if (rc || a.splits == 1) return rc;
    CCB_LAUNCH(tc_splitk_sum_kernel, dim3((unsigned)((numel + 255) / 256)), dim3(256), 0, st, (const float*)work, dw, numel, a.splits);
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
long long tc_workspace_floats(const ccb_conv_desc*, int) { return 0; }
int tc_fprop(const ccb_conv_desc*, const float*, const float*, const float*, const float*, float*, float*, long long, int,
             cudaStream_t) { return CCB_ERR_UNSUPPORTED; }
int tc_dgrad(const ccb_conv_desc*, const float*, const float*, const float*, const float*, float*, float*, long long, int,
             cudaStream_t) { return CCB_ERR_UNSUPPORTED; }
int tc_wgrad(const ccb_conv_desc*, const float*, const float*, float*, float*, long long, int, cudaStream_t) {
    return CCB_ERR_UNSUPPORTED;
}
}  // namespace ccb

extern "C" int ccb_debug_tc_plan(int, int*) { return CCB_ERR_UNSUPPORTED; }

#endif
