// conv_ffma.cu - CUDA-core (FFMA) implicit-GEMM convolution: forward, data-gradient (also the
// ConvTranspose2d forward) and weight-gradient, with fused bias / residual / activation epilogues.
//
// Role: (a) exact-fp32 baseline and fallback for shapes the wgmma tensor-core path does not take (C_in = 3,
// C_out <= 4 heads, tiny deep levels), (b) numerical cross-check for the tensor-core kernels
// (conv_tc.cu).  Replaces the cuDNN calls behind nn.Conv2d / nn.ConvTranspose2d in
// models/{DispResNet6,PoseNetB6,MaskNet6,back2future}.py (SURVEY.md 2a K6/K7).
//
// GEMM views (NCHW fp32, weights [Co,Ci,kh,kw]):
//   FPROP : C[m=(b,oy,ox)][n=co]      = sum_k A[m][k=(ci,ky,kx)] * W[co][k]
//   DGRAD : C[m=(b,jy,jx)][n=ci]      = sum_k dy[b,co,oy,ox] * W[co][ci][ky][kx], one launch per
//           stride-parity class (py,px): only the taps that hit integer output coordinates are
//           enumerated, so stride-2 layers waste no MACs.  ConvTranspose2d forward == DGRAD.
//   WGRAD : C[m=(ci,ky,kx)][n=co]     = sum_k=(b,oy,ox) x[...] * dy[b,co,oy,ox], split-K.
#include "conv.cuh"

namespace ccb {

enum { MODE_FPROP = 0, MODE_DGRAD = 1, MODE_WGRAD = 2 };

struct ConvArgs {
    const float* x;      // FPROP/WGRAD: input activations [B,Ci,Hi,Wi];  DGRAD: unused
    const float* w;      // [Co,Ci,kh,kw]
    const float* dy;     // DGRAD/WGRAD: [B,Co,Ho,Wo]
    const float* bias;   // epilogue (FPROP: per co, DGRAD-as-forward: per ci) or null
    const float* res;    // residual added before the activation (same layout as out) or null
    float* out;          // FPROP: y [B,Co,Ho,Wo]; DGRAD: dx [B,Ci,Hi,Wi]; WGRAD: dw [Co,Ci,kh,kw]
    float* work;         // split-K partials [splits][numel(out)]
    int B, Ci, Hi, Wi, Co, Ho, Wo, kh, kw, stride, pad;
    int act;             // CCB_ACT_*
    float slope;
    int splits;
    DgradClass dc;       // DGRAD: the parity class of this launch
    int M, N, K;
};

// Tile configuration: BM x BN outputs per CTA, TM x TN per thread, 256 threads, BK = 16.
template <int BM_, int BN_, int TM_, int TN_>
struct Cfg {
    static constexpr int BM = BM_, BN = BN_, TM = TM_, TN = TN_, BK = 16, NT = 256;
    static_assert((BM / TM) * (BN / TN) == NT, "thread tiling must cover the CTA tile");
};

// Decoded K index (one per k of the current tile), filled cooperatively.
struct KInfo { int off; int a; int b; int off2; };

template <int MODE>
__device__ __forceinline__ KInfo decode_k(const ConvArgs& a, int k) {
    KInfo r;
    r.off = -1; r.a = 0; r.b = 0; r.off2 = 0;
    if (k >= a.K) return r;
    if (MODE == MODE_FPROP) {
        int kk = a.kh * a.kw;
        int ci = k / kk, rem = k - ci * kk;
        int ky = rem / a.kw, kx = rem - ky * a.kw;
        r.off = ci * a.Hi * a.Wi; r.a = ky; r.b = kx; r.off2 = 0;
    } else if (MODE == MODE_DGRAD) {
        int nt = a.dc.nky * a.dc.nkx;
        int co = k / nt, rem = k - co * nt;
        int tky = rem / a.dc.nkx, tkx = rem - tky * a.dc.nkx;
        int ky = a.dc.ky0 + tky * a.stride, kx = a.dc.kx0 + tkx * a.stride;
        if (ky >= a.kh || kx >= a.kw) return r;          // parity class without a valid tap
        r.off = co * a.Ho * a.Wo; r.a = ky; r.b = kx;
        r.off2 = co * a.Ci * a.kh * a.kw + ky * a.kw + kx;
    } else {
        int hw = a.Ho * a.Wo;
        int b = k / hw, rem = k - b * hw;
        int oy = rem / a.Wo, ox = rem - oy * a.Wo;
        r.off = b; r.a = oy; r.b = ox; r.off2 = 0;
    }
    return r;
}

// Per-thread decoded M index (fixed across the K loop).
struct MInfo { int valid; int b; int y; int x; int c; };

template <int MODE>
__device__ __forceinline__ MInfo decode_m(const ConvArgs& a, int m) {
    MInfo r;
    r.valid = m < a.M; r.b = r.y = r.x = r.c = 0;
    if (!r.valid) return r;
    if (MODE == MODE_FPROP) {
        int hw = a.Ho * a.Wo;
        r.b = m / hw;
        int rem = m - r.b * hw;
        r.y = rem / a.Wo; r.x = rem - r.y * a.Wo;
    } else if (MODE == MODE_DGRAD) {
        int hw = a.dc.Hc * a.dc.Wc;
        r.b = m / hw;
        int rem = m - r.b * hw;
        int jy = rem / a.dc.Wc, jx = rem - jy * a.dc.Wc;
        r.y = a.dc.py + jy * a.stride; r.x = a.dc.px + jx * a.stride;
    } else {
        int kk = a.kh * a.kw;
        r.c = m / kk;
        int rem = m - r.c * kk;
        r.y = rem / a.kw; r.x = rem - r.y * a.kw;   // (ky, kx)
    }
    return r;
}

template <int MODE>
__device__ __forceinline__ float fetch_a(const ConvArgs& a, const MInfo& mi, const KInfo& ki) {
    if (!mi.valid || ki.off < 0) return 0.f;
    if (MODE == MODE_FPROP) {
        int iy = mi.y * a.stride - a.pad + ki.a, ix = mi.x * a.stride - a.pad + ki.b;
        if (iy < 0 || iy >= a.Hi || ix < 0 || ix >= a.Wi) return 0.f;
        return __ldg(a.x + (long long)mi.b * a.Ci * a.Hi * a.Wi + ki.off + iy * a.Wi + ix);
    } else if (MODE == MODE_DGRAD) {
        int ty = mi.y + a.pad - ki.a, tx = mi.x + a.pad - ki.b;     // divisible by stride by construction
        int oy = ty / a.stride, ox = tx / a.stride;
        if (ty < 0 || tx < 0 || oy >= a.Ho || ox >= a.Wo) return 0.f;
        return __ldg(a.dy + (long long)mi.b * a.Co * a.Ho * a.Wo + ki.off + oy * a.Wo + ox);
    } else {
        int iy = ki.a * a.stride - a.pad + mi.y, ix = ki.b * a.stride - a.pad + mi.x;
        if (iy < 0 || iy >= a.Hi || ix < 0 || ix >= a.Wi) return 0.f;
        return __ldg(a.x + ((long long)ki.off * a.Ci + mi.c) * a.Hi * a.Wi + iy * a.Wi + ix);
    }
}

template <int MODE>
__device__ __forceinline__ float fetch_b(const ConvArgs& a, const KInfo& ki, int k, int n) {
    if (n >= a.N || ki.off < 0) return 0.f;
    if (MODE == MODE_FPROP) return __ldg(a.w + (long long)n * a.K + k);
    if (MODE == MODE_DGRAD) return __ldg(a.w + ki.off2 + (long long)n * a.kh * a.kw);
    return __ldg(a.dy + ((long long)ki.off * a.Co + n) * a.Ho * a.Wo + ki.a * a.Wo + ki.b);
}

// linear offset of output element (m, n) in `out`
template <int MODE>
__device__ __forceinline__ long long out_offset(const ConvArgs& a, const MInfo& mi, int m, int n) {
    if (MODE == MODE_FPROP) return ((long long)mi.b * a.Co + n) * a.Ho * a.Wo + mi.y * a.Wo + mi.x;
    if (MODE == MODE_DGRAD) return ((long long)mi.b * a.Ci + n) * a.Hi * a.Wi + mi.y * a.Wi + mi.x;
    return (long long)n * a.M + m;   // dw[co][(ci,ky,kx)]
}

template <int MODE, class C>
__global__ void __launch_bounds__(256) conv_gemm_kernel(const ConvArgs a) {
    CCB_PDL_WAIT();
    constexpr int BM = C::BM, BN = C::BN, BK = C::BK, TM = C::TM, TN = C::TN;
    __shared__ __align__(16) float As[BK][BM + 4];
    __shared__ __align__(16) float Bs[BK][BN + 4];
    __shared__ KInfo s_k[2][BK];
    const int tid = threadIdx.x;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    // K range of this split (in tiles)
    const int ktiles = cdiv(a.K, BK);
    const int per = cdiv(ktiles, a.splits);
    const int kt_beg = blockIdx.z * per, kt_end = min(ktiles, kt_beg + per);

    // loader mapping: A element (kk = tid / BM + e * (256 / BM), m = tid % BM)
    constexpr int A_E = BM * BK / 256, A_KSTEP = 256 / BM;
    constexpr int B_E = BN * BK / 256;
    const int am = tid % BM, ak0 = tid / BM;
    const MInfo ami = decode_m<MODE>(a, m0 + am);
    const int bk = tid % BK, bn0 = tid / BK;     // B element (kk = bk, n = bn0 + e * 16)

    const int tx = tid % (BN / TN), ty = tid / (BN / TN);
    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    if (tid < BK && kt_beg < kt_end) s_k[0][tid] = decode_k<MODE>(a, kt_beg * BK + tid);
    __syncthreads();
    int buf = 0;
    for (int kt = kt_beg; kt < kt_end; ++kt) {
        const int k0 = kt * BK;
#pragma unroll
        for (int e = 0; e < A_E; ++e) {
            int kk = ak0 + e * A_KSTEP;
            As[kk][am] = fetch_a<MODE>(a, ami, s_k[buf][kk]);
        }
#pragma unroll
        for (int e = 0; e < B_E; ++e) {
            int n = bn0 + e * (256 / BK);
            Bs[bk][n] = fetch_b<MODE>(a, s_k[buf][bk], k0 + bk, n0 + n);
        }
        __syncthreads();
        if (tid < BK && kt + 1 < kt_end) s_k[buf ^ 1][tid] = decode_k<MODE>(a, (kt + 1) * BK + tid);
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float av[TM], bv[TN];
#pragma unroll
            for (int i = 0; i < TM; ++i) av[i] = As[kk][ty * TM + i];
#pragma unroll
            for (int j = 0; j < TN; ++j) bv[j] = Bs[kk][tx * TN + j];
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
        buf ^= 1;
    }

    // epilogue
    const long long out_numel = (MODE == MODE_FPROP) ? (long long)a.B * a.Co * a.Ho * a.Wo
                              : (MODE == MODE_DGRAD) ? (long long)a.B * a.Ci * a.Hi * a.Wi
                                                     : (long long)a.M * a.N;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        int m = m0 + ty * TM + i;
        if (m >= a.M) continue;
        MInfo mi = decode_m<MODE>(a, m);
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            int n = n0 + tx * TN + j;
            if (n >= a.N) continue;
            long long o = out_offset<MODE>(a, mi, m, n);
            float v = acc[i][j];
            if (a.splits > 1) {
                a.work[(long long)blockIdx.z * out_numel + o] = v;
            } else {
                if (MODE != MODE_WGRAD) {
                    if (a.bias) v += __ldg(a.bias + n);
                    if (a.res) v += __ldg(a.res + o);
                    v = apply_act(v, a.act, a.slope);
                }
                a.out[o] = v;
            }
        }
    }
}

// out[i] = epilogue(sum_s work[s][i]);  channel = (i / plane) % C for the bias
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ work, float* __restrict__ out,
                                                            const float* __restrict__ bias, const float* __restrict__ res,
                                                            long long numel, int splits, int plane, int C, int act,
                                                            float slope) {
    CCB_PDL_WAIT();
    long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= numel) return;
    float v = 0.f;
    for (int s = 0; s < splits; ++s) v += __ldg(work + (long long)s * numel + i);
    if (bias) v += __ldg(bias + (int)((i / plane) % C));
    if (res) v += __ldg(res + i);
    out[i] = apply_act(v, act, slope);
}

// dz = dy * act'(y) and db[c] = sum_{b,px} dz in ONE pass over the gradient (act_bwd + bias_grad read it twice and cost
// ~200 launches per step).  Large planes: grid (chunks, B, C), 256 threads x float4, per-CTA partial -> abb_merge_kernel;
// small planes (B * plane <= ABB_SMALL): one CTA per channel does everything.  Fixed summation order.
constexpr int ABB_CHUNK = 4096, ABB_SMALL = 8192;
__device__ __forceinline__ float act_grad(float g, float yv, int act, float slope) {
    switch (act) {
        case CCB_ACT_RELU: return (yv > 0.f) ? g : 0.f;
        case CCB_ACT_LEAKY: return (yv > 0.f) ? g : g * slope;
        case CCB_ACT_SIGMOID: return g * yv * (1.f - yv);
        default: return g;
    }
}
__global__ void __launch_bounds__(256) abb_large_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dz,
                                                        float* __restrict__ part, int C, int plane, int nchunk, int act, float slope) {
    CCB_PDL_WAIT();
    __shared__ float s_red[32];
    const int chunk = blockIdx.x, b = blockIdx.y, c = blockIdx.z;
    const long long base = ((long long)b * C + c) * plane;
    const int beg = chunk * ABB_CHUNK, end = min(plane, beg + ABB_CHUNK);
    float v[1] = {0.f};
    if ((plane & 3) == 0) {
        for (int i = beg + threadIdx.x * 4; i < end; i += 1024) {
            float4 g = __ldg((const float4*)(dy + base + i));
            if (act != CCB_ACT_NONE) {
                const float4 yv = __ldg((const float4*)(y + base + i));
                g.x = act_grad(g.x, yv.x, act, slope); g.y = act_grad(g.y, yv.y, act, slope);
                g.z = act_grad(g.z, yv.z, act, slope); g.w = act_grad(g.w, yv.w, act, slope);
                *(float4*)(dz + base + i) = g;
            }
            v[0] += (g.x + g.y) + (g.z + g.w);
        }
    } else {
        for (int i = beg + threadIdx.x; i < end; i += 256) {
            float g = __ldg(dy + base + i);
            if (act != CCB_ACT_NONE) { g = act_grad(g, __ldg(y + base + i), act, slope); dz[base + i] = g; }
            v[0] += g;
        }
    }
    if (part == nullptr) return;
    block_sum<1>(v, s_red);
    if (threadIdx.x == 0) part[((long long)c * gridDim.y + b) * nchunk + chunk] = v[0];
}
__global__ void __launch_bounds__(128) abb_merge_kernel(const float* __restrict__ part, float* __restrict__ db, int C, int n) {
    CCB_PDL_WAIT();
    const int c = blockIdx.x * 128 + threadIdx.x;
    if (c >= C) return;
    float a = 0.f;
    for (int s = 0; s < n; ++s) a += part[(long long)c * n + s];
    db[c] = a;
}
__global__ void __launch_bounds__(256) abb_small_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dz,
                                                        float* __restrict__ db, int B, int C, int plane, int act, float slope) {
    CCB_PDL_WAIT();
    __shared__ float s_red[32];
    const int c = blockIdx.x;
    float v[1] = {0.f};
    for (int b = 0; b < B; ++b) {
        const long long base = ((long long)b * C + c) * plane;
        for (int i = threadIdx.x; i < plane; i += 256) {
            float g = __ldg(dy + base + i);
            if (act != CCB_ACT_NONE) { g = act_grad(g, __ldg(y + base + i), act, slope); dz[base + i] = g; }
            v[0] += g;
        }
    }
    if (db == nullptr) return;
    block_sum<1>(v, s_red);
    if (threadIdx.x == 0) db[c] = v[0];
}

void launch_splitk_reduce(const float* work, float* out, const float* bias, const float* res, long long numel, int splits,
                          int plane, int C, int act, float slope, cudaStream_t st) {
    CCB_LAUNCH(splitk_reduce_kernel, dim3((unsigned)((numel + 255) / 256)), dim3(256), 0, st, work, out, bias, res, numel, splits,
               plane, C, act, slope);
}

// ------------------------------------------------------------------------------------------------
template <int MODE>
static int launch_gemm(const ConvArgs& a, long long out_numel, cudaStream_t st, const char* what) {
    const bool narrow = a.N <= 16;
    dim3 grid(cdiv(a.M, narrow ? 128 : 64), cdiv(a.N, narrow ? 16 : 64), a.splits);
    auto k_narrow = conv_gemm_kernel<MODE, Cfg<128, 16, 8, 1>>;
    auto k_wide = conv_gemm_kernel<MODE, Cfg<64, 64, 4, 4>>;
    if (narrow) CCB_LAUNCH(k_narrow, grid, dim3(256), 0, st, a);
    else CCB_LAUNCH(k_wide, grid, dim3(256), 0, st, a);
    int rc = check_launch(what);
    if (rc) return rc;
    if (a.splits > 1) {
        int plane = (MODE == MODE_FPROP) ? a.Ho * a.Wo : (MODE == MODE_DGRAD) ? a.Hi * a.Wi : 1;
        int C = (MODE == MODE_FPROP) ? a.Co : (MODE == MODE_DGRAD) ? a.Ci : 1;
        launch_splitk_reduce(a.work, a.out, (MODE == MODE_WGRAD) ? nullptr : a.bias, (MODE == MODE_WGRAD) ? nullptr : a.res,
                             out_numel, a.splits, plane, C, (MODE == MODE_WGRAD) ? CCB_ACT_NONE : a.act, a.slope, st);
        rc = check_launch("splitk_reduce");
    }
    return rc;
}

// Split-K count of an FFMA call: about 4 CTAs per SM (launch_gemm's tiles), at least 2 k-tiles per split and none empty,
// at most 64 splits and 64 MiB of partials.  The strided data gradient never splits: its parity classes would share the
// partials.
static int ffma_splits(const ccb_conv_desc* d, int op, long long out_numel) {
    if (op == CCB_CONV_DGRAD && d->stride > 1) return 1;
    const int kk = d->kh * d->kw;
    const int M = op == CCB_CONV_FPROP ? d->B * d->Ho * d->Wo : op == CCB_CONV_DGRAD ? d->B * d->Hi * d->Wi : d->Ci * kk;
    const int N = op == CCB_CONV_DGRAD ? d->Ci : d->Co;
    const int K = op == CCB_CONV_FPROP ? d->Ci * kk : op == CCB_CONV_DGRAD ? d->Co * kk : d->B * d->Ho * d->Wo;
    const bool narrow = N <= 16;
    const int tiles = cdiv(M, narrow ? 128 : 64) * cdiv(N, narrow ? 16 : 64), ktiles = cdiv(K, 16);
    if (tiles >= 4 * NUM_SMS || ktiles <= 2) return 1;
    long long s = 4 * NUM_SMS / tiles;
    if (s > ktiles / 2) s = ktiles / 2;
    if (s > 64) s = 64;
    if (s > (16ll << 20) / out_numel) s = (16ll << 20) / out_numel;
    while (s > 1 && cdiv(ktiles, (int)s) * (s - 1) >= ktiles) --s;
    return s < 1 ? 1 : (int)s;
}

static int check_desc(const ccb_conv_desc* d) {
    CCB_REQUIRE(d != nullptr, CCB_ERR_ARG, "conv: null descriptor");
    CCB_REQUIRE(d->B >= 1 && d->Ci >= 1 && d->Co >= 1 && d->Hi >= 1 && d->Wi >= 1, CCB_ERR_ARG, "conv: bad sizes");
    CCB_REQUIRE(d->kh >= 1 && d->kw >= 1 && d->stride >= 1 && d->pad >= 0, CCB_ERR_ARG, "conv: bad kernel/stride/pad");
    CCB_REQUIRE(d->Ho >= 1 && d->Wo >= 1, CCB_ERR_ARG, "conv: bad output size");
    // consistency of (Hi, Ho): Hi may exceed the minimal size by up to stride-1 (ConvTranspose output_padding)
    CCB_REQUIRE((d->Hi + 2 * d->pad - d->kh) / d->stride + 1 == d->Ho && (d->Wi + 2 * d->pad - d->kw) / d->stride + 1 == d->Wo,
                CCB_ERR_ARG, "conv: Ho/Wo inconsistent with Hi/Wi (%d,%d -> %d,%d, k %d s %d p %d)", d->Hi, d->Wi, d->Ho,
                d->Wo, d->kh, d->stride, d->pad);
    CCB_REQUIRE(d->impl >= CCB_CONV_IMPL_AUTO && d->impl <= CCB_CONV_IMPL_TC, CCB_ERR_ARG, "conv: unknown impl %d", d->impl);
    return CCB_OK;
}

static ConvArgs ffma_args(const ccb_conv_desc* d, int splits, float* work) {
    ConvArgs a;
    memset(&a, 0, sizeof(a));
    a.B = d->B; a.Ci = d->Ci; a.Hi = d->Hi; a.Wi = d->Wi; a.Co = d->Co; a.Ho = d->Ho; a.Wo = d->Wo;
    a.kh = d->kh; a.kw = d->kw; a.stride = d->stride; a.pad = d->pad;
    a.act = d->act; a.slope = d->slope; a.splits = splits; a.work = work;
    return a;
}

// the weight cache of the conv call in flight (wprep_get looks it up); sim builds have none
struct WCacheScope {
#ifndef CCB_CPU_SIM
    explicit WCacheScope(void* h) { g_cur_wcache = (WCache*)h; }
    ~WCacheScope() { g_cur_wcache = nullptr; }
#else
    explicit WCacheScope(void*) {}
#endif
};

// rows of W floats -> rows of Wp >= W floats, zero tail
__global__ void __launch_bounds__(256) pad_rows_kernel(const float* __restrict__ src, float* __restrict__ dst, long long rows, int W,
                                                       int Wp) {
    CCB_PDL_WAIT();
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= rows * Wp) return;
    const long long r = i / Wp;
    const int x = (int)(i - r * Wp);
    dst[i] = (x < W) ? __ldg(src + r * W + x) : 0.f;
}

// WGRAD on small feature maps whose width is not a multiple of 4 (26, 13, 7 ...): the tensor-core kernel reads
// 16-byte pixel chunks, so x and dy are first copied into rows padded to a multiple of 4 with zeros - a zero dy
// column contributes nothing and a zero x column is exactly what the convolution's own zero padding would read.
// dp: the padded call; xpf, dypf: floats of the padded copies of x and dy.
static void wgrad_pad_desc(const ccb_conv_desc* d, ccb_conv_desc& dp, long long& xpf, long long& dypf) {
    dp = *d;
    dp.Wo = (d->Wo + 3) & ~3;
    dp.Wi = (d->Wi + 3) & ~3;
    xpf = (long long)d->B * d->Ci * d->Hi * dp.Wi;
    dypf = (long long)d->B * d->Co * d->Ho * dp.Wo;
}

enum { PATH_FFMA, PATH_TC, PATH_TC_PADDED };
struct ConvPlan {
    int path;               // PATH_*
    int splits;             // split-K count (the data gradient's parity classes share it)
    long long head_floats;  // workspace ahead of the split-K partials: the prepared weights (tensor-core fprop / dgrad)
                            // or the padded copies of x and dy (PATH_TC_PADDED)
    long long work_floats;  // head + partials: the workspace the call needs
    const char* kernel;     // what ccb_debug_last_conv_kernel() reports after the call
};
static const char* const CONV_OP_NAME[3] = {"conv2d_fprop", "conv2d_dgrad", "conv2d_wgrad"};

// How one call runs, from the descriptor alone (shape + impl) and never from the workspace the caller passes, so that a
// call sums in the same order whatever ran before it.  AUTO takes the tensor cores where they pay off, TC wherever the
// kernels can express the shape, both take them for the weight gradient of a small map whose width is not a multiple
// of 4 through padded rows; everything else runs on the FFMA kernels.
static ConvPlan conv_plan(const ccb_conv_desc* d, int op) {
    ConvPlan p = {PATH_FFMA, 1, 0, 0, CONV_OP_NAME[op]};
    const long long numel = op == CCB_CONV_FPROP ? (long long)d->B * d->Co * d->Ho * d->Wo
                          : op == CCB_CONV_DGRAD ? (long long)d->B * d->Ci * d->Hi * d->Wi
                                                 : (long long)d->Co * d->Ci * d->kh * d->kw;
    if (d->impl == CCB_CONV_IMPL_TC ? tc_supported(d, op) : d->impl == CCB_CONV_IMPL_AUTO && tc_profitable(d, op)) {
        p.path = PATH_TC;
        p.splits = tc_plan(d, op, p.head_floats);
        p.kernel = op == CCB_CONV_WGRAD ? "conv_tc_wgrad" : "conv_tc";
    } else if (op == CCB_CONV_WGRAD && d->impl != CCB_CONV_IMPL_FFMA && d->Wo % 4 != 0) {
        ccb_conv_desc dp;
        long long xpf, dypf;
        wgrad_pad_desc(d, dp, xpf, dypf);
        if (xpf + dypf <= (8ll << 20) && tc_profitable(&dp, op)) {     // small maps only (<= 32 MiB of copies)
            p.path = PATH_TC_PADDED;
            p.splits = tc_plan(&dp, op, p.head_floats);
            p.head_floats = xpf + dypf;
            p.kernel = "conv_tc_wgrad";
        }
    }
    if (p.path == PATH_FFMA) p.splits = ffma_splits(d, op, numel);
    p.work_floats = p.head_floats + (p.splits > 1 ? p.splits * numel : 0);
    return p;
}

// Checks the call and its workspace against its plan; from then on the call is labelled with the plan's kernel.
static int start_conv(const ccb_conv_desc* d, int op, const float* work, long long work_floats, ConvPlan& p) {
    int rc = check_desc(d);
    if (rc) return rc;
    p = conv_plan(d, op);
    const long long have = work ? work_floats : 0;
    CCB_REQUIRE(have >= p.work_floats, CCB_ERR_ARG, "%s: workspace of %lld floats, the call needs %lld (ccb_conv_workspace_floats)",
                CONV_OP_NAME[op], have, p.work_floats);
    g_last_conv = p.kernel;
    return CCB_OK;
}

}  // namespace ccb

using namespace ccb;

extern "C" long long ccb_conv_workspace_floats(const ccb_conv_desc* d, int op) {
    if (op < CCB_CONV_FPROP || op > CCB_CONV_WGRAD || check_desc(d)) return -1;
    return conv_plan(d, op).work_floats;
}

extern "C" int ccb_debug_conv_plan(const ccb_conv_desc* d, int op, int* out2) {
    if (op < CCB_CONV_FPROP || op > CCB_CONV_WGRAD || !out2) return CCB_ERR_ARG;
    const int rc = check_desc(d);
    if (rc) return rc;
    const ConvPlan p = conv_plan(d, op);
    out2[0] = p.path;
    out2[1] = p.splits;
    return CCB_OK;
}

extern "C" int ccb_conv2d_fprop(const ccb_conv_desc* d, const float* x, const float* w, const float* bias,
                                const float* res, float* y, float* work, long long work_floats, ccb_stream_t stream) {
    CCB_REQUIRE(x && w && y, CCB_ERR_ARG, "conv2d_fprop: null pointer");
    ConvPlan p;
    int rc = start_conv(d, CCB_CONV_FPROP, work, work_floats, p);
    if (rc) return rc;
    WCacheScope wc_scope(d->wcache);
    if (p.path == PATH_TC) return tc_fprop(d, x, w, bias, res, y, work, work + p.head_floats, p.splits, (cudaStream_t)stream);
    ConvArgs a = ffma_args(d, p.splits, work);
    a.x = x; a.w = w; a.bias = bias; a.res = res; a.out = y;
    a.M = a.B * a.Ho * a.Wo; a.N = a.Co; a.K = a.Ci * a.kh * a.kw;
    return launch_gemm<MODE_FPROP>(a, (long long)a.M * a.N, (cudaStream_t)stream, p.kernel);
}

// dx[B,Ci,Hi,Wi] = conv_transpose(dy, w); with bias/res/act this is the ConvTranspose2d forward.
extern "C" int ccb_conv2d_dgrad(const ccb_conv_desc* d, const float* dy, const float* w, const float* bias,
                                const float* res, float* dx, float* work, long long work_floats, ccb_stream_t stream) {
    CCB_REQUIRE(dy && w && dx, CCB_ERR_ARG, "conv2d_dgrad: null pointer");
    ConvPlan p;
    int rc = start_conv(d, CCB_CONV_DGRAD, work, work_floats, p);
    if (rc) return rc;
    WCacheScope wc_scope(d->wcache);
    if (p.path == PATH_TC) return tc_dgrad(d, dy, w, bias, res, dx, work, work + p.head_floats, p.splits, (cudaStream_t)stream);
    ConvArgs a = ffma_args(d, p.splits, work);
    a.dy = dy; a.w = w; a.bias = bias; a.res = res; a.out = dx;
    const int s = a.stride;
    for (int py = 0; py < s && py < a.Hi; ++py)
        for (int px = 0; px < s && px < a.Wi; ++px) {
            ConvArgs c = a;
            c.dc = dgrad_class(d, py, px);
            c.M = a.B * c.dc.Hc * c.dc.Wc; c.N = a.Ci; c.K = a.Co * c.dc.nky * c.dc.nkx;
            if (c.K == 0) { c.K = 1; c.dc.nky = c.dc.nkx = 1; c.dc.ky0 = a.kh; c.dc.kx0 = a.kw; }   // no tap hits: output = epilogue(0)
            rc = launch_gemm<MODE_DGRAD>(c, (long long)a.B * a.Ci * a.Hi * a.Wi, (cudaStream_t)stream, p.kernel);
            if (rc) return rc;
        }
    return CCB_OK;
}

extern "C" int ccb_conv2d_wgrad(const ccb_conv_desc* d, const float* x, const float* dy, float* dw, float* work,
                                long long work_floats, ccb_stream_t stream) {
    CCB_REQUIRE(x && dy && dw, CCB_ERR_ARG, "conv2d_wgrad: null pointer");
    ConvPlan p;
    int rc = start_conv(d, CCB_CONV_WGRAD, work, work_floats, p);
    if (rc) return rc;
    if (p.path == PATH_TC) return tc_wgrad(d, x, dy, dw, work, p.splits, (cudaStream_t)stream);
    if (p.path == PATH_TC_PADDED) {
        ccb_conv_desc dp;
        long long xpf, dypf;
        wgrad_pad_desc(d, dp, xpf, dypf);
        float* xp = work;
        float* dyp = work + xpf;
        CCB_LAUNCH(pad_rows_kernel, dim3((unsigned)((xpf + 255) / 256)), dim3(256), 0, stream, x, xp, (long long)d->B * d->Ci * d->Hi,
                   d->Wi, dp.Wi);
        CCB_LAUNCH(pad_rows_kernel, dim3((unsigned)((dypf + 255) / 256)), dim3(256), 0, stream, dy, dyp, (long long)d->B * d->Co * d->Ho,
                   d->Wo, dp.Wo);
        rc = check_launch("conv2d_wgrad pad");
        if (rc) return rc;
        return tc_wgrad(&dp, xp, dyp, dw, work + p.head_floats, p.splits, (cudaStream_t)stream);
    }
    ConvArgs a = ffma_args(d, p.splits, work);
    a.x = x; a.dy = dy; a.out = dw; a.act = CCB_ACT_NONE;
    a.M = a.Ci * a.kh * a.kw; a.N = a.Co; a.K = a.B * a.Ho * a.Wo;
    return launch_gemm<MODE_WGRAD>(a, (long long)a.M * a.N, (cudaStream_t)stream, p.kernel);
}

extern "C" long long ccb_act_bwd_bias_workspace_floats(int B, int C, int plane) {
    if (B < 1 || C < 1 || plane < 1) return -1;
    if ((long long)B * plane <= ABB_SMALL) return 0;
    return (long long)C * B * cdiv(plane, ABB_CHUNK);
}
// dz = dy * act'(y) (skipped, dz untouched, when act == NONE) and, when db != NULL, db[c] = sum over (b, pixel) of dz.
extern "C" int ccb_act_bwd_bias(const float* dy, const float* y, float* dz, float* db, int B, int C, int plane, int act, float slope,
                                float* work, long long work_floats, ccb_stream_t stream) {
    CCB_REQUIRE(dy && B >= 1 && C >= 1 && plane >= 1, CCB_ERR_ARG, "act_bwd_bias: bad argument");
    CCB_REQUIRE(act == CCB_ACT_NONE || (y && dz), CCB_ERR_ARG, "act_bwd_bias: y and dz required with an activation");
    if (act == CCB_ACT_NONE && db == nullptr) return CCB_OK;
    if ((long long)B * plane <= ABB_SMALL) {
        CCB_LAUNCH(abb_small_kernel, dim3(C), dim3(256), 0, stream, dy, y, dz, db, B, C, plane, act, slope);
        return check_launch("act_bwd_bias");
    }
    const int nchunk = cdiv(plane, ABB_CHUNK);
    CCB_REQUIRE_WORK("act_bwd_bias", "work", work, work_floats, db ? ccb_act_bwd_bias_workspace_floats(B, C, plane) : 0);
    CCB_REQUIRE(C <= 65535 && B <= 65535, CCB_ERR_ARG, "act_bwd_bias: grid too large");
    CCB_LAUNCH(abb_large_kernel, dim3(nchunk, B, C), dim3(256), 0, stream, dy, y, dz, db ? work : nullptr, C, plane, nchunk, act, slope);
    if (db) CCB_LAUNCH(abb_merge_kernel, dim3(cdiv(C, 128)), dim3(128), 0, stream, (const float*)work, db, C, B * nchunk);
    return check_launch("act_bwd_bias");
}
