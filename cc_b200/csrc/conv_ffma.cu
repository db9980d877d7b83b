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
#include "ccb_common.cuh"

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
    // DGRAD parity class
    int py, px, Hc, Wc, ky0, kx0, nky, nkx;
    int M, N, K;
};

__device__ __forceinline__ float apply_act(float v, int act, float slope) {
    switch (act) {
        case CCB_ACT_RELU: return fmaxf(v, 0.f);
        case CCB_ACT_LEAKY: return v > 0.f ? v : v * slope;
        case CCB_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
        default: return v;
    }
}

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
        int nt = a.nky * a.nkx;
        int co = k / nt, rem = k - co * nt;
        int tky = rem / a.nkx, tkx = rem - tky * a.nkx;
        int ky = a.ky0 + tky * a.stride, kx = a.kx0 + tkx * a.stride;
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
        int hw = a.Hc * a.Wc;
        r.b = m / hw;
        int rem = m - r.b * hw;
        int jy = rem / a.Wc, jx = rem - jy * a.Wc;
        r.y = a.py + jy * a.stride; r.x = a.px + jx * a.stride;
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

// dz = dy * act'(y)  (in terms of the activation OUTPUT y), optionally accumulating a second grad
__global__ void __launch_bounds__(256) act_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y,
                                                      float* __restrict__ dz, long long numel, int act, float slope) {
    CCB_PDL_WAIT();
    long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= numel) return;
    float g = __ldg(dy + i), yv = __ldg(y + i);
    switch (act) {
        case CCB_ACT_RELU: g = (yv > 0.f) ? g : 0.f; break;
        case CCB_ACT_LEAKY: g = (yv > 0.f) ? g : g * slope; break;
        case CCB_ACT_SIGMOID: g = g * yv * (1.f - yv); break;
        default: break;
    }
    dz[i] = g;
}

// db[c] = sum_{b,y,x} dy[b,c,y,x] : one CTA per channel, fixed-order two-level sum
__global__ void __launch_bounds__(256) bias_grad_kernel(const float* __restrict__ dy, float* __restrict__ db, int B,
                                                        int C, int plane) {
    CCB_PDL_WAIT();
    __shared__ float s_red[32];
    const int c = blockIdx.x;
    float v[1] = {0.f};
    for (int b = 0; b < B; ++b) {
        const float* p = dy + ((long long)b * C + c) * plane;
        for (int i = threadIdx.x; i < plane; i += 256) v[0] += __ldg(p + i);
    }
    block_sum<1>(v, s_red);
    if (threadIdx.x == 0) db[c] = v[0];
}

// parallel variant for few channels x large planes: grid (C, nsplit) partials, then a per-channel merge
constexpr int BG_CHUNK = 16384;
__global__ void __launch_bounds__(256) bias_grad_partial_kernel(const float* __restrict__ dy, float* __restrict__ part, int B,
                                                                int C, int plane, int nsplit) {
    CCB_PDL_WAIT();
    __shared__ float s_red[32];
    const int c = blockIdx.x, sp = blockIdx.y;
    const long long per = (long long)B * plane;
    const long long beg = (long long)sp * BG_CHUNK, end = min(per, beg + (long long)BG_CHUNK);
    float v[1] = {0.f};
    for (long long i = beg + threadIdx.x; i < end; i += 256) {
        int b = (int)(i / plane), o = (int)(i - (long long)b * plane);
        v[0] += __ldg(dy + ((long long)b * C + c) * plane + o);
    }
    block_sum<1>(v, s_red);
    if (threadIdx.x == 0) part[(long long)c * nsplit + sp] = v[0];
}
__global__ void bias_grad_merge_kernel(const float* __restrict__ part, float* __restrict__ db, int C, int nsplit) {
    CCB_PDL_WAIT();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float a = 0.f;
    for (int s = 0; s < nsplit; ++s) a += part[(long long)c * nsplit + s];
    db[c] = a;
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

static int launch_bias_grad(const float* dy, float* db, int B, int C, int plane, float* work, long long work_floats,
                            cudaStream_t st) {
    const long long per = (long long)B * plane;
    const int nsplit = (int)((per + BG_CHUNK - 1) / BG_CHUNK);
    if (nsplit > 1 && work && (long long)C * nsplit <= work_floats) {
        CCB_LAUNCH(bias_grad_partial_kernel, dim3(C, nsplit), dim3(256), 0, st, dy, work, B, C, plane, nsplit);
        CCB_LAUNCH(bias_grad_merge_kernel, dim3(cdiv(C, 128)), dim3(128), 0, st, (const float*)work, db, C, nsplit);
    } else {
        CCB_LAUNCH(bias_grad_kernel, dim3(C), dim3(256), 0, st, dy, db, B, C, plane);
    }
    return check_launch("bias_grad");
}

void launch_splitk_reduce(const float* work, float* out, const float* bias, const float* res, long long numel, int splits,
                          int plane, int C, int act, float slope, cudaStream_t st) {
    CCB_LAUNCH(splitk_reduce_kernel, dim3((unsigned)((numel + 255) / 256)), dim3(256), 0, st, work, out, bias, res, numel, splits,
               plane, C, act, slope);
}

// ------------------------------------------------------------------------------------------------
static int pick_splits(int tiles, int ktiles, int max_splits) {
    const int target = NUM_SMS * 4;
    if (tiles >= target || ktiles <= 2) return 1;
    int s = target / tiles;
    if (s > ktiles / 2) s = ktiles / 2;
    if (s > max_splits) s = max_splits;
    return s < 1 ? 1 : s;
}

template <int MODE>
static int launch_gemm(ConvArgs& a, long long out_numel, long long work_floats, cudaStream_t st, const char* what) {
    const bool narrow = a.N <= 16;
    const int BM = narrow ? 128 : 64, BN = narrow ? 16 : 64;
    const int mt = cdiv(a.M, BM), nt = cdiv(a.N, BN), ktiles = cdiv(a.K, 16);
    int max_splits = (a.work && out_numel > 0) ? (int)(work_floats / out_numel) : 1;
    if (max_splits > 64) max_splits = 64;
    a.splits = pick_splits(mt * nt, ktiles, max_splits);
    // make sure no split is empty
    while (a.splits > 1 && cdiv(ktiles, a.splits) * (a.splits - 1) >= ktiles) --a.splits;
    dim3 grid(mt, nt, a.splits);
    auto k_narrow = conv_gemm_kernel<MODE, Cfg<128, 16, 8, 1>>;
    auto k_wide = conv_gemm_kernel<MODE, Cfg<64, 64, 4, 4>>;
    if (narrow) CCB_LAUNCH(k_narrow, grid, dim3(256), 0, st, a);
    else CCB_LAUNCH(k_wide, grid, dim3(256), 0, st, a);
    int rc = check_launch(what);
    if (rc) return rc;
    if (a.splits > 1) {
        int plane = (MODE == MODE_FPROP) ? a.Ho * a.Wo : (MODE == MODE_DGRAD) ? a.Hi * a.Wi : 1;
        int C = (MODE == MODE_FPROP) ? a.Co : (MODE == MODE_DGRAD) ? a.Ci : 1;
        CCB_LAUNCH(splitk_reduce_kernel, dim3((unsigned)((out_numel + 255) / 256)), dim3(256), 0, st,
                   a.work, a.out, (MODE == MODE_WGRAD) ? nullptr : a.bias, (MODE == MODE_WGRAD) ? nullptr : a.res,
                   out_numel, a.splits, plane, C, (MODE == MODE_WGRAD) ? CCB_ACT_NONE : a.act, a.slope);
        rc = check_launch("splitk_reduce");
    }
    return rc;
}

static int fill_conv(ConvArgs& a, const ccb_conv_desc* d) {
    CCB_REQUIRE(d != nullptr, CCB_ERR_ARG, "conv: null descriptor");
    CCB_REQUIRE(d->B >= 1 && d->Ci >= 1 && d->Co >= 1 && d->Hi >= 1 && d->Wi >= 1, CCB_ERR_ARG, "conv: bad sizes");
    CCB_REQUIRE(d->kh >= 1 && d->kw >= 1 && d->stride >= 1 && d->pad >= 0, CCB_ERR_ARG, "conv: bad kernel/stride/pad");
    CCB_REQUIRE(d->Ho >= 1 && d->Wo >= 1, CCB_ERR_ARG, "conv: bad output size");
    // consistency of (Hi, Ho): Hi may exceed the minimal size by up to stride-1 (ConvTranspose output_padding)
    CCB_REQUIRE((d->Hi + 2 * d->pad - d->kh) / d->stride + 1 == d->Ho && (d->Wi + 2 * d->pad - d->kw) / d->stride + 1 == d->Wo,
                CCB_ERR_ARG, "conv: Ho/Wo inconsistent with Hi/Wi (%d,%d -> %d,%d, k %d s %d p %d)", d->Hi, d->Wi, d->Ho,
                d->Wo, d->kh, d->stride, d->pad);
    memset(&a, 0, sizeof(a));
    a.B = d->B; a.Ci = d->Ci; a.Hi = d->Hi; a.Wi = d->Wi; a.Co = d->Co; a.Ho = d->Ho; a.Wo = d->Wo;
    a.kh = d->kh; a.kw = d->kw; a.stride = d->stride; a.pad = d->pad;
    a.act = d->act; a.slope = d->slope; a.splits = 1;
    return CCB_OK;
}

// tensor-core path (conv_tc.cu)
bool tc_supported(const ccb_conv_desc* d, int op);
bool tc_profitable(const ccb_conv_desc* d, int op);
long long tc_workspace_floats(const ccb_conv_desc* d, int op);
int tc_fprop(const ccb_conv_desc* d, const float* x, const float* w, const float* bias, const float* res, float* y,
             float* work, long long work_floats, int three, cudaStream_t st);
int tc_dgrad(const ccb_conv_desc* d, const float* dy, const float* w, const float* bias, const float* res, float* dx,
             float* work, long long work_floats, int three, cudaStream_t st);

int tc_wgrad(const ccb_conv_desc* d, const float* x, const float* dy, float* dw, float* work, long long work_floats,
             int three, cudaStream_t st);

// the weight cache of the conv call in flight (wprep_get looks it up); sim builds have none
struct WCacheScope {
#ifndef CCB_CPU_SIM
    explicit WCacheScope(void* h) { g_cur_wcache = (WCache*)h; }
    ~WCacheScope() { g_cur_wcache = nullptr; }
#else
    explicit WCacheScope(void*) {}
#endif
};

// 0: FFMA, 1: wgmma 3xTF32, 2: wgmma single TF32
static int pick_impl(const ccb_conv_desc* d, int op) {
    switch (d->impl) {
        case CCB_CONV_IMPL_FFMA: return 0;
        // forcing the tensor-core path falls back to FFMA only for shapes it cannot express at all
        case CCB_CONV_IMPL_TC: return tc_supported(d, op) ? 1 : 0;
        case CCB_CONV_IMPL_TC_TF32: return tc_supported(d, op) ? 2 : 0;
        default: return tc_profitable(d, op) ? 1 : 0;
    }
}

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
static bool wgrad_pad_desc(const ccb_conv_desc* d, ccb_conv_desc& dp, long long& xpf, long long& dypf) {
    if (d->impl == CCB_CONV_IMPL_FFMA || (d->Wo % 4) == 0) return false;
    dp = *d;
    dp.Wo = (d->Wo + 3) & ~3;
    dp.Wi = (d->Wi + 3) & ~3;
    xpf = (long long)d->B * d->Ci * d->Hi * dp.Wi;
    dypf = (long long)d->B * d->Co * d->Ho * dp.Wo;
    if (xpf + dypf > (8ll << 20)) return false;                    // small maps only (<= 32 MiB of copies)
    return tc_profitable(&dp, CCB_CONV_WGRAD);
}

}  // namespace ccb

using namespace ccb;

extern "C" long long ccb_conv_workspace_floats(const ccb_conv_desc* d, int op) {
    if (!d) return -1;
    const long long bias_need = (op == CCB_CONV_WGRAD) ? (long long)d->Co * (((long long)d->B * d->Ho * d->Wo + BG_CHUNK - 1) / BG_CHUNK) : 0;
    if (op == CCB_CONV_WGRAD) {
        ccb_conv_desc dp;
        long long xpf, dypf;
        if (wgrad_pad_desc(d, dp, xpf, dypf)) {
            const long long t = xpf + dypf + tc_workspace_floats(&dp, op);
            return t > bias_need ? t : bias_need;
        }
    }
    if (d->impl != CCB_CONV_IMPL_FFMA && tc_supported(d, op) && pick_impl(d, op) > 0) {
        const long long t = tc_workspace_floats(d, op);
        return t > bias_need ? t : bias_need;
    }
    long long numel = (op == CCB_CONV_FPROP) ? (long long)d->B * d->Co * d->Ho * d->Wo
                    : (op == CCB_CONV_DGRAD) ? (long long)d->B * d->Ci * d->Hi * d->Wi
                                             : (long long)d->Co * d->Ci * d->kh * d->kw;
    // enough for up to 16 splits, capped at 64 MiB of floats
    long long cap = 16ll * 1024 * 1024;
    long long want = numel * 16;
    if (want > cap) want = (cap / numel) * numel;
    if (want < numel) want = 0;
    return want > bias_need ? want : bias_need;
}

extern "C" int ccb_conv2d_fprop(const ccb_conv_desc* d, const float* x, const float* w, const float* bias,
                                const float* res, float* y, float* work, long long work_floats, ccb_stream_t stream) {
    ConvArgs a;
    int rc = fill_conv(a, d);
    if (rc) return rc;
    CCB_REQUIRE(x && w && y, CCB_ERR_ARG, "conv2d_fprop: null pointer");
    WCacheScope wc_scope(d->wcache);
    {
        int impl = pick_impl(d, CCB_CONV_FPROP);
        CCB_REQUIRE(impl >= 0, CCB_ERR_UNSUPPORTED, "conv2d_fprop: shape not supported by the tensor-core path");
        if (impl > 0) return tc_fprop(d, x, w, bias, res, y, work, work_floats, impl == 1, (cudaStream_t)stream);
    }
    a.x = x; a.w = w; a.bias = bias; a.res = res; a.out = y; a.work = work;
    a.M = a.B * a.Ho * a.Wo; a.N = a.Co; a.K = a.Ci * a.kh * a.kw;
    return launch_gemm<MODE_FPROP>(a, (long long)a.M * a.N, work_floats, (cudaStream_t)stream, "conv2d_fprop");
}

// dx[B,Ci,Hi,Wi] = conv_transpose(dy, w); with bias/res/act this is the ConvTranspose2d forward.
extern "C" int ccb_conv2d_dgrad(const ccb_conv_desc* d, const float* dy, const float* w, const float* bias,
                                const float* res, float* dx, float* work, long long work_floats, ccb_stream_t stream) {
    ConvArgs a;
    int rc = fill_conv(a, d);
    if (rc) return rc;
    CCB_REQUIRE(dy && w && dx, CCB_ERR_ARG, "conv2d_dgrad: null pointer");
    WCacheScope wc_scope(d->wcache);
    {
        int impl = pick_impl(d, CCB_CONV_DGRAD);
        CCB_REQUIRE(impl >= 0, CCB_ERR_UNSUPPORTED, "conv2d_dgrad: shape not supported by the tensor-core path");
        if (impl > 0) return tc_dgrad(d, dy, w, bias, res, dx, work, work_floats, impl == 1, (cudaStream_t)stream);
    }
    a.dy = dy; a.w = w; a.bias = bias; a.res = res; a.out = dx; a.work = work;
    const int s = a.stride;
    for (int py = 0; py < s && py < a.Hi; ++py)
        for (int px = 0; px < s && px < a.Wi; ++px) {
            ConvArgs c = a;
            c.py = py; c.px = px;
            c.Hc = (a.Hi - py + s - 1) / s; c.Wc = (a.Wi - px + s - 1) / s;
            c.ky0 = (py + a.pad) % s; c.kx0 = (px + a.pad) % s;
            c.nky = (a.kh > c.ky0) ? (a.kh - c.ky0 + s - 1) / s : 0;
            c.nkx = (a.kw > c.kx0) ? (a.kw - c.kx0 + s - 1) / s : 0;
            c.M = a.B * c.Hc * c.Wc; c.N = a.Ci; c.K = a.Co * c.nky * c.nkx;
            if (c.K == 0) { c.K = 1; c.nky = c.nkx = 1; c.ky0 = a.kh; c.kx0 = a.kw; }   // no tap hits: output = epilogue(0)
            // split-K partials of different parity classes must not alias: no split-K for strided dgrad
            float* wk = (s == 1) ? work : nullptr;
            c.work = wk;
            rc = launch_gemm<MODE_DGRAD>(c, (long long)a.B * a.Ci * a.Hi * a.Wi, wk ? work_floats : 0, (cudaStream_t)stream,
                                         "conv2d_dgrad");
            if (rc) return rc;
        }
    return CCB_OK;
}

extern "C" int ccb_conv2d_wgrad(const ccb_conv_desc* d, const float* x, const float* dy, float* dw, float* db,
                                float* work, long long work_floats, ccb_stream_t stream) {
    ConvArgs a;
    int rc = fill_conv(a, d);
    if (rc) return rc;
    CCB_REQUIRE(x && dy && dw, CCB_ERR_ARG, "conv2d_wgrad: null pointer");
    {
        int impl = pick_impl(d, CCB_CONV_WGRAD);
        CCB_REQUIRE(impl >= 0, CCB_ERR_UNSUPPORTED, "conv2d_wgrad: shape not supported by the tensor-core path");
        if (impl > 0) {
            rc = tc_wgrad(d, x, dy, dw, work, work_floats, impl == 1, (cudaStream_t)stream);
            if (rc) return rc;
            if (db) rc = launch_bias_grad(dy, db, d->B, d->Co, d->Ho * d->Wo, work, work_floats, (cudaStream_t)stream);
            return rc;
        }
    }
    {
        ccb_conv_desc dp;
        long long xpf, dypf;
        const bool padded = wgrad_pad_desc(d, dp, xpf, dypf);
        const long long inner = padded ? tc_workspace_floats(&dp, CCB_CONV_WGRAD) : 0;
        if (padded && work && xpf + dypf + inner <= work_floats) {
            float* xp = work;
            float* dyp = work + xpf;
            CCB_LAUNCH(pad_rows_kernel, dim3((unsigned)((xpf + 255) / 256)), dim3(256), 0, stream, x, xp, (long long)d->B * d->Ci * d->Hi,
                       d->Wi, dp.Wi);
            CCB_LAUNCH(pad_rows_kernel, dim3((unsigned)((dypf + 255) / 256)), dim3(256), 0, stream, dy, dyp, (long long)d->B * d->Co * d->Ho,
                       d->Wo, dp.Wo);
            rc = check_launch("conv2d_wgrad pad");
            if (rc) return rc;
            rc = tc_wgrad(&dp, xp, dyp, dw, work + xpf + dypf, work_floats - xpf - dypf, d->impl != CCB_CONV_IMPL_TC_TF32,
                          (cudaStream_t)stream);
            if (rc) return rc;
            if (db) rc = launch_bias_grad(dy, db, d->B, d->Co, d->Ho * d->Wo, work, work_floats, (cudaStream_t)stream);
            return rc;
        }
    }
    a.x = x; a.dy = dy; a.out = dw; a.work = work; a.act = CCB_ACT_NONE;
    a.M = a.Ci * a.kh * a.kw; a.N = a.Co; a.K = a.B * a.Ho * a.Wo;
    rc = launch_gemm<MODE_WGRAD>(a, (long long)a.M * a.N, work_floats, (cudaStream_t)stream, "conv2d_wgrad");
    if (rc) return rc;
    if (db) rc = launch_bias_grad(dy, db, a.B, a.Co, a.Ho * a.Wo, work, work_floats, (cudaStream_t)stream);
    return rc;
}

extern "C" int ccb_act_bwd(const float* dy, const float* y, float* dz, long long numel, int act, float slope,
                           ccb_stream_t stream) {
    CCB_REQUIRE(dy && y && dz && numel >= 0, CCB_ERR_ARG, "act_bwd: null pointer");
    if (numel == 0) return CCB_OK;
    CCB_LAUNCH(act_bwd_kernel, dim3((unsigned)((numel + 255) / 256)), dim3(256), 0, stream, dy, y, dz, numel, act, slope);
    return check_launch("act_bwd");
}

extern "C" long long ccb_act_bwd_bias_workspace_floats(int B, int C, int plane) {
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
    CCB_REQUIRE(db == nullptr || (work && work_floats >= (long long)C * B * nchunk), CCB_ERR_ARG, "act_bwd_bias: workspace too small");
    CCB_REQUIRE(C <= 65535 && B <= 65535, CCB_ERR_ARG, "act_bwd_bias: grid too large");
    CCB_LAUNCH(abb_large_kernel, dim3(nchunk, B, C), dim3(256), 0, stream, dy, y, dz, db ? work : nullptr, C, plane, nchunk, act, slope);
    if (db) CCB_LAUNCH(abb_merge_kernel, dim3(cdiv(C, 128)), dim3(128), 0, stream, (const float*)work, db, C, B * nchunk);
    return check_launch("act_bwd_bias");
}

extern "C" long long ccb_bias_grad_workspace_floats(int B, int C, int plane) {
    const long long nsplit = ((long long)B * plane + BG_CHUNK - 1) / BG_CHUNK;
    return nsplit > 1 ? (long long)C * nsplit : 0;
}
extern "C" int ccb_bias_grad(const float* dy, float* db, int B, int C, int plane, float* work, long long work_floats,
                             ccb_stream_t stream) {
    CCB_REQUIRE(dy && db, CCB_ERR_ARG, "bias_grad: null pointer");
    return launch_bias_grad(dy, db, B, C, plane, work, work_floats, (cudaStream_t)stream);
}
