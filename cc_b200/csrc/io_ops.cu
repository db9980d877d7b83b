// io_ops.cu - the callers either side of the training step (SURVEY.md 8f "next" rows N1 / N2):
//
//   N2  validation metrics as fused masked reductions
//         flow:  flow_diff / compute_epe / outlier_err / compute_all_epes   (loss_functions.py:355-427)
//         depth: compute_errors with median scaling and the Garg crop        (loss_functions.py:430-467)
//   N1  input pipeline on the device: uint8 HWC frames -> normalised fp32 NCHW frames with the reference's
//       augmentations (ArrayToTensor /255, Normalize mean .5 std .5, RandomHorizontalFlip, RandomScaleCrop;
//       custom_transforms.py:21-30,47-118) applied per sample from host-drawn parameters, plus the matching
//       intrinsics update.  H2D traffic drops 4x (uint8 instead of fp32).
//       The reference's other transforms, bit-exact with Pillow (behind scipy.misc.imrotate / imresize):
//       RandomRotate (:75-85) as Pillow's bilinear affine transform, Scale (:120-137) as Pillow's 8-bit resampler,
//       NormalizeLocally (:33-44) as per-sample channel statistics.
//
//   N3  motion segmentation scores: the three rigidity masks and the IoU counts of test_mask.py:129-156,224-262
//       depth evaluation of test_disp.py:98-141: the velodyne ground truth, scipy's cubic zoom, both scalings' errors
//       Make3D depth evaluation of test_make3d.py:97-148: imresize's contrast stretch, the capped median scaling, log10
//
// All floating-point reductions are two-stage and deterministic (per-block partials in double, fixed-order finalize); the
// segmentation counts are integer sums (atomics, the same in any order).
#include "ccb_common.cuh"

#ifdef CCB_CPU_SIM
// The fp64 round-to-nearest intrinsics the Pillow restatements below use, for the host build of this file: one IEEE
// operation each, kept apart by the volatile store so that the host compiler cannot fuse them either.
static inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }
static inline double __dsub_rn(double a, double b) { volatile double r = a - b; return r; }
static inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }
static inline double __ddiv_rn(double a, double b) { volatile double r = a / b; return r; }
static inline double __dsqrt_rn(double a) { volatile double r = sqrt(a); return r; }
static inline double __fma_rn(double a, double b, double c) { return fma(a, b, c); }
static inline long long __double_as_longlong(double d) { long long i; memcpy(&i, &d, 8); return i; }
static inline double __longlong_as_double(long long i) { double d; memcpy(&d, &i, 8); return d; }
#endif

namespace ccb {

// ------------------------------------------------------------------------------------------------
// ATen's upsample_bilinear2d(align_corners=False) source index (area_pixel_compute_source_index):
// src = scale * (dst + 0.5) - 0.5, clamped below at 0; scale = in / out in fp32.
struct Lin { int i0, i1; float w0, w1; };
__device__ __forceinline__ Lin lin_src(int dst, int in_size, float scale) {
    float s = scale * ((float)dst + 0.5f) - 0.5f;
    if (s < 0.f) s = 0.f;
    Lin l;
    l.i0 = (int)s;
    if (l.i0 > in_size - 1) l.i0 = in_size - 1;
    l.i1 = l.i0 + ((l.i0 < in_size - 1) ? 1 : 0);
    l.w1 = s - (float)l.i0;
    l.w0 = 1.f - l.w1;
    return l;
}
__device__ __forceinline__ float bilerp(const float* __restrict__ p, int w, const Lin& ly, const Lin& lx) {
    // ATen order: w0y * (w0x * v00 + w1x * v01) + w1y * (w0x * v10 + w1x * v11)
    return ly.w0 * (lx.w0 * __ldg(p + ly.i0 * w + lx.i0) + lx.w1 * __ldg(p + ly.i0 * w + lx.i1)) +
           ly.w1 * (lx.w0 * __ldg(p + ly.i1 * w + lx.i0) + lx.w1 * __ldg(p + ly.i1 * w + lx.i1));
}

// s[j] = the sum over blocks k < nblk of p[k * stride + j], j < NV: the fp64 block partials of one reduction in block order,
// a fixed order that gives the same bits on every run.
template <int NV>
__device__ __forceinline__ void sum_partials(const double* p, int nblk, int stride, double (&s)[NV]) {
    for (int j = 0; j < NV; ++j) s[j] = 0.0;
    for (int k = 0; k < nblk; ++k)
        for (int j = 0; j < NV; ++j) s[j] += p[(long long)k * stride + j];
}

// The maximum of m over the warp, then one atomicMax per warp into *dst.  The callers' keys are in the order they want,
// and a maximum is the same in any order.
template <class T>
__device__ __forceinline__ void warp_max_into(unsigned long long* dst, T m) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const T k = __shfl_xor_sync(0xffffffffu, m, o);
        m = (k > m) ? k : m;
    }
    if ((threadIdx.x & 31) == 0) atomicMax(dst, (unsigned long long)m);
}

// Order-preserving keys: the unsigned order of the key is the value order of the float / double (NaN is not ordered).
__device__ __forceinline__ unsigned ordered_key32(float f) {
    const unsigned k = __float_as_uint(f);
    return (k >> 31) ? ~k : (k | 0x80000000u);
}
__device__ __forceinline__ float ordered_value32(unsigned k) {
    return __uint_as_float((k >> 31) ? (k & 0x7fffffffu) : ~k);
}
__device__ __forceinline__ unsigned long long ordered_key(double d) {
    const unsigned long long k = (unsigned long long)__double_as_longlong(d);
    return (k >> 63) ? ~k : (k | 0x8000000000000000ull);
}
__device__ __forceinline__ double ordered_value(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// ================================================================================================
// Per-sample medians by radix select, for compute_errors (loss_functions.py:430-467), test_disp.py:124-141 and
// test_make3d.py:141-148.  The argument struct A of a caller gives
//   A::Key         the key type: 32 bits take 3 passes (11, 11, 10 bits), 64 bits 6 passes (11 x 5, then 9)
//   A::SEL         the selections per sample
//   A::UPPER       bit s set: selection s takes the upper middle rank n/2 (numpy's second middle value), else the lower
//                  middle (n-1)/2 (torch.median, numpy's first); the two are the same rank when n is odd
//   a.median_keys  the valid flag and the SEL order-preserving keys of element i of sample b
//   a.med          the select's state
// Each pass histograms, in block-shared memory, the keys that match the prefix found so far (median_hist_kernel); then one
// thread per (sample, selection) finds the bin holding its rank, extends the prefix and clears the histogram
// (median_select_kernel).  The first pass also counts the valid elements.  Integer counts: the same on every run.
struct MedianState {
    unsigned* hist;                 // [B][SEL][2048]
    unsigned long long* sel;        // [B][SEL][3]: key prefix, prefix mask, remaining rank
    unsigned long long* count;      // [B] valid elements
};

template <class Key> __host__ __device__ constexpr int radix_passes() { return (8 * (int)sizeof(Key) + 10) / 11; }
template <class Key> __device__ __forceinline__ int radix_shift(int pass) {
    return pass < radix_passes<Key>() - 1 ? 8 * (int)sizeof(Key) - 11 * (pass + 1) : 0;
}
template <class Key> __device__ __forceinline__ unsigned radix_bins(int pass) {
    return pass < radix_passes<Key>() - 1 ? 2048u : 1u << (8 * (int)sizeof(Key) - 11 * pass);
}

template <class A>
__global__ void __launch_bounds__(256) median_hist_kernel(const A a, int pass) {
    CCB_PDL_WAIT();
    using Key = typename A::Key;
    constexpr int S = A::SEL;
    __shared__ unsigned h[S * 2048];
    const int b = blockIdx.y;
    const int shift = radix_shift<Key>(pass);
    const Key bin_mask = (Key)(radix_bins<Key>(pass) - 1);
    for (int i = threadIdx.x; i < S * 2048; i += 256) h[i] = 0;
    __syncthreads();
    const unsigned long long* s = a.med.sel + (long long)b * S * 3;
    Key pre[S], msk[S];
#pragma unroll
    for (int k = 0; k < S; ++k) { pre[k] = (Key)s[3 * k]; msk[k] = (Key)s[3 * k + 1]; }
    const long long hw = (long long)a.H * a.W;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < hw; i += (long long)gridDim.x * 256) {
        Key key[S];
        if (!a.median_keys(b, i, key)) continue;
#pragma unroll
        for (int k = 0; k < S; ++k)
            if ((key[k] & msk[k]) == pre[k]) atomicAdd(h + k * 2048 + (unsigned)((key[k] >> shift) & bin_mask), 1u);
    }
    __syncthreads();
    unsigned* g = a.med.hist + (long long)b * S * 2048;
    for (int i = threadIdx.x; i < S * 2048; i += 256)
        if (h[i]) atomicAdd(g + i, h[i]);
}

template <class A>
__global__ void median_select_kernel(const A a, int pass) {
    CCB_PDL_WAIT();
    using Key = typename A::Key;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.B * A::SEL) return;
    const int b = t / A::SEL, k = t % A::SEL;
    unsigned* h = a.med.hist + (long long)t * 2048;
    unsigned long long* s = a.med.sel + (long long)t * 3;
    const int shift = radix_shift<Key>(pass);
    const unsigned nbins = radix_bins<Key>(pass);
    if (pass == 0) {
        unsigned long long n = 0;
        for (unsigned i = 0; i < nbins; ++i) n += h[i];
        if (k == 0) a.med.count[b] = n;
        s[2] = (n == 0) ? 0 : (((A::UPPER >> k) & 1u) ? n / 2 : (n - 1) / 2);
    }
    const unsigned long long rank = s[2];
    unsigned long long cum = 0;
    unsigned bin = 0;
    for (unsigned i = 0; i < nbins; ++i) {
        bin = i;
        if (cum + h[i] > rank) break;
        cum += h[i];
    }
    s[2] = rank - cum;
    s[0] |= (unsigned long long)bin << shift;
    s[1] |= (unsigned long long)(nbins - 1) << shift;
    for (unsigned i = 0; i < 2048; ++i) h[i] = 0;
}

// ================================================================================================
// Flow metrics.  One pass over the ground-truth grid:
//   total  = mask ? (m_pred > T ? rigid : 0) + (m_pred <= T ? non_rigid : 0) at prediction resolution : rigid
//   all / rigid / non-rigid EPE sums + their valid counts, outlier count (compute_all_epes :409-427)
struct FlowMetArgs {
    const float* gt;          // [B, nc, Hg, Wg], nc 2 or 3 (3rd = valid)
    const float* pa;          // [B, 2, hp, wp]  rigid (or the only) prediction
    const float* pb;          // [B, 2, hp, wp]  non-rigid prediction, or null
    const float* mask;        // [B, 1, hm, wm]  rigidity mask, or null
    double* partials;         // [blocks][8]
    float* epe_map;           // optional [B, Hg, Wg]: flow_diff of `pa` alone (null otherwise)
    int B, nc, Hg, Wg, hp, wp, hm, wm;
    float thresh, tau0, tau1;
};

__device__ __forceinline__ float mask_at_pred(const FlowMetArgs& a, const float* m, int y, int x, float sy, float sx) {
    Lin ly = lin_src(y, a.hm, sy), lx = lin_src(x, a.wm, sx);
    return bilerp(m, a.wm, ly, lx);
}

__global__ void __launch_bounds__(256) flow_metrics_kernel(const FlowMetArgs a) {
    CCB_PDL_WAIT();
    __shared__ double scratch[8 * 32];
    const long long npx = (long long)a.B * a.Hg * a.Wg;
    const float sy_p = (float)a.hp / (float)a.Hg, sx_p = (float)a.wp / (float)a.Wg;          // pred -> gt
    const float fu = (float)((double)a.Wg / (double)a.wp), fv = (float)((double)a.Hg / (double)a.hp);   // python float ratio, cast on use
    const float sy_mg = a.mask ? (float)a.hm / (float)a.Hg : 0.f, sx_mg = a.mask ? (float)a.wm / (float)a.Wg : 0.f;   // mask -> gt
    const float sy_mp = a.mask ? (float)a.hm / (float)a.hp : 0.f, sx_mp = a.mask ? (float)a.wm / (float)a.wp : 0.f;   // mask -> pred
    double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // epe_all, den_all, epe_rig, den_rig, epe_non, den_non, n_err, (unused)
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < npx; i += (long long)gridDim.x * 256) {
        const int x = (int)(i % a.Wg);
        const int y = (int)((i / a.Wg) % a.Hg);
        const int b = (int)(i / ((long long)a.Wg * a.Hg));
        const float* g = a.gt + (long long)b * a.nc * a.Hg * a.Wg + (long long)y * a.Wg + x;
        const float ug = __ldg(g), vg = __ldg(g + (long long)a.Hg * a.Wg);
        const float valid = (a.nc == 3) ? __ldg(g + 2ll * a.Hg * a.Wg) : 1.f;
        const Lin ly = lin_src(y, a.hp, sy_p), lx = lin_src(x, a.wp, sx_p);
        const float* pa = a.pa + (long long)b * 2 * a.hp * a.wp;
        float ua, va, ur = 0.f, vr = 0.f, un = 0.f, vn = 0.f;      // total, rigid-only, non-rigid-only (upsampled, unscaled)
        if (!a.mask) {
            ua = bilerp(pa, a.wp, ly, lx);
            va = bilerp(pa + a.hp * a.wp, a.wp, ly, lx);
        } else {
            const float* pb = a.pb + (long long)b * 2 * a.hp * a.wp;
            const float* m = a.mask + (long long)b * a.hm * a.wm;
            // the composite is formed at prediction resolution, then upsampled: evaluate the four corner pixels
            const int ys[2] = {ly.i0, ly.i1}, xs[2] = {lx.i0, lx.i1};
            const float wy[2] = {ly.w0, ly.w1}, wx[2] = {lx.w0, lx.w1};
            float rr[2][2][2], nn[2][2][2];
#pragma unroll
            for (int cy = 0; cy < 2; ++cy)
#pragma unroll
                for (int cx = 0; cx < 2; ++cx) {
                    const float mp = mask_at_pred(a, m, ys[cy], xs[cx], sy_mp, sx_mp);
                    const float sr = (mp > a.thresh) ? 1.f : 0.f, sn = (mp <= a.thresh) ? 1.f : 0.f;
                    const int o = ys[cy] * a.wp + xs[cx];
                    rr[cy][cx][0] = sr * __ldg(pa + o); rr[cy][cx][1] = sr * __ldg(pa + a.hp * a.wp + o);
                    nn[cy][cx][0] = sn * __ldg(pb + o); nn[cy][cx][1] = sn * __ldg(pb + a.hp * a.wp + o);
                }
            auto up = [&](float (&q)[2][2][2], int ch) {
                return wy[0] * (wx[0] * q[0][0][ch] + wx[1] * q[0][1][ch]) + wy[1] * (wx[0] * q[1][0][ch] + wx[1] * q[1][1][ch]);
            };
            float tt[2][2][2];
#pragma unroll
            for (int cy = 0; cy < 2; ++cy)
#pragma unroll
                for (int cx = 0; cx < 2; ++cx) { tt[cy][cx][0] = nn[cy][cx][0] + rr[cy][cx][0]; tt[cy][cx][1] = nn[cy][cx][1] + rr[cy][cx][1]; }
            ua = up(tt, 0); va = up(tt, 1);
            ur = up(rr, 0); vr = up(rr, 1);
            un = up(nn, 0); vn = up(nn, 1);
        }
        const float du = ug - ua * fu, dv = vg - va * fv;
        const float epe = sqrtf(du * du + dv * dv);
        if (a.epe_map) a.epe_map[i] = epe;
        const float ev = epe * valid;
        acc[0] += ev;
        acc[1] += valid;
        const float mag = sqrtf(ug * ug + vg * vg);
        const float e0 = (ev > a.tau0) ? 1.f : 0.f, e1 = ((ev / (mag + 1e-8f)) > a.tau1) ? 1.f : 0.f;
        acc[6] += e0 * e1 * valid;
        if (a.mask) {
            const Lin my = lin_src(y, a.hm, sy_mg), mx = lin_src(x, a.wm, sx_mg);
            const float mg = bilerp(a.mask + (long long)b * a.hm * a.wm, a.wm, my, mx);
            const float sr = (mg > a.thresh) ? 1.f : 0.f, sn = (mg <= a.thresh) ? 1.f : 0.f;
            {   // compute_epe(gt_rigid, rigid_pred): gt (all channels, valid included) times the gt-resolution mask
                const float d0 = ug * sr - ur * fu, d1 = vg * sr - vr * fv, vv = valid * sr;
                acc[2] += sqrtf(d0 * d0 + d1 * d1) * vv;
                acc[3] += vv;
            }
            {
                const float d0 = ug * sn - un * fu, d1 = vg * sn - vn * fv, vv = valid * sn;
                acc[4] += sqrtf(d0 * d0 + d1 * d1) * vv;
                acc[5] += vv;
            }
        }
    }
    block_sum<8>(acc, scratch);
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < 8; ++k) a.partials[(long long)blockIdx.x * 8 + k] = acc[k];
}

// out[0..3] = all_epe, rigid_epe, non_rigid_epe, outlier ratio   (nc == 2: plain mean over B*Hg*Wg, :384-385)
__global__ void flow_metrics_finalize(const double* __restrict__ partials, int nblocks, int nc, long long npx, float* __restrict__ out) {
    CCB_PDL_WAIT();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double s[8];
    sum_partials(partials, nblocks, 8, s);
    if (nc == 3) {
        out[0] = (float)s[0] / ((float)s[1] + 1e-8f);
        out[1] = (float)s[2] / ((float)s[3] + 1e-8f);
        out[2] = (float)s[4] / ((float)s[5] + 1e-8f);
    } else {
        out[0] = (float)s[0] / (float)npx;
        out[1] = (float)s[2] / (float)npx;
        out[2] = (float)s[4] / (float)npx;
    }
    out[3] = (float)s[6] / ((float)s[1] + 1e-8f);
}

// ================================================================================================
// Depth metrics (compute_errors :430-467).  Per sample: valid = 0 < gt < 80 (and inside the Garg crop);
// pred clamped to [1e-3, 80]; pred *= median(gt) / median(pred) (torch.median = LOWER median); then
// abs_diff, abs_rel, sq_rel, a1, a2, a3, each a mean over the valid pixels, averaged over the batch.
struct DepthArgs {
    using Key = unsigned;            // the medians: the lower middle of gt and of the clamped pred
    static constexpr int SEL = 2;
    static constexpr unsigned UPPER = 0;
    const float* gt;
    const float* pred;
    int B, H, W, y1, y2, x1, x2;     // crop window (whole image when crop is off)
    MedianState med;
    double* partials;                // [B][blocks][6]
    float* out;                      // [6]
    __device__ __forceinline__ bool median_keys(int b, long long i, Key (&k)[SEL]) const;
};

__device__ __forceinline__ bool depth_valid(const DepthArgs& a, float g, int y, int x) {
    return (g > 0.f) && (g < 80.f) && (y >= a.y1) && (y < a.y2) && (x >= a.x1) && (x < a.x2);
}
__device__ __forceinline__ float clamp_pred(float p) { return fminf(fmaxf(p, 1e-3f), 80.f); }

__device__ __forceinline__ bool DepthArgs::median_keys(int b, long long i, Key (&k)[SEL]) const {
    const long long hw = (long long)H * W;
    const int y = (int)(i / W), x = (int)(i - (long long)y * W);
    const float g = __ldg(gt + b * hw + i);
    if (!depth_valid(*this, g, y, x)) return false;
    k[0] = ordered_key32(g);
    k[1] = ordered_key32(clamp_pred(__ldg(pred + b * hw + i)));
    return true;
}

__global__ void __launch_bounds__(256) depth_errors_kernel(const DepthArgs a) {
    CCB_PDL_WAIT();
    __shared__ double scratch[6 * 32];
    const int b = blockIdx.y;
    const long long hw = (long long)a.H * a.W;
    const float med_g = ordered_value32((unsigned)a.med.sel[(long long)b * 6]);
    const float med_p = ordered_value32((unsigned)a.med.sel[(long long)b * 6 + 3]);
    double acc[6] = {0, 0, 0, 0, 0, 0};
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < hw; i += (long long)gridDim.x * 256) {
        const int y = (int)(i / a.W), x = (int)(i - (long long)y * a.W);
        const float g = __ldg(a.gt + b * hw + i);
        if (!depth_valid(a, g, y, x)) continue;
        const float p = __fdiv_rn(__fmul_rn(clamp_pred(__ldg(a.pred + b * hw + i)), med_g), med_p);   // (p * med_g) / med_p
        const float th = fmaxf(__fdiv_rn(g, p), __fdiv_rn(p, g));
        const float d = fabsf(g - p);
        acc[0] += d;
        acc[1] += __fdiv_rn(d, g);
        acc[2] += __fdiv_rn((g - p) * (g - p), g);
        acc[3] += (th < 1.25f) ? 1.0 : 0.0;
        acc[4] += (th < 1.5625f) ? 1.0 : 0.0;
        acc[5] += (th < 1.953125f) ? 1.0 : 0.0;
    }
    block_sum<6>(acc, scratch);
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < 6; ++k) a.partials[((long long)b * gridDim.x + blockIdx.x) * 6 + k] = acc[k];
}

__global__ void depth_errors_finalize(const DepthArgs a, int nblocks) {
    CCB_PDL_WAIT();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double tot[6] = {0, 0, 0, 0, 0, 0};
    for (int b = 0; b < a.B; ++b) {
        double s[6];
        sum_partials(a.partials + (long long)b * nblocks * 6, nblocks, 6, s);
        const double n = (double)a.med.count[b];
        for (int j = 0; j < 6; ++j) tot[j] += (double)(float)(s[j] / n);      // per-sample fp32 means, summed (:453-463)
    }
    for (int j = 0; j < 6; ++j) a.out[j] = (float)(tot[j] / (double)a.B);
}

// ================================================================================================
// N1: uint8 HWC frames -> normalised fp32 NCHW, with per-sample flip / scale-crop.
//   src [B][F][Hs][Ws][3] uint8 (F frames per sample: target + references), dst F tensors [B][3][H][W] (dst[f]).
//   params [B][4] = {flip (0/1), scale_x = scaled_w / Ws, scale_y, unused}, offs [B][2] = {crop x0, crop y0} in the
//   scaled image.  RandomScaleCrop (custom_transforms.py:98-118): resize to (scaled_h, scaled_w) then crop H x W at
//   (y0, x0); the resize is sampled here as a bilinear lookup with half-pixel centres (PIL / scipy.misc.imresize
//   'bilinear' convention for up-scaling) - no uint8 re-quantisation of the resized image.  Flip is applied first
//   (custom_transforms.py:47-58), as in the reference's Compose order.   out = (v / 255 - 0.5) / 0.5.
struct PrepArgs {
    const unsigned char* src;
    float* dst[8];
    const float* params;
    const int* offs;
    int B, F, Hs, Ws, H, W;
};

// UNIT: ArrayToTensor alone (v / 255), for NormalizeLocally to follow; otherwise Normalize(.5, .5) as well.
template <bool UNIT>
__global__ void __launch_bounds__(256) prep_frames_kernel(const PrepArgs a) {
    CCB_PDL_WAIT();
    const long long n = (long long)a.B * a.F * a.H * a.W;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const int x = (int)(i % a.W);
        const int y = (int)((i / a.W) % a.H);
        const int f = (int)((i / ((long long)a.W * a.H)) % a.F);
        const int b = (int)(i / ((long long)a.W * a.H * a.F));
        const float flip = __ldg(a.params + b * 4), sx = __ldg(a.params + b * 4 + 1), sy = __ldg(a.params + b * 4 + 2);
        const int ox = __ldg(a.offs + b * 2), oy = __ldg(a.offs + b * 2 + 1);
        // coordinates in the scaled image -> source coordinates (half-pixel centres), clamped to the frame
        float fx = ((float)(x + ox) + 0.5f) / sx - 0.5f, fy = ((float)(y + oy) + 0.5f) / sy - 0.5f;
        fx = fminf(fmaxf(fx, 0.f), (float)(a.Ws - 1));
        fy = fminf(fmaxf(fy, 0.f), (float)(a.Hs - 1));
        const int x0 = (int)fx, y0 = (int)fy;
        const int x1 = min(x0 + 1, a.Ws - 1), y1 = min(y0 + 1, a.Hs - 1);
        const float wx = fx - (float)x0, wy = fy - (float)y0;
        const int xa = (flip != 0.f) ? (a.Ws - 1 - x0) : x0, xb = (flip != 0.f) ? (a.Ws - 1 - x1) : x1;
        const unsigned char* s = a.src + (((long long)b * a.F + f) * a.Hs) * a.Ws * 3;
        float* d = a.dst[f] + (long long)b * 3 * a.H * a.W + (long long)y * a.W + x;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float v00 = (float)s[((long long)y0 * a.Ws + xa) * 3 + c], v01 = (float)s[((long long)y0 * a.Ws + xb) * 3 + c];
            const float v10 = (float)s[((long long)y1 * a.Ws + xa) * 3 + c], v11 = (float)s[((long long)y1 * a.Ws + xb) * 3 + c];
            const float v = (1.f - wy) * ((1.f - wx) * v00 + wx * v01) + wy * ((1.f - wx) * v10 + wx * v11);
            d[(long long)c * a.H * a.W] = UNIT ? v / 255.f : (v / 255.f - 0.5f) / 0.5f;
        }
    }
}

// ================================================================================================
// RandomRotate (custom_transforms.py:75-85) = scipy.misc.imrotate = Pillow Image.rotate(angle, BILINEAR), restated from
// Pillow's ImagingGenericTransform with affine_transform and bilinear_filter32RGB.  affine [B][6] maps an output pixel
// centre to an input point (the host builds it as Pillow does, with cos / sin rounded to 15 decimals; the identity leaves a
// frame unchanged).  Every operation is an explicit _rn intrinsic: Pillow's x86-64 build does not fuse multiply-adds, and
// a fused one moves some samples across a uint8 truncation step.
struct RotArgs {
    const unsigned char* src;   // [B][F][H][W][3]
    const double* affine;       // [B][6]
    unsigned char* dst;         // [B][F][H][W][3]
    int B, F, H, W;
};

__global__ void __launch_bounds__(256) rotate_frames_kernel(const RotArgs a) {
    CCB_PDL_WAIT();
    const long long n = (long long)a.B * a.F * a.H * a.W;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const int x = (int)(i % a.W);
        const int y = (int)((i / a.W) % a.H);
        const long long bf = i / ((long long)a.W * a.H);
        const double* m = a.affine + (bf / a.F) * 6;
        const double xo = (double)x + 0.5, yo = (double)y + 0.5;
        double xin = __dadd_rn(__dadd_rn(__dmul_rn(__ldg(m + 0), xo), __dmul_rn(__ldg(m + 1), yo)), __ldg(m + 2));
        double yin = __dadd_rn(__dadd_rn(__dmul_rn(__ldg(m + 3), xo), __dmul_rn(__ldg(m + 4), yo)), __ldg(m + 5));
        unsigned char* d = a.dst + i * 3;
        if (xin < 0.0 || xin >= (double)a.W || yin < 0.0 || yin >= (double)a.H) {   // outside: the fill colour 0
            d[0] = 0; d[1] = 0; d[2] = 0;
            continue;
        }
        xin = __dsub_rn(xin, 0.5);
        yin = __dsub_rn(yin, 0.5);
        const int xf = (int)floor(xin), yf = (int)floor(yin);
        const double dx = __dsub_rn(xin, (double)xf), dy = __dsub_rn(yin, (double)yf);
        const int x0 = min(max(xf, 0), a.W - 1), x1 = min(max(xf + 1, 0), a.W - 1);
        const bool row2 = (yf + 1 >= 0) && (yf + 1 < a.H);          // first row clamped; a missing second row repeats it
        const unsigned char* r0 = a.src + (bf * a.H + min(max(yf, 0), a.H - 1)) * (long long)a.W * 3;
        const unsigned char* r1 = row2 ? a.src + (bf * a.H + yf + 1) * (long long)a.W * 3 : r0;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const int p0 = r0[x0 * 3 + c], p1 = r0[x1 * 3 + c];
            const double v1 = __dadd_rn((double)p0, __dmul_rn((double)(p1 - p0), dx));
            double v2 = v1;
            if (row2) {
                const int q0 = r1[x0 * 3 + c], q1 = r1[x1 * 3 + c];
                v2 = __dadd_rn((double)q0, __dmul_rn((double)(q1 - q0), dx));
            }
            d[c] = (unsigned char)(int)__dadd_rn(v1, __dmul_rn(__dsub_rn(v2, v1), dy));   // truncated, as Pillow's (UINT8) cast
        }
    }
}

// ================================================================================================
// Scale (custom_transforms.py:120-137) / RandomScaleCrop's resize = scipy.misc.imresize = Pillow resize(BILINEAR):
// ImagingResample with 8-bit precision.  Per axis, output index i takes input samples [xmin, xmin + cnt) with the
// triangle filter widened by the scale factor on a downscale (antialiasing), normalised, in 22-bit fixed point
// (precompute_coeffs / normalize_coeffs_8bpc).  The horizontal pass runs first and is rounded back to uint8; a pass whose
// size does not change is skipped.
constexpr int RESAMPLE_BITS = 22;

struct CoeffArgs {
    int in_x, out_x, ks_x, in_y, out_y, ks_y;
    int* kk_x; int* bounds_x;     // [out_x][ks_x] weights, [out_x][2] = {xmin, count}
    int* kk_y; int* bounds_y;
};

__device__ __forceinline__ double tri_filter(double t) {
    if (t < 0.0) t = -t;
    return (t < 1.0) ? __dsub_rn(1.0, t) : 0.0;
}

// one thread per output index of either axis (threads [0, out_x) the horizontal one), fp64 in Pillow's operation order
__global__ void resample_coeffs_kernel(const CoeffArgs a) {
    CCB_PDL_WAIT();
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    const bool hx = t < a.out_x;
    if (!hx) t -= a.out_x;
    const int in_size = hx ? a.in_x : a.in_y, out_size = hx ? a.out_x : a.out_y, ksize = hx ? a.ks_x : a.ks_y;
    if (t >= out_size) return;
    int* k = (hx ? a.kk_x : a.kk_y) + (long long)t * ksize;
    int* bounds = (hx ? a.bounds_x : a.bounds_y) + 2 * t;
    const double scale = __ddiv_rn((double)in_size, (double)out_size);
    const double support = scale < 1.0 ? 1.0 : scale;           // the triangle's support 1, times the filter scale
    const double ss = __ddiv_rn(1.0, support);
    const double center = __dmul_rn(__dadd_rn((double)t, 0.5), scale);
    const int xmin = max((int)__dadd_rn(__dsub_rn(center, support), 0.5), 0);
    const int cnt = min((int)__dadd_rn(__dadd_rn(center, support), 0.5), in_size) - xmin;
    double ww = 0.0;
    for (int x = 0; x < cnt; ++x)
        ww = __dadd_rn(ww, tri_filter(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss)));
    for (int x = 0; x < ksize; ++x) {
        int q = 0;
        if (x < cnt) {
            double w = tri_filter(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss));
            if (ww != 0.0) w = __ddiv_rn(w, ww);
            q = (int)__dadd_rn(0.5, __dmul_rn(w, (double)(1 << RESAMPLE_BITS)));
        }
        k[x] = q;
    }
    bounds[0] = xmin;
    bounds[1] = cnt;
}

// One pass over [outer][len][inner][3] uint8 along `len` (horizontal: inner 1; vertical: inner = row width).
struct ResampleArgs {
    const unsigned char* src;   // [outer][in_len][inner][3]
    unsigned char* dst;         // [outer][out_len][inner][3]
    const int* kk;              // [out_len][ksize]
    const int* bounds;          // [out_len][2]
    long long outer;
    int in_len, out_len, inner, ksize;
};

__device__ __forceinline__ unsigned char clip8(int v) {
    return (unsigned char)min(max(v >> RESAMPLE_BITS, 0), 255);
}

__global__ void __launch_bounds__(256) resample_pass_kernel(const ResampleArgs a) {
    CCB_PDL_WAIT();
    const long long n = a.outer * a.out_len * a.inner;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const int ii = (int)(i % a.inner);
        const int l = (int)((i / a.inner) % a.out_len);
        const long long o = i / ((long long)a.inner * a.out_len);
        const int xmin = __ldg(a.bounds + 2 * l), cnt = __ldg(a.bounds + 2 * l + 1);
        const int* k = a.kk + (long long)l * a.ksize;
        const long long step = (long long)a.inner * 3;
        const unsigned char* s = a.src + ((o * a.in_len + xmin) * a.inner + ii) * 3;
        int s0 = 1 << (RESAMPLE_BITS - 1), s1 = s0, s2 = s0;
        for (int j = 0; j < cnt; ++j) {
            const int kj = __ldg(k + j);
            s0 += (int)s[0] * kj;
            s1 += (int)s[1] * kj;
            s2 += (int)s[2] * kj;
            s += step;
        }
        unsigned char* d = a.dst + i * 3;
        d[0] = clip8(s0); d[1] = clip8(s1); d[2] = clip8(s2);
    }
}

// ================================================================================================
// NormalizeLocally (custom_transforms.py:33-44): per sample b and channel c, mean and unbiased std over the F frames'
// H x W values (fp64 block partials, fixed-order finalize: the same bits on every run), rounded to fp32; then
// x = (x - m) / s in fp32 (t.sub_(m).div_(s)).  A zero std gives inf / nan, as in the reference.
struct NormLocalArgs {
    float* x[8];                // F frames [B][3][H][W], normalised in place
    double* partials;           // [B*3][nblk][2]
    float* stats;               // [B][3][2] = {mean, std}
    int B, F;
    long long hw;
};

__global__ void __launch_bounds__(256) normlocal_partials_kernel(const NormLocalArgs a) {
    CCB_PDL_WAIT();
    __shared__ double scratch[2 * 32];
    const int bc = blockIdx.y;
    double acc[2] = {0.0, 0.0};
    for (int f = 0; f < a.F; ++f) {
        const float* p = a.x[f] + bc * a.hw;
        for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < a.hw; i += (long long)gridDim.x * 256) {
            const double v = (double)__ldg(p + i);
            acc[0] += v;
            acc[1] += v * v;
        }
    }
    block_sum<2>(acc, scratch);
    if (threadIdx.x == 0) {
        a.partials[((long long)bc * gridDim.x + blockIdx.x) * 2 + 0] = acc[0];
        a.partials[((long long)bc * gridDim.x + blockIdx.x) * 2 + 1] = acc[1];
    }
}

__global__ void normlocal_finalize_kernel(const NormLocalArgs a, int nblk) {
    CCB_PDL_WAIT();
    const int bc = blockIdx.x * blockDim.x + threadIdx.x;
    if (bc >= a.B * 3) return;
    double s[2];
    sum_partials(a.partials + (long long)bc * nblk * 2, nblk, 2, s);
    const double n = (double)a.F * (double)a.hw;
    const double mean = s[0] / n;
    const double var = (s[1] - s[0] * mean) / (n - 1.0);
    a.stats[bc * 2 + 0] = (float)mean;
    a.stats[bc * 2 + 1] = (float)sqrt(var);
}

__global__ void __launch_bounds__(256) normlocal_apply_kernel(const NormLocalArgs a) {
    CCB_PDL_WAIT();
    const int bc = blockIdx.y;
    const float m = a.stats[bc * 2 + 0], s = a.stats[bc * 2 + 1];
    for (int f = 0; f < a.F; ++f) {
        float* p = a.x[f] + bc * a.hw;
        for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < a.hw; i += (long long)gridDim.x * 256)
            p[i] = __fdiv_rn(__fsub_rn(p[i], m), s);
    }
}

// ================================================================================================
// Motion segmentation scores (test_mask.py:129-134 and mask_error :224-262).  Per sample, at the nets' resolution h x w:
//   bare     = 1 - (1 - e1)(1 - e2) > 0.5                        e1, e2: channels 1 and 2 of the mask net's eval output
//   soft     = 1 - d / max(d),  d = sqrt(sum_c (flow_cam - flow)^2)   the maximum over the sample's whole map
//   census   = soft > thresh,   combined = bare or census
// and, over the ground-truth grid Hg x Wg, the confusion matrix n[pred][gt] of each mask read at the source pixel that
// scipy.ndimage.zoom(order=0) reads, against gt = (obj_map != 0), counted where semantic_map == car_label.  A mask value 1
// (rigid) is class 0: argmax([mask, 1 - mask]).
// The census comparison decides integer counts, so d, the division and the subtraction are single correctly rounded
// fp32 operations (no contraction): the counts are those of an IEEE evaluation of the expressions, operation by operation.
// max(d) == 0 gives 0/0 = NaN and an empty census, as in the reference.
struct MaskIouArgs {
    const float* emask;             // [B, C, h, w]
    const float* flow_cam;          // [B, 2, h, w]
    const float* flow;              // [B, 2, h, w]
    const float* obj;               // [B, Hg, Wg]
    const float* sem;               // [B, Hg, Wg]
    float* masks;                   // [B, 4, h, w] or null
    unsigned long long* dmax;       // [B]: bit pattern of max(d), zero-extended
    unsigned long long* counts;     // [B, 3, 2, 2]
    int B, C, h, w, Hg, Wg;
    float thresh, car;
};

__device__ __forceinline__ float flow_gap(const MaskIouArgs& a, int b, long long p) {
    const long long hw = (long long)a.h * a.w;
    const float du = __fsub_rn(__ldg(a.flow_cam + 2ll * b * hw + p), __ldg(a.flow + 2ll * b * hw + p));
    const float dv = __fsub_rn(__ldg(a.flow_cam + (2ll * b + 1) * hw + p), __ldg(a.flow + (2ll * b + 1) * hw + p));
    return __fsqrt_rn(__fadd_rn(__fmul_rn(du, du), __fmul_rn(dv, dv)));
}

// bit 0 combined, bit 1 census, bit 2 bare of source pixel p
__device__ __forceinline__ unsigned mask_bits(const MaskIouArgs& a, int b, long long p, float dmax, float* soft_out) {
    const long long hw = (long long)a.h * a.w;
    const float e1 = __ldg(a.emask + ((long long)b * a.C + 1) * hw + p), e2 = __ldg(a.emask + ((long long)b * a.C + 2) * hw + p);
    const bool bare = __fsub_rn(1.f, __fmul_rn(__fsub_rn(1.f, e1), __fsub_rn(1.f, e2))) > 0.5f;
    const float soft = __fsub_rn(1.f, __fdiv_rn(flow_gap(a, b, p), dmax));
    const bool census = soft > a.thresh;
    *soft_out = soft;
    return ((bare || census) ? 1u : 0u) | (census ? 2u : 0u) | (bare ? 4u : 0u);
}

// max(d) per sample on the bit patterns: d is non-negative or NaN, so unsigned order is value order with NaN on top
// (torch's max propagates NaN too), and a maximum is the same in any order.
__global__ void __launch_bounds__(256) mask_iou_max_kernel(const MaskIouArgs a) {
    CCB_PDL_WAIT();
    const int b = blockIdx.y;
    const long long hw = (long long)a.h * a.w;
    unsigned m = 0;
    for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < hw; p += (long long)gridDim.x * 256) {
        const unsigned k = __float_as_uint(flow_gap(a, b, p));
        m = (k > m) ? k : m;
    }
    warp_max_into(a.dmax + b, m);
}

__global__ void __launch_bounds__(256) mask_iou_masks_kernel(const MaskIouArgs a) {
    CCB_PDL_WAIT();
    const int b = blockIdx.y;
    const long long hw = (long long)a.h * a.w;
    const float dmax = __uint_as_float((unsigned)a.dmax[b]);
    float* out = a.masks + 4ll * b * hw;
    for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < hw; p += (long long)gridDim.x * 256) {
        float soft;
        const unsigned bits = mask_bits(a, b, p, dmax, &soft);
        out[p] = (bits & 1u) ? 1.f : 0.f;
        out[hw + p] = (bits & 2u) ? 1.f : 0.f;
        out[2 * hw + p] = (bits & 4u) ? 1.f : 0.f;
        out[3 * hw + p] = soft;
    }
}

// scipy.ndimage.zoom(order=0) with its default grid_mode=False: output index o reads the input at coordinate
// o * (n_in - 1) / (n_out - 1), evaluated in fp64 as (quotient first, then the product) and rounded half up.
__device__ __forceinline__ int zoom_nearest(int o, double step, int n_in) {
    return min((int)floor(__dadd_rn(__dmul_rn((double)o, step), 0.5)), n_in - 1);
}

// One thread per ground-truth pixel; per-thread counters, one warp + block reduction at the end, then 64-bit integer
// atomics: integer sums do not depend on the order, so the counts are the same on every run.
__global__ void __launch_bounds__(256) mask_iou_count_kernel(const MaskIouArgs a) {
    CCB_PDL_WAIT();
    __shared__ unsigned scratch[12 * 8];
    const int b = blockIdx.y;
    const long long ng = (long long)a.Hg * a.Wg;
    const float dmax = __uint_as_float((unsigned)a.dmax[b]);
    const double step_y = (a.Hg > 1) ? __ddiv_rn((double)(a.h - 1), (double)(a.Hg - 1)) : 1.0;
    const double step_x = (a.Wg > 1) ? __ddiv_rn((double)(a.w - 1), (double)(a.Wg - 1)) : 1.0;
    unsigned n[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};      // [mask][pred][gt]
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < ng; i += (long long)gridDim.x * 256) {
        if (__ldg(a.sem + b * ng + i) != a.car) continue;        // the ignore label of mask_error
        const int y = (int)(i / a.Wg), x = (int)(i - (long long)y * a.Wg);
        const long long p = (long long)zoom_nearest(y, step_y, a.h) * a.w + zoom_nearest(x, step_x, a.w);
        float soft;
        const unsigned bits = mask_bits(a, b, p, dmax, &soft);
        const unsigned gt = (__ldg(a.obj + b * ng + i) != 0.f) ? 1u : 0u;
#pragma unroll
        for (int m = 0; m < 3; ++m) {
            const unsigned cell = (((bits >> m) & 1u) ? 0u : 2u) + gt;
#pragma unroll
            for (int k = 0; k < 4; ++k) n[m * 4 + k] += (cell == (unsigned)k) ? 1u : 0u;
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < 12; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) n[k] += __shfl_xor_sync(0xffffffffu, n[k], o);
        if (lane == 0) scratch[k * 8 + warp] = n[k];
    }
    __syncthreads();
    if (threadIdx.x < 12) {
        unsigned long long s = 0;
        for (int wi = 0; wi < 8; ++wi) s += scratch[threadIdx.x * 8 + wi];
        if (s) atomicAdd(a.counts + b * 12 + threadIdx.x, s);
    }
}

// ================================================================================================
// KITTI-2015 flow submission (submit_flow.py:119-156).  Per sample, at the nets' resolution h x w:
//   bare     = 1 - (1 - e1)(1 - e2) > 0.5,   census = |cam_u - fwd_u| < T and |cam_v - fwd_v| < T
//   combined = 1 - (1 - bare)(1 - census)                       (0 or 1; its bilinear resize to h x w is the identity)
//   total    = (combined <= T) * fwd + (combined > T) * cam
// then total, fwd and cam each resized bilinearly to Hg x Wg and u, v scaled by (float)(Wg / w), (float)(Hg / h).
// The resize restates torch's CPU upsample_bilinear2d(align_corners=False) for float NCHW operation by operation: source
// index fma(in/out, dst + 0.5, -0.5) clamped at 0, lambda1 = src - floor(src), lambda0 = 1 - lambda1, and per axis
// fma(v0, lambda0, v1 * lambda1), the x axis inside the y axis.  Each output pixel composites its four taps.
struct FlowSubmitArgs {
    const float* emask;             // [B, C, h, w]
    const float* cam;               // [B, 2, h, w]
    const float* fwd;               // [B, 2, h, w]
    float* mask;                    // [B, 1, h, w]
    float* full;                    // [B, 3, 2, Hg, Wg] cam, fwd, total, or null
    unsigned short* png;            // [B, Hg, Wg, 3]
    float* flo;                     // [B, Hg, Wg, 2]
    int B, C, h, w, Hg, Wg;
    float thresh, fu, fv;
};

struct Tap { int i0, i1; float l0, l1; };
__device__ __forceinline__ Tap aten_tap(int dst, int in_size, float scale) {
    float s = __fmaf_rn(scale, __fadd_rn((float)dst, 0.5f), -0.5f);
    if (s < 0.f) s = 0.f;
    Tap t;
    t.i0 = min((int)floorf(s), in_size - 1);
    t.i1 = t.i0 + ((t.i0 < in_size - 1) ? 1 : 0);
    t.l1 = fminf(fmaxf(__fsub_rn(s, (float)t.i0), 0.f), 1.f);
    t.l0 = __fsub_rn(1.f, t.l1);
    return t;
}
__device__ __forceinline__ float aten_lerp(float v0, float v1, float l0, float l1) {
    return __fmaf_rn(v0, l0, __fmul_rn(v1, l1));
}

__device__ __forceinline__ float submit_combined(const FlowSubmitArgs& a, int b, long long p) {
    const long long hw = (long long)a.h * a.w;
    const float e1 = __ldg(a.emask + ((long long)b * a.C + 1) * hw + p), e2 = __ldg(a.emask + ((long long)b * a.C + 2) * hw + p);
    const bool bare = __fsub_rn(1.f, __fmul_rn(__fsub_rn(1.f, e1), __fsub_rn(1.f, e2))) > 0.5f;
    const float* c = a.cam + 2ll * b * hw + p;
    const float* f = a.fwd + 2ll * b * hw + p;
    const bool census = (fabsf(__fsub_rn(__ldg(c), __ldg(f))) < a.thresh) && (fabsf(__fsub_rn(__ldg(c + hw), __ldg(f + hw))) < a.thresh);
    return (bare || census) ? 1.f : 0.f;
}

__global__ void __launch_bounds__(256) flow_submit_mask_kernel(const FlowSubmitArgs a) {
    CCB_PDL_WAIT();
    const long long hw = (long long)a.h * a.w, n = (long long)a.B * hw;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
        a.mask[i] = submit_combined(a, (int)(i / hw), i % hw);
}

// numpy's float64 -> uint16 cast on x86-64: truncation to int32 (cvttsd2si; NaN and values outside the int32 range give
// INT_MIN), then the low 16 bits.
__device__ __forceinline__ unsigned short kitti_u16(float v) {
    const double x = __dadd_rn(__dmul_rn((double)v, 64.0), 32768.0);
    const int t = (x > -2147483649.0 && x < 2147483648.0) ? (int)x : (int)0x80000000u;
    return (unsigned short)((unsigned)t & 0xffffu);
}

__global__ void __launch_bounds__(256) flow_submit_kernel(const FlowSubmitArgs a) {
    CCB_PDL_WAIT();
    const long long hw = (long long)a.h * a.w, ng = (long long)a.Hg * a.Wg, n = (long long)a.B * ng;
    const float sy = (float)a.h / (float)a.Hg, sx = (float)a.w / (float)a.Wg;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const int b = (int)(i / ng);
        const long long q = i - (long long)b * ng;
        const int y = (int)(q / a.Wg), x = (int)(q - (long long)y * a.Wg);
        const Tap ty = aten_tap(y, a.h, sy), tx = aten_tap(x, a.w, sx);
        const long long taps[4] = {(long long)ty.i0 * a.w + tx.i0, (long long)ty.i0 * a.w + tx.i1,
                                   (long long)ty.i1 * a.w + tx.i0, (long long)ty.i1 * a.w + tx.i1};
        float v[3][2][4];       // [cam, fwd, total][u, v][tap]
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float m = submit_combined(a, b, taps[k]);
            const float sr = (m > a.thresh) ? 1.f : 0.f, sn = (m <= a.thresh) ? 1.f : 0.f;
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const float cam = __ldg(a.cam + (2ll * b + c) * hw + taps[k]), fwd = __ldg(a.fwd + (2ll * b + c) * hw + taps[k]);
                v[0][c][k] = cam;
                v[1][c][k] = fwd;
                v[2][c][k] = __fadd_rn(__fmul_rn(sn, fwd), __fmul_rn(sr, cam));
            }
        }
        float o[3][2];
#pragma unroll
        for (int f = 0; f < 3; ++f)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const float r0 = aten_lerp(v[f][c][0], v[f][c][1], tx.l0, tx.l1);
                const float r1 = aten_lerp(v[f][c][2], v[f][c][3], tx.l0, tx.l1);
                o[f][c] = __fmul_rn(aten_lerp(r0, r1, ty.l0, ty.l1), c == 0 ? a.fu : a.fv);
            }
        if (a.full)
#pragma unroll
            for (int f = 0; f < 3; ++f) {
                a.full[((3ll * b + f) * 2 + 0) * ng + q] = o[f][0];
                a.full[((3ll * b + f) * 2 + 1) * ng + q] = o[f][1];
            }
        a.png[3 * i + 0] = kitti_u16(o[2][0]);
        a.png[3 * i + 1] = kitti_u16(o[2][1]);
        a.png[3 * i + 2] = 1;
        a.flo[2 * i + 0] = o[2][0];
        a.flo[2 * i + 1] = o[2][1];
    }
}

// ================================================================================================
// Middlebury flow colours (flowlib.py flow_to_image :189-226, compute_color :345-386, make_color_wheel :389-436).
// Per image, P panels of [2, H, W] stacked along H (np.hstack of CHW arrays) share one maximum radius:
//   pass 1  |u| or |v| > 1e7 (fp32) -> unknown, zeroed; rad = sqrt(u^2 + v^2) in fp32; maxrad = max(rad), and any NaN
//           makes python's max(-1, nan) -1
//   pass 2  u / (maxrad + DBL_EPSILON) in fp64, then the colour wheel in fp64; NaN and unknown pixels are black.
// The levels are floor(255 * col) as uint8 (the reference returns them / 255).
__constant__ double c_wheel[55][3] = {      // RY 15, YG 6, GC 4, CB 11, BM 13, MR 6 steps; ramps floor(255 k / n)
    {255, 0, 0}, {255, 17, 0}, {255, 34, 0}, {255, 51, 0}, {255, 68, 0}, {255, 85, 0}, {255, 102, 0}, {255, 119, 0},
    {255, 136, 0}, {255, 153, 0}, {255, 170, 0}, {255, 187, 0}, {255, 204, 0}, {255, 221, 0}, {255, 238, 0},
    {255, 255, 0}, {213, 255, 0}, {170, 255, 0}, {128, 255, 0}, {85, 255, 0}, {43, 255, 0},
    {0, 255, 0}, {0, 255, 63}, {0, 255, 127}, {0, 255, 191},
    {0, 255, 255}, {0, 232, 255}, {0, 209, 255}, {0, 186, 255}, {0, 163, 255}, {0, 140, 255}, {0, 116, 255},
    {0, 93, 255}, {0, 70, 255}, {0, 47, 255}, {0, 24, 255},
    {0, 0, 255}, {19, 0, 255}, {39, 0, 255}, {58, 0, 255}, {78, 0, 255}, {98, 0, 255}, {117, 0, 255}, {137, 0, 255},
    {156, 0, 255}, {176, 0, 255}, {196, 0, 255}, {215, 0, 255}, {235, 0, 255},
    {255, 0, 255}, {255, 0, 213}, {255, 0, 170}, {255, 0, 128}, {255, 0, 85}, {255, 0, 43}};

struct FlowColorArgs {
    const float* flow;              // [B, P, 2, H, W]
    unsigned long long* maxrad;     // [B]: bit pattern of max(rad), ~0 for NaN
    unsigned char* out;             // [B, 3, P*H, W]
    int B, P, H, W;
};

__device__ __forceinline__ bool flow_unknown(float u, float v) { return fabsf(u) > 1e7f || fabsf(v) > 1e7f; }

__global__ void __launch_bounds__(256) flow_color_max_kernel(const FlowColorArgs a) {
    CCB_PDL_WAIT();
    const int b = blockIdx.y;
    const long long hw = (long long)a.H * a.W, n = (long long)a.P * hw;
    unsigned long long m = 0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const long long pnl = i / hw, p = i - pnl * hw;
        const float* f = a.flow + ((long long)b * a.P + pnl) * 2 * hw + p;
        float u = __ldg(f), v = __ldg(f + hw);
        if (flow_unknown(u, v)) u = v = 0.f;
        const float rad = __fsqrt_rn(__fadd_rn(__fmul_rn(u, u), __fmul_rn(v, v)));
        const unsigned long long k = (rad != rad) ? ~0ull : (unsigned long long)__float_as_uint(rad);
        m = (k > m) ? k : m;
    }
    warp_max_into(a.maxrad + b, m);
}

__global__ void __launch_bounds__(256) flow_color_kernel(const FlowColorArgs a) {
    CCB_PDL_WAIT();
    const int b = blockIdx.y;
    const long long hw = (long long)a.H * a.W, n = (long long)a.P * hw;
    const unsigned long long mk = a.maxrad[b];
    const double den = __dadd_rn(mk == ~0ull ? -1.0 : (double)__uint_as_float((unsigned)mk), 2.220446049250313e-16);
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const long long pnl = i / hw, p = i - pnl * hw;
        const float* f = a.flow + ((long long)b * a.P + pnl) * 2 * hw + p;
        float uf = __ldg(f), vf = __ldg(f + hw);
        const bool unknown = flow_unknown(uf, vf);
        if (unknown) uf = vf = 0.f;
        double u = __ddiv_rn((double)uf, den), v = __ddiv_rn((double)vf, den);
        const bool nan = (u != u) || (v != v);
        if (nan) u = v = 0.0;
        const double rad = __dsqrt_rn(__dadd_rn(__dmul_rn(u, u), __dmul_rn(v, v)));
        const double ang = __ddiv_rn(atan2(-v, -u), 3.141592653589793);
        const double fk = __dadd_rn(__dmul_rn(__ddiv_rn(__dadd_rn(ang, 1.0), 2.0), 54.0), 1.0);
        const int k0 = min(max((int)floor(fk), 1), 55);
        const int k1 = (k0 + 1 == 56) ? 1 : k0 + 1;
        const double fr = __dsub_rn(fk, (double)k0);
        unsigned char* o = a.out + (long long)b * 3 * n + i;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const double col0 = __ddiv_rn(c_wheel[k0 - 1][c], 255.0), col1 = __ddiv_rn(c_wheel[k1 - 1][c], 255.0);
            double col = __dadd_rn(__dmul_rn(__dsub_rn(1.0, fr), col0), __dmul_rn(fr, col1));
            col = (rad <= 1.0) ? __dsub_rn(1.0, __dmul_rn(rad, __dsub_rn(1.0, col))) : __dmul_rn(col, 0.75);
            const double level = floor(__dmul_rn(__dmul_rn(255.0, col), nan ? 0.0 : 1.0));
            o[c * n] = unknown ? (unsigned char)0 : (unsigned char)(int)level;
        }
    }
}

// ================================================================================================
// KITTI flow scores of decoded 16-bit PNGs (evaluate_flow.py compute_err :44-53, flow_io.flow_read_png :96-117), fp64:
//   u = (U - 2^15) / 64,  epe = sqrt(du^2 + dv^2) * valid_gt,  aepe = sum(epe) / sum(valid_gt)
//   Fl = sum([epe > 3] [epe / (|F_gt| + 1e-8) > 0.05] valid_gt) / sum(valid_gt)
// Per-block fp64 partials (the two counts are integers, exact in fp64 below 2^53), one fixed-order finalize per image.
struct KittiErrArgs {
    const unsigned short* gt;       // [B, H, W, 3]
    const unsigned short* pred;     // [B, H, W, 3]
    double* partials;               // [B][blocks][3]: sum epe, sum valid, outliers
    double* out;                    // [B, 2]
    long long* counts;              // [B, 2] outliers, valid; or null
    int B, H, W;
};

__global__ void __launch_bounds__(256) kitti_err_kernel(const KittiErrArgs a) {
    CCB_PDL_WAIT();
    __shared__ double scratch[3 * 32];
    const int b = blockIdx.y;
    const long long n = (long long)a.H * a.W;
    double acc[3] = {0, 0, 0};
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
        const unsigned short* g = a.gt + 3 * (b * n + i);
        const unsigned short* p = a.pred + 3 * (b * n + i);
        const double ug = __ddiv_rn((double)g[0] - 32768.0, 64.0), vg = __ddiv_rn((double)g[1] - 32768.0, 64.0);
        const double up = __ddiv_rn((double)p[0] - 32768.0, 64.0), vp = __ddiv_rn((double)p[1] - 32768.0, 64.0);
        const double valid = (double)g[2];
        const double du = __dsub_rn(ug, up), dv = __dsub_rn(vg, vp);
        const double epe = __dmul_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(du, du), __dmul_rn(dv, dv))), valid);
        const double mag = __dsqrt_rn(__dadd_rn(__dmul_rn(ug, ug), __dmul_rn(vg, vg)));
        acc[0] += epe;
        acc[1] += valid;
        if (epe > 3.0 && __ddiv_rn(epe, __dadd_rn(mag, 1e-8)) > 0.05) acc[2] += valid;
    }
    block_sum<3>(acc, scratch);
    if (threadIdx.x == 0) {
        double* o = a.partials + ((long long)b * gridDim.x + blockIdx.x) * 3;
        o[0] = acc[0]; o[1] = acc[1]; o[2] = acc[2];
    }
}

__global__ void kitti_err_finalize(const KittiErrArgs a, int nblk) {
    CCB_PDL_WAIT();
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.B) return;
    double s[3];
    sum_partials(a.partials + (long long)b * nblk * 3, nblk, 3, s);
    a.out[2 * b + 0] = __ddiv_rn(s[0], s[1]);
    a.out[2 * b + 1] = __ddiv_rn(s[2], s[1]);
    if (a.counts) {
        a.counts[2 * b + 0] = (long long)s[2];
        a.counts[2 * b + 1] = (long long)s[1];
    }
}

// ================================================================================================
// KITTI depth ground truth from a velodyne sweep (kitti_eval/depth_evaluation_utils.py generate_depth_map :148-191), fp64:
//   keep x >= 0;  (X, Y, Z) = P_velo2im (x, y, z, 1), each row summed as OpenBLAS's dgemm sums it (an fma chain over the
//   columns);  u = rint(X / Z) - 1, v = rint(Y / Z) - 1 (numpy's round: half to even);  keep 0 <= u < W, 0 <= v < H
//   depth[v, u] = Z of the LAST kept point on the pixel (numpy's fancy assignment)
//   duplicates grouped by the reference's sub2ind key v * (W - 1) + u - 1 (which also joins (v, W-1) with (v+1, 0)): for a
//   key with more than one point, the pixel of its FIRST point gets the least Z of the group;  finally depth < 0 -> 0.
// Integer atomics only (largest index, count, smallest index, least Z as an order-preserving key): the same bits on every
// run.  Pass 1 scatters the points, pass 2 writes every pixel.
struct VeloArgs {
    const float* pts;               // [total, 4]; column 3 is not read (the reference sets it to 1)
    const long long* offs;          // [B + 1] first point of each sample
    const double* P;                // [B, 3, 4]
    unsigned long long* last;       // [B, H*W]   1 + index of the last kept point on the pixel, 0 for none
    unsigned long long* cnt;        // [B, K]     kept points per key, indexed by key + 1 (K = H*(W-1) + 1 keys)
    unsigned long long* first;      // [B, K]     ~index of the first point of the key
    unsigned long long* zmin;       // [B, K]     ~ordered key of the least Z of the key
    double* depth;                  // [B, H, W]
    long long total;
    int B, H, W;
};

struct VeloPt { double z; int u, v; bool keep; };

__device__ __forceinline__ VeloPt velo_project(const VeloArgs& a, int b, long long i) {
    VeloPt r;
    r.keep = false; r.u = r.v = 0; r.z = 0.0;
    const float* q = a.pts + 4 * i;
    if (!(__ldg(q) >= 0.f)) return r;
    const double x = (double)__ldg(q), y = (double)__ldg(q + 1), z = (double)__ldg(q + 2);
    const double* P = a.P + 12ll * b;
    double c[3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
        c[k] = __dadd_rn(__fma_rn(__ldg(P + 4 * k + 2), z, __fma_rn(__ldg(P + 4 * k + 1), y, __dmul_rn(__ldg(P + 4 * k), x))),
                         __ldg(P + 4 * k + 3));
    const double u = __dsub_rn(rint(__ddiv_rn(c[0], c[2])), 1.0), v = __dsub_rn(rint(__ddiv_rn(c[1], c[2])), 1.0);
    if (!(u >= 0.0 && v >= 0.0 && u < (double)a.W && v < (double)a.H)) return r;
    r.keep = true; r.u = (int)u; r.v = (int)v; r.z = c[2];
    return r;
}

__device__ __forceinline__ bool velo_range(const VeloArgs& a, int b, long long* i0, long long* i1) {
    *i0 = a.offs[b];
    *i1 = a.offs[b + 1];
    return *i0 >= 0 && *i0 <= *i1 && *i1 <= a.total;       // malformed offsets: the sample gets no point
}

__global__ void __launch_bounds__(256) velo_scatter_kernel(const VeloArgs a) {
    CCB_PDL_WAIT();
    const int b = blockIdx.y;
    long long i0, i1;
    if (!velo_range(a, b, &i0, &i1)) return;
    const long long hw = (long long)a.H * a.W, K = (long long)a.H * (a.W - 1) + 1;
    for (long long i = i0 + (long long)blockIdx.x * 256 + threadIdx.x; i < i1; i += (long long)gridDim.x * 256) {
        const VeloPt p = velo_project(a, b, i);
        if (!p.keep) continue;
        const long long key = (long long)p.v * (a.W - 1) + p.u;     // sub2ind + 1
        atomicMax(a.last + b * hw + (long long)p.v * a.W + p.u, (unsigned long long)(i - i0 + 1));
        atomicAdd(a.cnt + b * K + key, 1ull);
        atomicMax(a.first + b * K + key, ~(unsigned long long)(i - i0));
        atomicMax(a.zmin + b * K + key, ~ordered_key(p.z));       // a NaN z never gets here: its u fails the bounds
    }
}

__global__ void __launch_bounds__(256) velo_depth_kernel(const VeloArgs a) {
    CCB_PDL_WAIT();
    const int b = blockIdx.y;
    long long i0, i1;
    const bool ok = velo_range(a, b, &i0, &i1);
    const long long hw = (long long)a.H * a.W, K = (long long)a.H * (a.W - 1) + 1;
    for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < hw; p += (long long)gridDim.x * 256) {
        double d = 0.0;
        const unsigned long long last = ok ? a.last[b * hw + p] : 0ull;
        if (last) {
            d = velo_project(a, b, i0 + (long long)last - 1).z;
            const int v = (int)(p / a.W), u = (int)(p - (long long)v * a.W);
            const long long key = (long long)v * (a.W - 1) + u;
            if (a.cnt[b * K + key] > 1) {
                const VeloPt f = velo_project(a, b, i0 + (long long)~a.first[b * K + key]);
                if (f.v == v && f.u == u) d = ordered_value(~a.zmin[b * K + key]);
            }
        }
        a.depth[b * hw + p] = (d < 0.0) ? 0.0 : d;
    }
}

// ================================================================================================
// scipy.ndimage.zoom(x, (H/h, W/w), order=3) (mode 'constant', grid_mode False, prefilter on) of fp32 images, in fp64:
//   prefilter  per axis (0 then 1) the cubic B-spline recursion, pole z = sqrt(3) - 2, gain (1 - z)(1 - 1/z), causal and
//              anti-causal initialisation with the mirror boundary (scipy's ni_splines.c for mode 'constant'); a line of
//              length 1 is left as it is
//   evaluate   at o * ((n - 1) / (m - 1)) per axis (1 when m == 1), 4 x 4 tensor-product B-spline weights, coefficient
//              indices outside the line mirrored
// then rounded to fp32 and clipped to [lo, hi] in fp32 (numpy's clip: NaN stays NaN).  One fp64 thread per line for the
// recursions, one thread per output pixel for the evaluation.
struct ZoomArgs {
    const float* src;               // [N, h, w]
    double* coef;                   // [N, h, w]
    float* dst;                     // [N, H, W]
    int N, h, w, H, W;
    float lo, hi;
};

__device__ __forceinline__ void spline_line(double* c, int n, long long stride) {
    if (n == 1) return;
    const double z = -0.2679491924311227;       // sqrt(3) - 2
    const double gain = (1.0 - z) * (1.0 - 1.0 / z);
    for (int i = 0; i < n; ++i) c[i * stride] *= gain;
    const double zn1 = pow(z, (double)(n - 1));
    double c0 = c[0] + zn1 * c[(long long)(n - 1) * stride];
    double zi = z;
    for (int i = 1; i < n - 1; ++i) {
        c0 += zi * (c[i * stride] + zn1 * c[(long long)(n - 1 - i) * stride]);
        zi *= z;
    }
    c[0] = c0 / (1.0 - zn1 * zn1);
    for (int i = 1; i < n; ++i) c[i * stride] += z * c[(i - 1) * stride];
    c[(long long)(n - 1) * stride] = (z * c[(long long)(n - 2) * stride] + c[(long long)(n - 1) * stride]) * z / (z * z - 1.0);
    for (int i = n - 2; i >= 0; --i) c[i * stride] = z * (c[(i + 1) * stride] - c[i * stride]);
}

// pass 0: one thread per column (copies the input and filters along axis 0); pass 1: one thread per row (axis 1)
__global__ void __launch_bounds__(256) zoom_prefilter_kernel(const ZoomArgs a, int pass) {
    CCB_PDL_WAIT();
    const long long hw = (long long)a.h * a.w;
    const long long nlines = (long long)a.N * (pass == 0 ? a.w : a.h);
    for (long long t = (long long)blockIdx.x * 256 + threadIdx.x; t < nlines; t += (long long)gridDim.x * 256) {
        if (pass == 0) {
            const long long n = t / a.w, x = t - n * a.w;
            double* c = a.coef + n * hw + x;
            const float* s = a.src + n * hw + x;
            for (int y = 0; y < a.h; ++y) c[(long long)y * a.w] = (double)__ldg(s + (long long)y * a.w);
            spline_line(c, a.h, a.w);
        } else {
            spline_line(a.coef + t * a.w, a.w, 1);
        }
    }
}

// scipy's mirror of a coefficient index (period 2n - 2; a line of length 1 has one coefficient)
__device__ __forceinline__ int mirror_index(int j, int n) {
    if (n == 1) return 0;
    const int period = 2 * n - 2;
    j = j % period;
    if (j < 0) j += period;
    return (j >= n) ? period - j : j;
}

__device__ __forceinline__ void cubic_weights(double t, double (&wt)[4]) {
    const double s = 1.0 - t;
    wt[0] = s * s * s / 6.0;
    wt[1] = (t * t * (t - 2.0) * 3.0 + 4.0) / 6.0;
    wt[2] = (s * s * (s - 2.0) * 3.0 + 4.0) / 6.0;
    wt[3] = t * t * t / 6.0;
}

__global__ void __launch_bounds__(256) zoom_eval_kernel(const ZoomArgs a) {
    CCB_PDL_WAIT();
    const long long HW = (long long)a.H * a.W, n_out = (long long)a.N * HW;
    const double step_y = (a.H > 1) ? (double)(a.h - 1) / (double)(a.H - 1) : 1.0;
    const double step_x = (a.W > 1) ? (double)(a.w - 1) / (double)(a.W - 1) : 1.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n_out; i += (long long)gridDim.x * 256) {
        const long long n = i / HW, q = i - n * HW;
        const int oy = (int)(q / a.W), ox = (int)(q - (long long)oy * a.W);
        const double cy = __dmul_rn((double)oy, step_y), cx = __dmul_rn((double)ox, step_x);
        const double fy = floor(cy), fx = floor(cx);
        double wy[4], wx[4];
        cubic_weights(cy - fy, wy);
        cubic_weights(cx - fx, wx);
        int xs[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) xs[k] = mirror_index((int)fx - 1 + k, a.w);
        const double* c = a.coef + n * a.h * (long long)a.w;
        double acc = 0.0;
#pragma unroll
        for (int ky = 0; ky < 4; ++ky) {
            const double* row = c + (long long)mirror_index((int)fy - 1 + ky, a.h) * a.w;
            double r = 0.0;
#pragma unroll
            for (int kx = 0; kx < 4; ++kx) r += wx[kx] * row[xs[kx]];
            acc += wy[ky] * r;
        }
        const float v = (float)acc;
        a.dst[i] = (v < a.lo) ? a.lo : ((v > a.hi) ? a.hi : v);
    }
}

// ================================================================================================
// One sample of test_disp.py:124-141 + compute_errors :171-187, in fp64.  mask = min_depth < gt < max_depth inside the
// crop rows [y1, y2) and columns [x1, x2);  per row r of the output the prediction is (double)pred * scale_r:
//   row 1  scale = median(gt[mask]) / median(pred[mask]), numpy medians (an even count averages the two middle values, in
//          fp64 for gt and in fp32 for the fp32 prediction)
//   row 0  scale = mean(s1 / |pose[:3]|) over the references with s1 > 0 (0 when there is none); zeros without poses
//   errors abs_rel sq_rel rms log_rms a1 a2 a3;  a* are exact counts over n, the rest fp64 block partials summed in a
//          fixed order.
// The medians: the lower and upper middle of gt and of pred.
struct EigenArgs {
    using Key = unsigned long long;
    static constexpr int SEL = 4;                   // gt lower, gt upper, pred lower, pred upper
    static constexpr unsigned UPPER = 0xa;
    const double* gt;               // [B, H, W]
    const float* pred;              // [B, H, W]
    const float* poses;             // [B, R, 6] or null
    const double* disp;             // [B, R] or null
    MedianState med;
    double* scale;                  // [B][2]
    double* partials;               // [B][blocks][2][7]
    double* out;                    // [B, 2, 7]
    double min_depth, max_depth;
    double cap;                     // scaled predictions above it become it (test_make3d.py:147; +inf: no cap)
    int log10;                      // log_rms of log10 (test_make3d.py:183) instead of ln
    int B, H, W, R, y1, y2, x1, x2;
    __device__ __forceinline__ bool median_keys(int b, long long i, Key (&k)[SEL]) const;
};

__device__ __forceinline__ bool eigen_valid(const EigenArgs& a, double g, int y, int x) {
    return (g > a.min_depth) && (g < a.max_depth) && (y >= a.y1) && (y < a.y2) && (x >= a.x1) && (x < a.x2);
}

__device__ __forceinline__ bool EigenArgs::median_keys(int b, long long i, Key (&k)[SEL]) const {
    const long long hw = (long long)H * W;
    const int y = (int)(i / W), x = (int)(i - (long long)y * W);
    const double g = __ldg(gt + b * hw + i);
    if (!eigen_valid(*this, g, y, x)) return false;
    k[0] = k[1] = ordered_key(g);
    k[2] = k[3] = ordered_key32(__ldg(pred + b * hw + i));
    return true;
}

// one thread per sample: both scales
__global__ void eigen_scale_kernel(const EigenArgs a) {
    CCB_PDL_WAIT();
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.B) return;
    const unsigned long long* s = a.med.sel + (long long)b * 12;
    const double g0 = ordered_value(s[0]), g1 = ordered_value(s[3]);
    const float p0 = ordered_value32((unsigned)s[6]), p1 = ordered_value32((unsigned)s[9]);
    const bool even = (a.med.count[b] & 1ull) == 0;
    const double med_g = even ? __ddiv_rn(__dadd_rn(g0, g1), 2.0) : g0;
    const float med_p = even ? __fdiv_rn(__fadd_rn(p0, p1), 2.f) : p0;
    a.scale[2 * b + 1] = __ddiv_rn(med_g, (double)med_p);
    double sum = 0.0;
    int n = 0;
    if (a.poses)
        for (int r = 0; r < a.R; ++r) {
            const double s1 = a.disp[(long long)b * a.R + r];
            if (!(s1 > 0.0)) continue;
            const float* p = a.poses + ((long long)b * a.R + r) * 6;
            const double x = p[0], y = p[1], z = p[2];
            const float norm = (float)__dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
            sum = __dadd_rn(sum, __ddiv_rn(s1, (double)norm));
            ++n;
        }
    a.scale[2 * b] = n ? __ddiv_rn(sum, (double)n) : 0.0;
}

__device__ __forceinline__ double nan_max(double p, double q) { return (p != p || p > q) ? p : q; }   // np.maximum

__global__ void __launch_bounds__(256) eigen_errors_kernel(const EigenArgs a) {
    CCB_PDL_WAIT();
    __shared__ double scratch[14 * 32];
    const int b = blockIdx.y;
    const long long hw = (long long)a.H * a.W;
    const int r0 = a.poses ? 0 : 1;
    const double sc[2] = {a.scale[2 * b], a.scale[2 * b + 1]};
    double acc[14];
#pragma unroll
    for (int k = 0; k < 14; ++k) acc[k] = 0.0;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < hw; i += (long long)gridDim.x * 256) {
        const int y = (int)(i / a.W), x = (int)(i - (long long)y * a.W);
        const double g = __ldg(a.gt + b * hw + i);
        if (!eigen_valid(a, g, y, x)) continue;
        const double p32 = (double)__ldg(a.pred + b * hw + i);
        const double lg = a.log10 ? log10(g) : log(g);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            if (r < r0) continue;
            double p = __dmul_rn(p32, sc[r]);
            if (p > a.cap) p = a.cap;
            const double th = nan_max(__ddiv_rn(g, p), __ddiv_rn(p, g));
            const double d = __dsub_rn(g, p), d2 = __dmul_rn(d, d), dl = __dsub_rn(lg, a.log10 ? log10(p) : log(p));
            double* o = acc + 7 * r;
            o[0] += __ddiv_rn(fabs(d), g);
            o[1] += __ddiv_rn(d2, g);
            o[2] += d2;
            o[3] += __dmul_rn(dl, dl);
            o[4] += (th < 1.25) ? 1.0 : 0.0;
            o[5] += (th < 1.5625) ? 1.0 : 0.0;
            o[6] += (th < 1.953125) ? 1.0 : 0.0;
        }
    }
    block_sum<14>(acc, scratch);
    if (threadIdx.x == 0) {
        double* o = a.partials + ((long long)b * gridDim.x + blockIdx.x) * 14;
#pragma unroll
        for (int k = 0; k < 14; ++k) o[k] = acc[k];
    }
}

// one thread per (sample, row), the block partials in block order
__global__ void eigen_finalize_kernel(const EigenArgs a, int nblk) {
    CCB_PDL_WAIT();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.B * 2) return;
    const int b = t >> 1, r = t & 1;
    double* o = a.out + (long long)t * 7;
    if (r == 0 && !a.poses) {
        for (int k = 0; k < 7; ++k) o[k] = 0.0;
        return;
    }
    double s[7];
    sum_partials(a.partials + (long long)b * nblk * 14 + 7 * r, nblk, 14, s);
    const double n = (double)a.med.count[b];
    o[0] = __ddiv_rn(s[0], n);
    o[1] = __ddiv_rn(s[1], n);
    o[2] = __dsqrt_rn(__ddiv_rn(s[2], n));
    o[3] = __dsqrt_rn(__ddiv_rn(s[3], n));
    for (int j = 4; j < 7; ++j) o[j] = __ddiv_rn(s[j], n);
}

// ================================================================================================
// The contrast stretch scipy.misc.imresize gives a float32 image before Pillow resizes it (test_make3d.py:100-102; scipy
// 1.1 imresize -> toimage -> bytescale): over the whole HxWx3 image, in float32 with each operation rounded on its own,
//   cscale = cmax - cmin (1 when 0), scale = 255 / cscale, u8 = trunc(clip((x - cmin) * scale, 0, 255) + 0.5).
// The frames hold the integers 0..255, so a table of the 256 values is the whole map.  The range is taken with integer
// atomics (the largest value and the largest 255 - value), the same in any order.
struct ByteScaleArgs {
    const unsigned char* src;       // [N][len]
    unsigned char* dst;             // [N][len]
    unsigned long long* range;      // [N][2]: max, 255 - min
    long long len;                  // H * W * 3
};

__global__ void __launch_bounds__(256) bytescale_range_kernel(const ByteScaleArgs a) {
    CCB_PDL_WAIT();
    __shared__ unsigned red[2][256];
    const int n = blockIdx.y, t = threadIdx.x;
    const unsigned char* s = a.src + (long long)n * a.len;
    unsigned hi = 0, lo = 0;
    for (long long i = (long long)blockIdx.x * 256 + t; i < a.len; i += (long long)gridDim.x * 256) {
        const unsigned v = s[i];
        hi = v > hi ? v : hi;
        lo = 255u - v > lo ? 255u - v : lo;
    }
    red[0][t] = hi;
    red[1][t] = lo;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (t < o) {
            red[0][t] = red[0][t + o] > red[0][t] ? red[0][t + o] : red[0][t];
            red[1][t] = red[1][t + o] > red[1][t] ? red[1][t + o] : red[1][t];
        }
        __syncthreads();
    }
    if (t == 0) {
        atomicMax(a.range + 2 * n, (unsigned long long)red[0][0]);
        atomicMax(a.range + 2 * n + 1, (unsigned long long)red[1][0]);
    }
}

// 256 threads: every block builds its image's table, then maps its share of the bytes
__global__ void __launch_bounds__(256) bytescale_apply_kernel(const ByteScaleArgs a) {
    CCB_PDL_WAIT();
    __shared__ unsigned char table[256];
    const int n = blockIdx.y, t = threadIdx.x;
    const float cmax = (float)a.range[2 * n], cmin = (float)(255ull - a.range[2 * n + 1]);
    float cscale = __fsub_rn(cmax, cmin);
    if (cscale == 0.f) cscale = 1.f;
    const float scale = __fdiv_rn(255.f, cscale);
    float v = __fmul_rn(__fsub_rn((float)t, cmin), scale);
    v = v < 0.f ? 0.f : (v > 255.f ? 255.f : v);
    table[t] = (unsigned char)__fadd_rn(v, 0.5f);
    __syncthreads();
    const unsigned char* s = a.src + (long long)n * a.len;
    unsigned char* d = a.dst + (long long)n * a.len;
    for (long long i = (long long)blockIdx.x * 256 + t; i < a.len; i += (long long)gridDim.x * 256) d[i] = table[s[i]];
}

}  // namespace ccb

using namespace ccb;

// blocks of a grid-stride loop over n elements: per_block elements each, at least 1 and at most cap.  A reduction's grid
// fixes the order of its fp64 partial sums, so each entry point keeps its constants.
static int blocks_for(long long n, int per_block, int cap) {
    const long long g = (n + per_block - 1) / per_block;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// A MedianState of B samples: the selections and the counts, then the histograms
static long long median_state_bytes(int B, int sel) { return (long long)B * (3 * sel + 1) * 8 + (long long)B * sel * 2048 * 4; }

// lays a.med out at `state` and clears it, then launches the passes of the select, nb histogram blocks per sample
template <class A>
static void median_select(A& a, char* state, int nb, ccb_stream_t stream) {
    a.med.sel = (unsigned long long*)state;
    a.med.count = a.med.sel + (long long)a.B * A::SEL * 3;
    a.med.hist = (unsigned*)(a.med.count + a.B);
    cudaMemsetAsync(state, 0, (size_t)median_state_bytes(a.B, A::SEL), (cudaStream_t)stream);
    for (int pass = 0; pass < radix_passes<typename A::Key>(); ++pass) {
        CCB_LAUNCH(median_hist_kernel<A>, dim3(nb, a.B), dim3(256), 0, stream, a, pass);
        CCB_LAUNCH(median_select_kernel<A>, dim3((a.B * A::SEL + 63) / 64), dim3(64), 0, stream, a, pass);
    }
}

extern "C" long long ccb_flow_metrics_workspace_bytes(int B, int Hg, int Wg) {
    if (B <= 0 || Hg <= 0 || Wg <= 0) return -1;
    return (long long)blocks_for((long long)B * Hg * Wg, 256, NUM_SMS * 8) * 8 * (long long)sizeof(double);
}

extern "C" int ccb_flow_metrics(const float* gt, const float* pred_rigid, const float* pred_nonrigid, const float* rigidity_mask,
                                int B, int nc, int Hg, int Wg, int hp, int wp, int hm, int wm, float thresh, float tau0,
                                float tau1, float* epe_map, void* work, long long work_bytes, float* out4, ccb_stream_t stream) {
    CCB_REQUIRE(gt && pred_rigid && out4, CCB_ERR_ARG, "flow_metrics: null pointer");
    CCB_REQUIRE(nc == 2 || nc == 3, CCB_ERR_ARG, "flow_metrics: ground truth must have 2 or 3 channels, got %d", nc);
    CCB_REQUIRE((rigidity_mask == nullptr) == (pred_nonrigid == nullptr), CCB_ERR_ARG,
                "flow_metrics: rigidity mask and non-rigid prediction come together");
    CCB_REQUIRE(B > 0 && Hg > 0 && Wg > 0 && hp > 0 && wp > 0, CCB_ERR_ARG, "flow_metrics: bad sizes");
    CCB_REQUIRE_WORK("flow_metrics", "work", work, work_bytes, ccb_flow_metrics_workspace_bytes(B, Hg, Wg));
    FlowMetArgs a;
    a.gt = gt; a.pa = pred_rigid; a.pb = pred_nonrigid; a.mask = rigidity_mask; a.partials = (double*)work; a.epe_map = epe_map;
    a.B = B; a.nc = nc; a.Hg = Hg; a.Wg = Wg; a.hp = hp; a.wp = wp; a.hm = hm; a.wm = wm;
    a.thresh = thresh; a.tau0 = tau0; a.tau1 = tau1;
    const int nb = blocks_for((long long)B * Hg * Wg, 256, NUM_SMS * 8);
    CCB_LAUNCH(flow_metrics_kernel, dim3(nb), dim3(256), 0, stream, a);
    CCB_LAUNCH(flow_metrics_finalize, dim3(1), dim3(32), 0, stream, (const double*)work, nb, nc, (long long)B * Hg * Wg, out4);
    return check_launch("flow_metrics");
}

extern "C" long long ccb_depth_errors_workspace_bytes(int B, int H, int W) {
    if (B <= 0 || H <= 0 || W <= 0) return -1;
    return (long long)B * blocks_for((long long)H * W, 256, 64) * 6 * 8 + median_state_bytes(B, DepthArgs::SEL);
}

extern "C" int ccb_depth_errors(const float* gt, const float* pred, int B, int H, int W, int crop, void* work, long long work_bytes,
                                float* out6, ccb_stream_t stream) {
    CCB_REQUIRE(gt && pred && out6, CCB_ERR_ARG, "depth_errors: null pointer");
    CCB_REQUIRE(B > 0 && H > 0 && W > 0, CCB_ERR_ARG, "depth_errors: bad sizes");
    CCB_REQUIRE_WORK("depth_errors", "work", work, work_bytes, ccb_depth_errors_workspace_bytes(B, H, W));
    DepthArgs a;
    a.gt = gt; a.pred = pred; a.B = B; a.H = H; a.W = W; a.out = out6;
    a.y1 = 0; a.y2 = H; a.x1 = 0; a.x2 = W;
    if (crop) {            // int(0.40810811 * H) etc. evaluated in double like python (:441-442)
        a.y1 = (int)(0.40810811 * H); a.y2 = (int)(0.99189189 * H);
        a.x1 = (int)(0.03594771 * W); a.x2 = (int)(0.96405229 * W);
    }
    const int nb = blocks_for((long long)H * W, 256, 64);
    a.partials = (double*)work;
    median_select(a, (char*)work + (long long)B * nb * 6 * 8, nb, stream);
    CCB_LAUNCH(depth_errors_kernel, dim3(nb, B), dim3(256), 0, stream, a);
    CCB_LAUNCH(depth_errors_finalize, dim3(1), dim3(32), 0, stream, a, nb);
    return check_launch("depth_errors");
}

extern "C" long long ccb_mask_iou_workspace_bytes(int B, int h, int w, int Hg, int Wg) {
    if (B <= 0 || h <= 0 || w <= 0 || Hg <= 0 || Wg <= 0) return -1;
    return (long long)B * (long long)sizeof(unsigned long long);
}

extern "C" int ccb_mask_iou(const float* emask, const float* flow_cam, const float* flow, const float* obj_map,
                            const float* semantic_map, int B, int C, int h, int w, int Hg, int Wg, float thresh, int car_label,
                            float* masks, void* work, long long work_bytes, long long* counts, ccb_stream_t stream) {
    CCB_REQUIRE(emask && flow_cam && flow && obj_map && semantic_map && counts, CCB_ERR_ARG, "mask_iou: null pointer");
    CCB_REQUIRE(C >= 3, CCB_ERR_ARG, "mask_iou: the mask net output needs channels 1 and 2, got %d channels", C);
    CCB_REQUIRE(B > 0 && h > 0 && w > 0 && Hg > 0 && Wg > 0, CCB_ERR_ARG, "mask_iou: bad sizes");
    const long long need = ccb_mask_iou_workspace_bytes(B, h, w, Hg, Wg);
    CCB_REQUIRE_WORK("mask_iou", "work", work, work_bytes, need);
    MaskIouArgs a;
    a.emask = emask; a.flow_cam = flow_cam; a.flow = flow; a.obj = obj_map; a.sem = semantic_map; a.masks = masks;
    a.dmax = (unsigned long long*)work; a.counts = (unsigned long long*)counts;
    a.B = B; a.C = C; a.h = h; a.w = w; a.Hg = Hg; a.Wg = Wg; a.thresh = thresh; a.car = (float)car_label;
    cudaMemsetAsync(a.dmax, 0, (size_t)need, (cudaStream_t)stream);
    cudaMemsetAsync(a.counts, 0, (size_t)B * 12 * sizeof(unsigned long long), (cudaStream_t)stream);
    const int nb = blocks_for((long long)h * w, 256, NUM_SMS * 4);
    CCB_LAUNCH(mask_iou_max_kernel, dim3(nb, B), dim3(256), 0, stream, a);
    if (masks) CCB_LAUNCH(mask_iou_masks_kernel, dim3(nb, B), dim3(256), 0, stream, a);
    CCB_LAUNCH(mask_iou_count_kernel, dim3(blocks_for((long long)Hg * Wg, 256, NUM_SMS * 4), B), dim3(256), 0, stream, a);
    return check_launch("mask_iou");
}

extern "C" int ccb_flow_submit(const float* emask, const float* flow_cam, const float* flow_fwd, int B, int C, int h, int w,
                               int Hg, int Wg, float thresh, float* mask, float* full, unsigned short* png, float* flo,
                               ccb_stream_t stream) {
    CCB_REQUIRE(emask && flow_cam && flow_fwd && mask && png && flo, CCB_ERR_ARG, "flow_submit: null pointer");
    CCB_REQUIRE(C >= 3, CCB_ERR_ARG, "flow_submit: the mask net output needs channels 1 and 2, got %d channels", C);
    CCB_REQUIRE(B > 0 && h > 0 && w > 0 && Hg > 0 && Wg > 0, CCB_ERR_ARG, "flow_submit: bad sizes");
    FlowSubmitArgs a;
    a.emask = emask; a.cam = flow_cam; a.fwd = flow_fwd; a.mask = mask; a.full = full; a.png = png; a.flo = flo;
    a.B = B; a.C = C; a.h = h; a.w = w; a.Hg = Hg; a.Wg = Wg; a.thresh = thresh;
    a.fu = (float)((double)Wg / (double)w);        // u * (w_gt / w_pred): the python float, cast to fp32 by torch's mul
    a.fv = (float)((double)Hg / (double)h);
    CCB_LAUNCH(flow_submit_mask_kernel, dim3(blocks_for((long long)B * h * w, 256, NUM_SMS * 8)), dim3(256), 0, stream, a);
    CCB_LAUNCH(flow_submit_kernel, dim3(blocks_for((long long)B * Hg * Wg, 256, NUM_SMS * 8)), dim3(256), 0, stream, a);
    return check_launch("flow_submit");
}

extern "C" long long ccb_flow_color_workspace_bytes(int B, int P, int H, int W) {
    if (B <= 0 || P <= 0 || H <= 0 || W <= 0) return -1;
    return (long long)B * (long long)sizeof(unsigned long long);
}

extern "C" int ccb_flow_color(const float* flow, int B, int P, int H, int W, void* work, long long work_bytes, unsigned char* out,
                              ccb_stream_t stream) {
    CCB_REQUIRE(flow && out, CCB_ERR_ARG, "flow_color: null pointer");
    CCB_REQUIRE(B > 0 && P > 0 && H > 0 && W > 0, CCB_ERR_ARG, "flow_color: bad sizes");
    const long long need = ccb_flow_color_workspace_bytes(B, P, H, W);
    CCB_REQUIRE_WORK("flow_color", "work", work, work_bytes, need);
    FlowColorArgs a;
    a.flow = flow; a.maxrad = (unsigned long long*)work; a.out = out; a.B = B; a.P = P; a.H = H; a.W = W;
    cudaMemsetAsync(a.maxrad, 0, (size_t)need, (cudaStream_t)stream);
    const int nb = blocks_for((long long)P * H * W, 256, NUM_SMS * 4);
    CCB_LAUNCH(flow_color_max_kernel, dim3(nb, B), dim3(256), 0, stream, a);
    CCB_LAUNCH(flow_color_kernel, dim3(nb, B), dim3(256), 0, stream, a);
    return check_launch("flow_color");
}

extern "C" long long ccb_kitti_flow_errors_workspace_bytes(int B, int H, int W) {
    if (B <= 0 || H <= 0 || W <= 0) return -1;
    return (long long)B * blocks_for((long long)H * W, 2048, 128) * 3 * (long long)sizeof(double);
}

extern "C" int ccb_kitti_flow_errors(const unsigned short* gt, const unsigned short* pred, int B, int H, int W, void* work,
                                     long long work_bytes, double* out, long long* counts, ccb_stream_t stream) {
    CCB_REQUIRE(gt && pred && out, CCB_ERR_ARG, "kitti_flow_errors: null pointer");
    CCB_REQUIRE(B > 0 && H > 0 && W > 0, CCB_ERR_ARG, "kitti_flow_errors: bad sizes");
    const long long need = ccb_kitti_flow_errors_workspace_bytes(B, H, W);
    CCB_REQUIRE_WORK("kitti_flow_errors", "work", work, work_bytes, need);
    KittiErrArgs a;
    a.gt = gt; a.pred = pred; a.partials = (double*)work; a.out = out; a.counts = counts; a.B = B; a.H = H; a.W = W;
    const int nb = blocks_for((long long)H * W, 2048, 128);
    CCB_LAUNCH(kitti_err_kernel, dim3(nb, B), dim3(256), 0, stream, a);
    CCB_LAUNCH(kitti_err_finalize, dim3((B + 63) / 64), dim3(64), 0, stream, a, nb);
    return check_launch("kitti_flow_errors");
}

// keys -1 .. H*(W-1) - 1 of the reference's sub2ind, stored at key + 1
static long long velo_keys(int H, int W) { return (long long)H * (W - 1) + 1; }

extern "C" long long ccb_velo_depth_workspace_bytes(int B, int H, int W) {
    if (B <= 0 || H <= 0 || W <= 0) return -1;
    return (long long)B * ((long long)H * W + 3 * velo_keys(H, W)) * (long long)sizeof(unsigned long long);
}

extern "C" int ccb_velo_depth(const float* points, const long long* offsets, const double* P_velo2im, long long total, int B, int H,
                              int W, void* work, long long work_bytes, double* depth, ccb_stream_t stream) {
    CCB_REQUIRE(offsets && P_velo2im && depth && (points || total == 0), CCB_ERR_ARG, "velo_depth: null pointer");
    CCB_REQUIRE(B > 0 && H > 0 && W > 0 && total >= 0, CCB_ERR_ARG, "velo_depth: bad sizes");
    const long long need = ccb_velo_depth_workspace_bytes(B, H, W);
    CCB_REQUIRE_WORK("velo_depth", "work", work, work_bytes, need);
    const long long hw = (long long)H * W, K = velo_keys(H, W);
    VeloArgs a;
    a.pts = points; a.offs = offsets; a.P = P_velo2im; a.depth = depth; a.total = total; a.B = B; a.H = H; a.W = W;
    a.last = (unsigned long long*)work;
    a.cnt = a.last + (long long)B * hw;
    a.first = a.cnt + (long long)B * K;
    a.zmin = a.first + (long long)B * K;
    cudaMemsetAsync(work, 0, (size_t)need, (cudaStream_t)stream);
    const int nbp = blocks_for((total + B - 1) / B, 256, NUM_SMS * 4);
    if (total > 0) CCB_LAUNCH(velo_scatter_kernel, dim3(nbp, B), dim3(256), 0, stream, a);
    CCB_LAUNCH(velo_depth_kernel, dim3(blocks_for((long long)H * W, 256, NUM_SMS * 4), B), dim3(256), 0, stream, a);
    return check_launch("velo_depth");
}

extern "C" long long ccb_spline_zoom_workspace_bytes(int N, int h, int w) {
    if (N <= 0 || h <= 0 || w <= 0) return -1;
    return (long long)N * h * w * (long long)sizeof(double);
}

extern "C" int ccb_spline_zoom(const float* src, int N, int h, int w, int H, int W, float lo, float hi, void* work,
                               long long work_bytes, float* dst, ccb_stream_t stream) {
    CCB_REQUIRE(src && dst, CCB_ERR_ARG, "spline_zoom: null pointer");
    CCB_REQUIRE(N > 0 && h > 0 && w > 0 && H > 0 && W > 0, CCB_ERR_ARG, "spline_zoom: bad sizes");
    CCB_REQUIRE_WORK("spline_zoom", "work", work, work_bytes, ccb_spline_zoom_workspace_bytes(N, h, w));
    ZoomArgs a;
    a.src = src; a.coef = (double*)work; a.dst = dst; a.N = N; a.h = h; a.w = w; a.H = H; a.W = W; a.lo = lo; a.hi = hi;
    CCB_LAUNCH(zoom_prefilter_kernel, dim3(blocks_for((long long)N * w, 256, NUM_SMS * 8)), dim3(256), 0, stream, a, 0);
    CCB_LAUNCH(zoom_prefilter_kernel, dim3(blocks_for((long long)N * h, 256, NUM_SMS * 8)), dim3(256), 0, stream, a, 1);
    CCB_LAUNCH(zoom_eval_kernel, dim3(blocks_for((long long)N * H * W, 256, NUM_SMS * 8)), dim3(256), 0, stream, a);
    return check_launch("spline_zoom");
}

// nb blocks per sample; workspace: block partials, the scales, then the median select's state
struct EigenPlan { int nb; long long partials, scale, med, bytes; };
static EigenPlan eigen_plan(int B, int H, int W) {
    EigenPlan p;
    p.nb = blocks_for((long long)H * W, 2048, 64);
    p.partials = 0;
    p.scale = p.partials + (long long)B * p.nb * 14 * 8;
    p.med = p.scale + (long long)B * 2 * 8;
    p.bytes = p.med + median_state_bytes(B, EigenArgs::SEL);
    return p;
}

extern "C" long long ccb_eigen_depth_errors_workspace_bytes(int B, int H, int W) {
    if (B <= 0 || H <= 0 || W <= 0) return -1;
    return eigen_plan(B, H, W).bytes;
}

// a (validated) EigenArgs with the workspace laid out and the selections cleared, then the launches
static int eigen_errors_launch(const char* what, EigenArgs a, void* work, ccb_stream_t stream) {
    const EigenPlan p = eigen_plan(a.B, a.H, a.W);
    char* w = (char*)work;
    a.partials = (double*)(w + p.partials); a.scale = (double*)(w + p.scale);
    const int B = a.B, nb = p.nb;
    median_select(a, w + p.med, nb, stream);
    CCB_LAUNCH(eigen_scale_kernel, dim3((B + 63) / 64), dim3(64), 0, stream, a);
    CCB_LAUNCH(eigen_errors_kernel, dim3(nb, B), dim3(256), 0, stream, a);
    CCB_LAUNCH(eigen_finalize_kernel, dim3((B * 2 + 63) / 64), dim3(64), 0, stream, a, nb);
    return check_launch(what);
}

extern "C" int ccb_eigen_depth_errors(const double* gt, const float* pred, int B, int H, int W, double min_depth, double max_depth,
                                      const double* crop, const float* poses, const double* displacements, int R, void* work,
                                      long long work_bytes, double* out, ccb_stream_t stream) {
    CCB_REQUIRE(gt && pred && crop && out, CCB_ERR_ARG, "eigen_depth_errors: null pointer");
    CCB_REQUIRE((poses == nullptr) == (displacements == nullptr), CCB_ERR_ARG,
                "eigen_depth_errors: poses and displacements come together");
    CCB_REQUIRE(B > 0 && H > 0 && W > 0 && (poses == nullptr || R > 0), CCB_ERR_ARG, "eigen_depth_errors: bad sizes");
    for (int k = 0; k < 4; ++k)
        CCB_REQUIRE(crop[k] >= 0.0 && crop[k] <= 1.0, CCB_ERR_ARG, "eigen_depth_errors: crop fraction %d outside [0, 1]", k);
    CCB_REQUIRE_WORK("eigen_depth_errors", "work", work, work_bytes, eigen_plan(B, H, W).bytes);
    EigenArgs a;
    a.gt = gt; a.pred = pred; a.poses = poses; a.disp = displacements; a.out = out;
    a.min_depth = min_depth; a.max_depth = max_depth; a.cap = HUGE_VAL; a.log10 = 0;
    a.B = B; a.H = H; a.W = W; a.R = poses ? R : 0;
    // generate_mask: np.array([f0 * H, f1 * H, f2 * W, f3 * W]).astype(np.int32), fp64 products truncated
    a.y1 = (int)(crop[0] * H); a.y2 = (int)(crop[1] * H); a.x1 = (int)(crop[2] * W); a.x2 = (int)(crop[3] * W);
    return eigen_errors_launch("eigen_depth_errors", a, work, stream);
}

extern "C" long long ccb_make3d_depth_errors_workspace_bytes(int B, int H, int W) {
    return ccb_eigen_depth_errors_workspace_bytes(B, H, W);
}

extern "C" int ccb_make3d_depth_errors(const double* gt, const float* pred, int B, int H, int W, double min_depth, double max_depth,
                                       void* work, long long work_bytes, double* out, ccb_stream_t stream) {
    CCB_REQUIRE(gt && pred && out, CCB_ERR_ARG, "make3d_depth_errors: null pointer");
    CCB_REQUIRE(B > 0 && H > 0 && W > 0, CCB_ERR_ARG, "make3d_depth_errors: bad sizes");
    CCB_REQUIRE_WORK("make3d_depth_errors", "work", work, work_bytes, eigen_plan(B, H, W).bytes);
    EigenArgs a;
    a.gt = gt; a.pred = pred; a.poses = nullptr; a.disp = nullptr; a.out = out;
    a.min_depth = min_depth; a.max_depth = max_depth; a.cap = max_depth; a.log10 = 1;
    a.B = B; a.H = H; a.W = W; a.R = 0;
    a.y1 = 0; a.y2 = H; a.x1 = 0; a.x2 = W;        // no crop: the mask is the depth range alone
    return eigen_errors_launch("make3d_depth_errors", a, work, stream);
}

template <bool UNIT>
static int prep_frames_launch(const char* what, const unsigned char* src_u8, float* const* dst, const float* params, const int* offs,
                              int B, int F, int Hs, int Ws, int H, int W, ccb_stream_t stream) {
    CCB_REQUIRE(src_u8 && dst && params && offs, CCB_ERR_ARG, "%s: null pointer", what);
    CCB_REQUIRE(F >= 1 && F <= 8, CCB_ERR_ARG, "%s: 1..8 frames per sample, got %d", what, F);
    CCB_REQUIRE(B > 0 && Hs > 0 && Ws > 0 && H > 0 && W > 0, CCB_ERR_ARG, "%s: bad sizes", what);
    PrepArgs a;
    a.src = src_u8; a.params = params; a.offs = offs; a.B = B; a.F = F; a.Hs = Hs; a.Ws = Ws; a.H = H; a.W = W;
    for (int f = 0; f < 8; ++f) a.dst[f] = (f < F) ? dst[f] : nullptr;
    for (int f = 0; f < F; ++f) CCB_REQUIRE(a.dst[f] != nullptr, CCB_ERR_ARG, "%s: dst[%d] is null", what, f);
    CCB_LAUNCH(prep_frames_kernel<UNIT>, dim3(blocks_for((long long)B * F * H * W, 256, NUM_SMS * 8)), dim3(256), 0, stream, a);
    return check_launch(what);
}

extern "C" int ccb_prep_frames(const unsigned char* src_u8, float* const* dst, const float* params, const int* offs, int B, int F,
                               int Hs, int Ws, int H, int W, ccb_stream_t stream) {
    return prep_frames_launch<false>("prep_frames", src_u8, dst, params, offs, B, F, Hs, Ws, H, W, stream);
}

extern "C" int ccb_prep_frames_unit(const unsigned char* src_u8, float* const* dst, const float* params, const int* offs, int B,
                                    int F, int Hs, int Ws, int H, int W, ccb_stream_t stream) {
    return prep_frames_launch<true>("prep_frames_unit", src_u8, dst, params, offs, B, F, Hs, Ws, H, W, stream);
}

extern "C" int ccb_rotate_frames_u8(const unsigned char* src, const double* affine, unsigned char* dst, int B, int F, int H, int W,
                                    ccb_stream_t stream) {
    CCB_REQUIRE(src && affine && dst, CCB_ERR_ARG, "rotate_frames_u8: null pointer");
    CCB_REQUIRE(src != dst, CCB_ERR_ARG, "rotate_frames_u8: cannot rotate in place");
    CCB_REQUIRE(B > 0 && F > 0 && H > 0 && W > 0, CCB_ERR_ARG, "rotate_frames_u8: bad sizes");
    RotArgs a;
    a.src = src; a.affine = affine; a.dst = dst; a.B = B; a.F = F; a.H = H; a.W = W;
    CCB_LAUNCH(rotate_frames_kernel, dim3(blocks_for((long long)B * F * H * W, 256, NUM_SMS * 8)), dim3(256), 0, stream, a);
    return check_launch("rotate_frames_u8");
}

// Workspace of ccb_resize_u8: both coefficient tables, then (when both passes run) the uint8 intermediate.
struct ResizePlan {
    int ks_x, ks_y;
    long long kk_x, bounds_x, kk_y, bounds_y, tmp, bytes;   // byte offsets; bytes = total
};

static int resample_ksize(int in_size, int out_size) {
    const double scale = (double)in_size / (double)out_size;
    return (int)ceil(scale < 1.0 ? 1.0 : scale) * 2 + 1;
}

static ResizePlan resize_plan(int N, int Hs, int Ws, int H, int W) {
    auto up = [](long long v) { return (v + 255) / 256 * 256; };
    ResizePlan p;
    p.ks_x = resample_ksize(Ws, W);
    p.ks_y = resample_ksize(Hs, H);
    p.kk_x = 0;
    p.bounds_x = up(p.kk_x + 4LL * W * p.ks_x);
    p.kk_y = up(p.bounds_x + 8LL * W);
    p.bounds_y = up(p.kk_y + 4LL * H * p.ks_y);
    p.tmp = up(p.bounds_y + 8LL * H);
    p.bytes = p.tmp + ((W != Ws && H != Hs) ? up((long long)N * Hs * W * 3) : 0);
    return p;
}

extern "C" long long ccb_resize_u8_workspace_bytes(int N, int Hs, int Ws, int H, int W) {
    if (N <= 0 || Hs <= 0 || Ws <= 0 || H <= 0 || W <= 0) return -1;
    return resize_plan(N, Hs, Ws, H, W).bytes;
}

extern "C" int ccb_resize_u8(const unsigned char* src, unsigned char* dst, int N, int Hs, int Ws, int H, int W, void* work,
                             long long work_bytes, ccb_stream_t stream) {
    CCB_REQUIRE(src && dst, CCB_ERR_ARG, "resize_u8: null pointer");
    CCB_REQUIRE(src != dst, CCB_ERR_ARG, "resize_u8: cannot resize in place");
    CCB_REQUIRE(N > 0 && Hs > 0 && Ws > 0 && H > 0 && W > 0, CCB_ERR_ARG, "resize_u8: bad sizes");
    const ResizePlan p = resize_plan(N, Hs, Ws, H, W);
    CCB_REQUIRE_WORK("resize_u8", "work", work, work_bytes, p.bytes);
    const bool hpass = W != Ws, vpass = H != Hs;
    if (!hpass && !vpass) {
        cudaMemcpyAsync(dst, src, (size_t)N * H * W * 3, cudaMemcpyDeviceToDevice, (cudaStream_t)stream);
        return check_launch("resize_u8");
    }
    char* w = (char*)work;
    CoeffArgs c;
    c.in_x = Ws; c.out_x = W; c.ks_x = p.ks_x; c.in_y = Hs; c.out_y = H; c.ks_y = p.ks_y;
    c.kk_x = (int*)(w + p.kk_x); c.bounds_x = (int*)(w + p.bounds_x); c.kk_y = (int*)(w + p.kk_y); c.bounds_y = (int*)(w + p.bounds_y);
    CCB_LAUNCH(resample_coeffs_kernel, dim3((W + H + 127) / 128), dim3(128), 0, stream, c);
    unsigned char* mid = (hpass && vpass) ? (unsigned char*)(w + p.tmp) : dst;
    if (hpass) {
        ResampleArgs r;
        r.src = src; r.dst = mid; r.kk = c.kk_x; r.bounds = c.bounds_x;
        r.outer = (long long)N * Hs; r.in_len = Ws; r.out_len = W; r.inner = 1; r.ksize = p.ks_x;
        CCB_LAUNCH(resample_pass_kernel, dim3(blocks_for((long long)N * Hs * W, 256, NUM_SMS * 8)), dim3(256), 0, stream, r);
    }
    if (vpass) {
        ResampleArgs r;
        r.src = hpass ? mid : src; r.dst = dst; r.kk = c.kk_y; r.bounds = c.bounds_y;
        r.outer = N; r.in_len = Hs; r.out_len = H; r.inner = W; r.ksize = p.ks_y;
        CCB_LAUNCH(resample_pass_kernel, dim3(blocks_for((long long)N * H * W, 256, NUM_SMS * 8)), dim3(256), 0, stream, r);
    }
    return check_launch("resize_u8");
}

extern "C" long long ccb_bytescale_u8_workspace_bytes(int N, int H, int W) {
    if (N <= 0 || H <= 0 || W <= 0) return -1;
    return (long long)N * 2 * (long long)sizeof(unsigned long long);
}

extern "C" int ccb_bytescale_u8(const unsigned char* src, int N, int H, int W, void* work, long long work_bytes, unsigned char* dst,
                                ccb_stream_t stream) {
    CCB_REQUIRE(src && dst, CCB_ERR_ARG, "bytescale_u8: null pointer");
    CCB_REQUIRE(N > 0 && H > 0 && W > 0, CCB_ERR_ARG, "bytescale_u8: bad sizes");
    CCB_REQUIRE_WORK("bytescale_u8", "work", work, work_bytes, ccb_bytescale_u8_workspace_bytes(N, H, W));
    ByteScaleArgs a;
    a.src = src; a.dst = dst; a.range = (unsigned long long*)work; a.len = (long long)H * W * 3;
    cudaMemsetAsync(work, 0, (size_t)N * 2 * sizeof(unsigned long long), (cudaStream_t)stream);
    const dim3 grid(blocks_for(a.len, 8192, 256), N);
    CCB_LAUNCH(bytescale_range_kernel, grid, dim3(256), 0, stream, a);
    CCB_LAUNCH(bytescale_apply_kernel, grid, dim3(256), 0, stream, a);
    return check_launch("bytescale_u8");
}

extern "C" long long ccb_normalize_local_workspace_bytes(int B, int H, int W) {
    if (B <= 0 || H <= 0 || W <= 0) return -1;
    return (long long)B * 3 * blocks_for((long long)H * W, 2048, 64) * 2 * (long long)sizeof(double) + (long long)B * 3 * 2 * (long long)sizeof(float);
}

extern "C" int ccb_normalize_local(float* const* frames, int B, int F, int H, int W, float* stats, void* work, long long work_bytes,
                                   ccb_stream_t stream) {
    CCB_REQUIRE(frames, CCB_ERR_ARG, "normalize_local: null pointer");
    CCB_REQUIRE(F >= 1 && F <= 8, CCB_ERR_ARG, "normalize_local: 1..8 frames per sample, got %d", F);
    CCB_REQUIRE(B > 0 && H > 0 && W > 0, CCB_ERR_ARG, "normalize_local: bad sizes");
    const long long need = ccb_normalize_local_workspace_bytes(B, H, W);
    CCB_REQUIRE_WORK("normalize_local", "work", work, work_bytes, need);
    NormLocalArgs a;
    for (int f = 0; f < 8; ++f) a.x[f] = (f < F) ? frames[f] : nullptr;
    for (int f = 0; f < F; ++f) CCB_REQUIRE(a.x[f] != nullptr, CCB_ERR_ARG, "normalize_local: frames[%d] is null", f);
    const int nblk = blocks_for((long long)H * W, 2048, 64);
    a.partials = (double*)work;
    a.stats = stats ? stats : (float*)((char*)work + (long long)B * 3 * nblk * 2 * sizeof(double));
    a.B = B; a.F = F; a.hw = (long long)H * W;
    CCB_LAUNCH(normlocal_partials_kernel, dim3(nblk, B * 3), dim3(256), 0, stream, a);
    CCB_LAUNCH(normlocal_finalize_kernel, dim3((B * 3 + 63) / 64), dim3(64), 0, stream, a, nblk);
    CCB_LAUNCH(normlocal_apply_kernel, dim3(nblk, B * 3), dim3(256), 0, stream, a);
    return check_launch("normalize_local");
}
