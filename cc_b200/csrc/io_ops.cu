// io_ops.cu - the callers either side of the training step (SURVEY.md 8f "next" rows N1 / N2):
//
//   N2  validation metrics as fused masked reductions
//         flow:  flow_diff / compute_epe / outlier_err / compute_all_epes   (loss_functions.py:355-427)
//         depth: compute_errors with median scaling and the Garg crop        (loss_functions.py:430-467)
//   N1  input pipeline on the device: uint8 HWC frames -> normalised fp32 NCHW frames with the reference's
//       augmentations (ArrayToTensor /255, Normalize mean .5 std .5, RandomHorizontalFlip, RandomScaleCrop;
//       custom_transforms.py:21-30,47-118) applied per sample from host-drawn parameters, plus the matching
//       intrinsics update.  H2D traffic drops 4x (uint8 instead of fp32).
//
// All reductions are two-stage and deterministic (per-block partials in double, fixed-order finalize).
#include "ccb_common.cuh"

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

template <int NV>
__device__ __forceinline__ void block_sum_d(double (&v)[NV], double* scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int i = 0; i < NV; ++i)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[i] += __shfl_xor_sync(0xffffffffu, v[i], o);
    __syncthreads();
    if (lane == 0)
#pragma unroll
        for (int i = 0; i < NV; ++i) scratch[i * 32 + warp] = v[i];
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int i = 0; i < NV; ++i) {
            double x = (lane < nwarps) ? scratch[i * 32 + lane] : 0.0;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
            v[i] = x;
        }
    }
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
    block_sum_d<8>(acc, scratch);
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < 8; ++k) a.partials[(long long)blockIdx.x * 8 + k] = acc[k];
}

// out[0..3] = all_epe, rigid_epe, non_rigid_epe, outlier ratio   (nc == 2: plain mean over B*Hg*Wg, :384-385)
__global__ void flow_metrics_finalize(const double* __restrict__ partials, int nblocks, int nc, long long npx, float* __restrict__ out) {
    CCB_PDL_WAIT();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int b = 0; b < nblocks; ++b)
        for (int k = 0; k < 8; ++k) s[k] += partials[(long long)b * 8 + k];
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
// Medians by a 3-pass radix select over the float bit patterns (all keys are positive: bit order == value order).
struct DepthArgs {
    const float* gt;
    const float* pred;
    int B, H, W, y1, y2, x1, x2;     // crop window (whole image when crop is off)
    unsigned* hist;                  // [B][2][2048]
    unsigned* sel;                   // [B][2][4]: prefix bits, prefix mask, remaining rank k, count
    double* partials;                // [B][blocks][6]
    float* out;                      // [6]
};

__device__ __forceinline__ bool depth_valid(const DepthArgs& a, float g, int y, int x) {
    return (g > 0.f) && (g < 80.f) && (y >= a.y1) && (y < a.y2) && (x >= a.x1) && (x < a.x2);
}
__device__ __forceinline__ float clamp_pred(float p) { return fminf(fmaxf(p, 1e-3f), 80.f); }

// pass 0: count valid + histogram of the top 11 bits; pass 1/2: histogram of the next 11 / 10 bits among keys
// matching the prefix found so far
__global__ void __launch_bounds__(256) depth_hist_kernel(const DepthArgs a, int pass) {
    CCB_PDL_WAIT();
    const int b = blockIdx.y;
    const int shift = (pass == 0) ? 21 : (pass == 1 ? 10 : 0);
    const unsigned nb_mask = (pass == 2) ? 1023u : 2047u;
    const long long hw = (long long)a.H * a.W;
    unsigned* hg = a.hist + ((long long)b * 2 + 0) * 2048;
    unsigned* hp = a.hist + ((long long)b * 2 + 1) * 2048;
    const unsigned* sg = a.sel + ((long long)b * 2 + 0) * 4;
    const unsigned* sp = a.sel + ((long long)b * 2 + 1) * 4;
    const unsigned pg = sg[0], mg = sg[1], pp = sp[0], mp = sp[1];
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < hw; i += (long long)gridDim.x * 256) {
        const int y = (int)(i / a.W), x = (int)(i - (long long)y * a.W);
        const float g = __ldg(a.gt + b * hw + i);
        if (!depth_valid(a, g, y, x)) continue;
        const unsigned kg = __float_as_uint(g), kp = __float_as_uint(clamp_pred(__ldg(a.pred + b * hw + i)));
        if ((kg & mg) == pg) atomicAdd(hg + ((kg >> shift) & nb_mask), 1u);
        if ((kp & mp) == pp) atomicAdd(hp + ((kp >> shift) & nb_mask), 1u);
    }
}

// one thread per (sample, which): find the bin holding rank k, extend the prefix, clear the histogram
__global__ void depth_select_kernel(const DepthArgs a, int pass) {
    CCB_PDL_WAIT();
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.B * 2) return;
    unsigned* h = a.hist + (long long)t * 2048;
    unsigned* s = a.sel + (long long)t * 4;
    const int shift = (pass == 0) ? 21 : (pass == 1 ? 10 : 0);
    const int nbins = (pass == 2) ? 1024 : 2048;
    if (pass == 0) {
        unsigned n = 0;
        for (int i = 0; i < nbins; ++i) n += h[i];
        s[3] = n;
        s[2] = (n > 0) ? (n - 1) / 2 : 0;             // torch.median: lower median = sorted[(n-1)//2]
    }
    unsigned k = s[2], cum = 0;
    int bin = 0;
    for (int i = 0; i < nbins; ++i) {
        if (cum + h[i] > k) { bin = i; break; }
        cum += h[i];
        bin = i;
    }
    s[2] = k - cum;
    s[0] |= ((unsigned)bin) << shift;
    s[1] |= ((pass == 2) ? 1023u : 2047u) << shift;
    for (int i = 0; i < 2048; ++i) h[i] = 0;
}

__global__ void __launch_bounds__(256) depth_errors_kernel(const DepthArgs a) {
    CCB_PDL_WAIT();
    __shared__ double scratch[6 * 32];
    const int b = blockIdx.y;
    const long long hw = (long long)a.H * a.W;
    const float med_g = __uint_as_float(a.sel[((long long)b * 2 + 0) * 4]);
    const float med_p = __uint_as_float(a.sel[((long long)b * 2 + 1) * 4]);
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
    block_sum_d<6>(acc, scratch);
    if (threadIdx.x == 0)
#pragma unroll
        for (int k = 0; k < 6; ++k) a.partials[((long long)b * gridDim.x + blockIdx.x) * 6 + k] = acc[k];
}

__global__ void depth_errors_finalize(const DepthArgs a, int nblocks) {
    CCB_PDL_WAIT();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    double tot[6] = {0, 0, 0, 0, 0, 0};
    for (int b = 0; b < a.B; ++b) {
        double s[6] = {0, 0, 0, 0, 0, 0};
        for (int k = 0; k < nblocks; ++k)
            for (int j = 0; j < 6; ++j) s[j] += a.partials[((long long)b * nblocks + k) * 6 + j];
        const double n = (double)a.sel[((long long)b * 2) * 4 + 3];
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
            d[(long long)c * a.H * a.W] = (v / 255.f - 0.5f) / 0.5f;
        }
    }
}

}  // namespace ccb

using namespace ccb;

static int grid_for(long long n) {
    long long g = (n + 255) / 256;
    const long long cap = NUM_SMS * 8;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

extern "C" long long ccb_flow_metrics_workspace_bytes(int B, int Hg, int Wg) {
    return (long long)grid_for((long long)B * Hg * Wg) * 8 * (long long)sizeof(double);
}

extern "C" int ccb_flow_metrics(const float* gt, const float* pred_rigid, const float* pred_nonrigid, const float* rigidity_mask,
                                int B, int nc, int Hg, int Wg, int hp, int wp, int hm, int wm, float thresh, float tau0,
                                float tau1, float* epe_map, void* work, float* out4, ccb_stream_t stream) {
    CCB_REQUIRE(gt && pred_rigid && work && out4, CCB_ERR_ARG, "flow_metrics: null pointer");
    CCB_REQUIRE(nc == 2 || nc == 3, CCB_ERR_ARG, "flow_metrics: ground truth must have 2 or 3 channels, got %d", nc);
    CCB_REQUIRE((rigidity_mask == nullptr) == (pred_nonrigid == nullptr), CCB_ERR_ARG,
                "flow_metrics: rigidity mask and non-rigid prediction come together");
    CCB_REQUIRE(B > 0 && Hg > 0 && Wg > 0 && hp > 0 && wp > 0, CCB_ERR_ARG, "flow_metrics: bad sizes");
    FlowMetArgs a;
    a.gt = gt; a.pa = pred_rigid; a.pb = pred_nonrigid; a.mask = rigidity_mask; a.partials = (double*)work; a.epe_map = epe_map;
    a.B = B; a.nc = nc; a.Hg = Hg; a.Wg = Wg; a.hp = hp; a.wp = wp; a.hm = hm; a.wm = wm;
    a.thresh = thresh; a.tau0 = tau0; a.tau1 = tau1;
    const int nb = grid_for((long long)B * Hg * Wg);
    CCB_LAUNCH(flow_metrics_kernel, dim3(nb), dim3(256), 0, stream, a);
    CCB_LAUNCH(flow_metrics_finalize, dim3(1), dim3(32), 0, stream, (const double*)work, nb, nc, (long long)B * Hg * Wg, out4);
    return check_launch("flow_metrics");
}

static int depth_blocks(int H, int W) {
    int g = (int)(((long long)H * W + 255) / 256);
    return g < 1 ? 1 : (g > 64 ? 64 : g);
}

extern "C" long long ccb_depth_errors_workspace_bytes(int B, int H, int W) {
    return (long long)B * 2 * 2048 * 4 + (long long)B * 2 * 4 * 4 + (long long)B * depth_blocks(H, W) * 6 * 8 + 64;
}

extern "C" int ccb_depth_errors(const float* gt, const float* pred, int B, int H, int W, int crop, void* work, float* out6,
                                ccb_stream_t stream) {
    CCB_REQUIRE(gt && pred && work && out6, CCB_ERR_ARG, "depth_errors: null pointer");
    CCB_REQUIRE(B > 0 && H > 0 && W > 0, CCB_ERR_ARG, "depth_errors: bad sizes");
    DepthArgs a;
    a.gt = gt; a.pred = pred; a.B = B; a.H = H; a.W = W; a.out = out6;
    a.y1 = 0; a.y2 = H; a.x1 = 0; a.x2 = W;
    if (crop) {            // int(0.40810811 * H) etc. evaluated in double like python (:441-442)
        a.y1 = (int)(0.40810811 * H); a.y2 = (int)(0.99189189 * H);
        a.x1 = (int)(0.03594771 * W); a.x2 = (int)(0.96405229 * W);
    }
    char* p = (char*)work;
    a.partials = (double*)p;   p += (long long)B * depth_blocks(H, W) * 6 * 8;
    a.hist = (unsigned*)p;     p += (long long)B * 2 * 2048 * 4;
    a.sel = (unsigned*)p;
    const int nb = depth_blocks(H, W);
#ifdef CCB_CPU_SIM
    memset(a.hist, 0, (size_t)B * 2 * 2048 * 4 + (size_t)B * 2 * 4 * 4);
#else
    cudaMemsetAsync(a.hist, 0, (size_t)B * 2 * 2048 * 4 + (size_t)B * 2 * 4 * 4, (cudaStream_t)stream);
#endif
    for (int pass = 0; pass < 3; ++pass) {
        CCB_LAUNCH(depth_hist_kernel, dim3(nb, B), dim3(256), 0, stream, a, pass);
        CCB_LAUNCH(depth_select_kernel, dim3((B * 2 + 63) / 64), dim3(64), 0, stream, a, pass);
    }
    CCB_LAUNCH(depth_errors_kernel, dim3(nb, B), dim3(256), 0, stream, a);
    CCB_LAUNCH(depth_errors_finalize, dim3(1), dim3(32), 0, stream, a, nb);
    return check_launch("depth_errors");
}

extern "C" int ccb_prep_frames(const unsigned char* src_u8, float* const* dst, const float* params, const int* offs, int B, int F,
                               int Hs, int Ws, int H, int W, ccb_stream_t stream) {
    CCB_REQUIRE(src_u8 && dst && params && offs, CCB_ERR_ARG, "prep_frames: null pointer");
    CCB_REQUIRE(F >= 1 && F <= 8, CCB_ERR_ARG, "prep_frames: 1..8 frames per sample, got %d", F);
    CCB_REQUIRE(B > 0 && Hs > 0 && Ws > 0 && H > 0 && W > 0, CCB_ERR_ARG, "prep_frames: bad sizes");
    PrepArgs a;
    a.src = src_u8; a.params = params; a.offs = offs; a.B = B; a.F = F; a.Hs = Hs; a.Ws = Ws; a.H = H; a.W = W;
    for (int f = 0; f < 8; ++f) a.dst[f] = (f < F) ? dst[f] : nullptr;
    for (int f = 0; f < F; ++f) CCB_REQUIRE(a.dst[f] != nullptr, CCB_ERR_ARG, "prep_frames: dst[%d] is null", f);
    CCB_LAUNCH(prep_frames_kernel, dim3(grid_for((long long)B * F * H * W)), dim3(256), 0, stream, a);
    return check_launch("prep_frames");
}
