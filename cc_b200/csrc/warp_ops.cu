// warp_ops.cu - image pyramid and the stand-alone warp-layer ops the reference exports by name
// (train.py:22: inverse_warp, pose2flow, flow2oob, flow_warp; loss_functions.py:10: ssim).
#include "ssim_tile.cuh"

namespace ccb {

// ------------------------------------------------------------------------------------------------
// Image pyramid: one CTA reduces a 32x32 full-res tile of one plane through every level
// (2x2 means of 2x2 means == exact 2^l box mean up to fp32 summation order).
struct PyrArgs {
    const float* img;
    float* out[CCB_MAX_LEVELS];
    int H, W, nlevels;
};

__global__ void __launch_bounds__(256) pyramid_kernel(const PyrArgs a) {
    CCB_PDL_WAIT();
    __shared__ float s[2][16 * 16];
    const int plane = blockIdx.z, ty0 = blockIdx.y * 32, tx0 = blockIdx.x * 32;
    const int tid = threadIdx.x;
    const float* src = a.img + (long long)plane * a.H * a.W;
    int n = 16;   // side of the current level inside the tile
    {
        int qy = tid >> 4, qx = tid & 15;
        int y = ty0 + 2 * qy, x = tx0 + 2 * qx;
        float v = 0.f;
        if (y + 1 < a.H + 0 && x + 1 < a.W + 0 && y < a.H && x < a.W) {
            const float* p = src + (long long)y * a.W + x;
            v = 0.25f * ((__ldg(p) + __ldg(p + 1)) + (__ldg(p + a.W) + __ldg(p + a.W + 1)));
            int h1 = a.H >> 1, w1 = a.W >> 1;
            a.out[1][(long long)plane * h1 * w1 + (long long)(y >> 1) * w1 + (x >> 1)] = v;
        }
        s[0][tid] = v;
    }
    int cur = 0;
    for (int l = 2; l < a.nlevels; ++l) {
        __syncthreads();
        int m = n >> 1;
        if (tid < m * m) {
            int qy = tid / m, qx = tid - qy * m;
            const float* p = &s[cur][(2 * qy) * n + 2 * qx];
            float v = 0.25f * ((p[0] + p[1]) + (p[n] + p[n + 1]));
            s[cur ^ 1][qy * m + qx] = v;
            int hl = a.H >> l, wl = a.W >> l;
            int y = (ty0 >> l) + qy, x = (tx0 >> l) + qx;
            if (y < hl && x < wl) a.out[l][(long long)plane * hl * wl + (long long)y * wl + x] = v;
        }
        cur ^= 1;
        n = m;
    }
}

// ------------------------------------------------------------------------------------------------
struct WarpArgs {
    const float* img;
    const float* depth;
    const float* pose;
    int pose_stride;
    const float* K;
    const float* Kinv;
    const float* flow;
    const float* grad_out;
    float* out;
    float* d_depth;
    float* d_flow;
    float* d_img;
    unsigned long long* d_img_fx;   // flow-warp backward: fixed-point accumulators of d_img, then max |grad_out| bits
    float* d_pose;
    float* pose_partials;
    int B, C, h, w, rot, pad;
    int b2f_norm;     // 1: Back2Future.warp normalisation 2*(x+u)/max(W-1,1)-1 (back2future.py:305-306)
};

constexpr int WNT = 256;

// inverse_warp forward (inverse_warp.py:250-283) / pose2flow forward (:195-220)
template <bool FLOW_OUT>
__global__ void __launch_bounds__(WNT) rigid_fwd_kernel(const WarpArgs a) {
    CCB_PDL_WAIT();
    __shared__ Cam cam;
    const int b = blockIdx.y;
    if (threadIdx.x == 0)
        make_cam(a.pose + (long long)b * a.pose_stride, a.K + b * 9, a.Kinv + b * 9, 1.f, a.rot, a.w, a.h, cam);
    __syncthreads();
    const long long hw = (long long)a.h * a.w;
    long long idx = (long long)blockIdx.x * WNT + threadIdx.x;
    if (idx >= hw) return;
    int y = (int)(idx / a.w), x = (int)(idx - (long long)y * a.w);
    float dep = __ldg(a.depth + b * hw + idx);
    Proj p = project(cam, (float)x, (float)y, dep, a.pad == CCB_PAD_ZEROS);
    if (FLOW_OUT) {
        float u, v;
        coords_to_flow(cam, p.Xn, p.Yn, (float)x, (float)y, u, v);
        a.out[(long long)b * 2 * hw + idx] = u;
        a.out[(long long)b * 2 * hw + hw + idx] = v;
    } else {
        Samp s = make_samp(p.Xn, p.Yn, a.w, a.h, a.pad);
        const float* im = a.img + (long long)b * 3 * hw;
#pragma unroll
        for (int c = 0; c < 3; ++c) a.out[(long long)b * 3 * hw + c * hw + idx] = interp(fetch(im + c * hw, s, a.w), s);
    }
}

template <bool FLOW_OUT>
__global__ void __launch_bounds__(WNT) rigid_bwd_kernel(const WarpArgs a) {
    CCB_PDL_WAIT();
    __shared__ Cam cam;
    __shared__ float s_red[12 * 32];
    const int b = blockIdx.y;
    if (threadIdx.x == 0)
        make_cam(a.pose + (long long)b * a.pose_stride, a.K + b * 9, a.Kinv + b * 9, 1.f, a.rot, a.w, a.h, cam);
    __syncthreads();
    const long long hw = (long long)a.h * a.w;
    long long idx = (long long)blockIdx.x * WNT + threadIdx.x;
    float acc[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) acc[k] = 0.f;
    if (idx < hw) {
        int y = (int)(idx / a.w), x = (int)(idx - (long long)y * a.w);
        float dep = __ldg(a.depth + b * hw + idx);
        Proj p = project(cam, (float)x, (float)y, dep, a.pad == CCB_PAD_ZEROS);
        float gXn, gYn;
        if (FLOW_OUT) {
            gXn = __ldg(a.grad_out + (long long)b * 2 * hw + idx) * cam.w1 * 0.5f;
            gYn = __ldg(a.grad_out + (long long)b * 2 * hw + hw + idx) * cam.h1 * 0.5f;
        } else {
            Samp s = make_samp(p.Xn, p.Yn, a.w, a.h, a.pad);
            const float* im = a.img + (long long)b * 3 * hw;
            float gix = 0.f, giy = 0.f;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                Corners cr = fetch(im + c * hw, s, a.w);
                float g = __ldg(a.grad_out + (long long)b * 3 * hw + c * hw + idx);
                gix += g * interp_dx(cr, s);
                giy += g * interp_dy(cr, s);
            }
            gXn = gix * s.gmx;
            gYn = giy * s.gmy;
        }
        a.d_depth[b * hw + idx] = project_bwd(cam, p, gXn, gYn, acc);
    }
    block_sum<12>(acc, s_red);
    if (threadIdx.x == 0) {
        float* po = a.pose_partials + ((long long)b * gridDim.x + blockIdx.x) * 12;
#pragma unroll
        for (int k = 0; k < 12; ++k) po[k] = acc[k];
    }
}

__global__ void rigid_pose_finalize(const WarpArgs a, int nblk) {
    CCB_PDL_WAIT();
    const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (wid >= a.B) return;
    float dP[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) dP[k] = 0.f;
    for (int t = lane; t < nblk; t += 32) {
        const float* p = a.pose_partials + ((long long)wid * nblk + t) * 12;
#pragma unroll
        for (int k = 0; k < 12; ++k) dP[k] += p[k];
    }
#pragma unroll
    for (int k = 0; k < 12; ++k) dP[k] = warp_sum(dP[k]);
    if (lane == 0) {
        Cam cm;
        make_cam(a.pose + (long long)wid * a.pose_stride, a.K + wid * 9, a.Kinv + wid * 9, 1.f, a.rot, a.w, a.h, cm);
        float dpose[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        pose_grad_from_dP(cm, dP, a.rot, dpose);
#pragma unroll
        for (int k = 0; k < 6; ++k) a.d_pose[wid * 6 + k] = dpose[k];
    }
}

__device__ __forceinline__ void warp_coords(const WarpArgs& a, float x, float y, float u, float v, float& Xn, float& Yn) {
    if (a.b2f_norm) {
        Xn = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, __fadd_rn(x, u)), (float)max(a.w - 1, 1)), 1.f);
        Yn = __fsub_rn(__fdiv_rn(__fmul_rn(2.f, __fadd_rn(y, v)), (float)max(a.h - 1, 1)), 1.f);
    } else {
        flow_coords(x, y, u, v, (float)(a.w - 1), (float)(a.h - 1), Xn, Yn);
    }
}

// ------------------------------------------------------------------------------------------------
// The image gradient of a bilinear sample is a scatter: an arbitrary flow can send any number of output pixels to one
// source pixel.  Float atomics would make the sum depend on the order the hardware serialises them in, and the training
// step (DispResNet6's chaotic gradient above all) would not compute the same thing twice.  The scatter therefore adds
// 64-bit fixed-point integers - integer addition is associative, so the result is independent of the order:
//   pass 1  max |grad_out| over the finite values (an order-free max, as integer bits)
//   pass 2  each contribution v -> round(v * 2^s) added to its accumulator, s = 62 - e - c with grad_out < 2^e and
//           h*w < 2^c: at most h*w contributions of magnitude <= max |grad_out| reach one accumulator, so none overflows,
//           and the resolution is 2^-(62 - c) of max |grad_out| (2^-44 at 256x832), far below fp32 rounding of the sum
//   pass 3  d_img += accumulator * 2^-s
// A non-finite contribution (inf / NaN in grad_out) cannot be held in fixed point: it goes straight into its own d_img
// element with a float atomic, as an unfixed scatter would put it - an inf / NaN sum does not depend on the order either.
__device__ __forceinline__ double fx_scale(const WarpArgs& a) {
    const float gmax = __uint_as_float((unsigned)a.d_img_fx[(long long)a.B * a.C * a.h * a.w]);
    if (!(gmax > 0.f)) return 1.0;
    const long long hw = (long long)a.h * a.w;
    const int e = ilogbf(gmax) + 1, c = 64 - __clzll(hw);
    return ldexp(1.0, 62 - e - c);
}
__device__ __forceinline__ void fx_add(const WarpArgs& a, long long i, float v, double scale) {
    if (isfinite(v)) atomicAdd(a.d_img_fx + i, (unsigned long long)__double2ll_rn((double)v * scale));
    else atomicAdd(a.d_img + i, v);
}
__device__ __forceinline__ void fx_scatter(const WarpArgs& a, long long plane_off, const Samp& s, float g, double scale) {
    const long long i = plane_off + (long long)s.y0 * a.w + s.x0;
    if (s.oky0 && s.okx0) fx_add(a, i, g * s.wy0 * s.wx0, scale);
    if (s.oky0 && s.okx1) fx_add(a, i + 1, g * s.wy0 * s.wx1, scale);
    if (s.oky1 && s.okx0) fx_add(a, i + a.w, g * s.wy1 * s.wx0, scale);
    if (s.oky1 && s.okx1) fx_add(a, i + a.w + 1, g * s.wy1 * s.wx1, scale);
}

__global__ void __launch_bounds__(WNT) fx_absmax_kernel(const WarpArgs a, long long n) {
    CCB_PDL_WAIT();
    unsigned m = 0;
    for (long long i = (long long)blockIdx.x * WNT + threadIdx.x; i < n; i += (long long)gridDim.x * WNT) {
        const unsigned bits = __float_as_uint(__ldg(a.grad_out + i)) & 0x7fffffffu;   // |g| as bits: ordered like the values
        if (bits < 0x7f800000u) m = max(m, bits);                                        // finite only
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) atomicMax(a.d_img_fx + n, (unsigned long long)m);
}

__global__ void __launch_bounds__(WNT) fx_finish_kernel(const WarpArgs a, long long n) {
    CCB_PDL_WAIT();
    const long long i = (long long)blockIdx.x * WNT + threadIdx.x;
    if (i >= n) return;
    a.d_img[i] += (float)((double)(long long)a.d_img_fx[i] / fx_scale(a));
}

// flow_warp (inverse_warp.py:164-192), any channel count
__global__ void __launch_bounds__(WNT) flow_warp_fwd_kernel(const WarpArgs a) {
    CCB_PDL_WAIT();
    const int b = blockIdx.y;
    const long long hw = (long long)a.h * a.w;
    long long idx = (long long)blockIdx.x * WNT + threadIdx.x;
    if (idx >= hw) return;
    int y = (int)(idx / a.w), x = (int)(idx - (long long)y * a.w);
    float Xn, Yn;
    warp_coords(a, (float)x, (float)y, __ldg(a.flow + (long long)b * 2 * hw + idx), __ldg(a.flow + (long long)b * 2 * hw + hw + idx),
                Xn, Yn);
    Samp s = make_samp(Xn, Yn, a.w, a.h, a.pad);
    const float* im = a.img + (long long)b * a.C * hw;
    for (int c = 0; c < a.C; ++c) a.out[(long long)b * a.C * hw + c * hw + idx] = interp(fetch(im + c * hw, s, a.w), s);
}

__global__ void __launch_bounds__(WNT) flow_warp_bwd_kernel(const WarpArgs a) {
    CCB_PDL_WAIT();
    const int b = blockIdx.y;
    const long long hw = (long long)a.h * a.w;
    long long idx = (long long)blockIdx.x * WNT + threadIdx.x;
    if (idx >= hw) return;
    int y = (int)(idx / a.w), x = (int)(idx - (long long)y * a.w);
    float Xn, Yn;
    const float w1 = (float)max(a.w - 1, 1), h1 = (float)max(a.h - 1, 1);
    warp_coords(a, (float)x, (float)y, __ldg(a.flow + (long long)b * 2 * hw + idx), __ldg(a.flow + (long long)b * 2 * hw + hw + idx),
                Xn, Yn);
    Samp s = make_samp(Xn, Yn, a.w, a.h, a.pad);
    const float* im = a.img + (long long)b * a.C * hw;
    float gix = 0.f, giy = 0.f;
    const double scale = a.d_img ? fx_scale(a) : 1.0;
    for (int c = 0; c < a.C; ++c) {
        float g = __ldg(a.grad_out + (long long)b * a.C * hw + c * hw + idx);
        if (a.d_flow) {
            Corners cr = fetch(im + c * hw, s, a.w);
            gix += g * interp_dx(cr, s);
            giy += g * interp_dy(cr, s);
        }
        if (a.d_img) fx_scatter(a, (long long)b * a.C * hw + c * hw, s, g, scale);
    }
    if (a.d_flow) {
        a.d_flow[(long long)b * 2 * hw + idx] = gix * s.gmx * (2.f / w1);
        a.d_flow[(long long)b * 2 * hw + hw + idx] = giy * s.gmy * (2.f / h1);
    }
}

// ------------------------------------------------------------------------------------------------
// Stand-alone SSIM (ssim.py:68-76).  One CTA = one plane x one 64x20 tile.
struct SsimArgs {
    const float* x;
    const float* y;
    const float* gout;
    float* out;
    float* dx;
    float* dy;
    float* work;       // [5][planes*h*w]
    int planes, h, w;
    float taps[CCB_SSIM_TAPS];
};

__device__ __forceinline__ void stage_plane(const float* __restrict__ src, float* __restrict__ dst, int h, int w,
                                            int x0, int y0) {
    using T = Tile<6>;
    for (int idx = threadIdx.x; idx < T::RH * T::RW; idx += NT) {
        int ry = idx / T::RW, rx = idx - ry * T::RW;
        int gy = y0 - 6 + ry, gx = x0 - 6 + rx;
        bool in = (gy >= 0) && (gy < h) && (gx >= 0) && (gx < w);
        dst[ry * T::PITCH + rx] = in ? __ldg(src + (long long)gy * w + gx) : 0.f;
    }
}

// PASS 0: write the SSIM map.  PASS 1: write grad_out * dS/d(mu1,Exx,mu2,Eyy,Exy) into work.
template <int PASS>
__global__ void __launch_bounds__(NT, 2) ssim_map_kernel(const SsimArgs a) {
    CCB_PDL_WAIT();
    using T = Tile<6>;
    CCB_DYN_SMEM(smem_raw);
    float* sx = reinterpret_cast<float*>(smem_raw);
    float* sy = sx + T::PLANE;
    float* sH = sy + T::PLANE;
    __shared__ float s_g[CCB_SSIM_TAPS];
    const int plane = blockIdx.z, x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    const long long hw = (long long)a.h * a.w;
    if (threadIdx.x < CCB_SSIM_TAPS) s_g[threadIdx.x] = a.taps[threadIdx.x];
    stage_plane(a.x + plane * hw, sx, a.h, a.w, x0, y0);
    stage_plane(a.y + plane * hw, sy, a.h, a.w, x0, y0);
    __syncthreads();
    float mx[2][PXT], my[3][PXT];
    hpass<0>(sx, nullptr, nullptr, sH, s_g);
    __syncthreads();
    vpass<2>(sH, s_g, mx);
    __syncthreads();
    hpass<1>(sx, sy, nullptr, sH, s_g);
    __syncthreads();
    vpass<3>(sH, s_g, my);
    const int col = threadIdx.x & 63, rg = threadIdx.x >> 6;
#pragma unroll
    for (int j = 0; j < PXT; ++j) {
        int py = y0 + rg * PXT + j, px = x0 + col;
        if (py < a.h && px < a.w) {
            float d2, dyy, dxy, d1, dxx, dxy2;
            float S = ssim_point(mx[0][j], mx[1][j], my[0][j], my[1][j], my[2][j], d2, dyy, dxy);
            long long o = plane * hw + (long long)py * a.w + px;
            if (PASS == 0) {
                a.out[o] = S;
            } else {
                ssim_point(my[0][j], my[1][j], mx[0][j], mx[1][j], my[2][j], d1, dxx, dxy2);   // roles swapped
                const long long n = (long long)a.planes * hw;
                float g = __ldg(a.gout + o);
                a.work[o] = g * d1;
                a.work[n + o] = g * dxx;
                a.work[2 * n + o] = g * d2;
                a.work[3 * n + o] = g * dyy;
                a.work[4 * n + o] = g * dxy;
            }
        }
    }
}

// d img1 = G*(g dmu1) + 2 x G*(g dExx) + y G*(g dExy);  d img2 symmetric (SURVEY A.4)
__global__ void __launch_bounds__(NT, 2) ssim_bwd_kernel(const SsimArgs a) {
    CCB_PDL_WAIT();
    using T = Tile<6>;
    CCB_DYN_SMEM(smem_raw);
    float* sD = reinterpret_cast<float*>(smem_raw);   // 3 planes
    float* sH = sD + 3 * T::PLANE;
    __shared__ float s_g[CCB_SSIM_TAPS];
    const int plane = blockIdx.z, x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
    const long long hw = (long long)a.h * a.w, n = (long long)a.planes * hw;
    if (threadIdx.x < CCB_SSIM_TAPS) s_g[threadIdx.x] = a.taps[threadIdx.x];
    float b1[3][PXT], b2[3][PXT];
    // maps 0 (dmu1), 1 (dExx), 4 (dExy)
    stage_plane(a.work + plane * hw, sD, a.h, a.w, x0, y0);
    stage_plane(a.work + n + plane * hw, sD + T::PLANE, a.h, a.w, x0, y0);
    stage_plane(a.work + 4 * n + plane * hw, sD + 2 * T::PLANE, a.h, a.w, x0, y0);
    __syncthreads();
    hpass<2>(sD, sD + T::PLANE, sD + 2 * T::PLANE, sH, s_g);
    __syncthreads();
    vpass<3>(sH, s_g, b1);
    __syncthreads();
    // maps 2 (dmu2), 3 (dEyy)  (third slot reuses dExy: ignored)
    stage_plane(a.work + 2 * n + plane * hw, sD, a.h, a.w, x0, y0);
    stage_plane(a.work + 3 * n + plane * hw, sD + T::PLANE, a.h, a.w, x0, y0);
    __syncthreads();
    hpass<2>(sD, sD + T::PLANE, sD + 2 * T::PLANE, sH, s_g);
    __syncthreads();
    vpass<3>(sH, s_g, b2);
    const int col = threadIdx.x & 63, rg = threadIdx.x >> 6;
#pragma unroll
    for (int j = 0; j < PXT; ++j) {
        int py = y0 + rg * PXT + j, px = x0 + col;
        if (py < a.h && px < a.w) {
            long long o = plane * hw + (long long)py * a.w + px;
            float xv = __ldg(a.x + o), yv = __ldg(a.y + o);
            if (a.dx) a.dx[o] = b1[0][j] + 2.f * xv * b1[1][j] + yv * b1[2][j];
            if (a.dy) a.dy[o] = b2[0][j] + 2.f * yv * b2[1][j] + xv * b1[2][j];
        }
    }
}

}  // namespace ccb

using namespace ccb;

extern "C" int ccb_image_pyramid(const float* img, int planes, int H, int W, int nlevels,
                                 float* const* out_levels, ccb_stream_t stream) {
    CCB_REQUIRE(img && out_levels, CCB_ERR_ARG, "image_pyramid: null pointer");
    CCB_REQUIRE(nlevels >= 1 && nlevels <= 6, CCB_ERR_ARG, "image_pyramid: nlevels %d not in [1,6]", nlevels);
    if (nlevels == 1) return CCB_OK;
    int div = 1 << (nlevels - 1);
    CCB_REQUIRE(H % div == 0 && W % div == 0, CCB_ERR_ARG, "image_pyramid: %dx%d not divisible by %d", H, W, div);
    PyrArgs a;
    a.img = img; a.H = H; a.W = W; a.nlevels = nlevels;
    a.out[0] = nullptr;
    for (int l = 1; l < nlevels; ++l) {
        CCB_REQUIRE(out_levels[l - 1] != nullptr, CCB_ERR_ARG, "image_pyramid: out level %d null", l);
        a.out[l] = out_levels[l - 1];
    }
    CCB_LAUNCH(pyramid_kernel, dim3(cdiv(W, 32), cdiv(H, 32), planes), dim3(256), 0, stream, a);
    return check_launch("image_pyramid");
}

static int warp_common(WarpArgs& a, const float* depth, const float* pose, int pose_stride, const float* K,
                       const float* Kinv, int B, int h, int w, int rot, int pad) {
    CCB_REQUIRE(depth && pose && K && Kinv, CCB_ERR_ARG, "warp: null input");
    CCB_REQUIRE(B >= 1 && h >= 2 && w >= 2, CCB_ERR_ARG, "warp: bad size B=%d h=%d w=%d", B, h, w);
    CCB_REQUIRE(rot == CCB_ROT_EULER || rot == CCB_ROT_QUAT, CCB_ERR_ARG, "warp: bad rotation_mode %d", rot);
    memset(&a, 0, sizeof(a));
    a.depth = depth; a.pose = pose; a.pose_stride = pose_stride; a.K = K; a.Kinv = Kinv;
    a.B = B; a.C = 3; a.h = h; a.w = w; a.rot = rot; a.pad = pad;
    return CCB_OK;
}

extern "C" long long ccb_warp_pose_partials_floats(int B, int h, int w) {
    if (B < 1 || h < 1 || w < 1) return -1;
    return (long long)B * cdiv(h * w, WNT) * 12;
}

extern "C" int ccb_inverse_warp_fwd(const float* img, const float* depth, const float* pose, int pose_stride,
                                    const float* K, const float* Kinv, int B, int h, int w, int rotation_mode,
                                    int padding_mode, float* out, ccb_stream_t stream) {
    WarpArgs a;
    int rc = warp_common(a, depth, pose, pose_stride, K, Kinv, B, h, w, rotation_mode, padding_mode);
    if (rc) return rc;
    CCB_REQUIRE(img && out, CCB_ERR_ARG, "inverse_warp_fwd: null img/out");
    CCB_REQUIRE(padding_mode == CCB_PAD_ZEROS || padding_mode == CCB_PAD_BORDER, CCB_ERR_ARG, "inverse_warp: bad padding_mode");
    a.img = img; a.out = out;
    CCB_LAUNCH(rigid_fwd_kernel<false>, dim3(cdiv(h * w, WNT), B), dim3(WNT), 0, stream, a);
    return check_launch("inverse_warp_fwd");
}

extern "C" int ccb_inverse_warp_bwd(const float* img, const float* depth, const float* pose, int pose_stride,
                                    const float* K, const float* Kinv, int B, int h, int w, int rotation_mode,
                                    int padding_mode, const float* grad_out, float* d_depth, float* d_pose,
                                    float* pose_partials, long long pose_partials_floats, ccb_stream_t stream) {
    WarpArgs a;
    int rc = warp_common(a, depth, pose, pose_stride, K, Kinv, B, h, w, rotation_mode, padding_mode);
    if (rc) return rc;
    CCB_REQUIRE(img && grad_out && d_depth && d_pose, CCB_ERR_ARG, "inverse_warp_bwd: null pointer");
    CCB_REQUIRE_WORK("inverse_warp_bwd", "pose_partials", pose_partials, pose_partials_floats, ccb_warp_pose_partials_floats(B, h, w));
    a.img = img; a.grad_out = grad_out; a.d_depth = d_depth; a.d_pose = d_pose; a.pose_partials = pose_partials;
    int nblk = cdiv(h * w, WNT);
    CCB_LAUNCH(rigid_bwd_kernel<false>, dim3(nblk, B), dim3(WNT), 0, stream, a);
    rc = check_launch("inverse_warp_bwd");
    if (rc) return rc;
    CCB_LAUNCH(rigid_pose_finalize, dim3(cdiv(B * 32, 128)), dim3(128), 0, stream, a, nblk);
    return check_launch("inverse_warp_pose_finalize");
}

extern "C" int ccb_pose2flow_fwd(const float* depth, const float* pose, int pose_stride, const float* K,
                                 const float* Kinv, int B, int h, int w, int rotation_mode, int padding_mode,
                                 float* flow, ccb_stream_t stream) {
    WarpArgs a;
    int rc = warp_common(a, depth, pose, pose_stride, K, Kinv, B, h, w, rotation_mode, padding_mode);
    if (rc) return rc;
    CCB_REQUIRE(flow, CCB_ERR_ARG, "pose2flow_fwd: null out");
    a.out = flow;
    CCB_LAUNCH(rigid_fwd_kernel<true>, dim3(cdiv(h * w, WNT), B), dim3(WNT), 0, stream, a);
    return check_launch("pose2flow_fwd");
}

extern "C" int ccb_pose2flow_bwd(const float* depth, const float* pose, int pose_stride, const float* K,
                                 const float* Kinv, int B, int h, int w, int rotation_mode, int padding_mode,
                                 const float* grad_flow, float* d_depth, float* d_pose, float* pose_partials,
                                 long long pose_partials_floats, ccb_stream_t stream) {
    WarpArgs a;
    int rc = warp_common(a, depth, pose, pose_stride, K, Kinv, B, h, w, rotation_mode, padding_mode);
    if (rc) return rc;
    CCB_REQUIRE(grad_flow && d_depth && d_pose, CCB_ERR_ARG, "pose2flow_bwd: null pointer");
    CCB_REQUIRE_WORK("pose2flow_bwd", "pose_partials", pose_partials, pose_partials_floats, ccb_warp_pose_partials_floats(B, h, w));
    a.grad_out = grad_flow; a.d_depth = d_depth; a.d_pose = d_pose; a.pose_partials = pose_partials;
    int nblk = cdiv(h * w, WNT);
    CCB_LAUNCH(rigid_bwd_kernel<true>, dim3(nblk, B), dim3(WNT), 0, stream, a);
    rc = check_launch("pose2flow_bwd");
    if (rc) return rc;
    CCB_LAUNCH(rigid_pose_finalize, dim3(cdiv(B * 32, 128)), dim3(128), 0, stream, a, nblk);
    return check_launch("pose2flow_pose_finalize");
}

// Small maps with many channels (Back2Future's feature warps at 8x26 .. 16x52 with 96-128 channels): a thread per pixel
// leaves 4-16 CTAs looping serially over the channels (measured: 70-92 us per call on 4-16 CTAs).  Here a WARP takes a
// pixel and its lanes take the channels; the flow gradient is a shuffle reduction (fixed order).
__global__ void __launch_bounds__(WNT) flow_warp_fwd_wpp_kernel(const WarpArgs a) {
    CCB_PDL_WAIT();
    const long long hw = (long long)a.h * a.w;
    const long long pix = (long long)blockIdx.x * (WNT / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (pix >= hw * a.B) return;
    const int b = (int)(pix / hw);
    const long long idx = pix - (long long)b * hw;
    const int y = (int)(idx / a.w), x = (int)(idx - (long long)y * a.w);
    float Xn, Yn;
    warp_coords(a, (float)x, (float)y, __ldg(a.flow + (long long)b * 2 * hw + idx), __ldg(a.flow + (long long)b * 2 * hw + hw + idx), Xn, Yn);
    const Samp s = make_samp(Xn, Yn, a.w, a.h, a.pad);
    const float* im = a.img + (long long)b * a.C * hw;
    for (int c = lane; c < a.C; c += 32) a.out[(long long)b * a.C * hw + c * hw + idx] = interp(fetch(im + c * hw, s, a.w), s);
}

__global__ void __launch_bounds__(WNT) flow_warp_bwd_wpp_kernel(const WarpArgs a) {
    CCB_PDL_WAIT();
    const long long hw = (long long)a.h * a.w;
    const long long pix = (long long)blockIdx.x * (WNT / 32) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (pix >= hw * a.B) return;                              // whole warps leave together
    const int b = (int)(pix / hw);
    const long long idx = pix - (long long)b * hw;
    const int y = (int)(idx / a.w), x = (int)(idx - (long long)y * a.w);
    float Xn, Yn;
    const float w1 = (float)max(a.w - 1, 1), h1 = (float)max(a.h - 1, 1);
    warp_coords(a, (float)x, (float)y, __ldg(a.flow + (long long)b * 2 * hw + idx), __ldg(a.flow + (long long)b * 2 * hw + hw + idx), Xn, Yn);
    const Samp s = make_samp(Xn, Yn, a.w, a.h, a.pad);
    const float* im = a.img + (long long)b * a.C * hw;
    float gix = 0.f, giy = 0.f;
    const double scale = a.d_img ? fx_scale(a) : 1.0;
    for (int c = lane; c < a.C; c += 32) {
        const float g = __ldg(a.grad_out + (long long)b * a.C * hw + c * hw + idx);
        if (a.d_flow) {
            const Corners cr = fetch(im + c * hw, s, a.w);
            gix += g * interp_dx(cr, s);
            giy += g * interp_dy(cr, s);
        }
        if (a.d_img) fx_scatter(a, (long long)b * a.C * hw + c * hw, s, g, scale);
    }
    if (a.d_flow) {
        gix = warp_sum(gix);
        giy = warp_sum(giy);
        if (lane == 0) {
            a.d_flow[(long long)b * 2 * hw + idx] = gix * s.gmx * (2.f / w1);
            a.d_flow[(long long)b * 2 * hw + hw + idx] = giy * s.gmy * (2.f / h1);
        }
    }
}

// The image gradient's fixed-point scatter buffer: one accumulator per element, then max |grad_out| (pass 1 above).
static long long scatter_words(int B, int C, int h, int w) { return (long long)B * C * h * w + 1; }
static bool warp_per_pixel(int B, int C, int h, int w) { return C >= 16 && (long long)B * h * w < 32768; }
static void launch_flow_warp(const WarpArgs& a, bool bwd, cudaStream_t st) {
    const long long n = (long long)a.B * a.C * a.h * a.w;
    if (bwd && a.d_img) {
        cudaMemsetAsync(a.d_img_fx, 0, (size_t)scatter_words(a.B, a.C, a.h, a.w) * sizeof(unsigned long long), st);
        const long long nb = (n + WNT - 1) / WNT;
        CCB_LAUNCH(fx_absmax_kernel, dim3((unsigned)(nb < 4 * NUM_SMS ? nb : 4 * NUM_SMS)), dim3(WNT), 0, st, a, n);
    }
    if (warp_per_pixel(a.B, a.C, a.h, a.w)) {
        const unsigned nb = (unsigned)cdiv((int)((long long)a.B * a.h * a.w), WNT / 32);
        if (bwd) CCB_LAUNCH(flow_warp_bwd_wpp_kernel, dim3(nb), dim3(WNT), 0, st, a);
        else CCB_LAUNCH(flow_warp_fwd_wpp_kernel, dim3(nb), dim3(WNT), 0, st, a);
    } else {
        if (bwd) CCB_LAUNCH(flow_warp_bwd_kernel, dim3(cdiv(a.h * a.w, WNT), a.B), dim3(WNT), 0, st, a);
        else CCB_LAUNCH(flow_warp_fwd_kernel, dim3(cdiv(a.h * a.w, WNT), a.B), dim3(WNT), 0, st, a);
    }
    if (bwd && a.d_img) CCB_LAUNCH(fx_finish_kernel, dim3((unsigned)((n + WNT - 1) / WNT)), dim3(WNT), 0, st, a, n);
}

extern "C" int ccb_flow_warp_fwd(const float* img, const float* flow, int B, int C, int h, int w,
                                 int padding_mode, float* out, ccb_stream_t stream) {
    CCB_REQUIRE(img && flow && out, CCB_ERR_ARG, "flow_warp_fwd: null pointer");
    CCB_REQUIRE(B >= 1 && C >= 1 && h >= 2 && w >= 2, CCB_ERR_ARG, "flow_warp_fwd: bad size");
    WarpArgs a;
    memset(&a, 0, sizeof(a));
    a.img = img; a.flow = flow; a.out = out; a.B = B; a.C = C; a.h = h; a.w = w; a.pad = padding_mode;
    launch_flow_warp(a, false, (cudaStream_t)stream);
    return check_launch("flow_warp_fwd");
}

extern "C" int ccb_flow_warp_bwd(const float* img, const float* flow, int B, int C, int h, int w,
                                 int padding_mode, const float* grad_out, float* d_flow, float* d_img,
                                 unsigned long long* work, long long work_words, ccb_stream_t stream) {
    CCB_REQUIRE(img && flow && grad_out, CCB_ERR_ARG, "flow_warp_bwd: null pointer");
    CCB_REQUIRE(B >= 1 && C >= 1 && h >= 1 && w >= 1, CCB_ERR_ARG, "flow_warp_bwd: bad size");
    CCB_REQUIRE_WORK("flow_warp_bwd", "work", work, work_words, d_img ? scatter_words(B, C, h, w) : 0);
    WarpArgs a;
    memset(&a, 0, sizeof(a));
    a.img = img; a.flow = flow; a.grad_out = grad_out; a.d_flow = d_flow; a.d_img = d_img; a.d_img_fx = work;
    a.B = B; a.C = C; a.h = h; a.w = w; a.pad = padding_mode;
    launch_flow_warp(a, true, (cudaStream_t)stream);
    return check_launch("flow_warp_bwd");
}

// Back2Future.warp (back2future.py:287-321): border padding, b2f coordinate normalisation
extern "C" int ccb_featwarp_fwd(const float* x, const float* flow, int B, int C, int h, int w, float* out,
                                ccb_stream_t stream) {
    CCB_REQUIRE(x && flow && out, CCB_ERR_ARG, "featwarp_fwd: null pointer");
    WarpArgs a;
    memset(&a, 0, sizeof(a));
    a.img = x; a.flow = flow; a.out = out; a.B = B; a.C = C; a.h = h; a.w = w; a.pad = CCB_PAD_BORDER; a.b2f_norm = 1;
    launch_flow_warp(a, false, (cudaStream_t)stream);
    return check_launch("featwarp_fwd");
}

extern "C" int ccb_featwarp_bwd(const float* x, const float* flow, int B, int C, int h, int w, const float* grad_out,
                                float* d_flow, float* d_x, unsigned long long* work, long long work_words, ccb_stream_t stream) {
    CCB_REQUIRE(x && flow && grad_out, CCB_ERR_ARG, "featwarp_bwd: null pointer");
    CCB_REQUIRE(B >= 1 && C >= 1 && h >= 1 && w >= 1, CCB_ERR_ARG, "featwarp_bwd: bad size");
    CCB_REQUIRE_WORK("featwarp_bwd", "work", work, work_words, d_x ? scatter_words(B, C, h, w) : 0);
    WarpArgs a;
    memset(&a, 0, sizeof(a));
    a.img = x; a.flow = flow; a.grad_out = grad_out; a.d_flow = d_flow; a.d_img = d_x; a.d_img_fx = work;
    a.B = B; a.C = C; a.h = h; a.w = w; a.pad = CCB_PAD_BORDER; a.b2f_norm = 1;
    launch_flow_warp(a, true, (cudaStream_t)stream);
    return check_launch("featwarp_bwd");
}

static size_t ssim_smem_fwd() { return (size_t)(2 * Tile<6>::PLANE + 3 * Tile<6>::RH * HP) * sizeof(float); }
static size_t ssim_smem_bwd() { return (size_t)(3 * Tile<6>::PLANE + 3 * Tile<6>::RH * HP) * sizeof(float); }

extern "C" int ccb_ssim_fwd(const float* img1, const float* img2, int planes, int h, int w, const float* taps_host,
                            float* out, ccb_stream_t stream) {
    CCB_REQUIRE(img1 && img2 && out && taps_host, CCB_ERR_ARG, "ssim_fwd: null pointer");
    SsimArgs a;
    memset(&a, 0, sizeof(a));
    a.x = img1; a.y = img2; a.out = out; a.planes = planes; a.h = h; a.w = w;
    for (int k = 0; k < CCB_SSIM_TAPS; ++k) a.taps[k] = taps_host[k];
    auto kfn = ssim_map_kernel<0>;
    { static bool once = false; if (!once) { cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssim_smem_fwd()); once = true; } }
    CCB_LAUNCH(kfn, dim3(cdiv(w, TW), cdiv(h, TH), planes), dim3(NT), ssim_smem_fwd(), stream, a);
    return check_launch("ssim_fwd");
}

extern "C" long long ccb_ssim_bwd_workspace_floats(int planes, int h, int w) {
    if (planes < 1 || h < 1 || w < 1) return -1;
    return 5LL * planes * h * w;
}

extern "C" int ccb_ssim_bwd(const float* img1, const float* img2, int planes, int h, int w, const float* taps_host,
                            const float* grad_out, float* d_img1, float* d_img2, float* work, long long work_floats,
                            ccb_stream_t stream) {
    CCB_REQUIRE(img1 && img2 && grad_out && taps_host, CCB_ERR_ARG, "ssim_bwd: null pointer");
    CCB_REQUIRE(planes >= 1 && h >= 1 && w >= 1, CCB_ERR_ARG, "ssim_bwd: bad size");
    CCB_REQUIRE_WORK("ssim_bwd", "work", work, work_floats, ccb_ssim_bwd_workspace_floats(planes, h, w));
    SsimArgs a;
    memset(&a, 0, sizeof(a));
    a.x = img1; a.y = img2; a.gout = grad_out; a.dx = d_img1; a.dy = d_img2; a.work = work;
    a.planes = planes; a.h = h; a.w = w;
    for (int k = 0; k < CCB_SSIM_TAPS; ++k) a.taps[k] = taps_host[k];
    auto k1 = ssim_map_kernel<1>;
    { static bool once = false; if (!once) { cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssim_smem_fwd()); once = true; } }
    CCB_LAUNCH(k1, dim3(cdiv(w, TW), cdiv(h, TH), planes), dim3(NT), ssim_smem_fwd(), stream, a);
    int rc = check_launch("ssim_bwd_maps");
    if (rc) return rc;
    auto k2 = ssim_bwd_kernel;
    { static bool once = false; if (!once) { cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ssim_smem_bwd()); once = true; } }
    CCB_LAUNCH(k2, dim3(cdiv(w, TW), cdiv(h, TH), planes), dim3(NT), ssim_smem_bwd(), stream, a);
    return check_launch("ssim_bwd");
}
