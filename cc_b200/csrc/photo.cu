// photo.cu - fused multi-scale photometric loss (warp + valid/occlusion masks + 13x13 SSIM +
// robust L1 + reductions) forward and hand-derived backward, plus the consensus-target variant.
//
// One launch covers every pyramid level: block -> (level, batch, 64x20 tile) through a prefix table.
// Each CTA stages the target tile (+6 px halo) in shared memory once, then loops over the reference
// frames: warp the reference into a second shared tile (projection + bilinear gather, or flow
// coordinates), run the separable 13-tap Gaussian moments out of shared memory
// (rows -> smem, columns -> registers), and finish SSIM / robust-L1 / mask terms in registers.
//
// Roofline note: with the reference's real 13x13 window the kernel is FP32-FMA bound
// (~1.4 kFMA per level-pixel forward), not HBM bound; with wssim == 0 the SSIM stage is compiled
// out (template SSIM=false) and the kernel is a pure streaming pass.
//
// Reference: loss_functions.py:27-128,132-137,160-202,343-352; inverse_warp.py:164-283; ssim.py:9-36.
#include "ssim_tile.cuh"

namespace ccb {

struct PhotoArgs {
    ccb_photo_desc d;
    int blk_off[CCB_MAX_LEVELS + 1];
    float omw;               // (1 - wssim) evaluated in double on the host, like the reference
};

__device__ __forceinline__ void locate_block(const PhotoArgs& a, int& l, int& b, int& x0, int& y0, int& local) {
    int blk = blockIdx.x;
    l = 0;
    while (l + 1 < a.d.nlevels && blk >= a.blk_off[l + 1]) ++l;
    local = blk - a.blk_off[l];
    const int w = a.d.w[l], h = a.d.h[l];
    const int tx_n = cdiv(w, TW), ty_n = cdiv(h, TH);
    b = local / (tx_n * ty_n);
    int t = local - b * tx_n * ty_n;
    y0 = (t / tx_n) * TH;
    x0 = (t % tx_n) * TW;
}

// depth_occlusion_masks of one pixel (loss_functions.py:132-137): the four rigid flows with the UNSCALED cameras
// cams[0..3], pairs (0,3) and (1,2); returns (1 - occ) of the two pairs.  Not inlined: five call sites per thread
// share one copy of the four projections (instruction-cache footprint of the fused kernel).
__device__ __noinline__ float2 rigid_occ_pairs(const Cam* cams, float x, float y, float dep) {
    float u[CCB_MAX_REFS], v[CCB_MAX_REFS];
#pragma unroll
    for (int i = 0; i < CCB_MAX_REFS; ++i) {
        Proj pp = project(cams[i], x, y, dep, false);
        coords_to_flow(cams[i], pp.Xn, pp.Yn, x, y, u[i], v[i]);
    }
    return make_float2(1.f - occ_mask(u[0], v[0], u[3], v[3]), 1.f - occ_mask(u[1], v[1], u[2], v[2]));
}

// ================================================================================================
// Forward.  MODE: CCB_PHOTO_RIGID / FLOW / CONSENSUS.  SSIM=false compiles the 13x13 stage out.
template <int MODE, bool SSIM>
__global__ void __launch_bounds__(NT, 2) photo_fwd_kernel(const PhotoArgs a) {
    CCB_PDL_WAIT();
    constexpr int HALO = SSIM ? 6 : 0;
    using T = Tile<HALO>;
    CCB_DYN_SMEM(smem_raw);
    float* sx = reinterpret_cast<float*>(smem_raw);   // [3][PLANE] target
    float* sy = sx + 3 * T::PLANE;                    // [3][PLANE] warped reference
    float* sH = sy + 3 * T::PLANE;                    // [3][RH*HP]  (SSIM only)
    __shared__ Cam s_cam[2 * CCB_MAX_REFS];           // [i]: level-scaled cam of ref i; [R+i]: unscaled cam (occlusion)
    __shared__ float s_red[4 * 32];

    const ccb_photo_desc& d = a.d;
    const float* s_g = a.d.taps;                       // kernel-parameter (constant-bank) operands of the tap FMAs
    int l, b, x0, y0, local;
    locate_block(a, l, b, x0, y0, local);
    const int h = d.h[l], w = d.w[l], R = d.R;
    const int hw = h * w;                              // per-tensor offsets fit 32 bits (<= 2^31 elements)
    const int tid = threadIdx.x;
    const int col = tid & 63, rg = tid >> 6;
    const float w1 = (float)(w - 1), h1 = (float)(h - 1);
    // ---- all cameras of this (level, batch) at once: threads 64.. build one each
    if (MODE == CCB_PHOTO_RIGID && tid >= 64 && tid < 64 + 2 * R) {
        const int k = tid - 64, i = (k < R) ? k : k - R;
        make_cam(d.pose + (b * R + i) * 6, d.K + b * 9, d.Kinv + b * 9, (k < R) ? (float)d.H / (float)h : 1.f,
                 d.rotation_mode, w, h, s_cam[k]);
    }

    // ---- stage the target tile (+halo); zero outside the image == conv zero padding
    const float* tgt = d.tgt[l] + b * 3 * hw;
    for (int idx = tid; idx < T::RH * T::RW; idx += NT) {
        int ry = idx / T::RW, rx = idx - ry * T::RW;
        int gy = y0 - HALO + ry, gx = x0 - HALO + rx;
        bool in = (gy >= 0) && (gy < h) && (gx >= 0) && (gx < w);
        int off = gy * w + gx;
#pragma unroll
        for (int c = 0; c < 3; ++c) sx[c * T::PLANE + ry * T::PITCH + rx] = in ? __ldg(tgt + c * hw + off) : 0.f;
    }
    __syncthreads();

    // ---- target moments, shared by all reference frames.  The channel loops below stay LOOPS: fully unrolled the
    // kernel was 12.6 k SASS instructions (200 KB) and 22 % of its stall samples were instruction fetch (ncu r01)
    float mu1[3][PXT], exx[3][PXT];
    if (SSIM) {
#pragma unroll 1
        for (int c = 0; c < 3; ++c) {
            hpass<0>(sx + c * Tile<6>::PLANE, nullptr, nullptr, sH, s_g);
            __syncthreads();
            float o[2][PXT];
            vpass<2>(sH, s_g, o);
#pragma unroll
            for (int j = 0; j < PXT; ++j) { mu1[c][j] = o[0][j]; exx[c][j] = o[1][j]; }
            __syncthreads();
        }
    }

    // consensus accumulators: first rigid error / validity, then the combined rigid error
    float cons_e0[PXT], cons_v0[PXT], cons_cam[PXT];

    // ---- occlusion masks of the centre pixels, once per pair (refs i and R-1-i share one: SURVEY F5)
    bool inimg[PXT];
    float om_pair[2][PXT];     // (1 - occ) of pair (0,R-1) and pair (1,R-2)
#pragma unroll
    for (int j = 0; j < PXT; ++j) {
        const int py = y0 + rg * PXT + j, px = x0 + col;
        inimg[j] = (py < h) && (px < w);
        om_pair[0][j] = om_pair[1][j] = 1.f;
        if (inimg[j] && d.has_occ && MODE != CCB_PHOTO_CONSENSUS) {
            const int off = py * w + px;
            if (MODE == CCB_PHOTO_RIGID) {
                const float2 om = rigid_occ_pairs(s_cam + R, (float)px, (float)py, __ldg(d.depth[l] + b * hw + off));
                om_pair[0][j] = om.x;
                om_pair[1][j] = om.y;
            } else {
                const float* fb = d.flow[l][0] + b * 2 * hw + off;
                const float* ff = d.flow[l][1] + b * 2 * hw + off;
                om_pair[0][j] = om_pair[1][j] = 1.f - occ_mask(__ldg(fb), __ldg(fb + hw), __ldg(ff), __ldg(ff + hw));
            }
        }
    }

    for (int i = 0; i < R; ++i) {
        // ---- warp the reference into sy over the staged region
        const float* ref = d.ref[l][i] + b * 3 * hw;
        for (int idx = tid; idx < T::RH * T::RW; idx += NT) {
            int ry = idx / T::RW, rx = idx - ry * T::RW;
            int gy = y0 - HALO + ry, gx = x0 - HALO + rx;
            float v0 = 0.f, v1 = 0.f, v2 = 0.f;
            if ((gy >= 0) && (gy < h) && (gx >= 0) && (gx < w)) {
                float Xn, Yn;
                int pad = CCB_PAD_ZEROS;
                if (MODE == CCB_PHOTO_RIGID) {
                    float dep = __ldg(d.depth[l] + b * hw + gy * w + gx);
                    Proj p = project(s_cam[i], (float)gx, (float)gy, dep, d.padding_mode == CCB_PAD_ZEROS);
                    Xn = p.Xn; Yn = p.Yn;
                    pad = d.padding_mode;
                } else {
                    const float* fl = d.flow[l][i] + b * 2 * hw + gy * w + gx;
                    flow_coords((float)gx, (float)gy, __ldg(fl), __ldg(fl + hw), w1, h1, Xn, Yn);
                }
                Samp s = make_samp(Xn, Yn, w, h, pad);
                v0 = interp(fetch(ref, s, w), s);
                v1 = interp(fetch(ref + hw, s, w), s);
                v2 = interp(fetch(ref + 2 * hw, s, w), s);
            }
            int o = ry * T::PITCH + rx;
            sy[o] = v0; sy[T::PLANE + o] = v1; sy[2 * T::PLANE + o] = v2;
        }
        __syncthreads();

        // ---- centre-pixel scalars (valid, occlusion, mask)
        float valid[PXT], om[PXT], mk[PXT];   // om = (1-occ)
        const int pair = (i == 0 || i == R - 1) ? 0 : 1;
#pragma unroll
        for (int j = 0; j < PXT; ++j) {
            int py = y0 + rg * PXT + j, px = x0 + col;
            int o = (rg * PXT + j + HALO) * T::PITCH + col + HALO;
            float wv0 = sy[o], wv1 = sy[T::PLANE + o], wv2 = sy[2 * T::PLANE + o];
            valid[j] = ((wv0 != 0.f) || (wv1 != 0.f) || (wv2 != 0.f)) ? 1.f : 0.f;
            om[j] = pair ? om_pair[1][j] : om_pair[0][j];
            mk[j] = 1.f;
            if (inimg[j] && MODE != CCB_PHOTO_CONSENSUS && d.has_mask)
                mk[j] = __ldg(d.mask[l] + (b * R + i) * hw + py * w + px);
        }

        // ---- per-channel SSIM + loss terms
        float s_l1 = 0.f, s_ss = 0.f, s_va = 0.f, s_ob = 0.f;
        float gm[PXT], e_l1[PXT], e_ss[PXT];
#pragma unroll
        for (int j = 0; j < PXT; ++j) { gm[j] = 0.f; e_l1[j] = 0.f; e_ss[j] = 0.f; }
#pragma unroll 1
        for (int c = 0; c < 3; ++c) {
            float o3[3][PXT];
            if (SSIM) {
                hpass<1>(sx + c * Tile<6>::PLANE, sy + c * Tile<6>::PLANE, nullptr, sH, s_g);
                __syncthreads();
                vpass<3>(sH, s_g, o3);
            }
#pragma unroll
            for (int j = 0; j < PXT; ++j) {
                int o = c * T::PLANE + (rg * PXT + j + HALO) * T::PITCH + col + HALO;
                float tv = sx[o], wv = sy[o];
                float S = 0.f, dmu2 = 0.f, deyy = 0.f, dexy = 0.f;
                if (SSIM) S = ssim_point(mu1[c][j], exx[c][j], o3[0][j], o3[1][j], o3[2][j], dmu2, deyy, dexy);
                if (MODE == CCB_PHOTO_CONSENSUS) {
                    e_l1[j] += rl1(tv - wv, 0.5f);
                    e_ss[j] += (1.f - S);
                } else if (inimg[j]) {
                    float e = (tv - wv) * valid[j] * om[j];      // (1-occ) in {0,1}: order-free
                    float df = e * mk[j];
                    s_l1 += rl1(df, d.qch);
                    float sl = (1.f - S * valid[j]) * om[j];
                    s_ss += sl * mk[j];
                    if (d.has_mask) gm[j] += rl1_d(df, d.qch) * e + d.wssim * sl;
                    if (SSIM) {
                        float gam = -valid[j] * om[j] * mk[j];
                        int off = (y0 + rg * PXT + j) * w + (x0 + col);
                        float* dm = d.dmaps[l] + ((b * R + i) * 9 + c * 3) * hw + off;
                        dm[0] = gam * dmu2;
                        dm[hw] = gam * deyy;
                        dm[2 * hw] = gam * dexy;
                    }
                }
            }
            if (SSIM) __syncthreads();   // sH is rewritten by the next channel / ref
        }

        if (MODE == CCB_PHOTO_CONSENSUS) {
#pragma unroll
            for (int j = 0; j < PXT; ++j) {
                // loss_functions.py:184-198: min over (fwd,bwd) rigid errors vs the flow error
                float e = a.omw * (e_l1[j] / 3.f) + d.wssim * (e_ss[j] / 3.f);
                if (i == 0) { cons_e0[j] = e; cons_v0[j] = valid[j]; }
                else if (i == 1) {
                    float vcam = 1.f - (1.f - cons_v0[j]) * (1.f - valid[j]);
                    cons_cam[j] = fminf(cons_e0[j], e) * vcam;
                } else {
                    int py = y0 + rg * PXT + j, px = x0 + col;
                    if ((py < h) && (px < w))
                        d.target[l][b * hw + py * w + px] =
                            (d.wrig * cons_cam[j] <= (e + 1e-8f)) ? 1.f : 0.f;
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < PXT; ++j) {
                if (!inimg[j]) continue;
                int off = (b * R + i) * hw + (y0 + rg * PXT + j) * w + (x0 + col);
                s_va += valid[j];
                s_ob += rl1(1.f - valid[j], d.qch);
                d.vo[l][off] = valid[j] * om[j];
                if (d.has_mask) d.gmask[l][off] = gm[j];
            }
            float red[4] = {s_l1, s_ss, s_va, s_ob};
            block_sum<4>(red, s_red);
            if (tid == 0) {
                float* po = d.partials + ((long long)blockIdx.x * R + i) * 4;
                po[0] = red[0]; po[1] = red[1]; po[2] = red[2]; po[3] = red[3];
            }
        }
        __syncthreads();   // sy reuse
    }

}

// ------------------------------------------------------------------------------------------------
// Forward finalize: per (level, ref) sums -> oob normalisation, loss terms, total loss.
// loss_functions.py:48,58-59 / 103,114
__global__ void __launch_bounds__(1024) photo_fwd_finalize(const PhotoArgs a) {
    CCB_PDL_WAIT();
    __shared__ float s_L[CCB_MAX_LEVELS * CCB_MAX_REFS];
    const ccb_photo_desc& d = a.d;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    const int ncombo = d.nlevels * d.R;
    for (int cb = warp; cb < ncombo; cb += nwarps) {       // one warp per (level, ref): fixed summation order
        const int l = cb / d.R, i = cb - l * d.R;
        const int nblk = a.blk_off[l + 1] - a.blk_off[l];
        float v0 = 0.f, v1 = 0.f, v2 = 0.f, v3 = 0.f;
        for (int k = lane; k < nblk; k += 32) {
            const float* p = d.partials + ((long long)(a.blk_off[l] + k) * d.R + i) * 4;
            v0 += p[0]; v1 += p[1]; v2 += p[2]; v3 += p[3];
        }
        v0 = warp_sum(v0); v1 = warp_sum(v1); v2 = warp_sum(v2); v3 = warp_sum(v3);
        if (lane == 0) {
            float npx = (float)((long long)d.B * d.h[l] * d.w[l]);
            float n = 3.f * npx;
            float oob = npx / v2;
            float L = a.omw * oob * (v0 / n + d.wssim * (v1 / n)) + d.lambda_oob * (v3 / npx);
            float* sc = d.scal + (l * d.R + i) * 4;
            sc[0] = a.omw * oob / n;
            sc[1] = oob;
            sc[2] = v2;
            sc[3] = L;
            s_L[cb] = L;
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int cb = 0; cb < ncombo; ++cb) t += s_L[cb];
        d.loss[0] = t;
    }
}

// ================================================================================================
// Backward.  Blurs the saved gamma*dS maps (halo 6), recomputes the centre-pixel warp, and chains to
// depth / pose (rigid) or flow; mask gradient is a scale of the saved unscaled term.
template <int MODE, bool SSIM>
__global__ void __launch_bounds__(NT, 2) photo_bwd_kernel(const PhotoArgs a) {
    CCB_PDL_WAIT();
    using T = Tile<6>;
    CCB_DYN_SMEM(smem_raw);
    float* sD = reinterpret_cast<float*>(smem_raw);   // [3][PLANE] dS maps of one channel
    float* sH = sD + 3 * T::PLANE;                    // [3][RH*HP]
    __shared__ Cam s_cam[CCB_MAX_REFS];
    __shared__ float s_red[12 * 32];

    const ccb_photo_desc& d = a.d;
    const float* s_g = a.d.taps;                       // constant-bank operands of the tap FMAs
    int l, b, x0, y0, local;
    locate_block(a, l, b, x0, y0, local);
    const int h = d.h[l], w = d.w[l], R = d.R;
    const int hw = h * w;
    const int tid = threadIdx.x;
    const int col = tid & 63, rg = tid >> 6;
    const float w1 = (float)(w - 1), h1 = (float)(h - 1);
    const float go = __ldg(d.grad_out);
    const float* tgt = d.tgt[l] + b * 3 * hw;
    if (MODE == CCB_PHOTO_RIGID && tid >= 64 && tid < 64 + R)
        make_cam(d.pose + (b * R + (tid - 64)) * 6, d.K + b * 9, d.Kinv + b * 9, (float)d.H / (float)h, d.rotation_mode, w, h,
                 s_cam[tid - 64]);

    float gd[PXT];
#pragma unroll
    for (int j = 0; j < PXT; ++j) gd[j] = 0.f;
    __syncthreads();

    for (int i = 0; i < R; ++i) {
        const float c_l = go * __ldg(d.scal + (l * R + i) * 4);
        const float c_s = c_l * d.wssim;
        // ---- blur the three dS maps of every channel
        // channel and pixel loops are kept as loops (bl / gd live in local memory, L1-resident): unrolled, the kernel
        // was 9.2 k SASS instructions and instruction fetch showed up as its top stall reason
        float bl[3][3][PXT];
        if (SSIM) {
#pragma unroll 1
            for (int c = 0; c < 3; ++c) {
                const float* dm = d.dmaps[l] + ((b * R + i) * 9 + c * 3) * hw;
                for (int idx = tid; idx < T::RH * T::RW; idx += NT) {
                    int ry = idx / T::RW, rx = idx - ry * T::RW;
                    int gy = y0 - 6 + ry, gx = x0 - 6 + rx;
                    bool in = (gy >= 0) && (gy < h) && (gx >= 0) && (gx < w);
                    int off = gy * w + gx;
                    int o = ry * T::PITCH + rx;
                    sD[o] = in ? __ldg(dm + off) : 0.f;
                    sD[T::PLANE + o] = in ? __ldg(dm + hw + off) : 0.f;
                    sD[2 * T::PLANE + o] = in ? __ldg(dm + 2 * hw + off) : 0.f;
                }
                __syncthreads();
                hpass<2>(sD, sD + T::PLANE, sD + 2 * T::PLANE, sH, s_g);
                __syncthreads();
                vpass<3>(sH, s_g, bl[c]);
            }
        }
        __syncthreads();   // sD/sH free

        const float* ref = d.ref[l][i] + b * 3 * hw;
        float acc[12];
#pragma unroll
        for (int k = 0; k < 12; ++k) acc[k] = 0.f;
#pragma unroll 1
        for (int j = 0; j < PXT; ++j) {
            int py = y0 + rg * PXT + j, px = x0 + col;
            if ((py < h) && (px < w)) {
                int off = py * w + px;
                int moff = (b * R + i) * hw + off;
                float Xn, Yn;
                Proj p;
                int pad = CCB_PAD_ZEROS;
                if (MODE == CCB_PHOTO_RIGID) {
                    float dep = __ldg(d.depth[l] + b * hw + off);
                    p = project(s_cam[i], (float)px, (float)py, dep, d.padding_mode == CCB_PAD_ZEROS);
                    Xn = p.Xn; Yn = p.Yn;
                    pad = d.padding_mode;
                } else {
                    const float* fl = d.flow[l][i] + b * 2 * hw + off;
                    flow_coords((float)px, (float)py, __ldg(fl), __ldg(fl + hw), w1, h1, Xn, Yn);
                }
                Samp s = make_samp(Xn, Yn, w, h, pad);
                float vo = __ldg(d.vo[l] + moff);
                float mk = d.has_mask ? __ldg(d.mask[l] + moff) : 1.f;
                float M = vo * mk;
                float gix = 0.f, giy = 0.f;
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    Corners cr = fetch(ref + c * hw, s, w);
                    float wv = interp(cr, s);
                    float tv = __ldg(tgt + c * hw + off);
                    float df = (tv - wv) * M;
                    float gw = -c_l * rl1_d(df, d.qch) * M;
                    if (SSIM) gw += c_s * (bl[c][0][j] + 2.f * wv * bl[c][1][j] + tv * bl[c][2][j]);
                    gix += gw * interp_dx(cr, s);
                    giy += gw * interp_dy(cr, s);
                }
                float gXn = gix * s.gmx, gYn = giy * s.gmy;
                if (MODE == CCB_PHOTO_RIGID) {
                    gd[j] += project_bwd(s_cam[i], p, gXn, gYn, acc);
                } else {
                    float* df = d.d_flow[l][i] + b * 2 * hw + off;
                    df[0] = gXn * (2.f / w1);
                    df[hw] = gYn * (2.f / h1);
                }
                if (d.has_mask) d.d_mask[l][moff] = c_l * __ldg(d.gmask[l] + moff);
            }
        }
        if (MODE == CCB_PHOTO_RIGID) {
            block_sum<12>(acc, s_red);
            if (tid == 0) {
                float* po = d.pose_partials + ((long long)blockIdx.x * R + i) * 12;
#pragma unroll
                for (int k = 0; k < 12; ++k) po[k] = acc[k];
            }
        }
        __syncthreads();
    }
    if (MODE == CCB_PHOTO_RIGID) {
#pragma unroll
        for (int j = 0; j < PXT; ++j) {
            int py = y0 + rg * PXT + j, px = x0 + col;
            if ((py < h) && (px < w)) d.d_depth[l][b * hw + py * w + px] = gd[j];
        }
    }
}

// One warp per (b, ref): sum the per-tile dP partials of every level, chain to the 6-DoF pose.
__global__ void photo_pose_finalize(const PhotoArgs a) {
    CCB_PDL_WAIT();
    const ccb_photo_desc& d = a.d;
    const int wid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (wid >= d.B * d.R) return;
    const int b = wid / d.R, i = wid - b * d.R;
    float dpose[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int l = 0; l < d.nlevels; ++l) {
        const int per_b = (a.blk_off[l + 1] - a.blk_off[l]) / d.B;
        float dP[12];
#pragma unroll
        for (int k = 0; k < 12; ++k) dP[k] = 0.f;
        for (int t = lane; t < per_b; t += 32) {
            const float* p = d.pose_partials + ((long long)(a.blk_off[l] + b * per_b + t) * d.R + i) * 12;
#pragma unroll
            for (int k = 0; k < 12; ++k) dP[k] += p[k];
        }
#pragma unroll
        for (int k = 0; k < 12; ++k) dP[k] = warp_sum(dP[k]);
        if (lane == 0) {
            Cam cm;
            make_cam(d.pose + ((long long)b * d.R + i) * 6, d.K + b * 9, d.Kinv + b * 9,
                     (float)d.H / (float)d.h[l], d.rotation_mode, d.w[l], d.h[l], cm);
            pose_grad_from_dP(cm, dP, d.rotation_mode, dpose);
        }
    }
    if (lane == 0) {
        float* o = d.d_pose + ((long long)b * d.R + i) * 6;
#pragma unroll
        for (int k = 0; k < 6; ++k) o[k] = dpose[k];
    }
}

// ------------------------------------------------------------------------------------------------
static int fill_args(const ccb_photo_desc* d, PhotoArgs& a) {
    CCB_REQUIRE(d != nullptr, CCB_ERR_ARG, "photo: null descriptor");
    CCB_REQUIRE(d->nlevels >= 1 && d->nlevels <= CCB_MAX_LEVELS, CCB_ERR_ARG, "photo: nlevels %d out of range", d->nlevels);
    CCB_REQUIRE(d->B >= 1 && d->R >= 1 && d->R <= CCB_MAX_REFS, CCB_ERR_ARG, "photo: bad B=%d R=%d", d->B, d->R);
    a.d = *d;
    a.omw = d->one_minus_wssim;
    a.blk_off[0] = 0;
    for (int l = 0; l < d->nlevels; ++l) {
        CCB_REQUIRE(d->h[l] >= 2 && d->w[l] >= 2, CCB_ERR_ARG, "photo: level %d size %dx%d too small", l, d->h[l], d->w[l]);
        a.blk_off[l + 1] = a.blk_off[l] + d->B * cdiv(d->w[l], TW) * cdiv(d->h[l], TH);
    }
    for (int l = d->nlevels + 1; l <= CCB_MAX_LEVELS; ++l) a.blk_off[l] = a.blk_off[d->nlevels];
    return CCB_OK;
}

template <int HALO>
static size_t fwd_smem() { return (size_t)(6 * Tile<HALO>::PLANE + (HALO ? 3 * Tile<HALO>::RH * HP : 0)) * sizeof(float); }
static size_t bwd_smem() { return (size_t)(3 * Tile<6>::PLANE + 3 * Tile<6>::RH * HP) * sizeof(float); }

template <int MODE, bool SSIM>
static int launch_fwd(const PhotoArgs& a, cudaStream_t st) {
    auto k = photo_fwd_kernel<MODE, SSIM>;
    size_t sm = SSIM ? fwd_smem<6>() : fwd_smem<0>();
    { static bool once = false; if (!once) { cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm); once = true; } }
    CCB_LAUNCH(k, dim3(a.blk_off[a.d.nlevels]), dim3(NT), sm, st, a);
    return check_launch("photo_fwd");
}
template <int MODE, bool SSIM>
static int launch_bwd(const PhotoArgs& a, cudaStream_t st) {
    auto k = photo_bwd_kernel<MODE, SSIM>;
    size_t sm = bwd_smem();
    { static bool once = false; if (!once) { cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm); once = true; } }
    CCB_LAUNCH(k, dim3(a.blk_off[a.d.nlevels]), dim3(NT), sm, st, a);
    return check_launch("photo_bwd");
}

}  // namespace ccb

using namespace ccb;

extern "C" long long ccb_photo_partials_floats(const ccb_photo_desc* d) {
    PhotoArgs a;
    if (fill_args(d, a) != CCB_OK) return -1;
    return (long long)a.blk_off[d->nlevels] * d->R * 4;
}
extern "C" long long ccb_photo_pose_partials_floats(const ccb_photo_desc* d) {
    PhotoArgs a;
    if (fill_args(d, a) != CCB_OK) return -1;
    return (long long)a.blk_off[d->nlevels] * d->R * 12;
}

static int check_common(const ccb_photo_desc* d, bool bwd) {
    for (int l = 0; l < d->nlevels; ++l) {
        CCB_REQUIRE(d->tgt[l] != nullptr, CCB_ERR_ARG, "photo: tgt[%d] is null", l);
        for (int i = 0; i < d->R; ++i) {
            CCB_REQUIRE(d->ref[l][i] != nullptr, CCB_ERR_ARG, "photo: ref[%d][%d] is null", l, i);
            if (d->mode != CCB_PHOTO_RIGID) CCB_REQUIRE(d->flow[l][i] != nullptr, CCB_ERR_ARG, "photo: flow[%d][%d] is null", l, i);
        }
        if (d->mode == CCB_PHOTO_RIGID) CCB_REQUIRE(d->depth[l] != nullptr, CCB_ERR_ARG, "photo: depth[%d] is null", l);
        if (d->has_mask) CCB_REQUIRE(d->mask[l] != nullptr, CCB_ERR_ARG, "photo: mask[%d] is null", l);
        if (d->mode != CCB_PHOTO_CONSENSUS) {
            CCB_REQUIRE(d->vo[l] != nullptr, CCB_ERR_ARG, "photo: vo[%d] is null", l);
            if (d->wssim != 0.f) CCB_REQUIRE(d->dmaps[l] != nullptr, CCB_ERR_ARG, "photo: dmaps[%d] is null", l);
            if (d->has_mask) CCB_REQUIRE(d->gmask[l] != nullptr, CCB_ERR_ARG, "photo: gmask[%d] is null", l);
        }
    }
    if (d->mode == CCB_PHOTO_RIGID) {
        CCB_REQUIRE(d->pose && d->K && d->Kinv, CCB_ERR_ARG, "photo: pose/K/Kinv null");
        CCB_REQUIRE(!d->has_occ || d->R == 4, CCB_ERR_ARG,
                    "photo: rigid occlusion masks need 4 reference frames (loss_functions.py:133-135), got %d", d->R);
        CCB_REQUIRE(d->padding_mode == CCB_PAD_ZEROS || d->padding_mode == CCB_PAD_BORDER, CCB_ERR_ARG, "photo: bad padding_mode");
    }
    if (d->mode == CCB_PHOTO_FLOW) CCB_REQUIRE(!d->has_occ || d->R == 2, CCB_ERR_ARG, "photo: flow occlusion needs R == 2");
    (void)bwd;
    return CCB_OK;
}

extern "C" int ccb_photo_loss_fwd(const ccb_photo_desc* d, ccb_stream_t stream) {
    PhotoArgs a;
    int rc = fill_args(d, a);
    if (rc) return rc;
    CCB_REQUIRE(d->mode == CCB_PHOTO_RIGID || d->mode == CCB_PHOTO_FLOW, CCB_ERR_ARG, "photo_loss_fwd: bad mode %d", d->mode);
    rc = check_common(d, false);
    if (rc) return rc;
    CCB_REQUIRE(d->partials && d->scal && d->loss, CCB_ERR_ARG, "photo_loss_fwd: partials/scal/loss null");
    cudaStream_t st = (cudaStream_t)stream;
    const bool ss = d->wssim != 0.f;
    if (d->mode == CCB_PHOTO_RIGID) rc = ss ? launch_fwd<CCB_PHOTO_RIGID, true>(a, st) : launch_fwd<CCB_PHOTO_RIGID, false>(a, st);
    else rc = ss ? launch_fwd<CCB_PHOTO_FLOW, true>(a, st) : launch_fwd<CCB_PHOTO_FLOW, false>(a, st);
    if (rc) return rc;
    CCB_LAUNCH(photo_fwd_finalize, dim3(1), dim3(1024), 0, st, a);
    return check_launch("photo_fwd_finalize");
}

extern "C" int ccb_photo_loss_bwd(const ccb_photo_desc* d, ccb_stream_t stream) {
    PhotoArgs a;
    int rc = fill_args(d, a);
    if (rc) return rc;
    CCB_REQUIRE(d->mode == CCB_PHOTO_RIGID || d->mode == CCB_PHOTO_FLOW, CCB_ERR_ARG, "photo_loss_bwd: bad mode %d", d->mode);
    rc = check_common(d, true);
    if (rc) return rc;
    CCB_REQUIRE(d->grad_out && d->scal, CCB_ERR_ARG, "photo_loss_bwd: grad_out/scal null");
    for (int l = 0; l < d->nlevels; ++l) {
        if (d->mode == CCB_PHOTO_RIGID) CCB_REQUIRE(d->d_depth[l] != nullptr, CCB_ERR_ARG, "photo_loss_bwd: d_depth[%d] null", l);
        else for (int i = 0; i < d->R; ++i) CCB_REQUIRE(d->d_flow[l][i] != nullptr, CCB_ERR_ARG, "photo_loss_bwd: d_flow[%d][%d] null", l, i);
        if (d->has_mask) CCB_REQUIRE(d->d_mask[l] != nullptr, CCB_ERR_ARG, "photo_loss_bwd: d_mask[%d] null", l);
    }
    cudaStream_t st = (cudaStream_t)stream;
    const bool ss = d->wssim != 0.f;
    if (d->mode == CCB_PHOTO_RIGID) {
        CCB_REQUIRE(d->d_pose && d->pose_partials, CCB_ERR_ARG, "photo_loss_bwd: d_pose/pose_partials null");
        rc = ss ? launch_bwd<CCB_PHOTO_RIGID, true>(a, st) : launch_bwd<CCB_PHOTO_RIGID, false>(a, st);
        if (rc) return rc;
        int nw = d->B * d->R;
        CCB_LAUNCH(photo_pose_finalize, dim3(cdiv(nw * 32, 128)), dim3(128), 0, st, a);
        return check_launch("photo_pose_finalize");
    }
    return ss ? launch_bwd<CCB_PHOTO_FLOW, true>(a, st) : launch_bwd<CCB_PHOTO_FLOW, false>(a, st);
}

extern "C" int ccb_consensus_targets(const ccb_photo_desc* d, ccb_stream_t stream) {
    PhotoArgs a;
    int rc = fill_args(d, a);
    if (rc) return rc;
    CCB_REQUIRE(d->mode == CCB_PHOTO_CONSENSUS && d->R == 3, CCB_ERR_ARG, "consensus_targets: mode must be CONSENSUS with R == 3");
    rc = check_common(d, false);
    if (rc) return rc;
    for (int l = 0; l < d->nlevels; ++l) CCB_REQUIRE(d->target[l] != nullptr, CCB_ERR_ARG, "consensus_targets: target[%d] null", l);
    cudaStream_t st = (cudaStream_t)stream;
    return (d->wssim != 0.f) ? launch_fwd<CCB_PHOTO_CONSENSUS, true>(a, st) : launch_fwd<CCB_PHOTO_CONSENSUS, false>(a, st);
}
