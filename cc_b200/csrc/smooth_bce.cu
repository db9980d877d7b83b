// smooth_bce.cu - smoothness terms and mask cross-entropies of the CC loss, every pyramid level in
// one launch, two-stage deterministic reductions (no atomics).
//   edge_aware_smoothness_loss  loss_functions.py:287-319
//   smooth_loss                 loss_functions.py:323-341
//   explainability_loss         loss_functions.py:148-155
//   consensus_depth_flow_mask + weighted_binary_cross_entropy   loss_functions.py:221-261
#include "ccb_common.cuh"

namespace ccb {

constexpr int PNT = 256;

struct LevelTab {
    int nlevels, B;
    int h[CCB_MAX_LEVELS], w[CCB_MAX_LEVELS];
    int blk_off[CCB_MAX_LEVELS + 1];
};

static void make_tab(LevelTab& t, int nlevels, int B, const int* h, const int* w) {
    t.nlevels = nlevels;
    t.B = B;
    t.blk_off[0] = 0;
    for (int l = 0; l < CCB_MAX_LEVELS; ++l) {
        if (l < nlevels) {
            t.h[l] = h[l]; t.w[l] = w[l];
            t.blk_off[l + 1] = t.blk_off[l] + B * cdiv(h[l] * w[l], PNT);
        } else {
            t.h[l] = t.w[l] = 0;
            t.blk_off[l + 1] = t.blk_off[l];
        }
    }
}

// block -> (level, batch, first pixel)
__device__ __forceinline__ bool locate(const LevelTab& t, int& l, int& b, int& y, int& x) {
    int blk = blockIdx.x;
    l = 0;
    while (l + 1 < t.nlevels && blk >= t.blk_off[l + 1]) ++l;
    int local = blk - t.blk_off[l];
    int per_b = cdiv(t.h[l] * t.w[l], PNT);
    b = local / per_b;
    int idx = (local - b * per_b) * PNT + threadIdx.x;
    y = idx / t.w[l];
    x = idx - y * t.w[l];
    return idx < t.h[l] * t.w[l];
}

__device__ __forceinline__ float sgn(float v) { return (v > 0.f) ? 1.f : ((v < 0.f) ? -1.f : 0.f); }

// ------------------------------------------------------------------------------------------------
struct SmoothArgs {
    ccb_smooth_desc d;
    LevelTab t;
    float lw[CCB_MAX_LEVELS];   // per-level weight (1 for edge-aware; 1/2.3^l for second order)
};

// exp(-mean_c |I(y,x) - I(y+dy,x+dx)|)
__device__ __forceinline__ float edge_w(const float* __restrict__ im, long long hw, int w, int y, int x, int dy, int dx) {
    long long o = (long long)y * w + x, o2 = (long long)(y + dy) * w + (x + dx);
    float s = fabsf(__ldg(im + o) - __ldg(im + o2));
    s += fabsf(__ldg(im + hw + o) - __ldg(im + hw + o2));
    s += fabsf(__ldg(im + 2 * hw + o) - __ldg(im + 2 * hw + o2));
    return expf(-(s / 3.f));
}

template <int KIND>
__global__ void __launch_bounds__(PNT) smooth_fwd_kernel(const SmoothArgs a) {
    CCB_PDL_WAIT();
    __shared__ float s_red[4 * 32];
    int l, b, y, x;
    bool in = locate(a.t, l, b, y, x);
    const int h = a.t.h[l], w = a.t.w[l], C = a.d.C;
    const long long hw = (long long)h * w;
    float v[4] = {0.f, 0.f, 0.f, 0.f};
    if (in) {
        const float* p = a.d.pred[l] + (long long)b * C * hw + (long long)y * w + x;
        if (KIND == CCB_SMOOTH_EDGE) {
            const float* im = a.d.img[l] + (long long)b * 3 * hw;
            float wx = (y < h - 1) ? edge_w(im, hw, w, y, x, 1, 0) : 0.f;
            float wy = (x < w - 1) ? edge_w(im, hw, w, y, x, 0, 1) : 0.f;
            for (int c = 0; c < C; ++c) {
                const float* q = p + c * hw;
                float p0 = __ldg(q);
                if (y < h - 1) v[0] += fabsf(p0 - __ldg(q + w)) * wx;
                if (x < w - 1) v[1] += fabsf(p0 - __ldg(q + 1)) * wy;
            }
        } else {
            for (int c = 0; c < C; ++c) {
                const float* q = p + c * hw;
                float p00 = __ldg(q);
                if (x < w - 2) v[0] += fabsf((__ldg(q + 2) - __ldg(q + 1)) - (__ldg(q + 1) - p00));
                if (y < h - 2) v[3] += fabsf((__ldg(q + 2 * w) - __ldg(q + w)) - (__ldg(q + w) - p00));
                if (x < w - 1 && y < h - 1) {
                    float p01 = __ldg(q + 1), p10 = __ldg(q + w), p11 = __ldg(q + w + 1);
                    v[1] += fabsf((p11 - p10) - (p01 - p00));   // dxdy
                    v[2] += fabsf((p11 - p01) - (p10 - p00));   // dydx
                }
            }
        }
    }
    block_sum<4>(v, s_red);
    if (threadIdx.x == 0) {
        float* po = a.d.partials + (long long)blockIdx.x * 4;
        po[0] = v[0]; po[1] = v[1]; po[2] = v[2]; po[3] = v[3];
    }
}

template <int KIND>
__device__ __forceinline__ void smooth_counts(const SmoothArgs& a, int l, float* n) {
    float B = (float)a.t.B, C = (float)a.d.C, h = (float)a.t.h[l], w = (float)a.t.w[l];
    if (KIND == CCB_SMOOTH_EDGE) {
        n[0] = B * C * (h - 1.f) * w; n[1] = B * C * h * (w - 1.f); n[2] = 1.f; n[3] = 1.f;
    } else {
        n[0] = B * C * h * (w - 2.f); n[1] = B * C * (h - 1.f) * (w - 1.f); n[2] = n[1]; n[3] = B * C * (h - 2.f) * w;
    }
}

template <int KIND>
__global__ void smooth_finalize(const SmoothArgs a) {
    CCB_PDL_WAIT();
    __shared__ float s_red[4 * 32];
    __shared__ float s_total;
    if (threadIdx.x == 0) s_total = 0.f;
    __syncthreads();
    for (int l = 0; l < a.t.nlevels; ++l) {
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        for (int k = a.t.blk_off[l] + threadIdx.x; k < a.t.blk_off[l + 1]; k += blockDim.x) {
            const float* p = a.d.partials + (long long)k * 4;
            v[0] += p[0]; v[1] += p[1]; v[2] += p[2]; v[3] += p[3];
        }
        block_sum<4>(v, s_red);
        if (threadIdx.x == 0) {
            float n[4];
            smooth_counts<KIND>(a, l, n);
            float L = (KIND == CCB_SMOOTH_EDGE) ? (v[0] / n[0] + v[1] / n[1])
                                                : (v[0] / n[0] + v[1] / n[1] + v[2] / n[2] + v[3] / n[3]) * a.lw[l];
            s_total += L;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) a.d.loss[0] = s_total;
}

template <int KIND>
__global__ void __launch_bounds__(PNT) smooth_bwd_kernel(const SmoothArgs a) {
    CCB_PDL_WAIT();
    int l, b, y, x;
    if (!locate(a.t, l, b, y, x)) return;
    const int h = a.t.h[l], w = a.t.w[l], C = a.d.C;
    const long long hw = (long long)h * w;
    const float go = __ldg(a.d.grad_out) * a.lw[l];
    float n[4];
    smooth_counts<KIND>(a, l, n);
    const float* p = a.d.pred[l] + (long long)b * C * hw + (long long)y * w + x;
    float* dp = a.d.d_pred[l] + (long long)b * C * hw + (long long)y * w + x;
    if (KIND == CCB_SMOOTH_EDGE) {
        const float* im = a.d.img[l] + (long long)b * 3 * hw;
        float wx0 = (y < h - 1) ? edge_w(im, hw, w, y, x, 1, 0) / n[0] : 0.f;
        float wx1 = (y > 0) ? edge_w(im, hw, w, y - 1, x, 1, 0) / n[0] : 0.f;
        float wy0 = (x < w - 1) ? edge_w(im, hw, w, y, x, 0, 1) / n[1] : 0.f;
        float wy1 = (x > 0) ? edge_w(im, hw, w, y, x - 1, 0, 1) / n[1] : 0.f;
        for (int c = 0; c < C; ++c) {
            const float* q = p + c * hw;
            float p0 = __ldg(q), g = 0.f;
            if (y < h - 1) g += sgn(p0 - __ldg(q + w)) * wx0;
            if (y > 0) g -= sgn(__ldg(q - w) - p0) * wx1;
            if (x < w - 1) g += sgn(p0 - __ldg(q + 1)) * wy0;
            if (x > 0) g -= sgn(__ldg(q - 1) - p0) * wy1;
            dp[c * hw] = go * g;
        }
    } else {
        for (int c = 0; c < C; ++c) {
            const float* q = p + c * hw;
            auto P = [&](int dy, int dx) { return __ldg(q + dy * w + dx); };
            float g = 0.f;
            // dx2 at x' = x, x-1, x-2 with coefficients +1, -2, +1
            if (x <= w - 3) g += sgn((P(0, 2) - P(0, 1)) - (P(0, 1) - P(0, 0))) / n[0];
            if (x >= 1 && x <= w - 2) g -= 2.f * sgn((P(0, 1) - P(0, 0)) - (P(0, 0) - P(0, -1))) / n[0];
            if (x >= 2) g += sgn((P(0, 0) - P(0, -1)) - (P(0, -1) - P(0, -2))) / n[0];
            if (y <= h - 3) g += sgn((P(2, 0) - P(1, 0)) - (P(1, 0) - P(0, 0))) / n[3];
            if (y >= 1 && y <= h - 2) g -= 2.f * sgn((P(1, 0) - P(0, 0)) - (P(0, 0) - P(-1, 0))) / n[3];
            if (y >= 2) g += sgn((P(0, 0) - P(-1, 0)) - (P(-1, 0) - P(-2, 0))) / n[3];
            // mixed terms at (y',x') in {(y,x):+1, (y,x-1):-1, (y-1,x):-1, (y-1,x-1):+1}
            auto mixed = [&](int oy, int ox) {
                float p00 = P(oy, ox), p01 = P(oy, ox + 1), p10 = P(oy + 1, ox), p11 = P(oy + 1, ox + 1);
                return sgn((p11 - p10) - (p01 - p00)) / n[1] + sgn((p11 - p01) - (p10 - p00)) / n[2];
            };
            if (y <= h - 2 && x <= w - 2) g += mixed(0, 0);
            if (y <= h - 2 && x >= 1) g -= mixed(0, -1);
            if (y >= 1 && x <= w - 2) g -= mixed(-1, 0);
            if (y >= 1 && x >= 1) g += mixed(-1, -1);
            dp[c * hw] = go * g;
        }
    }
}

// ------------------------------------------------------------------------------------------------
struct BceArgs {
    ccb_bce_desc d;
    LevelTab t;
};

__device__ __forceinline__ void consensus_target(const BceArgs& a, int l, int b, long long hw, long long o, float* t4) {
    const float th = a.d.thresh;
    const float* cf = a.d.census_fwd[l] + (long long)b * 2 * hw + o;
    const float* cb = a.d.census_bwd[l] + (long long)b * 2 * hw + o;
    float f = ((__ldg(cf) < th) ? 1.f : 0.f) * ((__ldg(cf + hw) < th) ? 1.f : 0.f);
    float bw = ((__ldg(cb) < th) ? 1.f : 0.f) * ((__ldg(cb + hw) < th) ? 1.f : 0.f);
    f = 1.f - (1.f - f) * (1.f - __ldg(a.d.target_fwd[l] + (long long)b * hw + o));
    bw = 1.f - (1.f - bw) * (1.f - __ldg(a.d.target_bwd[l] + (long long)b * hw + o));
    t4[0] = bw; t4[1] = bw; t4[2] = f; t4[3] = f;
}

template <int KIND>
__global__ void __launch_bounds__(PNT) bce_fwd_kernel(const BceArgs a) {
    CCB_PDL_WAIT();
    __shared__ float s_red[32];
    int l, b, y, x;
    bool in = locate(a.t, l, b, y, x);
    const int h = a.t.h[l], w = a.t.w[l], C = a.d.C;
    const long long hw = (long long)h * w;
    float v[1] = {0.f};
    if (in) {
        long long o = (long long)y * w + x;
        const float* m = a.d.mask[l] + (long long)b * C * hw + o;
        if (KIND == CCB_BCE_ONES) {
            for (int c = 0; c < C; ++c) v[0] += -fmaxf(logf(__ldg(m + c * hw)), -100.f);
        } else {
            float t4[4];
            consensus_target(a, l, b, hw, o, t4);
            const float w0 = a.d.wbce, w1 = 1.f - a.d.wbce;
            for (int c = 0; c < 4; ++c) {
                float mv = __ldg(m + c * hw);
                v[0] += w1 * (t4[c] * logf(mv + 1e-8f)) + w0 * ((1.f - t4[c]) * logf((1.f - mv) + 1e-8f));
            }
        }
    }
    block_sum<1>(v, s_red);
    if (threadIdx.x == 0) a.d.partials[blockIdx.x] = v[0];
}

template <int KIND>
__global__ void bce_finalize(const BceArgs a) {
    CCB_PDL_WAIT();
    __shared__ float s_red[32];
    __shared__ float s_total;
    if (threadIdx.x == 0) s_total = 0.f;
    __syncthreads();
    for (int l = 0; l < a.t.nlevels; ++l) {
        float v[1] = {0.f};
        for (int k = a.t.blk_off[l] + threadIdx.x; k < a.t.blk_off[l + 1]; k += blockDim.x) v[0] += a.d.partials[k];
        block_sum<1>(v, s_red);
        if (threadIdx.x == 0) {
            float n = (float)a.t.B * (float)a.d.C * (float)a.t.h[l] * (float)a.t.w[l];
            s_total += (KIND == CCB_BCE_ONES) ? (v[0] / n) : -(v[0] / n);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) a.d.loss[0] = s_total;
}

template <int KIND>
__global__ void __launch_bounds__(PNT) bce_bwd_kernel(const BceArgs a) {
    CCB_PDL_WAIT();
    int l, b, y, x;
    if (!locate(a.t, l, b, y, x)) return;
    const int h = a.t.h[l], w = a.t.w[l], C = a.d.C;
    const long long hw = (long long)h * w;
    const float n = (float)a.t.B * (float)C * (float)h * (float)w;
    const float go = __ldg(a.d.grad_out) / n;
    long long o = (long long)y * w + x;
    const float* m = a.d.mask[l] + (long long)b * C * hw + o;
    float* dm = a.d.d_mask[l] + (long long)b * C * hw + o;
    if (KIND == CCB_BCE_ONES) {
        for (int c = 0; c < C; ++c) {
            float mv = __ldg(m + c * hw);
            dm[c * hw] = go * (mv - 1.f) / fmaxf((1.f - mv) * mv, 1e-12f);   // torch BCE backward
        }
    } else {
        float t4[4];
        consensus_target(a, l, b, hw, o, t4);
        const float w0 = a.d.wbce, w1 = 1.f - a.d.wbce;
        for (int c = 0; c < 4; ++c) {
            float mv = __ldg(m + c * hw);
            dm[c * hw] = -go * (w1 * t4[c] / (mv + 1e-8f) - w0 * (1.f - t4[c]) / ((1.f - mv) + 1e-8f));
        }
    }
}

}  // namespace ccb

using namespace ccb;

static int smooth_args(const ccb_smooth_desc* d, SmoothArgs& a, bool bwd) {
    CCB_REQUIRE(d != nullptr, CCB_ERR_ARG, "smooth: null descriptor");
    CCB_REQUIRE(d->nlevels >= 1 && d->nlevels <= CCB_MAX_LEVELS, CCB_ERR_ARG, "smooth: nlevels %d", d->nlevels);
    CCB_REQUIRE(d->kind == CCB_SMOOTH_EDGE || d->kind == CCB_SMOOTH_SECOND, CCB_ERR_ARG, "smooth: kind %d", d->kind);
    CCB_REQUIRE(d->B >= 1 && d->C >= 1, CCB_ERR_ARG, "smooth: bad B/C");
    a.d = *d;
    make_tab(a.t, d->nlevels, d->B, d->h, d->w);
    double wgt = 1.0;
    for (int l = 0; l < CCB_MAX_LEVELS; ++l) {
        a.lw[l] = (d->kind == CCB_SMOOTH_SECOND) ? (float)wgt : 1.f;
        wgt /= 2.3;
    }
    for (int l = 0; l < d->nlevels; ++l) {
        CCB_REQUIRE(d->h[l] >= 1 && d->w[l] >= 1, CCB_ERR_ARG, "smooth: level %d size %dx%d", l, d->h[l], d->w[l]);
        CCB_REQUIRE(d->pred[l] != nullptr, CCB_ERR_ARG, "smooth: pred[%d] null", l);
        if (d->kind == CCB_SMOOTH_EDGE) CCB_REQUIRE(d->img[l] != nullptr, CCB_ERR_ARG, "smooth: img[%d] null", l);
        if (bwd) CCB_REQUIRE(d->d_pred[l] != nullptr, CCB_ERR_ARG, "smooth: d_pred[%d] null", l);
    }
    return CCB_OK;
}

extern "C" long long ccb_smooth_partials_floats(const ccb_smooth_desc* d) {
    SmoothArgs a;
    if (smooth_args(d, a, false)) return -1;
    return (long long)a.t.blk_off[d->nlevels] * 4;
}

extern "C" int ccb_smooth_fwd(const ccb_smooth_desc* d, ccb_stream_t stream) {
    SmoothArgs a;
    int rc = smooth_args(d, a, false);
    if (rc) return rc;
    CCB_REQUIRE(d->loss, CCB_ERR_ARG, "smooth_fwd: loss null");
    CCB_REQUIRE_WORK("smooth_fwd", "partials", d->partials, d->partials_floats, ccb_smooth_partials_floats(d));
    dim3 grid(a.t.blk_off[d->nlevels]);
    if (d->kind == CCB_SMOOTH_EDGE) {
        CCB_LAUNCH(smooth_fwd_kernel<CCB_SMOOTH_EDGE>, grid, dim3(PNT), 0, stream, a);
        CCB_LAUNCH(smooth_finalize<CCB_SMOOTH_EDGE>, dim3(1), dim3(256), 0, stream, a);
    } else {
        CCB_LAUNCH(smooth_fwd_kernel<CCB_SMOOTH_SECOND>, grid, dim3(PNT), 0, stream, a);
        CCB_LAUNCH(smooth_finalize<CCB_SMOOTH_SECOND>, dim3(1), dim3(256), 0, stream, a);
    }
    return check_launch("smooth_fwd");
}

extern "C" int ccb_smooth_bwd(const ccb_smooth_desc* d, ccb_stream_t stream) {
    SmoothArgs a;
    int rc = smooth_args(d, a, true);
    if (rc) return rc;
    CCB_REQUIRE(d->grad_out, CCB_ERR_ARG, "smooth_bwd: grad_out null");
    dim3 grid(a.t.blk_off[d->nlevels]);
    if (d->kind == CCB_SMOOTH_EDGE) CCB_LAUNCH(smooth_bwd_kernel<CCB_SMOOTH_EDGE>, grid, dim3(PNT), 0, stream, a);
    else CCB_LAUNCH(smooth_bwd_kernel<CCB_SMOOTH_SECOND>, grid, dim3(PNT), 0, stream, a);
    return check_launch("smooth_bwd");
}

static int bce_args(const ccb_bce_desc* d, BceArgs& a, bool bwd) {
    CCB_REQUIRE(d != nullptr, CCB_ERR_ARG, "bce: null descriptor");
    CCB_REQUIRE(d->nlevels >= 1 && d->nlevels <= CCB_MAX_LEVELS, CCB_ERR_ARG, "bce: nlevels %d", d->nlevels);
    CCB_REQUIRE(d->kind == CCB_BCE_ONES || d->kind == CCB_BCE_CONSENSUS, CCB_ERR_ARG, "bce: kind %d", d->kind);
    CCB_REQUIRE(d->kind == CCB_BCE_ONES || d->C == 4, CCB_ERR_ARG, "bce: consensus needs 4 mask channels, got %d", d->C);
    a.d = *d;
    make_tab(a.t, d->nlevels, d->B, d->h, d->w);
    for (int l = 0; l < d->nlevels; ++l) {
        CCB_REQUIRE(d->mask[l] != nullptr, CCB_ERR_ARG, "bce: mask[%d] null", l);
        if (d->kind == CCB_BCE_CONSENSUS)
            CCB_REQUIRE(d->census_bwd[l] && d->census_fwd[l] && d->target_bwd[l] && d->target_fwd[l], CCB_ERR_ARG,
                        "bce: consensus inputs null at level %d", l);
        if (bwd) CCB_REQUIRE(d->d_mask[l] != nullptr, CCB_ERR_ARG, "bce: d_mask[%d] null", l);
    }
    return CCB_OK;
}

extern "C" long long ccb_bce_partials_floats(const ccb_bce_desc* d) {
    BceArgs a;
    if (bce_args(d, a, false)) return -1;
    return (long long)a.t.blk_off[d->nlevels];
}

extern "C" int ccb_bce_fwd(const ccb_bce_desc* d, ccb_stream_t stream) {
    BceArgs a;
    int rc = bce_args(d, a, false);
    if (rc) return rc;
    CCB_REQUIRE(d->loss, CCB_ERR_ARG, "bce_fwd: loss null");
    CCB_REQUIRE_WORK("bce_fwd", "partials", d->partials, d->partials_floats, ccb_bce_partials_floats(d));
    dim3 grid(a.t.blk_off[d->nlevels]);
    if (d->kind == CCB_BCE_ONES) {
        CCB_LAUNCH(bce_fwd_kernel<CCB_BCE_ONES>, grid, dim3(PNT), 0, stream, a);
        CCB_LAUNCH(bce_finalize<CCB_BCE_ONES>, dim3(1), dim3(256), 0, stream, a);
    } else {
        CCB_LAUNCH(bce_fwd_kernel<CCB_BCE_CONSENSUS>, grid, dim3(PNT), 0, stream, a);
        CCB_LAUNCH(bce_finalize<CCB_BCE_CONSENSUS>, dim3(1), dim3(256), 0, stream, a);
    }
    return check_launch("bce_fwd");
}

extern "C" int ccb_bce_bwd(const ccb_bce_desc* d, ccb_stream_t stream) {
    BceArgs a;
    int rc = bce_args(d, a, true);
    if (rc) return rc;
    CCB_REQUIRE(d->grad_out, CCB_ERR_ARG, "bce_bwd: grad_out null");
    dim3 grid(a.t.blk_off[d->nlevels]);
    if (d->kind == CCB_BCE_ONES) CCB_LAUNCH(bce_bwd_kernel<CCB_BCE_ONES>, grid, dim3(PNT), 0, stream, a);
    else CCB_LAUNCH(bce_bwd_kernel<CCB_BCE_CONSENSUS>, grid, dim3(PNT), 0, stream, a);
    return check_launch("bce_bwd");
}
