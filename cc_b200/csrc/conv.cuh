// conv.cuh - what the CUDA-core (conv_ffma.cu) and tensor-core (conv_tc.cu) convolution paths share.
#pragma once
#include "ccb_common.cuh"

namespace ccb {

// the epilogue activation (CCB_ACT_*), applied after bias and residual
__device__ __forceinline__ float apply_act(float v, int act, float slope) {
    switch (act) {
        case CCB_ACT_RELU: return fmaxf(v, 0.f);
        case CCB_ACT_LEAKY: return v > 0.f ? v : v * slope;
        case CCB_ACT_SIGMOID: return 1.f / (1.f + expf(-v));
        default: return v;
    }
}

// out[i] = act(sum_s work[s][i] + bias[(i / plane) % C] + res[i]) over split-K partials work[splits][numel], summed in
// s order from 0.f; bias and res may be null (conv_ffma.cu)
void launch_splitk_reduce(const float* work, float* out, const float* bias, const float* res, long long numel, int splits,
                          int plane, int C, int act, float slope, cudaStream_t st);

// tensor-core path (conv_tc.cu)
bool tc_supported(const ccb_conv_desc* d, int op);
bool tc_profitable(const ccb_conv_desc* d, int op);
int tc_plan(const ccb_conv_desc* d, int op, long long& panel_floats);
int tc_fprop(const ccb_conv_desc* d, const float* x, const float* w, const float* bias, const float* res, float* y,
             float* wp, float* partial, int splits, cudaStream_t st);
int tc_dgrad(const ccb_conv_desc* d, const float* dy, const float* w, const float* bias, const float* res, float* dx,
             float* wp, float* partial, int splits, cudaStream_t st);
int tc_wgrad(const ccb_conv_desc* d, const float* x, const float* dy, float* dw, float* partial, int splits, cudaStream_t st);

// Stride-parity class (py, px) of a data gradient: the Hc x Wc pixels dx[.., py + jy*s, px + jx*s], which only the
// filter taps ky = ky0 + j*s (j < nky) and kx = kx0 + j*s (j < nkx) reach; nky or nkx is 0 where no tap does.
struct DgradClass { int py, px, Hc, Wc, ky0, kx0, nky, nkx; };

inline DgradClass dgrad_class(const ccb_conv_desc* d, int py, int px) {
    const int s = d->stride;
    DgradClass c;
    c.py = py; c.px = px;
    c.Hc = (d->Hi - py + s - 1) / s; c.Wc = (d->Wi - px + s - 1) / s;
    c.ky0 = (py + d->pad) % s; c.kx0 = (px + d->pad) % s;
    c.nky = (d->kh > c.ky0) ? (d->kh - c.ky0 + s - 1) / s : 0;
    c.nkx = (d->kw > c.kx0) ? (d->kw - c.kx0 + s - 1) / s : 0;
    return c;
}

}  // namespace ccb
