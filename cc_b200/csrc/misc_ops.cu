// misc_ops.cu - the small non-GEMM layers of the four networks and the optimiser:
//   BatchNorm2d (train-mode batch statistics) fwd/bwd   models/DispResNet6.py:45-52 (13 layers)
//   bilinear x2 upsample (align_corners=False) fwd/bwd  models/DispResNet6.py:174,180,186; back2future.py:60
//   fused multi-tensor Adam over one flat buffer         train.py:307-310,568
#include "ccb_common.cuh"

namespace ccb {

// ---- BatchNorm (training) ---------------------------------------------------------------------------
// Three fully parallel passes (the 1x1-downsample BNs of the decoder see 16-64 channels x 3.4 M values:
// one CTA per channel would serialise the whole plane):
//   1. bn_partial_kernel  : grid (C, nsplit): per-(channel, split) count / mean / M2 (two-pass inside the split)
//   2. bn_merge_kernel    : Chan merge of the splits -> stats[c] = {mean, invstd}; running-stat update
//   3. bn_apply_kernel    : y = (x - mean) * invstd * gamma + beta, elementwise
constexpr int BN_CHUNK = 8192;       // elements of one (batch, channel) plane handled per split-CTA

__global__ void __launch_bounds__(256) bn_partial_kernel(const float* __restrict__ x, float* __restrict__ part, int B, int C,
                                                         int plane, int nsplit) {
    CCB_PDL_WAIT();
    __shared__ float s_red[32];
    __shared__ float s_mean;
    const int c = blockIdx.x, sp = blockIdx.y;
    const long long per = (long long)B * plane;                 // values of this channel
    const long long beg = (long long)sp * BN_CHUNK, end = min(per, beg + (long long)BN_CHUNK);
    float v[1] = {0.f};
    for (long long i = beg + threadIdx.x; i < end; i += 256) {
        int b = (int)(i / plane), o = (int)(i - (long long)b * plane);
        v[0] += __ldg(x + ((long long)b * C + c) * plane + o);
    }
    block_sum<1>(v, s_red);
    const float n = (float)(end - beg);
    if (threadIdx.x == 0) s_mean = v[0] / n;
    __syncthreads();
    const float mean = s_mean;
    v[0] = 0.f;
    for (long long i = beg + threadIdx.x; i < end; i += 256) {
        int b = (int)(i / plane), o = (int)(i - (long long)b * plane);
        float d = __ldg(x + ((long long)b * C + c) * plane + o) - mean;
        v[0] += d * d;
    }
    block_sum<1>(v, s_red);
    if (threadIdx.x == 0) {
        float* p = part + ((long long)c * nsplit + sp) * 3;
        p[0] = n; p[1] = mean; p[2] = v[0];
    }
}

__global__ void bn_merge_kernel(const float* __restrict__ part, float* __restrict__ stats, float* __restrict__ run_mean,
                                float* __restrict__ run_var, int C, int nsplit, float eps, float momentum) {
    CCB_PDL_WAIT();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float n = 0.f, mean = 0.f, m2 = 0.f;
    for (int s = 0; s < nsplit; ++s) {                          // Chan et al. pairwise merge, fixed order
        const float* p = part + ((long long)c * nsplit + s) * 3;
        float nb = p[0], mb = p[1], m2b = p[2];
        float nt = n + nb, delta = mb - mean;
        mean += delta * (nb / nt);
        m2 += m2b + delta * delta * (n * nb / nt);
        n = nt;
    }
    float var = m2 / n;
    stats[2 * c] = mean;
    stats[2 * c + 1] = 1.f / sqrtf(var + eps);
    if (run_mean) {
        run_mean[c] = (1.f - momentum) * run_mean[c] + momentum * mean;
        float unb = (n > 1.f) ? m2 / (n - 1.f) : var;
        run_var[c] = (1.f - momentum) * run_var[c] + momentum * unb;
    }
}

__global__ void __launch_bounds__(256) bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, const float* __restrict__ stats,
                                                       float* __restrict__ y, long long numel, int C, int plane) {
    CCB_PDL_WAIT();
    long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= numel) return;
    int c = (int)((i / plane) % C);
    y[i] = (__ldg(x + i) - __ldg(stats + 2 * c)) * __ldg(stats + 2 * c + 1) * __ldg(gamma + c) + __ldg(beta + c);
}

// eval mode: y = (x - running_mean) / sqrt(running_var + eps) * gamma + beta
__global__ void __launch_bounds__(256) bn_eval_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                      const float* __restrict__ beta, const float* __restrict__ rm,
                                                      const float* __restrict__ rv, float* __restrict__ y, int B, int C,
                                                      int plane, float eps) {
    CCB_PDL_WAIT();
    const int c = blockIdx.x;
    const float mean = __ldg(rm + c), inv = 1.f / sqrtf(__ldg(rv + c) + eps), g = __ldg(gamma + c), bt = __ldg(beta + c);
    for (int b = 0; b < B; ++b) {
        const float* p = x + ((long long)b * C + c) * plane;
        float* q = y + ((long long)b * C + c) * plane;
        for (int i = threadIdx.x; i < plane; i += 256) q[i] = (__ldg(p + i) - mean) * inv * g + bt;
    }
}

// backward: partial sums of (dy, dy * xhat) per (channel, split) -> reduce -> elementwise dx
__global__ void __launch_bounds__(256) bn_bwd_partial_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                             const float* __restrict__ stats, float* __restrict__ part, int B,
                                                             int C, int plane, int nsplit) {
    CCB_PDL_WAIT();
    __shared__ float s_red[2 * 32];
    const int c = blockIdx.x, sp = blockIdx.y;
    const long long per = (long long)B * plane;
    const long long beg = (long long)sp * BN_CHUNK, end = min(per, beg + (long long)BN_CHUNK);
    const float mean = __ldg(stats + 2 * c), inv = __ldg(stats + 2 * c + 1);
    float v[2] = {0.f, 0.f};
    for (long long i = beg + threadIdx.x; i < end; i += 256) {
        int b = (int)(i / plane), o = (int)(i - (long long)b * plane);
        long long off = ((long long)b * C + c) * plane + o;
        float d = __ldg(dy + off);
        v[0] += d;
        v[1] += d * (__ldg(x + off) - mean) * inv;
    }
    block_sum<2>(v, s_red);
    if (threadIdx.x == 0) {
        float* p = part + ((long long)c * nsplit + sp) * 2;
        p[0] = v[0]; p[1] = v[1];
    }
}

__global__ void bn_bwd_merge_kernel(const float* __restrict__ part, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                    float* __restrict__ sums, int C, int nsplit) {
    CCB_PDL_WAIT();
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float a = 0.f, b = 0.f;
    for (int s = 0; s < nsplit; ++s) { a += part[((long long)c * nsplit + s) * 2]; b += part[((long long)c * nsplit + s) * 2 + 1]; }
    dbeta[c] = a;
    dgamma[c] = b;
    sums[2 * c] = a;
    sums[2 * c + 1] = b;
}

__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ dy,
                                                           const float* __restrict__ gamma, const float* __restrict__ stats,
                                                           const float* __restrict__ sums, float* __restrict__ dx,
                                                           long long numel, int C, int plane, float inv_n) {
    CCB_PDL_WAIT();
    long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= numel) return;
    int c = (int)((i / plane) % C);
    const float mean = __ldg(stats + 2 * c), inv = __ldg(stats + 2 * c + 1);
    float xh = (__ldg(x + i) - mean) * inv;
    dx[i] = __ldg(gamma + c) * inv * (__ldg(dy + i) - __ldg(sums + 2 * c) * inv_n - xh * __ldg(sums + 2 * c + 1) * inv_n);
}

// ---- bilinear x2 upsample, align_corners=False (F.interpolate scale_factor=2) ---------------------
// out [planes, 2h, 2w]; source index = (o + 0.5)/2 - 0.5 clamped at 0 (ATen area_pixel_compute_source_index)
__device__ __forceinline__ void up2_src(int o, int n, int& i0, int& i1, float& l1) {
    float s = ((float)o + 0.5f) * 0.5f - 0.5f;
    if (s < 0.f) s = 0.f;
    i0 = (int)s;
    i1 = i0 + ((i0 < n - 1) ? 1 : 0);
    l1 = s - (float)i0;
}

__global__ void __launch_bounds__(256) upsample2x_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int planes,
                                                             int h, int w) {
    CCB_PDL_WAIT();
    const int H = 2 * h, W = 2 * w;
    long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= (long long)planes * H * W) return;
    int ox = (int)(i % W), oy = (int)((i / W) % H), p = (int)(i / ((long long)W * H));
    int y0, y1, x0, x1;
    float ly, lx;
    up2_src(oy, h, y0, y1, ly);
    up2_src(ox, w, x0, x1, lx);
    const float* s = x + (long long)p * h * w;
    float hy = 1.f - ly, hx = 1.f - lx;
    y[i] = hy * (hx * __ldg(s + y0 * w + x0) + lx * __ldg(s + y0 * w + x1)) +
           ly * (hx * __ldg(s + y1 * w + x0) + lx * __ldg(s + y1 * w + x1));
}

// gather form of the transpose: each source pixel collects from the <= 4x4 outputs that read it
__global__ void __launch_bounds__(256) upsample2x_bwd_kernel(const float* __restrict__ dy, float* __restrict__ dx, int planes,
                                                             int h, int w) {
    CCB_PDL_WAIT();
    const int H = 2 * h, W = 2 * w;
    long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= (long long)planes * h * w) return;
    int sx = (int)(i % w), sy = (int)((i / w) % h), p = (int)(i / ((long long)w * h));
    const float* g = dy + (long long)p * H * W;
    float acc = 0.f;
    for (int oy = max(0, 2 * sy - 2); oy <= min(H - 1, 2 * sy + 2); ++oy) {
        int y0, y1;
        float ly;
        up2_src(oy, h, y0, y1, ly);
        float wy = ((y0 == sy) ? (1.f - ly) : 0.f) + ((y1 == sy) ? ly : 0.f);
        if (wy == 0.f) continue;
        for (int ox = max(0, 2 * sx - 2); ox <= min(W - 1, 2 * sx + 2); ++ox) {
            int x0, x1;
            float lx;
            up2_src(ox, w, x0, x1, lx);
            float wx = ((x0 == sx) ? (1.f - lx) : 0.f) + ((x1 == sx) ? lx : 0.f);
            if (wx != 0.f) acc += wy * wx * __ldg(g + (long long)oy * W + ox);
        }
    }
    dx[i] = acc;
}

// ---- Adam over a flat parameter / gradient buffer (torch.optim.Adam semantics, no weight decay) ----
// The step counters and bias corrections live in device memory (group g: state[4g..4g+2] = step, 1-b1^t, sqrt(1-b2^t))
// so that the whole training step can be captured once in a CUDA graph and replayed.  One thread per group; groups
// whose `active` flag is zero (a fixed network) keep their count.
__global__ void adam_prep_kernel(float* __restrict__ state, const int* __restrict__ active, int ngroups, float b1, float b2) {
    CCB_PDL_WAIT();
    const int grp = blockIdx.x * blockDim.x + threadIdx.x;
    if (grp < ngroups && (active == nullptr || __ldg(active + grp) != 0)) {
        float* s = state + 4 * grp;
        float t = s[0] + 1.f;
        s[0] = t;
        s[1] = (float)(1.0 - pow((double)b1, (double)t));
        s[2] = (float)sqrt(1.0 - pow((double)b2, (double)t));
    }
}

// grad_scale multiplies the gradient first (1/world_size after the NCCL sum).
// Block -> range: the largest entry whose first_block <= blockIdx.x (binary search over the table).  The range decides
// only which elements and which group's bias corrections a thread uses, never the per-element arithmetic.
__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                   float* __restrict__ v, const long long* __restrict__ ranges, int nranges,
                                                   const float* __restrict__ state,
                                                   float lr, float b1, float b2, float eps, float grad_scale) {
    CCB_PDL_WAIT();
    long long blk = blockIdx.x;
    int lo = 0, hi = nranges - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(ranges + 4 * mid + 3) <= blk) lo = mid;
        else hi = mid - 1;
    }
    const long long off = __ldg(ranges + 4 * lo), cnt = __ldg(ranges + 4 * lo + 1);
    const int grp = (int)__ldg(ranges + 4 * lo + 2);
    blk -= __ldg(ranges + 4 * lo + 3);
    const long long j = blk * 256 + threadIdx.x;
    if (j >= cnt) return;
    const long long i = off + j;
    const float bc1 = __ldg(state + 4 * grp + 1), bc2_sqrt = __ldg(state + 4 * grp + 2);
    float gi = __ldg(g + i) * grad_scale;
    float mi = b1 * m[i] + (1.f - b1) * gi;
    float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    float denom = sqrtf(vi) / bc2_sqrt + eps;
    p[i] = p[i] - (lr / bc1) * (mi / denom);
}

}  // namespace ccb

using namespace ccb;

extern "C" long long ccb_bn_workspace_floats(int B, int C, int plane) {
    if (B < 1 || C < 1 || plane < 1) return -1;
    long long nsplit = ((long long)B * plane + BN_CHUNK - 1) / BN_CHUNK;
    return (long long)C * nsplit * 3 + 2 * C;
}

extern "C" int ccb_bn_fwd(const float* x, const float* gamma, const float* beta, float* y, float* stats,
                          float* running_mean, float* running_var, int B, int C, int plane, float eps, float momentum,
                          int training, float* work, long long work_floats, ccb_stream_t stream) {
    CCB_REQUIRE(x && gamma && beta && y, CCB_ERR_ARG, "bn_fwd: null pointer");
    CCB_REQUIRE(B >= 1 && C >= 1 && plane >= 1, CCB_ERR_ARG, "bn_fwd: bad size");
    CCB_REQUIRE_WORK("bn_fwd", "work", work, work_floats, training ? ccb_bn_workspace_floats(B, C, plane) : 0);
    if (training) {
        CCB_REQUIRE(stats != nullptr, CCB_ERR_ARG, "bn_fwd: stats null in training mode");
        const int nsplit = (int)(((long long)B * plane + BN_CHUNK - 1) / BN_CHUNK);
        const long long numel = (long long)B * C * plane;
        CCB_LAUNCH(bn_partial_kernel, dim3(C, nsplit), dim3(256), 0, stream, x, work, B, C, plane, nsplit);
        CCB_LAUNCH(bn_merge_kernel, dim3(cdiv(C, 128)), dim3(128), 0, stream, (const float*)work, stats, running_mean, running_var, C,
                   nsplit, eps, momentum);
        CCB_LAUNCH(bn_apply_kernel, dim3((unsigned)((numel + 255) / 256)), dim3(256), 0, stream, x, gamma, beta, (const float*)stats, y,
                   numel, C, plane);
    } else {
        CCB_REQUIRE(running_mean && running_var, CCB_ERR_ARG, "bn_fwd: running stats null in eval mode");
        CCB_LAUNCH(bn_eval_kernel, dim3(C), dim3(256), 0, stream, x, gamma, beta, (const float*)running_mean,
                   (const float*)running_var, y, B, C, plane, eps);
    }
    return check_launch("bn_fwd");
}

extern "C" int ccb_bn_bwd(const float* x, const float* dy, const float* gamma, const float* stats, float* dx,
                          float* dgamma, float* dbeta, int B, int C, int plane, float* work, long long work_floats,
                          ccb_stream_t stream) {
    CCB_REQUIRE(x && dy && gamma && stats && dx && dgamma && dbeta, CCB_ERR_ARG, "bn_bwd: null pointer");
    CCB_REQUIRE(B >= 1 && C >= 1 && plane >= 1, CCB_ERR_ARG, "bn_bwd: bad size");
    CCB_REQUIRE_WORK("bn_bwd", "work", work, work_floats, ccb_bn_workspace_floats(B, C, plane));
    const int nsplit = (int)(((long long)B * plane + BN_CHUNK - 1) / BN_CHUNK);
    const long long numel = (long long)B * C * plane;
    float* sums = work + (long long)C * nsplit * 3;
    CCB_LAUNCH(bn_bwd_partial_kernel, dim3(C, nsplit), dim3(256), 0, stream, x, dy, stats, work, B, C, plane, nsplit);
    CCB_LAUNCH(bn_bwd_merge_kernel, dim3(cdiv(C, 128)), dim3(128), 0, stream, (const float*)work, dgamma, dbeta, sums, C, nsplit);
    CCB_LAUNCH(bn_bwd_apply_kernel, dim3((unsigned)((numel + 255) / 256)), dim3(256), 0, stream, x, dy, gamma, stats,
               (const float*)sums, dx, numel, C, plane, 1.f / ((float)B * (float)plane));
    return check_launch("bn_bwd");
}

extern "C" int ccb_upsample2x_fwd(const float* x, float* y, int planes, int h, int w, ccb_stream_t stream) {
    CCB_REQUIRE(x && y && planes >= 1 && h >= 1 && w >= 1, CCB_ERR_ARG, "upsample2x_fwd: bad argument");
    long long n = (long long)planes * 4 * h * w;
    CCB_LAUNCH(upsample2x_fwd_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, x, y, planes, h, w);
    return check_launch("upsample2x_fwd");
}

extern "C" int ccb_upsample2x_bwd(const float* dy, float* dx, int planes, int h, int w, ccb_stream_t stream) {
    CCB_REQUIRE(dy && dx && planes >= 1 && h >= 1 && w >= 1, CCB_ERR_ARG, "upsample2x_bwd: bad argument");
    long long n = (long long)planes * h * w;
    CCB_LAUNCH(upsample2x_bwd_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, dy, dx, planes, h, w);
    return check_launch("upsample2x_bwd");
}

extern "C" int ccb_adam_step_ranges(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                                    const long long* ranges, int nranges, long long nblocks, const int* group_active,
                                    int ngroups, float* group_state, float lr, float beta1, float beta2, float eps,
                                    float grad_scale, ccb_stream_t stream) {
    CCB_REQUIRE(params && grads && exp_avg && exp_avg_sq && group_state && ngroups >= 1 && nranges >= 0 && nblocks >= 0,
                CCB_ERR_ARG, "adam_step_ranges: bad argument");
    CCB_REQUIRE(nranges == 0 || (ranges != nullptr && nblocks >= 1), CCB_ERR_ARG, "adam_step_ranges: empty range table");
    CCB_REQUIRE(nblocks < (1LL << 31), CCB_ERR_ARG, "adam_step_ranges: %lld blocks", nblocks);
    CCB_LAUNCH(adam_prep_kernel, dim3(cdiv(ngroups, 32)), dim3(32), 0, stream, group_state, group_active, ngroups, beta1, beta2);
    int rc = check_launch("adam_prep");
    if (rc || nranges == 0) return rc;
    CCB_LAUNCH(adam_kernel, dim3((unsigned)nblocks), dim3(256), 0, stream, params, grads, exp_avg, exp_avg_sq, ranges, nranges,
               (const float*)group_state, lr, beta1, beta2, eps, grad_scale);
    return check_launch("adam_step_ranges");
}
