// b2f_ops.cu - the two non-conv operators of Back2Future (models/back2future.py):
//   correlate():  9x9 cost volume (third-party spatial_correlation_sample, kernel_size=1, patch_size=9)
//                 + the reference's channel permutation idx_fwd / idx_bwd, back2future.py:15-25,56-59,173-176
//   Model.warp(): feature warp = grid_sample(border, align_corners=False) of (grid + flow), :287-321
//                 (implemented by the flow_warp kernels in warp_ops.cu with the b2f normalisation)
#include "ccb_common.cuh"

namespace ccb {

// output channel p reads displacement (i, j):  idx_fwd[p] = (80 - p/9) - 9*(p%9);  idx_bwd[p] = idx_fwd[80-p]
__host__ __device__ __forceinline__ int corr_src(int p, int reversed) {
    int q = reversed ? 80 - p : p;
    return (80 - q / 9) - 9 * (q % 9);
}

__host__ __device__ __forceinline__ int corr_dst(int k, int reversed) {      // inverse of corr_src: natural displacement k -> output channel p
    // corr_src(q) = (80 - q/9) - 9*(q%9)  =>  k = 80 - a - 9 r with a = q/9, r = q%9  =>  r = (80-k)/9, a = (80-k)%9
    const int m = 80 - k;
    const int q = (m % 9) * 9 + m / 9;
    return reversed ? 80 - q : q;
}

constexpr int CT = 16;        // 16x16 pixel tile
constexpr int CH = CT + 8;    // + 4 px halo each side
constexpr int CG = 4;         // channels staged per barrier pair

// How many channel chunks a launch is cut into: the coarse pyramid levels have a handful of 16x16 tiles (4x13 map: ONE
// per sample) but up to 192 channels, so the channel loop is what has to be spread over the SMs.
__host__ __device__ __forceinline__ int corr_chunks(int B, int C, int h, int w) {
    const int tiles = cdiv(w, CT) * cdiv(h, CT) * B;
    int chunks = cdiv(2 * NUM_SMS, tiles);
    const int maxc = cdiv(C, CG);                  // at least one staged group per chunk
    if (chunks > maxc) chunks = maxc;
    if (chunks > 32) chunks = 32;
    return chunks < 1 ? 1 : chunks;
}

__device__ __forceinline__ void corr_stage(float (*s)[CH][CH + 1], const float* __restrict__ src, long long hw, int c0, int nc, int y0,
                                           int x0, int h, int w) {
    for (int idx = threadIdx.x; idx < CG * CH * CH; idx += CT * CT) {
        const int q = idx / (CH * CH), r = idx - q * (CH * CH);
        const int ry = r / CH, rx = r - ry * CH;
        const int gy = y0 - 4 + ry, gx = x0 - 4 + rx;
        s[q][ry][rx] = (q < nc && gy >= 0 && gy < h && gx >= 0 && gx < w) ? __ldg(src + (long long)(c0 + q) * hw + (long long)gy * w + gx) : 0.f;
    }
}

// out[b,p,y,x] = (1/C) sum_c f1[b,c,y,x] * f2[b,c,y+i-4,x+j-4],  (i,j) = divmod(corr_src(p), 9)
// grid (tiles_x, tiles_y, B * chunks): a CTA sums its chunk of the channels.  chunks == 1: the permuted, scaled result goes
// straight to `out`; else the raw sums go to part[chunk][b][k][y][x] (natural displacement order) and corr81_sum_kernel
// adds the chunks in a fixed order.
__global__ void __launch_bounds__(CT * CT) corr81_fwd_kernel(const float* __restrict__ f1, const float* __restrict__ f2,
                                                             float* __restrict__ out, float* __restrict__ part, int B, int C, int h,
                                                             int w, int reversed, int chunks) {
    CCB_PDL_WAIT();
    __shared__ float s2[CG][CH][CH + 1];
    const int b = blockIdx.z / chunks, chunk = blockIdx.z - b * chunks;
    const int x0 = blockIdx.x * CT, y0 = blockIdx.y * CT;
    const int tx = threadIdx.x % CT, ty = threadIdx.x / CT;
    const int x = x0 + tx, y = y0 + ty;
    const long long hw = (long long)h * w;
    const bool in = (y < h) && (x < w);
    const int per = cdiv(cdiv(C, chunks), CG) * CG;              // channels per chunk, a multiple of the staged group
    const int cbeg = chunk * per, cend = min(C, cbeg + per);
    float acc[81];
#pragma unroll
    for (int k = 0; k < 81; ++k) acc[k] = 0.f;
    for (int c = cbeg; c < cend; c += CG) {
        const int nc = min(CG, cend - c);
        __syncthreads();
        corr_stage(s2, f2 + (long long)b * C * hw, hw, c, nc, y0, x0, h, w);
        __syncthreads();
#pragma unroll
        for (int q = 0; q < CG; ++q) {
            const float a = (in && q < nc) ? __ldg(f1 + ((long long)b * C + c + q) * hw + (long long)y * w + x) : 0.f;
#pragma unroll
            for (int i = 0; i < 9; ++i)
#pragma unroll
                for (int j = 0; j < 9; ++j) acc[i * 9 + j] = fmaf(a, s2[q][ty + i][tx + j], acc[i * 9 + j]);
        }
    }
    if (!in) return;
    if (chunks == 1) {
#pragma unroll
        for (int k = 0; k < 81; ++k) out[((long long)b * 81 + corr_dst(k, reversed)) * hw + (long long)y * w + x] = acc[k] / (float)C;
    } else {
#pragma unroll
        for (int k = 0; k < 81; ++k) part[(((long long)chunk * B + b) * 81 + k) * hw + (long long)y * w + x] = acc[k];
    }
}

__global__ void __launch_bounds__(256) corr81_sum_kernel(const float* __restrict__ part, float* __restrict__ out, int B, int C, int h,
                                                         int w, int reversed, int chunks) {
    CCB_PDL_WAIT();
    const long long hw = (long long)h * w, n = (long long)B * 81 * hw;
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const long long px = i % hw;
    const int p = (int)((i / hw) % 81), b = (int)(i / (hw * 81));
    const int k = corr_src(p, reversed);
    float a = 0.f;
    for (int ch = 0; ch < chunks; ++ch) a += __ldg(part + (((long long)ch * B + b) * 81 + k) * hw + px);
    out[i] = a / (float)C;
}

// Backward.  d f1[b,c,y,x] = (1/C) sum_p g[b,p,y,x] f2[b,c,y+di,x+dj]        (di,dj) = displacement of channel p
//            d f2[b,c,y,x] = (1/C) sum_p g[b,p,y-di,x-dj] f1[b,c,y-di,x-dj]
// Both are ONE tiled kernel: d[c](y,x) = (1/C) sum_k G[k](y,x) * F[c](y + k/9 - 4, x + k%9 - 4) over the 81 NATURAL
// displacements k, with the thread's 81 G values held in registers and F[c] staged per channel in shared memory (tile
// + 4 px halo), exactly like the forward.  d f1 uses G[k] = g[p(k)] read in place; d f2 uses the mirrored problem
// (corr(f1,f2)[(i,j)](y,x) == corr(f2,f1)[(8-i,8-j)](y+i-4,x+j-4)): G'[80-k](y,x) = g[p(k)](y-di,x-dj), materialised
// by corr81_mirror_kernel (81 shifted copies of g, a streaming pass) and F = f1.
__global__ void __launch_bounds__(256) corr81_mirror_kernel(const float* __restrict__ g, float* __restrict__ gm, int B, int h, int w,
                                                            int reversed) {
    CCB_PDL_WAIT();
    const long long hw = (long long)h * w, n = (long long)B * 81 * hw;
    for (long long i0 = (long long)blockIdx.x * 256 + threadIdx.x; i0 < n; i0 += (long long)gridDim.x * 256) {
        const int x = (int)(i0 % w), y = (int)((i0 / w) % h);
        const int kk = (int)((i0 / hw) % 81), b = (int)(i0 / (hw * 81));      // kk = 80 - k: mirrored natural index
        const int k = 80 - kk;
        const int di = k / 9 - 4, dj = k % 9 - 4;
        const int ys = y - di, xs = x - dj;
        float v = 0.f;
        if (ys >= 0 && ys < h && xs >= 0 && xs < w) v = __ldg(g + ((long long)b * 81 + corr_dst(k, reversed)) * hw + (long long)ys * w + xs);
        gm[i0] = v;
    }
}

// natural != 0: G is already in natural displacement order (the mirrored buffer); else G[k] = g[corr_dst(k)].
// grid (tiles_x, tiles_y, B * chunks): the channels are independent outputs, a CTA takes its chunk of them.
__global__ void __launch_bounds__(CT * CT) corr81_dgrad_kernel(const float* __restrict__ G, const float* __restrict__ F,
                                                               float* __restrict__ d, int B, int C, int h, int w, int reversed,
                                                               int natural, int chunks) {
    CCB_PDL_WAIT();
    __shared__ float sf[CG][CH][CH + 1];
    const int b = blockIdx.z / chunks, chunk = blockIdx.z - b * chunks;
    const int x0 = blockIdx.x * CT, y0 = blockIdx.y * CT;
    const int tx = threadIdx.x % CT, ty = threadIdx.x / CT;
    const int x = x0 + tx, y = y0 + ty;
    const long long hw = (long long)h * w;
    const bool in = (y < h) && (x < w);
    const int per = cdiv(cdiv(C, chunks), CG) * CG;
    const int cbeg = chunk * per, cend = min(C, cbeg + per);
    float gk[81];
#pragma unroll
    for (int k = 0; k < 81; ++k) {
        const int p = natural ? k : corr_dst(k, reversed);
        gk[k] = in ? __ldg(G + ((long long)b * 81 + p) * hw + (long long)y * w + x) : 0.f;
    }
    const float invC = 1.f / (float)C;
    for (int c = cbeg; c < cend; c += CG) {
        const int nc = min(CG, cend - c);
        __syncthreads();
        corr_stage(sf, F + (long long)b * C * hw, hw, c, nc, y0, x0, h, w);
        __syncthreads();
#pragma unroll
        for (int q = 0; q < CG; ++q) {
            float a = 0.f;
#pragma unroll
            for (int i = 0; i < 9; ++i)
#pragma unroll
                for (int j = 0; j < 9; ++j) a = fmaf(gk[i * 9 + j], sf[q][ty + i][tx + j], a);
            if (in && q < nc) d[((long long)b * C + c + q) * hw + (long long)y * w + x] = a * invC;
        }
    }
}

}  // namespace ccb

using namespace ccb;

extern "C" long long ccb_corr81_fwd_workspace_floats(int B, int C, int h, int w) {
    const int chunks = corr_chunks(B, C, h, w);
    return chunks > 1 ? (long long)chunks * B * 81 * h * w : 0;
}

extern "C" int ccb_corr81_fwd(const float* f1, const float* f2, float* out, int B, int C, int h, int w, int reversed,
                              float* work, long long work_floats, ccb_stream_t stream) {
    CCB_REQUIRE(f1 && f2 && out && B >= 1 && C >= 1 && h >= 1 && w >= 1, CCB_ERR_ARG, "corr81_fwd: bad argument");
    const int chunks = corr_chunks(B, C, h, w);
    CCB_REQUIRE(chunks == 1 || (work && work_floats >= (long long)chunks * B * 81 * h * w), CCB_ERR_ARG,
                "corr81_fwd: workspace of ccb_corr81_fwd_workspace_floats() floats required");
    CCB_LAUNCH(corr81_fwd_kernel, dim3(cdiv(w, CT), cdiv(h, CT), B * chunks), dim3(CT * CT), 0, stream, f1, f2, out, work, B, C, h, w,
               reversed, chunks);
    if (chunks > 1) {
        const long long n = (long long)B * 81 * h * w;
        CCB_LAUNCH(corr81_sum_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, (const float*)work, out, B, C, h, w, reversed,
                   chunks);
    }
    return check_launch("corr81_fwd");
}

extern "C" int ccb_corr81_bwd(const float* f1, const float* f2, const float* grad_out, float* d_f1, float* d_f2, int B,
                              int C, int h, int w, int reversed, float* work, ccb_stream_t stream) {
    CCB_REQUIRE(f1 && f2 && grad_out && (d_f1 || d_f2), CCB_ERR_ARG, "corr81_bwd: bad argument");
    CCB_REQUIRE(d_f2 == nullptr || work != nullptr, CCB_ERR_ARG, "corr81_bwd: d_f2 needs a workspace of B*81*h*w floats");
    const int chunks = corr_chunks(B, C, h, w);
    const dim3 grid(cdiv(w, CT), cdiv(h, CT), B * chunks);
    if (d_f1) CCB_LAUNCH(corr81_dgrad_kernel, grid, dim3(CT * CT), 0, stream, grad_out, f2, d_f1, B, C, h, w, reversed, 0, chunks);
    if (d_f2) {
        const long long n = (long long)B * 81 * h * w;
        long long nb = (n + 255) / 256;
        if (nb > NUM_SMS * 16) nb = NUM_SMS * 16;
        CCB_LAUNCH(corr81_mirror_kernel, dim3((unsigned)nb), dim3(256), 0, stream, grad_out, work, B, h, w, reversed);
        CCB_LAUNCH(corr81_dgrad_kernel, grid, dim3(CT * CT), 0, stream, (const float*)work, f1, d_f2, B, C, h, w, reversed, 1, chunks);
    }
    return check_launch("corr81_bwd");
}
