// b2f_ops.cu - the two non-conv operators of Back2Future (models/back2future.py):
//   correlate():  9x9 cost volume (third-party spatial_correlation_sample, kernel_size=1, patch_size=9)
//                 + the reference's channel permutation idx_fwd / idx_bwd, back2future.py:15-25,56-59,173-176
//   Model.warp(): feature warp = grid_sample(border, align_corners=False) of (grid + flow), :287-321
//                 (implemented by the flow_warp kernels in warp_ops.cu with the b2f normalisation)
// and FlowNetC6's 21x21 cost volume at dilation 2 (models/FlowNetC6.py:18-30), at the end of the file.
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
    if (B < 1 || C < 1 || h < 1 || w < 1) return -1;
    const int chunks = corr_chunks(B, C, h, w);
    return chunks > 1 ? (long long)chunks * B * 81 * h * w : 0;
}

extern "C" int ccb_corr81_fwd(const float* f1, const float* f2, float* out, int B, int C, int h, int w, int reversed,
                              float* work, long long work_floats, ccb_stream_t stream) {
    CCB_REQUIRE(f1 && f2 && out && B >= 1 && C >= 1 && h >= 1 && w >= 1, CCB_ERR_ARG, "corr81_fwd: bad argument");
    CCB_REQUIRE_WORK("corr81_fwd", "work", work, work_floats, ccb_corr81_fwd_workspace_floats(B, C, h, w));
    const int chunks = corr_chunks(B, C, h, w);
    CCB_LAUNCH(corr81_fwd_kernel, dim3(cdiv(w, CT), cdiv(h, CT), B * chunks), dim3(CT * CT), 0, stream, f1, f2, out, work, B, C, h, w,
               reversed, chunks);
    if (chunks > 1) {
        const long long n = (long long)B * 81 * h * w;
        CCB_LAUNCH(corr81_sum_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, stream, (const float*)work, out, B, C, h, w, reversed,
                   chunks);
    }
    return check_launch("corr81_fwd");
}

extern "C" long long ccb_corr81_bwd_workspace_floats(int B, int C, int h, int w) {
    if (B < 1 || C < 1 || h < 1 || w < 1) return -1;
    return (long long)B * 81 * h * w;
}

extern "C" int ccb_corr81_bwd(const float* f1, const float* f2, const float* grad_out, float* d_f1, float* d_f2, int B,
                              int C, int h, int w, int reversed, float* work, long long work_floats, ccb_stream_t stream) {
    CCB_REQUIRE(f1 && f2 && grad_out && (d_f1 || d_f2) && B >= 1 && C >= 1 && h >= 1 && w >= 1, CCB_ERR_ARG,
                "corr81_bwd: bad argument");
    CCB_REQUIRE_WORK("corr81_bwd", "work", work, work_floats, d_f2 ? ccb_corr81_bwd_workspace_floats(B, C, h, w) : 0);
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

// ---------------------------------------------------------------------------------------------------------------------
// FlowNetC6 (models/FlowNetC6.py:18-30,111-112): correlate() = spatial_correlation_sample(kernel 1, patch 21, stride 1,
// padding 0, dilation_patch 2) / C, followed by LeakyReLU(0.1).  441 displacements (2 (i - 10), 2 (j - 10)), i the
// vertical one; no channel permutation.  441 accumulators do not fit a thread, so a CTA of the forward takes ONE vertical
// displacement i and a 32x8 pixel tile, and each thread keeps the 21 horizontal displacements of its pixel.  The f2 rows
// that displacement reads are staged per channel group with a 20 px halo either side.  Every output sums its channels in
// order 0..C-1 in one thread: the result depends on the shape only, and no workspace or atomic is involved.
namespace ccb {

constexpr int CD_N = 21;                 // displacements per axis
constexpr int CD_R = 20;                 // largest |displacement| in pixels: dilation 2 * 10
constexpr int CD_TX = 32, CD_TY = 8;     // pixel tile: one warp per tile row
constexpr int CD_SW = CD_TX + 2 * CD_R;  // staged row: tile + halo
constexpr int CD_CGF = 8;                // channels staged per barrier pair, forward
constexpr int CD_CGB = 16;               // and backward (= channels one backward CTA produces)
constexpr float CD_SLOPE = 0.1f;         // corr_activation = nn.LeakyReLU(0.1)

// s[q][r][col] = src[c0 + q](y0 + r + dy, x0 - 20 + col); zero outside the map and for q >= nc
template <int NCG>
__device__ __forceinline__ void corr441d_stage(float (*s)[CD_TY][CD_SW], const float* __restrict__ src, long long hw, int c0, int nc,
                                               int y0, int dy, int x0, int h, int w) {
    for (int idx = threadIdx.x; idx < NCG * CD_TY * CD_SW; idx += CD_TX * CD_TY) {
        const int q = idx / (CD_TY * CD_SW), r = idx - q * (CD_TY * CD_SW);
        const int ry = r / CD_SW, rx = r - ry * CD_SW;
        const int gy = y0 + ry + dy, gx = x0 - CD_R + rx;
        s[q][ry][rx] = (q < nc && gy >= 0 && gy < h && gx >= 0 && gx < w) ? __ldg(src + (long long)(c0 + q) * hw + (long long)gy * w + gx) : 0.f;
    }
}

// grid (tiles_x, tiles_y, B * 21): out[b, 21 i + j, y, x] = leaky((1/C) sum_c f1[b,c,y,x] f2[b,c,y + 2(i-10),x + 2(j-10)])
__global__ void __launch_bounds__(CD_TX * CD_TY) corr441d_fwd_kernel(const float* __restrict__ f1, const float* __restrict__ f2,
                                                                     float* __restrict__ out, int C, int h, int w) {
    CCB_PDL_WAIT();
    __shared__ float s2[CD_CGF][CD_TY][CD_SW];
    const int b = blockIdx.z / CD_N, i = blockIdx.z - b * CD_N;
    const int x0 = blockIdx.x * CD_TX, y0 = blockIdx.y * CD_TY;
    const int tx = threadIdx.x % CD_TX, ty = threadIdx.x / CD_TX;
    const int x = x0 + tx, y = y0 + ty;
    const long long hw = (long long)h * w;
    const bool in = (y < h) && (x < w);
    const float* a1 = f1 + (long long)b * C * hw + (long long)y * w + x;
    float acc[CD_N];
#pragma unroll
    for (int j = 0; j < CD_N; ++j) acc[j] = 0.f;
    for (int c = 0; c < C; c += CD_CGF) {
        const int nc = min(CD_CGF, C - c);
        __syncthreads();
        corr441d_stage<CD_CGF>(s2, f2 + (long long)b * C * hw, hw, c, nc, y0, 2 * (i - 10), x0, h, w);
        __syncthreads();
#pragma unroll
        for (int q = 0; q < CD_CGF; ++q) {
            const float a = (in && q < nc) ? __ldg(a1 + (long long)(c + q) * hw) : 0.f;
#pragma unroll
            for (int j = 0; j < CD_N; ++j) acc[j] = fmaf(a, s2[q][ty][tx + 2 * j], acc[j]);
        }
    }
    if (!in) return;
    float* o = out + ((long long)b * CD_N * CD_N + i * CD_N) * hw + (long long)y * w + x;
#pragma unroll
    for (int j = 0; j < CD_N; ++j) {
        const float v = acc[j] / (float)C;
        o[(long long)j * hw] = v > 0.f ? v : v * CD_SLOPE;
    }
}

// Backward, both inputs with one kernel: d[c](y,x) = (1/C) sum_{i,j} G[i,j](y,x) F[c](y + 2(i-10), x + 2(j-10)), summed
// over i then j, with dz = g * leaky'(out) (the sign of the stored output, as ccb_act_bwd_bias).
//   d f1: F = f2, G[i,j](y,x) = dz[21 i + j](y,x).
//   d f2: F = f1 and the mirrored gradient G[i,j](y,x) = dz[21 (20-i) + (20-j)](y + 2(i-10), x + 2(j-10)) (zero outside the
//         map), gathered in place: corr(f1,f2)[i,j](y,x) reads f2 at the pixel that corr(f2,f1)[20-i,20-j] maps back to.
// grid (tiles_x, tiles_y, B * ceil(C / 16)): a CTA produces 16 channels of a pixel tile.
__global__ void __launch_bounds__(CD_TX * CD_TY) corr441d_bwd_kernel(const float* __restrict__ g, const float* __restrict__ out,
                                                                     const float* __restrict__ F, float* __restrict__ d, int C,
                                                                     int h, int w, int mirrored) {
    CCB_PDL_WAIT();
    __shared__ float sf[CD_CGB][CD_TY][CD_SW];
    const int groups = cdiv(C, CD_CGB);
    const int b = blockIdx.z / groups, c0 = (blockIdx.z - b * groups) * CD_CGB;
    const int nc = min(CD_CGB, C - c0);
    const int x0 = blockIdx.x * CD_TX, y0 = blockIdx.y * CD_TY;
    const int tx = threadIdx.x % CD_TX, ty = threadIdx.x / CD_TX;
    const int x = x0 + tx, y = y0 + ty;
    const long long hw = (long long)h * w;
    const bool in = (y < h) && (x < w);
    const long long gb = (long long)b * CD_N * CD_N * hw;
    float acc[CD_CGB];
#pragma unroll
    for (int q = 0; q < CD_CGB; ++q) acc[q] = 0.f;
    for (int i = 0; i < CD_N; ++i) {
        const int dy = 2 * (i - 10);
        float gk[CD_N];
#pragma unroll
        for (int j = 0; j < CD_N; ++j) {
            const int ys = mirrored ? y + dy : y, xs = mirrored ? x + 2 * (j - 10) : x;
            const int p = mirrored ? (CD_N - 1 - i) * CD_N + (CD_N - 1 - j) : i * CD_N + j;
            float v = 0.f;
            if (in && ys >= 0 && ys < h && xs >= 0 && xs < w) {
                const long long k = gb + (long long)p * hw + (long long)ys * w + xs;
                v = __ldg(g + k);
                v = __ldg(out + k) > 0.f ? v : v * CD_SLOPE;
            }
            gk[j] = v;
        }
        __syncthreads();
        corr441d_stage<CD_CGB>(sf, F + (long long)b * C * hw, hw, c0, nc, y0, dy, x0, h, w);
        __syncthreads();
#pragma unroll
        for (int q = 0; q < CD_CGB; ++q)
#pragma unroll
            for (int j = 0; j < CD_N; ++j) acc[q] = fmaf(gk[j], sf[q][ty][tx + 2 * j], acc[q]);
    }
    if (!in) return;
#pragma unroll
    for (int q = 0; q < CD_CGB; ++q)
        if (q < nc) d[((long long)b * C + c0 + q) * hw + (long long)y * w + x] = acc[q] / (float)C;
}

}  // namespace ccb

extern "C" int ccb_corr441d_fwd(const float* f1, const float* f2, float* out, int B, int C, int h, int w, ccb_stream_t stream) {
    CCB_REQUIRE(f1 && f2 && out && B >= 1 && C >= 1 && h >= 1 && w >= 1, CCB_ERR_ARG, "corr441d_fwd: bad argument");
    CCB_REQUIRE((long long)B * CD_N <= 65535, CCB_ERR_ARG, "corr441d_fwd: batch too large");
    CCB_LAUNCH(corr441d_fwd_kernel, dim3(cdiv(w, CD_TX), cdiv(h, CD_TY), B * CD_N), dim3(CD_TX * CD_TY), 0, stream, f1, f2, out, C, h, w);
    return check_launch("corr441d_fwd");
}

extern "C" int ccb_corr441d_bwd(const float* f1, const float* f2, const float* out, const float* grad_out, float* d_f1, float* d_f2,
                                int B, int C, int h, int w, ccb_stream_t stream) {
    CCB_REQUIRE(f1 && f2 && out && grad_out && (d_f1 || d_f2) && B >= 1 && C >= 1 && h >= 1 && w >= 1, CCB_ERR_ARG,
                "corr441d_bwd: bad argument");
    CCB_REQUIRE((long long)B * cdiv(C, CD_CGB) <= 65535, CCB_ERR_ARG, "corr441d_bwd: batch x channels too large");
    const dim3 grid(cdiv(w, CD_TX), cdiv(h, CD_TY), B * cdiv(C, CD_CGB));
    if (d_f1) CCB_LAUNCH(corr441d_bwd_kernel, grid, dim3(CD_TX * CD_TY), 0, stream, grad_out, out, f2, d_f1, C, h, w, 0);
    if (d_f2) CCB_LAUNCH(corr441d_bwd_kernel, grid, dim3(CD_TX * CD_TY), 0, stream, grad_out, out, f1, d_f2, C, h, w, 1);
    return check_launch("corr441d_bwd");
}
