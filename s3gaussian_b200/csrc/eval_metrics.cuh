// eval_metrics.cuh - per-view evaluation metrics of the reference's render_pixels (utils/video_utils.py:210-241):
// squared-error sums for PSNR and the SSIM map of skimage.metrics.structural_similarity, whole image and masked.
//
// The SSIM here is skimage's (>= 0.19, data_range = 1, float32 input), not the training SSIM of train_step.cuh
// (11-tap Gaussian window, zero padding, no covariance correction):
//   * 7x7 uniform window, scipy.ndimage.uniform_filter with mode 'reflect' (d c b a | a b c d | d c b a).  scipy
//     filters axis 0 then axis 1, each pass accumulating in double and storing float32; so does the stencil below;
//   * vx = 49/48 (uxx - ux^2), vy likewise, vxy = 49/48 (uxy - ux uy);
//   * S = (2 ux uy + C1)(2 vxy + C2) / ((ux^2 + uy^2 + C1)(vx + vy + C2)), C1 = 0.01^2, C2 = 0.03^2,
//     every operation rounded to float32 in numpy's order (no FMA contraction).
// Mean SSIM is over S cropped by 3 pixels on every side; the masked SSIM over the uncropped map (full=True).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "reduce.cuh"

namespace s3g {

constexpr int EV_T = 32;                    // output tile edge
constexpr int EV_R = 3;                     // window radius (7x7)
constexpr int EV_W = EV_T + 2 * EV_R;       // 38: staged tile edge
constexpr int EV_THREADS = 256;
constexpr int EV_PARTS = 5;                 // per block: sse, ssim (interior), masked sse, masked ssim, mask count

__device__ __forceinline__ int ev_reflect(int i, int n) {
    i = i < 0 ? -i - 1 : (i >= n ? 2 * n - 1 - i : i);
    return min(max(i, 0), n - 1);   // only positions outside the tile's window reach the clamp
}

// one 32x32 tile of one channel per block; partial[block][EV_PARTS]
__global__ void __launch_bounds__(EV_THREADS) eval_metrics_kernel(int H, int W, const float* __restrict__ x,
                                                                 const float* __restrict__ y,
                                                                 const uint8_t* __restrict__ mask,
                                                                 float* __restrict__ partial) {
    __shared__ float sx[EV_W][EV_W + 1], sy[EV_W][EV_W + 1];
    __shared__ float v[5][EV_T][EV_W + 1];   // vertical-pass means of x, y, x*x, y*y, x*y
    __shared__ float red[8];
    const int ch = blockIdx.z;
    const int x0 = blockIdx.x * EV_T, y0 = blockIdx.y * EV_T;
    const float* px = x + (size_t)ch * H * W;
    const float* py = y + (size_t)ch * H * W;
    for (int e = threadIdx.x; e < EV_W * EV_W; e += EV_THREADS) {
        const int r = e / EV_W, c = e - r * EV_W;
        const size_t o = (size_t)ev_reflect(y0 + r - EV_R, H) * W + ev_reflect(x0 + c - EV_R, W);
        sx[r][c] = __ldg(px + o);
        sy[r][c] = __ldg(py + o);
    }
    __syncthreads();
    // axis 0: EV_T rows x EV_W columns
    for (int e = threadIdx.x; e < EV_T * EV_W; e += EV_THREADS) {
        const int r = e / EV_W, c = e - r * EV_W;
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0, a4 = 0.0;
#pragma unroll
        for (int k = 0; k < 2 * EV_R + 1; ++k) {
            const float xv = sx[r + k][c], yv = sy[r + k][c];
            a0 += xv; a1 += yv;
            a2 += __fmul_rn(xv, xv); a3 += __fmul_rn(yv, yv); a4 += __fmul_rn(xv, yv);
        }
        v[0][r][c] = (float)(a0 / 7.0); v[1][r][c] = (float)(a1 / 7.0); v[2][r][c] = (float)(a2 / 7.0);
        v[3][r][c] = (float)(a3 / 7.0); v[4][r][c] = (float)(a4 / 7.0);
    }
    __syncthreads();
    const float cov_norm = (float)(49.0 / 48.0);
    const float C1 = (float)(0.01 * 0.01), C2 = (float)(0.03 * 0.03);
    float s_se = 0.f, s_ssim = 0.f, m_se = 0.f, m_ssim = 0.f, m_n = 0.f;
    for (int e = threadIdx.x; e < EV_T * EV_T; e += EV_THREADS) {
        const int r = e / EV_T, c = e - r * EV_T;
        const int gy = y0 + r, gx = x0 + c;
        if (gy >= H || gx >= W) continue;
        // axis 1
        double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0, a4 = 0.0;
#pragma unroll
        for (int k = 0; k < 2 * EV_R + 1; ++k) {
            a0 += v[0][r][c + k]; a1 += v[1][r][c + k]; a2 += v[2][r][c + k];
            a3 += v[3][r][c + k]; a4 += v[4][r][c + k];
        }
        const float ux = (float)(a0 / 7.0), uy = (float)(a1 / 7.0);
        const float uxx = (float)(a2 / 7.0), uyy = (float)(a3 / 7.0), uxy = (float)(a4 / 7.0);
        const float vx = __fmul_rn(cov_norm, __fsub_rn(uxx, __fmul_rn(ux, ux)));
        const float vy = __fmul_rn(cov_norm, __fsub_rn(uyy, __fmul_rn(uy, uy)));
        const float vxy = __fmul_rn(cov_norm, __fsub_rn(uxy, __fmul_rn(ux, uy)));
        const float A1 = __fadd_rn(__fmul_rn(__fmul_rn(2.f, ux), uy), C1);
        const float A2 = __fadd_rn(__fmul_rn(2.f, vxy), C2);
        const float B1 = __fadd_rn(__fadd_rn(__fmul_rn(ux, ux), __fmul_rn(uy, uy)), C1);
        const float B2 = __fadd_rn(__fadd_rn(vx, vy), C2);
        const float S = __fdiv_rn(__fmul_rn(A1, A2), __fmul_rn(B1, B2));
        const float d = __fsub_rn(sx[r + EV_R][c + EV_R], sy[r + EV_R][c + EV_R]);
        const float se = __fmul_rn(d, d);
        s_se += se;
        if (gy >= EV_R && gy < H - EV_R && gx >= EV_R && gx < W - EV_R) s_ssim += S;
        if (mask && mask[(size_t)gy * W + gx]) {
            m_se += se;
            m_ssim += S;
            m_n += 1.f;
        }
    }
    float* out = partial + (size_t)((blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) * EV_PARTS;
    const float t0 = block_sum_256(s_se, red);
    if (threadIdx.x == 0) out[0] = t0;
    const float t1 = block_sum_256(s_ssim, red);
    if (threadIdx.x == 0) out[1] = t1;
    const float t2 = block_sum_256(m_se, red);
    if (threadIdx.x == 0) out[2] = t2;
    const float t3 = block_sum_256(m_ssim, red);
    if (threadIdx.x == 0) out[3] = t3;
    const float t4 = block_sum_256(m_n, red);
    if (threadIdx.x == 0) out[4] = t4;
}

// block c sums the `tiles` partials of channel c in double: out[4c + 0..3]; block 0 also writes the mask count out[4C]
__global__ void __launch_bounds__(256) eval_reduce_kernel(int tiles, const float* __restrict__ partial,
                                                         double* __restrict__ out) {
    __shared__ double red[EV_PARTS][256];
    const int ch = blockIdx.x;
    const float* p = partial + (size_t)ch * tiles * EV_PARTS;
    double a[EV_PARTS] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < tiles; i += 256) {
#pragma unroll
        for (int k = 0; k < EV_PARTS; ++k) a[k] += p[(size_t)i * EV_PARTS + k];
    }
#pragma unroll
    for (int k = 0; k < EV_PARTS; ++k) red[k][threadIdx.x] = a[k];
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
#pragma unroll
            for (int k = 0; k < EV_PARTS; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x < 4) out[4 * ch + threadIdx.x] = red[threadIdx.x][0];
    if (ch == 0 && threadIdx.x == 4) out[4 * gridDim.x] = red[4][0];
}

}  // namespace s3g
