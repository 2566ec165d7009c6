// train_step.cuh - the per-iteration work either side of render() in the reference's training
// loop, each as one or two streaming kernels:
//   * multi-tensor Adam           (torch.optim.Adam(l, lr=0.0, eps=1e-15), scene/gaussian_model.py:189,
//                                  stepped at train.py:520-522)
//   * densification statistics    (train.py:489-491, scene/gaussian_model.py:693-695)
//   * image loss forward+backward (L1 + (1-SSIM) + masked depth L2; utils/loss_utils.py:20-96,
//                                  train.py:395-419)
// All of it is HBM-bound elementwise / stencil work: 16-byte accesses, no tensor cores.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "reduce.cuh"

namespace s3g {

// ---------------------------------------------------------------------------------------------
// Adam.  One launch updates every tensor of every param group: block b owns ADAM_CHUNK consecutive
// elements of one tensor (table lookup by binary search), 28 bytes of traffic per element.
// Arithmetic follows torch's _multi_tensor_adam (torch/optim/adam.py): exp_avg.lerp_(g, 1-b1);
// exp_avg_sq.mul_(b2).addcmul_(g, g, value=1-b2); denom = sqrt(exp_avg_sq)/sqrt(bc2) + eps;
// p.addcdiv_(exp_avg, denom, value=-lr/bc1).
// ---------------------------------------------------------------------------------------------
constexpr int ADAM_THREADS = 256;
constexpr int ADAM_VEC_PER_THREAD = 4;
constexpr int ADAM_CHUNK = ADAM_THREADS * ADAM_VEC_PER_THREAD * 4;   // 4096 elements per block
constexpr int ADAM_MAX_TENSORS = 40;

struct AdamTensor {
    float* p;
    const float* g;
    float* m;
    float* v;
    long long n;
    float step_size;      // lr / (1 - beta1^step)
    float bc2_sqrt;       // sqrt(1 - beta2^step)
};
struct AdamArgs {
    AdamTensor t[ADAM_MAX_TENSORS];
    int block_start[ADAM_MAX_TENSORS + 1];
    int count;
    float w1;             // 1 - beta1
    float beta2, omb2;    // beta2, 1 - beta2
    float eps;
};

__device__ __forceinline__ void adam_update(float& p, float g, float& m, float& v, float w1, float b2, float omb2,
                                            float eps, float step_size, float bc2_sqrt) {
    m = fmaf(w1, g - m, m);
    v = fmaf(omb2 * g, g, v * b2);
    const float denom = sqrtf(v) / bc2_sqrt + eps;
    p = p - step_size * (m / denom);
}

__global__ void __launch_bounds__(ADAM_THREADS) adam_multi_tensor_kernel(const __grid_constant__ AdamArgs a) {
    // which tensor does this block belong to?
    int lo = 0, hi = a.count;
    const int b = blockIdx.x;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (a.block_start[mid] <= b) lo = mid; else hi = mid;
    }
    const AdamTensor& t = a.t[lo];
    const long long base = (long long)(b - a.block_start[lo]) * ADAM_CHUNK;
    const float ss = t.step_size, bc = t.bc2_sqrt;
    const bool aligned = ((((uintptr_t)t.p) | ((uintptr_t)t.g) | ((uintptr_t)t.m) | ((uintptr_t)t.v)) & 15) == 0;
    if (aligned && base + ADAM_CHUNK <= t.n) {
        float4 P[ADAM_VEC_PER_THREAD], G[ADAM_VEC_PER_THREAD], M[ADAM_VEC_PER_THREAD], V[ADAM_VEC_PER_THREAD];
#pragma unroll
        for (int j = 0; j < ADAM_VEC_PER_THREAD; ++j) {
            const long long i = base + (long long)(j * ADAM_THREADS + threadIdx.x) * 4;
            G[j] = __ldcs(reinterpret_cast<const float4*>(t.g + i));
            P[j] = *reinterpret_cast<const float4*>(t.p + i);
            M[j] = *reinterpret_cast<const float4*>(t.m + i);
            V[j] = *reinterpret_cast<const float4*>(t.v + i);
        }
#pragma unroll
        for (int j = 0; j < ADAM_VEC_PER_THREAD; ++j) {
            adam_update(P[j].x, G[j].x, M[j].x, V[j].x, a.w1, a.beta2, a.omb2, a.eps, ss, bc);
            adam_update(P[j].y, G[j].y, M[j].y, V[j].y, a.w1, a.beta2, a.omb2, a.eps, ss, bc);
            adam_update(P[j].z, G[j].z, M[j].z, V[j].z, a.w1, a.beta2, a.omb2, a.eps, ss, bc);
            adam_update(P[j].w, G[j].w, M[j].w, V[j].w, a.w1, a.beta2, a.omb2, a.eps, ss, bc);
            const long long i = base + (long long)(j * ADAM_THREADS + threadIdx.x) * 4;
            *reinterpret_cast<float4*>(t.p + i) = P[j];
            *reinterpret_cast<float4*>(t.m + i) = M[j];
            *reinterpret_cast<float4*>(t.v + i) = V[j];
        }
    } else {
        const long long end = (base + ADAM_CHUNK < t.n) ? base + ADAM_CHUNK : t.n;
        for (long long i = base + threadIdx.x; i < end; i += ADAM_THREADS) {
            float p = t.p[i], m = t.m[i], v = t.v[i];
            adam_update(p, t.g[i], m, v, a.w1, a.beta2, a.omb2, a.eps, ss, bc);
            t.p[i] = p; t.m[i] = m; t.v[i] = v;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Selective Adam (upstream 3DGS --optimizer_type sparse_adam, Taming 3DGS, gsplat SelectiveAdam): the tensors with
// row_width[i] > 0 hold `rows` rows of row_width floats, and only the rows with visible[r] != 0 are updated; every
// other row keeps its parameter and both moments bit for bit, and its gradient is never read.  Tensors with
// row_width 0 get the dense update in the same launch.  Every updated element gets adam_multi_tensor_kernel's
// arithmetic and roundings (adam_update_exact), so an all-visible mask, and a dense tensor under any mask, equal the
// dense step bit for bit.
// Same chunking as the dense kernel, one float4 per thread at a time.  In a masked tensor each thread looks up the
// rows its float4 spans (at most 4; the mask is 1 byte per row and stays in L1 / L2) and skips a float4 with no
// visible row without touching p, g, m or v, so an invisible row costs no parameter, gradient or moment traffic
// beyond the sectors it shares with a visible one.  A float4 whose rows are all visible takes the vector path; one
// that mixes takes predicated scalar accesses, as does every element of a tensor that is not 16-byte aligned.
// ---------------------------------------------------------------------------------------------
struct AdamSelectiveArgs {
    AdamTensor t[ADAM_MAX_TENSORS];
    unsigned row_width[ADAM_MAX_TENSORS];     // 0: dense; masked tensors have n < 2^32
    int block_start[ADAM_MAX_TENSORS + 1];
    int count;
    float w1, beta2, omb2, eps;
    const unsigned char* visible;             // [rows]
};

// adam_update with every rounding spelled out.  ptxas contracts adam_update's last line, p - step_size * q, into one
// FFMA in some places of adam_multi_tensor_kernel and not in others: as compiled for sm_90a, the scalar path and the
// .w lane of the float4 path round once (fused), the .x, .y and .z lanes round the product and then the difference.
// Naming the rounding per element lets the selective kernel give every element the dense kernel's bits, whatever
// ptxas would choose here.
__device__ __forceinline__ void adam_update_exact(float& p, float g, float& m, float& v, float w1, float b2, float omb2,
                                                  float eps, float step_size, float bc2_sqrt, bool fused) {
    m = fmaf(w1, __fsub_rn(g, m), m);
    v = fmaf(__fmul_rn(omb2, g), g, __fmul_rn(v, b2));
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);
    const float q = __fdiv_rn(m, denom);
    p = fused ? fmaf(-step_size, q, p) : __fsub_rn(p, __fmul_rn(step_size, q));
}

__global__ void __launch_bounds__(ADAM_THREADS) adam_selective_kernel(const __grid_constant__ AdamSelectiveArgs a) {
    int lo = 0, hi = a.count;
    const int b = blockIdx.x;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (a.block_start[mid] <= b) lo = mid; else hi = mid;
    }
    const AdamTensor& t = a.t[lo];
    const unsigned w = a.row_width[lo];
    const unsigned char* __restrict__ vis = a.visible;
    const long long base = (long long)(b - a.block_start[lo]) * ADAM_CHUNK;
    const long long end = (base + ADAM_CHUNK < t.n) ? base + ADAM_CHUNK : t.n;
    const float ss = t.step_size, bc = t.bc2_sqrt;
    const bool aligned = ((((uintptr_t)t.p) | ((uintptr_t)t.g) | ((uintptr_t)t.m) | ((uintptr_t)t.v)) & 15) == 0;
    const bool dense_vec = aligned && base + ADAM_CHUNK <= t.n;     // the dense kernel's float4 path takes this chunk
    if (aligned) {
        // the mask bytes of all four float4s first, so their latency is paid once and not before each float4
        unsigned any = 0xfu, all = 0xfu;
        if (w != 0) {
            any = all = 0u;
#pragma unroll
            for (int j = 0; j < ADAM_VEC_PER_THREAD; ++j) {
                const long long i = base + (long long)(j * ADAM_THREADS + threadIdx.x) * 4;
                if (i >= end) break;
                const long long last = i + 3 < end ? i + 3 : end - 1;
                bool a_ = false, b_ = true;
                for (unsigned r = (unsigned)i / w, r1 = (unsigned)last / w; r <= r1; ++r) {
                    const bool s = __ldg(vis + r) != 0;
                    a_ |= s;
                    b_ &= s;
                }
                any |= (unsigned)a_ << j;
                all |= (unsigned)b_ << j;
            }
        }
        for (int j = 0; j < ADAM_VEC_PER_THREAD; ++j) {
            const long long i = base + (long long)(j * ADAM_THREADS + threadIdx.x) * 4;
            if (i >= end) break;
            const long long last = i + 3 < end ? i + 3 : end - 1;
            if (!((any >> j) & 1u)) continue;
            if (((all >> j) & 1u) && last == i + 3) {
                const float4 G = __ldcs(reinterpret_cast<const float4*>(t.g + i));
                float4 P = *reinterpret_cast<const float4*>(t.p + i);
                float4 M = *reinterpret_cast<const float4*>(t.m + i);
                float4 V = *reinterpret_cast<const float4*>(t.v + i);
                adam_update_exact(P.x, G.x, M.x, V.x, a.w1, a.beta2, a.omb2, a.eps, ss, bc, !dense_vec);
                adam_update_exact(P.y, G.y, M.y, V.y, a.w1, a.beta2, a.omb2, a.eps, ss, bc, !dense_vec);
                adam_update_exact(P.z, G.z, M.z, V.z, a.w1, a.beta2, a.omb2, a.eps, ss, bc, !dense_vec);
                adam_update_exact(P.w, G.w, M.w, V.w, a.w1, a.beta2, a.omb2, a.eps, ss, bc, true);
                *reinterpret_cast<float4*>(t.p + i) = P;
                *reinterpret_cast<float4*>(t.m + i) = M;
                *reinterpret_cast<float4*>(t.v + i) = V;
                continue;
            }
            for (long long e = i; e <= last; ++e) {
                if (w != 0 && !__ldg(vis + (unsigned)e / w)) continue;
                float p = t.p[e], m = t.m[e], v = t.v[e];
                adam_update_exact(p, t.g[e], m, v, a.w1, a.beta2, a.omb2, a.eps, ss, bc, !dense_vec || (e & 3) == 3);
                t.p[e] = p; t.m[e] = m; t.v[e] = v;
            }
        }
    } else {
        for (long long e = base + threadIdx.x; e < end; e += ADAM_THREADS) {
            if (w != 0 && !__ldg(vis + (unsigned)e / w)) continue;
            float p = t.p[e], m = t.m[e], v = t.v[e];
            adam_update_exact(p, t.g[e], m, v, a.w1, a.beta2, a.omb2, a.eps, ss, bc, true);
            t.p[e] = p; t.m[e] = m; t.v[e] = v;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Densification statistics (train.py:489-491 + GaussianModel.add_densification_stats):
//   vis = radii > 0 ; max_radii2D[vis] = max(max_radii2D[vis], radii[vis]) ;
//   xyz_gradient_accum[vis] += |viewspace_grad[vis, :2]| ; denom[vis] += 1
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) densify_stats_kernel(int P, const float* __restrict__ vgrad,
                                                           const int* __restrict__ radii, float* __restrict__ accum,
                                                           float* __restrict__ denom, float* __restrict__ max_radii) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int r = radii[i];
    if (r <= 0) return;
    const float gx = vgrad[3 * (size_t)i], gy = vgrad[3 * (size_t)i + 1];
    accum[i] += sqrtf(gx * gx + gy * gy);
    denom[i] += 1.0f;
    max_radii[i] = fmaxf(max_radii[i], (float)r);
}

// densify_stats_kernel plus the absolute-gradient statistic (AbsGS, gsplat absgrad) in the same pass:
//   xyz_gradient_accum_abs[vis] += |viewspace_absgrad[vis]|   (absgrad f32[P,2])
__global__ void __launch_bounds__(256) densify_stats_abs_kernel(int P, const float* __restrict__ vgrad,
                                                               const float* __restrict__ vabs,
                                                               const int* __restrict__ radii, float* __restrict__ accum,
                                                               float* __restrict__ accum_abs,
                                                               float* __restrict__ denom,
                                                               float* __restrict__ max_radii) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int r = radii[i];
    if (r <= 0) return;
    const float gx = vgrad[3 * (size_t)i], gy = vgrad[3 * (size_t)i + 1];
    const float ax = vabs[2 * (size_t)i], ay = vabs[2 * (size_t)i + 1];
    accum[i] += sqrtf(gx * gx + gy * gy);
    accum_abs[i] += sqrtf(ax * ax + ay * ay);
    denom[i] += 1.0f;
    max_radii[i] = fmaxf(max_radii[i], (float)r);
}

// ---------------------------------------------------------------------------------------------
// Image loss terms {mean|x - y|, mean(ssim_map(x, y)), depth_l2} and their gradients,
// with the reference's SSIM (11x11 Gaussian window sigma 1.5, zero padding, C1 = 0.01^2, C2 = 0.03^2,
// loss_utils.py:56-96) and depth_l2 = mean over valid pixels (0.01 < gt < max_depth) of
// (clamp(pred/max_depth,0,1) - clamp(gt/max_depth,0,1))^2 (loss_utils.py:20-45).
//
// Pass 1 (loss_stats_kernel): one 32x32 tile per block and (image, channel) plane; the five window
// moments come from a separable 11-tap filter in shared memory; writes the three SSIM derivative
// maps and per-block partial sums {sum|x-y|, sum ssim, sum depth sq err, #valid}.
// Pass 2 (loss_grad_kernel): filters the derivative maps with the same (symmetric) window and writes
// dL/dx; the depth gradient is elementwise.  Between the passes only the partial sums are reduced
// (loss_reduce_kernel) - the valid-pixel count normalises the depth gradient.
// ---------------------------------------------------------------------------------------------
constexpr int LOSS_T = 32;             // tile edge
constexpr int LOSS_HALO = 5;
constexpr int LOSS_W = LOSS_T + 2 * LOSS_HALO; // 42
constexpr int LOSS_THREADS = 256;

struct LossWin { float w[11]; };
static_assert(LOSS_THREADS == 256, "block_sum_256 reduces 256-thread blocks");

// x, y: [planes][H][W] (planes = B*3).  maps: 3 x [planes][H][W].  partial: [blocks][4]
__global__ void __launch_bounds__(LOSS_THREADS) loss_stats_kernel(int H, int W, const float* __restrict__ x,
                                                                 const float* __restrict__ y, LossWin win,
                                                                 float* __restrict__ dm_dmu1,
                                                                 float* __restrict__ dm_dsig1,
                                                                 float* __restrict__ dm_dsig12,
                                                                 float* __restrict__ partial) {
    __shared__ float sx[LOSS_W][LOSS_W + 1], sy[LOSS_W][LOSS_W + 1];
    __shared__ float h[5][LOSS_W][LOSS_T + 1];
    __shared__ float red[8];
    const int plane = blockIdx.z;
    const int x0 = blockIdx.x * LOSS_T, y0 = blockIdx.y * LOSS_T;
    const float* px = x + (size_t)plane * H * W;
    const float* py = y + (size_t)plane * H * W;
    for (int e = threadIdx.x; e < LOSS_W * LOSS_W; e += LOSS_THREADS) {
        const int r = e / LOSS_W, c = e - r * LOSS_W;
        const int gy = y0 + r - LOSS_HALO, gx = x0 + c - LOSS_HALO;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
        sx[r][c] = in ? __ldg(px + (size_t)gy * W + gx) : 0.f;
        sy[r][c] = in ? __ldg(py + (size_t)gy * W + gx) : 0.f;
    }
    __syncthreads();
    // horizontal pass: LOSS_W rows x LOSS_T columns
    for (int e = threadIdx.x; e < LOSS_W * LOSS_T; e += LOSS_THREADS) {
        const int r = e / LOSS_T, c = e - r * LOSS_T;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, a4 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float xv = sx[r][c + k], yv = sy[r][c + k], w = win.w[k];
            a0 = fmaf(w, xv, a0); a1 = fmaf(w, yv, a1);
            a2 = fmaf(w, xv * xv, a2); a3 = fmaf(w, yv * yv, a3); a4 = fmaf(w, xv * yv, a4);
        }
        h[0][r][c] = a0; h[1][r][c] = a1; h[2][r][c] = a2; h[3][r][c] = a3; h[4][r][c] = a4;
    }
    __syncthreads();
    float s_l1 = 0.f, s_ssim = 0.f;
    for (int e = threadIdx.x; e < LOSS_T * LOSS_T; e += LOSS_THREADS) {
        const int r = e / LOSS_T, c = e - r * LOSS_T;
        const int gy = y0 + r, gx = x0 + c;
        if (gy >= H || gx >= W) continue;
        float mu1 = 0.f, mu2 = 0.f, s11 = 0.f, s22 = 0.f, s12 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float w = win.w[k];
            mu1 = fmaf(w, h[0][r + k][c], mu1); mu2 = fmaf(w, h[1][r + k][c], mu2);
            s11 = fmaf(w, h[2][r + k][c], s11); s22 = fmaf(w, h[3][r + k][c], s22);
            s12 = fmaf(w, h[4][r + k][c], s12);
        }
        const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
        const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
        const float sig1 = s11 - mu1_sq, sig2 = s22 - mu2_sq, sig12 = s12 - mu12;
        const float A = 2.f * mu12 + C1, B = 2.f * sig12 + C2;
        const float C = mu1_sq + mu2_sq + C1, D = sig1 + sig2 + C2;
        const float inv_cd = 1.f / (C * D);
        s_ssim += A * B * inv_cd;
        const size_t o = (size_t)plane * H * W + (size_t)gy * W + gx;
        dm_dmu1[o] = 2.f * inv_cd * (mu2 * (B - A) - mu1 * A * B / C + mu1 * A * B / D);
        dm_dsig1[o] = -A * B * inv_cd / D;
        dm_dsig12[o] = 2.f * A * inv_cd;
        s_l1 += fabsf(sx[r + LOSS_HALO][c + LOSS_HALO] - sy[r + LOSS_HALO][c + LOSS_HALO]);
    }
    const int bid = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    const float t1 = block_sum_256(s_l1, red);
    if (threadIdx.x == 0) partial[(size_t)bid * 2 + 0] = t1;
    const float t2 = block_sum_256(s_ssim, red);
    if (threadIdx.x == 0) partial[(size_t)bid * 2 + 1] = t2;
}

// L1 term only (lambda_dssim == 0: train.py:417 skips SSIM then): partial[b] = {sum|x-y|, 0}; n = B*C*H*W
__global__ void __launch_bounds__(LOSS_THREADS) loss_l1_stats_kernel(size_t n, const float* __restrict__ x,
                                                                    const float* __restrict__ y,
                                                                    float* __restrict__ partial) {
    __shared__ float red[8];
    float s = 0.f;
    const size_t n4 = n / 4;
    const float4* x4 = reinterpret_cast<const float4*>(x);
    const float4* y4 = reinterpret_cast<const float4*>(y);
    const bool vec = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
    if (vec) {
        for (size_t i = (size_t)blockIdx.x * LOSS_THREADS + threadIdx.x; i < n4; i += (size_t)gridDim.x * LOSS_THREADS) {
            const float4 a = __ldg(x4 + i), b = __ldg(y4 + i);
            s += fabsf(a.x - b.x) + fabsf(a.y - b.y) + fabsf(a.z - b.z) + fabsf(a.w - b.w);
        }
        for (size_t i = n4 * 4 + (size_t)blockIdx.x * LOSS_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * LOSS_THREADS)
            s += fabsf(x[i] - y[i]);
    } else {
        for (size_t i = (size_t)blockIdx.x * LOSS_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * LOSS_THREADS)
            s += fabsf(x[i] - y[i]);
    }
    const float t1 = block_sum_256(s, red);
    if (threadIdx.x == 0) { partial[(size_t)blockIdx.x * 2 + 0] = t1; partial[(size_t)blockIdx.x * 2 + 1] = 0.f; }
}
// dL/dx = wts[0]/N * sign(x-y)
__global__ void __launch_bounds__(256) loss_l1_grad_kernel(size_t n, const float* __restrict__ x, const float* __restrict__ y,
                                                          const float* __restrict__ wts, float invN, float* __restrict__ g) {
    const float k = __ldg(wts) * invN;
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const float d = x[i] - y[i];
    g[i] = d > 0.f ? k : (d < 0.f ? -k : 0.f);
}

// depth term statistics: partial[b] = {sum sq err over valid, #valid}; n = B*H*W
__global__ void __launch_bounds__(LOSS_THREADS) loss_depth_stats_kernel(size_t n, const float* __restrict__ pred,
                                                                       const float* __restrict__ gt, float max_depth,
                                                                       float* __restrict__ partial) {
    __shared__ float red[8];
    float s = 0.f, c = 0.f;
    for (size_t i = (size_t)blockIdx.x * LOSS_THREADS + threadIdx.x; i < n; i += (size_t)gridDim.x * LOSS_THREADS) {
        const float g = gt[i];
        if (g > 0.01f && g < max_depth) {
            const float a = fminf(fmaxf(pred[i] / max_depth, 0.f), 1.f);
            const float b = fminf(fmaxf(g / max_depth, 0.f), 1.f);
            s += (a - b) * (a - b);
            c += 1.f;
        }
    }
    const float t1 = block_sum_256(s, red);
    if (threadIdx.x == 0) partial[(size_t)blockIdx.x * 2 + 0] = t1;
    const float t2 = block_sum_256(c, red);
    if (threadIdx.x == 0) partial[(size_t)blockIdx.x * 2 + 1] = t2;
}

// sums[0..3] = {sum|x-y|, sum ssim, sum depth sq err, #valid depth}; one block, double accumulation
__global__ void __launch_bounds__(256) loss_reduce_kernel(int n_img, const float* __restrict__ p_img, int n_dep,
                                                         const float* __restrict__ p_dep, double* __restrict__ sums) {
    __shared__ double red[4][256];
    double a[4] = {0.0, 0.0, 0.0, 0.0};
    for (int i = threadIdx.x; i < n_img; i += 256) { a[0] += p_img[2 * (size_t)i]; a[1] += p_img[2 * (size_t)i + 1]; }
    for (int i = threadIdx.x; i < n_dep; i += 256) { a[2] += p_dep[2 * (size_t)i]; a[3] += p_dep[2 * (size_t)i + 1]; }
#pragma unroll
    for (int k = 0; k < 4; ++k) red[k][threadIdx.x] = a[k];
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) {
#pragma unroll
            for (int k = 0; k < 4; ++k) red[k][threadIdx.x] += red[k][threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x < 4) sums[threadIdx.x] = red[threadIdx.x][0];
}

// dL/dx = wts[0]/N * sign(x-y) + wts[1]/N * [ conv(dm_dmu1) + 2 x conv(dm_dsig1) + y conv(dm_dsig12) ]
// wts (device) = dL/d{mean|x-y|, mean ssim, depth_l2}: the upstream gradients autograd hands to backward.
__global__ void __launch_bounds__(LOSS_THREADS) loss_grad_kernel(int H, int W, const float* __restrict__ x,
                                                                const float* __restrict__ y, LossWin win,
                                                                const float* __restrict__ dm_dmu1,
                                                                const float* __restrict__ dm_dsig1,
                                                                const float* __restrict__ dm_dsig12,
                                                                const float* __restrict__ wts, float invN,
                                                                float* __restrict__ gx_out) {
    const float k_l1 = __ldg(wts) * invN, k_ssim = __ldg(wts + 1) * invN;
    __shared__ float s[3][LOSS_W][LOSS_W + 1];
    __shared__ float h[3][LOSS_W][LOSS_T + 1];
    const int plane = blockIdx.z;
    const int x0 = blockIdx.x * LOSS_T, y0 = blockIdx.y * LOSS_T;
    const size_t pb = (size_t)plane * H * W;
    for (int e = threadIdx.x; e < LOSS_W * LOSS_W; e += LOSS_THREADS) {
        const int r = e / LOSS_W, c = e - r * LOSS_W;
        const int gy = y0 + r - LOSS_HALO, gx = x0 + c - LOSS_HALO;
        const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
        const size_t o = pb + (size_t)gy * W + gx;
        s[0][r][c] = in ? __ldg(dm_dmu1 + o) : 0.f;
        s[1][r][c] = in ? __ldg(dm_dsig1 + o) : 0.f;
        s[2][r][c] = in ? __ldg(dm_dsig12 + o) : 0.f;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < LOSS_W * LOSS_T; e += LOSS_THREADS) {
        const int r = e / LOSS_T, c = e - r * LOSS_T;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float w = win.w[k];
            a0 = fmaf(w, s[0][r][c + k], a0); a1 = fmaf(w, s[1][r][c + k], a1); a2 = fmaf(w, s[2][r][c + k], a2);
        }
        h[0][r][c] = a0; h[1][r][c] = a1; h[2][r][c] = a2;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < LOSS_T * LOSS_T; e += LOSS_THREADS) {
        const int r = e / LOSS_T, c = e - r * LOSS_T;
        const int gy = y0 + r, gx = x0 + c;
        if (gy >= H || gx >= W) continue;
        float c0 = 0.f, c1 = 0.f, c2 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float w = win.w[k];
            c0 = fmaf(w, h[0][r + k][c], c0); c1 = fmaf(w, h[1][r + k][c], c1); c2 = fmaf(w, h[2][r + k][c], c2);
        }
        const size_t o = pb + (size_t)gy * W + gx;
        const float xv = __ldg(x + o), yv = __ldg(y + o);
        const float d = xv - yv;
        const float sgn = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
        gx_out[o] = k_l1 * sgn + k_ssim * (c0 + 2.f * xv * c1 + yv * c2);
    }
}

// dL/dpred_depth = wts[2] * 2 (a - b) / (max_depth * #valid) inside the clamp, 0 elsewhere
__global__ void __launch_bounds__(256) loss_depth_grad_kernel(size_t n, const float* __restrict__ pred,
                                                             const float* __restrict__ gt, float max_depth,
                                                             const float* __restrict__ wts,
                                                             const double* __restrict__ sums,
                                                             float* __restrict__ g_out) {
    const float w_depth = __ldg(wts + 2);
    const size_t i = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const double cnt = sums[3];
    const float g = gt[i];
    float r = 0.f;
    if (cnt > 0.0 && g > 0.01f && g < max_depth) {
        const float q = pred[i] / max_depth;
        if (q >= 0.f && q <= 1.f) {     // torch.clamp backward passes the gradient on the closed interval
            const float b = fminf(fmaxf(g / max_depth, 0.f), 1.f);
            r = (float)((double)w_depth * 2.0 * (double)(q - b) / ((double)max_depth * cnt));
        }
    }
    g_out[i] = r;
}

// ---------------------------------------------------------------------------------------------
// HexPlane regularisers (GaussianModel.compute_regulation, scene/gaussian_model.py:710-749 with
// compute_plane_smoothness of scene/regulation.py:22-28):
//   total = sum over planes of  w_smooth * mean((t[h+2] - 2 t[h+1] + t[h])^2)  +  w_l1 * mean|1 - t|
// (second difference along dim 2 of the [1,C,H,W] tensor; w_smooth = plane_tv_weight on the spatial
// planes 0,1,3 and time_smoothness_weight on the time planes 2,4,5, which also carry the L1 term).
// Planes live channels-last ([H][W][C], the layout the sampling kernels use), so a step along H is a
// stride of W*C floats and every access below is a coalesced float4.  Forward = one read pass with
// per-block partial sums; backward = one read pass (5-tap stencil of the fourth difference) + one write.
// ---------------------------------------------------------------------------------------------
constexpr int REG_THREADS = 256;
constexpr int REG_VEC = 4;
constexpr int REG_CHUNK4 = REG_THREADS * REG_VEC;      // float4 elements per block
constexpr int REG_MAX_PLANES = 48;

struct RegPlane {
    const float* t;
    float* g;
    int H, W, C;
    float k_smooth;     // w_smooth / (C (H-2) W)
    float k_l1;         // w_l1 / (C H W)
};
struct RegArgs {
    RegPlane p[REG_MAX_PLANES];
    int block_start[REG_MAX_PLANES + 1];
    int count;
};

__device__ __forceinline__ int reg_find(const RegArgs& a, int b) {
    int lo = 0, hi = a.count;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (a.block_start[mid] <= b) lo = mid; else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ float4 ld4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 sd4(float4 a, float4 b, float4 c) {   // a - 2b + c
    return make_float4(a.x - 2.f * b.x + c.x, a.y - 2.f * b.y + c.y, a.z - 2.f * b.z + c.z, a.w - 2.f * b.w + c.w);
}

__global__ void __launch_bounds__(REG_THREADS) plane_reg_forward_kernel(const __grid_constant__ RegArgs a,
                                                                       double* __restrict__ partial) {
    __shared__ double red[REG_THREADS / 32];
    const int pi = reg_find(a, blockIdx.x);
    const RegPlane& pl = a.p[pi];
    const long long row4 = (long long)pl.W * pl.C / 4;          // float4 per H step
    const long long n4 = row4 * pl.H;
    const long long base = (long long)(blockIdx.x - a.block_start[pi]) * REG_CHUNK4;
    float s_sm = 0.f, s_l1 = 0.f;
#pragma unroll
    for (int j = 0; j < REG_VEC; ++j) {
        const long long i = base + j * REG_THREADS + threadIdx.x;
        if (i >= n4) continue;
        const int h = (int)(i / row4);
        const float4 t0 = ld4(pl.t + 4 * i);
        if (pl.k_l1 != 0.f) s_l1 += fabsf(1.f - t0.x) + fabsf(1.f - t0.y) + fabsf(1.f - t0.z) + fabsf(1.f - t0.w);
        if (h + 2 < pl.H) {
            const float4 d = sd4(t0, ld4(pl.t + 4 * (i + row4)), ld4(pl.t + 4 * (i + 2 * row4)));
            s_sm += d.x * d.x + d.y * d.y + d.z * d.z + d.w * d.w;
        }
    }
    double v = (double)s_sm * (double)pl.k_smooth + (double)s_l1 * (double)pl.k_l1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < REG_THREADS / 32; ++w) t += red[w];
        partial[blockIdx.x] = t;
    }
}

__global__ void __launch_bounds__(256) plane_reg_reduce_kernel(int n, const double* __restrict__ partial,
                                                              double* __restrict__ total) {
    __shared__ double red[256];
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 256) s += partial[i];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) total[0] = red[0];
}

// grad[h] = gscale * ( 2 k_smooth (d[h-2] - 2 d[h-1] + d[h]) - k_l1 sign(1 - t[h]) ),  d[j] = t[j] - 2 t[j+1] + t[j+2]
// for 0 <= j <= H-3 and 0 elsewhere.
__global__ void __launch_bounds__(REG_THREADS) plane_reg_backward_kernel(const __grid_constant__ RegArgs a,
                                                                        const float* __restrict__ gscale) {
    const int pi = reg_find(a, blockIdx.x);
    const RegPlane& pl = a.p[pi];
    const long long row4 = (long long)pl.W * pl.C / 4;
    const long long n4 = row4 * pl.H;
    const long long base = (long long)(blockIdx.x - a.block_start[pi]) * REG_CHUNK4;
    const float gs = __ldg(gscale);
    const float ks = 2.f * pl.k_smooth * gs, kl = pl.k_l1 * gs;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int j = 0; j < REG_VEC; ++j) {
        const long long i = base + j * REG_THREADS + threadIdx.x;
        if (i >= n4) continue;
        const int h = (int)(i / row4);
        const int H = pl.H;
        const float* c = pl.t + 4 * i;
        const float4 t0 = ld4(c);
        const float4 tm2 = h >= 2 ? ld4(c - 8 * row4) : z, tm1 = h >= 1 ? ld4(c - 4 * row4) : z;
        const float4 tp1 = h + 1 < H ? ld4(c + 4 * row4) : z, tp2 = h + 2 < H ? ld4(c + 8 * row4) : z;
        // d[h-2] exists if h-2 >= 0 (and h <= H-1 always holds for its last tap); d[h-1] if h-1 >= 0 and h+1 <= H-1;
        // d[h] if h+2 <= H-1
        const float4 dm2 = h >= 2 ? sd4(tm2, tm1, t0) : z;
        const float4 dm1 = (h >= 1 && h + 1 < H) ? sd4(tm1, t0, tp1) : z;
        const float4 d0 = (h + 2 < H) ? sd4(t0, tp1, tp2) : z;
        float4 g = sd4(dm2, dm1, d0);
        g.x *= ks; g.y *= ks; g.z *= ks; g.w *= ks;
        if (kl != 0.f) {
            g.x -= kl * (t0.x < 1.f ? 1.f : (t0.x > 1.f ? -1.f : 0.f));
            g.y -= kl * (t0.y < 1.f ? 1.f : (t0.y > 1.f ? -1.f : 0.f));
            g.z -= kl * (t0.z < 1.f ? 1.f : (t0.z > 1.f ? -1.f : 0.f));
            g.w -= kl * (t0.w < 1.f ? 1.f : (t0.w > 1.f ? -1.f : 0.f));
        }
        *reinterpret_cast<float4*>(pl.g + 4 * i) = g;
    }
}

// ---------------------------------------------------------------------------------------------
// Row gather for densify / prune (scene/gaussian_model.py:411-470: _prune_optimizer,
// cat_tensors_to_optimizer, prune_points, densification_postfix).  The reference rebuilds each of the six
// per-Gaussian parameters and their two Adam moments with boolean indexing + torch.cat, one tensor at a
// time (~60 launches and as many temporaries).  Here every tensor is rebuilt by ONE launch:
//   dst_t[r] = src_t[src_index[r]]                         for r < n_kept, and for parameters
//   dst_t[r] = 0                                           for r >= n_kept when t is optimizer state
// (rows >= n_kept are the appended clones / split children, whose moments start at zero).
// ---------------------------------------------------------------------------------------------
constexpr int ROWS_MAX_TENSORS = 32;
struct RowTensor {
    const float* src;
    float* dst;
    int row_floats;
    int zero_new;
};
struct RowArgs {
    RowTensor t[ROWS_MAX_TENSORS];
    int count;
    long long n_out, n_kept;
    const long long* src_index;
};

__global__ void __launch_bounds__(256) gather_rows_kernel(const __grid_constant__ RowArgs a) {
    const RowTensor& t = a.t[blockIdx.y];
    const long long total = a.n_out * t.row_floats;
    for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < total; e += (long long)gridDim.x * 256) {
        const long long r = e / t.row_floats;
        const int c = (int)(e - r * t.row_floats);
        float v = 0.f;
        if (r < a.n_kept || !t.zero_new) v = __ldg(t.src + __ldg(a.src_index + r) * t.row_floats + c);
        t.dst[e] = v;
    }
}

}  // namespace s3g
