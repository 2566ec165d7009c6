// filter3d.cuh - Mip-Splatting's 3-D smoothing filter (include/s3g_b200.h, "3-D smoothing filter"): each Gaussian's
// sampling-rate bound from the training cameras, and the filter applied to the activated scales and opacities.
//
//   compute: filter3d_depth_kernel writes d_i (min camera-space z over the cameras that see Gaussian i, +inf for none)
//            into filter_3d, the max over seen Gaussians into ws[0] and the max focal_x into ws[1];
//            filter3d_fill_kernel then turns d_i into d_i / F * sqrt(0.2) in place.
//   apply:   filter3d_apply_forward_kernel / filter3d_apply_backward_kernel, one thread per Gaussian.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace s3g {

constexpr int F3D_BLOCK = 256;
constexpr int F3D_CHUNK = 64;            // cameras staged in shared memory at a time (8 KB)
constexpr float F3D_SQRT_VAR = 0.44721359549995793f;   // sqrt(0.2), Mip-Splatting's fixed variance in px^2

// One camera as the depth kernel reads it: rows 0..2 of the world-to-view matrix and the screen bounds in multiplied
// form (|x fx| <= hx z  <=>  -0.15 w <= x / z fx + w / 2 <= 1.15 w for z > 0).
struct F3dCam {
    double r0[4], r1[4], r2[4];
    double fx, fy, hx, hy;
};

// The camera-space mean is formed in double: in float32 the rounding of a 50-80 m world coordinate alone is ~1e-5 m,
// which moves the depth of a Gaussian a few metres from the camera by more than 1e-6 of itself and shifts the
// z > 0.2 / screen-edge decisions of points close to them.
__global__ void __launch_bounds__(F3D_BLOCK)
filter3d_depth_kernel(int P, const float* __restrict__ xyz, int C, const float* __restrict__ views,
                      const float* __restrict__ cams, float* __restrict__ depth, uint32_t* __restrict__ ws) {
    __shared__ F3dCam cam[F3D_CHUNK];
    __shared__ uint32_t block_max[2];
    const int i = blockIdx.x * F3D_BLOCK + threadIdx.x;
    double X = 0.0, Y = 0.0, Z = 0.0;
    if (i < P) {
        X = xyz[3 * i + 0];
        Y = xyz[3 * i + 1];
        Z = xyz[3 * i + 2];
    }
    if (threadIdx.x < 2) block_max[threadIdx.x] = 0u;
    float best = __int_as_float(0x7f800000);   // +inf: no camera sees it yet
    float focal = 0.f;                          // max focal_x over the cameras this thread staged (block 0 only)
    for (int c0 = 0; c0 < C; c0 += F3D_CHUNK) {
        const int n = min(F3D_CHUNK, C - c0);
        __syncthreads();
        for (int j = threadIdx.x; j < n; j += F3D_BLOCK) {
            const float* m = views + 16 * (c0 + j);
            const float* k = cams + 4 * (c0 + j);
            F3dCam& s = cam[j];
            for (int c = 0; c < 4; ++c) {       // m[k] = M[k % 4][k / 4]
                s.r0[c] = m[4 * c + 0];
                s.r1[c] = m[4 * c + 1];
                s.r2[c] = m[4 * c + 2];
            }
            s.fx = k[2];
            s.fy = k[3];
            s.hx = 0.65 * (double)k[0];
            s.hy = 0.65 * (double)k[1];
            focal = fmaxf(focal, k[2]);
        }
        __syncthreads();
        if (i < P) {
            for (int j = 0; j < n; ++j) {
                const F3dCam& s = cam[j];
                const double z = fma(s.r2[0], X, fma(s.r2[1], Y, fma(s.r2[2], Z, s.r2[3])));
                if (!(z > 0.2)) continue;
                const double x = fma(s.r0[0], X, fma(s.r0[1], Y, fma(s.r0[2], Z, s.r0[3])));
                const double y = fma(s.r1[0], X, fma(s.r1[1], Y, fma(s.r1[2], Z, s.r1[3])));
                if (fabs(x * s.fx) <= s.hx * z && fabs(y * s.fy) <= s.hy * z) best = fminf(best, (float)z);
            }
        }
    }
    // max of the seen depths (positive floats order like their bit patterns) and, in block 0, of focal_x:
    // per warp, per block in shared memory, then one global atomic per block - all order-independent
    const uint32_t seen = (i < P && best < __int_as_float(0x7f800000)) ? __float_as_uint(best) : 0u;
    const uint32_t wmax = __reduce_max_sync(0xffffffffu, seen);
    const uint32_t fmax = __reduce_max_sync(0xffffffffu, __float_as_uint(focal));
    if ((threadIdx.x & 31) == 0) {
        atomicMax(&block_max[0], wmax);
        atomicMax(&block_max[1], fmax);
    }
    if (i < P) depth[i] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        if (block_max[0] != 0u) atomicMax(&ws[0], block_max[0]);
        if (blockIdx.x == 0) ws[1] = block_max[1];
    }
}

__global__ void __launch_bounds__(F3D_BLOCK)
filter3d_fill_kernel(int P, float* __restrict__ filter, const uint32_t* __restrict__ ws) {
    const int i = blockIdx.x * F3D_BLOCK + threadIdx.x;
    if (i >= P) return;
    float d = filter[i];
    if (d == __int_as_float(0x7f800000)) d = __uint_as_float(ws[0]);   // unseen: the max over seen (0 if none)
    filter[i] = d / __uint_as_float(ws[1]) * F3D_SQRT_VAR;
}

// s' = sqrt(s^2 + f^2), o' = o * prod_k s_k / s'_k (= o sqrt(prod s^2 / prod s'^2), taken per axis so that no product of
// three squares under- or overflows; where f = 0 every ratio is exactly 1).
__global__ void __launch_bounds__(F3D_BLOCK)
filter3d_apply_forward_kernel(int P, const float* __restrict__ scales, const float* __restrict__ opacity,
                              const float* __restrict__ filter, float* __restrict__ out_scales,
                              float* __restrict__ out_opacity) {
    const int i = blockIdx.x * F3D_BLOCK + threadIdx.x;
    if (i >= P) return;
    const float f = filter[i];
    const float f2 = f * f;
    float q = 1.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float s = scales[3 * i + k];
        const float sf = sqrtf(s * s + f2);
        out_scales[3 * i + k] = sf;
        q *= s / sf;
    }
    out_opacity[i] = opacity[i] * q;
}

// dL/ds_k = g_s'_k s_k / s'_k + g_o' o' f^2 / (s_k s'_k^2), dL/do = g_o' prod_k s_k / s'_k.  The second term is formed
// as (f / s'_k)^2 / s_k and left out where f = 0, so there the gradients pass through bitwise (-0 included).
__global__ void __launch_bounds__(F3D_BLOCK)
filter3d_apply_backward_kernel(int P, const float* __restrict__ scales, const float* __restrict__ opacity,
                               const float* __restrict__ filter, const float* __restrict__ g_out_scales,
                               const float* __restrict__ g_out_opacity, float* __restrict__ g_scales,
                               float* __restrict__ g_opacity) {
    const int i = blockIdx.x * F3D_BLOCK + threadIdx.x;
    if (i >= P) return;
    const float f = filter[i];
    const float f2 = f * f;
    float s[3], sf[3], q = 1.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        s[k] = scales[3 * i + k];
        sf[k] = sqrtf(s[k] * s[k] + f2);
        q *= s[k] / sf[k];
    }
    const float go = g_out_opacity[i];
    const float go_o = go * (opacity[i] * q);      // g_o' o'
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float r = f / sf[k];
        float g = g_out_scales[3 * i + k] * (s[k] / sf[k]);
        if (f != 0.f) g += go_o * (r * r) / s[k];
        g_scales[3 * i + k] = g;
    }
    g_opacity[i] = go * q;
}

}  // namespace s3g
