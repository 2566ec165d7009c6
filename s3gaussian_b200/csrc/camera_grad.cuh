// camera_grad.cuh - gradients of the loss with respect to the camera (viewmatrix, projmatrix, campos) (sm_90a).
//
// A separate pass after the backward: it reads the per-Gaussian screen-space gradients the preprocess backward
// exported (dL_dmean2D, dL_dconic, dL_ddepth, dL_dcolor) and the forward's inputs, and applies the chain rule at the
// points where the camera enters the forward (preprocess.cuh):
//   p_hom = projmatrix x~          -> mean2D = p_hom.xy / (p_hom.w + 1e-7)
//   t     = viewmatrix x~          -> J(t) (with the 1.3 tanfov clamp), depth = t.z
//   W     = viewmatrix[:3,:3]      -> cov2D = J W Sigma W^T J^T + 0.3 I -> conic
//   dir   = x - campos             -> SH colour (the clamped mask zeroes a channel)
// The derivatives up to dL/dt, dL/d(J W) and dL/d(normalised dir) are preprocess_backward_kernel's own: load_cov3d,
// ewa_jacobian, cov2d_backward and sh_ddir in preprocess.cuh (the same zero gradient through the clamped components
// of t), so these gradients and the per-Gaussian ones describe the same function.  What is left here is the chain
// rule from those to the camera's entries.
//
// Summation order, fixed by P alone: each warp adds its 32 Gaussians' contributions with one xor butterfly in double
// and keeps a running sum per component over the block's CAM_ITERS rounds; a block adds its warps in warp order; the
// one-block finish kernel adds the block partials, lane b taking blocks b, b+32, ... in order, then one butterfly.
// One cast to float at the end.  No atomics.
#pragma once
#include "common.cuh"
#include "preprocess.cuh"

namespace s3g {

constexpr int CAM_THREADS = 128;
constexpr int CAM_ITERS = 8;                                // rounds of CAM_THREADS Gaussians per block
constexpr int CAM_GAUSS_PER_BLOCK = CAM_THREADS * CAM_ITERS;
// the summed components: viewmatrix storage entries 4c + r (r < 3) as 3c + r, then projmatrix entries 4c + r
// (r = 0, 1, 3) as 12 + 3c + {0, 1, 2}, then campos.  The rest are exact zeros: the forward never reads viewmatrix's
// fourth row, and mean2D does not depend on the third row of projmatrix.
constexpr int CAM_NCOMP = 27;

struct CamBwdArgs {
    int P, D, M;
    const float* means3D;
    const int* radii;
    const float* shs;          // read only when campos is asked for in SH mode
    const uint8_t* clamped;
    const float* scales;
    const float* rotations;
    float scale_modifier;
    const float* cov3D_precomp;
    const float* view;
    const float* proj;
    const float* campos;
    float focal_x, focal_y, tan_fovx, tan_fovy;
    const float* dL_dmean2D;   // [P,3]
    const float* dL_dconic;    // [P,4]
    const float* dL_ddepth;    // [P]
    const float* dL_dcolor;    // [P,3]
    double* partial;           // [CAM_NCOMP][nblocks]
    int nblocks;
    const float* grad_rec;     // AA only: the composite's records, [P][GRAD_REC], slot 5 = dL/dalpha_eff
    const float4* Cod;         // AA only: the forward's records, .y = alpha_eff
};

__host__ __device__ inline int camera_grad_blocks(int P) { return (int)div_up64(P, CAM_GAUSS_PER_BLOCK); }

// One visible Gaussian's contribution to the CAM_NCOMP components.  sh: its staged coefficient row when CAMPOS.
// AA: after an antialiased forward, whose opacity factor depends on the 2-D covariance and so on the camera.
template <bool CAMPOS, bool AA>
__device__ __forceinline__ void camera_contrib(const CamBwdArgs& a, const Cam& cam, int idx, const float* sh,
                                               float c[CAM_NCOMP]) {
    const float* view = cam.view;
    const float* proj = cam.proj;
    const float3 mean = {a.means3D[3 * idx], a.means3D[3 * idx + 1], a.means3D[3 * idx + 2]};
    float cov3D[6];
    float3 scl;
    float4 rot;
    load_cov3d(a, idx, cov3D, scl, rot);
    const float4 dconic = reinterpret_cast<const float4*>(a.dL_dconic)[idx];   // {x, y, 0, z}

    // ---- conic -> cov2D -> T = J W and t, as the preprocess backward ------------------------------------------------
    const EwaJacobian e = ewa_jacobian(a, mean, view);
    const Cov2dGrad g = cov2d_backward<AA>(a, e, cov3D, make_float3(dconic.x, dconic.y, dconic.w),
                                           AA ? a.Cod[idx].y * a.grad_rec[(size_t)idx * GRAD_REC + 5] : 0.f);
    const M3& J = e.J;
    // dT[k][j] = dL/d(J W)[k][j] (row k of the 2x3 product, column j): T.c[k][j] in the glm layout
    const float (&dT)[2][3] = g.dL_dT;
    // dL/dt, the depth term (depth = t.z) included
    const float dt[3] = {g.dL_dt.x, g.dL_dt.y, g.dL_dt.z + a.dL_ddepth[idx]};
    // viewmatrix entry 4c + r = V[r][c]: t_r = sum_c V[r][c] x~_c, and (J W)[k][c] = sum_r J[k][r] V[r][c] with
    // J[0] = (J.c[0][0], 0, J.c[0][2]), J[1] = (0, J.c[1][1], J.c[1][2])
    const float xt[4] = {mean.x, mean.y, mean.z, 1.f};
#pragma unroll
    for (int cc_ = 0; cc_ < 4; ++cc_) {
        const float w0 = cc_ < 3 ? dT[0][cc_] : 0.f, w1 = cc_ < 3 ? dT[1][cc_] : 0.f;
        c[3 * cc_ + 0] = dt[0] * xt[cc_] + w0 * J.c[0][0];
        c[3 * cc_ + 1] = dt[1] * xt[cc_] + w1 * J.c[1][1];
        c[3 * cc_ + 2] = dt[2] * xt[cc_] + w0 * J.c[0][2] + w1 * J.c[1][2];
    }

    // ---- mean2D = p_hom.xy / (p_hom.w + 1e-7): projmatrix entry 4c + r = P[r][c] ----------------------------------
    const float4 p_hom = xform4x4(mean, proj);
    const float m_w = 1.0f / (p_hom.w + 0.0000001f);
    const float gx = a.dL_dmean2D[3 * idx], gy = a.dL_dmean2D[3 * idx + 1];
    const float dp[3] = {gx * m_w, gy * m_w, -(gx * p_hom.x + gy * p_hom.y) * m_w * m_w};   // rows 0, 1, 3
#pragma unroll
    for (int cc_ = 0; cc_ < 4; ++cc_)
#pragma unroll
        for (int r = 0; r < 3; ++r) c[12 + 3 * cc_ + r] = dp[r] * xt[cc_];

    // ---- SH colour through dir = x - campos ---------------------------------------------------------------------------
    if (CAMPOS) {
        const float3 dir_orig = {mean.x - cam.campos[0], mean.y - cam.campos[1], mean.z - cam.campos[2]};
        const float len = sqrtf(dir_orig.x * dir_orig.x + dir_orig.y * dir_orig.y + dir_orig.z * dir_orig.z);
        const uint8_t cl = a.clamped[idx];
        const float* dcol = a.dL_dcolor + 3 * idx;
        const float dRGB[3] = {(cl & 1) ? 0.f : dcol[0], (cl & 2) ? 0.f : dcol[1], (cl & 4) ? 0.f : dcol[2]};
        const float3 dm =
            dnormvdv3(dir_orig, sh_ddir(a.D, dir_orig.x / len, dir_orig.y / len, dir_orig.z / len, sh, dRGB));
        c[24] = -dm.x;
        c[25] = -dm.y;
        c[26] = -dm.z;
    } else {
        c[24] = c[25] = c[26] = 0.f;
    }
}

// Block b sums Gaussians [b * CAM_GAUSS_PER_BLOCK, (b + 1) * CAM_GAUSS_PER_BLOCK) into partial[k][b].
template <int MT, bool CAMPOS, bool AA = false>   // MT = 16: SH rows of 48 floats known at compile time; 0: runtime M
__global__ void __launch_bounds__(CAM_THREADS) camera_grad_partial_kernel(const __grid_constant__ CamBwdArgs a) {
    extern __shared__ float s_dyn[];
    __shared__ Cam s_cam;
    __shared__ double s_warp[CAM_THREADS / 32][CAM_NCOMP];
    load_cam(s_cam, a.view, a.proj, a.campos);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int L = 3 * (MT > 0 ? MT : a.M);
    float* rows = s_dyn + warp * 32 * row_stride(L);
    double acc = 0.0;   // lane k < CAM_NCOMP: the warp's running sum of component k
    for (int it = 0; it < CAM_ITERS; ++it) {
        const int idx = blockIdx.x * CAM_GAUSS_PER_BLOCK + it * CAM_THREADS + threadIdx.x;
        const int first = idx - lane;
        if (first >= a.P) break;   // warp-uniform
        const bool visible = idx < a.P && a.radii[idx] > 0;
        if (!__any_sync(0xffffffffu, visible)) continue;
        if (CAMPOS) {
            __syncwarp();   // the previous round's reads of the rows are done
            warp_rows_in<3 * MT>(a.shs + (size_t)first * L, rows, L, min(32, a.P - first), lane);
            __syncwarp();
        }
        float c[CAM_NCOMP];
        if (visible) {
            camera_contrib<CAMPOS, AA>(a, s_cam, idx, rows + lane * row_stride(L), c);
        } else {
#pragma unroll
            for (int k = 0; k < CAM_NCOMP; ++k) c[k] = 0.f;
        }
#pragma unroll
        for (int k = 0; k < CAM_NCOMP; ++k) {
            double v = (double)c[k];
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
            if (lane == k) acc += v;
        }
    }
    if (lane < CAM_NCOMP) s_warp[warp][lane] = acc;
    __syncthreads();
    if (threadIdx.x < CAM_NCOMP) {
        double s = 0.0;
#pragma unroll
        for (int w = 0; w < CAM_THREADS / 32; ++w) s += s_warp[w][threadIdx.x];
        a.partial[(size_t)threadIdx.x * a.nblocks + blockIdx.x] = s;
    }
}

// One block of CAM_NCOMP warps: warp k sums component k over the block partials, then the 35 outputs are written
// (exact zeros at the entries listed above CAM_NCOMP).
__global__ void __launch_bounds__(32 * CAM_NCOMP)
camera_grad_finish_kernel(const double* __restrict__ partial, int nblocks, float* __restrict__ dL_dview,
                          float* __restrict__ dL_dproj, float* __restrict__ dL_dcampos) {
    __shared__ double s_sum[CAM_NCOMP];
    const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double s = 0.0;
    for (int b = lane; b < nblocks; b += 32) s += partial[(size_t)k * nblocks + b];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) s_sum[k] = s;
    __syncthreads();
    const int t = threadIdx.x;
    if (t < 16) {
        const int r = t & 3, col = t >> 2;
        if (dL_dview) dL_dview[t] = r == 3 ? 0.f : (float)s_sum[3 * col + r];
    } else if (t < 32) {
        const int e = t - 16, r = e & 3, col = e >> 2;
        if (dL_dproj) dL_dproj[e] = r == 2 ? 0.f : (float)s_sum[12 + 3 * col + (r == 3 ? 2 : r)];
    } else if (t < 35) {
        if (dL_dcampos) dL_dcampos[t - 32] = (float)s_sum[24 + t - 32];
    }
}

}  // namespace s3g
