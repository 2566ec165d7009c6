// preprocess.cuh - per-Gaussian forward and backward kernels (sm_90a).
//
// Forward replaces checkFrustum + preprocessCUDA (DGR/cuda_rasterizer/
// rasterizer_impl.cu:54-66, forward.cu:155-256 with computeCov3D :118-152,
// computeCov2D :74-113, computeColorFromSH :20-71, auxiliary.h:41-77,139-164).
// Backward replaces computeCov2DCUDA + preprocessCUDA (backward.cu:144-274,
// :346-412 with computeColorFromSH :20-139 and computeCov3D :278-341) as ONE
// kernel that also writes the zeros the reference glue memsets
// (rasterize_points.cu:154-163).
//
// Bit-exactness: radii / tile rects / depth keys feed integer outputs that must
// equal the reference's, so the forward keeps the reference's expression trees
// (operand order, IEEE div/sqrt, double-precision ndc2Pix) and lets nvcc apply
// its default FMA contraction to the same trees.  The 3x3 helper below restates
// the column-major product order of the vendored glm
// (third_party/glm/glm/detail/type_mat3x3.inl:486-518) - it is not glm.
#pragma once
#include "common.cuh"

namespace s3g {

// column-major 3x3: c[col][row]
struct M3 {
    float c[3][3];
};
__device__ __forceinline__ M3 m3(float a0, float a1, float a2, float b0, float b1, float b2,
                                  float c0, float c1, float c2) {
    M3 m;
    m.c[0][0] = a0; m.c[0][1] = a1; m.c[0][2] = a2;
    m.c[1][0] = b0; m.c[1][1] = b1; m.c[1][2] = b2;
    m.c[2][0] = c0; m.c[2][1] = c1; m.c[2][2] = c2;
    return m;
}
__device__ __forceinline__ M3 m3_mul(const M3& a, const M3& b) {
    M3 r;
#pragma unroll
    for (int col = 0; col < 3; ++col)
#pragma unroll
        for (int row = 0; row < 3; ++row)
            r.c[col][row] = a.c[0][row] * b.c[col][0] + a.c[1][row] * b.c[col][1] +
                            a.c[2][row] * b.c[col][2];
    return r;
}
__device__ __forceinline__ M3 m3_t(const M3& a) {
    M3 r;
#pragma unroll
    for (int col = 0; col < 3; ++col)
#pragma unroll
        for (int row = 0; row < 3; ++row) r.c[col][row] = a.c[row][col];
    return r;
}

// SH basis constants (auxiliary.h:22-39)
__device__ constexpr float kC0 = 0.28209479177387814f;
__device__ constexpr float kC1 = 0.4886025119029199f;
__device__ constexpr float kC2[5] = {1.0925484305920792f, -1.0925484305920792f,
                                     0.31539156525252005f, -1.0925484305920792f,
                                     0.5462742152960396f};
__device__ constexpr float kC3[7] = {-0.5900435899266435f, 2.890611442640554f,
                                     -0.4570457994644658f, 0.3731763325901154f,
                                     -0.4570457994644658f, 1.445305721320277f,
                                     -0.5900435899266435f};

struct Cam {
    float view[16];
    float proj[16];
    float campos[3];
};

__device__ __forceinline__ void load_cam(Cam& s_cam, const float* view, const float* proj,
                                         const float* campos) {
    const int t = threadIdx.x;
    if (t < 16) s_cam.view[t] = view[t];
    else if (t < 32) s_cam.proj[t - 16] = proj[t - 16];
    else if (t < 35 && campos) s_cam.campos[t - 32] = campos[t - 32];
    __syncthreads();
}

// auxiliary.h:58-77
__device__ __forceinline__ float3 xform4x3(const float3& p, const float* m) {
    float3 r = {m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12],
                m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14]};
    return r;
}
__device__ __forceinline__ float4 xform4x4(const float3& p, const float* m) {
    float4 r = {m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12],
                m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
                m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14],
                m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15]};
    return r;
}

// auxiliary.h:41-44 : evaluated in double, rounded to float on return
__device__ __forceinline__ float ndc_to_pix(float v, int S) { return ((v + 1.0) * S - 1.0) * 0.5; }

// forward.cu:118-152.  Which product of each a*b + c*d is fused into an FMA is left to the compiler elsewhere, and
// ptxas decides it differently per architecture; here every rounding is spelled out (the _rn intrinsics are never
// re-fused) as the reference's compiled computeCov3D rounds (pinned by tests/golden/raster_*.npz), so the covariance
// - and the conic, radii and tile lists that follow from it - do not depend on the GPU the library is built for.
__device__ __forceinline__ void cov3d_from_scale_rot(const float3 scale, float mod, const float4 rot,
                                                     float* cov3D) {
    const float s[3] = {__fmul_rn(mod, scale.x), __fmul_rn(mod, scale.y), __fmul_rn(mod, scale.z)};
    const float r = rot.x, x = rot.y, y = rot.z, z = rot.w;
    // R.c[col][row] (glm column-major, as m3()); S * R scales row k by s[k] (the zeros of S add exactly)
    const float R[3][3] = {
        {1.f - 2.f * __fadd_rn(__fmul_rn(y, y), __fmul_rn(z, z)), 2.f * __fmaf_rn(x, y, __fmul_rn(-r, z)),
         2.f * __fmaf_rn(r, y, __fmul_rn(x, z))},
        {2.f * __fmaf_rn(x, y, __fmul_rn(r, z)), 1.f - 2.f * __fmaf_rn(x, x, __fmul_rn(z, z)),
         2.f * __fmaf_rn(y, z, __fmul_rn(-r, x))},
        {2.f * __fmaf_rn(-r, y, __fmul_rn(x, z)), 2.f * __fmaf_rn(y, z, __fmul_rn(r, x)),
         1.f - 2.f * __fmaf_rn(x, x, __fmul_rn(y, y))}};
    float M[3][3];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int k = 0; k < 3; ++k) M[c][k] = __fmul_rn(s[k], R[c][k]);
    // Sigma = M^T M: Sigma.c[col][row] = sum_k M.c[row][k] * M.c[col][k], as fma(k=2, fma(k=0, k=1 product))
    auto sig = [&](int col, int row) {
        return __fmaf_rn(M[row][2], M[col][2], __fmaf_rn(M[row][0], M[col][0], __fmul_rn(M[row][1], M[col][1])));
    };
    cov3D[0] = sig(0, 0);
    cov3D[1] = sig(0, 1);
    cov3D[2] = sig(0, 2);
    cov3D[3] = sig(1, 1);
    cov3D[4] = sig(1, 2);
    cov3D[5] = sig(2, 2);
}

// Gaussian idx's six cov3D values: the precomputed ones, or those of its scale and rotation, which are returned in
// scl / rot (zeros when precomputed).  a: PreFwdArgs, PreBwdArgs or CamBwdArgs.
template <class Args>
__device__ __forceinline__ void load_cov3d(const Args& a, int idx, float cov3D[6], float3& scl, float4& rot) {
    scl = {0.f, 0.f, 0.f};
    rot = {0.f, 0.f, 0.f, 0.f};
    if (a.cov3D_precomp != nullptr) {
#pragma unroll
        for (int i = 0; i < 6; ++i) cov3D[i] = a.cov3D_precomp[6 * idx + i];
    } else {
        scl = {a.scales[3 * idx], a.scales[3 * idx + 1], a.scales[3 * idx + 2]};
        rot = reinterpret_cast<const float4*>(a.rotations)[idx];
        cov3d_from_scale_rot(scl, a.scale_modifier, rot, cov3D);
    }
}

// The EWA projection's Jacobian at a mean (forward.cu:78-97): t = the camera-space mean with x/z and y/z clamped to
// 1.3 tanfov, J = d(image)/dt at that t, W = the view rotation, T = W J.  x/y_grad_mul are 0 where the clamp is
// active, so the backward passes no gradient through a clamped component.  a: PreFwdArgs, PreBwdArgs or CamBwdArgs.
struct EwaJacobian {
    float x_grad_mul, y_grad_mul;
    float3 t;
    M3 J, W, T;
};
template <class Args>
__device__ __forceinline__ EwaJacobian ewa_jacobian(const Args& a, const float3& mean, const float* view) {
    EwaJacobian e;
    float3 t = xform4x3(mean, view);
    const float limx = 1.3f * a.tan_fovx;
    const float limy = 1.3f * a.tan_fovy;
    const float txtz = t.x / t.z;
    const float tytz = t.y / t.z;
    t.x = min(limx, max(-limx, txtz)) * t.z;
    t.y = min(limy, max(-limy, tytz)) * t.z;
    e.t = t;
    e.x_grad_mul = txtz < -limx || txtz > limx ? 0.f : 1.f;
    e.y_grad_mul = tytz < -limy || tytz > limy ? 0.f : 1.f;
    e.J = m3(a.focal_x / t.z, 0.0f, -(a.focal_x * t.x) / (t.z * t.z), 0.0f, a.focal_y / t.z,
             -(a.focal_y * t.y) / (t.z * t.z), 0.f, 0.f, 0.f);
    e.W = m3(view[0], view[4], view[8], view[1], view[5], view[9], view[2], view[6], view[10]);
    e.T = m3_mul(e.W, e.J);
    return e;
}

__device__ __forceinline__ M3 vrk_of(const float* cov3D) {
    return m3(cov3D[0], cov3D[1], cov3D[2], cov3D[1], cov3D[3], cov3D[4], cov3D[2], cov3D[4], cov3D[5]);
}

// forward.cu:74-113 without the dilation: the EWA 2-D covariance {a, b, c}
template <class Args>
__device__ __forceinline__ float3 cov2d_ewa_raw(const Args& a, const float3& mean, const float* cov3D,
                                                const float* view) {
    const M3 T = ewa_jacobian(a, mean, view).T;
    const M3 cov = m3_mul(m3_mul(m3_t(T), m3_t(vrk_of(cov3D))), T);
    return {cov.c[0][0], cov.c[0][1], cov.c[1][1]};
}
// forward.cu:74-113: the 2-D covariance dilated by 0.3 px^2
template <class Args>
__device__ __forceinline__ float3 cov2d_ewa(const Args& a, const float3& mean, const float* cov3D, const float* view) {
    float3 cov = cov2d_ewa_raw(a, mean, cov3D, view);
    cov.x += 0.3f;
    cov.z += 0.3f;
    return cov;
}

// Antialiasing (Mip-Splatting's 2-D filter): the dilation by 0.3 px^2 grows a Gaussian's footprint, and with it the
// energy it puts on screen, the more the smaller it is against a pixel.  The antialiased forms scale its opacity by
// h = sqrt(max(rho, AA_RHO_MIN)), rho = det0 / det1 the ratio of the 2-D covariance's determinant before and after
// the dilation, so that the dilated Gaussian carries the energy of the undilated one.  a, b, c: the EWA covariance
// (cov2d_ewa_raw), det1: the dilated determinant.
constexpr float AA_RHO_MIN = 2.5e-5f;
__device__ __forceinline__ float aa_rho(float a, float b, float c, float det1) { return (a * c - b * b) / det1; }
__device__ __forceinline__ float aa_scale(float rho) { return sqrtf(fmaxf(rho, AA_RHO_MIN)); }

// The camera's own intrinsics and OpenCV radial-tangential distortion (s3g_rasterize_forward_lens).  For the
// camera-space mean t: x = t.x / t.z, y = t.y / t.z, s = x^2 + y^2, rho = 1 + k1 s + k2 s^2 + k3 s^3,
// xd = x rho + 2 p1 x y + p2 (s + 2 x^2), yd = y rho + p1 (s + 2 y^2) + 2 p2 x y and the pixel is
// (fx xd + cx - 0.5, fy yd + cy - 0.5).  The 2-D covariance takes J = F D J_n: F = diag(fx, fy), D = d(xd, yd)/d(x, y)
// at the unclamped (x, y), J_n the pinhole Jacobian of (x, y) at the mean clamped to [xlo, xhi] x [ylo, yhi].  The host
// fills the derived fields (lens_params in api.cu).
struct LensParams {
    float fx, fy, cx, cy, k1, k2, p1, p2, k3;
    float max_r2;                // s*: culled where s > s* (+inf: the radial map never folds back)
    float xlo, xhi, ylo, yhi;    // the 1.3-frustum clamp of x and y in J_n
    float ndc_x, ndc_y;          // 2 / W, 2 / H: d(ndc) / d(pixel), the units of dL_dmean2D
};

// (x, y) and everything the distortion, its Jacobian D = [[D00, D01], [D01, D11]] and D's derivatives need
struct LensPoint {
    float x, y, s, rho, drho, ddrho;
    float xd, yd;
    float D00, D01, D11;
};
__device__ __forceinline__ LensPoint lens_point(const LensParams& L, float x, float y) {
    LensPoint p;
    p.x = x;
    p.y = y;
    const float s = x * x + y * y;
    p.s = s;
    p.rho = 1.f + s * (L.k1 + s * (L.k2 + s * L.k3));
    p.drho = L.k1 + s * (2.f * L.k2 + 3.f * L.k3 * s);    // d rho / ds
    p.ddrho = 2.f * L.k2 + 6.f * L.k3 * s;                 // d^2 rho / ds^2
    p.xd = x * p.rho + 2.f * L.p1 * x * y + L.p2 * (s + 2.f * x * x);
    p.yd = y * p.rho + L.p1 * (s + 2.f * y * y) + 2.f * L.p2 * x * y;
    p.D00 = p.rho + 2.f * x * x * p.drho + 2.f * L.p1 * y + 6.f * L.p2 * x;
    p.D01 = 2.f * x * y * p.drho + 2.f * L.p1 * x + 2.f * L.p2 * y;
    p.D11 = p.rho + 2.f * y * y * p.drho + 6.f * L.p1 * y + 2.f * L.p2 * x;
    return p;
}

// ewa_jacobian's lens form: e.t is the camera-space mean with x, y clamped to the lens's limits, e.J = F D J_n (rows as
// ewa_jacobian's), e.T = W J; p holds the unclamped point.
struct LensJacobian {
    EwaJacobian e;
    LensPoint p;
};
__device__ __forceinline__ LensJacobian lens_jacobian(const LensParams& L, const float3& t_view, const float* view) {
    LensJacobian lj;
    const float x = t_view.x / t_view.z;
    const float y = t_view.y / t_view.z;
    lj.p = lens_point(L, x, y);
    EwaJacobian& e = lj.e;
    float3 t = t_view;
    t.x = min(L.xhi, max(L.xlo, x)) * t.z;
    t.y = min(L.yhi, max(L.ylo, y)) * t.z;
    e.t = t;
    e.x_grad_mul = x < L.xlo || x > L.xhi ? 0.f : 1.f;
    e.y_grad_mul = y < L.ylo || y > L.yhi ? 0.f : 1.f;
    const float iz = 1.f / t.z;
    const float n02 = -t.x * iz * iz, n12 = -t.y * iz * iz;   // J_n = [[1/z, 0, n02], [0, 1/z, n12]]
    const float a00 = L.fx * lj.p.D00, a01 = L.fx * lj.p.D01, a10 = L.fy * lj.p.D01, a11 = L.fy * lj.p.D11;
    e.J = m3(a00 * iz, a01 * iz, a00 * n02 + a01 * n12, a10 * iz, a11 * iz, a10 * n02 + a11 * n12, 0.f, 0.f, 0.f);
    e.W = m3(view[0], view[4], view[8], view[1], view[5], view[9], view[2], view[6], view[10]);
    e.T = m3_mul(e.W, e.J);
    return lj;
}

// the EWA 2-D covariance {a, b, c} of T = W J
__device__ __forceinline__ float3 cov2d_of_T(const M3& T, const float* cov3D) {
    const M3 cov = m3_mul(m3_mul(m3_t(T), m3_t(vrk_of(cov3D))), T);
    return {cov.c[0][0], cov.c[0][1], cov.c[1][1]};
}

// dL/dt of the lens's covariance path from dL/dJ (J = F D J_n, lens_jacobian): through J_n to the clamped mean (no
// gradient to a clamped component) and through D's dependence on the unclamped (x, y) to t.
__device__ __forceinline__ float3 lens_cov_dt(const LensParams& L, const LensJacobian& lj, const float dJ[2][3]) {
    const LensPoint& p = lj.p;
    const float3 t = lj.e.t;
    const float iz = 1.f / t.z, iz2 = iz * iz;
    const float a00 = L.fx * p.D00, a01 = L.fx * p.D01, a10 = L.fy * p.D01, a11 = L.fy * p.D11;
    // dL/dJ_n = (F D)^T dL/dJ; only the entries that are not constant are needed
    const float dn00 = a00 * dJ[0][0] + a10 * dJ[1][0];
    const float dn02 = a00 * dJ[0][2] + a10 * dJ[1][2];
    const float dn11 = a01 * dJ[0][1] + a11 * dJ[1][1];
    const float dn12 = a01 * dJ[0][2] + a11 * dJ[1][2];
    float3 dt;
    dt.x = lj.e.x_grad_mul * -dn02 * iz2;
    dt.y = lj.e.y_grad_mul * -dn12 * iz2;
    dt.z = -(dn00 + dn11) * iz2 + 2.f * (t.x * dn02 + t.y * dn12) * iz2 * iz;
    // dL/dD = F^T dL/dJ J_n^T, with D01 = D10 one variable
    const float n02 = -t.x * iz2, n12 = -t.y * iz2;
    const float dD00 = L.fx * (dJ[0][0] * iz + dJ[0][2] * n02);
    const float dD01 = L.fx * (dJ[0][1] * iz + dJ[0][2] * n12) + L.fy * (dJ[1][0] * iz + dJ[1][2] * n02);
    const float dD11 = L.fy * (dJ[1][1] * iz + dJ[1][2] * n12);
    // dD/dx, dD/dy (d rho/dx = 2 x rho', d rho'/dx = 2 x rho'')
    const float x = p.x, y = p.y;
    const float dD00_dx = 6.f * x * p.drho + 4.f * x * x * x * p.ddrho + 6.f * L.p2;
    const float pxy = 2.f * y * p.drho + 4.f * x * x * y * p.ddrho + 2.f * L.p1;   // dD00/dy = dD01/dx
    const float qxy = 2.f * x * p.drho + 4.f * x * y * y * p.ddrho + 2.f * L.p2;   // dD01/dy = dD11/dx
    const float dD11_dy = 6.f * y * p.drho + 4.f * y * y * y * p.ddrho + 6.f * L.p1;
    const float gx = dD00 * dD00_dx + dD01 * pxy + dD11 * qxy;
    const float gy = dD00 * pxy + dD01 * qxy + dD11 * dD11_dy;
    // (x, y) = (t.x, t.y) / t.z
    dt.x += gx * iz;
    dt.y += gy * iz;
    dt.z -= (gx * x + gy * y) * iz;
    return dt;
}

// conic -> cov2D -> T and t (backward.cu:144-264): the gradients of the loss with respect to cov2D's entries a, b, c
// (zero unless nonsingular, i.e. denom2inv != 0), to dL/d(W J)[k][j] = dL_dT[k][j] and to the clamped camera-space
// mean t (the depth term excluded).  dL_dconic = {x, y, z} of the conic {a', b', c'}.
// AA (antialiased forward): alpha_g = dL/dalpha_eff * alpha_eff, with alpha_eff = opacity * h the opacity the
// composite used; the filter's term dL/drho * drho/d{a, b, c} joins dL_da, dL_db, dL_dc, and aa_h returns h.
struct Cov2dGrad {
    float dL_da, dL_db, dL_dc;
    bool nonsingular;
    float dL_dT[2][3];
    float3 dL_dt;
    float aa_h;
};
// LENS (after a lens forward): e is lj->e, and dL_dt also carries D's dependence on the mean (lens_cov_dt).
template <bool AA = false, bool LENS = false, class Args>
__device__ __forceinline__ Cov2dGrad cov2d_backward(const Args& a, const EwaJacobian& e, const float* cov3D,
                                                    float3 dL_dconic, float alpha_g = 0.f,
                                                    const LensJacobian* lj = nullptr) {
    Cov2dGrad g;
    const float h_x = a.focal_x, h_y = a.focal_y;
    const M3& T = e.T;
    const M3& W = e.W;
    const M3 Vrk = vrk_of(cov3D);
    const M3 cov2D = m3_mul(m3_mul(m3_t(T), m3_t(Vrk)), T);
    const float ca = cov2D.c[0][0] + 0.3f;
    const float cb = cov2D.c[0][1];
    const float cc = cov2D.c[1][1] + 0.3f;
    const float denom = ca * cc - cb * cb;
    float dL_da = 0, dL_db = 0, dL_dc = 0;
    const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
    g.nonsingular = denom2inv != 0;
    if (g.nonsingular) {
        dL_da = denom2inv * (-cc * cc * dL_dconic.x + 2 * cb * cc * dL_dconic.y + (denom - ca * cc) * dL_dconic.z);
        dL_dc = denom2inv * (-ca * ca * dL_dconic.z + 2 * ca * cb * dL_dconic.y + (denom - ca * cc) * dL_dconic.x);
        dL_db = denom2inv * 2 * (cb * cc * dL_dconic.x - (denom + 2 * cb * cb) * dL_dconic.y + ca * cb * dL_dconic.z);
    }
    if (AA) {
        const float a0 = cov2D.c[0][0], c0 = cov2D.c[1][1];
        const float rho = aa_rho(a0, cb, c0, denom);
        g.aa_h = aa_scale(rho);
        if (g.nonsingular && rho > AA_RHO_MIN) {
            // dL/drho = opacity g / (2 h) = alpha_eff g / (2 rho), as h * h = rho here; drho/d{a, b, c} with
            // det0 = a c - b^2 and det1 = denom = (a + 0.3)(c + 0.3) - b^2
            const float det0 = a0 * c0 - cb * cb;
            const float k = alpha_g / (2.f * rho) / (denom * denom);
            dL_da += k * (c0 * denom - det0 * cc);
            dL_dc += k * (a0 * denom - det0 * ca);
            dL_db += k * (-2.f * cb * (0.3f * (a0 + c0) + 0.09f));
        }
    }
    g.dL_da = dL_da;
    g.dL_db = dL_db;
    g.dL_dc = dL_dc;
    // dL_dT[k][j] = 2 (row k of T . column j of Vrk) dL_d(a or c) + (the other row . column j) dL_db
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const float own = T.c[k][0] * Vrk.c[j][0] + T.c[k][1] * Vrk.c[j][1] + T.c[k][2] * Vrk.c[j][2];
            const float other = T.c[1 - k][0] * Vrk.c[j][0] + T.c[1 - k][1] * Vrk.c[j][1] + T.c[1 - k][2] * Vrk.c[j][2];
            g.dL_dT[k][j] = 2 * own * (k == 0 ? dL_da : dL_dc) + other * dL_db;
        }
    const float (&dT)[2][3] = g.dL_dT;
    if constexpr (LENS) {
        float dJ[2][3];
#pragma unroll
        for (int k = 0; k < 2; ++k)
#pragma unroll
            for (int i = 0; i < 3; ++i) dJ[k][i] = W.c[i][0] * dT[k][0] + W.c[i][1] * dT[k][1] + W.c[i][2] * dT[k][2];
        g.dL_dt = lens_cov_dt(a.lens, *lj, dJ);
        return g;
    }
    const float dL_dJ00 = W.c[0][0] * dT[0][0] + W.c[0][1] * dT[0][1] + W.c[0][2] * dT[0][2];
    const float dL_dJ02 = W.c[2][0] * dT[0][0] + W.c[2][1] * dT[0][1] + W.c[2][2] * dT[0][2];
    const float dL_dJ11 = W.c[1][0] * dT[1][0] + W.c[1][1] * dT[1][1] + W.c[1][2] * dT[1][2];
    const float dL_dJ12 = W.c[2][0] * dT[1][0] + W.c[2][1] * dT[1][1] + W.c[2][2] * dT[1][2];
    const float3 t = e.t;
    const float tz = 1.f / t.z;
    const float tz2 = tz * tz;
    const float tz3 = tz2 * tz;
    g.dL_dt.x = e.x_grad_mul * -h_x * tz2 * dL_dJ02;
    g.dL_dt.y = e.y_grad_mul * -h_y * tz2 * dL_dJ12;
    g.dL_dt.z = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * t.x) * tz3 * dL_dJ02 +
                (2 * h_y * t.y) * tz3 * dL_dJ12;
    return g;
}

// forward.cu:20-71. sh points at this Gaussian's M coefficients ([M][3]).
__device__ __forceinline__ float3 sh_to_rgb(int deg, const float3 pos, const float* campos,
                                            const float* sh, uint8_t& clamped) {
    float3 dir = {pos.x - campos[0], pos.y - campos[1], pos.z - campos[2]};
    float len = sqrtf(dir.x * dir.x + dir.y * dir.y + dir.z * dir.z);
    dir.x = dir.x / len;
    dir.y = dir.y / len;
    dir.z = dir.z / len;
    float res[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#define SH(i) sh[(i) * 3 + c]
        float result = kC0 * SH(0);
        if (deg > 0) {
            float x = dir.x, y = dir.y, z = dir.z;
            result = result - kC1 * y * SH(1) + kC1 * z * SH(2) - kC1 * x * SH(3);
            if (deg > 1) {
                float xx = x * x, yy = y * y, zz = z * z;
                float xy = x * y, yz = y * z, xz = x * z;
                result = result + kC2[0] * xy * SH(4) + kC2[1] * yz * SH(5) +
                         kC2[2] * (2.0f * zz - xx - yy) * SH(6) + kC2[3] * xz * SH(7) +
                         kC2[4] * (xx - yy) * SH(8);
                if (deg > 2) {
                    result = result + kC3[0] * y * (3.0f * xx - yy) * SH(9) +
                             kC3[1] * xy * z * SH(10) + kC3[2] * y * (4.0f * zz - xx - yy) * SH(11) +
                             kC3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * SH(12) +
                             kC3[4] * x * (4.0f * zz - xx - yy) * SH(13) +
                             kC3[5] * z * (xx - yy) * SH(14) + kC3[6] * x * (xx - 3.0f * yy) * SH(15);
                }
            }
        }
#undef SH
        res[c] = result + 0.5f;
    }
    clamped = (uint8_t)((res[0] < 0 ? 1 : 0) | (res[1] < 0 ? 2 : 0) | (res[2] < 0 ? 4 : 0));
    return {fmaxf(res[0], 0.0f), fmaxf(res[1], 0.0f), fmaxf(res[2], 0.0f)};
}

// dL/d(normalised dir) of the SH colour, summed over the channels (backward.cu:20-139).  (x, y, z): the normalised
// direction, sh: the Gaussian's [M][3] coefficients, dRGB: dL/dcolour with the clamped channels zeroed.
__device__ __forceinline__ float3 sh_ddir(int deg, float x, float y, float z, const float* sh, const float dRGB[3]) {
    float ddir[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#define SH(i) sh[(i) * 3 + c]
        float dx_ = 0.f, dy_ = 0.f, dz_ = 0.f;
        if (deg > 0) {
            dx_ = -kC1 * SH(3);
            dy_ = -kC1 * SH(1);
            dz_ = kC1 * SH(2);
            if (deg > 1) {
                dx_ += kC2[0] * y * SH(4) + kC2[2] * 2.f * -x * SH(6) + kC2[3] * z * SH(7) + kC2[4] * 2.f * x * SH(8);
                dy_ += kC2[0] * x * SH(4) + kC2[1] * z * SH(5) + kC2[2] * 2.f * -y * SH(6) + kC2[4] * 2.f * -y * SH(8);
                dz_ += kC2[1] * y * SH(5) + kC2[2] * 2.f * 2.f * z * SH(6) + kC2[3] * x * SH(7);
                if (deg > 2) {
                    float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                    dx_ += (kC3[0] * SH(9) * 3.f * 2.f * xy + kC3[1] * SH(10) * yz +
                            kC3[2] * SH(11) * -2.f * xy + kC3[3] * SH(12) * -3.f * 2.f * xz +
                            kC3[4] * SH(13) * (-3.f * xx + 4.f * zz - yy) +
                            kC3[5] * SH(14) * 2.f * xz + kC3[6] * SH(15) * 3.f * (xx - yy));
                    dy_ += (kC3[0] * SH(9) * 3.f * (xx - yy) + kC3[1] * SH(10) * xz +
                            kC3[2] * SH(11) * (-3.f * yy + 4.f * zz - xx) +
                            kC3[3] * SH(12) * -3.f * 2.f * yz + kC3[4] * SH(13) * -2.f * xy +
                            kC3[5] * SH(14) * -2.f * yz + kC3[6] * SH(15) * -3.f * 2.f * xy);
                    dz_ += (kC3[1] * SH(10) * xy + kC3[2] * SH(11) * 4.f * 2.f * yz +
                            kC3[3] * SH(12) * 3.f * (2.f * zz - xx - yy) +
                            kC3[4] * SH(13) * 4.f * 2.f * xz + kC3[5] * SH(14) * (xx - yy));
                }
            }
        }
#undef SH
        ddir[0] += dx_ * dRGB[c];
        ddir[1] += dy_ * dRGB[c];
        ddir[2] += dz_ * dRGB[c];
    }
    return make_float3(ddir[0], ddir[1], ddir[2]);
}

struct PreFwdArgs {
    int P, D, M;
    const float* means3D;
    const float* scales;
    float scale_modifier;
    const float* rotations;
    const float* opacities;
    const float* shs;
    const float* cov3D_precomp;
    const float* colors_precomp;
    const float* colors_aux;   // [P,3] second colour set (feature image of render_feat) or NULL
    const float* view;
    const float* proj;
    const float* campos;
    int W, H;
    float tan_fovx, tan_fovy, focal_x, focal_y;
    int* radii;
    float4* xyAB;
    float4* Cod;
    float4* rgb;
    float4* aux;
    uint32_t* depth_key;
    uint32_t* tiles_touched;
    ushort4* rect;
    uint8_t* clamped;
    uint32_t* order;   // identity permutation, input of the depth sort
    int grid_x, grid_y;
    // static/dynamic split (forward only): group [P] nonzero = dynamic, or NULL.  A dynamic Gaussian gets bit 31 of
    // its own-index word in Cod.w (P < 2^30 leaves it free); group_count (zeroed) receives the number of them.
    const uint8_t* group;
    uint32_t* group_count;
};

// Conservative per-Gaussian cull threshold used by the tile kernels: a pixel
// whose quadratic form q = -power exceeds tau can never reach alpha >= 1/255
// (forward.cu:346-348), with slack for fp32 rounding that grows with the
// conditioning of the conic.  +inf disables culling for this Gaussian.
__device__ __forceinline__ float cull_tau(float opacity, float A, float B, float C, float lam_max,
                                          float lam_min) {
    const float INF = __int_as_float(0x7f800000);
    if (!(opacity == opacity)) return INF;   // NaN opacity: fminf(0.99, NaN) = 0.99 in the reference
    if (!(A > 0.f) || !(C > 0.f) || !(A * C - B * B > 0.f)) return INF;   // not PD: never cull
    if (!(opacity * 255.0f >= 0.999f)) return -1.0f;  // alpha <= opacity < 1/255 everywhere
    float cond = lam_max / fmaxf(lam_min, 1e-12f);
    float eps = 1e-5f * cond;
    if (!(eps < 0.5f)) return INF;
    float tau = __logf(opacity * 255.0f);
    tau = fmaxf(tau, 0.f);
    return (tau + 2e-3f) / (1.0f - eps) + 2e-3f;
}

// ---- warp-cooperative row staging ------------------------------------------
// A warp owns 32 consecutive Gaussians, i.e. 32 consecutive rows of L floats
// (SH coefficients or their gradients: L = 3*M, 192 bytes at M = 16).  Reading
// or writing them one row per lane touches 32 different 32-byte sectors per
// instruction; instead the warp moves the contiguous 32*L-float block with
// fully coalesced (vector) accesses through a shared-memory tile whose row
// stride is odd, so the per-lane row accesses are bank-conflict free.
constexpr int PRE_THREADS = 128;
__host__ __device__ inline int row_stride(int L) { return L | 1; }

template <int LT>   // LT > 0: compile-time row length, 0: runtime
__device__ __forceinline__ void warp_rows_in(const float* __restrict__ g, float* s, int Lr, int rows,
                                             int lane) {
    const int L = LT > 0 ? LT : Lr;
    const int stride = row_stride(L);
    const int total = rows * L;
    if ((L & 3) == 0 && ((reinterpret_cast<uintptr_t>(g) & 15) == 0)) {
        const float4* g4 = reinterpret_cast<const float4*>(g);
        for (int q = lane; q < total / 4; q += 32) {
            const float4 v = __ldg(g4 + q);
            const int f = q * 4, r = f / L, j = f - r * L;
            float* d = s + r * stride + j;
            d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
        }
    } else {
        for (int f = lane; f < total; f += 32) {
            const int r = f / L, j = f - r * L;
            s[r * stride + j] = __ldg(g + f);
        }
    }
}
template <int LT>
__device__ __forceinline__ void warp_rows_out(float* __restrict__ g, const float* s, int Lr, int rows,
                                              int lane) {
    const int L = LT > 0 ? LT : Lr;
    const int stride = row_stride(L);
    const int total = rows * L;
    if ((L & 3) == 0 && ((reinterpret_cast<uintptr_t>(g) & 15) == 0)) {
        float4* g4 = reinterpret_cast<float4*>(g);
        for (int q = lane; q < total / 4; q += 32) {
            const int f = q * 4, r = f / L, j = f - r * L;
            const float* d = s + r * stride + j;
            g4[q] = make_float4(d[0], d[1], d[2], d[3]);
        }
    } else {
        for (int f = lane; f < total; f += 32) {
            const int r = f / L, j = f - r * L;
            g[f] = s[r * stride + j];
        }
    }
}

struct Projected {
    float2 pix;
    float3 conic;
    float depth, radius, lam_max, lam_min;
    unsigned rminx, rminy, rmaxx, rmaxy;
    float aa_h;   // AA: the opacity factor of the antialiasing filter
};

// Everything of forward.cu:182-237 up to (not including) the colour; false = culled.  LENS: a: PreFwdLensArgs, the
// mean and the covariance's Jacobian through the lens (LensParams), and the lens cull.
template <bool AA, bool LENS = false, class Args>
__device__ __forceinline__ bool project_gaussian(const Args& a, const Cam& cam, int idx, const float3 p_orig,
                                                 Projected& o) {
    // near cull (auxiliary.h:152-154)
    const float3 p_view = xform4x3(p_orig, cam.view);
    if (p_view.z <= 0.2f) return false;

    float2 point_image;
    LensJacobian lj;
    if constexpr (LENS) {
        lj = lens_jacobian(a.lens, p_view, cam.view);
        if (lj.p.s > a.lens.max_r2) return false;
        point_image = {a.lens.fx * lj.p.xd + a.lens.cx - 0.5f, a.lens.fy * lj.p.yd + a.lens.cy - 0.5f};
    }
    float3 p_proj;
    if constexpr (!LENS) {
        const float4 p_hom = xform4x4(p_orig, cam.proj);
        const float p_w = 1.0f / (p_hom.w + 0.0000001f);
        p_proj = {p_hom.x * p_w, p_hom.y * p_w, p_hom.z * p_w};
    }

    float cov3D[6];
    float3 scl;
    float4 rot;
    load_cov3d(a, idx, cov3D, scl, rot);
    float3 raw, cov;
    if constexpr (LENS) {
        raw = cov2d_of_T(lj.e.T, cov3D);
        cov = {raw.x + 0.3f, raw.y, raw.z + 0.3f};
    } else if (AA) {
        raw = cov2d_ewa_raw(a, p_orig, cov3D, cam.view);
        cov = {raw.x + 0.3f, raw.y, raw.z + 0.3f};
    } else {
        cov = cov2d_ewa(a, p_orig, cov3D, cam.view);
    }

    const float det = (cov.x * cov.z - cov.y * cov.y);
    if (det == 0.0f) return false;
    if (AA) o.aa_h = aa_scale(aa_rho(raw.x, raw.y, raw.z, det));
    const float det_inv = 1.f / det;
    o.conic = {cov.z * det_inv, -cov.y * det_inv, cov.x * det_inv};

    const float mid = 0.5f * (cov.x + cov.z);
    const float lambda1 = mid + sqrtf(max(0.1f, mid * mid - det));
    const float lambda2 = mid - sqrtf(max(0.1f, mid * mid - det));
    const float my_radius = ceilf(3.f * sqrtf(max(lambda1, lambda2)));
    if constexpr (!LENS) point_image = {ndc_to_pix(p_proj.x, a.W), ndc_to_pix(p_proj.y, a.H)};

    // getRect (auxiliary.h:46-56): radius is passed as int, float division, C truncation
    const int max_radius = (int)my_radius;
    const unsigned gx = (unsigned)a.grid_x, gy = (unsigned)a.grid_y;
    o.rminx = min(gx, (unsigned)max((int)0, (int)((point_image.x - max_radius) / TILE_X)));
    o.rminy = min(gy, (unsigned)max((int)0, (int)((point_image.y - max_radius) / TILE_Y)));
    o.rmaxx = min(gx, (unsigned)max((int)0, (int)((point_image.x + max_radius + TILE_X - 1) / TILE_X)));
    o.rmaxy = min(gy, (unsigned)max((int)0, (int)((point_image.y + max_radius + TILE_Y - 1) / TILE_Y)));
    if ((o.rmaxx - o.rminx) * (o.rmaxy - o.rminy) == 0) return false;
    o.pix = point_image;
    o.depth = p_view.z;
    o.radius = my_radius;
    o.lam_max = max(lambda1, lambda2);
    o.lam_min = min(lambda1, lambda2);
    return true;
}

// the lens forward's arguments: the plain ones and the lens
struct PreFwdLensArgs : PreFwdArgs {
    LensParams lens;
};

// MT = 16: SH rows of 48 floats known at compile time; 0: runtime M.  AA: the composite gets opacity * h (antialiasing).
// LENS: a is a PreFwdLensArgs (preprocess_forward_lens_kernel)
template <int MT, bool AA, bool LENS, class Args>
__device__ __forceinline__ void preprocess_forward(const Args& a) {
    extern __shared__ float s_dyn[];
    __shared__ Cam s_cam;
    load_cam(s_cam, a.view, a.proj, a.campos);
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool valid = idx < a.P;

    Projected po;
    float3 p_orig = {0.f, 0.f, 0.f};
    bool vis = false;
    if (valid) {
        a.radii[idx] = 0;
        a.tiles_touched[idx] = 0;
        a.depth_key[idx] = DEPTH_KEY_INVISIBLE;
        a.order[idx] = (uint32_t)idx;
        p_orig = {a.means3D[3 * idx], a.means3D[3 * idx + 1], a.means3D[3 * idx + 2]};
        vis = project_gaussian<AA, LENS>(a, s_cam, idx, p_orig, po);
    }
    uint32_t group_bit = 0;
    if (a.group) {
        const bool dyn = valid && a.group[idx] != 0;
        const uint32_t m = __ballot_sync(0xffffffffu, dyn);
        if (lane == 0 && m) atomicAdd(a.group_count, (uint32_t)__popc(m));
        group_bit = dyn ? 0x80000000u : 0u;
    }

    float3 col = {0.f, 0.f, 0.f};
    uint8_t clamped = 0;
    if (a.colors_precomp == nullptr) {
        if (__any_sync(0xffffffffu, vis)) {
            const int L = 3 * (MT > 0 ? MT : a.M);
            float* rows = s_dyn + warp * 32 * row_stride(L);
            const int first = idx - lane;
            const int nrows = min(32, a.P - first);
            warp_rows_in<3 * MT>(a.shs + (size_t)first * L, rows, L, nrows, lane);
            __syncwarp();
            if (vis) col = sh_to_rgb(a.D, p_orig, s_cam.campos, rows + lane * row_stride(L), clamped);
        }
    } else if (vis) {
        col = {a.colors_precomp[3 * idx], a.colors_precomp[3 * idx + 1], a.colors_precomp[3 * idx + 2]};
    }
    if (!vis) return;
    const float opacity = AA ? a.opacities[idx] * po.aa_h : a.opacities[idx];

    a.clamped[idx] = clamped;
    a.radii[idx] = (int)po.radius;
    a.depth_key[idx] = __float_as_uint(po.depth);
    a.xyAB[idx] = make_float4(po.pix.x, po.pix.y, po.conic.x, po.conic.y);
    // Cod.w carries the Gaussian's own index: the backward composite takes the target of its REDs from the
    // staged record instead of a second id table (bit 31: the Gaussian's group in a split forward)
    a.Cod[idx] = make_float4(po.conic.z, opacity,
                             cull_tau(opacity, po.conic.x, po.conic.y, po.conic.z, po.lam_max, po.lam_min),
                             __uint_as_float((uint32_t)idx | group_bit));
    a.rgb[idx] = make_float4(col.x, col.y, col.z, po.depth);
    if (a.colors_aux)
        a.aux[idx] = make_float4(a.colors_aux[3 * idx], a.colors_aux[3 * idx + 1], a.colors_aux[3 * idx + 2], 0.f);
    a.rect[idx] = make_ushort4((unsigned short)po.rminx, (unsigned short)po.rminy, (unsigned short)po.rmaxx,
                               (unsigned short)po.rmaxy);
    a.tiles_touched[idx] = (po.rmaxy - po.rminy) * (po.rmaxx - po.rminx);
}
template <int MT, bool AA = false>
__global__ void __launch_bounds__(PRE_THREADS) preprocess_forward_kernel(PreFwdArgs a) {
    preprocess_forward<MT, AA, false>(a);
}
template <int MT, bool AA>
__global__ void __launch_bounds__(PRE_THREADS) preprocess_forward_lens_kernel(PreFwdLensArgs a) {
    preprocess_forward<MT, AA, true>(a);
}

// rasterizer_impl.cu:54-66
__global__ void __launch_bounds__(256)
mark_visible_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ view,
                    const float* __restrict__ proj, uint8_t* __restrict__ present) {
    __shared__ Cam s_cam;
    load_cam(s_cam, view, proj, nullptr);
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const float3 p = {means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2]};
    const float3 p_view = xform4x3(p, s_cam.view);
    present[idx] = p_view.z <= 0.2f ? 0 : 1;
}

// ---------------------------------------------------------------------------
// Backward
// ---------------------------------------------------------------------------
// Data-parallel gradient exchange fused into this kernel (dp.FusedGradExchange, csrc/peer.cuh): instead of
// writing the five per-Gaussian gradient tensors locally for a later all-reduce, every VISIBLE Gaussian's values
// are stored straight into the staging area of the rank that owns that slice of the flat gradient bucket, over
// NVLink peer mappings - the reduce-scatter half of the all-reduce happens while the kernel runs, culled rows
// (27 % at the benchmark view) never cross the link.  stage[o] is rank o's staging area [world][chunk].
struct PeerSink {
    float* stage[16];
    int world, rank;
    long long chunk;                                                  // floats per owner slice, multiple of 4
    long long off_mean3D, off_sh, off_opacity, off_scale, off_rot;   // offsets in the flat bucket (floats, off_sh % 4 == 0)
};
__device__ __forceinline__ float* sink_ptr(const PeerSink& s, long long e) {
    const long long o = e / s.chunk;
    return s.stage[o] + (long long)s.rank * s.chunk + (e - o * s.chunk);
}

struct PreBwdArgs {
    int P, D, M;
    const float* means3D;
    const int* radii;
    const float* shs;
    const uint8_t* clamped;
    const float* scales;
    const float* rotations;
    float scale_modifier;
    const float* cov3D_precomp;
    const float* view;
    const float* proj;
    const float* campos;
    float focal_x, focal_y, tan_fovx, tan_fovy;
    const float* grad_rec;   // [P][GRAD_REC] accumulated by the backward composite
    float* dL_dmean2D;       // [P,3]
    float* dL_dconic;        // [P,4] or NULL
    float* dL_dopacity;      // [P]
    float* dL_dcolor;        // [P,3]
    float* dL_dcolor_aux;    // [P,3] or NULL
    float* dL_ddepth;        // [P] or NULL
    float* dL_dmean3D;       // [P,3]
    float* dL_dcov3D;        // [P,6]
    float* dL_dsh;           // [P,M,3] or NULL when M == 0
    float* dL_dscale;        // [P,3]
    float* dL_drot;          // [P,4]
    PeerSink sink;           // DP kernels only
    const float4* Cod;       // AA kernels only: the forward's records, .y = the opacity the composite used
};

__device__ __forceinline__ float3 dnormvdv3(float3 v, float3 dv) {   // auxiliary.h:107-117
    float sum2 = v.x * v.x + v.y * v.y + v.z * v.z;
    float invsum32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
    float3 r;
    r.x = ((+sum2 - v.x * v.x) * dv.x - v.y * v.x * dv.y - v.z * v.x * dv.z) * invsum32;
    r.y = (-v.x * v.y * dv.x + (sum2 - v.y * v.y) * dv.y - v.z * v.y * dv.z) * invsum32;
    r.z = (-v.x * v.z * dv.x - v.y * v.z * dv.y + (sum2 - v.z * v.z) * dv.z) * invsum32;
    return r;
}

// the lens backward's arguments: the plain ones and the lens of the forward
struct PreBwdLensArgs : PreBwdArgs {
    LensParams lens;
};

// MT = 16: compile-time SH row length; 0: runtime M.  DP: gradients go to a.sink.  AA: after an antialiased forward.
// LENS: after a lens forward, a is a PreBwdLensArgs (preprocess_backward_lens_kernel).
template <int MT, bool DP, bool AA, bool LENS, class Args>
__device__ __forceinline__ void preprocess_backward(const Args& a) {
    static_assert(!(DP && AA), "the fused gradient exchange does not take the antialiased backward");
    static_assert(!(DP && LENS), "the fused gradient exchange does not take the lens backward");
    extern __shared__ float s_dyn[];
    __shared__ Cam s_cam;
    load_cam(s_cam, a.view, a.proj, a.campos);
    const int idx_raw = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool valid = idx_raw < a.P;
    const int idx = valid ? idx_raw : a.P - 1;   // clamped for address arithmetic only
    const float* view = s_cam.view;
    const float* proj = s_cam.proj;

    const bool visible = valid && a.radii[idx] > 0;
    // SH rows (input coefficients, then reused for their gradients) staged per warp
    const int Msh = MT > 0 ? MT : a.M;
    const int L = 3 * Msh;
    float* rows = s_dyn + warp * 32 * row_stride(L);
    float* myrow = rows + lane * row_stride(L);
    const int first = idx_raw - lane;
    const int nrows = min(32, a.P - first);
    if (a.shs) {
        if (__any_sync(0xffffffffu, visible)) warp_rows_in<3 * MT>(a.shs + (size_t)first * L, rows, L, nrows, lane);
        __syncwarp();
    }
    float g[GRAD_REC];
    if (visible) {
        const float4* gr = reinterpret_cast<const float4*>(a.grad_rec + (size_t)idx * GRAD_REC);
#pragma unroll
        for (int i = 0; i < GRAD_REC / 4; ++i) {
            float4 v = gr[i];
            g[4 * i] = v.x; g[4 * i + 1] = v.y; g[4 * i + 2] = v.z; g[4 * i + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int i = 0; i < GRAD_REC; ++i) g[i] = 0.f;
    }
    if (valid) {
    // outputs that are plain copies of the composite's accumulators
    a.dL_dmean2D[3 * idx + 0] = g[0];
    a.dL_dmean2D[3 * idx + 1] = g[1];
    a.dL_dmean2D[3 * idx + 2] = 0.f;
    if (a.dL_dconic) {
        a.dL_dconic[4 * idx + 0] = g[2];
        a.dL_dconic[4 * idx + 1] = g[3];
        a.dL_dconic[4 * idx + 2] = 0.f;
        a.dL_dconic[4 * idx + 3] = g[4];
    }
    if (AA) {}   // dL_dopacity = h * g[5] is written below, once h is known
    else if (!DP) a.dL_dopacity[idx] = g[5];
    else if (visible) *sink_ptr(a.sink, a.sink.off_opacity + idx) = g[5];
    a.dL_dcolor[3 * idx + 0] = g[6];
    a.dL_dcolor[3 * idx + 1] = g[7];
    a.dL_dcolor[3 * idx + 2] = g[8];
    if (a.dL_ddepth) a.dL_ddepth[idx] = g[9];
    if (a.dL_dcolor_aux) {
        a.dL_dcolor_aux[3 * idx + 0] = g[10];
        a.dL_dcolor_aux[3 * idx + 1] = g[11];
        a.dL_dcolor_aux[3 * idx + 2] = g[12];
    }
    }

    float dmean[3] = {0.f, 0.f, 0.f};
    float dcov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float dscale[3] = {0.f, 0.f, 0.f};
    float drot[4] = {0.f, 0.f, 0.f, 0.f};
    float aa_h = 0.f;

    if (!visible) {
        if (a.dL_dsh)
            for (int i = 0; i < L; ++i) myrow[i] = 0.f;
    } else {
        const float3 mean = {a.means3D[3 * idx], a.means3D[3 * idx + 1], a.means3D[3 * idx + 2]};
        float cov3D[6];
        float3 scl;
        float4 rot;
        load_cov3d(a, idx, cov3D, scl, rot);
        LensJacobian lj;
        if constexpr (LENS) lj = lens_jacobian(a.lens, xform4x3(mean, view), view);
        // ---- conic -> cov2D -> cov3D, mean (backward.cu:144-274) ----------
        {
            EwaJacobian e;
            if constexpr (LENS) e = lj.e;
            else e = ewa_jacobian(a, mean, view);
            const Cov2dGrad cg = cov2d_backward<AA, LENS>(a, e, cov3D, make_float3(g[2], g[3], g[4]),
                                                          AA ? a.Cod[idx].y * g[5] : 0.f, &lj);
            if (AA) aa_h = cg.aa_h;
            if (cg.nonsingular) {
                const M3& T = e.T;
                const float dL_da = cg.dL_da, dL_db = cg.dL_db, dL_dc = cg.dL_dc;
                dcov[0] = (T.c[0][0] * T.c[0][0] * dL_da + T.c[0][0] * T.c[1][0] * dL_db +
                           T.c[1][0] * T.c[1][0] * dL_dc);
                dcov[3] = (T.c[0][1] * T.c[0][1] * dL_da + T.c[0][1] * T.c[1][1] * dL_db +
                           T.c[1][1] * T.c[1][1] * dL_dc);
                dcov[5] = (T.c[0][2] * T.c[0][2] * dL_da + T.c[0][2] * T.c[1][2] * dL_db +
                           T.c[1][2] * T.c[1][2] * dL_dc);
                dcov[1] = 2 * T.c[0][0] * T.c[0][1] * dL_da +
                          (T.c[0][0] * T.c[1][1] + T.c[0][1] * T.c[1][0]) * dL_db +
                          2 * T.c[1][0] * T.c[1][1] * dL_dc;
                dcov[2] = 2 * T.c[0][0] * T.c[0][2] * dL_da +
                          (T.c[0][0] * T.c[1][2] + T.c[0][2] * T.c[1][0]) * dL_db +
                          2 * T.c[1][0] * T.c[1][2] * dL_dc;
                dcov[4] = 2 * T.c[0][2] * T.c[0][1] * dL_da +
                          (T.c[0][1] * T.c[1][2] + T.c[0][2] * T.c[1][1]) * dL_db +
                          2 * T.c[1][1] * T.c[1][2] * dL_dc;
            }
            // transformVec4x3Transpose (auxiliary.h:89-97); assignment, backward.cu:273
            const float3 dt = cg.dL_dt;
            dmean[0] = view[0] * dt.x + view[1] * dt.y + view[2] * dt.z;
            dmean[1] = view[4] * dt.x + view[5] * dt.y + view[6] * dt.z;
            dmean[2] = view[8] * dt.x + view[9] * dt.y + view[10] * dt.z;
        }
        // ---- screen-space mean and depth terms (backward.cu:372-403) ------
        if constexpr (LENS) {
            // pixel = F (xd, yd) + c - 0.5: dL/d(x, y) = D^T F dL/dpixel, then (x, y) = (t.x, t.y) / t.z
            const LensParams& L = a.lens;
            const LensPoint& p = lj.p;
            const float gxd = L.fx * L.ndc_x * g[0], gyd = L.fy * L.ndc_y * g[1];
            const float gx = p.D00 * gxd + p.D01 * gyd, gy = p.D01 * gxd + p.D11 * gyd;
            const float iz = 1.f / lj.e.t.z;
            const float3 dt = {gx * iz, gy * iz, -(gx * p.x + gy * p.y) * iz};
            dmean[0] += view[0] * dt.x + view[1] * dt.y + view[2] * dt.z;
            dmean[1] += view[4] * dt.x + view[5] * dt.y + view[6] * dt.z;
            dmean[2] += view[8] * dt.x + view[9] * dt.y + view[10] * dt.z;
            const float3 m = mean;
            const float mul3 = view[2] * m.x + view[6] * m.y + view[10] * m.z + view[14];
            const float gd = g[9];
            dmean[0] += (view[2] - view[3] * mul3) * gd;
            dmean[1] += (view[6] - view[7] * mul3) * gd;
            dmean[2] += (view[10] - view[11] * mul3) * gd;
        } else {
            const float3 m = mean;
            const float4 m_hom = xform4x4(m, proj);
            const float m_w = 1.0f / (m_hom.w + 0.0000001f);
            const float mul1 = (proj[0] * m.x + proj[4] * m.y + proj[8] * m.z + proj[12]) * m_w * m_w;
            const float mul2 = (proj[1] * m.x + proj[5] * m.y + proj[9] * m.z + proj[13]) * m_w * m_w;
            const float gx = g[0], gy = g[1];
            dmean[0] += (proj[0] * m_w - proj[3] * mul1) * gx + (proj[1] * m_w - proj[3] * mul2) * gy;
            dmean[1] += (proj[4] * m_w - proj[7] * mul1) * gx + (proj[5] * m_w - proj[7] * mul2) * gy;
            dmean[2] += (proj[8] * m_w - proj[11] * mul1) * gx + (proj[9] * m_w - proj[11] * mul2) * gy;
            const float mul3 = view[2] * m.x + view[6] * m.y + view[10] * m.z + view[14];
            const float gd = g[9];
            dmean[0] += (view[2] - view[3] * mul3) * gd;
            dmean[1] += (view[6] - view[7] * mul3) * gd;
            dmean[2] += (view[10] - view[11] * mul3) * gd;
        }
        // ---- SH (backward.cu:20-139) ---------------------------------------
        if (a.shs) {
            const float* sh = myrow;   // staged coefficients; overwritten with dL/dsh below
            float* dsh = myrow;
            const float* campos = s_cam.campos;
            const float3 dir_orig = {mean.x - campos[0], mean.y - campos[1], mean.z - campos[2]};
            const float len = sqrtf(dir_orig.x * dir_orig.x + dir_orig.y * dir_orig.y + dir_orig.z * dir_orig.z);
            const float x = dir_orig.x / len, y = dir_orig.y / len, z = dir_orig.z / len;
            const uint8_t cl = a.clamped[idx];
            const float dRGB[3] = {(cl & 1) ? 0.f : g[6], (cl & 2) ? 0.f : g[7], (cl & 4) ? 0.f : g[8]};
            const int deg = a.D;
            float basis[16];
            basis[0] = kC0;
            int nb = 1;
            if (deg > 0) {
                basis[1] = -kC1 * y; basis[2] = kC1 * z; basis[3] = -kC1 * x;
                nb = 4;
                if (deg > 1) {
                    float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                    basis[4] = kC2[0] * xy; basis[5] = kC2[1] * yz;
                    basis[6] = kC2[2] * (2.f * zz - xx - yy);
                    basis[7] = kC2[3] * xz; basis[8] = kC2[4] * (xx - yy);
                    nb = 9;
                    if (deg > 2) {
                        basis[9] = kC3[0] * y * (3.f * xx - yy);
                        basis[10] = kC3[1] * xy * z;
                        basis[11] = kC3[2] * y * (4.f * zz - xx - yy);
                        basis[12] = kC3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy);
                        basis[13] = kC3[4] * x * (4.f * zz - xx - yy);
                        basis[14] = kC3[5] * z * (xx - yy);
                        basis[15] = kC3[6] * x * (xx - 3.f * yy);
                        nb = 16;
                    }
                }
            }
            const float3 dm = dnormvdv3(dir_orig, sh_ddir(deg, x, y, z, sh, dRGB));
            dmean[0] += dm.x; dmean[1] += dm.y; dmean[2] += dm.z;
            // all reads of this lane's coefficients are done: the row now carries dL/dsh
            for (int i = 0; i < Msh; ++i) {
                float b = i < nb ? basis[i] : 0.f;
#pragma unroll
                for (int c = 0; c < 3; ++c) dsh[i * 3 + c] = b * dRGB[c];
            }
        }
        // ---- cov3D -> scale, rotation (backward.cu:278-341) ----------------
        if (a.scales) {
            const float r = rot.x, x = rot.y, y = rot.z, z = rot.w;
            M3 R = m3(1.f - 2.f * (y * y + z * z), 2.f * (x * y - r * z), 2.f * (x * z + r * y),
                      2.f * (x * y + r * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z - r * x),
                      2.f * (x * z - r * y), 2.f * (y * z + r * x), 1.f - 2.f * (x * x + y * y));
            const float3 s = {a.scale_modifier * scl.x, a.scale_modifier * scl.y, a.scale_modifier * scl.z};
            M3 S = m3(s.x, 0.f, 0.f, 0.f, s.y, 0.f, 0.f, 0.f, s.z);
            M3 M = m3_mul(S, R);
            M3 dSigma = m3(dcov[0], 0.5f * dcov[1], 0.5f * dcov[2], 0.5f * dcov[1], dcov[3],
                           0.5f * dcov[4], 0.5f * dcov[2], 0.5f * dcov[4], dcov[5]);
            M3 dM = m3_mul(M, dSigma);
#pragma unroll
            for (int c = 0; c < 3; ++c)
#pragma unroll
                for (int rr = 0; rr < 3; ++rr) dM.c[c][rr] *= 2.0f;
            M3 Rt = m3_t(R);
            M3 dMt = m3_t(dM);
            dscale[0] = Rt.c[0][0] * dMt.c[0][0] + Rt.c[0][1] * dMt.c[0][1] + Rt.c[0][2] * dMt.c[0][2];
            dscale[1] = Rt.c[1][0] * dMt.c[1][0] + Rt.c[1][1] * dMt.c[1][1] + Rt.c[1][2] * dMt.c[1][2];
            dscale[2] = Rt.c[2][0] * dMt.c[2][0] + Rt.c[2][1] * dMt.c[2][1] + Rt.c[2][2] * dMt.c[2][2];
#pragma unroll
            for (int rr = 0; rr < 3; ++rr) {
                dMt.c[0][rr] *= s.x;
                dMt.c[1][rr] *= s.y;
                dMt.c[2][rr] *= s.z;
            }
            drot[0] = 2 * z * (dMt.c[0][1] - dMt.c[1][0]) + 2 * y * (dMt.c[2][0] - dMt.c[0][2]) +
                      2 * x * (dMt.c[1][2] - dMt.c[2][1]);
            drot[1] = 2 * y * (dMt.c[1][0] + dMt.c[0][1]) + 2 * z * (dMt.c[2][0] + dMt.c[0][2]) +
                      2 * r * (dMt.c[1][2] - dMt.c[2][1]) - 4 * x * (dMt.c[2][2] + dMt.c[1][1]);
            drot[2] = 2 * x * (dMt.c[1][0] + dMt.c[0][1]) + 2 * r * (dMt.c[2][0] - dMt.c[0][2]) +
                      2 * z * (dMt.c[1][2] + dMt.c[2][1]) - 4 * y * (dMt.c[2][2] + dMt.c[0][0]);
            drot[3] = 2 * r * (dMt.c[0][1] - dMt.c[1][0]) + 2 * x * (dMt.c[2][0] + dMt.c[0][2]) +
                      2 * y * (dMt.c[1][2] + dMt.c[2][1]) - 4 * z * (dMt.c[1][1] + dMt.c[0][0]);
        }
    }
    if (DP) {
        if (a.shs) {   // the warp's visible rows, 16 bytes at a time, each into its owner's staging slice
            __syncwarp();
            const unsigned vis_mask = __ballot_sync(0xffffffffu, visible);
            if (vis_mask && nrows > 0) {
                const int stride = row_stride(L);
                const long long e0 = a.sink.off_sh + (long long)first * L;
                if ((L & 3) == 0) {
                    for (int q = lane; q < nrows * L / 4; q += 32) {
                        const int f = q * 4, r = f / L, j = f - r * L;
                        if (!((vis_mask >> r) & 1u)) continue;
                        const float* d = rows + r * stride + j;
                        *reinterpret_cast<float4*>(sink_ptr(a.sink, e0 + f)) = make_float4(d[0], d[1], d[2], d[3]);
                    }
                } else {
                    for (int f = lane; f < nrows * L; f += 32) {
                        const int r = f / L, j = f - r * L;
                        if ((vis_mask >> r) & 1u) *sink_ptr(a.sink, e0 + f) = rows[r * stride + j];
                    }
                }
            }
        }
        if (!visible) return;
        for (int k = 0; k < 3; ++k) *sink_ptr(a.sink, a.sink.off_mean3D + 3ll * idx + k) = dmean[k];
        for (int k = 0; k < 3; ++k) *sink_ptr(a.sink, a.sink.off_scale + 3ll * idx + k) = dscale[k];
        for (int k = 0; k < 4; ++k) *sink_ptr(a.sink, a.sink.off_rot + 4ll * idx + k) = drot[k];
        return;
    }
    if (a.dL_dsh) {   // coalesced write-out of the warp's 32 gradient rows (zeros where invisible)
        __syncwarp();
        if (nrows > 0) warp_rows_out<3 * MT>(a.dL_dsh + (size_t)first * L, rows, L, nrows, lane);
    }
    if (!valid) return;
    if (AA) a.dL_dopacity[idx] = aa_h * g[5];
    // like the reference, dL_dscale is taken w.r.t. (scale_modifier * scale) and is
    // not multiplied by the modifier (backward.cu:322-325)
    a.dL_dmean3D[3 * idx + 0] = dmean[0];
    a.dL_dmean3D[3 * idx + 1] = dmean[1];
    a.dL_dmean3D[3 * idx + 2] = dmean[2];
#pragma unroll
    for (int i = 0; i < 6; ++i) a.dL_dcov3D[6 * idx + i] = dcov[i];
    a.dL_dscale[3 * idx + 0] = dscale[0];
    a.dL_dscale[3 * idx + 1] = dscale[1];
    a.dL_dscale[3 * idx + 2] = dscale[2];
    reinterpret_cast<float4*>(a.dL_drot)[idx] = make_float4(drot[0], drot[1], drot[2], drot[3]);
}
// Register budget capped for 8 resident blocks per SM (64 registers, 20 spilled words): the kernel is HBM-bound and
// gains from more loads in flight than the unconstrained 96 registers allow.
template <int MT, bool DP = false, bool AA = false>
__global__ void __launch_bounds__(PRE_THREADS, 8) preprocess_backward_kernel(const __grid_constant__ PreBwdArgs a) {
    preprocess_backward<MT, DP, AA, false>(a);
}
template <int MT, bool AA>
__global__ void __launch_bounds__(PRE_THREADS, 8)
preprocess_backward_lens_kernel(const __grid_constant__ PreBwdLensArgs a) {
    preprocess_backward<MT, false, AA, true>(a);
}

}  // namespace s3g
