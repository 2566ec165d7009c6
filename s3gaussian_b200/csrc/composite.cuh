// composite.cuh - per-tile front-to-back alpha composite, forward and backward
// (colour + depth), for sm_90a.
//
// Replaces renderCUDA forward (DGR/cuda_rasterizer/forward.cu:261-379) and
// backward (backward.cu:415-590).  Same tiles, same sorted lists, same per-pixel
// arithmetic and thresholds (power > 0, alpha < 1/255, T < 1e-4), so colour,
// depth, final_T and n_contrib reproduce the reference.  What changes is how the
// work is organised:
//
//  * a 16x16 tile is 8 warps, each owning an 8x4 pixel rectangle;
//  * batches of 256 instances are gathered global->shared with cp.async
//    (16-byte records, double buffered) while the previous batch is composited;
//  * per 32 instances, every lane tests ONE instance against the warp's
//    rectangle (exact minimum of the conic's quadratic form over the rectangle
//    vs. the Gaussian's 1/255 cut-off, see cull_tau()) and the warp only walks
//    the ballot's survivors - the all-pairs loop of the reference
//    (forward.cu:328-366) is what makes it issue-bound;
//  * a warp leaves the loop as soon as all its pixels are saturated, the block
//    as soon as all warps are;
//  * backward: two phases per warp - lane = pixel for the sequential recurrences, then
//    lane = instance for the sums over pixels (moments of X = G dL/dalpha in registers) -
//    and three vector REDs per (warp, instance) instead of 10 atomics per (pixel,
//    Gaussian) pair (backward.cu:550-587); see render_backward_kernel.
#pragma once
#include "common.cuh"

namespace s3g {

constexpr int CB = 256;          // instances per staged batch
constexpr int SUB_W = 8;         // warp rectangle
constexpr int SUB_H = 4;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// Minimum over the rectangle dx in [dxl,dxh], dy in [dyl,dyh] of
// q(dx,dy) = 0.5*(A dx^2 + C dy^2) + B dx dy  (= -power of forward.cu:338),
// for a positive-definite conic: the minimiser is the centre if it lies inside,
// otherwise it sits on one of the (at most two) edges facing the centre; the two
// clamped 1-D minimisations below cover every case.
__device__ __forceinline__ float rect_min_q(float A, float B, float C, float dxl, float dxh,
                                            float dyl, float dyh) {
    const float ddx = fminf(fmaxf(0.f, dxl), dxh);
    const float ddy = fminf(fmaxf(0.f, dyl), dyh);
    // edge dx = ddx, free dy
    const float y1 = fminf(fmaxf(__fdividef(-B * ddx, C), dyl), dyh);
    const float q1 = 0.5f * (A * ddx * ddx + C * y1 * y1) + B * ddx * y1;
    // edge dy = ddy, free dx
    const float x2 = fminf(fmaxf(__fdividef(-B * ddy, A), dxl), dxh);
    const float q2 = 0.5f * (A * x2 * x2 + C * ddy * ddy) + B * x2 * ddy;
    return fminf(q1, q2);
}

struct RenderFwdArgs {
    const uint2* ranges;
    const uint32_t* point_list;
    int W, H;
    const float4* xyAB;
    const float4* Cod;
    const float4* rgb;
    const float4* aux;       // second colour set composited on the same lists (AUX kernels), or NULL
    const float* bg;
    float* final_T;
    uint32_t* n_contrib;
    float* out_color;
    float* out_depth;
    float* out_aux;          // [3,H,W] or NULL
};

// One staged instance: 48 bytes = three 16-byte gathers.  Lane j of the cull
// test reads element j: LDS.128 at a 12-word stride is conflict-free per
// quarter-warp.
struct __align__(16) Rec {
    float4 a;   // pix.x, pix.y, conic.x, conic.y
    float4 b;   // conic.z, opacity, tau_cull, own index (bits)
    float4 c;   // r, g, b, depth
};

// AUX: a second colour set (the feature image of render(render_feat=True), train.py:373) is composited in the
// same walk - the reference runs its whole rasterizer a second time on identical geometry for it.
template <bool AUX>
__global__ void __launch_bounds__(TILE_PIX) render_forward_kernel(RenderFwdArgs a) {
    __shared__ Rec s_rec[2][CB];
    __shared__ float4 s_aux[AUX ? 2 : 1][AUX ? CB : 1];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tile = blockIdx.y * gridDim.x + blockIdx.x;
    const int X0 = blockIdx.x * TILE_X + (warp & 1) * SUB_W;
    const int Y0 = blockIdx.y * TILE_Y + (warp >> 1) * SUB_H;
    const int px = X0 + (lane & 7), py = Y0 + (lane >> 3);
    const bool inside = px < a.W && py < a.H;
    const float pixx = (float)px, pixy = (float)py;
    const uint32_t pix_id = (uint32_t)a.W * py + px;
    // rectangle of d = xy - pix over the warp's pixels
    const float rx0 = (float)X0, rx1 = (float)(X0 + SUB_W - 1);
    const float ry0 = (float)Y0, ry1 = (float)(Y0 + SUB_H - 1);

    const uint2 range = a.ranges[tile];
    const int n = (int)(range.y - range.x);
    const int nb = (n + CB - 1) / CB;

    float T = 1.0f;
    uint32_t last_contributor = 0;
    float C0 = 0.f, C1 = 0.f, C2 = 0.f, D = 0.f;
    float A0 = 0.f, A1 = 0.f, A2 = 0.f;
    bool alive = inside;

    // prologue: gather batch 0, fetch the id of batch 1
    uint32_t id_next = 0;
    if (tid < n) {
        const uint32_t id = a.point_list[range.x + tid];
        cp_async16(&s_rec[0][tid].a, &a.xyAB[id]);
        cp_async16(&s_rec[0][tid].b, &a.Cod[id]);
        cp_async16(&s_rec[0][tid].c, &a.rgb[id]);
        if (AUX) cp_async16(&s_aux[0][tid], &a.aux[id]);
    }
    cp_async_commit();
    if (CB + tid < n) id_next = a.point_list[range.x + CB + tid];
    cp_async_wait_all();
    __syncthreads();

    for (int b = 0; b < nb; ++b) {
        const int buf = b & 1;
        // prefetch batch b+1 into the other buffer, and the ids of batch b+2
        if ((b + 1) * CB + tid < n) {
            cp_async16(&s_rec[buf ^ 1][tid].a, &a.xyAB[id_next]);
            cp_async16(&s_rec[buf ^ 1][tid].b, &a.Cod[id_next]);
            cp_async16(&s_rec[buf ^ 1][tid].c, &a.rgb[id_next]);
            if (AUX) cp_async16(&s_aux[buf ^ 1][tid], &a.aux[id_next]);
        }
        cp_async_commit();
        if ((b + 2) * CB + tid < n) id_next = a.point_list[range.x + (b + 2) * CB + tid];

        const int cnt = min(CB, n - b * CB);
        const Rec* rec = s_rec[buf];
        bool warp_done = !__any_sync(0xffffffffu, alive);
        if (!warp_done) {
            for (int c0 = 0; c0 < cnt; c0 += 32) {
                const int j = c0 + lane;
                bool pass = false;
                if (j < cnt) {
                    const float4 g0 = rec[j].a;
                    const float4 g1 = rec[j].b;
                    const float q = rect_min_q(g0.z, g0.w, g1.x, g0.x - rx1, g0.x - rx0,
                                               g0.y - ry1, g0.y - ry0);
                    pass = !(q > g1.z);
                }
                uint32_t mask = __ballot_sync(0xffffffffu, pass);
                const uint32_t idx_base = (uint32_t)(b * CB + c0 + 1);
                // Branch-free body: the kernel is issue-bound and most lanes of a
                // surviving instance do blend, so predication beats divergence.
                while (mask) {
                    const int bit = __ffs(mask) - 1;
                    mask &= mask - 1;
                    const Rec& r = rec[c0 + bit];
                    const float4 g0 = r.a;
                    const float4 g1 = r.b;
                    const float4 col = r.c;
                    const float dx = g0.x - pixx, dy = g0.y - pixy;
                    const float power = -0.5f * (g0.z * dx * dx + g1.x * dy * dy) - g0.w * dx * dy;
                    const float alpha = min(0.99f, g1.y * expf(power));
                    const float test_T = T * (1 - alpha);
                    // forward.cu:339-354: skip power > 0, skip alpha < 1/255, stop at T < 1e-4
                    const bool ok = alive && !(power > 0.0f) && !(alpha < 1.0f / 255.0f);
                    const bool stop = ok && (test_T < 0.0001f);
                    const bool blend = ok && !stop;
                    // weight alpha * T once (the reference multiplies feature * alpha * T per channel,
                    // forward.cu:358-360: same value up to one rounding)
                    const float wgt = blend ? alpha * T : 0.0f;
                    C0 = fmaf(col.x, wgt, C0);
                    C1 = fmaf(col.y, wgt, C1);
                    C2 = fmaf(col.z, wgt, C2);
                    D = fmaf(col.w, wgt, D);
                    if (AUX) {
                        const float4 ax = s_aux[buf][c0 + bit];
                        A0 = fmaf(ax.x, wgt, A0);
                        A1 = fmaf(ax.y, wgt, A1);
                        A2 = fmaf(ax.z, wgt, A2);
                    }
                    T = blend ? test_T : T;
                    last_contributor = blend ? idx_base + (uint32_t)bit : last_contributor;
                    alive = alive && !stop;
                }
                if (!__any_sync(0xffffffffu, alive)) {
                    warp_done = true;
                    break;
                }
            }
        }
        cp_async_wait_all();
        if (__syncthreads_and(warp_done)) break;
    }

    if (inside) {
        const size_t HW = (size_t)a.H * a.W;
        a.final_T[pix_id] = T;
        a.n_contrib[pix_id] = last_contributor;
        a.out_color[0 * HW + pix_id] = C0 + T * a.bg[0];
        a.out_color[1 * HW + pix_id] = C1 + T * a.bg[1];
        a.out_color[2 * HW + pix_id] = C2 + T * a.bg[2];
        a.out_depth[pix_id] = D;
        if (AUX) {
            a.out_aux[0 * HW + pix_id] = A0 + T * a.bg[0];
            a.out_aux[1 * HW + pix_id] = A1 + T * a.bg[1];
            a.out_aux[2 * HW + pix_id] = A2 + T * a.bg[2];
        }
    }
}

// ---- static / dynamic decomposition (forward only) ----------------------------------------------------------------
// render(return_decomposition=True) composites the full image, the dynamic subset and the static subset.  A subset
// pass would produce the same preprocess records and, the depth and tile sorts being stable, the full tile lists with
// the other group's entries removed - so one walk over the full lists with three accumulator sets gives all three
// images.  Every instance blends into the full set and into its own group's set (bit 31 of Cod.w, set by the
// preprocess); each set runs the per-pixel sequence of render_forward_kernel on its own T and alive flag, so each image
// is what a separate pass over that subset computes.  The walk ends when all three sets are saturated.
struct RenderSplitArgs {
    RenderFwdArgs f;                 // full image (+ final_T / n_contrib, as the plain forward)
    float* out_color_d;              // [3,H,W] dynamic subset
    float* out_depth_d;
    float* out_color_s;              // [3,H,W] static subset
    float* out_depth_s;
    const uint32_t* group_count;     // dynamic Gaussians (device); a pass over no Gaussians leaves a zero image
    uint32_t P;
};

__global__ void __launch_bounds__(TILE_PIX) render_forward_split_kernel(RenderSplitArgs sa) {
    __shared__ Rec s_rec[2][CB];
    const RenderFwdArgs& a = sa.f;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tile = blockIdx.y * gridDim.x + blockIdx.x;
    const int X0 = blockIdx.x * TILE_X + (warp & 1) * SUB_W;
    const int Y0 = blockIdx.y * TILE_Y + (warp >> 1) * SUB_H;
    const int px = X0 + (lane & 7), py = Y0 + (lane >> 3);
    const bool inside = px < a.W && py < a.H;
    const float pixx = (float)px, pixy = (float)py;
    const uint32_t pix_id = (uint32_t)a.W * py + px;
    const float rx0 = (float)X0, rx1 = (float)(X0 + SUB_W - 1);
    const float ry0 = (float)Y0, ry1 = (float)(Y0 + SUB_H - 1);

    const uint2 range = a.ranges[tile];
    const int n = (int)(range.y - range.x);
    const int nb = (n + CB - 1) / CB;

    // full image, dynamic (_d) and static (_s) accumulators
    float T = 1.0f, Td = 1.0f, Ts = 1.0f;
    uint32_t last_contributor = 0;
    float C0 = 0.f, C1 = 0.f, C2 = 0.f, D = 0.f;
    float C0d = 0.f, C1d = 0.f, C2d = 0.f, Dd = 0.f;
    float C0s = 0.f, C1s = 0.f, C2s = 0.f, Ds = 0.f;
    bool alive = inside, alive_d = inside, alive_s = inside;

    uint32_t id_next = 0;
    if (tid < n) {
        const uint32_t id = a.point_list[range.x + tid];
        cp_async16(&s_rec[0][tid].a, &a.xyAB[id]);
        cp_async16(&s_rec[0][tid].b, &a.Cod[id]);
        cp_async16(&s_rec[0][tid].c, &a.rgb[id]);
    }
    cp_async_commit();
    if (CB + tid < n) id_next = a.point_list[range.x + CB + tid];
    cp_async_wait_all();
    __syncthreads();

    for (int b = 0; b < nb; ++b) {
        const int buf = b & 1;
        if ((b + 1) * CB + tid < n) {
            cp_async16(&s_rec[buf ^ 1][tid].a, &a.xyAB[id_next]);
            cp_async16(&s_rec[buf ^ 1][tid].b, &a.Cod[id_next]);
            cp_async16(&s_rec[buf ^ 1][tid].c, &a.rgb[id_next]);
        }
        cp_async_commit();
        if ((b + 2) * CB + tid < n) id_next = a.point_list[range.x + (b + 2) * CB + tid];

        const int cnt = min(CB, n - b * CB);
        const Rec* rec = s_rec[buf];
        bool warp_done = !__any_sync(0xffffffffu, alive || alive_d || alive_s);
        if (!warp_done) {
            for (int c0 = 0; c0 < cnt; c0 += 32) {
                const int j = c0 + lane;
                bool pass = false;
                if (j < cnt) {
                    const float4 g0 = rec[j].a;
                    const float4 g1 = rec[j].b;
                    const float q = rect_min_q(g0.z, g0.w, g1.x, g0.x - rx1, g0.x - rx0,
                                               g0.y - ry1, g0.y - ry0);
                    pass = !(q > g1.z);
                }
                uint32_t mask = __ballot_sync(0xffffffffu, pass);
                const uint32_t idx_base = (uint32_t)(b * CB + c0 + 1);
                while (mask) {
                    const int bit = __ffs(mask) - 1;
                    mask &= mask - 1;
                    const Rec& r = rec[c0 + bit];
                    const float4 g0 = r.a;
                    const float4 g1 = r.b;
                    const float4 col = r.c;
                    const bool dyn = (__float_as_uint(g1.w) >> 31) != 0;
                    const float dx = g0.x - pixx, dy = g0.y - pixy;
                    const float power = -0.5f * (g0.z * dx * dx + g1.x * dy * dy) - g0.w * dx * dy;
                    const float alpha = min(0.99f, g1.y * expf(power));
                    const bool vis = !(power > 0.0f) && !(alpha < 1.0f / 255.0f);
                    // full image: the sequence of render_forward_kernel
                    {
                        const float test_T = T * (1 - alpha);
                        const bool ok = alive && vis;
                        const bool stop = ok && (test_T < 0.0001f);
                        const bool blend = ok && !stop;
                        const float wgt = blend ? alpha * T : 0.0f;
                        C0 = fmaf(col.x, wgt, C0);
                        C1 = fmaf(col.y, wgt, C1);
                        C2 = fmaf(col.z, wgt, C2);
                        D = fmaf(col.w, wgt, D);
                        T = blend ? test_T : T;
                        last_contributor = blend ? idx_base + (uint32_t)bit : last_contributor;
                        alive = alive && !stop;
                    }
                    // the instance's own group: the same sequence on that group's accumulators (selected, never
                    // multiplied by zero, so the other group's image sees nothing of this instance)
                    {
                        const float Tg = dyn ? Td : Ts;
                        const bool alive_g = dyn ? alive_d : alive_s;
                        const float test_T = Tg * (1 - alpha);
                        const bool ok = alive_g && vis;
                        const bool stop = ok && (test_T < 0.0001f);
                        const bool blend = ok && !stop;
                        const float wgt = blend ? alpha * Tg : 0.0f;
                        const float n0 = fmaf(col.x, wgt, dyn ? C0d : C0s);
                        const float n1 = fmaf(col.y, wgt, dyn ? C1d : C1s);
                        const float n2 = fmaf(col.z, wgt, dyn ? C2d : C2s);
                        const float nd = fmaf(col.w, wgt, dyn ? Dd : Ds);
                        const float nT = blend ? test_T : Tg;
                        const bool nalive = alive_g && !stop;
                        if (dyn) { C0d = n0; C1d = n1; C2d = n2; Dd = nd; Td = nT; alive_d = nalive; }
                        else     { C0s = n0; C1s = n1; C2s = n2; Ds = nd; Ts = nT; alive_s = nalive; }
                    }
                }
                if (!__any_sync(0xffffffffu, alive || alive_d || alive_s)) {
                    warp_done = true;
                    break;
                }
            }
        }
        cp_async_wait_all();
        if (__syncthreads_and(warp_done)) break;
    }

    if (inside) {
        const size_t HW = (size_t)a.H * a.W;
        const uint32_t nd = *sa.group_count;
        const bool any_d = nd > 0, any_s = nd < sa.P;
        a.final_T[pix_id] = T;
        a.n_contrib[pix_id] = last_contributor;
        a.out_color[0 * HW + pix_id] = C0 + T * a.bg[0];
        a.out_color[1 * HW + pix_id] = C1 + T * a.bg[1];
        a.out_color[2 * HW + pix_id] = C2 + T * a.bg[2];
        a.out_depth[pix_id] = D;
        sa.out_color_d[0 * HW + pix_id] = any_d ? C0d + Td * a.bg[0] : 0.f;
        sa.out_color_d[1 * HW + pix_id] = any_d ? C1d + Td * a.bg[1] : 0.f;
        sa.out_color_d[2 * HW + pix_id] = any_d ? C2d + Td * a.bg[2] : 0.f;
        sa.out_depth_d[pix_id] = Dd;
        sa.out_color_s[0 * HW + pix_id] = any_s ? C0s + Ts * a.bg[0] : 0.f;
        sa.out_color_s[1 * HW + pix_id] = any_s ? C1s + Ts * a.bg[1] : 0.f;
        sa.out_color_s[2 * HW + pix_id] = any_s ? C2s + Ts * a.bg[2] : 0.f;
        sa.out_depth_s[pix_id] = Ds;
    }
}

struct RenderBwdArgs {
    const uint2* ranges;
    const uint32_t* point_list;
    int W, H;
    const float* bg;
    const float4* xyAB;
    const float4* Cod;
    const float4* rgb;
    const float* final_T;
    const uint32_t* n_contrib;
    const float* dL_dpix;        // [3,H,W]
    const float* dL_dpix_depth;  // [1,H,W]
    const float4* aux;           // second colour set (AUX kernels) or NULL
    const float* dL_dpix_aux;    // [3,H,W] or NULL
    float* grad_rec;             // [P][GRAD_REC], zeroed
};

__device__ __forceinline__ float rcp_approx(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
// one 16-byte / 8-byte reduction into a gradient record instead of four / two scalar REDs
__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d)
                 : "memory");
}
__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
    asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}

// ---- backward composite -----------------------------------------------------
// Two phases per warp (8x4 pixel rectangle), both without a cross-lane reduction per instance:
//
//  phase 1, lane = pixel (sequential in the list, as backward.cu:513-589): for every instance that survives the
//    rectangle cull the lane advances its pixel's T / accumulated-colour recurrences and leaves exactly two
//    numbers in shared memory: X = G * dL/dalpha and w = alpha * T.  Every per-Gaussian gradient the reference
//    accumulates with 10 atomics per (pixel, Gaussian) is linear in those two with pixel-only coefficients:
//        dL/dopacity = sum X            dL/dconic  = -0.5 o sum X (dx^2, dx dy, dy^2)
//        dL/dmean2D  = o sum X (-A dx - B dy, -C dy - B dx) * (W/2, H/2)
//        dL/dcolour_c = sum w dL/dpix_c        dL/ddepth = sum w dL/dpix_depth
//  phase 2, lane = (instance slot, half of the rectangle): after BKS survivors the roles flip - every lane walks
//    16 pixels of ONE instance, accumulating the six pixel-coordinate moments of X (separable: three per pixel,
//    six per row) and the four w * dL/dpix sums in registers; the halves meet with 10 shuffles, the moments are
//    shifted to the Gaussian's centre and land as three vector REDs per instance.
//
// Per surviving (warp, instance) that is ~12 issue slots of reduction instead of the 46-instruction shuffle
// butterfly + selects of a per-instance warp reduction.
constexpr int BCB = 128;          // instances per staged batch (backward)
constexpr int BKS = 16;           // survivor slots per warp
constexpr int BXW_STRIDE = 33;    // float2 row stride of the slot table: conflict-free for both phases

template <bool AUX>
struct RenderBwdSmem {
    Rec rec[2][BCB];                       // 12 KB
    float4 aux[AUX ? 2 : 1][AUX ? BCB : 1];
    float4 dpix_aux[AUX ? 8 : 1][AUX ? 32 : 1];   // dL/dpix of the second image
    float2 xw[8][BKS][BXW_STRIDE];         // 33 KB  {X, w} per (slot, pixel)
    float4 slot_a[8][BKS];                 // {pix.x, pix.y, conic.x, conic.y}
    float4 slot_b[8][BKS];                 // {conic.z, opacity, -, id bits}
    float4 dpix[8][32];                    // dL/dpix {r, g, b, depth} of the warp's pixels
    uint32_t max_contrib;
};

template <bool AUX>
__device__ __forceinline__ void bwd_flush(const RenderBwdSmem<AUX>& sm, int warp, int lane, int ns, float cx, float cy,
                                          float ddelx_dx, float ddely_dy, float* __restrict__ grad_rec) {
    const int j = lane & (BKS - 1), h = lane >> 4;
    const float2* row = &sm.xw[warp][j][h * 16];
    const float4* dp = &sm.dpix[warp][h * 16];
    float m00 = 0.f, m10 = 0.f, m20 = 0.f, m01 = 0.f, m11 = 0.f, m02 = 0.f;
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, cd = 0.f;
    float x0 = 0.f, x1 = 0.f, x2 = 0.f;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        float r0 = 0.f, r1 = 0.f, r2 = 0.f;
#pragma unroll
        for (int x = 0; x < 8; ++x) {
            const float2 v = row[rr * 8 + x];
            const float4 d = dp[rr * 8 + x];
            const float xc = (float)x - 3.5f;        // pixel x relative to the rectangle centre
            r0 += v.x;
            r1 = fmaf(v.x, xc, r1);
            r2 = fmaf(v.x, xc * xc, r2);
            c0 = fmaf(v.y, d.x, c0);
            c1 = fmaf(v.y, d.y, c1);
            c2 = fmaf(v.y, d.z, c2);
            cd = fmaf(v.y, d.w, cd);
            if (AUX) {
                const float4 e = sm.dpix_aux[warp][h * 16 + rr * 8 + x];
                x0 = fmaf(v.y, e.x, x0);
                x1 = fmaf(v.y, e.y, x1);
                x2 = fmaf(v.y, e.z, x2);
            }
        }
        const float yc = (float)(2 * h + rr) - 1.5f;
        m00 += r0; m10 += r1; m20 += r2;
        m01 = fmaf(yc, r0, m01);
        m11 = fmaf(yc, r1, m11);
        m02 = fmaf(yc * yc, r0, m02);
    }
    const uint32_t F = 0xffffffffu;
    m00 += __shfl_xor_sync(F, m00, 16); m10 += __shfl_xor_sync(F, m10, 16); m20 += __shfl_xor_sync(F, m20, 16);
    m01 += __shfl_xor_sync(F, m01, 16); m11 += __shfl_xor_sync(F, m11, 16); m02 += __shfl_xor_sync(F, m02, 16);
    c0 += __shfl_xor_sync(F, c0, 16); c1 += __shfl_xor_sync(F, c1, 16);
    c2 += __shfl_xor_sync(F, c2, 16); cd += __shfl_xor_sync(F, cd, 16);
    if (AUX) {
        x0 += __shfl_xor_sync(F, x0, 16); x1 += __shfl_xor_sync(F, x1, 16); x2 += __shfl_xor_sync(F, x2, 16);
    }
    if (j < ns) {
        const float4 ga = sm.slot_a[warp][j];
        const float4 gb = sm.slot_b[warp][j];
        // d = xy - pix = e - (pixel - centre)
        const float ex = ga.x - cx, ey = ga.y - cy;
        const float sx = ex * m00 - m10;
        const float sy = ey * m00 - m01;
        const float sxx = fmaf(ex, ex * m00 - 2.f * m10, m20);
        const float syy = fmaf(ey, ey * m00 - 2.f * m01, m02);
        const float sxy = fmaf(ex, ey * m00 - m01, m11 - ey * m10);
        const float o = gb.y, hf = -0.5f * o;
        float* g = grad_rec + (size_t)__float_as_uint(gb.w) * GRAD_REC;
        if (h == 0) {
            red_add_v4(g, o * ddelx_dx * (-ga.z * sx - ga.w * sy), o * ddely_dy * (-gb.x * sy - ga.w * sx), hf * sxx,
                       hf * sxy);
            if (AUX) red_add_v4(g + 8, c2, cd, x0, x1);
            else red_add_v2(g + 8, c2, cd);
        } else {
            red_add_v4(g + 4, hf * syy, m00, c0, c1);
            if (AUX) atomicAdd(g + 12, x2);
        }
    }
}

template <bool AUX>
__global__ void __launch_bounds__(TILE_PIX) render_backward_kernel(RenderBwdArgs a) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    RenderBwdSmem<AUX>& sm = *reinterpret_cast<RenderBwdSmem<AUX>*>(s_raw);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t tile = blockIdx.y * gridDim.x + blockIdx.x;
    const int X0 = blockIdx.x * TILE_X + (warp & 1) * SUB_W;
    const int Y0 = blockIdx.y * TILE_Y + (warp >> 1) * SUB_H;
    const int px = X0 + (lane & 7), py = Y0 + (lane >> 3);
    const bool inside = px < a.W && py < a.H;
    const float pixx = (float)px, pixy = (float)py;
    const uint32_t pix_id = (uint32_t)a.W * py + px;
    const float rx0 = (float)X0, rx1 = (float)(X0 + SUB_W - 1);
    const float ry0 = (float)Y0, ry1 = (float)(Y0 + SUB_H - 1);
    const float cx = (float)X0 + 3.5f, cy = (float)Y0 + 1.5f;
    const size_t HW = (size_t)a.H * a.W;

    const uint2 range = a.ranges[tile];

    const float T_final = inside ? a.final_T[pix_id] : 0.f;
    float T = T_final;
    const int last_contributor = inside ? (int)a.n_contrib[pix_id] : 0;
    float dpix0 = 0.f, dpix1 = 0.f, dpix2 = 0.f, dpixd = 0.f;
    if (inside) {
        dpix0 = a.dL_dpix[0 * HW + pix_id];
        dpix1 = a.dL_dpix[1 * HW + pix_id];
        dpix2 = a.dL_dpix[2 * HW + pix_id];
        dpixd = a.dL_dpix_depth[pix_id];
    }
    sm.dpix[warp][lane] = make_float4(dpix0, dpix1, dpix2, dpixd);
    float dax0 = 0.f, dax1 = 0.f, dax2 = 0.f;
    if (AUX) {
        if (inside) {
            dax0 = a.dL_dpix_aux[0 * HW + pix_id];
            dax1 = a.dL_dpix_aux[1 * HW + pix_id];
            dax2 = a.dL_dpix_aux[2 * HW + pix_id];
        }
        sm.dpix_aux[warp][lane] = make_float4(dax0, dax1, dax2, 0.f);
    }
    // -(T_final * sum_c bg_c dL/dpix_c): the background term of backward.cu:564-567 (both images share bg)
    const float nbg = -T_final * (a.bg[0] * (dpix0 + dax0) + a.bg[1] * (dpix1 + dax1) + a.bg[2] * (dpix2 + dax2));

    // only instances below the block's deepest contributor matter (backward.cu:513)
    if (tid == 0) sm.max_contrib = 0;
    __syncthreads();
    const int warp_max = (int)__reduce_max_sync(0xffffffffu, (uint32_t)last_contributor);
    if (lane == 0 && warp_max > 0) atomicMax(&sm.max_contrib, (uint32_t)warp_max);
    __syncthreads();
    const int m = (int)sm.max_contrib;   // instances [0, m) are walked back to front
    const int nb = (m + BCB - 1) / BCB;
    if (nb == 0) return;

    // per-pixel recurrences of backward.cu:529-563.  The reference keeps accum_rec per channel and forms
    // sum_c (c_c - accum_c) dL/dpix_c; the same quantity with the dot products taken first:
    //   cd_i = sum_c colour_c(i) dL/dpix_c + depth(i) dL/dpix_depth,   A <- last_alpha * last_cd + (1 - last_alpha) * A,
    //   dL/dalpha = cd_i - A
    float A = 0.f, last_alpha = 0.f, last_cd = 0.f;
    const float ddelx_dx = 0.5f * a.W, ddely_dy = 0.5f * a.H;
    int ns = 0;   // filled survivor slots (warp-uniform)

    // slot t of batch b holds list index m-1-(b*BCB+t); threads >= BCB only composite
    uint32_t id_next = 0;
    {
        const int i0 = m - 1 - tid;
        if (tid < BCB && i0 >= 0) {
            const uint32_t id = a.point_list[range.x + i0];
            cp_async16(&sm.rec[0][tid].a, &a.xyAB[id]);
            cp_async16(&sm.rec[0][tid].b, &a.Cod[id]);
            cp_async16(&sm.rec[0][tid].c, &a.rgb[id]);
            if (AUX) cp_async16(&sm.aux[0][tid], &a.aux[id]);
        }
        cp_async_commit();
        const int i1 = m - 1 - (BCB + tid);
        if (tid < BCB && i1 >= 0) id_next = a.point_list[range.x + i1];
        cp_async_wait_all();
        __syncthreads();
    }

    for (int b = 0; b < nb; ++b) {
        const int buf = b & 1;
        if (tid < BCB) {
            const int i1 = m - 1 - ((b + 1) * BCB + tid);
            if (i1 >= 0) {
                cp_async16(&sm.rec[buf ^ 1][tid].a, &a.xyAB[id_next]);
                cp_async16(&sm.rec[buf ^ 1][tid].b, &a.Cod[id_next]);
                cp_async16(&sm.rec[buf ^ 1][tid].c, &a.rgb[id_next]);
                if (AUX) cp_async16(&sm.aux[buf ^ 1][tid], &a.aux[id_next]);
            }
            const int i2 = m - 1 - ((b + 2) * BCB + tid);
            if (i2 >= 0) id_next = a.point_list[range.x + i2];
        }
        cp_async_commit();
        const int top = m - 1 - b * BCB;           // list index of slot 0
        const int cnt = min(BCB, top + 1);
        const Rec* rec = sm.rec[buf];
        // the warp has nothing to do for instances at or above warp_max
        if (top - (cnt - 1) < warp_max) {
            for (int c0 = 0; c0 < cnt; c0 += 32) {
                const int jc = c0 + lane;
                bool pass = false;
                if (jc < cnt && top - jc < warp_max) {
                    const float4 g0 = rec[jc].a;
                    const float4 g1 = rec[jc].b;
                    const float q = rect_min_q(g0.z, g0.w, g1.x, g0.x - rx1, g0.x - rx0,
                                               g0.y - ry1, g0.y - ry0);
                    pass = !(q > g1.z);
                }
                uint32_t mask = __ballot_sync(0xffffffffu, pass);
                while (mask) {
                    const int jj = c0 + __ffs(mask) - 1;
                    mask &= mask - 1;
                    const int contributor = top - jj;   // 0-based list index
                    const Rec& r = rec[jj];
                    const float4 g0 = r.a;
                    const float4 g1 = r.b;
                    const float dx = g0.x - pixx, dy = g0.y - pixy;
                    const float power = -0.5f * (g0.z * dx * dx + g1.x * dy * dy) - g0.w * dx * dy;
                    // (ex2.approx here with a fall-back to the exact sequence in a band around alpha = 1/255 - the one
                    //  decision that must agree with the forward, or T is off by that pair's factor - was measured
                    //  slower on an earlier GPU: the reconvergence point costs more than the instructions saved)
                    const float G = expf(power);
                    const float alpha = min(0.99f, g1.y * G);
                    const bool contrib = contributor < last_contributor && !(power > 0.0f) &&
                                         !(alpha < 1.0f / 255.0f);
                    if (!__any_sync(0xffffffffu, contrib)) continue;
                    float X = 0.f, w = 0.f;
                    if (contrib) {
                        const float4 col = r.c;
                        // 1/(1-alpha): alpha <= 0.99, approx reciprocal (1 ulp) instead of
                        // the two IEEE divisions of backward.cu:529,567
                        const float inv = rcp_approx(1.f - alpha);
                        T = T * inv;
                        w = alpha * T;
                        A = last_alpha * last_cd + (1.f - last_alpha) * A;
                        float cdv = col.x * dpix0 + col.y * dpix1 + col.z * dpix2 + col.w * dpixd;
                        if (AUX) {
                            const float4 ax = sm.aux[buf][jj];
                            cdv += ax.x * dax0 + ax.y * dax1 + ax.z * dax2;
                        }
                        last_cd = cdv;
                        last_alpha = alpha;
                        X = G * ((cdv - A) * T + nbg * inv);
                    }
                    sm.xw[warp][ns][lane] = make_float2(X, w);
                    if (lane == 0) {
                        sm.slot_a[warp][ns] = g0;
                        sm.slot_b[warp][ns] = g1;
                    }
                    if (++ns == BKS) {
                        __syncwarp();
                        bwd_flush(sm, warp, lane, BKS, cx, cy, ddelx_dx, ddely_dy, a.grad_rec);
                        __syncwarp();
                        ns = 0;
                    }
                }
            }
        }
        cp_async_wait_all();
        __syncthreads();
    }
    if (ns) {
        __syncwarp();
        bwd_flush(sm, warp, lane, ns, cx, cy, ddelx_dx, ddely_dy, a.grad_rec);
    }
}

}  // namespace s3g
