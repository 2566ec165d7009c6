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
//  * forward: one walk for the training image, the extra colour sets (feature or
//    flow images) and the static/dynamic decomposition; see render_forward_kernel;
//  * backward: two phases per warp - lane = pixel for the sequential recurrences, then
//    lane = instance for the sums over pixels (moments of X = G dL/dalpha in registers) -
//    and one record per (warp, instance) instead of 10 atomics per (pixel, Gaussian) pair
//    (backward.cu:550-587).  One walk, two destinations for the record: three vector REDs
//    into grad_rec, or (deterministic backward) per-warp shared-memory partials summed in a
//    fixed order; see render_backward_kernel.
#pragma once
#include <type_traits>

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
    const float4* aux;       // first extra colour set composited on the same lists (NA >= 1 kernels), or NULL
    const float* bg;
    float* final_T;
    uint32_t* n_contrib;
    float* out_color;
    float* out_depth;
    float* out_aux;          // [3,H,W] or NULL
};

// The second extra colour set of a two-set walk (the two flow images of an evaluation walk).  It is a kernel parameter
// of its own so that the forward's argument structs keep their layout, and the kernels with fewer sets their code.
struct AuxSet {
    const float4* colors;    // [P], rgb in .xyz, indexed by Gaussian
    float* out;              // [3,H,W]
};

// extra colour set k of a walk: set 0 travels in RenderFwdArgs (aux / out_aux), set 1 in the AuxSet parameter
__device__ __forceinline__ const float4* aux_colors(const RenderFwdArgs& a, const AuxSet& a1, int k) {
    return k == 0 ? a.aux : a1.colors;
}
__device__ __forceinline__ float* aux_out(const RenderFwdArgs& a, const AuxSet& a1, int k) {
    return k == 0 ? a.out_aux : a1.out;
}

// One staged instance: 48 bytes = three 16-byte gathers.  Lane j of the cull
// test reads element j: LDS.128 at a 12-word stride is conflict-free per
// quarter-warp.
struct __align__(16) Rec {
    float4 a;   // pix.x, pix.y, conic.x, conic.y
    float4 b;   // conic.z, opacity, tau_cull, own index (bits)
    float4 c;   // r, g, b, depth
};

// the split walk's outputs: the dynamic and static subset images
struct RenderSplitArgs : RenderFwdArgs {
    float* out_color_d;              // [3,H,W] dynamic subset
    float* out_depth_d;
    float* out_color_s;              // [3,H,W] static subset
    float* out_depth_s;
    const uint32_t* group_count;     // dynamic Gaussians (device); a pass over no Gaussians leaves a zero image
    uint32_t P;
};

// {dynamic Gaussians, P} of a split walk; the epilogue reads them before its stores, which may alias group_count
__device__ __forceinline__ uint2 split_counts(const RenderFwdArgs&) { return make_uint2(0u, 0u); }
__device__ __forceinline__ uint2 split_counts(const RenderSplitArgs& s) { return make_uint2(*s.group_count, s.P); }

// The opacity images of an opacity walk (render_forward_opacity_kernel), each [1,H,W] or NULL:
//   alpha(p)        = 1 - T_final(p), T_final the transmittance the background is blended with, so
//                     colour = colour with bg 0 + (1 - alpha) bg exactly;
//   median_depth(p) = depth of the first contributor, front to back, whose blend takes T from > 0.5 to <= 0.5, 0
//                     where T never gets there;
//   alpha_d, alpha_s (SPLIT) the alpha images of the dynamic and static subsets.
// median_contrib (NULL: not kept) receives the 1-based list position of the median contributor, 0 for none (the
// convention of n_contrib), which the opacity backward reads to route dL/dmedian.
struct OpacityOut {
    float* alpha;
    float* median_depth;
    float* alpha_d;
    float* alpha_s;
    uint32_t* median_contrib;
};

// One walk over a tile's sorted list composites the colour image and depth (with final_T and n_contrib), and also:
//  * NA extra colour sets with the colour image's weights and background: the feature image of render(render_feat=True)
//    (train.py:373; NA = 1) or the flow images of an evaluation walk (NA = 1 or 2), for each of which the reference
//    runs its whole rasterizer again on identical geometry;
//  * SPLIT: the dynamic and static subset images of render(return_decomposition=True).  A subset pass would produce
//    the same preprocess records and, the depth and tile sorts being stable, the full tile lists without the other
//    group's entries - so every instance blends into the full set and into its own group's set (bit 31 of Cod.w, set
//    by the preprocess), each set running the same per-pixel sequence on its own T and alive flag.  Each image is what
//    a separate pass over its subset computes; the walk ends when all three sets are saturated;
//  * OPA: the opacity images of OpacityOut.  Only the opacity kernels instantiate it; the others keep their code.
template <int NA, bool SPLIT, bool OPA>
__device__ __forceinline__ void render_forward_walk(std::conditional_t<SPLIT, RenderSplitArgs, RenderFwdArgs> args,
                                                    AuxSet a1, OpacityOut opa) {
    static_assert(NA >= 0 && NA <= 2, "at most two extra colour sets");
    __shared__ Rec s_rec[2][CB];
    __shared__ float4 s_aux[NA ? NA : 1][NA ? 2 : 1][NA ? CB : 1];
    const RenderFwdArgs& a = args;

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

    // full image, and (SPLIT) dynamic (_d) and static (_s) accumulators
    float T = 1.0f, Td = 1.0f, Ts = 1.0f;
    uint32_t last_contributor = 0;
    float C0 = 0.f, C1 = 0.f, C2 = 0.f, D = 0.f;
    float C0d = 0.f, C1d = 0.f, C2d = 0.f, Dd = 0.f;
    float C0s = 0.f, C1s = 0.f, C2s = 0.f, Ds = 0.f;
    float A[NA ? NA : 1][3] = {};
    bool alive = inside, alive_d = inside, alive_s = inside;
    float Dm = 0.f;                  // OPA: median depth and its list position
    uint32_t median_contrib = 0;

    // prologue: gather batch 0, fetch the id of batch 1
    uint32_t id_next = 0;
    if (tid < n) {
        const uint32_t id = a.point_list[range.x + tid];
        cp_async16(&s_rec[0][tid].a, &a.xyAB[id]);
        cp_async16(&s_rec[0][tid].b, &a.Cod[id]);
        cp_async16(&s_rec[0][tid].c, &a.rgb[id]);
#pragma unroll
        for (int k = 0; k < NA; ++k) cp_async16(&s_aux[k][0][tid], &aux_colors(a, a1, k)[id]);
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
#pragma unroll
            for (int k = 0; k < NA; ++k) cp_async16(&s_aux[k][buf ^ 1][tid], &aux_colors(a, a1, k)[id_next]);
        }
        cp_async_commit();
        if ((b + 2) * CB + tid < n) id_next = a.point_list[range.x + (b + 2) * CB + tid];

        const int cnt = min(CB, n - b * CB);
        const Rec* rec = s_rec[buf];
        bool warp_done = !__any_sync(0xffffffffu, SPLIT ? alive || alive_d || alive_s : alive);
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
                    const bool dyn = (__float_as_uint(g1.w) >> 31) != 0;   // SPLIT: the instance's group
                    const float dx = g0.x - pixx, dy = g0.y - pixy;
                    const float power = -0.5f * (g0.z * dx * dx + g1.x * dy * dy) - g0.w * dx * dy;
                    const float alpha = min(0.99f, g1.y * expf(power));
                    // forward.cu:339-354: skip power > 0, skip alpha < 1/255, stop at T < 1e-4
                    const bool vis = !(power > 0.0f) && !(alpha < 1.0f / 255.0f);
                    const float test_T = T * (1 - alpha);
                    // alive && vis (spelled out for the plain walk: through vis, nvcc 12.9 reorders its predicates)
                    const bool ok = SPLIT ? alive && vis : alive && !(power > 0.0f) && !(alpha < 1.0f / 255.0f);
                    const bool stop = ok && (test_T < 0.0001f);
                    const bool blend = ok && !stop;
                    // weight alpha * T once (the reference multiplies feature * alpha * T per channel,
                    // forward.cu:358-360: same value up to one rounding)
                    const float wgt = blend ? alpha * T : 0.0f;
                    C0 = fmaf(col.x, wgt, C0);
                    C1 = fmaf(col.y, wgt, C1);
                    C2 = fmaf(col.z, wgt, C2);
                    D = fmaf(col.w, wgt, D);
#pragma unroll
                    for (int k = 0; k < NA; ++k) {
                        const float4 ax = s_aux[k][buf][c0 + bit];
                        A[k][0] = fmaf(ax.x, wgt, A[k][0]);
                        A[k][1] = fmaf(ax.y, wgt, A[k][1]);
                        A[k][2] = fmaf(ax.z, wgt, A[k][2]);
                    }
                    if constexpr (OPA) {
                        // T only falls, so at most one blend per pixel crosses 0.5
                        const bool med = blend && T > 0.5f && test_T <= 0.5f;
                        Dm = med ? col.w : Dm;
                        median_contrib = med ? idx_base + (uint32_t)bit : median_contrib;
                    }
                    T = blend ? test_T : T;
                    last_contributor = blend ? idx_base + (uint32_t)bit : last_contributor;
                    alive = alive && !stop;
                    if constexpr (SPLIT) {
                        // the instance's own group: the same sequence on that group's accumulators (selected, never
                        // multiplied by zero, so the other group's image sees nothing of this instance)
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
                if (!__any_sync(0xffffffffu, SPLIT ? alive || alive_d || alive_s : alive)) {
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
        const uint2 gc = split_counts(args);
        const bool any_d = gc.x > 0, any_s = gc.x < gc.y;   // a pass over no Gaussians leaves a zero image
        a.final_T[pix_id] = T;
        a.n_contrib[pix_id] = last_contributor;
        a.out_color[0 * HW + pix_id] = C0 + T * a.bg[0];
        a.out_color[1 * HW + pix_id] = C1 + T * a.bg[1];
        a.out_color[2 * HW + pix_id] = C2 + T * a.bg[2];
        a.out_depth[pix_id] = D;
        if constexpr (SPLIT) {
            args.out_color_d[0 * HW + pix_id] = any_d ? C0d + Td * a.bg[0] : 0.f;
            args.out_color_d[1 * HW + pix_id] = any_d ? C1d + Td * a.bg[1] : 0.f;
            args.out_color_d[2 * HW + pix_id] = any_d ? C2d + Td * a.bg[2] : 0.f;
            args.out_depth_d[pix_id] = Dd;
            args.out_color_s[0 * HW + pix_id] = any_s ? C0s + Ts * a.bg[0] : 0.f;
            args.out_color_s[1 * HW + pix_id] = any_s ? C1s + Ts * a.bg[1] : 0.f;
            args.out_color_s[2 * HW + pix_id] = any_s ? C2s + Ts * a.bg[2] : 0.f;
            args.out_depth_s[pix_id] = Ds;
        }
#pragma unroll
        for (int k = 0; k < NA; ++k) {
            float* o = aux_out(a, a1, k);
            o[0 * HW + pix_id] = A[k][0] + T * a.bg[0];
            o[1 * HW + pix_id] = A[k][1] + T * a.bg[1];
            o[2 * HW + pix_id] = A[k][2] + T * a.bg[2];
        }
        if constexpr (OPA) {
            if (opa.alpha) opa.alpha[pix_id] = 1.f - T;
            if (opa.median_depth) opa.median_depth[pix_id] = Dm;
            if (opa.median_contrib) opa.median_contrib[pix_id] = median_contrib;
            if constexpr (SPLIT) {
                if (opa.alpha_d) {   // a subset with no Gaussians keeps T = 1: alpha 0, as a pass over it gives
                    opa.alpha_d[pix_id] = 1.f - Td;
                    opa.alpha_s[pix_id] = 1.f - Ts;
                }
            }
        }
    }
}

template <int NA, bool SPLIT>
__global__ void __launch_bounds__(TILE_PIX)
    render_forward_kernel(std::conditional_t<SPLIT, RenderSplitArgs, RenderFwdArgs> args, AuxSet a1) {
    render_forward_walk<NA, SPLIT, false>(args, a1, OpacityOut{});
}

// the same walk, also writing the opacity images (s3g_rasterize_forward_opacity)
template <int NA, bool SPLIT>
__global__ void __launch_bounds__(TILE_PIX)
    render_forward_opacity_kernel(std::conditional_t<SPLIT, RenderSplitArgs, RenderFwdArgs> args, AuxSet a1,
                                  OpacityOut opa) {
    render_forward_walk<NA, SPLIT, true>(args, a1, opa);
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
    float* grad_rec;             // [P][GRAD_REC], zeroed (default walk only)
    // OPA kernels: gradients of the opacity images (each [1,H,W] or NULL) and, with dL_dpix_median, the forward's
    // median list positions (OpacityOut::median_contrib)
    const float* dL_dpix_alpha;
    const float* dL_dpix_median;
    const uint32_t* median_contrib;
};
// the deterministic walk's destination
struct RenderBwdDetArgs : RenderBwdArgs {
    const ushort4* rect;         // [P] of the forward
    const uint32_t* base;        // [P], det_base_kernel
    float4* records;             // [R][GRAD_REC / 4]
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
//    six per row) and the four w * dL/dpix sums in registers; the halves meet with 10 shuffles and the moments are
//    shifted to the Gaussian's centre (bwd_flush).
//
// Per surviving (warp, instance) that is ~12 issue slots of reduction instead of the 46-instruction shuffle
// butterfly + selects of a per-instance warp reduction.
//
// The same walk has two destinations for a flushed record (bwd_store):
//  * default (s3g_rasterize_backward): three vector REDs per (warp, instance) into the Gaussian's grad_rec row, in
//    whatever order warps and tiles get there - so two calls on the same inputs differ in the last bits;
//  * deterministic (s3g_rasterize_backward_deterministic, DET): every sum is taken in an order fixed by the inputs.
//    A flush stores into the warp's shared-memory partial of the batch slot; at the end of each batch of DCB
//    instances the block adds the eight warps' partials in warp order and writes one record per (tile, instance)
//    to the workspace at its emit position.  Partials a warp never writes (no surviving pixel, a warp past its last
//    contributor) stay zero, and instances behind the tile's deepest contributor get a zero record, so no stale
//    workspace content is ever read.  Around the walk:
//      - det_base_kernel: base[g] = position of Gaussian g's first tile instance in emit order (the forward's
//        exclusive scan `offsets`, indexed through the depth order).  Instance (g, tile t) has emit position
//        base[g] + (row-major index of t in g's rect), exactly as emit_instances_kernel numbered it.
//      - grad_rec_gather_kernel: every Gaussian's records summed over its tiles in row-major order, written as its
//        full grad_rec row (this replaces the memset of the default path).
//    No global atomics anywhere; preprocess_backward then reads grad_rec as it does after the default path.
constexpr int BCB = 128;          // instances per staged batch (default)
constexpr int DCB = 64;           // instances per staged batch (deterministic)
constexpr int BKS = 16;           // survivor slots per warp
constexpr int BXW_STRIDE = 33;    // float2 row stride of the slot table: conflict-free for both phases

// deterministic workspace: [R][GRAD_REC] floats of per-(tile, instance) records in emit order, then [P] uint32 base
// offsets
__host__ __device__ inline size_t det_records_bytes(int64_t R) { return (size_t)R * GRAD_REC * sizeof(float); }

__global__ void det_base_kernel(uint32_t P, const uint32_t* __restrict__ order, const uint32_t* __restrict__ offsets,
                                uint32_t* __restrict__ base) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < P) base[order[k]] = offsets[k];
}

// emit position of instance (Gaussian g, tile tx, ty): emit_instances_kernel numbers a Gaussian's tiles row-major
// over its rect, starting at base[g]
__device__ __forceinline__ size_t det_emit_pos(const ushort4* __restrict__ rect, const uint32_t* __restrict__ base,
                                               uint32_t g, uint32_t tx, uint32_t ty) {
    const ushort4 r = rect[g];
    return (size_t)base[g] + (ty - r.y) * (uint32_t)(r.z - r.x) + (tx - r.x);
}

// shared memory of the walk, batches of NB instances
template <bool AUX, int NB>
struct BwdWalkSmem {
    Rec rec[2][NB];
    float4 aux[AUX ? 2 : 1][AUX ? NB : 1];
    float4 dpix_aux[AUX ? 8 : 1][AUX ? 32 : 1];   // dL/dpix of the second image
    float2 xw[8][BKS][BXW_STRIDE];         // 33 KB  {X, w} per (slot, pixel)
    float4 slot_a[8][BKS];                 // {pix.x, pix.y, conic.x, conic.y}
    float4 slot_b[8][BKS];                 // {conic.z, opacity, batch slot (bits) if DET, id bits}
    float4 dpix[8][32];                    // dL/dpix {r, g, b, depth} of the warp's pixels
};
// OPA: per (warp, slot), dL/dmedian summed over the warp's pixels whose median the slot's instance is (an empty base
// otherwise, so the other walks keep their layout)
template <bool OPA>
struct BwdMedianSlots {
    float med[8][BKS];
};
template <>
struct BwdMedianSlots<false> {};
// ABS: the walk also keeps the absolute screen-space gradients in record entries 13 and 14, so quarter 3 is written
// with or without AUX
template <bool AUX, bool DET, bool OPA, bool ABS = false>
struct RenderBwdSmem : BwdWalkSmem<AUX, BCB>, BwdMedianSlots<OPA> {
    uint32_t max_contrib;
};
template <bool AUX, bool OPA, bool ABS>
struct RenderBwdSmem<AUX, true, OPA, ABS> : BwdWalkSmem<AUX, DCB>, BwdMedianSlots<OPA> {
    float4 part[(AUX || ABS) ? 4 : 3][8][DCB];   // [record quarter][warp][batch slot]; zero unless written this batch
    uint32_t max_contrib;
};

// quarter q of a flushed record to its destination: row g of grad_rec, or this warp's partial of batch slot `slot`
// (DET).  Each batch slot is flushed at most once per warp and batch.
template <bool AUX, bool DET, bool OPA, bool ABS = false>
__device__ __forceinline__ void bwd_store(RenderBwdSmem<AUX, DET, OPA, ABS>& sm, int warp, float* g, int slot, int q,
                                          float4 v) {
    if constexpr (DET) {
        sm.part[q][warp][slot] = v;
    } else {
        if (q == 3 && ABS) red_add_v4(g + 4 * q, v.x, v.y, v.z, v.w);   // entry 13 is not 8-byte aligned
        else if (q == 3) atomicAdd(g + 4 * q, v.x);
        else if (q == 2 && !AUX) red_add_v2(g + 4 * q, v.x, v.y);
        else red_add_v4(g + 4 * q, v.x, v.y, v.z, v.w);
    }
}

// lane (j, h) sums slot j's moments over half h of the rectangle; after the shuffles it holds the record's quarters
// 0 and 2 (h == 0) or 1 and 3 (h == 1, quarter 3 with AUX or ABS only) and stores them.
// ABS: the lane also sums, per pixel p, |X_p (A dx_p + B dy_p)| and |X_p (C dy_p + B dx_p)| with d_p = mean2D - pixel,
// the absolute values of the pixel's signed dL/dmean2D terms before the factors o W/2 and o H/2 (o > 0, applied once
// at the end); they go to record entries 13 and 14.
template <bool AUX, bool DET, bool OPA, bool ABS = false>
__device__ __forceinline__ void bwd_flush(RenderBwdSmem<AUX, DET, OPA, ABS>& sm, int warp, int lane, int ns, float cx,
                                          float cy, float ddelx_dx, float ddely_dy, float* __restrict__ grad_rec) {
    const int j = lane & (BKS - 1), h = lane >> 4;
    const float2* row = &sm.xw[warp][j][h * 16];
    const float4* dp = &sm.dpix[warp][h * 16];
    float m00 = 0.f, m10 = 0.f, m20 = 0.f, m01 = 0.f, m11 = 0.f, m02 = 0.f;
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, cd = 0.f;
    float x0 = 0.f, x1 = 0.f, x2 = 0.f;
    float ax = 0.f, ay = 0.f;                    // ABS: the two absolute sums
    float ca = 0.f, cb = 0.f, cc = 0.f, ex0 = 0.f, ey0 = 0.f;
    if constexpr (ABS) {
        // slot j's conic and centre offset (stale for j >= ns: those lanes store nothing)
        const float4 ga = sm.slot_a[warp][j];
        ca = ga.z; cb = ga.w; cc = sm.slot_b[warp][j].x;
        ex0 = ga.x - cx; ey0 = ga.y - cy;
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
        float r0 = 0.f, r1 = 0.f, r2 = 0.f;
        float tx0 = 0.f, ty0 = 0.f;              // ABS: A dx + B dy and C dy + B dx at the row's centre column
        if constexpr (ABS) {
            const float dyr = ey0 - ((float)(2 * h + rr) - 1.5f);
            tx0 = fmaf(cb, dyr, ca * ex0);
            ty0 = fmaf(cb, ex0, cc * dyr);
        }
#pragma unroll
        for (int x = 0; x < 8; ++x) {
            const float2 v = row[rr * 8 + x];
            const float4 d = dp[rr * 8 + x];
            const float xc = (float)x - 3.5f;        // pixel x relative to the rectangle centre
            if constexpr (ABS) {
                // dx_p = ex0 - xc: the row's terms shifted by -xc along x
                ax += fabsf(v.x * fmaf(-ca, xc, tx0));
                ay += fabsf(v.x * fmaf(-cb, xc, ty0));
            }
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
    if (ABS) {
        ax += __shfl_xor_sync(F, ax, 16); ay += __shfl_xor_sync(F, ay, 16);
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
        // the record's destination: the Gaussian's grad_rec row, or (DET) its batch slot
        float* g = grad_rec + (size_t)__float_as_uint(gb.w) * GRAD_REC;
        const int slot = __float_as_int(gb.z);
        if (h == 0) {
            bwd_store(sm, warp, g, slot, 0, make_float4(o * ddelx_dx * (-ga.z * sx - ga.w * sy),
                                                        o * ddely_dy * (-gb.x * sy - ga.w * sx), hf * sxx, hf * sxy));
            if constexpr (OPA) cd += sm.med[warp][j];                        // the median depth's weight-1 term
            bwd_store(sm, warp, g, slot, 2, make_float4(c2, cd, x0, x1));   // x0 = x1 = 0 without AUX
        } else {
            bwd_store(sm, warp, g, slot, 1, make_float4(hf * syy, m00, c0, c1));
            if constexpr (ABS)   // x2 = 0 without AUX
                bwd_store(sm, warp, g, slot, 3, make_float4(x2, o * ddelx_dx * ax, o * ddely_dy * ay, 0.f));
            else if constexpr (AUX) bwd_store(sm, warp, g, slot, 3, make_float4(x2, 0.f, 0.f, 0.f));
        }
    }
}

// OPA: the gradients of the opacity images join the walk.  alpha = 1 - T_final has dalpha/dalpha_i = T_final / (1 -
// alpha_i), the form of the background term, so T_final dL/dalpha joins nbg; dL/dmedian goes, with weight 1, into the
// depth sum of the one instance at the pixel's median position.  Both end in the same records as every other term.
// ABS: the absolute screen-space gradients as well (bwd_flush), in record entries 13 and 14.
template <bool AUX, bool DET, bool OPA, bool ABS = false>
__global__ void __launch_bounds__(TILE_PIX)
    render_backward_kernel(std::conditional_t<DET, RenderBwdDetArgs, RenderBwdArgs> args) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    RenderBwdSmem<AUX, DET, OPA, ABS>& sm = *reinterpret_cast<RenderBwdSmem<AUX, DET, OPA, ABS>*>(s_raw);
    const RenderBwdArgs& a = args;
    constexpr int NB = DET ? DCB : BCB;          // instances per staged batch
    constexpr int NQ = (AUX || ABS) ? 4 : 3;     // record quarters written

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
    const int n = (int)(range.y - range.x);

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
    float nbg = -T_final * (a.bg[0] * (dpix0 + dax0) + a.bg[1] * (dpix1 + dax1) + a.bg[2] * (dpix2 + dax2));
    float dmed = 0.f;               // OPA: dL/dmedian of the pixel and its median's 1-based list position (0: none)
    int median_contrib = 0;
    if constexpr (OPA) {
        if (inside && a.dL_dpix_alpha) nbg = fmaf(T_final, a.dL_dpix_alpha[pix_id], nbg);
        if (inside && a.dL_dpix_median) {
            dmed = a.dL_dpix_median[pix_id];
            median_contrib = (int)a.median_contrib[pix_id];
        }
    }

    // only instances below the block's deepest contributor matter (backward.cu:513)
    if (tid == 0) sm.max_contrib = 0;
    if constexpr (DET)
        for (int i = tid; i < NQ * 8 * DCB; i += TILE_PIX) (&sm.part[0][0][0])[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    const int warp_max = (int)__reduce_max_sync(0xffffffffu, (uint32_t)last_contributor);
    if (lane == 0 && warp_max > 0) atomicMax(&sm.max_contrib, (uint32_t)warp_max);
    __syncthreads();
    const int m = (int)sm.max_contrib;   // instances [0, m) are walked back to front
    if constexpr (DET) {
        // instances behind the deepest contributor get a zero record
        for (int i = m + tid; i < n; i += TILE_PIX) {
            const uint32_t g = a.point_list[range.x + i];
            float4* dst =
                args.records + det_emit_pos(args.rect, args.base, g, blockIdx.x, blockIdx.y) * (GRAD_REC / 4);
#pragma unroll
            for (int q = 0; q < NQ; ++q) dst[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    }
    const int nb = (m + NB - 1) / NB;
    if (nb == 0) return;

    // per-pixel recurrences of backward.cu:529-563.  The reference keeps accum_rec per channel and forms
    // sum_c (c_c - accum_c) dL/dpix_c; the same quantity with the dot products taken first:
    //   cd_i = sum_c colour_c(i) dL/dpix_c + depth(i) dL/dpix_depth,   A <- last_alpha * last_cd + (1 - last_alpha) * A,
    //   dL/dalpha = cd_i - A
    float A = 0.f, last_alpha = 0.f, last_cd = 0.f;
    const float ddelx_dx = 0.5f * a.W, ddely_dy = 0.5f * a.H;
    int ns = 0;   // filled survivor slots (warp-uniform)

    // slot t of batch b holds list index m-1-(b*NB+t); threads >= NB only composite
    uint32_t id_next = 0;
    {
        const int i0 = m - 1 - tid;
        if (tid < NB && i0 >= 0) {
            const uint32_t id = a.point_list[range.x + i0];
            cp_async16(&sm.rec[0][tid].a, &a.xyAB[id]);
            cp_async16(&sm.rec[0][tid].b, &a.Cod[id]);
            cp_async16(&sm.rec[0][tid].c, &a.rgb[id]);
            if (AUX) cp_async16(&sm.aux[0][tid], &a.aux[id]);
        }
        cp_async_commit();
        const int i1 = m - 1 - (NB + tid);
        if (tid < NB && i1 >= 0) id_next = a.point_list[range.x + i1];
        cp_async_wait_all();
        __syncthreads();
    }

    for (int b = 0; b < nb; ++b) {
        const int buf = b & 1;
        if (tid < NB) {
            const int i1 = m - 1 - ((b + 1) * NB + tid);
            if (i1 >= 0) {
                cp_async16(&sm.rec[buf ^ 1][tid].a, &a.xyAB[id_next]);
                cp_async16(&sm.rec[buf ^ 1][tid].b, &a.Cod[id_next]);
                cp_async16(&sm.rec[buf ^ 1][tid].c, &a.rgb[id_next]);
                if (AUX) cp_async16(&sm.aux[buf ^ 1][tid], &a.aux[id_next]);
            }
            const int i2 = m - 1 - ((b + 2) * NB + tid);
            if (i2 >= 0) id_next = a.point_list[range.x + i2];
        }
        cp_async_commit();
        const int top = m - 1 - b * NB;            // list index of slot 0
        const int cnt = min(NB, top + 1);
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
                    if constexpr (OPA) {
                        // at most one instance per pixel is its median: the warp sum runs only on a hit
                        const bool is_med = contrib && contributor + 1 == median_contrib;
                        float mv = is_med ? dmed : 0.f;
                        if (__any_sync(0xffffffffu, is_med))
#pragma unroll
                            for (int o = 16; o > 0; o >>= 1) mv += __shfl_xor_sync(0xffffffffu, mv, o);
                        if (lane == 0) sm.med[warp][ns] = mv;
                    }
                    if (lane == 0) {
                        sm.slot_a[warp][ns] = g0;
                        sm.slot_b[warp][ns] = DET ? make_float4(g1.x, g1.y, __int_as_float(jj), g1.w) : g1;
                    }
                    if (++ns == BKS) {
                        __syncwarp();
                        bwd_flush<AUX, DET, OPA, ABS>(sm, warp, lane, BKS, cx, cy, ddelx_dx, ddely_dy, a.grad_rec);
                        __syncwarp();
                        ns = 0;
                    }
                }
            }
            // slots never span a deterministic batch: its partials are complete at the barrier below
            if constexpr (DET) {
                if (ns) {
                    __syncwarp();
                    bwd_flush<AUX, DET, OPA, ABS>(sm, warp, lane, ns, cx, cy, ddelx_dx, ddely_dy, a.grad_rec);
                    __syncwarp();
                    ns = 0;
                }
            }
        }
        cp_async_wait_all();
        __syncthreads();
        if constexpr (DET) {
            // quarter q of slot t: the eight warps' partials added in warp order, then zeroed for the next batch
            const int q = tid / DCB, t = tid % DCB;
            if (q < NQ && t < cnt) {
                float4 s = sm.part[q][0][t];
                sm.part[q][0][t] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int w = 1; w < 8; ++w) {
                    const float4 v = sm.part[q][w][t];
                    sm.part[q][w][t] = make_float4(0.f, 0.f, 0.f, 0.f);
                    s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
                }
                const uint32_t g = __float_as_uint(rec[t].b.w);
                args.records[det_emit_pos(args.rect, args.base, g, blockIdx.x, blockIdx.y) * (GRAD_REC / 4) + q] = s;
            }
            __syncthreads();
        }
    }
    if (!DET && ns) {
        __syncwarp();
        bwd_flush<AUX, DET, OPA, ABS>(sm, warp, lane, ns, cx, cy, ddelx_dx, ddely_dy, a.grad_rec);
    }
}

// four threads per Gaussian, one record quarter each: the sum over the Gaussian's tiles in row-major order of its
// rect, written as quarter q of its grad_rec row (quarters >= nq and Gaussians without tiles are written as zeros)
__global__ void grad_rec_gather_kernel(uint32_t P, int nq, const uint32_t* __restrict__ tiles_touched,
                                       const uint32_t* __restrict__ base, const float4* __restrict__ records,
                                       float4* __restrict__ grad_rec) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t g = (uint32_t)(i >> 2);
    const int q = (int)(i & 3);
    if (g >= P) return;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    const uint32_t nt = tiles_touched[g];
    if (q < nq && nt) {
        const float4* r = records + (size_t)base[g] * (GRAD_REC / 4) + q;
        for (uint32_t k = 0; k < nt; ++k) {
            const float4 v = r[(size_t)k * (GRAD_REC / 4)];
            s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        }
    }
    grad_rec[(size_t)g * (GRAD_REC / 4) + q] = s;
}

// dL_dmean2D_abs [P,2] of an absgrad backward: record entries 13 and 14 of the Gaussians with radii > 0, 0 elsewhere
__global__ void __launch_bounds__(256) absgrad_export_kernel(uint32_t P, const int* __restrict__ radii,
                                                             const float* __restrict__ grad_rec,
                                                             float* __restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const bool vis = radii[i] > 0;
    const float* r = grad_rec + (size_t)i * GRAD_REC;
    out[2 * (size_t)i] = vis ? r[13] : 0.f;
    out[2 * (size_t)i + 1] = vis ? r[14] : 0.f;
}

}  // namespace s3g
