/*
 * s3g_b200.h - C ABI of the H100-native differentiable 4D Gaussian splatting
 * hot path (libs3g_b200.so).
 *
 * This is the drop-in boundary for the render path of nnanhuang/S3Gaussian.
 * Every entry point takes plain device pointers,
 * sizes and scalars - no torch types - and replaces one reference interface,
 * cited as <file>:<line> relative to the reference tree
 * (DGR = submodules/depth-diff-gaussian-rasterization):
 *
 *   s3g_mark_visible        <- CudaRasterizer::Rasterizer::markVisible   DGR/cuda_rasterizer/rasterizer.h:24-29
 *                              (pybind: _C.mark_visible                  DGR/ext.cpp:18)
 *   s3g_rasterize_forward   <- CudaRasterizer::Rasterizer::forward       DGR/cuda_rasterizer/rasterizer.h:31-56
 *                              (pybind: _C.rasterize_gaussians           DGR/ext.cpp:16, DGR/rasterize_points.cu:35-117)
 *   s3g_rasterize_backward  <- CudaRasterizer::Rasterizer::backward      DGR/cuda_rasterizer/rasterizer.h:58-88
 *                              (pybind: _C.rasterize_gaussians_backward  DGR/ext.cpp:17, DGR/rasterize_points.cu:119-202)
 *                              both take the reference's parameters as fields of named structs: s3g_raster_scene
 *                              (what the two share) and s3g_raster_forward_args / s3g_raster_backward_args
 *   s3g_deform_forward_save /  <- deform_network.forward_dynamic         scene/deformation.py:216-231
 *   s3g_deform_backward_saved     + HexPlaneField.forward                scene/hexplane.py:160-183
 *                                 + activations / Python SH->RGB         gaussian_renderer/__init__.py:99-117
 *
 * Conventions (identical to the reference):
 *   - all pointers are DEVICE pointers unless the name says host;
 *   - 4x4 matrices are 16 floats, m[k] = M[k%4][k/4] (column-major of the
 *     mathematical matrix, i.e. the transposed torch tensors of scene/cameras.py:59-63);
 *   - a NULL shs / colors_precomp / scales / rotations / cov3D_precomp selects
 *     the code path exactly as nullptr does at forward.cu:205,241 and backward.cu:406,410;
 *   - `stream` is a cudaStream_t passed as void* (the reference launches on the
 *     legacy default stream; we take the caller's stream explicitly);
 *   - every function returns >= 0 on success and a negative S3G_ERR_* code on
 *     failure; s3g_last_error() returns a thread-local message.
 *
 * There is NO CPU fallback anywhere behind this ABI: without a CUDA device every
 * compute entry point fails with S3G_ERR_CUDA.
 */
#ifndef S3G_B200_H
#define S3G_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define S3G_ABI_VERSION 2
#define S3G_ERR_UNSUPPORTED (-5) /* configuration outside what the kernels are built for */

#define S3G_OK 0
#define S3G_ERR_ARG (-1)    /* bad argument (maps to the AT_ERROR / Exception paths of the reference glue) */
#define S3G_ERR_CUDA (-2)   /* a CUDA runtime call or kernel launch failed */
#define S3G_ERR_ALLOC (-3)  /* an allocator callback returned NULL */
#define S3G_ERR_STATE (-4)  /* inconsistent opaque buffers passed to backward */

/* Growable byte-arena callback: replaces the three std::function<char*(size_t)>
 * arguments of Rasterizer::forward (rasterizer.h:32-34, created by
 * resizeFunctional() at rasterize_points.cu:27-33).  Must return a device
 * pointer to at least `bytes` bytes, 128-byte aligned or better. */
typedef char* (*s3g_alloc_fn)(void* user, size_t bytes);

int s3g_abi_version(void);
const char* s3g_last_error(void);
/* name of the CUDA arch the kernels were compiled for, e.g. "sm_90a" */
const char* s3g_build_arch(void);

/* ---- visibility (rasterizer_impl.cu:54-66,141-153) ---------------------- */
int s3g_mark_visible(int P, const float* means3D, const float* viewmatrix,
                     const float* projmatrix, uint8_t* present, void* stream);

/* ---- the rasterizer (rasterizer_impl.cu:198-444) ----------------------------------------------------------------
 * One forward and one backward entry point, each taking its arguments in named structs.  Fields carry the parameter
 * names of Rasterizer::forward / ::backward (rasterizer.h:31-88); an optional extra is a field left NULL (0 for
 * n_flow), so zero-initialise the structs and set what you use.
 *
 * s3g_raster_scene is what forward and backward share; fill it the same way for both calls.  `opacities` is read by
 * the forward only, `cam_pos` is the backward's `campos`, and `prefiltered` only selects a device-side trap in the
 * reference (auxiliary.h:156-160), so it is accepted and ignored. */
typedef struct s3g_raster_scene {
    int P, D, M;
    const float* background;
    int width, height;
    const float* means3D;
    const float* shs;
    const float* colors_precomp;
    const float* opacities;
    const float* scales;
    float scale_modifier;
    const float* rotations;
    const float* cov3D_precomp;
    const float* viewmatrix;
    const float* projmatrix;
    const float* cam_pos;
    float tan_fovx, tan_fovy;
    int prefiltered;
    int debug;
} s3g_raster_scene;

/* ---- forward (rasterizer_impl.cu:198-339) -------------------------------
 * Returns num_rendered (>= 0) like the reference, or a negative error.
 * out_color [3,H,W], out_depth [1,H,W], radii [P] (may be NULL) are
 * caller-allocated; the three opaque state buffers are grown through the
 * callbacks and are the forward->backward contract (their LAYOUT is ours, not
 * the reference's; use s3g_state_field() to look inside).
 * num_rendered never stalls the GPU: the count stays on the device for the binning kernels and is ALSO stored by
 * the scan kernel into mapped pinned host memory; the host reads it there after the whole forward has been enqueued
 * against the binning capacity this thread requested last time (binning_alloc is called with that size first).  If
 * the count outgrew the capacity - writes were clamped - the arena is grown through binning_alloc and the tail
 * (emit, tile sort, composite) is enqueued again.  The very first call on a (thread, device) waits for the count
 * before sizing the arena, like rasterizer_impl.cu:282.  No cudaMemcpy, event or stream synchronisation inside.
 *
 * Optional extras, composited in the same preprocess, sort and composite walk; out_color / out_depth / radii stay
 * exactly those of the plain call:
 *   colors_aux, out_color_aux: both or neither.  render(render_feat=True) rasterizes the same Gaussians twice - once
 *     with the RGB colours, once with the three-channel feature colours (gaussian_renderer/__init__.py:173-186,
 *     train.py:373) - and the reference runs its whole rasterizer again for the second image.  Here `colors_aux`
 *     [P,3] -> `out_color_aux` [3,H,W] (same background) comes from the one pass, and the aux pair of
 *     s3g_raster_backward_args is its backward.
 *   The reference's evaluation (utils/video_utils.py:170-299) renders each view once per image: the full image, with
 *   render(return_decomposition=True) the images of the dynamic and of the static Gaussians alone
 *   (gaussian_renderer/__init__.py:177-192), and once more per deformation-flow image, with the flow colours as
 *   override_color on the same geometry.  These two extras give those images from the one pass, FORWARD ONLY:
 *   group, out_color_d, out_depth_d, out_color_s, out_depth_s: either the four outputs are all given or all five
 *     pointers are NULL.  `group` is a DEVICE uint8 [P] (nonzero = dynamic; may be NULL only when P == 0);
 *     out_color_d / out_depth_d and out_color_s / out_depth_s ([3,H,W] / [1,H,W]) equal the plain forward on
 *     the dynamic / static subset alone - a subset with no Gaussians gives zero images, as P == 0 does;
 *   n_flow in {0, 1, 2}; for k < n_flow, flow_colors[k] is a DEVICE float [P,4], 16-byte aligned, rgb in .xyz (as
 *     s3g_flow_colors writes it), and out_flow[k] a [3,H,W] image equal to the plain forward with
 *     colors_precomp = that rgb (same geometry and background); pointers with k >= n_flow must be NULL.
 * The aux pair combines with neither the decomposition nor the flow sets.  After a forward with the decomposition
 * or a flow set, the state buffers it leaves (with a group, the staged records carry it) must not be passed to the
 * backward. */
typedef struct s3g_raster_forward_args {
    s3g_alloc_fn geom_alloc; void* geom_user;
    s3g_alloc_fn binning_alloc; void* binning_user;
    s3g_alloc_fn image_alloc; void* image_user;
    float* out_color;
    float* out_depth;
    int* radii;
    const float* colors_aux;
    float* out_color_aux;
    const uint8_t* group;
    float* out_color_d;
    float* out_depth_d;
    float* out_color_s;
    float* out_depth_s;
    int n_flow;
    const float* flow_colors[2];
    float* out_flow[2];
} s3g_raster_forward_args;
int64_t s3g_rasterize_forward(const s3g_raster_scene* scene, const s3g_raster_forward_args* fwd, void* stream);

/* ---- the backward's fused first half of the data-parallel gradient exchange -------------------------------------
 * View-parallel training (one camera per GPU, replicated Gaussians; reference batch loop train.py:372-392) sums the
 * per-Gaussian gradients over the ranks every step.  With a peer sink the backward's last kernel does not write
 * dL_dmean3D / dL_dsh / dL_dopacity / dL_dscale / dL_drot locally: every VISIBLE Gaussian's values are stored over
 * NVLink straight into the staging area of the rank that owns that slice of the flat gradient bucket
 * (stage[o] = rank o's area, laid out [world][chunk] floats, pre-zeroed; element e of the bucket lives in slice
 * e / chunk).  s3g_peer_reduce_gather() on every rank then sums its `world` sub-slices in rank order, stores the sums
 * into every rank's bucket (multimem.st through the multicast mapping, or peer stores) and re-zeroes the staging.
 * The five pointers named above may be NULL; dL_dmean2D and dL_dcolor stay local and must be given, and precomputed
 * 3-D covariances are not exchanged.  The caller provides the two device-side barriers (all ranks: backward |
 * barrier | reduce_gather | barrier).  off_* are float offsets of the tensors inside the bucket (off_shs % 4 == 0;
 * off_shs ignored with colors_precomp). */
typedef struct s3g_peer_sink {
    int world, rank;
    int64_t chunk;                 /* floats per owner slice, multiple of 4, world * chunk >= bucket size */
    void* stage[16];               /* peer-mapped staging base of every rank */
    int64_t off_means3D, off_shs, off_opacities, off_scales, off_rotations;
} s3g_peer_sink;

/* ---- backward (rasterizer_impl.cu:343-444) ------------------------------
 * R, radii and the three state buffers are what the forward returned and left.
 * All dL_* outputs are written for every Gaussian (zeros where radii <= 0), so
 * the caller need NOT pre-zero them (the reference glue zero-fills ten tensors,
 * rasterize_points.cu:154-163).  dL_dconic [P,4] and dL_ddepth [P] are the
 * reference's internal intermediates; pass NULL unless you want them exported
 * (parity tests do).  dL_dmean2D is [P,3] with z untouched = 0
 * (backward.cu:578-579).  dL_drot [P,4] must be 16-byte aligned (S3G_ERR_ARG
 * before any launch otherwise; not read with a peer sink).
 * Optional extras:
 *   dL_dpix_aux, dL_dcolor_aux: both or neither, after a forward with colors_aux: `dL_dpix_aux` [3,H,W] ->
 *     `dL_dcolor_aux` [P,3]; the geometry gradients are then those of the SUM of both images' losses;
 *   sink: the peer sink above.  It does not combine with the aux pair. */
typedef struct s3g_raster_backward_args {
    int64_t R;
    const int* radii;
    char* geom_buffer;
    char* binning_buffer;
    char* image_buffer;
    const float* dL_dpix;
    const float* dL_dpix_depth;
    float* dL_dmean2D;
    float* dL_dconic;
    float* dL_dopacity;
    float* dL_dcolor;
    float* dL_ddepth;
    float* dL_dmean3D;
    float* dL_dcov3D;
    float* dL_dsh;
    float* dL_dscale;
    float* dL_drot;
    const float* dL_dpix_aux;
    float* dL_dcolor_aux;
    const s3g_peer_sink* sink;
} s3g_raster_backward_args;
int s3g_rasterize_backward(const s3g_raster_scene* scene, const s3g_raster_backward_args* bwd, void* stream);

/* Deterministic backward: s3g_rasterize_backward with every sum taken in an order fixed by the inputs, so two calls
 * on the same forward give bitwise equal dL_* outputs (s3g_rasterize_backward adds the per-Gaussian contributions
 * of the composite with unordered atomic reductions and differs in the last bits from call to call).  The same
 * scene, backward arguments and contract; the gradients agree with s3g_rasterize_backward's up to float rounding.
 * The composite writes one gradient record per (tile, instance) into the workspace and a second kernel sums each
 * Gaussian's records over its tiles in row-major order; no global atomics, no host synchronisation.
 * workspace: s3g_rasterize_backward_deterministic_workspace_bytes(P, R, width, height) bytes (0 for invalid sizes),
 * 16-byte aligned: 64 bytes per tile instance (R, the forward's return value) plus 4 bytes per Gaussian, e.g.
 * 0.65 GB for 10 M instances and 2 M Gaussians.  It may be NULL when R == 0; its contents on entry do not matter.
 * S3G_ERR_ARG before any launch: every case of s3g_rasterize_backward, a non-NULL `sink` (the fused gradient
 * exchange is not deterministic), or a NULL or unaligned workspace when R > 0. */
size_t s3g_rasterize_backward_deterministic_workspace_bytes(int P, int64_t R, int width, int height);
int s3g_rasterize_backward_deterministic(const s3g_raster_scene* scene, const s3g_raster_backward_args* bwd,
                                         void* workspace, void* stream);

/* ---- accumulated opacity and median depth --------------------------------------------------------------------------
 * Not in the reference rasterizer, whose evaluation declares opacities / median_depths / static_opacities /
 * dynamic_opacities (utils/video_utils.py:144-149) and a sky-mask panel of 1 - opacity (:407-417) with nothing to fill
 * them.  Per pixel p, from the same walk, thresholds and per-Gaussian records as the colour and depth images:
 *   alpha(p)        = 1 - T_final(p), T_final the transmittance the background is blended with (power > 0 and
 *                     alpha < 1/255 skipped, stop before T < 1e-4), so out_color = (the bg = 0 image) + (1 - alpha) bg;
 *   median_depth(p) = the depth (the per-Gaussian camera z of out_depth) of the first contributor, front to back,
 *                     whose blend takes T from > 0.5 to <= 0.5; 0 where alpha never passes 0.5.  Its gradient goes
 *                     to that one Gaussian's depth with weight 1; which Gaussian is chosen gets none;
 *   alpha_d, alpha_s (decomposition, forward only): the alpha images of the dynamic and static subsets, each what a
 *                     separate pass over that subset computes (0 for an empty subset).
 * out_depth is sum_i w_i z_i, not normalised: expected depth is out_depth / alpha.
 *
 * The three calls below are s3g_rasterize_forward, s3g_rasterize_backward and s3g_rasterize_backward_deterministic
 * with the same scene, arguments, contract and results, plus one s3g_raster_opacity_args.  The forward reads its out_*
 * fields, the backwards their dL_dpix_* fields; each call rejects the other's fields.  A NULL `opa` or one with every
 * field NULL gives results identical to the plain call.
 *   forward: out_alpha, out_median_depth: [1,H,W] each, either may be NULL.  out_alpha_d, out_alpha_s: [1,H,W], both
 *     or neither, only with the decomposition (group).  They combine with the aux pair and the flow sets.  A forward
 *     with out_median_depth and neither the decomposition nor a flow set also keeps each pixel's median position in
 *     the image state (s3g_state_field "median_contrib") for the backward.
 *   backward: dL_dpix_alpha, dL_dpix_median: [1,H,W] each or NULL; they add T_final dL/dalpha to every contributor's
 *     alpha gradient and dL/dmedian to the median contributor's depth gradient, so dL_dmean3D, dL_dmean2D,
 *     dL_dopacity, dL_dscale, dL_drot, dL_dcov3D and the exported dL_dconic / dL_ddepth include them, and so does
 *     s3g_rasterize_camera_backward called afterwards.  The deterministic call stays bitwise repeatable.
 * S3G_ERR_ARG before any launch: every case of the plain call; alpha_d / alpha_s given alone or without `group`;
 * dL_dpix_* given to the forward or out_* to a backward (the decomposition is forward only); dL_dpix_median after a
 * forward that kept no median state for this image buffer and size (the last 1024 such forwards are remembered per
 * process); a peer sink with dL_dpix_alpha or dL_dpix_median (the fused gradient exchange does not take them). */
typedef struct s3g_raster_opacity_args {
    float* out_alpha;
    float* out_median_depth;
    float* out_alpha_d;
    float* out_alpha_s;
    const float* dL_dpix_alpha;
    const float* dL_dpix_median;
} s3g_raster_opacity_args;
int64_t s3g_rasterize_forward_opacity(const s3g_raster_scene* scene, const s3g_raster_forward_args* fwd,
                                      const s3g_raster_opacity_args* opa, void* stream);
int s3g_rasterize_backward_opacity(const s3g_raster_scene* scene, const s3g_raster_backward_args* bwd,
                                   const s3g_raster_opacity_args* opa, void* stream);
int s3g_rasterize_backward_deterministic_opacity(const s3g_raster_scene* scene, const s3g_raster_backward_args* bwd,
                                                 const s3g_raster_opacity_args* opa, void* workspace, void* stream);

/* ---- antialiasing (Mip-Splatting's 2-D screen-space filter) --------------------------------------------------------
 * Not in the reference rasterizer; upstream 3DGS calls it `antialiasing`, gsplat rasterize_mode="antialiased".  Every
 * Gaussian's 2-D covariance is dilated by 0.3 px^2, so one smaller than a pixel is drawn as a blob of at least that
 * size and grows brighter and thicker as the pixels grow (a model rendered below its training resolution, distant
 * geometry).  The antialiased forward keeps that dilation and scales the opacity by the ratio of the footprints:
 *   with a, b, c the EWA 2-D covariance before the dilation, det0 = a c - b^2, det1 = (a + 0.3)(c + 0.3) - b^2,
 *   h = sqrt(max(det0 / det1, 2.5e-5)), the composite uses alpha_eff = opacity * h wherever it reads an opacity (the
 *   blend weight, the 1/255 cut-off, the tile culling, the alpha and median images).
 * Conic, radii, tile rectangles and depth keys are those of the plain forward.
 * s3g_rasterize_forward_antialiased is s3g_rasterize_forward_opacity (so, with a NULL `opa` or every field NULL,
 * s3g_rasterize_forward) with the filter on: the same scene, arguments, contract and extras (aux pair, decomposition,
 * flow sets, opacity images).  The choice is made once, at the forward: the library remembers per geometry buffer
 * whether its last forward was antialiased (every forward updates that record), and s3g_rasterize_backward, its
 * deterministic and *_opacity forms and s3g_rasterize_camera_backward then apply that forward's chain rule: dL_dopacity
 * is h dL/dalpha_eff, and the term of h's dependence on the 2-D covariance reaches dL_dmean3D, dL_dscale, dL_drot,
 * dL_dcov3D and the camera gradients (dL_dmean2D, dL_dconic and dL_ddepth are the composite's, as before).  They read
 * the record through bwd->geom_buffer, so the camera pass needs it after an antialiased forward.
 * S3G_ERR_ARG before any launch: every case of s3g_rasterize_forward_opacity; in a backward, a peer sink after an
 * antialiased forward (the fused gradient exchange does not take its gradients). */
int64_t s3g_rasterize_forward_antialiased(const s3g_raster_scene* scene, const s3g_raster_forward_args* fwd,
                                          const s3g_raster_opacity_args* opa /* may be NULL */, void* stream);

/* ---- absolute screen-space gradients (AbsGS; gsplat rasterization(absgrad=True), means2d.absgrad) ------------------
 * Not in the reference.  Densification selects on the norm of the signed dL/dmean2D summed over pixels; over a large
 * Gaussian on a textured surface the pixels pull in opposite directions, the sum cancels and the Gaussian is never
 * split.  The absolute statistic sums each pixel's contribution's magnitude instead.  For Gaussian i, in the units of
 * dL_dmean2D (the pixel offset times width/2 or height/2):
 *   dL_dmean2D_abs[i] = ( sum_p |dL_p/dmean2D_x[i]|, sum_p |dL_p/dmean2D_y[i]| )
 * over the pixels p it contributes to, where dL_p/dmean2D is pixel p's whole share of dL_dmean2D: every image of the
 * call (colour, depth, the aux image, alpha and median depth) and the background term.  With X_p = G dL/dalpha_p,
 * d_p = mean2D - pixel, (A, B, C) the conic and o the opacity the composite used (opacity * h after an antialiased
 * forward):
 *   x: o (width/2)  sum_p |X_p (A dx_p + B dy_p)|        y: o (height/2) sum_p |X_p (C dy_p + B dx_p)|
 * The signed dL_dmean2D is the same sum without the absolute values, so |dL_dmean2D| <= dL_dmean2D_abs componentwise.
 * The statistic belongs to one call: with the aux pair, each pixel's colour and aux terms are added before the absolute
 * value; two separate calls for the two images add two sums of absolute values, which is never less.
 *
 * s3g_rasterize_backward_absgrad is s3g_rasterize_backward_opacity (`opa` may be NULL: s3g_rasterize_backward) or,
 * with deterministic != 0, s3g_rasterize_backward_deterministic_opacity with `workspace` as there: the same scene,
 * arguments, contract and every other output, the chain rule of an antialiased forward included.  It also writes
 * dL_dmean2D_abs DEVICE float [P,2], zero where radii <= 0.  The composite keeps the two sums in entries 13 and 14 of
 * each Gaussian's gradient record, which the other walks leave unused, so the geometry buffer and the workspace sizes
 * are unchanged.  The deterministic form stays bitwise repeatable, dL_dmean2D_abs included; the default form adds
 * with unordered atomics and differs in the last bits from call to call.  With a peer sink (deterministic = 0),
 * dL_dmean2D_abs stays local like dL_dmean2D.
 * S3G_ERR_ARG before any launch: every case of the call it extends; a NULL dL_dmean2D_abs when P > 0; deterministic
 * with a peer sink. */
int s3g_rasterize_backward_absgrad(const s3g_raster_scene* scene, const s3g_raster_backward_args* bwd,
                                   const s3g_raster_opacity_args* opa /* may be NULL */,
                                   float* dL_dmean2D_abs /* DEVICE [P,2] */, int deterministic,
                                   void* workspace /* deterministic: as s3g_rasterize_backward_deterministic */,
                                   void* stream);

/* ---- camera intrinsics and lens distortion (OpenCV radial-tangential) ---------------------------------------------
 * Not in the reference, which projects through the symmetric pinhole of tan_fovx / tan_fovy (principal point at the
 * image centre, no distortion); gsplat and upstream 3DGS forks take K and OpenCV distortion.  Street-scene cameras
 * (Waymo) have an off-centre principal point and five distortion coefficients.
 * The lens, in pixels of the render size: fx, fy, cx, cy, k1, k2, p1, p2, k3.  K convention: pixel j's centre is at
 * j + 0.5, so a centred camera has cx = width / 2 (the sky model's convention); an OpenCV K, whose pixel centres are
 * at j, needs cx + 0.5 and cy + 0.5.  For a Gaussian with camera-space mean t = view . p:
 *   1. near cull as before: t.z <= 0.2 is invisible;
 *   2. x = t.x / t.z, y = t.y / t.z, s = x^2 + y^2, rho = 1 + k1 s + k2 s^2 + k3 s^3,
 *      xd = x rho + 2 p1 x y + p2 (s + 2 x^2),  yd = y rho + p1 (s + 2 y^2) + 2 p2 x y;
 *   3. lens cull: s* is the smallest positive root of 1 + 3 k1 s + 5 k2 s^2 + 7 k3 s^3, the radius where the radial
 *      map r rho(r^2) stops increasing; where it exists, s > s* is culled (radius 0), since beyond it the polynomial
 *      folds points from outside the frustum back into the image.  The tangential terms do not enter the bound.
 *      s3g_lens_max_radius2 returns s* (computed in double, as the forward does once per call), or +inf;
 *   4. mean2D = (fx xd + cx - 0.5, fy yd + cy - 0.5) in the rasterizer's pixel coordinates; dL_dmean2D keeps its
 *      units, the gradient with respect to (2 u + 1) / width - 1 (and likewise v);
 *   5. the 2-D covariance is (F D J_n) W Sigma W^T (F D J_n)^T, then the 0.3 px^2 dilation and, antialiased, the
 *      filter as above.  F = diag(fx, fy); J_n = [[1/z, 0, -x_c/z], [0, 1/z, -y_c/z]] with x_c, y_c = x, y clamped
 *      to [-1.3 cx/fx, 1.3 (width - cx)/fx] and [-1.3 cy/fy, 1.3 (height - cy)/fy] (the plain 1.3 tanfov when
 *      cx = width / 2); D = d(xd, yd)/d(x, y) at the unclamped (x, y).  With zero coefficients D = I and, with
 *      fx = width / (2 tan_fovx), cx = width / 2 (likewise y), this is the plain forward's projection;
 *   6. depth, SH colour, radii, tile rectangles and the composite follow as in the plain forward.
 * viewmatrix still places the camera; projmatrix and tan_fovx / tan_fovy are not used by the projection.
 * s3g_rasterize_forward_lens is s3g_rasterize_forward_opacity (`opa` may be NULL: s3g_rasterize_forward) or, with
 * antialiased != 0, s3g_rasterize_forward_antialiased, through the lens: the same scene, arguments, contract and
 * extras (aux pair, decomposition, flow sets, opacity images).  The library remembers per geometry buffer the lens of
 * its last forward (every forward updates that record), and s3g_rasterize_backward, its deterministic, *_opacity and
 * absgrad forms then apply the chain rule of that projection: the mean's path through D^T F, the covariance's through
 * F D J_n with D's own dependence on the mean.  The lens gets no gradient.
 * S3G_ERR_ARG before any launch: every case of the call it extends; a NULL lens; fx or fy not finite and positive; cx,
 * cy or a coefficient not finite; after a lens forward, s3g_rasterize_camera_backward (camera gradients through the
 * lens are not implemented) and a backward with a peer sink (the fused gradient exchange does not take its
 * gradients). */
typedef struct s3g_raster_lens {
    float fx, fy, cx, cy;
    float k1, k2, p1, p2, k3;
} s3g_raster_lens;
int64_t s3g_rasterize_forward_lens(const s3g_raster_scene* scene, const s3g_raster_forward_args* fwd,
                                   const s3g_raster_opacity_args* opa /* may be NULL */, int antialiased,
                                   const s3g_raster_lens* lens, void* stream);
double s3g_lens_max_radius2(const s3g_raster_lens* lens);

/* ---- 3-D smoothing filter (Mip-Splatting's compute_3D_filter, get_scaling / get_opacity_with_3D_filter) ----------
 * Not in the reference.  Extends the model side of render(): optimisation lets a Gaussian shrink far below the finest
 * sampling interval any training camera had at its position, and a view closer than every training camera (a lane
 * change, a frame between two training frames) then shows it as a needle or speck.  The filter gives each Gaussian a
 * world-space lower bound on its size from the training cameras' sampling rates; it is applied to the activated scales
 * and opacities before the rasterizer (and its scale_modifier) and complements the 2-D antialiasing filter above, which
 * handles the opposite case (a model rendered coarser than it was trained).
 *
 * s3g_filter3d_compute: xyz DEVICE float [P,3] the Gaussian means (in the fine stage the canonical, undeformed
 * positions); C training cameras: viewmatrices DEVICE float [C,16], each the world-to-view matrix in the rasterizer's
 * viewmatrix layout (m[k] = M[k%4][k/4]), cams DEVICE float [C,4] = (width, height, focal_x, focal_y) with
 * focal_x = width / (2 tan(FoVx / 2)), focal_y likewise, all positive.  Writes filter_3d DEVICE float [P]:
 *   1. for camera c and Gaussian i, (x, y, z) the camera-space mean, u = x / z focal_x + width / 2,
 *      v = y / z focal_y + height / 2;
 *   2. the pair is valid when z > 0.2, -0.15 width <= u <= 1.15 width and -0.15 height <= v <= 1.15 height (taken in
 *      the multiplied form |x focal_x| <= 0.65 width z, the camera-space mean in double);
 *   3. d_i = min over the valid cameras of z;
 *   4. F = max over ALL cameras of focal_x - Mip-Splatting's choice: one focal for the whole camera set, not the min
 *      of z / focal per camera;
 *   5. a Gaussian no camera sees gets d_i = the max of d over the Gaussians that have one; when no Gaussian is seen,
 *      every filter value is 0 (Mip-Splatting raises there);
 *   6. filter_3d[i] = d_i / F * sqrt(0.2), 0.2 px^2 being Mip-Splatting's fixed variance.
 * Only min and max are taken, so two calls give bitwise equal results.  Three launches (a 4-byte memset, the depth
 * pass with the cameras staged through shared memory 64 at a time, the fill pass); no host synchronisation.
 * workspace: s3g_filter3d_compute_workspace_bytes(P) bytes (16 for P > 0, 0 otherwise), 16-byte aligned.  P == 0
 * does nothing and returns S3G_OK.
 * S3G_ERR_ARG before any launch: P < 0; C < 1 with P > 0; a NULL pointer; an unaligned workspace; P > INT_MAX / 3 or
 * C > INT_MAX / 16 (32-bit element indices).
 *
 * s3g_filter3d_apply_forward: scales DEVICE float [P,3] (activated, > 0), opacity [P] (activated), filter_3d [P] ->
 *   out_scales[i,k]  = sqrt(scales[i,k]^2 + f^2),
 *   out_opacity[i]   = opacity[i] sqrt(prod_k scales[i,k]^2 / prod_k out_scales[i,k]^2)   (f = filter_3d[i]),
 * which keeps opacity * prod scales, the Gaussian's integrated density.  Where f = 0 (and scales^2 is a normal
 * float) the outputs equal the inputs bitwise.
 * s3g_filter3d_apply_backward: the same inputs and the upstream gradients g_out_scales [P,3], g_out_opacity [P] ->
 *   g_scales[i,k] = g_out_scales[i,k] s_k / s'_k + g_out_opacity[i] o' f^2 / (s_k s'_k^2),
 *   g_opacity[i]  = g_out_opacity[i] sqrt(prod_k s_k^2 / prod_k s'_k^2)
 * (s = scales, s' = out_scales, o' = out_opacity); the filter is a constant and gets no gradient.  Where f = 0 the
 * gradients pass through bitwise.
 * One launch each; every output is written in full and must not alias an input.  P == 0 does nothing.
 * S3G_ERR_ARG before any launch: P < 0, a NULL pointer, P > INT_MAX / 3. */
size_t s3g_filter3d_compute_workspace_bytes(int P);
int s3g_filter3d_compute(int P, const float* xyz, int C, const float* viewmatrices, const float* cams,
                         float* filter_3d, void* workspace, void* stream);
int s3g_filter3d_apply_forward(int P, const float* scales, const float* opacity, const float* filter_3d,
                               float* out_scales, float* out_opacity, void* stream);
int s3g_filter3d_apply_backward(int P, const float* scales, const float* opacity, const float* filter_3d,
                                const float* g_out_scales, const float* g_out_opacity, float* g_scales,
                                float* g_opacity, void* stream);

/* ---- camera gradients ---------------------------------------------------------------------------------------------
 * Extends the backward of _RasterizeGaussians (DGR/diff_gaussian_rasterization/__init__.py:101-156), which returns no
 * gradient for raster_settings, and Rasterizer::backward (rasterizer.h:58-88): the gradient of the same loss with
 * respect to viewmatrix, projmatrix and campos, so a camera pose or extrinsic can be refined through the rasterizer.
 * Call it after s3g_rasterize_backward or s3g_rasterize_backward_deterministic with the same `scene` and `bwd`: it
 * reads the per-Gaussian dL_dmean2D, dL_dconic, dL_ddepth and (SH mode) dL_dcolor that call wrote, so dL_dconic and
 * dL_ddepth must have been exported.  With the aux pair those are the gradients of the sum of both images' losses,
 * and so is the camera gradient.  With a peer sink the four stay local (the sink only takes dL_dmean3D, dL_dsh,
 * dL_dopacity, dL_dscale, dL_drot), so the call works there too and gives this rank's camera gradient.
 * Outputs (DEVICE, each may be NULL, not all three): dL_dviewmatrix [16] and dL_dprojmatrix [16] in the layout the
 * matrices are read (m[k] = M[k%4][k/4], see the conventions above), dL_dcampos [3].  viewmatrix entries 3, 7, 11, 15
 * (never read by the forward) and projmatrix entries 2, 6, 10, 14 (mean2D does not depend on them) are exact zeros;
 * so is dL_dcampos with precomputed colours.  The tanfov values, culling and tile assignment get no gradient; through
 * the 1.3 tanfov clamp of J the clamped components of the camera-space mean get none, as in the backward.
 * The per-Gaussian contributions are summed in double in an order fixed by P (within a block in warp order, then a
 * one-block kernel over the block partials), cast to float once: the result repeats bit for bit whenever its
 * per-Gaussian inputs do, e.g. after the deterministic backward.  No atomics, no host synchronisation.
 * workspace: s3g_rasterize_camera_backward_workspace_bytes(P) bytes, 16-byte aligned (216 bytes per 1024 Gaussians,
 * 0 for P <= 0); it may be NULL when P == 0, and then the outputs are zero-filled.
 * S3G_ERR_ARG before any launch: dL_dconic or dL_ddepth NULL, all three outputs NULL, a NULL or unaligned workspace
 * when P > 0, or an input the chain rule needs missing. */
typedef struct s3g_raster_camera_grads {
    float* dL_dviewmatrix;   /* [16] or NULL */
    float* dL_dprojmatrix;   /* [16] or NULL */
    float* dL_dcampos;       /* [3]  or NULL */
} s3g_raster_camera_grads;
size_t s3g_rasterize_camera_backward_workspace_bytes(int P);
int s3g_rasterize_camera_backward(const s3g_raster_scene* scene, const s3g_raster_backward_args* bwd,
                                  const s3g_raster_camera_grads* out, void* workspace, void* stream);

/* ---- evaluation metrics (utils/video_utils.py:210-241 do them in torch and, for SSIM, on the host) ------------
 * One pass over an image pair, image / gt: DEVICE float [C,H,W] (1 <= C <= 4, H >= 7, W >= 7); mask: DEVICE uint8
 * [H,W] (nonzero = in) or NULL.  Writes, without host synchronisation, DEVICE double out[4*C+1]:
 *   out[4c+0] sum of squared errors of channel c        out[4c+1] sum of the SSIM map over the interior
 *   out[4c+2] the same squared errors summed over mask  out[4c+3] the SSIM map summed over the mask
 *   out[4C]   number of mask pixels (masked sums are 0 without a mask).
 * The SSIM map is skimage.metrics.structural_similarity's (>= 0.19, data_range 1, float32 input): 7x7 uniform window
 * with 'reflect' borders, K1 = 0.01, K2 = 0.03, sample covariances (x 49/48).  "Interior" is the map cropped by 3
 * pixels on every side (skimage's mean SSIM); the masked sum uses the uncropped map (full=True).
 * workspace: s3g_eval_metrics_workspace_bytes(C, H, W) bytes. */
size_t s3g_eval_metrics_workspace_bytes(int C, int H, int W);
int s3g_eval_metrics(int C, int H, int W, const float* image, const float* gt, const uint8_t* mask,
                     double* out, void* workspace, void* stream);

/* ---- deformation-flow colours (utils/video_utils.py:34-42,255-281; utils/visualization_tools.py:240-322) ------
 * out[i] = flow_visualizer(dx_to - dx_from)[i] for Gaussian i: dx_to, dx_from DEVICE float [P,3]; out DEVICE float
 * [P,4], 16-byte aligned, rgb in .xyz and 0 in .w.  The colour is scene_flow_to_rgb with the bright background and
 * flow_max_radius 1: the flow is min-max normalised over all 3P values, (x, y) picks a hue of the 55-entry colour
 * wheel by angle and a saturation (radius <= 1) or value (radius > 1) by radius.  normalize != 0 also applies the
 * reference's debug normalisation (c - min) / (max - min + 1e-6) over the 3P colour values.  Every rounding follows
 * the reference's torch operations.  No host synchronisation.  P == 0 does nothing.
 * workspace: s3g_flow_colors_workspace_bytes(P) bytes, 4-byte aligned. */
size_t s3g_flow_colors_workspace_bytes(int P);
int s3g_flow_colors(int P, const float* dx_to, const float* dx_from, int normalize, float* out, void* workspace,
                    void* stream);

/* ---- LPIPS v0.1, AlexNet backbone (utils/video_utils.py:221 calls lpips(rgb, gt_rgb, net_type='alex')) ----------
 * Restates lpipsPyTorch (csrc/lpips.cuh):
 *   lpipsPyTorch/__init__.py:19-21          lpips(): LPIPS('alex', '0.1') on x's device, criterion(x, y)
 *   lpipsPyTorch/modules/networks.py:50-51   z = (x - shift) / scale, shift = [-.030, -.088, -.188],
 *                                            scale = [.458, .448, .450] (true division; the input is used as given)
 *   lpipsPyTorch/modules/networks.py:53-63,77-83
 *                                            torchvision alexnet().features up to the fifth ReLU, taps after the ReLUs
 *                                            of conv 3->64 11x11/4 pad 2, conv 64->192 5x5 pad 2 (each followed by a
 *                                            3/2 max-pool, no padding, floor), conv 192->384, 384->256, 256->256 3x3
 *                                            pad 1; zero padding applies to the z-scored tensor
 *   lpipsPyTorch/modules/utils.py:6-8        n = f / (sqrt(sum_c f^2) + 1e-10) at each tap
 *   lpipsPyTorch/modules/lpips.py:30-34      d_l = mean over layer l's grid of sum_c lin_l[c] (n_x - n_y)^2
 *   lpipsPyTorch/modules/lpips.py:36         sum over the layers and the batch: for N > 1 images, the batch sum
 * The convolutions are implicit GEMMs on the tensor cores in 3xTF32 with fp32 accumulation; taps, normalisation and
 * lin weights in fp32; the means and their sum in double.
 *
 * s3g_lpips_alex_prepare: once per model, puts the convolution weights into the kernels' K order as tf32 hi/lo tiles
 * and copies the biases and lin weights, all into `prepared` (DEVICE, s3g_lpips_alex_prepared_bytes(), 16-byte
 * aligned).  The weights stay the caller's; `prepared` alone is read by s3g_lpips_alex.
 *
 * s3g_lpips_alex: x, y DEVICE float [N,3,H,W] (contiguous), N >= 1, H, W >= 31 (smaller sides make the second
 * max-pool's output empty; torch raises).  Writes, without host synchronisation, DEVICE double out[6]: out[l] the
 * term of layer l (0..4) summed over the N images, out[5] = out[0] + ... + out[4], the value of lpips(x, y).
 * Deterministic: no atomics, two calls give bitwise equal results.
 * workspace: s3g_lpips_alex_workspace_bytes(N, H, W) bytes (0 for invalid sizes).  It holds, for the 2N images (x's,
 * then y's), every convolution's ReLU output and the two max-pool outputs, channels-last float32, plus the taps'
 * per-block partial sums: about 0.24 GB for one 1920x1280 pair.
 * S3G_ERR_ARG before any launch: N < 1, a side below 31, a null pointer, or sizes whose element indices do not fit
 * 32 bits. */
typedef struct s3g_lpips_alex_weights {
    const float* conv_w[5];   /* features.{0,3,6,8,10}.weight, [Cout,Cin,k,k] */
    const float* conv_b[5];   /* features.{0,3,6,8,10}.bias, [Cout] */
    const float* lin_w[5];    /* lin{i}.model.1.weight, [1,C,1,1] (C floats) */
} s3g_lpips_alex_weights;
size_t s3g_lpips_alex_prepared_bytes(void);
int s3g_lpips_alex_prepare(const s3g_lpips_alex_weights* weights, void* prepared, void* stream);
size_t s3g_lpips_alex_workspace_bytes(int N, int H, int W);
int s3g_lpips_alex(int N, int H, int W, const float* x, const float* y, const void* prepared, double* out,
                   void* workspace, void* stream);

/* LPIPS backward: the gradients of s3g_lpips_alex's out[6] with respect to x and / or y (the weights are frozen, as
 * in lpipsPyTorch).  grad_out: DEVICE double [6], the upstream gradient of out; layer l's taps are weighed by
 * grad_out[l] + grad_out[5], so any mix of the layer terms and the total differentiates correctly.
 *
 * s3g_lpips_alex_backward_prepare: once per model, after or independently of s3g_lpips_alex_prepare, writes the
 * backward's weight layout into `prepared_bwd` (DEVICE, s3g_lpips_alex_backward_prepared_bytes(), 16-byte aligned):
 * conv 1's weights as given and, for convolutions 2-5, the flipped and transposed kernels as tf32 hi/lo tiles.  Only
 * weights->conv_w is read.
 *
 * s3g_lpips_alex_backward: N, H, W, `prepared` are those of the s3g_lpips_alex call being differentiated, and
 * fwd_workspace MUST be that call's workspace, unchanged since: the backward reads the saved activations (every
 * ReLU output, for the masks, the taps and the max-pool argmaxes) and never the images.  grad_x / grad_y: DEVICE
 * float [N,3,H,W], written (not accumulated); NULL = not wanted, and the work of that side is skipped.
 * workspace: s3g_lpips_alex_backward_workspace_bytes(N, H, W) bytes (0 for invalid sizes), about 0.1 GB for one
 * 1920x1280 pair.  No host synchronisation; deterministic: no atomics, two calls give bitwise equal gradients.
 * The dgrads of convolutions 2-5 are implicit GEMMs on the tensor cores in the forward's 3xTF32 arithmetic; conv 1's
 * (3 output channels) runs on the CUDA cores in fp32.
 * S3G_ERR_ARG before any launch: the size rules of s3g_lpips_alex, a null prepared / prepared_bwd / fwd_workspace /
 * grad_out / workspace, both gradients NULL, or an unaligned buffer (prepared and prepared_bwd 16 bytes, grad_out 8,
 * grad_x / grad_y 4). */
size_t s3g_lpips_alex_backward_prepared_bytes(void);
int s3g_lpips_alex_backward_prepare(const s3g_lpips_alex_weights* weights, void* prepared_bwd, void* stream);
size_t s3g_lpips_alex_backward_workspace_bytes(int N, int H, int W);
int s3g_lpips_alex_backward(int N, int H, int W, const void* prepared, const void* prepared_bwd,
                            const void* fwd_workspace, const double* grad_out, float* grad_x, float* grad_y,
                            void* workspace, void* stream);

/* ---- LPIPS v0.1, VGG16 backbone (metrics.py:74 calls lpips(renders[idx], gts[idx], net_type='vgg')) ---------------
 * The same computation as s3g_lpips_alex on another network (csrc/lpips_vgg.cuh), forward only:
 *   lpipsPyTorch/modules/networks.py:50-51   the same z-score
 *   lpipsPyTorch/modules/networks.py:53-63,88-96
 *                                            torchvision vgg16().features up to relu5_3: 3x3 pad 1 convolutions
 *                                            3->64, 64->64 | 64->128, 128->128 | 128->256, 256->256 x2 |
 *                                            256->512, 512->512 x2 | 512->512 x3, each followed by a ReLU, a 2/2
 *                                            max-pool (floor) between the groups; taps after the last ReLU of each
 *                                            group (64, 128, 256, 512, 512 channels)
 *   lpipsPyTorch/modules/utils.py:6-8, lpips.py:30-36   taps, lin weights, layer means and sums as above
 * 3xTF32 implicit GEMMs with fp32 accumulation, 128-channel tiles where Cout >= 128.
 *
 * s3g_lpips_vgg_prepare / s3g_lpips_vgg: as the AlexNet pair, with `prepared` of s3g_lpips_vgg_prepared_bytes()
 * (about 118 MB) and H, W >= 16 (smaller sides make the fourth max-pool's output empty; torch raises).  out[l] is the
 * term of tap l (0..4) summed over the N images, out[5] their sum.  No host synchronisation, no atomics: two calls give
 * bitwise equal results.  Nothing is kept for a backward.
 * workspace: s3g_lpips_vgg_workspace_bytes(N, H, W) bytes (0 for invalid sizes): two buffers of 2N * H * W * 64 floats
 * that the layers ping-pong between (x's and y's images walk each layer together) plus the taps' partial sums, 2.52 GB
 * for one 1920x1280 pair.
 * S3G_ERR_ARG before any launch: N < 1, a side below 16, a null pointer, an unaligned `prepared`, or 2N * H * W * 64
 * >= 2^31 (32-bit element indices). */
typedef struct s3g_lpips_vgg_weights {
    const float* conv_w[13];  /* features.{0,2,5,7,10,12,14,17,19,21,24,26,28}.weight, [Cout,Cin,3,3] */
    const float* conv_b[13];  /* the same indices' .bias, [Cout] */
    const float* lin_w[5];    /* lin{i}.model.1.weight, [1,C,1,1] (C floats) */
} s3g_lpips_vgg_weights;
size_t s3g_lpips_vgg_prepared_bytes(void);
int s3g_lpips_vgg_prepare(const s3g_lpips_vgg_weights* weights, void* prepared, void* stream);
size_t s3g_lpips_vgg_workspace_bytes(int N, int H, int W);
int s3g_lpips_vgg(int N, int H, int W, const float* x, const float* y, const void* prepared, double* out,
                  void* workspace, void* stream);

/* ---- state-buffer introspection (tests / debugging) ---------------------
 * buffer: 0 = geometry, 1 = binning, 2 = image.  Looks up a named field of our
 * layout for the given problem size and returns its byte offset from the
 * (128-byte aligned) buffer base, its element size and element count.
 * Fields: geometry: "xyAB","Cod","rgb","depth_key","tiles_touched","rect","clamped"
 *         binning : "point_list" (first field: its offset does not depend on the arena capacity; the sorted tile
 *                   ids are not materialised - "ranges" delimits every tile's slice of the list)
 *         image   : "final_T","n_contrib","ranges","median_contrib" (written only by an opacity forward that keeps
 *                   the median state)
 * Returns S3G_OK or S3G_ERR_ARG. */
int s3g_state_field(int buffer, const char* name, int64_t P, int64_t R, int width, int height,
                    size_t* offset, size_t* elem_bytes, size_t* count);

/* sizes of the three arenas (bytes) for a problem size; R may be 0 */
size_t s3g_geom_bytes(int64_t P);
size_t s3g_binning_bytes(int64_t R);
size_t s3g_image_bytes(int width, int height);

/* ---- HexPlane + deformation decoder + render() front-end -------------------
 * Replaces (forward: hexplane_sample_kernel -> wgmma decoder kernel; backward: mma.sync decoder kernel ->
 * hexplane_scatter_kernel; csrc/deform.cuh, csrc/deform_tc.cuh):
 *   deform_network.forward_dynamic / Deformation.forward_dynamic   scene/deformation.py:108-166,216-231
 *   HexPlaneField.get_density / interpolate_ms_features             scene/hexplane.py:73-106,160-175
 *   scaling/rotation/opacity activations + convert_SHs_python      gaussian_renderer/__init__.py:99-117,
 *                                                                  scene/gaussian_model.py:39-47, utils/sh_utils.py:57-112
 * Planes are CHANNELS-LAST: plane (a,b) of a level is float[res_b][res_a][32], i.e. the
 * reference's [1,32,res_b,res_a] parameter in torch.channels_last memory format.
 * Linear layers keep the PyTorch layout: weight [out][in], bias [out].  A NULL first-layer
 * weight disables that head (no_dx / no_ds / no_dr / no_do / no_dshs / feat_head=False). */
#define S3G_MAX_LEVELS 8
typedef struct s3g_deform_net {
    int num_levels;                        /* len(multires) */
    int feat_dim;                          /* output_coordinate_dim, must be 32 */
    int width;                             /* net_width, must be 64 */
    int reso[S3G_MAX_LEVELS][4];           /* per level: resolution of x, y, z, t */
    const float* planes[S3G_MAX_LEVELS][6];/* (0,1),(0,2),(0,3),(1,2),(1,3),(2,3) */
    float aabb[6];                         /* aabb[0] (max corner) then aabb[1] (min corner), hexplane.py:152-157 */
    const float *w_feat, *b_feat;          /* feature_out.0: [64][32*L] */
    const float *w_pos1, *b_pos1, *w_pos2, *b_pos2;      /* pos_deform.{1,3}:       [64][64], [3][64]  */
    const float *w_scl1, *b_scl1, *w_scl2, *b_scl2;      /* scales_deform.{1,3}:    [64][64], [3][64]  */
    const float *w_rot1, *b_rot1, *w_rot2, *b_rot2;      /* rotations_deform.{1,3}: [64][64], [4][64]  */
    const float *w_opa1, *b_opa1, *w_opa2, *b_opa2;      /* opacity_deform.{1,3}:   [64][64], [1][64]  */
    const float *w_shs1, *b_shs1, *w_shs2, *b_shs2;      /* shs_deform.{1,3}:       [64][64], [48][64] */
    const float *w_dino0, *b_dino0, *w_dino2, *b_dino2, *w_dino4, *b_dino4;   /* dino_head.{0,2,4} */
} s3g_deform_net;

/* Same shape, writable: parameter gradients.  Plane gradients are ACCUMULATED (+=) with
 * atomics and must be zeroed by the caller; Linear gradients are overwritten. */
typedef struct s3g_deform_net_grads {
    float* planes[S3G_MAX_LEVELS][6];
    float *w_feat, *b_feat;
    float *w_pos1, *b_pos1, *w_pos2, *b_pos2;
    float *w_scl1, *b_scl1, *w_scl2, *b_scl2;
    float *w_rot1, *b_rot1, *w_rot2, *b_rot2;
    float *w_opa1, *b_opa1, *w_opa2, *b_opa2;
    float *w_shs1, *b_shs1, *w_shs2, *b_shs2;
    float *w_dino0, *b_dino0, *w_dino2, *b_dino2, *w_dino4, *b_dino4;
} s3g_deform_net_grads;

/* Forward.  Inputs are the RAW Gaussian parameters (pre-activation) [P,*]; `time` is the
 * camera time in [0,1] (all Gaussians share it, gaussian_renderer/__init__.py:58).
 * Outputs (all fully written): means3D [P,3] = xyz + dx, scales_act [P,3] = exp(scales+ds),
 * rot_act [P,4] = normalize(rot+dr), opacity_act [P,1] = sigmoid(opacity+do),
 * colors [P,3] = clamp_min(SH(shs+dshs, dir(xyz - campos)) + 0.5, 0) with the UNDEFORMED xyz,
 * dx [P,3], dshs [P,16,3], feat [P,3].  Pointers of disabled heads may be NULL.
 * features [P, 32*num_levels] receives the sampled HexPlane features (the hand-over between the
 * sampling and the decoder kernel); keep it for s3g_deform_backward_saved.
 * acts receives the decoder's hidden activations (h = feature_out(f) and the hidden layer of every enabled head,
 * scene/deformation.py:56-76 - what autograd keeps for the reference): an opaque buffer of
 * s3g_deform_saved_bytes(net, P) bytes that s3g_deform_backward_saved reads.  acts may be NULL when no backward
 * will follow.
 * campos: device float[3]; sh_degree: active degree (0..3).  (1 <= num_levels <= 4; feat_dim 32; width 64.) */
size_t s3g_deform_saved_bytes(const s3g_deform_net* net, int P);
int s3g_deform_forward_save(const s3g_deform_net* net, int P, const float* xyz, const float* scales,
                            const float* rotations, const float* opacity, const float* shs, float time,
                            const float* campos, int sh_degree,
                            float* means3D, float* scales_act, float* rot_act, float* opacity_act,
                            float* colors, float* dx, float* dshs, float* feat, float* features, float* acts,
                            void* workspace, void* stream);
/* bytes of `workspace` for s3g_deform_forward_save (tensor-core-ready copies of the Linear weights) */
size_t s3g_deform_forward_workspace_bytes(const s3g_deform_net* net);

/* Backward of the above.  g_* are dL/d(output) (NULL = zero).  Writes dL/d(raw inputs)
 * [P,*] in full, overwrites the Linear gradients in `grads` and accumulates the plane
 * gradients.  `features` and `acts` are the buffers the forward filled; acts is required for P > 0.
 * `workspace` must hold s3g_deform_workspace_bytes(net, P) bytes. */
size_t s3g_deform_workspace_bytes(const s3g_deform_net* net, int P);
int s3g_deform_backward_saved(const s3g_deform_net* net, int P, const float* xyz, const float* scales,
                              const float* rotations, const float* opacity, const float* shs, float time,
                              const float* campos, int sh_degree, const float* features, const float* acts,
                              const float* g_means3D, const float* g_scales_act, const float* g_rot_act,
                              const float* g_opacity_act, const float* g_colors, const float* g_dx,
                              const float* g_dshs, const float* g_feat,
                              float* d_xyz, float* d_scales, float* d_rotations, float* d_opacity, float* d_shs,
                              const s3g_deform_net_grads* grads, void* workspace, void* stream);

/* ---- wgmma building-block self-test (csrc/umma_test.cu) -------------------
 * D[128,N] = A[128,K] * B[N,K]^T on the Hopper warpgroup tensor cores (wgmma tf32, accumulators in
 * registers), single pass or 3xTF32.  K % 8 == 0, K <= 128, N in {16, 32, 48, 64}.  Device pointers. */
int s3g_umma_selftest(const float* A, const float* B, float* D, int K, int N, int three_pass, void* stream);

/* ---- per-stage device timing (bench.py roofline leg) ----------------------
 * When enabled, forward/backward bracket every kernel stage with cudaEvents on
 * the caller's stream.  s3g_profile_read() synchronises those events and copies
 * the last call's stage times (milliseconds) into `ms`; returns the number of
 * stages written (names via s3g_profile_stage_name).  `which`: 0 = forward,
 * 1 = backward. */
int s3g_profile_enable(int on);
int s3g_profile_read(int which, float* ms, int capacity);
const char* s3g_profile_stage_name(int which, int index);

/* ---- standalone device radix sort (exposed for tests) -------------------
 * Stable LSD sort of n (key,value) u32 pairs on key bits [begin_bit,end_bit).
 * keys_out/vals_out receive the result; keys_in/vals_in are clobbered; `temp`
 * must hold s3g_sort_temp_bytes(n) bytes. */
size_t s3g_sort_temp_bytes(int64_t n);
int s3g_sort_pairs_u32(int64_t n, uint32_t* keys_in, uint32_t* vals_in,
                       uint32_t* keys_out, uint32_t* vals_out,
                       int begin_bit, int end_bit, void* temp, void* stream);

/* ---- training-step kernels either side of render() ------------------------------------------
 *
 * s3g_adam_step       <- torch.optim.Adam(l, lr=0.0, eps=1e-15).step()   scene/gaussian_model.py:189, train.py:520-522
 *                        (torch/optim/adam.py _multi_tensor_adam: no weight decay, no amsgrad)
 * s3g_adam_step_selective <- the same step restricted to the visible rows of the per-Gaussian tensors (not in the
 *                        reference)
 * s3g_densify_stats   <- max_radii2D update + add_densification_stats    train.py:489-491, scene/gaussian_model.py:693-695
 * s3g_image_loss_*    <- l1_loss + ssim + compute_depth("l2")            utils/loss_utils.py:20-96, train.py:395-419
 */
typedef struct s3g_adam_tensor {
    float* param;          /* updated in place */
    const float* grad;
    float* exp_avg;        /* updated in place */
    float* exp_avg_sq;     /* updated in place */
    int64_t numel;
    double lr;             /* the param group's current lr */
    int64_t step;          /* state['step'] AFTER this step's increment (>= 1) */
} s3g_adam_tensor;

/* `tensors` is a HOST array of n descriptors (device pointers inside).  One kernel launch per
 * 40 tensors.  Tensors with numel == 0 are skipped. */
int s3g_adam_step(int n, const s3g_adam_tensor* tensors, double beta1, double beta2, double eps, void* stream);

/* Selective Adam (upstream 3DGS --optimizer_type sparse_adam, Taming 3DGS, gsplat SelectiveAdam): s3g_adam_step in which
 * the per-Gaussian tensors update only the rows the step's views see.  row_width: HOST int32[n].  row_width[i] == 0
 * marks a dense tensor (the s3g_adam_step update); row_width[i] > 0 a masked one of `rows` rows of row_width[i] floats
 * (numel == rows * row_width[i], fewer than 2^31 elements).  visible: DEVICE uint8[rows] (a torch bool tensor's
 * storage).  A masked row with visible[r] != 0 gets exactly the s3g_adam_step update; one with visible[r] == 0 keeps
 * its param, exp_avg and exp_avg_sq bit for bit and its grad is not read.  `step` is the tensor's global counter, as
 * in s3g_adam_step, so an all-visible mask gives s3g_adam_step's bits.  One launch per 40 tensors, dense and masked
 * together; no host synchronisation.  S3G_ERR_ARG before any launch: n < 0, a NULL table, rows < 0, row_width < 0,
 * numel < 0 or != rows * row_width, and, for a tensor with numel > 0, a NULL pointer, step < 1, or a NULL visible
 * with row_width > 0. */
int s3g_adam_step_selective(int n, const s3g_adam_tensor* tensors, const int32_t* row_width, int64_t rows,
                            const uint8_t* visible, double beta1, double beta2, double eps, void* stream);

/* radii i32[P] (max over the step's views), viewspace_grad f32[P,3] (summed over the views);
 * for radii > 0: max_radii2D = max(max_radii2D, radii); xyz_gradient_accum += |grad[:2]|; denom += 1. */
int s3g_densify_stats(int P, const float* viewspace_grad, const int* radii, float* xyz_gradient_accum,
                      float* denom, float* max_radii2D, void* stream);

/* s3g_densify_stats in the same launch, and for radii > 0 also xyz_gradient_accum_abs += |viewspace_absgrad|, the
 * L2 norm of the absolute screen-space gradient f32[P,2] (s3g_rasterize_backward_absgrad, summed over the views). */
int s3g_densify_stats_abs(int P, const float* viewspace_grad, const float* viewspace_absgrad, const int* radii,
                          float* xyz_gradient_accum, float* xyz_gradient_accum_abs, float* denom, float* max_radii2D,
                          void* stream);

/* image, gt_image: f32[B,C,H,W] (or C == 0 and NULL: depth term only); depth, gt_depth: f32[B,H,W] or
 * both NULL (no depth term).
 * forward: sums (DEVICE double[4]) = {sum|image-gt|, sum ssim_map, sum over valid of
 *   (clamp(d/max,0,1)-clamp(gt/max,0,1))^2, #valid (0.01 < gt < max_depth)} - the caller forms
 *   l1 = sums[0]/N, ssim = sums[1]/N, depth_l2 = sums[2]/sums[3] on the device (no host sync) - and
 *   keeps the SSIM derivative maps in `workspace` (s3g_image_loss_workspace_bytes bytes).
 * backward: weights (DEVICE float[3]) = dL/d{l1, ssim, depth_l2} as autograd delivers them;
 *   writes g_image [B,C,H,W] and, with depth, g_depth [B,H,W].  Same workspace and sums. */
size_t s3g_image_loss_workspace_bytes(int B, int C, int H, int W);
int s3g_image_loss_forward(int B, int C, int H, int W, const float* image, const float* gt_image,
                           const float* depth, const float* gt_depth, float max_depth,
                           double* sums, void* workspace, void* stream);
int s3g_image_loss_backward(int B, int C, int H, int W, const float* image, const float* gt_image,
                            const float* depth, const float* gt_depth, float max_depth,
                            const float* weights, const double* sums, const void* workspace,
                            float* g_image, float* g_depth, void* stream);

/* The same terms with lambda_dssim == 0 (train.py:417 skips SSIM then): sums[1] = 0, no derivative maps;
 * workspace: 256 + 16 * 592 * 4 bytes are enough (s3g_image_loss_workspace_bytes(...) is an upper bound). */
int s3g_image_l1_depth_forward(int B, int C, int H, int W, const float* image, const float* gt_image,
                               const float* depth, const float* gt_depth, float max_depth,
                               double* sums, void* workspace, void* stream);
int s3g_image_l1_depth_backward(int B, int C, int H, int W, const float* image, const float* gt_image,
                                const float* depth, const float* gt_depth, float max_depth,
                                const float* weights, const double* sums, float* g_image, float* g_depth,
                                void* stream);

/* ---- HexPlane regularisers -------------------------------------------------------------
 * s3g_plane_reg_*  <- GaussianModel.compute_regulation                 scene/gaussian_model.py:710-749
 *                     + compute_plane_smoothness                        scene/regulation.py:22-28
 * total = sum_planes  w_smooth * mean((t[h+2]-2t[h+1]+t[h])^2 over [1,C,H-2,W]) + w_l1 * mean|1-t|
 * Each plane is the [1,C,H,W] tensor stored channels-last, i.e. physically [H][W][C]; C % 4 == 0, H >= 3;
 * plane and grad pointers 16-byte aligned (S3G_ERR_ARG before any launch otherwise).
 * `planes` is a HOST array (device pointers inside), n <= 48.  forward: total = DEVICE double[1],
 * workspace of s3g_plane_reg_workspace_bytes(...) bytes.  backward: gscale = DEVICE float[1] (the
 * upstream gradient); OVERWRITES planes[i].grad (same physical layout) with gscale * d total/d plane. */
typedef struct s3g_plane_desc {
    const float* plane;
    float* grad;          /* backward only */
    int H, W, C;
    float w_smooth;
    float w_l1;
} s3g_plane_desc;
size_t s3g_plane_reg_workspace_bytes(int n, const s3g_plane_desc* planes);
int s3g_plane_reg_forward(int n, const s3g_plane_desc* planes, double* total, void* workspace, void* stream);
int s3g_plane_reg_backward(int n, const s3g_plane_desc* planes, const float* gscale, void* stream);

/* ---- bilateral-grid colour correction (Wang et al., SIGGRAPH 2024; gsplat lib_bilagrid) ----------------------------
 * Not in the reference.  Each training image n gets a grid [12, L, GY, GX] of 3x4 affine colour transforms, indexed by
 * pixel position and luminance; the render is corrected through it before the photometric loss, so per-camera
 * exposure and white balance stop being explained by geometry.  grids: DEVICE float [N, 12, L, GY, GX], channel c is
 * entry (c / 4, c % 4) of the matrix A.  Images rgb / out: DEVICE float [B, 3, H, W].  image_ids: HOST int32 [B], the
 * grid of each image, distinct, in [0, N).
 *
 * s3g_bilagrid_slice_forward  <- gsplat lib_bilagrid slice(bil_grids, xy, rgb, grid_idx) at the pixel centres, through
 *                                BilateralGrid.forward (F.grid_sample, align_corners=True, padding_mode="border")
 * For pixel (i, j) of image b with colour (r, g, bl): x = (j + 0.5) / W (GX - 1), y = (i + 0.5) / H (GY - 1),
 * z = (0.299 r + 0.587 g + 0.114 bl) (L - 1), each clamped to [0, size - 1]; A = the trilinear interpolation of grid
 * image_ids[b] at (x, y, z); out = A[:, :3] (r, g, bl) + A[:, 3].  One launch per 512 images, one thread per pixel; no
 * intermediate in global memory.  out must not alias rgb.
 *
 * s3g_bilagrid_slice_backward  <- the autograd backward of the same formula
 * With grad_out [B, 3, H, W]: writes grad_rgb [B, 3, H, W] (may be NULL: not computed) and, for every listed image, the
 * row image_ids[b] of grad_grids [N, 12, L, GY, GX] (stored, not added: the caller zeroes the buffer; other rows are
 * not touched).  grad_rgb flows through A and through the luminance guide z, whose gradient is 0 where the unclamped
 * z is <= 0 or >= L - 1 (torch's border rule; so also for L == 1).  Two launches per 512 images: a gather over each
 * grid cell column's pixel support that writes fixed-order partial sums into the workspace, and their sum in split
 * order.  No atomics: two calls on the same inputs give bitwise equal results.  workspace:
 * s3g_bilagrid_slice_backward_workspace_bytes(...) bytes, 16-byte aligned.
 *
 * s3g_bilagrid_tv_forward / _backward  <- gsplat total_variation_loss(bil_grids.grids)
 * loss = (1/N) sum over the axes d in {L, GY, GX} of sum (grids shifted by one along d - grids)^2 / (12 L GY GX (n_d - 1)
 * / n_d) (an axis of size 1 adds 0).  forward: writes the DEVICE float scalar `loss`; workspace of
 * s3g_bilagrid_tv_workspace_bytes(...) bytes, 8-byte aligned; two launches, a fixed partition summed in double.
 * backward: gscale = DEVICE float[1] (the upstream gradient; no host synchronisation), OVERWRITES grad
 * [N, 12, L, GY, GX] with gscale * d loss / d grids; one launch.
 *
 * Every size works (L, GY, GX >= 1; the grid need not fit in shared memory).  S3G_ERR_ARG before any launch: a size
 * <= 0, a NULL pointer, an id outside [0, N), duplicate ids, N 12 L GY GX or 3 H W above INT_MAX, an unaligned
 * workspace. */
int s3g_bilagrid_slice_forward(int N, int L, int GY, int GX, const float* grids, int B, int H, int W,
                               const int32_t* image_ids, const float* rgb, float* out, void* stream);
size_t s3g_bilagrid_slice_backward_workspace_bytes(int N, int L, int GY, int GX, int B, int H, int W);
int s3g_bilagrid_slice_backward(int N, int L, int GY, int GX, const float* grids, int B, int H, int W,
                                const int32_t* image_ids, const float* rgb, const float* grad_out, float* grad_rgb,
                                float* grad_grids, void* workspace, void* stream);
size_t s3g_bilagrid_tv_workspace_bytes(int N, int L, int GY, int GX);
int s3g_bilagrid_tv_forward(int N, int L, int GY, int GX, const float* grids, float* loss, void* workspace,
                            void* stream);
int s3g_bilagrid_tv_backward(int N, int L, int GY, int GX, const float* grids, const float* gscale, float* grad,
                             void* stream);

/* ---- sky model (EmerNeRF's sky head; scene/background_model.py SkyModel, Background_Model(model_type="mlp")) --------
 * A direction MLP behind the Gaussians.  For pixel (x, y) of an H x W image, R = c2w[:3, :3]:
 *   d = R ((x - cx + 0.5) / fx, (y - cy + 0.5) / fy, 1),  v = d / (|d| + 1e-8)
 *   enc = [v, sin(xb), sin(xb + pi/2)], xb = (v, 2v, 4v, 8v, 16v) scale-major          (33 features)
 *   h1 = relu(W0 enc + b0), h2 = relu(W1 [h1, enc] + b1), sky = sigmoid(W2 h2 + b2)
 * Weights in PyTorch's fp32 layout: W0 [width, 33], W1 [width, width + 33], W2 [3, width]; width = 64, 128, 192 or
 * 256.  c2w: DEVICE float [4, 4] row-major, intrinsic: DEVICE float [3, 3] ((fx, 0, cx), (0, fy, cy), (0, 0, 1)); no
 * host synchronisation.  The parameters are read on every call (no prepared copy outlives a call).
 *
 * s3g_sky_forward   writes out_sky [3, H, W].  The wide layers run as 3xTF32 mma.sync; nothing per pixel but the output
 *                   is written to global memory.
 * s3g_sky_backward  with dL_dsky [3, H, W], writes (stores; the caller does not zero them) every weight and bias
 *                   gradient.  No gradient for the camera.  Recomputes the forward in chunks of 65536 pixels inside the
 *                   workspace; the weight gradients are fixed-order sums of per-CTA partials, so two calls give bitwise
 *                   equal results.
 * workspace: s3g_sky_workspace_bytes(width, H, W) bytes (0 for invalid sizes), 16-byte aligned; one buffer serves both
 * calls.  S3G_ERR_ARG before any launch: a width that is not a multiple of 64 in [64, 256], H < 1 or W < 1, 3 H W above
 * INT_MAX, a NULL pointer, a NULL or unaligned workspace. */
typedef struct s3g_sky_net {
    int width;
    const float* w0;   /* [width, 33] */
    const float* b0;   /* [width] */
    const float* w1;   /* [width, width + 33] */
    const float* b1;   /* [width] */
    const float* w2;   /* [3, width] */
    const float* b2;   /* [3] */
} s3g_sky_net;
typedef struct s3g_sky_net_grads {
    float* w0;
    float* b0;
    float* w1;
    float* b1;
    float* w2;
    float* b2;
} s3g_sky_net_grads;
size_t s3g_sky_workspace_bytes(int width, int H, int W);
int s3g_sky_forward(const s3g_sky_net* net, int H, int W, const float* c2w, const float* intrinsic, float* out_sky,
                    void* workspace, void* stream);
int s3g_sky_backward(const s3g_sky_net* net, int H, int W, const float* c2w, const float* intrinsic,
                     const float* dL_dsky, const s3g_sky_net_grads* grads, void* workspace, void* stream);

/* ---- densify / prune row gather -----------------------------------------------------------
 * s3g_gather_rows  <- _prune_optimizer / cat_tensors_to_optimizer / prune_points / densification_postfix
 *                     scene/gaussian_model.py:411-470 (boolean indexing + torch.cat per tensor)
 * For every tensor t (HOST array of descriptors, n <= 32; src/dst are device pointers to [rows, row_floats]
 * float32, dst has n_out rows):  dst[r] = src[src_index[r]] for r < n_kept or zero_new == 0, else 0.
 * src_index: DEVICE int64[n_out], each value a valid source row. */
typedef struct s3g_row_tensor {
    const float* src;
    float* dst;
    int row_floats;
    int zero_new;      /* 1 for optimizer state (exp_avg, exp_avg_sq): appended rows start at zero */
} s3g_row_tensor;
int s3g_gather_rows(int n, const s3g_row_tensor* tensors, int64_t n_out, int64_t n_kept, const int64_t* src_index,
                    void* stream);

/* ---- MCMC densification (3DGS-MCMC, Kheradmand et al. 2024; gsplat MCMCStrategy) ---------------------------------
 * Not in the reference, whose densification is the clone / split / prune heuristics.  3DGS-MCMC replaces them with
 * relocating near-transparent Gaussians onto live ones, growing to a fixed budget, and position noise.
 *
 * s3g_mcmc_relocate  <- the opacity / scale update of 3DGS-MCMC's relocate_gs and add_new_gs
 *                       (scene/gaussian_model.py: _update_params with the compute_relocation CUDA kernel) and its
 *                       replace_tensors_to_optimizer; gsplat strategy/ops.py relocate / sample_add
 * For the n pairs (src[j], dst[j]) (DEVICE int64 [n]) with ratio[j] (DEVICE int32 [n]: 1 + the number of times src[j]
 * was drawn): the caller has already copied row src[j] to row dst[j] of every per-Gaussian tensor.  With x the raw
 * opacity of row dst[j], o = sigmoid(x), N = min(ratio[j], 51):
 *   o' = 1 - (1 - o)^(1/N),
 *   D  = sum_{i=1..N} sum_{k=0..i-1} C(i-1,k) (-1)^k o'^(k+1) / sqrt(k+1),
 *   opacity <- logit(clamp(o', min_opacity, 1 - 2^-23)),   scaling[k] <- log((o / D) exp(scaling[k]))
 * written to rows dst[j] AND src[j] of opacity [rows,1] and scaling [rows,3] (raw, in place).  Everything is evaluated
 * in double (the published kernels use float32, where the alternating sum cancels badly at large N); D uses the
 * unclamped o'.  N = 1 keeps the raw values unless the clamp applies.  1 - (1 - o')^N = o before the clamp.
 * zero: HOST array of n_zero <= 32 descriptors; descriptor t's dst [rows, row_floats] float32 is zeroed at row dst[j],
 * and also at row src[j] when zero_new != 0 (the twelve Adam moments; the densification accumulators pass 0).  Its
 * src field is not read.
 * Rows dst[.] must be distinct and disjoint from rows src[.] (the same src may repeat): thread j reads only row dst[j].
 * One launch, no host synchronisation.  n == 0 does nothing.
 * S3G_ERR_ARG before any launch: n < 0; n_zero outside 0..32 or a NULL descriptor array with n_zero > 0; with n > 0, a
 * NULL pointer, a descriptor with a NULL dst or row_floats <= 0, or min_opacity outside (0, 1).
 *
 * s3g_mcmc_noise  <- the noise block after optimizer.step() in 3DGS-MCMC's train.py (build_scaling_rotation,
 *                    op_sigmoid, torch.bmm); gsplat MCMCStrategy inject_noise_to_position
 * xyz DEVICE float [P,3] (in place), the raw scaling [P,3], rotation [P,4] (w,x,y,z, not normalised) and opacity [P],
 * eps [P,3] (standard normal):
 *   gate = 1 / (1 + exp(-100 ((1 - sigmoid(opacity)) - 0.995))),  Sigma = R(q) diag(exp(scaling)^2) R(q)^T,
 *   xyz += step * gate * Sigma eps,   step = xyz_lr * noise_lr.
 * One elementwise launch: 56 bytes read and 12 written per Gaussian.  P == 0 does nothing.
 * S3G_ERR_ARG before any launch: P < 0, a NULL pointer, P > INT_MAX / 4. */
int s3g_mcmc_relocate(int n, const int64_t* src, const int64_t* dst, const int32_t* ratio, float min_opacity,
                      float* opacity, float* scaling, int n_zero, const s3g_row_tensor* zero, void* stream);
int s3g_mcmc_noise(int P, float* xyz, const float* scaling, const float* rotation, const float* opacity,
                   const float* eps, float step, void* stream);

/* ---- initialisation -------------------------------------------------------------------------
 * s3g_knn_mean_dist2  <- simple_knn._C.distCUDA2 (SimpleKNN::knn)   submodules/simple-knn/simple_knn.cu:185-221,
 *                        called at scene/gaussian_model.py:153 to initialise the scales
 * mean_dist2[i] = mean of the squared distances from points[i] to its 3 nearest OTHER points
 * (exact; coincident points count with distance 0).  points: f32[P,3]; workspace:
 * s3g_knn_workspace_bytes(P) bytes.  No host synchronisation. */
size_t s3g_knn_workspace_bytes(int P);
int s3g_knn_mean_dist2(int P, const float* points, float* mean_dist2, void* workspace, void* stream);

/* ---- gradient all-reduce over peer-mapped memory --------------------------------------------
 * The view-parallel step ends with sum(grads) over ranks; the reference has no distributed code, the
 * baseline is ncclAllReduce.  bufs: HOST array of `world` DEVICE pointers, bufs[p] = rank p's copy of the
 * same symmetric float32 buffer of `numel` elements (multiple of 4), peer-mapped into this process
 * (torch.distributed._symmetric_memory / cuMem VMM / cudaIpc).  Rank `rank` calls, on its own device:
 *     <all ranks wrote their contribution; cross-rank barrier>
 *     s3g_peer_reduce_scatter   - sums slice `rank` over all peers (direct NVLink loads) into bufs[rank]
 *     <barrier>
 *     s3g_peer_all_gather       - pulls the other reduced slices from their owners into bufs[rank]
 *     <barrier before the buffer is written again>
 * The kernels never wait on remote state; ordering is the caller's barriers (s3gaussian_b200/dp.py). */
int s3g_peer_reduce_scatter(int world, int rank, const void* const* bufs, int64_t numel, void* stream);
int s3g_peer_all_gather(int world, int rank, const void* const* bufs, int64_t numel, void* stream);
/* NVLS variant: one kernel on the MULTICAST address of the same symmetric buffer (multimem.ld_reduce +
 * multimem.st on slice `rank`), barriers before and after as above.  Not measured on H100. */
int s3g_peer_nvls_all_reduce(int world, int rank, void* multicast_ptr, int64_t numel, void* stream);
/* second half of the exchange started by s3g_rasterize_backward with a peer sink: stage_local = this rank's staging
 * [world][chunk]; results go to bucket_multicast (multimem.st) when non-NULL, else to bucket_ptrs[0..world-1]. */
int s3g_peer_reduce_gather(int world, int rank, void* stage_local, const void* const* bucket_ptrs,
                           void* bucket_multicast, int64_t numel, int64_t chunk, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* S3G_B200_H */
