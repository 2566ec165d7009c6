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
 *   s3g_deform_forward /    <- deform_network.forward_dynamic            scene/deformation.py:216-231
 *   s3g_deform_backward        + HexPlaneField.forward                   scene/hexplane.py:160-183
 *                              + activations / Python SH->RGB            gaussian_renderer/__init__.py:99-117
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

#define S3G_ABI_VERSION 1
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
 * before sizing the arena, like rasterizer_impl.cu:282.  No cudaMemcpy, event or stream synchronisation inside. */
int64_t s3g_rasterize_forward(
    s3g_alloc_fn geom_alloc, void* geom_user,
    s3g_alloc_fn binning_alloc, void* binning_user,
    s3g_alloc_fn image_alloc, void* image_user,
    int P, int D, int M,
    const float* background,
    int width, int height,
    const float* means3D,
    const float* shs,
    const float* colors_precomp,
    const float* opacities,
    const float* scales,
    float scale_modifier,
    const float* rotations,
    const float* cov3D_precomp,
    const float* viewmatrix,
    const float* projmatrix,
    const float* cam_pos,
    float tan_fovx, float tan_fovy,
    int prefiltered,
    float* out_color,
    float* out_depth,
    int* radii,
    int debug,
    void* stream);

/* ---- backward (rasterizer_impl.cu:343-444) ------------------------------
 * All dL_* outputs are written for every Gaussian (zeros where radii <= 0), so
 * the caller need NOT pre-zero them (the reference glue zero-fills ten tensors,
 * rasterize_points.cu:154-163).  dL_dconic [P,4] and dL_ddepth [P] are the
 * reference's internal intermediates; pass NULL unless you want them exported
 * (parity tests do).  dL_dmean2D is [P,3] with z untouched = 0
 * (backward.cu:578-579). */
int s3g_rasterize_backward(
    int P, int D, int M, int64_t R,
    const float* background,
    int width, int height,
    const float* means3D,
    const float* shs,
    const float* colors_precomp,
    const float* scales,
    float scale_modifier,
    const float* rotations,
    const float* cov3D_precomp,
    const float* viewmatrix,
    const float* projmatrix,
    const float* campos,
    float tan_fovx, float tan_fovy,
    const int* radii,
    char* geom_buffer,
    char* binning_buffer,
    char* image_buffer,
    const float* dL_dpix,
    const float* dL_dpix_depth,
    float* dL_dmean2D,
    float* dL_dconic,
    float* dL_dopacity,
    float* dL_dcolor,
    float* dL_ddepth,
    float* dL_dmean3D,
    float* dL_dcov3D,
    float* dL_dsh,
    float* dL_dscale,
    float* dL_drot,
    int debug,
    void* stream);

/* ---- backward fused with the first half of the data-parallel gradient exchange ----------------------------------
 * View-parallel training (one camera per GPU, replicated Gaussians; reference batch loop train.py:372-392) sums the
 * per-Gaussian gradients over the ranks every step.  With a peer sink the backward's last kernel does not write
 * dL_dmean3D / dL_dsh / dL_dopacity / dL_dscale / dL_drot locally: every VISIBLE Gaussian's values are stored over
 * NVLink straight into the staging area of the rank that owns that slice of the flat gradient bucket
 * (stage[o] = rank o's area, laid out [world][chunk] floats, pre-zeroed; element e of the bucket lives in slice
 * e / chunk).  s3g_peer_reduce_gather() on every rank then sums its `world` sub-slices in rank order, stores the sums
 * into every rank's bucket (multimem.st through the multicast mapping, or peer stores) and re-zeroes the staging.
 * The five pointers named above may be NULL; everything else is as in s3g_rasterize_backward.  The caller provides
 * the two device-side barriers (all ranks: backward_dp | barrier | reduce_gather | barrier).  off_* are float
 * offsets of the tensors inside the bucket (off_shs % 4 == 0; off_shs ignored with colors_precomp). */
typedef struct s3g_peer_sink {
    int world, rank;
    int64_t chunk;                 /* floats per owner slice, multiple of 4, world * chunk >= bucket size */
    void* stage[16];               /* peer-mapped staging base of every rank */
    int64_t off_means3D, off_shs, off_opacities, off_scales, off_rotations;
} s3g_peer_sink;
int s3g_rasterize_backward_dp(
    int P, int D, int M, int64_t R,
    const float* background,
    int width, int height,
    const float* means3D,
    const float* shs,
    const float* colors_precomp,
    const float* scales,
    float scale_modifier,
    const float* rotations,
    const float* cov3D_precomp,
    const float* viewmatrix,
    const float* projmatrix,
    const float* campos,
    float tan_fovx, float tan_fovy,
    const int* radii,
    char* geom_buffer,
    char* binning_buffer,
    char* image_buffer,
    const float* dL_dpix,
    const float* dL_dpix_depth,
    float* dL_dmean2D,
    float* dL_dconic,
    float* dL_dopacity,
    float* dL_dcolor,
    float* dL_ddepth,
    float* dL_dmean3D,
    float* dL_dcov3D,
    float* dL_dsh,
    float* dL_dscale,
    float* dL_drot,
    int debug,
    void* stream,
    const s3g_peer_sink* sink);

/* ---- one binning, two colour sets -------------------------------------------------
 * render(render_feat=True) rasterizes the same Gaussians twice - once with the RGB colours, once with the
 * three-channel feature colours (gaussian_renderer/__init__.py:173-186, train.py:373) - and the reference runs its
 * whole rasterizer again for the second image.  The *_aux entry points composite both colour sets in ONE pass over
 * one preprocess + one sort: `colors_aux` [P,3] -> `out_color_aux` [3,H,W] (same background), and in the backward
 * `dL_dpix_aux` [3,H,W] -> `dL_dcolor_aux` [P,3]; every other argument and output means what it means in
 * s3g_rasterize_forward / s3g_rasterize_backward, the geometry gradients are those of the SUM of both images'
 * losses. */
int64_t s3g_rasterize_forward_aux(
    s3g_alloc_fn geom_alloc, void* geom_user,
    s3g_alloc_fn binning_alloc, void* binning_user,
    s3g_alloc_fn image_alloc, void* image_user,
    int P, int D, int M,
    const float* background,
    int width, int height,
    const float* means3D,
    const float* shs,
    const float* colors_precomp,
    const float* opacities,
    const float* scales,
    float scale_modifier,
    const float* rotations,
    const float* cov3D_precomp,
    const float* viewmatrix,
    const float* projmatrix,
    const float* cam_pos,
    float tan_fovx, float tan_fovy,
    int prefiltered,
    float* out_color,
    float* out_depth,
    int* radii,
    int debug,
    void* stream,
    const float* colors_aux,
    float* out_color_aux);
int s3g_rasterize_backward_aux(
    int P, int D, int M, int64_t R,
    const float* background,
    int width, int height,
    const float* means3D,
    const float* shs,
    const float* colors_precomp,
    const float* scales,
    float scale_modifier,
    const float* rotations,
    const float* cov3D_precomp,
    const float* viewmatrix,
    const float* projmatrix,
    const float* campos,
    float tan_fovx, float tan_fovy,
    const int* radii,
    char* geom_buffer,
    char* binning_buffer,
    char* image_buffer,
    const float* dL_dpix,
    const float* dL_dpix_depth,
    float* dL_dmean2D,
    float* dL_dconic,
    float* dL_dopacity,
    float* dL_dcolor,
    float* dL_ddepth,
    float* dL_dmean3D,
    float* dL_dcov3D,
    float* dL_dsh,
    float* dL_dscale,
    float* dL_drot,
    int debug,
    void* stream,
    const float* dL_dpix_aux,
    float* dL_dcolor_aux);

/* ---- static / dynamic decomposition in one pass (FORWARD ONLY) -------------------------------
 * render(return_decomposition=True) (gaussian_renderer/__init__.py:177-192) composites the full image, the image of
 * the dynamic Gaussians alone and that of the static ones alone, and the reference runs its whole rasterizer once per
 * image.  This entry point does one preprocess, one sort and one composite walk with three accumulator sets.
 * `group` is a DEVICE uint8 [P] (nonzero = dynamic; may be NULL only when P == 0).  out_color / out_depth / radii
 * are exactly those of s3g_rasterize_forward on all P Gaussians; out_color_d / out_depth_d and out_color_s /
 * out_depth_s ([3,H,W] / [1,H,W], all four required) equal s3g_rasterize_forward on the dynamic / static subset
 * alone - a subset with no Gaussians gives zero images, as P == 0 does.
 * FORWARD ONLY: the state buffers it leaves carry the group in the staged records and must not be passed to any
 * backward.  Returns num_rendered of the full image. */
int64_t s3g_rasterize_forward_split(
    s3g_alloc_fn geom_alloc, void* geom_user,
    s3g_alloc_fn binning_alloc, void* binning_user,
    s3g_alloc_fn image_alloc, void* image_user,
    int P, int D, int M,
    const float* background,
    int width, int height,
    const float* means3D,
    const float* shs,
    const float* colors_precomp,
    const float* opacities,
    const float* scales,
    float scale_modifier,
    const float* rotations,
    const float* cov3D_precomp,
    const float* viewmatrix,
    const float* projmatrix,
    const float* cam_pos,
    float tan_fovx, float tan_fovy,
    int prefiltered,
    float* out_color,
    float* out_depth,
    int* radii,
    int debug,
    void* stream,
    const uint8_t* group,
    float* out_color_d,
    float* out_depth_d,
    float* out_color_s,
    float* out_depth_s);

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

/* ---- state-buffer introspection (tests / debugging) ---------------------
 * buffer: 0 = geometry, 1 = binning, 2 = image.  Looks up a named field of our
 * layout for the given problem size and returns its byte offset from the
 * (128-byte aligned) buffer base, its element size and element count.
 * Fields: geometry: "xyAB","Cod","rgb","depth_key","tiles_touched","rect","clamped"
 *         binning : "point_list" (first field: its offset does not depend on the arena capacity; the sorted tile
 *                   ids are not materialised - "ranges" delimits every tile's slice of the list)
 *         image   : "final_T","n_contrib","ranges"
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
 * sampling and the decoder kernel); keep it for s3g_deform_backward.
 * campos: device float[3]; sh_degree: active degree (0..3). */
int s3g_deform_forward(const s3g_deform_net* net, int P, const float* xyz, const float* scales,
                       const float* rotations, const float* opacity, const float* shs, float time,
                       const float* campos, int sh_degree,
                       float* means3D, float* scales_act, float* rot_act, float* opacity_act,
                       float* colors, float* dx, float* dshs, float* feat, float* features,
                       void* workspace, void* stream);
/* bytes of `workspace` for s3g_deform_forward (tensor-core-ready copies of the Linear weights) */
size_t s3g_deform_forward_workspace_bytes(const s3g_deform_net* net);

/* Training variant: the same forward, which also keeps the decoder's hidden activations (h = feature_out(f) and the
 * hidden layer of every enabled head, scene/deformation.py:56-76 - what autograd keeps for the reference) in the
 * opaque buffer `acts` of s3g_deform_saved_bytes(net, P) bytes, so that s3g_deform_backward_saved does not
 * recompute them.  acts == NULL: identical to s3g_deform_forward.  (1 <= num_levels <= 4; feat_dim 32; width 64.) */
size_t s3g_deform_saved_bytes(const s3g_deform_net* net, int P);
int s3g_deform_forward_save(const s3g_deform_net* net, int P, const float* xyz, const float* scales,
                            const float* rotations, const float* opacity, const float* shs, float time,
                            const float* campos, int sh_degree,
                            float* means3D, float* scales_act, float* rot_act, float* opacity_act,
                            float* colors, float* dx, float* dshs, float* feat, float* features, float* acts,
                            void* workspace, void* stream);

/* Backward of the above.  g_* are dL/d(output) (NULL = zero).  Writes dL/d(raw inputs)
 * [P,*] in full, overwrites the Linear gradients in `grads` and accumulates the plane
 * gradients.  `features` is the buffer the forward filled.  `workspace` must hold
 * s3g_deform_workspace_bytes(net, P) bytes. */
size_t s3g_deform_workspace_bytes(const s3g_deform_net* net, int P);
int s3g_deform_backward(const s3g_deform_net* net, int P, const float* xyz, const float* scales,
                        const float* rotations, const float* opacity, const float* shs, float time,
                        const float* campos, int sh_degree, const float* features,
                        const float* g_means3D, const float* g_scales_act, const float* g_rot_act,
                        const float* g_opacity_act, const float* g_colors, const float* g_dx,
                        const float* g_dshs, const float* g_feat,
                        float* d_xyz, float* d_scales, float* d_rotations, float* d_opacity, float* d_shs,
                        const s3g_deform_net_grads* grads, void* workspace, void* stream);
/* Same with the hidden activations s3g_deform_forward_save stored (acts == NULL: recompute, as above). */
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

/* radii i32[P] (max over the step's views), viewspace_grad f32[P,3] (summed over the views);
 * for radii > 0: max_radii2D = max(max_radii2D, radii); xyz_gradient_accum += |grad[:2]|; denom += 1. */
int s3g_densify_stats(int P, const float* viewspace_grad, const int* radii, float* xyz_gradient_accum,
                      float* denom, float* max_radii2D, void* stream);

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
 * Each plane is the [1,C,H,W] tensor stored channels-last, i.e. physically [H][W][C]; C % 4 == 0, H >= 3.
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
/* second half of the exchange started by s3g_rasterize_backward_dp: stage_local = this rank's staging
 * [world][chunk]; results go to bucket_multicast (multimem.st) when non-NULL, else to bucket_ptrs[0..world-1]. */
int s3g_peer_reduce_gather(int world, int rank, void* stage_local, const void* const* bucket_ptrs,
                           void* bucket_multicast, int64_t numel, int64_t chunk, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* S3G_B200_H */
