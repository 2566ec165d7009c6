"""Evaluation on the GPU: drop-in for the reference's ``utils/video_utils.py:render_pixels`` (:74-103, render_func
:106-350) and the per-view metrics it computes (:210-241).

Per view the reference renders three times (full image, dynamic Gaussians, static Gaussians), copies the image to
the host, takes PSNR in torch and SSIM twice with ``skimage.metrics.structural_similarity`` on the CPU.  In the fine
stage it then renders two deformation-flow images per view (render_func :243-299), each a complete render() with the
flow colours as override_color, the colours made by a torch colour wheel and taken through host numpy.

Here each view's deformation runs once (gaussian_renderer.fine_front), and one rasterizer walk
(s3g_rasterize_forward with its forward-only extras) gives its image, depth, static/dynamic decomposition and flow
images; one metrics kernel (s3g_eval_metrics) takes squared errors and the skimage SSIM map, whole image and inside the dynamic mask.  The flow
colours F(a, a+3) = flow_visualizer(dx_{a+3} - dx_a) come from s3g_flow_colors on the device, once per a.  View u
needs dx_{u+3}, so the front end runs up to three views ahead and the deformed geometry of views not yet walked waits
in a ring.  Memory beyond the reference's per-view state: dx_list is V*P*12 bytes, as the reference keeps it; the ring
holds at most four views' geometry; each live colour array is 16 bytes per Gaussian, and at most four are live.  The
per-view numbers stay on the device until the end of the pass.

    from s3gaussian_b200.evaluation import render_pixels     # instead of utils.video_utils.render_pixels
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

SSIM_WIN = 7                   # skimage's default win_size
NUM_CAMS = 3                   # render_func's num_cams; render_pixels never passes it
_CROP = (SSIM_WIN - 1) // 2


def _eval_sums(image: torch.Tensor, gt: torch.Tensor, mask: torch.Tensor | None) -> torch.Tensor:
    """DEVICE float64 [4C+1] of s3g_eval_metrics: per channel {sse, ssim sum over the interior, masked sse,
    masked ssim sum}, then the mask pixel count."""
    lib = _lib.load()
    Cn, H, W = image.shape
    dev = image.device
    ws = torch.empty(int(lib.s3g_eval_metrics_workspace_bytes(Cn, H, W)), dtype=torch.uint8, device=dev)
    out = torch.empty(4 * Cn + 1, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.s3g_eval_metrics(Cn, H, W, image.data_ptr(), gt.data_ptr(),
                                        mask.data_ptr() if mask is not None else None, out.data_ptr(),
                                        ws.data_ptr(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "eval_metrics")
    return out


def _psnr_of_mse(mse: torch.Tensor) -> torch.Tensor:
    # utils/image_utils.py:17-19, per channel; identical images give inf
    return 20 * torch.log10(1.0 / torch.sqrt(mse))


def _view_metrics(sums: torch.Tensor, Cn: int, H: int, W: int) -> torch.Tensor:
    """DEVICE float64 [5] = {psnr, ssim, masked psnr, masked ssim, mask pixels}; the masked values are NaN when
    the mask is empty.  Every value is the mean over channels of the per-channel value, as the reference's."""
    s = sums[:4 * Cn].view(Cn, 4)
    n = sums[4 * Cn]
    psnr = _psnr_of_mse(s[:, 0] / (H * W)).mean()
    ssim = (s[:, 1] / ((H - 2 * _CROP) * (W - 2 * _CROP))).mean()
    mpsnr = _psnr_of_mse(s[:, 2] / n).mean()
    mssim = (s[:, 3] / n).mean()
    return torch.stack([psnr, ssim, mpsnr, mssim, n])


def _check_pair(image: torch.Tensor, gt: torch.Tensor):
    if image.dim() != 3 or tuple(image.shape) != tuple(gt.shape):
        raise ValueError(f"image and gt must both be [C,H,W], got {tuple(image.shape)} and {tuple(gt.shape)}")
    if not image.is_cuda or gt.device != image.device:
        raise RuntimeError("s3gaussian_b200 has no CPU path: image and gt must be CUDA tensors on one device")
    Cn, H, W = image.shape
    if H < SSIM_WIN or W < SSIM_WIN:
        raise ValueError(f"image sides must be >= {SSIM_WIN} for the SSIM window, got {H}x{W}")
    return image.float().contiguous(), gt.float().contiguous()


def _mask_u8(mask, H: int, W: int, dev) -> torch.Tensor:
    m = torch.as_tensor(mask)
    if m.numel() != H * W:
        raise ValueError(f"dynamic_mask must have H*W = {H * W} elements, got {tuple(m.shape)}")
    return m.reshape(H, W).to(device=dev, dtype=torch.bool, non_blocking=True).contiguous().view(torch.uint8)


def image_metrics(image: torch.Tensor, gt: torch.Tensor, dynamic_mask=None) -> dict:
    """PSNR and SSIM of a [C,H,W] image against its ground truth, as render_pixels computes them
    (utils/video_utils.py:210-241): {"psnr", "ssim"} and, when `dynamic_mask` ([H,W] or [1,H,W], nonzero = in)
    selects at least one pixel, {"masked_psnr", "masked_ssim"} - 0-d float64 tensors on the image's device.
    ssim is skimage's mean SSIM (7x7 uniform window, map cropped by 3 pixels); masked_ssim averages the uncropped
    map over the mask (full=True).  Deciding whether a device mask is empty reads one number back."""
    image, gt = _check_pair(image, gt)
    Cn, H, W = image.shape
    mask = _mask_u8(dynamic_mask, H, W, image.device) if dynamic_mask is not None else None
    v = _view_metrics(_eval_sums(image, gt, mask), Cn, H, W)
    out = {"psnr": v[0], "ssim": v[1]}
    if mask is not None and bool(mask.any()):
        out.update({"masked_psnr": v[2], "masked_ssim": v[3]})
    return out


def _non_zero_mean(x):
    # utils/video_utils.py:44-46
    return sum(x) / len(x) if len(x) > 0 else -1


def _hwc(t: torch.Tensor) -> np.ndarray:
    # get_numpy(x.permute(1, 2, 0)) of the reference: an HWC host array
    return t.permute(1, 2, 0).cpu().numpy()


def flow_plan(V: int):
    """(forward_flows, backward_flows) of render_func (utils/video_utils.py:253-299) on V views: for each image, in
    the reference's order, (view, a) - the image renders `view` coloured by F(a, a + 3).  For V >= 6, forward_flows[u]
    uses F(u, u+3) and, for the last three views, F(u-3, u); backward_flows[u] uses F(u-3, u) and, for the first three
    views, F(u, u+3).  For V = 4 and 5 the reference's hard-coded boundary tests pair views as restated here."""
    n = NUM_CAMS
    fwd = [(t, t) for t in range(V - n)]
    fwd += [(V - n + i, a) for i, a in enumerate(range(max(V - 2 * n, 0), V - n))]
    bwd = [(i, t - n) for i, t in enumerate(range(n, min(2 * n, V)))]
    bwd += [(t, t - n) for t in range(n, V)]
    return fwd, bwd


def flow_colors(dx_to: torch.Tensor, dx_from: torch.Tensor, normalize: bool = False) -> torch.Tensor:
    """DEVICE float32 [P,4] (rgb in [:, :3]) = flow_visualizer(dx_to - dx_from) of the reference
    (utils/video_utils.py:34-42), with `normalize` also its debug min-max normalisation (s3g_flow_colors)."""
    lib = _lib.load()
    if dx_to.shape != dx_from.shape or dx_to.dim() != 2 or dx_to.size(1) != 3:
        raise ValueError(f"dx_to and dx_from must both be [P,3], got {tuple(dx_to.shape)} and {tuple(dx_from.shape)}")
    if not dx_to.is_cuda or dx_from.device != dx_to.device:
        raise RuntimeError("s3gaussian_b200 has no CPU path: dx_to and dx_from must be CUDA tensors on one device")
    dev = dx_to.device
    P = dx_to.size(0)
    dx_to, dx_from = dx_to.float().contiguous(), dx_from.float().contiguous()
    out = torch.empty((P, 4), dtype=torch.float32, device=dev)
    ws = torch.empty(int(lib.s3g_flow_colors_workspace_bytes(P)), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.s3g_flow_colors(P, dx_to.data_ptr(), dx_from.data_ptr(), int(bool(normalize)), out.data_ptr(),
                                       ws.data_ptr(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "flow_colors")
    return out


def render_pixels(viewpoint_stack, gaussians, bg, pipe, compute_metrics: bool = True,
                  return_decomposition: bool = True, debug: bool = False, lpips_fn=None, with_opacity: bool = False,
                  sky_model=None):
    """Drop-in for utils/video_utils.py:render_pixels: renders every camera of `viewpoint_stack` (the fine stage,
    under no_grad) and returns the reference's result dict:

      psnr, ssim, masked_psnr, masked_ssim, lpips - means over the views (non_zero_mean, -1 without values);
        masked metrics count only views whose dynamic_mask selects at least one pixel;
      rgbs, depths (normalised by their max), gt_rgbs, static_rgbs, dynamic_rgbs - lists of HWC numpy arrays,
        the lists train.py's render_keys reads; opacities (empty, as in the reference, unless with_opacity).

    with_opacity also fills the lists the reference declares but never fills: opacities and median_depths and, with
    the decomposition, static_opacities and dynamic_opacities, one HxW numpy array per view (the alpha and median-depth
    images of GaussianRasterizer.forward_opacity, and the static / dynamic subsets' alpha images) - what save_videos'
    sky_masks panel (1 - opacity) stacks.

    Each camera needs the attributes render() reads plus original_image ([3,H,W]) and, with compute_metrics,
    dynamic_mask ([H,W] or [1,H,W]).  The per-view metrics stay on the device and are read once at the end; the
    images go to host memory view by view, as the reference keeps them.

    With the fine stage's dx (not no_dx), also dx_list (the per-view dx, device tensors) and, from four views on,
    forward_flows / backward_flows (lists of HWC numpy arrays in the reference's order, see flow_plan); `debug`
    min-max normalises the flow colours, as the reference's.  lpips is -1 unless `lpips_fn(rgb, gt)` (-> tensor) is
    given; s3gaussian_b200.lpips.LPIPS() computes the reference's LPIPS on the device.  Not covered: save_seperate_pcd (render_func
    :243-249), which render_pixels never enables.

    sky_model (a s3gaussian_b200.sky.Background_Model at the views' image size): each view's rgbs image, and the
    PSNR / SSIM / LPIPS computed on it, is the render over a zero background plus (1 - alpha) times the view's sky
    (sky.sky_camera gives its c2w / intrinsic); the alpha image comes from the same walk.  The static / dynamic
    images are unchanged.
    """
    from .gaussian_renderer import (dynamic_mask_of, fine_front, pipe_lens_kwargs, pipe_rasterizer_kwargs,
                                    raster_settings_for)
    from .diff_gaussian_rasterization import GaussianRasterizer
    rgbs, gt_rgbs, depths, static_rgbs, dynamic_rgbs = [], [], [], [], []
    opacities, median_depths, static_opacities, dynamic_opacities = [], [], [], []
    per_view, lpipss, dx_list = [], [], []
    V = len(viewpoint_stack)
    plan_fwd, plan_bwd = flow_plan(V)
    flow_images = {}                          # (view, a) -> HWC array
    with torch.no_grad():
        ring = {}                             # view -> (settings, geometry) of views run ahead, not yet walked
        colours = {}                          # a -> F(a, a + 3), dropped after its last view
        last_use = {}
        for view, a in plan_fwd + plan_bwd:
            last_use[a] = max(last_use.get(a, -1), view)

        def front(i):
            cam = viewpoint_stack[i]
            rs = raster_settings_for(cam, gaussians, pipe, bg)
            geo = fine_front(cam, gaussians, pipe, rs.campos, gaussians.get_features)
            if geo[6] is not None:
                dx_list.append(geo[6])
            ring[i] = (rs, geo)

        n_front = 0
        for u, cam in enumerate(viewpoint_stack):
            if n_front == u:
                front(u)
                n_front += 1
            with_flows = bool(plan_fwd) and len(dx_list) > 0
            while with_flows and n_front < min(V, u + NUM_CAMS + 1):   # view u needs dx_{u+3}
                front(n_front)
                n_front += 1
            rs, (means3D, scales, rotations, opacity, shs, colors_precomp, dx, _, _) = ring.pop(u)
            need = sorted({a for v, a in plan_fwd + plan_bwd if v == u}) if with_flows else []
            for a in need:
                if a not in colours:
                    colours[a] = flow_colors(dx_list[a + NUM_CAMS], dx_list[a], normalize=debug)
            group = dynamic_mask_of(dx) if return_decomposition and dx is not None else None
            out = GaussianRasterizer(raster_settings=rs, **pipe_rasterizer_kwargs(pipe),
                                     **pipe_lens_kwargs(pipe, cam)).forward_eval(
                means3D=means3D, means2D=torch.zeros_like(means3D), opacities=opacity, group=group,
                flow_colors=[colours[a] for a in need], shs=shs, colors_precomp=colors_precomp, scales=scales,
                rotations=rotations, **({"with_opacity": True} if with_opacity or sky_model is not None else {}))
            rgb, _, depth_t, decomposition, flows = out[:5]
            if sky_model is not None:
                # rgb = render_bg0 + (1 - alpha) bg (the forward-opacity contract), so the sky composite swaps bg out
                from .sky import sky_camera
                alpha = out[5][0]
                sky = sky_model(*sky_camera(cam))
                rgb = rgb + (1.0 - alpha) * (sky - rs.bg.reshape(-1, 1, 1))
            if with_opacity:
                alpha, median, alpha_d, alpha_s = out[5]
                opacities.append(alpha[0].cpu().numpy())
                median_depths.append(median[0].cpu().numpy())
                if alpha_d is not None:
                    dynamic_opacities.append(alpha_d[0].cpu().numpy())
                    static_opacities.append(alpha_s[0].cpu().numpy())
            for a in [a for a in colours if last_use[a] <= u]:
                del colours[a]
            dev = rgb.device
            gt_rgb = torch.as_tensor(cam.original_image).to(dev, non_blocking=True)
            if compute_metrics:
                image, gt = _check_pair(rgb, gt_rgb)
                Cn, H, W = image.shape
                mask = _mask_u8(cam.dynamic_mask, H, W, dev)
                per_view.append(_view_metrics(_eval_sums(image, gt, mask), Cn, H, W))
                if lpips_fn is not None:
                    lpipss.append(torch.as_tensor(lpips_fn(rgb, gt_rgb)).mean())
            rgbs.append(_hwc(rgb))
            gt_rgbs.append(_hwc(gt_rgb))
            if decomposition is not None:
                static_rgbs.append(_hwc(decomposition[2]))
                dynamic_rgbs.append(_hwc(decomposition[0]))
            depth = _hwc(depth_t)
            depth /= depth.max()   # :198
            depths.append(depth)
            for a, img in zip(need, flows):
                flow_images[(u, a)] = _hwc(img)
        metrics = torch.stack(per_view).cpu().numpy() if per_view else np.zeros((0, 5))   # the one metrics read
        lp = [float(v) for v in torch.stack(lpipss).cpu()] if lpipss else []

    # the reference renders a boundary (view, colours) pair twice: the same image, copied
    used = set()

    def image_of(key):
        img = flow_images[key]
        if key in used:
            return img.copy()
        used.add(key)
        return img
    forward_flows = [image_of(k) for k in plan_fwd] if flow_images else []
    backward_flows = [image_of(k) for k in plan_bwd] if flow_images else []

    res = {}
    if compute_metrics:
        masked = metrics[metrics[:, 4] > 0]
        res["psnr"] = _non_zero_mean([float(v) for v in metrics[:, 0]])
        res["ssim"] = _non_zero_mean([float(v) for v in metrics[:, 1]])
        res["lpips"] = _non_zero_mean(lp) if lpips_fn is not None else -1
        res["masked_psnr"] = _non_zero_mean([float(v) for v in masked[:, 2]])
        res["masked_ssim"] = _non_zero_mean([float(v) for v in masked[:, 3]])
        n = len(viewpoint_stack)
        print(f"Eval over {n} images:")
        for k, name in (("psnr", "PSNR"), ("ssim", "SSIM"), ("lpips", "LPIPS"), ("masked_psnr", "Masked PSNR"),
                        ("masked_ssim", "Masked SSIM")):
            print(f"\t{name}: {res[k]:.4f}")
    else:
        res.update({k: -1 for k in ("psnr", "ssim", "lpips", "masked_psnr", "masked_ssim")})
    res["rgbs"] = rgbs
    res["depths"] = depths
    res["opacities"] = opacities
    if with_opacity:
        res["median_depths"] = median_depths
    if static_opacities:
        res["static_opacities"] = static_opacities
        res["dynamic_opacities"] = dynamic_opacities
    if gt_rgbs:
        res["gt_rgbs"] = gt_rgbs
    if static_rgbs:
        res["static_rgbs"] = static_rgbs
    if dynamic_rgbs:
        res["dynamic_rgbs"] = dynamic_rgbs
    if forward_flows:
        res["forward_flows"] = forward_flows
    if backward_flows:
        res["backward_flows"] = backward_flows
    if dx_list:
        res["dx_list"] = dx_list
    return res
