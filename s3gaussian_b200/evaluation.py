"""Evaluation on the GPU: drop-in for the reference's ``utils/video_utils.py:render_pixels`` (:74-103, render_func
:106-350) and the per-view metrics it computes (:210-241).

Per view the reference renders three times (full image, dynamic Gaussians, static Gaussians), copies the image to
the host, takes PSNR in torch and SSIM twice with ``skimage.metrics.structural_similarity`` on the CPU.  Here the
view is one split rasterizer pass (render() under no_grad, s3g_rasterize_forward_split) and one metrics kernel
(s3g_eval_metrics): squared errors and the skimage SSIM map, whole image and inside the dynamic mask.  The per-view
numbers stay on the device until the end of the pass.

    from s3gaussian_b200.evaluation import render_pixels     # instead of utils.video_utils.render_pixels
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

SSIM_WIN = 7                   # skimage's default win_size
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


def render_pixels(viewpoint_stack, gaussians, bg, pipe, compute_metrics: bool = True,
                  return_decomposition: bool = True, debug: bool = False, lpips_fn=None):
    """Drop-in for utils/video_utils.py:render_pixels: renders every camera of `viewpoint_stack` (the fine stage,
    under no_grad) and returns the reference's result dict:

      psnr, ssim, masked_psnr, masked_ssim, lpips - means over the views (non_zero_mean, -1 without values);
        masked metrics count only views whose dynamic_mask selects at least one pixel;
      rgbs, depths (normalised by their max), gt_rgbs, static_rgbs, dynamic_rgbs - lists of HWC numpy arrays,
        the lists train.py's render_keys reads; opacities (empty, as in the reference).

    Each camera needs the attributes render() reads plus original_image ([3,H,W]) and, with compute_metrics,
    dynamic_mask ([H,W] or [1,H,W]).  The per-view metrics stay on the device and are read once at the end; the
    images go to host memory view by view, as the reference keeps them.

    lpips is -1 unless `lpips_fn(rgb, gt)` (-> tensor) is given: the reference's LPIPS needs downloaded AlexNet
    weights.  Not covered: the deformation-flow renders (forward_flows / backward_flows, dx_list) and
    save_seperate_pcd (render_func :243-299), which train.py's render_keys do not use; `debug` only affects those.
    """
    from .gaussian_renderer import render
    rgbs, gt_rgbs, depths, static_rgbs, dynamic_rgbs = [], [], [], [], []
    per_view, lpipss = [], []
    with torch.no_grad():
        for cam in viewpoint_stack:
            pkg = render(cam, gaussians, pipe, bg, return_decomposition=return_decomposition, return_dx=True)
            rgb = pkg["render"]
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
            if "render_s" in pkg:
                static_rgbs.append(_hwc(pkg["render_s"]))
            if "render_d" in pkg:
                dynamic_rgbs.append(_hwc(pkg["render_d"]))
            depth = _hwc(pkg["depth"])
            depth /= depth.max()   # :198
            depths.append(depth)
        metrics = torch.stack(per_view).cpu().numpy() if per_view else np.zeros((0, 5))   # the one metrics read
        lp = [float(v) for v in torch.stack(lpipss).cpu()] if lpipss else []

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
    res["opacities"] = []
    if gt_rgbs:
        res["gt_rgbs"] = gt_rgbs
    if static_rgbs:
        res["static_rgbs"] = static_rgbs
    if dynamic_rgbs:
        res["dynamic_rgbs"] = dynamic_rgbs
    return res
