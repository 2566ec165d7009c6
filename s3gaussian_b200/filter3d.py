"""Mip-Splatting's 3-D smoothing filter on the device (csrc/filter3d.cuh; include/s3g_b200.h, "3-D smoothing filter").

``compute_filter_3d(xyz, cameras)`` gives every Gaussian the world-space size below which no training camera could
have resolved it (``filter_3D`` of Mip-Splatting's ``GaussianModel.compute_3D_filter``), and
``apply_filter_3d(scales, opacity, filter_3d)`` widens the activated scales by it and lowers the opacities so that
``opacity * prod(scales)`` is kept (``get_scaling_with_3D_filter`` / ``get_opacity_with_3D_filter``).  The filter is a
constant: it gets no gradient.  CUDA only; there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
import math

import torch

from . import _lib


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def camera_tensors(cameras, device):
    """-> (viewmatrices [C,16], cams [C,4] = (width, height, focal_x, focal_y)) as float32 on `device`, from anything
    with world_view_transform, image_width, image_height, FoVx and FoVy (the reference's Camera, SyntheticCamera)."""
    views = torch.stack([c.world_view_transform.detach().to("cpu", torch.float32).reshape(16) for c in cameras])
    cams = torch.tensor([[float(c.image_width), float(c.image_height),
                          c.image_width / (2.0 * math.tan(c.FoVx * 0.5)), c.image_height / (2.0 * math.tan(c.FoVy * 0.5))]
                         for c in cameras], dtype=torch.float32)
    return views.to(device).contiguous(), cams.to(device).contiguous()


def compute_filter_3d(xyz: torch.Tensor, cameras) -> torch.Tensor:
    """[P,1] float32 filter of the means `xyz` [P,3] (CUDA) seen from the training `cameras`: d / F * sqrt(0.2), with d
    the smallest depth at which a camera sees the mean (z > 0.2, inside the image widened by 15 % on every side) and F
    the largest focal_x of the set; a mean no camera sees takes the largest d of the seen ones, and with none seen the
    filter is 0."""
    cameras = list(cameras)
    if not xyz.is_cuda:
        raise RuntimeError("compute_filter_3d: CUDA tensors only (there is no CPU path)")
    if not cameras:
        raise ValueError("compute_filter_3d: needs at least one camera")
    lib = _lib.load()
    with torch.no_grad():
        xyz = xyz.detach().to(torch.float32).contiguous()
        P = xyz.shape[0]
        views, cams = camera_tensors(cameras, xyz.device)
        out = torch.empty((P, 1), dtype=torch.float32, device=xyz.device)
        ws = torch.empty(max(lib.s3g_filter3d_compute_workspace_bytes(P), 1), dtype=torch.uint8, device=xyz.device)
        with torch.cuda.device(xyz.device):
            _lib.check(lib.s3g_filter3d_compute(P, xyz.data_ptr(), len(cameras), views.data_ptr(), cams.data_ptr(),
                                                out.data_ptr(), ws.data_ptr(), _stream()), "s3g_filter3d_compute")
    return out


class _ApplyFilter3D(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scales, opacity, filter_3d):
        lib = _lib.load()
        P = scales.shape[0]
        out_scales = torch.empty_like(scales)
        out_opacity = torch.empty_like(opacity)
        with torch.cuda.device(scales.device):
            _lib.check(lib.s3g_filter3d_apply_forward(P, scales.data_ptr(), opacity.data_ptr(), filter_3d.data_ptr(),
                                                      out_scales.data_ptr(), out_opacity.data_ptr(), _stream()),
                       "s3g_filter3d_apply_forward")
        ctx.save_for_backward(scales, opacity, filter_3d)
        return out_scales, out_opacity

    @staticmethod
    def backward(ctx, g_scales_out, g_opacity_out):
        lib = _lib.load()
        scales, opacity, filter_3d = ctx.saved_tensors
        g_scales_out, g_opacity_out = g_scales_out.contiguous(), g_opacity_out.contiguous()
        g_scales, g_opacity = torch.empty_like(scales), torch.empty_like(opacity)
        with torch.cuda.device(scales.device):
            _lib.check(lib.s3g_filter3d_apply_backward(
                scales.shape[0], scales.data_ptr(), opacity.data_ptr(), filter_3d.data_ptr(), g_scales_out.data_ptr(),
                g_opacity_out.data_ptr(), g_scales.data_ptr(), g_opacity.data_ptr(), _stream()),
                "s3g_filter3d_apply_backward")
        return g_scales, g_opacity, None


def apply_filter_3d(scales: torch.Tensor, opacity: torch.Tensor, filter_3d: torch.Tensor):
    """(sqrt(scales^2 + f^2), opacity * sqrt(prod scales^2 / prod (scales^2 + f^2))) for the activated `scales` [P,3] and
    `opacity` [P,1] and the filter f = `filter_3d` [P,1] (or [P]); differentiable in scales and opacity."""
    P = scales.shape[0]
    if scales.shape != (P, 3) or opacity.numel() != P or filter_3d.numel() != P:
        raise ValueError(f"apply_filter_3d: scales {tuple(scales.shape)}, opacity {tuple(opacity.shape)} and "
                         f"filter_3d {tuple(filter_3d.shape)} must be [P,3], [P,1] and [P,1] for one P")
    if not (scales.is_cuda and opacity.is_cuda and filter_3d.is_cuda):
        raise RuntimeError("apply_filter_3d: CUDA tensors only (there is no CPU path)")
    if not scales.device == opacity.device == filter_3d.device:
        raise RuntimeError(f"apply_filter_3d: scales, opacity and filter_3d are on {scales.device}, {opacity.device} and "
                           f"{filter_3d.device}; they must share one device")
    if scales.dtype != torch.float32 or opacity.dtype != torch.float32 or filter_3d.dtype != torch.float32:
        raise TypeError("apply_filter_3d: float32 tensors only")
    return _ApplyFilter3D.apply(scales.contiguous(), opacity.contiguous(), filter_3d.detach().contiguous())
