"""Per-image bilateral-grid colour correction on the device (csrc/bilagrid.cuh; include/s3g_b200.h, "bilateral-grid
colour correction").

Wang et al., *Bilateral Guided Radiance Field Processing* (SIGGRAPH 2024), as gsplat's ``lib_bilagrid`` offers it
(``--use_bilateral_grid``): every training image gets a small grid of 3x4 affine colour transforms indexed by pixel
position and luminance, the render is corrected through its image's grid before the photometric loss, and a
total-variation term keeps the grids smooth.  Per-camera exposure and white balance are then absorbed by the grids
instead of by floaters and view-dependent colour.

``BilateralGrid(num, grid_X=16, grid_Y=16, grid_W=8)`` holds ``grids`` ``[num, 12, grid_W, grid_Y, grid_X]`` in
gsplat's layout and initialisation (the identity at every cell), so a gsplat ``bil_grids.state_dict()`` loads
unchanged.  ``slice(rgb, image_ids)`` corrects images, ``tv_loss()`` is the regulariser; both are differentiable and
their gradients repeat bit for bit.  CUDA only; there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
import numbers

import torch
from torch import nn

from . import _lib


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ids_array(ids):
    return (C.c_int32 * len(ids))(*ids)


class _Slice(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grids, rgb, ids):
        out = _slice_forward(grids, rgb, ids)
        ctx.ids = ids
        ctx.save_for_backward(grids, rgb)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        grids, rgb = ctx.saved_tensors
        ids = ctx.ids
        lib = _lib.load()
        N, _, L, GY, GX = grids.shape
        B, _, H, W = rgb.shape
        grad_out = grad_out.contiguous()
        grad_grids = torch.zeros_like(grids)
        grad_rgb = torch.empty_like(rgb) if ctx.needs_input_grad[1] else None
        ws = torch.empty(lib.s3g_bilagrid_slice_backward_workspace_bytes(N, L, GY, GX, B, H, W), dtype=torch.uint8,
                         device=rgb.device)
        with torch.cuda.device(rgb.device):
            _lib.check(lib.s3g_bilagrid_slice_backward(
                N, L, GY, GX, grids.data_ptr(), B, H, W, _ids_array(ids), rgb.data_ptr(), grad_out.data_ptr(),
                grad_rgb.data_ptr() if grad_rgb is not None else None, grad_grids.data_ptr(), ws.data_ptr(),
                _stream()), "s3g_bilagrid_slice_backward")
        return (grad_grids if ctx.needs_input_grad[0] else None), grad_rgb, None


def _slice_forward(grids, rgb, ids):
    lib = _lib.load()
    N, _, L, GY, GX = grids.shape
    B, _, H, W = rgb.shape
    out = torch.empty_like(rgb)
    with torch.cuda.device(rgb.device):
        _lib.check(lib.s3g_bilagrid_slice_forward(N, L, GY, GX, grids.data_ptr(), B, H, W, _ids_array(ids),
                                                  rgb.data_ptr(), out.data_ptr(), _stream()),
                   "s3g_bilagrid_slice_forward")
    return out


class _TvLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, grids):
        lib = _lib.load()
        N, _, L, GY, GX = grids.shape
        loss = torch.empty((), dtype=torch.float32, device=grids.device)
        ws = torch.empty(lib.s3g_bilagrid_tv_workspace_bytes(N, L, GY, GX), dtype=torch.uint8, device=grids.device)
        with torch.cuda.device(grids.device):
            _lib.check(lib.s3g_bilagrid_tv_forward(N, L, GY, GX, grids.data_ptr(), loss.data_ptr(), ws.data_ptr(),
                                                   _stream()), "s3g_bilagrid_tv_forward")
        ctx.save_for_backward(grids)
        return loss

    @staticmethod
    def backward(ctx, g):
        (grids,) = ctx.saved_tensors
        lib = _lib.load()
        N, _, L, GY, GX = grids.shape
        gs = g.reshape(1).to(torch.float32).contiguous()
        grad = torch.empty_like(grids)
        with torch.cuda.device(grids.device):
            _lib.check(lib.s3g_bilagrid_tv_backward(N, L, GY, GX, grids.data_ptr(), gs.data_ptr(), grad.data_ptr(),
                                                    _stream()), "s3g_bilagrid_tv_backward")
        return grad


def _check_grids(grids):
    if grids.dim() != 5 or grids.shape[1] != 12 or min(grids.shape) < 1:
        raise ValueError(f"BilateralGrid: grids must be [N, 12, L, GY, GX] with every size >= 1, got "
                         f"{tuple(grids.shape)}")
    if grids.dtype != torch.float32 or not grids.is_contiguous():
        raise ValueError("BilateralGrid: grids must be contiguous float32")


def _check_device(grids):
    if not grids.is_cuda:
        raise RuntimeError("BilateralGrid: the grids must be on a CUDA device (there is no CPU path); call .cuda()")


class BilateralGrid(nn.Module):
    """``num`` bilateral grids of ``grid_W`` luminance levels x ``grid_Y`` x ``grid_X`` cells (gsplat's
    ``BilateralGrid``), one per training image.  Memory: ``num * 12 * grid_W * grid_Y * grid_X * 4`` bytes, plus twice
    that for Adam's moments."""

    def __init__(self, num, grid_X=16, grid_Y=16, grid_W=8):
        super().__init__()
        for name, v in (("num", num), ("grid_X", grid_X), ("grid_Y", grid_Y), ("grid_W", grid_W)):
            if not isinstance(v, numbers.Integral) or isinstance(v, bool) or v < 1:
                raise ValueError(f"BilateralGrid: {name} must be an integer >= 1, got {v!r}")
        self.grid_width, self.grid_height, self.grid_guidance = grid_X, grid_Y, grid_W
        eye = torch.tensor([1.0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0])
        self.grids = nn.Parameter(eye.reshape(1, 12, 1, 1, 1).repeat(num, 1, grid_W, grid_Y, grid_X).contiguous())

    @property
    def num(self):
        return self.grids.shape[0]

    def _ids(self, image_ids, B):
        if isinstance(image_ids, numbers.Integral) and not isinstance(image_ids, bool):
            ids = [int(image_ids)]
        elif isinstance(image_ids, torch.Tensor):
            raise ValueError("BilateralGrid.slice: image_ids must be a Python int or a sequence of ints (checked on "
                             "the host), not a tensor")
        else:
            try:
                ids = list(image_ids)
            except TypeError:
                raise ValueError(f"BilateralGrid.slice: image_ids must be an int or a sequence of ints, got "
                                 f"{type(image_ids).__name__}") from None
            if not all(isinstance(i, numbers.Integral) and not isinstance(i, bool) for i in ids):
                raise ValueError("BilateralGrid.slice: image_ids must all be ints")
            ids = [int(i) for i in ids]
        if len(ids) != B:
            raise ValueError(f"BilateralGrid.slice: {len(ids)} image ids for {B} images")
        bad = [i for i in ids if not 0 <= i < self.num]
        if bad:
            raise ValueError(f"BilateralGrid.slice: image ids {bad} outside [0, {self.num})")
        if len(set(ids)) != len(ids):
            raise ValueError(f"BilateralGrid.slice: duplicate image ids in {ids}")
        return ids

    def slice(self, rgb: torch.Tensor, image_ids) -> torch.Tensor:
        """``rgb`` [3,H,W] or [B,3,H,W] (CUDA float32 contiguous, on the grids' device) corrected through the grids
        ``image_ids`` (an int, or B distinct ints): ``A[:, :3] rgb + A[:, 3]`` per pixel, A the trilinear
        interpolation of the image's grid at the pixel centre and luminance.  Same shape as ``rgb``; differentiable
        with respect to ``rgb`` and ``grids``."""
        grids = self.grids
        _check_grids(grids)
        if not isinstance(rgb, torch.Tensor) or rgb.dim() not in (3, 4) or rgb.shape[-3] != 3 or rgb.numel() == 0:
            raise ValueError(f"BilateralGrid.slice: rgb must be [3,H,W] or [B,3,H,W] and not empty, got "
                             f"{tuple(rgb.shape) if isinstance(rgb, torch.Tensor) else type(rgb).__name__}")
        if rgb.dtype != torch.float32:
            raise ValueError(f"BilateralGrid.slice: rgb must be float32, got {rgb.dtype}")
        if not rgb.is_contiguous():
            raise ValueError("BilateralGrid.slice: rgb must be contiguous")
        x = rgb if rgb.dim() == 4 else rgb.unsqueeze(0)
        ids = self._ids(image_ids, x.shape[0])
        _check_device(grids)
        if rgb.device != grids.device:
            raise RuntimeError(f"BilateralGrid.slice: rgb is on {rgb.device}, the grids on {grids.device}; CUDA "
                               "tensors on one device only (there is no CPU path)")
        if torch.is_grad_enabled() and (x.requires_grad or grids.requires_grad):
            out = _Slice.apply(grids, x, tuple(ids))
        else:
            out = _slice_forward(grids.detach(), x.detach(), ids)
        return out if rgb.dim() == 4 else out.squeeze(0)

    def tv_loss(self) -> torch.Tensor:
        """gsplat's ``total_variation_loss(grids)`` as a 0-d float32 tensor, differentiable in ``grids``."""
        _check_grids(self.grids)
        _check_device(self.grids)
        return _TvLoss.apply(self.grids)
