"""3DGS-MCMC's densification on the device (csrc/mcmc.cuh; include/s3g_b200.h, "MCMC densification").

``relocate(opacity, scaling, src, dst, ratio, min_opacity, zero)`` gives the pairs (src[j], dst[j]) the relocated raw
opacity and scales of 3DGS-MCMC's ``compute_relocation`` (evaluated in double) and zeroes the rows of the tensors in
`zero`; ``inject_noise(xyz, scaling, rotation, opacity, step, eps)`` adds 3DGS-MCMC's covariance-shaped position noise.
``GaussianModel.relocate_gs`` / ``add_new_gs`` / ``inject_noise`` are the users.  CUDA only; there is no CPU path.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check_raw(opacity, scaling):
    if not (opacity.is_cuda and scaling.is_cuda):
        raise RuntimeError("mcmc: CUDA tensors only (there is no CPU path)")
    rows = opacity.shape[0]
    if opacity.numel() != rows or scaling.shape != (rows, 3):
        raise ValueError(f"mcmc: opacity {tuple(opacity.shape)} and scaling {tuple(scaling.shape)} must be [P,1] and "
                         "[P,3] for one P")
    for t in (opacity, scaling):
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise TypeError("mcmc: contiguous float32 tensors only")


def relocate(opacity: torch.Tensor, scaling: torch.Tensor, src: torch.Tensor, dst: torch.Tensor, ratio: torch.Tensor,
             min_opacity: float, zero=()):
    """In place on the raw `opacity` [P,1] and `scaling` [P,3]: rows dst[j] and src[j] <- the relocation of row dst[j]
    (which the caller made a copy of row src[j]) with N = min(ratio[j], 51).  `zero`: (tensor [P,...], at_src) pairs,
    each tensor zeroed at rows dst[j] and, with at_src, at rows src[j] too.  One launch."""
    _check_raw(opacity, scaling)
    n = int(dst.numel())
    if src.numel() != n or ratio.numel() != n:
        raise ValueError(f"mcmc.relocate: src {src.numel()}, dst {n} and ratio {ratio.numel()} must have one length")
    if n == 0:
        return
    lib = _lib.load()
    src = src.to(opacity.device, torch.int64).contiguous()
    dst = dst.to(opacity.device, torch.int64).contiguous()
    ratio = ratio.to(opacity.device, torch.int32).contiguous()
    descs = []
    for t, at_src in zero:
        if t.dtype != torch.float32 or not t.is_contiguous() or t.device != opacity.device:
            raise TypeError("mcmc.relocate: zeroed tensors must be contiguous float32 on the opacity's device")
        rf = t[0].numel() if t.dim() > 1 else 1
        if rf:      # zero-width rows (_features_rest at max_sh_degree == 0) hold nothing
            descs.append(_lib.RowTensor(None, t.data_ptr(), int(rf), 1 if at_src else 0))
    arr = (_lib.RowTensor * max(len(descs), 1))(*descs)
    with torch.cuda.device(opacity.device):
        _lib.check(lib.s3g_mcmc_relocate(n, src.data_ptr(), dst.data_ptr(), ratio.data_ptr(), float(min_opacity),
                                         opacity.data_ptr(), scaling.data_ptr(), len(descs), arr, _stream()),
                   "s3g_mcmc_relocate")


def inject_noise(xyz: torch.Tensor, scaling: torch.Tensor, rotation: torch.Tensor, opacity: torch.Tensor, step: float,
                 eps: torch.Tensor):
    """xyz [P,3] += step * gate(o) * R diag(s^2) R^T eps, in place, from the raw scaling [P,3], rotation [P,4] and
    opacity [P,1]; gate = 1 / (1 + exp(-100 ((1 - o) - 0.995))), step = xyz_lr * noise_lr.  One launch."""
    _check_raw(opacity, scaling)
    P = xyz.shape[0]
    if xyz.shape != (P, 3) or opacity.shape[0] != P or rotation.shape != (P, 4) or eps.shape != (P, 3):
        raise ValueError(f"mcmc.inject_noise: xyz {tuple(xyz.shape)}, rotation {tuple(rotation.shape)} and eps "
                         f"{tuple(eps.shape)} must be [P,3], [P,4] and [P,3] for the opacity's P = {opacity.shape[0]}")
    for t in (xyz, rotation, eps):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.device != opacity.device:
            raise TypeError("mcmc.inject_noise: contiguous float32 tensors on one device only")
    lib = _lib.load()
    with torch.cuda.device(xyz.device):
        _lib.check(lib.s3g_mcmc_noise(P, xyz.data_ptr(), scaling.data_ptr(), rotation.data_ptr(), opacity.data_ptr(),
                                      eps.data_ptr(), float(step), _stream()), "s3g_mcmc_noise")
