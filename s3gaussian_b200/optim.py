"""Optimizer step and densification statistics of the reference's training loop as single
CUDA launches.

``FusedAdam`` is a drop-in for the optimizer the reference builds in
``GaussianModel.training_setup`` (scene/gaussian_model.py:170-189):

    self.optimizer = torch.optim.Adam(l, lr=0.0, eps=1e-15)

Same constructor, same param-group dicts (extra keys such as ``"name"`` are kept), same
``state[p] = {"step", "exp_avg", "exp_avg_sq"}`` layout - so the reference's optimizer-state surgery
(``replace_tensor_to_optimizer``, ``_prune_optimizer``, ``cat_tensors_to_optimizer``,
scene/gaussian_model.py:397-470) and ``state_dict()`` checkpoints keep working - but ``step()`` is one
kernel over every tensor of every group (28 B of HBM traffic per element) instead of torch's
per-op foreach launches.  Semantics: torch.optim.Adam with amsgrad=False, weight_decay=0,
maximize=False (anything else raises).  CUDA fp32 tensors only; no CPU path.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


class FusedAdam(torch.optim.Optimizer):
    """``selective_groups``: names of the param groups whose tensors hold one row per Gaussian (``[P, ...]``,
    contiguous).  ``step(visibility=v)`` with ``v`` a bool CUDA tensor ``[P]`` (``radii > 0`` of the step's render, or
    the union over its views) is then selective Adam (upstream 3DGS ``sparse_adam``, gsplat ``SelectiveAdam``): in
    those groups only the rows with ``v[i]`` are updated and every other row keeps its parameter and both moments
    bit for bit (its gradient is not read); the other groups get the dense update in the same launch.  The step
    counter and the bias correction stay global, so an all-true ``v`` gives ``step()``'s bits.  A tensor without a
    gradient is skipped as in ``step()``.  The names are a constructor argument, not a param-group key, so they
    survive ``load_state_dict`` of a torch.optim.Adam checkpoint."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *,
                 maximize=False, selective_groups=()):
        if weight_decay != 0 or amsgrad or maximize:
            raise NotImplementedError("FusedAdam: weight_decay / amsgrad / maximize are not used by the "
                                      "reference (scene/gaussian_model.py:189) and not implemented")
        if lr < 0.0 or eps < 0.0 or not (0.0 <= betas[0] < 1.0) or not (0.0 <= betas[1] < 1.0):
            raise ValueError("FusedAdam: invalid lr / eps / betas")
        if isinstance(selective_groups, str):
            raise TypeError("FusedAdam: selective_groups is a collection of group names")
        self.selective_groups = frozenset(selective_groups)
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,
                                      maximize=maximize))

    def _init_state(self, p):
        st = self.state[p]
        if len(st) == 0:
            st["step"] = torch.tensor(0.0, dtype=torch.float32)       # host scalar, as torch.optim.Adam keeps it
            st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
        return st

    def _check_visibility(self, v):
        if not isinstance(v, torch.Tensor) or v.dtype != torch.bool or v.dim() != 1 or not v.is_contiguous():
            raise RuntimeError("FusedAdam.step: visibility must be a contiguous 1-D bool tensor")
        if not any(g.get("name") in self.selective_groups for g in self.param_groups):
            raise RuntimeError("FusedAdam.step: visibility given, but the optimizer has no per-Gaussian group "
                               f"(selective_groups={sorted(self.selective_groups)})")

    @torch.no_grad()
    def step(self, closure=None, *, visibility=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        v = visibility
        if v is not None:
            self._check_visibility(v)
        # every check runs before any state changes or any launch
        todo = []
        for group in self.param_groups:
            masked = v is not None and group.get("name") in self.selective_groups
            for p in group["params"]:
                if p.grad is None:
                    continue
                if masked:
                    if p.dim() == 0 or p.shape[0] != v.numel():
                        raise RuntimeError(f"FusedAdam.step: group {group.get('name')!r} has {tuple(p.shape)} rows "
                                           f"for a visibility of {v.numel()}")
                    if p.device != v.device:
                        raise RuntimeError("FusedAdam.step: visibility must be on the parameters' device")
                if not p.is_cuda or p.dtype != torch.float32:
                    raise RuntimeError("FusedAdam: CUDA float32 parameters only (there is no CPU path)")
                if p.grad.is_sparse:
                    raise RuntimeError("FusedAdam does not support sparse gradients")
                # the update is elementwise: any dense layout works as long as all four tensors share it
                # (HexPlane planes are channels_last); masked rows must be contiguous
                if p.is_contiguous():
                    fmt = torch.contiguous_format
                elif not masked and p.dim() == 4 and p.is_contiguous(memory_format=torch.channels_last):
                    fmt = torch.channels_last
                else:
                    raise RuntimeError("FusedAdam: parameters must be dense (contiguous or channels_last)" +
                                       ("; per-Gaussian ones contiguous" if masked else ""))
                todo.append((group, p, fmt, p.numel() // p.shape[0] if masked and p.numel() else 0))
        lib = _lib.load()
        by_key = {}     # (device index, betas, eps) -> (descriptors, row widths); one launch per 40 tensors each
        keep = []
        for group, p, fmt, width in todo:
            b1, b2 = group["betas"]
            g = p.grad
            if g.stride() != p.stride():
                g = g.contiguous(memory_format=fmt)
            st = self._init_state(p)
            for k in ("exp_avg", "exp_avg_sq"):
                if st[k].stride() != p.stride():
                    st[k] = st[k].contiguous(memory_format=fmt)
            st["step"] += 1
            keep.append(g)
            descs, widths = by_key.setdefault((p.device.index, float(b1), float(b2), float(group["eps"])), ([], []))
            descs.append(_lib.AdamTensor(p.data_ptr(), g.data_ptr(), st["exp_avg"].data_ptr(),
                                         st["exp_avg_sq"].data_ptr(), p.numel(), float(group["lr"]), int(st["step"])))
            widths.append(width)
        for (dev, b1, b2, eps), (descs, widths) in by_key.items():
            arr = (_lib.AdamTensor * len(descs))(*descs)
            with torch.cuda.device(dev):
                stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
                if v is None:
                    _lib.check(lib.s3g_adam_step(len(descs), arr, b1, b2, eps, stream), "s3g_adam_step")
                else:
                    w = (C.c_int32 * len(widths))(*widths)
                    _lib.check(lib.s3g_adam_step_selective(len(descs), arr, w, v.numel(), v.data_ptr(), b1, b2, eps,
                                                           stream), "s3g_adam_step_selective")
        return loss


def add_densification_stats(viewspace_grad: torch.Tensor, radii: torch.Tensor, xyz_gradient_accum: torch.Tensor,
                            denom: torch.Tensor, max_radii2D: torch.Tensor, viewspace_absgrad: torch.Tensor | None = None,
                            xyz_gradient_accum_abs: torch.Tensor | None = None) -> None:
    """train.py:489-491 in one launch: for ``radii > 0`` update ``max_radii2D`` and call
    ``GaussianModel.add_densification_stats`` (scene/gaussian_model.py:693-695).  In place.
    With ``viewspace_absgrad`` (float32 [P,2], the rasterizer's absgrad) and ``xyz_gradient_accum_abs`` [P,1], both or
    neither, the same launch also adds ``||viewspace_absgrad||`` to ``xyz_gradient_accum_abs`` (s3g_densify_stats_abs)."""
    P = radii.shape[0]
    if (viewspace_absgrad is None) != (xyz_gradient_accum_abs is None):
        raise RuntimeError("add_densification_stats: viewspace_absgrad and xyz_gradient_accum_abs go together")
    extra = () if viewspace_absgrad is None else (viewspace_absgrad, xyz_gradient_accum_abs)
    for t in (viewspace_grad, radii, xyz_gradient_accum, denom, max_radii2D) + extra:
        if not t.is_cuda or not t.is_contiguous():
            raise RuntimeError("add_densification_stats: contiguous CUDA tensors only (there is no CPU path)")
    if radii.dtype != torch.int32 or viewspace_grad.dtype != torch.float32 or viewspace_grad.shape != (P, 3):
        raise RuntimeError("add_densification_stats: radii int32 [P], viewspace_grad float32 [P,3]")
    if xyz_gradient_accum.numel() != P or denom.numel() != P or max_radii2D.numel() != P:
        raise RuntimeError("add_densification_stats: accumulator sizes do not match P")
    if extra:
        if viewspace_absgrad.dtype != torch.float32 or viewspace_absgrad.shape != (P, 2):
            raise RuntimeError("add_densification_stats: viewspace_absgrad float32 [P,2]")
        if xyz_gradient_accum_abs.dtype != torch.float32 or xyz_gradient_accum_abs.numel() != P:
            raise RuntimeError("add_densification_stats: xyz_gradient_accum_abs float32 with P elements")
        _lib.check(_lib.load().s3g_densify_stats_abs(P, viewspace_grad.data_ptr(), viewspace_absgrad.data_ptr(),
                                                     radii.data_ptr(), xyz_gradient_accum.data_ptr(),
                                                     xyz_gradient_accum_abs.data_ptr(), denom.data_ptr(),
                                                     max_radii2D.data_ptr(),
                                                     C.c_void_p(torch.cuda.current_stream().cuda_stream)),
                   "s3g_densify_stats_abs")
        return
    _lib.check(_lib.load().s3g_densify_stats(P, viewspace_grad.data_ptr(), radii.data_ptr(),
                                             xyz_gradient_accum.data_ptr(), denom.data_ptr(), max_radii2D.data_ptr(),
                                             C.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "s3g_densify_stats")


def get_expon_lr_func(lr_init, lr_final, lr_delay_steps=0, lr_delay_mult=1.0, max_steps=1000000):
    """Log-linear learning-rate schedule with optional delay (utils/general_utils.py:196-229)."""
    import math

    def helper(step):
        if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
            return 0.0
        if lr_delay_steps > 0:
            delay_rate = lr_delay_mult + (1 - lr_delay_mult) * math.sin(
                0.5 * math.pi * min(max(step / lr_delay_steps, 0.0), 1.0))
        else:
            delay_rate = 1.0
        t = min(max(step / max_steps, 0.0), 1.0)
        log_lerp = math.exp(math.log(lr_init) * (1 - t) + math.log(lr_final) * t)
        return delay_rate * log_lerp
    return helper
