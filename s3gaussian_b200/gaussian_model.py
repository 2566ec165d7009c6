"""Training state of the Gaussians: the part of the reference's ``GaussianModel``
(scene/gaussian_model.py) that the training loop touches every iteration or every
densification interval - parameters, optimizer, densification statistics, densify / prune.

Same attribute and method names as the reference so ``train.py``-style loops read the same
(``training_setup``, ``update_learning_rate``, ``add_densification_stats``, ``densify``, ``prune``,
``prune_points``, ``reset_opacity``, ``compute_regulation`` ...).  What differs is how the work runs:

* the optimizer is ``FusedAdam`` (one launch per step, optim.py) with the reference's eight groups
  and learning rates (scene/gaussian_model.py:176-189).  Its per-Gaussian groups are the six of ``PARAM_GROUPS``, so
  ``optimizer.step(visibility=radii > 0)`` is selective Adam (only the rows the step's views see are updated);
  ``optimizer.step()`` is the reference's dense step;
* densify / prune rebuild the six parameters, their twelve Adam moments and the four per-Gaussian
  accumulators with ONE row-gather launch per operation (``s3g_gather_rows``) instead of boolean
  indexing + ``torch.cat`` per tensor (gaussian_model.py:411-470); the small mask / index arithmetic
  stays in torch;
* ``prune`` does not call ``torch.cuda.empty_cache()`` (gaussian_model.py:672): nothing is freed to
  the driver, so there is no allocator stall afterwards.

Row order after every operation, Adam moments of kept / new rows, the random samples of
``densify_and_split`` (same ``torch.normal`` call, so the same values for the same generator state)
match the reference bit for bit (tests/test_gpu_train.py runs the reference's own methods side by side).

``create_from_pcd`` uses our distCUDA2 (simple_knn.py, csrc/knn.cuh); ``save_ply`` / ``load_ply`` keep the
reference's attribute layout (io_ply.py).  CUDA only; no CPU path.

Not in the reference: Mip-Splatting's 3-D smoothing filter (filter3d.py).  ``compute_3D_filter(cameras)`` fills
``filter_3D`` [P,1]; ``get_scaling_with_3D_filter`` / ``get_opacity_with_3D_filter`` apply it, and render() does with
``pipe.filter_3d``.  Densify, prune and ``spatial_sort`` carry it (a new row takes its source row's value) until the
loop recomputes it.  It is not saved: ``capture()`` / ``restore()`` and the .ply files keep the reference's layout, so
recompute it from the training cameras after loading.

Not in the reference either: the absolute screen-space gradient statistic (AbsGS; gsplat ``DefaultStrategy(absgrad=True)``).
``densification_step(grad, radii, absgrad)`` also accumulates ``||absgrad||`` into ``xyz_gradient_accum_abs`` [P,1],
which prune and ``spatial_sort`` carry and densify resets like ``xyz_gradient_accum``; ``densify(..., max_grad_abs=T)``
then selects clones and splits on ``||xyz_gradient_accum_abs / denom|| >= T``.  It is not saved: ``capture()`` keeps the
reference's 14-tuple and ``restore()`` starts the accumulator from zero.

Not in the reference either: 3DGS-MCMC's densification (Kheradmand et al. 2024; gsplat ``MCMCStrategy``; mcmc.py), an
alternative to densify / prune with the same names as 3DGS-MCMC.  ``relocate_gs()`` moves every Gaussian with opacity
<= 0.005 onto an alive one drawn by opacity, ``add_new_gs(cap_max)`` grows the model by at most 5 % up to ``cap_max``,
and ``inject_noise(xyz_lr)`` adds covariance-shaped position noise to low-opacity Gaussians after each optimizer step.
Each row copy is the one ``s3g_gather_rows`` launch of densify, followed by one ``s3g_mcmc_relocate`` launch that sets
the drawn rows' and their copies' opacity and scales, zeroes the Adam moments of both and zeroes the copies'
accumulators.  Zeroing the copies' moments differs from the published code, which zeroes only the drawn rows' and lets a
relocated row keep the moments of the Gaussian it replaced.  ``filter_3D`` and ``_deformation_table`` follow the copies.
``capture()`` keeps the reference's 14-tuple: the budget is the loop's to keep.
"""
from __future__ import annotations

import ctypes as C
import math
from argparse import Namespace

import torch
import torch.nn as nn

from . import _lib
from .optim import FusedAdam, add_densification_stats, get_expon_lr_func

PARAM_GROUPS = ("xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation")      # names of gaussian_model.py:176-186
_ATTR = {"xyz": "_xyz", "f_dc": "_features_dc", "f_rest": "_features_rest", "opacity": "_opacity",
         "scaling": "_scaling", "rotation": "_rotation"}


def default_optimization_params(**over) -> Namespace:
    """The fields of OptimizationParams the model reads (arguments/__init__.py:100-141)."""
    d = dict(position_lr_init=0.00016, position_lr_final=0.0000016, position_lr_delay_mult=0.01,
             position_lr_max_steps=30_000, deformation_lr_init=0.000016, deformation_lr_final=0.0000016,
             deformation_lr_delay_mult=0.01, grid_lr_init=0.00016, grid_lr_final=0.000016, feature_lr=0.0025,
             opacity_lr=0.05, scaling_lr=0.005, rotation_lr=0.001, percent_dense=0.01)
    d.update(over)
    return Namespace(**d)


def inverse_sigmoid(x):
    return torch.log(x / (1 - x))                # utils/general_utils.py:115-116


def build_rotation(r):
    """Unit-quaternion (w,x,y,z) rows -> rotation matrices (utils/general_utils.py:245-266)."""
    q = r / torch.sqrt(r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1] + r[:, 2] * r[:, 2] + r[:, 3] * r[:, 3])[:, None]
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.zeros((q.size(0), 3, 3), device=r.device)
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 0, 1] = 2 * (x * y - w * z)
    R[:, 0, 2] = 2 * (x * z + w * y)
    R[:, 1, 0] = 2 * (x * y + w * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 1, 2] = 2 * (y * z - w * x)
    R[:, 2, 0] = 2 * (x * z - w * y)
    R[:, 2, 1] = 2 * (y * z + w * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def split_plan(selected: torch.Tensor):
    """Row plan of densify_and_split + prune_points (gaussian_model.py:496-522): kept rows in order, then the
    selected rows twice (``repeat(N, 1)`` with N = 2).  -> (src_index int64 [n_kept + 2 n_sel], n_kept, sel)."""
    sel = torch.nonzero(selected, as_tuple=False).squeeze(1)
    keep = torch.nonzero(~selected, as_tuple=False).squeeze(1)
    return torch.cat((keep, sel, sel)), int(keep.numel()), sel


class GaussianModel:
    def __init__(self, sh_degree: int, args=None, deformation=None):
        self.active_sh_degree = 0
        self.max_sh_degree = sh_degree
        if deformation is None and args is not None:
            from .deformation import deform_network
            deformation = deform_network(args)
        self._deformation = deformation
        e = torch.empty(0)
        self._xyz = self._features_dc = self._features_rest = self._scaling = self._rotation = self._opacity = e
        self.max_radii2D = self.xyz_gradient_accum = self.denom = self._deformation_accum = e
        self.xyz_gradient_accum_abs = e
        self._deformation_table = e
        self.filter_3D = e              # [P,1] once compute_3D_filter() ran; empty until then
        self.optimizer = None
        self.percent_dense = 0
        self.spatial_lr_scale = 0
        self.scaling_activation = torch.exp
        self.scaling_inverse_activation = torch.log
        self.opacity_activation = torch.sigmoid
        self.inverse_opacity_activation = inverse_sigmoid
        self.rotation_activation = torch.nn.functional.normalize

    # ---- construction ---------------------------------------------------------------------------
    def create_from_tensors(self, xyz, features_dc, features_rest, scaling, rotation, opacity, spatial_lr_scale=1.0):
        """The tail of create_from_pcd (gaussian_model.py:141-169) for already-initialised raw parameters
        (log-scales, raw quaternions, logit opacities)."""
        dev = xyz.device
        if dev.type != "cuda":
            raise RuntimeError("GaussianModel: CUDA tensors only (there is no CPU path)")
        self.spatial_lr_scale = spatial_lr_scale
        mk = lambda t: nn.Parameter(t.detach().clone().float().contiguous().requires_grad_(True))
        self._xyz, self._features_dc, self._features_rest = mk(xyz), mk(features_dc), mk(features_rest)
        self._scaling, self._rotation, self._opacity = mk(scaling), mk(rotation), mk(opacity)
        if self._deformation is not None:
            self._deformation = self._deformation.to(dev)
        P = xyz.shape[0]
        self.max_radii2D = torch.zeros(P, device=dev)
        self._deformation_table = torch.ones(P, dtype=torch.bool, device=dev)
        self.filter_3D = torch.empty(0, device=dev)
        return self

    def create_from_pcd(self, pcd, spatial_lr_scale: float):
        """gaussian_model.py:141-169: positions and colours from a point cloud (anything with ``.points`` and
        ``.colors`` [P,3] arrays, colours in [0,1]); isotropic scales from the mean squared distance to the three
        nearest neighbours (our distCUDA2), identity rotations, opacity 0.1."""
        import numpy as np
        from .simple_knn import distCUDA2
        dev = torch.device("cuda")
        xyz = torch.tensor(np.asarray(pcd.points)).float().to(dev)
        colour = (torch.tensor(np.asarray(pcd.colors)).float().to(dev) - 0.5) / 0.28209479177387814   # RGB2SH, sh_utils.py:114
        P, K = xyz.shape[0], (self.max_sh_degree + 1) ** 2
        features = torch.zeros((P, 3, K), device=dev)
        features[:, :3, 0] = colour
        dist2 = torch.clamp_min(distCUDA2(xyz), 0.0000001)
        scales = torch.log(torch.sqrt(dist2))[..., None].repeat(1, 3)
        rots = torch.zeros((P, 4), device=dev)
        rots[:, 0] = 1
        opacities = inverse_sigmoid(0.1 * torch.ones((P, 1), dtype=torch.float, device=dev))
        return self.create_from_tensors(xyz, features[:, :, 0:1].transpose(1, 2), features[:, :, 1:].transpose(1, 2),
                                        scales, rots, opacities, spatial_lr_scale)

    # ---- .ply / deformation checkpoints (gaussian_model.py:241-275,355-395) ------------------------
    def save_ply(self, path):
        from .io_ply import write_gaussian_ply
        write_gaussian_ply(path, self._xyz, self._features_dc, self._features_rest, self._opacity, self._scaling,
                           self._rotation)

    def load_ply(self, path, device="cuda"):
        from .io_ply import read_gaussian_ply
        d = read_gaussian_ply(path, self.max_sh_degree)
        dev = torch.device(device)
        self.create_from_tensors(d["xyz"].to(dev), d["features_dc"].to(dev), d["features_rest"].to(dev),
                                 d["scaling"].to(dev), d["rotation"].to(dev), d["opacity"].to(dev),
                                 self.spatial_lr_scale or 1.0)
        self.active_sh_degree = self.max_sh_degree
        return self

    def save_deformation(self, path):
        import os
        os.makedirs(path, exist_ok=True)
        torch.save(self._deformation.state_dict(), os.path.join(path, "deformation.pth"))
        torch.save(self._deformation_table, os.path.join(path, "deformation_table.pth"))
        torch.save(self._deformation_accum, os.path.join(path, "deformation_accum.pth"))

    def load_model(self, path):
        import os
        dev = self._xyz.device if self._xyz.numel() else torch.device("cuda")
        self._deformation.load_state_dict(torch.load(os.path.join(path, "deformation.pth"), map_location=dev))
        self._deformation = self._deformation.to(dev)
        P = self._xyz.shape[0]
        self._deformation_table = torch.ones(P, dtype=torch.bool, device=dev)
        self._deformation_accum = torch.zeros((P, 3), device=dev)
        for name, attr in (("deformation_table.pth", "_deformation_table"), ("deformation_accum.pth", "_deformation_accum")):
            f = os.path.join(path, name)
            if os.path.exists(f):
                setattr(self, attr, torch.load(f, map_location=dev))
        self.max_radii2D = torch.zeros(P, device=dev)

    # ---- the accessors render() and the loop read (gaussian_model.py:113-140) --------------------
    @property
    def get_scaling(self):
        return self.scaling_activation(self._scaling)

    @property
    def get_rotation(self):
        return self.rotation_activation(self._rotation)

    @property
    def get_xyz(self):
        return self._xyz

    @property
    def get_features(self):
        return torch.cat((self._features_dc, self._features_rest), dim=1)

    @property
    def get_opacity(self):
        return self.opacity_activation(self._opacity)

    # ---- Mip-Splatting's 3-D smoothing filter (filter3d.py) -------------------------------------------------------
    def compute_3D_filter(self, cameras):
        """filter_3D <- the filter of the current (canonical) positions from the training cameras."""
        from .filter3d import compute_filter_3d
        self.filter_3D = compute_filter_3d(self.get_xyz, cameras)

    def _require_filter_3D(self):
        if self.filter_3D.dim() != 2 or self.filter_3D.shape[0] != self._xyz.shape[0]:
            raise RuntimeError(f"filter_3D has {tuple(self.filter_3D.shape)} rows for {self._xyz.shape[0]} Gaussians: "
                               "call compute_3D_filter(cameras) first")

    # Each of the two properties runs the apply kernel and keeps half of its result, as Mip-Splatting's pair does; to
    # read both in one launch, call filter3d.apply_filter_3d(self.get_scaling, self.get_opacity, self.filter_3D).
    @property
    def get_scaling_with_3D_filter(self):
        from .filter3d import apply_filter_3d
        self._require_filter_3D()
        return apply_filter_3d(self.get_scaling, self.get_opacity, self.filter_3D)[0]

    @property
    def get_opacity_with_3D_filter(self):
        from .filter3d import apply_filter_3d
        self._require_filter_3D()
        return apply_filter_3d(self.get_scaling, self.get_opacity, self.filter_3D)[1]

    def get_covariance(self, scaling_modifier=1):
        from .gaussian_renderer import GaussianModelLite
        return GaussianModelLite.get_covariance(self, scaling_modifier)

    def oneupSHdegree(self):
        if self.active_sh_degree < self.max_sh_degree:
            self.active_sh_degree += 1

    def compute_regulation(self, time_smoothness_weight, l1_time_planes_weight, plane_tv_weight):
        from .regulation import compute_regulation
        return compute_regulation(self._deformation.deformation_net.grid.grids, time_smoothness_weight,
                                  l1_time_planes_weight, plane_tv_weight)

    # ---- optimizer (gaussian_model.py:170-215) ----------------------------------------------------
    def training_setup(self, training_args):
        dev = self._xyz.device
        P = self._xyz.shape[0]
        self.percent_dense = training_args.percent_dense
        self.xyz_gradient_accum = torch.zeros((P, 1), device=dev)
        self.xyz_gradient_accum_abs = torch.zeros((P, 1), device=dev)
        self.denom = torch.zeros((P, 1), device=dev)
        self._deformation_accum = torch.zeros((P, 3), device=dev)
        s = self.spatial_lr_scale
        groups = [{"params": [self._xyz], "lr": training_args.position_lr_init * s, "name": "xyz"}]
        if self._deformation is not None:
            groups += [{"params": list(self._deformation.get_mlp_parameters()),
                        "lr": training_args.deformation_lr_init * s, "name": "deformation"},
                       {"params": list(self._deformation.get_grid_parameters()),
                        "lr": training_args.grid_lr_init * s, "name": "grid"}]
        groups += [{"params": [self._features_dc], "lr": training_args.feature_lr, "name": "f_dc"},
                   {"params": [self._features_rest], "lr": training_args.feature_lr / 20.0, "name": "f_rest"},
                   {"params": [self._opacity], "lr": training_args.opacity_lr, "name": "opacity"},
                   {"params": [self._scaling], "lr": training_args.scaling_lr, "name": "scaling"},
                   {"params": [self._rotation], "lr": training_args.rotation_lr, "name": "rotation"}]
        self.optimizer = FusedAdam(groups, lr=0.0, eps=1e-15, selective_groups=PARAM_GROUPS)
        self.xyz_scheduler_args = get_expon_lr_func(training_args.position_lr_init * s, training_args.position_lr_final * s,
                                                    lr_delay_mult=training_args.position_lr_delay_mult,
                                                    max_steps=training_args.position_lr_max_steps)
        self.deformation_scheduler_args = get_expon_lr_func(training_args.deformation_lr_init * s,
                                                            training_args.deformation_lr_final * s,
                                                            lr_delay_mult=training_args.deformation_lr_delay_mult,
                                                            max_steps=training_args.position_lr_max_steps)
        self.grid_scheduler_args = get_expon_lr_func(training_args.grid_lr_init * s, training_args.grid_lr_final * s,
                                                     lr_delay_mult=training_args.deformation_lr_delay_mult,
                                                     max_steps=training_args.position_lr_max_steps)

    def update_learning_rate(self, iteration):
        """gaussian_model.py:203-218: the xyz, grid and deformation groups follow their exponential schedules;
        returns the xyz learning rate (train.py:321)."""
        lr_pos = None
        for group in self.optimizer.param_groups:
            if group["name"] == "xyz":
                lr_pos = group["lr"] = self.xyz_scheduler_args(iteration)
            if "grid" in group["name"]:
                group["lr"] = self.grid_scheduler_args(iteration)
            elif group["name"] == "deformation":
                group["lr"] = self.deformation_scheduler_args(iteration)
        return lr_pos

    # ---- checkpoints (gaussian_model.py:71-111; written by train.py:231,531, read by train.py:617) -------
    def capture(self):
        """The reference's 14-tuple, same order, so torch.save((gaussians.capture(), iteration), path) files are
        interchangeable with the reference's."""
        return (self.active_sh_degree, self._xyz, self._deformation.state_dict(), self._deformation_table,
                self._features_dc, self._features_rest, self._scaling, self._rotation, self._opacity, self.max_radii2D,
                self.xyz_gradient_accum, self.denom, self.optimizer.state_dict(), self.spatial_lr_scale)

    def restore(self, model_args, training_args):
        """gaussian_model.py:89-111.  Accepts a tuple captured by the reference class (its optimizer state dict is
        torch.optim.Adam's, which FusedAdam shares) or by this one."""
        (self.active_sh_degree, xyz, deform_state, table, f_dc, f_rest, scaling, rotation, opacity, max_radii2D,
         xyz_gradient_accum, denom, opt_dict, self.spatial_lr_scale) = model_args
        dev = xyz.device if xyz.is_cuda else torch.device("cuda")
        mk = lambda t: nn.Parameter(t.detach().to(dev).float().contiguous().requires_grad_(True))
        self._xyz, self._features_dc, self._features_rest = mk(xyz), mk(f_dc), mk(f_rest)
        self._scaling, self._rotation, self._opacity = mk(scaling), mk(rotation), mk(opacity)
        self._deformation_table = table.to(dev)
        self.filter_3D = torch.empty(0, device=dev)     # not in the tuple: recompute it from the cameras
        self.max_radii2D = max_radii2D.to(dev)
        self._deformation = self._deformation.to(dev)
        self._deformation.load_state_dict(deform_state)
        self.training_setup(training_args)     # xyz_gradient_accum_abs, not in the tuple, starts from zero
        self.xyz_gradient_accum = xyz_gradient_accum.to(dev)
        self.denom = denom.to(dev)
        self.optimizer.load_state_dict(opt_dict)

    # ---- per-iteration statistics (train.py:489-491, gaussian_model.py:693-695) --------------------
    def add_densification_stats(self, viewspace_point_tensor, update_filter):
        scratch = torch.zeros_like(self.max_radii2D)
        add_densification_stats(viewspace_point_tensor.contiguous(), update_filter.to(torch.int32), self.xyz_gradient_accum,
                                self.denom, scratch)

    def densification_step(self, viewspace_point_tensor_grad, radii, absgrad=None):
        """max_radii2D update + add_densification_stats with visibility_filter = radii > 0, one launch.  absgrad
        (float32 [P,2], viewspace_points.absgrad summed over the step's views) also goes into xyz_gradient_accum_abs."""
        if absgrad is None:
            add_densification_stats(viewspace_point_tensor_grad.contiguous(), radii, self.xyz_gradient_accum,
                                    self.denom, self.max_radii2D)
            return
        add_densification_stats(viewspace_point_tensor_grad.contiguous(), radii, self.xyz_gradient_accum, self.denom,
                                self.max_radii2D, absgrad.contiguous(), self.xyz_gradient_accum_abs)

    # ---- row surgery --------------------------------------------------------------------------------
    def _group(self, name):
        for g in self.optimizer.param_groups:
            if g["name"] == name:
                return g
        raise KeyError(name)

    def _rebuild(self, src_index: torch.Tensor, n_kept: int, keep_accumulators: bool):
        """Every per-Gaussian tensor <- rows ``src_index`` of itself; rows >= n_kept are new (Adam moments zero)."""
        lib = _lib.load()
        dev = self._xyz.device
        n_out = int(src_index.numel())
        src_index = src_index.to(torch.int64).contiguous()
        descs, new_params, new_states, hold = [], {}, {}, []

        def add(src, zero_new):
            src = src.contiguous()
            rf = math.prod(src.shape[1:])
            dst = torch.empty((n_out, *src.shape[1:]), device=dev, dtype=torch.float32)
            if rf == 0:      # zero-width rows (_features_rest at max_sh_degree == 0): nothing to gather
                return dst
            descs.append(_lib.RowTensor(src.data_ptr(), dst.data_ptr(), int(rf), 1 if zero_new else 0))
            hold.append(src)
            return dst
        for name in PARAM_GROUPS:
            p = getattr(self, _ATTR[name])
            new_params[name] = add(p.data, False)
            st = self.optimizer.state.get(p, None) if self.optimizer is not None else None
            if st:
                new_states[name] = (st["step"], add(st["exp_avg"], True), add(st["exp_avg_sq"], True))
        acc = None
        P_old = self._xyz.shape[0]
        # the 3-D filter, while it matches the rows: new rows take their source row's value
        filt = (add(self.filter_3D.to(dev, torch.float32), False)
                if self.filter_3D.dim() == 2 and self.filter_3D.shape[0] == P_old else None)
        have_acc = all(t.numel() > 0 and t.shape[0] == P_old for t in
                       (self.xyz_gradient_accum, self.denom, self._deformation_accum, self.max_radii2D))
        if keep_accumulators and not have_acc:      # training_setup() not called yet: nothing to carry over
            keep_accumulators = False
        if keep_accumulators:
            acc = [add(self.xyz_gradient_accum, False), add(self.denom, False), add(self._deformation_accum, False),
                   add(self.max_radii2D.unsqueeze(1), False)]
            # the absolute-gradient accumulator, when it matches the rows (zeros otherwise)
            acc_abs = self.xyz_gradient_accum_abs
            acc.append(add(acc_abs, False) if acc_abs.dim() == 2 and acc_abs.shape[0] == P_old else None)
        if n_out > 0:
            arr = (_lib.RowTensor * len(descs))(*descs)
            _lib.check(lib.s3g_gather_rows(len(descs), arr, n_out, int(n_kept), src_index.data_ptr(),
                                           C.c_void_p(torch.cuda.current_stream().cuda_stream)), "s3g_gather_rows")
        for name in PARAM_GROUPS:
            old = getattr(self, _ATTR[name])
            newp = nn.Parameter(new_params[name].requires_grad_(True))
            if self.optimizer is not None:
                group = self._group(name)
                self.optimizer.state.pop(old, None)
                group["params"][0] = newp
                if name in new_states:
                    step, m, v = new_states[name]
                    self.optimizer.state[newp] = {"step": step, "exp_avg": m, "exp_avg_sq": v}
            setattr(self, _ATTR[name], newp)
        self._deformation_table = self._deformation_table[src_index]
        self.filter_3D = filt if filt is not None else torch.empty(0, device=dev)
        if keep_accumulators:
            self.xyz_gradient_accum, self.denom, self._deformation_accum = acc[0], acc[1], acc[2]
            self.max_radii2D = acc[3].squeeze(1)
            self.xyz_gradient_accum_abs = acc[4] if acc[4] is not None else torch.zeros((n_out, 1), device=dev)
        else:       # densification_postfix resets them (gaussian_model.py:490-494)
            self.xyz_gradient_accum = torch.zeros((n_out, 1), device=dev)
            self.xyz_gradient_accum_abs = torch.zeros((n_out, 1), device=dev)
            self._deformation_accum = torch.zeros((n_out, 3), device=dev)
            self.denom = torch.zeros((n_out, 1), device=dev)
            self.max_radii2D = torch.zeros(n_out, device=dev)

    def spatial_sort(self):
        """Reorder every per-Gaussian tensor (parameters, Adam moments, densification accumulators) along a Morton
        curve of the positions (10 bits per axis over the bounding box).  Not in the reference - its Gaussians stay
        in LiDAR / append order - and a no-op for the maths: every kernel is order-independent up to the order of
        fp32 additions.  What it buys: consecutive warps of the HexPlane sample / scatter kernels (one warp per
        Gaussian) then touch neighbouring texels, so L1 absorbs most of the 12 KB-per-Gaussian plane traffic that
        otherwise goes to L2.  Cheap (one radix sort + one row gather); call it after densify / prune.  Returns the
        permutation (new row i = old row order[i])."""
        lib = _lib.load()
        with torch.no_grad():
            xyz = self._xyz.data
            P = xyz.shape[0]
            if P < 2:
                return torch.arange(P, device=xyz.device)
            lo, hi = xyz.min(0).values, xyz.max(0).values
            q = ((xyz - lo) / (hi - lo).clamp_min(1e-12) * 1023.999).to(torch.int64).clamp_(0, 1023)

            def spread(v):      # 10 bits -> every third bit
                v = (v | (v << 16)) & 0x030000FF
                v = (v | (v << 8)) & 0x0300F00F
                v = (v | (v << 4)) & 0x030C30C3
                return (v | (v << 2)) & 0x09249249
            key = (spread(q[:, 0]) | (spread(q[:, 1]) << 1) | (spread(q[:, 2]) << 2)).to(torch.int32).contiguous()
            idx = torch.arange(P, device=xyz.device, dtype=torch.int32)
            ko, vo = torch.empty_like(key), torch.empty_like(idx)
            tmp = torch.empty(lib.s3g_sort_temp_bytes(P), dtype=torch.uint8, device=xyz.device)
            _lib.check(lib.s3g_sort_pairs_u32(P, key.data_ptr(), idx.data_ptr(), ko.data_ptr(), vo.data_ptr(), 0, 30,
                                              tmp.data_ptr(), C.c_void_p(torch.cuda.current_stream().cuda_stream)),
                       "s3g_sort_pairs_u32")
            order = vo.to(torch.int64)
            self._rebuild(order, P, keep_accumulators=True)
        return order

    def prune_points(self, mask):
        """gaussian_model.py:441-455."""
        keep = torch.nonzero(~mask, as_tuple=False).squeeze(1)
        self._rebuild(keep, int(keep.numel()), keep_accumulators=True)

    def densify_and_clone(self, grads, grad_threshold, scene_extent):
        """gaussian_model.py:524-563: small Gaussians with a large view-space gradient are duplicated in place."""
        selected = torch.logical_and(torch.norm(grads, dim=-1) >= grad_threshold,
                                     torch.max(self.get_scaling, dim=1).values <= self.percent_dense * scene_extent)
        P = self._xyz.shape[0]
        sel = torch.nonzero(selected, as_tuple=False).squeeze(1)
        self._rebuild(torch.cat((torch.arange(P, device=sel.device), sel)), P, keep_accumulators=False)

    def densify_and_split(self, grads, grad_threshold, scene_extent, N=2):
        """gaussian_model.py:496-522: large Gaussians with a large gradient are replaced by N = 2 samples of
        themselves, 1.6x smaller."""
        if N != 2:
            raise NotImplementedError("densify_and_split: the reference calls it with N = 2 only")
        P = self._xyz.shape[0]
        dev = self._xyz.device
        padded_grad = torch.zeros(P, device=dev)
        padded_grad[:grads.shape[0]] = grads.squeeze()
        selected = torch.logical_and(padded_grad >= grad_threshold,
                                     torch.max(self.get_scaling, dim=1).values > self.percent_dense * scene_extent)
        if not selected.any():
            return
        with torch.no_grad():
            stds = self.get_scaling[selected].repeat(N, 1)
            samples = torch.normal(mean=torch.zeros((stds.size(0), 3), device=dev), std=stds)
            rots = build_rotation(self._rotation[selected]).repeat(N, 1, 1)
            new_xyz = torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1) + self.get_xyz[selected].repeat(N, 1)
            new_scaling = self.scaling_inverse_activation(self.get_scaling[selected].repeat(N, 1) / (0.8 * N))
            src_index, n_kept, _ = split_plan(selected)
            self._rebuild(src_index, n_kept, keep_accumulators=False)
            self._xyz.data[n_kept:] = new_xyz
            self._scaling.data[n_kept:] = new_scaling

    def densify(self, max_grad, min_opacity, extent, max_screen_size, *unused, max_grad_abs=None, **unused_kw):
        """gaussian_model.py:674-679.  max_grad_abs: clone and split select on the absolute-gradient statistic,
        ||xyz_gradient_accum_abs / denom|| >= max_grad_abs, instead of the signed one (gsplat's absgrad rule)."""
        if max_grad_abs is None:
            grads = self.xyz_gradient_accum / self.denom
        else:
            grads, max_grad = self.xyz_gradient_accum_abs / self.denom, max_grad_abs
        grads[grads.isnan()] = 0.0
        with torch.no_grad():
            self.densify_and_clone(grads, max_grad, extent)
        self.densify_and_split(grads, max_grad, extent)

    def prune(self, max_grad, min_opacity, extent, max_screen_size):
        """gaussian_model.py:661-672 (without the empty_cache() call)."""
        with torch.no_grad():
            prune_mask = (self.get_opacity < min_opacity).squeeze()
            if max_screen_size:
                big_points_vs = self.max_radii2D > max_screen_size
                big_points_ws = self.get_scaling.max(dim=1).values > 0.1 * extent
                prune_mask = torch.logical_or(torch.logical_or(prune_mask, big_points_vs), big_points_ws)
            self.prune_points(prune_mask)

    # ---- 3DGS-MCMC densification (mcmc.py) ---------------------------------------------------------------------------
    def _mcmc_relocate_rows(self, src, dst, min_opacity):
        """After _rebuild copied row src[j] to row dst[j]: both get the relocated opacity and scales, the Adam moments
        of both and the accumulators of dst[j] become zero.  One launch."""
        from .mcmc import relocate
        counts = torch.bincount(src, minlength=self._xyz.shape[0])
        zero = []
        if self.optimizer is not None:
            for name in PARAM_GROUPS:
                st = self.optimizer.state.get(getattr(self, _ATTR[name]), None)
                if st:
                    zero += [(st["exp_avg"], True), (st["exp_avg_sq"], True)]
        zero += [(t, False) for t in (self.xyz_gradient_accum, self.xyz_gradient_accum_abs, self.denom,
                                      self._deformation_accum, self.max_radii2D)]
        relocate(self._opacity.data, self._scaling.data, src, dst, counts[src] + 1, min_opacity, zero)

    def relocate_gs(self, min_opacity=0.005, generator=None):
        """3DGS-MCMC's relocate_gs: every dead Gaussian (opacity <= min_opacity) becomes a copy of an alive one drawn
        with probability proportional to its opacity (with replacement); the drawn Gaussian and its copies share the
        relocated opacity and scales.  P is unchanged.  Unlike the published code, the copies' Adam moments are zeroed
        too, not only the drawn rows'."""
        with torch.no_grad():
            o = self.get_opacity.squeeze(1)
            dead = o <= min_opacity
            dead_idx = torch.nonzero(dead, as_tuple=False).squeeze(1)
            alive_idx = torch.nonzero(~dead, as_tuple=False).squeeze(1)
            if dead_idx.numel() == 0 or alive_idx.numel() == 0:
                return
            drawn = alive_idx[torch.multinomial(o[alive_idx], dead_idx.numel(), replacement=True, generator=generator)]
            idx = torch.arange(o.shape[0], device=o.device)
            idx[dead_idx] = drawn
            self._rebuild(idx, o.shape[0], keep_accumulators=True)
            self._mcmc_relocate_rows(drawn, dead_idx, min_opacity)

    def add_new_gs(self, cap_max, generator=None, min_opacity=0.005):
        """3DGS-MCMC's add_new_gs: grow by min(cap_max, int(1.05 P)) - P Gaussians (none once P >= cap_max), each a
        copy of a row drawn with probability proportional to its opacity; drawn rows and copies share the relocated
        opacity and scales (its opacity clamped below at min_opacity).  Returns the number added."""
        P = self._xyz.shape[0]
        n = max(0, min(int(cap_max), int(1.05 * P)) - P)
        if n == 0:
            return 0
        with torch.no_grad():
            o = self.get_opacity.squeeze(1)
            drawn = torch.multinomial(o, n, replacement=True, generator=generator)
            self._rebuild(torch.cat((torch.arange(P, device=o.device), drawn)), P, keep_accumulators=True)
            self._mcmc_relocate_rows(drawn, torch.arange(P, P + n, device=o.device), min_opacity)
        return n

    def inject_noise(self, xyz_lr, noise_lr=5e5, generator=None):
        """3DGS-MCMC's position noise, after optimizer.step(): xyz += xyz_lr * noise_lr * gate(o) * Sigma eps with
        Sigma = R diag(s^2) R^T of the canonical parameters (not the 3-D-filtered scales), eps ~ N(0, I) [P,3] from
        torch.randn with `generator`, gate = 1 / (1 + exp(-100 ((1 - o) - 0.995))).  One launch besides the randn."""
        from .mcmc import inject_noise
        with torch.no_grad():
            eps = torch.randn(self._xyz.shape, device=self._xyz.device, generator=generator)
            inject_noise(self._xyz.data, self._scaling.data, self._rotation.data, self._opacity.data,
                         float(xyz_lr) * float(noise_lr), eps)

    def replace_tensor_to_optimizer(self, tensor, name):
        """gaussian_model.py:397-409: new parameter values, Adam moments reset to zero, step kept."""
        group = self._group(name)
        old = group["params"][0]
        st = self.optimizer.state.pop(old, None)
        newp = nn.Parameter(tensor.detach().clone().contiguous().requires_grad_(True))
        group["params"][0] = newp
        if st is not None:
            st["exp_avg"] = torch.zeros_like(newp)
            st["exp_avg_sq"] = torch.zeros_like(newp)
            self.optimizer.state[newp] = st
        return {name: newp}

    def reset_opacity(self):
        """gaussian_model.py:350-353."""
        with torch.no_grad():
            new = inverse_sigmoid(torch.min(self.get_opacity, torch.ones_like(self.get_opacity) * 0.01))
        self._opacity = self.replace_tensor_to_optimizer(new, "opacity")["opacity"]
