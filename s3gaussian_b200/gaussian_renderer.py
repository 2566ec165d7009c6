"""Drop-in for the reference's ``gaussian_renderer.render``
(gaussian_renderer/__init__.py:23-210): same signature, same result dict, same
control flow; the work runs in two fused CUDA stages instead of ~150 PyTorch
launches + the reference extension:

  fine stage : deform_network.render_front  (HexPlane + decoder + activations + SH->RGB, one kernel)
  both stages: GaussianRasterizer            (preprocess, sort, composite; C ABI of libs3g_b200.so)

``pc`` is anything with the attributes the reference reads from ``GaussianModel``
(get_xyz, _scaling, _rotation, _opacity, get_features, active_sh_degree, max_sh_degree,
_deformation, get_covariance); ``GaussianModelLite`` below is the minimal such object
used by the tests and bench.py.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn

from .diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
from .filter3d import apply_filter_3d


class GaussianModelLite(nn.Module):
    """The slice of scene/gaussian_model.py the render path touches (:32-60,113-140)."""

    def __init__(self, cloud, deformation=None, sh_degree=3):
        super().__init__()
        self.max_sh_degree = sh_degree
        self.active_sh_degree = sh_degree
        self._xyz = nn.Parameter(cloud.xyz.clone())
        self._features_dc = nn.Parameter(cloud.features_dc.clone())
        self._features_rest = nn.Parameter(cloud.features_rest.clone())
        self._scaling = nn.Parameter(cloud.scaling.clone())
        self._rotation = nn.Parameter(cloud.rotation.clone())
        self._opacity = nn.Parameter(cloud.opacity.clone())
        self._deformation = deformation
        self.scaling_activation = torch.exp
        self.opacity_activation = torch.sigmoid
        self.rotation_activation = torch.nn.functional.normalize

    @property
    def get_xyz(self):
        return self._xyz

    @property
    def get_features(self):
        return torch.cat((self._features_dc, self._features_rest), dim=1)

    @property
    def _deformation_table(self):
        return torch.ones(self._xyz.shape[0], dtype=torch.bool, device=self._xyz.device)

    def compute_regulation(self, time_smoothness_weight, l1_time_planes_weight, plane_tv_weight):
        """scene/gaussian_model.py:748-749, one fused launch per direction (regulation.py)."""
        from .regulation import compute_regulation
        return compute_regulation(self._deformation.deformation_net.grid.grids, time_smoothness_weight,
                                  l1_time_planes_weight, plane_tv_weight)

    def get_covariance(self, scaling_modifier=1):
        s = scaling_modifier * torch.exp(self._scaling)
        q = torch.nn.functional.normalize(self._rotation)
        r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                         2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                         2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
        Lm = R * s[:, None, :]
        S = Lm @ Lm.transpose(1, 2)
        return torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1)


class PipelineParams:       # arguments/__init__.py:93-98 defaults
    convert_SHs_python = True
    compute_cov3D_python = False
    debug = False
    shared_binning = True   # ours: colour + feature image in one rasterizer pass (False = two passes, as upstream)
    render_opacity = False  # ours: render() also returns the alpha and median-depth images (and alpha_d / alpha_s)
    antialiasing = False    # ours: the rasterizer's antialiasing filter (GaussianRasterizer(antialiasing=True))
    filter_3d = False       # ours: Mip-Splatting's 3-D smoothing filter on the scales and opacities (pc.filter_3D)
    absgrad = False         # ours: the backward also sets viewspace_points.absgrad (GaussianRasterizer(absgrad=True))
    lens = False            # ours: project through the camera's intrinsic and distortion (GaussianRasterizer(lens=...))


def pipe_shared_binning(pipe) -> bool:
    return bool(getattr(pipe, "shared_binning", True))


def pipe_render_opacity(pipe) -> bool:
    return bool(getattr(pipe, "render_opacity", False))


def pipe_rasterizer_kwargs(pipe) -> dict:
    """The keyword arguments GaussianRasterizer takes from the pipeline parameters: none unless pipe.antialiasing or
    pipe.absgrad is set."""
    kw = {"antialiasing": True} if getattr(pipe, "antialiasing", False) else {}
    if getattr(pipe, "absgrad", False):
        kw["absgrad"] = True
    return kw


def camera_lens(viewpoint_camera):
    """The Lens of a camera: fx, fy, cx, cy from its 3x3 `intrinsic` (the reference's Camera.intrinsic, principal point
    with pixel centres at j + 0.5) and k1, k2, p1, p2, k3 from its `distortion` (zeros when it has none)."""
    from .diff_gaussian_rasterization import Lens
    K = getattr(viewpoint_camera, "intrinsic", None)
    if K is None:
        raise RuntimeError("pipe.lens: the camera has no intrinsic (3x3 K) to build the lens from")
    K = torch.as_tensor(K, dtype=torch.float64).reshape(3, 3).cpu()
    dist = getattr(viewpoint_camera, "distortion", None)
    dist = [0.0] * 5 if dist is None else [float(v) for v in torch.as_tensor(dist, dtype=torch.float64).reshape(-1)]
    if len(dist) != 5:
        raise RuntimeError(f"pipe.lens: camera.distortion must hold k1, k2, p1, p2, k3 ({len(dist)} values)")
    return Lens(float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), *dist)


def pipe_lens_kwargs(pipe, viewpoint_camera) -> dict:
    """{"lens": camera_lens(viewpoint_camera)} when pipe.lens is set, else nothing."""
    return {"lens": camera_lens(viewpoint_camera)} if getattr(pipe, "lens", False) else {}


def pipe_filter_3d(pipe, pc) -> bool:
    """Whether pipe.filter_3d is set; when it is, checks before any launch that `pc` has a filter_3D for its P
    Gaussians and that precomputed covariances are not asked for."""
    if not getattr(pipe, "filter_3d", False):
        return False
    if pipe.compute_cov3D_python:
        raise NotImplementedError("pipe.filter_3d with compute_cov3D_python: the 3-D filter applies to scales, not "
                                  "precomputed covariances")
    P = pc.get_xyz.shape[0]
    f = getattr(pc, "filter_3D", None)
    if f is None or f.dim() != 2 or f.shape[0] != P:
        raise RuntimeError(f"pipe.filter_3d: the model has no filter_3D for its {P} Gaussians "
                           f"({None if f is None else tuple(f.shape)}); call compute_3D_filter(cameras) first")
    return True


def render(viewpoint_camera, pc, pipe, bg_color: torch.Tensor, scaling_modifier=1.0, override_color=None,
           stage="fine", return_decomposition=False, return_dx=False, render_feat=False):
    """Render the scene.  Background tensor (bg_color) must be on GPU!

    With pipe.lens, every rasterizer call projects through the camera's `intrinsic` and `distortion` (camera_lens).
    With pipe.absgrad, the backward of the result also sets result["viewspace_points"].absgrad (float32 [P,2]), the
    absolute screen-space gradient of the call(s) that drew "render" and "feat" (GaussianRasterizer(absgrad=True)).
    The differentiable decomposition passes index means2D and leave their statistic on those temporaries."""
    filter_3d = pipe_filter_3d(pipe, pc)
    xyz = pc.get_xyz
    dev = xyz.device
    # gradient carrier for the 2-D means (gaussian_renderer/__init__.py:31-35)
    screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=dev) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass

    raster_settings = raster_settings_for(viewpoint_camera, pc, pipe, bg_color, scaling_modifier)
    campos = raster_settings.campos
    rasterizer = GaussianRasterizer(raster_settings=raster_settings, **pipe_rasterizer_kwargs(pipe),
                                    **pipe_lens_kwargs(pipe, viewpoint_camera))

    means2D = screenspace_points
    shs = pc.get_features
    cov3D_precomp = None
    dx = feat = dshs = None

    if "coarse" in stage:
        means3D_final = xyz
        if pipe.compute_cov3D_python:
            cov3D_precomp = pc.get_covariance(scaling_modifier)
            scales_final = rotations_final = None
        else:
            scales_final = pc.scaling_activation(pc._scaling)
            rotations_final = pc.rotation_activation(pc._rotation)
        opacity = pc.opacity_activation(pc._opacity)
        if filter_3d:
            scales_final, opacity = apply_filter_3d(scales_final, opacity, pc.filter_3D)
        shs_final, colors_precomp = shs, None
        # convert_SHs_python evaluates the same polynomial with dir = xyz - campos; in the coarse
        # stage the rasterized mean IS xyz, so the in-kernel SH path gives the same colours
    elif "fine" in stage:
        (means3D_final, scales_final, rotations_final, opacity, shs_final, colors_precomp, dx, dshs,
         feat) = fine_front(viewpoint_camera, pc, pipe, campos, shs)
    else:
        raise NotImplementedError

    if override_color is not None:
        colors_precomp, shs_final = override_color, None

    want_feat = render_feat and "fine" in stage and feat is not None
    rendered_image2 = None
    # pipe.render_opacity: the same walks through their opacity forms, which add "alpha" and "median_depth" (and with a
    # decomposition "alpha_d" / "alpha_s") to the result
    opa = pipe_render_opacity(pipe)
    opacity_out = {}
    # Without autograd (evaluation, utils/video_utils.py:169) the decomposition's full, dynamic and static images come
    # from one rasterizer pass; with grad enabled the three differentiable passes below stay the only path.
    split = return_decomposition and dx is not None and not torch.is_grad_enabled()
    if split:
        dynamic_mask = dynamic_mask_of(dx)
        out = rasterizer.forward_eval(
            means3D=means3D_final, means2D=means2D, opacities=opacity, group=dynamic_mask, shs=shs_final,
            colors_precomp=colors_precomp, scales=scales_final, rotations=rotations_final, cov3D_precomp=cov3D_precomp,
            **({"with_opacity": True} if opa else {}))
        rendered_image, radii, depth, decomposition = out[:4]
        rendered_image_d, depth_d, rendered_image_s, depth_s = decomposition
        if opa:
            opacity_out = dict(zip(("alpha", "median_depth", "alpha_d", "alpha_s"), out[5]))
    elif want_feat and hasattr(rasterizer, "forward_aux") and pipe_shared_binning(pipe):
        # the feature image shares preprocess, sort and the per-pixel alpha evaluation with the colour image
        # (the reference rasterizes the same geometry a second time, gaussian_renderer/__init__.py:173-186)
        if opa:
            rendered_image, radii, depth, alpha, median_depth, rendered_image2 = rasterizer.forward_opacity(
                means3D=means3D_final, means2D=means2D, opacities=opacity, colors_aux=feat, shs=shs_final,
                colors_precomp=colors_precomp, scales=scales_final, rotations=rotations_final,
                cov3D_precomp=cov3D_precomp)
            opacity_out = {"alpha": alpha, "median_depth": median_depth}
        else:
            rendered_image, radii, depth, rendered_image2 = rasterizer.forward_aux(
                means3D=means3D_final, means2D=means2D, opacities=opacity, colors_aux=feat, shs=shs_final,
                colors_precomp=colors_precomp, scales=scales_final, rotations=rotations_final,
                cov3D_precomp=cov3D_precomp)
    elif opa:
        rendered_image, radii, depth, alpha, median_depth = rasterizer.forward_opacity(
            means3D=means3D_final, means2D=means2D, shs=shs_final, colors_precomp=colors_precomp, opacities=opacity,
            scales=scales_final, rotations=rotations_final, cov3D_precomp=cov3D_precomp)
        opacity_out = {"alpha": alpha, "median_depth": median_depth}
    else:
        rendered_image, radii, depth = rasterizer(
            means3D=means3D_final, means2D=means2D, shs=shs_final, colors_precomp=colors_precomp, opacities=opacity,
            scales=scales_final, rotations=rotations_final, cov3D_precomp=cov3D_precomp)

    result_dict = {"render": rendered_image, "viewspace_points": screenspace_points,
                   "visibility_filter": radii > 0, "radii": radii, "depth": depth}
    if opa:
        result_dict.update({k: opacity_out[k] for k in ("alpha", "median_depth")})

    if want_feat:
        if rendered_image2 is None:
            rendered_image2, _, _ = rasterizer(
                means3D=means3D_final, means2D=means2D, shs=None, colors_precomp=feat, opacities=opacity,
                scales=scales_final, rotations=rotations_final, cov3D_precomp=cov3D_precomp)
        result_dict.update({"feat": rendered_image2})

    if split:
        visible = radii > 0
        result_dict.update({"render_d": rendered_image_d, "depth_d": depth_d, "visibility_filter_d": visible[dynamic_mask],
                            "render_s": rendered_image_s, "depth_s": depth_s, "visibility_filter_s": visible[~dynamic_mask]})
        if opa:
            result_dict.update({"alpha_d": opacity_out["alpha_d"], "alpha_s": opacity_out["alpha_s"]})
    elif return_decomposition and dx is not None:
        dynamic_mask = dynamic_mask_of(dx)
        cols = colors_precomp if colors_precomp is not None else None

        def sub(mask):
            return (rasterizer.forward_opacity if opa else rasterizer)(
                means3D=means3D_final[mask], means2D=means2D[mask],
                shs=shs_final[mask] if shs_final is not None else None,
                colors_precomp=cols[mask] if cols is not None else None, opacities=opacity[mask],
                scales=scales_final[mask], rotations=rotations_final[mask],
                cov3D_precomp=cov3D_precomp[mask] if cov3D_precomp is not None else None)
        out_d, out_s = sub(dynamic_mask), sub(~dynamic_mask)
        (rendered_image_d, radii_d, depth_d), (rendered_image_s, radii_s, depth_s) = out_d[:3], out_s[:3]
        result_dict.update({"render_d": rendered_image_d, "depth_d": depth_d, "visibility_filter_d": radii_d > 0,
                            "render_s": rendered_image_s, "depth_s": depth_s, "visibility_filter_s": radii_s > 0})
        if opa:
            result_dict.update({"alpha_d": out_d[3], "alpha_s": out_s[3]})

    if return_dx and "fine" in stage:
        result_dict.update({"dx": dx})
        result_dict.update({"dshs": dshs})
    return result_dict


def raster_settings_for(viewpoint_camera, pc, pipe, bg_color, scaling_modifier=1.0):
    """The rasterizer settings render() uses for a camera (gaussian_renderer/__init__.py:37-53)."""
    dev = pc.get_xyz.device
    return GaussianRasterizationSettings(
        image_height=int(viewpoint_camera.image_height), image_width=int(viewpoint_camera.image_width),
        tanfovx=math.tan(viewpoint_camera.FoVx * 0.5), tanfovy=math.tan(viewpoint_camera.FoVy * 0.5), bg=bg_color,
        scale_modifier=scaling_modifier, viewmatrix=viewpoint_camera.world_view_transform.to(dev),
        projmatrix=viewpoint_camera.full_proj_transform.to(dev), sh_degree=pc.active_sh_degree,
        campos=viewpoint_camera.camera_center.to(dev), prefiltered=False, debug=pipe.debug)


def fine_front(viewpoint_camera, pc, pipe, campos, shs):
    """The fine stage's front end of render() (gaussian_renderer/__init__.py:85-117): deformation at the camera's time,
    activations and the colours or SHs the rasterizer takes; `shs` is pc.get_features.  One deformation forward.
    -> (means3D, scales, rotations, opacity, shs, colors_precomp, dx, dshs, feat); exactly one of shs /
    colors_precomp is None.  With pipe.filter_3d the scales and opacities are those after pc.filter_3D."""
    filter_3d = pipe_filter_3d(pipe, pc)
    if pipe.compute_cov3D_python:
        raise NotImplementedError("compute_cov3D_python with the deformation stage (reference default: False)")
    xyz = pc.get_xyz
    deform = pc._deformation
    time = float(viewpoint_camera.time)
    if hasattr(deform, "render_front"):
        (means3D_final, scales_final, rotations_final, opacity, colors_front, dx, dshs, feat) = \
            deform.render_front(xyz, pc._scaling, pc._rotation, pc._opacity, shs, time, campos,
                                pc.active_sh_degree)
        shs_final = None
        colors_precomp = colors_front
        if not pipe.convert_SHs_python:
            # SHs go to the rasterizer, which uses the DEFORMED mean for the view direction
            colors_precomp, shs_final = None, (shs if dshs is None else shs + dshs)
    else:   # any module with the reference signature (scene/deformation.py:216)
        t = torch.full((xyz.shape[0], 1), time, device=xyz.device)
        means3D_final, sc, ro, op, shs_final, dx, feat, dshs = deform(xyz, pc._scaling, pc._rotation,
                                                                      pc._opacity, shs, t)
        scales_final = pc.scaling_activation(sc)
        rotations_final = pc.rotation_activation(ro)
        opacity = pc.opacity_activation(op)
        colors_precomp = None
        if pipe.convert_SHs_python:
            colors_precomp = _sh_python(pc, shs_final, xyz, campos)
            shs_final = None
    if filter_3d:
        scales_final, opacity = apply_filter_3d(scales_final, opacity, pc.filter_3D)
    return means3D_final, scales_final, rotations_final, opacity, shs_final, colors_precomp, dx, dshs, feat


def dynamic_mask_of(dx):
    """The decomposition's dynamic Gaussians (gaussian_renderer/__init__.py:177-178): max |dx| above its mean."""
    max_values = torch.max(torch.abs(dx), dim=1)[0]
    return max_values > torch.mean(max_values)


def _sh_python(pc, shs_final, xyz, campos):
    """convert_SHs_python (gaussian_renderer/__init__.py:107-115) in torch, for non-fused deformation modules."""
    K = (pc.active_sh_degree + 1) ** 2
    d = xyz - campos
    d = d / d.norm(dim=1, keepdim=True)
    x, y, z = d[:, 0:1], d[:, 1:2], d[:, 2:3]
    b = [torch.full_like(x, 0.28209479177387814)]
    if K > 1:
        b += [-0.4886025119029199 * y, 0.4886025119029199 * z, -0.4886025119029199 * x]
    if K > 4:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        b += [1.0925484305920792 * xy, -1.0925484305920792 * yz, 0.31539156525252005 * (2 * zz - xx - yy),
              -1.0925484305920792 * xz, 0.5462742152960396 * (xx - yy)]
    if K > 9:
        b += [-0.5900435899266435 * y * (3 * xx - yy), 2.890611442640554 * xy * z,
              -0.4570457994644658 * y * (4 * zz - xx - yy), 0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy),
              -0.4570457994644658 * x * (4 * zz - xx - yy), 1.445305721320277 * z * (xx - yy),
              -0.5900435899266435 * x * (xx - 3 * yy)]
    B = torch.cat(b, dim=1)
    rgb = (B.unsqueeze(2) * shs_final[:, :K, :]).sum(1)
    return torch.clamp_min(rgb + 0.5, 0.0)
