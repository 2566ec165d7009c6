"""Drop-in for the reference's ``diff_gaussian_rasterization`` module.

Same public surface as DGR/diff_gaussian_rasterization/__init__.py
(``GaussianRasterizationSettings`` :158-170, ``GaussianRasterizer`` :172-221,
``rasterize_gaussians`` :21-42), same argument meaning and error behaviour, but
the work is done by libs3g_b200.so through its C ABI (include/s3g_b200.h):
torch only owns the tensors and the stream.

    from s3gaussian_b200.diff_gaussian_rasterization import (
        GaussianRasterizationSettings, GaussianRasterizer)

`s3gaussian_b200.install_as_reference_module()` registers this module under the
name ``diff_gaussian_rasterization`` so the reference's
``gaussian_renderer/__init__.py:18`` import resolves to it unchanged.
"""
from __future__ import annotations

import ctypes as C
import warnings
from typing import NamedTuple

import torch
import torch.nn as nn

from .. import _lib


def cpu_deep_copy_tuple(input_tuple):
    copied_tensors = [item.cpu().clone() if isinstance(item, torch.Tensor) else item
                      for item in input_tuple]
    return tuple(copied_tensors)


class _Arena:
    """A growable device byte buffer handed to the C side as an s3g_alloc_fn
    (what resizeFunctional() does with a torch tensor, rasterize_points.cu:27-33).
    It only ever grows, so a recycled arena makes no allocator traffic."""

    def __init__(self, device):
        self.device = device
        self.tensor = torch.empty(0, dtype=torch.uint8, device=device)
        self.cb = _lib.ALLOC_FN(self._alloc)

    def _alloc(self, _user, nbytes):
        try:
            nbytes = int(nbytes)
            if self.tensor.numel() < nbytes:
                # 12 % headroom: num_rendered moves a little from view to view
                self.tensor = None
                self.tensor = torch.empty(nbytes + nbytes // 8, dtype=torch.uint8, device=self.device)
            return self.tensor.data_ptr()
        except Exception:   # pragma: no cover - surfaced as S3G_ERR_ALLOC
            return 0


class _ArenaSet:
    """The three opaque state buffers of one forward (geometry, binning, image)."""
    __slots__ = ("geom", "binning", "img", "key")

    def __init__(self, device, key):
        self.geom, self.binning, self.img, self.key = _Arena(device), _Arena(device), _Arena(device), key


# Recycling pool.  The reference allocates three fresh byte tensors per forward
# (rasterize_points.cu:72-79); at 2M Gaussians that is ~0.5 GB of differently
# sized blocks per step interleaved with the gradient tensors, which fragments
# torch's caching allocator into one cudaMalloc (~15 ms) per step.  A set is
# leased to one autograd node and comes back when that node dies; reuse is
# ordered by the CUDA stream, so the pool is keyed by (device, stream).
_POOL: dict = {}
_POOL_MAX_FREE = 4


class _Lease:
    def __init__(self, device):
        key = (device.index, torch.cuda.current_stream(device).cuda_stream)
        free = _POOL.setdefault(key, [])
        self.aset = free.pop() if free else _ArenaSet(device, key)

    def __del__(self):
        aset, self.aset = self.aset, None
        if aset is not None and _POOL is not None:
            free = _POOL.setdefault(aset.key, [])
            if len(free) < _POOL_MAX_FREE:
                free.append(aset)


def release_cached_arenas():
    """Drop all pooled state buffers (they are plain torch tensors)."""
    _POOL.clear()


# Optional gradient sink.  By default the backward allocates its gradient tensors (rasterize_points.cu:154-163 does
# the same); a data-parallel caller can instead route them into a communication buffer - e.g. a symmetric-memory
# bucket that our peer all-reduce kernels sum in place (dp.PeerAllReduce) - so no gather copy sits between the
# backward kernel and the collective.  The sink is any callable (name, shape, device) -> float32 tensor or None;
# names: means3D, means2D, colors_precomp, opacities, cov3D_precomp, shs, scales, rotations.
_GRAD_SINK = None


def set_grad_sink(sink):
    """Install (or with None remove) the gradient sink; returns the previous one."""
    global _GRAD_SINK
    prev, _GRAD_SINK = _GRAD_SINK, sink
    return prev


def _ptr(t: torch.Tensor | None):
    """device pointer, or NULL for the reference's 'absent' empty tensors
    (torch.Tensor([]), DGR/.../__init__.py:198-208)."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


def _f32c(t: torch.Tensor, device) -> torch.Tensor:
    if t.numel() == 0:
        return t
    if t.dtype != torch.float32:
        raise TypeError(f"expected float32 tensor, got {t.dtype}")
    if t.device != device:
        raise RuntimeError(f"tensor on {t.device}, expected {device}")
    return t.contiguous()   # rasterize_points.cu:95-113


def _stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _camera_inputs(raster_settings):
    """(viewmatrix, projmatrix, campos) of the settings when autograd is to reach the camera - grad mode is on and one
    of them requires grad - else None.  They then go to _RasterizeGaussians.apply as extra trailing inputs, so that
    its backward can return their gradients (s3g_rasterize_camera_backward)."""
    if not torch.is_grad_enabled():
        return None
    cam = (raster_settings.viewmatrix, raster_settings.projmatrix, raster_settings.campos)
    if any(isinstance(t, torch.Tensor) and t.requires_grad for t in cam):
        return cam
    return None


class Lens(NamedTuple):
    """A camera's intrinsics and OpenCV radial-tangential distortion, in pixels of the render size (s3g_raster_lens,
    include/s3g_b200.h).  Pixel j's centre is at j + 0.5, so a centred camera has cx = width / 2; an OpenCV K, whose
    pixel centres are at j, needs cx + 0.5 and cy + 0.5."""
    fx: float
    fy: float
    cx: float
    cy: float
    k1: float = 0.0
    k2: float = 0.0
    p1: float = 0.0
    p2: float = 0.0
    k3: float = 0.0


def _lens_struct(lens):
    return _lib.RasterLens(*(float(v) for v in lens))


def _lens_apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings,
                colors_aux, opacity, antialiasing, absgrad, lens):
    """_RasterizeGaussians.apply of a lens forward: every input given, the lens last.  Camera gradients do not pass
    through the lens."""
    if _camera_inputs(raster_settings) is not None:
        raise NotImplementedError("camera gradients through a lens are not implemented: detach viewmatrix, projmatrix "
                                  "and campos, or render without the lens")
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings, colors_aux, None, None, None, opacity,
                                     bool(antialiasing), bool(absgrad), Lens(*lens))


def _antialiased_apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                       raster_settings, colors_aux, opacity, antialiasing=True, absgrad=False):
    """_RasterizeGaussians.apply of an antialiased or absgrad forward: every optional input given, then the opacity
    switch, antialiasing and, with absgrad only, absgrad=True last."""
    cam = _camera_inputs(raster_settings)
    switches = (opacity, bool(antialiasing), True) if absgrad else (opacity, True)
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings, colors_aux,
                                     *(cam if cam is not None else (None, None, None)), *switches)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                        cov3Ds_precomp, raster_settings, antialiasing=False, absgrad=False, lens=None):
    if lens is not None:
        return _lens_apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                           raster_settings, None, False, antialiasing, absgrad, lens)
    if antialiasing or absgrad:
        return _antialiased_apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                  cov3Ds_precomp, raster_settings, None, False, antialiasing, absgrad)
    cam = _camera_inputs(raster_settings)
    if cam is not None:
        return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales,
                                         rotations, cov3Ds_precomp, raster_settings, None, *cam)
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales,
                                     rotations, cov3Ds_precomp, raster_settings)


def rasterize_gaussians_aux(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                            cov3Ds_precomp, raster_settings, colors_aux, antialiasing=False, absgrad=False, lens=None):
    """(color, radii, depth, color_aux): both colour sets composited on ONE preprocess + sort
    (the aux pair of s3g_rasterize_forward / s3g_rasterize_backward)."""
    if lens is not None:
        return _lens_apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                           raster_settings, colors_aux, False, antialiasing, absgrad, lens)
    if antialiasing or absgrad:
        return _antialiased_apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                  cov3Ds_precomp, raster_settings, colors_aux, False, antialiasing, absgrad)
    cam = _camera_inputs(raster_settings)
    if cam is not None:
        return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales,
                                         rotations, cov3Ds_precomp, raster_settings, colors_aux, *cam)
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales,
                                     rotations, cov3Ds_precomp, raster_settings, colors_aux)


def rasterize_gaussians_opacity(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                cov3Ds_precomp, raster_settings, colors_aux=None, antialiasing=False, absgrad=False,
                                lens=None):
    """(color, radii, depth, alpha, median_depth[, color_aux]): the opacity images of s3g_rasterize_forward_opacity
    from the same walk, differentiable like the others (the *_opacity backwards)."""
    if lens is not None:
        return _lens_apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                           raster_settings, colors_aux, True, antialiasing, absgrad, lens)
    if antialiasing or absgrad:
        return _antialiased_apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                  cov3Ds_precomp, raster_settings, colors_aux, True, antialiasing, absgrad)
    cam = _camera_inputs(raster_settings)
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                     cov3Ds_precomp, raster_settings, colors_aux,
                                     *(cam if cam is not None else (None, None, None)), True)


def _scene(rs, dev, means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp):
    """The s3g_raster_scene of one forward or backward call, from the settings and the float32 contiguous inputs.
    It holds (as `keep`) the float32 copies of the settings' tensors it points to; the input tensors must be kept
    alive by the caller until the call returns."""
    keep = tuple(_f32c(t, dev) for t in (rs.bg, rs.viewmatrix, rs.projmatrix, rs.campos))
    bg, view, proj, campos = keep
    scene = _lib.RasterScene(
        P=means3D.size(0), D=int(rs.sh_degree), M=sh.size(1) if sh.numel() != 0 else 0, background=_ptr(bg),
        width=int(rs.image_width), height=int(rs.image_height), means3D=_ptr(means3D), shs=_ptr(sh),
        colors_precomp=_ptr(colors_precomp), opacities=_ptr(opacities), scales=_ptr(scales),
        scale_modifier=float(rs.scale_modifier), rotations=_ptr(rotations), cov3D_precomp=_ptr(cov3Ds_precomp),
        viewmatrix=_ptr(view), projmatrix=_ptr(proj), cam_pos=_ptr(campos), tan_fovx=float(rs.tanfovx),
        tan_fovy=float(rs.tanfovy), prefiltered=int(bool(rs.prefiltered)), debug=int(bool(rs.debug)))
    scene.keep = keep
    return scene


def _forward_args(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs):
    """Checks, float32 contiguous inputs, outputs and state buffers of every forward, and its scene and forward
    arguments with no optional extra set.
    -> (scene, fwd, lease, (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp), color, depth,
    radii); the lease goes back to the pool when dropped: later users of the arenas are ordered by the stream."""
    if means3D.dim() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:57-59
    if not means3D.is_cuda:
        raise RuntimeError("s3gaussian_b200 has no CPU path: means3D must be a CUDA tensor")
    dev = means3D.device
    P = means3D.size(0)
    H, W = int(rs.image_height), int(rs.image_width)
    inputs = tuple(_f32c(t, dev) for t in (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp))
    scene = _scene(rs, dev, *inputs)

    color = torch.empty((3, H, W), dtype=torch.float32, device=dev)
    depth = torch.empty((1, H, W), dtype=torch.float32, device=dev)
    radii = torch.empty((P,), dtype=torch.int32, device=dev)
    lease = _Lease(dev)
    aset = lease.aset
    fwd = _lib.RasterForwardArgs(geom_alloc=aset.geom.cb, binning_alloc=aset.binning.cb, image_alloc=aset.img.cb,
                                 out_color=color.data_ptr(), out_depth=depth.data_ptr(), radii=_ptr(radii))
    return scene, fwd, lease, inputs, color, depth, radii


def rasterize_gaussians_eval(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                             raster_settings, group=None, flow_colors=(), with_opacity=False, antialiasing=False,
                             lens=None):
    """s3g_rasterize_forward with its forward-only extras: (color, radii, depth, decomposition, flows) from one
    preprocess, one sort and one composite walk.  decomposition is (color_d, depth_d, color_s, depth_s) when
    `group` (bool or uint8 [P] on the device) is given, else None: the images forward() gives for the Gaussians
    with group != 0 (dynamic) and group == 0 (static) alone.  flows holds one [3,H,W] image per entry of
    `flow_colors` (at most two float32 [P,4] device tensors, rgb in [:, :3], as s3g_flow_colors writes them), each
    the image forward() gives with colors_precomp = that rgb.  with_opacity adds a sixth element, (alpha,
    median_depth, alpha_d, alpha_s) as forward_opacity() defines them; alpha_d / alpha_s are the dynamic and static
    subsets' alpha images, None without `group`.  antialiasing: s3g_rasterize_forward_antialiased instead.  lens (a
    Lens): s3g_rasterize_forward_lens, through the camera's intrinsics and distortion.  Forward only: there is no
    autograd node."""
    lib = _lib.load()
    flow_colors = tuple(flow_colors)
    if len(flow_colors) > 2:
        raise RuntimeError("forward_eval composites at most two flow colour sets")
    if torch.is_grad_enabled() and any(t.requires_grad for t in (means3D, means2D, sh, colors_precomp, opacities,
                                                                 scales, rotations, cov3Ds_precomp)):
        raise RuntimeError("forward_eval has no backward: call it under torch.no_grad() or with detached inputs")
    scene, fwd, lease, _, color, depth, radii = _forward_args(means3D, sh, colors_precomp, opacities, scales,
                                                               rotations, cov3Ds_precomp, raster_settings)
    dev, P = means3D.device, means3D.size(0)
    decomposition = None
    if group is not None:
        if group.dtype not in (torch.bool, torch.uint8) or tuple(group.shape) != (P,) or group.device != dev:
            raise RuntimeError("group must be a bool or uint8 tensor of shape (num_points,) on the Gaussians' device")
        group = group.contiguous().view(torch.uint8)
        decomposition = tuple(torch.empty_like(t) for t in (color, depth, color, depth))
        fwd.group = _ptr(group)
        fwd.out_color_d, fwd.out_depth_d, fwd.out_color_s, fwd.out_depth_s = (t.data_ptr() for t in decomposition)
    for fc in flow_colors:
        if fc.dtype != torch.float32 or tuple(fc.shape) != (P, 4) or not fc.is_contiguous() or fc.device != dev:
            raise RuntimeError("flow colours must be contiguous float32 tensors of shape (num_points, 4) on the "
                               "Gaussians' device")
    flows = [torch.empty_like(color) for _ in flow_colors]
    fwd.n_flow = len(flows)
    for k, (fc, out) in enumerate(zip(flow_colors, flows)):
        fwd.flow_colors[k], fwd.out_flow[k] = _ptr(fc), out.data_ptr()
    with torch.cuda.device(dev):
        if lens is not None:
            opacity = None
            if with_opacity:
                opacity = tuple(torch.empty_like(depth) if i < 2 or group is not None else None for i in range(4))
                opa = _lib.RasterOpacityArgs(*(_ptr(t) for t in opacity))
            lens_s = _lens_struct(lens)
            _lib.check(lib.s3g_rasterize_forward_lens(C.byref(scene), C.byref(fwd), C.byref(opa) if with_opacity
                                                      else None, 1 if antialiasing else 0, C.byref(lens_s),
                                                      _stream_ptr(dev)), "rasterize_gaussians_eval")
            out = (color, radii, depth, decomposition, flows)
            return out + (opacity,) if with_opacity else out
        if not with_opacity:
            if antialiasing:
                _lib.check(lib.s3g_rasterize_forward_antialiased(C.byref(scene), C.byref(fwd), None,
                                                                 _stream_ptr(dev)), "rasterize_gaussians_eval")
            else:
                _lib.check(lib.s3g_rasterize_forward(C.byref(scene), C.byref(fwd), _stream_ptr(dev)),
                           "rasterize_gaussians_eval")
            return color, radii, depth, decomposition, flows
        opacity = tuple(torch.empty_like(depth) if i < 2 or group is not None else None for i in range(4))
        opa = _lib.RasterOpacityArgs(*(_ptr(t) for t in opacity))
        forward = lib.s3g_rasterize_forward_antialiased if antialiasing else lib.s3g_rasterize_forward_opacity
        _lib.check(forward(C.byref(scene), C.byref(fwd), C.byref(opa), _stream_ptr(dev)), "rasterize_gaussians_eval")
    return color, radii, depth, decomposition, flows, opacity


_FUSED_EXCHANGE_WARNED = False


def _absgrad_backward_call(lib, scene, bwd, dev, P, H, W, opa, absgrad):
    """s3g_rasterize_backward_absgrad into `absgrad` (float32 [P,2]): its deterministic form, with a workspace from the
    caching allocator, under torch.use_deterministic_algorithms(True) as in _backward_call, and its default form with
    a peer sink (with the same one-time warning)."""
    global _FUSED_EXCHANGE_WARNED
    det = torch.are_deterministic_algorithms_enabled()
    workspace = None
    if det and not bwd.sink:
        nbytes = int(lib.s3g_rasterize_backward_deterministic_workspace_bytes(P, bwd.R, W, H))
        workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes > 0 else None
    elif det and not _FUSED_EXCHANGE_WARNED:
        _FUSED_EXCHANGE_WARNED = True
        warnings.warn("the fused gradient exchange (FusedGradExchange) is not deterministic: the rasterizer "
                      "backward runs its default, atomic-reduction path while it is installed", UserWarning,
                      stacklevel=4)
    _lib.check(lib.s3g_rasterize_backward_absgrad(C.byref(scene), C.byref(bwd), C.byref(opa) if opa is not None
                                                  else None, absgrad.data_ptr(), 1 if det and not bwd.sink else 0,
                                                  _ptr(workspace), _stream_ptr(dev)),
               "rasterize_gaussians_backward_absgrad")


def _backward_call(lib, scene, bwd, dev, P, H, W, opa=None):
    """s3g_rasterize_backward, or under torch.use_deterministic_algorithms(True) (warn_only or not) its deterministic
    twin with a workspace from the caching allocator; with `opa` (a RasterOpacityArgs) their *_opacity forms.  The
    fused gradient exchange has no deterministic form: with a peer sink the default path runs and a warning says so
    once per process."""
    global _FUSED_EXCHANGE_WARNED
    if torch.are_deterministic_algorithms_enabled():
        if not bwd.sink:
            nbytes = int(lib.s3g_rasterize_backward_deterministic_workspace_bytes(P, bwd.R, W, H))
            workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes > 0 else None
            if opa is not None:
                _lib.check(lib.s3g_rasterize_backward_deterministic_opacity(
                    C.byref(scene), C.byref(bwd), C.byref(opa), _ptr(workspace), _stream_ptr(dev)),
                    "rasterize_gaussians_backward_deterministic_opacity")
                return
            _lib.check(lib.s3g_rasterize_backward_deterministic(C.byref(scene), C.byref(bwd), _ptr(workspace),
                                                                _stream_ptr(dev)),
                       "rasterize_gaussians_backward_deterministic")
            return
        if not _FUSED_EXCHANGE_WARNED:
            _FUSED_EXCHANGE_WARNED = True
            warnings.warn("the fused gradient exchange (FusedGradExchange) is not deterministic: the rasterizer "
                          "backward runs its default, atomic-reduction path while it is installed", UserWarning,
                          stacklevel=4)
    if opa is not None:
        _lib.check(lib.s3g_rasterize_backward_opacity(C.byref(scene), C.byref(bwd), C.byref(opa), _stream_ptr(dev)),
                   "rasterize_gaussians_backward_opacity")
        return
    _lib.check(lib.s3g_rasterize_backward(C.byref(scene), C.byref(bwd), _stream_ptr(dev)),
               "rasterize_gaussians_backward")


def _camera_backward_call(lib, scene, bwd, dev, P, cam_shapes, needs):
    """s3g_rasterize_camera_backward after the backward call on the same scene and arguments: the gradients of
    (viewmatrix, projmatrix, campos) shaped like those tensors, None where `needs` is false."""
    if P == 0:   # nothing rendered and no per-Gaussian gradients to pass: the gradients are zero
        return tuple(torch.zeros(shape, dtype=torch.float32, device=dev) if need else None
                     for shape, need in zip(cam_shapes, needs))
    outs = tuple(torch.empty(n, dtype=torch.float32, device=dev) if need else None
                 for n, need in zip((16, 16, 3), needs))
    nbytes = int(lib.s3g_rasterize_camera_backward_workspace_bytes(P))
    workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes > 0 else None
    grads = _lib.RasterCameraGrads(*(_ptr(o) for o in outs))
    _lib.check(lib.s3g_rasterize_camera_backward(C.byref(scene), C.byref(bwd), C.byref(grads), _ptr(workspace),
                                                 _stream_ptr(dev)), "rasterize_gaussians_camera_backward")
    return tuple(o.view(shape) if o is not None else None for o, shape in zip(outs, cam_shapes))


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                cov3Ds_precomp, raster_settings, colors_aux=None, viewmatrix=None, projmatrix=None, campos=None,
                opacity=False, antialiasing=False, absgrad=False, lens=None):
        # viewmatrix / projmatrix / campos: raster_settings' own tensors, passed (by rasterize_gaussians*) only when
        # one of them requires grad; the backward then returns their gradients.  opacity (rasterize_gaussians_opacity):
        # alpha and median_depth follow depth in the outputs.  antialiasing: s3g_rasterize_forward_antialiased, whose
        # chain rule the backward calls apply by themselves.  absgrad: the backward is s3g_rasterize_backward_absgrad
        # and sets (or adds to) the `absgrad` attribute of the tensor object passed as means2D.  lens (a Lens):
        # s3g_rasterize_forward_lens, whose chain rule the backward calls apply by themselves
        lib = _lib.load()
        rs = raster_settings
        scene, fwd, lease, inputs, color, depth, radii = _forward_args(means3D, sh, colors_precomp, opacities, scales,
                                                                        rotations, cov3Ds_precomp, rs)
        means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp = inputs
        dev = means3D.device
        has_aux = colors_aux is not None
        if has_aux:
            colors_aux = _f32c(colors_aux, dev)
            if tuple(colors_aux.shape) != (means3D.size(0), 3):
                raise RuntimeError("colors_aux must have dimensions (num_points, 3)")
            color_aux = torch.empty_like(color)
            fwd.colors_aux, fwd.out_color_aux = _ptr(colors_aux), color_aux.data_ptr()
        if opacity:
            alpha, median_depth = torch.empty_like(depth), torch.empty_like(depth)
            opa = _lib.RasterOpacityArgs(out_alpha=alpha.data_ptr(), out_median_depth=median_depth.data_ptr())
        if lens is not None:
            if viewmatrix is not None:
                raise NotImplementedError("camera gradients through a lens are not implemented")
            lens_s = _lens_struct(lens)
            forward_call = lambda: lib.s3g_rasterize_forward_lens(
                C.byref(scene), C.byref(fwd), C.byref(opa) if opacity else None, 1 if antialiasing else 0,
                C.byref(lens_s), _stream_ptr(dev))
        elif antialiasing:
            forward_call = lambda: lib.s3g_rasterize_forward_antialiased(
                C.byref(scene), C.byref(fwd), C.byref(opa) if opacity else None, _stream_ptr(dev))
        elif opacity:
            forward_call = lambda: lib.s3g_rasterize_forward_opacity(C.byref(scene), C.byref(fwd), C.byref(opa),
                                                                     _stream_ptr(dev))
        else:
            forward_call = lambda: lib.s3g_rasterize_forward(C.byref(scene), C.byref(fwd), _stream_ptr(dev))
        with torch.cuda.device(dev):
            if rs.debug:
                cpu_args = cpu_deep_copy_tuple((rs.bg, means3D, colors_precomp, opacities, scales,
                                                rotations, rs.scale_modifier, cov3Ds_precomp,
                                                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy,
                                                rs.image_height, rs.image_width, sh, rs.sh_degree,
                                                rs.campos, rs.prefiltered, rs.debug))
                try:
                    num_rendered = _lib.check(forward_call(), "rasterize_gaussians")
                except Exception as ex:
                    torch.save(cpu_args, "snapshot_fw.dump")
                    print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
                    raise ex
            else:
                num_rendered = _lib.check(forward_call(), "rasterize_gaussians")

        ctx.raster_settings = rs
        ctx.num_rendered = int(num_rendered)
        # the three state buffers stay with the lease (not save_for_backward: they are ours,
        # opaque and recycled); saved[7:10] keeps the reference's tuple layout for callers
        # that peek at it
        ctx.lease = lease
        aset = lease.aset
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh,
                              aset.geom.tensor, aset.binning.tensor, aset.img.tensor)
        ctx.mark_non_differentiable(radii)
        ctx.has_aux = has_aux
        ctx.camera = viewmatrix is not None
        if ctx.camera:
            ctx.cam_shapes = (rs.viewmatrix.shape, rs.projmatrix.shape, rs.campos.shape)
        ctx.opacity = bool(opacity)
        ctx.antialiasing = bool(antialiasing)
        ctx.absgrad = bool(absgrad)
        ctx.lens = lens is not None
        if absgrad:
            ctx.means2D = means2D
        out = (color, radii, depth) + ((alpha, median_depth) if opacity else ()) + ((color_aux,) if has_aux else ())
        return out

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, *grad_rest):
        # grad_rest: (grad_alpha, grad_median_depth) of an opacity forward, then grad_out_aux with the aux set
        opacity = getattr(ctx, "opacity", False)
        antialiasing = getattr(ctx, "antialiasing", False)
        absgrad = getattr(ctx, "absgrad", False)
        lens = getattr(ctx, "lens", False)
        grad_alpha, grad_median = grad_rest[:2] if opacity else (None, None)
        grad_rest = grad_rest[2:] if opacity else grad_rest
        grad_out_aux = grad_rest[0] if grad_rest else None
        lib = _lib.load()
        rs = ctx.raster_settings
        (colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer,
         binningBuffer, imgBuffer) = ctx.saved_tensors
        dev = means3D.device
        P = means3D.size(0)
        H, W = int(rs.image_height), int(rs.image_width)
        M = sh.size(1) if sh.numel() != 0 else 0
        if grad_out_color is None:
            grad_out_color = torch.zeros((3, H, W), dtype=torch.float32, device=dev)
        if grad_depth is None:
            grad_depth = torch.zeros((1, H, W), dtype=torch.float32, device=dev)
        grad_out_color = _f32c(grad_out_color, dev)
        grad_depth = _f32c(grad_depth, dev)
        scene = _scene(rs, dev, means3D, sh, colors_precomp, None, scales, rotations, cov3Ds_precomp)

        has_cov_in = cov3Ds_precomp.numel() != 0

        def e(name, *shape):
            if _GRAD_SINK is not None:
                t = _GRAD_SINK(name, shape, dev)
                if t is not None:
                    if t.dtype != torch.float32 or tuple(t.shape) != shape or not t.is_contiguous() or t.device != dev:
                        raise RuntimeError(f"gradient sink returned an unusable tensor for {name}")
                    return t
            return torch.empty(shape, dtype=torch.float32, device=dev)

        # every element is written by the kernel (zeros where radii <= 0): no memsets
        grad_means3D, grad_means2D = e("means3D", P, 3), e("means2D", P, 3)
        grad_colors, grad_opacities = e("colors_precomp", P, 3), e("opacities", P, 1)
        grad_cov3D, grad_sh = e("cov3D_precomp", P, 6), e("shs", P, M, 3)
        grad_scales, grad_rotations = e("scales", P, 3), e("rotations", P, 4)
        grad_aux = None
        if ctx.has_aux:
            if grad_out_aux is None:
                grad_out_aux = torch.zeros((3, H, W), dtype=torch.float32, device=dev)
            grad_out_aux = _f32c(grad_out_aux, dev)
            grad_aux = e("colors_aux", P, 3)

        bwd = _lib.RasterBackwardArgs(
            R=ctx.num_rendered, radii=_ptr(radii), geom_buffer=_ptr(geomBuffer), binning_buffer=_ptr(binningBuffer),
            image_buffer=_ptr(imgBuffer), dL_dpix=grad_out_color.data_ptr(), dL_dpix_depth=grad_depth.data_ptr(),
            dL_dmean2D=_ptr(grad_means2D), dL_dopacity=_ptr(grad_opacities), dL_dcolor=_ptr(grad_colors),
            dL_dmean3D=_ptr(grad_means3D), dL_dcov3D=_ptr(grad_cov3D), dL_dsh=_ptr(grad_sh),
            dL_dscale=_ptr(grad_scales), dL_drot=_ptr(grad_rotations))
        # camera gradients: the backward also exports the per-Gaussian conic and depth gradients they are built from
        cam_needs = tuple(ctx.needs_input_grad[10:13]) if ctx.camera else (False, False, False)
        if any(cam_needs):
            grad_conic = torch.empty((P, 4), dtype=torch.float32, device=dev)
            grad_gdepth = torch.empty((P,), dtype=torch.float32, device=dev)
            bwd.dL_dconic, bwd.dL_ddepth = _ptr(grad_conic), _ptr(grad_gdepth)
        peer = getattr(_GRAD_SINK, "peer_sink_struct", None)
        opa = None
        if opacity and (grad_alpha is not None or grad_median is not None):
            if peer is not None:
                raise NotImplementedError("FusedGradExchange: the opacity-image gradients are not exchanged")
            grad_alpha = _f32c(grad_alpha, dev) if grad_alpha is not None else None
            grad_median = _f32c(grad_median, dev) if grad_median is not None else None
            opa = _lib.RasterOpacityArgs(dL_dpix_alpha=_ptr(grad_alpha), dL_dpix_median=_ptr(grad_median))
        if ctx.has_aux:
            bwd.dL_dpix_aux, bwd.dL_dcolor_aux = grad_out_aux.data_ptr(), grad_aux.data_ptr()
        elif peer is not None:
            # data-parallel exchange fused into the kernel (dp.FusedGradExchange): the gradient tensors returned
            # below are views of the exchange's bucket and hold the sums after its finish()
            if has_cov_in:
                raise NotImplementedError("FusedGradExchange: precomputed 3-D covariances are not exchanged")
            if antialiasing:
                raise NotImplementedError("FusedGradExchange: an antialiased forward's gradients are not exchanged")
            if lens:
                raise NotImplementedError("FusedGradExchange: a lens forward's gradients are not exchanged")
            _GRAD_SINK.note_backward()
            bwd.sink = C.pointer(peer)
        # the kernel stores dL_drot 16 bytes per row: a sink's view off a 16-byte boundary (a flat bucket holding the
        # tensors back to back, as bench.py lays it out for N > 1) receives the rows through an aligned tensor
        rot_out = grad_rotations
        if not bwd.sink and P > 0 and grad_rotations.data_ptr() % 16:
            rot_out = torch.empty_like(grad_rotations)
            bwd.dL_drot = _ptr(rot_out)
        grad_abs = None
        call = lambda: _backward_call(lib, scene, bwd, dev, P, H, W, opa)
        if absgrad:
            grad_abs = torch.empty((P, 2), dtype=torch.float32, device=dev)     # every row is written
            call = lambda: _absgrad_backward_call(lib, scene, bwd, dev, P, H, W, opa, grad_abs)
        with torch.cuda.device(dev):
            if P > 0:
                if rs.debug:
                    try:
                        call()
                    except Exception as ex:
                        print("\nAn error occured in backward.\n")
                        raise ex
                else:
                    call()
                if rot_out is not grad_rotations:
                    grad_rotations.copy_(rot_out)
            if any(cam_needs):
                cam_grads = _camera_backward_call(lib, scene, bwd, dev, P, ctx.cam_shapes, cam_needs)

        has_colors = colors_precomp.numel() != 0
        has_cov = cov3Ds_precomp.numel() != 0
        grads = (
            grad_means3D,
            grad_means2D,
            grad_sh if not has_colors else None,
            grad_colors if has_colors else None,
            grad_opacities,
            grad_scales if not has_cov else None,
            grad_rotations if not has_cov else None,
            grad_cov3D if has_cov else None,
            None,
        )
        if absgrad:
            # gsplat's means2d.absgrad: set on the tensor object passed as means2D, added to like .grad
            m2 = ctx.means2D
            prev = getattr(m2, "absgrad", None)
            m2.absgrad = grad_abs if prev is None else prev + grad_abs
        if lens:   # every input was given (_lens_apply)
            return grads + (grad_aux, None, None, None, None, None, None, None)
        if ctx.has_aux:
            grads = grads + (grad_aux,)
        if ctx.camera or opacity or antialiasing or absgrad:
            if not ctx.has_aux:
                grads = grads + (None,)
            grads = grads + (cam_grads if any(cam_needs) else (None, None, None))
        if opacity or antialiasing or absgrad:
            grads = grads + (None,)
        if antialiasing or absgrad:
            grads = grads + (None,)
        if absgrad:
            grads = grads + (None,)
        return grads


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


def _reference_inputs(shs, colors_precomp, scales, rotations, cov3D_precomp):
    """The reference's argument checks of GaussianRasterizer.forward (DGR/.../__init__.py:188-208), with each absent
    input replaced by an empty tensor."""
    if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
        raise Exception('Please provide excatly one of either SHs or precomputed colors!')

    if ((scales is None or rotations is None) and cov3D_precomp is None) or \
            ((scales is not None or rotations is not None) and cov3D_precomp is not None):
        raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')

    return tuple(torch.Tensor([]) if t is None else t for t in (shs, colors_precomp, scales, rotations, cov3D_precomp))


class GaussianRasterizer(nn.Module):
    """antialiasing=True: every forward applies Mip-Splatting's 2-D screen-space filter (s3g_rasterize_forward_antialiased,
    include/s3g_b200.h): each Gaussian's opacity is scaled by h = sqrt(max(det(cov2D) / det(cov2D + 0.3 I), 2.5e-5)),
    so a Gaussian smaller than a pixel keeps its on-screen energy at every resolution.  The backwards, camera
    gradients included, differentiate that forward.  Not in the reference (upstream 3DGS: `antialiasing`, gsplat:
    rasterize_mode="antialiased").

    absgrad=True: the backwards of forward(), forward_aux() and forward_opacity() also compute each Gaussian's absolute
    screen-space gradient (AbsGS; gsplat rasterization(absgrad=True)), sum over its pixels p of |dL_p/dmean2D| per
    component, in the units of means2D.grad, and store it as `means2D.absgrad` (float32 [P,2], zero for Gaussians
    with radii <= 0) on the tensor object passed as means2D.  A second backward into the same object adds to it, as
    .grad accumulates; set it to None to start again.  The statistic is per call: the aux pair's two images share one
    sum, two separate calls add two.  Not in the reference.

    lens (a Lens, or anything unpacking to fx, fy, cx, cy[, k1, k2, p1, p2, k3]): every forward projects through the
    camera's own intrinsics and OpenCV radial-tangential distortion (s3g_rasterize_forward_lens, include/s3g_b200.h)
    instead of the centred pinhole of tanfovx / tanfovy; viewmatrix still places the camera.  The backwards
    differentiate that projection; the lens gets no gradient, and camera gradients through it are not implemented
    (NotImplementedError when viewmatrix, projmatrix or campos requires grad).  Not in the reference."""

    def __init__(self, raster_settings, antialiasing=False, absgrad=False, lens=None):
        super().__init__()
        self.raster_settings = raster_settings
        self.antialiasing = bool(antialiasing)
        self.absgrad = bool(absgrad)
        self.lens = None if lens is None else Lens(*lens)

    def markVisible(self, positions):
        """bool[P]: passes the near-plane test (rasterizer_impl.cu:54-66)."""
        lib = _lib.load()
        with torch.no_grad():
            rs = self.raster_settings
            dev = positions.device
            if not positions.is_cuda:
                raise RuntimeError("s3gaussian_b200 has no CPU path: positions must be a CUDA tensor")
            positions = _f32c(positions, dev)
            P = positions.size(0)
            present = torch.zeros((P,), dtype=torch.bool, device=dev)
            with torch.cuda.device(dev):
                _lib.check(lib.s3g_mark_visible(P, _ptr(positions), _ptr(_f32c(rs.viewmatrix, dev)),
                                                _ptr(_f32c(rs.projmatrix, dev)), _ptr(present),
                                                _stream_ptr(dev)), "mark_visible")
        return present

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None,
                rotations=None, cov3D_precomp=None):
        shs, colors_precomp, scales, rotations, cov3D_precomp = _reference_inputs(shs, colors_precomp, scales,
                                                                                  rotations, cov3D_precomp)
        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales,
                                   rotations, cov3D_precomp, self.raster_settings, self.antialiasing, self.absgrad,
                                   self.lens)

    def forward_aux(self, means3D, means2D, opacities, colors_aux, shs=None, colors_precomp=None, scales=None,
                    rotations=None, cov3D_precomp=None):
        """forward() plus a second [P,3] colour set composited on the same binning:
        -> (color, radii, depth, color_aux).  Not in the reference (it calls forward() twice,
        gaussian_renderer/__init__.py:173-186); same arguments otherwise."""
        shs, colors_precomp, scales, rotations, cov3D_precomp = _reference_inputs(shs, colors_precomp, scales,
                                                                                  rotations, cov3D_precomp)
        return rasterize_gaussians_aux(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                       cov3D_precomp, self.raster_settings, colors_aux, self.antialiasing,
                                       self.absgrad, self.lens)

    def forward_opacity(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                        cov3D_precomp=None, colors_aux=None):
        """forward() (or forward_aux() with colors_aux) plus two [1,H,W] images from the same walk:
        -> (color, radii, depth, alpha, median_depth[, color_aux]).  alpha = 1 - the transmittance the background is
        blended with, so color = (the bg = 0 image) + (1 - alpha) * bg; median_depth = the depth of the first Gaussian,
        front to back, whose blend takes the transmittance from > 0.5 to <= 0.5 (0 where alpha stays <= 0.5).  Every
        output except radii is differentiable, the camera tensors included; the backward follows
        torch.use_deterministic_algorithms as forward()'s does.  Not in the reference."""
        shs, colors_precomp, scales, rotations, cov3D_precomp = _reference_inputs(shs, colors_precomp, scales,
                                                                                  rotations, cov3D_precomp)
        return rasterize_gaussians_opacity(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                           cov3D_precomp, self.raster_settings, colors_aux, self.antialiasing,
                                           self.absgrad, self.lens)

    def forward_eval(self, means3D, means2D, opacities, group=None, flow_colors=(), shs=None, colors_precomp=None,
                     scales=None, rotations=None, cov3D_precomp=None, with_opacity=False):
        """Every image of an evaluated view from one preprocess + sort + composite:
        -> (color, radii, depth, decomposition, flows).  decomposition is (color_d, depth_d, color_s, depth_s) when
        `group` (bool or uint8 [P] on the device) is given, else None: what forward() returns for the Gaussians with
        group != 0 (dynamic) / group == 0 (static) only.  flows has one [3,H,W] image per `flow_colors` entry (at
        most two float32 [P,4] device tensors, rgb in [:, :3]), equal to forward() with colors_precomp = that rgb.
        with_opacity=True appends (alpha, median_depth, alpha_d, alpha_s): forward_opacity()'s two images and the
        alpha images of the dynamic and static subsets (None without `group`).
        Forward only (no autograd node): raises if autograd would record through the inputs.  Not in the reference
        (its evaluation renders each view once per image, utils/video_utils.py:170-299, and its
        render(return_decomposition=True) calls forward() three times, gaussian_renderer/__init__.py:177-192)."""
        shs, colors_precomp, scales, rotations, cov3D_precomp = _reference_inputs(shs, colors_precomp, scales,
                                                                                  rotations, cov3D_precomp)
        return rasterize_gaussians_eval(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                        cov3D_precomp, self.raster_settings, group, flow_colors, with_opacity,
                                        self.antialiasing, self.lens)
