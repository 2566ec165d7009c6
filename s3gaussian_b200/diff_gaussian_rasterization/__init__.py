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


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                        cov3Ds_precomp, raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales,
                                     rotations, cov3Ds_precomp, raster_settings)


def rasterize_gaussians_aux(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                            cov3Ds_precomp, raster_settings, colors_aux):
    """(color, radii, depth, color_aux): both colour sets composited on ONE preprocess + sort
    (s3g_rasterize_forward_aux / s3g_rasterize_backward_aux)."""
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales,
                                     rotations, cov3Ds_precomp, raster_settings, colors_aux)


def rasterize_gaussians_split(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                              raster_settings, group):
    """(color, radii, depth, color_d, depth_d, color_s, depth_s) of s3g_rasterize_forward_split: the full image and
    the images of the Gaussians with group != 0 (dynamic) and group == 0 (static) alone, from one preprocess, one
    sort and one composite walk.  Forward only: there is no autograd node."""
    lib = _lib.load()
    tensors = (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp)
    if torch.is_grad_enabled() and any(t.requires_grad for t in tensors + (means2D,)):
        raise RuntimeError("forward_split has no backward: call it under torch.no_grad() or with detached inputs")
    if means3D.dim() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    if not means3D.is_cuda:
        raise RuntimeError("s3gaussian_b200 has no CPU path: means3D must be a CUDA tensor")
    dev = means3D.device
    rs = raster_settings
    P = means3D.size(0)
    H, W = int(rs.image_height), int(rs.image_width)
    if group.dtype not in (torch.bool, torch.uint8) or tuple(group.shape) != (P,) or group.device != dev:
        raise RuntimeError("group must be a bool or uint8 tensor of shape (num_points,) on the Gaussians' device")
    group = group.contiguous().view(torch.uint8)
    means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp = (_f32c(t, dev) for t in tensors)
    bg = _f32c(rs.bg, dev)
    view = _f32c(rs.viewmatrix, dev)
    proj = _f32c(rs.projmatrix, dev)
    campos = _f32c(rs.campos, dev)

    color, color_d, color_s = (torch.empty((3, H, W), dtype=torch.float32, device=dev) for _ in range(3))
    depth, depth_d, depth_s = (torch.empty((1, H, W), dtype=torch.float32, device=dev) for _ in range(3))
    radii = torch.empty((P,), dtype=torch.int32, device=dev)
    lease = _Lease(dev)   # back to the pool on return: later users of the arenas are ordered by the stream
    geom, binning, img = lease.aset.geom, lease.aset.binning, lease.aset.img
    M = sh.size(1) if sh.numel() != 0 else 0
    args = (geom.cb, None, binning.cb, None, img.cb, None, P, int(rs.sh_degree), M, _ptr(bg), W, H,
            _ptr(means3D), _ptr(sh), _ptr(colors_precomp), _ptr(opacities), _ptr(scales),
            float(rs.scale_modifier), _ptr(rotations), _ptr(cov3Ds_precomp), _ptr(view),
            _ptr(proj), _ptr(campos), float(rs.tanfovx), float(rs.tanfovy),
            int(bool(rs.prefiltered)), color.data_ptr(), depth.data_ptr(), _ptr(radii),
            int(bool(rs.debug)), _stream_ptr(dev), _ptr(group), color_d.data_ptr(), depth_d.data_ptr(),
            color_s.data_ptr(), depth_s.data_ptr())
    with torch.cuda.device(dev):
        _lib.check(lib.s3g_rasterize_forward_split(*args), "rasterize_gaussians_split")
    return color, radii, depth, color_d, depth_d, color_s, depth_s


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                cov3Ds_precomp, raster_settings, colors_aux=None):
        lib = _lib.load()
        if means3D.dim() != 2 or means3D.size(1) != 3:
            raise RuntimeError("means3D must have dimensions (num_points, 3)")  # rasterize_points.cu:57-59
        if not means3D.is_cuda:
            raise RuntimeError("s3gaussian_b200 has no CPU path: means3D must be a CUDA tensor")
        dev = means3D.device
        rs = raster_settings
        P = means3D.size(0)
        H, W = int(rs.image_height), int(rs.image_width)

        means3D = _f32c(means3D, dev)
        sh = _f32c(sh, dev)
        colors_precomp = _f32c(colors_precomp, dev)
        opacities = _f32c(opacities, dev)
        scales = _f32c(scales, dev)
        rotations = _f32c(rotations, dev)
        cov3Ds_precomp = _f32c(cov3Ds_precomp, dev)
        has_aux = colors_aux is not None
        if has_aux:
            colors_aux = _f32c(colors_aux, dev)
            if tuple(colors_aux.shape) != (P, 3):
                raise RuntimeError("colors_aux must have dimensions (num_points, 3)")
        bg = _f32c(rs.bg, dev)
        view = _f32c(rs.viewmatrix, dev)
        proj = _f32c(rs.projmatrix, dev)
        campos = _f32c(rs.campos, dev)

        color = torch.empty((3, H, W), dtype=torch.float32, device=dev)
        depth = torch.empty((1, H, W), dtype=torch.float32, device=dev)
        radii = torch.empty((P,), dtype=torch.int32, device=dev)
        color_aux = torch.empty((3, H, W), dtype=torch.float32, device=dev) if has_aux else None
        lease = _Lease(dev)
        geom, binning, img = lease.aset.geom, lease.aset.binning, lease.aset.img
        M = sh.size(1) if sh.numel() != 0 else 0

        args = (geom.cb, None, binning.cb, None, img.cb, None, P, int(rs.sh_degree), M, _ptr(bg), W, H,
                _ptr(means3D), _ptr(sh), _ptr(colors_precomp), _ptr(opacities), _ptr(scales),
                float(rs.scale_modifier), _ptr(rotations), _ptr(cov3Ds_precomp), _ptr(view),
                _ptr(proj), _ptr(campos), float(rs.tanfovx), float(rs.tanfovy),
                int(bool(rs.prefiltered)), color.data_ptr(), depth.data_ptr(), _ptr(radii),
                int(bool(rs.debug)), _stream_ptr(dev))
        fwd = lib.s3g_rasterize_forward
        if has_aux:
            args = args + (_ptr(colors_aux), color_aux.data_ptr())
            fwd = lib.s3g_rasterize_forward_aux
        with torch.cuda.device(dev):
            if rs.debug:
                cpu_args = cpu_deep_copy_tuple((rs.bg, means3D, colors_precomp, opacities, scales,
                                                rotations, rs.scale_modifier, cov3Ds_precomp,
                                                rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy,
                                                rs.image_height, rs.image_width, sh, rs.sh_degree,
                                                rs.campos, rs.prefiltered, rs.debug))
                try:
                    num_rendered = _lib.check(fwd(*args), "rasterize_gaussians")
                except Exception as ex:
                    torch.save(cpu_args, "snapshot_fw.dump")
                    print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
                    raise ex
            else:
                num_rendered = _lib.check(fwd(*args), "rasterize_gaussians")

        ctx.raster_settings = rs
        ctx.num_rendered = int(num_rendered)
        # the three state buffers stay with the lease (not save_for_backward: they are ours,
        # opaque and recycled); saved[7:10] keeps the reference's tuple layout for callers
        # that peek at it
        ctx.lease = lease
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh,
                              geom.tensor, binning.tensor, img.tensor)
        ctx.mark_non_differentiable(radii)
        ctx.has_aux = has_aux
        if has_aux:
            return color, radii, depth, color_aux
        return color, radii, depth

    @staticmethod
    def backward(ctx, grad_out_color, grad_radii, grad_depth, grad_out_aux=None):
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
        bg = _f32c(rs.bg, dev)
        view = _f32c(rs.viewmatrix, dev)
        proj = _f32c(rs.projmatrix, dev)
        campos = _f32c(rs.campos, dev)

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

        args = (P, int(rs.sh_degree), M, ctx.num_rendered, _ptr(bg), W, H, _ptr(means3D), _ptr(sh),
                _ptr(colors_precomp), _ptr(scales), float(rs.scale_modifier), _ptr(rotations),
                _ptr(cov3Ds_precomp), _ptr(view), _ptr(proj), _ptr(campos), float(rs.tanfovx),
                float(rs.tanfovy), _ptr(radii), _ptr(geomBuffer), _ptr(binningBuffer),
                _ptr(imgBuffer), grad_out_color.data_ptr(), grad_depth.data_ptr(),
                _ptr(grad_means2D), None, _ptr(grad_opacities), _ptr(grad_colors), None,
                _ptr(grad_means3D), _ptr(grad_cov3D), _ptr(grad_sh), _ptr(grad_scales),
                _ptr(grad_rotations), int(bool(rs.debug)), _stream_ptr(dev))
        bwd = lib.s3g_rasterize_backward
        peer = getattr(_GRAD_SINK, "peer_sink_struct", None)
        if ctx.has_aux:
            args = args + (grad_out_aux.data_ptr(), grad_aux.data_ptr())
            bwd = lib.s3g_rasterize_backward_aux
        elif peer is not None:
            # data-parallel exchange fused into the kernel (dp.FusedGradExchange): the gradient tensors returned
            # below are views of the exchange's bucket and hold the sums after its finish()
            if has_cov_in:
                raise NotImplementedError("FusedGradExchange: precomputed 3-D covariances are not exchanged")
            import ctypes as _C
            _GRAD_SINK.note_backward()
            args = args + (_C.byref(peer),)
            bwd = lib.s3g_rasterize_backward_dp
        with torch.cuda.device(dev):
            if P > 0:
                if rs.debug:
                    try:
                        _lib.check(bwd(*args), "rasterize_gaussians_backward")
                    except Exception as ex:
                        print("\nAn error occured in backward.\n")
                        raise ex
                else:
                    _lib.check(bwd(*args), "rasterize_gaussians_backward")

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
        if ctx.has_aux:
            grads = grads + (grad_aux,)
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


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

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
        raster_settings = self.raster_settings

        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')

        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')

        if shs is None:
            shs = torch.Tensor([])
        if colors_precomp is None:
            colors_precomp = torch.Tensor([])
        if scales is None:
            scales = torch.Tensor([])
        if rotations is None:
            rotations = torch.Tensor([])
        if cov3D_precomp is None:
            cov3D_precomp = torch.Tensor([])

        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales,
                                   rotations, cov3D_precomp, raster_settings)

    def forward_aux(self, means3D, means2D, opacities, colors_aux, shs=None, colors_precomp=None, scales=None,
                    rotations=None, cov3D_precomp=None):
        """forward() plus a second [P,3] colour set composited on the same binning:
        -> (color, radii, depth, color_aux).  Not in the reference (it calls forward() twice,
        gaussian_renderer/__init__.py:173-186); same arguments otherwise."""
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        E = torch.Tensor([])
        return rasterize_gaussians_aux(means3D, means2D, shs if shs is not None else E,
                                       colors_precomp if colors_precomp is not None else E, opacities,
                                       scales if scales is not None else E, rotations if rotations is not None else E,
                                       cov3D_precomp if cov3D_precomp is not None else E, self.raster_settings,
                                       colors_aux)

    def forward_split(self, means3D, means2D, opacities, group, shs=None, colors_precomp=None, scales=None,
                      rotations=None, cov3D_precomp=None):
        """forward() plus the images of the two Gaussian groups alone, from one preprocess + sort + composite:
        -> (color, radii, depth, color_d, depth_d, color_s, depth_s), where _d / _s are what forward() returns for
        the Gaussians with group != 0 / group == 0 only.  `group`: bool or uint8 [P] on the device.  Forward only
        (no autograd node): raises if autograd would record through the inputs.  Not in the reference (its
        render(return_decomposition=True) calls forward() three times, gaussian_renderer/__init__.py:177-192)."""
        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')
        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')
        E = torch.Tensor([])
        return rasterize_gaussians_split(means3D, means2D, shs if shs is not None else E,
                                         colors_precomp if colors_precomp is not None else E, opacities,
                                         scales if scales is not None else E, rotations if rotations is not None else E,
                                         cov3D_precomp if cov3D_precomp is not None else E, self.raster_settings,
                                         group)
