"""The sky model on the device (csrc/sky.cuh; include/s3g_b200.h, "sky model").

EmerNeRF's sky head as the reference declares it (``scene/background_model.py``: ``SkyModel``,
``Background_Model(model_type="mlp")``): every pixel's world-space ray direction goes through a sinusoidal encoding
and a 3-layer MLP with a skip connection, and a sigmoid gives the sky colour behind the Gaussians.  The caller
composites ``render_bg0 + (1 - alpha) * sky``, with ``render_bg0`` and ``alpha`` from ``render()`` with a zero
background and ``pipe.render_opacity``.

``Background_Model`` and ``SkyModel`` keep the reference's names and parameter layout, so a reference ``state_dict``
loads unchanged.  ``Background_Model.forward(c2w, intrinsic)`` is differentiable in the six MLP parameters (not in the
camera: the reference's encoder runs under no_grad); its weight gradients repeat bit for bit.  CUDA only; there is no
CPU path.
"""
from __future__ import annotations

import ctypes as C
import math
import numbers

import torch
from torch import nn

from . import _lib

WIDTHS = (64, 128, 192, 256)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


class SinusoidalEncoder(nn.Module):
    """The reference's ``SinusoidalEncoder(n_input_dims=3, min_deg=0, max_deg=4)``: [x, sin(x s), sin(x s + pi/2)],
    s = 1, 2, 4, 8, 16 (33 features).  Holds the ``scales`` buffer of the reference's state dict; the encoding itself
    runs inside the sky kernels."""

    def __init__(self, n_input_dims: int = 3, min_deg: int = 0, max_deg: int = 4):
        super().__init__()
        self.n_input_dims, self.min_deg, self.max_deg = n_input_dims, min_deg, max_deg
        self.register_buffer("scales", torch.tensor([2.0 ** i for i in range(min_deg, max_deg + 1)]))

    @property
    def n_output_dims(self) -> int:
        return (1 + (self.max_deg - self.min_deg + 1) * 2) * self.n_input_dims


class MLP(nn.Module):
    """The reference's ``MLP(in_dims=33, out_dims=3, num_layers=3, hidden_dims=width, skip_connections=[1])``: its
    ``layers`` are Linear(33, width), Linear(width + 33, width), Linear(width, 3)."""

    def __init__(self, in_dims: int, out_dims: int, hidden_dims: int):
        super().__init__()
        self.in_dims, self.hidden_dims, self.n_output_dims = in_dims, hidden_dims, out_dims
        self.num_layers, self.skip_connections = 3, [1]
        self.layers = nn.ModuleList([nn.Linear(in_dims, hidden_dims), nn.Linear(in_dims + hidden_dims, hidden_dims),
                                     nn.Linear(hidden_dims, out_dims)])


class SkyModel(nn.Module):
    """The reference's ``SkyModel(model_cfg)``: ``direction_encoding`` and ``sky_head``; ``model_cfg["mlp_width"]`` is
    the hidden width, a multiple of 64 from 64 to 256.  The parameters are nn.Linear's, initialised as nn.Linear
    initialises them."""

    def __init__(self, model_cfg: dict = {"mlp_width": 256}):   # noqa: B006 (the reference's default, never mutated)
        super().__init__()
        if "mlp_width" not in model_cfg:
            raise KeyError(f"SkyModel: model_cfg has no 'mlp_width' (the hidden width of the sky head); got keys "
                           f"{sorted(model_cfg)}")
        width = model_cfg["mlp_width"]
        if not isinstance(width, numbers.Integral) or isinstance(width, bool) or int(width) not in WIDTHS:
            raise ValueError(f"SkyModel: mlp_width must be one of {WIDTHS}, got {width!r}")
        self.model_cfg = model_cfg
        self.direction_encoding = SinusoidalEncoder(n_input_dims=3, min_deg=0, max_deg=4)
        self.sky_head = MLP(in_dims=self.direction_encoding.n_output_dims, out_dims=3, hidden_dims=int(width))

    @property
    def width(self) -> int:
        return self.sky_head.hidden_dims


def _net(params, width):
    w0, b0, w1, b1, w2, b2 = params
    return _lib.SkyNet(width, w0.data_ptr(), b0.data_ptr(), w1.data_ptr(), b1.data_ptr(), w2.data_ptr(),
                       b2.data_ptr())


def _workspace(lib, width, H, W, dev):
    return torch.empty(lib.s3g_sky_workspace_bytes(width, H, W), dtype=torch.uint8, device=dev)


def _forward(c2w, intrinsic, H, W, params):
    lib = _lib.load()
    width = params[0].shape[0]
    dev = c2w.device
    out = torch.empty(3, H, W, dtype=torch.float32, device=dev)
    ws = _workspace(lib, width, H, W, dev)
    net = _net(params, width)
    with torch.cuda.device(dev):
        _lib.check(lib.s3g_sky_forward(C.byref(net), H, W, c2w.data_ptr(), intrinsic.data_ptr(), out.data_ptr(),
                                       ws.data_ptr(), _stream()), "s3g_sky_forward")
    return out


class _Sky(torch.autograd.Function):
    @staticmethod
    def forward(ctx, c2w, intrinsic, H, W, *params):
        ctx.HW = (H, W)
        ctx.save_for_backward(c2w, intrinsic, *params)
        return _forward(c2w, intrinsic, H, W, params)

    @staticmethod
    def backward(ctx, grad_out):
        c2w, intrinsic, *params = ctx.saved_tensors
        H, W = ctx.HW
        lib = _lib.load()
        width = params[0].shape[0]
        dev = c2w.device
        g = grad_out.to(torch.float32).contiguous()
        grads = [torch.empty_like(p) for p in params]
        ws = _workspace(lib, width, H, W, dev)
        net = _net(params, width)
        gnet = _lib.SkyNetGrads(*(t.data_ptr() for t in grads))
        with torch.cuda.device(dev):
            _lib.check(lib.s3g_sky_backward(C.byref(net), H, W, c2w.data_ptr(), intrinsic.data_ptr(), g.data_ptr(),
                                            C.byref(gnet), ws.data_ptr(), _stream()), "s3g_sky_backward")
        return (None, None, None, None, *(gr if need else None for gr, need in zip(grads, ctx.needs_input_grad[4:])))


def _camera_tensor(x, name, n, dev):
    if not isinstance(x, torch.Tensor):
        raise ValueError(f"Background_Model: {name} must be a tensor, got {type(x).__name__}")
    if x.dim() == 3 and x.shape[0] == 1:
        x = x[0]
    if tuple(x.shape) != (n, n):
        raise ValueError(f"Background_Model: {name} must be [{n},{n}] (or [1,{n},{n}]), got {tuple(x.shape)}")
    if not x.is_floating_point():
        raise ValueError(f"Background_Model: {name} must be a floating-point tensor, got {x.dtype}")
    return x.detach().to(device=dev, dtype=torch.float32).contiguous()


class Background_Model(nn.Module):   # noqa: N801 (the reference's name)
    """The reference's ``Background_Model``: ``model_type="mlp"`` holds a ``SkyModel`` as ``sky_model`` and renders
    its sky image for a camera.  ``"gs"``, ``"rec_shell"`` and ``"sphere_shell"`` are not implemented here.
    ``aabb``, ``cam_norm`` and ``model_args`` are kept for the reference's signature; the MLP does not use them."""

    def __init__(self, img_width=960, img_height=640, aabb=None, cam_norm=None, model_type="mlp",
                 model_cfg: dict = {"head_mlp_layer_width": 256}, model_args: dict = {}):   # noqa: B006
        super().__init__()
        for name, v in (("img_width", img_width), ("img_height", img_height)):
            if not isinstance(v, numbers.Integral) or isinstance(v, bool) or v < 1:
                raise ValueError(f"Background_Model: {name} must be an integer >= 1, got {v!r}")
        if 3 * img_width * img_height > 2 ** 31 - 1:
            raise ValueError("Background_Model: 3 * img_width * img_height must fit 32-bit indices")
        if model_type != "mlp":
            raise NotImplementedError(f"Background_Model: model_type {model_type!r} is not implemented (only 'mlp')")
        self.aabb, self.model_args = aabb, model_args
        self.img_width, self.img_height = int(img_width), int(img_height)
        self.model_type, self.model_cfg = model_type, model_cfg
        self.sky_model = SkyModel(model_cfg)

    def _params(self):
        lay = self.sky_model.sky_head.layers
        return (lay[0].weight, lay[0].bias, lay[1].weight, lay[1].bias, lay[2].weight, lay[2].bias)

    def forward(self, c2w, intrinsic, img_idx=None) -> torch.Tensor:
        """The sky colour [3, img_height, img_width] seen by a camera with ``c2w`` [4,4] and pixel ``intrinsic``
        [3,3] (at this model's image size); differentiable in the MLP parameters.  ``img_idx`` is unused, as in the
        reference."""
        params = self._params()
        for p in params:
            if not p.is_cuda:
                raise RuntimeError("Background_Model: the parameters must be on a CUDA device (there is no CPU path); "
                                   "call .cuda()")
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise ValueError("Background_Model: the parameters must be contiguous float32")
        dev = params[0].device
        if any(p.device != dev for p in params):
            raise RuntimeError("Background_Model: the parameters are on more than one device")
        c2w = _camera_tensor(c2w, "c2w", 4, dev)
        intrinsic = _camera_tensor(intrinsic, "intrinsic", 3, dev)
        H, W = self.img_height, self.img_width
        if torch.is_grad_enabled() and any(p.requires_grad for p in params):
            return _Sky.apply(c2w, intrinsic, H, W, *params)
        return _forward(c2w, intrinsic, H, W, tuple(p.detach() for p in params))


def sky_camera(viewpoint_cam):
    """``(c2w [4,4], intrinsic [3,3])`` float32 of a camera: a reference camera's own ``c2w`` / ``intrinsic``
    (scene/cameras.py) when it has them; otherwise ``c2w`` derived from ``world_view_transform`` (W2C transposed) and
    the camera's own ``intrinsic`` when it has one, else one from the fields of view with the principal point at the
    image centre (``SyntheticCamera``).  With that intrinsic, the sky
    direction of pixel (x, y) projects through ``full_proj_transform`` onto the rasterizer's centre of that pixel."""
    c2w = getattr(viewpoint_cam, "c2w", None)
    K = getattr(viewpoint_cam, "intrinsic", None)
    if c2w is not None and K is not None:
        c2w, K = torch.as_tensor(c2w), torch.as_tensor(K)
        return c2w.to(torch.float32).reshape(4, 4).contiguous(), K.to(torch.float32).reshape(3, 3).contiguous()
    wvt = viewpoint_cam.world_view_transform
    c2w = torch.linalg.inv(wvt.transpose(0, 1).double()).to(torch.float32).contiguous()
    if K is not None:
        return c2w, torch.as_tensor(K).to(device=c2w.device, dtype=torch.float32).reshape(3, 3).contiguous()
    W, H = viewpoint_cam.image_width, viewpoint_cam.image_height
    fx = W / (2.0 * math.tan(viewpoint_cam.FoVx * 0.5))
    fy = H / (2.0 * math.tan(viewpoint_cam.FoVy * 0.5))
    K = torch.tensor([[fx, 0.0, W / 2.0], [0.0, fy, H / 2.0], [0.0, 0.0, 1.0]], dtype=torch.float32,
                     device=c2w.device)
    return c2w, K
