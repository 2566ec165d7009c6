"""LPIPS v0.1 with the AlexNet backbone on the device: drop-in for the reference's ``lpipsPyTorch`` (``lpips`` and
``LPIPS``), which utils/video_utils.py:221 calls once per evaluated view.

The network is the reference's: z-score with lpipsPyTorch's shift and scale, torchvision AlexNet ``features`` up to
the fifth ReLU, channel-normalised taps, the v0.1 ``lin`` weights, layer means summed (and, for a batch, summed over
the images).  The convolutions run as implicit GEMMs on the tensor cores in 3xTF32 (s3g_lpips_alex, csrc/lpips.cuh);
the result is a float32 [1,1,1,1] tensor on the inputs' device, computed without host synchronisation.

Like the reference's module, the result is differentiable with respect to x and y (the weights are frozen), so it can
be a training loss.  When grad is enabled and x or y requires grad, the call keeps the forward's activations (about
0.24 GB per 1920x1280 pair) until the backward, s3g_lpips_alex_backward: ReLU masks, max-pool argmaxes and taps from
those activations, the convolutions' input gradients as 3xTF32 implicit GEMMs on the tensor cores (conv 1's on the CUDA
cores).  Its weight layout is made on the first backward on a device.  Any other call keeps nothing.

Weights are never downloaded.  By default they are read from the files the reference's run leaves in the torch hub
cache, ``torch.hub.get_dir()/checkpoints``: ``alexnet-owt-7be5be79.pth`` (torchvision's AlexNet state dict; only
``features.{0,3,6,8,10}`` is used) and ``alex.pth`` (LPIPS v0.1 lin layers, ``lin{i}.model.1.weight``).

    from s3gaussian_b200.lpips import LPIPS, lpips
    fn = LPIPS()                     # once; weights prepared once per device
    d = fn(x, y)                     # x, y: [3,H,W] or [N,3,H,W] CUDA tensors, sides >= 31
    d = lpips(x, y, net_type='alex', version='0.1')
"""
from __future__ import annotations

import ctypes as C
import os

import torch
from torch.autograd.function import once_differentiable

from . import _lib

ALEXNET_FILE = "alexnet-owt-7be5be79.pth"
LIN_FILE = "alex.pth"
FEATURE_INDICES = (0, 3, 6, 8, 10)          # the convolutions of torchvision's alexnet().features
CONV_SHAPES = ((64, 3, 11, 11), (192, 64, 5, 5), (384, 192, 3, 3), (256, 384, 3, 3), (256, 256, 3, 3))
CHANNELS = tuple(s[0] for s in CONV_SHAPES)
MIN_SIDE = 31                               # below it the second max-pool has no output and torch raises


def default_paths() -> tuple[str, str]:
    """(AlexNet file, lin file) where the reference's torch.hub downloads leave them."""
    d = os.path.join(torch.hub.get_dir(), "checkpoints")
    return os.path.join(d, ALEXNET_FILE), os.path.join(d, LIN_FILE)


def _check_variant(net_type: str, version: str) -> None:
    # lpipsPyTorch/modules/lpips.py:19 asserts the version before get_network (networks.py:12-20) looks at the type
    assert version in ['0.1'], 'v0.1 is only supported now'
    if net_type != 'alex':
        raise NotImplementedError(f"net_type {net_type!r}: only 'alex' runs here ('vgg' is s3gaussian_b200.lpips_vgg, "
                                  f"forward only; 'squeeze' does not run on the device)")


def _load(path: str) -> dict:
    if not os.path.isfile(path):
        raise FileNotFoundError(f"LPIPS weight file not found: {path} (s3gaussian_b200 never downloads weights; "
                                f"put the file there or pass its path)")
    return torch.load(path, map_location="cpu", weights_only=True)


def _get(sd: dict, key: str, shape) -> torch.Tensor:
    """sd[key] as a contiguous float32 CPU tensor of `shape`."""
    if key not in sd:
        raise KeyError(f"LPIPS weights: missing {key!r}")
    t = torch.as_tensor(sd[key]).detach()
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"LPIPS weights: {key!r} has shape {tuple(t.shape)}, expected {tuple(shape)}")
    return t.to("cpu", torch.float32).contiguous()


class LPIPS:
    """LPIPS(net_type='alex', version='0.1', alexnet_path=None, lin_path=None): the reference's criterion on the
    device.  Without paths the weight files come from default_paths().  Calling it with x, y ([3,H,W] or [N,3,H,W],
    same shape, one CUDA device) returns float32 [1,1,1,1]: the LPIPS distance, summed over the N pairs."""

    def __init__(self, net_type: str = 'alex', version: str = '0.1', alexnet_path: str | None = None,
                 lin_path: str | None = None):
        _check_variant(net_type, version)
        da, dl = default_paths()
        features = _load(alexnet_path or da)
        lin = _load(lin_path or dl)
        self._set_weights(features, lin)

    @classmethod
    def from_state_dicts(cls, features_sd: dict, lin_sd: dict) -> "LPIPS":
        """From a torchvision AlexNet state dict (``features.{0,3,6,8,10}.{weight,bias}``; other keys are ignored)
        and an LPIPS v0.1 lin state dict (``lin{i}.model.1.weight``, [1,C,1,1])."""
        self = cls.__new__(cls)
        self._set_weights(features_sd, lin_sd)
        return self

    def _set_weights(self, features_sd: dict, lin_sd: dict) -> None:
        self._conv_w = [_get(features_sd, f"features.{i}.weight", s) for i, s in zip(FEATURE_INDICES, CONV_SHAPES)]
        self._conv_b = [_get(features_sd, f"features.{i}.bias", s[:1]) for i, s in zip(FEATURE_INDICES, CONV_SHAPES)]
        self._lin = [_get(lin_sd, f"lin{i}.model.1.weight", (1, c, 1, 1)) for i, c in enumerate(CHANNELS)]
        self._prepared = {}                 # device -> (prepared buffer, the device weights it was made from)
        self._prepared_bwd = {}             # device -> the backward's prepared buffer

    def _prepared_on(self, dev: torch.device) -> torch.Tensor:
        """The weights in the kernels' layout on `dev`, made once (pinned host copies, so no host synchronisation)."""
        if dev not in self._prepared:
            lib = _lib.load()
            ws = [t.pin_memory().to(dev, non_blocking=True) for t in self._conv_w + self._conv_b + self._lin]
            buf = torch.empty(int(lib.s3g_lpips_alex_prepared_bytes()), dtype=torch.uint8, device=dev)
            desc = _lib.LpipsAlexWeights()
            for i in range(5):
                desc.conv_w[i] = ws[i].data_ptr()
                desc.conv_b[i] = ws[5 + i].data_ptr()
                desc.lin_w[i] = ws[10 + i].data_ptr()
            _lib.check(lib.s3g_lpips_alex_prepare(C.byref(desc), buf.data_ptr(),
                                                  C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                       "lpips_alex_prepare")
            self._prepared[dev] = (buf, ws)
        return self._prepared[dev][0]

    def _prepared_bwd_on(self, dev: torch.device) -> torch.Tensor:
        """The backward's weight layout on `dev`, made the first time a backward runs there, from the device weight
        copies _prepared_on keeps (no host synchronisation)."""
        if dev not in self._prepared_bwd:
            lib = _lib.load()
            ws = self._prepared[dev][1]
            buf = torch.empty(int(lib.s3g_lpips_alex_backward_prepared_bytes()), dtype=torch.uint8, device=dev)
            desc = _lib.LpipsAlexWeights()
            for i in range(5):
                desc.conv_w[i] = ws[i].data_ptr()
                desc.conv_b[i] = ws[5 + i].data_ptr()
                desc.lin_w[i] = ws[10 + i].data_ptr()
            _lib.check(lib.s3g_lpips_alex_backward_prepare(C.byref(desc), buf.data_ptr(),
                                                           C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                       "lpips_alex_backward_prepare")
            self._prepared_bwd[dev] = buf
        return self._prepared_bwd[dev]

    def _run(self, N: int, H: int, W: int, xf: torch.Tensor, yf: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
        """(out [6], the workspace holding every activation) of one s3g_lpips_alex call on the current device."""
        lib = _lib.load()
        dev = xf.device
        prepared = self._prepared_on(dev)
        ws = torch.empty(int(lib.s3g_lpips_alex_workspace_bytes(N, H, W)), dtype=torch.uint8, device=dev)
        out = torch.empty(6, dtype=torch.float64, device=dev)
        _lib.check(lib.s3g_lpips_alex(N, H, W, xf.data_ptr(), yf.data_ptr(), prepared.data_ptr(), out.data_ptr(),
                                      ws.data_ptr(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                   "lpips_alex")
        return out, ws

    def terms(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        """DEVICE float64 [6]: the five layer terms (each summed over the N pairs), then their sum.  Differentiable
        with respect to x and y (not the frozen weights) when grad is enabled and either requires grad."""
        if x.dim() not in (3, 4) or tuple(x.shape) != tuple(y.shape):
            raise ValueError(f"x and y must both be [3,H,W] or [N,3,H,W], got {tuple(x.shape)} and {tuple(y.shape)}")
        N, Cn, H, W = (1, *x.shape) if x.dim() == 3 else tuple(x.shape)
        if Cn != 3:
            raise ValueError(f"LPIPS takes RGB images: 3 channels expected, got {Cn}")
        if H < MIN_SIDE or W < MIN_SIDE:
            raise ValueError(f"image sides must be >= {MIN_SIDE} for AlexNet's second max-pool, got {H}x{W}")
        if N < 1:
            raise ValueError("x and y hold no images")
        if not x.is_cuda or y.device != x.device:
            raise RuntimeError("s3gaussian_b200 has no CPU path: x and y must be CUDA tensors on one device")
        lib = _lib.load()
        nbytes = int(lib.s3g_lpips_alex_workspace_bytes(N, H, W))
        if nbytes == 0:
            raise ValueError(f"{N} images of {H}x{W} are too large for one LPIPS call (32-bit indices)")
        dev = x.device
        with torch.cuda.device(dev):
            xf, yf = x.float().contiguous(), y.float().contiguous()
            if torch.is_grad_enabled() and (xf.requires_grad or yf.requires_grad):
                return _LpipsAlexFunction.apply(xf, yf, self, (N, H, W))
            out, _ = self._run(N, H, W, xf, yf)
        return out

    def __call__(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        return self.terms(x, y)[5:].to(torch.float32).view(1, 1, 1, 1)


class _LpipsAlexFunction(torch.autograd.Function):
    """terms() with gradients for x and y: the forward keeps its workspace (every activation, about 0.24 GB per
    1920x1280 pair) until the backward, which reads it in s3g_lpips_alex_backward on the current stream."""

    @staticmethod
    def forward(ctx, xf, yf, fn, shape):
        out, ws = fn._run(*shape, xf, yf)
        ctx.save_for_backward(ws)
        ctx.fn, ctx.shape, ctx.in_shape = fn, shape, xf.shape
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        (ws,) = ctx.saved_tensors
        fn, (N, H, W) = ctx.fn, ctx.shape
        dev = ws.device
        lib = _lib.load()
        with torch.cuda.device(dev):
            prepared, prepared_bwd = fn._prepared_on(dev), fn._prepared_bwd_on(dev)
            # written as [N,3,H,W]; a [3,H,W] input gets a [3,H,W] gradient
            gx, gy = (torch.empty(ctx.in_shape, dtype=torch.float32, device=dev) if need else None
                      for need in ctx.needs_input_grad[:2])
            g = grad_out.to(dev, torch.float64).contiguous()
            work = torch.empty(int(lib.s3g_lpips_alex_backward_workspace_bytes(N, H, W)), dtype=torch.uint8,
                               device=dev)
            _lib.check(lib.s3g_lpips_alex_backward(N, H, W, prepared.data_ptr(), prepared_bwd.data_ptr(),
                                                   ws.data_ptr(), g.data_ptr(),
                                                   None if gx is None else gx.data_ptr(),
                                                   None if gy is None else gy.data_ptr(), work.data_ptr(),
                                                   C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                       "lpips_alex_backward")
        return gx, gy, None, None


_cached: dict = {}


def lpips(x: torch.Tensor, y: torch.Tensor, net_type: str = 'alex', version: str = '0.1') -> torch.Tensor:
    """Drop-in for lpipsPyTorch.lpips: the default weight files, one LPIPS per device kept for later calls (the
    reference builds and loads a new module per call)."""
    _check_variant(net_type, version)
    key = x.device
    if key not in _cached:
        _cached[key] = LPIPS(net_type, version)
    return _cached[key](x, y)
