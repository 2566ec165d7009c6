"""LPIPS v0.1 with the VGG16 backbone on the device: what the reference's metrics.py:74 reports,
``lpips(renders[idx], gts[idx], net_type='vgg')`` of ``lpipsPyTorch``.

The network is the reference's: z-score with lpipsPyTorch's shift and scale, torchvision VGG16 ``features`` up to
relu5_3 (thirteen 3x3 convolutions, four 2x2 max-pools), channel-normalised taps after relu1_2, 2_2, 3_3, 4_3 and 5_3,
the v0.1 ``lin`` weights, layer means summed (and, for a batch, summed over the images).  The convolutions run as
implicit GEMMs on the tensor cores in 3xTF32 (s3g_lpips_vgg, csrc/lpips_vgg.cuh); the result is a float32 [1,1,1,1]
tensor on the inputs' device, computed without host synchronisation.

Forward only: nothing is kept for a backward, and an input that requires grad while grad is enabled is refused rather
than answered with a value that does not differentiate.  A call allocates its workspace, 2.52 GB for one 1920x1280
pair (s3g_lpips_vgg_workspace_bytes).

Weights are never downloaded.  By default they are read from the files the reference's run leaves in the torch hub
cache, ``torch.hub.get_dir()/checkpoints``: ``vgg16-397923af.pth`` (torchvision's VGG16 state dict; only the thirteen
``features.*`` convolutions are used) and ``vgg.pth`` (LPIPS v0.1 lin layers, ``lin{i}.model.1.weight``).

    from s3gaussian_b200.lpips_vgg import LPIPSVGG, lpips_vgg
    fn = LPIPSVGG()                  # once; weights prepared once per device
    d = fn(x, y)                     # x, y: [3,H,W] or [N,3,H,W] CUDA tensors, sides >= 16
    d = lpips_vgg(x, y)              # metrics.py:74
"""
from __future__ import annotations

import ctypes as C
import os

import torch

from . import _lib
from .lpips import _get, _load

VGG16_FILE = "vgg16-397923af.pth"
LIN_FILE = "vgg.pth"
FEATURE_INDICES = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)   # the convolutions of torchvision's vgg16().features
CONV_CHANNELS = ((3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 512), (512, 512),
                 (512, 512), (512, 512), (512, 512), (512, 512))      # (Cin, Cout), every kernel 3x3
CHANNELS = (64, 128, 256, 512, 512)                                   # the taps: relu1_2, 2_2, 3_3, 4_3, 5_3
MIN_SIDE = 16                               # below it the fourth max-pool has no output and torch raises


def default_paths() -> tuple[str, str]:
    """(VGG16 file, lin file) where the reference's torch.hub downloads leave them."""
    d = os.path.join(torch.hub.get_dir(), "checkpoints")
    return os.path.join(d, VGG16_FILE), os.path.join(d, LIN_FILE)


class LPIPSVGG:
    """LPIPSVGG(vgg16_path=None, lin_path=None): the reference's LPIPS('vgg', '0.1') criterion on the device, forward
    only.  Without paths the weight files come from default_paths().  Calling it with x, y ([3,H,W] or [N,3,H,W], same
    shape, one CUDA device) returns float32 [1,1,1,1]: the LPIPS distance, summed over the N pairs."""

    def __init__(self, vgg16_path: str | None = None, lin_path: str | None = None):
        dv, dl = default_paths()
        self._set_weights(_load(vgg16_path or dv), _load(lin_path or dl))

    @classmethod
    def from_state_dicts(cls, features_sd: dict, lin_sd: dict) -> "LPIPSVGG":
        """From a torchvision VGG16 state dict (``features.{0,2,...,28}.{weight,bias}``; other keys are ignored) and
        an LPIPS v0.1 lin state dict (``lin{i}.model.1.weight``, [1,C,1,1])."""
        self = cls.__new__(cls)
        self._set_weights(features_sd, lin_sd)
        return self

    def _set_weights(self, features_sd: dict, lin_sd: dict) -> None:
        convs = list(zip(FEATURE_INDICES, CONV_CHANNELS))
        self._conv_w = [_get(features_sd, f"features.{i}.weight", (co, ci, 3, 3)) for i, (ci, co) in convs]
        self._conv_b = [_get(features_sd, f"features.{i}.bias", (co,)) for i, (ci, co) in convs]
        self._lin = [_get(lin_sd, f"lin{i}.model.1.weight", (1, c, 1, 1)) for i, c in enumerate(CHANNELS)]
        self._prepared = {}                 # device -> the prepared buffer

    def _prepared_on(self, dev: torch.device) -> torch.Tensor:
        """The weights in the kernels' layout on `dev`, made once (pinned host copies, so no host synchronisation;
        the device copies of the weights go back to the allocator, which keeps them for this stream until the
        preparation queued on it has run)."""
        if dev not in self._prepared:
            lib = _lib.load()
            ws = [t.pin_memory().to(dev, non_blocking=True) for t in self._conv_w + self._conv_b + self._lin]
            buf = torch.empty(int(lib.s3g_lpips_vgg_prepared_bytes()), dtype=torch.uint8, device=dev)
            desc = _lib.LpipsVggWeights()
            for i in range(13):
                desc.conv_w[i] = ws[i].data_ptr()
                desc.conv_b[i] = ws[13 + i].data_ptr()
            for i in range(5):
                desc.lin_w[i] = ws[26 + i].data_ptr()
            _lib.check(lib.s3g_lpips_vgg_prepare(C.byref(desc), buf.data_ptr(),
                                                 C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                       "lpips_vgg_prepare")
            self._prepared[dev] = buf
        return self._prepared[dev]

    def terms(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        """DEVICE float64 [6]: the five layer terms (each summed over the N pairs), then their sum."""
        if x.dim() not in (3, 4) or tuple(x.shape) != tuple(y.shape):
            raise ValueError(f"x and y must both be [3,H,W] or [N,3,H,W], got {tuple(x.shape)} and {tuple(y.shape)}")
        N, Cn, H, W = (1, *x.shape) if x.dim() == 3 else tuple(x.shape)
        if Cn != 3:
            raise ValueError(f"LPIPS takes RGB images: 3 channels expected, got {Cn}")
        if H < MIN_SIDE or W < MIN_SIDE:
            raise ValueError(f"image sides must be >= {MIN_SIDE} for VGG16's fourth max-pool, got {H}x{W}")
        if N < 1:
            raise ValueError("x and y hold no images")
        if torch.is_grad_enabled() and (x.requires_grad or y.requires_grad):
            raise NotImplementedError("LPIPS with the VGG16 backbone is forward-only here: call it under "
                                      "torch.no_grad() or pass x.detach(), y.detach() (s3gaussian_b200.lpips, the "
                                      "AlexNet backbone, is differentiable)")
        if not x.is_cuda or y.device != x.device:
            raise RuntimeError("s3gaussian_b200 has no CPU path: x and y must be CUDA tensors on one device")
        lib = _lib.load()
        nbytes = int(lib.s3g_lpips_vgg_workspace_bytes(N, H, W))
        if nbytes == 0:
            raise ValueError(f"{N} images of {H}x{W} are too large for one VGG LPIPS call (32-bit indices)")
        dev = x.device
        with torch.cuda.device(dev):
            xf, yf = x.detach().float().contiguous(), y.detach().float().contiguous()
            prepared = self._prepared_on(dev)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            out = torch.empty(6, dtype=torch.float64, device=dev)
            _lib.check(lib.s3g_lpips_vgg(N, H, W, xf.data_ptr(), yf.data_ptr(), prepared.data_ptr(), out.data_ptr(),
                                         ws.data_ptr(), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                       "lpips_vgg")
        return out

    def __call__(self, x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        return self.terms(x, y)[5:].to(torch.float32).view(1, 1, 1, 1)


_cached: dict = {}


def lpips_vgg(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """lpipsPyTorch.lpips(x, y, net_type='vgg') from the default weight files, one LPIPSVGG per device kept for later
    calls (the reference builds and loads a new module per call)."""
    key = x.device
    if key not in _cached:
        _cached[key] = LPIPSVGG()
    return _cached[key](x, y)
