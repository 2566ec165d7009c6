"""LPIPS v0.1 with the AlexNet backbone (lpipsPyTorch/modules/{lpips,networks,utils}.py) restated in float64 with
torch.nn.functional, on any device: the checker of csrc/lpips.cuh.  Does not import torchvision.

  z = (x - shift) / scale                       networks.py:41-44,50-51 (the float32 buffers, widened)
  AlexNet features to the fifth ReLU            networks.py:53-63,77-83 (torchvision alexnet().features[:12])
  n = f / (sqrt(sum_c f^2) + 1e-10)             utils.py:6-8
  d_l = mean_hw sum_c lin_l[c] (n_x - n_y)^2    lpips.py:30-34
  sum over layers and images                    lpips.py:36

Also the seeded weights every test and benchmark uses: Kaiming-scaled convolutions, non-negative lin weights, under
the real files' key names.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

FEATURE_INDICES = (0, 3, 6, 8, 10)
CONV_SHAPES = ((64, 3, 11, 11), (192, 64, 5, 5), (384, 192, 3, 3), (256, 384, 3, 3), (256, 256, 3, 3))
CONV_ARGS = ((4, 2), (1, 2), (1, 1), (1, 1), (1, 1))       # (stride, padding)
SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)


def random_state_dicts(seed: int = 0) -> tuple[dict, dict]:
    """(features_sd, lin_sd) with the key names of torchvision's AlexNet file and of LPIPS's alex.pth, float32."""
    g = torch.Generator().manual_seed(seed)
    feat, lin = {}, {}
    for i, s in zip(FEATURE_INDICES, CONV_SHAPES):
        fan_in = s[1] * s[2] * s[3]
        feat[f"features.{i}.weight"] = torch.randn(s, generator=g) * (2.0 / fan_in) ** 0.5
        feat[f"features.{i}.bias"] = 0.05 * torch.randn(s[0], generator=g)
    for i, s in enumerate(CONV_SHAPES):
        lin[f"lin{i}.model.1.weight"] = torch.rand((1, s[0], 1, 1), generator=g)
    return feat, lin


def features(x: torch.Tensor, features_sd: dict) -> list[torch.Tensor]:
    """The five normalised taps of [N,3,H,W] x, float64."""
    dev = x.device
    shift = torch.tensor(SHIFT, dtype=torch.float32).double().to(dev)[None, :, None, None]
    scale = torch.tensor(SCALE, dtype=torch.float32).double().to(dev)[None, :, None, None]
    h = (x.double() - shift) / scale
    taps = []
    for l, (i, (stride, pad)) in enumerate(zip(FEATURE_INDICES, CONV_ARGS)):
        w = features_sd[f"features.{i}.weight"].double().to(dev)
        b = features_sd[f"features.{i}.bias"].double().to(dev)
        h = F.relu(F.conv2d(h, w, b, stride=stride, padding=pad))
        taps.append(h / (torch.sqrt(torch.sum(h ** 2, dim=1, keepdim=True)) + 1e-10))
        if l < 2:
            h = F.max_pool2d(h, 3, 2)
    return taps


def lpips_terms(x: torch.Tensor, y: torch.Tensor, features_sd: dict, lin_sd: dict) -> torch.Tensor:
    """float64 [6]: each layer's term summed over the images, then the total (lpips(x, y) of the reference)."""
    if x.dim() == 3:
        x, y = x[None], y[None]
    terms = []
    for l, (fx, fy) in enumerate(zip(features(x, features_sd), features(y, features_sd))):
        w = lin_sd[f"lin{l}.model.1.weight"].double().to(x.device)
        terms.append(F.conv2d((fx - fy) ** 2, w).mean((2, 3)).sum())
    t = torch.stack(terms)
    return torch.cat([t, t.sum()[None]])
