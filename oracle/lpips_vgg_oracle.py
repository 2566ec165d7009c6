"""LPIPS v0.1 with the VGG16 backbone (lpipsPyTorch/modules/{lpips,networks,utils}.py) restated in float64 with
torch.nn.functional, on any device: the checker of csrc/lpips_vgg.cuh.  Does not import torchvision.

  z = (x - shift) / scale                       networks.py:41-44,50-51 (the float32 buffers, widened)
  VGG16 features to relu5_3                     networks.py:53-63,88-96 (torchvision vgg16().features[:30])
  n = f / (sqrt(sum_c f^2) + 1e-10)             utils.py:6-8, after relu1_2, 2_2, 3_3, 4_3, 5_3
  d_l = mean_hw sum_c lin_l[c] (n_x - n_y)^2    lpips.py:30-34
  sum over layers and images                    lpips.py:36

Also the seeded weights every VGG test and benchmark uses, under the real files' key names.  Thirteen random ReLU
layers die or blow up easily, so the convolutions are He-scaled (variance 2 / fan_in keeps the second moment of the
activations from layer to layer) and every bias is a small positive number: about half of the activations are non-zero
at every tap (tests/test_lpips_vgg_host.py asserts the terms are far above the comparison tolerance).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .lpips_oracle import SCALE, SHIFT

# torchvision vgg16().features: the convolutions' indices, group by group; a 2x2 max-pool follows all but the last
GROUPS = ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21), (24, 26, 28))
CHANNELS = (64, 128, 256, 512, 512)
FEATURE_INDICES = tuple(i for g in GROUPS for i in g)
CONV_SHAPES = tuple((CHANNELS[g], 3 if (g, j) == (0, 0) else CHANNELS[g - (j == 0)], 3, 3)
                    for g, idx in enumerate(GROUPS) for j in range(len(idx)))


def random_state_dicts(seed: int = 0) -> tuple[dict, dict]:
    """(features_sd, lin_sd) with the key names of torchvision's VGG16 file and of LPIPS's vgg.pth, float32."""
    g = torch.Generator().manual_seed(seed)
    feat, lin = {}, {}
    for i, s in zip(FEATURE_INDICES, CONV_SHAPES):
        fan_in = s[1] * s[2] * s[3]
        feat[f"features.{i}.weight"] = torch.randn(s, generator=g) * (2.0 / fan_in) ** 0.5
        feat[f"features.{i}.bias"] = 0.02 + 0.02 * torch.rand(s[0], generator=g)
    for i, c in enumerate(CHANNELS):
        lin[f"lin{i}.model.1.weight"] = torch.rand((1, c, 1, 1), generator=g)
    return feat, lin


def features(x: torch.Tensor, features_sd: dict) -> list[torch.Tensor]:
    """The five normalised taps of [N,3,H,W] x, float64."""
    dev = x.device
    shift = torch.tensor(SHIFT, dtype=torch.float32).double().to(dev)[None, :, None, None]
    scale = torch.tensor(SCALE, dtype=torch.float32).double().to(dev)[None, :, None, None]
    h = (x.double() - shift) / scale
    taps = []
    for g, idx in enumerate(GROUPS):
        if g > 0:
            h = F.max_pool2d(h, 2, 2)
        for i in idx:
            w = features_sd[f"features.{i}.weight"].double().to(dev)
            b = features_sd[f"features.{i}.bias"].double().to(dev)
            h = F.relu(F.conv2d(h, w, b, padding=1))
        taps.append(h / (torch.sqrt(torch.sum(h ** 2, dim=1, keepdim=True)) + 1e-10))
    return taps


def lpips_terms(x: torch.Tensor, y: torch.Tensor, features_sd: dict, lin_sd: dict) -> torch.Tensor:
    """float64 [6]: each layer's term summed over the images, then the total (lpips(x, y, net_type='vgg') of the
    reference)."""
    if x.dim() == 3:
        x, y = x[None], y[None]
    terms = []
    for l, (fx, fy) in enumerate(zip(features(x, features_sd), features(y, features_sd))):
        w = lin_sd[f"lin{l}.model.1.weight"].double().to(x.device)
        terms.append(F.conv2d((fx - fy) ** 2, w).mean((2, 3)).sum())
    t = torch.stack(terms)
    return torch.cat([t, t.sum()[None]])
