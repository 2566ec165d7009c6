"""float64 torch restatement of the rasterizer's lens projection (s3g_rasterize_forward_lens: the camera's intrinsics
and OpenCV radial-tangential distortion), written from the model in include/s3g_b200.h (test infrastructure).  It
extends aa_ref.project64: the same 3-D covariance, dilation and filter, with the mean and the covariance's Jacobian
taken through the lens."""
from __future__ import annotations

import math

import torch

from aa_ref import cov3d_matrix, filter64

NEAR = 0.2


def distort(lens, x, y):
    """(xd, yd, s) of normalised coordinates: the radial-tangential model."""
    fx, fy, cx, cy, k1, k2, p1, p2, k3 = lens
    s = x * x + y * y
    rho = 1 + k1 * s + k2 * s * s + k3 * s * s * s
    xd = x * rho + 2 * p1 * x * y + p2 * (s + 2 * x * x)
    yd = y * rho + p1 * (s + 2 * y * y) + 2 * p2 * x * y
    return xd, yd, s


def max_radius2(k1, k2, k3):
    """s*: the smallest positive real root of 1 + 3 k1 s + 5 k2 s^2 + 7 k3 s^3 (numpy.roots), or +inf."""
    import numpy as np
    c = [7 * k3, 5 * k2, 3 * k1, 1.0]
    while c and c[0] == 0:
        c = c[1:]
    if len(c) <= 1:
        return math.inf
    r = np.roots(c)
    pos = [z.real for z in r if abs(z.imag) <= 1e-12 * max(1.0, abs(z)) and z.real > 0]
    return min(pos) if pos else math.inf


def project64(d, leaf, lens, aa=False):
    """The lens preprocess of the Gaussians in leaf (float64 tensors: means3D, opacities, scales + rotations or cov3D,
    view; settings tensors stored transposed): -> dict of pix [n,2] (the rasterizer's pixel coordinates), ndc [n,2]
    (the units of dL_dmean2D), conic [n,3], depth [n], alpha_eff [n] (opacity * h when aa, else opacity), h [n] and
    visible [n] (near plane and lens cull).  Through the clamp of J_n the clamped component of the camera-space mean
    is a constant; D is taken at the unclamped point."""
    fx, fy, cx, cy, k1, k2, p1, p2, k3 = (float(v) for v in lens)
    W, H = d["W"], d["H"]
    p = leaf["means3D"]
    t = torch.cat([p, torch.ones_like(p[:, :1])], 1) @ leaf["view"]
    tz = t[:, 2]
    x, y = t[:, 0] / tz, t[:, 1] / tz
    xd, yd, s = distort((fx, fy, cx, cy, k1, k2, p1, p2, k3), x, y)
    pix = torch.stack([fx * xd + cx - 0.5, fy * yd + cy - 0.5], 1)
    ndc = torch.stack([(2 * pix[:, 0] + 1) / W - 1, (2 * pix[:, 1] + 1) / H - 1], 1)
    smax = max_radius2(k1, k2, k3)
    visible = (tz > NEAR) & (s <= smax)
    # D = d(xd, yd) / d(x, y), written out as the header states it
    rho = 1 + k1 * s + k2 * s * s + k3 * s * s * s
    drho = k1 + 2 * k2 * s + 3 * k3 * s * s
    D00 = rho + 2 * x * x * drho + 2 * p1 * y + 6 * p2 * x
    D01 = 2 * x * y * drho + 2 * p1 * x + 2 * p2 * y
    D11 = rho + 2 * y * y * drho + 6 * p1 * y + 2 * p2 * x
    xlo, xhi = -1.3 * cx / fx, 1.3 * (W - cx) / fx
    ylo, yhi = -1.3 * cy / fy, 1.3 * (H - cy) / fy
    inx, iny = (x >= xlo) & (x <= xhi), (y >= ylo) & (y <= yhi)
    tx = torch.where(inx, t[:, 0], (x.clamp(xlo, xhi) * tz).detach())
    ty = torch.where(iny, t[:, 1], (y.clamp(ylo, yhi) * tz).detach())
    zero = torch.zeros_like(tz)
    Jn = torch.stack([torch.stack([1 / tz, zero, -tx / tz ** 2], 1),
                      torch.stack([zero, 1 / tz, -ty / tz ** 2], 1)], 1)
    FD = torch.stack([torch.stack([fx * D00, fx * D01], 1), torch.stack([fy * D01, fy * D11], 1)], 1)
    T = FD @ Jn @ leaf["view"][:3, :3].T
    cov = T @ cov3d_matrix(leaf) @ T.transpose(1, 2)
    a, b, c = cov[:, 0, 0], cov[:, 0, 1], cov[:, 1, 1]
    op = leaf["opacities"].reshape(-1)
    conic, alpha_aa, h = filter64(a, b, c, op)
    return dict(pix=pix, ndc=ndc, conic=conic, depth=tz, alpha_eff=alpha_aa if aa else op, h=h, visible=visible,
                a=a, b=b, c=c, s=s)
