"""Float64 torch restatement of Mip-Splatting's 3-D smoothing filter (include/s3g_b200.h, "3-D smoothing filter"):
compute_3D_filter over a camera set and get_scaling / get_opacity_with_3D_filter, plus the closed-form backward."""
import math

import torch

SQRT_VAR = math.sqrt(0.2)


def camera_space64(xyz, views):
    """[C,P,3] camera-space means: views [C,16] in the rasterizer's layout (m[k] = M[k%4][k/4])."""
    M = views.double().reshape(-1, 4, 4).transpose(1, 2)          # [C,4,4], M[c][row][col]
    X = xyz.double()
    return torch.einsum("crk,pk->cpr", M[:, :3, :3], X) + M[:, None, :3, 3]


def valid64(xyz, views, cams):
    """[C,P] bool: z > 0.2 and the projection within [-0.15, 1.15] of the image on both axes; and [C,P] z."""
    p = camera_space64(xyz, views)
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    w, h, fx, fy = (cams.double()[:, k:k + 1] for k in range(4))
    zc = z.clamp_min(1e-3)
    u = x / zc * fx + w / 2
    v = y / zc * fy + h / 2
    ok = (z > 0.2) & (u >= -0.15 * w) & (u <= 1.15 * w) & (v >= -0.15 * h) & (v <= 1.15 * h)
    return ok, z


def margin64(xyz, views, cams):
    """[P] smallest relative distance of any (camera, Gaussian) pair to one of the validity thresholds."""
    p = camera_space64(xyz, views)
    x, y, z = p[..., 0], p[..., 1], p[..., 2]
    w, h, fx, fy = (cams.double()[:, k:k + 1] for k in range(4))
    mz = (z - 0.2).abs() / 0.2
    zc = z.clamp_min(1e-3)
    mu = ((x / zc * fx).abs() - 0.65 * w).abs() / (0.65 * w)
    mv = ((y / zc * fy).abs() - 0.65 * h).abs() / (0.65 * h)
    screen = torch.minimum(mu, mv)
    # the screen test only matters where z > 0.2
    m = torch.where(z > 0.2, torch.minimum(mz, screen), mz)
    return m.min(0).values


def compute64(xyz, views, cams):
    """-> ([P] float64 filter, [P] bool seen by some camera)."""
    ok, z = valid64(xyz, views, cams)
    d = torch.where(ok, z, torch.full_like(z, math.inf)).min(0).values
    seen = ok.any(0)
    F = cams.double()[:, 2].max()
    fill = d[seen].max() if bool(seen.any()) else torch.zeros((), dtype=torch.float64, device=d.device)
    d = torch.where(seen, d, fill)
    return d / F * SQRT_VAR, seen


def apply64(scales, opacity, f):
    """(sqrt(s^2 + f^2), o sqrt(prod s^2 / prod s'^2)); f [P] or [P,1]."""
    f2 = f.reshape(-1, 1) ** 2
    s2 = scales * scales
    sf2 = s2 + f2
    return torch.sqrt(sf2), opacity * torch.sqrt(s2.prod(1, keepdim=True) / sf2.prod(1, keepdim=True))


def apply_backward64(scales, opacity, f, g_scales, g_opacity):
    """The closed form: dL/ds_k = g_s'_k s_k / s'_k + g_o' o' f^2 / (s_k s'_k^2), dL/do = g_o' sqrt(prod s^2 / prod s'^2)."""
    sf, of = apply64(scales, opacity, f)
    f2 = f.reshape(-1, 1) ** 2
    ds = g_scales * scales / sf + g_opacity * of * f2 / (scales * sf * sf)
    do = g_opacity * (of / opacity)
    return ds, do
