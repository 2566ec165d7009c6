"""float64 torch restatement of the rasterizer's antialiasing filter (Mip-Splatting's 2-D filter) and of the preprocess
it is part of, written from the formulas in include/s3g_b200.h (test infrastructure)."""
from __future__ import annotations

import torch

DILATION = 0.3
RHO_MIN = 2.5e-5


def filter64(a, b, c, opacity):
    """(conic, alpha_eff, h) of EWA covariances {a, b, c} before the dilation: conic = the inverse of the dilated
    covariance as {x, y, z} (y = -b / det1, the one off-diagonal value), alpha_eff = opacity * h."""
    det0 = a * c - b * b
    ap, cp = a + DILATION, c + DILATION
    det1 = ap * cp - b * b
    h = torch.sqrt(torch.clamp(det0 / det1, min=RHO_MIN))
    conic = torch.stack([cp / det1, -b / det1, ap / det1], -1)
    return conic, opacity * h, h


def drho_closed_form(a, b, c):
    """d rho / d{a, b, c} as the header's chain rule states them."""
    det0 = a * c - b * b
    det1 = (a + DILATION) * (c + DILATION) - b * b
    d2 = det1 * det1
    return ((c * det1 - det0 * (c + DILATION)) / d2, -2 * b * (DILATION * (a + c) + DILATION * DILATION) / d2,
            (a * det1 - det0 * (a + DILATION)) / d2)


def cov3d_matrix(leaf):
    """[n,3,3] Sigma from leaf["cov3D"] ([n,6], upper triangle) or leaf["scales"] / leaf["rotations"] (the quaternion
    as given, not normalised, as the kernel reads it)."""
    if "cov3D" in leaf:
        c = leaf["cov3D"]
        return torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]],
                           1).view(-1, 3, 3)
    q = leaf["rotations"]
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
                     2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
                     2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1).view(-1, 3, 3)
    L = R * leaf["scales"][:, None, :]
    return L @ L.transpose(1, 2)


def project64(d, leaf):
    """The preprocess of the Gaussians in leaf (float64 tensors: means3D, opacities, scales + rotations or cov3D,
    view, proj; settings tensors stored transposed): -> dict of ndc [n,2] (mean2D before the pixel mapping), conic
    [n,3], depth [n], alpha_eff [n], h [n] and the EWA covariance a, b, c.  Through the 1.3 tanfov clamp the clamped
    component of the camera-space mean is a constant, the backward's convention."""
    x = leaf["means3D"]
    xt = torch.cat([x, torch.ones_like(x[:, :1])], 1)
    t = xt @ leaf["view"]
    p = xt @ leaf["proj"]
    ndc = p[:, :2] / (p[:, 3:4] + 1e-7)
    tz = t[:, 2]
    fx, fy = d["W"] / (2 * d["tanfovx"]), d["H"] / (2 * d["tanfovy"])
    limx, limy = 1.3 * d["tanfovx"], 1.3 * d["tanfovy"]
    rx, ry = t[:, 0] / tz, t[:, 1] / tz
    tx = torch.where(rx.abs() <= limx, t[:, 0], (rx.clamp(-limx, limx) * tz).detach())
    ty = torch.where(ry.abs() <= limy, t[:, 1], (ry.clamp(-limy, limy) * tz).detach())
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, zero, -fx * tx / tz ** 2], 1),
                     torch.stack([zero, fy / tz, -fy * ty / tz ** 2], 1)], 1)
    T = J @ leaf["view"][:3, :3].T
    cov = T @ cov3d_matrix(leaf) @ T.transpose(1, 2)
    a, b, c = cov[:, 0, 0], cov[:, 0, 1], cov[:, 1, 1]
    conic, alpha_eff, h = filter64(a, b, c, leaf["opacities"].reshape(-1))
    return dict(ndc=ndc, conic=conic, depth=tz, alpha_eff=alpha_eff, h=h, a=a, b=b, c=c)


def h_of(d, dev="cuda"):
    """h of every Gaussian of a scene dict (tests/util.scene_inputs), float64 [P] on dev."""
    leaf = {k: d[k].to(dev).double() for k in ("means3D", "opacities")}
    leaf.update({"cov3D": d["cov3D_precomp"].to(dev).double()} if d["cov3D_precomp"] is not None else
                {"scales": d["scales"].to(dev).double(), "rotations": d["rotations"].to(dev).double()})
    leaf["view"], leaf["proj"] = d["viewmatrix"].to(dev).double(), d["projmatrix"].to(dev).double()
    return torch.nan_to_num(project64(d, leaf)["h"], nan=1.0)   # NaN only at t.z = 0, culled by the near plane
