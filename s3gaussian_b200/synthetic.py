"""Synthetic workloads for tests and bench.py.

The reference ships no scene generator and there is no dataset here, so the
clouds and cameras are builder-defined, seeded, and frozen in this file.

Cameras follow the reference's conventions exactly (scene/cameras.py:53-64,
utils/graphics_utils.py:40-80): ``world_view_transform`` is W2C transposed,
``full_proj_transform`` = W2C^T @ P^T, ``camera_center`` is row 3 of the
inverse, znear = 0.01, zfar = 100, principal point at the image centre.

World frame is Waymo-like: x forward, y left, z up; camera frame is OpenCV
(x right, y down, z forward).
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

ZNEAR, ZFAR = 0.01, 100.0
WAYMO_FOCAL = 2055.0     # pixels at 1920 wide  ->  FoVx = 2 atan(1920 / (2*2055)) ~ 50.1 deg


def projection_matrix(znear, zfar, fovx, fovy) -> torch.Tensor:
    """utils/graphics_utils.py:54-74 (4x4, maps camera space to NDC with w = z)."""
    t, r = math.tan(fovy / 2) * znear, math.tan(fovx / 2) * znear
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (2 * r)
    P[1, 1] = 2.0 * znear / (2 * t)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


@dataclass
class SyntheticCamera:
    """The attributes gaussian_renderer.render() reads (gaussian_renderer/__init__.py:38-58)."""
    image_width: int
    image_height: int
    FoVx: float
    FoVy: float
    world_view_transform: torch.Tensor   # [4,4] = W2C^T
    full_proj_transform: torch.Tensor    # [4,4]
    camera_center: torch.Tensor          # [3]
    time: float = 0.0
    # optional, for render(pipe.lens): the 3x3 K (pixel centres at j + 0.5) and OpenCV k1, k2, p1, p2, k3
    intrinsic: torch.Tensor | None = None
    distortion: torch.Tensor | None = None

    def to(self, device):
        return SyntheticCamera(self.image_width, self.image_height, self.FoVx, self.FoVy,
                               self.world_view_transform.to(device),
                               self.full_proj_transform.to(device), self.camera_center.to(device),
                               self.time, self.intrinsic, self.distortion)

    @property
    def tanfovx(self):
        return math.tan(self.FoVx * 0.5)

    @property
    def tanfovy(self):
        return math.tan(self.FoVy * 0.5)


def make_camera(width, height, position, yaw_deg=0.0, pitch_deg=0.0, time=0.0,
                focal=None) -> SyntheticCamera:
    focal = WAYMO_FOCAL * width / 1920.0 if focal is None else focal
    fovx = 2 * math.atan(width / (2 * focal))
    fovy = 2 * math.atan(height / (2 * focal))
    yaw, pitch = math.radians(yaw_deg), math.radians(pitch_deg)
    fwd = np.array([math.cos(yaw) * math.cos(pitch), math.sin(yaw) * math.cos(pitch), math.sin(pitch)])
    right = np.array([math.sin(yaw), -math.cos(yaw), 0.0])
    down = np.cross(fwd, right)
    c2w_R = np.stack([right, down, fwd], axis=1)          # columns = camera axes in world
    w2c = np.eye(4)
    w2c[:3, :3] = c2w_R.T
    w2c[:3, 3] = -c2w_R.T @ np.asarray(position, dtype=np.float64)
    wvt = torch.tensor(np.float32(w2c)).transpose(0, 1).contiguous()
    proj = projection_matrix(ZNEAR, ZFAR, fovx, fovy).transpose(0, 1)
    full = (wvt.unsqueeze(0).bmm(proj.unsqueeze(0))).squeeze(0).contiguous()
    center = wvt.inverse()[3, :3].contiguous()
    return SyntheticCamera(width, height, fovx, fovy, wvt, full, center, float(time))


def waymo_ring(width=1920, height=1280, frames=50, cams_per_frame=3) -> list[SyntheticCamera]:
    """50 frames x 3 cameras (front, front-left, front-right; order [1,0,2] as
    scene/dataset_readers.py:619), ego moving +x at 1 m/frame, time = k/(frames-1)."""
    yaws = {0: 0.0, 1: 45.0, 2: -45.0}
    order = [1, 0, 2][:cams_per_frame]
    out = []
    for k in range(frames):
        for c in order:
            out.append(make_camera(width, height, (float(k), 0.0, 2.0), yaw_deg=yaws[c],
                                   time=k / max(frames - 1, 1)))
    return out


@dataclass
class GaussianCloud:
    """Raw (pre-activation) parameters, laid out like scene/gaussian_model.py:53-60."""
    xyz: torch.Tensor            # [P,3]
    features_dc: torch.Tensor    # [P,1,3]
    features_rest: torch.Tensor  # [P,15,3]
    scaling: torch.Tensor        # [P,3]  log-scale
    rotation: torch.Tensor       # [P,4]  un-normalised quaternion (r,x,y,z)
    opacity: torch.Tensor        # [P,1]  logit

    @property
    def P(self):
        return self.xyz.shape[0]

    def to(self, device):
        return GaussianCloud(*(t.to(device) for t in (self.xyz, self.features_dc, self.features_rest,
                                                      self.scaling, self.rotation, self.opacity)))

    def morton_sorted(self):
        """The same cloud with its rows permuted along a Morton curve of the positions (what
        GaussianModel.spatial_sort() does to a live model; host-side torch, data preparation only)."""
        xyz = self.xyz.detach().cpu()
        lo, hi = xyz.min(0).values, xyz.max(0).values
        q = ((xyz - lo) / (hi - lo).clamp_min(1e-12) * 1023.999).to(torch.int64).clamp_(0, 1023)

        def spread(v):
            v = (v | (v << 16)) & 0x030000FF
            v = (v | (v << 8)) & 0x0300F00F
            v = (v | (v << 4)) & 0x030C30C3
            return (v | (v << 2)) & 0x09249249
        key = spread(q[:, 0]) | (spread(q[:, 1]) << 1) | (spread(q[:, 2]) << 2)
        order = torch.argsort(key, stable=True).to(self.xyz.device)
        return GaussianCloud(*(t[order] for t in (self.xyz, self.features_dc, self.features_rest, self.scaling,
                                                  self.rotation, self.opacity)))

    # the reference's activations (scene/gaussian_model.py:39-47)
    def get_scaling(self):
        return torch.exp(self.scaling)

    def get_rotation(self):
        return torch.nn.functional.normalize(self.rotation)

    def get_opacity(self):
        return torch.sigmoid(self.opacity)

    def get_features(self):
        return torch.cat((self.features_dc, self.features_rest), dim=1)


# Frozen workload constants (tuned once so the front camera at 1920x1280 sees
# V/P ~ 0.7 and R/V ~ 5).
CLOUD_DEPTH_RANGE = (4.0, 80.0)     # metres in front of the frame-0 front camera
CLOUD_FRUSTUM_MARGIN = 1.12         # sample 12 % wider than the frustum so some Gaussians are culled
CLOUD_SCALE_MEDIAN = 0.035          # metres
CLOUD_SCALE_SIGMA = 0.6


def make_cloud(P: int, seed: int = 0, width=1920, height=1280) -> GaussianCloud:
    """Seeded cloud inside (a bit more than) the frame-0 front-camera frustum.

    Depth is drawn so that the density per unit depth grows linearly (between a
    uniform-in-depth and a uniform-in-volume fill), positions uniform across the
    widened frustum cross-section; a 10 % slice sits behind / beside the camera
    and is culled by the near plane or the tile-rect test.
    """
    g = torch.Generator().manual_seed(seed)
    focal = WAYMO_FOCAL * width / 1920.0
    tx, ty = width / (2 * focal), height / (2 * focal)
    z0, z1 = CLOUD_DEPTH_RANGE
    u = torch.rand(P, generator=g)
    z = torch.sqrt(z0 * z0 + u * (z1 * z1 - z0 * z0))          # pdf ~ z
    m = CLOUD_FRUSTUM_MARGIN
    cx = (torch.rand(P, generator=g) * 2 - 1) * tx * m * z     # camera right
    cy = (torch.rand(P, generator=g) * 2 - 1) * ty * m * z     # camera down
    behind = torch.rand(P, generator=g) < 0.10
    z = torch.where(behind, -z * 0.25, z)
    # camera (right, down, fwd) at (0,0,2) yaw 0 -> world (x fwd, y left, z up)
    xyz = torch.stack([z, -cx, 2.0 - cy], dim=1).float()
    s = torch.exp(math.log(CLOUD_SCALE_MEDIAN) + CLOUD_SCALE_SIGMA * torch.randn(P, 3, generator=g))
    scaling = torch.log(s).float()
    rotation = torch.randn(P, 4, generator=g).float()
    op = 0.05 + 0.9 * torch.rand(P, 1, generator=g)
    opacity = torch.log(op / (1 - op)).float()
    f_dc = torch.randn(P, 1, 3, generator=g).float()
    f_rest = (0.1 * torch.randn(P, 15, 3, generator=g)).float()
    return GaussianCloud(xyz, f_dc, f_rest, scaling, rotation, opacity)


def make_small_scene(P=256, width=64, height=48, seed=1):
    """A tiny scene for CPU-checkable tests: one camera looking down +x at a blob."""
    g = torch.Generator().manual_seed(seed)
    cam = make_camera(width, height, (0.0, 0.0, 0.0), focal=0.9 * width)
    xyz = torch.stack([2.0 + 6.0 * torch.rand(P, generator=g),
                       (torch.rand(P, generator=g) * 2 - 1) * 3.0,
                       (torch.rand(P, generator=g) * 2 - 1) * 2.0], dim=1).float()
    xyz[: max(P // 16, 1), 0] = -1.0 - torch.rand(max(P // 16, 1), generator=g)   # some behind
    s = torch.exp(math.log(0.12) + 0.5 * torch.randn(P, 3, generator=g))
    op = 0.05 + 0.9 * torch.rand(P, 1, generator=g)
    cloud = GaussianCloud(xyz, torch.randn(P, 1, 3, generator=g).float(),
                          (0.2 * torch.randn(P, 15, 3, generator=g)).float(), torch.log(s).float(),
                          torch.randn(P, 4, generator=g).float(), torch.log(op / (1 - op)).float())
    return cloud, cam


# ---------------------------------------------------------------------------
# HexPlane + decoder parameters (reference state_dict names, scene/deformation.py,
# scene/hexplane.py:48-70).  Seeded and frozen like the clouds.
# ---------------------------------------------------------------------------
DEFAULT_RESOLUTION = (64, 64, 64, 25)       # arguments/__init__.py:218-223
DEFAULT_MULTIRES = (1, 2, 4, 8)
PLANE_COMBS = ((0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3))
WAYMO_AABB = ((80.0, 40.0, 15.0), (-20.0, -40.0, -5.0))   # set_aabb(xyz_max, xyz_min), scene/__init__.py:150-151


def make_deform_state(seed=0, resolution=DEFAULT_RESOLUTION, multires=DEFAULT_MULTIRES, width=64, feat_dim=32,
                      aabb=WAYMO_AABB, all_heads=True, weight_scale=1.0):
    """state_dict of the reference's deform_network (the keys the hot path reads).

    Spatial planes ~ U(0.1,0.5), time planes near 1 with a small perturbation (so the
    time coordinate matters), Linear layers Xavier-like; `weight_scale` shrinks the last
    layers so the synthetic deformations stay realistic (cm-scale)."""
    g = torch.Generator().manual_seed(seed)
    st = {"deformation_net.grid.aabb": torch.tensor(aabb, dtype=torch.float32)}
    for li, m in enumerate(multires):
        reso = [r * m for r in resolution[:3]] + [resolution[3]]
        for ci, (a, b) in enumerate(PLANE_COMBS):
            shape = (1, feat_dim, reso[b], reso[a])
            if 3 in (a, b):
                pl = 1.0 + 0.1 * (torch.rand(shape, generator=g) - 0.5)
            else:
                pl = 0.1 + 0.4 * torch.rand(shape, generator=g)
            st[f"deformation_net.grid.grids.{li}.{ci}"] = pl.float()

    def lin(name, fan_out, fan_in, scale=1.0):
        bound = scale * math.sqrt(6.0 / (fan_in + fan_out))
        st[name + ".weight"] = ((torch.rand(fan_out, fan_in, generator=g) * 2 - 1) * bound).float()
        st[name + ".bias"] = ((torch.rand(fan_out, generator=g) * 2 - 1) / math.sqrt(fan_in) * scale).float()

    D = feat_dim * len(multires)
    lin("deformation_net.feature_out.0", width, D)
    heads = [("pos_deform", 3), ("shs_deform", 48)]
    if all_heads:
        heads += [("scales_deform", 3), ("rotations_deform", 4), ("opacity_deform", 1)]
    for name, k in heads:
        lin(f"deformation_net.{name}.1", width, width)
        lin(f"deformation_net.{name}.3", k, width, weight_scale)
    lin("deformation_net.dino_head.0", width, width)
    lin("deformation_net.dino_head.2", width, width)
    lin("deformation_net.dino_head.4", 3, width, weight_scale)
    return st
