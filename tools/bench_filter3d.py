"""3-D smoothing filter: (a) s3g_filter3d_compute against a torch per-camera loop that restates Mip-Splatting's
compute_3D_filter, (b) the apply kernels forward and backward, (c) coarse render() forward and forward + backward with
pipe.filter_3d off and on.  Prints one JSON line.

Shapes: 2 M Gaussians (make_cloud(2_000_000)), the 150 cameras of waymo_ring(1920, 1280, frames=50) as the training
set, and bench.py's camera waymo_ring[1] for render().  After warm-up the arms of each group alternate in rounds; each
round times --calls calls of one arm between two CUDA events (the torch loop gets --calls-loop, it is ~100x slower).
The card's name and power limit are read in the same run.  The compute kernel does P x C = 3e8 point-camera tests;
the apply forward reads 20 and writes 16 bytes per Gaussian, the backward reads 36 and writes 16.

    python tools/bench_filter3d.py [--calls 20] [--calls-loop 2] [--rounds 5]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_raster_camera import card, time_arms   # noqa: E402


def mip_splatting_loop(xyz, cameras):
    """Mip-Splatting's GaussianModel.compute_3D_filter in torch (float32, boolean indexing as upstream)."""
    distance = torch.ones((xyz.shape[0]), device=xyz.device) * 100000.0
    valid_points = torch.zeros((xyz.shape[0]), device=xyz.device, dtype=torch.bool)
    focal_length = 0.0
    for cam in cameras:
        W2C = cam.world_view_transform.t()
        xyz_cam = xyz @ W2C[:3, :3].t() + W2C[:3, 3][None, :]
        valid_depth = xyz_cam[:, 2] > 0.2
        x, y, z = xyz_cam[:, 0], xyz_cam[:, 1], xyz_cam[:, 2]
        z = torch.clamp(z, min=0.001)
        fx = cam.image_width / (2 * math.tan(cam.FoVx / 2))
        fy = cam.image_height / (2 * math.tan(cam.FoVy / 2))
        x = x / z * fx + cam.image_width / 2.0
        y = y / z * fy + cam.image_height / 2.0
        in_screen = torch.logical_and(torch.logical_and(x >= -0.15 * cam.image_width, x <= cam.image_width * 1.15),
                                      torch.logical_and(y >= -0.15 * cam.image_height, y <= 1.15 * cam.image_height))
        valid = torch.logical_and(valid_depth, in_screen)
        distance[valid] = torch.min(distance[valid], z[valid])
        valid_points = torch.logical_or(valid_points, valid)
        focal_length = max(focal_length, fx)
    distance[~valid_points] = distance[valid_points].max()
    return (distance / focal_length * (0.2 ** 0.5))[..., None]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--calls-loop", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is no CPU path")
    from s3gaussian_b200 import _lib, filter3d, synthetic as syn
    from s3gaussian_b200.gaussian_renderer import GaussianModelLite, PipelineParams, render
    dev = torch.device("cuda:0")
    lib = _lib.load()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    result = {"card": card()}
    P = 2_000_000
    cloud = syn.make_cloud(P, seed=0).to(dev)
    cams = [c.to(dev) for c in syn.waymo_ring(1920, 1280, frames=50)]

    # (a) compute
    xyz = cloud.xyz.contiguous()
    views, k = filter3d.camera_tensors(cams, dev)
    out = torch.empty(P, device=dev)
    ws = torch.empty(lib.s3g_filter3d_compute_workspace_bytes(P), dtype=torch.uint8, device=dev)
    kernel = lambda: _lib.check(lib.s3g_filter3d_compute(P, xyz.data_ptr(), len(cams), views.data_ptr(), k.data_ptr(),
                                                         out.data_ptr(), ws.data_ptr(), stream), "compute")
    kernel()
    loop = mip_splatting_loop(xyz, cams)[:, 0]
    # the float64 restatement, 2e5 Gaussians at a time (its [C, P] temporaries)
    import filter3d_ref
    d, seen, margin = [], [], []
    for i in range(0, P, 200_000):
        ok, z = filter3d_ref.valid64(xyz[i:i + 200_000], views, k)
        d.append(torch.where(ok, z, torch.full_like(z, math.inf)).min(0).values)
        seen.append(ok.any(0))
        margin.append(filter3d_ref.margin64(xyz[i:i + 200_000], views, k))
    d, seen, margin = torch.cat(d), torch.cat(seen), torch.cat(margin)
    want = torch.where(seen, d, d[seen].max()) / k[:, 2].double().max() * math.sqrt(0.2)
    del d
    torch.cuda.synchronize()
    rel = lambda a, b: ((a.double() - b.double()).abs() / b.double().abs())
    r = {"P": P, "C": len(cams), "tests": P * len(cams),
         "max_rel_diff_vs_float64": float(rel(out, want).max()),
         "max_rel_diff_vs_float64_margin_gt_1e-4": float(rel(out, want)[margin > 1e-4].max()),
         "max_rel_diff_vs_loop": float(rel(out, loop).max()),
         "frac_diff_vs_loop_gt_1e-5": float((rel(out, loop) > 1e-5).double().mean()),
         "max_rel_diff_loop_vs_float64": float(rel(loop, want).max()),
         **time_arms({"kernel": kernel}, a.calls, a.rounds),
         **time_arms({"torch_loop": lambda: mip_splatting_loop(xyz, cams)}, a.calls_loop, a.rounds)}
    r["loop_over_kernel"] = r["torch_loop"]["ms_median"] / r["kernel"]["ms_median"]
    r["tests_per_ns"] = P * len(cams) / (r["kernel"]["ms_median"] * 1e6)
    result["compute"] = r

    # (b) apply
    filt = out[:, None].contiguous()
    s, o = cloud.get_scaling().contiguous(), cloud.get_opacity().contiguous()
    e = lambda t: torch.empty_like(t)
    so, oo, gs, go, ds, do = e(s), e(o), torch.randn_like(s), torch.randn_like(o), e(s), e(o)
    arms = {
        "forward": lambda: _lib.check(lib.s3g_filter3d_apply_forward(P, s.data_ptr(), o.data_ptr(), filt.data_ptr(),
                                                                     so.data_ptr(), oo.data_ptr(), stream), "fwd"),
        "backward": lambda: _lib.check(lib.s3g_filter3d_apply_backward(
            P, s.data_ptr(), o.data_ptr(), filt.data_ptr(), gs.data_ptr(), go.data_ptr(), ds.data_ptr(), do.data_ptr(),
            stream), "bwd"),
    }
    r = time_arms(arms, a.calls, a.rounds)
    for name, nbytes in (("forward", 36 * P), ("backward", 52 * P)):
        r[name]["GB_per_s"] = nbytes / (r[name]["ms_median"] * 1e6)
    result["apply"] = r

    # (c) coarse render() at the bench.py headline camera
    pc = GaussianModelLite(cloud, sh_degree=3).to(dev)
    pc.filter_3D = filt
    cam = cams[1]
    bg = torch.zeros(3, device=dev)
    off, on = PipelineParams(), PipelineParams()
    on.filter_3d = True
    gimg = torch.randn(3, 1280, 1920, device=dev)

    def fwd(pipe):
        with torch.no_grad():
            render(cam, pc, pipe, bg, stage="coarse")

    def fwd_bwd(pipe):
        img = render(cam, pc, pipe, bg, stage="coarse")["render"]
        (img * gimg).sum().backward()
        for p in pc.parameters():
            p.grad = None
    r = time_arms({"forward_off": lambda: fwd(off), "forward_on": lambda: fwd(on),
                   "forward_backward_off": lambda: fwd_bwd(off), "forward_backward_on": lambda: fwd_bwd(on)},
                  a.calls, a.rounds)
    with torch.no_grad():
        r["visible_off"] = int((render(cam, pc, off, bg, stage="coarse")["radii"] > 0).sum())
        r["visible_on"] = int((render(cam, pc, on, bg, stage="coarse")["radii"] > 0).sum())
    result["render_coarse"] = r
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
