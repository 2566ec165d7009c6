"""Bilateral-grid colour correction: the fused slice and TV loss (s3gaussian_b200.bilateral_grid) against the torch
restatement of gsplat's formulas (tests/bilagrid_ref.py in float32: 5-D F.grid_sample, permute, batched 3x4 matmul;
total_variation_loss), which is what a user would otherwise paste into train.py.  Prints one JSON line.

(a) N = 150 grids of 16x16x8, one image of 960x640 (the reference's Waymo training size) and of 1920x1280:
    slice forward, slice forward + backward (grad_rgb and the grid gradient) and TV forward + backward, every arm
    alternating with the others in each round between CUDA events, after warm-up; the median of the rounds is
    reported.  Fused-against-torch parity is checked at the same sizes.  Bytes bounds from the shapes, not measured:
    the forward reads rgb and writes the output, 24 B per pixel; the backward reads rgb and grad_out and writes
    grad_rgb, 36 B per pixel (the grids, 0.1 MB each, are not counted).
(b) examples/train_loop.py (coarse) with and without --bilateral-grid, one subprocess per arm, alternating; each run
    reports its own time per iteration.
The card's name and power limit are read in the same run.

    python tools/bench_bilagrid.py [--calls 50] [--rounds 5] [--loop-rounds 2] [--loop-points 500000] [--loop-iters 300]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_raster_camera import card, time_arms   # noqa: E402

N, GRID = 150, (16, 16, 8)          # (GX, GY, L), gsplat's default
FWD_BYTES, BWD_BYTES = 24, 36       # per pixel


def image_arms(W, H, dev):
    import bilagrid_ref as ref
    from s3gaussian_b200.bilateral_grid import BilateralGrid
    GX, GY, L = GRID
    g = torch.Generator().manual_seed(0)
    bil = BilateralGrid(N, grid_X=GX, grid_Y=GY, grid_W=L).to(dev)
    with torch.no_grad():
        bil.grids.add_(0.1 * torch.randn(bil.grids.shape, generator=g).to(dev))
    rgb = (torch.rand(1, 3, H, W, generator=g) * 1.2 - 0.1).to(dev)
    go = torch.randn(1, 3, H, W, generator=g).to(dev)
    x = rgb.clone().requires_grad_(True)
    ids = [77]

    def fused_fwd():
        with torch.no_grad():
            return bil.slice(rgb, ids)

    def torch_fwd():
        with torch.no_grad():
            return ref.slice64(bil.grids, rgb, ids)

    def fused_fb():
        return torch.autograd.grad(bil.slice(x, ids), (x, bil.grids), go)

    def torch_fb():
        return torch.autograd.grad(ref.slice64(bil.grids, x, ids), (x, bil.grids), go)

    # parity at the timed size: fused against the float32 torch restatement, relative to each tensor's max
    parity = {}
    for name, a, b in (("forward", fused_fwd(), torch_fwd()),) + tuple(
            (n, u, v) for n, u, v in zip(("grad_rgb", "grad_grids"), fused_fb(), torch_fb())):
        parity[name] = float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)
    arms = {"fused_fwd": fused_fwd, "torch_fwd": torch_fwd, "fused_fwd_bwd": fused_fb, "torch_fwd_bwd": torch_fb}
    return arms, parity


def tv_arms(dev):
    import bilagrid_ref as ref
    from s3gaussian_b200.bilateral_grid import BilateralGrid
    GX, GY, L = GRID
    bil = BilateralGrid(N, grid_X=GX, grid_Y=GY, grid_W=L).to(dev)
    with torch.no_grad():
        bil.grids.add_(0.1 * torch.randn(bil.grids.shape, generator=torch.Generator().manual_seed(1)).to(dev))
    fused = lambda: torch.autograd.grad(10.0 * bil.tv_loss(), bil.grids)
    torch_ = lambda: torch.autograd.grad(10.0 * ref.tv64(bil.grids), bil.grids)
    (a,), (b,) = fused(), torch_()
    with torch.no_grad():
        lf, lt = float(bil.tv_loss()), float(ref.tv64(bil.grids))
    parity = {"tv_loss": abs(lf - lt) / lt,
              "tv_grad": float((a - b).abs().max()) / float(b.abs().max())}
    return {"fused_tv_fwd_bwd": fused, "torch_tv_fwd_bwd": torch_}, parity


def loop_runs(points, iters, rounds):
    arms = {"coarse": [], "coarse_bilateral_grid": []}
    for _ in range(rounds):
        for name in arms:
            cmd = [sys.executable, os.path.join(ROOT, "examples", "train_loop.py"), "--points", str(points), "--iters",
                   str(iters)] + (["--bilateral-grid"] if name.endswith("grid") else [])
            r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
            if r.returncode != 0:
                raise RuntimeError(r.stdout + r.stderr)
            arms[name].append(float(re.search(r"([\d.]+) ms per iteration", r.stdout).group(1)))
    return {k: {"ms_per_iter_median": float(np.median(v)), "ms_rounds": v} for k, v in arms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--loop-rounds", type=int, default=2)
    ap.add_argument("--loop-points", type=int, default=500_000)
    ap.add_argument("--loop-iters", type=int, default=300)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"card_before": card(), "grids": f"{N} x 16x16x8"}
    for W, H in ((960, 640), (1920, 1280)):
        arms, parity = image_arms(W, H, dev)
        t = time_arms(arms, a.calls, a.rounds)
        px = W * H
        res[f"{W}x{H}"] = {
            "ms": {k: v["ms_median"] for k, v in t.items()},
            "speedup_fwd": t["torch_fwd"]["ms_median"] / t["fused_fwd"]["ms_median"],
            "speedup_fwd_bwd": t["torch_fwd_bwd"]["ms_median"] / t["fused_fwd_bwd"]["ms_median"],
            "fwd_bound_MB": FWD_BYTES * px / 1e6, "bwd_bound_MB": BWD_BYTES * px / 1e6,
            "fused_fwd_GBps_of_bound": FWD_BYTES * px / (t["fused_fwd"]["ms_median"] * 1e6),
            "fused_fwd_bwd_GBps_of_bound": (FWD_BYTES + BWD_BYTES) * px / (t["fused_fwd_bwd"]["ms_median"] * 1e6),
            "parity_rel_to_max": parity}
        del arms
    arms, parity = tv_arms(dev)
    t = time_arms(arms, a.calls, a.rounds)
    res["tv"] = {"ms": {k: v["ms_median"] for k, v in t.items()}, "parity_rel": parity}
    torch.cuda.synchronize()
    if a.loop_rounds > 0:
        res["train_loop"] = dict(loop_runs(a.loop_points, a.loop_iters, a.loop_rounds), points=a.loop_points,
                                 iters=a.loop_iters, size="960x640")
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
