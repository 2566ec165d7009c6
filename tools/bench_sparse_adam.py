"""Selective Adam: (a) the optimizer step alone, dense FusedAdam.step() against step(visibility=mask), (b) the training
loop with and without --sparse-adam.  Prints one JSON line.

(a) 2 M Gaussians (make_cloud(2_000_000)), SH degree 3, the six per-Gaussian groups only (59 floats per Gaussian).
    The model is Morton-sorted (spatial_sort, as the training loop keeps it).  Masks:
      * radii > 0 of every camera of waymo_ring(1920, 1280, frames=50), rendered from the sorted model (each visible
        fraction is printed); timed as one arm that steps through all 150 masks in turn;
      * fixed fractions 1 %, 10 %, 50 %, 100 %: the rows nearest one point in space, which a Morton-ordered model
        holds in a few long runs;
      * each of these with its rows shuffled (the same count, scattered as in a model that is not sorted).
    Every arm alternates with the others in each round between CUDA events, after warm-up; the median of the rounds
    is reported.  Bytes model: 28 B per updated element (read p, g, m, v; write p, m, v) plus 1 B of mask per row.
(b) examples/train_loop.py --points 2000000, coarse and --fine, as a subprocess per arm, alternating; each run reports
    its own time per iteration (events over iterations 11..--iters) and its last logged loss.
The card's name and power limit are read in the same run, before and after.

    python tools/bench_sparse_adam.py [--calls 20] [--rounds 5] [--loop-rounds 3] [--loop-points 2000000]
                                      [--loop-iters 300]
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

from bench_raster_camera import card, time_arms   # noqa: E402

ROW_FLOATS = 59          # xyz 3, f_dc 3, f_rest 45, opacity 1, scaling 3, rotation 4


def step_bytes(n_rows_updated, P, masked):
    return 28 * ROW_FLOATS * n_rows_updated + (P if masked else 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--loop-rounds", type=int, default=3)
    ap.add_argument("--loop-points", type=int, default=2_000_000)
    ap.add_argument("--loop-iters", type=int, default=300)
    ap.add_argument("--skip-loop", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is no CPU path")
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_model import GaussianModel, default_optimization_params
    from s3gaussian_b200.gaussian_renderer import PipelineParams, render
    dev = torch.device("cuda:0")
    result = {"card": card()}
    P = 2_000_000

    # (a) the step alone
    cloud = syn.make_cloud(P, seed=0)
    g = GaussianModel(3).create_from_tensors(*(t.to(dev) for t in (cloud.xyz, cloud.features_dc, cloud.features_rest,
                                                                  cloud.scaling, cloud.rotation, cloud.opacity)))
    g.active_sh_degree = 3
    g.training_setup(default_optimization_params())
    g.spatial_sort()
    gen = torch.Generator(dev).manual_seed(1)
    params = [p for grp in g.optimizer.param_groups for p in grp["params"]]
    assert sum(p[0].numel() for p in params) == ROW_FLOATS
    for p in params:
        p.grad = torch.randn(p.shape, device=dev, generator=gen) * 0.01
    g.optimizer.step()          # creates the moments
    with torch.no_grad():
        cams = [c.to(dev) for c in syn.waymo_ring(1920, 1280, frames=50)]
        cam_masks = [(render(c, g, PipelineParams(), torch.zeros(3, device=dev), stage="coarse")["radii"] > 0)
                     for c in cams]
    fractions = [float(m.float().mean()) for m in cam_masks]
    perm = torch.randperm(P, device=dev, generator=gen)
    xyz = g.get_xyz.detach()
    centre = xyz[int(torch.randint(P, (1,), device=dev, generator=gen))]
    order = torch.argsort(((xyz - centre) ** 2).sum(1))
    fixed = {}
    for f in (0.01, 0.10, 0.50, 1.00):
        m = torch.zeros(P, dtype=torch.bool, device=dev)
        m[order[:int(round(f * P))]] = True
        fixed[f"{int(f * 100)}pct_morton"] = m
        fixed[f"{int(f * 100)}pct_shuffled"] = m[perm].contiguous()
    runs = {k: int(((m[1:] != m[:-1]).sum() + 1) // 2) for k, m in fixed.items()}
    cams_shuffled = [m[perm].contiguous() for m in cam_masks]
    opt = g.optimizer

    def cycle(masks):
        it = [0]

        def fn():
            opt.step(visibility=masks[it[0] % len(masks)])
            it[0] += 1
        return fn
    arms = {"dense": lambda: opt.step()}
    arms.update({k: (lambda m=m: opt.step(visibility=m)) for k, m in fixed.items()})
    arms["cameras_morton"] = cycle(cam_masks)
    arms["cameras_shuffled"] = cycle(cams_shuffled)
    # time_arms takes one call count; the camera arms cycle through all 150 masks per round
    r = time_arms({k: v for k, v in arms.items() if not k.startswith("cameras")}, a.calls, a.rounds)
    r.update(time_arms({k: v for k, v in arms.items() if k.startswith("cameras")}, len(cam_masks), a.rounds))
    vis_mean = float(np.mean(fractions))
    for k, v in r.items():
        if k == "dense":
            n = P
        elif k.startswith("cameras"):
            n = vis_mean * P
        else:
            n = int(fixed[k].sum())
        v["rows_updated"] = n
        v["TB_per_s"] = step_bytes(n, P, k != "dense") / (v["ms_median"] * 1e9)
        v["over_dense"] = v["ms_median"] / r["dense"]["ms_median"] if k != "dense" else 1.0
    result["step"] = r
    result["step_P"] = P
    result["visible_runs_of_fixed_masks"] = runs
    result["camera_visible_fraction"] = {"min": min(fractions), "median": float(np.median(fractions)),
                                         "mean": vis_mean, "max": max(fractions),
                                         "per_camera": [round(f, 4) for f in fractions]}
    del g, opt, params, cam_masks, cams_shuffled, fixed, arms
    torch.cuda.empty_cache()

    # (b) the training loop
    if not a.skip_loop:
        base = [sys.executable, os.path.join(ROOT, "examples", "train_loop.py"), "--points", str(a.loop_points),
                "--iters", str(a.loop_iters)]
        loop_arms = {"coarse_dense": base, "coarse_sparse": base + ["--sparse-adam"],
                     "fine_dense": base + ["--fine"], "fine_sparse": base + ["--fine", "--sparse-adam"]}
        res = {k: [] for k in loop_arms}
        loss = {k: [] for k in loop_arms}
        for _ in range(a.loop_rounds):
            for name, c in loop_arms.items():
                out = subprocess.run(c, capture_output=True, text=True)
                if out.returncode != 0:
                    raise RuntimeError(f"{name}: {out.stdout}{out.stderr}")
                res[name].append(float(re.search(r"([\d.]+) ms per iteration", out.stdout).group(1)))
                loss[name].append(float(re.findall(r"iter\s+\d+\s+loss ([\d.]+)", out.stdout)[-1]))
        result["train_loop"] = {k: {"ms_per_iter_median": float(np.median(v)), "ms_rounds": v,
                                    "spread": (max(v) - min(v)) / float(np.median(v)), "final_loss": loss[k]}
                                for k, v in res.items()}
        result["train_loop"]["iters"] = a.loop_iters
        result["train_loop"]["points"] = a.loop_points
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
