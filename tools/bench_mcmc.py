"""3DGS-MCMC densification: (a) s3g_mcmc_noise against a torch restatement of 3DGS-MCMC's noise block, (b) one
relocate_gs + add_new_gs on a trained-state model with about 5 % dead rows, (c) the coarse examples/train_loop.py
iteration with and without --mcmc-cap.  Prints one JSON line.

Shapes: 2 M Gaussians (make_cloud(2_000_000)).  (a) and (b) alternate their arms in rounds between CUDA events after
warm-up; (b) rebuilds the model from the same state before every timed call (outside the events), since each call
changes it.  (c) runs the loop as a subprocess per arm, alternating, and reads its own per-iteration time (events over
iterations 11..--iters).  The noise kernel moves 68 bytes per Gaussian (reads xyz 12, scaling 12, rotation 16, opacity
4, eps 12; writes xyz 12).  The card's name and power limit are read in the same run.

    python tools/bench_mcmc.py [--calls 20] [--rounds 5] [--loop-rounds 2] [--loop-points 2000000] [--loop-iters 300]
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

NOISE_BYTES = 68


def torch_noise(xyz, scaling, rotation, opacity, step, eps):
    """3DGS-MCMC's noise block in torch (its train.py: build_scaling_rotation, L L^T, op_sigmoid, bmm), eps given."""
    from s3gaussian_b200.gaussian_model import build_rotation
    R = build_rotation(torch.nn.functional.normalize(rotation))
    L = R * torch.exp(scaling)[:, None, :]
    cov = L @ L.transpose(1, 2)
    gate = 1 / (1 + torch.exp(-100 * ((1 - torch.sigmoid(opacity)) - 0.995)))
    noise = eps * gate * step
    xyz.add_(torch.bmm(cov, noise.unsqueeze(-1)).squeeze(-1))


def model_state(P, dev):
    """Raw parameters and Adam moments of a 2 M model after two FusedAdam steps, ~5 % of rows at opacity 0.003."""
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_model import GaussianModel, default_optimization_params
    cloud = syn.make_cloud(P, seed=0)
    g = GaussianModel(3).create_from_tensors(*(t.to(dev) for t in (cloud.xyz, cloud.features_dc, cloud.features_rest,
                                                                  cloud.scaling, cloud.rotation, cloud.opacity)))
    g.training_setup(default_optimization_params())
    gen = torch.Generator(dev).manual_seed(1)
    for _ in range(2):
        for name in ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"):
            p = getattr(g, name)
            p.grad = torch.randn(p.shape, device=dev, generator=gen) * 0.1
        g.optimizer.step()
        g.optimizer.zero_grad(set_to_none=True)
    dead = torch.rand(P, device=dev, generator=gen) < 0.05
    g._opacity.data[dead] = float(np.log(0.003 / 0.997))
    return g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--loop-rounds", type=int, default=2)
    ap.add_argument("--loop-points", type=int, default=2_000_000)
    ap.add_argument("--loop-iters", type=int, default=300)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is no CPU path")
    from s3gaussian_b200 import mcmc, synthetic as syn
    dev = torch.device("cuda:0")
    result = {"card": card()}
    P = 2_000_000

    # (a) noise
    cloud = syn.make_cloud(P, seed=0).to(dev)
    xyz0 = cloud.xyz.contiguous()
    sc, rot = cloud.scaling.contiguous(), cloud.rotation.contiguous()
    op = (cloud.opacity - 5.0).contiguous()            # o in ~(0.0003, 0.1): the gate's whole range is exercised
    eps = torch.randn(P, 3, device=dev, generator=torch.Generator(dev).manual_seed(2))
    step = 1.6e-4 * 5e5
    x_k, x_t = xyz0.clone(), xyz0.clone()
    mcmc.inject_noise(x_k, sc, rot, op, step, eps)
    torch_noise(x_t, sc, rot, op, step, eps)
    d_k, d_t = (x_k - xyz0).double(), (x_t - xyz0).double()
    r = time_arms({"kernel": lambda: mcmc.inject_noise(x_k, sc, rot, op, step, eps),
                   "torch": lambda: torch_noise(x_t, sc, rot, op, step, eps)}, a.calls, a.rounds)
    r["kernel"]["GB_per_s"] = NOISE_BYTES * P / (r["kernel"]["ms_median"] * 1e6)
    r["torch_over_kernel"] = r["torch"]["ms_median"] / r["kernel"]["ms_median"]
    r["max_abs_diff_of_displacement_vs_torch"] = float((d_k - d_t).abs().max())
    r["max_abs_displacement"] = float(d_t.abs().max())
    r["P"] = P
    result["noise"] = r
    del x_k, x_t, cloud

    # (b) relocate + add
    base = model_state(P, dev)
    n_dead = int((base.get_opacity <= 0.005).sum())
    saved = {k: getattr(base, k).detach().clone() for k in ("_xyz", "_features_dc", "_features_rest", "_opacity",
                                                            "_scaling", "_rotation")}
    saved_state = {k: base.optimizer.state[getattr(base, k)] for k in saved}
    from s3gaussian_b200.gaussian_model import GaussianModel, default_optimization_params

    def fresh():
        g = GaussianModel(3).create_from_tensors(*(saved[k] for k in ("_xyz", "_features_dc", "_features_rest",
                                                                      "_scaling", "_rotation", "_opacity")))
        g.training_setup(default_optimization_params())
        for k in saved:
            st = saved_state[k]
            g.optimizer.state[getattr(g, k)] = {"step": st["step"].clone(), "exp_avg": st["exp_avg"].clone(),
                                                "exp_avg_sq": st["exp_avg_sq"].clone()}
        return g

    arms = {"relocate": lambda g: g.relocate_gs(), "add": lambda g: g.add_new_gs(2 * P),
            "relocate_add": lambda g: (g.relocate_gs(), g.add_new_gs(2 * P))}
    times = {k: [] for k in arms}
    for rnd in range(a.rounds + 1):          # round 0 is warm-up
        for name, fn in arms.items():
            g = fresh()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn(g)
            e1.record()
            torch.cuda.synchronize()
            if rnd:
                times[name].append(e0.elapsed_time(e1))
            del g
    result["relocate_add"] = {k: {"ms_median": float(np.median(v)), "ms_min": float(np.min(v)), "ms_rounds": v}
                              for k, v in times.items()}
    result["relocate_add"].update(P=P, n_dead=n_dead, n_added=int(1.05 * P) - P)
    del base

    # (c) the coarse training loop, with and without --mcmc-cap
    cmd = [sys.executable, os.path.join(ROOT, "examples", "train_loop.py"), "--points", str(a.loop_points),
           "--iters", str(a.loop_iters)]
    loop_arms = {"default": cmd, "mcmc": cmd + ["--mcmc-cap", str(2 * a.loop_points)]}
    res = {k: [] for k in loop_arms}
    points = {}
    for _ in range(a.loop_rounds):
        for name, c in loop_arms.items():
            out = subprocess.run(c, capture_output=True, text=True)
            if out.returncode != 0:
                raise RuntimeError(f"{name}: {out.stdout}{out.stderr}")
            res[name].append(float(re.search(r"([\d.]+) ms per iteration", out.stdout).group(1)))
            points[name] = [int(p) for p in re.findall(r"points (\d+)", out.stdout)]
    result["train_loop_coarse"] = {k: {"ms_per_iter_median": float(np.median(v)), "ms_rounds": v,
                                       "points_every_50": points[k]} for k, v in res.items()}
    result["train_loop_coarse"]["iters"] = a.loop_iters
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
