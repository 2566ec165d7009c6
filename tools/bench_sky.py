"""Sky model: the kernels behind s3gaussian_b200.sky.Background_Model against the same model written in torch float32
(the reference's get_directions, encoding and nn.Linear chain, through autograd), which is what running the
reference's Background_Model would cost.  Prints one JSON line.

(a) Widths 64 and 256 at 960x640 (the reference's Waymo load size) and 1920x1280: forward, and forward + backward
    (every weight gradient), each arm alternating with the others in each round between CUDA events, after warm-up.
    Reported: the mean over the rounds and their spread (min, max), the peak memory each arm allocates above what it
    starts with, and the achieved TFLOP/s from the FLOP counts computed below from the shapes (fp32 FLOPs of the
    model; the 3xTF32 kernels issue three tensor-core products for each).
(b) examples/train_loop.py (coarse) with and without --sky, one subprocess per arm, alternating; each run reports its
    own time per iteration.
The card's name and power limit are read in the same run.

    python tools/bench_sky.py [--calls 10] [--rounds 5] [--loop-rounds 2] [--loop-points 500000] [--loop-iters 300]
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

from bench_raster_camera import card   # noqa: E402


def flops(width, px):
    """Multiply-adds x 2 per pixel: the forward's three layers; the backward's weight gradients of all three layers
    plus the input gradients of the two upper ones (the sigmoid, relu and encoding are not counted)."""
    macs_fwd = 33 * width + (width + 33) * width + 3 * width
    macs_bwd = macs_fwd + width * width + 3 * width
    return 2.0 * macs_fwd * px, 2.0 * (macs_fwd + macs_bwd) * px


def arms(width, W, H, dev):
    from s3gaussian_b200.sky import Background_Model
    torch.manual_seed(0)
    m = Background_Model(img_width=W, img_height=H, model_cfg={"mlp_width": width}).to(dev)
    params = [p for p in m.parameters()]
    tp = [p.detach().clone().requires_grad_(True) for p in params]
    c2w = torch.eye(4, device=dev)
    f = 0.9 * W
    K = torch.tensor([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], device=dev)
    g = torch.randn(3, H, W, device=dev)
    y, x = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32),
                          torch.arange(W, device=dev, dtype=torch.float32), indexing="ij")
    scales = torch.tensor([1.0, 2, 4, 8, 16], device=dev)

    def torch_sky():
        W0, b0, W1, b1, W2, b2 = tp
        with torch.no_grad():
            cam = torch.stack([(x - K[0, 2] + 0.5) / K[0, 0], (y - K[1, 2] + 0.5) / K[1, 1], torch.ones_like(x)], -1)
            d = (cam.reshape(-1, 1, 3) * c2w[:3, :3]).sum(-1)
            v = d / (torch.linalg.norm(d, dim=-1, keepdim=True) + 1e-8)
            xb = (v[:, None, :] * scales[:, None]).reshape(-1, 15)
            e = torch.cat([v, torch.sin(torch.cat([xb, xb + 0.5 * torch.pi], -1))], -1)
        h1 = torch.relu(torch.nn.functional.linear(e, W0, b0))
        h2 = torch.relu(torch.nn.functional.linear(torch.cat([h1, e], -1), W1, b1))
        return torch.sigmoid(torch.nn.functional.linear(h2, W2, b2)).reshape(H, W, 3).permute(2, 0, 1)

    def ours_fwd():
        with torch.no_grad():
            return m(c2w, K)

    def ours_fwd_bwd():
        return torch.autograd.grad(m(c2w, K), params, g)

    def torch_fwd():
        with torch.no_grad():
            return torch_sky()

    def torch_fwd_bwd():
        return torch.autograd.grad(torch_sky(), tp, g)

    with torch.no_grad():
        a, b = m(c2w, K), torch_sky()
        parity = float((a - b).abs().max() / b.abs().max())
    ga, gb = ours_fwd_bwd(), torch_fwd_bwd()
    gpar = max(float((u - w).abs().max() / w.abs().max()) for u, w in zip(ga, gb))
    return {"ours_fwd": ours_fwd, "ours_fwd_bwd": ours_fwd_bwd, "torch_fwd": torch_fwd,
            "torch_fwd_bwd": torch_fwd_bwd}, {"sky_rel_to_max": parity, "grad_rel_to_max": gpar}


def time_arms(fns, calls, rounds):
    for fn in fns.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    res = {k: [] for k in fns}
    for _ in range(rounds):
        for name, fn in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(calls):
                fn()
            e1.record()
            torch.cuda.synchronize()
            res[name].append(e0.elapsed_time(e1) / calls)
    return {k: {"ms_mean": float(np.mean(v)), "ms_min": float(np.min(v)), "ms_max": float(np.max(v))}
            for k, v in res.items()}


def peak_mb(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def loop_runs(points, iters, rounds):
    res = {"plain": [], "sky": []}
    for _ in range(rounds):
        for name in res:
            cmd = [sys.executable, os.path.join(ROOT, "examples", "train_loop.py"), "--points", str(points), "--iters",
                   str(iters)] + (["--sky"] if name == "sky" else [])
            r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
            if r.returncode != 0:
                raise RuntimeError(r.stdout + r.stderr)
            res[name].append(float(re.search(r"([\d.]+) ms per iteration", r.stdout).group(1)))
    return {k: {"ms_per_iter_mean": float(np.mean(v)), "ms_rounds": v} for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--loop-rounds", type=int, default=2)
    ap.add_argument("--loop-points", type=int, default=500_000)
    ap.add_argument("--loop-iters", type=int, default=300)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {"card_before": card()}
    for width in (64, 256):
        for W, H in ((960, 640), (1920, 1280)):
            fns, parity = arms(width, W, H, dev)
            t = time_arms(fns, a.calls, a.rounds)
            f_fwd, f_all = flops(width, W * H)
            res[f"w{width}_{W}x{H}"] = {
                "ms": t,
                "peak_MB": {k: peak_mb(fn) for k, fn in fns.items()},
                "GFLOP": {"fwd": f_fwd / 1e9, "fwd_bwd": f_all / 1e9},
                "TFLOPs": {k: (f_fwd if k.endswith("fwd") else f_all) / (v["ms_mean"] * 1e9) for k, v in t.items()},
                "parity": parity}
            del fns
            torch.cuda.empty_cache()
    if a.loop_rounds > 0:
        res["train_loop"] = dict(loop_runs(a.loop_points, a.loop_iters, a.loop_rounds), points=a.loop_points,
                                 iters=a.loop_iters, size="960x640")
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
