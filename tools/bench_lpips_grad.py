"""LPIPS (AlexNet, v0.1) forward + backward per call on the device, four arms, and the cost of an LPIPS loss term in a
fine-stage render + loss + backward iteration (prints one JSON line).

  ours         : s3gaussian_b200.lpips.LPIPS - s3g_lpips_alex, then s3g_lpips_alex_backward (3xTF32 dgrads)
  cudnn_tf32   : autograd of the reference's lpipsPyTorch module, cuDNN at torch's default (TF32 allowed)
  cudnn_fp32   : the same with torch.backends.cudnn.allow_tf32 = False
  oracle_fp64  : autograd of oracle/lpips_oracle.py in float64 on the device

One image pair per call (tools/bench_lpips.py's smooth image and a noisy copy), the gradient taken with respect to x
(the rendered image of a training loss).  After warm-up the arms alternate in rounds; each round times --calls calls
between two CUDA events.  GFLOP from the layer shapes: the forward's five convolutions for both images, plus the
input-gradient convolutions for x (as many multiply-adds as the forward's for one image).  Each arm's gradient is
compared with the float64 one (relative L2 and max |difference| / max |g64|).

The iteration part renders a fine-stage view (500k Gaussians, 1920x1280 by default, set up as tools/bench_lpips.py
does), takes the L1 loss to a ground truth and runs the backward, with and without `+ 0.05 * lpips(image, gt)`,
alternating; the optimiser step is not included (it does not depend on the loss).

    python tools/bench_lpips_grad.py [--sizes 960x640,1920x1280] [--calls 20] [--rounds 5] [--points 500000]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_lpips import gflop, image_pair, time_calls  # noqa: E402


def gflop_fwd_bwd(H: int, W: int) -> float:
    """forward for x and y, input gradients for x: the dgrads of convs 2-5 on the tensor cores and conv 1's on the
    CUDA cores do as many multiply-adds as the forward's convolutions of one image"""
    return gflop(H, W, images=2) + gflop(H, W, images=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="960x640,1920x1280")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--points", type=int, default=500_000)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--skip-train", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lpips_grad needs a CUDA device")

    import lpips_ref
    from bench_eval import power_limit_w
    from oracle import lpips_oracle as lo
    from s3gaussian_b200.lpips import LPIPS

    dev = torch.device("cuda:0")
    feat, lin = lo.random_state_dicts(0)
    ours = LPIPS.from_state_dicts(feat, lin)
    ref = lpips_ref.reference_module(feat, lin).to(dev) if lpips_ref.available() else None
    default_tf32 = torch.backends.cudnn.allow_tf32

    def grad_of(f, dtype=torch.float32):
        def run(x, y):
            xr = x.detach().to(dtype).clone().requires_grad_(True)
            f(xr, y.detach().to(dtype)).sum().backward()
            return xr.grad
        return run

    def cudnn(tf32):
        def run(x, y):
            torch.backends.cudnn.allow_tf32 = tf32
            return grad_of(ref)(x, y)
        return run
    arms = {"ours": grad_of(ours),
            "oracle_fp64": grad_of(lambda x, y: lo.lpips_terms(x, y, feat, lin)[5], torch.float64)}
    if ref is not None:
        arms["cudnn_tf32"] = cudnn(True)
        arms["cudnn_fp32"] = cudnn(False)

    sizes = []
    for sz in a.sizes.split(","):
        W, H = (int(v) for v in sz.split("x"))
        x, y = image_pair(H, W, W + H, dev)
        g64 = arms["oracle_fp64"](x, y)
        for f in arms.values():
            for _ in range(a.warmup):
                f(x, y)
        torch.cuda.synchronize()
        ms = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, f in arms.items():
                calls = a.calls if k != "oracle_fp64" else max(2, a.calls // 10)
                ms[k].append(time_calls(lambda: f(x, y), calls))
        gf = gflop_fwd_bwd(H, W)
        res = {}
        for k, f in arms.items():
            t = float(np.median(ms[k]))
            d = f(x, y).double() - g64
            res[k] = {"ms": round(t, 3), "ms_rounds": [round(m, 3) for m in ms[k]], "gflop": round(gf, 2),
                      "tflop_per_s": round(gf / t, 2), "grad_rel_l2_vs_fp64": float(d.norm() / g64.norm()),
                      "grad_max_vs_fp64": float(d.abs().max() / g64.abs().max())}
        torch.backends.cudnn.allow_tf32 = default_tf32
        sizes.append({"resolution": f"{W}x{H}", "arms": res})

    train = None if a.skip_train else bench_iteration(a, dev, ours)
    print(json.dumps({"metric": "LPIPS alex v0.1 forward + backward (grad for x) ms per call, one image pair",
                      "gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(),
                      "calls_per_round": a.calls, "rounds": a.rounds, "sizes": sizes, "iteration": train}))


def bench_iteration(a, dev, ours):
    import ref_ext
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.deformation import deform_network
    from s3gaussian_b200.gaussian_renderer import PipelineParams, GaussianModelLite, render
    W, H = 1920, 1280
    cam = syn.waymo_ring(W, H, frames=50)[30].to(dev)
    gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(0)).to(dev)
    net = deform_network(ref_ext.ref_deform_args(syn.DEFAULT_RESOLUTION, syn.DEFAULT_MULTIRES))
    net.deformation_net.set_aabb(*[list(x) for x in syn.WAYMO_AABB])
    net.load_state_dict(syn.make_deform_state(0, weight_scale=0.2), strict=False)
    pc = GaussianModelLite(syn.make_cloud(a.points, seed=0), net).to(dev)
    pipe, bg = PipelineParams(), torch.zeros(3, device=dev)

    def step(lam):
        image = render(cam, pc, pipe, bg, stage="fine")["render"]
        loss = (image - gt).abs().mean()
        if lam:
            loss = loss + lam * ours(image, gt).squeeze()
        loss.backward()
        for p in pc.parameters():
            p.grad = None
    arms = {"l1": 0.0, "l1_plus_0.05_lpips": 0.05}
    for lam in arms.values():
        for _ in range(a.warmup):
            step(lam)
    torch.cuda.synchronize()
    ms = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, lam in arms.items():
            ms[k].append(time_calls(lambda: step(lam), a.iters))
    med = {k: float(np.median(v)) for k, v in ms.items()}
    return {"gaussians": a.points, "resolution": f"{W}x{H}", "stage": "fine", "iters_per_round": a.iters,
            "ms_per_iteration": {k: round(v, 3) for k, v in med.items()},
            "ms_rounds": {k: [round(t, 3) for t in v] for k, v in ms.items()},
            "extra_ms_for_lpips": round(med["l1_plus_0.05_lpips"] - med["l1"], 3)}


if __name__ == "__main__":
    main()
