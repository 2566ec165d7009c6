"""LPIPS (v0.1; AlexNet, or VGG16 with --net vgg) per call on the device, four arms, and render_pixels per view with
LPIPS (prints one JSON line).

  ours         : s3gaussian_b200.lpips.LPIPS - implicit-GEMM convolutions in 3xTF32 (s3g_lpips_alex)
  cudnn_tf32   : the reference's lpipsPyTorch LPIPS module, built once, cuDNN at torch's default (TF32 allowed)
  cudnn_fp32   : the same module with torch.backends.cudnn.allow_tf32 = False (the accuracy class of `ours`)
  oracle_fp64  : oracle/lpips_oracle.py in float64 on the device, timed too but run for its value

Seeded random weights (Kaiming-scaled convolutions, non-negative lin weights), one image pair per call: a rendered-
like smooth image and a noisy copy.  After warm-up the arms alternate in rounds; each round times --calls calls of an
arm between two CUDA events.  Useful GFLOP counts the five convolutions (2 * M * N * K, x and y) from the layer
shapes.  The distance of each arm's value from the float64 result is reported.

The render_pixels part times render_pixels per view (fine stage, 12 waymo_ring views at 1920x1280, 500k Gaussians,
set up as tools/bench_eval_flow.py does) with lpips_fn set to `ours` and to the cuDNN module (TF32 default),
alternating, and without lpips_fn for the baseline.

--net vgg times s3gaussian_b200.lpips_vgg.LPIPSVGG (s3g_lpips_vgg) against the reference's module built with the
VGG16 backbone, the same arms and rounds, without the render_pixels part; GFLOP counts the thirteen convolutions.
`tflop_per_s` counts each multiply-add pair once for every arm: in `ours` the tensor cores execute three times that
(3xTF32).

    python tools/bench_lpips.py [--net alex] [--sizes 960x640,1920x1280] [--calls 50] [--rounds 5] [--points 500000]
                                [--views 12]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

CONVS = ((3, 64, 11, 4, 2), (64, 192, 5, 1, 2), (192, 384, 3, 1, 1), (384, 256, 3, 1, 1), (256, 256, 3, 1, 1))
# VGG16: (Cin, Cout) of the 3x3 / stride 1 / pad 1 convolutions, group by group; a 2x2 max-pool between the groups
VGG_GROUPS = (((3, 64), (64, 64)), ((64, 128), (128, 128)), ((128, 256), (256, 256), (256, 256)),
              ((256, 512), (512, 512), (512, 512)), ((512, 512), (512, 512), (512, 512)))


def gflop_vgg(H: int, W: int, images: int = 2) -> float:
    """2 x multiply-adds of the thirteen convolutions for `images` images of HxW (1503 per 1920x1280 image)."""
    total, h, w = 0, H, W
    for group in VGG_GROUPS:
        total += sum(2 * h * w * cout * cin * 9 for cin, cout in group)
        h, w = h // 2, w // 2
    return images * total / 1e9


def gflop(H: int, W: int, images: int = 2) -> float:
    """2 x multiply-adds of the five convolutions for `images` images of HxW (70.6 per 1920x1280 image)."""
    total, h, w = 0, H, W
    for l, (cin, cout, k, s, p) in enumerate(CONVS):
        h, w = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        total += 2 * h * w * cout * cin * k * k
        if l < 2:
            h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
    return images * total / 1e9


def image_pair(H, W, seed, dev):
    g = torch.Generator().manual_seed(seed)
    base = torch.nn.functional.interpolate(torch.rand(1, 3, H // 16, W // 16, generator=g), size=(H, W),
                                           mode="bilinear", align_corners=False)[0]
    return base.to(dev), (base + 0.05 * torch.randn(base.shape, generator=g)).clamp(0, 1).to(dev)


def time_calls(f, calls):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(calls):
        f()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--net", choices=("alex", "vgg"), default="alex")
    ap.add_argument("--sizes", default="960x640,1920x1280")
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--points", type=int, default=500_000)
    ap.add_argument("--views", type=int, default=12)
    ap.add_argument("--skip-render", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lpips needs a CUDA device")

    from bench_eval import power_limit_w
    if a.net == "vgg":
        import lpips_vgg_ref as lpips_ref
        from oracle import lpips_vgg_oracle as lo
        from s3gaussian_b200.lpips_vgg import LPIPSVGG as LPIPS
    else:
        import lpips_ref
        from oracle import lpips_oracle as lo
        from s3gaussian_b200.lpips import LPIPS

    dev = torch.device("cuda:0")
    feat, lin = lo.random_state_dicts(0)
    ours = LPIPS.from_state_dicts(feat, lin)
    ref = lpips_ref.reference_module(feat, lin).to(dev) if lpips_ref.available() else None

    def cudnn(tf32):
        def run(x, y):
            torch.backends.cudnn.allow_tf32 = tf32
            with torch.no_grad():
                return ref(x, y)
        return run
    arms = {"ours": lambda x, y: ours(x, y), "oracle_fp64": lambda x, y: lo.lpips_terms(x, y, feat, lin)[5]}
    if ref is not None:
        arms["cudnn_tf32"] = cudnn(True)
        arms["cudnn_fp32"] = cudnn(False)
    default_tf32 = torch.backends.cudnn.allow_tf32

    sizes = []
    for sz in a.sizes.split(","):
        W, H = (int(v) for v in sz.split("x"))
        x, y = image_pair(H, W, W + H, dev)
        exact = float(lo.lpips_terms(x, y, feat, lin)[5])
        for f in arms.values():
            for _ in range(a.warmup):
                f(x, y)
        torch.cuda.synchronize()
        ms = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, f in arms.items():
                calls = a.calls if k != "oracle_fp64" else max(3, a.calls // 10)
                ms[k].append(time_calls(lambda: f(x, y), calls))
        torch.backends.cudnn.allow_tf32 = default_tf32
        gf = (gflop_vgg if a.net == "vgg" else gflop)(H, W)
        res = {}
        for k, f in arms.items():
            t = float(np.median(ms[k]))
            v = float(f(x, y))
            res[k] = {"ms": round(t, 3), "ms_rounds": [round(m, 3) for m in ms[k]], "gflop": round(gf, 2),
                      "tflop_per_s": round(gf / t, 2), "value": v, "abs_err_vs_fp64": abs(v - exact),
                      "rel_err_vs_fp64": abs(v - exact) / abs(exact)}
        torch.backends.cudnn.allow_tf32 = default_tf32
        sizes.append({"resolution": f"{W}x{H}", "fp64_value": exact, "arms": res})

    render = None
    if not a.skip_render and a.net == "alex":
        render = bench_render_pixels(a, dev, ours, cudnn(True) if ref is not None else None)
        torch.backends.cudnn.allow_tf32 = default_tf32
    print(json.dumps({"metric": f"LPIPS {a.net} v0.1 ms per call (one image pair)", "gpu": torch.cuda.get_device_name(dev),
                      "power_limit_w": power_limit_w(), "calls_per_round": a.calls, "rounds": a.rounds,
                      "sizes": sizes, "render_pixels": render}))


def bench_render_pixels(a, dev, ours, cudnn_tf32):
    import ref_ext
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.deformation import deform_network
    from s3gaussian_b200.evaluation import render_pixels
    from s3gaussian_b200.gaussian_renderer import PipelineParams, GaussianModelLite
    W, H = 1920, 1280
    cams = [c.to(dev) for c in syn.waymo_ring(W, H, frames=50)[30:30 + a.views]]
    g = torch.Generator().manual_seed(0)
    for i, cam in enumerate(cams):
        cam.original_image = torch.rand(3, H, W, generator=g).to(dev)
        m = torch.zeros(H, W, dtype=torch.bool)
        if i % 3:
            m[200 + 40 * i:500 + 40 * i, 300:900 + 50 * i] = True
        cam.dynamic_mask = m.to(dev)
    pipe = PipelineParams()
    bg = torch.zeros(3, device=dev)
    net = deform_network(ref_ext.ref_deform_args(syn.DEFAULT_RESOLUTION, syn.DEFAULT_MULTIRES))
    net.deformation_net.set_aabb(*[list(x) for x in syn.WAYMO_AABB])
    net.load_state_dict(syn.make_deform_state(0, weight_scale=0.2), strict=False)
    pc = GaussianModelLite(syn.make_cloud(a.points, seed=0), net).to(dev)
    paths = {"no_lpips": None, "ours": ours}
    if cudnn_tf32 is not None:
        paths["cudnn_tf32"] = cudnn_tf32
    ms = {k: [] for k in paths}
    lp = {}
    import contextlib
    import io
    with torch.no_grad():
        for k, f in paths.items():
            with contextlib.redirect_stdout(io.StringIO()):
                render_pixels(cams, pc, bg, pipe, lpips_fn=f)
        for _ in range(a.rounds):
            for k, f in paths.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                with contextlib.redirect_stdout(io.StringIO()):
                    r = render_pixels(cams, pc, bg, pipe, lpips_fn=f)
                torch.cuda.synchronize()
                ms[k].append((time.perf_counter() - t0) * 1e3 / a.views)
                lp[k] = r["lpips"]
    return {"gaussians": a.points, "resolution": f"{W}x{H}", "views": a.views,
            "ms_per_view": {k: round(float(np.median(v)), 2) for k, v in ms.items()},
            "ms_per_view_rounds": {k: [round(t, 2) for t in v] for k, v in ms.items()}, "lpips": lp}


if __name__ == "__main__":
    main()
