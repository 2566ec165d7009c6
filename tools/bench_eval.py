"""Per-view evaluation time: the reference's render_pixels step vs the fused one (prints one JSON line).

  current : render(return_decomposition=True, return_dx=True) as three rasterizer passes (full image, dynamic
            subset, static subset - what render() did without autograd before the split pass, and still does with
            it), PSNR in torch, image to the host, SSIM and the masked SSIM map with the skimage algorithm on the
            CPU (oracle/eval_oracle.py, the restatement of skimage.metrics.structural_similarity), masked PSNR in torch
            (utils/video_utils.py:170-241 without LPIPS)
  fused   : render() under no_grad (one split rasterizer pass) + the evaluation-metrics kernel, numbers left on the
            device (s3gaussian_b200.evaluation)

Fine stage, waymo_ring cameras at 1920x1280, 500k and 2M Gaussians by default.  The two paths alternate view by
view after warm-up; each per-view time is wall clock between two device synchronisations.  The render part alone is
also timed with CUDA events.  Both paths' images and metrics are compared on the timed views.

    python tools/bench_eval.py [--points 500000,2000000] [--views 6] [--rounds 3]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def power_limit_w():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=20)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def three_pass_render(cam, pc, pipe, bg):
    """render(stage='fine', return_decomposition=True, return_dx=True) with the decomposition as two extra
    rasterizer passes over the boolean-indexed subsets (gaussian_renderer.render's grad-enabled branch)."""
    import math
    from s3gaussian_b200.diff_gaussian_rasterization import GaussianRasterizationSettings, GaussianRasterizer
    xyz = pc.get_xyz
    dev = xyz.device
    campos = cam.camera_center.to(dev)
    rs = GaussianRasterizationSettings(
        image_height=int(cam.image_height), image_width=int(cam.image_width), tanfovx=math.tan(cam.FoVx * 0.5),
        tanfovy=math.tan(cam.FoVy * 0.5), bg=bg, scale_modifier=1.0, viewmatrix=cam.world_view_transform.to(dev),
        projmatrix=cam.full_proj_transform.to(dev), sh_degree=pc.active_sh_degree, campos=campos, prefiltered=False,
        debug=False)
    rast = GaussianRasterizer(rs)
    m2d = torch.zeros_like(xyz)
    m3, sc, ro, op, col, dx, dshs, feat = pc._deformation.render_front(
        xyz, pc._scaling, pc._rotation, pc._opacity, pc.get_features, float(cam.time), campos, pc.active_sh_degree)
    img, radii, depth = rast(means3D=m3, means2D=m2d, opacities=op, colors_precomp=col, scales=sc, rotations=ro)
    mx = torch.max(torch.abs(dx), dim=1)[0]
    mask = mx > torch.mean(mx)

    def sub(m):
        return rast(means3D=m3[m], means2D=m2d[m], opacities=op[m], colors_precomp=col[m], scales=sc[m],
                    rotations=ro[m])
    img_d, _, depth_d = sub(mask)
    img_s, _, depth_s = sub(~mask)
    return {"render": img, "depth": depth, "render_d": img_d, "depth_d": depth_d, "render_s": img_s, "depth_s": depth_s}


def psnr(img1, img2):
    # utils/image_utils.py:17-19
    mse = (((img1 - img2)) ** 2).view(img1.shape[0], -1).mean(1, keepdim=True)
    return 20 * torch.log10(1.0 / torch.sqrt(mse))


def host_metrics(rgb, gt, mask_np):
    """utils/video_utils.py:210-241 without LPIPS: torch PSNR, SSIM twice on the host"""
    from oracle import eval_oracle as eo
    out = {"psnr": psnr(rgb, gt).mean().double().item()}
    rgb_np, gt_np = rgb.cpu().numpy(), gt.cpu().numpy()
    out["ssim"] = eo.ssim(rgb_np, gt_np)
    if mask_np.sum() > 0:
        m = torch.from_numpy(mask_np).to(rgb.device)
        out["masked_psnr"] = psnr(rgb.permute(1, 2, 0)[m].permute(1, 0), gt.permute(1, 2, 0)[m].permute(1, 0)).mean().double().item()
        out["masked_ssim"] = eo.masked_ssim(rgb_np, gt_np, mask_np)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", default="500000,2000000")
    ap.add_argument("--views", type=int, default=6)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()

    import ref_ext
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.deformation import deform_network
    from s3gaussian_b200.evaluation import _eval_sums, _mask_u8, _view_metrics
    from s3gaussian_b200.gaussian_renderer import render, PipelineParams, GaussianModelLite

    dev = torch.device("cuda:0")
    W, H = 1920, 1280
    cams = [c.to(dev) for c in syn.waymo_ring(W, H, frames=50)[30:30 + a.views]]
    g = torch.Generator().manual_seed(0)
    gts, masks = [], []
    for i in range(a.views):
        gts.append(torch.rand(3, H, W, generator=g).to(dev))
        m = np.zeros((H, W), bool)
        if i % 3:
            m[200 + 40 * i:500 + 40 * i, 300:900 + 50 * i] = True
        masks.append(m)
    pipe = PipelineParams()
    bg = torch.zeros(3, device=dev)
    results = []
    for P in [int(p) for p in a.points.split(",")]:
        net = deform_network(ref_ext.ref_deform_args(syn.DEFAULT_RESOLUTION, syn.DEFAULT_MULTIRES))
        net.deformation_net.set_aabb(*[list(x) for x in syn.WAYMO_AABB])
        net.load_state_dict(syn.make_deform_state(0, weight_scale=0.2), strict=False)
        pc = GaussianModelLite(syn.make_cloud(P, seed=0), net).to(dev)

        def current(i):
            r = three_pass_render(cams[i], pc, pipe, bg)
            return r, host_metrics(r["render"], gts[i], masks[i])

        def fused(i):
            r = render(cams[i], pc, pipe, bg, stage="fine", return_decomposition=True, return_dx=True)
            img = r["render"]
            v = _view_metrics(_eval_sums(img, gts[i], _mask_u8(masks[i], H, W, dev)), 3, H, W)
            return r, v

        def wall(fn, i):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn(i)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3, out

        def events(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            out = fn()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1), out

        ms_cur, ms_fus, ms_r3, ms_r1 = [], [], [], []
        worst = {"image_relerr": 0.0, "psnr": 0.0, "ssim": 0.0, "masked_psnr": 0.0, "masked_ssim": 0.0}
        bitwise = True
        with torch.no_grad():
            for _ in range(a.warmup):
                current(0)
                fused(0)
            for rnd in range(a.rounds):
                for i in range(a.views):
                    t_c, (rc, mc) = wall(current, i)
                    t_f, (rf, mf) = wall(fused, i)
                    ms_cur.append(t_c)
                    ms_fus.append(t_f)
                    t3, _ = events(lambda: three_pass_render(cams[i], pc, pipe, bg))
                    t1, _ = events(lambda: render(cams[i], pc, pipe, bg, stage="fine", return_decomposition=True,
                                                  return_dx=True))
                    ms_r3.append(t3)
                    ms_r1.append(t1)
                    if rnd == 0:
                        for k in ("render", "depth", "render_d", "depth_d", "render_s", "depth_s"):
                            if not torch.equal(rc[k], rf[k]):
                                bitwise = False
                                e = float((rc[k] - rf[k]).abs().max() / rc[k].abs().max().clamp_min(1e-30))
                                worst["image_relerr"] = max(worst["image_relerr"], e)
                        mf = mf.cpu().numpy()
                        worst["psnr"] = max(worst["psnr"], abs(mc["psnr"] - mf[0]))
                        worst["ssim"] = max(worst["ssim"], abs(mc["ssim"] - mf[1]))
                        if "masked_psnr" in mc:
                            worst["masked_psnr"] = max(worst["masked_psnr"], abs(mc["masked_psnr"] - mf[2]))
                            worst["masked_ssim"] = max(worst["masked_ssim"], abs(mc["masked_ssim"] - mf[3]))
        results.append({"gaussians": P, "resolution": f"{W}x{H}", "views": a.views, "rounds": a.rounds,
                        "ms_per_view_current": round(float(np.median(ms_cur)), 3),
                        "ms_per_view_fused": round(float(np.median(ms_fus)), 3),
                        "speedup": round(float(np.median(ms_cur) / np.median(ms_fus)), 2),
                        "ms_render_three_pass": round(float(np.median(ms_r3)), 3),
                        "ms_render_split": round(float(np.median(ms_r1)), 3),
                        "images_bitwise_equal": bitwise,
                        "max_abs_metric_diff": {k: float(v) for k, v in worst.items()}})
        del pc, net
        torch.cuda.empty_cache()
    print(json.dumps({"metric": "ms per evaluated view (render with decomposition + PSNR/SSIM/masked metrics, no LPIPS)",
                      "gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(),
                      "workloads": results}))


if __name__ == "__main__":
    main()
