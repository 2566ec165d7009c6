"""Rasterizer backward with and without the absolute screen-space gradients: s3g_rasterize_backward against
s3g_rasterize_backward_absgrad (deterministic = 0), and s3g_rasterize_backward_deterministic against
s3g_rasterize_backward_absgrad (deterministic = 1), on the state of one plain forward, in the same process.  Prints one
JSON line.

Shapes: the bench.py headline (2 M Gaussians, SH degree 3, 1920x1280, bench.py's camera waymo_ring[1]) and the
rasterizer shape of config 3 (500 k Gaussians, 1920x1280, precomputed colours + the feature image through the aux pair
that render(render_feat=True) uses).  After warm-up the arms alternate in rounds; each round times --calls calls of
one arm between two CUDA events.  The card's name and power limit are read in the same run.

    python tools/bench_raster_absgrad.py [--calls 20] [--rounds 5]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_raster_camera import card, time_arms   # noqa: E402


def setup(P, W, H, aux, dev):
    import util
    from s3gaussian_b200 import _lib, synthetic as syn
    from s3gaussian_b200 import diff_gaussian_rasterization as ours
    cloud = syn.make_cloud(P, seed=0)
    cam = syn.waymo_ring(W, H, frames=50)[1]
    d = util.scene_inputs(cloud, cam, mode="rgb" if aux else "sh", sh_degree=3, bg=(0.0, 0.0, 0.0))

    class Ctx:
        def save_for_backward(self, *a):
            self.saved = a

        def mark_non_differentiable(self, *a):
            pass
    E = torch.Tensor([])
    g = lambda k: d[k].to(dev).contiguous() if d[k] is not None else E
    inputs = [g(k) for k in ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")]
    rs = util.settings_for(ours, d, dev)
    gen = torch.Generator().manual_seed(3)
    colors_aux = torch.rand(P, 3, generator=gen).to(dev) if aux else None
    lib = _lib.load()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    means3D, sh, cp, op, sc, ro, cov = inputs

    ctx = Ctx()
    ours._RasterizeGaussians.forward(ctx, means3D, torch.zeros_like(means3D), *inputs[1:], rs, colors_aux)
    bscene = ours._scene(rs, means3D.device, means3D, sh, cp, None, sc, ro, cov)
    e = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
    outs = [e(P, 3), e(P, 1), e(P, 3), e(P, 3), e(P, 6), e(P, 16, 3), e(P, 3), e(P, 4), e(P, 3)]
    absgrad = e(P, 2)
    gc, gd, gf = (torch.randn(ch, H, W, generator=gen).to(dev) for ch in (3, 1, 3))
    s = ctx.saved
    bwd = _lib.RasterBackwardArgs(
        R=ctx.num_rendered, radii=s[5].data_ptr(), geom_buffer=s[7].data_ptr(), binning_buffer=s[8].data_ptr(),
        image_buffer=s[9].data_ptr(), dL_dpix=gc.data_ptr(), dL_dpix_depth=gd.data_ptr(),
        dL_dmean2D=outs[0].data_ptr(), dL_dopacity=outs[1].data_ptr(), dL_dcolor=outs[2].data_ptr(),
        dL_dmean3D=outs[3].data_ptr(), dL_dcov3D=outs[4].data_ptr(), dL_dsh=outs[5].data_ptr(),
        dL_dscale=outs[6].data_ptr(), dL_drot=outs[7].data_ptr())
    if aux:
        bwd.dL_dpix_aux, bwd.dL_dcolor_aux = gf.data_ptr(), outs[8].data_ptr()
    nbytes = int(lib.s3g_rasterize_backward_deterministic_workspace_bytes(P, ctx.num_rendered, W, H))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    S, B = C.byref(bscene), C.byref(bwd)
    arms = {
        "backward": lambda: _lib.check(lib.s3g_rasterize_backward(S, B, stream), "bwd"),
        "backward_absgrad": lambda: _lib.check(lib.s3g_rasterize_backward_absgrad(
            S, B, None, absgrad.data_ptr(), 0, None, stream), "bwd absgrad"),
        "deterministic": lambda: _lib.check(lib.s3g_rasterize_backward_deterministic(
            S, B, ws.data_ptr(), stream), "det"),
        "deterministic_absgrad": lambda: _lib.check(lib.s3g_rasterize_backward_absgrad(
            S, B, None, absgrad.data_ptr(), 1, ws.data_ptr(), stream), "det absgrad"),
    }
    keep = (ctx, bwd, inputs, colors_aux, bscene, outs, absgrad, ws, gc, gd, gf)
    return arms, ctx.num_rendered, keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: there is no CPU path")
    dev = torch.device("cuda:0")
    result = {"card": card()}
    for name, (P, W, H, aux) in {"headline_2M_1920x1280_sh": (2_000_000, 1920, 1280, False),
                                 "config3_500k_1920x1280_aux": (500_000, 1920, 1280, True)}.items():
        arms, R, keep = setup(P, W, H, aux, dev)
        r = {"P": P, "R": R, **time_arms(arms, a.calls, a.rounds)}
        r["absgrad_over_backward"] = r["backward_absgrad"]["ms_median"] / r["backward"]["ms_median"]
        r["absgrad_over_deterministic"] = r["deterministic_absgrad"]["ms_median"] / r["deterministic"]["ms_median"]
        result[name] = r
        del arms, keep
        torch.cuda.empty_cache()
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
