"""Rasterizer with the lens off, an identity lens and a distorting lens: the forward (s3g_rasterize_forward against
s3g_rasterize_forward_lens) and the backward (s3g_rasterize_backward on the state of each kind of forward, which runs
the lens's chain rule after a lens forward), in the same process.  Prints one JSON line.  The identity lens is the
camera's own pinhole (fx = width / (2 tan_fovx), cx = width / 2); the distorting one moves the principal point by
(+12, -8) px and takes k1 = -0.12, k2 = 0.03, p1 = 1e-3, p2 = -5e-4, k3 = 0 (no finite lens cull).

Shapes: the bench.py headline (2 M Gaussians, SH degree 3, 1920x1280, bench.py's camera waymo_ring[1]) and the
rasterizer shape of config 3 (500 k Gaussians, 1920x1280, the fine stage's precomputed colours + feature image through
the aux pair that render(render_feat=True) uses).  After warm-up the arms alternate in rounds; each round times --calls
calls of one arm between two CUDA events.  The forward arms share their own state buffers; each backward arm has the
state of one forward of its kind.  The card's name and power limit are read in the same run.

    python tools/bench_raster_lens.py [--calls 20] [--rounds 5]
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

    # forward arms: their own state buffers and outputs
    scene, fwd, lease, _, color, depth, radii = ours._forward_args(means3D, sh, cp, op, sc, ro, cov, rs)
    if aux:
        color_aux = torch.empty_like(color)
        fwd.colors_aux, fwd.out_color_aux = colors_aux.data_ptr(), color_aux.data_ptr()

    W_, H_ = d["W"], d["H"]
    fx, fy = W_ / (2 * d["tanfovx"]), H_ / (2 * d["tanfovy"])
    lenses = {"identity": ours.Lens(fx, fy, W_ / 2, H_ / 2),
              "distorting": ours.Lens(fx, fy, W_ / 2 + 12, H_ / 2 - 8, -0.12, 0.03, 1e-3, -5e-4, 0.0)}
    lens_s = {k: ours._lens_struct(v) for k, v in lenses.items()}

    # backward arms: the state of one forward of each kind
    bscene = ours._scene(rs, means3D.device, means3D, sh, cp, None, sc, ro, cov)
    e = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
    outs = [e(P, 3), e(P, 1), e(P, 3), e(P, 3), e(P, 6), e(P, 16, 3), e(P, 3), e(P, 4), e(P, 3)]
    gc, gd, gf = (torch.randn(ch, H, W, generator=gen).to(dev) for ch in (3, 1, 3))
    ctxs, bwds = [], []
    for lens in (None, lenses["identity"], lenses["distorting"]):
        ctx = Ctx()
        ours._RasterizeGaussians.forward(ctx, means3D, torch.zeros_like(means3D), *inputs[1:], rs, colors_aux, None,
                                         None, None, False, False, False, lens)
        s = ctx.saved
        bwd = _lib.RasterBackwardArgs(
            R=ctx.num_rendered, radii=s[5].data_ptr(), geom_buffer=s[7].data_ptr(), binning_buffer=s[8].data_ptr(),
            image_buffer=s[9].data_ptr(), dL_dpix=gc.data_ptr(), dL_dpix_depth=gd.data_ptr(),
            dL_dmean2D=outs[0].data_ptr(), dL_dopacity=outs[1].data_ptr(), dL_dcolor=outs[2].data_ptr(),
            dL_dmean3D=outs[3].data_ptr(), dL_dcov3D=outs[4].data_ptr(), dL_dsh=outs[5].data_ptr(),
            dL_dscale=outs[6].data_ptr(), dL_drot=outs[7].data_ptr())
        if aux:
            bwd.dL_dpix_aux, bwd.dL_dcolor_aux = gf.data_ptr(), outs[8].data_ptr()
        ctxs.append(ctx)
        bwds.append(bwd)
    torch.cuda.synchronize()

    arms = {
        "forward": lambda: _lib.check(lib.s3g_rasterize_forward(C.byref(scene), C.byref(fwd), stream), "fwd"),
        "forward_lens_identity": lambda: _lib.check(lib.s3g_rasterize_forward_lens(
            C.byref(scene), C.byref(fwd), None, 0, C.byref(lens_s["identity"]), stream), "fwd lens identity"),
        "forward_lens_distorting": lambda: _lib.check(lib.s3g_rasterize_forward_lens(
            C.byref(scene), C.byref(fwd), None, 0, C.byref(lens_s["distorting"]), stream), "fwd lens distorting"),
        "backward": lambda: _lib.check(lib.s3g_rasterize_backward(C.byref(bscene), C.byref(bwds[0]), stream), "bwd"),
        "backward_lens_identity": lambda: _lib.check(lib.s3g_rasterize_backward(
            C.byref(bscene), C.byref(bwds[1]), stream), "bwd lens identity"),
        "backward_lens_distorting": lambda: _lib.check(lib.s3g_rasterize_backward(
            C.byref(bscene), C.byref(bwds[2]), stream), "bwd lens distorting"),
    }
    keep = (ctxs, bwds, lens_s, inputs, colors_aux, scene, fwd, lease, color, depth, radii, bscene, outs, gc, gd, gf) + (
        (color_aux,) if aux else ())
    return arms, [c.num_rendered for c in ctxs], keep


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
        r = {"P": P, "R_plain": R[0], "R_lens_identity": R[1], "R_lens_distorting": R[2],
             **time_arms(arms, a.calls, a.rounds)}
        for pas in ("forward", "backward"):
            for lens in ("identity", "distorting"):
                r[f"{pas}_lens_{lens}_over_{pas}"] = r[f"{pas}_lens_{lens}"]["ms_median"] / r[pas]["ms_median"]
        result[name] = r
        del arms, keep
        torch.cuda.empty_cache()
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
