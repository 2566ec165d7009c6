"""Generate tests/golden/raster_*.npz from the REAL reference extension.

Runs on a GPU (the reference rasterizer is CUDA-only), with the reference built into oracle/_ref:

    python tools/make_golden_raster.py OUTDIR [CASE ...]

then copy OUTDIR/*.npz to tests/golden/ and commit.  Each file holds
the inputs of one rasterizer call and everything the reference produced for it:
colour, depth, radii, the decoded internal state (means2D, conic_opacity, depth,
tiles_touched, sorted point_list + keys, ranges, n_contrib, final_T) and all
gradients for a seeded dL/dout.  The CPU oracle (oracle/splat_oracle.c) and the
CUDA path are both tested against these files.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

from s3gaussian_b200 import synthetic as syn
import ref_ext
import util

CASES = [
    # name, P, W, H, mode, sh_degree, seed, cov_precomp[, fy / fx, SH coefficients M, scale_modifier]
    ("small_sh3", 300, 64, 48, "sh", 3, 1, False),
    ("small_rgb", 300, 64, 48, "rgb", 0, 2, False),
    ("ragged_sh1", 500, 70, 45, "sh", 1, 3, False),       # image not a multiple of 16
    ("covpre_rgb", 200, 48, 32, "rgb", 0, 4, True),       # precomputed 3D covariance path
    ("dense_sh2", 1500, 96, 64, "sh", 2, 5, False),       # saturating pixels (T < 1e-4 early stop)
    # fx != fy (the Waymo reader scales them separately), fewer than 16 SH coefficients, scale_modifier != 1
    ("aniso_sh2_m9", 400, 70, 45, "sh", 2, 6, False, 1.448, 9, 0.8),
    ("aniso_sh1_m4", 300, 48, 80, "sh", 1, 7, False, 0.69, 4, 1.3),          # portrait
    ("aniso_covpre_rgb", 200, 64, 48, "rgb", 0, 8, True, 1.2, 0, 0.5),      # scale_modifier ignored with cov3D
    ("sh0_m1", 300, 64, 48, "sh", 0, 9, False, 1.0, 1, 1.0),
]


def case_inputs(name, P, W, H, mode, deg, seed, covpre, fy_over_fx=None, M=16, scale_modifier=None):
    """The scene dict of one case: make_small_scene's cloud; its camera, or with fy_over_fx the camera at the same pose
    with fx = 0.9 W and fy = fy_over_fx * fx; the first M SH coefficients; and scale_modifier when given."""
    cloud, cam = syn.make_small_scene(P=P, width=W, height=H, seed=seed)
    if name == "dense_sh2":
        cloud.opacity += 2.0
    if fy_over_fx is not None:
        cam = util.anisotropic_camera(W, H, 0.9 * W, fy_over_fx * 0.9 * W, (0.0, 0.0, 0.0))
    d = util.scene_inputs(cloud, cam, mode=mode, sh_degree=deg, cov_precomp=covpre)
    if d["shs"] is not None:
        d["shs"] = d["shs"][:, :M].contiguous()
    if scale_modifier is not None:
        d["scale_modifier"] = float(scale_modifier)
    return d


def main(outdir, names=None):
    os.makedirs(outdir, exist_ok=True)
    dev = torch.device("cuda:0")
    ref = ref_ext.load()
    for case in CASES:
        name, P, W, H, mode, deg, seed = case[:7]
        if names and name not in names:
            continue
        d = case_inputs(*case)
        gc, gd = util.seeded_grads(d, seed=seed + 100)
        out = util.run_module(ref, d, dev, gc, gd)
        # internal state through the raw extension entry point
        E = torch.Tensor([])
        g = lambda k: d[k].to(dev).contiguous() if d[k] is not None else E
        R, _, _, _, gb, bb, ib = ref._C.rasterize_gaussians(
            d["bg"].to(dev), g("means3D"), g("colors_precomp"), g("opacities"), g("scales"), g("rotations"),
            d.get("scale_modifier", 1.0), g("cov3D_precomp"), d["viewmatrix"].to(dev), d["projmatrix"].to(dev), d["tanfovx"],
            d["tanfovy"], H, W, g("shs"), deg, d["campos"].to(dev), False, False)
        torch.cuda.synchronize()
        rg, rb, ri = ref_ext.decode_geom(gb, P), ref_ext.decode_binning(bb, R), ref_ext.decode_image(ib, W * H)
        tiles = ((W + 15) // 16) * ((H + 15) // 16)
        save = {f"in_{k}": (v.numpy() if isinstance(v, torch.Tensor) else np.asarray(v))
                for k, v in d.items() if v is not None}
        save.update(in_grad_color=gc.numpy(), in_grad_depth=gd.numpy(),
                    color=out["color"].cpu().numpy(), depth=out["depth"].cpu().numpy(),
                    radii=out["radii"].cpu().numpy(), num_rendered=np.int64(R),
                    means2D=rg["means2D"].reshape(P, 2), conic_opacity=rg["conic_opacity"].reshape(P, 4),
                    depths=rg["depths"], tiles_touched=rg["tiles_touched"], cov3D=rg["cov3D"].reshape(P, 6),
                    rgb=rg["rgb"].reshape(P, 3), point_list=rb["point_list"], point_list_keys=rb["point_list_keys"],
                    ranges=ri["ranges"].reshape(-1, 2)[:tiles], n_contrib=ri["n_contrib"], final_T=ri["accum_alpha"])
        for k, v in out["grads"].items():
            save[f"grad_{k}"] = v.cpu().numpy()
        path = os.path.join(outdir, f"raster_{name}.npz")
        np.savez_compressed(path, **save)
        print(name, "R", R, "V", int((out["radii"] > 0).sum()), "->", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    # python tools/make_golden_raster.py OUTDIR [CASE ...]: only the named cases when any are given
    if len(sys.argv) < 2:
        sys.exit("usage: python tools/make_golden_raster.py OUTDIR [CASE ...]")
    main(sys.argv[1], sys.argv[2:])
