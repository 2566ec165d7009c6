"""CPU: the oracle (oracle/splat_oracle.c) against the golden vectors captured from
the real reference extension (tests/golden/README.md).  This is what pins the
oracle; the GPU tests then pin the CUDA path against both."""
import glob
import os

import numpy as np
import pytest
import torch

import util

GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "raster_*.npz")))


def load_case(path):
    z = np.load(path)
    d = {}
    for k in ("means3D", "opacities", "scales", "rotations", "shs", "colors_precomp", "cov3D_precomp",
              "viewmatrix", "projmatrix", "campos", "bg"):
        d[k] = torch.from_numpy(z["in_" + k]) if ("in_" + k) in z.files else None
    for k in ("W", "H", "sh_degree"):
        d[k] = int(z["in_" + k])
    for k in ("tanfovx", "tanfovy"):
        d[k] = float(z["in_" + k])
    if "in_scale_modifier" in z.files:
        d["scale_modifier"] = float(z["in_scale_modifier"])
    return z, d


def test_golden_present():
    assert len(GOLD) >= 5, "golden vectors missing"


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p)[7:-4] for p in GOLD])
def test_oracle_forward_matches_reference(path, oracle_lib):
    z, d = load_case(path)
    o = util.oracle_run(oracle_lib, d)
    # integer / index outputs: bit-exact
    assert o["R"] == int(z["num_rendered"])
    np.testing.assert_array_equal(o["radii"], z["radii"])
    np.testing.assert_array_equal(o["geometry"]["tiles_touched"], z["tiles_touched"])
    np.testing.assert_array_equal(o["binning"]["point_list"], z["point_list"])
    np.testing.assert_array_equal(o["binning"]["keys"], z["point_list_keys"])
    np.testing.assert_array_equal(o["binning"]["ranges"], z["ranges"])
    np.testing.assert_array_equal(o["image"]["n_contrib"], z["n_contrib"])
    # floating point: 1e-4 relative (north_star), in practice ~1e-6
    vis = z["radii"] > 0
    assert util.relerr(o["geometry"]["xy"][vis], z["means2D"][vis]) < 1e-5
    assert util.relerr(o["geometry"]["conic_opacity"][vis], z["conic_opacity"][vis]) < 1e-4
    assert util.relerr(o["geometry"]["depth"][vis], z["depths"][vis]) < 1e-6
    assert util.relerr(o["color"], z["color"]) < 1e-4
    assert util.relerr(o["depth"], z["depth"]) < 1e-4
    assert util.relerr(o["image"]["final_T"], z["final_T"]) < 1e-4


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p)[7:-4] for p in GOLD])
def test_oracle_backward_matches_reference(path, oracle_lib):
    z, d = load_case(path)
    gc, gd = torch.from_numpy(z["in_grad_color"]), torch.from_numpy(z["in_grad_depth"])
    o = util.oracle_run(oracle_lib, d, gc, gd)
    g = o["grads"]
    names = {"means3D": "means3D", "means2D": "means2D", "opacities": "opacity", "scales": "scales",
             "rotations": "rotations", "shs": "sh", "colors_precomp": "colors", "cov3D_precomp": "cov3D"}
    checked = 0
    for gk, ok in names.items():
        key = "grad_" + gk
        if key not in z.files:
            continue
        ref = z[key]
        mine = g[ok].reshape(ref.shape)
        # the reference sums with unordered fp32 atomics; 1e-4 of the tensor's max is the bar
        assert util.relerr(mine, ref) < 1e-4, (gk, util.relerr(mine, ref))
        checked += 1
    assert checked >= 5
