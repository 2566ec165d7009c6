"""CPU: the integer binning restatement (tests/binning_ref.py) pinned to the real reference.

The golden vectors hold the reference extension's own projected centres, radii, depths, sorted point list, sorted
64-bit keys and ranges; the restatement rebuilds the last three from the first three alone and must reproduce them
bit for bit.  Two seeded scenes also go through the CPU oracle's binning, which is pinned by the same goldens."""
import os

import numpy as np
import pytest

import binning_ref as br
import util
from test_oracle_golden import GOLD, load_case


def _restate_golden(z, W, H):
    gx, gy = br.grid_of(W, H)
    radii = z["radii"]
    rect = br.rects_from_means2d(z["means2D"], radii, gx, gy)
    key = np.where(radii > 0, z["depths"].view(np.uint32), np.uint32(br.DEPTH_KEY_INVISIBLE)).astype(np.uint32)
    return br.binning(key, rect, gx, gx * gy), rect


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p)[7:-4] for p in GOLD])
def test_restatement_reproduces_reference_golden(path):
    z, d = load_case(path)
    ref, rect = _restate_golden(z, d["W"], d["H"])
    area = (rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1])
    np.testing.assert_array_equal(area, z["tiles_touched"].astype(np.int64))
    np.testing.assert_array_equal(ref["tiles_touched"], z["tiles_touched"])
    assert ref["R"] == int(z["num_rendered"])
    np.testing.assert_array_equal(ref["point_list"], z["point_list"])
    np.testing.assert_array_equal(ref["point_list_keys"], z["point_list_keys"])
    np.testing.assert_array_equal(ref["ranges"], z["ranges"])


@pytest.mark.parametrize("P,W,H,seed", [(700, 97, 61, 51), (3000, 256, 160, 52)])
def test_restatement_matches_cpu_oracle(P, W, H, seed, oracle_lib):
    from s3gaussian_b200 import synthetic as syn
    cloud, cam = syn.make_small_scene(P=P, width=W, height=H, seed=seed)
    d = util.scene_inputs(cloud, cam, mode="rgb")
    o = util.oracle_run(oracle_lib, d)
    gx, gy = br.grid_of(W, H)
    geo = o["geometry"]
    radii = o["radii"]
    rect = br.rects_from_means2d(geo["xy"], radii, gx, gy)
    key = np.where(radii > 0, np.asarray(geo["depth"], np.float32).view(np.uint32),
                   np.uint32(br.DEPTH_KEY_INVISIBLE)).astype(np.uint32)
    ref = br.binning(key, rect, gx, gx * gy)
    assert ref["R"] == o["R"] > 0
    np.testing.assert_array_equal(ref["tiles_touched"], geo["tiles_touched"])
    np.testing.assert_array_equal(ref["point_list"], o["binning"]["point_list"])
    np.testing.assert_array_equal(ref["point_list_keys"], o["binning"]["keys"])
    np.testing.assert_array_equal(ref["ranges"], o["binning"]["ranges"])


def test_restatement_ties_keep_index_order_and_offsets_scan_depth_order():
    """Hand-built case: equal depth keys, a culled Gaussian with a stale rect, a rect on the last tile column."""
    gx, gy = 3, 2
    key = np.array([7, 5, 7, br.DEPTH_KEY_INVISIBLE, 5, 7], np.uint32)
    rect = np.array([[0, 0, 2, 1], [1, 0, 3, 2], [2, 1, 3, 2], [0, 0, 3, 2], [1, 1, 2, 2], [0, 0, 1, 1]])
    ref = br.binning(key, rect, gx, gx * gy)
    np.testing.assert_array_equal(ref["tiles_touched"], [2, 4, 1, 0, 1, 1])
    np.testing.assert_array_equal(ref["order"], [1, 4, 0, 2, 5, 3])
    np.testing.assert_array_equal(ref["offsets"], [0, 4, 5, 7, 8, 9])
    assert ref["R"] == 9
    # tile 0: g0 (7), g5 (7); tile 1: g1 (5), g0 (7); tile 2: g1; tile 4: g1, g4 (both 5); tile 5: g1 (5), g2 (7)
    np.testing.assert_array_equal(ref["point_list"], [0, 5, 1, 0, 1, 1, 4, 1, 2])
    np.testing.assert_array_equal(ref["ranges"], [[0, 2], [2, 4], [4, 5], [0, 0], [5, 7], [7, 9]])
    np.testing.assert_array_equal(ref["point_list_keys"] >> np.uint64(32), [0, 0, 1, 1, 2, 4, 4, 5, 5])
