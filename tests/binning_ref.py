"""Integer restatement of the forward's binning (test infrastructure).

Binning is everything between the preprocess and the composite: the depth sort, the offset scan, the tile-instance
emission, the tile-id sort and the per-tile ranges.  Its result is fully determined by three per-Gaussian outputs of
the preprocess: the depth key (the float bits of the view-space depth, 0xFFFFFFFF for a culled Gaussian), the tile
rect and the rect's area.  This module recomputes every integer the binning produces from those, in numpy int64,
with no tolerance and no float arithmetic, so a test can compare the device's buffers exactly.

The instance list is restated the way the reference rasterizer builds it, not the way this project does: one
(tile << 32 | depth bits) key per touched tile, emitted in Gaussian-index order, then one stable sort on the 64-bit
keys (DGR/cuda_rasterizer/rasterizer_impl.cu:70-138).  The device instead sorts the depths over the Gaussians first
and sorts only the tile ids over the instances; the two agree exactly when every pass is stable.
"""
from __future__ import annotations

import numpy as np

DEPTH_KEY_INVISIBLE = 0xFFFFFFFF
TILE = 16


def grid_of(W: int, H: int) -> tuple[int, int]:
    return (W + TILE - 1) // TILE, (H + TILE - 1) // TILE


def key_bits(n_tiles: int) -> int:
    """Bits of the tile-id sort key (getHigherMsb, rasterizer_impl.cu:35-50): enough for every tile id, at least 1."""
    return max(1, int(n_tiles).bit_length())


def rects_from_means2d(means2D, radii, grid_x: int, grid_y: int) -> np.ndarray:
    """[P, 4] int64 (x0, y0, x1, y1) in tiles: the reference's getRect (auxiliary.h:46-56) in float32 - the integer
    radius converted to float, one float32 add or subtract at a time, the division by the tile size (exact) and C
    truncation toward zero, clamped to [0, grid].  Rows with radius 0 (culled) are zero."""
    p = np.asarray(means2D, np.float32).reshape(-1, 2)
    rad = np.asarray(radii).reshape(-1)
    vis = rad > 0
    r = rad.astype(np.float32)
    t = np.float32(TILE)
    with np.errstate(invalid="ignore", over="ignore"):
        lo_x = (p[:, 0] - r) / t
        lo_y = (p[:, 1] - r) / t
        hi_x = ((p[:, 0] + r) + np.float32(TILE - 1)) / t
        hi_y = ((p[:, 1] + r) + np.float32(TILE - 1)) / t
    out = np.zeros((p.shape[0], 4), np.int64)
    for c, (v, g) in enumerate(((lo_x, grid_x), (lo_y, grid_y), (hi_x, grid_x), (hi_y, grid_y))):
        out[vis, c] = np.clip(np.trunc(v[vis]), 0, g).astype(np.int64)
    return out


def binning(depth_key, rect, grid_x: int, n_tiles: int) -> dict:
    """depth_key [P] u32, rect [P, 4] (x0, y0, x1, y1) in tiles.  A Gaussian is culled when its depth key is
    DEPTH_KEY_INVISIBLE; its rect is then ignored (the device does not write it).  Returns

      tiles_touched [P]  the rect area of a visible Gaussian, 0 for a culled one
      order [P]          stable argsort of depth_key over all P Gaussians
      offsets [P]        exclusive cumulative sum of tiles_touched[order]
      R                  total instance count
      point_list [R]     Gaussian of every (tile, Gaussian) instance, sorted by (tile, depth key, Gaussian index)
      point_list_keys [R] u64 (tile << 32 | depth key) in the same order
      ranges [n_tiles, 2] [start, end) of every touched tile in point_list, (0, 0) for every other tile
    """
    key = np.asarray(depth_key, np.uint32).reshape(-1).astype(np.int64)
    r = np.asarray(rect).reshape(-1, 4).astype(np.int64)
    P = key.shape[0]
    vis = key != DEPTH_KEY_INVISIBLE
    w = r[:, 2] - r[:, 0]
    h = r[:, 3] - r[:, 1]
    touched = np.where(vis, w * h, 0)
    if np.any(touched < 0):
        raise ValueError("rect with x1 < x0 or y1 < y0")

    order = np.argsort(key, kind="stable")
    t_sorted = touched[order]
    offsets = np.cumsum(t_sorted) - t_sorted
    R = int(touched.sum())

    # duplicateWithKeys: every visible Gaussian, in index order, writes one key per tile of its rect
    g_vis = np.nonzero(touched)[0]
    n = touched[g_vis]
    g = np.repeat(g_vis, n)
    start = np.cumsum(n) - n
    i = np.arange(R, dtype=np.int64) - np.repeat(start, n)
    wr = np.repeat(w[g_vis], n)
    tile = (np.repeat(r[g_vis, 1], n) + i // wr) * grid_x + np.repeat(r[g_vis, 0], n) + i % wr
    del i, wr, start
    if R and (tile.min() < 0 or tile.max() >= n_tiles):
        raise ValueError("rect outside the tile grid")
    keys = (tile << 32) | key[g]
    perm = np.argsort(keys, kind="stable")
    point_list = g[perm]
    keys = keys[perm]
    tile = tile[perm]
    del perm

    counts = np.bincount(tile, minlength=n_tiles).astype(np.int64)
    ends = np.cumsum(counts)
    ranges = np.stack([ends - counts, ends], 1)
    ranges[counts == 0] = 0
    return dict(tiles_touched=touched.astype(np.uint32), order=order.astype(np.uint32),
                offsets=offsets.astype(np.uint32), R=R, point_list=point_list.astype(np.uint32),
                point_list_keys=keys.astype(np.uint64), ranges=ranges.astype(np.uint32))
