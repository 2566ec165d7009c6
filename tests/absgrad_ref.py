"""float64 torch restatement of the absolute screen-space gradient (s3g_rasterize_backward_absgrad), written from the
definition in include/s3g_b200.h after the composite restatement of test_gpu_raster_opacity._restated_images
(test infrastructure).

Every (pixel, list slot) pair gets its own zero leaf offsets ex, ey added to the Gaussian's pixel-space mean, so one
backward of sum(dL/dpix * images) gives, per pair, pixel p's share of dL/dmean2D.  The signed statistic is their
scatter-sum, the absolute one the scatter-sum of their absolute values, both times W/2 (x) or H/2 (y)."""
from __future__ import annotations

import numpy as np
import torch


def tile_pixels(W, H):
    """[tiles, 256] pixel ids (-1 outside the image) in tile order (16x16 tiles, row-major)."""
    tx, ty = (W + 15) // 16, (H + 15) // 16
    out = np.full((tx * ty, 256), -1, np.int64)
    for t in range(tx * ty):
        x0, y0 = (t % tx) * 16, (t // tx) * 16
        yy, xx = np.mgrid[y0:y0 + 16, x0:x0 + 16]
        ok = (xx < W) & (yy < H)
        out[t] = np.where(ok, yy * W + xx, -1).reshape(-1)
    return out


def pixel_lists(W, H, ranges, point_list):
    """(pix [n], idx [n,K]): every pixel of the image and its tile's depth-ordered list (-1 padded), from the forward's
    per-tile ranges and point list."""
    tiles = tile_pixels(W, H)
    K = max(1, int((ranges[:, 1] - ranges[:, 0]).max()))
    pix_all, idx_all = [], []
    for tt, (s0, e0) in enumerate(ranges):
        pix = tiles[tt][tiles[tt] >= 0]
        row = np.full(K, -1, np.int64)
        row[:e0 - s0] = point_list[s0:e0]
        pix_all.append(pix)
        idx_all.append(np.repeat(row[None], pix.size, 0))
    return torch.from_numpy(np.concatenate(pix_all)), torch.from_numpy(np.concatenate(idx_all))


def composite64(W, H, mx, my, conic, op, col, tz, bg, pix, idx, aux=None, ex=None, ey=None):
    """The composite of test_gpu_raster_opacity._restated_images on pixel-space means (mx, my), conics [P,3] and the
    opacities the composite uses (op, opacity * h after an antialiased forward), with ex / ey [n,K] added to each
    pair's offset: -> per-pixel (color [n,3], depth [n], alpha [n], median [n], aux [n,3] or None).  Blend decisions
    are taken on the values."""
    dev = mx.device
    valid = idx >= 0
    gi = idx.clamp_min(0)
    px, py = (pix % W).double()[:, None], (pix // W).double()[:, None]
    dx, dy = mx[gi] - px, my[gi] - py
    if ex is not None:
        dx, dy = dx + ex, dy + ey
    cA, cB, cC = conic[:, 0], conic[:, 1], conic[:, 2]
    power = -0.5 * (cA[gi] * dx * dx + cC[gi] * dy * dy) - cB[gi] * dx * dy
    alpha = torch.clamp_max(op[gi] * torch.exp(power), 0.99)
    vis = valid & (power.detach() <= 0) & (alpha.detach() >= 1 / 255)
    n, K = idx.shape
    T = torch.ones(n, dtype=torch.float64, device=dev)
    alive = torch.ones(n, dtype=torch.bool, device=dev)
    Cimg = torch.zeros(n, 3, dtype=torch.float64, device=dev)
    Aimg = torch.zeros(n, 3, dtype=torch.float64, device=dev)
    D = torch.zeros(n, dtype=torch.float64, device=dev)
    med = torch.zeros(n, dtype=torch.float64, device=dev)
    for k in range(K):
        a = alpha[:, k]
        test_T = T * (1 - a)
        ok = alive & vis[:, k]
        stop = ok & (test_T.detach() < 1e-4)
        blend = ok & ~stop
        w = torch.where(blend, a * T, torch.zeros_like(T))
        g = gi[:, k]
        Cimg = Cimg + w[:, None] * col[g]
        if aux is not None:
            Aimg = Aimg + w[:, None] * aux[g]
        D = D + w * tz[g]
        hit = blend & (T.detach() > 0.5) & (test_T.detach() <= 0.5)
        med = torch.where(hit, tz[g], med)
        T = torch.where(blend, test_T, T)
        alive = alive & ~stop
    return (Cimg + T[:, None] * bg, D, 1 - T, med, (Aimg + T[:, None] * bg) if aux is not None else None)


def pixel_loss(images, pix, dL):
    """sum over pixels of dL/dpix . images; dL: dict of [C,H,W] float64 gradients for any of color, depth, alpha,
    median, aux (absent: 0)."""
    color, depth, alpha, median, aux = images
    at = lambda g: g.reshape(g.shape[0], -1)[:, pix].T
    loss = 0.0
    for name, v in (("color", color), ("depth", depth[:, None]), ("alpha", alpha[:, None]),
                    ("median", median[:, None]), ("aux", aux)):
        if name in dL and v is not None:
            loss = loss + (v * at(dL[name])).sum()
    return loss


def mean2d_grads64(W, H, mx, my, conic, op, col, tz, bg, pix, idx, dL, aux=None):
    """-> (signed [P,2], absgrad [P,2]) in the units of dL_dmean2D: the scatter-sums over (pixel, slot) pairs of each
    pixel's dL_p/dmean2D and of its absolute value."""
    P = mx.shape[0]
    ex = torch.zeros(idx.shape, dtype=torch.float64, device=mx.device, requires_grad=True)
    ey = torch.zeros_like(ex, requires_grad=True)
    loss = pixel_loss(composite64(W, H, mx.detach(), my.detach(), conic.detach(), op.detach(), col.detach(),
                                  tz.detach(), bg, pix, idx, None if aux is None else aux.detach(), ex, ey), pix, dL)
    gx, gy = torch.autograd.grad(loss, (ex, ey), allow_unused=True)
    gx = torch.zeros_like(ex) if gx is None else gx
    gy = torch.zeros_like(ey) if gy is None else gy
    valid = idx >= 0
    g = idx[valid]
    out = torch.zeros(2, 2, P, dtype=torch.float64, device=mx.device)
    for c, (gv, scale) in enumerate(((gx[valid], 0.5 * W), (gy[valid], 0.5 * H))):
        out[0, c].index_add_(0, g, gv * scale)
        out[1, c].index_add_(0, g, gv.abs() * scale)
    return out[0].T.contiguous(), out[1].T.contiguous()
