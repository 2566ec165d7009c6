"""GPU: the accumulated-opacity and median-depth images of the rasterizer (s3g_rasterize_forward_opacity and the two
*_opacity backwards) through GaussianRasterizer.forward_opacity, forward_eval(with_opacity=True), render() with
pipe.render_opacity and render_pixels(with_opacity=True).

1. On the golden scenes and on tile-edge and ragged shapes: colour, depth and radii bitwise those of forward(); alpha
   bitwise 1 - final_T; colour - (1 - alpha) bg equal to the bg = 0 image; the median depth bitwise the depth of the
   Gaussian at the stored median position, which a CPU walk over the sorted lists picks too.
2. dL_ddepth of loss = sum g * median is, per Gaussian, the sum of g over the pixels it is the median of.
3. Gradients of losses on alpha, on the median, and on both with colour, depth and aux against a float64 torch
   restatement of preprocess + composite (P <= 64, multi-tile images), camera gradients included.
4. Determinism, render() and render_pixels().
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import util
from test_oracle_golden import GOLD, load_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ours(built_lib):
    from s3gaussian_b200 import diff_gaussian_rasterization as mod
    return mod


class _Ctx:
    def save_for_backward(self, *a):
        self.saved = a

    def mark_non_differentiable(self, *a):
        pass


def _inputs(d):
    E = torch.Tensor([])
    g = lambda k: d[k].to(DEV).contiguous() if d[k] is not None else E
    return [g(k) for k in ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")]


def _opacity_forward(ours, d):
    """_RasterizeGaussians.forward(opacity=True) keeping the state: -> (outputs, ctx, views of the state)."""
    from s3gaussian_b200 import _lib
    inputs = _inputs(d)
    ctx = _Ctx()
    out = ours._RasterizeGaussians.forward(ctx, inputs[0], torch.zeros_like(inputs[0]), *inputs[1:],
                                           util.settings_for(ours, d, DEV), None, None, None, None, True)
    torch.cuda.synchronize()
    P, R, W, H = inputs[0].shape[0], ctx.num_rendered, d["W"], d["H"]
    bufs = {0: ctx.saved[7], 1: ctx.saved[8], 2: ctx.saved[9]}

    def view(bid, name, dt):
        off, eb, cnt = _lib.state_field(bid, name, P, R, W, H)
        buf = bufs[bid]
        a = ((buf.data_ptr() + 127) & ~127) - buf.data_ptr() + off
        return buf[a:a + eb * cnt].cpu().numpy().view(dt).copy()

    views = dict(final_T=view(2, "final_T", np.float32), median_contrib=view(2, "median_contrib", np.uint32),
                 ranges=view(2, "ranges", np.uint32).reshape(-1, 2),
                 point_list=view(1, "point_list", np.uint32) if R > 0 else np.zeros(0, np.uint32),
                 xyAB=view(0, "xyAB", np.float32).reshape(-1, 4), Cod=view(0, "Cod", np.float32).reshape(-1, 4),
                 rgb=view(0, "rgb", np.float32).reshape(-1, 4))
    return out, ctx, views


def _small(P, W, H, seed, mode="rgb", deg=0, cov=False):
    from s3gaussian_b200 import synthetic as syn
    cloud, cam = syn.make_small_scene(P=P, width=W, height=H, seed=seed)
    return util.scene_inputs(cloud, cam, mode=mode, sh_degree=deg, cov_precomp=cov)


# golden scenes, a 16x16 single tile, tile-edge (multiples of 16) and ragged shapes
SHAPES = [("sh", 3, 400, 80, 64, 11), ("sh", 0, 257, 33, 17, 12), ("rgb", 0, 1000, 128, 96, 13),
          ("sh", 2, 64, 16, 16, 14), ("rgb", 0, 600, 47, 31, 15), ("sh", 1, 900, 96, 48, 16)]
CASES = [("golden", p) for p in GOLD] + [("shape", s) for s in SHAPES]


def _case(kind, spec):
    if kind == "golden":
        return load_case(spec)[1]
    mode, deg, P, W, H, seed = spec
    return _small(P, W, H, seed, mode, deg)


def _tile_pixels(W, H):
    """[tiles, 256] pixel ids (-1 outside the image) in tile order"""
    tx, ty = (W + 15) // 16, (H + 15) // 16
    out = np.full((tx * ty, 256), -1, np.int64)
    for t in range(tx * ty):
        x0, y0 = (t % tx) * 16, (t // tx) * 16
        yy, xx = np.mgrid[y0:y0 + 16, x0:x0 + 16]
        ok = (xx < W) & (yy < H)
        out[t] = np.where(ok, yy * W + xx, -1).reshape(-1)
    return out


def _cpu_median_walk(views, W, H):
    """float64 walk over every pixel's sorted list with the forward's float32 records: -> (1-based median position per
    pixel, 0 for none; smallest distance of any decision in the pixel's walk from its threshold)"""
    pos = np.zeros(W * H, np.int64)
    margin = np.full(W * H, np.inf)
    xy, Cod, tiles = views["xyAB"].astype(np.float64), views["Cod"].astype(np.float64), _tile_pixels(W, H)
    for t, (s, e) in enumerate(views["ranges"]):
        pix = tiles[t][tiles[t] >= 0]
        if e == s or pix.size == 0:
            continue
        px, py = (pix % W).astype(np.float64), (pix // W).astype(np.float64)
        T, alive, p, m = np.ones(pix.size), np.ones(pix.size, bool), np.zeros(pix.size, np.int64), margin[pix]
        for k, g in enumerate(views["point_list"][s:e]):
            dx, dy = xy[g, 0] - px, xy[g, 1] - py
            power = -0.5 * (xy[g, 2] * dx * dx + Cod[g, 0] * dy * dy) - xy[g, 3] * dx * dy
            a = np.minimum(0.99, Cod[g, 1] * np.exp(power))
            test_T = T * (1 - a)
            ok = alive & (power <= 0) & (a >= 1 / 255)
            stop = ok & (test_T < 1e-4)
            blend = ok & ~stop
            hit = blend & (T > 0.5) & (test_T <= 0.5)
            p = np.where(hit, k + 1, p)
            live = alive & (power <= 0)
            m = np.where(live, np.minimum(m, np.minimum(np.abs(a - 1 / 255), np.abs(test_T - 1e-4))), m)
            m = np.where(blend, np.minimum(m, np.abs(test_T - 0.5)), m)
            T = np.where(blend, test_T, T)
            alive = alive & ~stop
        pos[pix], margin[pix] = p, m
    return pos, margin


@pytest.mark.parametrize("kind,spec", CASES, ids=[f"golden-{p.split('/')[-1][7:-4]}" if k == "golden" else
                                                  "x".join(map(str, p[2:5])) + f"-{p[0]}" for k, p in CASES])
def test_forward_images(kind, spec, ours):
    d = _case(kind, spec)
    W, H = d["W"], d["H"]
    color0, radii0, depth0, _, _ = util.ours_forward_state(d, DEV)
    (color, radii, depth, alpha, median), ctx, v = _opacity_forward(ours, d)
    assert torch.equal(color, color0) and torch.equal(depth, depth0) and torch.equal(radii, radii0)
    a = alpha.cpu().numpy().reshape(-1)
    assert np.array_equal(a.view(np.uint32), (np.float32(1) - v["final_T"]).view(np.uint32))
    assert a.min() >= 0 and a.max() < 1
    color_bg0, _, _, _, _ = util.ours_forward_state(dict(d, bg=torch.zeros(3)), DEV)
    bg = d["bg"].to(DEV).view(3, 1, 1)
    torch.testing.assert_close(color - (1 - alpha) * bg, color_bg0, rtol=0, atol=1e-6)
    # the median: the depth of the Gaussian at the stored position, bitwise
    med, pos = median.cpu().numpy().reshape(-1), v["median_contrib"].astype(np.int64)
    tiles = _tile_pixels(W, H)
    start = np.zeros(W * H, np.int64)
    for t in range(tiles.shape[0]):
        start[tiles[t][tiles[t] >= 0]] = v["ranges"][t, 0]
    has = pos > 0
    assert has.any()
    g = v["point_list"][start[has] + pos[has] - 1]
    assert np.array_equal(med[has].view(np.uint32), v["rgb"][g, 3].view(np.uint32))
    assert (med[~has] == 0).all()
    assert ((a >= 0.5) == has).all()         # a median exactly where T fell to 0.5 or below
    # a CPU walk picks the same Gaussian, except where a decision sits within float32 rounding of its threshold
    cpu, margin = _cpu_median_walk(v, W, H)
    differ = cpu != pos
    assert (margin[differ] < 1e-5).all(), (np.nonzero(differ)[0][:8], margin[differ][:8])
    assert differ.sum() <= max(2, W * H // 2000)


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("spec", SHAPES[:3] + SHAPES[4:5])
def test_median_gradient_goes_to_the_median_gaussian(spec, det, ours):
    from s3gaussian_b200 import _lib
    lib = _lib.load()
    mode, deg, P, W, H, seed = spec
    d = _small(P, W, H, seed, mode, deg)
    (color, radii, depth, alpha, median), ctx, v = _opacity_forward(ours, d)
    gen = torch.Generator().manual_seed(seed)
    gm = torch.randn(1, H, W, generator=gen).to(DEV)
    means3D, sh, cp, op, sc, ro, cov = _inputs(d)
    M = sh.shape[1] if sh.numel() else 0
    scene = ours._scene(util.settings_for(ours, d, DEV), means3D.device, means3D, sh, cp, None, sc, ro, cov)
    e = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device=DEV)
    o = dict(mean2D=e(P, 3), conic=e(P, 4), opacity=e(P, 1), color=e(P, 3), depth=e(P), mean3D=e(P, 3), cov3D=e(P, 6),
             sh=e(P, max(M, 1), 3), scale=e(P, 3), rot=e(P, 4))
    z3, z1 = torch.zeros(3, H, W, device=DEV), torch.zeros(1, H, W, device=DEV)
    s = ctx.saved
    bwd = _lib.RasterBackwardArgs(
        R=ctx.num_rendered, radii=s[5].data_ptr(), geom_buffer=s[7].data_ptr(), binning_buffer=s[8].data_ptr(),
        image_buffer=s[9].data_ptr(), dL_dpix=z3.data_ptr(), dL_dpix_depth=z1.data_ptr(),
        dL_dmean2D=o["mean2D"].data_ptr(), dL_dconic=o["conic"].data_ptr(), dL_dopacity=o["opacity"].data_ptr(),
        dL_dcolor=o["color"].data_ptr(), dL_ddepth=o["depth"].data_ptr(), dL_dmean3D=o["mean3D"].data_ptr(),
        dL_dcov3D=o["cov3D"].data_ptr(), dL_dsh=o["sh"].data_ptr() if M else None, dL_dscale=o["scale"].data_ptr(),
        dL_drot=o["rot"].data_ptr())
    opa = _lib.RasterOpacityArgs(dL_dpix_median=gm.data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    if det:
        nb = int(lib.s3g_rasterize_backward_deterministic_workspace_bytes(P, ctx.num_rendered, W, H))
        ws = torch.empty(max(nb, 16), dtype=torch.uint8, device=DEV)
        _lib.check(lib.s3g_rasterize_backward_deterministic_opacity(C.byref(scene), C.byref(bwd), C.byref(opa),
                                                                    ws.data_ptr(), stream), "det")
    else:
        _lib.check(lib.s3g_rasterize_backward_opacity(C.byref(scene), C.byref(bwd), C.byref(opa), stream), "bwd")
    torch.cuda.synchronize()
    pos = v["median_contrib"].astype(np.int64)
    tiles = _tile_pixels(W, H)
    start = np.zeros(W * H, np.int64)
    for t in range(tiles.shape[0]):
        start[tiles[t][tiles[t] >= 0]] = v["ranges"][t, 0]
    has = pos > 0
    expect = np.zeros(P, np.float64)
    np.add.at(expect, v["point_list"][start[has] + pos[has] - 1].astype(np.int64),
              gm.cpu().numpy().reshape(-1)[has].astype(np.float64))
    got = o["depth"].cpu().numpy()
    assert (expect != 0).sum() > 3
    assert (got[expect == 0] == 0).all()
    np.testing.assert_allclose(got, expect, rtol=1e-5, atol=1e-6 * np.abs(expect).max())
    # the alpha-free, colour-free loss moves the Gaussians only through their depth: no opacity / conic gradient
    assert float(o["opacity"].abs().max()) == 0 and float(o["conic"].abs().max()) == 0


# ---- gradients against a float64 restatement ------------------------------------------------------------------------
def _restated_images(d, leaf, lists, aux=None):
    """float64 restatement of preprocess + composite (preprocess.cuh, composite.cuh), the tile lists taken from the
    forward: -> (color [3,H,W], depth, alpha, median, aux image or None).  Blend decisions are taken on the values."""
    W, H = d["W"], d["H"]
    x, V, Pm = leaf["means3D"], leaf["view"], leaf["proj"]
    xt = torch.cat([x, torch.ones_like(x[:, :1])], 1)
    t, p = xt @ V, xt @ Pm
    ndc = p[:, :2] / (p[:, 3:4] + 1e-7)
    mx, my = ((ndc[:, 0] + 1) * W - 1) * 0.5, ((ndc[:, 1] + 1) * H - 1) * 0.5
    tz = t[:, 2]
    if "cov3D" in leaf:
        c = leaf["cov3D"]
    else:
        s, q = leaf["scales"], leaf["rotations"]
        r, qx, qy, qz = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
        R = torch.stack([1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - r * qz), 2 * (qx * qz + r * qy),
                         2 * (qx * qy + r * qz), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - r * qx),
                         2 * (qx * qz - r * qy), 2 * (qy * qz + r * qx), 1 - 2 * (qx * qx + qy * qy)], 1).view(-1, 3, 3)
        L = R * s[:, None, :]
        S = L @ L.transpose(1, 2)
        c = torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1)
    Sig = torch.stack([c[:, 0], c[:, 1], c[:, 2], c[:, 1], c[:, 3], c[:, 4], c[:, 2], c[:, 4], c[:, 5]], 1).view(-1, 3, 3)
    fx, fy = W / (2 * d["tanfovx"]), H / (2 * d["tanfovy"])
    limx, limy = 1.3 * d["tanfovx"], 1.3 * d["tanfovy"]
    rx, ry = t[:, 0] / tz, t[:, 1] / tz
    tx = torch.where(rx.abs() <= limx, t[:, 0], (rx.clamp(-limx, limx) * tz).detach())
    ty = torch.where(ry.abs() <= limy, t[:, 1], (ry.clamp(-limy, limy) * tz).detach())
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, zero, -fx * tx / tz ** 2], 1),
                     torch.stack([zero, fy / tz, -fy * ty / tz ** 2], 1)], 1)
    Tm = J @ V[:3, :3].T
    cov = Tm @ Sig @ Tm.transpose(1, 2)
    a_, b_, c_ = cov[:, 0, 0] + 0.3, cov[:, 0, 1], cov[:, 1, 1] + 0.3
    det = a_ * c_ - b_ * b_
    cA, cB, cC = c_ / det, -b_ / det, a_ / det
    op, col = leaf["opacities"][:, 0], leaf["colors"]
    tiles = _tile_pixels(W, H)
    pix_all, idx_all = [], []
    K = max(1, int((lists["ranges"][:, 1] - lists["ranges"][:, 0]).max()))
    for tt, (s0, e0) in enumerate(lists["ranges"]):
        pix = tiles[tt][tiles[tt] >= 0]
        row = np.full(K, -1, np.int64)
        row[:e0 - s0] = lists["point_list"][s0:e0]
        pix_all.append(pix)
        idx_all.append(np.repeat(row[None], pix.size, 0))
    pix = torch.from_numpy(np.concatenate(pix_all)).to(DEV)
    idx = torch.from_numpy(np.concatenate(idx_all)).to(DEV)
    valid = idx >= 0
    gi = idx.clamp_min(0)
    px, py = (pix % W).double()[:, None], (pix // W).double()[:, None]
    dx, dy = mx[gi] - px, my[gi] - py
    power = -0.5 * (cA[gi] * dx * dx + cC[gi] * dy * dy) - cB[gi] * dx * dy
    alpha = torch.clamp_max(op[gi] * torch.exp(power), 0.99)
    vis = valid & (power <= 0) & (alpha >= 1 / 255)
    n = pix.numel()
    T = torch.ones(n, dtype=torch.float64, device=DEV)
    alive = torch.ones(n, dtype=torch.bool, device=DEV)
    Cimg = torch.zeros(n, 3, dtype=torch.float64, device=DEV)
    Aimg = torch.zeros(n, 3, dtype=torch.float64, device=DEV)
    D = torch.zeros(n, dtype=torch.float64, device=DEV)
    med = torch.zeros(n, dtype=torch.float64, device=DEV)
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
    bg = d["bg"].to(DEV).double()
    order = torch.argsort(pix)
    img = lambda v: v[order].T.reshape(-1, H, W)
    color = img(Cimg + T[:, None] * bg)
    aux_img = img(Aimg + T[:, None] * bg) if aux is not None else None
    return color, img(D[:, None]), img((1 - T)[:, None]), img(med[:, None]), aux_img


def _grad_case(P, W, H, seed, cov):
    from s3gaussian_b200 import synthetic as syn
    cloud, cam = syn.make_small_scene(P=P, width=W, height=H, seed=seed)
    cloud.scaling += math.log(2.5)          # fewer, larger Gaussians: most pixels see several and alpha passes 0.5
    return util.scene_inputs(cloud, cam, mode="rgb", cov_precomp=cov)


LOSSES = ["alpha", "median", "all"]


@pytest.mark.parametrize("loss_kind", LOSSES)
@pytest.mark.parametrize("P,W,H,seed,cov", [(48, 48, 40, 3, False), (64, 40, 33, 5, True), (32, 64, 32, 9, False)])
def test_gradients_match_float64_restatement(P, W, H, seed, cov, loss_kind, ours):
    check_gradients_against_restatement(ours, _grad_case(P, W, H, seed, cov), seed, loss_kind)


def check_gradients_against_restatement(ours, d, seed, loss_kind):
    """forward_opacity's gradients (Gaussians and camera) for `loss_kind` against _restated_images in float64; d holds
    precomputed colours."""
    P, W, H, cov = d["means3D"].shape[0], d["W"], d["H"], d["cov3D_precomp"] is not None
    _, _, _, _, lists = util.ours_forward_state(d, DEV)
    gen = torch.Generator().manual_seed(seed + 100)
    gc, gd, ga, gm = (torch.randn(ch, H, W, generator=gen, dtype=torch.float64) for ch in (3, 1, 1, 1))
    gx = torch.randn(3, H, W, generator=gen, dtype=torch.float64)
    aux_cols = torch.rand(P, 3, generator=gen)
    use_aux = loss_kind == "all"

    def loss_of(color, depth, alpha, median, aux_img, dt):
        c = lambda t: t.to(DEV, dt)
        if loss_kind == "alpha":
            return (alpha * c(ga)).sum()
        if loss_kind == "median":
            return (median * c(gm)).sum()
        return ((alpha * c(ga)).sum() + (median * c(gm)).sum() + (color * c(gc)).sum() + (depth * c(gd)).sum() +
                (aux_img * c(gx)).sum())

    names = ["means3D", "opacities", "colors_precomp"] + (["cov3D_precomp"] if cov else ["scales", "rotations"])
    t32 = {k: d[k].to(DEV).clone().requires_grad_(True) for k in names}
    rs = util.settings_for(ours, d, DEV)
    cam32 = {k: getattr(rs, k).clone().requires_grad_(True) for k in ("viewmatrix", "projmatrix", "campos")}
    rs = rs._replace(**cam32)
    aux32 = aux_cols.to(DEV).requires_grad_(True) if use_aux else None
    out = ours.GaussianRasterizer(rs).forward_opacity(
        means3D=t32["means3D"], means2D=torch.zeros_like(t32["means3D"], requires_grad=True),
        opacities=t32["opacities"], colors_precomp=t32["colors_precomp"], scales=t32.get("scales"),
        rotations=t32.get("rotations"), cov3D_precomp=t32.get("cov3D_precomp"), colors_aux=aux32)
    color, radii, depth, alpha, median = out[:5]
    loss_of(color, depth, alpha, median, out[5] if use_aux else None, torch.float32).backward()

    leaf = {"means3D": d["means3D"], "opacities": d["opacities"], "colors": d["colors_precomp"],
            "view": d["viewmatrix"], "proj": d["projmatrix"]}
    leaf.update({"cov3D": d["cov3D_precomp"]} if cov else {"scales": d["scales"], "rotations": d["rotations"]})
    leaf = {k: v.to(DEV).double().clone().requires_grad_(True) for k, v in leaf.items()}
    aux64 = aux_cols.to(DEV).double().requires_grad_(True) if use_aux else None
    images = _restated_images(d, leaf, lists, aux64)
    # the restatement reproduces the images first (same blend decisions)
    for got, ref in zip((color, depth, alpha, median), images[:4]):
        assert util.relerr(got.detach().cpu().numpy(), ref.detach().cpu().numpy()) < 1e-4
    assert float((median > 0).float().mean()) > 0.2
    loss_of(*images, torch.float64).backward()
    pairs = [(t32["means3D"], leaf["means3D"], "means3D"), (t32["opacities"], leaf["opacities"], "opacities"),
             (cam32["viewmatrix"], leaf["view"], "viewmatrix"), (cam32["projmatrix"], leaf["proj"], "projmatrix")]
    pairs += [(t32["cov3D_precomp"], leaf["cov3D"], "cov3D")] if cov else [
        (t32["scales"], leaf["scales"], "scales"), (t32["rotations"], leaf["rotations"], "rotations")]
    if loss_kind == "all":
        pairs += [(t32["colors_precomp"], leaf["colors"], "colors"), (aux32, aux64, "aux")]
    vis = (radii > 0).cpu()
    for g32, g64, name in pairs:
        got = g32.grad
        ref = g64.grad if g64.grad is not None else torch.zeros_like(g64)   # not in the median's graph
        if got.dim() == 2 and got.shape[0] == P:
            got, ref = got[vis.to(got.device)], ref[vis.to(ref.device)]
        got, ref = got.double().cpu().numpy(), ref.detach().cpu().numpy()
        if np.abs(ref).max() == 0:   # the median depends on neither the 2-D footprint nor the projection matrix
            assert loss_kind == "median" and np.abs(got).max() == 0, (name, np.abs(got).max())
            continue
        assert util.relerr(got, ref) < 1e-3, (loss_kind, name, util.relerr(got, ref))
    if loss_kind == "median":    # the median moves the Gaussians only through their depth
        assert float(t32["opacities"].grad.abs().max()) == 0


# ---- determinism ----------------------------------------------------------------------------------------------------
class _deterministic:
    def __enter__(self):
        self.prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
        torch.use_deterministic_algorithms(True)

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.prev[0], warn_only=self.prev[1])


def _autograd_run(ours, d, seed, aux=False):
    t = {k: d[k].to(DEV).clone().requires_grad_(True) for k in util.TENSOR_KEYS if d[k] is not None}
    m2d = torch.zeros_like(t["means3D"], requires_grad=True)
    rs = util.settings_for(ours, d, DEV)
    cam = {k: getattr(rs, k).clone().requires_grad_(True) for k in ("viewmatrix", "projmatrix", "campos")}
    rs = rs._replace(**cam)
    gen = torch.Generator().manual_seed(seed)
    H, W = d["H"], d["W"]
    gc, gd, ga, gm, gx = (torch.randn(ch, H, W, generator=gen).to(DEV) for ch in (3, 1, 1, 1, 3))
    colors_aux = torch.rand(d["means3D"].shape[0], 3, generator=gen).to(DEV).requires_grad_(True) if aux else None
    out = ours.GaussianRasterizer(rs).forward_opacity(means2D=m2d, colors_aux=colors_aux, **t)
    loss = (out[0] * gc).sum() + (out[2] * gd).sum() + (out[3] * ga).sum() + (out[4] * gm).sum()
    if aux:
        loss = loss + (out[5] * gx).sum()
    loss.backward()
    res = {k: v.grad.clone() for k, v in list(t.items()) + list(cam.items())}
    res["means2D"] = m2d.grad.clone()
    if aux:
        res["aux"] = colors_aux.grad.clone()
    return res


@pytest.mark.parametrize("aux", [False, True])
def test_deterministic_backward_repeats_bitwise(aux, ours):
    from s3gaussian_b200 import synthetic as syn
    cloud = syn.make_cloud(60_000, seed=4, width=640, height=416)
    cam = syn.make_camera(640, 416, (0, 0, 2.0))
    d = util.scene_inputs(cloud, cam, mode="sh", sh_degree=3)
    with _deterministic():
        runs = [_autograd_run(ours, d, 21, aux) for _ in range(2)]
    default = _autograd_run(ours, d, 21, aux)
    for k in runs[0]:
        assert torch.isfinite(runs[0][k]).all() and float(runs[0][k].abs().max()) > 0, k
        assert torch.equal(runs[0][k].view(torch.int32), runs[1][k].view(torch.int32)), k
        scale = float(runs[0][k].abs().max())
        torch.testing.assert_close(default[k], runs[0][k], rtol=1e-3, atol=1e-3 * scale)


def test_empty_cloud_gives_zero_images(ours):
    d = _small(8, 40, 24, 2)
    for k in ("means3D", "opacities", "scales", "rotations", "colors_precomp"):
        d[k] = d[k][:0]
    rs = util.settings_for(ours, d, DEV)
    t = {k: d[k].to(DEV) for k in util.TENSOR_KEYS if d[k] is not None}
    color, radii, depth, alpha, median = ours.GaussianRasterizer(rs).forward_opacity(
        means2D=torch.zeros_like(t["means3D"]), **t)
    assert float(alpha.abs().max()) == 0 and float(median.abs().max()) == 0


# ---- render() and render_pixels() -----------------------------------------------------------------------------------
def _model(P=30_000, seed=3, fine=True):
    from ref_ext import ref_deform_args
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.deformation import deform_network
    from s3gaussian_b200.gaussian_model import GaussianModel
    dev = torch.device(DEV)
    cloud = syn.make_cloud(P, seed=seed)
    net = None
    if fine:
        net = deform_network(ref_deform_args(syn.DEFAULT_RESOLUTION, syn.DEFAULT_MULTIRES))
        net.deformation_net.set_aabb(*[list(x) for x in syn.WAYMO_AABB])
    g = GaussianModel(3, deformation=net).create_from_tensors(
        cloud.xyz.to(dev), cloud.features_dc.to(dev), cloud.features_rest.to(dev), cloud.scaling.to(dev),
        cloud.rotation.to(dev), cloud.opacity.to(dev))
    g.active_sh_degree = 3
    if fine:
        g._deformation.to(dev)
    return g


RENDER_CASES = [("coarse", False, False), ("fine", False, False), ("fine", True, False), ("fine", False, True),
                ("fine", True, True)]


@pytest.mark.parametrize("stage,feat,decomp", RENDER_CASES)
@pytest.mark.parametrize("grad", [False, True])
def test_render_switch(stage, feat, decomp, grad, ours):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_renderer import (PipelineParams, dynamic_mask_of, fine_front, raster_settings_for,
                                                   render)
    g = _model(fine=stage == "fine")
    cam = syn.waymo_ring(320, 208, frames=10)[4].to(DEV)
    bg = torch.tensor([0.2, 0.1, 0.3], device=DEV)
    off, on = PipelineParams(), PipelineParams()
    on.render_opacity = True
    with torch.set_grad_enabled(grad):
        r_off = render(cam, g, off, bg, stage=stage, render_feat=feat, return_decomposition=decomp, return_dx=True)
        r_on = render(cam, g, on, bg, stage=stage, render_feat=feat, return_decomposition=decomp, return_dx=True)
    extra = {"alpha", "median_depth"} | ({"alpha_d", "alpha_s"} if decomp and stage == "fine" else set())
    assert set(r_on) == set(r_off) | extra and not (set(r_off) & extra)
    for k, v in r_off.items():
        if isinstance(v, torch.Tensor) and k != "viewspace_points":
            assert torch.equal(v, r_on[k]), k
    # the images are forward_opacity's on the same inputs
    with torch.no_grad():
        rs = raster_settings_for(cam, g, on, bg)
        rast = ours.GaussianRasterizer(rs)
        if stage == "coarse":
            geo = dict(means3D=g.get_xyz, shs=g.get_features, scales=g.scaling_activation(g._scaling),
                       rotations=g.rotation_activation(g._rotation), opacities=g.opacity_activation(g._opacity))
            aux = None
        else:
            means3D, scales, rotations, opacity, shs, colors_precomp, dx, _, featc = fine_front(cam, g, on, rs.campos,
                                                                                               g.get_features)
            geo = dict(means3D=means3D, shs=shs, colors_precomp=colors_precomp, scales=scales, rotations=rotations,
                       opacities=opacity)
            aux = featc if feat else None
        m2d = torch.zeros_like(geo["means3D"])
        ref = rast.forward_opacity(means2D=m2d, colors_aux=aux, **geo)
        assert torch.equal(r_on["alpha"], ref[3]) and torch.equal(r_on["median_depth"], ref[4])
        if "alpha_d" in extra:
            mask = dynamic_mask_of(dx)
            for key, m in (("alpha_d", mask), ("alpha_s", ~mask)):
                sub = {k: v[m] if v is not None else None for k, v in geo.items()}
                assert torch.equal(r_on[key], rast.forward_opacity(means2D=m2d[m], **sub)[3]), key
    if grad:
        (r_on["alpha"].sum() + r_on["median_depth"].mean() + r_on["render"].sum()).backward()
        assert torch.isfinite(g._xyz.grad).all() and float(g._opacity.grad.abs().max()) > 0


def test_render_pixels_fills_the_opacity_lists(ours):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.evaluation import render_pixels
    from s3gaussian_b200.gaussian_renderer import PipelineParams, render
    g = _model()
    cams = syn.waymo_ring(160, 112, frames=2)[:5]      # five views: the walks also carry flow sets
    for c in cams:
        c.original_image = torch.rand(3, 112, 160)
    bg, pipe = torch.zeros(3, device=DEV), PipelineParams()
    base = render_pixels(cams, g, bg, pipe, compute_metrics=False)
    res = render_pixels(cams, g, bg, pipe, compute_metrics=False, with_opacity=True)
    assert base["opacities"] == [] and "median_depths" not in base and "static_opacities" not in base
    for k in ("rgbs", "depths", "static_rgbs", "dynamic_rgbs"):
        assert all(np.array_equal(a, b) for a, b in zip(base[k], res[k])), k
    on = PipelineParams()
    on.render_opacity = True
    for key in ("opacities", "median_depths", "static_opacities", "dynamic_opacities"):
        assert len(res[key]) == len(cams) and all(a.shape == (112, 160) for a in res[key]), key
    with torch.no_grad():
        for i, c in enumerate(cams):
            r = render(c, g, on, bg, stage="fine", return_decomposition=True)
            for key, rk in (("opacities", "alpha"), ("median_depths", "median_depth"),
                            ("dynamic_opacities", "alpha_d"), ("static_opacities", "alpha_s")):
                assert np.array_equal(res[key][i], r[rk][0].cpu().numpy()), (key, i)
