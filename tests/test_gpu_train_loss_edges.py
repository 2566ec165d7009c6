"""GPU (run with -m gpu): the fused image loss (L1 + SSIM + masked depth L2, csrc/train_step.cuh) and the HexPlane
regulariser against the float64 oracle (oracle/train_oracle.py, pinned to the reference by test_oracle_train.py)
run on the device, where a stencil or reduction kernel goes wrong: 1-pixel, window-sized and tile +/- 1 images,
C in {1, 3, 4} and up to 12 planes, every entry point backwarded on its own, depth exactly on the mask and clamp
bounds, non-contiguous / channels_last / unbatched inputs, and regulariser planes at the stencil ends, the
1024-float4 block chunk and the 48-plane table.  Nothing here needs oracle/_ref.

Bars, from the arithmetic of the kernels (float32 separable stencils, float32 per-block partial sums of at most a
few thousand terms, one reduction of the partials in double, scalars divided in double):
  * scalars: L1 and depth L2 within 1e-6 absolute: means of values <= 1.5^2 summed in float32 over <= 4096
    terms per block (relative rounding <~ 1e-7) and in double across blocks.  SSIM within 1e-5: each map value
    carries the cancellation of sigma = E[x^2] - mu^2 (float32, ~1e-7 absolute) against D >= C2 = 9e-4.
  * gradients, max |ours - oracle| over max |oracle|: 1e-4 on the SSIM path (the derivative maps inherit the same
    sigma cancellation, and the backward is a second 11+11-tap float32 stencil); 1e-6 where only the L1 term
    reaches the image (sign(x - y) is exact in float32, the only rounding is of w/N); 1e-5 for depth.
  * element-wise: |ours - oracle| <= rel * |oracle| + floor, with
      SSIM path  rel 1e-4, floor 1e-5 * max|oracle|: a pixel's error is a few float32 ulps of its stencil terms,
                 which for these inputs stay within ~10x the largest gradient;
      L1 only    rel 1e-6, floor 0: the same sign and the same w/N everywhere, exact zeros where x == y;
      depth      rel 1e-5, floor 2^-22 * 2|w| / (max_depth * #valid): q = pred/max_depth and b = gt/max_depth
                 are float32 values in [0, 1], each rounded once, and q - b once more.
Flat images (sigma = 0, test_constant_images) are the one place where the float32 cancellation in
sigma = E[x^2] - mu^2 against C2 exceeds the SSIM bars; that test states its own bars from the same arithmetic.
"""
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_golden_train as mg                  # noqa: E402 (input generators only)
from oracle import train_oracle as tro          # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

SSIM_BAR, SSIM_REL, SSIM_FLOOR = 1e-4, 1e-4, 1e-5
L1_BAR, L1_REL = 1e-6, 1e-6
DEPTH_BAR, DEPTH_REL = 1e-5, 1e-5


def check_grad(got, want, bar, rel, floor, what):
    """max-norm error <= bar * max|want| and element-wise |got - want| <= rel |want| + floor (absolute)."""
    assert got is not None and tuple(got.shape) == tuple(want.shape), (what, None if got is None else got.shape)
    got, want = got.detach().double(), want.detach().double()
    err = (got - want).abs()
    m = float(want.abs().max())
    e_max = float(err.max()) / m if m > 0 else float(err.max())
    need = float((err - rel * want.abs()).max())
    assert e_max <= bar, f"{what}: max error {e_max:.3e} of max|oracle| (bar {bar:.0e})"
    assert need <= floor, f"{what}: element-wise needs an absolute floor {need:.3e} = {need / max(m, 1e-300):.3e} " \
                          f"of max|oracle| (floor {floor:.3e})"


def check_ssim_grad(got, want, what):
    check_grad(got, want, SSIM_BAR, SSIM_REL, SSIM_FLOOR * float(want.abs().max()), what)


def check_l1_grad(got, want, what):
    check_grad(got, want, L1_BAR, L1_REL, 0.0, what)


def check_depth_grad(got, want, w, gt_depth, max_depth, what):
    gtd = gt_depth.double()
    cnt = int(((gtd > 0.01) & (gtd < max_depth)).sum())
    floor = 2.0 ** -22 * 2.0 * abs(w) / (max_depth * max(cnt, 1))
    check_grad(got, want, DEPTH_BAR, DEPTH_REL, floor, what)


def close(a, b, tol):
    """|a - b| < tol, or both NaN (the depth term of an image with no valid depth pixel)."""
    a, b = float(a), float(b)
    return (math.isnan(a) and math.isnan(b)) or abs(a - b) < tol


def check_scalars(ours, ref, what):
    for name, u, v, tol in zip(("l1", "ssim", "depth_l2"), ours, ref, (1e-6, 1e-5, 1e-6)):
        assert close(u, v, tol), (what, name, float(u), float(v))


def inputs(B, C, H, W, seed):
    return [t.to(DEV) for t in mg.loss_inputs(B, C, H, W, seed)]


def leaf(t, dtype=None):
    return t.detach().to(dtype or t.dtype).clone().requires_grad_(True)


def oracle_terms(x, gt, d, gt_depth, max_depth=80.0):
    """The oracle's three terms in float64 on the device; x and d are float64 leaves (or None)."""
    l1 = tro.l1_mean(x, gt.double()) if x is not None else torch.zeros((), dtype=torch.float64, device=DEV)
    ss = tro.ssim_mean(x, gt.double()) if x is not None else torch.zeros((), dtype=torch.float64, device=DEV)
    dl2 = tro.depth_l2(d, gt_depth.double(), max_depth) if d is not None else \
        torch.zeros((), dtype=torch.float64, device=DEV)
    return l1, ss, dl2


def grad_of(out, inp, w=1.0):
    return torch.autograd.grad(out, inp, grad_outputs=torch.full_like(out, w), retain_graph=True)[0]


# ---- shape matrix ----------------------------------------------------------------------------------------------
# every size appears as H and as W, non-square, with (B, C) cycling through {1, 3} x {1, 3, 4}; (3, 3, 33, 97) and
# (3, 4, 65, 11) cross tile boundaries with the 42-wide halo on up to 12 planes
SIZES = (1, 5, 10, 11, 12, 31, 32, 33, 42, 43, 64, 65, 97)
BC = ((1, 1), (3, 3), (1, 4), (3, 1), (1, 3), (3, 4))
SHAPES = [(*BC[i % 6], h, SIZES[(i + 5) % len(SIZES)]) for i, h in enumerate(SIZES)] + \
         [(1, 3, 1, 1), (3, 4, 11, 11), (1, 1, 32, 32), (3, 3, 43, 42)]


@pytest.mark.parametrize("B,C,H,W", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
def test_loss_terms_and_each_gradient_against_oracle(B, C, H, W, built_lib):
    from s3gaussian_b200 import losses
    img, gt, depth, gt_depth = inputs(B, C, H, W, 100 + H * 7 + W)
    x, d = leaf(img), leaf(depth)
    ours = losses.image_loss_terms(x, gt, d, gt_depth)
    xo, do = leaf(img, torch.float64), leaf(depth, torch.float64)
    ref = oracle_terms(xo, gt, do, gt_depth)
    what = f"{B}x{C}x{H}x{W}"
    check_scalars(ours, ref, what)
    # each term's gradient on its own: upstream weights (1, 0, 0), (0, 1, 0), (0, 0, 1)
    check_l1_grad(grad_of(ours[0], x), grad_of(ref[0], xo), what + " dl1/dx")
    check_ssim_grad(grad_of(ours[1], x), grad_of(ref[1], xo), what + " dssim/dx")
    check_depth_grad(grad_of(ours[2], d), grad_of(ref[2], do), 1.0, gt_depth, 80.0, what + " ddepth/dd")
    assert float(grad_of(ours[2], x).abs().max()) == 0.0 and float(grad_of(ours[0], d).abs().max()) == 0.0
    # the training combination
    loss = losses.training_loss(x, gt, d, gt_depth)
    rloss = tro.training_loss(xo, gt.double(), do, gt_depth.double())
    assert close(loss, rloss, 1e-5), (what, loss.item(), rloss.item())
    check_ssim_grad(grad_of(loss, x), grad_of(rloss, xo), what + " dloss/dx")


def test_four_full_size_views_against_oracle(built_lib):
    """B = 4 at 1280x1920: 12 planes, B*C*H*W = 29.5 M > 2^24."""
    from s3gaussian_b200 import losses
    img, gt, depth, gt_depth = inputs(4, 3, 1280, 1920, 6)
    x, d = leaf(img), leaf(depth)
    ours = losses.image_loss_terms(x, gt, d, gt_depth)
    loss = ours[0] + 0.5 * ours[2] + 0.2 * (1.0 - ours[1])
    loss.backward()
    xo, do = leaf(img, torch.float64), leaf(depth, torch.float64)
    ref = oracle_terms(xo, gt, do, gt_depth)
    check_scalars(ours, ref, "4x3x1280x1920")
    rloss = ref[0] + 0.5 * ref[2] + 0.2 * (1.0 - ref[1])
    rloss.backward()
    check_ssim_grad(x.grad, xo.grad, "4x3x1280x1920 dloss/dx")
    check_depth_grad(d.grad, do.grad, 0.5, gt_depth, 80.0, "4x3x1280x1920 dloss/dd")
    del xo, do, ref, rloss
    # the L1-only path at the same size
    x2, d2 = leaf(img), leaf(depth)
    losses.training_loss(x2, gt, d2, gt_depth, lambda_dssim=0.0).backward()
    n = img.numel()
    want = torch.sign(img.double() - gt.double()) / n
    check_l1_grad(x2.grad, want, "4x3x1280x1920 L1-only dloss/dx")
    assert torch.equal(d2.grad, d.grad)


# ---- every entry point ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lambda_dssim", [0.2, 0.0])
def test_training_loss_against_oracle(lambda_dssim, built_lib):
    from s3gaussian_b200 import losses
    for B, C, H, W in ((2, 3, 45, 70), (1, 3, 37, 53), (3, 1, 33, 97)):
        img, gt, depth, gt_depth = inputs(B, C, H, W, 21)
        x, d = leaf(img), leaf(depth)
        loss = losses.training_loss(x, gt, d, gt_depth, lambda_dssim=lambda_dssim, lambda_depth=0.5)
        loss.backward()
        xo, do = leaf(img, torch.float64), leaf(depth, torch.float64)
        rloss = tro.training_loss(xo, gt.double(), do, gt_depth.double(), lambda_dssim=lambda_dssim)
        rloss.backward()
        what = f"lambda_dssim={lambda_dssim} {B}x{C}x{H}x{W}"
        if lambda_dssim == 0:
            assert abs(loss.item() - rloss.item()) < 1e-6, (what, loss.item(), rloss.item())
            check_l1_grad(x.grad, xo.grad, what)
        else:
            assert abs(loss.item() - rloss.item()) < 1e-5, (what, loss.item(), rloss.item())
            check_ssim_grad(x.grad, xo.grad, what)
        check_depth_grad(d.grad, do.grad, 0.5, gt_depth, 80.0, what)


@pytest.mark.parametrize("with_ssim", [True, False])
def test_image_only_and_depth_only_calls(with_ssim, built_lib):
    """image_loss_terms with depth None (null depth pointers) and with image None (C = 0)."""
    from s3gaussian_b200 import losses
    img, gt, depth, gt_depth = inputs(2, 3, 40, 75, 22)
    x = leaf(img)
    l1, ss, dl2 = losses.image_loss_terms(x, gt, with_ssim=with_ssim)
    assert float(dl2) == 0.0
    xo = leaf(img, torch.float64)
    rl1, rss, _ = oracle_terms(xo, gt, None, None)
    assert abs(l1.item() - rl1.item()) < 1e-6
    if with_ssim:
        assert abs(ss.item() - rss.item()) < 1e-5
        (l1 - 0.3 * ss).backward()
        (rl1 - 0.3 * rss).backward()
        check_ssim_grad(x.grad, xo.grad, "image only")
    else:
        assert float(ss) == 0.0
        (2.0 * l1).backward()
        (2.0 * rl1).backward()
        check_l1_grad(x.grad, xo.grad, "image only, no SSIM")
    d = leaf(depth)
    l1, ss, dl2 = losses.image_loss_terms(None, None, d, gt_depth, with_ssim=with_ssim)
    assert float(l1) == 0.0 and float(ss) == 0.0
    do = leaf(depth, torch.float64)
    rdl2 = tro.depth_l2(do, gt_depth.double())
    assert abs(dl2.item() - rdl2.item()) < 1e-6
    (-3.0 * dl2).backward()
    (-3.0 * rdl2).backward()
    check_depth_grad(d.grad, do.grad, -3.0, gt_depth, 80.0, "depth only")


def test_reference_named_wrappers_each_backwarded(built_lib):
    """l1_loss, ssim and compute_depth each with its own backward, and two wrapper calls on one image summed."""
    from s3gaussian_b200 import losses
    img, gt, depth, gt_depth = inputs(1, 3, 50, 66, 23)
    xo_all = leaf(img, torch.float64)
    for name, fn, rfn, check in (("l1_loss", losses.l1_loss, tro.l1_mean, check_l1_grad),
                                 ("ssim", losses.ssim, tro.ssim_mean, check_ssim_grad)):
        x, xo = leaf(img), leaf(img, torch.float64)
        v, rv = fn(x, gt), rfn(xo, gt.double())
        assert abs(v.item() - rv.item()) < (1e-6 if name == "l1_loss" else 1e-5), name
        v.backward()
        rv.backward()
        check(x.grad, xo.grad, name)
    d, do = leaf(depth), leaf(depth, torch.float64)
    v, rv = losses.compute_depth("l2", d, gt_depth), tro.depth_l2(do, gt_depth.double())
    assert abs(v.item() - rv.item()) < 1e-6
    v.backward()
    rv.backward()
    check_depth_grad(d.grad, do.grad, 1.0, gt_depth, 80.0, "compute_depth")
    # two calls on the same image: autograd adds their gradients
    x = leaf(img)
    (losses.l1_loss(x, gt) + 0.7 * (1.0 - losses.ssim(x, gt))).backward()
    (tro.l1_mean(xo_all, gt.double()) + 0.7 * (1.0 - tro.ssim_mean(xo_all, gt.double()))).backward()
    check_ssim_grad(x.grad, xo_all.grad, "l1_loss + ssim")


@pytest.mark.parametrize("weights", [(-1.5, 0.0, -2.0), (0.0, -0.4, 0.0), (0.0, 0.0, 0.0), (2.5, 1.0, -0.25)])
def test_zero_and_negative_upstream_weights(weights, built_lib):
    from s3gaussian_b200 import losses
    img, gt, depth, gt_depth = inputs(2, 4, 35, 44, 24)
    x, d = leaf(img), leaf(depth)
    xo, do = leaf(img, torch.float64), leaf(depth, torch.float64)
    ours = losses.image_loss_terms(x, gt, d, gt_depth)
    ref = oracle_terms(xo, gt, do, gt_depth)
    gx, gd = torch.autograd.grad(ours, (x, d), [torch.tensor(w, device=DEV) for w in weights])
    rx, rd = torch.autograd.grad(ref, (xo, do), [torch.tensor(w, device=DEV, dtype=torch.float64) for w in weights])
    if weights == (0.0, 0.0, 0.0):
        assert float(gx.abs().max()) == 0.0 and float(gd.abs().max()) == 0.0
        return
    if weights[1] == 0.0:
        check_l1_grad(gx, rx, f"weights {weights}")
    else:
        check_ssim_grad(gx, rx, f"weights {weights}")
    if weights[2] == 0.0:
        assert float(gd.abs().max()) == 0.0
    else:
        check_depth_grad(gd, rd, weights[2], gt_depth, 80.0, f"weights {weights}")


# ---- depth mask and clamp bounds ---------------------------------------------------------------------------------
def depth_edges(B, H, W, max_depth, seed):
    """gt and pred [B, H, W] with pixels exactly on the mask bounds (0.01 and max_depth excluded, their neighbours
    towards the inside included) and on the clamp bounds (pred = 0 and max_depth pass the gradient, beyond do not)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    gt = (0.05 + 0.9 * torch.rand(B, H, W, device=DEV, generator=g)) * max_depth
    pred = (torch.rand(B, H, W, device=DEV, generator=g) * 1.2 - 0.1) * max_depth
    f32 = lambda v: torch.tensor(v, dtype=torch.float32, device=DEV)
    lo, hi = f32(0.01), f32(max_depth)
    gf, pf = gt.view(-1), pred.view(-1)
    edges = {
        0: (lo, None), 1: (torch.nextafter(lo, f32(1.0)), f32(0.0)), 2: (hi, None),
        3: (torch.nextafter(hi, f32(0.0)), f32(0.0)), 4: (f32(0.0), None), 5: (f32(-1.0), None),
        6: (2.0 * hi, None), 7: (None, f32(0.0)), 8: (None, hi), 9: (None, -0.5 * hi), 10: (None, 1.5 * hi),
        11: (torch.nextafter(lo, f32(1.0)), hi), 12: (torch.nextafter(hi, f32(0.0)), hi),
    }
    for i, (gv, pv) in edges.items():
        if gv is not None:
            gf[i] = gv
        if pv is not None:
            pf[i] = pv
    return pred, gt


@pytest.mark.parametrize("max_depth", [80.0, 1.0])
@pytest.mark.parametrize("layout", ["HW", "1HW", "B1HW"])
def test_depth_mask_and_clamp_bounds(layout, max_depth, built_lib):
    from s3gaussian_b200 import losses
    B = 3 if layout == "B1HW" else 1
    H, W = 9, 13
    pred, gt = depth_edges(B, H, W, max_depth, 31)
    shape = {"HW": (H, W), "1HW": (1, H, W), "B1HW": (B, 1, H, W)}[layout]
    pred, gt = pred.reshape(shape), gt.reshape(shape)
    # the mask decisions the edges were built for, in the oracle itself
    gf = gt.reshape(-1).double()
    valid = (gf > 0.01) & (gf < max_depth)
    assert valid[[1, 3, 11, 12]].all() and not valid[[0, 2, 4, 5, 6]].any()
    d, do = leaf(pred), leaf(pred, torch.float64)
    v = losses.compute_depth("l2", d, gt, max_depth=max_depth)
    rv = tro.depth_l2(do, gt.double(), max_depth)
    assert abs(v.item() - rv.item()) < 1e-6, (v.item(), rv.item())
    v.backward()
    rv.backward()
    what = f"depth {layout} max_depth={max_depth}"
    check_depth_grad(d.grad, do.grad, 1.0, gt, max_depth, what)
    gd, rd = d.grad.reshape(-1), do.grad.reshape(-1)
    assert tuple(d.grad.shape) == shape
    assert torch.equal(gd == 0, rd == 0), what                  # the same pixels pass the gradient
    assert (rd[[1, 3, 7, 8, 11]] != 0).all() and (rd[[0, 2, 4, 5, 6, 9, 10]] == 0).all()
    # the same depth with an image beside it (B from the image)
    img, gimg, _, _ = inputs(B, 3, H, W, 32)
    x, d2 = leaf(img), leaf(pred)
    l1, ss, dl2 = losses.image_loss_terms(x, gimg, d2, gt, max_depth=max_depth)
    assert dl2.item() == v.item()
    (0.5 * dl2 + l1).backward()
    check_depth_grad(d2.grad, 0.5 * do.grad, 0.5, gt, max_depth, what + " beside an image")


@pytest.mark.parametrize("with_ssim", [True, False])
def test_depth_with_no_valid_pixel_is_nan_with_zero_gradient(with_ssim, built_lib):
    """The reference's mean over an empty selection is NaN and its gradient zero."""
    from s3gaussian_b200 import losses
    img, gimg, depth, _ = inputs(2, 3, 20, 30, 33)
    gt = torch.zeros_like(depth)
    gt[0, 0, :5] = 80.0                      # excluded at the upper bound
    gt[1, 0, :5] = 0.01                      # excluded at the lower bound
    gt[1, 0, 5:7] = 1e4
    d, do = leaf(depth), leaf(depth, torch.float64)
    v = losses.compute_depth("l2", d, gt)
    rv = tro.depth_l2(do, gt.double())
    assert math.isnan(v.item()) and math.isnan(rv.item())
    v.backward()
    rv.backward()
    assert torch.equal(d.grad, torch.zeros_like(d)) and torch.equal(do.grad, torch.zeros_like(do))
    x, d2 = leaf(img), leaf(depth)
    loss = losses.training_loss(x, gimg, d2, gt, lambda_dssim=0.2 if with_ssim else 0.0)
    assert math.isnan(loss.item())
    loss.backward()
    assert torch.equal(d2.grad, torch.zeros_like(d2)) and bool(torch.isfinite(x.grad).all())
    xo = leaf(img, torch.float64)
    rl = tro.l1_mean(xo, gimg.double()) + (0.2 * (1.0 - tro.ssim_mean(xo, gimg.double())) if with_ssim else 0.0)
    rl.backward()
    (check_ssim_grad if with_ssim else check_l1_grad)(x.grad, xo.grad, "image beside an empty depth mask")


# ---- input layouts and values -------------------------------------------------------------------------------
def _compare_layout(x_ours, gt_ours, img, gt, what):
    from s3gaussian_b200 import losses
    l1, ss, _ = losses.image_loss_terms(x_ours, gt_ours)
    (l1 + 0.2 * (1.0 - ss)).backward()
    xo = leaf(img.reshape(1, *img.shape[-3:]) if img.dim() == 3 else img, torch.float64)
    g64 = (gt.reshape(1, *gt.shape[-3:]) if gt.dim() == 3 else gt).double()
    rl1, rss = tro.l1_mean(xo, g64), tro.ssim_mean(xo, g64)
    assert abs(l1.item() - rl1.item()) < 1e-6 and abs(ss.item() - rss.item()) < 1e-5, what
    (rl1 + 0.2 * (1.0 - rss)).backward()
    return xo.grad


def test_non_contiguous_channels_last_and_unbatched_inputs(built_lib):
    img, gt, _, _ = inputs(2, 3, 47, 61, 41)
    g = torch.Generator(device=DEV).manual_seed(41)
    # gt[:, :3] of a 4-channel tensor (train.py slices the alpha channel off); the image too
    gt4 = torch.cat([gt, torch.rand(2, 1, 47, 61, device=DEV, generator=g)], 1)
    img4 = leaf(torch.cat([img, torch.rand(2, 1, 47, 61, device=DEV, generator=g)], 1))
    assert not gt4[:, :3].is_contiguous()
    want = _compare_layout(img4[:, :3], gt4[:, :3], img, gt, "sliced")
    check_ssim_grad(img4.grad[:, :3], want, "sliced")
    assert float(img4.grad[:, 3].abs().max()) == 0.0
    # channels_last
    x = leaf(img.contiguous(memory_format=torch.channels_last))
    want = _compare_layout(x, gt.contiguous(memory_format=torch.channels_last), img, gt, "channels_last")
    check_ssim_grad(x.grad, want, "channels_last")
    # unbatched [3, H, W]: the gradient comes back in that shape
    x = leaf(img[1])
    want = _compare_layout(x, gt[1], img[1], gt[1], "unbatched")
    assert tuple(x.grad.shape) == (3, 47, 61)
    check_ssim_grad(x.grad, want[0], "unbatched")


def test_values_outside_unit_range(built_lib):
    from s3gaussian_b200 import losses
    g = torch.Generator(device=DEV).manual_seed(42)
    img = torch.rand(3, 3, 38, 70, device=DEV, generator=g) * 2.0 - 0.5
    gt = (img + 0.3 * torch.randn(img.shape, device=DEV, generator=g)).clamp(-0.5, 1.5)
    x = leaf(img)
    want = _compare_layout(x, gt, img, gt, "[-0.5, 1.5]")
    check_ssim_grad(x.grad, want, "[-0.5, 1.5]")
    assert losses.l1_loss(img, gt).item() == losses.l1_loss(gt, img).item()


@pytest.mark.parametrize("a,b", [(0.5, 0.5), (0.25, 0.75), (1.0, 0.0)])
def test_constant_images(a, b, built_lib):
    """sigma = 0 inside the image: only C2 keeps B and D away from zero, and the float32 arithmetic of the reference's
    formulation, not the kernel, sets the error.  sigma = E[x^2] - mu^2 cancels to ~eps (a + b)^2 absolute
    (eps = 2^-24), i.e. ~eps (a + b)^2 / C2 relative in each SSIM value and each derivative map; the gradient is
    the sum of three stencil terms, conv(dm/dmu1) + 2x conv(dm/dsig1) + y conv(dm/dsig12), of size T each (below)
    that cancel to ~1e-3 T.  The bars are the defaults or 8 float32 roundings of these magnitudes, whichever is
    wider.  Identical images: SSIM 1, B = D and A = C to rounding, so the gradient is rounding of T alone."""
    from s3gaussian_b200 import losses
    B, C, H, W = 2, 3, 40, 50
    eps, C1, C2 = 2.0 ** -24, 0.01 ** 2, 0.03 ** 2
    img = torch.full((B, C, H, W), a, device=DEV)
    gt = torch.full((B, C, H, W), b, device=DEV)
    x = leaf(img)
    l1, ss, _ = losses.image_loss_terms(x, gt)
    xo = leaf(img, torch.float64)
    rss = tro.ssim_mean(xo, gt.double())
    ss_bar = max(1e-5, 8 * eps * (abs(a) + abs(b)) ** 2 / C2 * abs(rss.item()))
    assert abs(ss.item() - rss.item()) <= ss_bar, (ss.item(), rss.item(), ss_bar)
    assert l1.item() == abs(a - b)
    ss.backward()
    rss.backward()
    # the three terms' size at an interior pixel (mu1 = a, mu2 = b, sigma = 0), times k = 1/N
    A, Cc = 2 * a * b + C1, a * a + b * b + C1
    dmu1 = 2 / (Cc * C2) * (b * (C2 - A) - a * A * C2 / Cc + a * A)
    T = (abs(dmu1) + 2 * abs(a) * A / (Cc * C2) + abs(b) * 2 * A / (Cc * C2)) / img.numel()
    if a == b:
        assert abs(ss.item() - 1.0) < 1e-6
        assert float(x.grad.abs().max()) <= 8 * eps * T, (float(x.grad.abs().max()), T)
        return
    m = float(xo.grad.abs().max())
    arith = 8 * eps * ((abs(a) + abs(b)) ** 2 / C2 + T / m)           # relative to max|oracle|
    check_grad(x.grad, xo.grad, max(SSIM_BAR, arith), SSIM_REL, max(SSIM_FLOOR, arith) * m, f"constant {a} vs {b}")


# ---- determinism -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_ssim", [True, False])
def test_forward_and_retained_backward_are_bitwise_repeatable(with_ssim, built_lib):
    """Block partials and one reducer, no atomics: the same sums on every call; the backward reads the derivative
    maps kept in the saved workspace, so a second backward of the same graph gives the same bits."""
    from s3gaussian_b200 import losses
    img, gt, depth, gt_depth = inputs(2, 3, 300, 430, 51)
    x, d = leaf(img), leaf(depth)
    first = losses.image_loss_terms(x, gt, d, gt_depth, with_ssim=with_ssim)
    again = losses.image_loss_terms(x, gt, d, gt_depth, with_ssim=with_ssim)
    for u, v in zip(first, again):
        assert torch.equal(u, v)
    loss = first[0] + 0.5 * first[2] + 0.2 * (1.0 - first[1])
    loss.backward(retain_graph=True)
    gx, gd = x.grad.clone(), d.grad.clone()
    x.grad, d.grad = None, None
    loss.backward(retain_graph=True)
    assert torch.equal(x.grad, gx) and torch.equal(d.grad, gd)
    # a forward in between (new derivative maps in a new workspace) does not disturb the retained graph
    other = losses.image_loss_terms(x, torch.flip(gt, (-1,)), d, gt_depth, with_ssim=with_ssim)
    x.grad, d.grad = None, None
    loss.backward()
    assert torch.equal(x.grad, gx) and torch.equal(d.grad, gd)
    del other


# ---- HexPlane regulariser ----------------------------------------------------------------------------------------
def _plane(H, W, Cc, g, offset=1.0):
    t = torch.rand(1, Cc, H, W, device=DEV, generator=g) * 0.8 + offset - 0.4      # straddles 1 for the L1 sign
    t.view(-1)[:: 7] = 1.0                                                         # |1 - t| at its kink
    return t.contiguous(memory_format=torch.channels_last).requires_grad_(True)


# (H, W, C): one second-difference row (H = 3); the 5-tap backward stencil reaching both ends (H = 4, 5); W = 1 and
# C = 4; 1023 / 1024 / 1025 float4 (one block chunk -1, 0, +1); chunks ending inside a row (7 x 300 x 8)
EDGE_PLANES = [(3, 1, 4), (3, 7, 8), (4, 5, 4), (5, 3, 12), (4, 1, 4), (5, 1, 4),
               (1023, 1, 4), (1024, 1, 4), (1025, 1, 4), (7, 300, 8), (3, 683, 4), (6, 2, 32)]


def _reg_check(levels, weights, upstream, what):
    from s3gaussian_b200 import regulation
    total = regulation.compute_regulation(levels, *weights)
    ref_levels = [[p.detach().double().requires_grad_(True) for p in lv] for lv in levels]
    ref = tro.compute_regulation(ref_levels, *weights)
    assert abs(total.item() - ref.item()) <= 2e-6 * abs(ref.item()), (what, total.item(), ref.item())
    (upstream * total).backward()
    (upstream * ref).backward()
    for l, (lv, rlv) in enumerate(zip(levels, ref_levels)):
        for k, (p, r) in enumerate(zip(lv, rlv)):
            if len(lv) == 3:
                assert p.grad is None, (what, "3-plane level", l)
                continue
            assert p.grad.stride() == p.stride(), (what, l, k, p.grad.stride(), p.stride())
            m = float(r.grad.abs().max())
            check_grad(p.grad, r.grad, 1e-5, 1e-4, 1e-6 * m, f"{what} level {l} plane {k} {tuple(p.shape)}")


@pytest.mark.parametrize("upstream", [1.0, -2.5, 0.0])
def test_plane_regulation_edges_against_oracle(upstream, built_lib):
    g = torch.Generator(device=DEV).manual_seed(61)
    levels = [[_plane(*s, g) for s in EDGE_PLANES[:6]],
              [_plane(*s, g) for s in (EDGE_PLANES[1], (4, 4, 4), (3, 9, 8))],      # 3 planes: no regulariser
              [_plane(*s, g) for s in EDGE_PLANES[6:]]]
    # weights chosen so that the smoothness and L1 parts of the gradient are of comparable size
    _reg_check(levels, (0.05, 0.02, 0.01), upstream, f"edges, upstream {upstream}")
    g2 = torch.Generator(device=DEV).manual_seed(62)
    single = _plane(5, 1, 4, g2)
    from s3gaussian_b200 import regulation
    v = regulation.compute_plane_smoothness(single)
    assert abs(v.item() - tro.plane_smoothness(single.detach().double()).item()) <= 2e-6 * abs(v.item())


def test_plane_regulation_48_planes_and_mixed_levels(built_lib):
    g = torch.Generator(device=DEV).manual_seed(63)
    shapes = EDGE_PLANES + [(8 + i, 3 + (i * 5) % 17, 4 * (1 + i % 4)) for i in range(36)]
    levels, it = [], iter(shapes)
    for l in range(10):
        if l in (2, 7):
            levels.append([_plane(4, 4, 4, g) for _ in range(3)])
        else:
            levels.append([_plane(*next(it), g) for _ in range(6)])
    assert sum(len(lv) for lv in levels if len(lv) == 6) == 48
    # the reference's default weights (time_smoothness 0.01, l1_time_planes 1e-4, plane_tv 1e-4)
    _reg_check(levels, (0.01, 0.0001, 0.0001), -1.0, "48 planes")
