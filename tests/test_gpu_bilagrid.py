"""GPU: the bilateral-grid slice and TV loss (s3g_bilagrid_*, s3gaussian_b200.bilateral_grid) against the float64
restatement in tests/bilagrid_ref.py.

1. Slice forward, grad_rgb and grad_grids within 1e-4 of each tensor's max, for grids (16,16,8), (1,1,1), (5,3,2) and
   (32,32,16) (GX, GY, L), images 960x640, 97x61 and 8x6, B = 1 and B = 3 with unsorted ids at N = 150, colours in
   [-0.2, 1.3] with exact 0 and 1 pixels.  Pixels whose luminance level lies within 1e-5 of an integer (where the
   z-gradient jumps) without being exactly black or white are nudged off it.  Rows of grids not sliced stay exactly
   0, and two backward calls are bitwise equal.
2. TV forward and backward against float64, bitwise repeatable.
3. A coarse render -> slice -> image_loss_terms backward, bitwise repeatable under torch.use_deterministic_algorithms.
4. Recovering three per-image affine colour transforms with FusedAdam on the grids alone.
5. examples/train_loop.py --bilateral-grid.
"""
import os
import re
import subprocess
import sys

import pytest
import torch

import bilagrid_ref as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N = 150
GRIDS = [(16, 16, 8), (1, 1, 1), (5, 3, 2), (32, 32, 16)]      # (GX, GY, L)
IMAGES = [(960, 640), (97, 61), (8, 6)]
IDS = {1: [73], 3: [149, 0, 73]}


def _bar(got, want, rel=1e-4):
    err = float((got.double() - want.double()).abs().max())
    scale = float(want.double().abs().max())
    assert err <= rel * max(scale, 1e-30), (err, scale)


def _module(shape, seed):
    from s3gaussian_b200.bilateral_grid import BilateralGrid
    GX, GY, L = shape
    m = BilateralGrid(N, grid_X=GX, grid_Y=GY, grid_W=L).to(DEV)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        m.grids.add_(0.3 * torch.randn(m.grids.shape, generator=g).to(DEV))
    return m


def _image(B, W, H, L, seed):
    g = torch.Generator().manual_seed(seed)
    rgb = torch.rand(B, 3, H, W, generator=g) * 1.5 - 0.2
    # the background: whole pixels of exact 0 and exact 1
    bgmask = torch.rand(B, 1, H, W, generator=g)
    rgb = torch.where(bgmask < 0.1, torch.zeros(()), torch.where(bgmask > 0.9, torch.ones(()), rgb))
    gray = 0.299 * rgb[:, 0] + 0.587 * rgb[:, 1] + 0.114 * rgb[:, 2]
    z = gray * (L - 1)
    near = ((z - z.round()).abs() < 1e-5) & (bgmask[:, 0] >= 0.1) & (bgmask[:, 0] <= 0.9)
    rgb = rgb + 1e-4 * near[:, None].float()
    return rgb.contiguous().to(DEV)


def _ref(m, rgb, ids, go):
    G = m.grids.detach().double().requires_grad_(True)
    x = rgb.double().requires_grad_(True)
    out = ref.slice64(G, x, ids)
    gG, gx = torch.autograd.grad(out, (G, x), go.double())
    return out.detach(), gx, gG


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("size", IMAGES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("shape", GRIDS, ids=lambda s: "x".join(map(str, s)))
def test_slice_against_float64(shape, size, B):
    W, H = size
    m = _module(shape, seed=hash((shape, B)) % 1000)
    rgb = _image(B, W, H, shape[2], seed=W + B)
    ids = IDS[B]
    x = rgb.clone().requires_grad_(True)
    out = m.slice(x, ids)
    go = torch.randn(out.shape, generator=torch.Generator().manual_seed(3)).to(DEV)
    gx, gG = torch.autograd.grad(out, (x, m.grids), go)
    want, wgx, wgG = _ref(m, rgb, ids, go)
    _bar(out.detach(), want)
    _bar(gx, wgx)
    _bar(gG[ids], wgG[ids])
    others = torch.ones(N, dtype=torch.bool)
    others[ids] = False
    assert float(gG[others.to(DEV)].abs().max()) == 0.0
    # repeatable bit for bit
    gx2, gG2 = torch.autograd.grad(m.slice(x, ids), (x, m.grids), go)
    assert torch.equal(gx, gx2) and torch.equal(gG, gG2)


def test_slice_shapes_and_no_grad():
    m = _module((16, 16, 8), 1)
    rgb = _image(1, 40, 30, 8, 2)[0]
    out = m.slice(rgb, 5)
    assert out.shape == rgb.shape and out.grad_fn is not None
    with torch.no_grad():
        out2 = m.slice(rgb, 5)
    assert out2.grad_fn is None and torch.equal(out.detach(), out2)
    m.grids.requires_grad_(False)
    out3 = m.slice(rgb, [5])
    assert out3.grad_fn is None and torch.equal(out3, out2)
    # grad through rgb only
    m.grids.requires_grad_(False)
    x = rgb.clone().requires_grad_(True)
    (gx,) = torch.autograd.grad(m.slice(x, 5).sum(), x)
    _, wgx, _ = _ref(m, rgb[None], [5], torch.ones(1, 3, 30, 40, device=DEV))
    _bar(gx, wgx[0])
    # the identity grid gives back its input
    from s3gaussian_b200.bilateral_grid import BilateralGrid
    ident = BilateralGrid(2).to(DEV)
    torch.testing.assert_close(ident.slice(rgb, 1), rgb, rtol=0, atol=1e-6)


@pytest.mark.parametrize("shape", GRIDS, ids=lambda s: "x".join(map(str, s)))
def test_tv_against_float64(shape):
    m = _module(shape, 11)
    loss = m.tv_loss()
    (g,) = torch.autograd.grad(10.0 * loss, m.grids)
    G = m.grids.detach().double().requires_grad_(True)
    want = ref.tv64(G)
    (wg,) = torch.autograd.grad(10.0 * want, G)
    assert loss.dtype == torch.float32 and loss.shape == ()
    lf, lw = float(loss.detach()), float(want.detach())
    assert abs(lf - lw) <= 1e-5 * max(abs(lw), 1e-30), (lf, lw)
    _bar(g, wg)
    loss2 = m.tv_loss()
    (g2,) = torch.autograd.grad(10.0 * loss2, m.grids)
    assert torch.equal(loss, loss2) and torch.equal(g, g2)


def _scene(seed=0):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_model import GaussianModel
    cloud = syn.make_cloud(20000, seed=seed, width=320, height=200)
    gm = GaussianModel(3).create_from_tensors(*(t.to(DEV) for t in (cloud.xyz, cloud.features_dc, cloud.features_rest,
                                                                      cloud.scaling, cloud.rotation, cloud.opacity)))
    gm.active_sh_degree = 3
    cam = syn.waymo_ring(320, 200, frames=2)[0].to(DEV)
    return gm, cam


def _step(gm, cam, bil, target):
    from s3gaussian_b200 import losses
    from s3gaussian_b200.gaussian_renderer import PipelineParams, render
    for p in (gm._xyz, gm._features_dc, gm._opacity, bil.grids):
        p.grad = None
    out = render(cam, gm, PipelineParams(), torch.zeros(3, device=DEV), stage="coarse")
    image = bil.slice(out["render"], 2)
    l1, ssim_value, _ = losses.image_loss_terms(image, target)
    loss = l1 + 0.2 * (1.0 - ssim_value) + 10.0 * bil.tv_loss()
    loss.backward()
    return [p.grad.clone() for p in (gm._xyz, gm._features_dc, gm._opacity, bil.grids)]


def test_render_slice_loss_end_to_end_and_deterministic():
    gm, cam = _scene()
    for p in (gm._xyz, gm._features_dc, gm._opacity):
        p.requires_grad_(True)
    bil = _module((16, 16, 8), 5)
    with torch.no_grad():
        from s3gaussian_b200.gaussian_renderer import PipelineParams, render
        target = render(cam, gm, PipelineParams(), torch.zeros(3, device=DEV), stage="coarse")["render"] * 1.1 + 0.02
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    torch.use_deterministic_algorithms(True)
    try:
        a = _step(gm, cam, bil, target)
        b = _step(gm, cam, bil, target)
    finally:
        torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
    for x, y in zip(a, b):
        assert torch.isfinite(x).all() and torch.equal(x, y)
    assert float(a[0].abs().max()) > 0 and float(a[3][2].abs().max()) > 0
    others = torch.ones(N, dtype=torch.bool, device=DEV)
    others[2] = False
    # only the TV term reaches the other rows
    (tvg,) = torch.autograd.grad(10.0 * bil.tv_loss(), bil.grids)
    assert torch.equal(a[3][others], tvg[others])


def test_fit_recovers_per_image_affine_transforms():
    """Three images, each the same random colours under a known affine 3x4 transform; the grids alone, FusedAdam at
    lr 0.01 for 400 steps on the L2 loss, must reproduce every target to a mean absolute error below 2e-3 (the
    identity starts above 0.05)."""
    from s3gaussian_b200.bilateral_grid import BilateralGrid
    from s3gaussian_b200.optim import FusedAdam
    g = torch.Generator().manual_seed(0)
    rgb = (torch.rand(3, 3, 64, 96, generator=g) * 0.9 + 0.05).to(DEV)
    M = torch.eye(3, 4).repeat(3, 1, 1) + 0.15 * torch.randn(3, 3, 4, generator=g)
    M = M.to(DEV)
    target = torch.einsum("bij,bjhw->bihw", M[:, :, :3], rgb) + M[:, :, 3, None, None]
    bil = BilateralGrid(3, grid_X=8, grid_Y=8, grid_W=4).to(DEV)
    opt = FusedAdam([{"params": [bil.grids], "lr": 0.01, "name": "bilagrid"}], lr=0.01, eps=1e-15)
    start = float((bil.slice(rgb, [0, 1, 2]) - target).abs().mean())
    for _ in range(400):
        order = [2, 0, 1]
        loss = ((bil.slice(rgb[order].contiguous(), order) - target[order]) ** 2).mean()
        loss.backward()
        opt.step()
        opt.zero_grad(set_to_none=True)
    with torch.no_grad():
        err = float((bil.slice(rgb, [0, 1, 2]) - target).abs().mean())
    print(f"fit: mean |error| {start:.4f} -> {err:.6f}")
    assert start > 0.05 and err < 2e-3, (start, err)


def test_train_loop_with_bilateral_grid():
    cmd = [sys.executable, os.path.join(ROOT, "examples", "train_loop.py"), "--points", "20000", "--iters", "200",
           "--width", "480", "--height", "320", "--bilateral-grid"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    rows = [(int(m.group(1)), float(m.group(2))) for m in re.finditer(r"iter\s+(\d+)\s+loss ([\d.]+)", r.stdout)]
    assert [it for it, _ in rows] == [50, 100, 150, 200], r.stdout
    assert rows[-1][1] < rows[0][1], rows
