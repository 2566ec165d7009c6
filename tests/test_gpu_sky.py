"""GPU: the sky model (s3g_sky_*, s3gaussian_b200.sky) against the float64 restatement in tests/sky_ref.py and the
goldens made from the reference module.

1. Forward and every weight / bias gradient within 1e-4 of each tensor's max, widths 64, 128 and 256, sizes 1x1,
   37x23, 960x640 and 1920x1280, with a rotated c2w, fx != fy and an off-centre principal point; and every golden.
2. Two backward calls bitwise equal; no host synchronisation in the forward or the backward.
3. A forward under grad keeps no per-pixel memory but its output until the backward.
4. sky_camera: a point along each pixel's sky direction projects through full_proj_transform onto the pixel's centre.
5. render -> composite -> loss backward against the same composite built with the torch float32 restatement, and
   bitwise repeatable under torch.use_deterministic_algorithms in the coarse stage.
6. Twenty Adam steps fitting the sky alone follow the torch float32 restatement's loss trajectory.
7. render_pixels with and without sky_model; examples/train_loop.py --sky.
"""
import glob
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import sky_ref as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(1, 1), (37, 23), (960, 640), (1920, 1280)]       # (W, H)


def _bar(got, want, rel=1e-4):
    err = float((got.double() - want.double()).abs().max())
    scale = float(want.double().abs().max())
    assert err <= rel * max(scale, 1e-30), (err, scale)


def _camera(W, H, seed):
    g = torch.Generator().manual_seed(seed)
    A = torch.linalg.qr(torch.randn(3, 3, generator=g, dtype=torch.float64))[0]
    c2w = torch.eye(4, dtype=torch.float64)
    c2w[:3, :3] = A * torch.sign(torch.det(A))
    c2w[:3, 3] = torch.randn(3, generator=g, dtype=torch.float64)
    f = 0.8 * max(W, H)
    K = torch.tensor([[f, 0, 0.37 * W], [0, 1.3 * f, 0.61 * H], [0, 0, 1]], dtype=torch.float64)
    return c2w.float().to(DEV), K.float().to(DEV)


def _model(width, W, H, seed):
    from s3gaussian_b200.sky import Background_Model
    torch.manual_seed(seed)
    m = Background_Model(img_width=W, img_height=H, model_cfg={"mlp_width": width}).to(DEV)
    with torch.no_grad():
        for p in m.parameters():
            if p.dim() == 2:
                p.normal_(0.0, 1.5 / math.sqrt(p.shape[1]))
            elif p.numel() > 5:
                p.normal_(0.0, 0.2)
    return m


def _params(m):
    lay = m.sky_model.sky_head.layers
    return [lay[0].weight, lay[0].bias, lay[1].weight, lay[1].bias, lay[2].weight, lay[2].bias]


def _run(m, c2w, K, g):
    out = m(c2w, K)
    grads = torch.autograd.grad(out, _params(m), g)
    return out.detach(), grads


@pytest.mark.parametrize("size", SIZES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("width", [64, 128, 256])
def test_against_float64(width, size):
    W, H = size
    m = _model(width, W, H, seed=width + W)
    c2w, K = _camera(W, H, seed=W + 3)
    # a loss gradient with a mean, as a photometric loss has: with a zero-mean one the weight gradients are sums that
    # cancel to ~sqrt(HW) terms, and the few pixels whose pre-activation lies within fp32 rounding of a ReLU's kink
    # (their mask differs between fp32 and float64, in torch's float32 as here) stand out against that
    g = 0.5 + torch.randn(3, H, W, device=DEV)
    out, grads = _run(m, c2w, K, g)
    want, wgrads = ref.sky_grads64([p.detach() for p in _params(m)], c2w, K, H, W, g)
    _bar(out, want)
    for a, b in zip(grads, wgrads):
        _bar(a, b)
    # two backward calls are bitwise equal
    _, grads2 = _run(m, c2w, K, g)
    assert all(torch.equal(a, b) for a, b in zip(grads, grads2))


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "sky_*.npz"))),
                         ids=os.path.basename)
def test_against_the_reference_goldens(path):
    from s3gaussian_b200.sky import Background_Model
    z = np.load(path)
    H, W = int(z["H"]), int(z["W"])
    m = Background_Model(img_width=W, img_height=H, model_cfg={"mlp_width": int(z["width"])})
    with torch.no_grad():
        for i, lay in enumerate(m.sky_model.sky_head.layers):
            lay.weight.copy_(torch.from_numpy(z[f"w{i}"]))
            lay.bias.copy_(torch.from_numpy(z[f"b{i}"]))
    m = m.to(DEV)
    out, grads = _run(m, torch.from_numpy(z["c2w"]).to(DEV), torch.from_numpy(z["intrinsic"]).to(DEV),
                      torch.from_numpy(z["dL_dsky"]).to(DEV))
    _bar(out.cpu(), torch.from_numpy(z["sky"]))
    for got, name in zip(grads, ("grad_w0", "grad_b0", "grad_w1", "grad_b1", "grad_w2", "grad_b2")):
        _bar(got.cpu(), torch.from_numpy(z[name]))


def test_no_host_synchronisation_and_memory_kept():
    W, H = 960, 640
    m = _model(256, W, H, seed=1)
    c2w, K = _camera(W, H, seed=2)
    g = torch.randn(3, H, W, device=DEV)
    _run(m, c2w, K, g)                      # warm: library load, allocator
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = m(c2w, K)
        kept = torch.cuda.memory_allocated() - before
        grads = torch.autograd.grad(out, _params(m), g)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    # the output itself (3 x H x W floats) is all a forward under grad keeps until the backward
    assert kept <= 3 * H * W * 4 + 4096, kept
    assert all(torch.isfinite(x).all() for x in grads)


def test_sky_camera_directions_project_onto_pixel_centres():
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.sky import sky_camera
    for cam in syn.waymo_ring(96, 64, frames=2)[:4]:
        c2w, K = sky_camera(cam)
        H, W = cam.image_height, cam.image_width
        v = ref.directions(c2w, K, H, W)
        centre = c2w[:3, 3].double()
        pts = centre + 7.0 * v
        hom = torch.cat([pts, torch.ones(H * W, 1, dtype=torch.float64)], 1) @ cam.full_proj_transform.double()
        ndc = hom[:, :2] / hom[:, 3:4]
        px = ((ndc[:, 0] + 1.0) * W - 1.0) * 0.5
        py = ((ndc[:, 1] + 1.0) * H - 1.0) * 0.5
        pix = torch.arange(H * W)
        assert float((px - (pix % W).double()).abs().max()) < 1e-3
        assert float((py - (pix // W).double()).abs().max()) < 1e-3


def _scene(seed=0):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_model import GaussianModel
    cloud = syn.make_cloud(20000, seed=seed, width=320, height=200)
    gm = GaussianModel(3).create_from_tensors(*(t.to(DEV) for t in (cloud.xyz, cloud.features_dc, cloud.features_rest,
                                                                      cloud.scaling, cloud.rotation, cloud.opacity)))
    gm.active_sh_degree = 3
    cam = syn.waymo_ring(320, 200, frames=2)[0].to(DEV)
    return gm, cam


def _torch_sky(params, c2w, K, H, W):
    """The torch float32 restatement: get_directions, the encoding and the nn.Linear chain, through autograd."""
    W0, b0, W1, b1, W2, b2 = params
    v = ref.directions(c2w, K, H, W).float()
    xb = torch.cat([v * s for s in ref.SCALES], -1)
    e = torch.cat([v, torch.sin(torch.cat([xb, xb + 0.5 * torch.pi], -1))], -1)
    h1 = torch.relu(e @ W0.T + b0)
    h2 = torch.relu(torch.cat([h1, e], -1) @ W1.T + b1)
    return torch.sigmoid(h2 @ W2.T + b2).T.reshape(3, H, W)


def _composite_step(gm, cam, sky_fn, sky_params, target, mask):
    from s3gaussian_b200 import losses
    from s3gaussian_b200.gaussian_renderer import PipelineParams, render
    pipe = PipelineParams()
    pipe.render_opacity = True
    out = render(cam, gm, pipe, torch.zeros(3, device=DEV), stage="coarse")
    alpha = out["alpha"]
    image = out["render"] + (1.0 - alpha) * sky_fn()
    l1, ssim_value, _ = losses.image_loss_terms(image, target)
    loss = l1 + 0.2 * (1.0 - ssim_value) + 0.05 * torch.nn.functional.binary_cross_entropy(
        alpha.clamp(1e-6, 1 - 1e-6), 1.0 - mask)
    tensors = [gm._xyz, gm._features_dc, gm._opacity, *sky_params]
    return [t.clone() for t in torch.autograd.grad(loss, tensors)]


def test_render_composite_loss_against_torch_and_deterministic():
    from s3gaussian_b200.sky import sky_camera
    gm, cam = _scene()
    for p in (gm._xyz, gm._features_dc, gm._opacity):
        p.requires_grad_(True)
    H, W = cam.image_height, cam.image_width
    m = _model(64, W, H, seed=3)
    c2w, K = (t.to(DEV) for t in sky_camera(cam))
    g = torch.Generator().manual_seed(4)
    target = (torch.rand(3, H, W, generator=g) * 0.8 + 0.1).to(DEV)
    mask = (torch.rand(1, H, W, generator=g) < 0.3).float().to(DEV)
    ours = _params(m)
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    torch.use_deterministic_algorithms(True)
    try:
        a = _composite_step(gm, cam, lambda: m(c2w, K), ours, target, mask)
        b = _composite_step(gm, cam, lambda: m(c2w, K), ours, target, mask)
    finally:
        torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    tp = [p.detach().clone().requires_grad_(True) for p in ours]
    t = _composite_step(gm, cam, lambda: _torch_sky(tp, c2w, K, H, W), tp, target, mask)
    for x, y in zip(a, t):
        assert torch.isfinite(x).all()
        _bar(x, y, rel=1e-3)
    assert all(float(x.abs().max()) > 0 for x in a)


def test_adam_fit_follows_the_torch_trajectory():
    """P = 0: the render is empty, so the composite is the sky itself; 20 Adam steps on an analytic sky."""
    W, H = 160, 96
    m = _model(128, W, H, seed=5)
    c2w, K = _camera(W, H, seed=6)
    v = ref.directions(c2w, K, H, W).float().T.reshape(3, H, W)
    target = torch.stack([0.5 + 0.4 * v[2], 0.6 - 0.3 * v[0], 0.3 + 0.2 * v[1] * v[0]]).clamp(0, 1)
    ours = _params(m)
    theirs = [p.detach().clone().requires_grad_(True) for p in ours]
    runs = []
    for params, fn in ((ours, lambda: m(c2w, K)), (theirs, lambda: _torch_sky(theirs, c2w, K, H, W))):
        opt = torch.optim.Adam(params, lr=3e-3)
        losses = []
        for _ in range(20):
            loss = ((fn() - target) ** 2).mean()
            opt.zero_grad()
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        runs.append(losses)
    print("sky fit:", runs[0][0], "->", runs[0][-1])
    assert runs[0][-1] < 0.7 * runs[0][0]
    for a, b in zip(*runs):
        assert abs(a - b) <= 1e-3 * b, runs


def test_render_pixels_with_and_without_sky():
    import ref_ext
    from s3gaussian_b200 import evaluation
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.deformation import deform_network
    from s3gaussian_b200.gaussian_renderer import GaussianModelLite, PipelineParams, render
    from s3gaussian_b200.sky import sky_camera
    cloud = syn.make_cloud(5000, seed=2, width=160, height=96)
    net = deform_network(ref_ext.ref_deform_args(syn.DEFAULT_RESOLUTION, syn.DEFAULT_MULTIRES))
    net.deformation_net.set_aabb(*[list(a) for a in syn.WAYMO_AABB])
    net.load_state_dict(syn.make_deform_state(0, weight_scale=0.2), strict=False)
    gm = GaussianModelLite(cloud, net).to(DEV)
    cams = []
    for c in syn.waymo_ring(160, 96, frames=2)[:3]:
        c = c.to(DEV)
        c.original_image = torch.rand(3, 96, 160, device=DEV)
        c.dynamic_mask = torch.zeros(96, 160, dtype=torch.bool, device=DEV)
        cams.append(c)
    m = _model(64, 160, 96, seed=7)
    bg = torch.tensor([0.2, 0.3, 0.4], device=DEV)
    pipe = PipelineParams()
    plain = evaluation.render_pixels(cams, gm, bg, pipe, return_decomposition=False)
    with_sky = evaluation.render_pixels(cams, gm, bg, pipe, return_decomposition=False, sky_model=m)
    opa = PipelineParams()
    opa.render_opacity = True
    for i, c in enumerate(cams):
        with torch.no_grad():
            out = render(c, gm, opa, torch.zeros(3, device=DEV), stage="fine")
            want = out["render"] + (1 - out["alpha"]) * m(*sky_camera(c))
        np.testing.assert_allclose(with_sky["rgbs"][i], want.permute(1, 2, 0).cpu().numpy(), atol=2e-5)
        np.testing.assert_allclose(plain["depths"][i], with_sky["depths"][i], rtol=1e-5, atol=1e-6)
        assert not np.allclose(plain["rgbs"][i], with_sky["rgbs"][i])
    assert with_sky["opacities"] == [] and with_sky["psnr"] != plain["psnr"]


def test_train_loop_with_sky():
    cmd = [sys.executable, os.path.join(ROOT, "examples", "train_loop.py"), "--points", "20000", "--iters", "200",
           "--width", "480", "--height", "320", "--sky"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    rows = [(int(m.group(1)), float(m.group(2))) for m in re.finditer(r"iter\s+(\d+)\s+loss ([\d.]+)", r.stdout)]
    assert [it for it, _ in rows] == [50, 100, 150, 200], r.stdout
    assert rows[-1][1] < rows[0][1], rows
