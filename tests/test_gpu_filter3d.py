"""GPU: Mip-Splatting's 3-D smoothing filter (s3g_filter3d_compute / _apply_forward / _apply_backward, filter3d.py,
GaussianModel.compute_3D_filter, pipe.filter_3d).

1. The compute kernel against the float64 restatement (tests/filter3d_ref.py): Waymo-ring cameras, mixed camera sizes
   and focal lengths, Gaussians no camera sees, a cloud nobody sees, P = 0, C = 1, C beyond one shared-memory chunk,
   points 1e-3 either side of every threshold; repeat calls bitwise equal.
2. The apply kernels against the float64 formula, bitwise identity where f = 0, the integrated density kept.
3. render() / render_pixels() with the switch against the rasterizer on the filtered tensors, and gradients against
   autograd through a float32 torch restatement of the apply.
4. Densify, prune and spatial_sort carry filter_3D rows.
5. The property the filter exists for: a Gaussian far below its filter, seen 8x closer than in training.
"""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import filter3d_ref as ref
from test_gpu_raster_opacity import _model

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def f3d(built_lib):
    from s3gaussian_b200 import filter3d
    return filter3d


def _check_compute(f3d, xyz, cams, what, margin=1e-4):
    """Kernel vs restatement: within 1e-6 relative where every pair is > `margin` from a threshold; repeat calls
    bitwise equal.  Returns (kernel values, restated values, seen)."""
    xyz = xyz.to(DEV).float().contiguous()
    got = f3d.compute_filter_3d(xyz, cams)
    assert got.shape == (xyz.shape[0], 1) and got.dtype == torch.float32
    assert torch.equal(got, f3d.compute_filter_3d(xyz, cams)), what
    views, k = f3d.camera_tensors(cams, DEV)
    want, seen = ref.compute64(xyz, views, k)
    far = ref.margin64(xyz, views, k) > margin
    got = got[:, 0].double()
    err = ((got - want).abs() / want.abs().clamp_min(1e-30))[far]
    assert float(err.max()) <= 1e-6, (what, float(err.max()))
    return got, want, seen


def test_compute_on_the_waymo_ring(f3d):
    """2 x 10^5 Gaussians of make_cloud (10 % behind the first camera) x the 150 cameras of waymo_ring (three 64-camera
    chunks, the last one partial)."""
    from s3gaussian_b200 import synthetic as syn
    cams = syn.waymo_ring(1920, 1280, frames=50)
    got, want, seen = _check_compute(f3d, syn.make_cloud(200_000, seed=4).xyz, cams, "waymo ring")
    assert 0.5 < float(seen.double().mean()) < 0.999
    # the ones nobody sees take the largest seen value
    assert torch.equal(got[~seen], torch.full_like(got[~seen], float(got[seen].max())))


def test_compute_with_mixed_cameras(f3d):
    """Cameras of different sizes and focal lengths; F is the max focal_x over ALL cameras, including one that sees
    nothing of the cloud (it is 1 km above it)."""
    from s3gaussian_b200 import synthetic as syn
    cams = [syn.make_camera(640, 480, (0.0, 0.0, 2.0), focal=500.0), syn.make_camera(1920, 1080, (5.0, 1.0, 2.0),
                                                                                   yaw_deg=10.0, focal=1500.0),
            syn.make_camera(320, 640, (-3.0, -1.0, 1.5), yaw_deg=-5.0, pitch_deg=3.0, focal=300.0),
            syn.make_camera(800, 600, (0.0, 0.0, 1000.0), focal=4000.0)]
    xyz = syn.make_cloud(50_000, seed=5).xyz
    got, want, seen = _check_compute(f3d, xyz, cams, "mixed cameras")
    _, k = f3d.camera_tensors(cams, DEV)
    assert float(k[:, 2].max()) == float(k[3, 2])
    # the camera looking away sees nothing, yet sets F
    ok, _ = ref.valid64(xyz.to(DEV), *f3d.camera_tensors(cams[3:], DEV))
    assert not bool(ok.any())
    f_without = ref.compute64(xyz.to(DEV), *f3d.camera_tensors(cams[:3], DEV))[0]
    torch.testing.assert_close(want, f_without * float(k[:3, 2].max()) / float(k[3, 2]), rtol=1e-12, atol=0)


def test_compute_unseen_nobody_p0_c1_and_many_cameras(f3d):
    from s3gaussian_b200 import synthetic as syn
    cam = syn.make_camera(320, 240, (0.0, 0.0, 0.0), focal=300.0)
    g = torch.Generator().manual_seed(6)
    front = torch.stack([torch.empty(4000).uniform_(2, 30, generator=g), torch.empty(4000).uniform_(-5, 5, generator=g),
                         torch.empty(4000).uniform_(-3, 3, generator=g)], 1)
    behind = front * torch.tensor([-1.0, 1.0, 1.0])
    beside = front * torch.tensor([0.05, 1.0, 1.0]) + torch.tensor([0.0, 40.0, 0.0])
    xyz = torch.cat([front, behind, beside])
    got, want, seen = _check_compute(f3d, xyz, [cam], "C = 1")             # one camera
    assert bool(seen[:1000].any()) and not bool(seen[4000:].any())
    assert torch.equal(got[4000:], torch.full_like(got[4000:], float(got[seen].max())))
    got, _, seen = _check_compute(f3d, xyz[4000:], [cam], "nobody")           # nobody sees anything: zeros
    assert not bool(seen.any()) and torch.equal(got, torch.zeros_like(got))
    assert f3d.compute_filter_3d(torch.zeros(0, 3, device=DEV), [cam]).shape == (0, 1)   # P = 0
    # 200 cameras (three full 64-camera chunks and a partial one), each at its own position
    cams = [syn.make_camera(320, 240, (0.1 * i, 0.05 * (i % 7), 0.02 * (i % 5)), yaw_deg=0.2 * (i % 11),
                            focal=250.0 + i) for i in range(200)]
    _check_compute(f3d, xyz, cams, "C = 200")


def test_compute_threshold_decisions(f3d):
    """One camera with camera space = world space (W = 200, H = 100, focal 100): points 1e-3 (relative) inside and
    outside z > 0.2 and each of the four screen bounds.  Inside ones are valid (d = their z), outside ones are not
    (d = the anchor's 50)."""
    W, H, fpx = 200, 100, 100.0
    cam = SimpleNamespace(world_view_transform=torch.eye(4), image_width=W, image_height=H,
                          FoVx=2 * math.atan(W / (2 * fpx)), FoVy=2 * math.atan(H / (2 * fpx)))
    pts, inside = [[0.0, 0.0, 50.0]], [True]
    for e, ins in ((1e-3, True), (-1e-3, False)):
        pts.append([0.0, 0.0, 0.2 * (1 + e)])
        inside.append(ins)
        z = 5.0
        for axis, half, foc in ((0, 0.65 * W, fpx), (1, 0.65 * H, fpx)):
            for sign in (1.0, -1.0):
                p = [0.0, 0.0, z]
                p[axis] = sign * half * (1 - e) * z / foc          # |x f / z| = 0.65 w (1 -+ 1e-3)
                pts.append(p)
                inside.append(ins)
    xyz = torch.tensor(pts, dtype=torch.float32)
    got, want, seen = _check_compute(f3d, xyz, [cam], "thresholds", margin=5e-4)
    assert seen.tolist() == inside
    _, k = f3d.camera_tensors([cam], DEV)
    d = torch.tensor([p[2] if ins else 50.0 for p, ins in zip(pts, inside)], dtype=torch.float64, device=DEV)
    torch.testing.assert_close(got, d / float(k[0, 2]) * math.sqrt(0.2), rtol=1e-6, atol=0)


# ---- apply ------------------------------------------------------------------------------------------------------------
def _apply_inputs(P, seed, zero_every=3):
    g = torch.Generator().manual_seed(seed)
    s = torch.exp(torch.empty(P, 3).uniform_(-9, 0, generator=g))
    o = torch.empty(P, 1).uniform_(0.01, 0.99, generator=g)
    f = torch.exp(torch.empty(P, 1).uniform_(-9, -1, generator=g))
    f[::zero_every] = 0.0
    return s.to(DEV), o.to(DEV), f.to(DEV)


def test_apply_against_the_formula(f3d):
    P = 300_000
    s, o, f = _apply_inputs(P, 1)
    s.requires_grad_(True)
    o.requires_grad_(True)
    sf, of = f3d.apply_filter_3d(s, o, f)
    g = torch.Generator().manual_seed(2)
    gs, go = torch.randn(P, 3, generator=g).to(DEV), torch.randn(P, 1, generator=g).to(DEV)
    gs[::7] = -0.0
    ds, do = torch.autograd.grad((sf, of), (s, o), (gs, go))
    s64, o64, f64 = s.detach().double(), o.detach().double(), f.double()
    rs, ro = ref.apply64(s64, o64, f64)
    cs, co = ref.apply_backward64(s64, o64, f64, gs.double(), go.double())
    rel = lambda a, b: float(((a.double() - b).abs() / b.abs().clamp_min(1e-30)).max())
    assert rel(sf, rs) <= 1e-5 and rel(of, ro) <= 1e-5, (rel(sf, rs), rel(of, ro))
    # dL/ds has two terms that may cancel: relative to the sum of their magnitudes
    bound = gs.double().abs() * s64 / rs + go.double().abs() * ro * f64 ** 2 / (s64 * rs * rs)
    e_ds = float(((ds.double() - cs).abs() / bound.clamp_min(1e-30)).max())
    assert e_ds <= 1e-5 and rel(do, co) <= 1e-5, (e_ds, rel(do, co))
    # the integrated density o prod s is kept
    assert rel(of * sf.prod(1, keepdim=True), (o64 * s64.prod(1, keepdim=True))) <= 1e-5
    # where f = 0: the inputs and upstream gradients come through bitwise (signed zeros included)
    z = f[:, 0] == 0
    assert int(z.sum()) == (P + 2) // 3
    as_bits = lambda t: t.contiguous().view(torch.int32)
    assert torch.equal(as_bits(sf[z]), as_bits(s[z])) and torch.equal(as_bits(of[z]), as_bits(o[z]))
    assert torch.equal(as_bits(ds[z]), as_bits(gs[z])) and torch.equal(as_bits(do[z]), as_bits(go[z]))
    # a filter of shape [P] works the same
    sf1, of1 = f3d.apply_filter_3d(s.detach(), o.detach(), f[:, 0])
    assert torch.equal(sf1, sf) and torch.equal(of1, of)


# ---- render() ---------------------------------------------------------------------------------------------------------
def _train_cams():
    from s3gaussian_b200 import synthetic as syn
    return syn.waymo_ring(320, 208, frames=10)


def _apply_torch32(scales, opacity, f):
    """The apply restated in float32 torch (autograd gives its backward)."""
    s2 = scales * scales
    sf2 = s2 + f * f
    return torch.sqrt(sf2), opacity * torch.sqrt(s2.prod(1, keepdim=True) / sf2.prod(1, keepdim=True))


class _KernelValuesTorchBackward(torch.autograd.Function):
    """Forward: the apply kernel's values, so the rasterizer receives bitwise the tensors render() gives it.  Backward:
    autograd of the float32 torch restatement on the same inputs and upstream gradients.  Comparing render() against
    render() with this in place of apply_filter_3d isolates the apply's backward: the rasterizer's forward and backward
    see identical inputs, so none of its thresholds (the 1/255 cut-off, the T < 1e-4 stop) can decide differently."""

    @staticmethod
    def forward(ctx, scales, opacity, f):
        from s3gaussian_b200.filter3d import apply_filter_3d
        ctx.save_for_backward(scales, opacity, f)
        with torch.no_grad():
            return apply_filter_3d(scales, opacity, f)

    @staticmethod
    def backward(ctx, g_scales, g_opacity):
        scales, opacity, f = ctx.saved_tensors
        with torch.enable_grad():
            s, o = scales.detach().requires_grad_(True), opacity.detach().requires_grad_(True)
            ds, do = torch.autograd.grad(_apply_torch32(s, o, f), (s, o), (g_scales, g_opacity))
        return ds, do, None


def _seeded_model(**kw):
    """_model with the deformation network initialised from a fixed seed, whatever ran before."""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(11)
        return _model(**kw)


RENDER_CASES = [("coarse", False, False, False, False), ("coarse", False, True, True, False),
                ("fine", False, False, False, False), ("fine", True, False, False, False),
                ("fine", True, True, True, False), ("fine", False, True, False, True), ("fine", True, False, True, True)]


@pytest.mark.parametrize("stage,feat,opacity,aa,decomp", RENDER_CASES)
def test_render_with_the_switch(stage, feat, opacity, aa, decomp, f3d):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200 import diff_gaussian_rasterization as ours
    from s3gaussian_b200.gaussian_renderer import PipelineParams, fine_front, raster_settings_for, render
    g = _seeded_model(fine=stage == "fine")
    g.compute_3D_filter(_train_cams())
    assert g.filter_3D.shape == (g.get_xyz.shape[0], 1)
    cam = syn.waymo_ring(320, 208, frames=10)[4].to(DEV)
    bg = torch.tensor([0.2, 0.1, 0.3], device=DEV)
    on, off = PipelineParams(), PipelineParams()
    on.filter_3d = True
    on.render_opacity = off.render_opacity = opacity
    on.antialiasing = off.antialiasing = aa
    with torch.no_grad():
        r = render(cam, g, on, bg, stage=stage, render_feat=feat, return_decomposition=decomp, return_dx=True)
        r_off = render(cam, g, off, bg, stage=stage, render_feat=feat, return_decomposition=decomp, return_dx=True)
        assert float((r["render"] - r_off["render"]).abs().max()) > 1e-3
        # the rasterizer called directly on the filtered tensors
        rs = raster_settings_for(cam, g, on, bg)
        rast = ours.GaussianRasterizer(rs, **({"antialiasing": True} if aa else {}))
        if stage == "coarse":
            sc, op = f3d.apply_filter_3d(g.get_scaling, g.get_opacity, g.filter_3D)
            geo = dict(means3D=g.get_xyz, shs=g.get_features, colors_precomp=None, scales=sc,
                       rotations=g.get_rotation, opacities=op)
            featc = dx = None
        else:
            means3D, sc, ro, op, shs, cp, dx, _, featc = fine_front(cam, g, on, rs.campos, g.get_features)
            geo = dict(means3D=means3D, shs=shs, colors_precomp=cp, scales=sc, rotations=ro, opacities=op)
        m2d = torch.zeros_like(geo["means3D"])
        want = rast.forward_opacity(means2D=m2d, colors_aux=featc if feat else None, **geo)
        assert torch.equal(r["render"], want[0]) and torch.equal(r["radii"], want[1]) and torch.equal(r["depth"], want[2])
        if opacity:
            assert torch.equal(r["alpha"], want[3]) and torch.equal(r["median_depth"], want[4])
        if feat:
            assert torch.equal(r["feat"], want[5])
        if decomp and dx is not None:
            assert not torch.equal(r["render_d"], r_off["render_d"]) and not torch.equal(r["render_s"], r_off["render_s"])
    # gradients: render() against the same render whose apply backward is autograd of the float32 restatement (same
    # forward values, deterministic rasterizer backward, so only the apply's backward differs)
    import s3gaussian_b200.gaussian_renderer as gr
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        grads = []
        for restated in (False, True):
            for p in (g._xyz, g._scaling, g._opacity):
                p.grad = None
            if restated:
                orig = gr.apply_filter_3d
                gr.apply_filter_3d = _KernelValuesTorchBackward.apply
            try:
                out = render(cam, g, on, bg, stage=stage, render_feat=feat, return_dx=True)
            finally:
                if restated:
                    gr.apply_filter_3d = orig
            gen = torch.Generator().manual_seed(9)
            loss = (out["render"] * torch.randn(out["render"].shape, generator=gen).to(DEV)).sum()
            if opacity:
                loss = loss + out["alpha"].sum()
            if feat:
                loss = loss + out["feat"].sum()
            loss.backward()
            grads.append([p.grad.clone() for p in (g._xyz, g._scaling, g._opacity)])
    finally:
        torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
    for name, a, b in zip(("_xyz", "_scaling", "_opacity"), *grads):
        scale = float(b.abs().max())
        assert scale > 0, name
        assert float((a - b).abs().max()) <= 1e-5 * scale, (name, float((a - b).abs().max()), scale)


def test_render_pixels_follows_the_switch(f3d):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.evaluation import render_pixels
    from s3gaussian_b200.gaussian_renderer import PipelineParams, render
    g = _seeded_model()
    g.compute_3D_filter(_train_cams())
    cams = syn.waymo_ring(160, 112, frames=2)[:4]
    for c in cams:
        c.original_image = torch.rand(3, 112, 160)
    bg = torch.zeros(3, device=DEV)
    on = PipelineParams()
    on.filter_3d = True
    base = render_pixels(cams, g, bg, PipelineParams(), compute_metrics=False)
    res = render_pixels(cams, g, bg, on, compute_metrics=False)
    assert any(not np.array_equal(a, b) for a, b in zip(base["rgbs"], res["rgbs"]))
    with torch.no_grad():
        for i, c in enumerate(cams):
            r = render(c, g, on, bg, stage="fine", return_decomposition=True)
            assert np.array_equal(res["rgbs"][i], r["render"].permute(1, 2, 0).cpu().numpy()), i
    g.filter_3D = g.filter_3D[:-1]
    with pytest.raises(RuntimeError, match="compute_3D_filter"):
        render_pixels(cams, g, bg, on, compute_metrics=False)


# ---- model bookkeeping ------------------------------------------------------------------------------------------------
def test_densify_prune_and_sort_carry_the_filter(f3d):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_model import default_optimization_params, split_plan
    from s3gaussian_b200.gaussian_renderer import PipelineParams, render
    g = _seeded_model(P=20_000, fine=False)
    g.training_setup(default_optimization_params())
    g.compute_3D_filter(_train_cams())
    P = g.get_xyz.shape[0]
    gen = torch.Generator().manual_seed(4)
    # prune
    old = g.filter_3D.clone()
    mask = (torch.rand(P, generator=gen) < 0.2).to(DEV)
    g.prune_points(mask)
    assert torch.equal(g.filter_3D, old[~mask])
    # clone: the selected rows are appended with their source's value
    old, P = g.filter_3D.clone(), g.get_xyz.shape[0]
    grads = torch.rand(P, 1, generator=gen).to(DEV)
    extent = float(g.get_scaling.max(dim=1).values.median()) / 0.01
    sel = torch.nonzero((torch.norm(grads, dim=-1) >= 0.5) & (g.get_scaling.max(dim=1).values <= 0.01 * extent))[:, 0]
    g.densify_and_clone(grads, 0.5, extent)
    assert 0 < sel.numel() and torch.equal(g.filter_3D, old[torch.cat((torch.arange(P, device=DEV), sel))])
    # split
    old, P = g.filter_3D.clone(), g.get_xyz.shape[0]
    grads = torch.rand(P, 1, generator=gen).to(DEV)
    selected = (grads[:, 0] >= 0.5) & (g.get_scaling.max(dim=1).values > 0.01 * extent)
    src, _, _ = split_plan(selected)
    g.densify_and_split(grads, 0.5, extent)
    assert int(selected.sum()) > 0 and torch.equal(g.filter_3D, old[src])
    # Morton sort
    old = g.filter_3D.clone()
    order = g.spatial_sort()
    assert torch.equal(g.filter_3D, old[order])
    # a stale filter: the documented error
    g.filter_3D = old[:-3]
    on = PipelineParams()
    on.filter_3d = True
    cam = syn.waymo_ring(320, 208, frames=10)[4].to(DEV)
    with pytest.raises(RuntimeError, match="compute_3D_filter"):
        render(cam, g, on, torch.zeros(3, device=DEV), stage="coarse")
    with pytest.raises(RuntimeError, match="compute_3D_filter"):
        g.get_scaling_with_3D_filter
    g.compute_3D_filter(_train_cams())
    sc, op = g.get_scaling_with_3D_filter, g.get_opacity_with_3D_filter
    assert sc.shape == (g.get_xyz.shape[0], 3) and op.shape == (g.get_xyz.shape[0], 1)
    # a filter assigned by hand in another dtype is gathered as its float32 values
    g.filter_3D = g.filter_3D.double() * (1 + 1e-12)
    old = g.filter_3D.clone()
    mask = (torch.rand(g.get_xyz.shape[0], generator=gen) < 0.2).to(DEV)
    g.prune_points(mask)
    assert g.filter_3D.dtype == torch.float32 and torch.equal(g.filter_3D, old[~mask].float())


# ---- what the filter is for -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ratio", [1e-3, 1.0])
def test_a_gaussian_below_its_filter_seen_8x_closer(ratio, f3d, capsys):
    """Trained from a camera at depth 16 m (focal 100 px), so f = 16 / 100 sqrt(0.2); the Gaussian's scale is `ratio`
    f.  Rendered from 2 m (8x closer), white on black, with the filter its screen std is 8 sqrt(0.2 (1 + ratio^2)) px
    and its opacity o (ratio^2 / (1 + ratio^2))^(3/2): the radius is the preprocess's for that std and the summed image
    is the analytic filtered Gaussian, sampled at the pixel centres with the rasterizer's 1/255 cut-off and 0.99 cap,
    within 1e-3 relative (+1e-6).  At ratio 1e-3 that opacity is ~1e-9 and the Gaussian vanishes; without the filter it
    is a speck of alpha ~0.99 whose lit pixels lie within 2 px of its centre."""
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_renderer import PipelineParams, render
    W = H = 65        # odd: the Gaussian's centre falls on a pixel centre
    fpx, z_train, z_view = 100.0, 16.0, 2.0
    train = syn.make_camera(W, H, (0.0, 0.0, 0.0), focal=fpx)
    view = syn.make_camera(W, H, (z_train - z_view, 0.0, 0.0), focal=fpx).to(DEV)
    _, k = f3d.camera_tensors([train], DEV)
    f = z_train / float(k[0, 2]) * math.sqrt(0.2)
    o = 0.99
    cloud = SimpleNamespace(xyz=torch.tensor([[z_train, 0.0, 0.0]]), features_dc=torch.zeros(1, 1, 3),
                            features_rest=torch.zeros(1, 15, 3), scaling=torch.full((1, 3), math.log(ratio * f)),
                            rotation=torch.tensor([[1.0, 0.0, 0.0, 0.0]]),
                            opacity=torch.tensor([[math.log(o / (1 - o))]]))
    from s3gaussian_b200.gaussian_model import GaussianModel
    g = GaussianModel(3).create_from_tensors(*(t.to(DEV) for t in (cloud.xyz, cloud.features_dc, cloud.features_rest,
                                                                   cloud.scaling, cloud.rotation, cloud.opacity)))
    g.compute_3D_filter([train])
    torch.testing.assert_close(float(g.filter_3D[0, 0]), f, rtol=1e-6, atol=0)
    white = torch.ones(1, 3, device=DEV)
    bg = torch.zeros(3, device=DEV)
    on, off = PipelineParams(), PipelineParams()
    on.filter_3d = True
    res = {}
    for name, pipe in (("filtered", on), ("plain", off)):
        with torch.no_grad():
            r = render(view, g, pipe, bg, stage="coarse", override_color=white)
        img = r["render"][0].double().cpu().numpy()
        lit = np.argwhere(img > 0)
        extent = float(np.sqrt(((lit - (H - 1) / 2) ** 2).sum(1)).max()) if len(lit) else 0.0
        res[name] = (int(r["radii"][0]), float(img.sum()), float(img.max()), extent)
    # analytic: on the optical axis J = diag(F / z), cov2D = (F s / z)^2 I + 0.3 I
    F = float(k[0, 2])
    fpx_view = W / (2 * math.tan(view.FoVx / 2))
    s_filt = math.sqrt((ratio * f) ** 2 + f ** 2)
    o_filt = o * (ratio * f / s_filt) ** 3
    var = (fpx_view * s_filt / z_view) ** 2 + 0.3
    radius = math.ceil(3 * math.sqrt(var + math.sqrt(0.1)))
    c = ((W - 1) / 2, (H - 1) / 2)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    alpha = np.minimum(0.99, o_filt * np.exp(-0.5 * ((xx - c[0]) ** 2 + (yy - c[1]) ** 2) / var))
    energy = float(alpha[alpha >= 1 / 255].sum())
    with capsys.disabled():
        print(f"\n[filter3d] ratio {ratio:g}: screen std {math.sqrt(var - 0.3):.3f} px (the filter's alone: 8 sqrt(0.2) "
              f"= {8 * math.sqrt(0.2):.3f}), opacity {o_filt:.3e}; filtered radius {res['filtered'][0]} (analytic {radius}),"
              f" energy {res['filtered'][1]:.5f} (analytic {energy:.5f}); plain radius {res['plain'][0]}, "
              f"peak {res['plain'][2]:.3f}, lit within {res['plain'][3]:.2f} px, energy {res['plain'][1]:.4f}")
    assert res["filtered"][0] == radius
    assert abs(res["filtered"][1] - energy) <= 1e-3 * energy + 1e-6, (res["filtered"][1], energy)
    if ratio == 1e-3:
        assert res["plain"][3] <= 2.0 and res["plain"][2] > 0.9
        assert res["filtered"][1] == 0.0
