"""GPU: the rasterizer through a camera's intrinsics and OpenCV distortion (s3g_rasterize_forward_lens,
GaussianRasterizer(lens=...)).

1. Identity: the centred lens without distortion gives the plain call's outputs, every forward form and gradients.
2. Principal point: an off-centre cx, cy equals the plain forward with the correspondingly shifted projmatrix.
3. Sky consistency: a Gaussian on the sky ray of pixel (x, y) lands at mean2D = (x, y).
4. Geometry: xyAB and the conic against the float64 restatement (tests/lens_ref.py), radii, the lens cull.
5. Per-Gaussian gradients against the float64 VJP of the restatement, absgrad against the walk without the lens.
6. The deterministic backward repeats bitwise.
7. A small Gaussian's intensity centroid lies at the OpenCV-projected pixel.
8. render() and render_pixels() with pipe.lens.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import lens_ref
import util
from test_gpu_raster_aa import _Ctx, _check, _close, _geo, _state
from test_gpu_raster_camera import _sh_rgb64
from test_gpu_raster_opacity import _model

pytestmark = pytest.mark.gpu
DEV = "cuda"

BARREL = (-0.25, 0.06, 0.0, 0.0, 0.0)
PINCUSHION = (0.18, 0.03, 0.0, 0.0, 0.0)
TANGENTIAL = (-0.05, 0.0, 0.012, -0.008, 0.0)
K3_FOLD = (0.0, 0.0, 0.0, 0.0, -0.9)      # s* = 1 / 6.3: a finite lens cull inside the 1.3 frustum


@pytest.fixture(scope="module")
def ours(built_lib):
    from s3gaussian_b200 import diff_gaussian_rasterization as mod
    return mod


def _scene(mode="sh", cov=False, deg=3, P=600, W=64, H=48, seed=7):
    from s3gaussian_b200 import synthetic as syn
    cloud, cam = syn.make_small_scene(P=P, width=W, height=H, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    cloud.scaling += torch.empty(P, 1).uniform_(-3.0, 0.5, generator=g)
    return util.scene_inputs(cloud, cam, mode=mode, sh_degree=deg, cov_precomp=cov)


def _centred(d, dist=(0.0,) * 5, dx=0.0, dy=0.0):
    from s3gaussian_b200.diff_gaussian_rasterization import Lens
    W, H = d["W"], d["H"]
    return Lens(W / (2 * d["tanfovx"]), H / (2 * d["tanfovy"]), W / 2 + dx, H / 2 + dy, *dist)


def _leaf(d, vis=None, grad=False):
    sel = (lambda t: t[vis]) if vis is not None else (lambda t: t)
    leaf = {k: sel(d[k].to(DEV).double()).clone().requires_grad_(grad) for k in ("means3D", "opacities")}
    if d["cov3D_precomp"] is not None:
        leaf["cov3D"] = sel(d["cov3D_precomp"].to(DEV).double()).clone().requires_grad_(grad)
    else:
        for k in ("scales", "rotations"):
            leaf[k] = sel(d[k].to(DEV).double()).clone().requires_grad_(grad)
    leaf["view"] = d["viewmatrix"].to(DEV).double()
    return leaf


def _forward_state(ours, d, lens, aa=False):
    """A lens forward through _RasterizeGaussians.forward: -> (ctx, radii, xyAB [P,4], Cod [P,4])."""
    E = torch.Tensor([])
    g = lambda k: d[k].to(DEV).contiguous() if d[k] is not None else E
    inputs = [g(k) for k in ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")]
    ctx = _Ctx()
    with torch.no_grad():
        ours._RasterizeGaussians.forward(ctx, inputs[0], torch.zeros_like(inputs[0]), *inputs[1:],
                                         util.settings_for(ours, d, DEV), None, None, None, None, False, aa, False,
                                         lens)
    torch.cuda.synchronize()
    P, R, W, H = inputs[0].shape[0], ctx.num_rendered, d["W"], d["H"]
    s = ctx.saved
    xyAB = _state(s[7], "xyAB", P, R, W, H, torch.float32).view(P, 4)
    Cod = _state(s[7], "Cod", P, R, W, H, torch.float32).view(P, 4)
    return ctx, inputs, s[5].clone(), xyAB, Cod


# ---- 1. identity ---------------------------------------------------------------------------------------------------

def _radii_equal_off_integers(got, ref, d, lens, aa):
    """Radii equal except where the float64 radius (3 sqrt(lambda_max)) lies within 1e-4 of an integer."""
    r = lens_ref.project64(d, _leaf(d), lens, aa)
    a, b, c = r["a"] + 0.3, r["b"], r["c"] + 0.3
    mid = 0.5 * (a + c)
    lam = mid + torch.sqrt(torch.clamp(mid * mid - (a * c - b * b), min=0.1))
    r64 = 3 * torch.sqrt(lam)
    near = (r64 - r64.round()).abs() < 1e-4
    differ = got != ref
    assert not bool((differ & ~near).any()), int((differ & ~near).sum())


FORWARD_CASES = [("sh", False, 3, False), ("rgb", False, 0, True), ("sh", True, 2, True), ("rgb", True, 0, False)]


@pytest.mark.parametrize("mode,cov,deg,aa", FORWARD_CASES)
def test_identity_lens_gives_the_plain_forward(mode, cov, deg, aa, ours):
    d = _scene(mode, cov, deg)
    rs = util.settings_for(ours, d, DEV)
    lens = _centred(d)
    lr, plain = ours.GaussianRasterizer(rs, antialiasing=aa, lens=lens), ours.GaussianRasterizer(rs, antialiasing=aa)
    geo = _geo(d)
    P = d["means3D"].shape[0]
    gen = torch.Generator().manual_seed(3)
    aux = torch.rand(P, 3, generator=gen).to(DEV)
    flows = [torch.rand(P, 4, generator=gen).to(DEV) for _ in range(2)]
    group = (torch.rand(P, generator=gen) < 0.4).to(DEV)
    with torch.no_grad():
        m2d = torch.zeros_like(geo["means3D"])
        got, ref = lr(means2D=m2d, **geo), plain(means2D=m2d, **geo)
        assert int((ref[1] > 0).sum()) > 50
        _radii_equal_off_integers(got[1], ref[1], d, lens, aa)
        for i in (0, 2):
            _close(got[i], ref[i], ("forward", i))
        got, ref = lr.forward_aux(means2D=m2d, colors_aux=aux, **geo), plain.forward_aux(means2D=m2d, colors_aux=aux,
                                                                                          **geo)
        for i in (0, 2, 3):
            _close(got[i], ref[i], ("aux", i))
        for colors_aux in (None, aux):
            got = lr.forward_opacity(means2D=m2d, colors_aux=colors_aux, **geo)
            ref = plain.forward_opacity(means2D=m2d, colors_aux=colors_aux, **geo)
            for i in range(len(ref)):
                if i != 1:
                    _close(got[i], ref[i], ("opacity", colors_aux is not None, i))
        got = lr.forward_eval(means2D=m2d, group=group, flow_colors=flows, with_opacity=True, **geo)
        ref = plain.forward_eval(means2D=m2d, group=group, flow_colors=flows, with_opacity=True, **geo)
        for i in (0, 2):
            _close(got[i], ref[i], ("eval", i))
        for k in range(4):
            _close(got[3][k], ref[3][k], ("decomposition", k))
            _close(got[5][k], ref[5][k], ("eval opacity", k))
        for k in range(2):
            _close(got[4][k], ref[4][k], ("flow", k))


def _grads(ours, d, lens=None, rs=None, aa=False, det=False, opacity=False, seed=5):
    """Gradients of a seeded loss on forward() (or forward_opacity()) through autograd."""
    t = {k: d[k].to(DEV).clone().requires_grad_(True) for k in util.TENSOR_KEYS if d[k] is not None}
    m2d = torch.zeros_like(t["means3D"], requires_grad=True)
    rs = rs if rs is not None else util.settings_for(ours, d, DEV)
    gen = torch.Generator().manual_seed(seed)
    gc, gd, ga = (torch.randn(ch, d["H"], d["W"], generator=gen).to(DEV) for ch in (3, 1, 1))
    r = ours.GaussianRasterizer(rs, antialiasing=aa, lens=lens)
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    torch.use_deterministic_algorithms(det)
    try:
        if opacity:
            out = r.forward_opacity(means2D=m2d, **t)
            loss = (out[0] * gc).sum() + (out[2] * gd).sum() + (out[3] * ga).sum()
        else:
            out = r(means2D=m2d, **t)
            loss = (out[0] * gc).sum() + (out[2] * gd).sum()
        loss.backward()
    finally:
        torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
    return {k: v.grad.clone() for k, v in list(t.items()) + [("means2D", m2d)]}, out[1]


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("mode,cov,aa", [("sh", False, False), ("rgb", True, True)])
def test_identity_lens_gives_the_plain_gradients(mode, cov, aa, det, ours):
    d = _scene(mode, cov, 3 if mode == "sh" else 0, seed=13)
    got, radii = _grads(ours, d, _centred(d), aa=aa, det=det, opacity=True)
    ref, radii_ref = _grads(ours, d, None, aa=aa, det=det, opacity=True)
    same = radii == radii_ref
    assert int(same.sum()) > 50
    for k in ref:
        _check(got[k][same], ref[k][same], k)


# ---- 2. principal point ----------------------------------------------------------------------------------------------

def test_principal_point_equals_the_shifted_projection(ours):
    from s3gaussian_b200 import synthetic as syn
    d = _scene("sh", False, 3, P=800, W=96, H=64, seed=21)
    d["means3D"] = d["means3D"].clone()
    dx, dy = 7.25, -4.5
    lens = _centred(d, dx=dx, dy=dy)
    P = syn.projection_matrix(syn.ZNEAR, syn.ZFAR, 2 * math.atan(d["tanfovx"]), 2 * math.atan(d["tanfovy"]))
    P[0, 2] = 2 * lens.cx / d["W"] - 1
    P[1, 2] = 2 * lens.cy / d["H"] - 1
    shifted = dict(d, projmatrix=(d["viewmatrix"].unsqueeze(0).bmm(P.transpose(0, 1).unsqueeze(0))).squeeze(0))
    # keep the cloud inside both clamps: the plain 1.3 tanfov one and the lens's
    r = lens_ref.project64(d, _leaf(d), lens)
    t = torch.cat([d["means3D"].double(), torch.ones(d["means3D"].shape[0], 1, dtype=torch.float64)], 1) @ \
        d["viewmatrix"].double()
    x, y = (t[:, 0] / t[:, 2]).abs(), (t[:, 1] / t[:, 2]).abs()
    lim = 1.3 * min(d["tanfovx"], d["tanfovy"]) - (abs(dx) + abs(dy)) / lens.fx - 0.05
    inside = (x < lim) & (y < lim)
    for k in util.TENSOR_KEYS:
        if d[k] is not None:
            d[k] = d[k][inside]
            shifted[k] = d[k]
    assert int(inside.sum()) > 300 and bool(r["visible"].any())
    rs = util.settings_for(ours, d, DEV)
    rs_shift = util.settings_for(ours, shifted, DEV)
    with torch.no_grad():
        m2d = torch.zeros_like(d["means3D"]).to(DEV)
        got = ours.GaussianRasterizer(rs, lens=lens).forward_opacity(means2D=m2d, **_geo(d))
        ref = ours.GaussianRasterizer(rs_shift).forward_opacity(means2D=m2d, **_geo(d))
    _radii_equal_off_integers(got[1], ref[1], d, lens, False)
    for i in (0, 2, 3, 4):
        _close(got[i], ref[i], ("shifted", i))
    g_got, rad = _grads(ours, d, lens, opacity=True)
    g_ref, rad_ref = _grads(ours, d, None, rs=rs_shift, opacity=True)
    same = rad == rad_ref
    for k in g_ref:
        _check(g_got[k][same], g_ref[k][same], k)


# ---- 3. sky consistency ------------------------------------------------------------------------------------------------

def test_gaussian_on_a_sky_ray_lands_on_its_pixel(ours):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.diff_gaussian_rasterization import Lens
    from s3gaussian_b200.sky import sky_camera
    W, H = 160, 96
    base = syn.make_camera(W, H, (0.0, 0.0, 1.5), yaw_deg=10.0, pitch_deg=-4.0)
    K = torch.tensor([[150.0, 0.0, 86.3], [0.0, 140.0, 41.7], [0.0, 0.0, 1.0]])
    cam = syn.SyntheticCamera(W, H, base.FoVx, base.FoVy, base.world_view_transform, base.full_proj_transform,
                              base.camera_center, 0.0, K)
    c2w, Kc = sky_camera(cam)
    assert torch.equal(Kc, K)
    pix = torch.tensor([[3.0, 5.0], [80.0, 40.0], [151.0, 90.0], [17.0, 77.0]])
    dirs = torch.stack([(pix[:, 0] + 0.5 - K[0, 2]) / K[0, 0], (pix[:, 1] + 0.5 - K[1, 2]) / K[1, 1],
                        torch.ones(4)], 1).double()
    depth = torch.tensor([4.0, 9.0, 6.0, 12.0], dtype=torch.float64)
    xyz = (dirs * depth[:, None]) @ c2w[:3, :3].double().T + c2w[:3, 3].double()
    n = xyz.shape[0]
    d = dict(W=W, H=H, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=torch.zeros(3), sh_degree=0,
             viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform, campos=cam.camera_center,
             means3D=xyz.float(), opacities=torch.full((n, 1), 0.5), scales=torch.full((n, 3), 0.01),
             rotations=torch.tensor([[1.0, 0, 0, 0]]).repeat(n, 1), shs=None, colors_precomp=torch.ones(n, 3),
             cov3D_precomp=None)
    lens = Lens(float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]))
    _, _, radii, xyAB, _ = _forward_state(ours, d, lens)
    assert bool((radii > 0).all())
    err = (xyAB[:, :2].cpu().double() - pix.double()).abs().max()
    assert float(err) <= 1e-3, float(err)


# ---- 4. geometry ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dist", [BARREL, PINCUSHION, TANGENTIAL, K3_FOLD], ids=["barrel", "pincushion", "tangential",
                                                                              "k3"])
def test_geometry_matches_the_float64_restatement(dist, ours):
    d = _scene("sh", False, 3, P=1500, W=96, H=64, seed=31)
    lens = _centred(d, dist, dx=3.0, dy=-2.0)
    _, _, radii, xyAB, Cod = _forward_state(ours, d, lens)
    r = lens_ref.project64(d, _leaf(d), lens)
    vis = (radii > 0)
    assert int(vis.sum()) > 100
    assert not bool((vis & ~r["visible"]).any())
    pix_err = (xyAB[vis, :2].double() - r["pix"][vis]).abs().max()
    assert float(pix_err) <= 2e-3, float(pix_err)
    conic = torch.stack([xyAB[:, 2], xyAB[:, 3], Cod[:, 0]], 1).double()[vis]
    rel = ((conic - r["conic"][vis]).abs() / r["conic"][vis].abs().amax(1, keepdim=True)).max()
    assert float(rel) <= 1e-4, float(rel)
    if dist is K3_FOLD:
        beyond = r["s"] > lens_ref.max_radius2(0.0, 0.0, -0.9)
        assert int((beyond & (r["depth"] > 0.2)).sum()) > 10
        assert int(radii[beyond].abs().sum()) == 0
    # the radius from the float64 covariance, except near an integer
    a, b, c = r["a"] + 0.3, r["b"], r["c"] + 0.3
    mid = 0.5 * (a + c)
    r64 = 3 * torch.sqrt(mid + torch.sqrt(torch.clamp(mid * mid - (a * c - b * b), min=0.1)))
    ok = vis & ((r64 - r64.round()).abs() > 1e-4)
    assert torch.equal(radii[ok].double(), torch.ceil(r64[ok]))



# ---- 5. gradients ------------------------------------------------------------------------------------------------------

def _explicit_backward(ours, d, gc, gd, lens, aa=False, det=False, absgrad=False):
    from s3gaussian_b200 import _lib
    lib = _lib.load()
    ctx, inputs, radii, _, _ = _forward_state(ours, d, lens, aa)
    means3D, sh, cp, op, sc, ro, cov = inputs
    P, H, W = means3D.shape[0], d["H"], d["W"]
    M = sh.shape[1] if sh.numel() else 0
    rs = util.settings_for(ours, d, DEV)
    scene = ours._scene(rs, means3D.device, means3D, sh, cp, None, sc, ro, cov)
    e = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device=DEV)
    o = dict(mean2D=e(P, 3), conic=e(P, 4), opacity=e(P, 1), color=e(P, 3), depth=e(P), mean3D=e(P, 3), cov3D=e(P, 6),
             sh=e(P, max(M, 1), 3), scale=e(P, 3), rot=e(P, 4), abs=e(P, 2))
    gc, gd = gc.to(DEV).contiguous(), gd.to(DEV).contiguous()
    s = ctx.saved
    bwd = _lib.RasterBackwardArgs(
        R=ctx.num_rendered, radii=s[5].data_ptr(), geom_buffer=s[7].data_ptr(), binning_buffer=s[8].data_ptr(),
        image_buffer=s[9].data_ptr(), dL_dpix=gc.data_ptr(), dL_dpix_depth=gd.data_ptr(),
        dL_dmean2D=o["mean2D"].data_ptr(), dL_dconic=o["conic"].data_ptr(), dL_dopacity=o["opacity"].data_ptr(),
        dL_dcolor=o["color"].data_ptr(), dL_ddepth=o["depth"].data_ptr(), dL_dmean3D=o["mean3D"].data_ptr(),
        dL_dcov3D=o["cov3D"].data_ptr(), dL_dsh=o["sh"].data_ptr() if M else None, dL_dscale=o["scale"].data_ptr(),
        dL_drot=o["rot"].data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    nb = int(lib.s3g_rasterize_backward_deterministic_workspace_bytes(P, ctx.num_rendered, W, H))
    ws = torch.empty(max(nb, 16), dtype=torch.uint8, device=DEV)
    if absgrad:
        _lib.check(lib.s3g_rasterize_backward_absgrad(C.byref(scene), C.byref(bwd), None, o["abs"].data_ptr(),
                                                      1 if det else 0, ws.data_ptr(), stream), "absgrad")
    elif det:
        _lib.check(lib.s3g_rasterize_backward_deterministic(C.byref(scene), C.byref(bwd), ws.data_ptr(), stream), "det")
    else:
        _lib.check(lib.s3g_rasterize_backward(C.byref(scene), C.byref(bwd), stream), "bwd")
    # camera gradients do not pass through the lens
    cws = torch.empty(max(int(lib.s3g_rasterize_camera_backward_workspace_bytes(P)), 16), dtype=torch.uint8, device=DEV)
    view = e(16)
    out = _lib.RasterCameraGrads(view.data_ptr(), None, None)
    assert lib.s3g_rasterize_camera_backward(C.byref(scene), C.byref(bwd), C.byref(out), cws.data_ptr(), stream) == -1
    assert b"lens" in lib.s3g_last_error()
    torch.cuda.synchronize()
    R = ctx.num_rendered
    o["clamped"] = _state(s[7], "clamped", P, R, W, H, torch.uint8)
    o["dalpha"] = _state(s[7], "grad_rec", P, R, W, H, torch.float32).view(P, -1)[:, 5]
    o["radii"] = radii
    return o


def _vjp64(d, o, lens, aa):
    vis = o["radii"] > 0
    leaf = _leaf(d, vis, grad=True)
    cp = d["campos"].to(DEV).double()
    r = lens_ref.project64(d, leaf, lens, aa)
    g = lambda k: o[k].double()[vis]
    gc = g("conic")
    loss = ((r["ndc"] * g("mean2D")[:, :2]).sum() + (r["conic"][:, 0] * gc[:, 0]).sum() +
            (r["conic"][:, 1] * 2 * gc[:, 1]).sum() + (r["conic"][:, 2] * gc[:, 3]).sum() +
            (r["depth"] * g("depth")).sum() + (r["alpha_eff"] * g("dalpha")).sum())
    grads = {}
    if d["shs"] is not None:
        sh = d["shs"].to(DEV).double()[vis].clone().requires_grad_(True)
        dirs = leaf["means3D"] - cp
        rgb = _sh_rgb64(d["sh_degree"], sh, dirs / dirs.norm(dim=1, keepdim=True))
        cl = o["clamped"][vis].long()
        keep = torch.stack([(cl & 1) == 0, (cl & 2) == 0, (cl & 4) == 0], 1).double()
        loss = loss + (rgb * keep * g("color")).sum()
        grads["sh"] = sh
    names = {"mean3D": "means3D", "opacity": "opacities", "cov3D": "cov3D", "scale": "scales", "rot": "rotations"}
    grads.update({k: leaf[v] for k, v in names.items() if v in leaf})
    keys = list(grads)
    res = torch.autograd.grad(loss, [grads[k] for k in keys], allow_unused=True)
    return {k: (v if v is not None else torch.zeros_like(grads[k])) for k, v in zip(keys, res)}, vis


GRAD_CASES = [("sh", False, 3, False, False, BARREL), ("sh", False, 3, True, True, TANGENTIAL),
              ("sh", True, 2, True, False, PINCUSHION), ("rgb", False, 0, False, True, K3_FOLD),
              ("rgb", True, 0, False, False, TANGENTIAL), ("sh", False, 1, True, True, BARREL)]


@pytest.mark.parametrize("mode,cov,deg,aa,det,dist", GRAD_CASES)
def test_gradients_match_float64_vjp(mode, cov, deg, aa, det, dist, ours):
    d = _scene(mode, cov, deg, seed=41 + deg)
    lens = _centred(d, dist, dx=2.5, dy=1.5)
    gc, gd = util.seeded_grads(d, 9 + deg)
    o = _explicit_backward(ours, d, gc, gd, lens, aa, det)
    ref, vis = _vjp64(d, o, lens, aa)
    for k in ("mean3D", "opacity", "cov3D", "scale", "rot", "sh"):
        if k in ref:
            got = o[k][vis] if k != "sh" else o["sh"][vis][:, :ref["sh"].shape[1]]
            _check(got, ref[k], k)
    assert bool((~vis).any()) and float(o["mean3D"][~vis].abs().max()) == 0


@pytest.mark.parametrize("det", [False, True])
def test_absgrad_after_a_lens_forward(det, ours):
    """The composite is the lens's own: the absgrad output equals the absgrad walk on the same geometry records; the
    other gradients equal the backward without absgrad."""
    d = _scene("sh", False, 3, seed=51)
    lens = _centred(d, BARREL, dx=-3.0)
    gc, gd = util.seeded_grads(d, 4)
    a = _explicit_backward(ours, d, gc, gd, lens, det=det, absgrad=True)
    b = _explicit_backward(ours, d, gc, gd, lens, det=True)
    vis = a["radii"] > 0
    assert float(a["abs"][vis].abs().max()) > 0 and float(a["abs"][~vis].abs().max()) == 0
    assert bool((a["abs"][vis] >= a["mean2D"][vis, :2].abs() * (1 - 1e-5)).all())
    for k in ("mean3D", "scale", "rot", "opacity", "mean2D"):
        _check(a[k][vis], b[k][vis].double(), k)


# ---- 6. determinism ------------------------------------------------------------------------------------------------

def test_deterministic_backward_repeats_bitwise(ours):
    from s3gaussian_b200 import synthetic as syn
    cloud = syn.make_cloud(60_000, seed=4, width=640, height=416)
    cam = syn.make_camera(640, 416, (0, 0, 2.0))
    d = util.scene_inputs(cloud, cam, mode="sh", sh_degree=3)
    lens = _centred(d, TANGENTIAL, dx=5.0, dy=-3.0)
    runs = [_grads(ours, d, lens, aa=True, det=True, opacity=True, seed=21)[0] for _ in range(2)]
    for k in runs[0]:
        assert torch.isfinite(runs[0][k]).all() and float(runs[0][k].abs().max()) > 0, k
        assert torch.equal(runs[0][k].view(torch.int32), runs[1][k].view(torch.int32)), k


# ---- 7. point projection ---------------------------------------------------------------------------------------------

def test_point_centroid_lies_at_the_opencv_projection(ours):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.diff_gaussian_rasterization import Lens
    W, H = 320, 240
    cam = syn.make_camera(W, H, (0.0, 0.0, 0.0), focal=280.0)
    lens = Lens(280.0, 275.0, 163.4, 117.8, -0.21, 0.05, 0.004, -0.003, 0.0)
    c2w = torch.linalg.inv(cam.world_view_transform.transpose(0, 1).double())
    for x, y in ((0.02, -0.03), (-0.5, -0.38), (0.5, 0.37)):
        depth = 5.0
        xyz = (torch.tensor([[x * depth, y * depth, depth, 1.0]], dtype=torch.float64) @ c2w.T)[:, :3]
        # OpenCV: distort the normalised point, then K with the pixel centre at j (cx - 0.5)
        fx, fy, cx, cy, k1, k2, p1, p2, k3 = lens
        r2 = x * x + y * y
        rad = 1 + k1 * r2 + k2 * r2 ** 2 + k3 * r2 ** 3
        u = fx * (x * rad + 2 * p1 * x * y + p2 * (r2 + 2 * x * x)) + (cx - 0.5)
        v = fy * (y * rad + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y) + (cy - 0.5)
        s = 1.6 * depth / fx     # about 1.6 px standard deviation
        d = dict(W=W, H=H, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=torch.zeros(3), sh_degree=0,
                 viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform, campos=cam.camera_center)
        rs = util.settings_for(ours, d, DEV)
        with torch.no_grad():
            img = ours.GaussianRasterizer(rs, lens=lens)(
                means3D=xyz.float().to(DEV), means2D=torch.zeros(1, 3, device=DEV), opacities=torch.full((1, 1), 0.5,
                                                                                                          device=DEV),
                colors_precomp=torch.ones(1, 3, device=DEV), scales=torch.full((1, 3), s, device=DEV),
                rotations=torch.tensor([[1.0, 0, 0, 0]], device=DEV))[0][0].double().cpu()
        w = img.sum()
        cu = float((img.sum(0) * torch.arange(W, dtype=torch.float64)).sum() / w)
        cv = float((img.sum(1) * torch.arange(H, dtype=torch.float64)).sum() / w)
        assert abs(cu - u) <= 0.05 and abs(cv - v) <= 0.05, ((x, y), (cu, cv), (u, v))


# ---- 8. render() and render_pixels() ---------------------------------------------------------------------------------

def _lens_camera(cam, dist=BARREL):
    from s3gaussian_b200 import synthetic as syn
    W, H = cam.image_width, cam.image_height
    fx, fy = W / (2 * cam.tanfovx), H / (2 * cam.tanfovy)
    K = torch.tensor([[fx, 0.0, W / 2 + 4.0], [0.0, fy, H / 2 - 3.0], [0.0, 0.0, 1.0]])
    return syn.SyntheticCamera(W, H, cam.FoVx, cam.FoVy, cam.world_view_transform, cam.full_proj_transform,
                               cam.camera_center, cam.time, K, torch.tensor(dist))


@pytest.mark.parametrize("stage,feat", [("coarse", False), ("fine", False), ("fine", True)])
def test_render_with_pipe_lens(stage, feat, ours):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_renderer import PipelineParams, camera_lens, fine_front, raster_settings_for, render
    g = _model(fine=stage == "fine")
    cam = _lens_camera(syn.waymo_ring(320, 208, frames=10)[4]).to(DEV)
    bg = torch.tensor([0.2, 0.1, 0.3], device=DEV)
    off, on = PipelineParams(), PipelineParams()
    on.lens = on.render_opacity = True
    with torch.no_grad():
        r_off = render(cam, g, off, bg, stage=stage, render_feat=feat)
        r_on = render(cam, g, on, bg, stage=stage, render_feat=feat)
    assert float((r_on["render"] - r_off["render"]).abs().max()) > 1e-3
    with torch.no_grad():
        rs = raster_settings_for(cam, g, on, bg)
        rast = ours.GaussianRasterizer(rs, lens=camera_lens(cam))
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
        ref = rast.forward_opacity(means2D=torch.zeros_like(geo["means3D"]), colors_aux=aux, **geo)
    assert torch.equal(r_on["render"], ref[0]) and torch.equal(r_on["alpha"], ref[3])
    if feat:
        assert torch.equal(r_on["feat"], ref[5])
    r = render(cam, g, on, bg, stage=stage, render_feat=feat)
    (r["render"].sum() + r["alpha"].sum()).backward()
    assert torch.isfinite(g._xyz.grad).all() and float(g._opacity.grad.abs().max()) > 0


def test_render_pixels_with_pipe_lens(ours):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.evaluation import render_pixels
    from s3gaussian_b200.gaussian_renderer import PipelineParams, render
    g = _model()
    cams = [_lens_camera(c, TANGENTIAL) for c in syn.waymo_ring(160, 112, frames=2)[:4]]
    for c in cams:
        c.original_image = torch.rand(3, 112, 160)
    bg = torch.zeros(3, device=DEV)
    on = PipelineParams()
    on.lens = True
    base = render_pixels(cams, g, bg, PipelineParams(), compute_metrics=False)
    res = render_pixels(cams, g, bg, on, compute_metrics=False)
    assert any(not np.array_equal(a, b) for a, b in zip(base["rgbs"], res["rgbs"]))
    with torch.no_grad():
        for i, c in enumerate(cams):
            r = render(c, g, on, bg, stage="fine", return_decomposition=True)
            assert np.array_equal(res["rgbs"][i], r["render"].permute(1, 2, 0).cpu().numpy()), i
            assert np.array_equal(res["static_rgbs"][i], r["render_s"].permute(1, 2, 0).cpu().numpy()), i
