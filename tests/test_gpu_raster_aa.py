"""GPU: the rasterizer's antialiasing (s3g_rasterize_forward_antialiased, GaussianRasterizer(antialiasing=True)).

1. Forward identity: every forward form with the filter on gives the plain call's outputs with the opacities
   pre-multiplied by h (h from the float64 restatement in tests/aa_ref.py), radii bitwise equal.
2. Per-Gaussian and camera gradients against the float64 VJP of the restated preprocess (aa_ref.project64 plus the SH
   colour), applied to the composite gradients the backward exports (dL_dmean2D, dL_dconic, dL_ddepth, dL_dcolor and
   dL/dalpha_eff, read from the geometry state's gradient records).
3. The deterministic backward repeats bitwise.
4. Sub-pixel Gaussians rendered at two resolutions with one field of view keep their brightness.
5. render() and render_pixels() with pipe.antialiasing.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import aa_ref
import util
from test_gpu_raster_camera import _sh_rgb64, _with_edge_gaussians
from test_gpu_raster_opacity import _model

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def ours(built_lib):
    from s3gaussian_b200 import diff_gaussian_rasterization as mod
    return mod


def _scene(mode="sh", cov=False, deg=3, P=600, W=64, H=48, seed=7):
    """A small scene whose Gaussians span sub-pixel (h at its floor) to large (h near 1), plus 8 beyond the clamp."""
    from s3gaussian_b200 import synthetic as syn
    cloud, cam = syn.make_small_scene(P=P, width=W, height=H, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    cloud.scaling += torch.empty(P, 1).uniform_(-4.0, 1.0, generator=g)
    cloud = _with_edge_gaussians(cloud)
    return util.scene_inputs(cloud, cam, mode=mode, sh_degree=deg, cov_precomp=cov)


def _geo(d, opacities=None):
    t = {k: d[k].to(DEV).contiguous() for k in util.TENSOR_KEYS if d[k] is not None}
    if opacities is not None:
        t["opacities"] = opacities
    return t


def _premultiplied(d):
    """The opacities times h, as float32 on the device."""
    return (d["opacities"].to(DEV).double().reshape(-1) * aa_ref.h_of(d)).float().reshape(-1, 1)


def _close(got, ref, what):
    got, ref = got.double(), ref.double()
    scale = float(ref.abs().max())
    assert scale > 0, what
    assert float((got - ref).abs().max()) <= 1e-4 * scale, (what, float((got - ref).abs().max()), scale)


FORWARD_CASES = [("sh", False, 3), ("rgb", False, 0), ("sh", True, 2), ("rgb", True, 0)]


@pytest.mark.parametrize("mode,cov,deg", FORWARD_CASES)
def test_forward_forms_equal_the_plain_call_with_premultiplied_opacities(mode, cov, deg, ours):
    d = _scene(mode, cov, deg)
    rs = util.settings_for(ours, d, DEV)
    aa, plain = ours.GaussianRasterizer(rs, antialiasing=True), ours.GaussianRasterizer(rs)
    geo, pre = _geo(d), _geo(d, _premultiplied(d))
    P = d["means3D"].shape[0]
    gen = torch.Generator().manual_seed(3)
    aux = torch.rand(P, 3, generator=gen).to(DEV)
    flows = [torch.rand(P, 4, generator=gen).to(DEV) for _ in range(2)]
    group = (torch.rand(P, generator=gen) < 0.4).to(DEV)
    with torch.no_grad():
        m2d = torch.zeros_like(geo["means3D"])
        got, ref = aa(means2D=m2d, **geo), plain(means2D=m2d, **pre)
        assert torch.equal(got[1], ref[1])
        assert int((got[1] > 0).sum()) > 50
        for i in (0, 2):
            _close(got[i], ref[i], ("forward", i))
        # the filter changes the image: the plain call with the original opacities differs
        orig = plain(means2D=m2d, **geo)[0]
        assert float((orig - got[0]).abs().max()) > 1e-2
        got, ref = aa.forward_aux(means2D=m2d, colors_aux=aux, **geo), plain.forward_aux(means2D=m2d, colors_aux=aux,
                                                                                          **pre)
        assert torch.equal(got[1], ref[1])
        for i in (0, 2, 3):
            _close(got[i], ref[i], ("aux", i))
        for colors_aux in (None, aux):
            got = aa.forward_opacity(means2D=m2d, colors_aux=colors_aux, **geo)
            ref = plain.forward_opacity(means2D=m2d, colors_aux=colors_aux, **pre)
            assert torch.equal(got[1], ref[1])
            for i in range(len(ref)):
                if i != 1:
                    _close(got[i], ref[i], ("opacity", colors_aux is not None, i))
        got = aa.forward_eval(means2D=m2d, group=group, flow_colors=flows, with_opacity=True, **geo)
        ref = plain.forward_eval(means2D=m2d, group=group, flow_colors=flows, with_opacity=True, **pre)
        assert torch.equal(got[1], ref[1])
        for i in (0, 2):
            _close(got[i], ref[i], ("eval", i))
        for k in range(4):
            _close(got[3][k], ref[3][k], ("decomposition", k))
            _close(got[5][k], ref[5][k], ("eval opacity", k))
        for k in range(2):
            _close(got[4][k], ref[4][k], ("flow", k))


class _Ctx:
    def save_for_backward(self, *a):
        self.saved = a

    def mark_non_differentiable(self, *a):
        pass


def _state(buf, name, P, R, W, H, dtype):
    from s3gaussian_b200 import _lib
    off, eb, cnt = _lib.state_field(0, name, P, R, W, H)
    a = ((buf.data_ptr() + 127) & ~127) - buf.data_ptr() + off
    return buf[a:a + cnt * eb].view(dtype).clone()


def _explicit_backward(ours, d, gc, gd, det=False):
    """Antialiased forward + s3g_rasterize_backward{,_deterministic} exporting every per-Gaussian gradient, then the
    camera pass.  -> dict of device tensors: radii, clamped, the composite's dL/dalpha_eff (grad_rec slot 5), the
    per-Gaussian gradients and the three camera gradients."""
    from s3gaussian_b200 import _lib
    lib = _lib.load()
    E = torch.Tensor([])
    g = lambda k: d[k].to(DEV).contiguous() if d[k] is not None else E
    inputs = [g(k) for k in ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")]
    rs = util.settings_for(ours, d, DEV)
    ctx = _Ctx()
    ours._RasterizeGaussians.forward(ctx, inputs[0], torch.zeros_like(inputs[0]), *inputs[1:], rs, None, None, None,
                                     None, False, True)
    means3D, sh, cp, op, sc, ro, cov = inputs
    P, H, W = means3D.shape[0], d["H"], d["W"]
    M = sh.shape[1] if sh.numel() else 0
    scene = ours._scene(rs, means3D.device, means3D, sh, cp, None, sc, ro, cov)
    e = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device=DEV)
    o = dict(mean2D=e(P, 3), conic=e(P, 4), opacity=e(P, 1), color=e(P, 3), depth=e(P), mean3D=e(P, 3), cov3D=e(P, 6),
             sh=e(P, max(M, 1), 3), scale=e(P, 3), rot=e(P, 4), view=e(16), proj=e(16), campos=e(3))
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
    if det:
        nb = int(lib.s3g_rasterize_backward_deterministic_workspace_bytes(P, ctx.num_rendered, W, H))
        ws = torch.empty(max(nb, 16), dtype=torch.uint8, device=DEV)
        _lib.check(lib.s3g_rasterize_backward_deterministic(C.byref(scene), C.byref(bwd), ws.data_ptr(), stream), "det")
    else:
        _lib.check(lib.s3g_rasterize_backward(C.byref(scene), C.byref(bwd), stream), "bwd")
    cws = torch.empty(max(int(lib.s3g_rasterize_camera_backward_workspace_bytes(P)), 16), dtype=torch.uint8, device=DEV)
    out = _lib.RasterCameraGrads(o["view"].data_ptr(), o["proj"].data_ptr(), o["campos"].data_ptr())
    _lib.check(lib.s3g_rasterize_camera_backward(C.byref(scene), C.byref(bwd), C.byref(out), cws.data_ptr(), stream),
               "camera")
    torch.cuda.synchronize()
    R = ctx.num_rendered
    o["clamped"] = _state(s[7], "clamped", P, R, W, H, torch.uint8)
    o["dalpha"] = _state(s[7], "grad_rec", P, R, W, H, torch.float32).view(P, -1)[:, 5]
    o["radii"] = s[5].clone()
    return o


def _vjp64(d, o):
    """float64 VJP of the restated preprocess over the visible Gaussians with the exported composite gradients: the
    gradients of the Gaussians' inputs and of (viewmatrix, projmatrix, campos).  dL/dconic.y is exported for the
    symmetric pair, so it weighs twice against the one off-diagonal value."""
    vis = o["radii"] > 0
    leaf = {k: d[k].to(DEV).double()[vis].clone().requires_grad_(True) for k in ("means3D", "opacities")}
    if d["cov3D_precomp"] is not None:
        leaf["cov3D"] = d["cov3D_precomp"].to(DEV).double()[vis].clone().requires_grad_(True)
    else:
        for k in ("scales", "rotations"):
            leaf[k] = d[k].to(DEV).double()[vis].clone().requires_grad_(True)
    leaf["view"] = d["viewmatrix"].to(DEV).double().clone().requires_grad_(True)
    leaf["proj"] = d["projmatrix"].to(DEV).double().clone().requires_grad_(True)
    cp = d["campos"].to(DEV).double().clone().requires_grad_(True)
    r = aa_ref.project64(d, leaf)
    assert bool((r["h"] > 0.9).any()) and bool((r["h"] < 0.05).any())   # the filter matters here
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
    names = {"mean3D": "means3D", "opacity": "opacities", "cov3D": "cov3D", "scale": "scales", "rot": "rotations",
             "view": "view", "proj": "proj"}
    grads.update({k: leaf[v] for k, v in names.items() if v in leaf})
    grads["campos"] = cp
    keys = list(grads)
    res = torch.autograd.grad(loss, [grads[k] for k in keys], allow_unused=True)
    return {k: (v if v is not None else torch.zeros_like(grads[k])) for k, v in zip(keys, res)}, vis


def _check(got, ref, name):
    got, ref = got.double().cpu().numpy().reshape(ref.shape), ref.detach().cpu().numpy()
    assert np.isfinite(got).all(), name
    scale = np.abs(ref).max()
    if scale == 0:
        assert np.abs(got).max() == 0, name
        return
    assert util.relerr(got, ref) <= 1e-4, (name, util.relerr(got, ref))
    frac, worst, i = util.elementwise(got, ref, rtol=1e-4, atol=1e-5 * scale)
    assert frac == 0.0, (name, worst, i, got.reshape(-1)[i], ref.reshape(-1)[i])


GRAD_CASES = [("sh", False, 3, False), ("sh", False, 3, True), ("sh", False, 1, False), ("sh", True, 3, False),
              ("rgb", False, 0, False), ("rgb", True, 0, True)]


@pytest.mark.parametrize("mode,cov,deg,det", GRAD_CASES)
def test_gradients_match_float64_vjp(mode, cov, deg, det, ours):
    d = _scene(mode, cov, deg, seed=11 + deg)
    gc, gd = util.seeded_grads(d, 5 + deg)
    o = _explicit_backward(ours, d, gc, gd, det)
    ref, vis = _vjp64(d, o)
    # dL/dopacity is h times the composite's dL/dalpha_eff
    assert float(o["dalpha"][vis].abs().max()) > 0
    for k in ("mean3D", "opacity", "cov3D", "scale", "rot", "sh"):
        if k in ref:
            got = o[k][vis] if k != "sh" else o["sh"][vis][:, :ref["sh"].shape[1]]
            _check(got, ref[k], k)
    assert bool((~vis).any()) and float(o["opacity"][~vis].abs().max()) == 0
    for k in ("view", "proj", "campos"):
        if k == "campos" and d["shs"] is None:
            assert float(o[k].abs().max()) == 0
            continue
        _check(o[k], ref[k].reshape(-1), k)


def test_deterministic_backward_repeats_bitwise(ours):
    from s3gaussian_b200 import synthetic as syn
    cloud = syn.make_cloud(60_000, seed=4, width=640, height=416)
    cam = syn.make_camera(640, 416, (0, 0, 2.0))
    d = util.scene_inputs(cloud, cam, mode="sh", sh_degree=3)

    def run():
        t = {k: d[k].to(DEV).clone().requires_grad_(True) for k in util.TENSOR_KEYS if d[k] is not None}
        m2d = torch.zeros_like(t["means3D"], requires_grad=True)
        rs = util.settings_for(ours, d, DEV)
        cam_t = {k: getattr(rs, k).clone().requires_grad_(True) for k in ("viewmatrix", "projmatrix", "campos")}
        gen = torch.Generator().manual_seed(21)
        gc, gd, ga = (torch.randn(ch, 416, 640, generator=gen).to(DEV) for ch in (3, 1, 1))
        out = ours.GaussianRasterizer(rs._replace(**cam_t), antialiasing=True).forward_opacity(means2D=m2d, **t)
        ((out[0] * gc).sum() + (out[2] * gd).sum() + (out[3] * ga).sum()).backward()
        return {k: v.grad.clone() for k, v in list(t.items()) + list(cam_t.items()) + [("means2D", m2d)]}

    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    torch.use_deterministic_algorithms(True)
    try:
        runs = [run() for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
    for k in runs[0]:
        assert torch.isfinite(runs[0][k]).all() and float(runs[0][k].abs().max()) > 0, k
        assert torch.equal(runs[0][k].view(torch.int32), runs[1][k].view(torch.int32)), k


def _subpixel_cloud(n, focal, seed):
    """n white Gaussians of about 0.3 px standard deviation at full resolution (depth 4 to 8, focal `focal` px), spread
    over the view of a camera at the origin looking down +x, at opacity 0.6 - sparse enough that few overlap."""
    g = torch.Generator().manual_seed(seed)
    depth = 4 + 4 * torch.rand(n, generator=g)
    xyz = torch.stack([depth, (torch.rand(n, generator=g) * 2 - 1) * 0.45 * depth,
                       (torch.rand(n, generator=g) * 2 - 1) * 0.3 * depth], 1)
    s = (0.3 * depth / focal)[:, None].expand(n, 3).contiguous()
    rot = torch.zeros(n, 4)
    rot[:, 0] = 1
    return xyz, s, rot, torch.full((n, 1), 0.6), torch.ones(n, 3)


def test_subpixel_gaussians_keep_their_brightness_across_resolutions(ours):
    """Mean image intensity of 3000 sub-pixel Gaussians (white on black) at 512x384 and at 256x192, same field of view.
    Measured on an H100 80GB HBM3: with antialiasing the half-resolution image is 0.936x as bright, without it 3.138x,
    since the 0.3 px^2 dilation dominates a Gaussian's footprint there."""
    from s3gaussian_b200 import synthetic as syn
    W, H = 512, 384
    focal = 0.9 * W
    xyz, s, rot, op, col = (t.to(DEV) for t in _subpixel_cloud(3000, focal, 2))
    means = {}
    for aa in (False, True):
        for w, h in ((W, H), (W // 2, H // 2)):
            cam = syn.make_camera(w, h, (0.0, 0.0, 0.0), focal=focal * w / W)
            d = dict(W=w, H=h, tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=torch.zeros(3), sh_degree=0,
                     viewmatrix=cam.world_view_transform, projmatrix=cam.full_proj_transform, campos=cam.camera_center)
            rs = util.settings_for(ours, d, DEV)
            with torch.no_grad():
                img = ours.GaussianRasterizer(rs, antialiasing=aa)(means3D=xyz, means2D=torch.zeros_like(xyz),
                                                                   opacities=op, colors_precomp=col, scales=s,
                                                                   rotations=rot)[0]
            means[(aa, w)] = float(img.mean())
    ratio_aa = means[(True, W // 2)] / means[(True, W)]
    ratio_plain = means[(False, W // 2)] / means[(False, W)]
    print(f"half/full mean intensity: antialiased {ratio_aa:.3f}, plain {ratio_plain:.3f}")
    assert 1 / 1.25 < ratio_aa < 1.25, ratio_aa
    assert ratio_plain > 2.0, ratio_plain


# ---- render() and render_pixels() -----------------------------------------------------------------------------------

@pytest.mark.parametrize("stage,feat", [("coarse", False), ("fine", False), ("fine", True)])
def test_render_switch(stage, feat, ours):
    from s3gaussian_b200 import synthetic as syn
    from types import SimpleNamespace
    from s3gaussian_b200.gaussian_renderer import PipelineParams, fine_front, raster_settings_for, render
    g = _model(fine=stage == "fine")
    cam = syn.waymo_ring(320, 208, frames=10)[4].to(DEV)
    bg = torch.tensor([0.2, 0.1, 0.3], device=DEV)
    off, on = PipelineParams(), PipelineParams()
    on.antialiasing = on.render_opacity = True
    legacy = SimpleNamespace(convert_SHs_python=True, compute_cov3D_python=False, debug=False)
    with torch.no_grad():
        r_off = render(cam, g, off, bg, stage=stage, render_feat=feat)
        r_legacy = render(cam, g, legacy, bg, stage=stage, render_feat=feat)
        r_on = render(cam, g, on, bg, stage=stage, render_feat=feat)
    for k, v in r_off.items():   # switch off: bitwise what a pipe without the attribute gives
        if isinstance(v, torch.Tensor) and k != "viewspace_points":
            assert torch.equal(v, r_legacy[k]), k
    assert float((r_on["render"] - r_off["render"]).abs().max()) > 1e-3
    # the antialiased rasterizer on the same inputs gives render()'s images
    with torch.no_grad():
        rs = raster_settings_for(cam, g, on, bg)
        rast = ours.GaussianRasterizer(rs, antialiasing=True)
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
    # with autograd: the antialiased backward runs and reaches the model
    r = render(cam, g, on, bg, stage=stage, render_feat=feat)
    (r["render"].sum() + r["alpha"].sum()).backward()
    assert torch.isfinite(g._xyz.grad).all() and float(g._opacity.grad.abs().max()) > 0


def test_render_pixels_follows_the_switch(ours):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.evaluation import render_pixels
    from s3gaussian_b200.gaussian_renderer import PipelineParams, render
    g = _model()
    cams = syn.waymo_ring(160, 112, frames=2)[:5]
    for c in cams:
        c.original_image = torch.rand(3, 112, 160)
    bg = torch.zeros(3, device=DEV)
    on = PipelineParams()
    on.antialiasing = True
    base = render_pixels(cams, g, bg, PipelineParams(), compute_metrics=False)
    res = render_pixels(cams, g, bg, on, compute_metrics=False)
    assert any(not np.array_equal(a, b) for a, b in zip(base["rgbs"], res["rgbs"]))
    with torch.no_grad():
        for i, c in enumerate(cams):
            r = render(c, g, on, bg, stage="fine", return_decomposition=True)
            assert np.array_equal(res["rgbs"][i], r["render"].permute(1, 2, 0).cpu().numpy()), i
            assert np.array_equal(res["static_rgbs"][i], r["render_s"].permute(1, 2, 0).cpu().numpy()), i
