"""GPU: the absolute screen-space gradient (s3g_rasterize_backward_absgrad, GaussianRasterizer(absgrad=True),
render() with pipe.absgrad, GaussianModel.densify(max_grad_abs=...)).

1. means2D.absgrad against the float64 restatement of tests/absgrad_ref.py (per (pixel, slot) leaves) at three small
   shapes with partial tiles, RGB and precomputed covariances, three losses, plain and antialiased forwards, the
   default and the deterministic walk; exactly 0 for Gaussians with radii == 0.
2. Every other output of the deterministic absgrad backward is bitwise that of the deterministic opacity backward; the
   default walk's match to float rounding.
3. The deterministic absgrad repeats bitwise.
4. A Gaussian whose pixel gradients cancel has a vanishing signed statistic and a large absolute one; densify selects
   it only with max_grad_abs, and a one-sided Gaussian in both modes.
5. render() sets viewspace_points.absgrad in both stages, with and without render_feat, and is unchanged with the
   switch off.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import aa_ref
import absgrad_ref
import util
from test_gpu_raster_opacity import _grad_case, _model

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def ours(built_lib):
    from s3gaussian_b200 import diff_gaussian_rasterization as mod
    return mod


class _deterministic:
    def __init__(self, on=True):
        self.on = on

    def __enter__(self):
        self.prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
        torch.use_deterministic_algorithms(self.on)

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.prev[0], warn_only=self.prev[1])


LOSSES = {"color_depth": ("color", "depth"), "alpha_median": ("alpha", "median"),
          "all": ("color", "depth", "alpha", "median", "aux")}
SHAPES = [(48, 48, 40, 3, False), (64, 40, 33, 5, True), (32, 64, 32, 9, False)]


def _absgrad_run(ours, d, dL, aa, det, aux_cols=None, m2d=None):
    """forward_opacity(absgrad=True) + backward of sum(dL * images) -> (means2D tensor, radii)."""
    names = ["means3D", "opacities", "colors_precomp"] + (["cov3D_precomp"] if d["cov3D_precomp"] is not None
                                                           else ["scales", "rotations"])
    t = {k: d[k].to(DEV).clone().requires_grad_(True) for k in names}
    if m2d is None:
        m2d = torch.zeros_like(t["means3D"], requires_grad=True)
    aux = aux_cols.to(DEV).requires_grad_(True) if aux_cols is not None else None
    rast = ours.GaussianRasterizer(util.settings_for(ours, d, DEV), antialiasing=aa, absgrad=True)
    out = rast.forward_opacity(means3D=t["means3D"], means2D=m2d, opacities=t["opacities"],
                               colors_precomp=t["colors_precomp"], scales=t.get("scales"),
                               rotations=t.get("rotations"), cov3D_precomp=t.get("cov3D_precomp"), colors_aux=aux)
    images = dict(color=out[0], depth=out[2], alpha=out[3], median=out[4], aux=out[5] if aux is not None else None)
    loss = sum((images[k] * dL[k].to(DEV, torch.float32)).sum() for k in dL)
    with _deterministic(det):
        loss.backward()
    return m2d, out[1]


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("loss_kind", list(LOSSES))
@pytest.mark.parametrize("P,W,H,seed,cov", SHAPES)
def test_absgrad_matches_float64_oracle(P, W, H, seed, cov, loss_kind, aa, det, ours):
    check_absgrad_against_restatement(ours, _grad_case(P, W, H, seed, cov), seed, loss_kind, aa, det)


def check_absgrad_against_restatement(ours, d, seed, loss_kind, aa, det):
    """means2D.absgrad of forward_opacity(absgrad=True) for `loss_kind` against absgrad_ref in float64; d holds
    precomputed colours."""
    P, W, H, cov = d["means3D"].shape[0], d["W"], d["H"], d["cov3D_precomp"] is not None
    _, _, _, _, lists = util.ours_forward_state(d, DEV)
    gen = torch.Generator().manual_seed(seed + 200)
    dL = {k: torch.randn(3 if k in ("color", "aux") else 1, H, W, generator=gen, dtype=torch.float64)
          for k in LOSSES[loss_kind]}
    aux_cols = torch.rand(P, 3, generator=gen) if "aux" in dL else None
    m2d, radii = _absgrad_run(ours, d, dL, aa, det, aux_cols)
    absg = m2d.absgrad
    assert absg.dtype == torch.float32 and tuple(absg.shape) == (P, 2)

    leaf = {k: d[k].to(DEV).double() for k in ("means3D", "opacities")}
    leaf.update({"cov3D": d["cov3D_precomp"].to(DEV).double()} if cov else
                {"scales": d["scales"].to(DEV).double(), "rotations": d["rotations"].to(DEV).double()})
    leaf["view"], leaf["proj"] = d["viewmatrix"].to(DEV).double(), d["projmatrix"].to(DEV).double()
    pr = aa_ref.project64(d, leaf)
    mx, my = ((pr["ndc"][:, 0] + 1) * W - 1) * 0.5, ((pr["ndc"][:, 1] + 1) * H - 1) * 0.5
    op = pr["alpha_eff"] if aa else leaf["opacities"].reshape(-1)
    pix, idx = (t.to(DEV) for t in absgrad_ref.pixel_lists(W, H, lists["ranges"], lists["point_list"]))
    signed, ref = absgrad_ref.mean2d_grads64(
        W, H, torch.nan_to_num(mx), torch.nan_to_num(my), torch.nan_to_num(pr["conic"]), torch.nan_to_num(op),
        d["colors_precomp"].to(DEV).double(), torch.nan_to_num(pr["depth"]), d["bg"].to(DEV).double(), pix, idx,
        {k: v.to(DEV) for k, v in dL.items()}, aux_cols.to(DEV).double() if aux_cols is not None else None)
    vis = (radii > 0)
    assert int(vis.sum()) > 5
    assert float(absg[~vis].abs().max()) == 0 if bool((~vis).any()) else True
    got, want = absg[vis].double().cpu().numpy(), ref[vis].cpu().numpy()
    assert util.relerr(got, want) < 1e-3, (loss_kind, aa, det, util.relerr(got, want))
    # the restatement's signed sum is the backward's dL_dmean2D, and the triangle inequality holds
    sg = m2d.grad[:, :2][vis].double().cpu().numpy()
    assert util.relerr(sg, signed[vis].cpu().numpy()) < 1e-3
    assert (np.abs(sg) <= got * (1 + 1e-5) + 1e-6 * np.abs(got).max()).all()


# ---- the other outputs ----------------------------------------------------------------------------------------------
def _c_backward(ours, d, det, absgrad, aa=False, seed=4):
    """One forward (opacity form, antialiased or not) and one backward through the C ABI with every output exported:
    the deterministic or default *_opacity backward, or s3g_rasterize_backward_absgrad.  -> dict of outputs."""
    from s3gaussian_b200 import _lib
    lib = _lib.load()
    P, W, H = d["means3D"].shape[0], d["W"], d["H"]
    E = torch.Tensor([])
    g = lambda k: d[k].to(DEV).contiguous() if d[k] is not None else E
    inputs = [g(k) for k in ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")]
    rs = util.settings_for(ours, d, DEV)

    class Ctx:
        def save_for_backward(self, *a):
            self.saved = a

        def mark_non_differentiable(self, *a):
            pass
    ctx = Ctx()
    ours._RasterizeGaussians.forward(ctx, inputs[0], torch.zeros_like(inputs[0]), *inputs[1:], rs, None, None, None,
                                     None, True, aa)
    scene = ours._scene(rs, torch.device(DEV), inputs[0], inputs[1], inputs[2], None, inputs[4], inputs[5], inputs[6])
    gen = torch.Generator().manual_seed(seed)
    gc, gd, ga = (torch.randn(ch, H, W, generator=gen).to(DEV) for ch in (3, 1, 1))
    e = lambda *s: torch.zeros(s, dtype=torch.float32, device=DEV)
    M = inputs[1].size(1) if inputs[1].numel() else 0
    o = dict(mean2D=e(P, 3), conic=e(P, 4), opacity=e(P, 1), color=e(P, 3), depth=e(P), mean3D=e(P, 3), cov3D=e(P, 6),
             sh=e(P, max(M, 1), 3), scale=e(P, 3), rot=e(P, 4))
    s = ctx.saved
    bwd = _lib.RasterBackwardArgs(
        R=ctx.num_rendered, radii=s[5].data_ptr(), geom_buffer=s[7].data_ptr(), binning_buffer=s[8].data_ptr(),
        image_buffer=s[9].data_ptr(), dL_dpix=gc.data_ptr(), dL_dpix_depth=gd.data_ptr(),
        dL_dmean2D=o["mean2D"].data_ptr(), dL_dconic=o["conic"].data_ptr(), dL_dopacity=o["opacity"].data_ptr(),
        dL_dcolor=o["color"].data_ptr(), dL_ddepth=o["depth"].data_ptr(), dL_dmean3D=o["mean3D"].data_ptr(),
        dL_dcov3D=o["cov3D"].data_ptr(), dL_dsh=o["sh"].data_ptr() if M else None, dL_dscale=o["scale"].data_ptr(),
        dL_drot=o["rot"].data_ptr())
    opa = _lib.RasterOpacityArgs(dL_dpix_alpha=ga.data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    nb = int(lib.s3g_rasterize_backward_deterministic_workspace_bytes(P, ctx.num_rendered, W, H))
    ws = torch.empty(max(nb, 16), dtype=torch.uint8, device=DEV)
    if absgrad:
        o["abs"] = e(P, 2)
        _lib.check(lib.s3g_rasterize_backward_absgrad(C.byref(scene), C.byref(bwd), C.byref(opa), o["abs"].data_ptr(),
                                                      int(det), ws.data_ptr() if det else None, stream), "absgrad")
    elif det:
        _lib.check(lib.s3g_rasterize_backward_deterministic_opacity(C.byref(scene), C.byref(bwd), C.byref(opa),
                                                                    ws.data_ptr(), stream), "det")
    else:
        _lib.check(lib.s3g_rasterize_backward_opacity(C.byref(scene), C.byref(bwd), C.byref(opa), stream), "bwd")
    torch.cuda.synchronize()
    if not M:
        o.pop("sh")
    o["radii"] = s[5].clone()
    return o


SCENES = [("small_rgb", dict(P=600, width=96, height=64, seed=5), "rgb", False),
          ("covpre_sh", dict(P=900, width=83, height=61, seed=7), "sh", True)]


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("name,kw,mode,cov", SCENES)
def test_other_outputs_are_those_of_the_backward_it_extends(name, kw, mode, cov, aa, ours):
    """Deterministic: bitwise equal.  The signed moments of the absgrad walk are the same source expressions as the
    plain walk's, and the abs sums are independent accumulators, so the compiled arithmetic of every other output is
    the same.  Default walk: equal to float rounding (unordered atomics)."""
    from s3gaussian_b200 import synthetic as syn
    cloud, cam = syn.make_small_scene(**kw)
    d = util.scene_inputs(cloud, cam, mode=mode, sh_degree=2, cov_precomp=cov)
    ref = _c_backward(ours, d, True, False, aa)
    got = _c_backward(ours, d, True, True, aa)
    for k, v in ref.items():
        assert torch.equal(v, got[k]), k
    vis = got["radii"] > 0
    assert float(got["abs"][~vis].abs().max()) == 0 if bool((~vis).any()) else True
    assert bool((got["mean2D"][:, :2].abs() <= got["abs"] * (1 + 1e-5) + 1e-7).all())
    ref_d = _c_backward(ours, d, False, False, aa)
    got_d = _c_backward(ours, d, False, True, aa)
    for k, v in ref_d.items():
        if k == "radii":
            assert torch.equal(v, got_d[k])
            continue
        assert util.relerr(got_d[k].cpu().numpy(), v.cpu().numpy()) < 1e-5, k
    assert util.relerr(got_d["abs"].cpu().numpy(), got["abs"].cpu().numpy()) < 1e-5


def test_deterministic_absgrad_repeats_bitwise(ours):
    d = _grad_case(64, 40, 33, 5, False)
    gen = torch.Generator().manual_seed(1)
    dL = {k: torch.randn(3 if k == "color" else 1, 33, 40, generator=gen, dtype=torch.float64)
          for k in ("color", "depth", "alpha")}
    runs = [_absgrad_run(ours, d, dL, False, True)[0] for _ in range(2)]
    assert torch.equal(runs[0].absgrad, runs[1].absgrad) and torch.equal(runs[0].grad, runs[1].grad)
    assert float(runs[0].absgrad.abs().max()) > 0


def test_absgrad_accumulates_like_grad(ours):
    d = _grad_case(48, 48, 40, 3, False)
    gen = torch.Generator().manual_seed(2)
    dL = {"color": torch.randn(3, 40, 48, generator=gen, dtype=torch.float64)}
    m2d, _ = _absgrad_run(ours, d, dL, False, True)
    first = m2d.absgrad.clone()
    _absgrad_run(ours, d, dL, False, True, m2d=m2d)        # the same deterministic call into the same tensor
    assert torch.equal(m2d.absgrad, first + first) and float(first.abs().max()) > 0
    m2d.absgrad = None
    _absgrad_run(ours, d, dL, False, True, m2d=m2d)
    assert torch.equal(m2d.absgrad, first)


# ---- the property the statistic exists for --------------------------------------------------------------------------
W2 = H2 = 97          # (W - 1) / 2 = 48: the optical axis projects onto a pixel centre
Z2 = 4.85             # 1 world unit at this depth is 97 / 4.85 = 20 px (tan(fov / 2) = 0.5)


def _two_gaussians(ours):
    """G0 on the optical axis (pixel (48, 48)), isotropic; G1 20 px to its right.  -> (settings, raw tensors)."""
    n, f, tan = 0.01, 100.0, 0.5
    Pm = torch.zeros(4, 4)
    Pm[0, 0] = Pm[1, 1] = 1 / tan
    Pm[3, 2] = 1.0
    Pm[2, 2] = f / (f - n)
    Pm[2, 3] = -(f * n) / (f - n)
    rs = ours.GaussianRasterizationSettings(
        image_height=H2, image_width=W2, tanfovx=tan, tanfovy=tan, bg=torch.zeros(3, device=DEV), scale_modifier=1.0,
        viewmatrix=torch.eye(4, device=DEV), projmatrix=Pm.T.contiguous().to(DEV), sh_degree=0,
        campos=torch.zeros(3, device=DEV), prefiltered=False, debug=False)
    xyz = torch.tensor([[0.0, 0.0, Z2], [1.0, 0.0, Z2]], device=DEV)
    return rs, xyz


def _two_gaussian_grads(ours, rs, xyz, scale_g1):
    """dL/dpix: 1 on G0's 21x21 window (symmetric about its mean), scale_g1 on the 10x21 window right of G1's column
    (one-sided).  -> (means2D tensor, radii)."""
    P = xyz.shape[0]
    m2d = torch.zeros(P, 3, device=DEV, requires_grad=True)
    t = dict(means3D=xyz, opacities=torch.full((P, 1), 0.8, device=DEV), colors_precomp=torch.full((P, 3), 0.5, device=DEV),
             scales=torch.full((P, 3), 0.1, device=DEV), rotations=torch.tensor([[1.0, 0, 0, 0]] * P, device=DEV))
    color, radii, _ = ours.GaussianRasterizer(rs, absgrad=True)(means2D=m2d, **t)
    g = torch.zeros(3, H2, W2, device=DEV)
    g[0, 38:59, 38:59] = 1.0
    g[0, 38:59, 69:79] = scale_g1
    with _deterministic():
        (color * g).sum().backward()
    return m2d, radii


def test_cancelling_gradients_vanish_only_in_the_signed_statistic(ours):
    from s3gaussian_b200.gaussian_model import GaussianModel, default_optimization_params
    rs, xyz = _two_gaussians(ours)
    m2d, radii = _two_gaussian_grads(ours, rs, xyz, 1.0)
    a0, a1 = (float(v) for v in m2d.absgrad.norm(dim=1))
    m2d, radii = _two_gaussian_grads(ours, rs, xyz, a0 / a1)       # the same absolute magnitude for both
    assert bool((radii > 0).all())
    signed, absg = m2d.grad[:, :2].norm(dim=1), m2d.absgrad.norm(dim=1)
    assert float(signed[0]) <= 1e-4 * float(absg[0]), (float(signed[0]), float(absg[0]))
    assert abs(float(absg[1]) / float(absg[0]) - 1) < 1e-3
    thr = 0.5 * float(absg[0])
    assert float(signed[1]) >= thr           # the one-sided Gaussian passes the signed threshold

    def model():
        g = GaussianModel(0).create_from_tensors(
            xyz, torch.zeros(2, 1, 3, device=DEV), torch.zeros(2, 0, 3, device=DEV),
            torch.full((2, 3), math.log(0.1), device=DEV), torch.tensor([[1.0, 0, 0, 0]] * 2, device=DEV),
            torch.zeros(2, 1, device=DEV))
        g.training_setup(default_optimization_params())
        g.densification_step(m2d.grad, radii, m2d.absgrad)
        torch.testing.assert_close(g.xyz_gradient_accum[:, 0], m2d.grad[:, :2].norm(dim=1), rtol=1e-6, atol=0)
        torch.testing.assert_close(g.xyz_gradient_accum_abs[:, 0], absg, rtol=1e-6, atol=0)
        return g
    # clone (small Gaussians: extent 100) and split (large: extent 1)
    for extent, grow in ((100.0, 1), (1.0, 2)):
        g = model()
        g.densify(thr, 0.005, extent, None)
        assert g.get_xyz.shape[0] == 2 + grow * 1 - (1 if grow == 2 else 0)
        if grow == 1:
            assert torch.equal(g.get_xyz[2], xyz[1])
        else:
            assert torch.equal(g.get_xyz[0], xyz[0])          # G0 kept, G1 replaced by two samples
        g = model()
        g.densify(thr, 0.005, extent, None, max_grad_abs=thr)
        assert g.get_xyz.shape[0] == (4 if grow == 1 else 4)
        if grow == 1:
            assert torch.equal(g.get_xyz[2:], xyz)
        assert float(g.xyz_gradient_accum_abs.abs().max()) == 0     # reset with the other accumulators


# ---- render() -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stage,feat,shared", [("coarse", False, True), ("fine", False, True), ("fine", True, True),
                                               ("fine", True, False)])
def test_render_sets_viewspace_absgrad(stage, feat, shared, ours):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_renderer import PipelineParams, render
    g = _model(P=20_000, fine=stage == "fine")
    cam = syn.waymo_ring(320, 208, frames=10)[4].to(DEV)
    bg = torch.tensor([0.2, 0.1, 0.3], device=DEV)
    off, on = PipelineParams(), PipelineParams()
    on.absgrad = True
    off.shared_binning = on.shared_binning = shared
    res = {}
    for name, pipe in (("off", off), ("on", on)):
        with _deterministic():
            r = render(cam, g, pipe, bg, stage=stage, render_feat=feat, return_dx=True)
            loss = r["render"].sum() + 0.1 * r["depth"].mean() + (r["feat"].square().mean() if feat else 0)
            loss.backward()
        res[name] = (r, {k: v.grad.clone() for k, v in (("xyz", g._xyz), ("opacity", g._opacity),
                                                          ("scaling", g._scaling))})
        for p in (g._xyz, g._opacity, g._scaling, g._rotation, g._features_dc, g._features_rest):
            p.grad = None
    (r_off, g_off), (r_on, g_on) = res["off"], res["on"]
    assert getattr(r_off["viewspace_points"], "absgrad", None) is None
    for k, v in r_off.items():
        if isinstance(v, torch.Tensor) and k != "viewspace_points":
            assert torch.equal(v, r_on[k]), k
    for k in g_off:
        assert torch.equal(g_off[k], g_on[k]), k
    vs = r_on["viewspace_points"]
    assert torch.equal(vs.grad, r_off["viewspace_points"].grad)
    a = vs.absgrad
    P = g.get_xyz.shape[0]
    assert tuple(a.shape) == (P, 2) and a.dtype == torch.float32 and bool(torch.isfinite(a).all())
    vis = r_on["visibility_filter"]
    assert float(a[~vis].abs().max()) == 0 and float(a[vis].max()) > 0
    assert bool((vs.grad[:, :2].abs() <= a * (1 + 1e-4) + 1e-9).all())


def test_densify_stats_abs_matches_torch(ours):
    from s3gaussian_b200.optim import add_densification_stats
    P = 5000
    gen = torch.Generator().manual_seed(7)
    vg = torch.randn(P, 3, generator=gen).to(DEV)
    va = torch.rand(P, 2, generator=gen).to(DEV)
    radii = (torch.randint(-2, 6, (P,), generator=gen)).to(DEV, torch.int32)
    acc, acc_abs, den, mr = (torch.rand(P, 1, generator=gen).to(DEV), torch.rand(P, 1, generator=gen).to(DEV),
                             torch.rand(P, 1, generator=gen).to(DEV), torch.rand(P, generator=gen).to(DEV))
    ref = [t.clone() for t in (acc, den, mr)]
    add_densification_stats(vg, radii, *ref)
    add_densification_stats(vg, radii, acc, den, mr, va, acc_abs_got := acc_abs.clone())
    assert torch.equal(acc, ref[0]) and torch.equal(den, ref[1]) and torch.equal(mr, ref[2])
    vis = radii > 0
    want = acc_abs.clone()
    want[vis] += torch.sqrt((va[vis] ** 2).sum(1, keepdim=True))
    torch.testing.assert_close(acc_abs_got, want, rtol=1e-6, atol=0)
    assert torch.equal(acc_abs_got[~vis], acc_abs[~vis])
