"""GPU: the static/dynamic split rasterizer pass, render()'s decomposition under no_grad, the evaluation-metrics
kernel and render_pixels (run with -m gpu).

Checkers: the existing rasterizer (s3g_rasterize_forward) on all Gaussians and on each subset - the three passes the
decomposition made so far, and still makes with grad enabled; where oracle/_ref is built, the reference extension on
each subset; for the metrics, oracle/eval_oracle.py (skimage's SSIM and the reference's PSNR restated in numpy)."""
import numpy as np
import pytest
import torch

import ref_ext
import util
from oracle import eval_oracle as eo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4            # the suite's image bar against the reference extension
SPLIT_TOL = 1e-6      # split images vs the masked passes: bitwise is the target
SSIM_TOL, PSNR_TOL = 1e-5, 1e-4


def _dgr():
    from s3gaussian_b200 import diff_gaussian_rasterization as dgr
    return dgr


def _scene(case):
    from s3gaussian_b200 import synthetic as syn
    if case == "small":
        cloud, cam = syn.make_small_scene(P=3000, width=96, height=64, seed=7)
        return util.scene_inputs(cloud, cam, mode="sh", sh_degree=3, bg=(0.1, 0.2, 0.3))
    P, W, H = {"200k_960x640": (200_000, 960, 640), "500k_1920x1280": (500_000, 1920, 1280)}[case]
    cloud = syn.make_cloud(P, seed=0, width=W, height=H)
    cam = syn.make_camera(W, H, (0, 0, 2.0))
    return util.scene_inputs(cloud, cam, mode="rgb", sh_degree=0, bg=(0.1, 0.2, 0.3))


def _mask(kind, P, seed=0):
    g = torch.Generator().manual_seed(seed)
    if kind == "random10":
        return (torch.rand(P, generator=g) < 0.1).to(DEV)
    if kind == "random50":
        return (torch.rand(P, generator=g) < 0.5).to(DEV)
    if kind == "all_static":
        return torch.zeros(P, dtype=torch.bool, device=DEV)
    return torch.ones(P, dtype=torch.bool, device=DEV)


def _tensors(d, sel=None):
    out = {}
    for k in util.TENSOR_KEYS:
        t = d[k]
        out[k] = None if t is None else (t.to(DEV) if sel is None else t.to(DEV)[sel])
    return out


def _call(rast, t, **extra):
    m2d = torch.zeros_like(t["means3D"])
    return (rast.forward_split if extra else rast)(means3D=t["means3D"], means2D=m2d, opacities=t["opacities"],
                                                   shs=t["shs"], colors_precomp=t["colors_precomp"],
                                                   scales=t["scales"], rotations=t["rotations"],
                                                   cov3D_precomp=t["cov3D_precomp"], **extra)


def _close(a, b, tol):
    """bitwise, or within `tol` relative; returns (ok, bitwise, relerr)"""
    if torch.equal(a, b):
        return True, True, 0.0
    e = util.relerr(a.cpu().numpy(), b.cpu().numpy())
    return e <= tol, False, e


def _check_split(d, group):
    dgr = _dgr()
    rast = dgr.GaussianRasterizer(util.settings_for(dgr, d, DEV))
    with torch.no_grad():
        t = _tensors(d)
        color, radii, depth = _call(rast, t)
        color2, radii2, depth2, color_d, depth_d, color_s, depth_s = _call(rast, t, group=group)
        subs = [_call(rast, _tensors(d, m)) for m in (group, ~group)]
    torch.cuda.synchronize()
    assert torch.equal(color2, color) and torch.equal(depth2, depth) and torch.equal(radii2, radii)
    report = {}
    for name, mine, ref in (("color_d", color_d, subs[0][0]), ("depth_d", depth_d, subs[0][2]),
                            ("color_s", color_s, subs[1][0]), ("depth_s", depth_s, subs[1][2])):
        ok, bitwise, e = _close(mine, ref, SPLIT_TOL)
        assert ok, (name, e)
        report[name] = bitwise
    for m, sub in ((group, subs[0]), (~group, subs[1])):
        assert torch.equal(sub[1], radii[m])   # per-Gaussian preprocess: a subset keeps its radii
    return report, subs


@pytest.mark.parametrize("kind", ["random10", "random50", "all_static", "all_dynamic"])
@pytest.mark.parametrize("case", ["small", "200k_960x640", "500k_1920x1280"])
def test_split_render_equals_masked_passes(case, kind, built_lib):
    d = _scene(case)
    P = d["means3D"].shape[0]
    group = _mask(kind, P)
    report, subs = _check_split(d, group)
    assert all(report.values()), report    # bitwise in practice: the same instruction sequence per image
    if kind in ("all_static", "all_dynamic"):
        empty = subs[0] if kind == "all_static" else subs[1]
        assert not empty[0].any() and not empty[2].any()   # a pass over no Gaussians: zero images
    if kind == "random50" and ref_ext.available():
        ref = ref_ext.load()
        for m in (group, ~group):
            dm = dict(d)
            sel = m.cpu()
            for k in util.TENSOR_KEYS:
                if d[k] is not None:
                    dm[k] = d[k][sel]
            r = util.run_module(ref, dm, DEV)
            mine = util.run_module(_dgr(), dm, DEV)
            assert np.array_equal(mine["radii"].cpu().numpy(), r["radii"].cpu().numpy())
            assert util.relerr(mine["color"].cpu().numpy(), r["color"].cpu().numpy()) < TOL
            assert util.relerr(mine["depth"].cpu().numpy(), r["depth"].cpu().numpy()) < TOL


def test_split_render_with_no_gaussians(built_lib):
    d = _scene("small")
    for k in util.TENSOR_KEYS:
        if d[k] is not None:
            d[k] = d[k][:0]
    dgr = _dgr()
    rast = dgr.GaussianRasterizer(util.settings_for(dgr, d, DEV))
    with torch.no_grad():
        out = _call(rast, _tensors(d), group=torch.zeros(0, dtype=torch.bool, device=DEV))
    assert out[1].numel() == 0
    for t in out[:1] + out[2:]:
        assert not t.any()


def test_forward_split_refuses_autograd(built_lib):
    d = _scene("small")
    dgr = _dgr()
    rast = dgr.GaussianRasterizer(util.settings_for(dgr, d, DEV))
    t = _tensors(d)
    t["means3D"].requires_grad_(True)
    with pytest.raises(RuntimeError, match="no backward"):
        _call(rast, t, group=_mask("random50", t["means3D"].shape[0]))


def _fine_model(P, W, H, seed=0):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.deformation import deform_network
    from s3gaussian_b200.gaussian_renderer import GaussianModelLite
    cloud = syn.make_cloud(P, seed=seed, width=W, height=H)
    net = deform_network(ref_ext.ref_deform_args(syn.DEFAULT_RESOLUTION, syn.DEFAULT_MULTIRES))
    net.deformation_net.set_aabb(*[list(a) for a in syn.WAYMO_AABB])
    net.load_state_dict(syn.make_deform_state(0, weight_scale=0.2), strict=False)
    return GaussianModelLite(cloud, net).to(DEV)


@pytest.mark.parametrize("P,W,H", [(20_000, 240, 160), (500_000, 1920, 1280)], ids=["20k_240x160", "500k_1920x1280"])
def test_render_decomposition_without_grad_equals_grad_path(P, W, H, built_lib):
    """render(return_decomposition=True, return_dx=True): the split pass under no_grad returns the keys and
    values of the three differentiable passes (the dx-threshold mask of the fine stage)"""
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_renderer import render, PipelineParams
    pc = _fine_model(P, W, H)
    cam = syn.waymo_ring(W, H, frames=3)[4].to(DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    ref = render(cam, pc, PipelineParams(), bg, stage="fine", return_decomposition=True, return_dx=True)
    with torch.no_grad():
        out = render(cam, pc, PipelineParams(), bg, stage="fine", return_decomposition=True, return_dx=True)
    assert list(out) == list(ref)
    m = ref["visibility_filter_d"].numel()
    assert 0 < m < P   # the dx threshold splits the cloud
    for k in out:
        if k == "viewspace_points":
            continue
        a, b = out[k], ref[k].detach()
        assert a.shape == b.shape and torch.equal(a, b), k


def _pair(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(3, H, W, generator=g)
    y = (x + 0.1 * torch.randn(3, H, W, generator=g)).clamp(0, 1)
    return x, y


def _masks(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return {"empty": torch.zeros(H, W, dtype=torch.bool), "full": torch.ones(H, W, dtype=torch.bool),
            "random": torch.rand(H, W, generator=g) < 0.3}


@pytest.mark.parametrize("H,W", [(7, 7), (643, 965), (1280, 1920)], ids=["7x7", "965x643", "1920x1280"])
def test_metrics_kernel_matches_oracle(H, W, built_lib):
    from s3gaussian_b200.evaluation import image_metrics
    x, y = _pair(H, W, H + W)
    xn, yn = x.numpy(), y.numpy()
    ref_psnr, ref_ssim = eo.psnr(xn, yn), eo.ssim(xn, yn)
    for name, m in _masks(H, W, 5).items():
        out = image_metrics(x.to(DEV), y.to(DEV), m.to(DEV))
        assert abs(float(out["psnr"]) - ref_psnr) <= PSNR_TOL, (name, float(out["psnr"]), ref_psnr)
        assert abs(float(out["ssim"]) - ref_ssim) <= SSIM_TOL, (name, float(out["ssim"]), ref_ssim)
        if name == "empty":
            assert "masked_psnr" not in out and "masked_ssim" not in out
            continue
        mn = m.numpy()
        assert abs(float(out["masked_psnr"]) - eo.masked_psnr(xn, yn, mn)) <= PSNR_TOL, name
        assert abs(float(out["masked_ssim"]) - eo.masked_ssim(xn, yn, mn)) <= SSIM_TOL, name
    # identical images: PSNR inf, SSIM 1
    same = image_metrics(x.to(DEV), x.to(DEV), _masks(H, W, 5)["random"].to(DEV))
    assert float(same["psnr"]) == float("inf") and float(same["masked_psnr"]) == float("inf")
    assert abs(float(same["ssim"]) - 1.0) <= 1e-12 and abs(float(same["masked_ssim"]) - 1.0) <= 1e-12


def test_metrics_kernel_without_mask(built_lib):
    from s3gaussian_b200.evaluation import image_metrics
    x, y = _pair(50, 70, 1)
    out = image_metrics(x.to(DEV), y.to(DEV))
    assert set(out) == {"psnr", "ssim"}
    assert abs(float(out["ssim"]) - eo.ssim(x.numpy(), y.numpy())) <= SSIM_TOL


def test_render_pixels_matches_oracle_on_three_pass_render(built_lib):
    """9-view ring (3 frames x 3 cameras) with per-view dynamic masks, two of them empty: render_pixels' metrics
    equal the oracle's on the images of the existing three-pass render (grad enabled), and its image lists are
    those images"""
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.evaluation import render_pixels
    from s3gaussian_b200.gaussian_renderer import render, PipelineParams
    W, H = 240, 160
    pc = _fine_model(60_000, W, H, seed=2)
    pipe = PipelineParams()
    bg = torch.zeros(3, device=DEV)
    cams = syn.waymo_ring(W, H, frames=3)
    g = torch.Generator().manual_seed(9)
    refs, per_view = [], []
    for i, cam in enumerate(cams):
        r = render(cam.to(DEV), pc, pipe, bg, stage="fine", return_decomposition=True, return_dx=True)
        img = r["render"].detach().cpu()
        cam.original_image = (img + 0.05 * torch.randn(img.shape, generator=g)).clamp(0, 1)
        m = torch.zeros(1, H, W, dtype=torch.bool)
        if i not in (0, 4):
            y0, x0 = int(torch.randint(0, H // 2, (1,), generator=g)), int(torch.randint(0, W // 2, (1,), generator=g))
            m[0, y0:y0 + 10 + 5 * i, x0:x0 + 20 + 7 * i] = True
        cam.dynamic_mask = m
        refs.append({k: r[k].detach().cpu() for k in ("render", "render_d", "render_s", "depth")})
        per_view.append(eo.view_metrics(img.numpy(), cam.original_image.numpy(), m[0].numpy()))
    res = render_pixels(cams, pc, bg, pipe)

    def mean(k):
        v = [p[k] for p in per_view if k in p]
        return sum(v) / len(v) if v else -1
    assert abs(res["psnr"] - mean("psnr")) <= PSNR_TOL
    assert abs(res["ssim"] - mean("ssim")) <= SSIM_TOL
    assert abs(res["masked_psnr"] - mean("masked_psnr")) <= PSNR_TOL
    assert abs(res["masked_ssim"] - mean("masked_ssim")) <= SSIM_TOL
    assert res["lpips"] == -1
    for key, rk in (("rgbs", "render"), ("dynamic_rgbs", "render_d"), ("static_rgbs", "render_s")):
        assert len(res[key]) == 9
        for a, r in zip(res[key], refs):
            assert np.array_equal(a, r[rk].permute(1, 2, 0).numpy()), key
    for a, r in zip(res["depths"], refs):
        dn = r["depth"].permute(1, 2, 0).numpy()
        assert np.array_equal(a, dn / dn.max())
    for a, cam in zip(res["gt_rgbs"], cams):
        assert np.array_equal(a, cam.original_image.permute(1, 2, 0).numpy())
