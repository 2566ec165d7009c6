"""GPU: VGG16 LPIPS (s3g_lpips_vgg) against the float64 oracle and the reference's own module, its exact cases, the
absence of host synchronisation, and render_pixels with lpips_fn."""
import numpy as np
import pytest
import torch

import lpips_vgg_ref
import util
from oracle import lpips_vgg_oracle as vo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _tol(ours, ref):
    return abs(ours - ref) <= 1e-5 + 1e-4 * abs(ref)


def _check_terms(ours, ref, what):
    ours, ref = ours.cpu().tolist(), ref.cpu().tolist()
    for l in range(6):
        assert _tol(ours[l], ref[l]), (what, l, ours[l], ref[l])


@pytest.fixture(scope="module")
def weights():
    return vo.random_state_dicts(11)


@pytest.fixture(scope="module")
def fn(weights, built_lib):
    from s3gaussian_b200.lpips_vgg import LPIPSVGG
    return LPIPSVGG.from_state_dicts(*weights)


def _random_pair(H, W, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(3, H, W, generator=g), torch.rand(3, H, W, generator=g)


def _rendered_pair(H, W, seed):
    """a rasterised image and a noisy copy of it"""
    from s3gaussian_b200 import synthetic as syn
    cloud, cam = syn.make_small_scene(P=20_000, width=W, height=H, seed=seed)
    color = util.ours_forward_state(util.scene_inputs(cloud, cam, mode="sh", sh_degree=3), DEV)[0].float().cpu()
    g = torch.Generator().manual_seed(seed)
    return color, (color + 0.05 * torch.randn(color.shape, generator=g)).clamp(0, 1)


def _oracle_terms(x, y, weights):
    """the float64 oracle; its activations (gigabytes at 1920x1280) go back to the driver before the next case"""
    t = vo.lpips_terms(x, y, *weights)
    torch.cuda.empty_cache()
    return t


@pytest.mark.parametrize("H,W,case", [(16, 16, "random"), (47, 33, "random"), (33, 47, "rendered"),
                                      (160, 240, "random"), (160, 240, "rendered"), (640, 960, "random"),
                                      (640, 960, "rendered"), (1280, 1920, "rendered")],
                         ids=["16x16-random", "33x47-random", "47x33-rendered", "240x160-random", "240x160-rendered",
                              "960x640-random", "960x640-rendered", "1920x1280-rendered"])
def test_matches_fp64_oracle(H, W, case, fn, weights):
    x, y = (_random_pair if case == "random" else _rendered_pair)(H, W, H + W)
    x, y = x.to(DEV), y.to(DEV)
    ours = fn.terms(x, y)
    ref = _oracle_terms(x, y, weights)
    _check_terms(ours, ref, (H, W, case))
    d = fn(x, y)
    assert d.shape == (1, 1, 1, 1) and d.dtype == torch.float32 and d.device == x.device
    assert float(d) == float(np.float32(ours[5].item()))


def test_exact_cases(fn):
    H, W = 47, 66
    x, y = _random_pair(H, W, 5)
    x, y = x.to(DEV), y.to(DEV)
    assert torch.all(fn.terms(x, x) == 0)
    a = fn.terms(x, y)
    assert torch.equal(a, fn.terms(x, y))                         # two calls
    assert torch.equal(a, fn.terms(x[None], y[None]))             # [3,H,W] is [1,3,H,W]
    x2, y2 = _random_pair(H, W, 6)
    x2, y2 = x2.to(DEV), y2.to(DEV)
    b = fn.terms(x2, y2)
    batch = fn.terms(torch.stack([x, x2]), torch.stack([y, y2]))  # the batch sum
    assert torch.allclose(batch, a + b, rtol=1e-12, atol=0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        on_s = fn.terms(x, y)
    torch.cuda.current_stream().wait_stream(s)
    assert torch.equal(a, on_s)


def test_grad_inputs_are_refused_or_detached_under_no_grad(fn):
    x, y = _random_pair(32, 48, 4)
    x, y = x.to(DEV).requires_grad_(), y.to(DEV)
    with pytest.raises(NotImplementedError, match="forward-only"):
        fn(x, y)
    with torch.no_grad():
        d = fn(x, y)
    assert not d.requires_grad and torch.equal(d, fn(x.detach(), y))


def test_inputs_outside_unit_range_are_not_clamped(fn, weights):
    g = torch.Generator().manual_seed(3)
    x = (2.0 * torch.randn(2, 3, 80, 120, generator=g)).to(DEV)
    y = (x + torch.randn(x.shape, generator=g).to(DEV)).to(DEV)
    _check_terms(fn.terms(x, y), vo.lpips_terms(x, y, *weights), "outside [0,1]")
    assert not _tol(float(fn.terms(x, y)[5]), float(fn.terms(x.clamp(0, 1), y.clamp(0, 1))[5]))


def test_no_host_synchronisation(weights, built_lib):
    from s3gaussian_b200.lpips_vgg import LPIPSVGG
    x, y = _random_pair(96, 128, 8)
    x, y = x.to(DEV), y.to(DEV)
    torch.cuda.synchronize()
    fresh = LPIPSVGG.from_state_dicts(*weights)
    torch.cuda.set_sync_debug_mode("error")
    try:
        d1 = fresh(x, y)        # includes the once-per-device weight preparation
        d2 = fresh(x, y)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(d1, d2)


@pytest.mark.skipif(not lpips_vgg_ref.available(),
                    reason="torchvision or oracle/_ref/s3g_ref/lpipsPyTorch (oracle/build_ref_lpips.sh) missing")
@pytest.mark.parametrize("shape", [(3, 47, 66), (2, 3, 160, 240)], ids=["66x47", "2x240x160"])
def test_matches_reference_module_on_device(shape, fn, weights):
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.rand(shape, generator=g).to(DEV)
    y = (x + 0.1 * torch.randn(shape, generator=g).to(DEV)).clamp(0, 1)
    ref = lpips_vgg_ref.reference_module(*weights).to(DEV)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            r = float(ref(x, y))
    finally:
        torch.backends.cudnn.allow_tf32 = old
    assert _tol(float(fn(x, y)), r), (float(fn(x, y)), r)


def test_render_pixels_with_lpips_fn(fn, weights):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.evaluation import render_pixels
    from s3gaussian_b200.gaussian_renderer import PipelineParams
    from test_gpu_eval import _fine_model
    W, H = 240, 160
    pc = _fine_model(60_000, W, H, seed=2)
    pipe = PipelineParams()
    bg = torch.zeros(3, device=DEV)
    cams = syn.waymo_ring(W, H, frames=3)
    g = torch.Generator().manual_seed(9)
    for i, cam in enumerate(cams):
        cam.original_image = torch.rand(3, H, W, generator=g)
        m = torch.zeros(1, H, W, dtype=torch.bool)
        m[0, 10 * i:10 * i + 30, 20:80] = True
        cam.dynamic_mask = m
    plain = render_pixels(cams, pc, bg, pipe)
    res = render_pixels(cams, pc, bg, pipe, lpips_fn=fn)
    per_view = [float(vo.lpips_terms(torch.from_numpy(r).permute(2, 0, 1).to(DEV), cam.original_image.to(DEV),
                                     *weights)[5]) for r, cam in zip(res["rgbs"], cams)]
    ref = sum(per_view) / len(per_view)
    assert plain["lpips"] == -1
    assert _tol(res["lpips"], ref), (res["lpips"], ref)
    assert list(res) == list(plain)
    for k, v in plain.items():
        if k == "lpips":
            continue
        if isinstance(v, list):
            assert len(res[k]) == len(v), k
            for a, b in zip(res[k], v):
                assert (torch.equal(a, b) if torch.is_tensor(a) else np.array_equal(a, b)), k
        else:
            assert res[k] == v, k
