"""GPU: the gradients of LPIPS (s3g_lpips_alex_backward through LPIPS.terms' autograd Function) against autograd of the
float64 oracle and of the reference's own module, the exact cases, the absence of host synchronisation and a
backward through render()."""
import pytest
import torch

import lpips_ref
from oracle import lpips_oracle as lo
from test_gpu_lpips import _random_pair, _rendered_pair

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def weights():
    return lo.random_state_dicts(11)


@pytest.fixture(scope="module")
def fn(weights, built_lib):
    from s3gaussian_b200.lpips import LPIPS
    return LPIPS.from_state_dicts(*weights)


# An isolated max-pool argmax flip (two window values within float32 rounding of each other) sends one pooled
# element's gradient to a neighbour, which moves the image gradient over that element's receptive field.  fp32
# autograd of the same network on the CPU shows it too: one flip among 35k pool-1 windows of an independent random
# 240x160 pair puts it 4.2e-3 (relative L2) and 3.6e-2 (max) from float64.  Independent random pairs and the noisy
# rendered pairs of the size sweep measured up to 1.8e-2 / 0.145 on an H100; where no window flips, the error is below
# 1e-4 / 1e-3, which the other tests hold.
FLIP_REL, FLIP_MAX = 3e-2, 0.25


def _check_grad(ours, ref, what, rel_max=1e-4, worst_max=1e-3):
    """relative L2 error <= rel_max and max |difference| <= worst_max * max |ref|"""
    assert ours.shape == ref.shape and ours.dtype == torch.float32, what
    assert torch.isfinite(ours).all(), what
    d = ours.double() - ref
    rel = float(d.norm() / ref.norm())
    worst = float(d.abs().max() / ref.abs().max())
    assert rel <= rel_max and worst <= worst_max, (what, rel, worst)


def _pairs(H, W, N, case, seed):
    make = _random_pair if case == "random" else _rendered_pair
    ps = [make(H, W, seed + i) for i in range(N)]
    x, y = torch.stack([p[0] for p in ps]), torch.stack([p[1] for p in ps])
    return x.to(DEV), y.to(DEV)


def _grads(terms_of, x, y, wants, weigh=lambda t: t[5]):
    """(terms, gx, gy) of weigh(terms_of(x, y)) with grad on the inputs named in `wants`"""
    xr = x.detach().clone().requires_grad_("x" in wants)
    yr = y.detach().clone().requires_grad_("y" in wants)
    t = terms_of(xr, yr)
    weigh(t).backward()
    return t.detach(), xr.grad, yr.grad


def _oracle(weights, x, y, wants, weigh=lambda t: t[5]):
    return _grads(lambda a, b: lo.lpips_terms(a, b, *weights), x.double(), y.double(), wants, weigh)


@pytest.mark.parametrize("H,W", [(31, 31), (64, 97), (160, 240), (640, 960), (1280, 1920)],
                         ids=["31x31", "97x64", "240x160", "960x640", "1920x1280"])
@pytest.mark.parametrize("case", ["random", "rendered"])
@pytest.mark.parametrize("N,wants", [(1, "x"), (1, "y"), (1, "xy"), (2, "xy")], ids=["N1-x", "N1-y", "N1-xy", "N2-xy"])
def test_gradients_match_fp64_oracle(H, W, case, N, wants, fn, weights):
    x, y = _pairs(H, W, N, case, H + W)
    _, gx, gy = _grads(fn.terms, x, y, wants)
    _, ox, oy = _oracle(weights, x, y, wants)
    for g, o, side in ((gx, ox, "x"), (gy, oy, "y")):
        if side in wants:
            _check_grad(g, o, (H, W, case, N, side), FLIP_REL, FLIP_MAX)
        else:
            assert g is None and o is None


@pytest.mark.parametrize("N,wants", [(2, "x"), (2, "y")], ids=["N2-x", "N2-y"])
def test_one_sided_batch_matches_fp64_oracle(N, wants, fn, weights):
    x, y = _pairs(160, 240, N, "random", 3)
    _, gx, gy = _grads(fn.terms, x, y, wants)
    _, ox, oy = _oracle(weights, x, y, wants)
    g, o = (gx, ox) if wants == "x" else (gy, oy)
    _check_grad(g, o, wants, FLIP_REL, FLIP_MAX)


def test_layer_terms_and_mixtures(fn, weights):
    x, y = _pairs(64, 97, 2, "random", 21)
    for l in range(5):
        pick = lambda t, l=l: t[l]
        _, gx, gy = _grads(fn.terms, x, y, "xy", pick)
        _, ox, oy = _oracle(weights, x, y, "xy", pick)
        _check_grad(gx, ox, ("layer", l, "x"))
        _check_grad(gy, oy, ("layer", l, "y"))
    v = torch.randn(6, generator=torch.Generator().manual_seed(4), dtype=torch.float64).to(DEV)
    mix = lambda t: (t * v).sum()
    _, gx, gy = _grads(fn.terms, x, y, "xy", mix)
    _, ox, oy = _oracle(weights, x, y, "xy", mix)
    _check_grad(gx, ox, "mix x")
    _check_grad(gy, oy, "mix y")


@pytest.mark.skipif(not lpips_ref.available(),
                    reason="torchvision or oracle/_ref/s3g_ref/lpipsPyTorch (oracle/build_ref_lpips.sh) missing")
@pytest.mark.parametrize("shape", [(3, 64, 97), (2, 3, 160, 240)], ids=["97x64", "2x240x160"])
def test_gradients_match_reference_module_on_device(shape, fn, weights):
    g = torch.Generator().manual_seed(sum(shape))
    x = torch.rand(shape, generator=g).to(DEV)
    y = (x + 0.1 * torch.randn(shape, generator=g).to(DEV)).clamp(0, 1)
    ref = lpips_ref.reference_module(*weights).to(DEV)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        xr, yr = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
        ref(xr, yr).sum().backward()
    finally:
        torch.backends.cudnn.allow_tf32 = old
    xo, yo = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    fn(xo, yo).sum().backward()
    assert xo.grad.shape == x.shape and yo.grad.shape == y.shape
    _check_grad(xo.grad, xr.grad.double(), "x")
    _check_grad(yo.grad, yr.grad.double(), "y")


def test_exact_cases(fn, weights):
    from s3gaussian_b200.lpips import LPIPS
    x, y = _pairs(64, 97, 1, "random", 5)
    # x == y: every tap difference is exactly 0
    _, gx, gy = _grads(fn.terms, x, x.clone(), "xy")
    assert torch.all(gx == 0) and torch.all(gy == 0)
    # two forward + backward calls: bitwise equal
    t1, gx1, gy1 = _grads(fn.terms, x, y, "xy")
    t2, gx2, gy2 = _grads(fn.terms, x, y, "xy")
    assert torch.equal(gx1, gx2) and torch.equal(gy1, gy2)
    # the value with grad is the value without
    with torch.no_grad():
        assert torch.equal(t1, fn.terms(x, y))
    assert torch.equal(t1, fn.terms(x, y))
    # conv 3 dead (every output 0): finite gradients, the oracle's
    feat, lin = weights
    dead = dict(feat)
    dead["features.6.bias"] = torch.full_like(feat["features.6.bias"], -1e3)
    fd = LPIPS.from_state_dicts(dead, lin)
    t, gx, gy = _grads(fd.terms, x, y, "xy")
    assert float(t[2]) == 0.0
    _, ox, oy = _oracle((dead, lin), x, y, "xy")
    assert torch.isfinite(ox).all() and torch.isfinite(oy).all()
    _check_grad(gx, ox, "dead x")
    _check_grad(gy, oy, "dead y")


def test_unbatched_input_gets_unbatched_gradient_and_dtype_is_autograds(fn, weights):
    x, y = _pairs(64, 97, 1, "random", 9)
    xh = x[0].half().requires_grad_(True)
    d = fn(xh, y[0])
    d.backward()
    assert xh.grad.shape == (3, 64, 97) and xh.grad.dtype == torch.float16
    _, ox, _ = _oracle(weights, xh.detach().float()[None], y, "x")
    assert torch.allclose(xh.grad.float(), ox[0].float().half().float(), rtol=1e-2, atol=1e-3 * float(ox.abs().max()))


def test_memory_kept_only_between_forward_and_backward(fn):
    x, y = _pairs(160, 240, 1, "random", 12)
    xr = x.clone().requires_grad_(True)
    fn.terms(xr, y)[5].backward()        # weights of both directions prepared
    xr.grad = None
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    with torch.no_grad():
        t = fn.terms(xr, y)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() - base == 512      # the float64 [6] result alone
    del t
    assert torch.cuda.memory_allocated() == base
    t = fn.terms(xr, y)
    from s3gaussian_b200 import _lib
    assert torch.cuda.memory_allocated() - base >= int(_lib.load().s3g_lpips_alex_workspace_bytes(1, 160, 240))
    t[5].backward()
    xr.grad = None
    del t
    assert torch.cuda.memory_allocated() == base


def test_no_host_synchronisation(weights, built_lib):
    from s3gaussian_b200.lpips import LPIPS
    x, y = _pairs(96, 128, 1, "random", 8)
    torch.cuda.synchronize()
    fresh = LPIPS.from_state_dicts(*weights)
    xr = x.clone().requires_grad_(True)
    yr = y.clone().requires_grad_(True)
    torch.cuda.set_sync_debug_mode("error")
    try:
        fresh(xr, yr).backward()         # includes both once-per-device weight preparations
        g1 = xr.grad.clone()
        xr.grad = None
        fresh(xr, yr).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(g1, xr.grad)


def test_backward_through_render(fn, weights):
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_renderer import render, PipelineParams
    from test_gpu_eval import _fine_model
    W, H = 240, 160
    pc = _fine_model(20_000, W, H, seed=3)
    cam = syn.waymo_ring(W, H, frames=3)[1].to(DEV)
    bg = torch.tensor([0.1, 0.2, 0.3], device=DEV)
    gt = torch.rand(3, H, W, generator=torch.Generator().manual_seed(2)).to(DEV)
    params = [p for p in pc.parameters() if p.requires_grad]

    def grads():
        out = [None if p.grad is None else p.grad.detach().clone() for p in params]
        for p in params:
            p.grad = None
        return out

    image = render(cam, pc, PipelineParams(), bg, stage="fine")["render"]
    fn(image, gt).backward()
    ours = grads()
    image = render(cam, pc, PipelineParams(), bg, stage="fine")["render"]
    xo = image.detach().double().requires_grad_(True)
    lo.lpips_terms(xo, gt.double(), *weights)[5].backward()
    image.backward(xo.grad.float())
    ref = grads()
    checked = 0
    for a, b in zip(ours, ref):
        assert (a is None) == (b is None)
        if b is None or float(b.norm()) == 0.0:
            continue
        # the image gradients themselves differ by isolated max-pool flips (FLIP_REL); the rasterizer adds its atomics
        rel = float((a.double() - b.double()).norm() / b.double().norm())
        assert rel <= FLIP_REL, rel
        checked += 1
    assert checked > 0
