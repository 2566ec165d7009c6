"""CPU: the float64 oracle's LPIPS gradients against the reference module's autograd, the sizes and argument errors of
the backward's C entry points, and the CPU refusal of the differentiable path.  Nothing here launches GPU work."""
import ctypes as C

import pytest
import torch

import lpips_ref
from oracle import lpips_oracle as lo


@pytest.mark.skipif(not lpips_ref.available(),
                    reason="torchvision or oracle/_ref/s3g_ref/lpipsPyTorch (oracle/build_ref_lpips.sh) missing")
def test_oracle_gradients_match_reference_module():
    feat, lin = lo.random_state_dicts(3)
    ref = lpips_ref.reference_module(feat, lin)
    assert not any(p.requires_grad for p in ref.parameters())     # frozen, as in lpipsPyTorch
    g = torch.Generator().manual_seed(1)
    x = torch.rand(2, 3, 64, 97, generator=g)
    y = (x + 0.2 * torch.randn(x.shape, generator=g)).clamp(0, 1)
    xr, yr = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    ref(xr, yr).sum().backward()
    xo, yo = x.double().requires_grad_(True), y.double().requires_grad_(True)
    lo.lpips_terms(xo, yo, feat, lin)[5].backward()
    for r, o in ((xr.grad, xo.grad), (yr.grad, yo.grad)):
        d = r.double() - o
        assert float(d.norm() / o.norm()) <= 1e-5
        assert float(d.abs().max() / o.abs().max()) <= 1e-5


def _layer_sizes(H, W):
    """(conv output sizes, max-pool output sizes) of AlexNet's features on an H x W image"""
    conv, pool, h, w = [], [], H, W
    for l, (s, (stride, pad)) in enumerate(zip(lo.CONV_SHAPES, lo.CONV_ARGS)):
        h, w = (h + 2 * pad - s[2]) // stride + 1, (w + 2 * pad - s[3]) // stride + 1
        conv.append(s[0] * h * w)
        if l < 2:
            h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
            pool.append(s[0] * h * w)
    return conv, pool


def test_backward_size_queries(built_lib):
    lib = built_lib
    # conv 1's weights as given, then convs 2-5 as 64 x 32 hi | lo tiles
    tiles = sum(s[0] * s[1] * s[2] * s[3] // (64 * 32) for s in lo.CONV_SHAPES[1:])
    assert lib.s3g_lpips_alex_backward_prepared_bytes() == 4 * (64 * 3 * 11 * 11 + tiles * 2 * 64 * 32)
    r = lambda n: (n + 255) // 256 * 256
    for N, H, W in ((1, 31, 31), (2, 64, 97), (1, 1280, 1920), (3, 640, 960)):
        conv, pool = _layer_sizes(H, W)
        a = 2 * N * max(conv[4], conv[2], conv[1], conv[0])
        b = 2 * N * max(conv[3], pool[1], pool[0])
        assert lib.s3g_lpips_alex_backward_workspace_bytes(N, H, W) == r(4 * a) + r(4 * b) + 256, (N, H, W)
    assert 0.09e9 < lib.s3g_lpips_alex_backward_workspace_bytes(1, 1280, 1920) < 0.1e9
    for n, h, w in ((0, 64, 64), (1, 30, 64), (1, 64, 30), (1, 20000, 20000), (400, 1280, 1920)):
        assert lib.s3g_lpips_alex_workspace_bytes(n, h, w) == 0
        assert lib.s3g_lpips_alex_backward_workspace_bytes(n, h, w) == 0


def test_backward_argument_errors(built_lib):
    from s3gaussian_b200 import _lib
    lib = built_lib
    p = C.c_void_p(256)    # never dereferenced: every call below fails its argument checks first
    odd16, odd8, odd4 = C.c_void_p(256 + 4), C.c_void_p(256 + 4), C.c_void_p(256 + 2)
    ok = dict(N=1, H=64, W=64, prep=p, prep_bwd=p, fwd=p, gout=p, gx=p, gy=p, work=p)
    bad = [dict(N=0), dict(H=30), dict(W=30), dict(H=20000, W=20000), dict(N=400, H=1280, W=1920),
           dict(prep=None), dict(prep_bwd=None), dict(fwd=None), dict(gout=None), dict(work=None),
           dict(gx=None, gy=None), dict(prep=odd16), dict(prep_bwd=odd16), dict(gout=odd8), dict(gx=odd4),
           dict(gy=odd4), dict(gx=None, gy=odd4)]
    for change in bad:
        a = {**ok, **change}
        rc = lib.s3g_lpips_alex_backward(a["N"], a["H"], a["W"], a["prep"], a["prep_bwd"], a["fwd"], a["gout"],
                                         a["gx"], a["gy"], a["work"], None)
        assert rc == -1, change
        assert _lib.last_error()
    assert lib.s3g_lpips_alex_backward_prepare(None, p, None) == -1
    desc = _lib.LpipsAlexWeights()
    assert lib.s3g_lpips_alex_backward_prepare(C.byref(desc), p, None) == -1
    for i in range(5):
        desc.conv_w[i] = 256
    assert lib.s3g_lpips_alex_backward_prepare(C.byref(desc), None, None) == -1
    assert lib.s3g_lpips_alex_backward_prepare(C.byref(desc), odd16, None) == -1


def test_cpu_inputs_that_require_grad_have_no_cpu_path():
    from s3gaussian_b200.lpips import LPIPS
    fn = LPIPS.from_state_dicts(*lo.random_state_dicts(0))
    x = torch.rand(3, 40, 40, requires_grad=True)
    for a, b in ((x, torch.rand(3, 40, 40)), (torch.rand(3, 40, 40), x), (x, x)):
        with pytest.raises(RuntimeError, match="no CPU path"):
            fn(a, b)
    assert fn._prepared == {} and fn._prepared_bwd == {}
