"""CPU: the bilateral-grid restatement (tests/bilagrid_ref.py) against a hand-written trilinear loop, the identity,
gradcheck, hand-computed TV values and the border rule of the luminance guide; the C entry points' argument errors
before any launch; the header in C; and the Python checks that run before any launch."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import bilagrid_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20    # never dereferenced: every call below fails validation before any launch


def _loop_slice(grids, rgb, ids):
    """Per pixel, per corner: the definition written out with plain floats."""
    grids, rgb = grids.numpy(), rgb.numpy()
    B, _, H, W = rgb.shape
    _, _, L, GY, GX = grids.shape
    out = np.zeros_like(rgb)

    def axis(v, size):
        v = min(max(v, 0.0), size - 1.0)
        i0 = min(int(math.floor(v)), size - 1)
        return i0, v - i0

    for b in range(B):
        g = grids[ids[b]]
        for i in range(H):
            for j in range(W):
                r, gg, bl = rgb[b, :, i, j]
                x0, fx = axis((j + 0.5) / W * (GX - 1), GX)
                y0, fy = axis((i + 0.5) / H * (GY - 1), GY)
                z0, fz = axis((0.299 * r + 0.587 * gg + 0.114 * bl) * (L - 1), L)
                A = np.zeros(12)
                for dz, wz in ((0, 1 - fz), (1, fz)):
                    for dy, wy in ((0, 1 - fy), (1, fy)):
                        for dx, wx in ((0, 1 - fx), (1, fx)):
                            w = wz * wy * wx
                            if w == 0:
                                continue
                            A += w * g[:, z0 + dz, y0 + dy, x0 + dx]
                A = A.reshape(3, 4)
                out[b, :, i, j] = A[:, :3] @ np.array([r, gg, bl]) + A[:, 3]
    return torch.from_numpy(out)


@pytest.mark.parametrize("shape", [(4, 3, 5), (1, 1, 1), (2, 1, 3), (3, 4, 1)])
def test_restatement_matches_the_trilinear_loop(shape):
    L, GY, GX = shape
    g = torch.Generator().manual_seed(L * 100 + GY * 10 + GX)
    grids = ref.identity_grids(3, L, GY, GX) + 0.3 * torch.randn(3, 12, L, GY, GX, dtype=torch.float64, generator=g)
    rgb = torch.rand(2, 3, 7, 6, dtype=torch.float64, generator=g) * 1.5 - 0.2
    rgb[0, :, 0, 0] = 0.0      # black: z = 0
    rgb[1, :, 1, 1] = 1.0      # white: z = L - 1 (up to the rounding of the luminance weights)
    ids = [2, 0]
    torch.testing.assert_close(ref.slice64(grids, rgb, ids, torch.float64), _loop_slice(grids, rgb, ids), rtol=1e-12,
                               atol=1e-12)
    # the default float32 guide moves z by float32 rounding only
    torch.testing.assert_close(ref.slice64(grids, rgb, ids), _loop_slice(grids, rgb, ids), rtol=0, atol=1e-5)


def test_identity_grid_gives_back_its_input():
    rgb = torch.rand(2, 3, 9, 11, dtype=torch.float64) * 1.5 - 0.2
    for shape in ((8, 16, 16), (1, 1, 1), (5, 3, 2)):
        torch.testing.assert_close(ref.slice64(ref.identity_grids(2, *shape), rgb, [1, 0]), rgb, rtol=0, atol=1e-14)


def test_restatement_passes_gradcheck():
    g = torch.Generator().manual_seed(4)
    grids = (ref.identity_grids(2, 3, 3, 4) + 0.2 * torch.randn(2, 12, 3, 3, 4, dtype=torch.float64, generator=g))
    rgb = torch.rand(1, 3, 5, 4, dtype=torch.float64, generator=g) * 0.8 + 0.1     # luminance away from the clamps
    assert torch.autograd.gradcheck(lambda G, x: ref.slice64(G, x, [1], torch.float64),
                                    (grids.requires_grad_(True), rgb.requires_grad_(True)))
    assert torch.autograd.gradcheck(ref.tv64, (grids.detach().clone().requires_grad_(True),))


def test_tv_by_hand():
    # one grid, L = 1, GY = 1, GX = 2: only x differences, 12 channels of (1 - 0)^2 over count 12 * 1 * 1 * 1
    g = torch.zeros(1, 12, 1, 1, 2, dtype=torch.float64)
    g[..., 1] = 1.0
    assert float(ref.tv64(g)) == pytest.approx(1.0)
    # two grids, L = 2, GY = 1, GX = 1: only z differences; grid 0 differs by 2 in channel 0, grid 1 by 1 in every
    # channel; sum = 4 + 12 over count 12, halved for N = 2
    g = torch.zeros(2, 12, 2, 1, 1, dtype=torch.float64)
    g[0, 0, 1] = 2.0
    g[1, :, 1] = 1.0
    assert float(ref.tv64(g)) == pytest.approx((4.0 + 12.0) / 12.0 / 2.0)
    # every axis of size 1: 0
    assert float(ref.tv64(torch.randn(3, 12, 1, 1, 1, dtype=torch.float64))) == 0.0
    # the identity is constant: 0
    assert float(ref.tv64(ref.identity_grids(2, 8, 16, 16))) == 0.0
    # a ramp along y only, GY = 3, L = 2, GX = 4: per difference 0.25^2, 12 * 2 * 2 * 4 differences, count 12 * 2 * 2 * 4
    g = (0.5 * torch.arange(3, dtype=torch.float64) / 2).reshape(1, 1, 1, 3, 1).expand(1, 12, 2, 3, 4).contiguous()
    assert float(ref.tv64(g)) == pytest.approx(0.0625)


def test_border_rule_at_black_and_white():
    """At z = 0 (black) and z = L - 1 (white) the luminance guide passes no gradient: grad_rgb = A[:, :3]^T grad_out,
    with A the bilinear sample of the bottom or top level."""
    g = torch.Generator().manual_seed(5)
    L = 4
    grids = ref.identity_grids(1, L, 2, 2) + 0.5 * torch.randn(1, 12, L, 2, 2, dtype=torch.float64, generator=g)
    one = torch.ones((), dtype=torch.float32)
    assert float(0.299 * one + 0.587 * one + 0.114 * one) == 1.0     # white's float32 luminance is on the clamp
    for v, level in ((0.0, 0), (1.0, L - 1)):
        rgb = torch.full((1, 3, 1, 1), v, dtype=torch.float64, requires_grad=True)
        go = torch.randn(1, 3, 1, 1, dtype=torch.float64, generator=g)
        (gr,) = torch.autograd.grad(ref.slice64(grids, rgb, [0]), rgb, go)
        A = grids[0, :, level].mean(dim=(1, 2)).reshape(3, 4)          # the 1x1 image samples the 2x2 cells' centre
        torch.testing.assert_close(gr.reshape(3), A[:, :3].t() @ go.reshape(3), rtol=1e-12, atol=1e-12)
    # just inside the clamp the guide does pass a gradient
    rgb = torch.full((1, 3, 1, 1), 0.5, dtype=torch.float64, requires_grad=True)
    go = torch.randn(1, 3, 1, 1, dtype=torch.float64, generator=g)
    (gr,) = torch.autograd.grad(ref.slice64(grids, rgb, [0]), rgb, go)
    A = 0.5 * (grids[0, :, 1] + grids[0, :, 2]).mean(dim=(1, 2)).reshape(3, 4)
    assert float((gr.reshape(3) - A[:, :3].t() @ go.reshape(3)).abs().max()) > 1e-3


# ---- the C entry points -----------------------------------------------------------------------------------------------
def _ids(*v):
    return (C.c_int32 * len(v))(*v)


def test_slice_argument_errors_before_any_launch(built_lib):
    lib = built_lib

    def fwd(N=4, L=8, GY=16, GX=16, grids=FAKE, B=2, H=6, W=8, ids=None, rgb=FAKE, out=FAKE):
        return lib.s3g_bilagrid_slice_forward(N, L, GY, GX, grids, B, H, W, _ids(0, 3) if ids is None else ids, rgb,
                                              out, None)

    def bwd(N=4, L=8, GY=16, GX=16, grids=FAKE, B=2, H=6, W=8, ids=None, rgb=FAKE, go=FAKE, grgb=FAKE, gg=FAKE,
            ws=FAKE):
        return lib.s3g_bilagrid_slice_backward(N, L, GY, GX, grids, B, H, W, _ids(0, 3) if ids is None else ids, rgb,
                                               go, grgb, gg, ws, None)
    common = [({"N": 0}, b"size <= 0"), ({"L": 0}, b"size <= 0"), ({"GY": -1}, b"size <= 0"), ({"GX": 0}, b"size <= 0"),
              ({"B": 0}, b"size <= 0"), ({"H": 0}, b"size <= 0"), ({"W": -2}, b"size <= 0"),
              ({"grids": None}, b"null pointer"), ({"rgb": None}, b"null pointer"),
              ({"ids": _ids(0, 4)}, b"outside [0, N)"), ({"ids": _ids(-1, 2)}, b"outside [0, N)"),
              ({"ids": _ids(3, 3)}, b"duplicate"),
              ({"N": 1 << 20, "ids": _ids(0, 1)}, b"32-bit"), ({"H": 1 << 15, "W": 1 << 15}, b"32-bit")]
    for kw, msg in common + [({"out": None}, b"null pointer")]:
        assert fwd(**kw) == -1, kw
        assert msg in lib.s3g_last_error(), (kw, lib.s3g_last_error())
    for kw, msg in common + [({"go": None}, b"null pointer"), ({"gg": None}, b"null pointer"),
                             ({"ws": None}, b"null pointer"), ({"ws": FAKE + 4}, b"16-byte")]:
        assert bwd(**kw) == -1, kw
        assert msg in lib.s3g_last_error(), (kw, lib.s3g_last_error())
    # the NULL ids array is refused too
    assert lib.s3g_bilagrid_slice_forward(4, 8, 16, 16, FAKE, 2, 6, 8, None, FAKE, FAKE, None) == -1
    assert b"null pointer" in lib.s3g_last_error()


def test_workspace_sizes(built_lib):
    lib = built_lib
    # 16x16x8 at 960x640: each column's support is at most 2 * 960 / 15 + 6 by 2 * 640 / 15 + 6 pixels, 3 slices of
    # 4096; one level chunk; 12 * 8 floats per partial
    assert lib.s3g_bilagrid_slice_backward_workspace_bytes(150, 8, 16, 16, 1, 640, 960) == 4 * 256 * 3 * 96
    assert lib.s3g_bilagrid_slice_backward_workspace_bytes(150, 16, 16, 16, 2, 640, 960) == 4 * 2 * 2 * 256 * 3 * 96
    assert lib.s3g_bilagrid_slice_backward_workspace_bytes(1, 1, 1, 1, 1, 6, 8) == 4 * 96
    assert lib.s3g_bilagrid_slice_backward_workspace_bytes(0, 8, 16, 16, 1, 640, 960) == 0
    assert lib.s3g_bilagrid_tv_workspace_bytes(150, 8, 16, 16) == 8 * 1024
    assert lib.s3g_bilagrid_tv_workspace_bytes(1, 1, 1, 1) == 8
    assert lib.s3g_bilagrid_tv_workspace_bytes(1, 0, 1, 1) == 0


def test_tv_argument_errors_before_any_launch(built_lib):
    lib = built_lib
    fwd = lambda N=2, L=8, GY=4, GX=4, g=FAKE, loss=FAKE, ws=FAKE: lib.s3g_bilagrid_tv_forward(N, L, GY, GX, g, loss, ws,
                                                                                                None)
    bwd = lambda N=2, L=8, GY=4, GX=4, g=FAKE, gs=FAKE, out=FAKE: lib.s3g_bilagrid_tv_backward(N, L, GY, GX, g, gs, out,
                                                                                                None)
    for fn, ptrs in ((fwd, ("g", "loss", "ws")), (bwd, ("g", "gs", "out"))):
        for kw in ({"N": 0}, {"L": -1}, {"GY": 0}, {"GX": 0}):
            assert fn(**kw) == -1 and b"size <= 0" in lib.s3g_last_error(), kw
        assert fn(N=1 << 22) == -1 and b"32-bit" in lib.s3g_last_error()
        for p in ptrs:
            assert fn(**{p: None}) == -1 and b"null pointer" in lib.s3g_last_error(), p
    assert fwd(ws=FAKE + 4) == -1 and b"8-byte" in lib.s3g_last_error()


def test_header_declares_the_entry_points_in_c(built_lib, tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    from s3gaussian_b200 import _lib
    libdir = os.path.dirname(_lib.LIB_PATH)
    src = tmp_path / "bg.c"
    src.write_text('#include <stddef.h>\n#include <stdint.h>\n#include "s3g_b200.h"\n'
                   'int main(void) {\n'
                   '    float* p = NULL;\n'
                   '    int32_t ids[1] = {0};\n'
                   '    size_t ws = s3g_bilagrid_slice_backward_workspace_bytes(1, 1, 1, 1, 1, 6, 8);\n'
                   '    size_t wt = s3g_bilagrid_tv_workspace_bytes(1, 1, 1, 1);\n'
                   '    int a = s3g_bilagrid_slice_forward(1, 1, 1, 1, p, 1, 6, 8, ids, p, p, NULL);\n'
                   '    int b = s3g_bilagrid_slice_backward(1, 1, 1, 1, p, 1, 6, 8, ids, p, p, p, p, NULL, NULL);\n'
                   '    int c = s3g_bilagrid_tv_forward(0, 1, 1, 1, p, p, NULL, NULL);\n'
                   '    int d = s3g_bilagrid_tv_backward(0, 1, 1, 1, p, p, p, NULL);\n'
                   '    return (ws == 384 && wt == 8 && a == S3G_ERR_ARG && b == S3G_ERR_ARG && c == S3G_ERR_ARG &&\n'
                   '            d == S3G_ERR_ARG) ? 0 : 1;\n'
                   '}\n')
    exe = tmp_path / "bg"
    r = subprocess.run([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                        "-o", str(exe), "-L", libdir, "-ls3g_b200", f"-Wl,-rpath,{libdir}"], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = "/usr/local/cuda/lib64" + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    assert subprocess.run([str(exe)], env=env).returncode == 0


# ---- Python ----------------------------------------------------------------------------------------------------------
def test_module_layout_and_state_dict():
    from s3gaussian_b200.bilateral_grid import BilateralGrid
    m = BilateralGrid(5)
    assert tuple(m.grids.shape) == (5, 12, 8, 16, 16) and m.grids.is_contiguous() and m.grids.dtype == torch.float32
    assert torch.equal(m.grids.double(), ref.identity_grids(5, 8, 16, 16))
    m2 = BilateralGrid(3, grid_X=4, grid_Y=2, grid_W=1)
    assert tuple(m2.grids.shape) == (3, 12, 1, 2, 4) and list(m2.state_dict()) == ["grids"]
    # a state dict whose grids is a permuted (non-contiguous) view, as gsplat builds it, loads unchanged
    src = torch.randn(3, 1, 2, 4, 12).permute(0, 4, 1, 2, 3)
    m2.load_state_dict({"grids": src})
    assert torch.equal(m2.grids, src) and m2.grids.is_contiguous()
    for bad in ({"num": 0}, {"num": 2, "grid_X": 0}, {"num": 2, "grid_W": 1.5}, {"num": True}):
        with pytest.raises(ValueError, match="integer >= 1"):
            BilateralGrid(**bad)


def test_python_errors_before_any_launch():
    from s3gaussian_b200.bilateral_grid import BilateralGrid
    m = BilateralGrid(4, grid_X=4, grid_Y=4, grid_W=2)
    x = torch.rand(3, 6, 8)
    for rgb, match in ((torch.rand(4, 6, 8), r"\[3,H,W\]"), (torch.rand(6, 8), r"\[3,H,W\]"),
                       (torch.rand(1, 1, 3, 6, 8), r"\[3,H,W\]"), (torch.rand(3, 0, 8), "not empty"),
                       (x.double(), "float32"), (torch.rand(3, 8, 6).transpose(1, 2), "contiguous"),
                       ("image", r"\[3,H,W\]")):
        with pytest.raises(ValueError, match=match):
            m.slice(rgb, 0)
    for ids, match in ((4, "outside"), (-1, "outside"), ([0, 1], "2 image ids for 1"), ([], "0 image ids"),
                       (1.0, "int or a sequence"), ([0.0], "all be ints"), (True, "int or a sequence"),
                       (torch.tensor([0]), "not a tensor")):
        with pytest.raises(ValueError, match=match):
            m.slice(x, ids)
    xb = torch.rand(3, 3, 6, 8)
    with pytest.raises(ValueError, match="duplicate"):
        m.slice(xb, [0, 2, 0])
    with pytest.raises(ValueError, match="outside"):
        m.slice(xb, (0, 1, 4))
    # well-formed, but on the CPU
    with pytest.raises(RuntimeError, match="CUDA"):
        m.slice(x, 0)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.slice(xb, range(3))
    with pytest.raises(RuntimeError, match="CUDA"):
        m.tv_loss()
    with torch.no_grad():
        m.grids.data = m.grids.data.double()
    with pytest.raises(ValueError, match="float32"):
        m.tv_loss()
