"""CPU: the 3-D smoothing filter without a GPU - the float64 restatement (tests/filter3d_ref.py) on hand-computed cases,
gradcheck and the closed-form backward of the apply, argument errors of the three entry points before any launch, the
header in C, and the Python errors and dispatch that need no device."""
import ctypes as C
import math
import os
import shutil
import subprocess
from types import SimpleNamespace

import pytest
import torch

import filter3d_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20    # never dereferenced: every call below fails validation before any launch


# ---- the restatement --------------------------------------------------------------------------------------------------
def _cam(width, height, focal, R=None, t=(0.0, 0.0, 0.0)):
    """views [16] for x_cam = R x + t in the rasterizer's layout, cams [4]."""
    M = torch.eye(4, dtype=torch.float64)
    if R is not None:
        M[:3, :3] = torch.as_tensor(R, dtype=torch.float64)
    M[:3, 3] = torch.as_tensor(t, dtype=torch.float64)
    return M.t().reshape(16), torch.tensor([width, height, focal, focal], dtype=torch.float64)


def _cams(*cs):
    return torch.stack([c[0] for c in cs]), torch.stack([c[1] for c in cs])


def test_compute_restatement_by_hand():
    """Identity camera 100x80, focal 50: (0,0,5) is seen at z = 5, (0,0,2) at 2 from a second camera 3 m behind it
    ... F is the larger focal of the two, unseen points take the largest seen depth."""
    views, cams = _cams(_cam(100, 80, 50.0), _cam(200, 80, 70.0, t=(0.0, 0.0, -3.0)))
    xyz = torch.tensor([[0.0, 0.0, 5.0],      # camera 0 at z = 5, camera 1 at z = 2
                        [0.0, 0.0, 7.0],      # z = 7 and 4
                        [0.0, 0.0, -1.0],     # behind both
                        [100.0, 0.0, 10.0]])  # beside both: u = 100 / 10 * 50 + 50 = 550 > 115
    f, seen = ref.compute64(xyz, views, cams)
    assert seen.tolist() == [True, True, False, False]
    F = 70.0
    torch.testing.assert_close(f, torch.tensor([2.0, 4.0, 4.0, 4.0], dtype=torch.float64) / F * math.sqrt(0.2))
    f, seen = ref.compute64(xyz[2:], views, cams)            # nobody seen: zeros
    assert not seen.any() and torch.equal(f, torch.zeros(2, dtype=torch.float64))


def test_compute_restatement_matches_the_camera_loop():
    """compute64 against a per-camera loop in Mip-Splatting's form (x_cam = xyz @ R + T, one clamped division)."""
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.filter3d import camera_tensors
    cams_list = syn.waymo_ring(320, 200, frames=4)
    xyz = syn.make_cloud(3000, seed=2, width=320, height=200).xyz
    views, cams = camera_tensors(cams_list, "cpu")
    f, _ = ref.compute64(xyz, views, cams)
    X = xyz.double()
    distance = torch.full((X.shape[0],), 1e5, dtype=torch.float64)
    valid_points = torch.zeros(X.shape[0], dtype=torch.bool)
    focal_length = 0.0
    for c in cams_list:
        W2C = c.world_view_transform.double().t()
        p = X @ W2C[:3, :3].t() + W2C[:3, 3]
        fx = c.image_width / (2 * math.tan(c.FoVx / 2))
        fy = c.image_height / (2 * math.tan(c.FoVy / 2))
        valid_depth = p[:, 2] > 0.2
        z = p[:, 2].clamp(min=0.001)
        x = p[:, 0] / z * fx + c.image_width / 2.0
        y = p[:, 1] / z * fy + c.image_height / 2.0
        in_screen = (x >= -0.15 * c.image_width) & (x <= c.image_width * 1.15) & (y >= -0.15 * c.image_height) & (
            y <= 1.15 * c.image_height)
        valid = valid_depth & in_screen
        distance[valid] = torch.min(distance[valid], z[valid])
        valid_points |= valid
        focal_length = max(focal_length, fx)
    distance[~valid_points] = distance[valid_points].max()
    assert 0 < int((~valid_points).sum()) < X.shape[0]
    torch.testing.assert_close(f, distance / float(torch.tensor(focal_length, dtype=torch.float32)) * 0.2 ** 0.5,
                               rtol=1e-7, atol=0)


def _apply_inputs(n, seed):
    g = torch.Generator().manual_seed(seed)
    s = torch.exp(torch.empty(n, 3, dtype=torch.float64).uniform_(-8, 0, generator=g))
    o = torch.empty(n, 1, dtype=torch.float64).uniform_(0.05, 0.99, generator=g)
    f = torch.exp(torch.empty(n, 1, dtype=torch.float64).uniform_(-7, -2, generator=g))
    return s, o, f


def test_apply_restatement_passes_gradcheck():
    s, o, f = _apply_inputs(32, 1)
    assert torch.autograd.gradcheck(lambda s, o: ref.apply64(s, o, f), (s.requires_grad_(True), o.requires_grad_(True)))


def test_apply_backward_matches_the_closed_form():
    s, o, f = _apply_inputs(4096, 2)
    s.requires_grad_(True)
    o.requires_grad_(True)
    g = torch.Generator().manual_seed(3)
    gs, go = torch.randn(4096, 3, dtype=torch.float64, generator=g), torch.randn(4096, 1, dtype=torch.float64, generator=g)
    sf, of = ref.apply64(s, o, f)
    ds, do = torch.autograd.grad((sf * gs).sum() + (of * go).sum(), (s, o))
    cs, co = ref.apply_backward64(s.detach(), o.detach(), f, gs, go)
    torch.testing.assert_close(ds, cs, rtol=1e-10, atol=0)
    torch.testing.assert_close(do, co, rtol=1e-10, atol=0)
    # the integrated density o prod s is kept
    torch.testing.assert_close(of * sf.prod(1, keepdim=True), o * s.prod(1, keepdim=True), rtol=1e-12, atol=0)


# ---- the C entry points -----------------------------------------------------------------------------------------------
def test_compute_argument_errors_before_any_launch(built_lib):
    lib = built_lib
    ws = FAKE

    def call(P=8, xyz=FAKE, Cn=2, views=FAKE, cams=FAKE, out=FAKE, ws=ws):
        return lib.s3g_filter3d_compute(P, xyz, Cn, views, cams, out, ws, None)
    assert lib.s3g_filter3d_compute_workspace_bytes(8) == 16 and lib.s3g_filter3d_compute_workspace_bytes(0) == 0
    assert call(P=0, xyz=None, Cn=0, views=None, cams=None, out=None, ws=None) == 0    # nothing to do
    for kw, msg in (({"P": -1}, b"P < 0"), ({"Cn": 0}, b"C < 1"), ({"Cn": -3}, b"C < 1"),
                    ({"xyz": None}, b"null pointer"), ({"views": None}, b"null pointer"),
                    ({"cams": None}, b"null pointer"), ({"out": None}, b"null pointer"), ({"ws": None}, b"null pointer"),
                    ({"ws": FAKE + 4}, b"not 16-byte aligned"), ({"P": (1 << 31) // 3 + 1}, b"32-bit"),
                    ({"Cn": (1 << 31) // 16 + 1}, b"32-bit")):
        assert call(**kw) == -1, kw
        assert msg in lib.s3g_last_error(), (kw, lib.s3g_last_error())


def test_apply_argument_errors_before_any_launch(built_lib):
    lib = built_lib
    fwd = lambda P, *p: lib.s3g_filter3d_apply_forward(P, *p, None)
    bwd = lambda P, *p: lib.s3g_filter3d_apply_backward(P, *p, None)
    for fn, n in ((fwd, 5), (bwd, 7)):
        assert fn(0, *([None] * n)) == 0
        assert fn(-1, *([FAKE] * n)) == -1 and b"P < 0" in lib.s3g_last_error()
        assert fn((1 << 31) // 3 + 1, *([FAKE] * n)) == -1 and b"32-bit" in lib.s3g_last_error()
        for k in range(n):
            p = [FAKE] * n
            p[k] = None
            assert fn(4, *p) == -1 and b"null pointer" in lib.s3g_last_error(), k


def test_header_declares_the_entry_points_in_c(built_lib, tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    from s3gaussian_b200 import _lib
    libdir = os.path.dirname(_lib.LIB_PATH)
    src = tmp_path / "f3d.c"
    src.write_text('#include <stddef.h>\n#include "s3g_b200.h"\n'
                   'int main(void) {\n'
                   '    float* p = NULL;\n'
                   '    size_t ws = s3g_filter3d_compute_workspace_bytes(8);\n'
                   '    int a = s3g_filter3d_compute(8, p, 0, p, p, p, NULL, NULL);\n'
                   '    int b = s3g_filter3d_apply_forward(-1, p, p, p, p, p, NULL);\n'
                   '    int c = s3g_filter3d_apply_backward(-1, p, p, p, p, p, p, p, NULL);\n'
                   '    return (ws == 16 && a == S3G_ERR_ARG && b == S3G_ERR_ARG && c == S3G_ERR_ARG) ? 0 : 1;\n'
                   '}\n')
    exe = tmp_path / "f3d"
    r = subprocess.run([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                        "-o", str(exe), "-L", libdir, "-ls3g_b200", f"-Wl,-rpath,{libdir}"], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = "/usr/local/cuda/lib64" + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    assert subprocess.run([str(exe)], env=env).returncode == 0


# ---- Python ----------------------------------------------------------------------------------------------------------
def test_camera_tensors_layout():
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.filter3d import camera_tensors
    cams = [syn.make_camera(640, 400, (1.0, 2.0, 3.0), yaw_deg=20.0), syn.make_camera(320, 240, (0.0, 0.0, 0.0),
                                                                                       focal=111.0)]
    views, k = camera_tensors(cams, "cpu")
    assert views.shape == (2, 16) and k.shape == (2, 4) and views.dtype == k.dtype == torch.float32
    assert torch.equal(views[0], cams[0].world_view_transform.reshape(16))
    torch.testing.assert_close(k[0], torch.tensor([640.0, 400.0, syn.WAYMO_FOCAL / 3, syn.WAYMO_FOCAL / 3]))
    torch.testing.assert_close(k[1], torch.tensor([320.0, 240.0, 111.0, 111.0]))


def test_python_errors_without_a_device():
    from s3gaussian_b200.filter3d import apply_filter_3d, compute_filter_3d
    from s3gaussian_b200.gaussian_model import GaussianModel
    s, o, f = torch.ones(4, 3), torch.ones(4, 1), torch.zeros(4, 1)
    with pytest.raises(RuntimeError, match="CUDA"):
        apply_filter_3d(s, o, f)
    with pytest.raises(ValueError, match="must be"):
        apply_filter_3d(s, o, torch.zeros(5, 1))
    with pytest.raises(ValueError, match="must be"):
        apply_filter_3d(torch.ones(4, 2), o, f)
    with pytest.raises(RuntimeError, match="CUDA"):
        compute_filter_3d(torch.zeros(4, 3), [object()])
    g = GaussianModel(0)
    assert g.filter_3D.numel() == 0
    for prop in ("get_scaling_with_3D_filter", "get_opacity_with_3D_filter"):
        with pytest.raises(RuntimeError, match="compute_3D_filter"):
            getattr(g, prop)


def _fake_render(monkeypatch):
    """render() with a recording rasterizer and apply_filter_3d on CPU tensors."""
    from s3gaussian_b200 import gaussian_renderer as gr
    calls = []

    class FakeRasterizer:
        def __init__(self, raster_settings, **kw):
            calls.append(("rasterizer", kw))

        def __call__(self, means3D, **kw):
            calls.append(("raster", kw["scales"], kw["opacities"]))
            z = torch.zeros(1, 4, 4)
            return torch.zeros(3, 4, 4), torch.ones(means3D.shape[0], dtype=torch.int32), z

    def fake_apply(scales, opacity, filter_3d):
        calls.append(("apply", scales, opacity, filter_3d))
        return scales + 1, opacity * 0.5
    monkeypatch.setattr(gr, "GaussianRasterizer", FakeRasterizer)
    monkeypatch.setattr(gr, "apply_filter_3d", fake_apply)
    monkeypatch.setattr(gr, "raster_settings_for", lambda *a, **k: SimpleNamespace(campos=torch.zeros(3)))
    pc = SimpleNamespace(get_xyz=torch.zeros(5, 3), get_features=torch.zeros(5, 16, 3), _scaling=torch.zeros(5, 3),
                         _rotation=torch.ones(5, 4), _opacity=torch.zeros(5, 1), scaling_activation=torch.exp,
                         rotation_activation=torch.nn.functional.normalize, opacity_activation=torch.sigmoid)
    return gr, pc, calls


def test_render_switch_dispatch(monkeypatch):
    """Off or absent: no apply; on: the rasterizer receives apply_filter_3d's outputs of the activated tensors."""
    gr, pc, calls = _fake_render(monkeypatch)
    pipe = gr.PipelineParams()
    assert pipe.filter_3d is False
    gr.render(None, pc, pipe, torch.zeros(3), stage="coarse")
    legacy = SimpleNamespace(compute_cov3D_python=False, convert_SHs_python=False, debug=False)
    gr.render(None, pc, legacy, torch.zeros(3), stage="coarse")
    assert [c[0] for c in calls] == ["rasterizer", "raster"] * 2
    calls.clear()
    pipe.filter_3d = True
    pc.filter_3D = torch.full((5, 1), 0.25)
    gr.render(None, pc, pipe, torch.zeros(3), stage="coarse")
    assert [c[0] for c in calls] == ["rasterizer", "apply", "raster"]
    _, s, o, f = calls[1]
    assert torch.equal(s, torch.ones(5, 3)) and torch.equal(o, torch.full((5, 1), 0.5)) and f is pc.filter_3D
    assert torch.equal(calls[2][1], s + 1) and torch.equal(calls[2][2], o * 0.5)


def test_render_switch_errors_before_any_call(monkeypatch):
    gr, pc, calls = _fake_render(monkeypatch)
    pipe = gr.PipelineParams()
    pipe.filter_3d = True
    for filt in (None, torch.empty(0), torch.zeros(4, 1)):
        if filt is not None:
            pc.filter_3D = filt
        for stage in ("coarse", "fine"):
            with pytest.raises(RuntimeError, match="compute_3D_filter"):
                gr.render(None, pc, pipe, torch.zeros(3), stage=stage)
    pc.filter_3D = torch.zeros(5, 1)
    pipe.compute_cov3D_python = True
    for stage in ("coarse", "fine"):
        with pytest.raises(NotImplementedError, match="precomputed covariances"):
            gr.render(None, pc, pipe, torch.zeros(3), stage=stage)
    assert calls == []
