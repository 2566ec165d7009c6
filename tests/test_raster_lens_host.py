"""CPU: the rasterizer's lens projection without a GPU - the float64 restatement (gradcheck, OpenCV's formula), the
host's lens-cull bound against numpy.roots, argument errors of s3g_rasterize_forward_lens and of the backwards after
it (before any launch), the header, and the Python dispatch with a fake library object."""
import ctypes as C
import math
import os
import shutil
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import lens_ref
from test_raster_aa_host import FAKE, _bwd, _Ctx, _FakeLib, _fwd, _scene, _settings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LENS = (120.0, 110.0, 35.5, 22.0, -0.2, 0.05, 0.01, -0.004, 0.02)


# ---- the restatement ---------------------------------------------------------------------------------------------------
def _leaf(n, seed, cov=False):
    g = torch.Generator().manual_seed(seed)
    u = lambda *s, lo=-1.0, hi=1.0: torch.empty(*s, dtype=torch.float64).uniform_(lo, hi, generator=g)
    z = u(n, lo=2.0, hi=6.0)
    # inside the clamp of J_n, where the restatement is differentiable
    leaf = {"means3D": torch.stack([u(n, lo=-0.2, hi=0.2) * z, u(n, lo=-0.15, hi=0.15) * z, z], 1),
            "opacities": u(n, 1, lo=0.1, hi=0.9)}
    if cov:
        L = u(n, 3, 3, lo=-0.1, hi=0.1) + 0.1 * torch.eye(3, dtype=torch.float64)
        S = L @ L.transpose(1, 2)
        leaf["cov3D"] = torch.stack([S[:, 0, 0], S[:, 0, 1], S[:, 0, 2], S[:, 1, 1], S[:, 1, 2], S[:, 2, 2]], 1)
    else:
        leaf["scales"] = u(n, 3, lo=0.02, hi=0.2)
        leaf["rotations"] = u(n, 4)
    c, s = math.cos(0.05), math.sin(0.05)
    R = torch.tensor([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=torch.float64)
    V = torch.eye(4, dtype=torch.float64)
    V[:3, :3] = R
    V[:3, 3] = torch.tensor([0.1, -0.2, 0.3])
    leaf["view"] = V.T.contiguous()   # stored transposed, as the rasterizer's viewmatrix
    return leaf


@pytest.mark.parametrize("cov,aa", [(False, False), (True, True)])
def test_restatement_passes_gradcheck(cov, aa):
    d = dict(W=72, H=48)
    leaf = _leaf(12, 3, cov)
    keys = [k for k in ("means3D", "opacities", "scales", "rotations", "cov3D") if k in leaf]

    def f(*args):
        lf = dict(leaf, **dict(zip(keys, args)))
        r = lens_ref.project64(d, lf, LENS, aa)
        return r["ndc"], r["conic"], r["depth"], r["alpha_eff"]
    assert torch.autograd.gradcheck(f, tuple(leaf[k].clone().requires_grad_(True) for k in keys))


def test_distortion_equals_the_opencv_formula():
    """OpenCV's documented radial-tangential model (calib3d, projectPoints), transcribed in numpy."""
    rng = np.random.default_rng(0)
    x, y = rng.uniform(-0.8, 0.8, 500), rng.uniform(-0.6, 0.6, 500)
    fx, fy, cx, cy, k1, k2, p1, p2, k3 = LENS
    r2 = x * x + y * y
    radial = 1 + k1 * r2 + k2 * r2 ** 2 + k3 * r2 ** 3
    xpp = x * radial + 2 * p1 * x * y + p2 * (r2 + 2 * x * x)
    ypp = y * radial + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y
    xd, yd, _ = lens_ref.distort(LENS, torch.from_numpy(x), torch.from_numpy(y))
    np.testing.assert_allclose(xd.numpy(), xpp, rtol=1e-14, atol=1e-15)
    np.testing.assert_allclose(yd.numpy(), ypp, rtol=1e-14, atol=1e-15)
    # the pixel with OpenCV's centre at j is ours with the centre at j + 0.5
    leaf = {"means3D": torch.from_numpy(np.stack([x * 3, y * 3, np.full(500, 3.0)], 1)),
            "opacities": torch.full((500, 1), 0.5, dtype=torch.float64),
            "scales": torch.full((500, 3), 0.05, dtype=torch.float64),
            "rotations": torch.tensor([[1.0, 0, 0, 0]], dtype=torch.float64).repeat(500, 1),
            "view": torch.eye(4, dtype=torch.float64)}
    pix = lens_ref.project64(dict(W=72, H=48), leaf, LENS)["pix"].numpy()
    np.testing.assert_allclose(pix[:, 0], fx * xpp + (cx - 0.5), rtol=1e-12)
    np.testing.assert_allclose(pix[:, 1], fy * ypp + (cy - 0.5), rtol=1e-12)


K_TABLE = [(0.0, 0.0, 0.0), (0.1, 0.02, 0.0), (-0.2, 0.0, 0.0), (-0.3, 0.1, 0.0), (-0.25, 0.06, -0.01),
           (0.2, -0.1, 0.0), (0.0, 0.0, -0.9), (0.0, 0.0, 0.5), (0.5, -2.0, 1.0), (-1e-3, 0.0, 0.0),
           (0.3, 0.0, -1e-4), (-0.4, 0.3, -0.06), (1.0, 1.0, 1.0)]


@pytest.mark.parametrize("k1,k2,k3", K_TABLE)
def test_lens_cull_bound_agrees_with_numpy_roots(k1, k2, k3, built_lib):
    from s3gaussian_b200 import _lib
    got = built_lib.s3g_lens_max_radius2(C.byref(_lib.RasterLens(100, 100, 50, 50, k1, k2, 0.3, -0.2, k3)))
    # the host takes the coefficients as float32, as the struct holds them
    f = lambda v: float(np.float32(v))
    ref = lens_ref.max_radius2(f(k1), f(k2), f(k3))
    if math.isinf(ref):
        assert math.isinf(got) and got > 0, got
    else:
        assert abs(got - ref) <= 1e-9 * ref, (got, ref)
    assert math.isnan(built_lib.s3g_lens_max_radius2(None))


# ---- argument errors -------------------------------------------------------------------------------------------------
def _lens(**kw):
    from s3gaussian_b200 import _lib
    v = dict(zip(("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2", "k3"), LENS))
    v.update(kw)
    return _lib.RasterLens(**v)


def test_forward_argument_errors_before_any_launch(built_lib):
    from s3gaussian_b200 import _lib
    lib = built_lib
    call = lambda lens, fwd=None, opa=None: lib.s3g_rasterize_forward_lens(
        C.byref(_scene()), C.byref(fwd or _fwd()), C.byref(opa) if opa is not None else None, 0,
        C.byref(lens) if lens is not None else None, None)
    assert lib.s3g_rasterize_forward_lens(None, C.byref(_fwd()), None, 0, C.byref(_lens()), None) == -1
    assert call(None) == -1 and b"null lens" in lib.s3g_last_error()
    for kw in ({"fx": 0.0}, {"fy": -1.0}, {"fx": math.inf}, {"fy": math.nan}):
        assert call(_lens(**kw)) == -1 and b"fx and fy" in lib.s3g_last_error(), kw
    for k in ("cx", "cy", "k1", "k2", "p1", "p2", "k3"):
        for v in (math.nan, math.inf):
            assert call(_lens(**{k: v})) == -1 and b"finite" in lib.s3g_last_error(), k
    # the checks of the call it extends
    assert call(_lens(), opa=_lib.RasterOpacityArgs(dL_dpix_alpha=FAKE)) == -1
    assert b"backward inputs" in lib.s3g_last_error()
    # everything valid: the failing image allocator is the first thing that stops it
    assert call(_lens()) == -3 and b"allocator returned NULL" in lib.s3g_last_error()


def test_backward_follows_the_last_forward_on_the_geometry_buffer(built_lib):
    """After a lens forward a peer-sink backward and the camera pass are S3G_ERR_ARG before any launch; after a plain
    forward on the same buffer they get past that check.  lens -> plain -> lens."""
    from s3gaussian_b200 import _lib
    lib = built_lib
    geom = FAKE + (1 << 17)
    sink = _lib.PeerSink(world=2, rank=0, chunk=4, off_means3D=0, off_opacities=0, off_scales=0, off_rotations=0)
    sink.stage[0] = sink.stage[1] = FAKE

    def backward(name, *extra):
        b = _bwd(geom)
        b.sink = C.pointer(sink)
        b.dL_dpix_aux, b.dL_dcolor_aux = FAKE, FAKE
        return getattr(lib, name)(C.byref(_scene()), C.byref(b), *extra, None)

    def camera():
        b = _bwd(geom)
        b.dL_dconic, b.dL_ddepth = FAKE, FAKE
        out = _lib.RasterCameraGrads(FAKE, None, None)
        return lib.s3g_rasterize_camera_backward(C.byref(_scene()), C.byref(b), C.byref(out), None, None)

    opa = _lib.RasterOpacityArgs()
    lens = _lens()
    for with_lens in (True, False, True):
        if with_lens:
            rc = lib.s3g_rasterize_forward_lens(C.byref(_scene()), C.byref(_fwd(geom)), None, 0, C.byref(lens), None)
        else:
            rc = lib.s3g_rasterize_forward(C.byref(_scene()), C.byref(_fwd(geom)), None)
        assert rc == -3
        for name, extra in (("s3g_rasterize_backward", ()), ("s3g_rasterize_backward_opacity", (C.byref(opa),))):
            assert backward(name, *extra) == -1
            err = lib.s3g_last_error()
            assert (b"lens forward" in err) == with_lens and (b"aux gradients do not combine" in err) != with_lens, err
        assert camera() == -1
        assert (b"lens forward" in lib.s3g_last_error()) == with_lens, lib.s3g_last_error()


def test_header_declares_the_entry_point_in_c(built_lib, tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    from s3gaussian_b200 import _lib
    libdir = os.path.dirname(_lib.LIB_PATH)
    src = tmp_path / "lens.c"
    src.write_text('#include <math.h>\n#include <stddef.h>\n#include "s3g_b200.h"\n'
                   'int main(void) { s3g_raster_lens l = {100.f, 100.f, 50.f, 50.f, -0.2f, 0.f, 0.f, 0.f, 0.f};\n'
                   '  if (s3g_rasterize_forward_lens(NULL, NULL, NULL, 0, &l, NULL) != S3G_ERR_ARG) return 1;\n'
                   '  if (!(s3g_lens_max_radius2(&l) > 1.6 && s3g_lens_max_radius2(&l) < 1.7)) return 2;\n'
                   '  return 0; }\n')
    exe = tmp_path / "lens"
    r = subprocess.run([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                        "-o", str(exe), "-L", libdir, "-ls3g_b200", f"-Wl,-rpath,{libdir}", "-lm"], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = "/usr/local/cuda/lib64" + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    assert subprocess.run([str(exe)], env=env).returncode == 0


# ---- Python dispatch -------------------------------------------------------------------------------------------------
class _LensLib(_FakeLib):
    def s3g_rasterize_forward_lens(self, scene, fwd, opa, antialiased, lens, stream):
        l = lens._obj
        self.calls.append(("s3g_rasterize_forward_lens", opa is not None, antialiased,
                           tuple(getattr(l, k) for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2", "k3"))))
        return 5


@pytest.fixture
def fake(monkeypatch):
    from s3gaussian_b200 import _lib
    from s3gaussian_b200 import diff_gaussian_rasterization as dgr
    lib = _LensLib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(dgr, "_stream_ptr", lambda dev: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: torch.autograd.profiler.record_function("cpu"))
    P, E = 4, torch.Tensor([])
    byte = torch.zeros(64, dtype=torch.uint8)

    def forward_args(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs):
        arena = SimpleNamespace(tensor=byte)
        lease = SimpleNamespace(aset=SimpleNamespace(geom=arena, binning=arena, img=arena))
        return (_lib.RasterScene(), _lib.RasterForwardArgs(), lease,
                (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp),
                torch.zeros(3, 16, 16), torch.zeros(1, 16, 16), torch.zeros(P, dtype=torch.int32))
    monkeypatch.setattr(dgr, "_forward_args", forward_args)
    x = torch.zeros(P, 3)
    return lib, dgr, (x, x, E, x, torch.zeros(P, 1), x, torch.zeros(P, 4), E)


def test_forward_dispatch(fake):
    lib, dgr, inputs = fake
    rs = _settings(dgr)
    lens = dgr.Lens(10.0, 11.0, 8.5, 7.5, 0.1, 0.0, 0.0, 0.0, -0.2)
    expect_lens = tuple(float(np.float32(v)) for v in lens)
    for aa in (False, True):
        for opacity in (False, True):
            ctx = _Ctx()
            out = dgr._RasterizeGaussians.forward(ctx, *inputs, rs, None, None, None, None, opacity, aa, False, lens)
            assert lib.calls[-1] == ("s3g_rasterize_forward_lens", opacity, int(aa), expect_lens)
            assert ctx.lens and len(out) == (5 if opacity else 3)
            out = dgr.rasterize_gaussians_eval(*inputs, rs, with_opacity=opacity, antialiasing=aa, lens=lens)
            assert lib.calls[-1] == ("s3g_rasterize_forward_lens", opacity, int(aa), expect_lens)
            assert len(out) == (6 if opacity else 5)
    # without a lens: the calls of before
    dgr._RasterizeGaussians.forward(_Ctx(), *inputs, rs, None, None, None, None, False, False)
    assert lib.calls[-1] == ("s3g_rasterize_forward", False)


def test_apply_arguments(monkeypatch):
    """lens=None: apply gets exactly the arguments of before; with a lens every input, then the lens last."""
    from s3gaussian_b200 import diff_gaussian_rasterization as dgr
    seen = []
    monkeypatch.setattr(dgr._RasterizeGaussians, "apply", staticmethod(lambda *a: seen.append(a)))
    rs = _settings(dgr)
    x = torch.zeros(4, 3)
    kw = dict(means3D=x, means2D=x, opacities=x, colors_precomp=x, scales=x, rotations=x)
    plain = dgr.GaussianRasterizer(rs)
    plain(**kw)
    assert len(seen[-1]) == 9
    lens = (10.0, 11.0, 8.0, 7.0)
    r = dgr.GaussianRasterizer(rs, antialiasing=True, lens=lens)
    for call, colors_aux, opacity in ((lambda: r(**kw), None, False), (lambda: r.forward_aux(colors_aux=x, **kw), x,
                                                                        False),
                                      (lambda: r.forward_opacity(**kw), None, True)):
        call()
        a = seen[-1]
        assert len(a) == 17 and a[9] is colors_aux and a[10:13] == (None, None, None) and a[13] is opacity
        assert a[14] is True and a[15] is False and a[16] == dgr.Lens(10.0, 11.0, 8.0, 7.0)


def test_not_implemented_cases(fake):
    lib, dgr, inputs = fake
    # a camera tensor that requires grad
    rs = _settings(dgr, cam_grad=True)
    x = torch.zeros(4, 3)
    r = dgr.GaussianRasterizer(rs, lens=(10.0, 10.0, 8.0, 8.0))
    with pytest.raises(NotImplementedError, match="lens"):
        r(means3D=x, means2D=x, opacities=x, colors_precomp=x, scales=x, rotations=x)
    # a fused gradient exchange after a lens forward
    P, E = 4, torch.Tensor([])
    byte = torch.zeros(64, dtype=torch.uint8)
    saved = (torch.zeros(P, 3), torch.zeros(P, 3), torch.zeros(P, 3), torch.zeros(P, 4), E,
             torch.ones(P, dtype=torch.int32), E, byte, byte, byte)
    ctx = SimpleNamespace(raster_settings=_settings(dgr), saved_tensors=saved, num_rendered=5, has_aux=False,
                          camera=False, opacity=False, antialiasing=False, lens=True, needs_input_grad=(True,) * 17)

    class Sink:
        peer_sink_struct = object()
        notes = 0

        def __call__(self, name, shape, dev):
            return None

        def note_backward(self):
            Sink.notes += 1
    prev = dgr.set_grad_sink(Sink())
    try:
        lib.calls.clear()
        with pytest.raises(NotImplementedError, match="lens"):
            dgr._RasterizeGaussians.backward(ctx, torch.zeros(3, 16, 16), None, torch.zeros(1, 16, 16))
        assert lib.calls == [] and Sink.notes == 0
    finally:
        dgr.set_grad_sink(prev)
    # without the sink: the usual backward call, one gradient per apply() input
    grads = dgr._RasterizeGaussians.backward(ctx, torch.zeros(3, 16, 16), None, torch.zeros(1, 16, 16))
    assert lib.calls[-1] == ("s3g_rasterize_backward", False) and len(grads) == 17


def test_render_switch(monkeypatch):
    """pipe.lens off: render() constructs the rasterizer as before; on: with the camera's lens; a camera without
    intrinsic raises."""
    from s3gaussian_b200 import gaussian_renderer as gr
    made = []

    class FakeRasterizer:
        def __init__(self, raster_settings, **kw):
            made.append(kw)

        def __call__(self, means3D, **kw):
            z = torch.zeros(1, 4, 4)
            return torch.zeros(3, 4, 4), torch.ones(means3D.shape[0], dtype=torch.int32), z

    monkeypatch.setattr(gr, "GaussianRasterizer", FakeRasterizer)
    monkeypatch.setattr(gr, "raster_settings_for", lambda *a, **k: SimpleNamespace(campos=torch.zeros(3)))
    pc = SimpleNamespace(get_xyz=torch.zeros(5, 3), get_features=torch.zeros(5, 16, 3), _scaling=torch.zeros(5, 3),
                         _rotation=torch.ones(5, 4), _opacity=torch.zeros(5, 1), scaling_activation=torch.exp,
                         rotation_activation=torch.nn.functional.normalize, opacity_activation=torch.sigmoid)
    K = torch.tensor([[100.0, 0.0, 50.5], [0.0, 90.0, 40.25], [0.0, 0.0, 1.0]])
    cam = SimpleNamespace(intrinsic=K)
    pipe = gr.PipelineParams()
    assert pipe.lens is False
    gr.render(cam, pc, pipe, torch.zeros(3), stage="coarse")
    pipe.lens = True
    gr.render(cam, pc, pipe, torch.zeros(3), stage="coarse")
    cam.distortion = [0.1, -0.02, 0.001, 0.002, 0.003]
    pipe.antialiasing = True
    gr.render(cam, pc, pipe, torch.zeros(3), stage="coarse")
    from s3gaussian_b200.diff_gaussian_rasterization import Lens
    assert made == [{}, {"lens": Lens(100.0, 90.0, 50.5, 40.25)},
                    {"antialiasing": True, "lens": Lens(100.0, 90.0, 50.5, 40.25, 0.1, -0.02, 0.001, 0.002, 0.003)}]
    with pytest.raises(RuntimeError, match="intrinsic"):
        gr.render(SimpleNamespace(), pc, pipe, torch.zeros(3), stage="coarse")


def test_sky_camera_keeps_a_synthetic_camera_intrinsic():
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.sky import sky_camera
    base = syn.make_camera(64, 48, (0.0, 0.0, 1.0))
    K = torch.tensor([[70.0, 0.0, 30.0], [0.0, 65.0, 20.0], [0.0, 0.0, 1.0]])
    cam = syn.SyntheticCamera(64, 48, base.FoVx, base.FoVy, base.world_view_transform, base.full_proj_transform,
                              base.camera_center, 0.0, K, torch.zeros(5))
    c2w, Kc = sky_camera(cam)
    assert torch.equal(Kc, K) and torch.equal(c2w, sky_camera(base)[0])
    assert cam.to("cpu").intrinsic is K
