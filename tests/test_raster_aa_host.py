"""CPU: the rasterizer's antialiasing without a GPU - argument errors of s3g_rasterize_forward_antialiased and of a
backward after it (before any launch), the Python dispatch with a fake library object, the code of the preprocess
and camera-pass kernels that existed before the filter, and the filter's float64 restatement and its closed-form
derivatives."""
import ctypes as C
import json
import os
import shutil
import subprocess
from types import SimpleNamespace

import pytest
import torch

import aa_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "preprocess_sass.json")
FAKE = 1 << 20    # never dereferenced: every call below fails validation or allocation first


def _scene():
    from s3gaussian_b200 import _lib
    return _lib.RasterScene(P=4, background=FAKE, width=16, height=16, means3D=FAKE, colors_precomp=FAKE,
                            opacities=FAKE, scales=FAKE, scale_modifier=1.0, rotations=FAKE, viewmatrix=FAKE,
                            projmatrix=FAKE, tan_fovx=1.0, tan_fovy=1.0)


def _fwd(geom=0):
    """Forward arguments whose geometry allocator returns `geom` and whose image allocator fails: the forward takes
    the geometry buffer, then stops with S3G_ERR_ALLOC before any launch."""
    from s3gaussian_b200 import _lib
    g = _lib.ALLOC_FN(lambda user, n: geom)
    never = _lib.ALLOC_FN(lambda user, n: 0)
    f = _lib.RasterForwardArgs(geom_alloc=g, binning_alloc=never, image_alloc=never, out_color=FAKE, out_depth=FAKE)
    f.keep = (g, never)
    return f


def _bwd(geom):
    from s3gaussian_b200 import _lib
    return _lib.RasterBackwardArgs(R=5, geom_buffer=geom, binning_buffer=FAKE, image_buffer=FAKE + 4096,
                                   dL_dpix=FAKE, dL_dpix_depth=FAKE, dL_dmean2D=FAKE, dL_dopacity=FAKE,
                                   dL_dcolor=FAKE, dL_dmean3D=FAKE, dL_dcov3D=FAKE, dL_dscale=FAKE, dL_drot=FAKE)


def test_forward_argument_errors_before_any_launch(built_lib):
    from s3gaussian_b200 import _lib
    lib = built_lib
    call = lambda fwd, opa: lib.s3g_rasterize_forward_antialiased(C.byref(_scene()), C.byref(fwd),
                                                                  C.byref(opa) if opa is not None else None, None)
    assert lib.s3g_rasterize_forward_antialiased(None, C.byref(_fwd()), None, None) == -1
    assert lib.s3g_rasterize_forward_antialiased(C.byref(_scene()), None, None, None) == -1
    assert b"forward_antialiased: null scene" in lib.s3g_last_error()
    # the opacity forward's checks, with and without opacity arguments
    for field, msg in (("dL_dpix_alpha", b"backward inputs"), ("out_alpha_d", b"go together")):
        assert call(_fwd(), _lib.RasterOpacityArgs(**{field: FAKE})) == -1, field
        assert msg in lib.s3g_last_error(), (field, lib.s3g_last_error())
    f = _fwd()
    f.out_color = None
    assert call(f, None) == -1 and b"null output" in lib.s3g_last_error()
    s = _scene()
    s.width = 0
    assert lib.s3g_rasterize_forward_antialiased(C.byref(s), C.byref(_fwd()), None, None) == -1
    assert b"bad sizes" in lib.s3g_last_error()
    # everything valid: the failing allocator is the first thing that stops it
    assert call(_fwd(), None) == -3 and b"allocator returned NULL" in lib.s3g_last_error()


def test_backward_follows_the_last_forward_on_the_geometry_buffer(built_lib):
    """A peer-sink backward after an antialiased forward is S3G_ERR_ARG before any launch; after a plain forward on the
    same geometry buffer it gets past that check (and stops at the next one, the aux pair with a sink)."""
    from s3gaussian_b200 import _lib
    lib = built_lib
    geom = FAKE + (1 << 16)
    sink = _lib.PeerSink(world=2, rank=0, chunk=4, off_means3D=0, off_opacities=0, off_scales=0, off_rotations=0)
    sink.stage[0] = sink.stage[1] = FAKE

    def backward(name, *extra):
        b = _bwd(geom)
        b.sink = C.pointer(sink)
        b.dL_dpix_aux, b.dL_dcolor_aux = FAKE, FAKE
        return getattr(lib, name)(C.byref(_scene()), C.byref(b), *extra, None)

    opa = _lib.RasterOpacityArgs()
    for forward in ("s3g_rasterize_forward_antialiased", "s3g_rasterize_forward", "s3g_rasterize_forward_antialiased",
                    "s3g_rasterize_forward_opacity"):
        args = (C.byref(opa),) if forward != "s3g_rasterize_forward" else ()
        assert getattr(lib, forward)(C.byref(_scene()), C.byref(_fwd(geom)), *args, None) == -3
        aa = forward.endswith("antialiased")
        for name, extra in (("s3g_rasterize_backward", ()), ("s3g_rasterize_backward_opacity", (C.byref(opa),))):
            assert backward(name, *extra) == -1, (forward, name)
            err = lib.s3g_last_error()
            assert (b"antialiased" in err) == aa and (b"aux gradients do not combine" in err) != aa, (forward, err)


def test_header_declares_the_entry_point_in_c(built_lib, tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    from s3gaussian_b200 import _lib
    libdir = os.path.dirname(_lib.LIB_PATH)
    src = tmp_path / "aa.c"
    src.write_text('#include <stddef.h>\n#include "s3g_b200.h"\n'
                   'int main(void) { return s3g_rasterize_forward_antialiased(NULL, NULL, NULL, NULL) == S3G_ERR_ARG '
                   '? 0 : 1; }\n')
    exe = tmp_path / "aa"
    r = subprocess.run([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                        "-o", str(exe), "-L", libdir, "-ls3g_b200", f"-Wl,-rpath,{libdir}"], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = "/usr/local/cuda/lib64" + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    assert subprocess.run([str(exe)], env=env).returncode == 0


# ---- Python dispatch -------------------------------------------------------------------------------------------------
def _settings(dgr, cam_grad=False):
    t = lambda *s: torch.zeros(s, requires_grad=cam_grad)
    return dgr.GaussianRasterizationSettings(
        image_height=16, image_width=16, tanfovx=1.0, tanfovy=1.0, bg=torch.zeros(3), scale_modifier=1.0,
        viewmatrix=t(4, 4), projmatrix=t(4, 4), sh_degree=0, campos=t(3), prefiltered=False, debug=False)


@pytest.mark.parametrize("cam_grad", [False, True])
def test_apply_arguments(monkeypatch, cam_grad):
    """antialiasing=False: forward / forward_aux / forward_opacity call apply exactly as before; True: every optional
    input, then antialiasing=True last."""
    from s3gaussian_b200 import diff_gaussian_rasterization as dgr
    seen = []
    monkeypatch.setattr(dgr._RasterizeGaussians, "apply", staticmethod(lambda *a: seen.append(a)))
    rs = _settings(dgr, cam_grad)
    x = torch.zeros(4, 3)
    kw = dict(means3D=x, means2D=x, opacities=x, colors_precomp=x, scales=x, rotations=x)
    cam = (rs.viewmatrix, rs.projmatrix, rs.campos) if cam_grad else (None, None, None)
    for aa in (False, True):
        r = dgr.GaussianRasterizer(rs, antialiasing=aa) if aa else dgr.GaussianRasterizer(rs)
        r(**kw)
        r.forward_aux(colors_aux=x, **kw)
        r.forward_opacity(**kw)
        r.forward_opacity(colors_aux=x, **kw)
        plain, aux, opa, opa_aux = seen[-4:]
        if not aa:
            assert len(plain) == (13 if cam_grad else 9) and len(aux) == (13 if cam_grad else 10)
            assert len(opa) == len(opa_aux) == 14 and opa[13] is True
            continue
        for a, colors_aux, opacity in ((plain, None, False), (aux, x, False), (opa, None, True), (opa_aux, x, True)):
            assert len(a) == 15 and a[8] is rs and a[9] is colors_aux and a[13] is opacity and a[14] is True
            assert all(u is v for u, v in zip(a[10:13], cam))


class _FakeLib:
    def __init__(self):
        self.calls = []

    def _rec(self, name, opa=None):
        self.calls.append((name, opa is not None))
        return 5

    def s3g_rasterize_forward(self, scene, fwd, stream):
        return self._rec("s3g_rasterize_forward")

    def s3g_rasterize_forward_opacity(self, scene, fwd, opa, stream):
        return self._rec("s3g_rasterize_forward_opacity", opa)

    def s3g_rasterize_forward_antialiased(self, scene, fwd, opa, stream):
        return self._rec("s3g_rasterize_forward_antialiased", opa)

    def s3g_rasterize_backward(self, scene, bwd, stream):
        return self._rec("s3g_rasterize_backward")

    def s3g_rasterize_backward_opacity(self, scene, bwd, opa, stream):
        return self._rec("s3g_rasterize_backward_opacity", opa)

    def s3g_rasterize_backward_deterministic_workspace_bytes(self, P, R, W, H):
        return 64

    def s3g_rasterize_backward_deterministic(self, scene, bwd, ws, stream):
        return self._rec("s3g_rasterize_backward_deterministic")

    def s3g_rasterize_backward_deterministic_opacity(self, scene, bwd, opa, ws, stream):
        return self._rec("s3g_rasterize_backward_deterministic_opacity", opa)


class _Ctx:
    def save_for_backward(self, *a):
        self.saved_tensors = a

    def mark_non_differentiable(self, *a):
        pass


@pytest.fixture
def fake(monkeypatch):
    """A fake library, and _forward_args without the CUDA checks: the forwards run on CPU tensors."""
    from s3gaussian_b200 import _lib
    from s3gaussian_b200 import diff_gaussian_rasterization as dgr
    lib = _FakeLib()
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
    for aa, opacity, expect in ((False, False, ("s3g_rasterize_forward", False)),
                                (False, True, ("s3g_rasterize_forward_opacity", True)),
                                (True, False, ("s3g_rasterize_forward_antialiased", False)),
                                (True, True, ("s3g_rasterize_forward_antialiased", True))):
        ctx = _Ctx()
        out = dgr._RasterizeGaussians.forward(ctx, *inputs, rs, None, None, None, None, opacity, aa)
        assert lib.calls[-1] == expect and ctx.antialiasing is aa and len(out) == (5 if opacity else 3)
        for with_opacity in (False, True):
            out = dgr.rasterize_gaussians_eval(*inputs, rs, with_opacity=with_opacity, antialiasing=aa)
            name = ("s3g_rasterize_forward_antialiased" if aa else
                    "s3g_rasterize_forward_opacity" if with_opacity else "s3g_rasterize_forward")
            assert lib.calls[-1] == (name, with_opacity) and len(out) == (6 if with_opacity else 5)


def _backward(dgr, opacity, grads_in, aa, aux=False):
    P, E = 4, torch.Tensor([])
    byte = torch.zeros(64, dtype=torch.uint8)
    saved = (torch.zeros(P, 3), torch.zeros(P, 3), torch.zeros(P, 3), torch.zeros(P, 4), E,
             torch.ones(P, dtype=torch.int32), E, byte, byte, byte)
    ctx = SimpleNamespace(raster_settings=_settings(dgr), saved_tensors=saved, num_rendered=5, has_aux=aux,
                          camera=False, opacity=opacity, antialiasing=aa, needs_input_grad=(True,) * 15)
    return dgr._RasterizeGaussians.backward(ctx, torch.zeros(3, 16, 16), None, torch.zeros(1, 16, 16), *grads_in)


def test_backward_dispatch(fake):
    """An antialiased forward is followed by the usual backward calls (the library applies the filter's chain rule
    itself) and its backward returns one gradient per apply() input."""
    lib, dgr, _ = fake
    z = torch.zeros(1, 16, 16)
    for aa in (False, True):
        lib.calls.clear()
        grads = _backward(dgr, False, (), aa)
        assert lib.calls == [("s3g_rasterize_backward", False)] and len(grads) == (15 if aa else 9)
        grads = _backward(dgr, True, (z, z), aa)
        assert lib.calls[-1] == ("s3g_rasterize_backward_opacity", True) and len(grads) == (15 if aa else 14)
        grads = _backward(dgr, False, (torch.zeros(3, 16, 16),), aa, aux=True)
        assert lib.calls[-1] == ("s3g_rasterize_backward", False) and len(grads) == (15 if aa else 10)
        assert grads[9] is not None
        prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
        torch.use_deterministic_algorithms(True)
        try:
            _backward(dgr, False, (), aa)
            assert lib.calls[-1] == ("s3g_rasterize_backward_deterministic", False)
            _backward(dgr, True, (None, z), aa)
            assert lib.calls[-1] == ("s3g_rasterize_backward_deterministic_opacity", True)
        finally:
            torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])


def test_peer_sink_after_an_antialiased_forward_is_not_implemented(fake):
    lib, dgr, _ = fake

    class Sink:
        peer_sink_struct = object()
        notes = 0

        def __call__(self, name, shape, dev):
            return None

        def note_backward(self):
            Sink.notes += 1
    prev = dgr.set_grad_sink(Sink())
    try:
        with pytest.raises(NotImplementedError, match="antialiased"):
            _backward(dgr, False, (), True)
        assert lib.calls == [] and Sink.notes == 0
    finally:
        dgr.set_grad_sink(prev)


def test_render_switch(monkeypatch):
    """pipe.antialiasing off or absent: render() constructs the rasterizer exactly as before; on: with
    antialiasing=True."""
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
    pipe = gr.PipelineParams()
    assert pipe.antialiasing is False
    gr.render(None, pc, pipe, torch.zeros(3), stage="coarse")
    legacy = SimpleNamespace(compute_cov3D_python=False, convert_SHs_python=False, debug=False)
    gr.render(None, pc, legacy, torch.zeros(3), stage="coarse")
    pipe.antialiasing = True
    gr.render(None, pc, pipe, torch.zeros(3), stage="coarse")
    assert made == [{}, {}, {"antialiasing": True}]


# ---- the kernels that existed before the filter ----------------------------------------------------------------------
def test_existing_preprocess_kernels_keep_their_code(built_lib):
    """The preprocess forward and backward (both data-parallel forms) and camera-pass kernels of the parent build,
    recorded in tests/golden/preprocess_sass.json (CUDA 12.9, sm_90a): the same SASS, instruction for instruction.
    They gained a defaulted `false` template argument, which changes their mangled names only."""
    from s3gaussian_b200 import _lib
    from test_flow_host import _sass_by_kernel, sass_digests
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    with open(GOLDEN) as f:
        golden = json.load(f)
    ver = subprocess.run(["cuobjdump", "--version"], capture_output=True, text=True).stdout
    if f"V{golden['cuda']}" not in ver:
        pytest.skip(f"recorded with CUDA {golden['cuda']}; SASS of another toolkit differs")
    sass = _sass_by_kernel(_lib.LIB_PATH)
    assert len(golden["kernels"]) == 10
    for name, rec in golden["kernels"].items():
        assert name in sass, f"{name} missing from the library"
        exact, multiset = sass_digests(sass[name])
        assert len(sass[name]) == rec["instructions"], name
        assert multiset == rec["multiset"] and exact == rec["exact"], f"{name}: SASS differs from the parent build"


# ---- the filter's restatement ----------------------------------------------------------------------------------------
def _abc(n, seed):
    """EWA covariances from sub-pixel to large, PSD with a margin: a, c in [5e-5, 30] px^2, |b| < sqrt(a c)."""
    g = torch.Generator().manual_seed(seed)
    a = torch.exp(torch.empty(n, dtype=torch.float64).uniform_(-10, 3.4, generator=g))
    c = torch.exp(torch.empty(n, dtype=torch.float64).uniform_(-10, 3.4, generator=g))
    b = torch.empty(n, dtype=torch.float64).uniform_(-0.95, 0.95, generator=g) * torch.sqrt(a * c)
    op = torch.empty(n, dtype=torch.float64).uniform_(0.05, 0.99, generator=g)
    return a, b, c, op


def test_filter_restatement_passes_gradcheck():
    a, b, c, op = (t.requires_grad_(True) for t in _abc(64, 1))
    rho = (a * c - b * b) / ((a + 0.3) * (c + 0.3) - b * b)
    assert bool((rho > aa_ref.RHO_MIN).any()) and bool((rho < aa_ref.RHO_MIN).any())   # both branches of the floor
    # away from the floor's kink: gradcheck's finite differences must not straddle it
    keep = ((rho - aa_ref.RHO_MIN).abs() > 1e-6).detach()
    args = tuple(t.detach()[keep].requires_grad_(True) for t in (a, b, c, op))
    f = lambda a, b, c, op: aa_ref.filter64(a, b, c, op)[:2]
    assert torch.autograd.gradcheck(f, args)


def test_filter_derivatives_match_the_closed_form():
    """dL/dopacity = h g and, above the floor, dL/d{a,b,c} gains opacity g / (2 h) drho/d{a,b,c}; below it, nothing."""
    a, b, c, op = (t.requires_grad_(True) for t in _abc(4096, 2))
    g = torch.randn(4096, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    _, alpha_eff, h = aa_ref.filter64(a, b, c, op)
    da, db, dc, dop = torch.autograd.grad((alpha_eff * g).sum(), (a, b, c, op))
    h = h.detach()
    torch.testing.assert_close(dop, h * g, rtol=1e-12, atol=0)
    ra, rb, rc = aa_ref.drho_closed_form(a.detach(), b.detach(), c.detach())
    rho = h * h
    above = (a * c - b * b).detach() / ((a + 0.3) * (c + 0.3) - b * b).detach() > aa_ref.RHO_MIN
    assert 100 < int(above.sum()) < 4000
    k = torch.where(above, op.detach() * g / (2 * h), torch.zeros_like(h))
    for got, closed in ((da, ra), (db, rb), (dc, rc)):
        torch.testing.assert_close(got, k * closed, rtol=1e-9, atol=1e-12)
    assert bool((rho[above] > aa_ref.RHO_MIN * (1 - 1e-12)).all())
