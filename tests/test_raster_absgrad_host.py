"""CPU: the absolute screen-space gradient without a GPU - argument errors of s3g_rasterize_backward_absgrad and
s3g_densify_stats_abs (before any launch), the header, the Python dispatch with a fake library object, render()'s
switch, add_densification_stats' checks, dp.sync_view_stats over gloo, GaussianModel's accumulator through _rebuild
and densify, the code of the backward composite kernels that existed before the feature, and the float64 oracle's
self-checks."""
import ctypes as C
import json
import os
import shutil
import socket
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import absgrad_ref
from test_raster_aa_host import FAKE, _FakeLib, _bwd, _scene, _settings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "composite_bwd_sass.json")


# ---- C ABI ----------------------------------------------------------------------------------------------------------
def test_backward_absgrad_argument_errors_before_any_launch(built_lib):
    from s3gaussian_b200 import _lib
    lib = built_lib
    geom = FAKE + (1 << 18)
    call = lambda b, out=FAKE, det=0, ws=None, scene=None, opa=None: lib.s3g_rasterize_backward_absgrad(
        C.byref(scene or _scene()), C.byref(b), C.byref(opa) if opa is not None else None, out, det, ws, None)
    assert lib.s3g_rasterize_backward_absgrad(None, C.byref(_bwd(geom)), None, FAKE, 0, None, None) == -1
    assert b"backward_absgrad: null scene" in lib.s3g_last_error()
    assert call(_bwd(geom), out=None) == -1 and b"null dL_dmean2D_abs" in lib.s3g_last_error()
    # P == 0: nothing to do, NULL output allowed
    s = _scene()
    s.P = 0
    assert call(_bwd(geom), out=None, scene=s) == 0
    # the checks of the calls it extends
    b = _bwd(geom)
    b.dL_dpix = None
    assert call(b) == -1 and b"null input" in lib.s3g_last_error()
    b = _bwd(geom)
    b.dL_dpix_aux = FAKE
    assert call(b) == -1 and b"go together" in lib.s3g_last_error()
    assert call(_bwd(geom), opa=_lib.RasterOpacityArgs(out_alpha=FAKE)) == -1
    assert b"forward outputs" in lib.s3g_last_error()
    assert call(_bwd(geom), det=1, ws=None) == -1 and b"workspace" in lib.s3g_last_error()
    assert call(_bwd(geom), det=1, ws=FAKE + 4) == -1 and b"aligned" in lib.s3g_last_error()
    # a peer sink: not with the deterministic walk
    sink = _lib.PeerSink(world=2, rank=0, chunk=4, off_means3D=0, off_opacities=0, off_scales=0, off_rotations=0)
    sink.stage[0] = sink.stage[1] = FAKE
    b = _bwd(geom)
    b.sink = C.pointer(sink)
    assert call(b, det=1, ws=FAKE) == -1 and b"not deterministic" in lib.s3g_last_error()


def test_densify_stats_abs_argument_errors(built_lib):
    lib = built_lib
    assert lib.s3g_densify_stats_abs(-1, None, None, None, None, None, None, None, None) == -1
    assert lib.s3g_densify_stats_abs(0, None, None, None, None, None, None, None, None) == 0
    assert lib.s3g_densify_stats_abs(4, FAKE, None, FAKE, FAKE, FAKE, FAKE, FAKE, None) == -1
    assert b"densify_stats_abs: null pointer" in lib.s3g_last_error()


def test_header_declares_the_entry_points_in_c(built_lib, tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    from s3gaussian_b200 import _lib
    for name in ("s3g_rasterize_backward_absgrad", "s3g_densify_stats_abs"):
        assert name in _lib.SIGNATURES
    libdir = os.path.dirname(_lib.LIB_PATH)
    src = tmp_path / "absgrad.c"
    src.write_text('#include <stddef.h>\n#include "s3g_b200.h"\n'
                   'int main(void) {\n'
                   '  if (s3g_rasterize_backward_absgrad(NULL, NULL, NULL, NULL, 0, NULL, NULL) != S3G_ERR_ARG) return 1;\n'
                   '  return s3g_densify_stats_abs(-1, NULL, NULL, NULL, NULL, NULL, NULL, NULL, NULL) == S3G_ERR_ARG '
                   '? 0 : 2;\n}\n')
    exe = tmp_path / "absgrad"
    r = subprocess.run([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                        "-o", str(exe), "-L", libdir, "-ls3g_b200", f"-Wl,-rpath,{libdir}"], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = "/usr/local/cuda/lib64" + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    assert subprocess.run([str(exe)], env=env).returncode == 0


def test_existing_backward_composite_kernels_keep_their_code(built_lib):
    """The eight render_backward_kernel<AUX, DET, OPA> instantiations, grad_rec_gather_kernel and densify_stats_kernel
    of the parent build, recorded in tests/golden/composite_bwd_sass.json (CUDA 12.9, sm_90a): the same SASS,
    instruction for instruction.  The composite kernels gained a defaulted `false` ABS template argument, which
    changes their mangled names only."""
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


# ---- Python dispatch ------------------------------------------------------------------------------------------------
class _AbsFakeLib(_FakeLib):
    def s3g_rasterize_backward_absgrad(self, scene, bwd, opa, out, det, ws, stream):
        self.calls.append(("s3g_rasterize_backward_absgrad", opa is not None))
        self.abs_args = (out, det, ws)
        self.abs_bwd = bwd._obj
        C.memmove(out, (C.c_float * 8)(*[float(i + 1) for i in range(8)]), 32)   # P = 4 rows of 2
        return 0


@pytest.fixture
def fake(monkeypatch):
    """A fake library, and _forward_args without the CUDA checks: the forwards run on CPU tensors."""
    from s3gaussian_b200 import _lib
    from s3gaussian_b200 import diff_gaussian_rasterization as dgr
    lib = _AbsFakeLib()
    monkeypatch.setattr(_lib, "load", lambda: lib)
    monkeypatch.setattr(dgr, "_stream_ptr", lambda dev: None)
    monkeypatch.setattr(torch.cuda, "device", lambda dev: torch.autograd.profiler.record_function("cpu"))
    P = 4
    byte = torch.zeros(64, dtype=torch.uint8)

    def forward_args(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs):
        arena = SimpleNamespace(tensor=byte)
        lease = SimpleNamespace(aset=SimpleNamespace(geom=arena, binning=arena, img=arena))
        return (_lib.RasterScene(), _lib.RasterForwardArgs(), lease,
                (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp),
                torch.zeros(3, 16, 16), torch.zeros(1, 16, 16), torch.ones(P, dtype=torch.int32))
    monkeypatch.setattr(dgr, "_forward_args", forward_args)
    return lib, dgr


def _leaves(P=4):
    return dict(means3D=torch.zeros(P, 3, requires_grad=True), opacities=torch.zeros(P, 1, requires_grad=True),
                colors_precomp=torch.zeros(P, 3, requires_grad=True), scales=torch.zeros(P, 3, requires_grad=True),
                rotations=torch.zeros(P, 4, requires_grad=True))


@pytest.mark.parametrize("cam_grad", [False, True])
def test_apply_arguments(monkeypatch, cam_grad):
    """absgrad=True: every optional input, then opacity, antialiasing and absgrad=True last; absgrad=False: the calls
    of the parent commit."""
    from s3gaussian_b200 import diff_gaussian_rasterization as dgr
    seen = []
    monkeypatch.setattr(dgr._RasterizeGaussians, "apply", staticmethod(lambda *a: seen.append(a)))
    rs = _settings(dgr, cam_grad)
    x = torch.zeros(4, 3)
    kw = dict(means3D=x, means2D=x, opacities=x, colors_precomp=x, scales=x, rotations=x)
    cam = (rs.viewmatrix, rs.projmatrix, rs.campos) if cam_grad else (None, None, None)
    for aa in (False, True):
        calls = []
        for absgrad in (False, True):
            r = dgr.GaussianRasterizer(rs, antialiasing=aa, absgrad=absgrad)
            r(**kw)
            r.forward_aux(colors_aux=x, **kw)
            r.forward_opacity(**kw)
            r.forward_opacity(colors_aux=x, **kw)
            calls.append(seen[-4:])
        off, on = calls
        legacy = []
        r = dgr.GaussianRasterizer(rs, antialiasing=aa) if aa else dgr.GaussianRasterizer(rs)
        r(**kw)
        r.forward_aux(colors_aux=x, **kw)
        r.forward_opacity(**kw)
        r.forward_opacity(colors_aux=x, **kw)
        legacy = seen[-4:]
        same = lambda u, v: u is v or (isinstance(u, torch.Tensor) and u.numel() == 0 and v.numel() == 0)
        for a, b in zip(off, legacy):     # absent inputs are fresh empty tensors on every call
            assert len(a) == len(b) and all(same(u, v) for u, v in zip(a, b))
        for a, colors_aux, opacity in zip(on, (None, x, None, x), (False, False, True, True)):
            assert len(a) == 16 and a[8] is rs and a[9] is colors_aux and a[13] is opacity
            assert a[14] is aa and a[15] is True and a[1] is x
            assert all(u is v for u, v in zip(a[10:13], cam))


def _run(dgr, absgrad, opacity=False, aa=False, m2d=None):
    rs = _settings(dgr)
    t = _leaves()
    m2d = torch.zeros(4, 3, requires_grad=True) if m2d is None else m2d
    r = dgr.GaussianRasterizer(rs, antialiasing=aa, absgrad=absgrad)
    out = (r.forward_opacity if opacity else r)(means2D=m2d, **t)
    loss = out[0].sum() + out[2].sum() + (out[3].sum() if opacity else 0)
    loss.backward()
    return m2d


def test_backward_dispatch_sets_and_accumulates_absgrad(fake):
    lib, dgr = fake
    for opacity in (False, True):
        for aa in (False, True):
            lib.calls.clear()
            m2d = _run(dgr, True, opacity, aa)
            assert lib.calls[-1] == ("s3g_rasterize_backward_absgrad", opacity)
            out, det, ws = lib.abs_args
            assert out == m2d.absgrad.data_ptr() and det == 0 and ws is None
            want = torch.arange(1.0, 9.0).view(4, 2)
            assert m2d.absgrad.dtype == torch.float32 and torch.equal(m2d.absgrad, want)
            assert m2d.grad is not None
            _run(dgr, True, opacity, aa, m2d=m2d)                       # a second backward adds
            assert torch.equal(m2d.absgrad, 2 * want)
            m2d.absgrad = None
            _run(dgr, True, opacity, aa, m2d=m2d)
            assert torch.equal(m2d.absgrad, want)


def test_backward_dispatch_deterministic(fake):
    lib, dgr = fake
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    torch.use_deterministic_algorithms(True)
    try:
        _run(dgr, True)
        out, det, ws = lib.abs_args
        assert lib.calls[-1] == ("s3g_rasterize_backward_absgrad", False) and det == 1 and ws is not None
    finally:
        torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])


def test_switch_off_makes_the_parent_calls(fake):
    """absgrad off: the same library calls with byte-identical backward arguments as a rasterizer built without the
    argument, and no attribute on means2D."""
    lib, dgr = fake
    from s3gaussian_b200 import _lib
    captured = []
    orig = lib.s3g_rasterize_backward

    def rec(scene, bwd, stream):
        # the argument struct with every pointer reduced to NULL / set (the tensors differ from call to call)
        o = bwd._obj
        captured.append(tuple((n, getattr(o, n) if n == "R" else bool(getattr(o, n))) for n, _ in o._fields_))
        return orig(scene, bwd, stream)
    lib.s3g_rasterize_backward = rec
    m_off = _run(dgr, False)
    rs = _settings(dgr)
    m_legacy = torch.zeros(4, 3, requires_grad=True)
    out = dgr.GaussianRasterizer(rs)(means2D=m_legacy, **_leaves())
    (out[0].sum() + out[2].sum()).backward()
    assert [c[0] for c in lib.calls] == ["s3g_rasterize_forward", "s3g_rasterize_backward"] * 2
    assert len(captured) == 2 and captured[0] == captured[1]
    assert not hasattr(m_off, "absgrad") and not hasattr(m_legacy, "absgrad")


def test_render_switch(monkeypatch):
    """pipe.absgrad off or absent: render() constructs the rasterizer exactly as before; on: with absgrad=True."""
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
    assert pipe.absgrad is False
    gr.render(None, pc, pipe, torch.zeros(3), stage="coarse")
    legacy = SimpleNamespace(compute_cov3D_python=False, convert_SHs_python=False, debug=False)
    gr.render(None, pc, legacy, torch.zeros(3), stage="coarse")
    pipe.absgrad = True
    gr.render(None, pc, pipe, torch.zeros(3), stage="coarse")
    pipe.antialiasing = True
    gr.render(None, pc, pipe, torch.zeros(3), stage="coarse")
    assert made == [{}, {}, {"absgrad": True}, {"antialiasing": True, "absgrad": True}]


def test_add_densification_stats_checks():
    from s3gaussian_b200.optim import add_densification_stats
    P = 4
    t = lambda *s: torch.zeros(*s)
    radii = torch.ones(P, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="go together"):
        add_densification_stats(t(P, 3), radii, t(P, 1), t(P, 1), t(P), viewspace_absgrad=t(P, 2))
    with pytest.raises(RuntimeError, match="go together"):
        add_densification_stats(t(P, 3), radii, t(P, 1), t(P, 1), t(P), xyz_gradient_accum_abs=t(P, 1))
    with pytest.raises(RuntimeError, match="CUDA"):
        add_densification_stats(t(P, 3), radii, t(P, 1), t(P, 1), t(P), t(P, 2), t(P, 1))


# ---- data parallel ---------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, results):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    from s3gaussian_b200 import dp
    dp.init_from_env("gloo")
    vgrad = torch.tensor([[3.0, -4.0, 0.0], [1.0, 0.0, 0.0]]) * (rank + 1)
    absgrad = torch.tensor([[3.0, 4.0], [2.0, 1.0]]) * (rank + 1)
    radii = torch.tensor([2 + rank, 0], dtype=torch.int32)
    out = dp.sync_view_stats(vgrad, radii, absgrad)
    results[rank] = (len(out), out[2] is absgrad, absgrad.clone(), vgrad.clone(), radii.clone(),
                     len(dp.sync_view_stats(vgrad.clone(), radii.clone())))
    dist.barrier()
    dist.destroy_process_group()


def test_sync_view_stats_sums_absgrad_over_gloo():
    import torch.multiprocessing as mp
    from s3gaussian_b200 import dp
    world, port = 2, _free_port()
    results = mp.Manager().dict()
    mp.spawn(_worker, args=(world, port, results), nprocs=world, join=True)
    for r in range(world):
        n, same, absgrad, vgrad, radii, n_plain = results[r]
        assert n == 3 and same and n_plain == 2
        assert torch.equal(absgrad, torch.tensor([[9.0, 12.0], [6.0, 3.0]]))
        assert torch.equal(vgrad, torch.tensor([[9.0, -12.0, 0.0], [3.0, 0.0, 0.0]]))
        assert torch.equal(radii, torch.tensor([3, 0], dtype=torch.int32))
    a = torch.ones(2, 2)
    assert dp.sync_view_stats(torch.ones(2, 3), torch.ones(2), a)[2] is a      # single process: untouched


# ---- GaussianModel --------------------------------------------------------------------------------------------------
def _fake_gather(monkeypatch):
    """s3g_gather_rows on CPU tensors (rows >= n_kept zeroed where asked), and a CPU stream."""
    from s3gaussian_b200 import _lib
    from s3gaussian_b200 import gaussian_model as gm

    def gather(n, descs, n_out, n_kept, src_index, stream):
        idx = np.ctypeslib.as_array((C.c_int64 * n_out).from_address(src_index)).copy()
        rows = int(idx.max()) + 1 if n_out else 0
        for k in range(n):
            dsc = descs[k]
            rf = dsc.row_floats
            src = np.ctypeslib.as_array((C.c_float * (rows * rf)).from_address(dsc.src)).reshape(rows, rf)
            dst = np.ctypeslib.as_array((C.c_float * (n_out * rf)).from_address(dsc.dst)).reshape(n_out, rf)
            dst[:] = src[idx]
            if dsc.zero_new:
                dst[n_kept:] = 0
        return 0
    monkeypatch.setattr(_lib, "load", lambda: SimpleNamespace(s3g_gather_rows=gather))
    monkeypatch.setattr(gm.torch.cuda, "current_stream", lambda *a: SimpleNamespace(cuda_stream=0))
    return gm


def _cpu_model(gm, P=5):
    g = gm.GaussianModel(0)
    g._xyz = torch.nn.Parameter(torch.arange(P * 3.0).view(P, 3))
    g._features_dc, g._features_rest = torch.nn.Parameter(torch.zeros(P, 1, 3)), torch.nn.Parameter(torch.zeros(P, 0, 3))
    g._scaling, g._rotation = torch.nn.Parameter(torch.zeros(P, 3)), torch.nn.Parameter(torch.ones(P, 4))
    g._opacity = torch.nn.Parameter(torch.zeros(P, 1))
    g.xyz_gradient_accum = torch.arange(P, dtype=torch.float32).view(P, 1)
    g.xyz_gradient_accum_abs = torch.arange(P, dtype=torch.float32).view(P, 1) * 10 + 1
    g.denom = torch.ones(P, 1)
    g._deformation_accum = torch.zeros(P, 3)
    g.max_radii2D = torch.zeros(P)
    g._deformation_table = torch.ones(P, dtype=torch.bool)
    return g


def test_rebuild_carries_and_resets_the_abs_accumulator(monkeypatch):
    gm = _fake_gather(monkeypatch)
    g = _cpu_model(gm)
    old = g.xyz_gradient_accum_abs.clone()
    g.prune_points(torch.tensor([False, True, False, False, True]))
    assert torch.equal(g.xyz_gradient_accum_abs, old[[0, 2, 3]])
    g._rebuild(torch.tensor([2, 0, 1]), 3, keep_accumulators=True)        # spatial_sort's reorder
    assert torch.equal(g.xyz_gradient_accum_abs, old[[3, 0, 2]])
    g._rebuild(torch.tensor([0, 1, 2, 1]), 3, keep_accumulators=False)    # densify: reset
    assert torch.equal(g.xyz_gradient_accum_abs, torch.zeros(4, 1))
    # an accumulator that does not match the rows (a model from before the feature) restarts from zero
    g = _cpu_model(gm)
    g.xyz_gradient_accum_abs = torch.empty(0)
    g.prune_points(torch.tensor([False, True, False, False, False]))
    assert torch.equal(g.xyz_gradient_accum_abs, torch.zeros(4, 1))


def test_densify_selects_on_the_abs_statistic(monkeypatch):
    gm = _fake_gather(monkeypatch)
    for max_grad_abs, want in ((None, [3, 4]), (35.0, [4])):
        g = _cpu_model(gm)
        g.percent_dense = 1.0
        g.densify(2.5, 0.005, 10.0, None, max_grad_abs=max_grad_abs)       # every Gaussian is small: clone
        xyz = torch.arange(15.0).view(5, 3)
        assert torch.equal(g.get_xyz.detach(), torch.cat([xyz, xyz[want]]))
        assert torch.equal(g.xyz_gradient_accum_abs, torch.zeros(5 + len(want), 1))


def test_capture_keeps_the_reference_tuple():
    from s3gaussian_b200.gaussian_model import GaussianModel
    import inspect
    src = inspect.getsource(GaussianModel.capture)
    assert "xyz_gradient_accum_abs" not in src
    assert "xyz_gradient_accum_abs" in inspect.getsource(GaussianModel.training_setup)


# ---- the float64 oracle ---------------------------------------------------------------------------------------------
def _oracle_scene(seed, P=12, W=40, H=33):
    g = torch.Generator().manual_seed(seed)
    f64 = dict(dtype=torch.float64)
    mx = (torch.rand(P, generator=g, **f64) * W).requires_grad_(True)
    my = (torch.rand(P, generator=g, **f64) * H).requires_grad_(True)
    s = torch.rand(P, generator=g, **f64) * 3 + 1
    b = (torch.rand(P, generator=g, **f64) - 0.5) * 0.4 / s
    conic = torch.stack([1 / s, b, 1 / (s * 1.3)], 1)
    op = torch.rand(P, generator=g, **f64) * 0.8 + 0.1
    col, aux = torch.rand(P, 3, generator=g, **f64), torch.rand(P, 3, generator=g, **f64)
    tz = torch.rand(P, generator=g, **f64) + 1
    order = torch.argsort(tz).numpy()
    nt = ((W + 15) // 16) * ((H + 15) // 16)
    ranges = np.array([[i * P, (i + 1) * P] for i in range(nt)])
    pix, idx = absgrad_ref.pixel_lists(W, H, ranges, np.tile(order, nt))
    dL = {k: torch.randn(3 if k in ("color", "aux") else 1, H, W, generator=g, **f64)
          for k in ("color", "depth", "alpha", "median", "aux")}
    bg = torch.tensor([0.1, 0.2, 0.3], **f64)
    return W, H, mx, my, conic, op, col, tz, bg, pix, idx, dL, aux


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_signed_sum_is_autograds_mean2d_gradient(seed):
    W, H, mx, my, conic, op, col, tz, bg, pix, idx, dL, aux = _oracle_scene(seed)
    signed, absg = absgrad_ref.mean2d_grads64(W, H, mx, my, conic, op, col, tz, bg, pix, idx, dL, aux)
    loss = absgrad_ref.pixel_loss(absgrad_ref.composite64(W, H, mx, my, conic, op, col, tz, bg, pix, idx, aux), pix,
                                  dL)
    gx, gy = torch.autograd.grad(loss, (mx, my))
    torch.testing.assert_close(signed, torch.stack([gx * W / 2, gy * H / 2], 1), rtol=1e-10, atol=1e-10)
    assert float(signed.abs().max()) > 1
    # the triangle inequality, strictly for Gaussians with pixels pulling both ways
    assert bool((signed.abs() <= absg + 1e-12).all()) and float((absg - signed.abs()).max()) > 1


def test_oracle_triangle_inequality_across_calls():
    """Two calls (colour, then aux) add two sums of absolute values: never less than one call's sum over both."""
    W, H, mx, my, conic, op, col, tz, bg, pix, idx, dL, aux = _oracle_scene(5)
    one = absgrad_ref.mean2d_grads64(W, H, mx, my, conic, op, col, tz, bg, pix, idx,
                                     {"color": dL["color"], "aux": dL["aux"]}, aux)[1]
    a = absgrad_ref.mean2d_grads64(W, H, mx, my, conic, op, col, tz, bg, pix, idx, {"color": dL["color"]})[1]
    b = absgrad_ref.mean2d_grads64(W, H, mx, my, conic, op, aux, tz, bg, pix, idx, {"color": dL["aux"]})[1]
    assert bool((one <= a + b + 1e-9).all()) and float((a + b - one).max()) > 0
