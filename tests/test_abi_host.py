"""CPU: the C-ABI library loads and exports every symbol include/s3g_b200.h
declares, the host-side mirror of the reference API validates arguments like the
reference, and the synthetic cameras follow the reference's conventions.  No
compute is launched here."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    h = open(os.path.join(ROOT, "include", "s3g_b200.h")).read()
    h = re.sub(r"/\*.*?\*/", "", h, flags=re.S)
    out = {}
    for m in re.finditer(r"\b(s3g_\w+)\s*\(([^;{]*?)\)\s*;", h, flags=re.S):
        params = [p.strip() for p in m.group(2).split(",") if p.strip() and p.strip() != "void"]
        out[m.group(1)] = len(params)
    return out


def test_library_exports_every_declared_symbol_at_abi_2(built_lib):
    from s3gaussian_b200 import _lib
    decl = header_functions()
    assert len(decl) >= 12
    raw = C.CDLL(_lib.LIB_PATH)
    for name, nparams in decl.items():
        assert hasattr(raw, name), f"{name} declared in the header but not exported"
        assert name in _lib.SIGNATURES, f"{name} has no ctypes binding"
        assert len(_lib.SIGNATURES[name][1]) == nparams, f"{name}: ctypes arity != header arity"
    assert built_lib.s3g_abi_version() == 2
    assert built_lib.s3g_build_arch() == b"sm_90a"


def test_library_is_sm90a_only(built_lib):
    import shutil
    import subprocess
    from s3gaussian_b200 import _lib
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    out = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\w+", out))
    assert archs == {"sm_90a"}, archs


def test_arena_sizes_and_field_lookup(built_lib):
    from s3gaussian_b200 import _lib
    lib = built_lib
    assert lib.s3g_geom_bytes(0) > 0
    g1, g2 = lib.s3g_geom_bytes(1000), lib.s3g_geom_bytes(2000)
    assert g2 > g1 > 1000 * 100
    assert lib.s3g_binning_bytes(10**6) >= 20 * 10**6      # point_list + two ping-pong (tile, id) pairs
    assert lib.s3g_image_bytes(1920, 1280) >= 1920 * 1280 * 8
    off, eb, cnt = _lib.state_field(2, "ranges", 10, 0, 1920, 1280)
    assert (eb, cnt) == (8, 120 * 80) and off % 128 == 0
    off, eb, cnt = _lib.state_field(1, "point_list", 10, 777, 64, 64)
    assert (off, eb, cnt) == (0, 4, 777)
    with pytest.raises(RuntimeError):
        _lib.state_field(0, "no_such_field", 10, 0, 64, 64)


def test_argument_errors_of_the_struct_abi_do_not_need_a_gpu(built_lib):
    from s3gaussian_b200 import _lib
    lib = built_lib
    assert lib.s3g_mark_visible(-1, None, None, None, None, None) == -1
    assert b"P < 0" in lib.s3g_last_error()
    assert lib.s3g_mark_visible(0, None, None, None, None, None) == 0          # P == 0 short-circuit
    assert lib.s3g_sort_pairs_u32(5, None, None, None, None, 8, 8, None, None) == -1
    cb = _lib.ALLOC_FN(lambda user, n: 0)
    scene = _lib.RasterScene(P=-5, width=16, height=16, scale_modifier=1.0, tan_fovx=1.0, tan_fovy=1.0)
    fwd = _lib.RasterForwardArgs(geom_alloc=cb, binning_alloc=cb, image_alloc=cb)
    rc = lib.s3g_rasterize_forward(C.byref(scene), C.byref(fwd), None)
    assert rc == -1
    scene.P = 3
    rc = lib.s3g_rasterize_backward(C.byref(scene), C.byref(_lib.RasterBackwardArgs()), None)
    assert rc in (-1, -4)
    assert lib.s3g_rasterize_forward(None, C.byref(fwd), None) == -1
    assert lib.s3g_rasterize_backward(C.byref(scene), None, None) == -1


def test_rasterizer_extras_that_do_not_combine_are_rejected(built_lib):
    """Each optional extra of the rasterizer is a field; the combinations no pass supports fail with S3G_ERR_ARG
    before anything is launched."""
    from s3gaussian_b200 import _lib
    lib = built_lib
    cb = _lib.ALLOC_FN(lambda user, n: 0)
    fake = 1 << 20    # never dereferenced: every call below fails validation first
    scene = _lib.RasterScene(P=4, background=fake, width=16, height=16, means3D=fake, colors_precomp=fake,
                             opacities=fake, scales=fake, scale_modifier=1.0, rotations=fake, viewmatrix=fake,
                             projmatrix=fake, tan_fovx=1.0, tan_fovy=1.0)
    fwd = _lib.RasterForwardArgs(geom_alloc=cb, binning_alloc=cb, image_alloc=cb, out_color=fake, out_depth=fake,
                                 colors_aux=fake, out_color_aux=fake)
    # aux colours with the static/dynamic decomposition
    fwd.group, fwd.out_color_d, fwd.out_depth_d, fwd.out_color_s, fwd.out_depth_s = (fake,) * 5
    assert lib.s3g_rasterize_forward(C.byref(scene), C.byref(fwd), None) == -1
    assert b"split and aux forwards do not combine" in lib.s3g_last_error()
    # aux colours with a flow colour set, which the composite would write through the aux slot
    fwd.group, fwd.out_color_d, fwd.out_depth_d, fwd.out_color_s, fwd.out_depth_s = (None,) * 5
    fwd.n_flow, fwd.flow_colors[0], fwd.out_flow[0] = 1, fake, fake
    assert lib.s3g_rasterize_forward(C.byref(scene), C.byref(fwd), None) == -1
    assert b"colors_aux and flow colours do not combine" in lib.s3g_last_error()
    # the peer sink with the aux gradients
    sink = _lib.PeerSink(world=2, rank=0, chunk=4)
    sink.stage[0] = sink.stage[1] = fake
    bwd = _lib.RasterBackwardArgs(geom_buffer=fake, image_buffer=fake, dL_dpix=fake, dL_dpix_depth=fake,
                                  dL_dmean2D=fake, dL_dcolor=fake, dL_dpix_aux=fake, dL_dcolor_aux=fake,
                                  sink=C.pointer(sink))
    assert lib.s3g_rasterize_backward(C.byref(scene), C.byref(bwd), None) == -1
    assert b"peer sink and the aux gradients do not combine" in lib.s3g_last_error()


def test_backward_rejects_an_unaligned_rotation_gradient(built_lib):
    """dL_drot is stored 16 bytes per row: an output off a 16-byte boundary is S3G_ERR_ARG before any launch, in the
    plain, deterministic and absgrad backwards (the Python glue hands such a sink view an aligned tensor instead)."""
    from s3gaussian_b200 import _lib
    lib = built_lib
    fake = 1 << 20    # never dereferenced: every call below fails validation first
    scene = _lib.RasterScene(P=4, background=fake, width=16, height=16, means3D=fake, colors_precomp=fake,
                             opacities=fake, scales=fake, scale_modifier=1.0, rotations=fake, viewmatrix=fake,
                             projmatrix=fake, tan_fovx=1.0, tan_fovy=1.0)
    for off in (4, 8, 12):
        bwd = _lib.RasterBackwardArgs(R=5, geom_buffer=fake, binning_buffer=fake, image_buffer=fake, dL_dpix=fake,
                                      dL_dpix_depth=fake, dL_dmean2D=fake, dL_dopacity=fake, dL_dcolor=fake,
                                      dL_dmean3D=fake, dL_dcov3D=fake, dL_dscale=fake, dL_drot=fake + off)
        for call in (lambda: lib.s3g_rasterize_backward(C.byref(scene), C.byref(bwd), None),
                     lambda: lib.s3g_rasterize_backward_deterministic(C.byref(scene), C.byref(bwd), fake, None),
                     lambda: lib.s3g_rasterize_backward_absgrad(C.byref(scene), C.byref(bwd), None, fake, 0, None,
                                                                None)):
            assert call() == -1, off
            assert b"dL_drot must be 16-byte aligned" in lib.s3g_last_error(), (off, lib.s3g_last_error())


def test_rasterizer_python_api_mirrors_reference_validation():
    from s3gaussian_b200 import diff_gaussian_rasterization as dgr
    assert dgr.GaussianRasterizationSettings._fields == (
        "image_height", "image_width", "tanfovx", "tanfovy", "bg", "scale_modifier", "viewmatrix",
        "projmatrix", "sh_degree", "campos", "prefiltered", "debug")
    rs = dgr.GaussianRasterizationSettings(8, 8, 1.0, 1.0, torch.zeros(3), 1.0, torch.eye(4), torch.eye(4), 0,
                                           torch.zeros(3), False, False)
    r = dgr.GaussianRasterizer(rs)
    x = torch.zeros(4, 3)
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(x, x, torch.zeros(4, 1), scales=x, rotations=torch.zeros(4, 4))
    with pytest.raises(Exception, match="excatly one of either SHs or precomputed colors"):
        r(x, x, torch.zeros(4, 1), shs=torch.zeros(4, 1, 3), colors_precomp=x, scales=x, rotations=torch.zeros(4, 4))
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(x, x, torch.zeros(4, 1), colors_precomp=x)
    with pytest.raises(Exception, match="scale/rotation pair or precomputed 3D covariance"):
        r(x, x, torch.zeros(4, 1), colors_precomp=x, scales=x, rotations=torch.zeros(4, 4),
          cov3D_precomp=torch.zeros(4, 6))
    # CPU tensors are refused loudly: there is no CPU path
    with pytest.raises(RuntimeError, match="no CPU path"):
        r(x, x, torch.zeros(4, 1), colors_precomp=x, scales=x, rotations=torch.zeros(4, 4))
    with pytest.raises(RuntimeError, match="no CPU path"):
        r.markVisible(x)
    with pytest.raises(RuntimeError, match="num_points, 3"):
        r(torch.zeros(4, 2), x, torch.zeros(4, 1), colors_precomp=x, scales=x, rotations=torch.zeros(4, 4))


def test_install_as_reference_module():
    import sys
    import s3gaussian_b200
    s3gaussian_b200.install_as_reference_module()
    import diff_gaussian_rasterization as m
    assert m is s3gaussian_b200.diff_gaussian_rasterization
    assert hasattr(m, "GaussianRasterizer") and hasattr(m, "GaussianRasterizationSettings")
    del sys.modules["diff_gaussian_rasterization"]


def test_product_never_imports_the_oracle():
    """tier rule: nothing under s3gaussian_b200/ may import, link or call oracle/."""
    pkg = os.path.join(ROOT, "s3gaussian_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(dp, f), errors="ignore").read()
                for pat in (r"^\s*(from|import)\s+oracle", r"oracle[/\\._]", r"liboracle|splat_oracle"):
                    assert not re.search(pat, src, flags=re.M), f"{f} references the oracle ({pat})"


def test_synthetic_camera_conventions():
    from s3gaussian_b200 import synthetic as syn
    cam = syn.make_camera(1920, 1280, (3.0, -1.0, 2.0), yaw_deg=30.0)
    assert abs(math.degrees(cam.FoVx) - 50.1) < 0.1
    V = cam.world_view_transform.T.numpy()          # W2C
    # camera centre maps to the origin, forward axis is +z of the camera
    c = np.array([3.0, -1.0, 2.0, 1.0])
    assert np.allclose(V @ c, [0, 0, 0, 1], atol=1e-5)
    fwd = np.array([math.cos(math.radians(30)), math.sin(math.radians(30)), 0.0])
    p = V @ np.append(c[:3] + 5 * fwd, 1.0)
    assert np.allclose(p[:3], [0, 0, 5], atol=1e-4)
    assert np.allclose(cam.camera_center.numpy(), c[:3], atol=1e-5)
    # full_proj: w component equals view depth
    q = np.append(c[:3] + 5 * fwd + np.array([0.3, 0.2, 0.1]), 1.0)
    hom = cam.full_proj_transform.T.numpy() @ q
    assert abs(hom[3] - (V @ q)[2]) < 1e-4
    ring = syn.waymo_ring(frames=50)
    assert len(ring) == 150 and ring[0].time == 0.0 and abs(ring[-1].time - 1.0) < 1e-9
    cloud = syn.make_cloud(1000, seed=0)
    again = syn.make_cloud(1000, seed=0)
    assert torch.equal(cloud.xyz, again.xyz) and cloud.get_features().shape == (1000, 16, 3)
