"""GPU: the rasterizer at settings the rest of the suite does not reach: cameras with fx != fy, scale_modifier != 1
and SH tensors of every coefficient count M the kernels accept.

launch_sh_rows (csrc/api.cu) runs the <16> instantiations of the preprocess forward, the preprocess backward and the
camera-gradient kernel for M == 16 and the runtime-M <0> ones for any other M.  Their rows are staged through
warp_rows_in, which reads float4 when the row length 3M is a multiple of 4 and the pointer is 16-byte aligned and one
float at a time otherwise.  Above 48 KB of staged rows the launch raises the kernel's dynamic shared-memory limit
(M >= 32), and above 200 KB it refuses the call (M >= 134).

A. Exact identities, bitwise with the deterministic backward, through six entry points (forward, forward_aux, the
   antialiased forward with camera gradients, forward_opacity, absgrad, forward with camera gradients):
   - M in {1, 4, 9} (every degree D <= sqrt(M) - 1), and M in {32, 133} with D = 3, against the same coefficients
     padded to a wider M.  The padding holds random values, not zeros: no kernel may read a coefficient beyond the
     degree.  Images, radii and every non-SH gradient are equal; dL/dsh equals on the shared coefficients and is
     exactly zero on the padding.
   - M = 134 is refused with S3G_ERR_ARG by the forward, the backward and the camera backward, and the next call
     works.
   - SH rows at a 4-byte storage offset give the aligned tensor's results.
   - (scales, mod) and (fl32(scales * mod), 1) agree for mod in {0.5, 0.8, 1.3}.  cov3d_from_scale_rot and the
     preprocess backward both round the product mod * scale once, so the two calls see the same float32 scales, and
     dL_dscales is taken with respect to mod * scale (the reference's convention), so it is the same tensor too.
B. Anisotropic cameras (fy / fx in {1.448, 0.69, 1.0007}) against the checkers the suite already trusts: the CPU
   oracle at the bars of test_gpu_raster.test_cuda_matches_cpu_oracle, the float64 restatements of the AA, camera,
   opacity / median and absgrad tests at their own bars, the reference extension at the bars of the benchmark-size
   test, and filter3d_ref for the 3-D filter's screen bound.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import ref_ext
import util

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4


@pytest.fixture(scope="module")
def ours(built_lib):
    from s3gaussian_b200 import diff_gaussian_rasterization as mod
    return mod


class _deterministic:
    def __init__(self, on=True):
        self.on = on

    def __enter__(self):
        self.prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
        torch.use_deterministic_algorithms(self.on)

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.prev[0], warn_only=self.prev[1])


def _scene(ratio=1.448, P=385, W=70, H=45, seed=6, mode="sh", deg=3, M=16, cov=False, mod=None):
    """make_small_scene's cloud seen by the camera at its pose with fx = 0.9 W and fy = ratio * fx.  The 8 first
    Gaussians are large ones beyond the 1.3 tanfov clamp, and the last one sits in the middle of the view: with
    P % 32 == 1 the last warp stages a single row, whose length 3M is odd for M in {1, 9}."""
    from s3gaussian_b200 import synthetic as syn
    from test_gpu_raster_camera import _with_edge_gaussians
    cloud, _ = syn.make_small_scene(P=P, width=W, height=H, seed=seed)
    cloud = _with_edge_gaussians(cloud)
    cloud.xyz[-1] = torch.tensor([4.0, 0.1, -0.1])
    cloud.opacity[-1] = 2.0
    cam = util.anisotropic_camera(W, H, 0.9 * W, ratio * 0.9 * W, (0.0, 0.0, 0.0))
    d = util.scene_inputs(cloud, cam, mode=mode, sh_degree=deg, cov_precomp=cov)
    if d["shs"] is not None:
        d["shs"] = d["shs"][:, :M].contiguous()
    if mod is not None:
        d["scale_modifier"] = float(mod)
    return d


def _padded(shs, M, seed=3):
    """shs [P,m,3] widened to [P,M,3] with random coefficients after the first m."""
    g = torch.Generator().manual_seed(seed)
    tail = torch.randn(shs.shape[0], M - shs.shape[1], 3, generator=g)
    return torch.cat([shs, tail], 1).contiguous()


# ---- A. exact identities --------------------------------------------------------------------------------------------
ENTRIES = ["forward", "aux", "aa_camera", "opacity", "absgrad", "camera"]


def _run(ours, d, entry, shs=None, det=True):
    """One forward and backward of `entry` with seeded image gradients -> dict of every output and gradient.
    shs: a device tensor used as the SH leaf as given (its storage offset included)."""
    P, H, W = d["means3D"].shape[0], d["H"], d["W"]
    t = {k: d[k].to(DEV).clone().requires_grad_(True) for k in util.TENSOR_KEYS if d[k] is not None}
    if shs is not None:
        t["shs"] = shs.requires_grad_(True)
    m2d = torch.zeros_like(t["means3D"], requires_grad=True)
    rs = util.settings_for(ours, d, DEV)
    cam = {}
    if entry in ("camera", "aa_camera"):
        cam = {k: getattr(rs, k).clone().requires_grad_(True) for k in ("viewmatrix", "projmatrix", "campos")}
        rs = rs._replace(**cam)
    rast = ours.GaussianRasterizer(rs, antialiasing=entry == "aa_camera", absgrad=entry == "absgrad")
    gen = torch.Generator().manual_seed(5)
    gc, gd, ga, gm, gx = (torch.randn(ch, H, W, generator=gen).to(DEV) for ch in (3, 1, 1, 1, 3))
    aux = None
    if entry == "aux":
        aux = torch.rand(P, 3, generator=gen).to(DEV).requires_grad_(True)
        out = rast.forward_aux(means2D=m2d, colors_aux=aux, **t)
        images = (out[0], out[2], out[3])
        weights = (gc, gd, gx)
    elif entry == "opacity":
        out = rast.forward_opacity(means2D=m2d, **t)
        images = (out[0], out[2], out[3], out[4])
        weights = (gc, gd, ga, gm)
    else:
        out = rast(means2D=m2d, **t)
        images = (out[0], out[2])
        weights = (gc, gd)
    loss = sum((img * w).sum() for img, w in zip(images, weights))
    with _deterministic(det):
        loss.backward()
    res = {f"image{i}": img.detach() for i, img in enumerate(images)}
    res["radii"] = out[1]
    res.update({"d_" + k: v.grad for k, v in t.items()})
    res["d_means2D"] = m2d.grad
    res.update({"d_" + k: v.grad for k, v in cam.items()})
    if aux is not None:
        res["d_aux"] = aux.grad
    if entry == "absgrad":
        res["absgrad"] = m2d.absgrad
    return res


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _assert_identical(got, want, skip=()):
    assert set(got) == set(want)
    for k in want:
        if k in skip:
            continue
        assert got[k] is not None and want[k] is not None, k
        assert torch.equal(_bits(got[k]), _bits(want[k])), (k, float((got[k].double() - want[k].double()).abs().max()))


def _assert_padding_identity(narrow, wide, m):
    """narrow: run with m coefficients; wide: the same coefficients padded with random ones."""
    _assert_identical(wide, narrow, skip=("d_shs",))
    assert torch.equal(_bits(wide["d_shs"][:, :m]), _bits(narrow["d_shs"])), \
        float((wide["d_shs"][:, :m] - narrow["d_shs"]).abs().max())
    assert float(wide["d_shs"][:, m:].abs().max()) == 0
    assert int((narrow["radii"] > 0).sum()) > 50 and float(narrow["d_shs"].abs().max()) > 0
    assert int(narrow["radii"][-1]) > 0      # the single row of the last warp is rendered


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("M,deg", [(1, 0), (4, 0), (4, 1), (9, 0), (9, 1), (9, 2)])
def test_fewer_sh_coefficients_equal_the_padded_tensor(M, deg, entry, ours):
    d = _scene(deg=deg, M=M)
    narrow = _run(ours, d, entry)
    wide = _run(ours, d, entry, shs=_padded(d["shs"], 16).to(DEV))
    _assert_padding_identity(narrow, wide, M)


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("M", [32, 133])
def test_more_sh_coefficients_equal_the_16_coefficient_tensor(M, entry, ours):
    """M = 32: the first M whose staged rows (128 x 97 floats) exceed 48 KB.  M = 133: 128 x 399 floats = 204 288
    bytes, the largest under the 200 KB refusal."""
    d = _scene(deg=3, M=16)
    narrow = _run(ours, d, entry)
    wide = _run(ours, d, entry, shs=_padded(d["shs"], M).to(DEV))
    _assert_padding_identity(narrow, wide, 16)


class _Ctx:
    def save_for_backward(self, *a):
        self.saved = a

    def mark_non_differentiable(self, *a):
        pass


def test_134_sh_coefficients_are_refused(ours):
    """3 x 134 floats per row, 128 rows: 206 336 bytes of shared memory > 200 KB.  The forward, the backward and the
    camera backward return S3G_ERR_ARG, and a call after them renders as before."""
    from s3gaussian_b200 import _lib
    lib = _lib.load()
    d = _scene(deg=3, M=16)
    before = _run(ours, d, "forward")
    sh134 = _padded(d["shs"], 134).to(DEV)
    rs = util.settings_for(ours, d, DEV)
    t = {k: d[k].to(DEV) for k in util.TENSOR_KEYS if d[k] is not None}
    with pytest.raises(RuntimeError, match="S3G_ERR_ARG"):
        ours.GaussianRasterizer(rs)(means2D=torch.zeros_like(t["means3D"]), **dict(t, shs=sh134))
    # a forward at M = 16, then the backward and the camera backward with a scene at M = 134
    E = torch.Tensor([])
    inputs = [t.get(k, E) for k in ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations",
                                    "cov3D_precomp")]
    ctx = _Ctx()
    ours._RasterizeGaussians.forward(ctx, inputs[0], torch.zeros_like(inputs[0]), *inputs[1:], rs)
    P, H, W = d["means3D"].shape[0], d["H"], d["W"]
    scene = ours._scene(rs, torch.device(DEV), inputs[0], sh134, inputs[2], None, inputs[4], inputs[5], inputs[6])
    e = lambda *s: torch.zeros(s, dtype=torch.float32, device=DEV)
    o = dict(mean2D=e(P, 3), conic=e(P, 4), opacity=e(P, 1), color=e(P, 3), depth=e(P), mean3D=e(P, 3), cov3D=e(P, 6),
             sh=e(P, 134, 3), scale=e(P, 3), rot=e(P, 4), view=e(16), proj=e(16), campos=e(3))
    gc, gd = e(3, H, W), e(1, H, W)
    s = ctx.saved
    bwd = _lib.RasterBackwardArgs(
        R=ctx.num_rendered, radii=s[5].data_ptr(), geom_buffer=s[7].data_ptr(), binning_buffer=s[8].data_ptr(),
        image_buffer=s[9].data_ptr(), dL_dpix=gc.data_ptr(), dL_dpix_depth=gd.data_ptr(),
        dL_dmean2D=o["mean2D"].data_ptr(), dL_dconic=o["conic"].data_ptr(), dL_dopacity=o["opacity"].data_ptr(),
        dL_dcolor=o["color"].data_ptr(), dL_ddepth=o["depth"].data_ptr(), dL_dmean3D=o["mean3D"].data_ptr(),
        dL_dcov3D=o["cov3D"].data_ptr(), dL_dsh=o["sh"].data_ptr(), dL_dscale=o["scale"].data_ptr(),
        dL_drot=o["rot"].data_ptr())
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.s3g_rasterize_backward(C.byref(scene), C.byref(bwd), stream) == -1
    assert "too many SH coefficients" in _lib.last_error()
    cws = torch.empty(max(int(lib.s3g_rasterize_camera_backward_workspace_bytes(P)), 16), dtype=torch.uint8,
                      device=DEV)
    grads = _lib.RasterCameraGrads(o["view"].data_ptr(), o["proj"].data_ptr(), o["campos"].data_ptr())
    assert lib.s3g_rasterize_camera_backward(C.byref(scene), C.byref(bwd), C.byref(grads), cws.data_ptr(),
                                             stream) == -1
    assert "too many SH coefficients" in _lib.last_error()
    torch.cuda.synchronize()
    _assert_identical(_run(ours, d, "forward"), before)


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("M,deg", [(16, 3), (9, 2)])
def test_unaligned_sh_rows_equal_the_aligned_tensor(M, deg, entry, ours):
    """An SH tensor 4 bytes into its storage takes warp_rows_in's scalar path even where 3M % 4 == 0."""
    d = _scene(deg=deg, M=M)
    aligned = _run(ours, d, entry)
    buf = torch.empty(d["shs"].numel() + 1, dtype=torch.float32, device=DEV)
    shs = buf[1:].view(d["shs"].shape)
    shs.copy_(d["shs"])
    assert shs.data_ptr() % 16 == 4 and shs.is_contiguous()
    _assert_identical(_run(ours, d, entry, shs=shs), aligned)


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("mod", [0.5, 0.8, 1.3])
def test_scale_modifier_equals_prescaled_scales(mod, entry, ours):
    d = _scene(deg=2, M=9, mod=mod)
    pre = dict(d, scales=d["scales"] * torch.tensor(mod, dtype=torch.float32), scale_modifier=1.0)
    got, want = _run(ours, d, entry), _run(ours, pre, entry)
    _assert_identical(got, want)
    # the modifier matters here: the unmodified call renders differently
    plain = _run(ours, dict(d, scale_modifier=1.0), "forward")
    assert not torch.equal(plain["image0"], got["image0"])


# ---- B. anisotropic cameras against the existing checkers -----------------------------------------------------------
# fy / fx, colours ("sh", "rgb", "cov": rgb with precomputed covariances), D, M, scale_modifier, P, W, H, seed
ORACLE_CASES = [
    (1.448, "sh", 3, 16, 1.0, 400, 80, 64, 11),
    (1.448, "sh", 2, 9, 0.8, 385, 70, 45, 12),         # ragged
    # seed 13 here puts one Gaussian's alpha at one pixel within 6e-7 (relative) of the 1/255 cut-off, where glibc's
    # expf and the device's differ in the decision; seed 23 keeps every decision 1.8e-5 or more from it
    (1.448, "rgb", 0, 0, 1.3, 300, 64, 48, 23),
    (1.448, "cov", 0, 0, 0.8, 200, 64, 48, 14),         # the modifier does not apply to precomputed covariances
    (1.448, "sh", 1, 4, 0.8, 100, 16, 16, 15),          # one tile
    (0.69, "sh", 1, 4, 1.3, 300, 48, 80, 16),           # portrait
    (0.69, "sh", 0, 1, 1.0, 257, 33, 17, 17),           # ragged, one coefficient
    (0.69, "sh", 3, 16, 0.8, 500, 96, 64, 18),
    (0.69, "cov", 0, 0, 1.0, 200, 40, 72, 19),          # portrait
    (1.0007, "sh", 2, 9, 1.0, 400, 64, 48, 20),
    (1.0007, "sh", 3, 16, 1.3, 300, 47, 31, 21),        # ragged
    (1.0007, "rgb", 0, 0, 0.8, 600, 128, 96, 22),
]


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("ratio,mode,deg,M,mod,P,W,H,seed", ORACLE_CASES)
def test_anisotropic_camera_matches_cpu_oracle(ratio, mode, deg, M, mod, P, W, H, seed, det, ours, oracle_lib):
    from test_gpu_raster import check_state_vs
    d = _scene(ratio, P, W, H, seed, "sh" if mode == "sh" else "rgb", deg, M, mode == "cov", mod)
    gc, gd = util.seeded_grads(d, seed)
    o = util.oracle_run(oracle_lib, d, gc, gd)
    color, radii, depth, R, views = util.ours_forward_state(d, DEV)
    check_state_vs(views, radii, R, dict(num_rendered=o["R"], radii=o["radii"],
                                         tiles_touched=o["geometry"]["tiles_touched"],
                                         point_list=o["binning"]["point_list"], keys=o["binning"]["keys"],
                                         ranges=o["binning"]["ranges"], n_contrib=o["image"]["n_contrib"]))
    assert int((radii > 0).sum()) > 10
    assert util.relerr(color.cpu().numpy(), o["color"]) < TOL
    assert util.relerr(depth.cpu().numpy(), o["depth"]) < TOL
    with _deterministic(det):
        out = util.run_module(ours, d, DEV, gc, gd)
    names = {"means3D": "means3D", "means2D": "means2D", "opacities": "opacity", "scales": "scales",
             "rotations": "rotations", "shs": "sh", "colors_precomp": "colors", "cov3D_precomp": "cov3D"}
    assert len(out["grads"]) >= 5
    for k, g in out["grads"].items():
        ref = o["grads"][names[k]].reshape(g.shape)
        if np.abs(ref).max() == 0:
            assert float(g.abs().max()) == 0, k
        else:
            assert util.relerr(g.cpu().numpy(), ref) < TOL, (k, util.relerr(g.cpu().numpy(), ref))


CAMERAS = [(1.448, 64, 48), (0.69, 48, 72)]     # fy / fx, W, H


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("ratio,W,H", CAMERAS)
def test_anisotropic_antialiased_gradients_match_float64_vjp(ratio, W, H, det, ours):
    """test_gpu_raster_aa's check: per-Gaussian and camera gradients against the float64 VJP, SH at D = 2, M = 9."""
    from test_gpu_raster_aa import _check, _explicit_backward, _vjp64
    d = _scene(ratio, 600, W, H, 23, deg=2, M=9)
    g = torch.Generator().manual_seed(24)
    scaled = dict(d, scales=d["scales"] * torch.exp(torch.empty(600, 1).uniform_(-4.0, 1.0, generator=g)))
    gc, gd = util.seeded_grads(scaled, 25)
    o = _explicit_backward(ours, scaled, gc, gd, det)
    ref, vis = _vjp64(scaled, o)
    for k in ("mean3D", "opacity", "scale", "rot", "sh"):
        got = o[k][vis] if k != "sh" else o["sh"][vis][:, :ref["sh"].shape[1]]
        _check(got, ref[k], k)
    for k in ("view", "proj", "campos"):
        _check(o[k], ref[k].reshape(-1), k)


@pytest.mark.parametrize("ratio,W,H", CAMERAS)
@pytest.mark.parametrize("cov", [False, True])
def test_anisotropic_camera_gradients_match_float64_oracle(ratio, W, H, cov, ours):
    """test_gpu_raster_camera's check, SH at D = 2, M = 9."""
    from test_gpu_raster_camera import _check_against_oracle
    _check_against_oracle(ours, _scene(ratio, 600, W, H, 26, deg=2, M=9, cov=cov), seed=27)


def _rgb_grad_scene(ratio, P, W, H, seed, cov):
    """test_gpu_raster_opacity._grad_case at an anisotropic camera."""
    from s3gaussian_b200 import synthetic as syn
    cloud, _ = syn.make_small_scene(P=P, width=W, height=H, seed=seed)
    cloud.scaling += math.log(2.5)
    cam = util.anisotropic_camera(W, H, 0.9 * W, ratio * 0.9 * W, (0.0, 0.0, 0.0))
    return util.scene_inputs(cloud, cam, mode="rgb", cov_precomp=cov)


GRAD_CASES = [(1.448, 48, 48, 40, 3, False), (0.69, 64, 40, 33, 5, True)]


@pytest.mark.parametrize("loss_kind", ["alpha", "median", "all"])
@pytest.mark.parametrize("ratio,P,W,H,seed,cov", GRAD_CASES)
def test_anisotropic_opacity_gradients_match_float64_restatement(ratio, P, W, H, seed, cov, loss_kind, ours):
    """test_gpu_raster_opacity's check (its restatement composites precomputed colours)."""
    from test_gpu_raster_opacity import check_gradients_against_restatement
    check_gradients_against_restatement(ours, _rgb_grad_scene(ratio, P, W, H, seed, cov), seed, loss_kind)


@pytest.mark.parametrize("aa,det", [(False, True), (True, False)])
@pytest.mark.parametrize("ratio,P,W,H,seed,cov", GRAD_CASES)
def test_anisotropic_absgrad_matches_float64_restatement(ratio, P, W, H, seed, cov, aa, det, ours):
    """test_gpu_raster_absgrad's check (its restatement composites precomputed colours)."""
    from test_gpu_raster_absgrad import check_absgrad_against_restatement
    check_absgrad_against_restatement(ours, _rgb_grad_scene(ratio, P, W, H, seed, cov), seed, "all", aa, det)


def test_anisotropic_camera_matches_reference_extension(ours):
    """100 k make_cloud Gaussians at 960x640, fy / fx = 1.448, D = 2, M = 9, scale_modifier 0.9, at the bars of
    test_gpu_raster.test_cuda_matches_reference_extension_at_benchmark_sizes."""
    from s3gaussian_b200 import synthetic as syn
    from test_gpu_raster import check_against_reference_extension
    if not ref_ext.available():
        pytest.skip("oracle/_ref (prebuilt reference extension) not present")
    W, H = 960, 640
    fx = syn.WAYMO_FOCAL * W / 1920.0
    cam = util.anisotropic_camera(W, H, fx, 1.448 * fx, (0.0, 0.0, 2.0))
    d = util.scene_inputs(syn.make_cloud(100_000, seed=0), cam, mode="sh", sh_degree=2, bg=(0.0, 0.0, 0.0))
    d["shs"] = d["shs"][:, :9].contiguous()
    d["scale_modifier"] = 0.9
    check_against_reference_extension(ref_ext.load(), ours, d, "aniso 1.448 M=9 mod=0.9")


def test_filter3d_screen_bound_uses_each_focal(built_lib):
    """compute_filter_3d over cameras with fx != fy against filter3d_ref.compute64; the same cameras with fy set to fx
    see a different set of Gaussians, so a y bound taken with fx would fail."""
    import filter3d_ref
    from s3gaussian_b200 import filter3d, synthetic as syn
    from test_gpu_filter3d import _check_compute
    cams = [util.anisotropic_camera(640, 320, 500.0, 1.448 * 500.0, (0.0, 0.0, 2.0)),
            util.anisotropic_camera(320, 640, 300.0, 0.69 * 300.0, (-3.0, -1.0, 1.5), yaw_deg=-5.0),
            util.anisotropic_camera(960, 640, 1027.5, 1.2 * 1027.5, (5.0, 1.0, 2.0), yaw_deg=10.0)]
    xyz = syn.make_cloud(50_000, seed=5).xyz
    got, want, seen = _check_compute(filter3d, xyz, cams, "anisotropic cameras")
    assert bool(seen.any())
    views, k = filter3d.camera_tensors(cams, DEV)
    assert bool((k[:, 2] != k[:, 3]).all())
    ok = filter3d_ref.valid64(xyz.to(DEV), views, k)[0]
    k_iso = k.clone()
    k_iso[:, 3] = k[:, 2]
    ok_iso = filter3d_ref.valid64(xyz.to(DEV), views, k_iso)[0]
    assert int((ok != ok_iso).sum()) > 1000
    assert not torch.equal(filter3d_ref.compute64(xyz.to(DEV), views, k_iso)[0], want)
