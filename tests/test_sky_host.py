"""CPU: the sky-model restatement (tests/sky_ref.py) against the goldens made from the reference module, gradcheck and
the closed-form gradients; state-dict round trips with the reference's key names; the C entry points' argument
errors before any launch; the header in C; and the Python checks that run before any launch."""
import ctypes as C
import glob
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import sky_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "sky_*.npz")))
FAKE = 1 << 20    # never dereferenced: every call below fails validation before any launch
KEYS = ["sky_model.direction_encoding.scales"] + [f"sky_model.sky_head.layers.{i}.{k}" for i in range(3)
                                                   for k in ("weight", "bias")]


def _golden(path):
    z = np.load(path)
    params = [torch.from_numpy(z[f"{k}{i}"]).double() for i in range(3) for k in ("w", "b")]
    return z, params


def test_goldens_exist():
    names = {os.path.basename(p) for p in GOLDEN}
    assert {"sky_w64_ragged.npz", "sky_w256_ragged.npz", "sky_w64_larger.npz", "sky_w256_larger.npz"} <= names


@pytest.mark.parametrize("path", GOLDEN, ids=os.path.basename)
def test_restatement_matches_the_reference_goldens(path):
    z, params = _golden(path)
    H, W = int(z["H"]), int(z["W"])
    c2w, K = torch.from_numpy(z["c2w"]), torch.from_numpy(z["intrinsic"])
    assert float(K[0, 0]) != float(K[1, 1]) and float(K[0, 2]) != W / 2
    out, grads = ref.sky_grads64(params, c2w, K, H, W, torch.from_numpy(z["dL_dsky"]), chunk=997)
    want = torch.from_numpy(z["sky"]).double()
    assert float((out - want).abs().max()) <= 1e-5 * float(want.abs().max())
    for i, name in enumerate(("grad_w0", "grad_b0", "grad_w1", "grad_b1", "grad_w2", "grad_b2")):
        w = torch.from_numpy(z[name]).double()
        assert float((grads[i] - w).abs().max()) <= 1e-4 * float(w.abs().max()), name
    # the autograd form gives the same image
    assert float((ref.sky64(params, c2w, K, H, W) - out).abs().max()) < 1e-12


def test_restatement_gradcheck_and_closed_form():
    torch.manual_seed(0)
    Wd, H, W = 8, 3, 5
    params = [torch.randn(Wd, 33), torch.randn(Wd) * 0.2, torch.randn(Wd, Wd + 33) * 0.3, torch.randn(Wd) * 0.2,
              torch.randn(3, Wd) * 0.4, torch.randn(3) * 0.2]
    params = [p.double().requires_grad_(True) for p in params]
    c2w = torch.eye(4, dtype=torch.float64)
    K = torch.tensor([[4.0, 0, 2.3], [0, 3.0, 1.4], [0, 0, 1]], dtype=torch.float64)
    assert torch.autograd.gradcheck(lambda *p: ref.sky64(p, c2w, K, H, W), params)
    g = torch.randn(3, H, W, dtype=torch.float64)
    want = torch.autograd.grad((ref.sky64(params, c2w, K, H, W) * g).sum(), params)
    _, got = ref.sky_grads64([p.detach() for p in params], c2w, K, H, W, g, chunk=4)
    for a, b in zip(got, want):
        assert torch.allclose(a, b, rtol=1e-10, atol=1e-12)


def test_encoding_layout():
    v = torch.tensor([[0.1, -0.2, 0.3]], dtype=torch.float64)
    e = ref.encode(v)[0]
    assert e.shape == (33,)
    assert torch.equal(e[:3], v[0])
    assert torch.allclose(e[3 + 3 * 2: 6 + 3 * 2], torch.sin(4 * v[0]))                 # scale 4, sin
    assert torch.allclose(e[18 + 3 * 4: 21 + 3 * 4], torch.cos(16 * v[0]))              # scale 16, sin(x + pi/2)


# ---- Python: layout, state dicts, checks -------------------------------------------------------------------------
def test_state_dict_uses_the_reference_keys_and_round_trips():
    from s3gaussian_b200.sky import Background_Model
    for width in (64, 128, 192, 256):
        m = Background_Model(img_width=37, img_height=23, model_cfg={"mlp_width": width})
        sd = m.state_dict()
        assert list(sd) == KEYS
        assert torch.equal(sd["sky_model.direction_encoding.scales"], torch.tensor([1.0, 2, 4, 8, 16]))
        shapes = [tuple(sd[k].shape) for k in KEYS[1:]]
        assert shapes == [(width, 33), (width,), (width, width + 33), (width,), (3, width), (3,)]
        m2 = Background_Model(img_width=37, img_height=23, model_cfg={"mlp_width": width})
        m2.load_state_dict({k: torch.randn_like(v) if k != KEYS[0] else v for k, v in sd.items()})
        m.load_state_dict(m2.state_dict())
        for k in KEYS:
            assert torch.equal(m.state_dict()[k], m2.state_dict()[k])


@pytest.mark.parametrize("path", GOLDEN[:1], ids=os.path.basename)
def test_reference_state_dict_loads_unchanged(path):
    """The golden's weights, under the reference's key names, load into Background_Model unchanged."""
    from s3gaussian_b200.sky import Background_Model
    z, _ = _golden(path)
    sd = {KEYS[0]: torch.tensor([1.0, 2, 4, 8, 16])}
    for i in range(3):
        sd[f"sky_model.sky_head.layers.{i}.weight"] = torch.from_numpy(z[f"w{i}"])
        sd[f"sky_model.sky_head.layers.{i}.bias"] = torch.from_numpy(z[f"b{i}"])
    m = Background_Model(img_width=int(z["W"]), img_height=int(z["H"]), model_cfg={"mlp_width": int(z["width"])})
    m.load_state_dict(sd)
    assert torch.equal(m.sky_model.sky_head.layers[1].weight, torch.from_numpy(z["w1"]))


def test_python_errors_before_any_launch():
    from s3gaussian_b200.sky import Background_Model, SkyModel
    with pytest.raises(KeyError, match="mlp_width"):
        Background_Model()                                   # the reference's own default model_cfg
    with pytest.raises(KeyError, match="mlp_width"):
        SkyModel({"head_mlp_layer_width": 256})
    for w in (32, 100, 320, 0, 64.0, True, "256"):
        with pytest.raises(ValueError, match="mlp_width"):
            SkyModel({"mlp_width": w})
    for t in ("gs", "rec_shell", "sphere_shell", "other"):
        with pytest.raises(NotImplementedError, match=t):
            Background_Model(model_type=t, model_cfg={"mlp_width": 64})
    for kw in ({"img_width": 0}, {"img_height": -1}, {"img_width": 2.0}, {"img_width": 1 << 16, "img_height": 1 << 15}):
        with pytest.raises(ValueError, match="img_"):
            Background_Model(model_cfg={"mlp_width": 64}, **kw)
    assert SkyModel().width == 256
    m = Background_Model(img_width=8, img_height=6, model_cfg={"mlp_width": 64})
    c2w, K = torch.eye(4), torch.tensor([[4.0, 0, 4], [0, 4, 3], [0, 0, 1]])
    with pytest.raises(RuntimeError, match="CUDA"):
        m(c2w, K)
    m.sky_model.sky_head.layers[0].weight.data = m.sky_model.sky_head.layers[0].weight.data.double()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(c2w, K)


def test_camera_argument_checks():
    from s3gaussian_b200 import sky
    for x, n, match in ((torch.eye(3), 4, r"\[4,4\]"), (torch.eye(4)[None].repeat(2, 1, 1), 4, r"\[4,4\]"),
                        (torch.eye(3, dtype=torch.int32), 3, "floating"), ([[1.0]], 3, "tensor")):
        with pytest.raises(ValueError, match=match):
            sky._camera_tensor(x, "c2w", n, "cpu")
    assert sky._camera_tensor(torch.eye(4, dtype=torch.float64)[None], "c2w", 4, "cpu").dtype == torch.float32


def test_sky_camera_of_a_synthetic_camera():
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.sky import sky_camera
    cam = syn.make_camera(96, 64, (1.0, 2.0, 0.5), yaw_deg=30.0, pitch_deg=-10.0)
    c2w, K = sky_camera(cam)
    w2c = cam.world_view_transform.transpose(0, 1)
    assert torch.allclose(c2w @ w2c, torch.eye(4), atol=1e-5)
    assert float(K[0, 2]) == 48.0 and float(K[1, 2]) == 32.0
    assert abs(float(K[0, 0]) - 96 / (2 * np.tan(cam.FoVx / 2))) < 1e-3
    ref_cam = type("Cam", (), {"c2w": torch.eye(4, dtype=torch.float64), "intrinsic": K.double()})()
    a, b = sky_camera(ref_cam)
    assert a.dtype == torch.float32 and torch.equal(a, torch.eye(4)) and torch.equal(b, K)


# ---- the C entry points --------------------------------------------------------------------------------------------
def _net(lib_mod, width=64, **null):
    ptr = {k: (None if null.get(k) else FAKE) for k in ("w0", "b0", "w1", "b1", "w2", "b2")}
    return lib_mod.SkyNet(width, **ptr)


def test_argument_errors_before_any_launch(built_lib):
    from s3gaussian_b200 import _lib
    lib = built_lib

    def fwd(net=None, H=6, W=8, c2w=FAKE, K=FAKE, out=FAKE, ws=FAKE):
        return lib.s3g_sky_forward(C.byref(net) if net is not None else None, H, W, c2w, K, out, ws, None)

    def bwd(net=None, H=6, W=8, c2w=FAKE, K=FAKE, g=FAKE, grads="ok", ws=FAKE):
        gr = _lib.SkyNetGrads(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE) if grads == "ok" else grads
        return lib.s3g_sky_backward(C.byref(net) if net is not None else None, H, W, c2w, K, g,
                                    C.byref(gr) if gr is not None else None, ws, None)
    ok = _net(_lib)
    common = [({"net": None}, b"null net"), ({"H": 0}, b">= 1"), ({"W": -3}, b">= 1"),
              ({"H": 1 << 15, "W": 1 << 15}, b"32-bit"), ({"c2w": None}, b"null pointer"), ({"K": None}, b"null pointer"),
              ({"ws": None}, b"null workspace"), ({"ws": FAKE + 4}, b"16-byte")]
    common += [({"net": _net(_lib, width=w)}, b"multiple of 64") for w in (0, 32, 96, 320, -64)]
    common += [({"net": _net(_lib, **{k: True})}, b"null pointer") for k in ("w0", "b0", "w1", "b1", "w2", "b2")]
    for kw, msg in common + [({"out": None}, b"null pointer")]:
        kw = {"net": ok, **kw}
        assert fwd(**kw) == -1, kw
        assert msg in lib.s3g_last_error(), (kw, lib.s3g_last_error())
    for kw, msg in common + [({"g": None}, b"null pointer"), ({"grads": None}, b"null pointer")] + \
            [({"grads": _lib.SkyNetGrads(*[None if j == i else FAKE for j in range(6)])}, b"null pointer")
             for i in range(6)]:
        kw = {"net": ok, **kw}
        assert bwd(**kw) == -1, kw
        assert msg in lib.s3g_last_error(), (kw, lib.s3g_last_error())


def test_workspace_bytes(built_lib):
    lib = built_lib
    for w in (0, 32, 96, 320):
        assert lib.s3g_sky_workspace_bytes(w, 6, 8) == 0
    assert lib.s3g_sky_workspace_bytes(64, 0, 8) == 0 and lib.s3g_sky_workspace_bytes(64, 1 << 15, 1 << 15) == 0
    a = lib.s3g_sky_workspace_bytes(64, 1, 1)
    assert a > 0 and a % 256 == 0
    # bounded by the backward's pixel chunk: the same from 65536 pixels on
    big = lib.s3g_sky_workspace_bytes(256, 640, 960)
    assert big == lib.s3g_sky_workspace_bytes(256, 1280, 1920) == lib.s3g_sky_workspace_bytes(256, 256, 256)
    assert big < 65536 * (4 * 256 + 56) * 4 + (16 << 20)        # the chunk's activations + weights and partials
    assert lib.s3g_sky_workspace_bytes(64, 640, 960) < big


def test_header_declares_the_entry_points_in_c(built_lib, tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    from s3gaussian_b200 import _lib
    libdir = os.path.dirname(_lib.LIB_PATH)
    src = tmp_path / "sky.c"
    src.write_text('#include <stddef.h>\n#include "s3g_b200.h"\n'
                   'int main(void) {\n'
                   '    float* p = NULL;\n'
                   '    s3g_sky_net net = {64, NULL, NULL, NULL, NULL, NULL, NULL};\n'
                   '    s3g_sky_net_grads g = {NULL, NULL, NULL, NULL, NULL, NULL};\n'
                   '    size_t ws = s3g_sky_workspace_bytes(64, 6, 8);\n'
                   '    int a = s3g_sky_forward(&net, 6, 8, p, p, p, NULL, NULL);\n'
                   '    int b = s3g_sky_backward(&net, 6, 8, p, p, p, &g, NULL, NULL);\n'
                   '    return (ws > 0 && a == S3G_ERR_ARG && b == S3G_ERR_ARG) ? 0 : 1;\n'
                   '}\n')
    exe = tmp_path / "sky"
    r = subprocess.run([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                        "-o", str(exe), "-L", libdir, "-ls3g_b200", f"-Wl,-rpath,{libdir}"], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = "/usr/local/cuda/lib64" + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    assert subprocess.run([str(exe)], env=env).returncode == 0
