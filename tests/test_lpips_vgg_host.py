"""CPU: the VGG16 LPIPS oracle against the reference's own module, weight-file loading, argument errors of the Python
API and of the C entry points.  Nothing here launches GPU work."""
import ctypes as C

import pytest
import torch

import lpips_vgg_ref
from oracle import lpips_vgg_oracle as vo


def _pair(shape, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(shape, generator=g)
    return x, (x + 0.2 * torch.randn(shape, generator=g)).clamp(0, 1)


@pytest.mark.skipif(not lpips_vgg_ref.available(),
                    reason="torchvision or oracle/_ref/s3g_ref/lpipsPyTorch (oracle/build_ref_lpips.sh) missing")
@pytest.mark.parametrize("shape", [(3, 48, 64), (3, 47, 33), (2, 3, 48, 64), (2, 3, 61, 35)],
                         ids=["64x48", "33x47", "2x64x48", "2x35x61"])
def test_oracle_matches_reference_module(shape):
    feat, lin = vo.random_state_dicts(3)
    ref = lpips_vgg_ref.reference_module(feat, lin)
    x, y = _pair(shape, sum(shape))
    with torch.no_grad():
        r = ref(x, y)
    assert r.shape == (1, 1, 1, 1) and r.dtype == torch.float32
    o = vo.lpips_terms(x, y, feat, lin)
    assert abs(float(r) - float(o[5])) <= 1e-6 * float(o[5]), (float(r), float(o[5]))
    if len(shape) == 4:   # the batch sum of lpips.py:36
        singles = sum(float(vo.lpips_terms(x[i], y[i], feat, lin)[5]) for i in range(shape[0]))
        assert abs(float(o[5]) - singles) <= 1e-12 * singles


def test_seeded_weights_keep_every_tap_alive():
    """Thirteen random ReLU layers: every layer term must stay far above the GPU comparison's absolute tolerance
    (1e-5), and a healthy share of every tap's activations non-zero, or those comparisons would be vacuous."""
    for seed in (0, 3, 11):
        feat, lin = vo.random_state_dicts(seed)
        x, y = _pair((3, 48, 64), seed)
        terms = vo.lpips_terms(x, y, feat, lin)
        assert all(float(t) > 1e-3 for t in terms[:5]), terms
        for tap in vo.features(x[None], feat):
            assert 0.25 < float((tap > 0).double().mean()) < 0.9


def _write_files(tmp_path, seed=1):
    feat, lin = vo.random_state_dicts(seed)
    full = dict(feat)
    g = torch.Generator().manual_seed(7)
    full["classifier.0.weight"] = torch.randn(16, 8, generator=g)   # the real file's classifier keys: ignored
    full["classifier.0.bias"] = torch.randn(16, generator=g)
    v, l = tmp_path / "vgg16-397923af.pth", tmp_path / "vgg.pth"
    torch.save(full, v)
    torch.save(lin, l)
    return feat, lin, str(v), str(l)


def _no_download(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("torch.hub.load_state_dict_from_url must not be called")
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)


def test_weight_files_load_with_real_key_names(tmp_path, monkeypatch):
    from s3gaussian_b200.lpips_vgg import LPIPSVGG, default_paths
    _no_download(monkeypatch)
    feat, lin, v, l = _write_files(tmp_path)
    assert vo.FEATURE_INDICES == (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
    for fn in (LPIPSVGG(vgg16_path=v, lin_path=l), LPIPSVGG.from_state_dicts(feat, lin)):
        assert len(fn._conv_w) == len(fn._conv_b) == 13 and len(fn._lin) == 5
        for w, b, i in zip(fn._conv_w, fn._conv_b, vo.FEATURE_INDICES):
            assert torch.equal(w, feat[f"features.{i}.weight"]) and torch.equal(b, feat[f"features.{i}.bias"])
        for i, w in enumerate(fn._lin):
            assert torch.equal(w, lin[f"lin{i}.model.1.weight"])
    # the default location is torch.hub.get_dir()/checkpoints
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    (tmp_path / "hub" / "checkpoints").mkdir(parents=True)
    assert default_paths() == (str(tmp_path / "hub" / "checkpoints" / "vgg16-397923af.pth"),
                               str(tmp_path / "hub" / "checkpoints" / "vgg.pth"))
    for src, dst in ((v, default_paths()[0]), (l, default_paths()[1])):
        with open(src, "rb") as fi, open(dst, "wb") as fo:
            fo.write(fi.read())
    assert torch.equal(LPIPSVGG()._conv_w[6], feat["features.14.weight"])


def test_bad_state_dicts():
    from s3gaussian_b200.lpips_vgg import LPIPSVGG
    feat, lin = vo.random_state_dicts(0)
    with pytest.raises(KeyError, match="features.28.bias"):
        LPIPSVGG.from_state_dicts({k: v for k, v in feat.items() if k != "features.28.bias"}, lin)
    with pytest.raises(ValueError, match="lin3.model.1.weight"):
        LPIPSVGG.from_state_dicts(feat, {**lin, "lin3.model.1.weight": torch.zeros(1, 256, 1, 1)})


def test_missing_file_names_the_path_and_never_downloads(tmp_path, monkeypatch):
    from s3gaussian_b200 import lpips_vgg as lv
    _no_download(monkeypatch)
    _, _, v, l = _write_files(tmp_path)
    missing = str(tmp_path / "nowhere" / "vgg.pth")
    with pytest.raises(FileNotFoundError, match=missing):
        lv.LPIPSVGG(vgg16_path=v, lin_path=missing)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "empty_hub"))
    with pytest.raises(FileNotFoundError, match="vgg16-397923af.pth"):
        lv.LPIPSVGG()
    monkeypatch.setattr(lv, "_cached", {})
    with pytest.raises(FileNotFoundError, match="empty_hub"):
        lv.lpips_vgg(torch.rand(3, 40, 40), torch.rand(3, 40, 40))


def test_argument_errors_before_any_gpu_work():
    from s3gaussian_b200.lpips_vgg import LPIPSVGG
    fn = LPIPSVGG.from_state_dicts(*vo.random_state_dicts(0))
    for x, y in (((3, 40, 40), (3, 40, 41)), ((1, 3, 40, 40), (3, 40, 40)), ((4, 40, 40), (4, 40, 40)),
                 ((1, 1, 40, 40), (1, 1, 40, 40)), ((3, 15, 40), (3, 15, 40)), ((2, 3, 40, 15), (2, 3, 40, 15)),
                 ((40, 40), (40, 40)), ((0, 3, 40, 40), (0, 3, 40, 40))):
        with pytest.raises(ValueError):
            fn(torch.rand(x), torch.rand(y))
    # forward only: an input that wants a gradient is refused, not answered with a value that has none
    for gx, gy in ((True, False), (False, True)):
        x, y = torch.rand(3, 40, 40, requires_grad=gx), torch.rand(3, 40, 40, requires_grad=gy)
        with pytest.raises(NotImplementedError, match=r"forward-only.*no_grad\(\).*detach\(\)"):
            fn(x, y)
        with torch.no_grad(), pytest.raises(RuntimeError, match="no CPU path"):
            fn(x, y)
    with pytest.raises(RuntimeError, match="no CPU path"):
        fn(torch.rand(3, 16, 16), torch.rand(3, 16, 16))
    assert fn._prepared == {}


def test_c_entry_points_sizes_and_argument_errors(built_lib):
    from s3gaussian_b200 import _lib
    lib = built_lib
    # every layer's weights as hi | lo over [Cout][K padded to 32], the biases, the five lin vectors
    weights = sum(2 * s[0] * (-(-s[1] * 9 // 32) * 32) for s in vo.CONV_SHAPES)
    floats = weights + sum(s[0] for s in vo.CONV_SHAPES) + sum(vo.CHANNELS)
    assert lib.s3g_lpips_vgg_prepared_bytes() == 4 * floats and 117e6 < 4 * floats < 119e6
    # 1920x1280 pair: two ping-pong buffers of 2 images x 64 channels at full resolution, and the taps' partials
    acts = 2 * (2 * 1280 * 1920 * 64 * 4)
    ws = lib.s3g_lpips_vgg_workspace_bytes(1, 1280, 1920)
    assert acts < ws < acts + 1_000_000 and 2.51e9 < ws < 2.53e9
    assert lib.s3g_lpips_vgg_workspace_bytes(2, 16, 16) > lib.s3g_lpips_vgg_workspace_bytes(1, 16, 16) > 0
    for n, h, w in ((0, 64, 64), (1, 15, 64), (1, 64, 15), (1, 20000, 20000), (7, 1280, 1920)):
        assert lib.s3g_lpips_vgg_workspace_bytes(n, h, w) == 0
    assert lib.s3g_lpips_vgg_workspace_bytes(6, 1280, 1920) > 0
    p = C.c_void_p(256)   # never dereferenced: every call below fails its argument checks first
    for n, h, w, ptrs in ((0, 64, 64, (p, p, p, p, p)), (1, 15, 64, (p, p, p, p, p)), (1, 64, 15, (p, p, p, p, p)),
                          (1, 20000, 20000, (p, p, p, p, p)), (1, 64, 64, (None, p, p, p, p)),
                          (1, 64, 64, (p, None, p, p, p)), (1, 64, 64, (p, p, None, p, p)),
                          (1, 64, 64, (p, p, p, None, p)), (1, 64, 64, (p, p, p, p, None)),
                          (1, 64, 64, (p, p, C.c_void_p(260), p, p))):
        x, y, prep, out, work = ptrs
        assert lib.s3g_lpips_vgg(n, h, w, x, y, prep, out, work, None) == -1, (n, h, w, ptrs)
        assert _lib.last_error()
    assert lib.s3g_lpips_vgg_prepare(None, p, None) == -1
    desc = _lib.LpipsVggWeights()
    assert lib.s3g_lpips_vgg_prepare(C.byref(desc), p, None) == -1
    for i in range(13):
        desc.conv_w[i] = desc.conv_b[i] = 256
    assert lib.s3g_lpips_vgg_prepare(C.byref(desc), p, None) == -1     # the lin pointers are still null
    assert lib.s3g_abi_version() == 2
