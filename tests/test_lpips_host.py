"""CPU: the LPIPS oracle against the reference's own module, weight-file loading, argument errors of the Python API
and of the C entry points.  Nothing here launches GPU work."""
import ctypes as C

import pytest
import torch

import lpips_ref
from oracle import lpips_oracle as lo


def _pair(shape, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(shape, generator=g)
    return x, (x + 0.2 * torch.randn(shape, generator=g)).clamp(0, 1)


@pytest.mark.skipif(not lpips_ref.available(),
                    reason="torchvision or oracle/_ref/s3g_ref/lpipsPyTorch (oracle/build_ref_lpips.sh) missing")
@pytest.mark.parametrize("shape", [(3, 48, 64), (3, 131, 97), (2, 3, 48, 64), (2, 3, 131, 97)],
                         ids=["64x48", "97x131", "2x64x48", "2x97x131"])
def test_oracle_matches_reference_module(shape):
    feat, lin = lo.random_state_dicts(3)
    ref = lpips_ref.reference_module(feat, lin)
    x, y = _pair(shape, sum(shape))
    with torch.no_grad():
        r = ref(x, y)
    assert r.shape == (1, 1, 1, 1) and r.dtype == torch.float32
    o = lo.lpips_terms(x, y, feat, lin)
    assert abs(float(r) - float(o[5])) <= 1e-6 * float(o[5]), (float(r), float(o[5]))
    if len(shape) == 4:   # the batch sum of lpips.py:36
        singles = sum(float(lo.lpips_terms(x[i], y[i], feat, lin)[5]) for i in range(shape[0]))
        assert abs(float(o[5]) - singles) <= 1e-12 * singles


def _write_files(tmp_path, seed=1):
    feat, lin = lo.random_state_dicts(seed)
    full = dict(feat)
    g = torch.Generator().manual_seed(7)
    full["classifier.1.weight"] = torch.randn(16, 8, generator=g)   # the real file's classifier keys: ignored
    full["classifier.1.bias"] = torch.randn(16, generator=g)
    a, l = tmp_path / "alexnet-owt-7be5be79.pth", tmp_path / "alex.pth"
    torch.save(full, a)
    torch.save(lin, l)
    return feat, lin, str(a), str(l)


def _no_download(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("torch.hub.load_state_dict_from_url must not be called")
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", refuse)


def test_weight_files_load_with_real_key_names(tmp_path, monkeypatch):
    from s3gaussian_b200.lpips import LPIPS, default_paths
    _no_download(monkeypatch)
    feat, lin, a, l = _write_files(tmp_path)
    for fn in (LPIPS(alexnet_path=a, lin_path=l), LPIPS.from_state_dicts(feat, lin)):
        for w, i in zip(fn._conv_w, lo.FEATURE_INDICES):
            assert torch.equal(w, feat[f"features.{i}.weight"])
        for b, i in zip(fn._conv_b, lo.FEATURE_INDICES):
            assert torch.equal(b, feat[f"features.{i}.bias"])
        for i, w in enumerate(fn._lin):
            assert torch.equal(w, lin[f"lin{i}.model.1.weight"])
    # the default location is torch.hub.get_dir()/checkpoints
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    (tmp_path / "hub" / "checkpoints").mkdir(parents=True)
    assert default_paths() == (str(tmp_path / "hub" / "checkpoints" / "alexnet-owt-7be5be79.pth"),
                               str(tmp_path / "hub" / "checkpoints" / "alex.pth"))
    for src, dst in ((a, default_paths()[0]), (l, default_paths()[1])):
        with open(src, "rb") as fi, open(dst, "wb") as fo:
            fo.write(fi.read())
    assert torch.equal(LPIPS()._conv_w[2], feat["features.6.weight"])


def test_missing_file_names_the_path_and_never_downloads(tmp_path, monkeypatch):
    from s3gaussian_b200 import lpips as lp
    _no_download(monkeypatch)
    _, _, a, l = _write_files(tmp_path)
    missing = str(tmp_path / "nowhere" / "alex.pth")
    with pytest.raises(FileNotFoundError, match=missing):
        lp.LPIPS(alexnet_path=a, lin_path=missing)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "empty_hub"))
    with pytest.raises(FileNotFoundError, match="alexnet-owt-7be5be79.pth"):
        lp.LPIPS()
    monkeypatch.setattr(lp, "_cached", {})
    with pytest.raises(FileNotFoundError, match="empty_hub"):
        lp.lpips(torch.rand(3, 40, 40), torch.rand(3, 40, 40))


def test_argument_errors_before_any_gpu_work():
    from s3gaussian_b200.lpips import LPIPS, lpips
    for net in ("vgg", "squeeze"):
        with pytest.raises(NotImplementedError):
            LPIPS(net_type=net)
        with pytest.raises(NotImplementedError):
            lpips(torch.rand(3, 40, 40), torch.rand(3, 40, 40), net_type=net)
    with pytest.raises(AssertionError):
        LPIPS(version="0.0")
    with pytest.raises(AssertionError):
        lpips(torch.rand(3, 40, 40), torch.rand(3, 40, 40), version="0.2")
    fn = LPIPS.from_state_dicts(*lo.random_state_dicts(0))
    for x, y in (((3, 40, 40), (3, 40, 41)), ((1, 3, 40, 40), (3, 40, 40)), ((4, 40, 40), (4, 40, 40)),
                 ((1, 1, 40, 40), (1, 1, 40, 40)), ((3, 30, 40), (3, 30, 40)), ((2, 3, 40, 30), (2, 3, 40, 30)),
                 ((40, 40), (40, 40)), ((0, 3, 40, 40), (0, 3, 40, 40))):
        with pytest.raises(ValueError):
            fn(torch.rand(x), torch.rand(y))
    with pytest.raises(RuntimeError, match="no CPU path"):
        fn(torch.rand(3, 40, 40), torch.rand(3, 40, 40))
    assert fn._prepared == {}


def test_c_entry_points_sizes_and_argument_errors(built_lib):
    from s3gaussian_b200 import _lib
    lib = built_lib
    tiles = sum((s[0] // 64) * (-(-s[1] * s[2] * s[3] // 32)) for s in lo.CONV_SHAPES)
    assert lib.s3g_lpips_alex_prepared_bytes() == 4 * (tiles * 2 * 64 * 32 + 2 * sum(s[0] for s in lo.CONV_SHAPES))
    # 1920x1280 pair: 64@319x479, 64@159x239, 192@159x239, 192@79x119, 384 + 256 + 256 @79x119, 2 images
    acts = 2 * 4 * (64 * 319 * 479 + 64 * 159 * 239 + 192 * 159 * 239 + 192 * 79 * 119 + 896 * 79 * 119)
    ws = lib.s3g_lpips_alex_workspace_bytes(1, 1280, 1920)
    assert acts < ws < acts + 200_000 and 0.23e9 < ws < 0.25e9
    assert lib.s3g_lpips_alex_workspace_bytes(2, 31, 31) > lib.s3g_lpips_alex_workspace_bytes(1, 31, 31) > 0
    for n, h, w in ((0, 64, 64), (1, 30, 64), (1, 64, 30), (1, 20000, 20000), (400, 1280, 1920)):
        assert lib.s3g_lpips_alex_workspace_bytes(n, h, w) == 0
    p = C.c_void_p(256)   # never dereferenced: every call below fails its argument checks first
    for n, h, w, ptrs in ((0, 64, 64, (p, p, p, p, p)), (1, 30, 64, (p, p, p, p, p)), (1, 64, 30, (p, p, p, p, p)),
                          (1, 20000, 20000, (p, p, p, p, p)), (1, 64, 64, (None, p, p, p, p)),
                          (1, 64, 64, (p, None, p, p, p)), (1, 64, 64, (p, p, None, p, p)),
                          (1, 64, 64, (p, p, p, None, p)), (1, 64, 64, (p, p, p, p, None))):
        x, y, prep, out, work = ptrs
        assert lib.s3g_lpips_alex(n, h, w, x, y, prep, out, work, None) == -1, (n, h, w, ptrs)
        assert _lib.last_error()
    assert lib.s3g_lpips_alex_prepare(None, p, None) == -1
    desc = _lib.LpipsAlexWeights()
    assert lib.s3g_lpips_alex_prepare(C.byref(desc), p, None) == -1
