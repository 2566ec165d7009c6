"""CPU: argument checks of the split forward and the evaluation-metrics entry points (no GPU needed), and
properties of the evaluation oracle (oracle/eval_oracle.py), including a cross-check against skimage where it is
installed."""
import numpy as np
import pytest

from oracle import eval_oracle as eo


def test_eval_metrics_argument_errors_do_not_need_a_gpu(built_lib):
    lib = built_lib
    fake = 1 << 20   # never dereferenced: every call below fails validation first
    for C, H, W in ((3, 6, 64), (3, 64, 6), (0, 64, 64), (5, 64, 64)):
        assert lib.s3g_eval_metrics(C, H, W, fake, fake, None, fake, fake, None) == -1, (C, H, W)
    assert b">= 7" in lib.s3g_last_error() or b"C <= 4" in lib.s3g_last_error()
    assert lib.s3g_eval_metrics(3, 7, 7, None, fake, None, fake, fake, None) == -1
    assert lib.s3g_eval_metrics(3, 7, 7, fake, fake, None, None, fake, None) == -1
    assert lib.s3g_eval_metrics(3, 7, 7, fake, fake, None, fake, None, None) == -1
    assert lib.s3g_eval_metrics_workspace_bytes(3, 1280, 1920) >= 3 * 40 * 60 * 5 * 4
    assert lib.s3g_eval_metrics_workspace_bytes(0, 7, 7) == 0


def test_forward_split_argument_errors_do_not_need_a_gpu(built_lib):
    from s3gaussian_b200 import _lib
    lib = built_lib
    cb = _lib.ALLOC_FN(lambda user, n: 0)
    fake = 1 << 20

    def call(P, group, cd, dd, cs, ds):
        return lib.s3g_rasterize_forward_split(cb, None, cb, None, cb, None, P, 0, 0, fake, 16, 16, *([None] * 5), 1.0,
                                               *([None] * 5), 1.0, 1.0, 0, fake, fake, None, 0, None,
                                               group, cd, dd, cs, ds)
    # mismatched null output pairs
    assert call(4, fake, fake, None, fake, fake) == -1
    assert call(4, fake, fake, fake, None, fake) == -1
    assert call(4, fake, None, fake, fake, fake) == -1
    assert b"null dynamic/static output" in lib.s3g_last_error()
    # no group with Gaussians to split
    assert call(4, None, fake, fake, fake, fake) == -1
    assert b"null group" in lib.s3g_last_error()
    # bad sizes, as the plain forward
    assert call(-5, fake, fake, fake, fake, fake) == -1


def _pair(H, W, seed):
    g = np.random.default_rng(seed)
    x = g.random((3, H, W), dtype=np.float32)
    y = np.clip(x + g.normal(0, 0.1, (3, H, W)).astype(np.float32), 0, 1).astype(np.float32)
    return x, y


def test_oracle_identical_images():
    x, _ = _pair(40, 33, 0)
    assert eo.ssim(x, x) == 1.0
    assert np.all(eo.ssim_map(x[0], x[0]) == 1.0)
    assert eo.psnr(x, x) == np.inf
    m = np.zeros((40, 33), bool)
    m[5:9, 7:20] = True
    assert eo.masked_psnr(x, x, m) == np.inf and eo.masked_ssim(x, x, m) == 1.0


def test_oracle_psnr_is_mean_of_per_channel_psnr():
    x, y = _pair(20, 30, 1)
    y[1] = x[1] + 0.5 * (y[1] - x[1])   # channels with different errors: mean of PSNRs != PSNR of the pooled MSE
    per = [eo.psnr(x[c:c + 1], y[c:c + 1]) for c in range(3)]
    assert eo.psnr(x, y) == pytest.approx(np.mean(per), abs=1e-12)
    pooled = 10 * np.log10(1.0 / np.mean((x.astype(np.float64) - y) ** 2))
    assert abs(eo.psnr(x, y) - pooled) > 1e-3


def test_oracle_masked_metrics_see_only_their_pixels():
    H, W = 48, 52
    x, y = _pair(H, W, 2)
    m = np.zeros((H, W), bool)
    m[10:20, 12:30] = True
    # PSNR: nothing outside the mask matters
    x2, y2 = x.copy(), y.copy()
    x2[:, ~m] = 0.25
    y2[:, ~m] = 0.75
    assert eo.masked_psnr(x, y, m) == eo.masked_psnr(x2, y2, m)
    # SSIM: nothing farther than the window radius from the mask matters
    near = np.zeros_like(m)
    near[10 - 3:20 + 3, 12 - 3:30 + 3] = True
    x3, y3 = x.copy(), y.copy()
    x3[:, ~near] = 0.25
    y3[:, ~near] = 0.75
    assert eo.masked_ssim(x, y, m) == eo.masked_ssim(x3, y3, m)
    # the full mask: masked PSNR is the PSNR, masked SSIM the mean of the uncropped map
    full = np.ones((H, W), bool)
    assert eo.masked_psnr(x, y, full) == pytest.approx(eo.psnr(x, y), abs=1e-12)
    S = np.stack([eo.ssim_map(x[c], y[c]) for c in range(3)])
    assert eo.masked_ssim(x, y, full) == pytest.approx(S.mean(dtype=np.float64), abs=1e-12)
    assert eo.ssim(x, y) == pytest.approx(S[:, 3:-3, 3:-3].mean(axis=(1, 2), dtype=np.float64).mean(), abs=1e-12)


def test_oracle_rejects_images_below_the_window():
    with pytest.raises(ValueError):
        eo.ssim_map(np.zeros((6, 10), np.float32), np.zeros((6, 10), np.float32))


@pytest.mark.parametrize("H,W", [(7, 7), (31, 45), (96, 64)])
def test_oracle_matches_skimage(H, W):
    skm = pytest.importorskip("skimage.metrics")
    x, y = _pair(H, W, 3)
    ref = skm.structural_similarity(x, y, data_range=1.0, channel_axis=0)
    assert abs(eo.ssim(x, y) - float(ref)) < 1e-6
    _, S = skm.structural_similarity(np.moveaxis(x, 0, -1), np.moveaxis(y, 0, -1), data_range=1.0, channel_axis=-1,
                                     full=True)
    m = np.random.default_rng(4).random((H, W)) < 0.3
    assert abs(eo.masked_ssim(x, y, m) - float(S[m].mean())) < 1e-6
