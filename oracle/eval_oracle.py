"""numpy / scipy restatement of the reference's evaluation metrics (utils/video_utils.py:210-241): the checker of
s3g_eval_metrics and s3gaussian_b200.evaluation.

SSIM is skimage.metrics.structural_similarity (>= 0.19) as the reference calls it - data_range=1.0, one channel at
a time, float32 input kept float32 - written from skimage's algorithm: 7x7 scipy.ndimage.uniform_filter (mode
'reflect'), K1 = 0.01, K2 = 0.03, sample covariances (x 49/48), the mean over the map cropped by 3 pixels taken in
float64.  It is cross-checked against skimage itself where skimage is installed (tests/test_eval_host.py).

PSNR is utils/image_utils.py:17-19 on [C,...] arrays: the mean over channels of the per-channel PSNR.
"""
from __future__ import annotations

import numpy as np
from scipy.ndimage import uniform_filter

WIN = 7
K1, K2 = 0.01, 0.03


def ssim_map(x: np.ndarray, y: np.ndarray) -> np.ndarray:
    """float32 SSIM map of two 2-D images (uncropped, what full=True returns)."""
    x = np.asarray(x, np.float32)
    y = np.asarray(y, np.float32)
    if min(x.shape) < WIN:
        raise ValueError("image sides must be >= 7")
    f = lambda a: uniform_filter(a, size=WIN, mode="reflect")   # float32 in, float32 out
    ux, uy = f(x), f(y)
    uxx, uyy, uxy = f(x * x), f(y * y), f(x * y)
    cov_norm = np.float32(WIN * WIN / (WIN * WIN - 1.0))
    vx = cov_norm * (uxx - ux * ux)
    vy = cov_norm * (uyy - uy * uy)
    vxy = cov_norm * (uxy - ux * uy)
    C1 = np.float32((K1 * 1.0) ** 2)
    C2 = np.float32((K2 * 1.0) ** 2)
    two = np.float32(2)
    A1, A2 = two * ux * uy + C1, two * vxy + C2
    B1, B2 = ux * ux + uy * uy + C1, vx + vy + C2
    S = (A1 * A2) / (B1 * B2)
    assert S.dtype == np.float32
    return S


def ssim(img: np.ndarray, gt: np.ndarray) -> float:
    """structural_similarity(img, gt, data_range=1.0, channel_axis=0) of [C,H,W] arrays."""
    p = (WIN - 1) // 2
    vals = [ssim_map(img[c], gt[c])[p:-p, p:-p].mean(dtype=np.float64) for c in range(img.shape[0])]
    return float(np.mean(vals))


def masked_ssim(img: np.ndarray, gt: np.ndarray, mask: np.ndarray) -> float:
    """structural_similarity(HWC, HWC, data_range=1.0, channel_axis=-1, full=True)[1][mask].mean() of [C,H,W]
    arrays and a boolean [H,W] mask (video_utils.py:233-241)."""
    m = np.asarray(mask, bool)
    S = np.stack([ssim_map(img[c], gt[c]) for c in range(img.shape[0])], -1)
    return float(S[m].mean(dtype=np.float64))


def psnr(img: np.ndarray, gt: np.ndarray) -> float:
    """psnr(img, gt).mean() of utils/image_utils.py for [C,...] arrays; identical images give inf."""
    a = np.asarray(img, np.float32).reshape(img.shape[0], -1)
    b = np.asarray(gt, np.float32).reshape(gt.shape[0], -1)
    mse = ((a - b) ** 2).mean(axis=1, dtype=np.float64)
    with np.errstate(divide="ignore"):
        return float(np.mean(20 * np.log10(1.0 / np.sqrt(mse))))


def masked_psnr(img: np.ndarray, gt: np.ndarray, mask: np.ndarray) -> float:
    """psnr of the [C,K] masked pixels (video_utils.py:223-231)."""
    m = np.asarray(mask, bool)
    return psnr(img[:, m], gt[:, m])


def view_metrics(img: np.ndarray, gt: np.ndarray, mask: np.ndarray | None) -> dict:
    """the per-view metrics of render_func; masked ones only for a non-empty mask."""
    out = {"psnr": psnr(img, gt), "ssim": ssim(img, gt)}
    if mask is not None and np.asarray(mask, bool).any():
        out["masked_psnr"] = masked_psnr(img, gt, mask)
        out["masked_ssim"] = masked_ssim(img, gt, mask)
    return out
