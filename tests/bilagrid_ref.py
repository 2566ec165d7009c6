"""Float64 restatement of the bilateral-grid slice and total-variation loss (gsplat lib_bilagrid: BilateralGrid.forward
through F.grid_sample, slice, total_variation_loss), written from their definition for the tests."""
import torch
import torch.nn.functional as F


def identity_grids(N, L, GY, GX, dtype=torch.float64):
    eye = torch.tensor([1.0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], dtype=dtype)
    return eye.reshape(1, 12, 1, 1, 1).repeat(N, 1, L, GY, GX)


def slice64(grids, rgb, ids, guide_dtype=torch.float32):
    """grids [N,12,L,GY,GX], rgb [B,3,H,W], ids a list of B ints -> [B,3,H,W], in grids' dtype; differentiable.

    The luminance guide is computed in `guide_dtype`.  gsplat computes it in float32, where a white pixel's luminance
    is exactly 1 and so lies on the upper clamp (in float64 it is 1 - 2^-52, just inside); the default keeps that.
    Everything after the guide is in grids' dtype.  gradcheck needs guide_dtype=torch.float64."""
    B, _, H, W = rgb.shape
    dt, dev = grids.dtype, grids.device
    ys, xs = torch.meshgrid((torch.arange(H, dtype=dt, device=dev) + 0.5) / H,
                            (torch.arange(W, dtype=dt, device=dev) + 0.5) / W, indexing="ij")
    r, g, b = rgb.to(guide_dtype).unbind(1)
    gray = (0.299 * r + 0.587 * g + 0.114 * b).to(dt)              # [B,H,W]
    # grid_sample's (x, y, z) in [-1, 1]: x indexes GX, y GY, z the L luminance levels
    coords = torch.stack([(xs * 2 - 1).expand(B, H, W), (ys * 2 - 1).expand(B, H, W), gray * 2 - 1], dim=-1)
    A = F.grid_sample(grids[list(ids)], coords[:, None], mode="bilinear", align_corners=True, padding_mode="border")
    A = A[:, :, 0].permute(0, 2, 3, 1).reshape(B, H, W, 3, 4)      # [B,H,W,3,4]
    x = rgb.to(dt).permute(0, 2, 3, 1)[..., None]                   # [B,H,W,3,1]
    out = (A[..., :3] @ x)[..., 0] + A[..., 3]
    return out.permute(0, 3, 1, 2)


def tv64(grids):
    """(1/N) sum over dims L, GY, GX of sum(diff^2) / max(numel of one shifted grid without the batch dim, 1)."""
    N = grids.shape[0]
    tv = grids.new_zeros(())
    for d in (2, 3, 4):
        n = grids.shape[d]
        x1 = grids.narrow(d, 1, n - 1)
        x2 = grids.narrow(d, 0, n - 1)
        count = max(x1[0].numel(), 1)
        tv = tv + ((x1 - x2) ** 2).sum() / count
    return tv / N
