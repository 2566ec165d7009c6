"""Float64 torch restatement of 3DGS-MCMC's densification (include/s3g_b200.h, "MCMC densification"): the relocation of
one row as the published definition writes it (the double sum, not the kernel's rearrangement), the row bookkeeping of
relocate_gs / add_new_gs given the draws, and the position noise given eps."""
import math

import torch

N_MAX = 51
O_MAX = 1.0 - 2.0 ** -23


def binom(n, k):
    return float(math.comb(n, k))


def relocation64(o, ratio, min_opacity=0.005):
    """o [n] float64 opacities, ratio [n] ints -> (o_new clamped, o' unclamped, D, N)."""
    o = o.double()
    N = ratio.to(torch.int64).clamp(max=N_MAX)
    op = 1.0 - (1.0 - o) ** (1.0 / N.double())
    D = torch.zeros_like(o)
    for i in range(1, int(N.max()) + 1 if N.numel() else 1):
        inner = torch.zeros_like(o)
        for k in range(i):
            inner += binom(i - 1, k) * (-1.0) ** k * op ** (k + 1) / math.sqrt(k + 1)
        D += torch.where(i <= N, inner, torch.zeros_like(inner))
    return op.clamp(min_opacity, O_MAX), op, D, N


def relocate_rows64(raw_opacity, raw_scaling, ratio, min_opacity=0.005):
    """Raw [n,1] / [n,3] of the drawn rows -> the relocated (opacity o_new [n], scales s' [n,3]), activated, float64."""
    o = torch.sigmoid(raw_opacity.double().reshape(-1))
    o_new, _, D, _ = relocation64(o, ratio, min_opacity)
    return o_new, (o / D)[:, None] * torch.exp(raw_scaling.double())


def plan_relocate(opacity, drawn, min_opacity=0.005):
    """relocate_gs given its draws: activated opacities [P], drawn [n_dead] rows (in dead-row order) ->
    (dead [n_dead], src_index [P] of the row copy, ratio [n_dead])."""
    dead = torch.nonzero(opacity <= min_opacity, as_tuple=False).squeeze(1)
    idx = torch.arange(opacity.numel(), device=opacity.device)
    idx[dead] = drawn
    return dead, idx, torch.bincount(drawn, minlength=opacity.numel())[drawn] + 1


def plan_add(P, cap_max, drawn):
    """add_new_gs given its draws -> (n, src_index [P + n], new rows [n], ratio [n])."""
    n = max(0, min(cap_max, int(1.05 * P)) - P)
    assert drawn.numel() == n
    dev = drawn.device
    return n, torch.cat((torch.arange(P, device=dev), drawn)), torch.arange(P, P + n, device=dev), \
        torch.bincount(drawn, minlength=P)[drawn] + 1


def build_rotation64(r):
    q = r.double() / r.double().norm(dim=1, keepdim=True)
    w, x, y, z = q.unbind(1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y),
                        2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                        2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], 1).reshape(-1, 3, 3)


def noise64(scaling, rotation, opacity, step, eps):
    """The displacement step * gate * R diag(s^2) R^T eps [P,3], float64."""
    o = torch.sigmoid(opacity.double().reshape(-1))
    gate = 1.0 / (1.0 + torch.exp(-100.0 * ((1.0 - o) - 0.995)))
    R = build_rotation64(rotation)
    S2 = torch.exp(scaling.double()) ** 2
    Sigma = R @ torch.diag_embed(S2) @ R.transpose(1, 2)
    return step * gate[:, None] * (Sigma @ eps.double()[:, :, None])[:, :, 0]
