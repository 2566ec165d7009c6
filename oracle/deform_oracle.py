"""CPU restatement of the reference's HexPlane field + deformation decoder +
render() front-end arithmetic.  TEST INFRASTRUCTURE ONLY (tier rule 3).

Restates (paths relative to /root/reference):
  normalize_aabb, grid_sample_wrapper, interpolate_ms_features, HexPlaneField.get_density
                                              scene/hexplane.py:19-46,73-106,160-175
  Deformation.query_time / forward_dynamic    scene/deformation.py:78-166 (default flags and the
                                              optional scales / rotations / opacity heads)
  activations + Python SH->RGB of render()    gaussian_renderer/__init__.py:99-117,
                                              utils/sh_utils.py:57-112
Third-party arithmetic restated from its documented behaviour: torch
F.grid_sample(bilinear, align_corners=True, padding_mode='border') - the sampling
coordinate is ((x+1)/2)*(size-1) clipped to [0,size-1], the four neighbours are
weighted by the opposite sub-rectangle areas, out-of-range neighbours contribute 0.

Written with plain torch indexing (no grid_sample, no nn.Linear) so it can run in
float64; pinned against the REAL reference module imported on the CPU
(tools/make_golden_deform.py -> tests/golden/deform_*.npz).
"""
from __future__ import annotations

import itertools

import torch

COMBS = list(itertools.combinations(range(4), 2))   # (0,1),(0,2),(0,3),(1,2),(1,3),(2,3)

C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
      -0.4570457994644658, 1.445305721320277, -0.5900435899266435]


def bilinear_border(plane, x, y):
    """plane [C,H,W]; x,y in normalised [-1,1] coordinates (x -> width). Returns [N,C]."""
    C, H, W = plane.shape
    ix = ((x + 1) / 2) * (W - 1)
    iy = ((y + 1) / 2) * (H - 1)
    ix = ix.clamp(0, W - 1)
    iy = iy.clamp(0, H - 1)
    x0 = torch.floor(ix)
    y0 = torch.floor(iy)
    x1 = x0 + 1
    y1 = y0 + 1
    w_nw = (x1 - ix) * (y1 - iy)
    w_ne = (ix - x0) * (y1 - iy)
    w_sw = (x1 - ix) * (iy - y0)
    w_se = (ix - x0) * (iy - y0)

    def tap(xx, yy, w):
        inb = (xx >= 0) & (xx <= W - 1) & (yy >= 0) & (yy <= H - 1)
        xi = xx.clamp(0, W - 1).long()
        yi = yy.clamp(0, H - 1).long()
        v = plane[:, yi, xi].transpose(0, 1)            # [N,C]
        return v * (w * inb.to(w.dtype)).unsqueeze(1)

    return tap(x0, y0, w_nw) + tap(x1, y0, w_ne) + tap(x0, y1, w_sw) + tap(x1, y1, w_se)


def hexplane_features(state, xyz, t):
    """[N,128] multi-level feature (scene/hexplane.py:73-106,160-175)."""
    aabb = state["deformation_net.grid.aabb"].to(xyz.dtype)
    p = (xyz - aabb[0]) * (2.0 / (aabb[1] - aabb[0])) - 1.0      # normalize_aabb (:19-20); aabb[0] is the MAX corner
    pts = torch.cat([p, t], dim=-1)
    feats = []
    level = 0
    while f"deformation_net.grid.grids.{level}.0" in state:
        f = None
        for ci, (a, b) in enumerate(COMBS):
            plane = state[f"deformation_net.grid.grids.{level}.{ci}"][0].to(xyz.dtype)
            s = bilinear_border(plane, pts[:, a], pts[:, b])
            f = s if f is None else f * s
        feats.append(f)
        level += 1
    return torch.cat(feats, dim=-1)


def _lin(state, name, x):
    return x @ state[name + ".weight"].to(x.dtype).t() + state[name + ".bias"].to(x.dtype)


def _head(state, prefix, h, kinks):     # Sequential(ReLU, Linear, ReLU, Linear)  scene/deformation.py:61-65
    a = _lin(state, prefix + ".1", torch.relu(h))
    kinks += [h, a]
    return _lin(state, prefix + ".3", torch.relu(a))


def deform_forward(state, xyz, scales, rotations, opacity, shs, t, *, no_dx=False, no_ds=True, no_dr=True,
                   no_do=True, no_dshs=False, feat_head=True):
    """Deformation.forward_dynamic (scene/deformation.py:108-166). t: [N,1].
    out["relu_margin"] [N]: the smallest |input| of any ReLU the enabled heads apply (inf if none) - how close the
    Gaussian sits to a kink of the decoder, where the derivative jumps."""
    f = hexplane_features(state, xyz, t)
    h = _lin(state, "deformation_net.feature_out.0", f)                         # D = 1: a single Linear
    out = {}
    kinks = []
    dx = None if no_dx else _head(state, "deformation_net.pos_deform", h, kinks)
    out["means3D"] = xyz if no_dx else xyz + dx                                  # mask == 1 (:117)
    out["scales"] = scales if no_ds else scales + _head(state, "deformation_net.scales_deform", h, kinks)
    out["rotations"] = rotations if no_dr else rotations + _head(state, "deformation_net.rotations_deform", h, kinks)
    out["opacity"] = opacity if no_do else opacity + _head(state, "deformation_net.opacity_deform", h, kinks)
    dshs = None if no_dshs else _head(state, "deformation_net.shs_deform", h, kinks).reshape(-1, 16, 3)
    out["shs"] = shs if no_dshs else shs + dshs
    feat = None
    if feat_head:                                                               # no leading ReLU (:66-76)
        a = _lin(state, "deformation_net.dino_head.0", h)
        b = _lin(state, "deformation_net.dino_head.2", torch.relu(a))
        feat = _lin(state, "deformation_net.dino_head.4", torch.relu(b))
        kinks += [a, b]
    margin = torch.full((xyz.shape[0],), float("inf"), dtype=xyz.dtype, device=xyz.device)
    if kinks:
        margin = torch.cat([k.detach().abs() for k in kinks], dim=1).amin(dim=1)
    out.update(dx=dx, dshs=dshs, feat=feat, hidden=h, features=f, relu_margin=margin)
    return out


def texel_margin(state, xyz):
    """[N]: distance, in normalised coordinates (the [-1,1] of grid_sample), from each Gaussian's spatial sampling
    coordinate to the nearest texel boundary or border of any level - where d(feature)/d(xyz) jumps."""
    aabb = state["deformation_net.grid.aabb"].to(xyz.dtype)
    p = (xyz.detach() - aabb[0]) * (2.0 / (aabb[1] - aabb[0])) - 1.0
    margin = torch.full((xyz.shape[0],), float("inf"), dtype=xyz.dtype, device=xyz.device)
    level = 0
    while f"deformation_net.grid.grids.{level}.0" in state:
        shape = {}
        for ci, (a, b) in enumerate(COMBS):            # width of plane (a,b) is axis a, height is axis b
            H, W = state[f"deformation_net.grid.grids.{level}.{ci}"].shape[-2:]
            shape[a], shape[b] = W, H
        for ax in range(3):
            m = shape[ax] - 1
            ix = (p[:, ax] + 1) / 2 * m
            d = (ix - ix.round().clamp(0, m)).abs() * (2.0 / m)
            margin = torch.minimum(margin, d)
        level += 1
    return margin


def sh_basis(deg, d):
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    b = [torch.full_like(x, C0)]
    if deg > 0:
        b += [-C1 * y, C1 * z, -C1 * x]
    if deg > 1:
        xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
        b += [C2[0] * xy, C2[1] * yz, C2[2] * (2 * zz - xx - yy), C2[3] * xz, C2[4] * (xx - yy)]
    if deg > 2:
        b += [C3[0] * y * (3 * xx - yy), C3[1] * xy * z, C3[2] * y * (4 * zz - xx - yy),
              C3[3] * z * (2 * zz - 3 * xx - 3 * yy), C3[4] * x * (4 * zz - xx - yy), C3[5] * z * (xx - yy),
              C3[6] * x * (xx - 3 * yy)]
    return torch.stack(b, dim=1)          # [N, (deg+1)^2]


def render_front(xyz_undeformed, d_out, campos, active_sh_degree):
    """activations + convert_SHs_python of render() (gaussian_renderer/__init__.py:99-117):
    exp / normalize(eps 1e-12) / sigmoid; SH evaluated with the UNDEFORMED position."""
    scales = torch.exp(d_out["scales"])
    rot = d_out["rotations"] / d_out["rotations"].norm(dim=1, keepdim=True).clamp_min(1e-12)
    opacity = torch.sigmoid(d_out["opacity"])
    dirs = xyz_undeformed - campos
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    B = sh_basis(active_sh_degree, dirs)                       # [N,K]
    K = B.shape[1]
    rgb = (B.unsqueeze(2) * d_out["shs"][:, :K, :]).sum(1)     # [N,3]
    colors = torch.clamp_min(rgb + 0.5, 0.0)
    # clamp_margin [N]: how close the colour is to the clamp's kink
    return dict(scales=scales, rotations=rot, opacity=opacity, colors_precomp=colors,
                clamp_margin=(rgb + 0.5).detach().abs().amin(dim=1))


OUTPUTS = ("means3D", "scales", "rotations", "opacity", "colors_precomp", "dx", "dshs", "feat")


def front_outputs(state, xyz, scales, rotations, opacity, shs, t, campos, active_sh_degree, raw=False, **flags):
    """The eight outputs of the fused front end (s3g_deform_forward_save), in OUTPUTS order; dx, dshs and feat are
    None when their head is off.  raw=True: scales / rotations / opacity before the activations, as
    deform_network.forward_dynamic returns them.  Also returns the per-Gaussian kink margins."""
    d = deform_forward(state, xyz, scales, rotations, opacity, shs, t, **flags)
    fr = render_front(xyz, d, campos, active_sh_degree)
    act = (d["scales"], d["rotations"], d["opacity"]) if raw else (fr["scales"], fr["rotations"], fr["opacity"])
    margins = dict(relu=d["relu_margin"], clamp=fr["clamp_margin"], texel=texel_margin(state, xyz))
    return (d["means3D"], *act, fr["colors_precomp"], d["dx"], d["dshs"], d["feat"]), margins


def chunked_front(state, inputs, time, campos, active_sh_degree, upstream, chunk=65536, raw=False, **flags):
    """front_outputs and its backward, run over the Gaussians in chunks so that millions fit in float64.

    state: {name: tensor} as front_outputs reads it; the trainable entries are leaves with requires_grad, and their
    .grad accumulates over the chunks' backward calls (zero them before).  inputs: (xyz, scales, rotations, opacity,
    shs), [P,*] each.  upstream: dL/d(output) for the eight OUTPUTS, [P,*] each, or None for an output nothing uses.
    Returns (outputs, input_grads, margins): the eight outputs (None for a disabled head), dL/d(input) for the five
    inputs (zeros where no gradient reaches) and the kink margins, each concatenated over the chunks."""
    P = inputs[0].shape[0]
    outs, grads, margins = [], [], []
    for s in range(0, max(P, 1), chunk):          # P == 0: one empty chunk, so that the shapes come out right
        e = min(P, s + chunk)
        leaves = [x[s:e].detach().clone().requires_grad_(True) for x in inputs]
        t = torch.full((e - s, 1), float(time), dtype=inputs[0].dtype, device=inputs[0].device)
        o, m = front_outputs(state, *leaves, t, campos, active_sh_degree, raw=raw, **flags)
        pairs = [(oi, g[s:e].reshape(oi.shape).to(oi.dtype)) for oi, g in zip(o, upstream)
                 if oi is not None and g is not None and oi.requires_grad]
        if pairs:
            torch.autograd.backward([p[0] for p in pairs], [p[1] for p in pairs])
        outs.append([None if oi is None else oi.detach() for oi in o])
        grads.append([torch.zeros_like(x) if x.grad is None else x.grad for x in leaves])
        margins.append(m)
    cat = lambda ts: None if ts[0] is None else torch.cat(ts)
    return ([cat([c[i] for c in outs]) for i in range(len(OUTPUTS))], [cat([c[i] for c in grads]) for i in range(5)],
            {k: torch.cat([m[k] for m in margins]) for k in margins[0]})
