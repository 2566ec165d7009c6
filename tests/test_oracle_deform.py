"""CPU: the deformation oracle (oracle/deform_oracle.py) against golden vectors produced by
importing the REAL reference deform_network (tools/make_golden_deform.py)."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import deform_oracle as do
from s3gaussian_b200 import synthetic as syn

GOLD = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "deform_*.npz")))


def load_deform_case(path):
    z = np.load(path)
    st = syn.make_deform_state(int(z["state_seed"]), tuple(int(v) for v in z["resolution"]),
                               tuple(int(v) for v in z["multires"]), weight_scale=0.2)
    flags = dict(no_ds=bool(z["flags"][0]), no_dr=bool(z["flags"][1]), no_do=bool(z["flags"][2]))
    return z, st, flags


def oracle_outputs(z, st, flags, dtype=torch.float64, need_grad=False):
    T = lambda k: torch.from_numpy(z[k]).to(dtype).requires_grad_(need_grad)
    xyz, scales, rot, opa, shs = T("in_xyz"), T("in_scales"), T("in_rot"), T("in_opacity"), T("in_shs")
    state = {k: v.to(dtype).requires_grad_(need_grad and k != "deformation_net.grid.aabb") for k, v in st.items()}
    t = torch.full((xyz.shape[0], 1), float(z["time"]), dtype=dtype)
    d = do.deform_forward(state, xyz, scales, rot, opa, shs, t, **flags)
    fr = do.render_front(xyz, d, torch.from_numpy(z["campos"]).to(dtype), 3)
    outs = (d["means3D"], fr["scales"], fr["rotations"], fr["opacity"], fr["colors_precomp"], d["dx"], d["feat"], d["dshs"])
    return outs, (xyz, scales, rot, opa, shs), state


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


def test_deform_golden_present():
    assert len(GOLD) >= 4


@pytest.mark.parametrize("path", GOLD, ids=[os.path.basename(p)[7:-4] for p in GOLD])
def test_deform_oracle_forward(path):
    z, st, flags = load_deform_case(path)
    outs, _, _ = oracle_outputs(z, st, flags)
    names = ("out_means3D", "out_scales", "out_rot", "out_opacity", "out_colors", "out_dx", "out_feat", "out_dshs")
    for o, n in zip(outs, names):
        assert rel(o.detach().numpy(), z[n]) < 2e-5, (n, rel(o.detach().numpy(), z[n]))


@pytest.mark.parametrize("path", [p for p in GOLD if "default_1k" not in p],
                         ids=[os.path.basename(p)[7:-4] for p in GOLD if "default_1k" not in p])
def test_deform_oracle_backward(path):
    z, st, flags = load_deform_case(path)
    outs, leaves, state = oracle_outputs(z, st, flags, need_grad=True)
    loss = sum((o * torch.from_numpy(z[f"w{i}"]).double()).sum() for i, o in enumerate(outs))
    loss.backward()
    for leaf, n in zip(leaves, ("g_xyz", "g_scales", "g_rot", "g_opacity", "g_shs")):
        assert rel(leaf.grad.numpy(), z[n]) < 1e-4, (n, rel(leaf.grad.numpy(), z[n]))
    checked = 0
    for k, v in state.items():
        key = "pg_" + k
        if key in z.files and v.grad is not None:
            assert rel(v.grad.numpy(), z[key]) < 1e-4, (k, rel(v.grad.numpy(), z[key]))
            checked += 1
    assert checked >= 20


@pytest.mark.parametrize("chunk", [64, 100])
def test_chunked_oracle_equals_single_pass(chunk):
    """do.chunked_front (the float64 oracle run in chunks, what the GPU tests use at 500 k and 2 M Gaussians) against one
    pass over all Gaussians: outputs, input gradients and the plane / Linear gradients that accumulate over the chunks'
    backward calls.  Chunk sizes that do not divide P, every head on, an SH degree below 3 and an unused output."""
    reso, multires = (6, 5, 4, 3), (1, 2)
    st = syn.make_deform_state(4, reso, multires, aabb=((9.0, 4.0, 3.0), (-2.0, -4.0, -3.0)), weight_scale=0.2)
    flags = dict(no_ds=False, no_dr=False, no_do=False)
    P = 301
    g = torch.Generator().manual_seed(9)
    xyz = torch.tensor([-2.0, -4.0, -3.0]) + torch.tensor([11.0, 8.0, 6.0]) * (torch.rand(P, 3, generator=g) * 1.2 - 0.1)
    inputs = [v.double() for v in (xyz, torch.randn(P, 3, generator=g) * 0.3 - 2, torch.randn(P, 4, generator=g),
                                   torch.randn(P, 1, generator=g), torch.randn(P, 16, 3, generator=g) * 0.3)]
    shapes = ((P, 3), (P, 3), (P, 4), (P, 1), (P, 3), (P, 3), (P, 16, 3), (P, 3))
    upstream = [torch.randn(*s, generator=g, dtype=torch.float64) for s in shapes]
    upstream[7] = None
    campos = torch.tensor([0.3, -0.2, 6.0], dtype=torch.float64)

    def run(c):
        state = {k: v.double().requires_grad_(k != "deformation_net.grid.aabb") for k, v in st.items()}
        outs, grads, margins = do.chunked_front(state, inputs, 0.37, campos, 2, upstream, chunk=c, **flags)
        return outs, grads, {k: v.grad for k, v in state.items() if v.grad is not None}, margins

    ref, mine = run(P), run(chunk)
    for a, b in zip(ref[0] + ref[1], mine[0] + mine[1]):
        assert a.shape == b.shape and rel(b.numpy(), a.numpy()) < 1e-12
    assert set(ref[2]) == set(mine[2]) and len(ref[2]) >= 6 * len(multires) + 20
    for k in ref[2]:
        assert rel(mine[2][k].numpy(), ref[2][k].numpy()) < 1e-12, k
    for k in ref[3]:
        assert torch.equal(ref[3][k], mine[3][k]), k
    # the single pass is the plain composition deform_forward -> render_front
    d = do.deform_forward({k: v.double() for k, v in st.items()}, *inputs, torch.full((P, 1), 0.37, dtype=torch.float64),
                          **flags)
    assert torch.equal(ref[0][4], do.render_front(inputs[0], d, campos, 2)["colors_precomp"])


def test_chunked_oracle_empty():
    st = syn.make_deform_state(4, (6, 5, 4, 3), (1,), aabb=((9.0, 4.0, 3.0), (-2.0, -4.0, -3.0)))
    state = {k: v.double().requires_grad_(k != "deformation_net.grid.aabb") for k, v in st.items()}
    inputs = [torch.zeros(0, *s, dtype=torch.float64) for s in ((3,), (3,), (4,), (1,), (16, 3))]
    upstream = [torch.zeros(0, *s, dtype=torch.float64) for s in ((3,), (3,), (4,), (1,), (3,), (3,), (16, 3), (3,))]
    outs, grads, _ = do.chunked_front(state, inputs, 0.5, torch.zeros(3, dtype=torch.float64), 3, upstream, chunk=7)
    assert [tuple(o.shape) for o in outs] == [(0, 3), (0, 3), (0, 4), (0, 1), (0, 3), (0, 3), (0, 16, 3), (0, 3)]
    assert [tuple(x.shape) for x in grads] == [(0, 3), (0, 3), (0, 4), (0, 1), (0, 16, 3)]
    assert all(v.grad is None or not v.grad.any() for v in state.values())
