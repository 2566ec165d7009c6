"""GPU: selective Adam (s3g_adam_step_selective, FusedAdam.step(visibility=...), examples/train_loop.py --sparse-adam).

1. Five steps with a fresh mask each against oracle.train_oracle.adam_step in float64, started from the float32 state
   before each step: the six per-Gaussian row widths and dense groups (a channels_last 4-D plane among them), P from 1
   to 100 003, masks from none to all.  Visible rows to 1e-6 relative; invisible rows bitwise unchanged in p, m and v
   with NaN in their gradients; the step counter global.
2. Bitwise identities with the dense step: an all-true mask, and the dense groups under any mask; also for tensor views
   off a 16-byte boundary (the scalar path).
3. No host synchronisation, and two runs from one seed bitwise equal.
4. GaussianModel: prune / densify / relocate_gs / add_new_gs followed by a step with the old mask, spatial_sort,
   capture() / restore(), and the training loop with --sparse-adam.
"""
import io
import os
import re
import subprocess
import sys

import pytest
import torch

from oracle.train_oracle import adam_step

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B1, B2, EPS = 0.9, 0.999, 1e-15

# the reference's per-Gaussian groups: row shapes of xyz, f_dc, f_rest (SH degree 3), opacity, scaling, rotation
ROW_SHAPES = {"xyz": (3,), "f_dc": (1, 3), "f_rest": (15, 3), "opacity": (1,), "scaling": (3,), "rotation": (4,)}
MASKS = ["none", "one", "10pct", "runs", "all"]


def _mask(kind, P, gen):
    if kind == "none":
        return torch.zeros(P, dtype=torch.bool)
    if kind == "one":
        m = torch.zeros(P, dtype=torch.bool)
        m[int(torch.randint(P, (1,), generator=gen))] = True
        return m
    if kind == "10pct":
        return torch.rand(P, generator=gen) < 0.1
    if kind == "runs":      # what a Morton-ordered model sees: a few long runs of visible rows
        m = torch.zeros(P, dtype=torch.bool)
        for _ in range(3):
            a = int(torch.randint(P, (1,), generator=gen))
            m[a:a + max(1, P // 7)] = True
        return m
    return torch.ones(P, dtype=torch.bool)


def _optimizer(P, gen, *, offset=0):
    """Per-Gaussian groups of P rows and dense groups (an MLP and a channels_last plane), random parameters and
    moments from two dense warm-up steps.  offset > 0 makes every per-Gaussian tensor a view `offset` floats into
    its storage, off a 16-byte boundary."""
    from s3gaussian_b200.optim import FusedAdam

    def param(shape):
        n = 1
        for s in shape:
            n *= s
        base = torch.randn(n + offset, generator=gen)
        return torch.nn.Parameter(base.to(DEV)[offset:].view(shape))
    groups = [{"params": [param((P, *shape))], "lr": 1e-3 * (k + 1), "name": name}
              for k, (name, shape) in enumerate(ROW_SHAPES.items())]
    plane = torch.nn.Parameter(torch.randn(1, 16, 24, 10, generator=gen).to(DEV).contiguous(
        memory_format=torch.channels_last))
    groups += [{"params": [torch.nn.Parameter(torch.randn(64, 27, generator=gen).to(DEV)),
                           torch.nn.Parameter(torch.randn(64, generator=gen).to(DEV))], "lr": 2e-4, "name": "deformation"},
               {"params": [plane], "lr": 3e-4, "name": "grid"}]
    opt = FusedAdam(groups, lr=0.0, eps=EPS, betas=(B1, B2), selective_groups=ROW_SHAPES)
    for _ in range(2):
        _grads(opt, gen)
        opt.step()
    return opt


def _params(opt):
    return [(g["name"], p) for g in opt.param_groups for p in g["params"]]


def _grads(opt, gen, mask=None):
    """Fresh gradients; with a mask, NaN in the rows it hides."""
    for name, p in _params(opt):
        g = torch.randn(p.shape, generator=gen).to(DEV)
        if p.dim() == 4:
            g = g.contiguous(memory_format=torch.channels_last)
        if mask is not None and name in ROW_SHAPES:
            g[~mask.to(DEV)] = float("nan")
        if p.storage_offset():      # keep the gradient as misaligned as the parameter
            buf = torch.empty(p.numel() + p.storage_offset(), device=DEV)
            g = buf[p.storage_offset():].view(p.shape).copy_(g)
        p.grad = g


def _snapshot(opt):
    return {id(p): (p.detach().clone(), opt.state[p]["exp_avg"].clone(), opt.state[p]["exp_avg_sq"].clone(),
                    int(opt.state[p]["step"])) for _, p in _params(opt)}


def _relerr(a, b, old):
    """Error relative to the larger of the result and the value it was updated from: one row's exp_avg can cancel to
    near zero (beta1 m + (1 - beta1) g), and float32 then keeps the absolute error of its operands."""
    scale = torch.maximum(b.abs().max(), old.double().abs().max())
    return float((a.double() - b).abs().max() / (scale + 1e-30))


@pytest.mark.parametrize("P", [1, 7, 4095, 4096, 4097, 100_003])
@pytest.mark.parametrize("kind", MASKS)
def test_five_steps_against_float64(P, kind, built_lib):
    gen = torch.Generator().manual_seed(P + 17 * MASKS.index(kind))
    opt = _optimizer(P, gen)
    for _ in range(5):
        mask = _mask(kind, P, gen).to(DEV)
        _grads(opt, gen, mask)
        before = _snapshot(opt)
        grads = {id(p): p.grad.clone() for _, p in _params(opt)}
        opt.step(visibility=mask)
        for (name, p), group in zip(_params(opt), [g for g in opt.param_groups for _ in g["params"]]):
            p0, m0, v0, step0 = before[id(p)]
            st = opt.state[p]
            assert int(st["step"]) == step0 + 1, name
            rows = mask if name in ROW_SHAPES else torch.ones(p.shape[0], dtype=torch.bool, device=DEV)
            want = adam_step(p0.double(), grads[id(p)].double(), m0.double(), v0.double(), step0 + 1, group["lr"],
                             B1, B2, EPS)
            for got, w, old, what in zip((p.detach(), st["exp_avg"], st["exp_avg_sq"]), want, (p0, m0, v0), "pmv"):
                if rows.any():
                    e = _relerr(got[rows], w[rows], old[rows])
                    assert e < 1e-6, (name, what, e)
                assert torch.equal(got[~rows], old[~rows]), (name, what, "an invisible row changed")


@pytest.mark.parametrize("P", [4097, 100_003])
def test_all_true_mask_and_dense_groups_equal_the_dense_step_bitwise(P, built_lib):
    gen = torch.Generator().manual_seed(P)
    opt_s, opt_d = _optimizer(P, torch.Generator().manual_seed(5)), _optimizer(P, torch.Generator().manual_seed(5))
    for it in range(4):
        mask = (torch.ones(P, dtype=torch.bool) if it % 2 == 0 else torch.rand(P, generator=gen) < 0.3).to(DEV)
        g_gen = torch.Generator().manual_seed(100 + it)
        _grads(opt_s, g_gen)
        for (_, a), (_, b) in zip(_params(opt_s), _params(opt_d)):
            b.grad = a.grad.clone()
        opt_s.step(visibility=mask)
        opt_d.step()
        for (name, a), (_, b) in zip(_params(opt_s), _params(opt_d)):
            sa, sb = opt_s.state[a], opt_d.state[b]
            if it % 2 == 0 or name not in ROW_SHAPES:
                for x, y in ((a, b), (sa["exp_avg"], sb["exp_avg"]), (sa["exp_avg_sq"], sb["exp_avg_sq"])):
                    assert torch.equal(x, y), (it, name)
        # re-align the per-Gaussian rows after a partial step so every all-true step starts from the same state
        for (_, a), (_, b) in zip(_params(opt_s), _params(opt_d)):
            with torch.no_grad():
                a.copy_(b)
            for k in ("exp_avg", "exp_avg_sq"):
                opt_s.state[a][k].copy_(opt_d.state[b][k])


def test_misaligned_views_take_the_scalar_path(built_lib):
    P = 9_001
    gen = torch.Generator().manual_seed(11)
    opt = _optimizer(P, gen, offset=1)
    assert all(p.data_ptr() % 16 == 4 for n, p in _params(opt) if n in ROW_SHAPES)
    mask = (torch.rand(P, generator=gen) < 0.4).to(DEV)
    _grads(opt, gen, mask)
    before = _snapshot(opt)
    grads = {id(p): p.grad.clone() for _, p in _params(opt)}
    opt.step(visibility=mask)
    for name, p in _params(opt):
        if name not in ROW_SHAPES:
            continue
        p0, m0, v0, step0 = before[id(p)]
        group = next(g for g in opt.param_groups if g["name"] == name)
        want = adam_step(p0.double(), grads[id(p)].double(), m0.double(), v0.double(), step0 + 1, group["lr"], B1, B2,
                         EPS)
        for got, w, old in zip((p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"]), want, (p0, m0, v0)):
            assert _relerr(got[mask], w[mask], old[mask]) < 1e-6, name
            assert torch.equal(got[~mask], old[~mask]), name
    # all-true on a misaligned view equals the dense step on the same view bit for bit
    a, b = _optimizer(P, torch.Generator().manual_seed(3), offset=3), _optimizer(P, torch.Generator().manual_seed(3),
                                                                                 offset=3)
    _grads(a, torch.Generator().manual_seed(4))
    for (_, x), (_, y) in zip(_params(a), _params(b)):
        y.grad = x.grad.clone()
    a.step(visibility=torch.ones(P, dtype=torch.bool, device=DEV))
    b.step()
    for (_, x), (_, y) in zip(_params(a), _params(b)):
        assert torch.equal(x, y) and torch.equal(a.state[x]["exp_avg_sq"], b.state[y]["exp_avg_sq"])


def test_no_host_synchronisation_and_bitwise_repeatable(built_lib):
    P = 50_000
    runs = []
    for _ in range(2):
        gen = torch.Generator().manual_seed(21)
        opt = _optimizer(P, gen)
        masks = [(torch.rand(P, generator=gen) < 0.2).to(DEV) for _ in range(3)]
        for m in masks:
            _grads(opt, gen, m)
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode("error")
            try:
                opt.step(visibility=m)
            finally:
                torch.cuda.set_sync_debug_mode(0)
        runs.append([t.clone() for _, p in _params(opt) for t in (p.detach(), opt.state[p]["exp_avg"],
                                                                   opt.state[p]["exp_avg_sq"])])
    assert all(torch.equal(x, y) for x, y in zip(*runs))


# ---- GaussianModel -------------------------------------------------------------------------------------------------
def _model(P, seed=0):
    from ref_ext import ref_deform_args
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.deformation import deform_network
    from s3gaussian_b200.gaussian_model import GaussianModel, default_optimization_params
    cloud = syn.make_cloud(P, seed=seed)
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        net = deform_network(ref_deform_args(syn.DEFAULT_RESOLUTION, syn.DEFAULT_MULTIRES))
    g = GaussianModel(3, deformation=net).create_from_tensors(
        cloud.xyz.to(DEV), cloud.features_dc.to(DEV), cloud.features_rest.to(DEV), cloud.scaling.to(DEV),
        cloud.rotation.to(DEV), cloud.opacity.to(DEV))
    g.training_setup(default_optimization_params())
    return g


def _model_grads(g, gen, dense=True):
    from s3gaussian_b200.gaussian_model import PARAM_GROUPS
    for group in g.optimizer.param_groups:
        if group["name"] in PARAM_GROUPS or dense:
            for p in group["params"]:
                p.grad = (torch.randn(p.shape, generator=gen) * 0.1).to(DEV).contiguous(
                    memory_format=torch.channels_last if p.dim() == 4 and not p.is_contiguous() else
                    torch.contiguous_format)


def _per_gaussian(g):
    from s3gaussian_b200.gaussian_model import _ATTR, PARAM_GROUPS
    out = []
    for name in PARAM_GROUPS:
        p = getattr(g, _ATTR[name])
        st = g.optimizer.state.get(p, {})
        out.append((name, p, st))
    return out


def _dense(g):
    return [p for grp in g.optimizer.param_groups if grp["name"] in ("deformation", "grid") for p in grp["params"]]


def test_model_steps_compose_with_densify_prune_mcmc_and_sort(built_lib):
    P = 30_000
    gen = torch.Generator().manual_seed(7)
    g = _model(P)
    assert g.optimizer.selective_groups == {"xyz", "f_dc", "f_rest", "opacity", "scaling", "rotation"}
    for _ in range(2):
        _model_grads(g, gen)
        g.optimizer.step()
    mask = (torch.rand(P, generator=gen) < 0.25).to(DEV)
    _model_grads(g, gen)
    before = [(n, p.detach().clone(), st["exp_avg"].clone()) for n, p, st in _per_gaussian(g)]
    g.optimizer.step(visibility=mask)
    for (n, p, st), (_, p0, m0) in zip(_per_gaussian(g), before):
        assert torch.equal(p[~mask], p0[~mask]) and torch.equal(st["exp_avg"][~mask], m0[~mask]), n
        assert not torch.equal(p[mask], p0[mask]), n
    g.optimizer.zero_grad(set_to_none=True)

    def step_after_surgery(op):
        """The loop's order: backward, surgery, step with the render's (old) mask.  The new per-Gaussian tensors have no
        gradient, so only the dense groups move, exactly as step() would move them."""
        _model_grads(g, gen)
        old_mask = (torch.rand(g.get_xyz.shape[0], generator=gen) < 0.3).to(DEV)
        dense_grads = [p.grad.clone() for p in _dense(g)]
        op()
        rows = [(n, p.detach().clone()) for n, p, _ in _per_gaussian(g)]
        assert all(p.grad is None for _, p, _ in _per_gaussian(g))
        ref = [(p.detach().clone(), {k: v.clone() for k, v in g.optimizer.state[p].items()}) for p in _dense(g)]
        g.optimizer.step(visibility=old_mask)
        assert all(torch.equal(p, p0) for (_, p, _), (_, p0) in zip(_per_gaussian(g), rows))
        from s3gaussian_b200.optim import FusedAdam
        for p, (p0, st0), gr in zip(_dense(g), ref, dense_grads):
            q = torch.nn.Parameter(p0.clone())
            q.grad = gr
            o = FusedAdam([{"params": [q], "lr": next(grp["lr"] for grp in g.optimizer.param_groups
                                                       if any(x is p for x in grp["params"]))}], lr=0.0, eps=1e-15)
            o.state[q] = {k: v.clone() for k, v in st0.items()}
            o.step()
            assert torch.equal(q, p)
        g.optimizer.zero_grad(set_to_none=True)

    step_after_surgery(lambda: g.prune_points(torch.rand(g.get_xyz.shape[0], generator=gen).to(DEV) < 0.1))
    step_after_surgery(lambda: g.densify_and_clone(torch.rand(g.get_xyz.shape[0], 1, generator=gen).to(DEV), 0.9, 1e9))
    with torch.no_grad():
        g._opacity.data[:500] = -10.0        # some dead rows for relocate_gs
    step_after_surgery(lambda: g.relocate_gs(generator=torch.Generator(DEV).manual_seed(1)))
    step_after_surgery(lambda: g.add_new_gs(g.get_xyz.shape[0] + 700, generator=torch.Generator(DEV).manual_seed(2)))
    step_after_surgery(g.spatial_sort)
    # after the surgery, a selective step on the new rows
    P2 = g.get_xyz.shape[0]
    mask = (torch.rand(P2, generator=gen) < 0.5).to(DEV)
    _model_grads(g, gen)
    before = [(n, p.detach().clone()) for n, p, _ in _per_gaussian(g)]
    g.optimizer.step(visibility=mask)
    for (n, p, _), (_, p0) in zip(_per_gaussian(g), before):
        assert torch.equal(p[~mask], p0[~mask]) and not torch.equal(p[mask], p0[mask]), n


def test_capture_restore_round_trip(built_lib):
    from s3gaussian_b200.gaussian_model import GaussianModel, default_optimization_params
    P = 20_000
    gen = torch.Generator().manual_seed(9)
    g = _model(P)
    masks = [(torch.rand(P, generator=gen) < 0.3).to(DEV) for _ in range(4)]
    for m in masks[:2]:
        _model_grads(g, gen)
        g.optimizer.step(visibility=m)
    buf = io.BytesIO()
    torch.save((g.capture(), 2), buf)        # train.py's checkpoint, so the two models share no tensor
    buf.seek(0)
    tup, _ = torch.load(buf, weights_only=False)
    assert isinstance(tup[12], dict) and set(tup[12]) == {"state", "param_groups"}
    h = GaussianModel(3, deformation=_model(P)._deformation)
    h.restore(tup, default_optimization_params())
    assert h.optimizer.selective_groups == g.optimizer.selective_groups
    for m in masks[2:]:
        seed = int(torch.randint(1 << 30, (1,), generator=gen))
        _model_grads(g, torch.Generator().manual_seed(seed))
        _model_grads(h, torch.Generator().manual_seed(seed))
        g.optimizer.step(visibility=m)
        h.optimizer.step(visibility=m)
    for (n, a, sa), (_, b, sb) in zip(_per_gaussian(g), _per_gaussian(h)):
        assert torch.equal(a, b) and torch.equal(sa["exp_avg"], sb["exp_avg"]) and int(sa["step"]) == int(sb["step"]), n


@pytest.mark.parametrize("fine", [False, True])
def test_train_loop_with_sparse_adam(fine):
    cmd = [sys.executable, os.path.join(ROOT, "examples", "train_loop.py"), "--points", "20000", "--iters", "200",
           "--width", "480", "--height", "320", "--sparse-adam"] + (["--fine"] if fine else [])
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    rows = [(int(m.group(1)), float(m.group(2))) for m in re.finditer(r"iter\s+(\d+)\s+loss ([\d.]+)", r.stdout)]
    assert [it for it, _ in rows] == [50, 100, 150, 200], r.stdout
    assert rows[-1][1] < rows[0][1], rows
