"""GPU: 3DGS-MCMC's densification (s3g_mcmc_relocate / s3g_mcmc_noise, mcmc.py, GaussianModel.relocate_gs /
add_new_gs / inject_noise, examples/train_loop.py --mcmc-cap).

1. The relocation kernel against the float64 restatement (tests/mcmc_ref.py): ratios 1..60 and opacities from 0.005 to
   1 - 2^-23, rows drawn up to 100 times; opacity and scales to 1e-6 relative, every other value bitwise.
2. relocate_gs / add_new_gs on a model after real Adam steps, against the bookkeeping of the restatement given the same
   draws: parameters, moments, accumulators, filter_3D, _deformation_table, the optimizer's Parameters, the budget,
   zero-width f_rest, the no-dead and all-dead cases, and two runs from one seed.
3. The noise kernel against the restatement for a given eps.
4. What relocation is for: a Gaussian and its N co-located relocated copies give the same alpha through the rasterizer.
5. examples/train_loop.py --mcmc-cap end to end.
"""
import math
import os
import re
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch

import mcmc_ref as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def mc(built_lib):
    from s3gaussian_b200 import mcmc
    return mcmc


def _logit(o):
    o = torch.as_tensor(o, dtype=torch.float64)
    return torch.log(o) - torch.log1p(-o)


def _opacity_grid(n, gen):
    """n opacities spread from 0.005 to 1 - 2^-23: uniform in logit, plus the two ends."""
    x = torch.rand(n, generator=gen, dtype=torch.float64) * float(_logit(ref.O_MAX) - _logit(0.005)) + float(_logit(0.005))
    x[:2] = torch.tensor([float(_logit(0.005)), float(_logit(ref.O_MAX))])
    return x.float()


def _check_relocated(opacity, scaling, rows, raw_o, raw_s, ratio, what):
    o_want, s_want = ref.relocate_rows64(raw_o, raw_s, ratio)
    o_got = torch.sigmoid(opacity[rows].double().reshape(-1))
    s_got = torch.exp(scaling[rows].double())
    torch.testing.assert_close(o_got, o_want, rtol=1e-6, atol=0, msg=lambda m: f"{what} opacity: {m}")
    torch.testing.assert_close(s_got, s_want, rtol=1e-6, atol=0, msg=lambda m: f"{what} scales: {m}")


# ---- 1. the kernel ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["ratio_1_to_60", "drawn_up_to_100"])
def test_relocate_kernel_against_the_restatement(layout, mc):
    gen = torch.Generator().manual_seed(3)
    if layout == "ratio_1_to_60":      # each source once, the ratio given freely
        n_src = 3000
        src = torch.arange(n_src)
        ratio = torch.arange(n_src) % 60 + 1
    else:                              # source k drawn k times, k = 1..100: its ratio is k + 1
        n_src = 100
        src = torch.arange(n_src).repeat_interleave(torch.arange(1, n_src + 1))
        ratio = torch.bincount(src, minlength=n_src)[src] + 1
    n = src.numel()
    P = n_src + n + 500                # sources, then destinations, then rows nobody touches
    dst = torch.arange(n_src, n_src + n)
    raw_o = torch.empty(P, 1)
    raw_o[:, 0] = _opacity_grid(P, gen)
    raw_s = torch.rand(P, 3, generator=gen) * 6 - 5
    raw_o[dst], raw_s[dst] = raw_o[src], raw_s[src]          # the caller's row copy
    moments = [torch.randn(P, w, generator=gen) for w in (3, 1, 48)]
    accs = [torch.rand(P, 1, generator=gen), torch.rand(P, generator=gen), torch.rand(P, 3, generator=gen)]
    t = {k: v.to(DEV) for k, v in dict(o=raw_o, s=raw_s).items()}
    m_dev = [m.to(DEV) for m in moments]
    a_dev = [a.to(DEV) for a in accs]
    mc.relocate(t["o"], t["s"], src.to(DEV), dst.to(DEV), ratio.to(DEV), 0.005,
                [(m, True) for m in m_dev] + [(a, False) for a in a_dev])
    o, s = t["o"].cpu(), t["s"].cpu()
    _check_relocated(o, s, dst, raw_o[src], raw_s[src], ratio, "dst")
    assert torch.equal(o[src], o[dst]) and torch.equal(s[src], s[dst])
    untouched = torch.arange(n_src + n, P)
    assert torch.equal(o[untouched], raw_o[untouched]) and torch.equal(s[untouched], raw_s[untouched])
    both = torch.cat((src.unique(), dst))
    rest = torch.ones(P, dtype=torch.bool)
    rest[both] = False
    for m, m0 in zip(m_dev, moments):
        m = m.cpu()
        assert bool((m[both] == 0).all()) and torch.equal(m[rest], m0[rest])
    rest_acc = torch.ones(P, dtype=torch.bool)
    rest_acc[dst] = False
    for a, a0 in zip(a_dev, accs):
        a = a.cpu()
        assert bool((a[dst] == 0).all()) and torch.equal(a[rest_acc], a0[rest_acc])
    # N = 1 keeps the raw values bitwise (no clamp inside (0.005, 1 - 2^-23))
    if layout == "ratio_1_to_60":
        one = ratio == 1
        inside = one & (torch.sigmoid(raw_o[src, 0].double()) > 0.005) & (torch.sigmoid(raw_o[src, 0].double()) < ref.O_MAX)
        assert int(inside.sum()) > 0
        assert torch.equal(o[dst[inside]], raw_o[src[inside]]) and torch.equal(s[dst[inside]], raw_s[src[inside]])


def test_relocate_kernel_with_n_zero_and_repeat_calls(mc):
    """No descriptors; the same inputs give bitwise equal results."""
    gen = torch.Generator().manual_seed(8)
    raw_o = _opacity_grid(64, gen)[:, None].to(DEV)
    raw_s = (torch.rand(64, 3, generator=gen) - 2).to(DEV)
    src, dst = torch.arange(32, device=DEV), torch.arange(32, 64, device=DEV)
    raw_o[32:], raw_s[32:] = raw_o[:32], raw_s[:32]
    outs = []
    for _ in range(2):
        o, s = raw_o.clone(), raw_s.clone()
        mc.relocate(o, s, src, dst, torch.full((32,), 7, device=DEV), 0.005)
        outs.append((o, s))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    _check_relocated(outs[0][0].cpu(), outs[0][1].cpu(), dst.cpu(), raw_o[:32].cpu(), raw_s[:32].cpu(),
                     torch.full((32,), 7), "n_zero = 0")


# ---- 2. the model -----------------------------------------------------------------------------------------------------
def _trained_model(P=6000, sh_degree=3, seed=5, dead_frac=0.05, fine=True):
    """A model after three FusedAdam steps on seeded gradients, every per-Gaussian side tensor filled, and about
    `dead_frac` of the rows at opacity 0.001-0.005."""
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_model import GaussianModel, default_optimization_params
    gen = torch.Generator().manual_seed(seed)
    cloud = syn.make_cloud(P, seed=seed)
    K = (sh_degree + 1) ** 2 - 1
    net = None
    if fine:
        from ref_ext import ref_deform_args
        from s3gaussian_b200.deformation import deform_network
        with torch.random.fork_rng(devices=[]):
            torch.manual_seed(seed)
            net = deform_network(ref_deform_args(syn.DEFAULT_RESOLUTION, syn.DEFAULT_MULTIRES))
    g = GaussianModel(sh_degree, deformation=net).create_from_tensors(
        cloud.xyz.to(DEV), cloud.features_dc.to(DEV), cloud.features_rest[:, :K].contiguous().to(DEV),
        cloud.scaling.to(DEV), cloud.rotation.to(DEV), cloud.opacity.to(DEV))
    g.training_setup(default_optimization_params())
    for _ in range(3):
        for name in ("_xyz", "_features_dc", "_features_rest", "_opacity", "_scaling", "_rotation"):
            p = getattr(g, name)
            if p.numel():        # zero-width f_rest gets no gradient and so no Adam state
                p.grad = (torch.randn(p.shape, generator=gen) * 0.1).to(DEV)
        g.optimizer.step()
        g.optimizer.zero_grad(set_to_none=True)
    with torch.no_grad():
        dead = torch.rand(P, generator=gen) < dead_frac
        o = torch.rand(P, generator=gen) * 0.004 + 0.001
        g._opacity.data[dead.to(DEV), 0] = _logit(o[dead]).float().to(DEV)
    g.xyz_gradient_accum = torch.rand(P, 1, generator=gen).to(DEV)
    g.xyz_gradient_accum_abs = torch.rand(P, 1, generator=gen).to(DEV)
    g.denom = torch.randint(0, 9, (P, 1), generator=gen).float().to(DEV)
    g.max_radii2D = torch.rand(P, generator=gen).to(DEV) * 30
    g._deformation_accum = torch.rand(P, 3, generator=gen).to(DEV)
    g._deformation_table = (torch.rand(P, generator=gen) < 0.7).to(DEV)
    g.filter_3D = torch.rand(P, 1, generator=gen).to(DEV)
    return g


PARAMS = (("xyz", "_xyz"), ("f_dc", "_features_dc"), ("f_rest", "_features_rest"), ("opacity", "_opacity"),
          ("scaling", "_scaling"), ("rotation", "_rotation"))
ACCS = ("xyz_gradient_accum", "xyz_gradient_accum_abs", "denom", "max_radii2D", "_deformation_accum")


def _snapshot(g):
    snap = {"params": {n: getattr(g, a).detach().clone() for n, a in PARAMS},
            "param_objs": {n: getattr(g, a) for n, a in PARAMS},
            "acc": {a: getattr(g, a).clone() for a in ACCS},
            "table": g._deformation_table.clone(), "filter": g.filter_3D.clone()}
    snap["state"] = {}
    for n, a in PARAMS:
        st = g.optimizer.state.get(getattr(g, a))
        snap["state"][n] = (st["step"].clone(), st["exp_avg"].clone(), st["exp_avg_sq"].clone()) if st else None
    return snap


def _assert_unchanged(g, snap):
    for n, a in PARAMS:
        assert getattr(g, a) is snap["param_objs"][n] and torch.equal(getattr(g, a).detach(), snap["params"][n])
    for a in ACCS:
        assert torch.equal(getattr(g, a), snap["acc"][a])
    assert torch.equal(g._deformation_table, snap["table"]) and torch.equal(g.filter_3D, snap["filter"])


def _check_after(g, snap, idx, src, dst, ratio):
    """The model after the row copy `idx` and the relocation of the pairs (src, dst) with `ratio`."""
    idx, src, dst = idx.to(DEV), src.to(DEV), dst.to(DEV)
    P = idx.numel()
    touched = torch.zeros(P, dtype=torch.bool, device=DEV)
    touched[src] = touched[dst] = True
    relocated = torch.zeros(P, dtype=torch.bool, device=DEV)
    relocated[dst] = True
    for n, a in PARAMS:
        p = getattr(g, a)
        group = g._group(n)
        assert group["params"][0] is p and isinstance(p, torch.nn.Parameter) and p.requires_grad
        want = snap["params"][n][idx]
        if n in ("opacity", "scaling"):
            assert torch.equal(p.detach()[~touched], want[~touched])
        else:
            assert torch.equal(p.detach(), want), n
        st = g.optimizer.state.get(p)
        if snap["state"][n] is None:
            assert not st and p.numel() == 0, n
            continue
        step0, m0, v0 = snap["state"][n]
        assert torch.equal(st["step"], step0)
        for m, m_old in ((st["exp_avg"], m0), (st["exp_avg_sq"], v0)):
            assert m.shape == p.shape
            assert bool((m[touched] == 0).all()) and torch.equal(m[~touched], m_old[idx][~touched]), n
    _check_relocated(g._opacity.detach().cpu(), g._scaling.detach().cpu(), dst.cpu(),
                     snap["params"]["opacity"][src].cpu(), snap["params"]["scaling"][src].cpu(), ratio.cpu(), "model")
    assert torch.equal(g._opacity.detach()[src], g._opacity.detach()[dst])
    assert torch.equal(g._scaling.detach()[src], g._scaling.detach()[dst])
    for a in ACCS:
        t, want = getattr(g, a), snap["acc"][a][idx]
        assert t.shape == want.shape and bool((t[relocated] == 0).all()) and torch.equal(t[~relocated], want[~relocated]), a
    assert torch.equal(g._deformation_table, snap["table"][idx]) and torch.equal(g.filter_3D, snap["filter"][idx])


@pytest.mark.parametrize("sh_degree", [3, 0])
def test_relocate_gs(sh_degree, mc):
    g = _trained_model(sh_degree=sh_degree, fine=sh_degree == 3)
    assert g._features_rest.shape[1] == (0 if sh_degree == 0 else 15)
    snap = _snapshot(g)
    P = g.get_xyz.shape[0]
    o = torch.sigmoid(snap["params"]["opacity"][:, 0])
    alive = torch.nonzero(o > 0.005)[:, 0]
    drawn = alive[torch.multinomial(o[alive], int((o <= 0.005).sum()), replacement=True,
                                    generator=torch.Generator(DEV).manual_seed(17))]
    dead, idx, ratio = ref.plan_relocate(o, drawn)
    assert 0.03 * P < dead.numel() < 0.07 * P and int(ratio.max()) >= 3
    g.relocate_gs(generator=torch.Generator(DEV).manual_seed(17))
    assert g.get_xyz.shape[0] == P
    assert bool((o[drawn] > 0.005).all())                               # draws only from alive rows
    _check_after(g, snap, idx, drawn, dead, ratio)
    assert float(g.get_opacity.detach().min()) >= 0.005 * (1 - 1e-6)


@pytest.mark.parametrize("sh_degree", [3, 0])
def test_add_new_gs(sh_degree, mc):
    g = _trained_model(sh_degree=sh_degree, fine=sh_degree == 3)
    P = g.get_xyz.shape[0]
    for cap in (P, P - 10, 0):                                          # cap_max <= P: nothing happens
        snap = _snapshot(g)
        assert g.add_new_gs(cap) == 0
        _assert_unchanged(g, snap)
    for cap in (P + 7, 2 * P):
        P = g.get_xyz.shape[0]
        snap = _snapshot(g)
        o = torch.sigmoid(snap["params"]["opacity"][:, 0])
        n_want = max(P, min(cap, int(1.05 * P))) - P
        drawn = torch.multinomial(o, n_want, replacement=True, generator=torch.Generator(DEV).manual_seed(cap))
        n, idx, new, ratio = ref.plan_add(P, cap, drawn)
        assert g.add_new_gs(cap, generator=torch.Generator(DEV).manual_seed(cap)) == n == n_want
        assert g.get_xyz.shape[0] == max(P, min(cap, int(1.05 * P)))
        _check_after(g, snap, idx, drawn, new, ratio)


def test_nothing_dead_or_nothing_alive_does_nothing(mc):
    for frac, opacity in ((0.0, 0.3), (1.0, 0.004)):
        g = _trained_model(P=2000, dead_frac=frac, fine=False)
        if frac == 0.0:
            g._opacity.data.clamp_(min=float(_logit(0.01)))
        else:
            g._opacity.data.fill_(float(_logit(opacity)))
        snap = _snapshot(g)
        g.relocate_gs()
        _assert_unchanged(g, snap)


def test_two_runs_from_one_seed_are_bitwise_equal(mc):
    runs = []
    for _ in range(2):
        g = _trained_model(P=4000)
        g.relocate_gs(generator=torch.Generator(DEV).manual_seed(1))
        g.add_new_gs(10_000, generator=torch.Generator(DEV).manual_seed(2))
        g.inject_noise(1e-4, generator=torch.Generator(DEV).manual_seed(3))
        runs.append(_snapshot(g))
    a, b = runs
    for n, _ in PARAMS:
        assert torch.equal(a["params"][n], b["params"][n])
        for x, y in zip(a["state"][n], b["state"][n]):
            assert torch.equal(x, y)
    for k in ACCS:
        assert torch.equal(a["acc"][k], b["acc"][k])
    assert torch.equal(a["table"], b["table"]) and torch.equal(a["filter"], b["filter"])


def test_relocate_without_training_setup(mc):
    """A model that never called training_setup(): no moments to zero; the accumulators start at zero."""
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200.gaussian_model import GaussianModel
    cloud = syn.make_cloud(500, seed=1)
    g = GaussianModel(3).create_from_tensors(cloud.xyz.to(DEV), cloud.features_dc.to(DEV),
                                             cloud.features_rest.to(DEV), cloud.scaling.to(DEV),
                                             cloud.rotation.to(DEV), cloud.opacity.to(DEV))
    g._opacity.data[:50] = -8.0
    g.relocate_gs(generator=torch.Generator(DEV).manual_seed(0))
    assert g.get_xyz.shape[0] == 500 and float(g.get_opacity.detach().min()) >= 0.005 * (1 - 1e-6)
    assert g.add_new_gs(600, generator=torch.Generator(DEV).manual_seed(0)) == 25
    assert g.xyz_gradient_accum.shape == (525, 1) and float(g.xyz_gradient_accum.abs().max()) == 0


# ---- 3. the noise -----------------------------------------------------------------------------------------------------
def test_noise_against_the_restatement(mc):
    from s3gaussian_b200 import synthetic as syn
    gen = torch.Generator().manual_seed(21)
    P = 200_000
    cloud = syn.make_cloud(P, seed=4)
    xyz0 = cloud.xyz.clone()
    scaling, rotation = cloud.scaling.clone(), cloud.rotation.clone()
    opacity = _logit(torch.rand(P, 1, generator=gen, dtype=torch.float64) * 0.0199 + 1e-4).float()
    opacity[:1000] = float(_logit(0.99))                  # opaque: gate ~1e-43
    eps = torch.randn(P, 3, generator=gen)
    step = 1.6e-4 * 5e5
    xyz = xyz0.to(DEV)
    mc.inject_noise(xyz, scaling.to(DEV), rotation.to(DEV), opacity.to(DEV), step, eps.to(DEV))
    got = xyz.cpu().double()
    d = ref.noise64(scaling, rotation, opacity, step, eps)
    want = xyz0.double() + d
    # the floor: one float32 rounding of the sum, and 2^-18 (64 float32 roundings) of the largest term of Sigma eps,
    # which the float32 products R^T eps, s^2 (.) and R (.) can lose to cancellation in a small component
    o = torch.sigmoid(opacity.double())
    gate = 1.0 / (1.0 + torch.exp(-100.0 * ((1.0 - o) - 0.995)))
    full = step * torch.exp(2 * scaling.double()).max(1, keepdim=True).values * eps.double().norm(dim=1, keepdim=True)
    floor = 2.0 ** -23 * want.abs() + 2.0 ** -18 * gate * full
    err = (got - want).abs()
    assert bool((err <= 1e-5 * d.abs() + floor).all()), float((err / (1e-5 * d.abs() + floor)).max())
    assert float(gate[1000:].min()) > 0.1 and float(d[1000:].abs().max()) > 1e-3      # the low-opacity rows do move
    moved = (got - xyz0.double()).abs()
    assert bool((moved[:1000] <= 1e-30 * full[:1000]).all())      # o = 0.99: gate ~ 2e-43
    # through the model, eps drawn from the generator
    from s3gaussian_b200.gaussian_model import GaussianModel
    g = GaussianModel(3).create_from_tensors(xyz0.to(DEV), cloud.features_dc.to(DEV), cloud.features_rest.to(DEV),
                                             scaling.to(DEV), rotation.to(DEV), opacity.to(DEV))
    g.inject_noise(1.6e-4, generator=torch.Generator(DEV).manual_seed(9))
    eps2 = torch.randn((P, 3), device=DEV, generator=torch.Generator(DEV).manual_seed(9))
    xyz2 = xyz0.to(DEV)
    mc.inject_noise(xyz2, scaling.to(DEV), rotation.to(DEV), opacity.to(DEV), step, eps2)
    assert torch.equal(g.get_xyz.detach(), xyz2)


# ---- 4. what relocation is for ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("o", [0.05, 0.3, 0.6, 0.9])
def test_relocated_copies_keep_the_alpha_at_the_centre(o, mc):
    """A Gaussian whose mean projects onto a pixel centre, and N co-located copies with the relocated opacity and
    scales: alpha at that pixel is 1 - (1 - o')^N = o to 1e-5 (every copy's alpha stays in [1/255, 0.99)); N = 1 keeps
    the image bitwise."""
    from s3gaussian_b200 import synthetic as syn
    from s3gaussian_b200 import diff_gaussian_rasterization as ours
    from s3gaussian_b200.gaussian_renderer import raster_settings_for
    W = H = 33
    cam = syn.make_camera(W, H, (0.0, 0.0, 0.0), focal=40.0).to(DEV)
    centre = torch.tensor([[6.0, 0.0, 0.0]], device=DEV)        # on the optical axis: pixel (16, 16)
    pc = SimpleNamespace(get_xyz=centre, active_sh_degree=0)
    rs = raster_settings_for(cam, pc, SimpleNamespace(debug=False), torch.zeros(3, device=DEV))

    def alpha_of(raw_o, raw_s, N):
        means = centre.repeat(N, 1)
        with torch.no_grad():
            out = ours.GaussianRasterizer(rs).forward_opacity(
                means, torch.zeros_like(means), torch.sigmoid(raw_o), colors_precomp=torch.ones(N, 3, device=DEV),
                scales=torch.exp(raw_s), rotations=torch.tensor([[0.9, 0.1, -0.3, 0.2]], device=DEV).repeat(N, 1))
        return out[3][0], out[0]

    raw_o = _logit(torch.tensor([[o]])).float().to(DEV)
    raw_s = torch.tensor([[-1.2, -2.0, -1.6]], device=DEV)
    base, colour = alpha_of(raw_o, raw_s, 1)
    assert abs(float(base[16, 16]) - o) < 1e-5
    for N in (1, 2, 3, 8):
        # row 0 drawn, rows 1.. its copies (at N = 1 one spare row takes the copy and is not drawn)
        rows = max(N, 2)
        ro, rsc = raw_o.repeat(rows, 1).contiguous(), raw_s.repeat(rows, 1).contiguous()
        mc.relocate(ro, rsc, torch.zeros(rows - 1, dtype=torch.int64, device=DEV), torch.arange(1, rows, device=DEV),
                    torch.full((rows - 1,), N, device=DEV), 0.005)
        ro, rsc = ro[:N].contiguous(), rsc[:N].contiguous()
        op = float(torch.sigmoid(ro[0].double()))
        assert 1 / 255 <= op * 0.999 and op < 0.99
        alpha, img = alpha_of(ro, rsc, N)
        assert abs(float(alpha[16, 16]) - float(base[16, 16])) <= 1e-5, (N, float(alpha[16, 16]), float(base[16, 16]))
        if N == 1:
            assert torch.equal(ro, raw_o) and torch.equal(rsc, raw_s)
            assert torch.equal(alpha, base) and torch.equal(img, colour)


# ---- 5. the training loop ---------------------------------------------------------------------------------------------
def test_train_loop_with_mcmc_cap():
    cap = 22_500
    r = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_loop.py"), "--points", "20000",
                        "--iters", "300", "--width", "480", "--height", "320", "--mcmc-cap", str(cap)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    rows = [(int(m.group(1)), float(m.group(2)), int(m.group(3)))
            for m in re.finditer(r"iter\s+(\d+)\s+loss ([\d.]+).*points (\d+)", r.stdout)]
    assert [it for it, _, _ in rows] == [50, 100, 150, 200, 250, 300], r.stdout
    points = [p for _, _, p in rows]
    assert max(points) <= cap and points[-1] == cap and points[0] == 20_000, points
    assert rows[-1][1] < rows[0][1], rows
    bad = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_loop.py"), "--mcmc-cap", "10",
                          "--absgrad-threshold", "0.1"], capture_output=True, text=True, timeout=300)
    assert bad.returncode != 0 and "--absgrad-threshold" in bad.stderr
