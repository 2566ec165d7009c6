"""Generate tests/golden/train_*.npz from the REAL reference code (CPU, build container).

  loss cases : utils/loss_utils.py of /root/reference imported as it is (l1_loss, ssim, compute_depth),
               composed as train.py:395-419 does, gradients from autograd.
  adam case  : the optimizer the reference constructs (scene/gaussian_model.py:176-189): torch.optim.Adam
               with its eight named groups, lr=0.0 default, eps=1e-15, stepped three times.
  reg case   : GaussianModel.compute_regulation + its three helpers (scene/gaussian_model.py:710-749) and
               compute_plane_smoothness (scene/regulation.py:22-28), all extracted with ast and run as they are.
  stats case : the two statements of train.py:489-491 executed verbatim around the reference's own
               GaussianModel.add_densification_stats, whose source is extracted from
               scene/gaussian_model.py with ast (the module itself needs simple_knn/open3d to import).

np.savez_compressed stamps each member with the time of writing, so a rerun changes the bytes of files whose values
are unchanged: to add a case, pass a scratch directory as the argument and copy only the new case's file into
tests/golden.
"""
import ast
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("REF", "/root/reference")
sys.path.insert(0, ROOT)
import numpy as np
import torch

LOSS_CASES = [
    # name, B, C, H, W, seed
    ("ragged", 1, 3, 37, 53, 11),
    ("batch2", 2, 3, 64, 96, 12),
    ("tiny", 1, 3, 7, 9, 13),          # smaller than the 11x11 window
    ("tile_edges", 1, 3, 65, 33, 14),  # one pixel past a 32x32 tile in both directions
    ("gray", 1, 1, 23, 29, 15),        # C = 1: one plane per image
    ("c4_batch3", 3, 4, 19, 35, 16),   # C = 4, B = 3: 12 planes
    ("window", 1, 3, 11, 11, 17),      # exactly the 11x11 window
    ("row", 1, 3, 1, 40, 18),          # a single row: every window tap but the centre row is padding
    ("tile_cross", 2, 3, 33, 97, 19),  # past one tile vertically and two horizontally, 6 planes
]


def import_loss_utils():
    m = types.ModuleType("utils")
    m.__path__ = [f"{REF}/utils"]
    sys.modules["utils"] = m
    from utils import loss_utils
    return loss_utils


def loss_inputs(B, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(B, C, H, W, generator=g)
    # smooth-ish prediction: gt blurred a little + noise, clipped like a rendered image
    img = (gt + 0.15 * torch.randn(B, C, H, W, generator=g)).clamp(0, 1.2)
    gt_depth = torch.rand(B, H, W, generator=g) * 100.0          # some > max_depth (invalid)
    gt_depth[torch.rand(B, H, W, generator=g) < 0.2] = 0.0       # sparse lidar: holes
    depth = (gt_depth + 5.0 * torch.randn(B, H, W, generator=g)).abs()
    depth[torch.rand(B, H, W, generator=g) < 0.05] = 95.0        # beyond the clamp
    return img, gt, depth.unsqueeze(1), gt_depth.unsqueeze(1)


def make_loss(outdir, lu):
    for name, B, C, H, W, seed in LOSS_CASES:
        img, gt, depth, gt_depth = loss_inputs(B, C, H, W, seed)
        img.requires_grad_(True)
        depth.requires_grad_(True)
        l1 = lu.l1_loss(img, gt)
        ss = lu.ssim(img, gt)
        dl2 = lu.compute_depth("l2", depth, gt_depth)
        loss = l1 + 0.5 * dl2 + 0.2 * (1.0 - ss)
        loss.backward()
        np.savez_compressed(os.path.join(outdir, f"train_loss_{name}.npz"), dims=np.array([B, C, H, W]), seed=seed,
                            l1=l1.item(), ssim=ss.item(), depth_l2=dl2.item(), loss=loss.item(),
                            g_image=img.grad.numpy(), g_depth=depth.grad.numpy())
        print(name, l1.item(), ss.item(), dl2.item())


ADAM_SHAPES = [("xyz", (300, 3), 1.6e-4), ("deformation", (64, 128), 1.6e-5), ("deformation", (64,), 1.6e-5),
               ("grid", (1, 32, 9, 16), 1.6e-3), ("f_dc", (300, 1, 3), 0.0025), ("f_rest", (300, 15, 3), 0.0025 / 20),
               ("opacity", (300, 1), 0.05), ("scaling", (300, 3), 0.005), ("rotation", (300, 4), 0.001),
               ("odd", (4099,), 0.01), ("nograd", (10,), 0.01)]


def adam_inputs(seed=21, steps=3):
    g = torch.Generator().manual_seed(seed)
    params = [torch.randn(*s, generator=g) for _, s, _ in ADAM_SHAPES]
    grads = [[torch.randn(*s, generator=g) * (10.0 ** float(torch.randint(-6, 1, (1,), generator=g)))
              for _, s, _ in ADAM_SHAPES] for _ in range(steps)]
    return params, grads


def make_adam(outdir):
    params, grads = adam_inputs()
    ps = [torch.nn.Parameter(p.clone()) for p in params]
    groups = {}
    for (name, _, lr), p in zip(ADAM_SHAPES, ps):
        groups.setdefault(name, {"params": [], "lr": lr, "name": name})["params"].append(p)
    opt = torch.optim.Adam(list(groups.values()), lr=0.0, eps=1e-15)
    out = {}
    for s, gs in enumerate(grads):
        for (name, _, _), p, g in zip(ADAM_SHAPES, ps, gs):
            p.grad = None if name == "nograd" else g.clone()
        if s == 2:      # a learning-rate change between steps, as update_learning_rate does
            for gr in opt.param_groups:
                if gr["name"] == "xyz":
                    gr["lr"] = 1.0e-4
        opt.step()
        for i, p in enumerate(ps):
            out[f"p{i}_s{s}"] = p.detach().numpy().copy()
    for i, p in enumerate(ps):
        st = opt.state.get(p, {})
        if st:
            out[f"m{i}"] = st["exp_avg"].numpy().copy()
            out[f"v{i}"] = st["exp_avg_sq"].numpy().copy()
    np.savez_compressed(os.path.join(outdir, "train_adam.npz"), seed=21, steps=3, **out)
    print("adam ok")


def reference_method(name, file="scene/gaussian_model.py", ns=None):
    src = open(f"{REF}/{file}").read()
    for node in ast.walk(ast.parse(src)):
        if isinstance(node, ast.FunctionDef) and node.name == name:
            mod = ast.Module(body=[node], type_ignores=[])
            ns = {"torch": torch} if ns is None else ns
            exec(compile(mod, f"{REF}/{file}", "exec"), ns)
            return ns[name]
    raise KeyError(name)


def reg_inputs(seed=41, resolution=(8, 6, 5, 7), multires=(1, 2), channels=32):
    """planes shaped like init_grid_param (scene/hexplane.py:48-70): [1,C,reso[b],reso[a]] per comb (a,b)."""
    import itertools
    g = torch.Generator().manual_seed(seed)
    levels = []
    for m in multires:
        reso = [r * m for r in resolution[:3]] + [resolution[3]]
        planes = []
        for ca, cb in itertools.combinations(range(4), 2):
            t = torch.rand(1, channels, reso[cb], reso[ca], generator=g) * 0.8 + 0.6      # straddles 1 for the L1 sign
            planes.append(t)
        levels.append(planes)
    return levels


def make_reg(outdir):
    ns = {"torch": torch}
    reference_method("compute_plane_smoothness", "scene/regulation.py", ns)
    for m in ("_plane_regulation", "_time_regulation", "_l1_regulation", "compute_regulation"):
        reference_method(m, ns=ns)
    levels = [[p.clone().requires_grad_(True) for p in lv] for lv in reg_inputs()]
    model = types.SimpleNamespace()
    model._deformation = types.SimpleNamespace(deformation_net=types.SimpleNamespace(grid=types.SimpleNamespace(grids=levels)))
    for m in ("_plane_regulation", "_time_regulation", "_l1_regulation"):
        setattr(model, m, types.MethodType(ns[m], model))
    total = ns["compute_regulation"](model, 0.01, 0.0001, 0.0001)       # arguments/__init__.py:213-215 defaults
    total.backward()
    out = {f"g{l}_{k}": p.grad.numpy() for l, lv in enumerate(levels) for k, p in enumerate(lv)}
    np.savez_compressed(os.path.join(outdir, "train_plane_reg.npz"), seed=41, total=total.item(), **out)
    print("reg", total.item())


def stats_inputs(P=5000, seed=31):
    g = torch.Generator().manual_seed(seed)
    radii = torch.randint(-1, 40, (P,), generator=g, dtype=torch.int32).clamp_min(0)
    vgrad = torch.randn(P, 3, generator=g) * 1e-3
    accum = torch.rand(P, 1, generator=g)
    denom = torch.randint(0, 5, (P, 1), generator=g).float()
    max_radii = torch.randint(0, 30, (P,), generator=g).float()
    return radii, vgrad, accum, denom, max_radii


def make_stats(outdir):
    add = reference_method("add_densification_stats")
    radii, vgrad, accum, denom, max_radii = stats_inputs()
    gaussians = types.SimpleNamespace(xyz_gradient_accum=accum.clone(), denom=denom.clone(), max_radii2D=max_radii.clone())
    visibility_filter = radii > 0
    viewspace_point_tensor_grad = vgrad
    # train.py:490-491, verbatim
    gaussians.max_radii2D[visibility_filter] = torch.max(gaussians.max_radii2D[visibility_filter], radii[visibility_filter])
    add(gaussians, viewspace_point_tensor_grad, visibility_filter)
    np.savez_compressed(os.path.join(outdir, "train_densify_stats.npz"), seed=31, P=5000,
                        accum=gaussians.xyz_gradient_accum.numpy(), denom=gaussians.denom.numpy(),
                        max_radii2D=gaussians.max_radii2D.numpy())
    print("stats ok")


if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden")
    os.makedirs(out, exist_ok=True)
    make_loss(out, import_loss_utils())
    make_adam(out)
    make_stats(out)
    make_reg(out)
