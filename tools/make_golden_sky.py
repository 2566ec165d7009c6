"""Generate tests/golden/sky_*.npz (described in tests/golden/SKY.md) by importing the REAL reference sky model.

Runs on the CPU: scene/background_model.py and scene/encodings.py of the reference are imported as they are, with
stand-ins only for the modules that cannot load here (simple_knn._C, plyfile, matplotlib, open3d,
scene.gaussian_model; the
`scene` / `utils` package __init__s are bypassed by registering bare package objects).  Background_Model builds its
pixel grid on "cuda", so the file's forward is restated from the reference's own pieces: get_directions over the
same row-major pixel coordinates, then SkyModel and the sigmoid, exactly as Background_Model.forward runs them.

Each file stores the seeds, the camera, the seeded weights (not nn.Linear's initialisation: every tensor is
redrawn), the seeded dL/dsky (0.5 + N(0, 1)) and the reference's float32 output and parameter gradients.

    python tools/make_golden_sky.py [OUTDIR]
"""
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("REF", "/root/reference")
import numpy as np
import torch


def import_reference():
    for name in ("scene", "utils"):
        m = types.ModuleType(name)
        m.__path__ = [f"{REF}/{name}"]
        sys.modules[name] = m
    knn = types.ModuleType("simple_knn")
    knn.__path__ = []
    knn_c = types.ModuleType("simple_knn._C")
    knn_c.distCUDA2 = None
    sys.modules["simple_knn"], sys.modules["simple_knn._C"] = knn, knn_c
    ply = types.ModuleType("plyfile")
    ply.PlyData = ply.PlyElement = None
    sys.modules["plyfile"] = ply
    sys.modules["open3d"] = types.ModuleType("open3d")     # utils/general_utils.py imports it at module level
    mpl = types.ModuleType("matplotlib")
    mpl.__path__ = []
    sys.modules["matplotlib"] = mpl
    sys.modules["matplotlib.pyplot"] = types.ModuleType("matplotlib.pyplot")
    gm = types.ModuleType("scene.gaussian_model")
    gm.GaussianModel = type("GaussianModel", (torch.nn.Module,), {})
    sys.modules["scene.gaussian_model"] = gm
    import scene.background_model as bm
    return bm


def rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


CASES = [
    # name, width, H, W, seed, rotation angles, (fx, fy, cx, cy)
    ("w64_ragged", 64, 23, 37, 1, (0.3, -0.7, 1.1), (30.0, 41.0, 15.2, 13.7)),
    ("w256_ragged", 256, 23, 37, 2, (-1.2, 0.4, 2.5), (25.0, 19.0, 21.0, 9.5)),
    ("w64_larger", 64, 80, 120, 3, (0.1, 1.3, -0.4), (95.0, 110.0, 52.0, 44.0)),
    ("w256_larger", 256, 80, 120, 4, (2.0, -0.2, 0.6), (70.0, 64.0, 66.5, 35.0)),
]


def make_case(bm, width, H, W, seed, angles, intr):
    g = torch.Generator().manual_seed(seed)
    model = bm.SkyModel({"mlp_width": width})
    with torch.no_grad():
        for p in model.sky_head.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * (1.5 / np.sqrt(p.shape[-1])) if p.dim() == 2 else
                    torch.randn(p.shape, generator=g) * 0.2)
    c2w = np.eye(4, dtype=np.float32)
    c2w[:3, :3] = rot(*angles)
    c2w[:3, 3] = torch.randn(3, generator=g).numpy()
    fx, fy, cx, cy = intr
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], dtype=np.float32)
    # a loss gradient with a mean, as a photometric loss has (a zero-mean one cancels the weight gradients down to the
    # few pixels whose ReLU decision is within float32 rounding of its kink)
    gsky = 0.5 + torch.randn(3, H, W, generator=g)
    # Background_Model.pixel_coord / get_ray_directions / forward, on the CPU
    x = torch.arange(0, W, dtype=torch.float32).long()
    y = torch.arange(0, H, dtype=torch.float32).long()
    pc = torch.stack(torch.meshgrid(x, y, indexing="xy")).float()
    v = bm.get_directions(pc[0].flatten(), pc[1].flatten(), torch.from_numpy(c2w), torch.from_numpy(K))
    sky = torch.sigmoid(model(v.reshape(H, W, 3))).permute(2, 0, 1)
    (sky * gsky).sum().backward()
    out = dict(width=width, H=H, W=W, seed=seed, c2w=c2w, intrinsic=K, dL_dsky=gsky.numpy(),
               sky=sky.detach().numpy())
    for i in range(3):
        lay = model.sky_head.layers[i]
        out[f"w{i}"], out[f"b{i}"] = lay.weight.detach().numpy(), lay.bias.detach().numpy()
        out[f"grad_w{i}"], out[f"grad_b{i}"] = lay.weight.grad.numpy(), lay.bias.grad.numpy()
    return out


def main(outdir):
    os.makedirs(outdir, exist_ok=True)
    bm = import_reference()
    for name, width, H, W, seed, angles, intr in CASES:
        d = make_case(bm, width, H, W, seed, angles, intr)
        np.savez_compressed(os.path.join(outdir, f"sky_{name}.npz"), **d)
        print(name, {k: v.shape for k, v in d.items() if hasattr(v, "shape")})


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden"))
