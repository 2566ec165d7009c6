"""Developer check (gpurun): fused deformation forward/backward vs the golden vectors of the real reference."""
import os, sys, glob, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
from argparse import Namespace
from s3gaussian_b200 import synthetic as syn
from s3gaussian_b200.deformation import deform_network
from test_oracle_deform import load_deform_case, rel

def make_args(reso, multires, **flags):
    d = dict(net_width=64, timebase_pe=4, defor_depth=1, posebase_pe=10, scale_rotation_pe=2, opacity_pe=2,
             timenet_width=64, timenet_output=32, bounds=1.6,
             kplanes_config={"grid_dimensions": 2, "input_coordinate_dim": 4, "output_coordinate_dim": 32, "resolution": list(reso)},
             multires=list(multires), no_dx=False, no_grid=False, no_ds=True, no_dr=True, no_do=True, no_dshs=False,
             feat_head=True, empty_voxel=False, grid_pe=0, static_mlp=False, apply_rotation=False)
    d.update(flags); return Namespace(**d)

dev = torch.device("cuda:0")
do_bwd = "--bwd" in sys.argv
for path in ([] if "--notest" in sys.argv else sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "deform_*.npz")))):
    z, st, flags = load_deform_case(path)
    net = deform_network(make_args([int(v) for v in z["resolution"]], [int(v) for v in z["multires"]], **flags))
    net.deformation_net.set_aabb(*[list(a) for a in syn.WAYMO_AABB])
    missing, unexpected = net.load_state_dict(st, strict=False)
    assert not unexpected, unexpected
    net = net.to(dev)
    for li, gp in enumerate(net.deformation_net.grid.grids):
        for p in gp: assert p.is_contiguous(memory_format=torch.channels_last)
    T = lambda k: torch.from_numpy(z[k]).to(dev).requires_grad_(do_bwd)
    xyz, sc, ro, op, shs = T("in_xyz"), T("in_scales"), T("in_rot"), T("in_opacity"), T("in_shs")
    campos = torch.from_numpy(z["campos"]).to(dev)
    outs = net.render_front(xyz, sc, ro, op, shs, float(z["time"]), campos, 3)
    torch.cuda.synchronize()
    names = ("out_means3D", "out_scales", "out_rot", "out_opacity", "out_colors", "out_dx", "out_dshs", "out_feat")
    print(os.path.basename(path), " ".join(f"{n[4:]}={rel(o.detach().cpu().numpy().reshape(z[n].shape), z[n]):.1e}" for o, n in zip(outs, names)))
    if do_bwd:
        order = (0, 1, 2, 3, 4, 5, 7, 6)   # golden weights w0..w7 follow (m3, sc, ro, op, colors, dx, feat, dshs)
        ws = [torch.from_numpy(z[f"w{i}"]).to(dev) for i in range(8)]
        o_by = dict(zip(("m3", "sc", "ro", "op", "col", "dx", "dshs", "feat"), outs))
        loss = sum((o_by[k] * w.reshape(o_by[k].shape)).sum() for k, w in zip(("m3", "sc", "ro", "op", "col", "dx", "feat", "dshs"), ws))
        loss.backward(); torch.cuda.synchronize()
        msg = []
        for leaf, n in zip((xyz, sc, ro, op, shs), ("g_xyz", "g_scales", "g_rot", "g_opacity", "g_shs")):
            msg.append(f"{n}={rel(leaf.grad.cpu().numpy(), z[n]):.1e}")
        worst = 0; cnt = 0
        for k, p in net.named_parameters():
            key = "pg_" + k
            if key in z.files and p.grad is not None:
                e = rel(p.grad.cpu().numpy(), z[key]); worst = max(worst, e); cnt += 1
                if e > 1e-4: msg.append(f"{k}={e:.1e}")
            elif key + "_sum" in z.files and p.grad is not None:
                gf = p.grad.reshape(-1).double()
                e = abs(float(gf.sum()) - float(z[key + "_sum"])) / (abs(float(z[key + "_abs"])) + 1e-30)
                e2 = rel(p.grad.reshape(-1)[::997].cpu().numpy(), z[key + "_sample"])
                worst = max(worst, e2); cnt += 1
                if e2 > 1e-4 or e > 1e-4: msg.append(f"{k}: sum {e:.1e} sample {e2:.1e}")
        print("   bwd:", " ".join(msg), f"| {cnt} param grads, worst {worst:.1e}")
# timing at 2M with the default config
if "--time" in sys.argv:
    P = int(os.environ.get("DEV_P", 2_000_000))
    st = syn.make_deform_state(0, weight_scale=0.2)
    net = deform_network(make_args(syn.DEFAULT_RESOLUTION, syn.DEFAULT_MULTIRES)); net.deformation_net.set_aabb(*[list(a) for a in syn.WAYMO_AABB])
    net.load_state_dict(st, strict=False); net = net.to(dev)
    cloud = syn.make_cloud(P, seed=0).to(dev)
    args = [cloud.xyz.requires_grad_(do_bwd), cloud.scaling.requires_grad_(do_bwd), cloud.rotation.requires_grad_(do_bwd), cloud.opacity.requires_grad_(do_bwd), cloud.get_features().detach().requires_grad_(do_bwd)]
    campos = torch.tensor([0., 0., 2.], device=dev)
    def step():
        outs = net.render_front(*args, 0.37, campos, 3)
        if do_bwd:
            torch.autograd.backward(list(outs), [torch.ones_like(o) for o in outs])
    for _ in range(3): step()
    torch.cuda.synchronize(); e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10): step()
    e1.record(); torch.cuda.synchronize()
    print(f"deform {'fwd+bwd' if do_bwd else 'fwd'} at P={P}: {e0.elapsed_time(e1)/10:.3f} ms")
