"""A minimal S3Gaussian-style training loop on the H100 path: the control flow of the reference's
train.py (scene_reconstruction, train.py:330-530) with every heavy step running through libs3g_b200.so.

    python examples/train_loop.py [--points 200000] [--iters 300] [--fine] [--filter-3d] [--densify-until N]
                                 [--absgrad-threshold T | --mcmc-cap N] [--sparse-adam] [--bilateral-grid]
                                 [--sky]

Synthetic data (there is no dataset reader here): a random cloud initialised through create_from_pcd
(3-NN scales), targets rendered from a perturbed copy of it.  Needs a CUDA device (sm_90a).
"""
import argparse
import os
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from s3gaussian_b200 import losses, synthetic as syn
from s3gaussian_b200.gaussian_model import GaussianModel, default_optimization_params
from s3gaussian_b200.gaussian_renderer import PipelineParams, render


def sky_directions(c2w, K, H, W):
    """Unit world-space ray directions [3, H, W] of the pixel grid (the sky model's step 1), float32 torch."""
    y, x = torch.meshgrid(torch.arange(H, device=c2w.device, dtype=torch.float32),
                          torch.arange(W, device=c2w.device, dtype=torch.float32), indexing="ij")
    cam = torch.stack([(x - K[0, 2] + 0.5) / K[0, 0], (y - K[1, 2] + 0.5) / K[1, 1], torch.ones_like(x)])
    d = torch.einsum("ij,jhw->ihw", c2w[:3, :3], cam)
    return d / (d.norm(dim=0, keepdim=True) + 1e-8)


def lens_camera(cam):
    """cam with a principal point 3 % of the width right and 2 % of the height up of the centre, and mild barrel
    distortion with tangential terms (the K convention of render(pipe.lens): pixel centres at j + 0.5)."""
    W, H = cam.image_width, cam.image_height
    fx, fy = W / (2 * cam.tanfovx), H / (2 * cam.tanfovy)
    K = torch.tensor([[fx, 0.0, 0.53 * W], [0.0, fy, 0.48 * H], [0.0, 0.0, 1.0]])
    return syn.SyntheticCamera(W, H, cam.FoVx, cam.FoVy, cam.world_view_transform, cam.full_proj_transform,
                               cam.camera_center, cam.time, K, torch.tensor([-0.1, 0.02, 5e-4, -3e-4, 0.0]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=200_000)
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--width", type=int, default=960)
    ap.add_argument("--height", type=int, default=640)
    ap.add_argument("--fine", action="store_true", help="train the HexPlane deformation stage too")
    ap.add_argument("--checkpoint", default="", help="write and re-load a reference-format checkpoint here (needs --fine)")
    ap.add_argument("--filter-3d", action="store_true",
                    help="Mip-Splatting's 3-D smoothing filter, recomputed on Mip-Splatting's schedule")
    ap.add_argument("--densify-until", type=int, default=0, help="last densification iteration (0: never stop)")
    ap.add_argument("--absgrad-threshold", type=float, default=0.0,
                    help="densify on the absolute screen-space gradient (AbsGS, gsplat absgrad) with this threshold "
                         "instead of the signed one (0: off)")
    ap.add_argument("--mcmc-cap", type=int, default=0,
                    help="3DGS-MCMC densification up to this many Gaussians instead of densify / prune: relocation, "
                         "5 %% growth per interval, position noise and the opacity / scale regularisers (0: off)")
    ap.add_argument("--sparse-adam", action="store_true",
                    help="selective Adam: update only the Gaussians the step's view sees (radii > 0), as upstream "
                         "3DGS --optimizer_type sparse_adam and gsplat SelectiveAdam")
    ap.add_argument("--bilateral-grid", action="store_true",
                    help="per-camera bilateral-grid colour correction (gsplat --use_bilateral_grid): every camera's "
                         "targets get a fixed exposure difference, and each render is sliced through its camera's "
                         "grid before the loss")
    ap.add_argument("--sky", action="store_true",
                    help="sky model (the reference's Background_Model(model_type='mlp')): the targets get an analytic, "
                         "direction-dependent sky behind the Gaussians; each render (zero background, alpha image) is "
                         "composited over the model's sky, and alpha is pulled towards 1 - the sky mask")
    ap.add_argument("--lens", action="store_true",
                    help="camera intrinsics and distortion: every camera gets an off-centre principal point and OpenCV "
                         "radial-tangential coefficients; the targets and the training renders go through them "
                         "(pipe.lens)")
    a = ap.parse_args()
    if a.sky and a.bilateral_grid:
        ap.error("--sky re-renders the targets over its sky, which would drop --bilateral-grid's exposure changes")
    if a.mcmc_cap and a.absgrad_threshold > 0:
        ap.error("--mcmc-cap replaces densify / prune, so --absgrad-threshold has nothing to select")
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device: s3gaussian_b200 has no CPU path")
    dev = torch.device("cuda:0")
    opt = default_optimization_params()
    cams = [c.to(dev) for c in syn.waymo_ring(a.width, a.height, frames=10)]
    bg = torch.zeros(3, device=dev)
    pipe = PipelineParams()
    train_pipe = PipelineParams()
    train_pipe.filter_3d = a.filter_3d
    train_pipe.absgrad = a.absgrad_threshold > 0
    if a.lens:
        cams = [lens_camera(c) for c in cams]
        pipe.lens = train_pipe.lens = True

    # ---- scene: "ground truth" cloud -> target images; training starts from a point cloud of it -------
    truth = syn.make_cloud(a.points, seed=0)
    gt = GaussianModel(3).create_from_tensors(truth.xyz.to(dev), truth.features_dc.to(dev), truth.features_rest.to(dev),
                                              truth.scaling.to(dev), truth.rotation.to(dev), truth.opacity.to(dev))
    gt.active_sh_degree = 3
    with torch.no_grad():
        targets = []
        for c in cams:
            out = render(c, gt, pipe, bg, stage="coarse")
            targets.append((out["render"].clone(), out["depth"].clone()))
    bil_grids = bil_opt = None
    if a.bilateral_grid:
        from s3gaussian_b200.bilateral_grid import BilateralGrid
        from s3gaussian_b200.optim import FusedAdam
        # each camera's own exposure and white balance: a fixed per-channel gain and offset on its targets
        g = torch.Generator().manual_seed(7)
        for k, (img, dep) in enumerate(targets):
            gain = (1.0 + 0.15 * torch.randn(3, 1, 1, generator=g)).to(dev)
            offset = (0.03 * torch.randn(3, 1, 1, generator=g)).to(dev)
            targets[k] = (img * gain + offset, dep)
        bil_grids = BilateralGrid(len(cams)).to(dev)
        # gsplat's schedule (its LinearLR and ExponentialLR chained, so their factors multiply): lr 2e-3, a linear
        # warm-up from 0.01x over the first 1000 iterations and an exponential decay to 0.01x at the last iteration
        bil_opt = FusedAdam([{"params": [bil_grids.grids], "lr": 2e-3, "name": "bilagrid"}], lr=2e-3, eps=1e-15)
    sky_model = sky_opt = None
    if a.sky:
        from s3gaussian_b200.optim import FusedAdam
        from s3gaussian_b200.sky import Background_Model, sky_camera
        # the ground truth's sky: a smooth colour of the world-space ray direction, behind the truth cloud; the sky
        # mask is where the truth's alpha is below 0.5
        opa_pipe = PipelineParams()
        opa_pipe.render_opacity = True
        with torch.no_grad():
            for k, c in enumerate(cams):
                out = render(c, gt, opa_pipe, bg, stage="coarse")
                v = sky_directions(*sky_camera(c), a.height, a.width)
                sky = torch.stack([0.45 + 0.35 * v[2], 0.6 + 0.25 * v[2] - 0.1 * v[0], 0.85 - 0.1 * v[1]]).clamp(0, 1)
                alpha = out["alpha"]
                targets[k] = (out["render"] + (1.0 - alpha) * sky, targets[k][1], (alpha < 0.5).float())
        train_pipe.render_opacity = True
        sky_model = Background_Model(img_width=a.width, img_height=a.height, model_cfg={"mlp_width": 64}).to(dev)
        # not tuned on real data: the learning rate and the mask-loss weight below only have to work on this scene
        sky_opt = FusedAdam([{"params": list(sky_model.parameters()), "lr": 1e-3, "name": "sky"}], lr=1e-3, eps=1e-15)
    colours = (truth.features_dc[:, 0] * 0.28209479177387814 + 0.5).clamp(0, 1)
    pcd = SimpleNamespace(points=truth.xyz.numpy(), colors=colours.numpy())

    deformation = None
    if a.fine:
        sys.path.insert(0, os.path.join(ROOT, "tests"))      # tests/ref_ext.py holds the ModelHiddenParams defaults
        from ref_ext import ref_deform_args
        from s3gaussian_b200.deformation import deform_network
        deformation = deform_network(ref_deform_args(syn.DEFAULT_RESOLUTION, syn.DEFAULT_MULTIRES))
        deformation.deformation_net.set_aabb(*[list(x) for x in syn.WAYMO_AABB])
    gaussians = GaussianModel(3, deformation=deformation).create_from_pcd(pcd, spatial_lr_scale=5.0)   # 3-NN scales
    gaussians.training_setup(opt)
    if a.filter_3d:
        gaussians.compute_3D_filter(cams)       # Mip-Splatting: once before training, from every training camera
    stage = "fine" if a.fine else "coarse"
    extent = 30.0

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for it in range(1, a.iters + 1):
        if it == 11:
            e0.record()
        xyz_lr = gaussians.update_learning_rate(it)
        if it % 100 == 0:
            gaussians.oneupSHdegree()
        k = (it - 1) % len(cams)
        out = render(cams[k], gaussians, train_pipe, bg, stage=stage, return_dx=a.fine, render_feat=False)
        image, depth = out["render"], out["depth"]
        if bil_grids is not None:
            image = bil_grids.slice(image, k)
        if sky_model is not None:     # bg is zero: image + (1 - alpha) sky is the render over a per-pixel sky
            alpha = out["alpha"]
            image = image + (1.0 - alpha) * sky_model(*sky_camera(cams[k]))
        l1, ssim_value, depth_l2 = losses.image_loss_terms(image, targets[k][0], depth, targets[k][1])
        loss = l1 + 0.5 * depth_l2 + 0.2 * (1.0 - ssim_value)                    # train.py:395-419
        if bil_grids is not None:
            loss = loss + 10.0 * bil_grids.tv_loss()
        if sky_model is not None:     # binary cross-entropy of alpha against 1 - sky mask
            loss = loss + 0.05 * torch.nn.functional.binary_cross_entropy(alpha.clamp(1e-6, 1 - 1e-6),
                                                                          1.0 - targets[k][2])
        if a.fine:
            loss = loss + 0.001 * out["dx"].abs().mean() + 0.001 * out["dshs"].abs().mean() + \
                gaussians.compute_regulation(0.01, 0.0001, 0.0001)
        if a.mcmc_cap:      # 3DGS-MCMC's opacity and scale regularisers (its train.py, opacity_reg = scale_reg = 0.01)
            loss = loss + 0.01 * gaussians.get_opacity.mean() + 0.01 * gaussians.get_scaling.mean()
        loss.backward()
        with torch.no_grad():
            vs = out["viewspace_points"]
            gaussians.densification_step(vs.grad, out["radii"], getattr(vs, "absgrad", None))   # train.py:489-491
            densifying = not a.densify_until or it < a.densify_until
            if a.mcmc_cap and densifying and it > 50 and it % 100 == 0:
                gaussians.relocate_gs()
                gaussians.add_new_gs(a.mcmc_cap)
                gaussians.spatial_sort()
                if a.filter_3d:
                    gaussians.compute_3D_filter(cams)
            elif densifying and it > 50 and it % 100 == 0:
                gaussians.densify(0.0002, 0.005, extent, 20 if it > 3000 else None,
                                  max_grad_abs=a.absgrad_threshold if a.absgrad_threshold > 0 else None)
                gaussians.prune(0.0002, 0.005, extent, 20 if it > 3000 else None)
                gaussians.spatial_sort()      # ours: keep the model in Morton order (densify appends at the end)
                if a.filter_3d:
                    gaussians.compute_3D_filter(cams)     # Mip-Splatting: after every densify and prune
            elif a.filter_3d and a.densify_until and it > a.densify_until and it % 100 == 0 and it < a.iters - 100:
                gaussians.compute_3D_filter(cams)         # then every 100 iterations, except near the end
        if a.sparse_adam:       # after densify / prune the per-Gaussian tensors have no gradient: dense groups only
            gaussians.optimizer.step(visibility=out["radii"] > 0)
        else:
            gaussians.optimizer.step()                                           # one launch over all groups
        gaussians.optimizer.zero_grad(set_to_none=True)
        if bil_opt is not None:
            warm = 0.01 + 0.99 * min((it - 1) / 1000.0, 1.0)
            decay = 0.01 ** ((it - 1) / a.iters)
            bil_opt.param_groups[0]["lr"] = 2e-3 * warm * decay
            bil_opt.step()
            bil_opt.zero_grad(set_to_none=True)
        if sky_opt is not None:
            sky_opt.step()
            sky_opt.zero_grad(set_to_none=True)
        if a.mcmc_cap:
            gaussians.inject_noise(xyz_lr)
        if it % 50 == 0:
            print(f"iter {it:5d}  loss {loss.item():.5f}  l1 {l1.item():.5f}  ssim {ssim_value.item():.4f}  "
                  f"points {gaussians.get_xyz.shape[0]}")
    e1.record()
    torch.cuda.synchronize()
    # checkpoint in the reference's format (train.py:531: torch.save((gaussians.capture(), iteration), path)) and back
    if a.checkpoint and not a.fine:
        print("--checkpoint needs --fine: capture() stores the deformation network's state_dict")
    elif a.checkpoint:
        torch.save((gaussians.capture(), a.iters), a.checkpoint)
        model_args, first_iter = torch.load(a.checkpoint, weights_only=False)
        resumed = GaussianModel(3, deformation=gaussians._deformation)
        resumed.restore(model_args, opt)
        assert torch.equal(resumed.get_xyz, gaussians.get_xyz) and first_iter == a.iters
        print(f"checkpoint {a.checkpoint}: {resumed.get_xyz.shape[0]} points restored (iteration {first_iter})")
    if a.iters > 10:
        print(f"{e0.elapsed_time(e1) / (a.iters - 10):.3f} ms per iteration over the last {a.iters - 10}")


if __name__ == "__main__":
    main()
