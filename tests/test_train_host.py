"""CPU: host-side behaviour of the training-step modules (no kernels run): argument validation, the
no-CPU-fallback rule, optimizer state layout, learning-rate schedule."""
import math

import pytest
import torch


def test_image_loss_rejects_cpu_tensors(built_lib):
    from s3gaussian_b200 import losses
    with pytest.raises(RuntimeError, match="no CPU path"):
        losses.l1_loss(torch.zeros(3, 8, 8), torch.zeros(3, 8, 8))
    with pytest.raises(RuntimeError, match="pairs"):
        losses.image_loss_terms(torch.zeros(3, 8, 8), torch.zeros(3, 8, 8), depth=torch.zeros(1, 8, 8))
    with pytest.raises(NotImplementedError):
        losses.compute_depth("smooth_l1", torch.zeros(1, 8, 8), torch.zeros(1, 8, 8))
    with pytest.raises(NotImplementedError):
        losses.ssim(torch.zeros(3, 8, 8), torch.zeros(3, 8, 8), window_size=7)


def test_fused_adam_rejects_cpu_and_unsupported(built_lib):
    from s3gaussian_b200.optim import FusedAdam
    p = torch.nn.Parameter(torch.zeros(4))
    p.grad = torch.ones(4)
    with pytest.raises(RuntimeError, match="no CPU path"):
        FusedAdam([p], lr=1e-3).step()
    with pytest.raises(NotImplementedError):
        FusedAdam([p], lr=1e-3, amsgrad=True)
    with pytest.raises(NotImplementedError):
        FusedAdam([p], lr=1e-3, weight_decay=0.1)
    with pytest.raises(ValueError):
        FusedAdam([p], lr=-1.0)


def test_fused_adam_keeps_the_reference_group_layout(built_lib):
    """The reference addresses groups by group['name'] and state by parameter (gaussian_model.py:397-470)."""
    from s3gaussian_b200.optim import FusedAdam
    a, b = torch.nn.Parameter(torch.zeros(5, 3)), torch.nn.Parameter(torch.zeros(5, 1))
    opt = FusedAdam([{"params": [a], "lr": 1.6e-4, "name": "xyz"}, {"params": [b], "lr": 0.05, "name": "opacity"}],
                    lr=0.0, eps=1e-15)
    assert [g["name"] for g in opt.param_groups] == ["xyz", "opacity"]
    assert opt.param_groups[0]["eps"] == 1e-15 and opt.param_groups[1]["lr"] == 0.05
    assert opt.state.get(a, None) is None
    opt.step()      # no gradients: nothing to do, no state created, no kernel launched
    assert len(opt.state) == 0
    sd = opt.state_dict()
    assert sd["param_groups"][0]["name"] == "xyz"


def test_densify_stats_rejects_cpu(built_lib):
    from s3gaussian_b200.optim import add_densification_stats
    with pytest.raises(RuntimeError, match="no CPU path"):
        add_densification_stats(torch.zeros(4, 3), torch.zeros(4, dtype=torch.int32), torch.zeros(4, 1),
                                torch.zeros(4, 1), torch.zeros(4))


def test_expon_lr_schedule():
    from s3gaussian_b200.optim import get_expon_lr_func
    f = get_expon_lr_func(1.6e-4, 1.6e-6, lr_delay_mult=0.01, max_steps=20000)
    assert f(0) == pytest.approx(1.6e-4) and f(20000) == pytest.approx(1.6e-6) and f(40000) == pytest.approx(1.6e-6)
    assert f(10000) == pytest.approx(math.sqrt(1.6e-4 * 1.6e-6))
    assert f(-1) == 0.0 and get_expon_lr_func(0.0, 0.0)(5) == 0.0
    d = get_expon_lr_func(1.0, 1.0, lr_delay_steps=100, lr_delay_mult=0.1)
    assert d(0) == pytest.approx(0.1) and d(100) == pytest.approx(1.0) and 0.1 < d(50) < 1.0


def test_split_plan_row_order():
    """kept rows in order, then the selected rows twice - the order densify_and_split + prune_points produce
    (scene/gaussian_model.py:496-522)."""
    from s3gaussian_b200.gaussian_model import split_plan
    sel = torch.tensor([False, True, False, False, True, False])
    src, n_kept, idx = split_plan(sel)
    assert n_kept == 4 and idx.tolist() == [1, 4]
    assert src.tolist() == [0, 2, 3, 5, 1, 4, 1, 4]
    # the same thing spelled the reference's way on a value tensor
    x = torch.arange(6.0)
    cat = torch.cat((x, x[sel].repeat(2)))
    pruned = cat[~torch.cat((sel, torch.zeros(2 * int(sel.sum()), dtype=torch.bool)))]
    assert torch.equal(pruned, x[src])


def test_gaussian_model_rejects_cpu_and_exposes_reference_names(built_lib):
    from s3gaussian_b200.gaussian_model import GaussianModel, default_optimization_params
    m = GaussianModel(3)
    with pytest.raises(RuntimeError, match="no CPU path"):
        m.create_from_tensors(torch.zeros(4, 3), torch.zeros(4, 1, 3), torch.zeros(4, 15, 3), torch.zeros(4, 3),
                              torch.zeros(4, 4), torch.zeros(4, 1))
    for name in ("create_from_pcd", "save_ply", "load_ply", "save_deformation", "load_model","training_setup", "update_learning_rate", "add_densification_stats", "densify", "prune", "prune_points",
                 "densify_and_clone", "densify_and_split", "reset_opacity", "replace_tensor_to_optimizer",
                 "compute_regulation", "oneupSHdegree", "get_covariance"):
        assert callable(getattr(m, name))
    a = default_optimization_params()
    assert a.position_lr_init == 0.00016 and a.percent_dense == 0.01 and a.opacity_lr == 0.05


def test_gather_rows_argument_checks(built_lib):
    import ctypes as C
    from s3gaussian_b200 import _lib
    lib = _lib.load()
    assert lib.s3g_gather_rows(0, None, 1, 1, None, None) == -1
    t = (_lib.RowTensor * 1)(_lib.RowTensor(1, 1, 3, 0))
    assert lib.s3g_gather_rows(1, t, 4, 5, None, None) == -1          # n_kept > n_out
    assert lib.s3g_gather_rows(1, t, 0, 0, None, None) == 0           # nothing to do


def test_image_loss_argument_checks(built_lib):
    """Every call below is refused before any launch; the fake device addresses are never dereferenced."""
    from s3gaussian_b200 import _lib
    lib = _lib.load()
    P = 256
    for fwd in (lib.s3g_image_loss_forward, lib.s3g_image_l1_depth_forward):
        assert fwd(1, 65536, 4, 4, P, P, None, None, 80.0, P, P, None) == -1      # B*C = 65536 planes
        assert fwd(65536, 1, 4, 4, P, P, None, None, 80.0, P, P, None) == -1
        assert fwd(1, 0, 4, 4, None, None, None, None, 80.0, P, P, None) == -1    # C = 0 and no depth
        assert fwd(1, 3, 4, 4, P, P, P, None, 80.0, P, P, None) == -1             # depth without gt_depth
        assert fwd(1, 3, 4, 4, P, P, None, P, 80.0, P, P, None) == -1             # gt_depth without depth
        assert fwd(1, 3, 4, 4, None, P, None, None, 80.0, P, P, None) == -1       # C > 0 and no image
        assert fwd(1, 3, 0, 4, P, P, None, None, 80.0, P, P, None) == -1          # empty image
        assert fwd(1, 3, 4, 4, P, P, None, None, 80.0, None, P, None) == -1       # no sums
        assert fwd(1, 3, 4, 4, P, P, None, None, 80.0, P, None, None) == -1       # no workspace
    bwd = lib.s3g_image_loss_backward
    assert bwd(1, 65536, 4, 4, P, P, None, None, 80.0, P, P, P, P, None, None) == -1
    assert bwd(1, 0, 4, 4, None, None, None, None, 80.0, P, P, P, None, None, None) == -1
    assert bwd(1, 3, 4, 4, P, P, P, None, 80.0, P, P, P, P, P, None) == -1
    assert bwd(1, 3, 4, 4, P, P, None, None, 80.0, P, P, P, None, None, None) == -1     # no g_image
    assert bwd(1, 0, 4, 4, None, None, P, P, 80.0, P, P, P, None, None, None) == -1     # no g_depth
    bl1 = lib.s3g_image_l1_depth_backward
    assert bl1(1, 65536, 4, 4, P, P, None, None, 80.0, P, P, P, None, None) == -1
    assert bl1(1, 0, 4, 4, None, None, None, None, 80.0, P, P, None, None, None) == -1
    assert bl1(1, 3, 4, 4, P, P, None, P, 80.0, P, P, P, None, None) == -1
    assert bl1(1, 3, 4, 4, P, P, None, None, 80.0, None, P, P, None, None) == -1       # no weights
    # the largest plane count is accepted (sizing only; nothing runs)
    assert lib.s3g_image_loss_workspace_bytes(65535, 1, 1, 1) > 0
    assert lib.s3g_image_loss_workspace_bytes(1, 3, 0, 4) == 0


def test_plane_reg_argument_checks(built_lib):
    """The 48-plane table limit, H >= 3, C % 4 == 0 and 16-byte alignment are checked before any launch; the
    workspace holds one double per 1024-float4 block."""
    from s3gaussian_b200 import _lib
    lib = _lib.load()
    P, G = 256, 512

    def table(*shapes, plane=P, grad=G):
        return (_lib.PlaneDesc * len(shapes))(*[_lib.PlaneDesc(plane, grad, H, W, Cc, 1.0, 0.5) for H, W, Cc in shapes])
    ok = table(*[(4, 2, 4)] * 48)
    assert lib.s3g_plane_reg_workspace_bytes(48, ok) == 256 + 8 * 48
    for n, t in ((49, table(*[(4, 2, 4)] * 49)), (0, ok), (1, table((2, 8, 4))), (1, table((3, 8, 6))),
                 (1, table((3, 8, 2))), (1, table((3, 0, 4))), (1, table((3, 8, 4), plane=P + 4))):
        assert lib.s3g_plane_reg_workspace_bytes(n, t) == 0
        assert lib.s3g_plane_reg_forward(n, t, P, P, None) == -1
        assert lib.s3g_plane_reg_backward(n, t, P, None) == -1
    unaligned_grad = table((3, 8, 4), grad=G + 8)
    assert lib.s3g_plane_reg_workspace_bytes(1, unaligned_grad) > 0     # the forward reads no gradient
    assert lib.s3g_plane_reg_backward(1, unaligned_grad, P, None) == -1
    assert lib.s3g_plane_reg_backward(1, table((3, 8, 4), grad=None), P, None) == -1
    assert lib.s3g_plane_reg_backward(1, table((3, 8, 4)), None, None) == -1           # no upstream gradient
    assert lib.s3g_plane_reg_forward(1, table((3, 8, 4)), None, P, None) == -1         # no total
    # blocks of 1024 float4: 1023 and 1024 float4 fit one block, 1025 take two
    for H, blocks in ((1023, 1), (1024, 1), (1025, 2)):
        assert lib.s3g_plane_reg_workspace_bytes(1, table((H, 1, 4))) == 256 + 8 * blocks
    assert lib.s3g_plane_reg_workspace_bytes(2, table((1025, 1, 4), (7, 300, 8))) == 256 + 8 * (2 + 5)


def test_peer_slices_cover_the_buffer_in_float4_units():
    from s3gaussian_b200.dp import peer_slices
    for numel, world in ((40, 3), (8, 8), (118_000_000, 8), (4, 2), (472, 5)):
        sl = peer_slices(numel, world)
        assert len(sl) == world and sl[0][0] == 0 and sl[-1][1] == numel
        assert all(b % 4 == 0 and e % 4 == 0 and b <= e for b, e in sl)
        assert all(sl[i][1] == sl[i + 1][0] for i in range(world - 1))
    with pytest.raises(ValueError):
        peer_slices(10, 2)


def test_peer_entry_points_check_arguments(built_lib):
    import ctypes as C
    from s3gaussian_b200 import _lib
    lib = _lib.load()
    two = (C.c_void_p * 2)(16, 32)
    assert lib.s3g_peer_reduce_scatter(1, 0, two, 8, None) == -1        # world < 2
    assert lib.s3g_peer_reduce_scatter(2, 2, two, 8, None) == -1        # rank out of range
    assert lib.s3g_peer_all_gather(2, 0, two, 6, None) == -1            # numel not a multiple of 4
    bad = (C.c_void_p * 2)(16, 36)
    assert lib.s3g_peer_all_gather(2, 0, bad, 8, None) == -1            # misaligned peer pointer
