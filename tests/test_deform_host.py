"""CPU: the deformation drop-in keeps the reference's parameter names/shapes (checkpoint
compatibility), stores planes channels-last, and refuses CPU tensors."""
import numpy as np
import pytest
import torch

import ref_ext
from s3gaussian_b200 import synthetic as syn
from s3gaussian_b200.deformation import deform_network


def make(reso=(16, 12, 10, 7), multires=(1, 2), **flags):
    return deform_network(ref_ext.ref_deform_args(reso, multires, **flags))


def test_state_dict_matches_reference_layout():
    net = make(syn.DEFAULT_RESOLUTION[:3] + (25,), (1, 2))
    sd = net.state_dict()
    st = syn.make_deform_state(0, syn.DEFAULT_RESOLUTION, (1, 2))
    for k, v in st.items():
        assert k in sd, k
        assert tuple(sd[k].shape) == tuple(v.shape), (k, sd[k].shape, v.shape)
    # names the reference has and the path never reads are still there for checkpoint loading
    for k in ("timenet.0.weight", "timenet.2.bias", "time_poc", "pos_poc", "rotation_scaling_poc", "opacity_poc",
              "deformation_net.grid.aabb"):
        assert k in sd
    assert sd["deformation_net.grid.grids.1.2"].shape == (1, 32, 25, 128)     # (x,t) plane of level x2
    missing, unexpected = net.load_state_dict(st, strict=False)
    assert not unexpected


def test_planes_are_channels_last_and_survive_load_state_dict():
    net = make()
    st = syn.make_deform_state(3, (16, 12, 10, 7), (1, 2))
    net.load_state_dict(st, strict=False)
    for gp in net.deformation_net.grid.grids:
        for p in gp:
            assert p.is_contiguous(memory_format=torch.channels_last)
    p = net.deformation_net.grid.grids[0][0]
    assert torch.equal(p.detach(), st["deformation_net.grid.grids.0.0"])
    # texel (y,x) is 32 contiguous floats
    assert p.stride() == (32 * p.shape[2] * p.shape[3], 1, 32 * p.shape[3], 32)
    assert sum(p.numel() for p in make(syn.DEFAULT_RESOLUTION, syn.DEFAULT_MULTIRES).parameters()) == 35_771_492


def test_unsupported_configs_and_cpu_inputs_fail_loudly():
    # switches that run through the PyTorch cold path (deformation_cold.py) construct; they refuse CPU tensors too
    for flag in ("empty_voxel", "static_mlp"):
        cold = make(**{flag: True})
        assert cold.deformation_net.cold
        z = torch.zeros(4, 3)
        with pytest.raises(RuntimeError, match="no CPU path"):
            cold(z, z, torch.zeros(4, 4), torch.zeros(4, 1), torch.zeros(4, 16, 3), torch.zeros(4, 1))
    with pytest.raises(NotImplementedError):
        make(no_grid=True)
    with pytest.raises(NotImplementedError):
        deform_network(ref_ext.ref_deform_args((8, 8, 8, 5), (1,), net_width=128))
    net = make()
    x = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="no CPU path"):
        net(x, x, torch.zeros(4, 4), torch.zeros(4, 1), torch.zeros(4, 16, 3), torch.zeros(4, 1))


def test_render_signature_matches_reference():
    import inspect
    from s3gaussian_b200 import gaussian_renderer as gr
    sig = inspect.signature(gr.render)
    assert list(sig.parameters) == ["viewpoint_camera", "pc", "pipe", "bg_color", "scaling_modifier", "override_color",
                                    "stage", "return_decomposition", "return_dx", "render_feat"]
    assert sig.parameters["stage"].default == "fine" and sig.parameters["scaling_modifier"].default == 1.0


def test_saved_activation_buffer_size_follows_the_enabled_heads(built_lib):
    """s3g_deform_saved_bytes (host logic, no GPU): one [ceil(P/128)*128][64] float tile set per kept hidden layer -
    h plus the hidden layer of every enabled head (the dino head has two) - and 0 for nets whose forward does not run
    on the wgmma kernel (unsupported level counts)."""
    import ctypes as C
    from s3gaussian_b200 import _lib
    from s3gaussian_b200.deformation import CNet
    lib = _lib.load()

    def saved(net, P):
        byname = {n: p.detach() for n, p in net._named_hot_params()}
        cnet = CNet()
        net._fill(cnet, byname)
        return int(lib.s3g_deform_saved_bytes(C.byref(cnet), P))

    per_slot = lambda P: ((P + 127) // 128) * 128 * 64 * 4
    default = make()                                        # pos + shs + dino: h, pos, shs, d0, d2
    assert saved(default, 1000) == 5 * per_slot(1000)
    assert saved(default, 128) == 5 * 128 * 64 * 4
    assert saved(default, 0) == 0
    allheads = make(no_ds=False, no_dr=False, no_do=False)  # + scales, rotation, opacity
    assert saved(allheads, 1000) == 8 * per_slot(1000)
    nofeat = make(feat_head=False, no_dshs=True)            # h + pos only
    assert saved(nofeat, 300) == 2 * per_slot(300)
    deep = make(reso=(8, 8, 8, 5), multires=(1, 2, 3, 4, 5))   # 5 levels: not a supported net -> 0, and the forward raises
    assert saved(deep, 1000) == 0


def test_backward_without_saved_activations_is_an_argument_error(built_lib):
    """s3g_deform_backward_saved reads the hidden activations the forward kept: with P > 0 a NULL `acts` returns
    S3G_ERR_ARG with a message, before any CUDA call (so no GPU is needed here)."""
    import ctypes as C
    from s3gaussian_b200.deformation import CNet, CNetGrads
    net = make()
    byname = {n: p.detach() for n, p in net._named_hot_params()}
    grads = {n: torch.zeros_like(p) for n, p in byname.items()}
    cnet, cg = CNet(), CNetGrads()
    net._fill(cnet, byname, grads=(cg, grads))
    dummy = C.c_void_p(256)      # never dereferenced: the call returns before it touches a device pointer
    rc = built_lib.s3g_deform_backward_saved(C.byref(cnet), 100, *[dummy] * 5, 0.5, dummy, 3, dummy, None,
                                             *[None] * 8, *[dummy] * 5, C.byref(cg), dummy, None)
    assert rc == -1
    assert b"null acts" in built_lib.s3g_last_error()
