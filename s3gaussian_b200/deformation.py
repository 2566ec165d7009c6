"""Drop-in for the reference's ``scene.deformation.deform_network`` (+ the
HexPlane field it owns), backed by the fused CUDA kernels of libs3g_b200.so.

Same constructor argument (an ``args`` namespace with the ``ModelHiddenParams``
fields, arguments/__init__.py:204-233), same parameter names and shapes as the
reference module (scene/deformation.py:16-76,179-200, scene/hexplane.py:48-70), so
``state_dict`` / checkpoints interchange; the planes are ``[1,32,H,W]`` parameters
stored in ``torch.channels_last`` memory format, which is the ``[H][W][32]`` texel
layout the kernels gather (one 128-byte load per bilinear tap).

``forward(point, scales, rotations, opacity, shs, times_sel)`` returns the
reference's 8-tuple ``(means3D, scales, rotations, opacity, shs, dx, feat, dshs)``
(scene/deformation.py:216-231).  ``render_front(...)`` is the fused form
``render()`` uses: it also applies the activations and the Python SH->RGB of
gaussian_renderer/__init__.py:99-117 inside the same kernel.

No CPU path: CPU tensors raise.
"""
from __future__ import annotations

import ctypes as C
import itertools
import math
import warnings

import torch
import torch.nn as nn

from . import _lib

MAX_LEVELS = 8
_PF = C.POINTER(C.c_float)

# every Linear the kernels read: reference module path, s3g_deform_net field suffix (w_<suffix>, b_<suffix>) and the
# args switch of its head (None: always on; a no_* switch turns the head off, feat_head turns it on)
_LAYERS = [
    ("feature_out.0", "feat", None),
    ("pos_deform.1", "pos1", "no_dx"), ("pos_deform.3", "pos2", "no_dx"),
    ("scales_deform.1", "scl1", "no_ds"), ("scales_deform.3", "scl2", "no_ds"),
    ("rotations_deform.1", "rot1", "no_dr"), ("rotations_deform.3", "rot2", "no_dr"),
    ("opacity_deform.1", "opa1", "no_do"), ("opacity_deform.3", "opa2", "no_do"),
    ("shs_deform.1", "shs1", "no_dshs"), ("shs_deform.3", "shs2", "no_dshs"),
    ("dino_head.0", "dino0", "feat_head"), ("dino_head.2", "dino2", "feat_head"), ("dino_head.4", "dino4", "feat_head"),
]
_FIELDS = [(f"{wb}_{suffix}", C.c_void_p) for _, suffix, _ in _LAYERS for wb in ("w", "b")]


def _head_on(args, switch):
    if switch is None:
        return True
    if switch.startswith("no_"):
        return not getattr(args, switch)
    return getattr(args, switch, True)


class CNet(C.Structure):           # s3g_deform_net (include/s3g_b200.h)
    _fields_ = [("num_levels", C.c_int), ("feat_dim", C.c_int), ("width", C.c_int),
                ("reso", (C.c_int * 4) * MAX_LEVELS), ("planes", (C.c_void_p * 6) * MAX_LEVELS),
                ("aabb", C.c_float * 6)] + _FIELDS


class CNetGrads(C.Structure):      # s3g_deform_net_grads
    _fields_ = [("planes", (C.c_void_p * 6) * MAX_LEVELS)] + _FIELDS


def _p(t):
    return None if t is None else t.data_ptr()


class HexPlaneField(nn.Module):
    """Parameter container with the reference's names (scene/hexplane.py:109-158)."""

    def __init__(self, bounds, planeconfig, multires):
        super().__init__()
        self.aabb = nn.Parameter(torch.tensor([[bounds] * 3, [-bounds] * 3], dtype=torch.float32), requires_grad=False)
        self.grid_config = [planeconfig]
        self.multiscale_res_multipliers = list(multires)
        self.concat_features = True
        self.grids = nn.ModuleList()
        self.feat_dim = 0
        out_dim = planeconfig["output_coordinate_dim"]
        assert planeconfig["grid_dimensions"] == 2 and planeconfig["input_coordinate_dim"] == 4
        for res in self.multiscale_res_multipliers:
            reso = [r * res for r in planeconfig["resolution"][:3]] + list(planeconfig["resolution"][3:])
            gp = nn.ParameterList()
            for comb in itertools.combinations(range(4), 2):
                shape = [1, out_dim] + [reso[cc] for cc in comb[::-1]]
                t = torch.empty(shape).contiguous(memory_format=torch.channels_last)
                if 3 in comb:
                    nn.init.ones_(t)                       # time planes start at 1 (hexplane.py:64-65)
                else:
                    nn.init.uniform_(t, a=0.1, b=0.5)
                gp.append(nn.Parameter(t))
            self.feat_dim += out_dim
            self.grids.append(gp)

    @property
    def get_aabb(self):
        return self.aabb[0], self.aabb[1]

    def set_aabb(self, xyz_max, xyz_min):
        self.aabb = nn.Parameter(torch.tensor([xyz_max, xyz_min], dtype=torch.float32).to(self.aabb.device),
                                 requires_grad=False)


class Deformation(nn.Module):
    """Parameter container mirroring scene/deformation.py:16-76 (default W=64, D=1)."""

    def __init__(self, D=1, W=64, args=None):
        super().__init__()
        if D != 1 or W != 64:
            raise NotImplementedError("the fused decoder is built for defor_depth=1, net_width=64")
        if getattr(args, "no_grid", False):
            raise NotImplementedError("no_grid=True: the reference itself cannot run it (query_time leaves `hidden` "
                                      "undefined, scene/deformation.py:80-91)")
        if getattr(args, "grid_pe", 0) != 0:
            raise NotImplementedError("grid_pe != 0: the reference sizes feature_out for 3x the features but feeds it "
                                      "1x or (1+2*grid_pe)x (scene/deformation.py:47-50,86-87); not runnable upstream")
        self.D, self.W, self.args = D, W, args
        # switches that stay in PyTorch: deformation_cold.py
        self.cold = bool(getattr(args, "empty_voxel", False) or getattr(args, "static_mlp", False) or
                         getattr(args, "apply_rotation", False))
        self.grid = HexPlaneField(args.bounds, args.kplanes_config, args.multires)
        if getattr(args, "empty_voxel", False):
            from .deformation_cold import DenseGrid
            self.empty_voxel = DenseGrid(channels=1, world_size=[64, 64, 64])
        if getattr(args, "static_mlp", False):
            self.static_mlp = nn.Sequential(nn.ReLU(), nn.Linear(W, W), nn.ReLU(), nn.Linear(W, 1))
        self.feature_out = nn.Sequential(nn.Linear(self.grid.feat_dim, W))

        def head(k):
            return nn.Sequential(nn.ReLU(), nn.Linear(W, W), nn.ReLU(), nn.Linear(W, k))
        self.pos_deform, self.scales_deform, self.rotations_deform = head(3), head(3), head(4)
        self.opacity_deform, self.shs_deform = head(1), head(16 * 3)
        if getattr(args, "feat_head", True):
            self.dino_head = nn.Sequential(nn.Linear(64, 64), nn.ReLU(), nn.Linear(64, 64), nn.ReLU(), nn.Linear(64, 3))

    @property
    def get_aabb(self):
        return self.grid.get_aabb

    def set_aabb(self, xyz_max, xyz_min):
        self.grid.set_aabb(xyz_max, xyz_min)
        if getattr(self.args, "empty_voxel", False):
            self.empty_voxel.set_aabb(xyz_max, xyz_min)

    def get_mlp_parameters(self):
        return [p for n, p in self.named_parameters() if "grid" not in n]

    def get_grid_parameters(self):
        return [p for n, p in self.named_parameters() if "grid" in n]


def initialize_weights(m):      # scene/deformation.py:237-243 (both branches touch the WEIGHT)
    if isinstance(m, nn.Linear):
        nn.init.xavier_uniform_(m.weight, gain=1)


class deform_network(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.args = args
        times_ch = 2 * args.timebase_pe + 1
        # present in the reference's state_dict but dead on the path (deformation.py:190-193,218-224)
        self.timenet = nn.Sequential(nn.Linear(times_ch, args.timenet_width), nn.ReLU(),
                                     nn.Linear(args.timenet_width, args.timenet_output))
        self.deformation_net = Deformation(W=args.net_width, D=args.defor_depth, args=args)
        self.register_buffer("time_poc", torch.FloatTensor([(2 ** i) for i in range(args.timebase_pe)]))
        self.register_buffer("pos_poc", torch.FloatTensor([(2 ** i) for i in range(args.posebase_pe)]))
        self.register_buffer("rotation_scaling_poc", torch.FloatTensor([(2 ** i) for i in range(args.scale_rotation_pe)]))
        self.register_buffer("opacity_poc", torch.FloatTensor([(2 ** i) for i in range(args.opacity_pe)]))
        self.apply(initialize_weights)

    # ---- reference API ------------------------------------------------------
    @property
    def get_aabb(self):
        return self.deformation_net.get_aabb

    def get_mlp_parameters(self):
        return self.deformation_net.get_mlp_parameters() + list(self.timenet.parameters())

    def get_grid_parameters(self):
        return self.deformation_net.get_grid_parameters()

    def forward(self, point, scales=None, rotations=None, opacity=None, shs=None, times_sel=None):
        return self.forward_dynamic(point, scales, rotations, opacity, shs, times_sel)

    def forward_dynamic(self, point, scales=None, rotations=None, opacity=None, shs=None, times_sel=None):
        """(means3D, scales, rotations, opacity, shs, dx, feat, dshs) - raw (pre-activation)
        scales / rotations / opacity, like scene/deformation.py:216-231."""
        t = float(times_sel.reshape(-1)[0]) if torch.is_tensor(times_sel) else float(times_sel)
        if self.deformation_net.cold:
            from . import deformation_cold
            if not point.is_cuda:
                raise RuntimeError("s3gaussian_b200 has no CPU path: point must be a CUDA tensor")
            return deformation_cold.forward_dynamic(self.deformation_net, point, scales, rotations, opacity, shs, t)
        zero3 = torch.zeros(3, device=point.device)
        out = _DeformFront.apply(self, t, zero3, 0, True, point, scales, rotations, opacity, shs,
                                 *self._param_list())
        means3D, sc, ro, op, _colors, dx, dshs, feat = out
        a = self.args
        shs_f = shs if a.no_dshs else shs + dshs
        return (means3D, sc, ro, op, shs_f, None if a.no_dx else dx,
                feat if getattr(a, "feat_head", True) else None, None if a.no_dshs else dshs)

    # ---- fused front-end of render() -----------------------------------------
    def render_front(self, xyz, scaling, rotation, opacity, shs, time, campos, active_sh_degree):
        """One kernel: deformation + activations + SH->RGB (gaussian_renderer/__init__.py:89-117).
        Returns (means3D_final, scales_act, rot_act, opacity_act, colors_precomp, dx, dshs, feat)."""
        if self.deformation_net.cold:
            from . import deformation_cold
            if not xyz.is_cuda:
                raise RuntimeError("s3gaussian_b200 has no CPU path: xyz must be a CUDA tensor")
            return deformation_cold.render_front(self.deformation_net, xyz, scaling, rotation, opacity, shs, float(time),
                                                 campos, active_sh_degree)
        return _DeformFront.apply(self, float(time), campos, int(active_sh_degree), False, xyz, scaling, rotation,
                                  opacity, shs, *self._param_list())

    # ---- plumbing ------------------------------------------------------------
    def _named_hot_params(self):
        d = self.deformation_net
        out = []
        for li, gp in enumerate(d.grid.grids):
            for ci, p in enumerate(gp):
                out.append((f"grid.{li}.{ci}", p))
        for lname, _, switch in _LAYERS:
            if not _head_on(self.args, switch):
                continue
            mod = d
            for part in lname.split("."):
                mod = getattr(mod, part) if not part.isdigit() else mod[int(part)]
            out.append((lname + ".weight", mod.weight))
            out.append((lname + ".bias", mod.bias))
        return out

    def _param_list(self):
        return [p for _, p in self._named_hot_params()]

    def _fill(self, cnet, tensors_by_name, grads=None):
        """fill a CNet (and optionally a CNetGrads) from {name: tensor}"""
        d = self.deformation_net
        L = len(d.grid.grids)
        cnet.num_levels, cnet.feat_dim, cnet.width = L, d.grid.grid_config[0]["output_coordinate_dim"], d.W
        base = d.grid.grid_config[0]["resolution"]
        for li, m in enumerate(d.grid.multiscale_res_multipliers):
            reso = [r * m for r in base[:3]] + list(base[3:])
            for c in range(4):
                cnet.reso[li][c] = reso[c]
            for ci in range(6):
                cnet.planes[li][ci] = tensors_by_name[f"grid.{li}.{ci}"].data_ptr()
                if grads is not None:
                    grads[0].planes[li][ci] = grads[1][f"grid.{li}.{ci}"].data_ptr()
        aabb = d.grid.aabb.detach().reshape(-1).tolist()
        for i in range(6):
            cnet.aabb[i] = aabb[i]
        for lname, suffix, switch in _LAYERS:
            on = _head_on(self.args, switch)
            wf, bf = "w_" + suffix, "b_" + suffix
            setattr(cnet, wf, tensors_by_name[lname + ".weight"].data_ptr() if on else None)
            setattr(cnet, bf, tensors_by_name[lname + ".bias"].data_ptr() if on else None)
            if grads is not None:
                setattr(grads[0], wf, grads[1][lname + ".weight"].data_ptr() if on else None)
                setattr(grads[0], bf, grads[1][lname + ".bias"].data_ptr() if on else None)


_NONDETERMINISTIC_WARNED = False


def _warn_if_deterministic_requested():
    """The deformation backward adds its gradients with atomic reductions; under
    torch.use_deterministic_algorithms(True) say so once per process (it still runs)."""
    global _NONDETERMINISTIC_WARNED
    if torch.are_deterministic_algorithms_enabled() and not _NONDETERMINISTIC_WARNED:
        _NONDETERMINISTIC_WARNED = True
        warnings.warn("the deformation backward is not deterministic: the HexPlane plane-gradient scatter and the "
                      "decoder weight gradients are summed with atomic reductions, so their last bits vary from run "
                      "to run", UserWarning, stacklevel=3)


def _check_plane(p):
    if p.dim() != 4 or p.shape[0] != 1:
        raise RuntimeError("plane parameter must be [1,C,H,W]")
    if not p.is_contiguous(memory_format=torch.channels_last):
        raise RuntimeError("plane parameters must be in torch.channels_last memory format "
                           "(HexPlaneField creates them that way; load_state_dict preserves it)")


class _DeformFront(torch.autograd.Function):
    """inputs: module, time, campos, sh_degree, raw_outputs, xyz, scaling, rotation, opacity, shs, *params
    outputs: means3D, scales, rot, opacity, colors, dx, dshs, feat
    (raw_outputs=True: scales/rot/opacity are returned WITHOUT activation, as forward_dynamic does)"""

    @staticmethod
    def forward(ctx, module, time, campos, sh_degree, raw_outputs, xyz, scaling, rotation, opacity, shs, *params):
        lib = _lib.load()
        if not xyz.is_cuda:
            raise RuntimeError("s3gaussian_b200 has no CPU path: xyz must be a CUDA tensor")
        dev = xyz.device
        P = xyz.shape[0]
        f32 = lambda t: t.detach().to(torch.float32).contiguous()
        xyz_, sc_, ro_, op_, shs_ = f32(xyz), f32(scaling), f32(rotation), f32(opacity), f32(shs)
        if shs_.shape[1:] != (16, 3):
            raise NotImplementedError("the fused SH path is built for max_sh_degree = 3 (16 coefficients)")
        names = [n for n, _ in module._named_hot_params()]
        byname = dict(zip(names, [p.detach() for p in params]))
        for n, p in byname.items():
            if n.startswith("grid."):
                _check_plane(p)
            elif not p.is_contiguous():
                raise RuntimeError(f"{n} must be contiguous")
        cnet = CNet()
        module._fill(cnet, byname)
        e = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        means, sc_o, ro_o, op_o = e(P, 3), e(P, 3), e(P, 4), e(P, 1)
        colors, dx, dshs, feat = e(P, 3), e(P, 3), e(P, 16, 3), e(P, 3)
        features = e(P, 32 * len(module.deformation_net.grid.grids))     # sampler -> decoder hand-over, kept for backward
        campos_ = campos.detach().to(device=dev, dtype=torch.float32).contiguous()
        fws = torch.empty(int(lib.s3g_deform_forward_workspace_bytes(C.byref(cnet))), dtype=torch.uint8, device=dev)
        # when a backward will follow, the decoder's hidden activations are kept for it (what autograd keeps for the
        # reference's nn.Sequential heads; opaque buffer, 256 B per Gaussian and hidden layer)
        nbytes = int(lib.s3g_deform_saved_bytes(C.byref(cnet), P)) if any(ctx.needs_input_grad) else 0
        acts = torch.empty(nbytes, dtype=torch.uint8, device=dev) if nbytes > 0 else None
        with torch.cuda.device(dev):
            _lib.check(lib.s3g_deform_forward_save(C.byref(cnet), P, _p(xyz_), _p(sc_), _p(ro_), _p(op_), _p(shs_),
                                                   float(time), _p(campos_), int(sh_degree), _p(means), _p(sc_o),
                                                   _p(ro_o), _p(op_o), _p(colors), _p(dx), _p(dshs), _p(feat), _p(features),
                                                   _p(acts), _p(fws), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                       "s3g_deform_forward_save")
        if raw_outputs:
            # forward_dynamic returns the un-activated values; with the default flags those are the inputs
            a = module.args
            if not (a.no_ds and a.no_dr and a.no_do):
                raise NotImplementedError("forward_dynamic with scale/rotation/opacity heads: use render_front()")
            sc_o, ro_o, op_o = sc_.clone(), ro_.clone(), op_.clone()
        ctx.module, ctx.time, ctx.sh_degree, ctx.raw, ctx.names = module, float(time), int(sh_degree), raw_outputs, names
        ctx.save_for_backward(xyz_, sc_, ro_, op_, shs_, campos_, features, acts, *[p.detach() for p in params])
        return means, sc_o, ro_o, op_o, colors, dx, dshs, feat

    @staticmethod
    def backward(ctx, g_means, g_sc, g_ro, g_op, g_col, g_dx, g_dshs, g_feat):
        lib = _lib.load()
        _warn_if_deterministic_requested()
        module = ctx.module
        xyz, sc, ro, op, shs, campos, features, acts, *params = ctx.saved_tensors     # acts is None only when P == 0
        dev = xyz.device
        P = xyz.shape[0]
        byname = dict(zip(ctx.names, params))
        gz = lambda g: None if g is None else g.to(torch.float32).contiguous()
        g_means, g_sc, g_ro, g_op, g_col, g_dx, g_dshs, g_feat = map(gz, (g_means, g_sc, g_ro, g_op, g_col, g_dx, g_dshs, g_feat))
        raw_sc = raw_ro = raw_op = None
        if ctx.raw:      # pass-through outputs: their gradient goes straight to the inputs
            raw_sc, raw_ro, raw_op, g_sc, g_ro, g_op = g_sc, g_ro, g_op, None, None, None
        e = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
        d_xyz, d_sc, d_ro, d_op, d_shs = e(P, 3), e(P, 3), e(P, 4), e(P, 1), e(P, 16, 3)
        pgrads = {}
        for n, p in byname.items():
            if n.startswith("grid."):
                pgrads[n] = torch.zeros_like(p, memory_format=torch.preserve_format)   # accumulated with atomics
            else:
                pgrads[n] = torch.empty_like(p)
        cnet, cg = CNet(), CNetGrads()
        module._fill(cnet, byname, grads=(cg, pgrads))
        ws = torch.empty(int(lib.s3g_deform_workspace_bytes(C.byref(cnet), P)), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.s3g_deform_backward_saved(C.byref(cnet), P, _p(xyz), _p(sc), _p(ro), _p(op), _p(shs), ctx.time,
                                                     _p(campos), ctx.sh_degree, _p(features), _p(acts), _p(g_means), _p(g_sc),
                                                     _p(g_ro), _p(g_op), _p(g_col), _p(g_dx), _p(g_dshs), _p(g_feat), _p(d_xyz),
                                                     _p(d_sc), _p(d_ro), _p(d_op), _p(d_shs), C.byref(cg), _p(ws),
                                                     C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)),
                       "s3g_deform_backward_saved")
        if ctx.raw:
            if raw_sc is not None:
                d_sc = d_sc + raw_sc
            if raw_ro is not None:
                d_ro = d_ro + raw_ro
            if raw_op is not None:
                d_op = d_op + raw_op
        return (None, None, None, None, None, d_xyz, d_sc, d_ro, d_op, d_shs, *[pgrads[n] for n in ctx.names])
