"""CPU: the buffer sizes the deformation stage asks for (forward workspace, kept activations, backward workspace)
for every head set and level count, pinned to known values, and the argument errors for an incomplete set of
Linear pointers.  All of it is host logic of libs3g_b200.so: no GPU is needed."""
import ctypes as C

import pytest
import torch

import ref_ext
from s3gaussian_b200.deformation import CNet, CNetGrads, deform_network

HEAD_SETS = {
    "default": dict(),                                            # no_ds / no_dr / no_do
    "all_heads": dict(no_ds=False, no_dr=False, no_do=False),
    "no_dx": dict(no_dx=True),
    "no_dshs": dict(no_dshs=True),
    "no_feat_head": dict(feat_head=False),
    "pos_only": dict(no_dshs=True, feat_head=False),
    "dino_only": dict(no_dx=True, no_dshs=True),
    "no_heads": dict(no_dx=True, no_dshs=True, feat_head=False),
}
RESO = (12, 10, 8, 6)
SIZES = (1, 333, 500_000)
# (heads, L): s3g_deform_forward_workspace_bytes, then s3g_deform_saved_bytes and s3g_deform_workspace_bytes for
# each P in SIZES; resolution RESO, multires 1..L
BYTES = {
    ("default", 1): [188928, 163840, 22803328, 491520, 22845824, 640122880, 86803200],
    ("default", 2): [205312, 163840, 24908288, 491520, 24993280, 640122880, 152908032],
    ("default", 3): [221696, 163840, 27017088, 491520, 27144576, 640122880, 219016704],
    ("default", 4): [238080, 163840, 29129728, 491520, 29299712, 640122880, 285129216],
    ("all_heads", 1): [311808, 262144, 36119424, 786432, 36161920, 1024196608, 100119296],
    ("all_heads", 2): [328192, 262144, 38224384, 786432, 38309376, 1024196608, 166224128],
    ("all_heads", 3): [344576, 262144, 40333184, 786432, 40460672, 1024196608, 232332800],
    ("all_heads", 4): [360960, 262144, 42445824, 786432, 42615808, 1024196608, 298445312],
    ("no_dx", 1): [147968, 131072, 18342784, 393216, 18385280, 512098304, 82342656],
    ("no_dx", 2): [164352, 131072, 20447744, 393216, 20532736, 512098304, 148447488],
    ("no_dx", 3): [180736, 131072, 22556544, 393216, 22684032, 512098304, 214556160],
    ("no_dx", 4): [197120, 131072, 24669184, 393216, 24839168, 512098304, 280668672],
    ("no_dshs", 1): [131584, 131072, 15348608, 393216, 15391104, 512098304, 79348480],
    ("no_dshs", 2): [147968, 131072, 17453568, 393216, 17538560, 512098304, 145453312],
    ("no_dshs", 3): [164352, 131072, 19562368, 393216, 19689856, 512098304, 211561984],
    ("no_dshs", 4): [180736, 131072, 21675008, 393216, 21844992, 512098304, 277674496],
    ("no_feat_head", 1): [115200, 98304, 14082944, 294912, 14125440, 384073728, 78082816],
    ("no_feat_head", 2): [131584, 98304, 16187904, 294912, 16272896, 384073728, 144187648],
    ("no_feat_head", 3): [147968, 98304, 18296704, 294912, 18424192, 384073728, 210296320],
    ("no_feat_head", 4): [164352, 98304, 20409344, 294912, 20579328, 384073728, 276408832],
    ("pos_only", 1): [57856, 65536, 6628224, 196608, 6670720, 256049152, 70628096],
    ("pos_only", 2): [74240, 65536, 8733184, 196608, 8818176, 256049152, 136732928],
    ("pos_only", 3): [90624, 65536, 10841984, 196608, 10969472, 256049152, 202841600],
    ("pos_only", 4): [107008, 65536, 12954624, 196608, 13124608, 256049152, 268954112],
    ("dino_only", 1): [90624, 98304, 10888064, 294912, 10930560, 384073728, 74887936],
    ("dino_only", 2): [107008, 98304, 12993024, 294912, 13078016, 384073728, 140992768],
    ("dino_only", 3): [123392, 98304, 15101824, 294912, 15229312, 384073728, 207101440],
    ("dino_only", 4): [139776, 98304, 17214464, 294912, 17384448, 384073728, 273213952],
    ("no_heads", 1): [16896, 32768, 2167680, 98304, 2210176, 128024576, 66167552],
    ("no_heads", 2): [33280, 32768, 4272640, 98304, 4357632, 128024576, 132272384],
    ("no_heads", 3): [49664, 32768, 6381440, 98304, 6508928, 128024576, 198381056],
    ("no_heads", 4): [66048, 32768, 8494080, 98304, 8664064, 128024576, 264493568],
}


def make(heads, L):
    return deform_network(ref_ext.ref_deform_args(RESO, tuple(range(1, L + 1)), **HEAD_SETS[heads]))


def c_structs(net, grads=False):
    byname = {n: p.detach() for n, p in net._named_hot_params()}
    cnet, cg = CNet(), CNetGrads()
    net._fill(cnet, byname, grads=(cg, {n: torch.zeros_like(p) for n, p in byname.items()}) if grads else None)
    return cnet, cg


@pytest.mark.parametrize("heads,L", list(BYTES), ids=[f"{h}-L{L}" for h, L in BYTES])
def test_buffer_sizes(heads, L, built_lib):
    cnet, _ = c_structs(make(heads, L))
    got = [int(built_lib.s3g_deform_forward_workspace_bytes(C.byref(cnet)))]
    for P in SIZES:
        got += [int(built_lib.s3g_deform_saved_bytes(C.byref(cnet), P)),
                int(built_lib.s3g_deform_workspace_bytes(C.byref(cnet), P))]
    assert got == BYTES[(heads, L)]


def backward_rc(lib, cnet, cg):
    """s3g_deform_backward_saved with P = 0: every argument check comes before its first CUDA call"""
    dummy = C.c_void_p(256)
    return lib.s3g_deform_backward_saved(C.byref(cnet), 0, *[None] * 5, 0.5, None, 3, None, None, *[None] * 8,
                                         *[None] * 5, C.byref(cg), dummy, None)


@pytest.mark.parametrize("field", ["w_feat", "b_feat", "w_pos1", "b_pos2", "w_shs2", "b_dino0", "w_dino4"])
def test_null_gradient_of_an_enabled_layer_is_an_argument_error(field, built_lib):
    cnet, cg = c_structs(make("default", 2), grads=True)
    setattr(cg, field, None)
    assert backward_rc(built_lib, cnet, cg) == -1
    assert b"null Linear gradient for an enabled layer" in built_lib.s3g_last_error()


@pytest.mark.parametrize("field,msg", [("b_feat", b"null feature_out"), ("b_pos1", b"incomplete head"),
                                       ("w_shs2", b"incomplete head"), ("b_dino4", b"incomplete dino head")])
def test_incomplete_layer_pointers_are_an_argument_error(field, msg, built_lib):
    cnet, _ = c_structs(make("default", 2))
    setattr(cnet, field, None)
    assert int(built_lib.s3g_deform_forward_workspace_bytes(C.byref(cnet))) == 0
    assert msg in built_lib.s3g_last_error()
