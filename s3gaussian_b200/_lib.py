"""ctypes binding of libs3g_b200.so (include/s3g_b200.h).

Loading fails loudly when the CUDA library has not been built: there is no CPU
or eager-PyTorch fallback anywhere in this package.
"""
from __future__ import annotations

import ctypes as C
import os

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "lib", "libs3g_b200.so")

ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_void_p, C.c_size_t)

S3G_OK = 0
ERR_NAMES = {-1: "S3G_ERR_ARG", -2: "S3G_ERR_CUDA", -3: "S3G_ERR_ALLOC", -4: "S3G_ERR_STATE"}

_lib = None

# every symbol include/s3g_b200.h declares: (name, restype, argtypes)
_F, _V, _I, _I64, _SZ, _D = C.c_float, C.c_void_p, C.c_int, C.c_int64, C.c_size_t, C.c_double
SIGNATURES = {
    "s3g_abi_version": (_I, []),
    "s3g_last_error": (C.c_char_p, []),
    "s3g_build_arch": (C.c_char_p, []),
    "s3g_mark_visible": (_I, [_I, _V, _V, _V, _V, _V]),
    "s3g_rasterize_forward": (_I64, [ALLOC_FN, _V, ALLOC_FN, _V, ALLOC_FN, _V, _I, _I, _I, _V, _I, _I,
                                      _V, _V, _V, _V, _V, _F, _V, _V, _V, _V, _V, _F, _F, _I, _V, _V,
                                      _V, _I, _V]),
    "s3g_rasterize_backward": (_I, [_I, _I, _I, _I64, _V, _I, _I, _V, _V, _V, _V, _F, _V, _V, _V, _V,
                                    _V, _F, _F, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V,
                                    _V, _V, _V, _I, _V]),
    "s3g_rasterize_forward_aux": (_I64, [ALLOC_FN, _V, ALLOC_FN, _V, ALLOC_FN, _V, _I, _I, _I, _V, _I, _I,
                                          _V, _V, _V, _V, _V, _F, _V, _V, _V, _V, _V, _F, _F, _I, _V, _V,
                                          _V, _I, _V, _V, _V]),
    "s3g_rasterize_backward_aux": (_I, [_I, _I, _I, _I64, _V, _I, _I, _V, _V, _V, _V, _F, _V, _V, _V, _V,
                                        _V, _F, _F, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V,
                                        _V, _V, _V, _I, _V, _V, _V]),
    "s3g_rasterize_forward_split": (_I64, [ALLOC_FN, _V, ALLOC_FN, _V, ALLOC_FN, _V, _I, _I, _I, _V, _I, _I,
                                            _V, _V, _V, _V, _V, _F, _V, _V, _V, _V, _V, _F, _F, _I, _V, _V,
                                            _V, _I, _V, _V, _V, _V, _V, _V]),
    "s3g_eval_metrics_workspace_bytes": (_SZ, [_I, _I, _I]),
    "s3g_eval_metrics": (_I, [_I, _I, _I, _V, _V, _V, _V, _V, _V]),
    "s3g_rasterize_backward_dp": (_I, [_I, _I, _I, _I64, _V, _I, _I, _V, _V, _V, _V, _F, _V, _V, _V, _V,
                                       _V, _F, _F, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V, _V,
                                       _V, _V, _V, _I, _V, _V]),
    "s3g_peer_reduce_gather": (_I, [_I, _I, _V, _V, _V, _I64, _I64, _V]),
    "s3g_state_field": (_I, [_I, C.c_char_p, _I64, _I64, _I, _I, C.POINTER(_SZ), C.POINTER(_SZ),
                             C.POINTER(_SZ)]),
    # struct pointers (s3g_deform_net / s3g_deform_net_grads) are passed with ctypes.byref()
    "s3g_deform_forward": (_I, [_V, _I] + [_V] * 5 + [_F, _V, _I] + [_V] * 9 + [_V, _V]),
    "s3g_deform_forward_workspace_bytes": (_SZ, [_V]),
    "s3g_deform_saved_bytes": (_SZ, [_V, _I]),
    "s3g_deform_forward_save": (_I, [_V, _I] + [_V] * 5 + [_F, _V, _I] + [_V] * 9 + [_V] + [_V, _V]),
    "s3g_deform_backward_saved": (_I, [_V, _I] + [_V] * 5 + [_F, _V, _I] + [_V, _V] + [_V] * 8 + [_V] * 5 + [_V, _V, _V]),
    "s3g_deform_workspace_bytes": (_SZ, [_V, _I]),
    "s3g_deform_backward": (_I, [_V, _I] + [_V] * 5 + [_F, _V, _I] + [_V] + [_V] * 8 + [_V] * 5 + [_V, _V, _V]),
    "s3g_umma_selftest": (_I, [_V, _V, _V, _I, _I, _I, _V]),
    "s3g_profile_enable": (_I, [_I]),
    "s3g_profile_read": (_I, [_I, _V, _I]),
    "s3g_profile_stage_name": (C.c_char_p, [_I, _I]),
    "s3g_geom_bytes": (_SZ, [_I64]),
    "s3g_binning_bytes": (_SZ, [_I64]),
    "s3g_image_bytes": (_SZ, [_I, _I]),
    "s3g_sort_temp_bytes": (_SZ, [_I64]),
    "s3g_sort_pairs_u32": (_I, [_I64, _V, _V, _V, _V, _I, _I, _V, _V]),
    # training-step kernels; s3g_adam_step takes a host array of AdamTensor (below)
    "s3g_adam_step": (_I, [_I, _V, _D, _D, _D, _V]),
    "s3g_densify_stats": (_I, [_I, _V, _V, _V, _V, _V, _V]),
    "s3g_image_loss_workspace_bytes": (_SZ, [_I, _I, _I, _I]),
    "s3g_image_loss_forward": (_I, [_I, _I, _I, _I, _V, _V, _V, _V, _F, _V, _V, _V]),
    "s3g_image_l1_depth_forward": (_I, [_I, _I, _I, _I, _V, _V, _V, _V, _F, _V, _V, _V]),
    "s3g_image_l1_depth_backward": (_I, [_I, _I, _I, _I, _V, _V, _V, _V, _F, _V, _V, _V, _V, _V]),
    "s3g_knn_workspace_bytes": (_SZ, [_I]),
    "s3g_knn_mean_dist2": (_I, [_I, _V, _V, _V, _V]),
    "s3g_peer_reduce_scatter": (_I, [_I, _I, _V, _I64, _V]),
    "s3g_peer_all_gather": (_I, [_I, _I, _V, _I64, _V]),
    "s3g_peer_nvls_all_reduce": (_I, [_I, _I, _V, _I64, _V]),
    "s3g_gather_rows": (_I, [_I, _V, _I64, _I64, _V, _V]),
    "s3g_plane_reg_workspace_bytes": (_SZ, [_I, _V]),
    "s3g_plane_reg_forward": (_I, [_I, _V, _V, _V, _V]),
    "s3g_plane_reg_backward": (_I, [_I, _V, _V, _V]),
    "s3g_image_loss_backward": (_I, [_I, _I, _I, _I, _V, _V, _V, _V, _F, _V, _V, _V, _V, _V, _V]),
}


class AdamTensor(C.Structure):
    """s3g_adam_tensor (include/s3g_b200.h)."""
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("numel", C.c_int64), ("lr", C.c_double), ("step", C.c_int64)]


def load():
    """Return the loaded library (builds nothing; see s3gaussian_b200.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -m s3gaussian_b200.build` "
            "(nvcc, sm_90a). s3gaussian_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.s3g_abi_version() != 1:
        raise RuntimeError("libs3g_b200.so ABI version mismatch; rebuild")
    _lib = lib
    return lib


def last_error() -> str:
    return load().s3g_last_error().decode()


def check(code: int, what: str) -> int:
    """status < 0 -> RuntimeError (the reference glue raises through AT_ERROR / std::runtime_error)."""
    if code < 0:
        raise RuntimeError(f"{what}: {ERR_NAMES.get(int(code), code)}: {last_error()}")
    return code


def state_field(buffer: int, name: str, P: int, R: int, W: int, H: int):
    off, eb, cnt = _SZ(), _SZ(), _SZ()
    check(load().s3g_state_field(buffer, name.encode(), P, R, W, H, C.byref(off), C.byref(eb),
                                 C.byref(cnt)), "s3g_state_field")
    return off.value, eb.value, cnt.value


def profile_enable(on: bool) -> None:
    load().s3g_profile_enable(1 if on else 0)


def profile_read(which: int) -> dict:
    """{stage name: milliseconds} of the last forward (0) / backward (1) call."""
    lib = load()
    buf = (C.c_float * 16)()
    n = check(lib.s3g_profile_read(which, buf, 16), "s3g_profile_read")
    return {lib.s3g_profile_stage_name(which, i).decode(): float(buf[i]) for i in range(n)}


class PeerSink(C.Structure):
    """s3g_peer_sink (include/s3g_b200.h)."""
    _fields_ = [("world", C.c_int), ("rank", C.c_int), ("chunk", C.c_int64), ("stage", C.c_void_p * 16),
                ("off_means3D", C.c_int64), ("off_shs", C.c_int64), ("off_opacities", C.c_int64),
                ("off_scales", C.c_int64), ("off_rotations", C.c_int64)]


class PlaneDesc(C.Structure):
    """s3g_plane_desc (include/s3g_b200.h)."""
    _fields_ = [("plane", C.c_void_p), ("grad", C.c_void_p), ("H", C.c_int), ("W", C.c_int), ("C", C.c_int),
                ("w_smooth", C.c_float), ("w_l1", C.c_float)]


class RowTensor(C.Structure):
    """s3g_row_tensor (include/s3g_b200.h)."""
    _fields_ = [("src", C.c_void_p), ("dst", C.c_void_p), ("row_floats", C.c_int), ("zero_new", C.c_int)]
