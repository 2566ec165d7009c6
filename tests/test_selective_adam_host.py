"""CPU: selective Adam without a GPU - the argument errors of s3g_adam_step_selective before any launch, the header
in C, and FusedAdam.step(visibility=...)'s checks, which raise before any state changes."""
import ctypes
import os
import shutil
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20    # never dereferenced: every call below fails validation before any launch


def _table(lib_mod, n, numel=12, step=1):
    return (lib_mod.AdamTensor * n)(*[lib_mod.AdamTensor(FAKE, FAKE, FAKE, FAKE, numel, 0.1, step)] * n)


def test_argument_errors_before_any_launch(built_lib):
    from s3gaussian_b200 import _lib
    lib = built_lib
    call = lambda n, t, w, rows, vis=FAKE: lib.s3g_adam_step_selective(
        n, t, None if w is None else (ctypes.c_int32 * len(w))(*w), rows, vis, 0.9, 0.999, 1e-15, None)
    t = _table(_lib, 2)
    assert call(-1, t, [3, 0], 4) == -1 and b"bad tensor table" in lib.s3g_last_error()
    assert call(2, None, [3, 0], 4) == -1 and b"bad tensor table" in lib.s3g_last_error()
    assert call(2, t, None, 4) == -1 and b"bad tensor table" in lib.s3g_last_error()
    assert call(2, t, [3, 0], -1) == -1 and b"rows < 0" in lib.s3g_last_error()
    assert call(2, t, [-3, 0], 4) == -1 and b"row_width < 0" in lib.s3g_last_error()
    # numel 12 is 4 rows of 3, not 5 rows of 3 nor 4 rows of 5 (12 % 5 != 0)
    assert call(2, t, [3, 0], 5) == -1 and b"numel == rows * row_width" in lib.s3g_last_error()
    assert call(2, t, [5, 0], 4) == -1 and b"numel == rows * row_width" in lib.s3g_last_error()
    assert call(2, t, [3, 0], 4, vis=None) == -1 and b"null visible" in lib.s3g_last_error()
    for field in ("param", "grad", "exp_avg", "exp_avg_sq"):
        bad = _table(_lib, 2)
        setattr(bad[1], field, None)
        assert call(2, bad, [3, 0], 4) == -1 and b"null pointer" in lib.s3g_last_error()
    assert call(2, _table(_lib, 2, step=0), [3, 0], 4) == -1 and b"step < 1" in lib.s3g_last_error()
    assert call(2, _table(_lib, 2, numel=-4), [0, 0], 4) == -1 and b"negative numel" in lib.s3g_last_error()
    big = _table(_lib, 1, numel=2 ** 31)
    assert call(1, big, [2], 2 ** 30) == -1 and b"2^31" in lib.s3g_last_error()
    # an error in the 41st tensor is found before the first launch (the first 40 would form one launch)
    many = _table(_lib, 41)
    many[40].grad = None
    assert call(41, many, [3] * 41, 4) == -1 and b"null pointer" in lib.s3g_last_error()
    # nothing to do: no tensors, empty tensors (with NULL pointers), or only masked tensors of zero rows
    assert call(0, None, None, 0, None) == 0
    empty = (_lib.AdamTensor * 2)(*[_lib.AdamTensor(None, None, None, None, 0, 0.1, 0)] * 2)
    assert call(2, empty, [3, 0], 0, None) == 0


def test_header_declaration_compiles_as_c(built_lib, tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    from s3gaussian_b200 import _lib
    src = tmp_path / "selective.c"
    src.write_text(r'''
#include <stdio.h>
#include "s3g_b200.h"
int main(void) {
    s3g_adam_tensor t[2] = {{NULL, NULL, NULL, NULL, 12, 0.1, 1}, {NULL, NULL, NULL, NULL, 0, 0.1, 1}};
    int32_t w[2] = {3, 0};
    if (s3g_adam_step_selective(-1, t, w, 4, NULL, 0.9, 0.999, 1e-15, NULL) != S3G_ERR_ARG) return 1;
    if (s3g_adam_step_selective(2, t, w, -1, NULL, 0.9, 0.999, 1e-15, NULL) != S3G_ERR_ARG) return 2;
    if (s3g_adam_step_selective(2, t, w, 5, NULL, 0.9, 0.999, 1e-15, NULL) != S3G_ERR_ARG) return 3;
    if (s3g_adam_step_selective(2, t, w, 4, NULL, 0.9, 0.999, 1e-15, NULL) != S3G_ERR_ARG) return 4;
    t[0].numel = 0;
    if (s3g_adam_step_selective(2, t, w, 0, NULL, 0.9, 0.999, 1e-15, NULL) != S3G_OK) return 5;
    printf("selective adam c ok\n");
    return 0;
}
''')
    exe = tmp_path / "selective"
    libdir = os.path.dirname(_lib.LIB_PATH)
    r = subprocess.run([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                        "-o", str(exe), "-L", libdir, "-ls3g_b200", f"-Wl,-rpath,{libdir}"], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = "/usr/local/cuda/lib64" + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    r = subprocess.run([str(exe)], env=env, capture_output=True, text=True)
    assert r.returncode == 0 and "selective adam c ok" in r.stdout, (r.returncode, r.stdout, r.stderr)


# ---- Python ----------------------------------------------------------------------------------------------------------
def _opt(P=5, with_dense=True, selective=("xyz", "opacity")):
    xyz = torch.nn.Parameter(torch.randn(P, 3))
    opa = torch.nn.Parameter(torch.randn(P, 1))
    groups = [{"params": [xyz], "lr": 0.1, "name": "xyz"}, {"params": [opa], "lr": 0.1, "name": "opacity"}]
    if with_dense:
        groups.append({"params": [torch.nn.Parameter(torch.randn(4, 4))], "lr": 0.1, "name": "deformation"})
    from s3gaussian_b200.optim import FusedAdam
    opt = FusedAdam(groups, lr=0.0, eps=1e-15, selective_groups=selective)
    for g in opt.param_groups:
        for p in g["params"]:
            p.grad = torch.randn_like(p)
    return opt


def _unchanged(opt, before):
    params = [p for g in opt.param_groups for p in g["params"]]
    return len(opt.state) == 0 and all(torch.equal(p, b) for p, b in zip(params, before))


@pytest.mark.parametrize("bad, match", [
    (torch.ones(5, dtype=torch.uint8), "bool"),
    (torch.ones(5), "bool"),
    (torch.ones(5, 1, dtype=torch.bool), "1-D"),
    (torch.ones(10, dtype=torch.bool)[::2], "contiguous"),
    ([True] * 5, "bool"),
    (torch.ones(4, dtype=torch.bool), "rows"),
    (torch.ones(6, dtype=torch.bool), "rows"),
])
def test_bad_visibility_raises_before_anything_changes(bad, match):
    opt = _opt()
    before = [p.detach().clone() for g in opt.param_groups for p in g["params"]]
    with pytest.raises(RuntimeError, match=match):
        opt.step(visibility=bad)
    assert _unchanged(opt, before)


def test_visibility_needs_a_per_gaussian_group():
    for sel in ((), ("f_rest",)):
        opt = _opt(selective=sel)
        before = [p.detach().clone() for g in opt.param_groups for p in g["params"]]
        with pytest.raises(RuntimeError, match="no per-Gaussian group"):
            opt.step(visibility=torch.ones(5, dtype=torch.bool))
        assert _unchanged(opt, before)


def test_rows_are_checked_only_where_there_is_a_gradient():
    """After densify / prune the per-Gaussian tensors are new ones without a gradient, while the mask has the old P.
    Then only the dense group is stepped, so the size check passes and the CPU parameter is what stops the step."""
    opt = _opt()
    for g in opt.param_groups[:2]:
        g["params"][0].grad = None
    with pytest.raises(RuntimeError, match="CUDA float32 parameters only"):
        opt.step(visibility=torch.ones(3, dtype=torch.bool))
    assert len(opt.state) == 0


def test_visibility_on_another_device_than_the_parameters():
    opt = _opt()
    with pytest.raises(RuntimeError, match="device"):
        opt.step(visibility=torch.ones(5, dtype=torch.bool, device="meta"))
    assert len(opt.state) == 0


def test_selective_groups_are_names_and_survive_load_state_dict():
    from s3gaussian_b200.optim import FusedAdam
    with pytest.raises(TypeError):
        FusedAdam([torch.nn.Parameter(torch.zeros(2))], selective_groups="xyz")
    opt = _opt()
    ref = torch.optim.Adam([{"params": [torch.nn.Parameter(torch.zeros(5, 3))], "lr": 0.2, "name": "xyz"},
                            {"params": [torch.nn.Parameter(torch.zeros(5, 1))], "lr": 0.2, "name": "opacity"},
                            {"params": [torch.nn.Parameter(torch.zeros(4, 4))], "lr": 0.2, "name": "deformation"}])
    sd = opt.state_dict()
    assert set(sd) == {"state", "param_groups"} and "selective_groups" not in sd["param_groups"][0]
    opt.load_state_dict(ref.state_dict())
    assert opt.selective_groups == {"xyz", "opacity"} and opt.param_groups[0]["lr"] == 0.2
