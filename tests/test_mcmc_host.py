"""CPU: 3DGS-MCMC's densification without a GPU - the float64 restatement (tests/mcmc_ref.py) on its defining properties
and closed forms, the single-sum form the kernel evaluates, argument errors of the two entry points before any launch,
the header in C, and the Python errors that need no device."""
import math
import os
import shutil
import subprocess

import pytest
import torch

import mcmc_ref as ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FAKE = 1 << 20    # never dereferenced: every call below fails validation before any launch

OPACITIES = torch.tensor([0.005, 0.0051, 0.01, 0.1, 0.3, 0.5, 0.7, 0.9, 0.99, 0.999, 1 - 1e-5, 1 - 2.0 ** -23],
                         dtype=torch.float64)


def _grid(ratios):
    o = OPACITIES.repeat(len(ratios))
    r = torch.tensor(ratios).repeat_interleave(OPACITIES.numel())
    return o, r


# ---- the restatement --------------------------------------------------------------------------------------------------
def test_one_draw_is_the_identity():
    o_new, op, D, N = ref.relocation64(OPACITIES, torch.ones(OPACITIES.numel(), dtype=torch.int64))
    assert torch.equal(N, torch.ones_like(N))
    torch.testing.assert_close(op, OPACITIES, rtol=1e-14, atol=0)
    torch.testing.assert_close(D, OPACITIES, rtol=1e-14, atol=0)          # s' = (o / D) s = s
    torch.testing.assert_close(o_new, OPACITIES.clamp(max=ref.O_MAX), rtol=1e-14, atol=0)


def test_n_copies_composite_to_the_original_opacity():
    """1 - (1 - o')^N = o before the clamp, for every N up to the cap."""
    o, r = _grid(list(range(1, 52)))
    _, op, _, N = ref.relocation64(o, r)
    torch.testing.assert_close(1.0 - (1.0 - op) ** N.double(), o, rtol=1e-12, atol=0)


def test_closed_forms_at_two_and_three():
    o, r = _grid([2, 3])
    _, op, D, _ = ref.relocation64(o, r)
    two, three = r == 2, r == 3
    torch.testing.assert_close(op[two], 1 - torch.sqrt(1 - o[two]), rtol=1e-14, atol=0)
    torch.testing.assert_close(op[three], 1 - (1 - o[three]) ** (1 / 3), rtol=1e-14, atol=0)
    x = op[two]
    torch.testing.assert_close(D[two], 2 * x - x ** 2 / math.sqrt(2), rtol=1e-14, atol=0)
    x = op[three]
    torch.testing.assert_close(D[three], 3 * x - 3 * x ** 2 / math.sqrt(2) + x ** 3 / math.sqrt(3), rtol=1e-14, atol=0)


def test_ratio_above_51_and_opacity_near_one_are_clamped():
    o = OPACITIES
    n = o.numel()
    at51 = ref.relocation64(o, torch.full((n,), 51))
    for r in (52, 60, 100):
        got = ref.relocation64(o, torch.full((n,), r))
        assert torch.equal(got[3], torch.full((n,), 51))
        for a, b in zip(got[:3], at51[:3]):
            assert torch.equal(a, b)
    near_one = torch.tensor([1 - 2.0 ** -30, 1 - 1e-12], dtype=torch.float64)
    o_new, op, _, _ = ref.relocation64(near_one, torch.ones(2, dtype=torch.int64))
    assert torch.equal(o_new, torch.full((2,), ref.O_MAX, dtype=torch.float64)) and bool((op > ref.O_MAX).all())
    # and the lower clamp: o = 0.006 split 3 ways is 0.002 < 0.005 per copy
    o_new, op, D, _ = ref.relocation64(torch.tensor([0.006], dtype=torch.float64), torch.tensor([3]))
    assert float(op) < 0.005 and float(o_new) == 0.005
    torch.testing.assert_close(D, 3 * op - 3 * op ** 2 / math.sqrt(2) + op ** 3 / math.sqrt(3), rtol=1e-14, atol=0)


def test_single_sum_form_of_the_kernel_equals_the_double_sum():
    """csrc/mcmc.cuh sums over i first: D = sum_m C(N,m) (-1)^(m-1) o'^m / sqrt(m)."""
    o, r = _grid([2, 3, 5, 8, 17, 33, 51])
    _, op, D, N = ref.relocation64(o, r)
    single = torch.zeros_like(op)
    for j in range(op.numel()):
        n, x = int(N[j]), float(op[j])
        single[j] = sum(math.comb(n, m) * (-1.0) ** (m - 1) * x ** m / math.sqrt(m) for m in range(1, n + 1))
    torch.testing.assert_close(single, D, rtol=1e-9, atol=0)


def test_plans_given_the_draws():
    o = torch.tensor([0.5, 0.001, 0.9, 0.005, 0.2])
    dead, idx, ratio = ref.plan_relocate(o, torch.tensor([2, 2]))
    assert dead.tolist() == [1, 3] and idx.tolist() == [0, 2, 2, 2, 4] and ratio.tolist() == [3, 3]
    n, idx, new, ratio = ref.plan_add(100, 1000, torch.tensor([7, 3, 7, 7, 0]))
    assert n == 5 and idx[100:].tolist() == [7, 3, 7, 7, 0] and new.tolist() == list(range(100, 105))
    assert ratio.tolist() == [4, 2, 4, 4, 2]
    assert ref.plan_add(100, 103, torch.tensor([1, 2, 3]))[0] == 3
    assert ref.plan_add(100, 90, torch.tensor([], dtype=torch.int64))[0] == 0


def test_noise_restatement_by_hand():
    """Identity rotation, s = (1, 2, 0.5): Sigma eps = (s^2 eps); o = 0.5 has gate 1 / (1 + exp(49.5))."""
    eps = torch.tensor([[1.0, 1.0, 1.0], [1.0, -2.0, 3.0]])
    scaling = torch.log(torch.tensor([[1.0, 2.0, 0.5], [1.0, 1.0, 1.0]], dtype=torch.float64))
    rot = torch.tensor([[2.0, 0.0, 0.0, 0.0], [math.cos(math.pi / 4), 0.0, 0.0, math.sin(math.pi / 4)]])
    opacity = torch.tensor([[0.0], [-20.0]])
    d = ref.noise64(scaling, rot, opacity, 3.0, eps)
    g = 1 / (1 + math.exp(49.5))
    torch.testing.assert_close(d[0], 3.0 * g * torch.tensor([1.0, 4.0, 0.25], dtype=torch.float64), rtol=1e-12, atol=0)
    gate = 1 / (1 + math.exp(-100 * ((1 - 1 / (1 + math.exp(20.0))) - 0.995)))
    torch.testing.assert_close(d[1], 3.0 * gate * eps[1].double(), rtol=1e-12, atol=1e-15)   # isotropic: R cancels


# ---- the C entry points ----------------------------------------------------------------------------------------------
def test_argument_errors_before_any_launch(built_lib):
    from s3gaussian_b200 import _lib
    lib = built_lib
    rt = (_lib.RowTensor * 33)(*[_lib.RowTensor(None, FAKE, 3, 1)] * 33)
    relocate = lambda n, src=FAKE, dst=FAKE, ratio=FAKE, mo=0.005, o=FAKE, s=FAKE, nz=1, z=rt: \
        lib.s3g_mcmc_relocate(n, src, dst, ratio, mo, o, s, nz, z, None)
    assert relocate(-1) == -1 and b"n < 0" in lib.s3g_last_error()
    assert relocate(0, None, None, None, 0.005, None, None, 0, None) == 0          # n == 0 does nothing
    for kw in ("src", "dst", "ratio", "o", "s"):
        assert relocate(4, **{kw: None}) == -1 and b"null pointer" in lib.s3g_last_error()
    assert relocate(4, nz=33) == -1 and b"0..32" in lib.s3g_last_error()
    assert relocate(4, nz=-1) == -1
    assert relocate(4, nz=2, z=None) == -1 and b"null descriptor array" in lib.s3g_last_error()
    bad = (_lib.RowTensor * 2)(_lib.RowTensor(None, FAKE, 3, 1), _lib.RowTensor(None, None, 3, 0))
    assert relocate(4, nz=2, z=bad) == -1 and b"null dst" in lib.s3g_last_error()
    bad[1] = _lib.RowTensor(None, FAKE, 0, 0)
    assert relocate(4, nz=2, z=bad) == -1 and b"row_floats" in lib.s3g_last_error()
    for mo in (0.0, 1.0, -0.1, float("nan")):
        assert relocate(4, mo=mo) == -1 and b"min_opacity" in lib.s3g_last_error()
    noise = lambda P, *ptrs: lib.s3g_mcmc_noise(P, *(ptrs or (FAKE,) * 5), 1.0, None)
    assert noise(-1) == -1 and b"P < 0" in lib.s3g_last_error()
    assert noise(0, None, None, None, None, None) == 0
    for k in range(5):
        ptrs = [FAKE] * 5
        ptrs[k] = None
        assert noise(8, *ptrs) == -1 and b"null pointer" in lib.s3g_last_error()
    assert noise(2 ** 31 // 4 + 1) == -1 and b"too large" in lib.s3g_last_error()


def test_header_declarations_compile_as_c(built_lib, tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("gcc not available")
    from s3gaussian_b200 import _lib
    src = tmp_path / "mcmc.c"
    src.write_text(r'''
#include <stdio.h>
#include "s3g_b200.h"
int main(void) {
    s3g_row_tensor z[1] = {{NULL, NULL, 3, 1}};
    if (s3g_mcmc_relocate(-1, NULL, NULL, NULL, 0.005f, NULL, NULL, 1, z, NULL) != S3G_ERR_ARG) return 1;
    if (s3g_mcmc_relocate(2, NULL, NULL, NULL, 0.005f, NULL, NULL, 1, z, NULL) != S3G_ERR_ARG) return 2;
    if (s3g_mcmc_noise(-1, NULL, NULL, NULL, NULL, NULL, 1.0f, NULL) != S3G_ERR_ARG) return 3;
    if (s3g_mcmc_noise(0, NULL, NULL, NULL, NULL, NULL, 1.0f, NULL) != S3G_OK) return 4;
    printf("mcmc c ok\n");
    return 0;
}
''')
    exe = tmp_path / "mcmc"
    libdir = os.path.dirname(_lib.LIB_PATH)
    r = subprocess.run([gcc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                        "-o", str(exe), "-L", libdir, "-ls3g_b200", f"-Wl,-rpath,{libdir}"], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    env = dict(os.environ)
    env["LD_LIBRARY_PATH"] = "/usr/local/cuda/lib64" + os.pathsep + env.get("LD_LIBRARY_PATH", "")
    assert subprocess.run([str(exe)], env=env).returncode == 0


# ---- Python ----------------------------------------------------------------------------------------------------------
def test_python_errors_without_a_device():
    from s3gaussian_b200 import mcmc
    from s3gaussian_b200.gaussian_model import GaussianModel
    o, s = torch.zeros(4, 1), torch.zeros(4, 3)
    i = torch.zeros(1, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="CUDA"):
        mcmc.relocate(o, s, i, i, i, 0.005)
    with pytest.raises(RuntimeError, match="CUDA"):
        mcmc.inject_noise(torch.zeros(4, 3), s, torch.zeros(4, 4), o, 1.0, torch.zeros(4, 3))
    g = GaussianModel(0)
    assert g.add_new_gs(100) == 0          # an empty model stays empty whatever the cap
