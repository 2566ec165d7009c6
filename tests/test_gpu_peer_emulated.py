"""GPU, one device: the view-parallel gradient exchange with W ranks emulated on one H100 - the peer kernels
(csrc/peer.cuh behind csrc/api_dp.cu), the DP instantiations of preprocess_backward_kernel that store each visible
Gaussian's gradients into the owner rank's staging slice, and the bucket layouts of dp.PeerAllReduce and
dp.FusedGradExchange.

The kernels take one plain device pointer per rank and never wait on remote state: the order between ranks comes
from the caller's barriers alone.  W buffers on one device, each rank's launch issued in turn on one stream, and
phase order (every rank's step k before any rank's step k+1) in place of the barriers therefore run the code a
W-GPU job runs; the ld.global.relaxed.sys loads and the plain stores do not care whether an address is local or
peer-mapped.  The oracle is the defined semantics: every element of the result is the float32 sum of the ranks'
values in rank order (s = v0; s += v1; ...), the same bits on every rank, and each rank's contribution is the
single-view backward that the rest of the suite checks against the CPU float64 oracle and the reference.

  * s3g_peer_reduce_scatter + s3g_peer_all_gather for W in {2, 3, 4, 5, 8, 16} (the <2>, <4>, <8> templates and
    the generic kernel) on data whose sum depends on the order: bitwise rank-order sums, nothing outside a rank's
    slice touched, empty and short slices, slices long enough for the all-gather's four-way unrolled loop and its
    tail; s3g_peer_reduce_gather on hand-filled staging areas, which it must leave zeroed;
  * dp.FusedGradExchange through the autograd path, with torch.distributed._symmetric_memory replaced by a fake
    that hands out the W emulated buffers: each rank's staged contribution against the plain backward of its view,
    the exchanged sums bitwise and within 1e-5 of float64, the staging re-zeroed over two steps, and the outputs
    that stay local (means2D, colors_precomp, absgrad, the camera gradients);
  * s3g_rasterize_backward with a hand-built s3g_peer_sink whose bucket order, gaps and chunk FusedGradExchange
    never produces;
  * bench.py's default path at N <= 3 (a plain gradient sink into a PeerAllReduce-sized buffer at unaligned
    offsets, then reduce-scatter and all-gather): under torch.use_deterministic_algorithms bitwise against the sum of
    the deterministic backwards run without a sink, and with the default backward.

Not covered here: the NVLS kernel (s3g_peer_nvls_all_reduce) and the multicast branch of peer_reduce_gather_kernel
need a multicast mapping of a symmetric allocation, which one GPU cannot provide.  tests/test_gpu_multi.py reaches
them on a box with two or more GPUs whose allocation has one.
"""
import ctypes as C
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import util

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
PEER_THREADS = 512          # csrc/peer.cuh
GUARD = 64                  # floats after every buffer that no kernel may touch
SENTINEL = 12345.0


@pytest.fixture(scope="module")
def lib(built_lib):
    return built_lib


@pytest.fixture(scope="module")
def ours(built_lib):
    from s3gaussian_b200 import diff_gaussian_rasterization as m
    return m


def _check(code, what):
    from s3gaussian_b200 import _lib
    _lib.check(code, what)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptrs(ts):
    return (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _all_zero_bits(t):
    return not bool(_bits(t).any())


def _rank_order_sum(vals):
    s = vals[0].clone()
    for v in vals[1:]:
        s += v
    return s


def _round4(n):
    return (n + 3) // 4 * 4


def _guarded(values):
    """A device buffer holding `values` followed by GUARD sentinel floats; -> (buffer, view of the first part)."""
    buf = torch.full((values.numel() + GUARD,), SENTINEL, dtype=torch.float32, device=DEV)
    buf[:values.numel()] = values
    return buf, buf[:values.numel()]


def _guard_intact(buf):
    return bool((buf[-GUARD:] == SENTINEL).all())


# ---- 1. collective kernels, bitwise -----------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _peer_grid(work4, sms):
    """api_dp.cu peer_grid: one thread per float4 of the work, at most four blocks per SM."""
    return max(1, min(-(-work4 // PEER_THREADS), sms * 4))


def _all_gather_stride(numel, world, sms):
    """Grid stride, in float4, of peer_all_gather_kernel as s3g_peer_all_gather launches it."""
    chunk4 = -(-(numel // 4) // world)
    per = max(1, _peer_grid(chunk4, sms) // (world - 1) * 2)
    return per * PEER_THREADS


def _long_slice_numel(world, sms):
    """A size whose full slices are more than four all-gather grid strides long and not a multiple of the stride
    (the unrolled loop and its tail both run), the last slice one float4 short."""
    chunk4 = sms * 4 * PEER_THREADS                # from here on the grid is at its cap: the stride stays put
    stride = _all_gather_stride(4 * world * chunk4, world, sms)
    if chunk4 <= 4 * stride or chunk4 % stride == 0:
        chunk4 = 4 * stride + stride // 2 + 1
    return 4 * (world * chunk4 - 1)


def _order_sensitive(numel, gen):
    """±1e8, 1 and N(0, 1) values: where ±1e8 and a small value meet, the float32 sum depends on the order."""
    pick = torch.randint(0, 4, (numel,), device=DEV, generator=gen, dtype=torch.int32)
    sign = torch.randint(0, 2, (numel,), device=DEV, generator=gen, dtype=torch.int32) * 2 - 1
    small = torch.randn(numel, device=DEV, generator=gen)
    return torch.where(pick < 2, sign * 1e8, torch.where(pick == 2, torch.ones_like(small), small))


WORLDS = [2, 3, 4, 5, 8, 16]


@pytest.mark.parametrize("world", WORLDS)
def test_reduce_scatter_then_all_gather_is_the_rank_order_sum(world, lib):
    from s3gaussian_b200 import dp
    sms = _sms()
    long_numel = _long_slice_numel(world, sms)
    stride4 = _all_gather_stride(long_numel, world, sms)
    long_slice4 = (dp.peer_slices(long_numel, world)[0][1]) // 4
    assert long_slice4 > 4 * stride4 and long_slice4 % stride4 != 0
    sizes = [4, 4 * (world - 1), 4 * (3 * world + 1), long_numel]
    gen = torch.Generator(device=DEV).manual_seed(1000 + world)
    differ = total = 0
    for numel in sizes:
        vals = [_order_sensitive(numel, gen) for _ in range(world)]
        want = _rank_order_sum(vals)
        differ += int((_bits(_rank_order_sum(vals[::-1])) != _bits(want)).sum())
        total += numel
        held = [_guarded(v) for v in vals]
        bufs = [h[1] for h in held]
        ptrs = _ptrs(bufs)
        for r in range(world):
            _check(lib.s3g_peer_reduce_scatter(world, r, ptrs, numel, _stream()), "s3g_peer_reduce_scatter")
        slices = dp.peer_slices(numel, world)
        assert slices[-1][1] == numel
        for r, (lo, hi) in enumerate(slices):
            assert _same_bits(bufs[r][lo:hi], want[lo:hi]), (world, numel, r, "reduced slice")
            assert _same_bits(bufs[r][:lo], vals[r][:lo]) and _same_bits(bufs[r][hi:], vals[r][hi:]), \
                (world, numel, r, "outside the slice")
        for r in range(world):
            _check(lib.s3g_peer_all_gather(world, r, ptrs, numel, _stream()), "s3g_peer_all_gather")
        for r in range(world):
            assert _same_bits(bufs[r], want), (world, numel, r, "after the all-gather")
            assert _guard_intact(held[r][0]), (world, numel, r, "guard")
        del vals, held, bufs, want
    # the data tells the rank order from its reverse (two terms add commutatively in float32: not at world 2)
    if world > 2:
        assert differ > 0.05 * total, (differ, total)


@pytest.mark.parametrize("world", WORLDS)
def test_reduce_gather_sums_staging_into_every_bucket_and_zeroes_it(world, lib):
    sms = _sms()
    cap4 = sms * 4 * PEER_THREADS
    gen = torch.Generator(device=DEV).manual_seed(2000 + world)
    cases = []
    for numel in (4, 4 * (world - 1), 4 * (3 * world + 1), 4 * 1003 * world + 8):
        c0 = _round4(-(-numel // world))
        cases += [(numel, c0), (numel, c0 + 4), (numel, _round4(numel) + 36)]
    cases.append((4 * (world * (cap4 + 777) - 1), 4 * (cap4 + 777)))    # a grid-stride loop over each slice
    for numel, chunk in cases:
        assert chunk % 4 == 0 and chunk * world >= numel
        contrib = [_order_sensitive(numel, gen) for _ in range(world)]
        want = _rank_order_sum(contrib)
        stages, before = [], []
        for r in range(world):
            lo = min(r * chunk, numel)
            n = min(numel - lo, chunk)
            st = torch.randn(world, chunk, device=DEV, generator=gen) + 7.0     # past `n`: never read, never zeroed
            for p in range(world):
                st[p, :n] = contrib[p][lo:lo + n]
            before.append(st.reshape(-1).clone())
            stages.append(_guarded(st.reshape(-1)))
        buckets = [_guarded(torch.full((numel,), float("nan"), device=DEV)) for _ in range(world)]
        bucket_ptrs = _ptrs([b[1] for b in buckets])
        for r in range(world):
            _check(lib.s3g_peer_reduce_gather(world, r, C.c_void_p(stages[r][1].data_ptr()), bucket_ptrs, None,
                                              numel, chunk, _stream()), "s3g_peer_reduce_gather")
        for r in range(world):
            assert _same_bits(buckets[r][1], want), (world, numel, chunk, r, "bucket")
            assert _guard_intact(buckets[r][0]), (world, numel, chunk, r, "bucket guard")
            lo = min(r * chunk, numel)
            n = min(numel - lo, chunk)
            exp = before[r].view(world, chunk).clone()
            exp[:, :n] = 0.0
            assert _same_bits(stages[r][1], exp.reshape(-1)), (world, numel, chunk, r, "staging")
            assert _guard_intact(stages[r][0]), (world, numel, chunk, r, "staging guard")
        del contrib, stages, before, buckets


# ---- 2. dp.FusedGradExchange through the autograd path ------------------------------------------------------------
class _Handle:
    def __init__(self, rank, world, ptrs):
        self.rank, self.world_size, self.buffer_ptrs, self.multicast_ptr = rank, world, ptrs, 0

    def barrier(self, channel=0):
        pass


class _EmulatedSymmetricMemory:
    """What dp.FusedGradExchange uses of torch.distributed._symmetric_memory, for `world` ranks on one device.  The
    first empty() allocates every rank's buffer (the sizes are symmetric) and each call returns the buffer of the
    rank being constructed (`rank`); rendezvous() hands out every rank's pointer and no multicast mapping."""

    def __init__(self, world):
        self.world, self.rank, self.buffers = world, 0, None

    def enable_symm_mem_for_group(self, name):
        pass

    def empty(self, *size, dtype=torch.float32, device=None):
        if self.buffers is None:
            self.buffers = [torch.empty(*size, dtype=dtype, device=device) for _ in range(self.world)]
        buf = self.buffers[self.rank]
        assert tuple(buf.shape) == tuple(size) and buf.dtype == dtype
        return buf

    def rendezvous(self, buffer, group):
        assert buffer is self.buffers[self.rank] and group.group_name == "emulated"
        return _Handle(self.rank, self.world, [b.data_ptr() for b in self.buffers])


def _exchanges(world, shapes, monkeypatch):
    """`world` dp.FusedGradExchange objects, one per emulated rank, over one fake symmetric allocation."""
    import torch.distributed._symmetric_memory  # noqa: F401  (the real module first; the attribute is then replaced)
    from s3gaussian_b200 import dp
    fake = _EmulatedSymmetricMemory(world)
    monkeypatch.setattr(torch.distributed, "_symmetric_memory", fake)
    monkeypatch.setattr(dp.dist, "get_world_size", lambda group=None: world)
    group = SimpleNamespace(group_name="emulated")
    exs = []
    for r in range(world):
        fake.rank = r
        ex = dp.FusedGradExchange(shapes, torch.device(DEV), group=group)
        assert ex.rank == r and ex.world == world and ex.mc == 0
        exs.append(ex)
    return exs


def _cloud_scene(P, seed, width, height):
    """make_cloud: a tenth of the Gaussians behind every camera below, more outside some of the frusta."""
    from s3gaussian_b200 import synthetic as syn
    cloud = syn.make_cloud(P, seed=seed, width=width, height=height)
    cams = [syn.make_camera(width, height, (0.06 * i, 0.3 * math.sin(i), 2.0 + 0.1 * math.cos(i)),
                            yaw_deg=7.0 * math.sin(1.3 * i)) for i in range(64)]
    return cloud, cams


def _small_scene(P, seed, width, height):
    """make_small_scene's blob cut to P Gaussians, keeping one of the rows behind the camera when P > 1."""
    from s3gaussian_b200 import synthetic as syn
    big, _ = syn.make_small_scene(P=64, width=width, height=height, seed=seed)   # rows 0..3 behind the camera
    rows = list(range(3, 3 + P)) if P > 1 else [10]
    cloud = syn.GaussianCloud(*(t[rows].clone() for t in (big.xyz, big.features_dc, big.features_rest, big.scaling,
                                                         big.rotation, big.opacity)))
    cams = [syn.make_camera(width, height, (0.03 * i, 0.4 * math.sin(i), 0.2 * math.cos(i)),
                            yaw_deg=6.0 * math.sin(1.7 * i), focal=0.9 * width) for i in range(64)]
    return cloud, cams


def _view_inputs(cloud, cam, mode, D, M):
    d = util.scene_inputs(cloud, cam, mode=mode, sh_degree=D)
    if mode == "sh":
        d["shs"] = d["shs"][:, :M].contiguous()
    return d


def _render_backward(ours, d, seed, extras):
    """forward + backward of one view through GaussianRasterizer under whatever gradient sink is installed: the
    view's radii, and the gradients of its inputs, of means2D and, with `extras`, means2D.absgrad and the camera
    tensors (viewmatrix / projmatrix / campos requiring grad)."""
    gc, gd = (g.to(DEV) for g in util.seeded_grads(d, seed))
    t = {k: d[k].to(DEV).clone().requires_grad_(True) for k in util.TENSOR_KEYS if d[k] is not None}
    m2d = torch.zeros_like(t["means3D"], requires_grad=True)
    rs = util.settings_for(ours, d, DEV)
    cam = {}
    if extras:
        cam = {k: getattr(rs, k).clone().requires_grad_(True) for k in ("viewmatrix", "projmatrix", "campos")}
        rs = rs._replace(**cam)
    color, radii, depth = ours.GaussianRasterizer(rs, absgrad=extras)(means2D=m2d, **t)
    ((color * gc).sum() + (depth * gd).sum()).backward()
    grads = {k: v.grad.detach().clone() for k, v in t.items()}
    grads["means2D"] = m2d.grad.detach().clone()
    if extras:
        grads["absgrad"] = m2d.absgrad.detach().clone()
        grads.update({k: v.grad.detach().clone() for k, v in cam.items()})
    return radii.detach(), grads


def _assert_close(got, ref, ref2, what):
    """Element-wise |got - ref| <= 1e-4 |ref| + atol, atol from the default backward's own run-to-run spread
    (util.grad_atol: its composite accumulates with unordered atomics); at most two elements of a tensor of 1000 or
    more outside, none of a smaller one."""
    got, ref, ref2 = (np.asarray(x.detach().cpu().numpy(), np.float64) for x in (got, ref, ref2))
    if ref.size == 0:
        return
    atol = util.grad_atol(ref, ref2)
    frac, worst, idx = util.elementwise(got, ref, 1e-4, atol)
    allowed = 2 if got.size >= 1000 else 0
    assert frac * got.size <= allowed + 1e-9, (what, frac, worst, idx, got.reshape(-1)[idx], ref.reshape(-1)[idx])


def _contributions(exs):
    """Each rank's contribution as it sits in the owners' staging areas: element e of rank r is
    stage_{e // chunk}[r * chunk + e % chunk]."""
    n, chunk, world = exs[0].numel, exs[0].chunk, exs[0].world
    stages = [ex.buffer[ex.stage_off:ex.stage_off + world * chunk].view(world, chunk) for ex in exs]
    out = []
    for r in range(world):
        c = torch.empty(n, dtype=torch.float32, device=DEV)
        for o in range(world):
            lo, hi = min(o * chunk, n), min((o + 1) * chunk, n)
            c[lo:hi] = stages[o][r, :hi - lo]
        out.append(c)
    return out


def _check_contribution(c, offsets, radii, plain_a, plain_b, what):
    """rank r's staged contribution: zero on the rows of Gaussians with radius 0 in its view and in the gaps of the
    bucket, its view's plain backward elsewhere."""
    covered = torch.zeros(c.numel(), dtype=torch.bool, device=DEV)
    hidden = radii <= 0
    for k, (o, cnt, shp) in offsets.items():
        got = c[o:o + cnt].view(shp)
        covered[o:o + cnt] = True
        assert _all_zero_bits(got[hidden]), (what, k, "rows of hidden Gaussians")
        _assert_close(got, plain_a[k], plain_b[k], (what, k))
    assert _all_zero_bits(c[~covered]), (what, "bucket gaps")


def _check_exchanged(buckets, contribs, offsets, plains, what):
    """After the reduce + gather: every bucket is the rank-order float32 sum of the contributions, bit for bit, within
    1e-5 (max-normalised) of their float64 sum, and within 1e-5 of the float64 sum of the ranks' plain backwards
    (`plains`: two runs per rank) plus the summed run-to-run spread of those backwards over the same scale: their
    composite accumulates with unordered atomics, so a staged contribution is its view's plain backward only to
    that spread."""
    want = _rank_order_sum(contribs)
    for r, b in enumerate(buckets):
        assert _same_bits(b, buckets[0]), (what, r, "buckets differ between ranks")
        assert _same_bits(b, want), (what, r, "bucket != rank-order sum of the contributions")
    for k, (o, cnt, shp) in offsets.items():
        got = buckets[0][o:o + cnt].double()
        exact64 = sum(c[o:o + cnt].double() for c in contribs)
        want64 = sum(p[0][k].double() for p in plains).reshape(-1)
        spread = sum(float((p[0][k].double() - p[1][k].double()).abs().max()) for p in plains)
        scale = float(want64.abs().max()) + 1e-30
        err_exact = float((got - exact64).abs().max()) / (float(exact64.abs().max()) + 1e-30)
        assert err_exact < 1e-5, (what, k, "vs float64 of the contributions", err_exact)
        err = float((got - want64).abs().max()) / scale
        assert err < 1e-5 + spread / scale, (what, k, "vs float64 of the plain backwards", err, spread / scale)


def _visibility_spread(radii_list):
    vis = torch.stack([r > 0 for r in radii_list]).sum(0)
    return int((vis == 0).sum()), int(((vis > 0) & (vis < len(radii_list))).sum())


FUSED_CASES = [
    # world, sh degree, SH coefficients (0: colors_precomp), P, absgrad + camera gradients
    (2, 3, 16, 20011, False), (3, 3, 16, 20011, True), (4, 3, 16, 20011, False), (8, 3, 16, 20011, True),
    (16, 3, 16, 20011, False),
    (3, 2, 9, 20011, True), (4, 2, 9, 20011, False),           # runtime M, scalar SH stores (L = 27)
    (3, 1, 4, 20011, False), (4, 1, 4, 20011, True),           # runtime M, float4 SH stores (L = 12)
    (3, 0, 1, 20011, True), (4, 0, 1, 20011, False),           # one coefficient (L = 3)
    (3, 0, 0, 20011, True), (4, 0, 0, 20011, False),           # colors_precomp: no shs in the bucket
    (16, 3, 16, 37, True), (16, 2, 9, 1, False),               # several owners with empty slices
]


@pytest.mark.parametrize("world,D,M,P,extras", FUSED_CASES)
def test_fused_exchange_two_steps(world, D, M, P, extras, ours, monkeypatch):
    """W FusedGradExchange objects on one fake symmetric allocation; per step, rank r installs its exchange and runs
    view r's forward + backward, then every rank calls finish().  Two steps with different views on the same
    exchanges, so a staging area that was not re-zeroed shows up in the second."""
    mode = "sh" if M else "rgb"
    width, height = 160, 112
    cloud, cams = (_cloud_scene if P > 1000 else _small_scene)(P, 11 + world, width, height)
    shapes = {"means3D": (P, 3), "opacities": (P, 1), "scales": (P, 3), "rotations": (P, 4)}
    if M:
        shapes["shs"] = (P, M, 3)
    exs = _exchanges(world, shapes, monkeypatch)
    offsets = exs[0].offsets
    for ex in exs[1:]:
        assert ex.offsets == offsets and ex.chunk == exs[0].chunk and ex.stage_off == exs[0].stage_off
    assert ("shs" in offsets) == bool(M) and exs[0].peer_sink_struct.off_shs == (offsets["shs"][0] if M else -1)
    local = ["means2D"] + (["colors_precomp"] if not M else []) + \
        (["absgrad", "viewmatrix", "projmatrix", "campos"] if extras else [])
    for step in range(2):
        views = [_view_inputs(cloud, cams[step * world + r], mode, D, M) for r in range(world)]
        seeds = [100 * step + r for r in range(world)]
        plain = [[_render_backward(ours, views[r], seeds[r], extras) for _ in range(2)] for r in range(world)]
        mine = []
        for r, ex in enumerate(exs):
            ex.install()
            try:
                mine.append(_render_backward(ours, views[r], seeds[r], extras))
            finally:
                ex.uninstall()
        torch.cuda.synchronize()
        radii = [m[0] for m in mine]
        for r in range(world):
            assert torch.equal(radii[r], plain[r][0][0]), (step, r, "radii")
        if P > 1000:
            nowhere, somewhere = _visibility_spread(radii)
            assert nowhere > 0 and somewhere > 0, (nowhere, somewhere)
        contribs = _contributions(exs)
        for r in range(world):
            what = (world, D, M, P, step, r)
            _check_contribution(contribs[r], offsets, radii[r], plain[r][0][1], plain[r][1][1], what)
            for k in local:
                _assert_close(mine[r][1][k], plain[r][0][1][k], plain[r][1][1][k], what + (k,))
        for ex in exs:
            ex.bucket.fill_(float("nan"))
        for ex in exs:
            ex.finish()
        torch.cuda.synchronize()
        _check_exchanged([ex.bucket for ex in exs], contribs, offsets, [(p[0][1], p[1][1]) for p in plain],
                         (world, step))
        for r, ex in enumerate(exs):
            assert _all_zero_bits(ex.buffer[ex.stage_off:]), (world, step, r, "staging not zeroed")


# ---- 3. a bucket layout FusedGradExchange never produces, through the C ABI ----------------------------------------
class _Ctx:
    def save_for_backward(self, *a):
        self.saved = a

    def mark_non_differentiable(self, *a):
        pass


def _forward_state(ours, d):
    E = torch.Tensor([])
    g = lambda k: d[k].to(DEV).contiguous() if d[k] is not None else E
    ctx = _Ctx()
    args = (ctx, g("means3D"), torch.zeros_like(g("means3D")), g("shs"), g("colors_precomp"), g("opacities"),
            g("scales"), g("rotations"), g("cov3D_precomp"), util.settings_for(ours, d, DEV))
    ours._RasterizeGaussians.forward(*args)
    ctx.inputs = args[1:8] + args[8:9]
    return ctx


def _c_backward(ours, ctx, d, seed, sink=None):
    """s3g_rasterize_backward (the default path) of one forward; every output NaN-filled on entry."""
    from s3gaussian_b200 import _lib
    lib = _lib.load()
    means3D, _, sh, colors_precomp, opacities, scales, rotations, cov3D = ctx.inputs
    P, M = means3D.shape[0], sh.size(1)
    e = lambda *s: torch.full(s, float("nan"), dtype=torch.float32, device=DEV)
    out = dict(means2D=e(P, 3), opacities=e(P, 1), colors=e(P, 3), means3D=e(P, 3), cov3D=e(P, 6), shs=e(P, M, 3),
               scales=e(P, 3), rotations=e(P, 4))
    out["means2D"].zero_()      # z is left untouched by contract
    gc, gd = (g.to(DEV).contiguous() for g in util.seeded_grads(d, seed))
    scene = ours._scene(util.settings_for(ours, d, DEV), means3D.device, means3D, sh, colors_precomp, None, scales,
                        rotations, cov3D)
    s = ctx.saved
    bwd = _lib.RasterBackwardArgs(
        R=ctx.num_rendered, radii=s[5].data_ptr(), geom_buffer=s[7].data_ptr(),
        binning_buffer=s[8].data_ptr() if s[8].numel() else None, image_buffer=s[9].data_ptr(),
        dL_dpix=gc.data_ptr(), dL_dpix_depth=gd.data_ptr(), dL_dmean2D=out["means2D"].data_ptr(),
        dL_dopacity=out["opacities"].data_ptr(), dL_dcolor=out["colors"].data_ptr(),
        dL_dmean3D=out["means3D"].data_ptr(), dL_dcov3D=out["cov3D"].data_ptr(), dL_dsh=out["shs"].data_ptr(),
        dL_dscale=out["scales"].data_ptr(), dL_drot=out["rotations"].data_ptr())
    if sink is not None:
        bwd.sink = C.pointer(sink)
    _check(lib.s3g_rasterize_backward(C.byref(scene), C.byref(bwd), _stream()), "s3g_rasterize_backward")
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("world,D,M", [(3, 3, 16), (4, 2, 9), (5, 1, 4)])
def test_hand_built_sink_with_a_scrambled_layout(world, D, M, ours, lib):
    """s3g_rasterize_backward with an s3g_peer_sink whose tensors sit in another order than dp's, with gaps, and whose
    chunk is larger than the layout needs: a mix-up between the off_* fields cannot cancel out here.  The exchanged
    tensors' local outputs stay untouched; dL_dmean2D and dL_dcolor are the plain backward's."""
    from s3gaussian_b200 import _lib
    P, width, height = 20011, 160, 112
    cloud, cams = _cloud_scene(P, 40 + world, width, height)
    shapes = {"rotations": (P, 4), "opacities": (P, 1), "shs": (P, M, 3), "scales": (P, 3), "means3D": (P, 3)}
    offsets, o = {}, 8
    for k, gap in zip(shapes, (12, 4, 16, 8, 20)):          # not dp's order, gaps of 4 to 20 floats
        cnt = math.prod(shapes[k])
        offsets[k] = (o, cnt, shapes[k])
        o = _round4(o + cnt) + gap
    numel = o
    chunk = _round4(-(-numel // world)) + 4 * 37                 # larger than the layout needs
    stages = [_guarded(torch.zeros(world * chunk, device=DEV)) for _ in range(world)]
    sink_of = []
    for r in range(world):
        s = _lib.PeerSink()
        s.world, s.rank, s.chunk = world, r, chunk
        for p in range(world):
            s.stage[p] = stages[p][1].data_ptr()
        s.off_means3D, s.off_shs, s.off_opacities = offsets["means3D"][0], offsets["shs"][0], offsets["opacities"][0]
        s.off_scales, s.off_rotations = offsets["scales"][0], offsets["rotations"][0]
        sink_of.append(s)
    plains, radii = [], []
    for r in range(world):
        d = _view_inputs(cloud, cams[r], "sh", D, M)
        ctx = _forward_state(ours, d)
        plain = [_c_backward(ours, ctx, d, 300 + r) for _ in range(2)]
        mine = _c_backward(ours, ctx, d, 300 + r, sink=sink_of[r])
        for k in ("means3D", "shs", "opacities", "scales", "rotations", "cov3D"):    # the exchanged tensors
            assert bool(torch.isnan(mine[k]).all()), (world, r, k, "written locally")
        for k in ("means2D", "colors"):                                             # the local ones
            _assert_close(mine[k], plain[0][k], plain[1][k], (world, r, k))
        plains.append(plain)
        radii.append(ctx.saved[5])
    for r in range(world):
        assert _guard_intact(stages[r][0]), (world, r, "staging guard")
    contribs = _contributions([SimpleNamespace(buffer=stages[o][1], stage_off=0, numel=numel, chunk=chunk,
                                               world=world) for o in range(world)])
    for r in range(world):
        _check_contribution(contribs[r], offsets, radii[r], plains[r][0], plains[r][1], (world, r))
    buckets = [_guarded(torch.full((numel,), float("nan"), device=DEV)) for _ in range(world)]
    bucket_ptrs = _ptrs([b[1] for b in buckets])
    for r in range(world):
        _check(lib.s3g_peer_reduce_gather(world, r, C.c_void_p(stages[r][1].data_ptr()), bucket_ptrs, None, numel,
                                          chunk, _stream()), "s3g_peer_reduce_gather")
    torch.cuda.synchronize()
    _check_exchanged([b[1] for b in buckets], contribs, offsets, plains, (world, "scrambled"))
    for r in range(world):
        assert _guard_intact(buckets[r][0]) and _guard_intact(stages[r][0]), (world, r, "guards")
        assert _all_zero_bits(stages[r][1]), (world, r, "staging not zeroed")


# ---- 4. bench.py's default N <= 3 path, end to end --------------------------------------------------------------
class _deterministic:
    def __init__(self, on=True):
        self.on = on

    def __enter__(self):
        self.prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
        torch.use_deterministic_algorithms(self.on)

    def __exit__(self, *exc):
        torch.use_deterministic_algorithms(self.prev[0], warn_only=self.prev[1])


@pytest.mark.parametrize("world,mode,det", [(2, "sh", True), (3, "sh", True), (3, "rgb", True), (3, "sh", False)])
def test_bench_default_exchange_is_the_rank_order_sum_of_the_backwards(world, mode, det, ours, lib):
    """bench.py at N <= 3: a plain callable sink (no peer_sink_struct) lays the tensors out back to back, offsets not
    rounded, in a buffer rounded up to 4 floats as dp.PeerAllReduce rounds it; then reduce-scatter and all-gather.
    At P = 20011 every tensor after means3D, rotations included, starts off a 16-byte boundary.  Under
    torch.use_deterministic_algorithms the sink path writes every element, bit for bit as the deterministic backward
    without a sink, and every buffer ends as the rank-order sum of those backwards, bit for bit.  With the default
    (atomic) backward bench.py times, each rank's buffer is its view's plain backward under the element-wise bar,
    and the exchanged buffers are the rank-order sum of what the ranks wrote, bit for bit."""
    P, width, height = 20011, 160, 112
    cloud, cams = _cloud_scene(P, 60 + world, width, height)
    views = [_view_inputs(cloud, cams[r], mode, 3, 16) for r in range(world)]
    names = ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations")
    offs, n_tot = {}, 0
    for k in names:
        if views[0][k] is not None:
            offs[k] = (n_tot, views[0][k].numel())
            n_tot += views[0][k].numel()
    numel = _round4(n_tot)
    assert numel > n_tot and offs["rotations"][0] % 4 != 0      # a rounded tail; an unaligned [P,4] gradient

    def flat(g):
        f = torch.zeros(numel, device=DEV)
        for k, (o, n) in offs.items():
            f[o:o + n] = g[k].reshape(-1)
        return f
    bufs = []
    with _deterministic(det):
        plains = [[flat(_render_backward(ours, views[r], 500 + r, False)[1]) for _ in range(1 if det else 2)]
                  for r in range(world)]
        for r in range(world):
            buf = torch.full((numel,), float("nan"), device=DEV)
            buf[n_tot:] = 0.0                               # PeerAllReduce's buffer starts zeroed

            def sink(name, shape, device, buf=buf):
                if name not in offs:
                    return None
                o, n = offs[name]
                return buf[o:o + n].view(shape)
            prev = ours.set_grad_sink(sink)
            try:
                _render_backward(ours, views[r], 500 + r, False)
            finally:
                ours.set_grad_sink(prev)
            torch.cuda.synchronize()
            if det:
                assert _same_bits(buf, plains[r][0]), (world, mode, r, "sink path != deterministic backward")
            else:
                for k, (o, n) in offs.items():
                    _assert_close(buf[o:o + n], plains[r][0][o:o + n], plains[r][1][o:o + n], (world, mode, r, k))
                assert _all_zero_bits(buf[n_tot:]), (world, mode, r, "tail")
            bufs.append(buf)
    want = _rank_order_sum(bufs)
    ptrs = _ptrs(bufs)
    for r in range(world):
        _check(lib.s3g_peer_reduce_scatter(world, r, ptrs, numel, _stream()), "s3g_peer_reduce_scatter")
    for r in range(world):
        _check(lib.s3g_peer_all_gather(world, r, ptrs, numel, _stream()), "s3g_peer_all_gather")
    for r in range(world):
        assert _same_bits(bufs[r], want), (world, mode, r)
