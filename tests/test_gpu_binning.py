"""GPU: the forward's binning checked exactly against the integer restatement in tests/binning_ref.py.

Each case runs one forward, reads the preprocess outputs the binning starts from (depth_key, rect, tiles_touched)
and everything it produces (the depth order, the offsets, the instance count, point_list, the tile ranges), and
recomputes the latter from the former in numpy.  No oracle preprocess is involved, so every integer is compared
with no tolerance.  The cases are chosen to reach the size-selected paths of the binning - the shared-memory and
global tile histograms, two and three tile-sort passes, the grid-barrier and ticket scans, the tile sort bounded by
a device-side count - and the layouts where a sort goes wrong first: depth ties across sort blocks, one Gaussian
with a very long emit segment, one tile whose list spans more than the look-back window.  Each case asserts the
size that puts it in its regime.
"""
import threading

import numpy as np
import pytest
import torch

import binning_ref as br
import ref_ext
import util

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
TOL = 1e-4
SORT_TILE = 4096           # items per onesweep block (radix_sort.cuh)
LOOKBACK_WINDOW = 8        # predecessor blocks one look-back round reads
SCAN_TILE = 2048           # items per scan block
SCAN_BLOCKS_PER_SM = 8     # 256-thread scan blocks: at most 2048 / 256 resident per SM
SMEM_DEFAULT = 48 * 1024   # dynamic shared memory without the opt-in
SMEM_OPT_IN_LIMIT = 64 * 1024   # largest tile histogram the emit kernel keeps in shared memory


@pytest.fixture(scope="module")
def ours(built_lib):
    from s3gaussian_b200 import diff_gaussian_rasterization as m
    return m


# ---------------------------------------------------------------------------------------------------- scenes
def scene(u, v, z, r_px, W, H, seed, focal=None):
    """Isotropic Gaussians centred on pixel (u, v) at view depth z with a screen radius of about r_px pixels, seen by
    an axis-aligned camera at the origin looking down +x (view z == world x exactly).  rgb colours, opacity in
    [0.1, 0.9]."""
    from s3gaussian_b200 import synthetic as syn
    P = len(u)
    f = float(focal if focal is not None else max(W, H) / 2)
    rng = np.random.default_rng(seed)
    z = np.asarray(z, np.float64)
    cx = (np.asarray(u, np.float64) - W / 2) / f * np.abs(z)
    cy = (np.asarray(v, np.float64) - H / 2) / f * np.abs(z)
    xyz = np.stack([z, -cx, -cy], 1).astype(np.float32)
    # screen sigma = s * f / z; the radius is 3 sigma (plus the 0.3 px^2 low-pass)
    s = (np.asarray(r_px, np.float64) / 3.0 * np.abs(z) / f).astype(np.float32)
    cam = syn.make_camera(W, H, (0.0, 0.0, 0.0), focal=f)
    rot = np.zeros((P, 4), np.float32)
    rot[:, 0] = 1.0
    d = dict(means3D=torch.from_numpy(xyz), opacities=torch.from_numpy(rng.uniform(0.1, 0.9, (P, 1)).astype(np.float32)),
             scales=torch.from_numpy(np.repeat(s[:, None], 3, 1)), rotations=torch.from_numpy(rot), shs=None,
             colors_precomp=torch.from_numpy(rng.uniform(0.0, 1.0, (P, 3)).astype(np.float32)), cov3D_precomp=None,
             viewmatrix=cam.world_view_transform.clone(), projmatrix=cam.full_proj_transform.clone(),
             campos=cam.camera_center.clone(), bg=torch.tensor((0.1, 0.2, 0.3)), W=W, H=H, tanfovx=cam.tanfovx,
             tanfovy=cam.tanfovy, sh_degree=0)
    return d


def random_scene(P, W, H, seed, r_px=(3.0, 24.0), depth=(2.0, 12.0), culled=True, focal=None):
    """P Gaussians spread over (a little more than) the image; with `culled`, every 7th is behind the camera and every
    11th far off screen (tiles_touched = 0), interleaved with the visible ones."""
    rng = np.random.default_rng(seed)
    u = rng.uniform(-0.1 * W, 1.1 * W, P)
    v = rng.uniform(-0.1 * H, 1.1 * H, P)
    z = rng.uniform(*depth, P)
    r = rng.uniform(*r_px, P)
    if culled:
        i = np.arange(P)
        z = np.where(i % 7 == 3, -z, z)
        u = np.where(i % 11 == 5, -4.0 * W - 1000.0, u)
    return scene(u, v, z, r, W, H, seed, focal)


# ---------------------------------------------------------------------------------------------- the forward
class _Ctx:
    def save_for_backward(self, *a):
        self.saved = a

    def mark_non_differentiable(self, *a):
        pass


GEOM_FIELDS = (("depth_key", np.uint32), ("rect", np.uint16), ("tiles_touched", np.uint32), ("order", np.uint32),
               ("offsets", np.uint32), ("rgb", np.float32))


def forward_state(ours, d):
    """One forward through the autograd Function (util.ours_forward_state's pattern) -> dict of numpy arrays: the
    preprocess outputs the binning reads, everything it writes, n_contrib, radii, colour, and R.  Only the fields
    are copied to the host, not the whole state buffers."""
    from s3gaussian_b200 import _lib
    E = torch.Tensor([])
    g = lambda k: d[k].to(DEV).contiguous() if d[k] is not None else E
    ctx = _Ctx()
    with torch.no_grad():
        color, radii, _ = ours._RasterizeGaussians.forward(
            ctx, g("means3D"), torch.zeros_like(g("means3D")), g("shs"), g("colors_precomp"), g("opacities"),
            g("scales"), g("rotations"), g("cov3D_precomp"), util.settings_for(ours, d, DEV))
    torch.cuda.synchronize()
    R = ctx.num_rendered
    P, W, H = d["means3D"].shape[0], d["W"], d["H"]
    bufs = {0: ctx.saved[7], 1: ctx.saved[8], 2: ctx.saved[9]}

    def view(bid, name, dt):
        off, eb, cnt = _lib.state_field(bid, name, P, R, W, H)
        buf = bufs[bid]
        if cnt == 0:
            return np.zeros(0, dt)
        a = ((buf.data_ptr() + 127) & ~127) - buf.data_ptr() + off
        return buf[a:a + eb * cnt].cpu().numpy().view(dt)

    s = {name: view(0, name, dt) for name, dt in GEOM_FIELDS}
    s["rect"] = s["rect"].reshape(-1, 4)
    s["rgb"] = s["rgb"].reshape(-1, 4)
    s["point_list"] = view(1, "point_list", np.uint32) if R > 0 else np.zeros(0, np.uint32)
    s["ranges"] = view(2, "ranges", np.uint32).reshape(-1, 2)
    s["n_contrib"] = view(2, "n_contrib", np.uint32)
    s.update(R=R, radii=radii.cpu().numpy(), color=color.cpu().numpy(), W=W, H=H)
    del ctx
    return s


def check_binning(s):
    """Every integer of the binning equals the restatement; returns the restatement."""
    W, H = s["W"], s["H"]
    gx, gy = br.grid_of(W, H)
    n_tiles = gx * gy
    key, rect = s["depth_key"], s["rect"].astype(np.int64)
    vis = key != br.DEPTH_KEY_INVISIBLE
    np.testing.assert_array_equal(vis, s["radii"] > 0)
    assert np.all(rect[vis, 2] <= gx) and np.all(rect[vis, 3] <= gy)
    area = (rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1])
    assert np.all(area[vis] > 0)
    np.testing.assert_array_equal(s["tiles_touched"][vis], area[vis])
    assert not np.any(s["tiles_touched"][~vis])
    np.testing.assert_array_equal(key[vis], s["rgb"][vis, 3].view(np.uint32))
    ref = br.binning(key, rect, gx, n_tiles)
    assert s["R"] == ref["R"]
    np.testing.assert_array_equal(s["order"], ref["order"])
    np.testing.assert_array_equal(s["offsets"], ref["offsets"])
    np.testing.assert_array_equal(s["point_list"], ref["point_list"])
    assert s["ranges"].shape == (n_tiles, 2)
    np.testing.assert_array_equal(s["ranges"], ref["ranges"])
    lens = s["ranges"][:, 1].astype(np.int64) - s["ranges"][:, 0].astype(np.int64)
    assert not np.any(s["ranges"][lens == 0])          # empty tiles are (0, 0)
    per_pixel = lens.reshape(gy, gx)[np.arange(H) // 16][:, np.arange(W) // 16]
    assert np.all(s["n_contrib"].reshape(H, W) <= per_pixel)
    return ref


def run_and_check(ours, d):
    s = forward_state(ours, d)
    ref = check_binning(s)
    return s, ref


# ---------------------------------------------------------------------------------------- tile-count regimes
# (W, H, tiles, key bits, tile-sort passes, emit histogram path)
REGIMES = [
    (1, 1, 1, 1, 1, "shared"),              # single tile
    (17, 1, 2, 2, 1, "shared"),             # ragged last tile column
    (256, 256, 256, 9, 2, "shared"),        # last pass 1 bit wide
    (1920, 1280, 9_600, 14, 2, "shared"),
    (2048, 1536, 12_288, 14, 2, "shared"),  # exactly 48 KB: the default shared-memory limit
    (2064, 1552, 12_513, 14, 2, "opt-in"),  # needs the > 48 KB opt-in
    (2048, 2048, 16_384, 15, 2, "opt-in"),  # exactly 64 KB
    (2064, 2048, 16_512, 15, 2, "global"),  # one tile row past 64 KB: global-memory histogram
    (4080, 4112, 65_535, 16, 2, "global"),
    (4096, 4096, 65_536, 17, 3, "global"),  # 17 key bits: three tile-sort passes
    (4112, 4112, 66_049, 17, 3, "global"),
    (16, 1_048_560, 65_535, 16, 2, "global"),   # a strip one tile wide and 65 535 tiles tall
]


def emit_path(n_tiles):
    b = 4 * n_tiles
    return "shared" if b <= SMEM_DEFAULT else "opt-in" if b <= SMEM_OPT_IN_LIMIT else "global"


@pytest.mark.parametrize("W,H,tiles,bits,passes,path", REGIMES, ids=[f"{r[0]}x{r[1]}" for r in REGIMES])
def test_tile_count_regimes(W, H, tiles, bits, passes, path, ours):
    gx, gy = br.grid_of(W, H)
    assert gx * gy == tiles
    assert br.key_bits(tiles) == bits and -(-bits // 8) == passes
    assert emit_path(tiles) == path
    P = 1 if tiles == 1 else 4000
    d = random_scene(P, W, H, seed=tiles, r_px=(3.0, 40.0))
    s, ref = run_and_check(ours, d)
    assert ref["R"] > 0
    if tiles > 1:
        assert np.count_nonzero(ref["ranges"][:, 1] > ref["ranges"][:, 0]) > 1


def test_image_too_tall_for_the_tile_grid_is_refused(ours):
    """65 536 tile rows do not fit the 16-bit rect and the launch grid: the forward refuses the call before it
    launches anything (no kernel and no memset of this library in the profile)."""
    W, H = 16, 65_536 * 16
    d = random_scene(64, W, H, seed=3)
    t = {k: d[k].to(DEV) for k in ("means3D", "opacities", "scales", "rotations", "colors_precomp")}
    m2d = torch.zeros_like(t["means3D"])
    rast = ours.GaussianRasterizer(util.settings_for(ours, d, DEV))
    sentinel = torch.zeros(16, device=DEV)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        with torch.no_grad(), pytest.raises(RuntimeError, match="image too large"):
            rast(means3D=t["means3D"], means2D=m2d, opacities=t["opacities"], scales=t["scales"],
                 rotations=t["rotations"], colors_precomp=t["colors_precomp"])
        sentinel.add_(1.0)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert names, "the profile recorded no device activity at all (not even the sentinel kernel)"
    assert not any("s3g" in n or "emset" in n for n in names), names


# ------------------------------------------------------------------------------- Gaussian counts at block edges
EDGE_P = [1, 31, 32, 33, 511, 512, 513, 2047, 2048, 2049, 4095, 4096, 4097, 8 * 4096 + 1, 9 * 4096]


@pytest.mark.parametrize("P", EDGE_P)
def test_gaussian_counts_at_block_edges(P, ours):
    d = random_scene(P, 320, 240, seed=P)
    s, ref = run_and_check(ours, d)
    assert s["depth_key"].shape[0] == P
    culled = int(np.count_nonzero(s["depth_key"] == br.DEPTH_KEY_INVISIBLE))
    if P >= 12:   # culled Gaussians behind the camera (index 3 mod 7) and off screen (5 mod 11) among visible ones
        assert 0 < culled < P and float(d["means3D"][:, 0].min()) < 0
    if P > LOOKBACK_WINDOW * SORT_TILE:
        assert -(-P // SORT_TILE) > LOOKBACK_WINDOW


# ---------------------------------------------------------------------------------------- adversarial layouts
def test_every_gaussian_at_one_depth(ours):
    """All depth keys equal: the depth sort must keep index order across 10 onesweep blocks (more than the
    look-back window), and every tile's list is in index order."""
    P, W, H = 40_000, 640, 480
    rng = np.random.default_rng(61)
    d = scene(rng.uniform(0, W, P), rng.uniform(0, H, P), np.full(P, 5.0), rng.uniform(3, 30, P), W, H, 61)
    s, ref = run_and_check(ours, d)
    vis = s["depth_key"] != br.DEPTH_KEY_INVISIBLE
    assert np.count_nonzero(vis) == P and np.unique(s["depth_key"]).size == 1
    assert -(-P // SORT_TILE) > LOOKBACK_WINDOW
    np.testing.assert_array_equal(s["order"], np.arange(P))


def test_a_few_distinct_depths(ours):
    P, W, H = 50_000, 800, 600
    rng = np.random.default_rng(62)
    z = rng.choice(np.array([3.0, 5.5, 9.25]), P)
    d = scene(rng.uniform(0, W, P), rng.uniform(0, H, P), z, rng.uniform(3, 30, P), W, H, 62)
    s, ref = run_and_check(ours, d)
    assert np.unique(s["depth_key"]).size == 3


def test_one_gaussian_covering_every_tile_among_tiny_ones(ours):
    """One warp's emit segment is the whole tile grid (3 072 instances) while its neighbours emit one to four."""
    P, W, H, big = 6000, 1024, 768, 2500
    rng = np.random.default_rng(63)
    u, v, z, r = rng.uniform(0, W, P), rng.uniform(0, H, P), rng.uniform(2, 12, P), np.full(P, 0.3)
    u[big], v[big], z[big], r[big] = W / 2, H / 2, 6.0, 2.0 * (W + H)
    d = scene(u, v, z, r, W, H, 63)
    s, ref = run_and_check(ours, d)
    gx, gy = br.grid_of(W, H)
    assert int(s["tiles_touched"][big]) == gx * gy
    assert int(np.sort(s["tiles_touched"])[-2]) <= 4


def test_one_tile_holding_more_than_100k_instances(ours):
    """120 000 Gaussians inside one tile, at 16 depths: that tile's list spans 30 onesweep blocks of the tile sort
    (more than the look-back window) and is full of depth ties."""
    W, H, tx, ty = 512, 384, 13, 9
    n_dense, n_rest = 120_000, 5000
    rng = np.random.default_rng(64)
    u = np.concatenate([tx * 16 + rng.uniform(5.5, 11.5, n_dense), rng.uniform(0, W, n_rest)])
    v = np.concatenate([ty * 16 + rng.uniform(5.5, 11.5, n_dense), rng.uniform(0, H, n_rest)])
    z = np.concatenate([rng.choice(np.linspace(3.0, 9.0, 16), n_dense), rng.uniform(2, 12, n_rest)])
    r = np.concatenate([np.full(n_dense, 0.3), rng.uniform(3, 30, n_rest)])
    perm = rng.permutation(n_dense + n_rest)       # the dense tile's Gaussians interleaved with the others
    d = scene(u[perm], v[perm], z[perm], r[perm], W, H, 64)
    s, ref = run_and_check(ours, d)
    gx, _ = br.grid_of(W, H)
    lens = ref["ranges"][:, 1].astype(np.int64) - ref["ranges"][:, 0]
    assert int(lens[ty * gx + tx]) >= n_dense > LOOKBACK_WINDOW * SORT_TILE
    assert int(lens[ty * gx + tx]) > 100_000


# ---------------------------------------------------------------------------------------------- scan regimes
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_scan_grid_barrier_regime(ours):
    """P <= SMs x 2048: one scan block per 2048 Gaussians, at most one per SM - the grid is resident whatever the
    occupancy, so the scan takes the grid-barrier path."""
    P = _sms() * SCAN_TILE
    d = random_scene(P, 1920, 1280, seed=71, r_px=(3.0, 8.0))
    s, ref = run_and_check(ours, d)
    assert -(-P // SCAN_TILE) <= _sms()


def test_scan_ticket_regime(ours):
    """P > SMs x 8 x 2048: more scan blocks than can ever be resident (8 per SM at most), so the scan hands out
    tickets and looks back.  ~3.2 M Gaussians with small radii keep R near 6 M."""
    P = 3_200_000
    assert -(-P // SCAN_TILE) > _sms() * SCAN_BLOCKS_PER_SM
    d = random_scene(P, 1920, 1280, seed=72, r_px=(3.0, 6.0))
    run_and_check(ours, d)


# -------------------------------------------------------------------------------------------------- capacity
def test_capacity_small_calls_after_a_big_one_and_growth(ours):
    """The binning arena is sized from the capacity this thread used last (R + R/8 + 1 of the first call, grown the
    same way whenever a count outgrows it); the tile sort is launched for the capacity and bounded by the count on
    the device.  In a fresh thread: a big call, small calls whose lists span several sort blocks far below the
    capacity, then calls that outgrow it and repeat their tail - once with the shared-memory tile histogram and once
    with the global one.  Every call is exact."""
    from s3gaussian_b200 import _lib
    steps = [  # (label, P, W, H, radius range, seed)
        ("big", 300_000, 1920, 1280, (3.0, 12.0), 81),
        ("small", 20_000, 1920, 1280, (3.0, 12.0), 82),
        ("small-global", 30_000, 2576, 1664, (3.0, 12.0), 83),
        ("grow-shared", 400_000, 1920, 1280, (3.0, 30.0), 84),
        ("small-after-growth", 20_000, 1920, 1280, (3.0, 12.0), 85),
        ("grow-global", 600_000, 2576, 1664, (3.0, 40.0), 86),
    ]
    scenes = [(label, random_scene(P, W, H, seed, r_px=rr)) for label, P, W, H, rr, seed in steps]
    out, err = [], []

    def body():
        try:
            for label, d in scenes:
                grow = label.startswith("grow")
                _lib.profile_enable(grow)
                try:
                    s = forward_state(ours, d)
                    stages = _lib.profile_read(0) if grow else {}
                finally:
                    _lib.profile_enable(False)
                out.append((label, s, stages))
        except BaseException as e:   # surfaced in the test's thread
            err.append(e)

    th = threading.Thread(target=body)
    th.start()
    th.join()
    if err:
        raise err[0]
    cap = None
    for label, s, stages in out:
        ref = check_binning(s)
        R = ref["R"]
        assert emit_path(np.prod(br.grid_of(s["W"], s["H"]))) == ("global" if "global" in label else "shared")
        if cap is None:
            cap = R + R // 8 + 1
        elif label.startswith("grow"):
            assert R > cap, (label, R, cap)
            assert "retry" in stages, (label, stages)
            cap = R + R // 8 + 1
        else:
            assert 2 * SORT_TILE < R < cap // 4, (label, R, cap)


# -------------------------------------------------------------------------------------------- reference extension
@pytest.mark.parametrize("W,H", [(2064, 1552), (4112, 4112)], ids=["12513_tiles", "66049_tiles"])
def test_tile_regime_matches_reference_extension(W, H, ours):
    """The opt-in shared-memory histogram and the three-pass tile sort against the reference extension: n_contrib
    bit for bit, the colour within 1e-4 of the image max."""
    if not ref_ext.available():
        pytest.skip("oracle/_ref (prebuilt reference extension) not present")
    ref = ref_ext.load()
    gx, gy = br.grid_of(W, H)
    assert emit_path(gx * gy) == ("opt-in" if gx * gy == 12_513 else "global")
    d = random_scene(4000, W, H, seed=gx * gy, r_px=(3.0, 40.0))
    s, _ = run_and_check(ours, d)
    E = torch.Tensor([])
    g = lambda k: d[k].to(DEV).contiguous() if d[k] is not None else E
    R0, rc, _, rrad, gb, bb, ib = ref._C.rasterize_gaussians(
        d["bg"].to(DEV), g("means3D"), g("colors_precomp"), g("opacities"), g("scales"), g("rotations"), 1.0,
        g("cov3D_precomp"), d["viewmatrix"].to(DEV), d["projmatrix"].to(DEV), d["tanfovx"], d["tanfovy"], H, W,
        g("shs"), d["sh_degree"], d["campos"].to(DEV), False, False)
    torch.cuda.synchronize()
    ri = ref_ext.decode_image(ib, W * H)
    assert int(R0) == s["R"]
    np.testing.assert_array_equal(rrad.cpu().numpy(), s["radii"])
    np.testing.assert_array_equal(s["n_contrib"], ri["n_contrib"])
    assert util.relerr(s["color"], rc.cpu().numpy()) < TOL
