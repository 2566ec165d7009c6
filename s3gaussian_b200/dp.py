"""View-parallel data parallelism for the render path.

The reference has no distributed code: it renders a batch of cameras in a sequential
loop and combines them at the loss (train.py:372-392).  Each view's forward+backward is
independent given replicated parameters, so the batch shards by CAMERA: one process per
GPU (torch.distributed, NCCL over NVLink/NVSwitch), rank r renders views r, r+G, ...,
and the only exchange is

  * one all-reduce (SUM) of the flat fp32 gradient bucket per step: per-Gaussian grads
    (59 floats = 236 B each) + the 35.8 M deformation parameters (143 MB);
  * the densify statistics (viewspace-gradient norm accumulates with SUM, radii with MAX,
    visibility with OR; gaussian_model.py:693-695, train.py:489-499);
  * a broadcast of the Gaussian tensors after rank 0 densifies/prunes
    (gaussian_model.py:496-561 samples with torch.normal, so ranks would diverge).

Host-side logic only; works with any backend (the CPU tests run it over gloo).
"""
from __future__ import annotations

import os
from typing import Iterable, Sequence

import torch
import torch.distributed as dist


def init_from_env(backend: str | None = None):
    """(rank, world, local_rank).  Reads RANK / WORLD_SIZE / LOCAL_RANK / MASTER_* (torchrun)."""
    rank = int(os.environ.get("RANK", 0))
    world = int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        kw = {}
        if backend == "nccl":
            torch.cuda.set_device(local)
            kw["device_id"] = torch.device(f"cuda:{local}")
        dist.init_process_group(backend, **kw)
    return rank, world, local


def shard_views(views: Sequence, rank: int, world: int) -> list:
    """Views of one step's batch owned by `rank` (round-robin; 8 views / 8 GPUs = 1 each)."""
    return [v for i, v in enumerate(views) if i % world == rank]


class GradBucket:
    """Flat fp32 bucket over a fixed parameter list: one collective per step.

    `attach()` points every p.grad at its slice of the bucket, so autograd accumulates the
    local gradients straight into it (no gather copy); `zero()` clears it; `all_reduce()`
    sums it over the ranks in place (optionally averaging)."""

    def __init__(self, params: Iterable[torch.Tensor]):
        self.params = [p for p in params]
        if not self.params:
            raise ValueError("GradBucket needs at least one parameter")
        dev, dt = self.params[0].device, torch.float32
        self.offsets, n = [], 0
        for p in self.params:
            if p.dtype != dt or p.device != dev:
                raise ValueError("all bucket parameters must be float32 on one device")
            self.offsets.append(n)
            n += p.numel()
        self.flat = torch.zeros(n, dtype=dt, device=dev)
        self.attach()

    def attach(self):
        for p, o in zip(self.params, self.offsets):
            g = self.flat[o:o + p.numel()]
            if p.is_contiguous():
                p.grad = g.view(p.shape)
            else:   # channels-last planes: same memory order as the parameter
                p.grad = g.as_strided(p.shape, p.stride())

    def zero(self):
        self.flat.zero_()

    @property
    def nbytes(self) -> int:
        return self.flat.numel() * 4

    def all_reduce(self, average: bool = False):
        if dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM)
            if average:
                self.flat.div_(dist.get_world_size())
        return self.flat


def sync_view_stats(viewspace_grad: torch.Tensor, radii: torch.Tensor, absgrad: torch.Tensor | None = None):
    """The batch statistics of ONE training step, combined over the ranks' views exactly as the reference
    combines the views of its sequential batch loop: the screen-space gradients ADD
    (train.py:435-437: viewspace_point_tensor_grad += viewspace_point_tensor_list[idx].grad) and the radii take
    the MAX (train.py:391 `radii = torch.cat(radii_list,0).max(dim=0).values`), so `radii > 0` is the OR of the
    per-view visibility filters (:392).  Call it ONCE per step on the local per-step tensors (in place), then
    make ONE `GaussianModel.densification_step(viewspace_grad, radii)` call on every rank: the accumulators
    `xyz_gradient_accum` / `denom` / `max_radii2D` themselves are never all-reduced (they would be re-summed
    every step).  `absgrad` (the rasterizer's absolute screen-space gradient, summed over the rank's views) ADDS like
    the signed gradient; when given it is synchronised too and returned third."""
    out = (viewspace_grad, radii) if absgrad is None else (viewspace_grad, radii, absgrad)
    if not (dist.is_initialized() and dist.get_world_size() > 1):
        return out
    dist.all_reduce(viewspace_grad, op=dist.ReduceOp.SUM)
    dist.all_reduce(radii, op=dist.ReduceOp.MAX)
    if absgrad is not None:
        dist.all_reduce(absgrad, op=dist.ReduceOp.SUM)
    return out


def broadcast_gaussians(tensors: dict, src: int = 0) -> dict:
    """After `src` densified / pruned: ship the new point count, then every per-Gaussian tensor
    (and whatever else is in `tensors`, e.g. Adam moments).  Non-source ranks get NEW tensors of
    the right size; returns the dict to install."""
    if not (dist.is_initialized() and dist.get_world_size() > 1):
        return tensors
    rank = dist.get_rank()
    names = sorted(tensors)
    dev = tensors[names[0]].device
    out = {}
    for k in names:
        t = tensors[k]
        shape = torch.tensor(list(t.shape) + [-1] * (8 - t.dim()), dtype=torch.int64, device=dev)
        dist.broadcast(shape, src)
        dims = [int(v) for v in shape.tolist() if v >= 0]
        buf = t.contiguous() if rank == src else torch.empty(dims, dtype=t.dtype, device=dev)
        dist.broadcast(buf, src)
        out[k] = buf
    return out


def max_over_ranks(value: float, device) -> float:
    """device-timed milliseconds -> the slowest rank's (what a step costs)."""
    if not (dist.is_initialized() and dist.get_world_size() > 1):
        return value
    t = torch.tensor([value], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t[0])


def peer_slices(numel: int, world: int):
    """[(begin, end)] in elements of the slice each rank reduces (float4 granularity, csrc/peer.cuh)."""
    if numel % 4:
        raise ValueError("peer all-reduce buffers hold a multiple of 4 floats")
    n4 = numel // 4
    chunk4 = (n4 + world - 1) // world
    return [(min(r * chunk4, n4) * 4, min((r + 1) * chunk4, n4) * 4) for r in range(world)]


class PeerAllReduce:
    """SUM all-reduce of one flat fp32 buffer over NVLink peer memory with our own kernels
    (csrc/peer.cuh): reduce-scatter by direct peer loads, then all-gather by direct peer loads.

    The buffer is a symmetric allocation (torch.distributed._symmetric_memory: the same size on every rank,
    peer-mapped into every process); rank order of the sum is fixed, so every rank gets bit-identical
    results.  The kernels never wait on remote state - the three device-side barriers between them
    (the handle's signal-pad barrier) provide the ordering:

        contributions written | barrier | reduce-scatter | barrier | all-gather | barrier | buffer reusable

    NCCL is the baseline this replaces for the 472 MB per-step gradient bucket; `available()`
    tells whether the symmetric-memory rendezvous worked on this system (callers fall back to
    dist.all_reduce and say so)."""

    def __init__(self, numel: int, device, group=None):
        import ctypes as C
        import torch.distributed._symmetric_memory as symm_mem
        from . import _lib
        self.numel = (int(numel) + 3) // 4 * 4
        self.group = group if group is not None else dist.group.WORLD
        import warnings
        try:        # older torch releases need the group registered first; newer ones deprecate the call (warning muted)
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                symm_mem.enable_symm_mem_for_group(self.group.group_name)
        except Exception:
            pass
        self.buffer = symm_mem.empty(self.numel, dtype=torch.float32, device=device)
        self.handle = symm_mem.rendezvous(self.buffer, self.group)
        self.rank, self.world = self.handle.rank, self.handle.world_size
        ptrs = list(self.handle.buffer_ptrs)
        self._ptrs = (C.c_void_p * self.world)(*ptrs)
        self._lib = _lib
        self.buffer.zero_()

    def nvls_all_reduce_(self) -> torch.Tensor:
        """In-switch (NVLS) variant: one kernel on the handle's multicast pointer.  Round-2 code path: not yet
        run on hardware, nothing calls it by default (tools/dev_peer.py --nvls)."""
        import ctypes as C
        mc = int(getattr(self.handle, "multicast_ptr", 0) or 0)
        if mc == 0:
            raise RuntimeError("PeerAllReduce: this symmetric allocation has no multicast mapping")
        lib = self._lib.load()
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        self.handle.barrier(channel=0)
        self._lib.check(lib.s3g_peer_nvls_all_reduce(self.world, self.rank, C.c_void_p(mc), self.numel, stream),
                        "s3g_peer_nvls_all_reduce")
        self.handle.barrier(channel=1)
        return self.buffer

    def flat(self, numel: int | None = None) -> torch.Tensor:
        return self.buffer if numel is None else self.buffer[:numel]

    def all_reduce_(self) -> torch.Tensor:
        import ctypes as C
        lib = self._lib.load()
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        h = self.handle
        h.barrier(channel=0)
        self._lib.check(lib.s3g_peer_reduce_scatter(self.world, self.rank, self._ptrs, self.numel, stream),
                        "s3g_peer_reduce_scatter")
        h.barrier(channel=1)
        self._lib.check(lib.s3g_peer_all_gather(self.world, self.rank, self._ptrs, self.numel, stream),
                        "s3g_peer_all_gather")
        h.barrier(channel=0)
        return self.buffer


def make_peer_all_reduce(numel: int, device):
    """PeerAllReduce, or None (with the reason) where symmetric memory cannot be set up."""
    try:
        return PeerAllReduce(numel, device), None
    except Exception as e:       # no NVLink peer access, old driver, non-NCCL group, ...
        return None, f"{type(e).__name__}: {e}"


class FusedGradExchange:
    """Per-Gaussian gradient all-reduce with its first half fused into the backward kernel.

    The plain path (PeerAllReduce / ncclAllReduce) lets the backward write its five gradient tensors and then moves
    the whole 236 B/Gaussian bucket twice over NVLink.  Here the backward's last kernel
    (preprocess_backward_kernel<.., DP>, sink of s3g_rasterize_backward) stores every VISIBLE Gaussian's gradient values
    straight into the staging area of the rank that owns that slice of the flat bucket - peer-mapped symmetric
    memory, plain stores - so the reduce-scatter traffic overlaps the kernel's own HBM work and culled rows never
    cross the link; `finish()` then runs ONE kernel per rank that sums the `world` staging sub-slices in rank order
    (bit-identical results on every rank), writes the sums into every rank's bucket (multimem.st through the
    NVSwitch multicast mapping when the allocation has one, direct peer stores otherwise) and re-zeroes the staging.

        ex = FusedGradExchange({"means3D": (P, 3), "shs": (P, 16, 3), "opacities": (P, 1), ...}, device)
        ex.install()                    # diff_gaussian_rasterization routes its backward through the sink
        loss.backward()                 # grads of the named inputs are VIEWS of ex.bucket (not yet summed)
        ex.finish()                     # barrier | reduce + gather | barrier  -> the views hold the sums

    Layout: one symmetric allocation [bucket | staging]; every tensor starts on a 16-byte boundary of the bucket;
    slice o of the bucket (chunk floats) is owned by rank o; staging = [world][chunk]."""

    NAMES = ("means3D", "shs", "opacities", "scales", "rotations")

    def __init__(self, shapes: dict, device, group=None):
        import ctypes as C
        import warnings
        import torch.distributed._symmetric_memory as symm_mem
        from . import _lib
        self._lib = _lib
        self.group = group if group is not None else dist.group.WORLD
        self.offsets, n = {}, 0
        for k in self.NAMES:
            if k in shapes and shapes[k] is not None:
                cnt = 1
                for v in shapes[k]:
                    cnt *= int(v)
                self.offsets[k] = (n, cnt, tuple(int(v) for v in shapes[k]))
                n = (n + cnt + 3) // 4 * 4
        for k in ("means3D", "opacities", "scales", "rotations"):
            if k not in self.offsets:
                raise ValueError(f"FusedGradExchange needs the shape of {k}")
        self.numel = n
        try:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                symm_mem.enable_symm_mem_for_group(self.group.group_name)
        except Exception:
            pass
        world = dist.get_world_size(self.group)
        self.chunk = ((n + world - 1) // world + 3) // 4 * 4
        self.stage_off = (n + 3) // 4 * 4
        total = self.stage_off + world * self.chunk
        self.buffer = symm_mem.empty(total, dtype=torch.float32, device=device)
        self.handle = symm_mem.rendezvous(self.buffer, self.group)
        self.rank, self.world = self.handle.rank, self.handle.world_size
        self.buffer.zero_()
        self.bucket = self.buffer[:n]
        ptrs = [int(p) for p in self.handle.buffer_ptrs]
        self._bucket_ptrs = (C.c_void_p * self.world)(*ptrs)
        self.mc = int(getattr(self.handle, "multicast_ptr", 0) or 0)
        sink = _lib.PeerSink()
        sink.world, sink.rank, sink.chunk = self.world, self.rank, self.chunk
        for p in range(self.world):
            sink.stage[p] = ptrs[p] + 4 * self.stage_off
        sink.off_means3D = self.offsets["means3D"][0]
        sink.off_shs = self.offsets["shs"][0] if "shs" in self.offsets else -1
        sink.off_opacities = self.offsets["opacities"][0]
        sink.off_scales = self.offsets["scales"][0]
        sink.off_rotations = self.offsets["rotations"][0]
        self.peer_sink_struct = sink            # read by diff_gaussian_rasterization's backward
        self._prev = None
        self._pending = False
        torch.cuda.synchronize(device)
        self.handle.barrier(channel=0)          # every rank's buffer is zeroed before anyone stores into it

    # gradient sink protocol of diff_gaussian_rasterization (name, shape, device) -> tensor or None
    def __call__(self, name, shape, device):
        if name not in self.offsets:
            return None
        o, cnt, shp = self.offsets[name]
        if tuple(shape) != shp:
            raise RuntimeError(f"FusedGradExchange: {name} has shape {tuple(shape)}, the bucket was laid out for {shp}")
        return self.bucket[o:o + cnt].view(shape)

    def note_backward(self):
        """called by the rasterizer's backward: the kernel STORES (not adds) this rank's rows into the owners'
        staging, so exactly one backward may run between two finish() calls"""
        if self._pending:
            raise RuntimeError("FusedGradExchange: a second backward before finish() would overwrite the first one's "
                               "rows in the staging areas (one view per rank and exchange)")
        self._pending = True

    def install(self):
        from . import diff_gaussian_rasterization as dgr
        self._prev = dgr.set_grad_sink(self)
        return self

    def uninstall(self):
        from . import diff_gaussian_rasterization as dgr
        dgr.set_grad_sink(self._prev)

    def finish(self) -> torch.Tensor:
        """All ranks call this after their backward: returns the bucket holding the summed gradients."""
        import ctypes as C
        lib = self._lib.load()
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        self.handle.barrier(channel=0)          # every rank's stores have landed
        stage_local = self.buffer.data_ptr() + 4 * self.stage_off
        self._lib.check(lib.s3g_peer_reduce_gather(self.world, self.rank, C.c_void_p(stage_local), self._bucket_ptrs,
                                                   C.c_void_p(self.mc) if self.mc else None, self.numel, self.chunk,
                                                   stream), "s3g_peer_reduce_gather")
        self.handle.barrier(channel=1)          # sums visible everywhere, staging zeroed everywhere
        self._pending = False
        return self.bucket


def make_fused_grad_exchange(shapes: dict, device):
    """FusedGradExchange, or (None, reason) where symmetric memory cannot be set up."""
    try:
        return FusedGradExchange(shapes, device), None
    except Exception as ex:      # pragma: no cover - depends on the system
        return None, f"{type(ex).__name__}: {ex}"
