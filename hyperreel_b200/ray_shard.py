"""Multi-GPU rendering: rays shard embarrassingly, the finished pixel tiles are gathered over NVLink.

The reference renders a frame on rank 0 only (nlf/__init__.py:810-811) and has no collective on this path.
Here every rank renders a contiguous ray range (image row tiles for a full frame -- neighbouring pixels hit
neighbouring texels, so locality per GPU is preserved) with replicated parameters.  12 bytes per ray and peer
cross the fabric; nothing else does (SURVEY.md section 8e).

Two ways to assemble ``[N,3]`` on every rank:

* **peer-memory epilogue** (NVSwitch, the default on CUDA): a gather buffer ``[N,3]`` lives in symmetric memory on
  every GPU (``torch.distributed._symmetric_memory``: one allocation per rank, peer-mapped over NVLink).  The render
  kernel's epilogue stores each finished pixel into *every* rank's buffer (``hr_render_scatter``): the gather is fused
  into the kernel, no collective kernel follows -- only a signal-pad barrier so that nobody reads before all tiles landed.
  Two buffers alternate, which makes one barrier per call enough (see ``TileGather``).
* **one collective** (``all_gather_into_tensor``; NCCL on GPUs, gloo in the CPU tests): for render functions that are not
  the fused model, for more than ``HR_MAX_PEERS`` ranks, or when symmetric memory is not available.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Dict, Optional, Tuple

import torch
import torch.distributed as dist

from . import lib as L


def shard_range(n: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous range [lo, hi) of rank ``rank``: the first ``n % world`` ranks get one extra ray."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


class TileGather:
    """Peer-mapped gather buffers for ``render_sharded``: two ``[capacity,3]`` fp32 buffers per rank in symmetric memory.

    Hazards: rank A's epilogue writes into rank B's buffer k.  (i) B must not read buffer k before every rank's tile has
    landed -> one barrier after the render kernel.  (ii) A must not overwrite buffer k while B still reads the previous
    frame from it -> buffers alternate: A's writes of call c+2 come after A left the barrier of call c+1, which B joins
    only after everything B enqueued for call c (its reads included, same stream) -- so one barrier per call suffices as
    long as consumers read on the rendering stream."""

    def __init__(self, capacity: int, device: torch.device, group=None):
        import torch.distributed._symmetric_memory as symm_mem

        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        if self.world > L.HR_MAX_PEERS:
            raise RuntimeError(f"peer-memory gather supports up to {L.HR_MAX_PEERS} ranks")
        self.capacity = int(capacity)
        self.bufs, self.hdls, self.ptrs = [], [], []
        for _ in range(2):
            t = symm_mem.empty((self.capacity, 3), dtype=torch.float32, device=device)
            hdl = symm_mem.rendezvous(t, self.group)
            self.bufs.append(t)
            self.hdls.append(hdl)
            self.ptrs.append((C.c_void_p * self.world)(*[int(p) for p in hdl.buffer_ptrs]))
        self.turn = 0

    def next(self):
        k = self.turn
        self.turn ^= 1
        return self.bufs[k], self.hdls[k], self.ptrs[k]


_gathers: Dict[tuple, TileGather] = {}
_p2p_broken = False


def _tile_gather(n: int, device: torch.device, group) -> Optional[TileGather]:
    """Cached TileGather with room for n rays, or None when symmetric memory cannot be set up (decided once, on all ranks
    together: the rendezvous is collective)."""
    global _p2p_broken
    if _p2p_broken:
        return None
    key = (device.index, id(group))
    g = _gathers.get(key)
    if g is not None and g.capacity >= n:
        return g
    ok = torch.ones(1, device=device)
    try:
        cap = max(n, 1 << 16)
        g = TileGather(cap, device, group)
    except Exception:  # no symmetric-memory support in this build / on this fabric
        g = None
        ok.zero_()
    dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
    if float(ok.item()) == 0.0:
        _p2p_broken = True
        return None
    _gathers[key] = g
    return g


def render_sharded(rays: torch.Tensor, render_fn: Callable[..., Dict[str, torch.Tensor]], group=None,
                   gather: str = "auto", **render_kwargs) -> torch.Tensor:
    """Render ``rays`` ([N,C], identical on every rank) cooperatively; returns the full ``rgb`` [N,3] on every
    rank.  Bit-identical to a single-rank render because no reduction crosses rays.

    ``gather``: ``'auto'`` (peer-memory epilogue when possible, else the collective), ``'p2p'`` (fail if it cannot be used)
    or ``'collective'``.  With the peer-memory path the returned tensor is a view of the gather buffer, valid until the
    call after next."""
    if not (dist.is_available() and dist.is_initialized()):
        return render_fn(rays, **render_kwargs)["rgb"]
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    n = rays.shape[0]
    lo, hi = shard_range(n, rank, world)
    model = getattr(render_fn, "model", None)
    fused = rays.is_cuda and hasattr(model, "render_scatter") and not render_kwargs and world <= L.HR_MAX_PEERS
    if gather == "p2p" and not fused:
        raise RuntimeError("peer-memory gather needs the fused CUDA model, no extra render kwargs and <= 8 ranks")
    if fused and gather in ("auto", "p2p"):
        g = _tile_gather(n, rays.device, group)
        if g is None and gather == "p2p":
            raise RuntimeError("symmetric memory is not available in this process group")
        if g is not None:
            buf, hdl, ptrs = g.next()
            model.render_scatter(rays[lo:hi], ptrs, g.world, lo)  # epilogue stores into every rank's buffer
            hdl.barrier()  # signal-pad barrier on the current stream: all tiles have landed everywhere
            return buf[:n]
    per = (n + world - 1) // world  # padded tile so that all_gather_into_tensor sees equal shapes
    tile = torch.zeros((per, 3), dtype=torch.float32, device=rays.device)
    if hi > lo:
        tile[: hi - lo] = render_fn(rays[lo:hi], **render_kwargs)["rgb"]
    gathered = torch.empty((world * per, 3), dtype=torch.float32, device=rays.device)
    dist.all_gather_into_tensor(gathered, tile, group=group)
    if n % world == 0:
        return gathered
    out = torch.empty((n, 3), dtype=torch.float32, device=rays.device)
    for r in range(world):
        a, b = shard_range(n, r, world)
        out[a:b] = gathered[r * per: r * per + (b - a)]
    return out
