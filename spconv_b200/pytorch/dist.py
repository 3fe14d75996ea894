"""Data-parallel plumbing for the hot path: one point cloud (or an equal slice of the batch) per
GPU, full weight replica per GPU, and ONE all-reduce of a single flat gradient bucket per step.

The reference has no distributed code at all (SURVEY section 5: no NCCL / torch.distributed call
sites); every op on the path is per-sample (the batch index is just ``indices[:, 0]``,
``spconv/pytorch/core.py:148``), so there is no feature collective -- only the weight (and bias)
gradients cross NVLink.  For a SECOND-style encoder the bucket is O(1 MB): latency-bound, hence a
single flat bucket rather than per-tensor collectives.
"""
from __future__ import annotations

import ctypes
from typing import Iterable, List, Optional, Tuple

import torch
import torch.distributed as dist

from .. import _cabi


def shard_batch(indices: torch.Tensor, features: torch.Tensor, batch_size: int, rank: int,
                world_size: int) -> Tuple[torch.Tensor, torch.Tensor, int]:
    """Samples ``b`` with ``b % world_size == rank`` go to ``rank``; batch ids are renumbered
    ``0..local_bs-1``.  Returns ``(indices, features, local_batch_size)``."""
    assert batch_size % world_size == 0, "batch must divide evenly across ranks"
    b = indices[:, 0].long()
    keep = (b % world_size) == rank
    local = indices[keep].clone()
    local[:, 0] = (b[keep] // world_size).to(indices.dtype)
    return local, features[keep], batch_size // world_size


class GradBucket:
    """Flat view over the gradients of ``params`` so a step needs exactly one collective."""

    def __init__(self, params: Iterable[torch.nn.Parameter]):
        self.params: List[torch.nn.Parameter] = [p for p in params if p.requires_grad]
        assert self.params, "no trainable parameters"
        dev, dt = self.params[0].device, self.params[0].dtype
        self.numel = sum(p.numel() for p in self.params)
        self.flat = torch.zeros(self.numel, device=dev, dtype=dt)
        self._views: List[torch.Tensor] = []
        off = 0
        for p in self.params:
            assert p.dtype == dt, "one bucket per dtype"
            self._views.append(self.flat[off:off + p.numel()].view_as(p))
            off += p.numel()
        self.attach()

    def attach(self) -> int:
        """(Re-)alias every ``p.grad`` to its slice of the bucket.  ``optimizer.zero_grad()`` and
        ``module.zero_grad()`` default to ``set_to_none=True``, which drops the aliases; the next
        backward then allocates fresh ``.grad`` tensors OUTSIDE the bucket.  A gradient found
        outside is copied in before it is re-aliased, so nothing is lost.  Returns how many
        parameters had to be re-attached."""
        fixed = 0
        for p, view in zip(self.params, self._views):
            g = p.grad
            if g is not None and g.data_ptr() == view.data_ptr() and g.shape == view.shape:
                continue
            if g is not None:
                view.copy_(g)
            p.grad = view
            fixed += 1
        return fixed

    def zero(self) -> None:
        """Zero the gradients in place (use instead of ``zero_grad(set_to_none=True)``)."""
        self.attach()
        self.flat.zero_()

    def all_reduce(self, group: Optional[dist.ProcessGroup] = None, average: bool = True,
                   async_op: bool = False):
        """Sum (or mean) the bucket over the data-parallel group: one NCCL launch per step."""
        self.attach()          # gradients produced after a zero_grad(set_to_none=True) are pulled in
        if not dist.is_initialized() or dist.get_world_size(group) == 1:
            return None
        if average:
            self.flat.div_(dist.get_world_size(group))
        return dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group, async_op=async_op)


def allreduce_gradients(module: torch.nn.Module, group: Optional[dist.ProcessGroup] = None,
                        average: bool = True) -> None:
    """Stateless variant: flatten existing ``.grad`` tensors, one all-reduce, copy back."""
    if not dist.is_initialized() or dist.get_world_size(group) == 1:
        return
    grads = [p.grad for p in module.parameters() if p.grad is not None]
    if not grads:
        return
    flat = torch.cat([g.reshape(-1) for g in grads])
    if average:
        flat.div_(dist.get_world_size(group))
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    off = 0
    for g in grads:
        g.copy_(flat[off:off + g.numel()].view_as(g))
        off += g.numel()


class PeerGroup:
    """The exchange buffers of a data-parallel group, for the weight-gradient all-reduce fused into the
    weight-gradient kernel (``csrc/peer.cu``; ``include/spconv_b200.h`` ``spx_peer_group``).

        peers = PeerGroup()                       # after init_process_group; one process per GPU of ONE node
        ops.set_peer_group(peers)                 # every conv dW now comes back summed (mean) over the ranks
        ...
        loss.backward()                           # conv weight gradients: no all-reduce call
        ops.peer_allreduce_(bucket.flat)          # everything else: biases, norms, heads (bucket = GradBucket)

    Only the weight gradients of the conv ops are exchanged.  Biases (added outside the op in training)
    and every other parameter keep rank-local gradients until ``ops.peer_allreduce_`` reduces them, one
    call per tensor or one per :class:`GradBucket` of them, on every rank in the same order.

    Every rank allocates one buffer (``2 x capacity`` bytes: two epochs of its own fp32 slices), exports a CUDA IPC handle, and maps
    the others' (NVLink peer access).  ``capacity_bytes`` bounds the largest weight tensor, counted as
    fp32 (default 8 MB = 27 x 256 x 256 and some).  ``scale`` multiplies the sum (``1 / world`` = mean, the
    DDP convention).  Raises if peer mapping is not possible -- callers that can live without the fused
    path catch that and fall back to :class:`GradBucket`."""

    def __init__(self, group: Optional[dist.ProcessGroup] = None, capacity_bytes: int = 8 << 20,
                 average: bool = True, timeout_ms: int = 20000, device: Optional[torch.device] = None):
        lib = _cabi.load()
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        assert self.world <= _cabi.SPX_MAX_PEERS, f"at most {_cabi.SPX_MAX_PEERS} ranks"
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.scale = 1.0 / self.world if average else 1.0
        self._lib = lib
        self._mapped: List[int] = []
        self._own = None
        self.group = _cabi.PeerGroup()
        failure: Optional[str] = None
        # Every rank takes part in every collective of this constructor exactly once, whatever fails locally: a rank
        # that cannot create or map a buffer must not leave the others waiting in a collective it never joins.
        with torch.cuda.device(self.device):
            handle = (ctypes.c_ubyte * 64)()
            try:
                own = ctypes.c_void_p()
                _cabi.check(lib.spx_peer_buffer_create(capacity_bytes, self.world, ctypes.byref(own), handle),
                            "peer_buffer_create")
                self._own = own.value
            except Exception as e:                       # noqa: BLE001 -- reported through the consensus below
                failure = f"{type(e).__name__}: {e}"
            handles: List[Optional[bytes]] = [None] * self.world
            if self.world > 1:
                dist.all_gather_object(handles, bytes(handle) if failure is None else None, group=group)
            else:
                handles[0] = bytes(handle) if failure is None else None
            g = self.group
            g.world, g.rank, g.timeout_ms, g.capacity_bytes = self.world, self.rank, timeout_ms, capacity_bytes
            if failure is None and any(h is None for h in handles):
                failure = "a peer could not create its exchange buffer"
            if failure is None:
                try:
                    for r, h in enumerate(handles):
                        if r == self.rank:
                            g.buffers[r] = self._own
                            continue
                        mapped = ctypes.c_void_p()
                        raw = (ctypes.c_ubyte * 64).from_buffer_copy(h)
                        _cabi.check(lib.spx_peer_buffer_open(raw, ctypes.byref(mapped)), f"peer_buffer_open(rank {r})")
                        self._mapped.append(mapped.value)
                        g.buffers[r] = mapped.value
                except Exception as e:                   # noqa: BLE001
                    failure = f"{type(e).__name__}: {e}"
            torch.cuda.synchronize()
            if self.world > 1:
                # consensus (also the barrier: nobody pushes before every buffer is mapped and zeroed)
                ok = torch.tensor([0 if failure else 1], dtype=torch.int32, device=self.device)
                dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=group)
                if int(ok.item()) == 0 and failure is None:
                    failure = "a peer could not map the exchange buffers"
        if failure is not None:
            self.close()
            raise RuntimeError(f"PeerGroup: peer-memory exchange unavailable on rank {self.rank}: {failure}")

    @classmethod
    def local_ring(cls, world: int, capacity_bytes: int = 8 << 20, average: bool = True,
                   timeout_ms: int = 5000) -> List["PeerGroup"]:
        """``world`` groups whose buffers all live on the CURRENT device of this process: the exchange
        protocol between "ranks" that are streams of one GPU.  Test fixture (single-GPU boxes)."""
        lib = _cabi.load()
        bufs = []
        for _ in range(world):
            own = ctypes.c_void_p()
            handle = (ctypes.c_ubyte * 64)()
            _cabi.check(lib.spx_peer_buffer_create(capacity_bytes, world, ctypes.byref(own), handle), "peer_buffer_create")
            bufs.append(own.value)
        out = []
        for r in range(world):
            pg = object.__new__(cls)
            pg.world, pg.rank, pg.scale = world, r, (1.0 / world if average else 1.0)
            pg.device = torch.device("cuda", torch.cuda.current_device())
            pg._lib, pg._mapped, pg._own = lib, [], bufs[r]
            g = _cabi.PeerGroup()
            g.world, g.rank, g.timeout_ms, g.capacity_bytes, g.colocated = world, r, timeout_ms, capacity_bytes, world
            for q in range(world):
                g.buffers[q] = bufs[q]
            pg.group = g
            out.append(pg)
        torch.cuda.synchronize()
        return out

    def error(self) -> int:
        """Sticky error word of this rank's buffer: 1 = a peer did not arrive within the timeout (the
        affected gradients are NaN).  Synchronises the device."""
        torch.cuda.synchronize(self.device)
        e = ctypes.c_int(0)
        _cabi.check(self._lib.spx_peer_error(ctypes.byref(self.group), ctypes.byref(e)), "peer_error")
        return e.value

    def close(self) -> None:
        """Unmap the peers' buffers and free this rank's (all ranks: after a barrier / synchronize)."""
        if getattr(self, "_lib", None) is None:
            return
        with torch.cuda.device(self.device):
            torch.cuda.synchronize()
            for m in self._mapped:
                self._lib.spx_peer_buffer_close(m)
            self._mapped = []
            if self._own:
                self._lib.spx_peer_buffer_destroy(self._own)
                self._own = None
        self._lib = None
