"""Ring communicator of the burst-attention drivers.

Mirrors the reference's ``Ring`` (comm.py:104-321): ops are queued with
``double_ring_send_recv`` / ``_ring_send_recv_base``, launched by ``commit`` and
awaited by ``wait``.  Two transports:

* ``native`` (CUDA tensors, the product path): the C-ABI ring of
  include/burst_attn_b200.h -- grouped ncclSend/ncclRecv on a library-owned
  high-priority side stream, event hand-off to the compute stream, no host
  sync (the reference's BMTrain side-stream variant, comm.py:267-283,313-317,
  is the model).  One communicator per (process group, tag), cached -- the
  reference builds a fresh ``Ring`` per call (burst_attn_interface.py:205,265,268).
  When all ranks share a node (``default_transport``; or ``BA_RING_TRANSPORT=ce``) the flat ring instead
  pushes its hops with the copy engines into a ring-owned, IPC-mapped receive arena
  (csrc/ring_ce.cu): zero SMs, so the hop neither slows the tile kernels down nor -- for short
  shards -- stays exposed behind them as NCCL's SM-resident kernels do.  Receive
  buffers then come from ``Ring.empty_like`` (a bump allocator over the arena that
  every rank drives identically, so offsets are symmetric).
* ``torch`` (CPU tensors under gloo, used by the world_size-2 CPU tests of the
  ring schedule): ``dist.batch_isend_irecv`` as in comm.py:159-171,269.

A ``Ring`` here is always ONE ring over ONE group.  The reference's intra/inter
"double ring" (comm.py:187-254) is composed by the drivers from up to three of
them -- intra-node hops, inter-node prefetch of the block that starts the next
cycle, inter-node chain of the dQ node sums (burst_attn_interface.py:
``_ring_forward`` / ``_bwd_rounds``) -- so each level has its own
communicator and side stream and is awaited independently.  8 GPUs on one
NVSwitch are a uniform fabric where the flat ring is as good; the hierarchy is for
W spanning several NVLink domains.
"""
from __future__ import annotations

import ctypes
import os
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from . import native as _n


def get_world_size(group=None) -> int:
    if not dist.is_available() or not dist.is_initialized():
        return 1
    return dist.get_world_size(group)


def get_rank(group=None) -> int:
    if not dist.is_available() or not dist.is_initialized():
        return 0
    return dist.get_rank(group)


def replicate(t: torch.Tensor) -> torch.Tensor:
    out = torch.empty_like(t)
    out.copy_(t)
    return out


# --------------------------------------------------------------------------- #
# native rings, cached per (process group, tag, device)
# --------------------------------------------------------------------------- #
class _DeviceBytes:
    """A raw device allocation presented through the CUDA array interface (zero-copy ``torch.as_tensor``)."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


def _align(n: int, a: int = 1024) -> int:
    return (n + a - 1) // a * a


class CopyEngineUnavailable(RuntimeError):
    """The copy-engine transport could not be set up on at least one rank (e.g. a process that cannot see its
    neighbours' GPUs, or no CUDA IPC in this container).  Raised on EVERY rank of the ring together."""


_ce_disabled = False  # set once the copy-engine transport failed in this process: later rings go over NCCL


class _NativeRing:
    def __init__(self, group, tag: str, device: torch.device, transport: str = "nccl"):
        self.lib = _n.lib()
        self.group = group
        self.device = device
        self.world = get_world_size(group)
        self.rank = get_rank(group)
        self.ce = transport == "ce" and self.world > 1
        self.arena: Optional[torch.Tensor] = None  # uint8 view of the receive arena (copy-engine transport)
        self.arena_off = 0
        self.handle = ctypes.c_void_p()
        idbuf = (ctypes.c_uint8 * _n.NCCL_UNIQUE_ID_BYTES)()
        if self.ce:
            idbuf = None  # no communicator: hops go through ba_ring_arena_* (csrc/ring_ce.cu)
        elif self.world > 1:
            payload = [None]
            if self.rank == 0:
                _n.check(self.lib.ba_ring_unique_id(idbuf), "ba_ring_unique_id")
                payload = [bytes(idbuf)]
            src = dist.get_global_rank(group, 0) if group is not None else 0
            dist.broadcast_object_list(payload, src=src, group=group, device=device)
            ctypes.memmove(idbuf, payload[0], _n.NCCL_UNIQUE_ID_BYTES)
        with torch.cuda.device(device):
            _n.check(self.lib.ba_ring_create(idbuf, self.rank, self.world, ctypes.byref(self.handle)),
                     "ba_ring_create")

    def post(self, srcs: Sequence[torch.Tensor], dsts: Sequence[torch.Tensor]) -> None:
        n = len(srcs)
        VP = ctypes.c_void_p * n
        I64 = ctypes.c_int64 * n
        for s, d in zip(srcs, dsts):
            assert s.is_contiguous() and d.is_contiguous() and s.numel() * s.element_size() == d.numel() * d.element_size()
        src = VP(*[s.data_ptr() for s in srcs])
        dst = VP(*[d.data_ptr() for d in dsts])
        nb = I64(*[s.numel() * s.element_size() for s in srcs])
        _n.check(self.lib.ba_ring_post(self.handle, src, dst, nb, n, _n.stream_ptr(srcs[0].device)), "ba_ring_post")

    def wait(self, device) -> None:
        _n.check(self.lib.ba_ring_wait(self.handle, _n.stream_ptr(device)), "ba_ring_wait")

    # ---- receive arena of the copy-engine transport
    def begin(self, nbytes: int) -> None:
        """Start of one driver call that will carve ``nbytes`` of receive buffers.  Every rank passes the
        same number (equal shards), so they all decide to grow in the same call."""
        if not self.ce:
            return
        if self.arena is None or nbytes > self.arena.numel():
            self._grow(nbytes + nbytes // 4)
        self.arena_off = 0

    def _grow(self, nbytes: int) -> None:
        # collective: nobody may still be pushing into (or reading from) the arena that is replaced
        torch.cuda.synchronize(self.device)
        dist.barrier(group=self.group)
        self.arena = None
        base = ctypes.c_void_p()
        hbuf = (ctypes.c_uint8 * _n.IPC_HANDLE_BYTES)()
        with torch.cuda.device(self.device):
            # Every rank goes through the same collectives whether or not its own step worked, and all ranks then
            # agree: either everyone has a connected arena or everyone raises CopyEngineUnavailable (-> NCCL).
            err = self._try(lambda: self.lib.ba_ring_arena_create(self.handle, nbytes, ctypes.byref(base), hbuf),
                            "ba_ring_arena_create")
            gathered: List[Optional[tuple]] = [None] * self.world
            dist.all_gather_object(gathered, (err is None, bytes(hbuf)), group=self.group)
            if not all(g[0] for g in gathered):
                raise CopyEngineUnavailable(err or "a peer rank could not create its receive arena")
            prv = (ctypes.c_uint8 * _n.IPC_HANDLE_BYTES).from_buffer_copy(gathered[(self.rank - 1) % self.world][1])
            nxt = (ctypes.c_uint8 * _n.IPC_HANDLE_BYTES).from_buffer_copy(gathered[(self.rank + 1) % self.world][1])
            err = self._try(lambda: self.lib.ba_ring_arena_connect(self.handle, prv, nxt), "ba_ring_arena_connect")
            connected: List[Optional[bool]] = [None] * self.world
            dist.all_gather_object(connected, err is None, group=self.group)
            if not all(connected):
                raise CopyEngineUnavailable(err or "a peer rank could not map its neighbours' arenas")
        self.arena = torch.as_tensor(_DeviceBytes(base.value, _align(nbytes)), device=self.device)
        dist.barrier(group=self.group)

    @staticmethod
    def _try(call, what: str) -> Optional[str]:
        """Run one C-ABI call; None on success, the error text otherwise (never raises)."""
        try:
            _n.check(call(), what)
            return None
        except _n.NativeLibraryError as e:
            return str(e)

    def empty(self, shape, dtype) -> torch.Tensor:
        n = 1
        for d in shape:
            n *= d
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        off = _align(self.arena_off)
        assert self.arena is not None and off + nbytes <= self.arena.numel(), \
            "receive arena exhausted: Ring.begin() was given too small a size"
        self.arena_off = off + nbytes
        return self.arena[off:off + nbytes].view(dtype).view(shape)


_native_rings: Dict[tuple, _NativeRing] = {}


def _group_identity(group) -> tuple:
    """A stable identity of a process group: its name and member ranks (NOT id(group): after a group is
    destroyed a new one can reuse the address and would silently inherit a communicator with stale peers)."""
    if group is None:
        return ("world", get_world_size(None))
    try:
        return (str(getattr(group, "group_name", "")), tuple(dist.get_process_group_ranks(group)))
    except Exception:
        return ("id", id(group))


def _native_ring(group, tag: str, device: torch.device, transport: str = "nccl") -> _NativeRing:
    key = (_group_identity(group), tag, device.index if device.index is not None else -1, transport)
    ring = _native_rings.get(key)
    if ring is None:
        ring = _NativeRing(group, tag, device, transport)
        _native_rings[key] = ring
    return ring


def destroy_rings() -> None:
    """Tear down every cached native ring (communicator, side stream, copy-engine arena).  Call it before
    ``dist.destroy_process_group()`` -- e.g. on elastic restarts -- so that a later re-init builds fresh
    communicators; all ranks must call it (device-synchronised) together."""
    if torch.cuda.is_available():
        torch.cuda.synchronize()
    for ring in _native_rings.values():
        ring.arena = None
        if ring.handle:
            ring.lib.ba_ring_destroy(ring.handle)
            ring.handle = ctypes.c_void_p()
    _native_rings.clear()


# --------------------------------------------------------------------------- #
def default_transport() -> str:
    """Transport of a flat ring when the caller does not name one: ``BA_RING_TRANSPORT`` if set; otherwise the copy
    engines (``ce``) when every rank of the job runs on this node -- torchrun's LOCAL_WORLD_SIZE equals the world
    size -- and NCCL in every other case (several nodes, or a launcher that does not say).  The copy engines take no
    SMs, whereas NCCL's SM-resident send/recv kernels slow the tile kernels down while they co-run."""
    env = os.environ.get("BA_RING_TRANSPORT")
    if env:
        return env
    if _ce_disabled:
        return "nccl"
    try:
        local = int(os.environ.get("LOCAL_WORLD_SIZE", "0"))
    except ValueError:
        local = 0
    world = get_world_size(None)
    return "ce" if (world > 1 and local == world) else "nccl"


class Ring:
    """Single flat ring over ``process_group``: send to (rank+1)%W, receive from (rank-1)%W."""

    def __init__(self, process_group=None, local_group=(None, None), dq: bool = False, tag: Optional[str] = None,
                 transport: Optional[str] = None):
        self.comm = process_group
        self.transport = transport or default_transport()
        # "local": measurement only (bench.py --ab-comm): every hop becomes a device-local copy src -> dst on the
        # compute stream, i.e. the ring is replaced by a local buffer swap -- same kernels, same bytes through HBM,
        # nothing over NVLink -- the A/B partner that isolates exposed communication time (results are wrong)
        assert self.transport in ("nccl", "ce", "local"), \
            f"BA_RING_TRANSPORT must be nccl, ce or local, got {self.transport!r}"
        self.world_size = get_world_size(process_group)
        self.rank = get_rank(process_group)
        self.tag = tag or ("dq" if dq else "kv")
        # reference field names kept for API compatibility (comm.py:137-141); hierarchy lives in the drivers
        self.local_group, self.local_group2 = local_group[0], local_group[1]
        self.double_ring = False
        self.intra_size = self.world_size
        self.inter_size = 1
        self._pending: List[Tuple[torch.Tensor, torch.Tensor]] = []
        self._reqs = []
        self._native: Optional[_NativeRing] = None
        self._device = None

    # ---- queue (comm.py:256-257)
    def _ring_send_recv_base(self, tensor_list, dest_list, group=None):
        self._pending += list(zip(tensor_list, dest_list))

    def double_ring_send_recv(self, tensor_list, dest_list, r=0):
        self._ring_send_recv_base(tensor_list, dest_list)

    def double_ring_send_recv_q(self, tensor_list, dest_list, r=0):
        self._ring_send_recv_base(tensor_list, dest_list)

    # ---- launch (comm.py:285-299)
    def commit(self):
        if not self._pending:
            return
        srcs = [s for s, _ in self._pending]
        dsts = [d for _, d in self._pending]
        self._pending = []
        if srcs[0].is_cuda and self.transport == "local":
            for s, d in zip(srcs, dsts):
                d.copy_(s)
            self._reqs = []
        elif srcs[0].is_cuda:
            self._device = srcs[0].device
            self._ensure_native(self._device)
            self._native.post(srcs, dsts)
            self._reqs = ["native"]
        else:
            self._reqs = self._commit_torch(srcs, dsts)

    def _commit_torch(self, srcs, dsts):
        W, rank = self.world_size, self.rank
        if W == 1:
            for s, d in zip(srcs, dsts):
                d.copy_(s)
            return []
        nxt, prv = (rank + 1) % W, (rank - 1 + W) % W
        if self.comm is not None:
            nxt, prv = dist.get_global_rank(self.comm, nxt), dist.get_global_rank(self.comm, prv)
        ops = []
        for s, d in zip(srcs, dsts):
            send = dist.P2POp(dist.isend, s, nxt, group=self.comm)
            recv = dist.P2POp(dist.irecv, d, prv, group=self.comm)
            ops += [send, recv] if rank % 2 == 0 else [recv, send]  # comm.py:166-171
        return dist.batch_isend_irecv(ops)

    # ---- await (comm.py:301-321)
    def wait(self, force_wait_inter=False):
        for r in self._reqs:
            if r == "native":
                self._native.wait(self._device)
            else:
                r.wait()
        self._reqs = []

    # ---- convenience used by the drivers
    def post(self, srcs, dsts):
        self._ring_send_recv_base(srcs, dsts)
        self.commit()

    def _ensure_native(self, device):
        if self._native is None:
            self._native = _native_ring(self.comm, self.tag, device, self.transport)

    def begin(self, like: torch.Tensor, recv_sizes: Sequence[int]) -> None:
        """Announce one driver call that will ask ``empty`` / ``empty_like`` for receive buffers of these byte
        sizes (only the copy-engine transport cares: its buffers come from the ring's arena)."""
        if like.is_cuda and self.world_size > 1 and self.transport == "ce":
            self._device = like.device
            self._ensure_native(like.device)
            try:
                self._native.begin(sum(_align(n) for n in recv_sizes))
            except CopyEngineUnavailable as e:
                if os.environ.get("BA_RING_TRANSPORT") == "ce":
                    raise  # asked for by name: fail loudly
                # the default picked it: every rank of the ring is here together -- all fall back to NCCL
                global _ce_disabled
                _ce_disabled = True
                import warnings
                warnings.warn(f"burst_attn: copy-engine ring transport unavailable ({e}); using NCCL")
                self.transport, self._native = "nccl", None

    def empty(self, shape, dtype, device) -> torch.Tensor:
        """A buffer that may be the DESTINATION of a hop on this ring."""
        if self._native is not None and self._native.ce:
            return self._native.empty(tuple(shape), dtype)
        return torch.empty(tuple(shape), dtype=dtype, device=device)

    def empty_like(self, t: torch.Tensor) -> torch.Tensor:
        return self.empty(t.shape, t.dtype, t.device)
