"""
Symmetric (peer-mapped) device memory.

One rendezvous replaces every per-edge NCCL communicator of the reference
(``gossip/graph_manager.py:22-32`` creates a 2-rank group + 2 warm-up
all-reduces per phone-book entry): each rank allocates its buffers with the
native runtime (``_C.symm_alloc`` -> cudaMalloc + cudaIpcGetMemHandle), the
64-byte handles are exchanged ONCE over the c10d control plane
(``all_gather_object``; NCCL or gloo, it only moves ~100 bytes), every peer
maps them (``cudaIpcOpenMemHandle``) and the resulting device pointers are
packed into an int64 device table that the kernels index by rank.  After that
NVSwitch makes every peer equidistant; any circulant offset costs the same.

Two worlds implement the same small interface (``alloc`` / ``ptr_table``):

* :class:`SymmetricWorld`   -- one process per GPU (production);
* :class:`LocalWorld`       -- N virtual ranks inside ONE process (all on one
  GPU = loop-back tests, or one per visible GPU via plain peer access).
"""

from __future__ import annotations

import threading
from typing import Dict, List, Optional

import torch
import torch.distributed as dist

from ..ops import native


class _Buffer(object):
    __slots__ = ('name', 'nbytes', 'local', 'peers', 'table', 'mc', 'vmm')

    def __init__(self, name, nbytes):
        self.name = name
        self.nbytes = nbytes
        self.local = None      # uint8 tensor owned by this rank
        self.peers = None      # list of uint8 tensors (index = rank)
        self.table = None      # int64 device tensor of base pointers
        self.mc = None         # uint8 tensor over the MULTICAST mapping (VmmSymmetricWorld), or None
        self.vmm = None        # the native VmmBuffer that owns the physical memory


class SymmetricWorld(object):
    """Symmetric allocator over a ``torch.distributed`` group, one rank per
    process.  ``ranks`` are the members (global ranks); position in the list
    is the *symmetric rank* used to index pointer tables."""

    def __init__(self, device=None, group=None):
        assert dist.is_initialized(), 'SymmetricWorld needs torch.distributed'
        C = native.load()
        self._C = C
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)
        if device is None:
            device = torch.device('cuda', torch.cuda.current_device())
        self.device = torch.device(device)
        assert self.world <= C.MAX_RANKS
        self.buffers: Dict[str, _Buffer] = {}

    def alloc(self, name: str, nbytes: int) -> _Buffer:
        """Collective: every rank allocates ``nbytes`` and maps everyone else's."""
        assert name not in self.buffers
        C = self._C
        buf = _Buffer(name, nbytes)
        buf.local, handle = C.symm_alloc(int(nbytes), self.device.index)
        if self.world > 1 and len(handle) == 0:
            raise RuntimeError('cudaIpcGetMemHandle failed; peer mapping unavailable')
        gathered = [None] * self.world
        if self.world > 1:
            dist.all_gather_object(gathered, (bytes(handle), int(nbytes)), group=self.group)
        buf.peers = []
        for r in range(self.world):
            if r == self.rank:
                buf.peers.append(buf.local)
            else:
                h, nb = gathered[r]
                assert nb == nbytes, 'symmetric allocations must have equal size'
                buf.peers.append(C.symm_open(h, int(nb), self.device.index))
        buf.table = torch.tensor([t.data_ptr() for t in buf.peers],
                                 dtype=torch.int64, device=self.device)
        self.buffers[name] = buf
        if self.world > 1:
            dist.barrier(group=self.group)    # nobody touches a peer before all mapped
        return buf

    def barrier(self):
        if self.world > 1:
            dist.barrier(group=self.group)


class VmmSymmetricWorld(SymmetricWorld):
    """Symmetric allocator on the CUDA virtual-memory-management API with an NVSwitch multicast
    view (``_C.VmmBuffer``, csrc/vmm_symm.cpp): ``alloc()`` returns a buffer whose ``peers`` /
    ``table`` are ordinary unicast P2P mappings (same contract as :class:`SymmetricWorld`) and
    whose ``mc`` is a tensor over the multicast address -- ``multimem.ld_reduce`` reads through it
    are summed inside the switch, ``multimem.st`` writes land in every GPU.  The POSIX file
    descriptors of the allocations are passed between the ranks with ``SCM_RIGHTS`` messages over
    abstract unix-domain sockets (``_C.FdChannel``; ``pidfd_getfd`` is refused inside GPU
    containers), named after a job token that travels over the c10d control plane (single host,
    one NVLink domain)."""

    @staticmethod
    def supported(device=None) -> bool:
        if not (torch.cuda.is_available() and native.available()):
            return False
        dev = torch.cuda.current_device() if device is None else torch.device(device).index
        caps = native.load().vmm_caps(int(dev))
        return bool(caps.get('multicast') and caps.get('posix_fd'))

    def _channel(self):
        """lazily created fd-passing channel (abstract unix sockets named after a job token that
        symmetric rank 0 draws and broadcasts over the control plane)"""
        if getattr(self, '_fdx', None) is None:
            import os
            import uuid
            tok = [None]
            if self.rank == 0:
                tok[0] = 'sgp_b200.%d.%s' % (os.getpid(), uuid.uuid4().hex[:12])
            if self.world > 1:
                src = dist.get_global_rank(self.group, 0) if self.group is not None else 0
                dist.broadcast_object_list(tok, src=src, group=self.group)
            self._fdx = self._C.FdChannel(tok[0], self.rank, self.world)
            if self.world > 1:
                dist.barrier(group=self.group)        # every rank listens before anybody connects
        return self._fdx

    def _exchange_fds(self, fd: int, tag: int):
        """everybody sends `fd` to every peer, then receives world-1 descriptors -> {rank: fd}"""
        ch = self._channel()
        for r in range(self.world):
            if r != self.rank:
                ch.send(r, tag, int(fd))
        got = {}
        for _ in range(self.world - 1):
            src, t, f = ch.recv()
            assert t == tag, 'fd channel out of step (tag %d, expected %d)' % (t, tag)
            got[int(src)] = int(f)
        return got

    def alloc(self, name: str, nbytes: int, multicast: bool = True) -> _Buffer:
        assert name not in self.buffers
        C = self._C
        buf = _Buffer(name, nbytes)
        vb = C.VmmBuffer(int(nbytes), self.device.index, self.world)
        buf.vmm = vb
        buf.local = vb.local()
        self._tag = getattr(self, '_tag', 0) + 2
        tag = self._tag
        fds = self._exchange_fds(vb.fd(), tag) if self.world > 1 else {}
        buf.peers = []
        for r in range(self.world):
            if r == self.rank:
                buf.peers.append(buf.local)
            else:
                buf.peers.append(vb.open_peer(0, fds[r]))       # pid 0: the descriptor is already ours
                C.close_fd(fds[r])
        buf.table = torch.tensor([t.data_ptr() for t in buf.peers], dtype=torch.int64, device=self.device)
        if self.world > 1:
            dist.barrier(group=self.group)
        if multicast and self.world > 1:
            ch = self._channel()
            if self.rank == 0:
                mc_fd = vb.mc_create()
                for r in range(1, self.world):
                    ch.send(r, tag + 1, int(mc_fd))
            else:
                src, t, f = ch.recv()
                assert src == 0 and t == tag + 1
                vb.mc_import(0, int(f))
                C.close_fd(int(f))
            dist.barrier(group=self.group)
            vb.mc_add_device()
            dist.barrier(group=self.group)            # all devices joined before anybody binds
            buf.mc = vb.mc_bind_and_map()
            dist.barrier(group=self.group)
        self.buffers[name] = buf
        return buf


class LocalWorld(object):
    """``world`` virtual ranks in this process.  ``devices[r]`` is the GPU of
    virtual rank r (default: all on the current device -> loop-back)."""

    def __init__(self, world: int, devices: Optional[List[int]] = None):
        C = native.load()
        self._C = C
        self.world = world
        cur = torch.cuda.current_device()
        self.devices = [cur] * world if devices is None else list(devices)
        for d in set(self.devices):
            for p in set(self.devices):
                if d != p and not C.enable_peer_access(d, p):
                    raise RuntimeError('no peer access %d -> %d' % (d, p))
        self.buffers: Dict[str, List[_Buffer]] = {}
        self.lock = threading.Lock()

    def alloc(self, name: str, nbytes: int) -> List[_Buffer]:
        C = self._C
        locals_ = [C.symm_alloc(int(nbytes), d)[0] for d in self.devices]
        out = []
        for r, d in enumerate(self.devices):
            b = _Buffer(name, nbytes)
            b.local = locals_[r]
            b.peers = locals_
            b.table = torch.tensor([t.data_ptr() for t in locals_], dtype=torch.int64,
                                   device=torch.device('cuda', d))
            out.append(b)
        self.buffers[name] = out
        return out

    def view(self, rank: int) -> '_LocalRankView':
        return _LocalRankView(self, rank)


class _LocalRankView(object):
    """What one virtual rank sees: same interface as :class:`SymmetricWorld`,
    with allocations shared through the parent (first caller allocates)."""

    def __init__(self, parent: LocalWorld, rank: int):
        self.parent = parent
        self.rank = rank
        self.world = parent.world
        self.device = torch.device('cuda', parent.devices[rank])
        self.group = None

    def alloc(self, name: str, nbytes: int) -> _Buffer:
        with self.parent.lock:          # virtual ranks may allocate from their own threads
            if name not in self.parent.buffers:
                self.parent.alloc(name, nbytes)
        b = self.parent.buffers[name][self.rank]
        assert b.nbytes == nbytes
        return b

    def barrier(self):
        torch.cuda.synchronize()
