"""
AllReduce-SGD comparator.

The reference's AR baseline is ``torch.nn.parallel.DistributedDataParallel``
(``gossip_sgd.py:179-180``): bucketed NCCL all-reduces + a separate optimizer.
Here the exact-averaging baseline is built from the same parts as the gossip
path so the comparison isolates the algorithm:

* parameters in one flat arena, gradients in ONE flat buffer that lives in
  NVSwitch-mapped symmetric memory;
* ``sgp_allreduce_sgd_kernel``: every rank pulls all peers' gradient buffers
  with 16-byte P2P loads, sums them in rank order (replicas stay bit-identical),
  scales by 1/world and applies SGD-momentum in the same pass -- one kernel,
  no NCCL call, no bucket copies;
* ``transport='nvls'`` (the default whenever the GPUs support NVSwitch multicast):
  ``sgp_nvls_allreduce_kernel`` -- parameters and gradients live in VMM symmetric
  memory with a multicast mapping; every rank reduces ITS 1/world slice of the
  gradients inside the switch (``multimem.ld_reduce``), applies SGD-momentum to
  that slice only (sharded optimizer step) and multicasts the new parameters to
  every replica (``multimem.st``): ~2 x 4n bytes over NVLink per GPU instead of
  (world-1) x 4n, bit-identical replicas, still one kernel and no NCCL call;
* ``transport='nccl'`` keeps a library path (one in-place ``all_reduce`` on the
  flat gradient + the fused local SGD kernel) as a second comparator.
"""

from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist
from torch.nn.modules import Module

from ..ops import native
from ..utils.arena import FlatArena
from .distributed import consensus_unsupported
from .trainer import GossipTrainer


class AllReduceDataParallel(Module):

    def __init__(self, module, rank=None, world_size=None, transport='auto',
                 grad_dtype=torch.float32, timeout_s=60.0, grid=None, gossip_dtype=None):
        super().__init__()
        from .distributed import check_gossip_dtype
        check_gossip_dtype(gossip_dtype, 'AllReduceDataParallel')
        self.module = module
        if rank is None or world_size is None:
            if dist.is_initialized():
                rank, world_size = dist.get_rank(), dist.get_world_size()
            else:
                rank, world_size = 0, 1
        self.rank, self.world_size = rank, world_size
        params = list(module.parameters())
        assert all(p.dtype == torch.float32 and p.is_cuda for p in params)
        self.device = params[0].device
        from .symmetric import LocalWorld, SymmetricWorld, VmmSymmetricWorld
        spans_hosts = False
        if transport == 'auto':
            # the NVLS / P2P kernels map every rank's buffers (fd passing, CUDA IPC): one host, one
            # NVLink domain.  Ranks on several hosts reduce with NCCL and keep the fused local step.
            from .distributed import _single_nvlink_domain
            if world_size > 1 and dist.is_initialized() and not _single_nvlink_domain(world_size, True):
                transport, spans_hosts = 'nccl', True
            else:
                transport = 'nvls' if (world_size > 1 and VmmSymmetricWorld.supported(self.device)) else 'p2p'
        if transport == 'nvls' and world_size == 1:
            transport = 'p2p'
        self.transport = transport
        self._timeout_s = float(timeout_s)
        self._z_buf = None
        if transport == 'nvls':
            self.world = VmmSymmetricWorld(self.device)

            def symmetric_alloc(numel, dtype, device):
                # the parameter arena itself lives in multicast-bound symmetric memory: the kernel
                # all-gathers the updated slices straight into every replica's parameters
                self._z_buf = self.world.alloc('ar.z', int(numel) * 4)
                return self._z_buf.local.view(dtype)
            self.arena = FlatArena(params, device=self.device, allocator=symmetric_alloc)
        else:
            self.arena = FlatArena(params, device=self.device)
        self.arena.adopt(params)
        if world_size > 1:          # AR replicas must start identical
            dist.broadcast(self.arena.flat, src=0)
            for b in module.buffers():
                dist.broadcast(b.data, src=0)
        C = native.load()
        self.C = C
        if transport != 'nvls':
            # (several hosts: nothing is peer-mapped, the buffers below are plain local allocations)
            self.world = (SymmetricWorld(self.device) if (world_size > 1 and not spans_hosts)
                          else LocalWorld(1, [self.device.index]).view(0))
        n = self.arena.total
        esize = 4 if grad_dtype == torch.float32 else 2
        self._grad_buf = self.world.alloc('ar.grad', n * esize)
        self.grad_flat = self._grad_buf.local.view(grad_dtype)[:n]
        self.grad_flat.zero_()
        self.arena.bind_grads(params, self.grad_flat)
        self.momentum = self.arena.new_buffer()
        self.pad = (self.world.alloc('ar.pad', C.PAD_BYTES, multicast=False) if transport == 'nvls'
                    else self.world.alloc('ar.pad', C.PAD_BYTES))
        self.state = torch.zeros(C.STATE_BYTES, dtype=torch.uint8, device=self.device)
        self.state.view(torch.float32)[C.STATE_OFF_PSW // 4: C.STATE_OFF_PSW // 4 + 2] = 1.0
        self.hyper = torch.zeros(C.HYPER_FLOATS, dtype=torch.float32, device=self.device)
        self._hyper_host = torch.zeros(C.HYPER_FLOATS, dtype=torch.float32).pin_memory()
        self._hyper_cache = None
        table = torch.zeros(1, C.TABLE_ROW, dtype=torch.int32, device=self.device)
        wtable = torch.zeros(1, C.WTABLE_ROW, dtype=torch.float32, device=self.device)
        wtable[0, 0] = 1.0
        self.ctx = C.GossipContext(
            z=self.arena.flat, g=self.grad_flat, m=self.momentum, shadow=None, residual=None,
            pad_ptrs=self.pad.table, outbox_ptrs=None, table=table, wtable=wtable,
            rank=self.world.rank, world=self.world.world, state=self.state, hyper=self.hyper,
            timeout_s=float(timeout_s))
        sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        if grid is None:
            grid = min(self.ctx.max_grid(), 2 * sms)
        self.grid = int(max(1, min(grid, n // C.CHUNK)))
        if transport == 'nvls':
            per_rank = -(-(n // C.CHUNK) // self.world.world)          # chunks of one rank's slice
            self.grid = int(max(1, min(self.grid, C.nvls_max_grid(self.device.index), per_rank)))
            self._z_mc = self._z_buf.mc.view(torch.float32)[:n]
            self._g_mc = self._grad_buf.mc.view(grad_dtype)[:n]
        self.steps = 0
        torch.cuda.synchronize(self.device)
        self.world.barrier()

    def forward(self, *a, **kw):
        return self.module(*a, **kw)

    # the replicas are identical by construction: there is no consensus distance to measure
    consensus_distance = average_model = averaged = consensus_unsupported('AllReduceDataParallel')

    def set_hyper(self, lr, momentum, weight_decay, nesterov, grad_scale=1.0):
        key = (float(lr), float(momentum), float(weight_decay), bool(nesterov), float(grad_scale))
        if key == self._hyper_cache:
            return
        self._hyper_cache = key
        h = self._hyper_host
        h[0], h[1], h[2], h[3], h[4], h[5] = key[0], key[1], key[2], float(key[3]), 1.0, key[4]
        self.hyper.copy_(h, non_blocking=True)

    def allreduce_step(self):
        """grads <- mean over ranks ; SGD-momentum ; grads <- 0   (current stream)"""
        C = self.C
        if self.transport == 'nccl' and self.world_size > 1:
            dist.all_reduce(self.grad_flat)
            self.set_hyper(*self._hyper_cache[:4], grad_scale=1.0 / self.world_size)
            self.ctx.step(C.F_SGD | C.F_ZERO_GRAD | C.F_PHASE1 | C.F_NO_ROTATE, self.grid)
        elif self.transport == 'nvls':
            # in-switch reduce of the owned slice + sharded SGD + multicast all-gather; the kernel
            # also clears the consumed gradient slice on every rank (multimem.st of zeros)
            C.nvls_allreduce(self.arena.flat, self._z_mc, self._g_mc, self.momentum, self.pad.table,
                             self.state, self.hyper, self.world.rank, self.world.world, self._timeout_s,
                             1.0, True, self.grid)
            self.steps += 1
        else:
            self.ctx.allreduce_sgd(self._grad_buf.table, 0, self.grid)
            C.zero_(self.grad_flat)
            self.steps += 1

    def check(self):
        st = int(self.state.view(torch.int32)[self.C.STATE_OFF_STATUS // 4].item())
        if st != 0:
            raise RuntimeError('all-reduce kernel error %d on rank %d' % (st, self.rank))


class _EngineShim(object):
    """The slice of GossipEngine that GossipTrainer touches."""

    def __init__(self, ar: AllReduceDataParallel):
        self.ar = ar
        self.device = ar.device
        self.steps = 0
        from ..ops import native
        self.C = native.load()

    def set_hyper(self, lr, momentum, weight_decay, nesterov, do_sgd=True, grad_scale=1.0):
        self.ar.set_hyper(lr, momentum, weight_decay, nesterov, grad_scale)

    def check(self):
        self.ar.check()


class ARTrainer(GossipTrainer):
    """Graph-captured forward/backward + the fused all-reduce+SGD kernel."""

    def __init__(self, model: AllReduceDataParallel, lr, momentum=0.9, weight_decay=1e-4,
                 nesterov=True, criterion=None, amp_dtype=torch.bfloat16, use_cuda_graph=True,
                 warmup_iters=3, channels_last=True, lars=False):
        if lars:
            raise ValueError('LARS is not supported by the all-reduce optimizer: its sharded fused step '
                             'holds 1/n of each tensor, so no rank sees a whole tensor\'s norm')
        self.model = model
        self.ar = model

        class _Opt(object):
            param_groups = [dict(lr=lr, momentum=momentum, weight_decay=weight_decay,
                                 nesterov=nesterov)]
            grad_scale = 1.0
        self.opt = _Opt()
        self.engine = _EngineShim(model)
        self.k = None
        self.overlap = False
        self.gossip = False
        self._init_runtime(model.device, criterion, amp_dtype, use_cuda_graph, warmup_iters, channels_last)

    def _one_step(self, first=False):
        self._fwd_bwd()
        self.ar.allreduce_step()

    def _after_replay(self):
        self.ar.steps += 1

    def finish(self):
        torch.cuda.synchronize(self.device)
        self.ar.check()

    def check(self):
        self.ar.check()
