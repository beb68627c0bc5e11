"""
GossipDataParallel: SGP / Overlap-SGP / D-PSGD model wrapper.

API parity with ``gossip/distributed.py:39-589`` (constructor arguments,
``forward``, ``transfer_params``, ``sync_comms``, ``block``, ``state_dict`` /
``load_state_dict``, ``train`` / ``eval``, ``update_gossiper``,
``ps_numerator`` / ``unbias``, ``_query_gossip_queue`` and the public
attributes ``ps_weight``, ``is_ps_numerator``, ``gossip_enable``,
``gossiping``, ``params_mixed``, ``overlap``, ``synch_freq``, ``asynch``,
``lazy_mixing``, ``num_updates``, ``dist_config``, ``gossip_stream``).

What is different underneath (H100-first):

* parameters are re-homed into ONE flat, 256-byte aligned arena at wrap time
  (``utils/arena.py``); there is no per-step flatten / unflatten / per-tensor
  copy (reference K4/K5/K8).
* there is no gossip *thread*.  The reference hands the parameters to a Python
  thread that drives NCCL broadcasts and synchronises a stream
  (``gossip/distributed.py:459-510``).  Here a gossip step is a kernel launch:
  in sync mode ONE fused kernel on the current stream, in overlap mode a
  publish kernel on the current stream plus a gather kernel on
  ``gossip_stream`` that runs concurrently with the next forward/backward; the
  "hand-off" is a CUDA event.
* the push-sum algebra (bias / de-bias / residual add / pre-scale) happens
  inside those kernels; with :class:`~..optim.FusedGossipSGD` so does the
  SGD-momentum update (reference K1-K9).
* on CPU tensors / the gloo backend the same state machine runs over
  ``isend/irecv`` (``transport='c10d'``), which is also the oracle the kernel
  path is tested against.

State convention: between launches the parameters always hold the de-biased
estimate ``z = x / w`` on the kernel transport (``is_ps_numerator`` is only
True between a backward pass and the next gossip launch when an *external*
optimizer is used); on the c10d transport they follow the reference's
numerator / de-biased alternation.
"""

from __future__ import annotations

import contextlib
import math
import numbers
import time
from collections import namedtuple
from typing import Dict

import torch
import torch.distributed as dist
from torch.autograd import Variable
from torch.nn.modules import Module

from ..gossiper import C10dTransport, bf16_message_numel, bf16_message_weight, pack_bf16_message
from ..mixing_manager import UniformMixing
from ..topology.graph_manager import NPeerDynamicDirectedExponentialGraph as NPDDEGraph
from ..utils import tracing
from ..utils.arena import FlatArena
from ..utils.helpers import communicate, create_process_group, group_by_dtype, make_logger

HEARTBEAT_TIMEOUT = 300  # seconds a rank waits for its in-neighbours (reference :36)


class ConsensusStats(namedtuple('ConsensusStats', ['distance_sq', 'average_norm_sq', 'rank_distance_sq'])):
    """Result of :meth:`GossipDataParallel.consensus_distance` / ``average_model``:
    ``distance_sq = (1/n) sum_i |z_i - zbar|^2``, ``average_norm_sq = |zbar|^2`` and, from
    ``average_model`` only, ``rank_distance_sq[i] = |z_i - zbar|^2`` (else None)."""
    __slots__ = ()

    @property
    def relative(self) -> float:
        """sqrt(distance_sq / average_norm_sq): the ranks' RMS spread relative to the average"""
        if self.average_norm_sq > 0:
            return math.sqrt(self.distance_sq / self.average_norm_sq)
        return 0.0 if self.distance_sq == 0 else math.inf


def consensus_unsupported(kind):
    """A ``consensus_distance`` / ``average_model`` / ``averaged`` stand-in for wrappers that do
    not implement them (AD-PSGD, all-reduce): raises ValueError."""
    def method(self, *args, **kwargs):
        raise ValueError('consensus_distance(), average_model() and averaged() are implemented by '
                         'GossipDataParallel (SGP, D-PSGD, Overlap-SGP), not by %s' % kind)
    return method


# --------------------------------------------------------------------------- #
# backends
# --------------------------------------------------------------------------- #
class _KernelBackend(object):
    """sm_90a data plane: GossipEngine over symmetric memory."""

    name = 'nvlink'

    def __init__(self, owner, arena: FlatArena, graph, mixing, world_view, overlap,
                 compute_dtype, timeout_s, grid, msg_dtype=None):
        from ..ops.peer_mix import GossipEngine
        self.owner = owner
        self.arena = arena
        self.shadow = None
        if compute_dtype is not None and compute_dtype != torch.float32:
            assert compute_dtype == torch.bfloat16, 'compute copies are bf16'
            self.shadow = arena.new_buffer(dtype=torch.bfloat16)
            self.shadow.copy_(arena.flat)
        self.engine = GossipEngine(world_view, arena.flat, graph, mixing, shadow=self.shadow,
                                   with_residual=msg_dtype is None, timeout_s=timeout_s, grid=grid,
                                   name=owner._symm_name, msg_dtype=msg_dtype)
        self.gather_event = None
        self.residual_pending = False       # a gather finished/launched and is not folded yet
        self.sgd_pending = False            # FusedGossipSGD.step() deferred into next launch

    # optimizer buffers are attached lazily by FusedGossipSGD
    def attach_sgd(self, grad_flat, momentum_flat, grad2=None):
        self.engine.set_sgd_buffers(grad_flat, momentum_flat, grad2)


class _C10dBackend(object):
    """Portable data plane: isend/irecv of edge-weighted snapshots (+ the
    push-sum weight as one extra element), residual folded at the next query.

    ``msg_bf16``: every message is Q(a_j * x) in bf16 with the fp32 weight in its tail (see
    ``gossiper.pack_bf16_message``); the sender subtracts what it sends instead of scaling by
    the self weight, so the local result is x - sum_out m_j + sum_in m_j, accumulated in fp32."""

    name = 'c10d'

    def __init__(self, owner, arenas: Dict[torch.dtype, FlatArena], graph, mixing,
                 comm_device, group=None, msg_bf16=False):
        self.owner = owner
        self.msg_bf16 = msg_bf16
        self._sent = []             # bf16: (arena, Q(a_j x)) subtracted by the last start()
        self.arenas = arenas
        self.graph = graph
        self.mixing = mixing
        self.comm_device = comm_device
        self.transport = C10dTransport(group)
        self.pending = None
        self.send_bufs, self.recv_bufs = {}, {}

    def _buf(self, store, key, numel, dtype):
        t = store.get(key)
        if t is None or t.numel() != numel:
            t = torch.empty(numel, dtype=dtype, device=self.comm_device)
            if self.comm_device.type == 'cpu' and torch.cuda.is_available():
                t = t.pin_memory()
            store[key] = t
        return t

    def start(self, ps_weight: float, pollable: bool = False, mix: bool = True):
        """Snapshot x (numerator, NOT yet self-scaled) and post the exchange.
        Returns the self-loop weight the caller applies locally.  ``mix=False`` (retry of an
        interrupted round): the local numerator already carries the self-loop scaling of the
        failed attempt, so the messages are rebuilt from ``x / self_w`` (== the pre-mix
        numerator) and the caller must NOT scale again.  With bf16 messages the numerator is
        never scaled by the caller: start() subtracts the messages itself (and a retry first
        adds back those of the failed attempt); only the weight follows the rule above."""
        out_edges, in_edges = self.graph.get_edges()
        self_w, edge_w = self.mixing.scalar_weights([e.dest for e in out_edges])
        undo = 1.0 if mix else 1.0 / float(self_w)
        if self.msg_bf16:
            if not mix:
                for arena, q in self._sent:
                    arena.flat.add_(q.to(arena.flat.dtype))
            self._sent = []
        reqs, recvs, keep, poll = [], [], [], []
        for dtype, arena in self.arenas.items():
            n = bf16_message_numel(arena.total) if self.msg_bf16 else arena.total + 1
            msg_dtype = torch.bfloat16 if self.msg_bf16 else dtype
            remote_in = [e for e in in_edges if e.src != e.dest]
            bufs = [self._buf(self.recv_bufs, (dtype, i), n, msg_dtype) for i in range(len(remote_in))]
            batched = getattr(self.transport, 'batched', False)   # NCCL: receives + sends as ONE grouped launch
            if batched:
                rr = []
            elif pollable:   # gloo cannot poll a plain irecv (see _PolledRecv)
                rr = [self.transport.post_polled_recv(b, e) for b, e in zip(bufs, remote_in)]
            else:
                rr = self.transport.post_recvs(bufs, remote_in)
            reqs += rr
            poll += rr
            local_add = []
            send_edges, send_msgs = [], []
            for i, e in enumerate(out_edges):
                msg = self._buf(self.send_bufs, (dtype, i), n, msg_dtype)
                if self.msg_bf16:
                    a = float(edge_w[e.dest])
                    q = pack_bf16_message(msg, arena.flat, a, float(ps_weight) * a * undo)
                    self._sent.append((arena, q))
                    if self.comm_device.type == 'cpu' and arena.flat.is_cuda:
                        torch.cuda.current_stream().synchronize()
                else:
                    msg[:-1].copy_(arena.flat, non_blocking=True)
                    if self.comm_device.type == 'cpu' and arena.flat.is_cuda:
                        torch.cuda.current_stream().synchronize()
                    msg[-1] = ps_weight
                    msg.mul_(edge_w[e.dest] * undo)
                if e.dest == e.src:
                    local_add.append(msg)
                else:
                    send_edges.append(e)
                    send_msgs.append(msg)
            if batched:
                # (symmetric exchanges -- in-peer == out-peer -- deadlock on NCCL when "irecv, then
                # isend" is launched op by op on both sides; see gossiper.C10dTransport)
                rr, _ = self.transport.exchange(bufs, remote_in, send_msgs, send_edges)
                reqs += rr
                poll += rr
            else:
                reqs += self.transport.post_sends(send_msgs, send_edges)
            recvs.append((arena, bufs + local_add))
            keep.append(send_msgs)
        for arena, q in self._sent:             # the sender keeps what it did not send
            arena.flat.sub_(q.to(arena.flat.dtype))
        self.pending = (reqs, recvs, keep, poll)
        if self.graph.is_dynamic_graph():
            self.graph.get_peers(rotate=True)
        return self_w

    def abort(self):
        """Drop an interrupted round (reference: ``gossiper.clean_msg_buffers_()`` after a
        RuntimeError in the gossip thread, ``gossip/distributed.py:494-498``)."""
        self.pending = None

    def done(self) -> bool:
        if self.pending is None:
            return True
        return all(_req_done(r) for r in self.pending[3])

    def finish(self, timeout_s: float = None):
        """Wait and fold: returns the residual push-sum weight.  ``timeout_s`` is the
        heartbeat: a peer that does not deliver in time raises ``NameError('Gossip flag
        timeout')`` like the reference's gossip-flag wait (``gossip/distributed.py:349-352``)
        instead of hanging until the process group's own (30 min) timeout."""
        reqs, recvs, _, _ = self.pending
        # NCCL works keep their stream-ordered wait() (and NCCL's own watchdog); the heartbeat
        # wrapper is for host-side (gloo) requests
        host_side = self.comm_device.type == 'cpu'
        deadline = time.time() + timeout_s if (timeout_s is not None and host_side) else None
        for i in range(len(reqs)):
            _wait_req(reqs, i, deadline)
        w_res = 0.0
        first = True
        staged = False
        for arena, bufs in recvs:
            for b in bufs:
                staged = staged or (b.device != arena.flat.device)
                if self.msg_bf16:
                    arena.flat.add_(b[:arena.total].to(arena.flat.device, non_blocking=True).to(arena.flat.dtype))
                    if first:
                        w_res += bf16_message_weight(b, arena.total)
                else:
                    arena.flat.add_(b[:-1].to(arena.flat.device, non_blocking=True))
                    if first:
                        w_res += float(b[-1])
            first = False
        if staged and torch.cuda.is_available():
            # pinned CPU receive buffers -> GPU arena: the async H2D copies read the buffers when
            # the STREAM reaches them.  start() re-posts irecvs into the same buffers right away
            # (overlap mode: finish and start run back to back), so a peer's next message could
            # land before the DMA of this round has run.  Wait for the copies first.
            for arena, _ in recvs:
                if arena.flat.is_cuda:
                    torch.cuda.current_stream(arena.flat.device).synchronize()
        self.pending = None
        self._sent = []
        return w_res


def _wait_req(reqs, i, deadline):
    """``reqs[i].wait()`` bounded by the heartbeat deadline.  gloo offers no usable timed wait
    (an expired ``Work.wait(timeout)`` closes the connection pair, and ``is_completed()`` never
    flips), so an unfinished request is parked in a helper thread (:class:`_PolledRecv`) and the
    wrapper replaces it in ``reqs`` -- a later retry waits on the same wrapper."""
    req = reqs[i]
    if deadline is None:
        req.wait()
        return
    if not hasattr(req, 'wait_for'):
        if _req_done(req):
            req.wait()
            return
        from ..gossiper import _PolledRecv
        req = reqs[i] = _PolledRecv(req)
    if not req.wait_for(max(deadline - time.time(), 1e-3)):
        raise NameError('Gossip flag timeout')


def _req_done(req) -> bool:
    try:
        return bool(req.is_completed())
    except Exception:
        return False


# --------------------------------------------------------------------------- #
# wrapper
# --------------------------------------------------------------------------- #
_INSTANCES = [0]


class GossipDataParallel(Module):
    """Distributed gossip model wrapper (SGP if ``push_sum`` else D-PSGD;
    ``overlap=True`` -> OSGP; ``synch_freq>0`` -> bounded-staleness async)."""

    def __init__(self, module, device_ids=None, rank=None, world_size=None,
                 graph=None, mixing=None, comm_device=None, push_sum=True,
                 overlap=False, synch_freq=0, verbose=False, use_streams=True,
                 nprocs_per_node=1, local_node_group=None,
                 transport='auto', compute_dtype=None, symmetric_world=None,
                 heartbeat_timeout=HEARTBEAT_TIMEOUT, grid=None, symmetric_name=None,
                 gossip_dtype=None, slowmo_frequency=0, slowmo_lr=1.0, slowmo_momentum=0.5):
        super(GossipDataParallel, self).__init__()
        # SlowMo (perform_slowmo): every slowmo_frequency optimizer steps, exact average + slow
        # momentum step with learning rate slowmo_lr and momentum slowmo_momentum; 0 = off
        self.slowmo_frequency, self.slowmo_lr, self.slowmo_momentum = check_slowmo_args(
            slowmo_frequency, slowmo_lr, slowmo_momentum)
        if self.slowmo_frequency and nprocs_per_node > 1:
            raise ValueError('SlowMo (slowmo_frequency > 0) is not implemented for nprocs_per_node > 1 '
                             '(hierarchical mode)')
        # bf16 gossip messages: half the bytes per in-neighbour, push-sum mass conserved exactly
        # (the sender keeps what it did not send); parameters and push-sum weights stay fp32
        self.gossip_dtype = check_gossip_dtype(
            gossip_dtype, 'overlap=True (OSGP)' if overlap else
            'nprocs_per_node > 1' if nprocs_per_node > 1 else None)
        _INSTANCES[0] += 1
        self._instance_id = _INSTANCES[0]
        self._timeout_s = float(heartbeat_timeout)
        # name of this wrapper's symmetric allocations: identical on every rank of the world
        # (one instance per process: the instance counter; several virtual ranks inside ONE process
        # -- LocalWorld loop-back -- must pass the same explicit name)
        self._symm_name = symmetric_name or ('gdp%d' % self._instance_id)
        self.last_consensus = None      # ConsensusStats of the last consensus_distance() / average_model()
        self._gossip_done = None        # consensus: event on gossip_stream (prepare_consensus)
        self.exposed_comm_s = 0.0       # c10d data plane: host seconds blocked waiting for peers
        self.gossip_retries = 0         # interrupted gossip rounds that were re-queued (soft retry)

        first_param = next(module.parameters())
        on_cuda = first_param.is_cuda
        # one process per GPU: the default device list is the module's device,
        # not "every visible GPU" (reference :49-52 drives 8 GPUs per process)
        if device_ids is None:
            device_ids = [first_param.device.index] if on_cuda else []
        self.device_ids = list(device_ids)
        self.output_device = self.device_ids[0] if self.device_ids else None
        self.nprocs_per_node = nprocs_per_node

        if world_size is None or rank is None:
            assert dist.is_initialized()
            rank, world_size = dist.get_rank(), dist.get_world_size()
        self.process_rank = rank

        self.local_node_group = local_node_group
        if self.nprocs_per_node > 1:
            self.local_rank = self.process_rank % self.nprocs_per_node
            world_size //= nprocs_per_node
            rank //= nprocs_per_node
            if local_node_group is None:
                for node in range(world_size):
                    ranks = list(range(node * nprocs_per_node, (node + 1) * nprocs_per_node))
                    grp = create_process_group(ranks)
                    if self.process_rank in ranks:
                        self.local_node_group = grp
        else:
            self.local_rank = 0
        self.is_local_master = (self.process_rank % self.nprocs_per_node == 0)

        self.module = module
        self._module_copies = [self.module]
        self._replica_arenas = []       # single-process multi-GPU mode: (arena, grad_flat) per replica
        first_param_dtype = first_param.dtype

        # -- communication device / transport ------------------------------- #
        backend_name = dist.get_backend() if dist.is_initialized() else None
        if comm_device is None:
            cpu_comm = (backend_name == 'gloo') or not on_cuda
            comm_device = torch.device('cpu') if cpu_comm else torch.device('cuda', first_param.device.index)
        comm_device = torch.device(comm_device)
        if comm_device.type == 'cuda' and comm_device.index is None and on_cuda:
            comm_device = torch.device('cuda', first_param.device.index)
        self.__cpu_comm = comm_device.type == 'cpu'

        if graph is None:
            graph = NPDDEGraph(rank, world_size, self.nprocs_per_node, self.local_rank)
        if mixing is None:
            mixing = UniformMixing(graph, comm_device)
        # push_sum=False is D-PSGD (the reference swaps in its PushPull gossiper,
        # gossip/distributed.py:145-150).  Plain averaging is only correct when the mixing matrix
        # is doubly stochastic -- on the circulant schedules of graph_manager that means every
        # phase is balanced (as many in- as out-neighbours), and then the push-sum weight stays
        # exactly 1.  Both data planes here always carry the weight (one scalar), so the flag
        # selects no different code path; it is validated instead of silently ignored.
        if not push_sum:
            for outs, ins in graph.phases():
                if len(outs) != len(ins):
                    raise ValueError('push_sum=False (D-PSGD) needs a balanced schedule (doubly '
                                     'stochastic mixing): phase with out-peers %s but in-peers %s'
                                     % (sorted(outs), sorted(ins)))

        self.dist_config = {
            'verbose': verbose, 'comm_device': comm_device, 'graph': graph,
            'mixing': mixing, 'push_sum': push_sum, 'rank': rank,
            'process_rank': self.process_rank, 'world_size': world_size,
            'cpu_comm': self.__cpu_comm,
        }
        self.overlap = overlap
        self.synch_freq = synch_freq
        self.num_updates = 0
        self.asynch = synch_freq > 0
        self.logger = make_logger(rank, verbose)

        # -- parameters -> flat arenas --------------------------------------- #
        params = [p for p in module.parameters()]
        by_dtype = group_by_dtype(params)
        self._arenas: Dict[torch.dtype, FlatArena] = {}
        self._hier = self._make_local_nvls_group(by_dtype, on_cuda, first_param.device)
        for dtype, group in by_dtype.items():
            alloc = self._hier.arena_allocator if (self._hier is not None and dtype == torch.float32) else None
            arena = FlatArena(group, device=group[0].device, allocator=alloc)
            arena.adopt(group)
            self._arenas[dtype] = arena
        self._params_by_dtype = by_dtype
        self._hier_grad = None
        if self._hier is not None:
            # the flat gradient of the local ranks lives in multicast-bound symmetric memory so
            # that the local-node average is one in-switch reduction (FusedGossipSGD reuses it)
            self._hier_grad = self._hier.finish(self._arenas[torch.float32])
            self._arenas[torch.float32].bind_grads(by_dtype[torch.float32], self._hier_grad)

        if len(self.device_ids) > 1:
            self._build_local_replicas()

        all_fp32 = list(by_dtype.keys()) == [torch.float32]
        # SlowMo state, fp32, arena-sized and identical on every rank: slow momentum u and the model
        # at the start of the outer iteration x_prev.  Allocated here because the collective must not
        # allocate (virtual loop-back ranks run it from threads, see prepare_consensus)
        self._slowmo_u = self._slowmo_x_prev = None
        self._slowmo_initialized = False
        self._slowmo_calls = 0
        if self.slowmo_frequency:
            if not all_fp32:
                raise ValueError('SlowMo (slowmo_frequency > 0) needs fp32 parameters')
            self._slowmo_u = torch.zeros_like(self._arenas[torch.float32].flat)
            self._slowmo_x_prev = torch.zeros_like(self._slowmo_u)
        if transport == 'auto':
            use_kernels = on_cuda and not self.__cpu_comm and all_fp32 and _native_ok()
            # the kernel data plane maps every peer's buffers over CUDA IPC / NVSwitch: it needs
            # ALL ranks on one host (one NVLink domain) and at most MAX_RANKS of them.  Anything
            # else (the multi-node SLURM scripts) falls back to the c10d data plane.
            if not _single_nvlink_domain(world_size * self.nprocs_per_node, use_kernels):
                if use_kernels:
                    self.logger.info('ranks span several hosts (or > %d ranks): using the c10d '
                                     'transport instead of the NVLink kernels' % _max_kernel_ranks())
                use_kernels = False
        else:
            use_kernels = transport in ('nvlink', 'kernel', 'peer')
        if use_kernels and not (on_cuda and all_fp32):
            raise RuntimeError('nvlink transport needs fp32 CUDA parameters')
        if use_kernels and not _native_ok():
            raise RuntimeError('nvlink transport requested but the sm_90a extension is '
                               'not available (python -m stochastic_gradient_push_b200.ops.build)')

        # push-sum weight (host mirror; the kernel transport keeps the truth on device)
        self._ps_weight = torch.ones(1, device=comm_device, dtype=first_param_dtype)
        self.is_ps_numerator = False
        self.gossip_enable = True
        self.gossiping = False
        self.params_mixed = True
        self.gossip_ps_factor = torch.zeros(1, device=comm_device, dtype=first_param_dtype)
        self.gossip_ps_weight = self._ps_weight.clone()
        self.lazy_mixing = (not self.asynch and mixing.is_regular() and not self.overlap)
        self.lazy_ps_factor = self.gossip_ps_factor.clone()
        self._w = 1.0                      # c10d transport: python mirror of ps_weight
        self._rounds_started = 0
        self._fused_optimizer = None

        if on_cuda and not self.__cpu_comm and use_streams:
            self.gossip_stream = torch.cuda.Stream(device=first_param.device)
        elif on_cuda:
            self.gossip_stream = torch.cuda.current_stream(first_param.device)
        else:
            self.gossip_stream = None

        # -- data plane ------------------------------------------------------- #
        self._kernel = None
        self._c10d = None
        # hierarchical mode: the node masters rendezvous among themselves; new_group is
        # collective over the WHOLE world, so every rank creates it
        self._masters_group = None
        if self.nprocs_per_node > 1 and world_size > 1 and dist.is_initialized():
            # (both data planes: the kernel rendezvous and the bounded-staleness drain of the
            # c10d plane are collectives among the node masters only)
            self._masters_group = dist.new_group(
                [r * self.nprocs_per_node for r in range(world_size)])
        if self.is_local_master:
            if use_kernels:
                if symmetric_world is None:
                    symmetric_world = self._make_symmetric_world(world_size, first_param.device)
                self._kernel = _KernelBackend(
                    self, self._arenas[torch.float32], graph, mixing, symmetric_world,
                    overlap, compute_dtype, self._timeout_s, grid, msg_dtype=self.gossip_dtype)
            else:
                self._c10d = _C10dBackend(self, self._arenas, graph, mixing, comm_device,
                                          msg_bf16=self.gossip_dtype is not None)
        self.transport = 'nvlink' if self._kernel is not None else 'c10d'
        self._twin = []          # [bf16 compute twin] (a list so it is not a registered submodule)
        if self._kernel is not None and self._kernel.shadow is not None:
            self._twin.append(self._build_compute_twin())
        self.dist_config['gossipers'] = {
            dtype: _GossiperView(self, dtype) for dtype in self._arenas}
        self.gossip_ps_factor.fill_(mixing.scalar_weights()[0])
        self.lazy_ps_factor.copy_(self.gossip_ps_factor)
        self.logger.debug('lazy mixing: {}; transport: {}'.format(self.lazy_mixing, self.transport))

        self.__register_hooks()

    # ------------------------------------------------------------------ #
    # construction helpers
    # ------------------------------------------------------------------ #
    def _build_compute_twin(self):
        """bf16 twin of ``self.module`` for the forward/backward pass.

        Its convolution / linear parameters are bf16 views of the SHADOW arena that
        the gossip kernel rewrites every step (``SGP_F_SHADOW``), so no cast kernel
        ever runs (autocast re-casts all 54 weight tensors forward and their gradients
        backward, every step); its normalisation parameters ARE the fp32 master views
        and its buffers (running statistics) ARE the master module's buffers."""
        import copy
        from torch.nn.modules.batchnorm import _NormBase
        arena = self._arenas[torch.float32]
        twin = copy.deepcopy(self.module)
        norm_ids = set(id(p) for m in twin.modules() if isinstance(m, _NormBase)
                       for p in m.parameters(recurse=False))
        shadow_views = arena.views_of(self._kernel.shadow)
        with torch.no_grad():
            for p, v_master, v_shadow in zip(twin.parameters(), arena.views, shadow_views):
                p.data = v_master if id(p) in norm_ids else v_shadow
                p.grad = None
        for m_t, m_m in zip(twin.modules(), self.module.modules()):
            for name in list(m_m._buffers):
                m_t._buffers[name] = m_m._buffers[name]
        return twin

    @property
    def compute_module(self):
        """The module the fast path runs: the bf16 twin if ``compute_dtype`` was given,
        else the wrapped module itself."""
        return self._twin[0] if self._twin else self.module

    def _make_symmetric_world(self, world_size, device):
        from .symmetric import LocalWorld, SymmetricWorld
        if world_size == 1:
            return LocalWorld(1, [device.index]).view(0)
        return SymmetricWorld(device, self._masters_group)

    # ------------------------------------------------------------------ #
    # properties
    # ------------------------------------------------------------------ #
    @property
    def ps_weight(self):
        if self._kernel is not None:
            self._ps_weight.fill_(self._kernel.engine.ps_weight)
        else:
            self._ps_weight.fill_(self._w)
        return self._ps_weight

    @ps_weight.setter
    def ps_weight(self, v):
        val = float(v.reshape(-1)[0]) if torch.is_tensor(v) else float(v)
        self._w = val
        self._ps_weight.fill_(val)
        if self._kernel is not None:
            self._kernel.engine.ps_weight = val

    @property
    def arena(self) -> FlatArena:
        """fp32 parameter arena (the flagship path)."""
        return self._arenas[torch.float32]

    @property
    def engine(self):
        return self._kernel.engine if self._kernel is not None else None

    @property
    def compute_shadow(self):
        return self._kernel.shadow if self._kernel is not None else None

    # ------------------------------------------------------------------ #
    # reference API
    # ------------------------------------------------------------------ #
    def update_gossiper(self, attr, val):
        """Set ``attr`` (in practice ``'peers_per_itr'``) on the gossipers."""
        self.logger.debug('updating gossiper {} -> {}'.format(attr, val))
        for gossiper in self.dist_config['gossipers'].values():
            if val == getattr(gossiper, attr):
                self.logger.debug('nothing to update')
                return
            setattr(gossiper, attr, val)

    def state_dict(self, finish_gossip=True, *args, **kwargs):
        if finish_gossip:
            if self.asynch:
                self._drain_async()
            self._query_gossip_queue()
            self._flush_pending(drain=True)
        super_dict = super(GossipDataParallel, self).state_dict(*args, **kwargs)
        out = {'state_dict': super_dict,
               'ps_weight': self.ps_weight.detach().cpu().clone(),
               'is_ps_numerator': self.is_ps_numerator}
        if self.gossip_dtype is not None:
            # informational: parameters are fp32 either way, so a checkpoint loads across dtypes
            out['gossip_dtype'] = 'bfloat16'
        if self.slowmo_frequency:
            out['slowmo'] = {'u': self._slowmo_u.detach().cpu().clone(),
                             'x_prev': self._slowmo_x_prev.detach().cpu().clone(),
                             'initialized': self._slowmo_initialized,
                             'calls': self._slowmo_calls}
        return out

    def load_state_dict(self, load_dict, *args, **kwargs):
        state_dict = load_dict['state_dict']
        super(GossipDataParallel, self).load_state_dict(state_dict, *args, **kwargs)
        self.ps_weight = load_dict['ps_weight']
        self.is_ps_numerator = load_dict['is_ps_numerator']
        if self._kernel is not None and self._kernel.shadow is not None:
            self._kernel.shadow.copy_(self.arena.flat)
        sm = load_dict.get('slowmo')
        if sm is not None and self.slowmo_frequency:
            self._slowmo_u.copy_(sm['u'])
            self._slowmo_x_prev.copy_(sm['x_prev'])
            self._slowmo_initialized = bool(sm['initialized'])
            self._slowmo_calls = int(sm['calls'])

    # -- SlowMo: slow momentum over periodic exact averaging ------------------- #
    def perform_slowmo(self, optimizer) -> bool:
        """SlowMo (Wang et al., ICLR 2020) on top of gossip.  Call it after every optimizer step
        (in synchronous mode after ``transfer_params()``).  Every ``slowmo_frequency``-th call it
        drains in-flight gossip (as :meth:`state_dict` does), takes the push-sum average
        zbar = sum_i w_i z_i / sum_i w_i of the ranks' de-biased parameters and, with
        gamma = ``optimizer.param_groups[0]['lr']``, alpha = ``slowmo_lr``, beta = ``slowmo_momentum``:

            u <- beta u + (x_prev - zbar) / gamma ;  x_prev <- x_prev - alpha gamma u ;  z_i <- x_prev

        and resets every push-sum weight to 1.  The first such call only averages (x_prev <- zbar,
        u <- 0): no collective is needed at construction, at the cost of one period of slow
        momentum (the paper starts x_prev at the initial point).  Afterwards every rank holds the
        same parameters, u and x_prev.  The base optimizer's momentum and the BatchNorm buffers are
        left alone; beta = 0, alpha = 1 is periodic exact averaging.

        Returns True when the step ran (collective on those calls), False otherwise (always with
        ``slowmo_frequency=0``).  With a :class:`GossipTrainer` do not call it: ``trainer.step()``
        runs the step itself."""
        gamma = self._slowmo_tick(optimizer)
        if gamma is None:
            return False
        if self.asynch:
            self._drain_async()
        self._query_gossip_queue()
        self._flush_pending(drain=True)
        self.unbias()
        if self._kernel is not None:
            e = self._kernel.engine
            self.prepare_consensus()
            if self.gossip_stream is not None:
                self._gossip_done.record(self.gossip_stream)
                torch.cuda.current_stream().wait_event(self._gossip_done)
            self._slowmo_launch(gamma)
            e.poll(blocking=True)
        else:
            self._slowmo_c10d(gamma)
        return True

    def _slowmo_tick(self, optimizer):
        """count one optimizer step: the base learning rate if a SlowMo step is due now, else None"""
        if not self.slowmo_frequency:
            return None
        calls = self._slowmo_calls + 1
        if calls % self.slowmo_frequency:
            self._slowmo_calls = calls
            return None
        gamma = float(optimizer.param_groups[0]['lr'])
        if any(float(g['lr']) != gamma for g in optimizer.param_groups):
            # u is the displacement over gamma: one gamma per model (groups may differ in weight
            # decay or momentum, as with no-bias-decay)
            raise ValueError('SlowMo needs one base learning rate; the parameter groups have lr %s'
                             % [float(g['lr']) for g in optimizer.param_groups])
        if not gamma > 0:
            raise ValueError('SlowMo needs a positive base learning rate, got %r' % gamma)
        self._slowmo_calls = calls
        return gamma

    def _slowmo_launch(self, gamma):
        """NVLink plane: enqueue the SlowMo collective on the current stream (no host sync)"""
        self._kernel.engine.slowmo(self._slowmo_u, self._slowmo_x_prev, gamma, self.slowmo_lr,
                                   self.slowmo_momentum, init=not self._slowmo_initialized)
        self._slowmo_initialized = True

    def _slowmo_c10d(self, gamma):
        """c10d plane: zbar from fp64 all-reduces of sum w z and sum w, the update in fp32 (the
        same operations on identical inputs on every rank)"""
        world = self.dist_config['world_size']
        flat = self.arena.flat
        with torch.no_grad():
            if world > 1:
                dev = self.dist_config['comm_device']
                grp = self._masters_group
                w = float(self._w)
                s = flat.detach().to(dev, torch.float64) * w
                wsum = torch.tensor([w], dtype=torch.float64, device=dev)
                dist.all_reduce(s, group=grp)
                dist.all_reduce(wsum, group=grp)
                zbar = s.div_(wsum).to(flat.device, torch.float32)
            else:
                zbar = flat.detach().clone()
            u, x_prev = self._slowmo_u, self._slowmo_x_prev
            if self._slowmo_initialized:
                u.mul_(self.slowmo_momentum).add_(x_prev.sub(zbar).div_(gamma))
                x_prev.sub_(u, alpha=self.slowmo_lr * gamma)
            else:
                u.zero_()
                x_prev.copy_(zbar)
            flat.copy_(x_prev)
        self._slowmo_initialized = True
        self.ps_weight = 1.0

    # -- consensus: distance and push-sum average model ----------------------- #
    def consensus_distance(self) -> 'ConsensusStats':
        """How far the ranks' models are apart.  With z_i the de-biased parameters of rank i and
        w_i its push-sum weight, zbar = sum_i w_i z_i / sum_i w_i (the point push-sum contracts
        to) and ``distance_sq = (1/n) sum_i |z_i - zbar|^2``; also ``average_norm_sq = |zbar|^2``
        and ``.relative = sqrt(distance_sq / average_norm_sq)``.  ``rank_distance_sq`` is None.
        Identical on every rank.

        Collective: every gossiping rank must call it.  In-flight gossip is drained first (as by
        :meth:`state_dict`).  With a :class:`GossipTrainer` call ``trainer.finish()`` first: under
        Overlap-SGP the trainer holds the last residual.  On the NVLink plane each rank reduces a
        1/n slice of the elements from every rank's snapshot; on the c10d plane it is three
        all-reduces.  Training continued afterwards is unaffected."""
        return self._consensus(None, full=False)[1]

    def average_model(self, out=None) -> torch.Tensor:
        """The push-sum average model zbar as a flat fp32 tensor in the arena's layout
        (``self.arena.views_of(t)`` gives per-parameter views), written into ``out`` if given.
        Same collective semantics as :meth:`consensus_distance`; its statistics, with
        ``rank_distance_sq[i] = |z_i - zbar|^2`` for every rank, are left in
        :attr:`last_consensus`.  BatchNorm buffers are not gossiped and are not averaged."""
        return self._consensus(out, full=True)[0]

    @contextlib.contextmanager
    def averaged(self):
        """Context manager: the parameters (and the bf16 compute copy, if there is one) hold the
        push-sum average model inside the block and are restored bit for bit on exit.  Yields
        the :class:`ConsensusStats` of the average.  Collective (calls :meth:`average_model`);
        buffers such as BatchNorm running statistics stay local."""
        avg = self.average_model()
        flat = self.arena.flat
        shadow = self.compute_shadow
        with torch.no_grad():
            saved = flat.clone()
            saved_shadow = shadow.clone() if shadow is not None else None
            flat.copy_(avg)
            if shadow is not None:
                shadow.copy_(avg)
        del avg
        try:
            yield self.last_consensus
        finally:
            with torch.no_grad():
                flat.copy_(saved)
                if shadow is not None:
                    shadow.copy_(saved_shadow)

    def prepare_consensus(self):
        """Create what the consensus collectives and :meth:`perform_slowmo` need on the NVLink
        plane (they do it on first use; collective).  A process that drives several virtual ranks
        from several threads calls it on every rank before any of them calls
        :meth:`consensus_distance` or :meth:`perform_slowmo`: creating a CUDA
        event or allocating memory can wait for the shared device, where another virtual rank's
        barrier kernel waits for this one (see ``GossipEngine.prepare_consensus``)."""
        if self._kernel is None or self._gossip_done is not None:
            return
        self._kernel.engine.prepare_consensus()
        self._kernel.engine.poll()                  # (allocates its pinned status words)
        self._gossip_done = torch.cuda.Event()
        if self.gossip_stream is not None:
            self._gossip_done.record(self.gossip_stream)     # (creates the event)

    def _consensus(self, out, full):
        what = 'average_model()' if full else 'consensus_distance()'
        if self.nprocs_per_node > 1:
            raise ValueError('%s is not implemented for nprocs_per_node > 1 (hierarchical mode)' % what)
        if list(self._arenas) != [torch.float32]:
            raise ValueError('%s needs fp32 parameters' % what)
        flat = self.arena.flat
        if full:
            if out is None:
                out = torch.empty_like(flat)
            elif out.dtype != torch.float32 or out.numel() != flat.numel() or out.device != flat.device \
                    or not out.is_contiguous():
                raise ValueError('out must be a contiguous fp32 tensor of %d elements on %s'
                                 % (flat.numel(), flat.device))
        # drain exactly like state_dict(): every received message folded, every deferred update
        # applied, parameters de-biased
        if self.asynch:
            self._drain_async()
        self._query_gossip_queue()
        self._flush_pending(drain=True)
        self.unbias()
        world = self.dist_config['world_size']
        if self._kernel is not None:
            e = self._kernel.engine
            self.prepare_consensus()
            if self.gossip_stream is not None:
                self._gossip_done.record(self.gossip_stream)
                torch.cuda.current_stream().wait_event(self._gossip_done)
            res = e.consensus(out, full).cpu()       # (synchronises)
            e.poll(blocking=True)
            vals = [float(v) for v in res]
            ranks = vals[2:2 + world] if full else None
            stats = ConsensusStats(vals[0], vals[1], ranks)
        elif world == 1:
            with torch.no_grad():
                if full:
                    out.copy_(flat)
                nrm = float(flat.double().pow(2).sum())
            stats = ConsensusStats(0.0, nrm, [0.0] if full else None)
        else:
            stats = self._consensus_c10d(out, full, world)
        self.last_consensus = stats
        return out, stats

    def _consensus_c10d(self, out, full, world):
        """c10d plane: sum w z and sum w (all-reduce), then sum |z - zbar|^2 (all-reduce of a
        per-rank vector, so that every rank also learns every rank's term), in fp64."""
        dev = self.dist_config['comm_device']
        grp = self._masters_group
        with torch.no_grad():
            z = self.arena.flat.detach().to(dev, torch.float64)
            w = float(self._w)
            s = z * w
            wsum = torch.tensor([w], dtype=torch.float64, device=dev)
            dist.all_reduce(s, group=grp)
            dist.all_reduce(wsum, group=grp)
            zbar = s.div_(wsum)
            per_rank = torch.zeros(world, dtype=torch.float64, device=dev)
            per_rank[self.dist_config['rank']] = (z - zbar).pow_(2).sum()
            dist.all_reduce(per_rank, group=grp)
            per_rank = [float(v) for v in per_rank.cpu()]
            dsq = 0.0
            for v in per_rank:                  # rank order: the same sum on every rank
                dsq += v
            nrm = float(zbar.pow(2).sum())
            if full:
                out.copy_(zbar.to(out.device, torch.float32))
        return ConsensusStats(dsq / world, nrm, per_rank if full else None)

    def forward(self, *inputs, **kwargs):
        if self.device_ids:
            inputs, kwargs = self.scatter(inputs, kwargs, self.device_ids)
        else:
            inputs, kwargs = (inputs,), (kwargs,)
        if self.nprocs_per_node > 1:
            self._sync_params_multiprocess()
        if len(self.device_ids) == 1 or len(self._module_copies) == 1:
            return self.module(*inputs[0], **kwargs[0])
        # single-process multi-GPU (reference :253-276): master -> replicas, one thread per GPU
        self._sync_params()
        n = min(len(inputs), len(self._module_copies))
        outputs = self.parallel_apply(self._module_copies[:n], inputs[:n], kwargs[:n])
        return self.gather(outputs, self.output_device)

    # ------------------------------------------------------------------ #
    # single-process multi-GPU replicas (reference :87-99, 231-276, 523-549; N10)
    # ------------------------------------------------------------------ #
    def _build_local_replicas(self):
        """One process drives ``device_ids`` (the reference's default launch mode: 8 GPUs per
        process).  Each extra GPU gets a deep copy of the module whose parameters are re-homed
        into ONE flat arena with ONE flat gradient buffer, so that the reference's
        ``broadcast_coalesced`` is a single peer-to-peer DMA copy of the arena per replica and
        its ``reduce_add_coalesced`` is a single kernel on the master GPU that sums the
        replicas' flat gradients with 16-byte P2P loads (``_C.peer_reduce_``).  Gossip runs on
        ``device_ids[0]``'s parameters, exactly as in the reference."""
        import copy
        assert list(self._params_by_dtype.keys()) == [torch.float32] or \
            len(self._params_by_dtype) == 1, 'multi-GPU replicas need single-dtype parameters'
        dtype = next(iter(self._arenas))
        master = self._arenas[dtype]
        params0 = self._params_by_dtype[dtype]
        self._master_grad = master.new_buffer()
        master.bind_grads(params0, self._master_grad)
        self._replica_arenas = [(master, self._master_grad)]
        for dev_idx in self.device_ids[1:]:
            dev = torch.device('cuda', dev_idx)
            rep = copy.deepcopy(self.module).to(dev)
            rparams = [p for p in rep.parameters()]
            arena = FlatArena(rparams, device=dev)
            arena.adopt(rparams)
            gflat = arena.new_buffer()
            arena.bind_grads(rparams, gflat)
            self._module_copies.append(rep)
            self._replica_arenas.append((arena, gflat))
        for m in self._module_copies[1:]:
            m.train(self.module.training)

    def _sync_params(self):
        """master parameters / buffers -> every local replica (reference :256-276)"""
        master, _ = self._replica_arenas[0]
        cur = torch.cuda.current_stream(master.flat.device)
        for (arena, _), rep in zip(self._replica_arenas[1:], self._module_copies[1:]):
            with torch.cuda.device(arena.flat.device):
                s = torch.cuda.current_stream(arena.flat.device)
                s.wait_stream(cur)
                arena.flat.copy_(master.flat, non_blocking=True)        # one P2P DMA copy
                for b_m, b_r in zip(self.module.buffers(), rep.buffers()):
                    b_r.copy_(b_m, non_blocking=True)

    def _master_grad_flat(self):
        """the flat buffer the master's ``p.grad`` views live in, or None if an optimizer
        replaced them (``zero_grad(set_to_none=True)``)"""
        dtype = next(iter(self._arenas))
        opt = self._fused_optimizer
        cand = opt.grad_flat[dtype] if (opt is not None and not self._twin) else self._master_grad
        arena = self._arenas[dtype]
        for p, v in zip(self._params_by_dtype[dtype], arena.views_of(cand)):
            if p.requires_grad:
                return cand if (p.grad is not None and p.grad.data_ptr() == v.data_ptr()) else None
        return None

    def _reduce_local_grads(self):
        """sum of the replicas' flat gradients -> the master's gradient (reference :523-549)"""
        from ..ops import native
        dtype = next(iter(self._arenas))
        arena0 = self._arenas[dtype]
        dev0 = arena0.flat.device
        cur = torch.cuda.current_stream(dev0)
        for _, g in self._replica_arenas[1:]:
            cur.wait_stream(torch.cuda.current_stream(g.device))
        replica_grads = [g for _, g in self._replica_arenas[1:]]
        g0 = self._master_grad_flat()
        fused = native.available() and arena0.flat.is_cuda
        if g0 is not None:
            if fused:
                native.load().peer_reduce_(g0, [g0] + replica_grads, 1.0)     # in place, ONE kernel
            else:
                for g in replica_grads:
                    g0.add_(g.to(dev0))
        else:
            # foreign per-tensor gradients on the master: reduce the replicas into a scratch arena,
            # then one add per tensor
            if getattr(self, '_grad_scratch', None) is None:
                self._grad_scratch = arena0.new_buffer()
            sc = self._grad_scratch
            if fused:
                native.load().peer_reduce_(sc, replica_grads, 1.0)
            else:
                sc.zero_()
                for g in replica_grads:
                    sc.add_(g.to(dev0))
            for p, v in zip(self._params_by_dtype[dtype], arena0.views_of(sc)):
                if not p.requires_grad:
                    continue
                if p.grad is None:
                    p.grad = v.clone()
                else:
                    p.grad.add_(v)
        for _, g in self._replica_arenas[1:]:
            with torch.cuda.device(g.device):
                torch.cuda.current_stream(g.device).wait_stream(cur)
                g.zero_()

    def scatter(self, inputs, kwargs, device_ids):
        from torch.nn.parallel.scatter_gather import scatter_kwargs
        return scatter_kwargs(inputs, kwargs, device_ids, dim=0)

    def parallel_apply(self, replicas, inputs, kwargs):
        from torch.nn.parallel.parallel_apply import parallel_apply
        return parallel_apply(replicas, inputs, kwargs, self.device_ids[:len(replicas)])

    def gather(self, outputs, output_device):
        from torch.nn.parallel.scatter_gather import gather
        return gather(outputs, output_device, dim=0)

    def _make_local_nvls_group(self, by_dtype, on_cuda, device):
        """hierarchical mode (``nprocs_per_node > 1``) on the kernel plane: the local ranks of a
        node share a VMM symmetric world with multicast mappings; None when unavailable (CPU,
        gloo-only hosts, no NVSwitch multicast) -> the c10d collectives of the reference."""
        if not (self.nprocs_per_node > 1 and on_cuda and dist.is_initialized()
                and self.local_node_group is not None and torch.float32 in by_dtype):
            return None
        from .symmetric import VmmSymmetricWorld
        ok = torch.tensor([1 if VmmSymmetricWorld.supported(device) else 0], device=device
                          if dist.get_backend() == 'nccl' else 'cpu')
        dist.all_reduce(ok, op=dist.ReduceOp.MIN, group=self.local_node_group)
        if int(ok.item()) == 0:
            return None
        return _LocalNvlsGroup(self, device)

    def _sync_params_multiprocess(self):
        """Node master -> local ranks (reference :278-296); the parameters are
        one flat arena per dtype so this is one broadcast per dtype -- on the kernel plane a
        ``multimem.st`` broadcast through the switch (``sgp_nvls_bcast_kernel``)."""
        src = self.dist_config['rank'] * self.nprocs_per_node
        for dtype, arena in self._arenas.items():
            if self._hier is not None and dtype == torch.float32:
                self._hier.broadcast_params(arena)
                continue
            dist.broadcast(arena.flat, src=src, group=self.local_node_group)
        buffers = [b.data for b in self.module.buffers()]
        if buffers:
            import functools
            communicate(buffers, functools.partial(dist.broadcast, src=src,
                                                   group=self.local_node_group))

    # -- bias / de-bias ----------------------------------------------------- #
    def ps_numerator(self):
        """Convert the parameters to the push-sum numerator ``x = z * w``."""
        if self.is_ps_numerator:
            return
        if self._kernel is not None and self._fused_optimizer is not None:
            return      # the fused kernels re-bias internally; params stay de-biased
        if not self.lazy_mixing:
            self._scale_params(invert=False)
        self.is_ps_numerator = True

    def unbias(self):
        """Convert the parameters to the de-biased estimate ``z = x / w``."""
        if not self.is_ps_numerator:
            return
        if not self.lazy_mixing:
            self._scale_params(invert=True)
        self.is_ps_numerator = False

    def _scale_params(self, invert):
        if self._kernel is not None:
            e = self._kernel.engine
            e.C.scale_(e.z, e.ps_weight_tensor(), invert, e.shadow)
        else:
            w = self._w
            if w == 1.0:
                return
            for arena in self._arenas.values():
                arena.flat.mul_(1.0 / w if invert else w)

    # -- train / eval -------------------------------------------------------- #
    def train(self, mode=True):
        super(GossipDataParallel, self).train(mode)
        self.gossip_enable = True
        for module in self._module_copies[1:]:
            module.train(mode)
        return self

    def eval(self):
        super(GossipDataParallel, self).eval()
        # drain BEFORE disabling (the reference disables first, which turns its
        # own drain into a no-op; SURVEY 3.4 quirk) so no peer message is lost
        self._query_gossip_queue(non_blocking=self.asynch)
        self._flush_pending(drain=True)
        self.gossip_enable = False
        for module in self._module_copies[1:]:
            module.eval()
        return self

    def block(self):
        self.logger.info('blocking')
        if dist.is_initialized():
            dist.barrier()

    def sync_comms(self):
        if self.asynch:
            self._drain_async()
        self._query_gossip_queue(non_blocking=False)
        self._flush_pending(drain=True)

    def _drain_async(self):
        """Collective drain for bounded-staleness runs, where ranks start different
        numbers of gossip rounds.  (1) Until EVERY rank has left its training loop
        (async barrier) keep serving: finish rounds non-blockingly and start
        gossip-only rounds, so a peer that is still inside a forced wait gets the
        message it needs.  (2) Agree on the furthest round anybody started and
        catch up to it; only then is a blocking drain safe.  The reference relies
        on its 300 s heartbeat in this situation."""
        if not (dist.is_initialized() and self.is_local_master and self.gossip_enable):
            return
        dev = 'cuda' if dist.get_backend() == 'nccl' else 'cpu'
        flag = torch.zeros(1, device=dev)
        grp = self._masters_group       # None (= world) unless nprocs_per_node > 1: only masters gossip
        left_loop = dist.all_reduce(flag, async_op=True, group=grp)
        t0 = time.time()
        while not left_loop.is_completed():
            if self._query_gossip_queue(non_blocking=True) is not False or not self.gossiping:
                self.transfer_params()
            time.sleep(0.0005)
            if time.time() - t0 > self._timeout_s:
                raise NameError('Gossip flag timeout')
        left_loop.wait()
        t = torch.tensor([self._rounds_started], dtype=torch.int64, device=dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=grp)
        target = int(t.item())
        while True:
            self._query_gossip_queue(non_blocking=False)
            if self._rounds_started >= target:
                break
            self.transfer_params()

    # -- gossip state machine ------------------------------------------------ #
    def _query_gossip_queue(self, non_blocking=False):
        """Fold the result of the in-flight gossip into the model.  Returns
        True when something was folded, False otherwise."""
        if not self.gossip_enable:
            return
        if not self.gossiping:
            if self.is_local_master:
                self.logger.debug('not gossiping right now')
            return False

        if self._kernel is not None:
            k = self._kernel
            # heartbeat: one 4-byte async read-back of the kernels' sticky status word per query;
            # raises NameError('Gossip flag timeout') like the reference (:349-352) as soon as a
            # timed-out wait has been observed (non-blocking: sees the previous launches' state)
            k.engine.poll(blocking=not non_blocking and self.overlap)
            if self.overlap and k.gather_event is not None:
                if non_blocking and not k.gather_event.query():
                    return False
                torch.cuda.current_stream().wait_event(k.gather_event)
                k.gather_event = None
                k.residual_pending = True       # folded by the next publish / flush
            # sync mode: the fused kernel already ran on this stream
            self.params_mixed = True
            self.gossiping = False
            return True

        c = self._c10d
        if non_blocking and not c.done():
            return False
        self.ps_numerator()
        t0 = time.time()
        try:
            with tracing.span('gossip.wait+fold'):
                self._w += c.finish(self._timeout_s)
        except RuntimeError as e:
            # "atomic gossip was interrupted so try again" (reference :358-364, 494-504): the
            # round is dropped -- nothing of it was folded -- and re-queued with mix=False: the
            # local share was already scaled when the failed round started, so the retry only
            # re-sends the out-messages.  (A heartbeat timeout is a NameError and is NOT retried.)
            self.logger.warning('received runtime error {}; re-queueing the gossip round'.format(e))
            c.abort()
            self.gossip_retries += 1
            self.params_mixed = True
            self.gossiping = False
            self.transfer_params(mix=False)
            return False
        # host time spent blocked on peers = communication NOT hidden behind compute
        self.exposed_comm_s += time.time() - t0
        tracing.counter('exposed_comm_ms', (time.time() - t0) * 1e3)
        self.params_mixed = True
        self.gossiping = False
        return True

    def transfer_params(self, mix=True):
        """Launch a gossip step with the current parameters."""
        if not self.gossip_enable or not self.is_local_master:
            return False
        if not self.params_mixed:
            self.logger.warning('params not mixed')
            return False

        if self._kernel is not None:
            with tracing.span('gossip.kernel'):
                self._launch_kernel_gossip()
        else:
            self.ps_numerator()
            c = self._c10d
            with tracing.span('gossip.post'):
                self_w = c.start(self._w, pollable=self.asynch, mix=mix)
            if mix:
                if not c.msg_bf16:                      # (bf16: start() subtracted the messages)
                    for arena in self._arenas.values():     # keep the self-loop share
                        arena.flat.mul_(self_w)
                self._w *= self_w
        self.params_mixed = False
        self.gossiping = True
        self._rounds_started += 1
        return True

    def _launch_kernel_gossip(self):
        k = self._kernel
        e = k.engine
        sgd = self._consume_pending_sgd()
        in_numer = self.is_ps_numerator
        if self.overlap:
            e.publish(sgd=sgd, fold=k.residual_pending, in_numerator=in_numer)
            k.residual_pending = False
            cur = torch.cuda.current_stream()
            ev = torch.cuda.Event()
            ev.record(cur)
            self.gossip_stream.wait_event(ev)
            with torch.cuda.stream(self.gossip_stream):
                e.gather()
                k.gather_event = torch.cuda.Event()
                k.gather_event.record(self.gossip_stream)
        else:
            e.mix(sgd=sgd, in_numerator=in_numer)
        self.is_ps_numerator = False

    def _consume_pending_sgd(self):
        k = self._kernel
        if k is not None and k.sgd_pending:
            k.sgd_pending = False
            return True
        return False

    def _flush_pending(self, drain=False):
        """Apply a deferred fused-SGD step and/or fold a gathered residual
        without starting a new gossip (eval / checkpoint / sync_comms).  ``drain=True`` (the
        explicit drain points) also synchronises and raises on a reported heartbeat failure; the
        per-iteration call from the forward pre-hook only does the non-blocking poll."""
        k = self._kernel
        if k is None:
            return
        if k.sgd_pending or k.residual_pending or self.is_ps_numerator:
            k.engine.local(sgd=self._consume_pending_sgd(), fold=k.residual_pending,
                           in_numerator=self.is_ps_numerator)
            k.residual_pending = False
            self.is_ps_numerator = False
        k.engine.poll(blocking=drain)

    # -- hooks ----------------------------------------------------------------- #
    def __register_hooks(self):
        self.register_forward_pre_hook(self.__make_forward_pre_hook())
        self.register_full_backward_pre_hook(self.__make_backward_hook())

    def __make_backward_hook(self):
        def hook(*unused):
            if len(self._module_copies) > 1:
                self._reduce_local_grads()
            if self.nprocs_per_node > 1 and self._hier is not None and self._hier.grads_in_place(self):
                # local-node gradient average: ONE in-switch all-reduce of the flat symmetric
                # gradient buffer (multimem.ld_reduce + multimem.st), scaled by 1/nprocs
                self._hier.allreduce_grads()
            elif self.nprocs_per_node > 1:
                grads = [p.grad.data for p in self.module.parameters()
                         if p.requires_grad and p.grad is not None]
                for g in grads:
                    g.div_(self.nprocs_per_node)
                import functools
                communicate(grads, functools.partial(dist.all_reduce,
                                                     group=self.local_node_group))
            self.ps_numerator()

        def queue_hook(*unused):
            # run once, at the END of this backward pass (reference :567-569)
            Variable._execution_engine.queue_callback(hook)
        return queue_hook

    def __make_forward_pre_hook(self):
        def hook(*unused):
            if self.gossip_enable:
                non_blocking = self.num_updates < self.synch_freq
                if self._query_gossip_queue(non_blocking):
                    self.num_updates = 0
                else:
                    self.num_updates += 1
                if self.overlap:
                    self.transfer_params()
            if self._kernel is not None:
                self._flush_pending()     # deferred SGD must land before forward
            self.unbias()
        return hook


class _LocalNvlsGroup(object):
    """NVLS data plane of one node's local ranks (hierarchical mode, reference :62-80, 278-296,
    551-562): parameter arena + flat gradient in multicast-bound symmetric memory, a signal pad,
    and the two launches -- ``multimem.st`` parameter broadcast from the node master and the
    in-switch gradient all-reduce."""

    def __init__(self, owner, device):
        from ..ops import native
        from .symmetric import VmmSymmetricWorld
        self.C = native.load()
        self.owner = owner
        self.device = device
        self.world = VmmSymmetricWorld(device, owner.local_node_group)
        self.tag = 'hier%d' % owner._instance_id
        self.z_buf = None
        self.g_buf = None
        self.timeout_s = owner._timeout_s

    def arena_allocator(self, numel, dtype, device):
        self.z_buf = self.world.alloc(self.tag + '.z', int(numel) * 4)
        return self.z_buf.local.view(dtype)

    def finish(self, arena):
        C = self.C
        n = arena.total
        self.n = n
        self.g_buf = self.world.alloc(self.tag + '.g', n * 4)
        self.pad = self.world.alloc(self.tag + '.pad', C.PAD_BYTES, multicast=False)
        self.state = torch.zeros(C.STATE_BYTES, dtype=torch.uint8, device=self.device)
        self.hyper = torch.zeros(C.HYPER_FLOATS, dtype=torch.float32, device=self.device)
        self.z_mc = self.z_buf.mc.view(torch.float32)[:n]
        self.g_mc = self.g_buf.mc.view(torch.float32)[:n]
        self.grad_flat = self.g_buf.local.view(torch.float32)[:n]
        self.grad_flat.zero_()
        sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        per_rank = -(-(n // C.CHUNK) // self.world.world)
        self.grid = int(max(1, min(2 * sms, C.nvls_max_grid(self.device.index), per_rank)))
        torch.cuda.synchronize(self.device)
        self.world.barrier()
        return self.grad_flat

    def grads_in_place(self, owner) -> bool:
        """are the module's ``.grad`` tensors still views of the symmetric flat buffer?"""
        arena = owner._arenas[torch.float32]
        for p, v in zip(owner._params_by_dtype[torch.float32], arena.views_of(self.grad_flat)):
            if p.requires_grad:
                return p.grad is not None and p.grad.data_ptr() == v.data_ptr()
        return False

    def broadcast_params(self, arena):
        self.C.nvls_bcast(self.z_mc, arena.flat, self.pad.table, self.state, self.world.rank,
                          self.world.world, 0, self.timeout_s, self.grid)

    def allreduce_grads(self):
        self.C.nvls_allreduce(None, None, self.g_mc, None, self.pad.table, self.state, self.hyper,
                              self.world.rank, self.world.world, self.timeout_s,
                              1.0 / self.world.world, False, self.grid)


def check_gossip_dtype(gossip_dtype, unsupported=None):
    """Validate a ``gossip_dtype`` argument -> ``torch.bfloat16`` or None (fp32 messages).
    ``unsupported``: the configuration bf16 messages would be combined with, if that
    combination is not implemented (the error names it)."""
    if gossip_dtype in (None, torch.float32):
        return None
    if gossip_dtype != torch.bfloat16:
        raise ValueError('gossip_dtype must be None, torch.float32 or torch.bfloat16, got %r'
                         % (gossip_dtype,))
    if unsupported:
        raise ValueError('gossip_dtype=torch.bfloat16 is not supported with %s; bf16 messages '
                         'are implemented for synchronous SGP and D-PSGD' % unsupported)
    return torch.bfloat16


def check_slowmo_args(frequency, lr, momentum):
    """Validate the SlowMo arguments -> (int frequency >= 0, float alpha > 0, float 0 <= beta < 1)."""
    if isinstance(frequency, bool) or not isinstance(frequency, numbers.Integral) or frequency < 0:
        raise ValueError('slowmo_frequency must be an int >= 0 (0 = off), got %r' % (frequency,))
    if not (isinstance(lr, numbers.Real) and math.isfinite(lr) and lr > 0):
        raise ValueError('slowmo_lr must be a finite number > 0, got %r' % (lr,))
    if not (isinstance(momentum, numbers.Real) and 0 <= momentum < 1):
        raise ValueError('slowmo_momentum must be in [0, 1), got %r' % (momentum,))
    return int(frequency), float(lr), float(momentum)


def _native_ok() -> bool:
    from ..ops import native
    return torch.cuda.is_available() and native.available()


def _max_kernel_ranks() -> int:
    from ..ops import native
    return int(native.load().MAX_RANKS) if native.available() else 0


def _single_nvlink_domain(total_ranks: int, local_ok: bool) -> bool:
    """Collective (when torch.distributed is up): True iff every rank wants the kernel transport,
    all ranks run on one host and there are at most MAX_RANKS of them.  Every rank must call it
    with the same arguments' meaning, so that all of them pick the same data plane."""
    if not (dist.is_initialized() and dist.get_world_size() > 1):
        return bool(local_ok)
    import socket
    info = (socket.gethostname(), bool(local_ok))
    gathered = [None] * dist.get_world_size()
    dist.all_gather_object(gathered, info)
    hosts = set(h for h, _ in gathered)
    return all(ok for _, ok in gathered) and len(hosts) == 1 and len(gathered) <= _max_kernel_ranks()


class _GossiperView(object):
    """What ``dist_config['gossipers'][dtype]`` exposes: the knobs of the
    reference's per-dtype gossiper (``peers_per_itr``, ``mixing_weights``,
    ``ps_weight``) routed to whichever data plane is active."""

    def __init__(self, owner: GossipDataParallel, dtype):
        self._owner = owner
        self.dtype = dtype

    @property
    def _graph(self):
        return self._owner.dist_config['graph']

    @property
    def peers_per_itr(self):
        return self._graph.peers_per_itr

    @peers_per_itr.setter
    def peers_per_itr(self, v):
        o = self._owner
        if v == self._graph.peers_per_itr:
            return
        # a schedule change is a global event: finish what is in flight first
        o._query_gossip_queue(non_blocking=False)
        o._flush_pending()
        if o._kernel is not None:
            torch.cuda.synchronize()
            o._kernel.engine.sync_graph()
        if dist.is_initialized():
            dist.barrier()
        self._graph.peers_per_itr = v
        if o._kernel is not None:
            o._kernel.engine.set_schedule(self._graph, o.dist_config['mixing'])
            torch.cuda.synchronize()
            if dist.is_initialized():
                dist.barrier()
        o.gossip_ps_factor.fill_(o.dist_config['mixing'].scalar_weights()[0])

    @property
    def mixing_weights(self):
        return self._owner.dist_config['mixing'].get_mixing_weights()

    @property
    def ps_weight(self):
        return self._owner.ps_weight

    @property
    def regular(self):
        return self._owner.dist_config['mixing'].is_regular()
