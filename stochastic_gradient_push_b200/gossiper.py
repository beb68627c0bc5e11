"""
Gossipers: one consensus-averaging step over the current graph window.

API parity with ``gossip/gossiper.py`` -- ``Gossiper`` (:31-173), ``PushSum``
(:176-219), ``PushPull`` (:222-275), ``BilatPushPull`` (:278-323): same
constructor, ``mix()`` signatures/returns, ``ps_weight`` / ``peers_per_itr``
properties, ``refresh_peers_``, ``refresh_mixing_weights_``, ``mix_out_msg_``,
``clean_msg_buffers_``, ``parse_in_msg_buffer`` and the public attributes
(``in_msg_buffer``, ``placeholder``, ``out_msg_buffer``, ``out_edges``,
``in_edges``, ``mixing_weights``, ``passive``, ``regular``, ``device``).

What is different underneath:

* The reference emulates point-to-point with ``dist.broadcast`` inside one
  2-rank process group per edge.  Here a gossiper owns a *transport*:

  - ``PeerMemoryTransport`` (CUDA, engine in ``ops/peer_mix.py``): the message lives in
    NVSwitch-mapped symmetric memory and ``mix`` is ONE sm_90a kernel that
    publishes the message, waits on the in-neighbours' sequence flags and
    accumulates their buffers with weighted 16-byte P2P loads.  No NCCL.
  - ``C10dTransport`` (any backend, CPU/gloo capable): true ``isend/irecv``
    on the world group.  It is the portable fallback and the numerical oracle
    for the kernels.

* Because receives are posted before sends and nothing blocks on a peer's
  *matching call order*, PushPull cannot deadlock on non-bipartite graphs
  (the reference deadlocks on gloo for e.g. a ring, SURVEY C12); the
  active/passive distinction is kept as an attribute for API parity only.
"""

from __future__ import annotations

import torch
import torch.distributed as dist

from .topology.graph_manager import GraphManager
from .mixing_manager import MixingManager, UniformMixing


# --------------------------------------------------------------------------- #
# bf16 message wire format (GossipDataParallel(gossip_dtype=torch.bfloat16), c10d plane)
# --------------------------------------------------------------------------- #
def bf16_message_numel(n: int) -> int:
    """bf16 elements of one message carrying ``n`` values: the payload, padded to an even
    length, then two slots holding the bit pattern of the fp32 push-sum weight (which must not
    be rounded)."""
    return n + (n & 1) + 2


def pack_bf16_message(msg: torch.Tensor, x: torch.Tensor, scale: float, weight: float) -> torch.Tensor:
    """Write Q(scale * x) and the fp32 ``weight`` into the bf16 buffer ``msg``.  Returns
    Q(scale * x) on ``x``'s device, which the sender subtracts from its own numerator: it loses
    exactly what the receiver gets, so push-sum mass is conserved."""
    n = x.numel()
    q = (x * scale).to(torch.bfloat16)
    msg[:n].copy_(q, non_blocking=True)
    msg[n:].zero_()
    msg[n + (n & 1):].view(torch.float32).fill_(weight)
    return q


def bf16_message_weight(msg: torch.Tensor, n: int) -> float:
    return float(msg[n + (n & 1):].view(torch.float32)[0])


# --------------------------------------------------------------------------- #
# transports
# --------------------------------------------------------------------------- #
class C10dTransport(object):
    """isend/irecv on a c10d group.  Tags disambiguate repeated edges between
    the same pair inside one step (phone books may contain duplicates).

    NCCL (GPU tensors between hosts) needs two things gloo does not:

    * a rank's receives and sends of ONE exchange must be launched as ONE group
      (``batch_isend_irecv``): NCCL runs the point-to-point operations of a pair of ranks on
      one stream in launch order, so "irecv then isend" on both sides of a symmetric exchange
      (a ring of 2, the ``n/2`` hop of the exponential graphs, every bipartite pairing) would
      leave both receive kernels waiting for sends that are queued behind them.
      ``exchange()`` does that when ``batched`` (default: the group's backend is NCCL);
    * sends and receives that are NOT issued together (the AD-PSGD loop sends early and
      receives when the partner has answered) must not share a communicator per direction:
      with ``reverse_group`` set, messages from a higher to a lower rank travel on that
      second group, so the two directions of a pair never queue behind each other.

    NCCL ignores tags; repeated edges are matched in posting order, which is the same
    (``k``-th send <-> ``k``-th receive) on both sides."""

    name = 'c10d'

    def __init__(self, group=None, batched=None, reverse_group=None):
        self.group = group
        self.reverse_group = reverse_group
        self._batched = batched

    @property
    def batched(self) -> bool:
        if self._batched is None:
            try:
                # ('nccl', or a per-device map such as 'cpu:gloo,cuda:nccl'; grouping is harmless on gloo)
                self._batched = bool(dist.is_initialized()) and \
                    'nccl' in str(dist.get_backend(self.group)).lower()
            except Exception:
                self._batched = False
        return self._batched

    def _group_for(self, src, dst):
        if self.reverse_group is not None and src > dst:
            return self.reverse_group
        return self.group

    def post_recvs(self, buffers, in_edges):
        reqs, seen = [], {}
        for buf, edge in zip(buffers, in_edges):
            k = seen.get(edge.src, 0)
            seen[edge.src] = k + 1
            reqs.append(dist.irecv(buf, src=edge.src, group=self._group_for(edge.src, edge.dest), tag=k))
        return reqs

    def post_sends(self, msgs, out_edges):
        reqs, seen = [], {}
        for msg, edge in zip(msgs, out_edges):
            k = seen.get(edge.dest, 0)
            seen[edge.dest] = k + 1
            reqs.append(dist.isend(msg, dst=edge.dest, group=self._group_for(edge.src, edge.dest), tag=k))
        return reqs

    def exchange(self, recv_bufs, in_edges, send_msgs, out_edges):
        """Post the receives and the sends of one step -> ``(recv_reqs, send_reqs)``.  Every
        request of ``recv_reqs`` must be waited for before ANY receive buffer is read (a batched
        launch returns requests that cover the whole group, not one per buffer)."""
        if not self.batched:
            return self.post_recvs(recv_bufs, in_edges), self.post_sends(send_msgs, out_edges)
        # (a grouped launch takes ONE process group; the direction split is pointless inside it)
        ops, seen = [], {}
        for buf, edge in zip(recv_bufs, in_edges):
            k = seen.get(edge.src, 0)
            seen[edge.src] = k + 1
            ops.append(dist.P2POp(dist.irecv, buf, edge.src, self.group, tag=k))
        seen = {}
        for msg, edge in zip(send_msgs, out_edges):
            k = seen.get(edge.dest, 0)
            seen[edge.dest] = k + 1
            ops.append(dist.P2POp(dist.isend, msg, edge.dest, self.group, tag=k))
        if not ops:
            return [], []
        return list(dist.batch_isend_irecv(ops)), []

    def post_polled_recv(self, buf, in_edge):
        """A receive whose completion can be polled without blocking.  gloo's
        ``Work.is_completed()`` never flips until ``wait()`` is called, so a
        helper thread parks in ``wait()`` and raises an event instead.  (NCCL works can be
        polled directly; parking a thread in their stream-level ``wait()`` would return at once.)"""
        req = self.post_recvs([buf], [in_edge])[0]
        return req if self.batched else _PolledRecv(req)


class _PolledRecv(object):

    def __init__(self, req):
        import threading
        self._req = req
        self._done = threading.Event()
        self._err = None
        self._thread = threading.Thread(target=self._park, daemon=True,
                                        name='Gossip-Recv-Poll')
        self._thread.start()

    def _park(self):
        try:
            self._req.wait()
        except Exception as e:       # surfaced to the caller in wait()
            self._err = e
        self._done.set()

    def is_completed(self):
        return self._done.is_set()

    def wait(self):
        self._done.wait()
        if self._err is not None:
            raise self._err

    def wait_for(self, seconds: float) -> bool:
        """Bounded wait: False when the message has not arrived within ``seconds``."""
        if not self._done.wait(seconds):
            return False
        if self._err is not None:
            raise self._err
        return True


class PeerMemoryTransport(object):
    """sm_90a data plane for STAND-ALONE gossipers (``README.md:67-68`` of the
    reference uses ``PushSum``/``PushPull`` directly on a tensor): the message is
    staged into a chunk-padded buffer whose outbox lives in NVSwitch peer-mapped
    memory and ``mix`` becomes kernel launches of :class:`~.ops.peer_mix.GossipEngine`
    -- ``residual=False`` -> the fused publish+pull+mix kernel, ``residual=True`` ->
    publish + gather (sum of the in-neighbours' weighted messages).  Collective
    construction (every rank of the world builds its gossiper)."""

    name = 'nvlink'

    def __init__(self, world=None, timeout_s=60.0, grid=None):
        self.world = world
        self.timeout_s = timeout_s
        self.grid = grid
        self.engine = None

    def bind(self, gossiper, msg):
        from .ops.peer_mix import GossipEngine, build_tables
        from .ops import native
        C = native.load()
        assert msg.is_cuda and msg.dtype == torch.float32, 'nvlink transport: fp32 CUDA messages'
        n = msg.numel()
        self.n = n
        padded = (n + C.CHUNK - 1) // C.CHUNK * C.CHUNK
        self.z = torch.zeros(padded, dtype=torch.float32, device=msg.device)
        world = self.world
        if world is None:
            from .parallel.symmetric import LocalWorld, SymmetricWorld
            if gossiper.world_size > 1:
                world = SymmetricWorld(msg.device)
            else:
                world = LocalWorld(1, [msg.device.index]).view(0)
        graph, mixing = gossiper._graph_manager, gossiper._mixing_manager
        self.engine = GossipEngine(world, self.z, graph, mixing, with_residual=True,
                                   timeout_s=self.timeout_s, grid=self.grid, name='gossiper')
        # residual=True exchanges are summed with unit edge weights (the caller
        # already scaled by lo; reference 'uniform' weight == 1, mixing_manager.py:47)
        table, wtable = build_tables(graph, mixing, msg.device)
        unit = wtable.clone()
        unit[:, 1:] = (wtable[:, 1:] != 0).float()
        self._tables = (table, wtable)
        self._unit_tables = (table, unit)

    def mix(self, gossiper, out_msg, ps_weight, residual):
        e = self.engine
        w = float(ps_weight.reshape(-1)[0]) if torch.is_tensor(ps_weight) else float(ps_weight)
        self.z[:self.n].copy_(out_msg.reshape(-1))
        e.ps_weight = w
        if residual:
            e.ctx.set_schedule(*self._unit_tables)
            e.publish(sgd=False, fold=False, in_numerator=True)
            e.gather()
            msg = e.residual[:self.n]
            psw = torch.full((1,), e.res_weight, dtype=out_msg.dtype, device=out_msg.device)
            e.ps_weight = w                          # publish keeps only the self-loop share
        else:
            e.ctx.set_schedule(*self._tables)
            e.mix(sgd=False, in_numerator=True)      # z <- xn / wn
            wn = e.ps_weight
            msg = self.z[:self.n] * wn               # numerator, like the c10d path
            psw = torch.full((1,), wn, dtype=out_msg.dtype, device=out_msg.device)
        e.check()
        e.sync_graph()
        gossiper.refresh_peers_(rotate=False)
        return msg, psw


# --------------------------------------------------------------------------- #
# base class
# --------------------------------------------------------------------------- #
class Gossiper(object):
    """Generic multi-peer gossip averaging object."""

    def __init__(self, msg, graph, device=None, mixing=None, logger=None,
                 rank=None, world_size=None, transport=None):
        self.logger = logger
        if rank is None or world_size is None:
            assert dist.is_initialized(), \
                'pass rank/world_size or initialise torch.distributed'
            rank, world_size = dist.get_rank(), dist.get_world_size()
        self.rank = rank
        self.world_size = world_size
        assert isinstance(graph, GraphManager)
        self._graph_manager = graph
        self.device = torch.device(device) if device is not None else msg.device
        self.passive = self._graph_manager.is_passive()
        self.refresh_peers_(rotate=False)

        if mixing is None:
            mixing = UniformMixing(self._graph_manager, self.device)
        assert isinstance(mixing, MixingManager)
        self._mixing_manager = mixing
        self.refresh_mixing_weights_()
        self.regular = self._mixing_manager.is_regular()

        self.out_msg_buffer = []
        self._ps_weight = torch.ones(1, dtype=msg.dtype, device=self.device)
        numel = msg.numel() + (0 if self.regular else 1)
        self.in_msg_buffer = torch.zeros(numel, dtype=msg.dtype, device=self.device)
        self.in_msg_buffer[:msg.numel()].copy_(msg.detach().reshape(-1))
        if not self.regular:
            self.in_msg_buffer[-1] = 1.0
        if self.device.type == 'cpu' and torch.cuda.is_available():
            try:
                self.in_msg_buffer = self.in_msg_buffer.pin_memory()
            except Exception as e:          # pragma: no cover
                if self.logger is not None:
                    self.logger.error(e)
        self.placeholder = self.in_msg_buffer.clone()
        self._extra_placeholders = []
        self._pending_req = None
        if transport == 'nvlink':
            transport = PeerMemoryTransport()
        self.transport = transport if transport is not None else C10dTransport()
        if isinstance(self.transport, PeerMemoryTransport):
            self.transport.bind(self, msg)

    # -- properties --------------------------------------------------------- #
    @property
    def ps_weight(self):
        return self._ps_weight

    @ps_weight.setter
    def ps_weight(self, v):
        if torch.is_tensor(v):
            self._ps_weight.copy_(v.reshape(-1)[:1])
        else:
            self._ps_weight.fill_(float(v))

    @property
    def peers_per_itr(self):
        return self._graph_manager.peers_per_itr

    @peers_per_itr.setter
    def peers_per_itr(self, v):
        self._graph_manager.peers_per_itr = v
        # the reference leaves a stale `peers_per_itr_device` and stale edges
        # behind here (SURVEY C10 quirk); we refresh so the new window is live
        self.refresh_peers_(rotate=False)

    @property
    def peers_per_itr_device(self):
        return torch.tensor([self._graph_manager.peers_per_itr],
                            device=self.device, dtype=self._ps_weight.dtype)

    # -- graph / weights ---------------------------------------------------- #
    def refresh_peers_(self, rotate=None):
        if rotate is None:
            rotate = self._graph_manager.is_dynamic_graph()
        assert not (rotate and not self._graph_manager.is_dynamic_graph())
        self.out_edges, self.in_edges = self._graph_manager.get_edges(rotate)

    def refresh_mixing_weights_(self, residual_adjusted=False):
        self.mixing_weights = self._mixing_manager.get_mixing_weights(
            residual_adjusted)

    def _weight(self, key, dtype):
        return self.mixing_weights[key].to(device=self.device, dtype=dtype)

    def mix_out_msg_(self, out_msg, ps_weight, residual=False):
        """Generator of outgoing messages: optional loop-back first, then one
        message per out-edge.  Uniform mixing scales ``out_msg`` IN PLACE and
        yields the same tensor for every edge (reference semantics,
        ``gossip/gossiper.py:139-143``)."""
        self.refresh_mixing_weights_(residual)
        self.ps_weight = ps_weight
        if not self.regular:
            out_msg = torch.cat([out_msg.reshape(-1),
                                 self.ps_weight.to(out_msg.dtype)])
        if not residual:
            yield out_msg.mul(self._weight('lo', out_msg.dtype))
        if self._mixing_manager.is_uniform():
            out_msg *= self._weight('uniform', out_msg.dtype)
            for _ in self.out_edges:
                yield out_msg
        else:
            for edge in self.out_edges:
                yield out_msg.mul(self._weight(edge.dest, out_msg.dtype))

    def clean_msg_buffers_(self):
        """Wait for every in-flight send, then drop the references."""
        while self.out_msg_buffer:
            req, _ = self.out_msg_buffer.pop()
            req.wait()

    def parse_in_msg_buffer(self, residual=False):
        msg = self.in_msg_buffer
        if not self.regular:
            return msg.narrow(0, 0, len(msg) - 1), msg[-1]
        if residual:
            return msg, self.ps_weight * self.peers_per_itr_device
        return msg, torch.ones(1, device=self.device, dtype=msg.dtype)

    # -- shared exchange ---------------------------------------------------- #
    def _recv_buffers(self, k):
        while len(self._extra_placeholders) < k - 1:
            self._extra_placeholders.append(torch.empty_like(self.placeholder))
        return ([self.placeholder] + self._extra_placeholders)[:k]

    def _exchange(self, out_msg, ps_weight, residual):
        """post irecvs -> post isends -> wait -> accumulate."""
        assert out_msg.device.type == self.device.type
        msgs = self.mix_out_msg_(out_msg, ps_weight, residual)
        loopback = None if residual else next(msgs)

        remote_in = [e for e in self.in_edges if e.src != e.dest]
        bufs = self._recv_buffers(len(remote_in))
        batched = getattr(self.transport, 'batched', False)
        if not batched:                    # receives first: the peers' messages can land while
            recv_reqs = self.transport.post_recvs(bufs, remote_in)      # ours are being built

        self_msgs, send_edges, send_msgs = [], [], []
        for edge in self.out_edges:
            m = next(msgs)
            if edge.dest == edge.src:      # self-edge (e.g. n=2, ppi=2)
                self_msgs.append(m)
            else:
                send_edges.append(edge)
                send_msgs.append(m)
        if batched:                        # NCCL: one grouped launch of all receives and sends
            # (its requests cover the sends too and are waited for exactly once, below -- a second
            # wait() on a completed gloo request never returns; `send_msgs` stays alive until then)
            recv_reqs, send_reqs = self.transport.exchange(bufs, remote_in, send_msgs, send_edges)
        else:
            send_reqs = self.transport.post_sends(send_msgs, send_edges)
        for req, m in zip(send_reqs, send_msgs):
            self.out_msg_buffer.append((req, m))

        if loopback is not None:
            self.in_msg_buffer.copy_(loopback)
        else:
            self.in_msg_buffer.zero_()
        for m in self_msgs:
            self.in_msg_buffer.add_(m)
        for req in recv_reqs:              # all of them before any buffer is read (see exchange())
            req.wait()
        for buf in bufs:
            self.in_msg_buffer.add_(buf)

        self.refresh_peers_()
        self.clean_msg_buffers_()
        return self.parse_in_msg_buffer(residual)

    def mix(self, *args, **kwargs):
        raise NotImplementedError


class PushSum(Gossiper):
    """Column-stochastic push (SGP).  ``mix(out_msg, ps_weight, residual)``
    returns ``(in_msg, in_ps_weight)``; with ``residual=True`` the result is
    the sum of what the in-neighbours pushed (the caller folds it into its own
    pre-scaled copy), otherwise it already contains the ``lo``-weighted
    loop-back."""

    def mix(self, out_msg, ps_weight, residual=False):
        if self.logger is not None:
            self.logger.debug('in/out -peers {}/{}'.format(
                self.in_edges, self.out_edges))
        if isinstance(self.transport, PeerMemoryTransport):
            return self.transport.mix(self, out_msg, ps_weight, residual)
        return self._exchange(out_msg, ps_weight, residual)


class PushPull(Gossiper):
    """Doubly-stochastic symmetric exchange (D-PSGD)."""

    def mix(self, out_msg, ps_weight, residual=False):
        if self.logger is not None:
            self.logger.debug('in/out -peers {}/{}'.format(
                self.in_edges, self.out_edges))
        if isinstance(self.transport, PeerMemoryTransport):
            return self.transport.mix(self, out_msg, ps_weight, residual)
        return self._exchange(out_msg, ps_weight, residual)


class BilatPushPull(Gossiper):
    """Bilateral exchange for AD-PSGD: active ranks send then receive; passive
    ranks keep one receive posted, poll it, and answer only once the partner's
    message has landed.  Returns ``(in_msg, ps_weight)`` on completion and
    ``(out_msg, False)`` when a passive rank has nothing yet (callers test the
    truthiness of the second element, ``gossip/ad_psgd.py:354-356``)."""

    def mix(self, out_msg):
        assert out_msg.device.type == self.device.type
        assert len(self.in_edges) == 1 and len(self.out_edges) == 1
        out_edge, in_edge = self.out_edges[0], self.in_edges[0]

        if not self.passive:
            msg = next(self.mix_out_msg_(out_msg, 1., residual=True))
            recv, send = self.transport.exchange([self.in_msg_buffer], [in_edge], [msg], [out_edge])
            for req in send + recv:
                req.wait()
            completed = True
        else:
            if self._pending_req is None:
                self._pending_req = self.transport.post_polled_recv(
                    self.in_msg_buffer, in_edge)
            if self._pending_req.is_completed():
                self._pending_req.wait()
                msg = next(self.mix_out_msg_(out_msg, 1., residual=True))
                self.transport.post_sends([msg], [out_edge])[0].wait()
                self._pending_req = None
                completed = True
            else:
                completed = False

        if completed:
            self.refresh_peers_()
            self.clean_msg_buffers_()
            return self.parse_in_msg_buffer(residual=True)
        return out_msg, completed
