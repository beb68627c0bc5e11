"""
BilatGossipDataParallel: asynchronous bilateral gossip (AD-PSGD).

API parity with ``gossip/ad_psgd.py:36-418``: same constructor arguments,
``forward``, ``update_lr``, ``enable_gossip`` / ``disable_gossip``, ``block``
(no-op), ``sync_comms``, ``train`` / ``eval``, ``_pull_model``,
``_transfer_grads``, ``communicator_warmup``.

The reference forks a separate gossip *process* that owns a second
``torch.distributed`` world, a shared-memory (CUDA-IPC / pinned) copy of the
model + gradients and its own ``torch.optim.SGD``, and loops forever
{apply new gradients; bilateral average with the next peer}.  On H100 none of
that needs a process:

* the "gossip copy" is a second flat arena on the same GPU; gradients reach it
  with one flat D2D copy, the model is pulled back with one flat D2D copy;
* the gossip-side optimizer is the fused SGD kernel (``engine.local``);
* the bilateral average is the pull kernel over NVSwitch peer memory, gated by
  a DEVICE-SIDE round state machine: ``sgp_bilat_decide_kernel`` (one CTA) reads
  the partner's publish flags / our ack flags with a bounded (~50 us) wait and
  writes what the following worker launch does -- publish the snapshot, pull
  ``x <- (x + x_partner)/2`` + ack + advance, both, or nothing.  Active ranks
  publish unconditionally, passive ranks only once their partner's snapshot is
  visible (``gossip/gossiper.py:290-316``); no kernel ever spins for long and the
  host never decides a transition;
* the loop that keeps enqueueing {decide, work} pairs is a NATIVE thread
  (``_C.BilatDaemon``, csrc/bindings.cpp): no GIL, no ``stream.synchronize()`` per
  poll -- it throttles itself with a ring of CUDA events and a pinned feedback
  word, on a dedicated lowest-priority stream with a small grid, so training
  kernels keep the SMs;
* the training thread takes the daemon's mutex to enqueue {pull the model, apply
  the new gradients with the fused SGD kernel} on the same stream, which orders
  them against whole gossip rounds exactly like the reference's ``gossip_lock``.

On CPU tensors / gloo the same loop runs over ``BilatPushPull`` (isend/irecv on
a dedicated process group) with plain torch SGD -- the oracle for the kernels.
"""

from __future__ import annotations

import threading
import time

import torch
import torch.distributed as dist
from torch.autograd import Variable
from torch.nn.modules import Module

from ..gossiper import BilatPushPull, C10dTransport
from ..ops import oracle
from ..utils.arena import FlatArena
from ..utils.helpers import make_logger
from ..utils.metering import Meter
from .distributed import consensus_unsupported


class BilatGossipDataParallel(Module):
    """Distributed bilateral-gossip model wrapper (AD-PSGD)."""

    def __init__(self, module, device_ids=None, master_addr=None, master_port=None,
                 backend=None, world_size=None, rank=None, graph_class=None,
                 mixing_class=None, num_peers=1, comm_device=None, lr=0.1, momentum=0.9,
                 weight_decay=1e-4, nesterov=True, verbose=True,
                 network_interface_type=None, tcp_interface_name=None,
                 transport='auto', poll_interval=2e-4, gossip_grid=32,
                 heartbeat_timeout=300.0, max_rounds_per_update=4, daemon_depth=2,
                 partner_wait_us=50.0, symmetric_world=None, gossip_dtype=None):
        super(BilatGossipDataParallel, self).__init__()
        from .distributed import check_gossip_dtype
        # (bf16 bilateral messages would need their own mass-correction term)
        check_gossip_dtype(gossip_dtype, 'BilatGossipDataParallel (AD-PSGD)')
        first = next(module.parameters())
        on_cuda = first.is_cuda
        if device_ids is None:
            device_ids = [first.device.index] if on_cuda else []
        self.device_ids = list(device_ids)
        self.output_device = self.device_ids[0] if self.device_ids else None
        self.module = module
        self._module_copies = [self.module]
        self._replicas = None           # single-process multi-GPU mode (device_ids with > 1 GPU)

        # control plane: reuse the caller's process group, or create the one the
        # reference's gossip process would have created (ad_psgd.py:280-284)
        if not dist.is_initialized() and world_size is not None and world_size > 1 \
                and symmetric_world is None:
            import os
            if master_addr is not None:
                os.environ['MASTER_ADDR'] = str(master_addr)
            if master_port is not None:
                os.environ['MASTER_PORT'] = str(master_port)
            dist.init_process_group(backend=backend or ('nccl' if on_cuda else 'gloo'),
                                    world_size=world_size, rank=rank)
        if rank is None or world_size is None:
            if dist.is_initialized():
                rank, world_size = dist.get_rank(), dist.get_world_size()
            else:
                rank, world_size = 0, 1

        if comm_device is None:
            comm_device = first.device if on_cuda else torch.device('cpu')
        comm_device = torch.device(comm_device)
        self.__cpu_comm = comm_device.type == 'cpu'
        self.dist_config = {
            'verbose': verbose, 'graph_class': graph_class, 'master_addr': master_addr,
            'master_port': master_port, 'backend': backend, 'world_size': world_size,
            'rank': rank, 'mixing_class': mixing_class, 'lr': lr, 'momentum': momentum,
            'nesterov': nesterov, 'weight_decay': weight_decay, 'comm_device': comm_device,
            'network_interface_type': network_interface_type, 'num_peers': num_peers,
        }
        self.num_updates = 0
        self.logger = make_logger(rank, verbose)
        self.gossip_enable = True
        self._poll = float(poll_interval)
        # the reference's gossip process averages as fast as it can, even when no new
        # gradient arrived; on NVLink that is ~18 rounds (1.8 GB of pulls) per training
        # step competing with the model for HBM and SMs.  Bound it (None = unbounded).
        self.max_rounds_per_update = max_rounds_per_update
        self._rounds_since_update = 0
        self._timeout_s = float(heartbeat_timeout)

        # graph / mixing are given as CLASSES (instantiated here, like the
        # reference instantiates them inside its gossip process)
        from ..topology.graph_manager import DynamicBipartiteExponentialGraph
        from ..mixing_manager import UniformMixing
        graph_class = graph_class or DynamicBipartiteExponentialGraph
        mixing_class = mixing_class or UniformMixing
        self.graph = graph_class(rank, world_size, peers_per_itr=num_peers)
        self.mixing = mixing_class(self.graph, comm_device)
        self.dist_config['graph'] = self.graph
        self.dist_config['mixing'] = self.mixing

        # train copy: flat arena (+ flat gradient)
        params = list(module.parameters())
        assert all(p.dtype == first.dtype for p in params), 'single-dtype models only'
        self.arena = FlatArena(params, device=first.device)
        self.arena.adopt(params)
        self.grad_flat = self.arena.new_buffer()
        self.arena.bind_grads(params, self.grad_flat)
        if len(self.device_ids) > 1:
            # the reference's launch mode (one process, several GPUs; gossip/ad_psgd.py:57-69,
            # 148-191, 378-404): flat-arena replicas, P2P DMA parameter sync, one P2P kernel that
            # sums the replicas' gradients into the master's before they go to the gossip side
            from .replicas import LocalReplicas
            self._replicas = LocalReplicas(module, self.device_ids, self.arena, params)
            self._module_copies = self._replicas.copies

        # gossip copy + its gradient / momentum buffers
        self.gossip_flat = self.arena.new_buffer()
        self.gossip_flat.copy_(self.arena.flat)
        self.gossip_params = self.arena.views_of(self.gossip_flat)
        self.gossip_grad_flat = self.arena.new_buffer()
        self.gossip_grads = self.arena.views_of(self.gossip_grad_flat)
        self.momentum_flat = self.arena.new_buffer()

        self.gossip_lock = threading.Lock()
        self.gossip_enable_flag = threading.Event()
        self.train_write_flag = threading.Event()    # train thread wrote new grads
        self.gossip_read_flag = threading.Event()    # gossip thread consumed them
        self.gossip_update_flag = threading.Event()  # learning rate changed
        self._stop = threading.Event()
        self._lr = float(lr)
        self._rounds_completed = 0
        self.grads_applied = 0
        self._error = None

        use_kernels = False
        if transport == 'auto':
            from .distributed import _native_ok, _single_nvlink_domain
            use_kernels = on_cuda and not self.__cpu_comm and first.dtype == torch.float32 \
                and _native_ok()
            # kernels need one NVLink domain (all ranks on one host); else the c10d loop
            use_kernels = _single_nvlink_domain(world_size, use_kernels)
        elif transport in ('nvlink', 'kernel', 'peer'):
            use_kernels = True
        self.transport = 'nvlink' if use_kernels else 'c10d'

        self.engine = None
        self.gossiper = None
        if use_kernels:
            from ..ops.peer_mix import GossipEngine
            from .symmetric import LocalWorld, SymmetricWorld
            if symmetric_world is not None:
                sw = symmetric_world            # e.g. a LocalWorld view: several ranks in one process
            else:
                sw = SymmetricWorld(first.device) if world_size > 1 \
                    else LocalWorld(1, [first.device.index]).view(0)
            self.engine = GossipEngine(sw, self.gossip_flat, self.graph, self.mixing,
                                       grad=self.gossip_grad_flat, momentum=self.momentum_flat,
                                       grid=gossip_grid, timeout_s=self._timeout_s, name='adpsgd')
            self.engine.set_hyper(lr, momentum, weight_decay, nesterov)
            self._hyper = (float(lr), momentum, weight_decay, nesterov)
            # gossip starts disabled (the reference's thread waits for enable_gossip()); a rank
            # may start `max_rounds_per_update` rounds per applied gradient
            self._budget = 0x7FFFFFFF if max_rounds_per_update is None else int(max_rounds_per_update)
            self.engine.ctx.bilat_ctl(self._budget, 0)
            torch.cuda.synchronize(first.device)
            C = self.engine.C
            self.daemon = C.BilatDaemon(self.engine.ctx, self.engine.grid, bool(self.graph.is_passive()),
                                        float(partner_wait_us), int(daemon_depth),
                                        max(20.0, float(poll_interval) * 1e6))
            # the daemon owns the (lowest-priority) gossip stream; torch sees it as an external stream
            self.gossip_stream = torch.cuda.ExternalStream(self.daemon.stream_handle(), device=first.device)
            self._apply_grid = int(min(self.engine.max_grid, C.MAX_CTAS, self.gossip_flat.numel() // C.CHUNK))
            self._grads_pending = False
            self._ev_main = torch.cuda.Event()
            self._ev_pulled = torch.cuda.Event()
            if world_size > 1:
                self.daemon.start()
        else:
            self.gossip_stream = None
            group = rev_group = None
            if dist.is_initialized() and world_size > 1:
                group = dist.new_group(list(range(world_size)))   # gossip-only channel
                import os
                if 'nccl' in str(dist.get_backend(group)).lower() \
                        or os.environ.get('SGP_B200_C10D_SPLIT', '0') == '1':      # (test / debug switch)
                    # this loop sends early and receives once the partner has answered: on NCCL
                    # the two directions of a pair must not share a communicator (a send queued
                    # in front of the receive its partner is waiting for would deadlock the pair;
                    # see gossiper.C10dTransport) -> second group for "higher rank -> lower rank"
                    rev_group = dist.new_group(list(range(world_size)))
            self._gossip_group = group
            if world_size > 1:
                # messages are staged on the communication device (pinned host memory for gloo
                # with a CUDA model, like the reference's comm_device, gossip/ad_psgd.py:351-352)
                self.gossiper = BilatPushPull(self.gossip_flat, graph=self.graph, mixing=self.mixing,
                                              device=comm_device, rank=rank, world_size=world_size,
                                              transport=C10dTransport(group, batched=False,
                                                                      reverse_group=rev_group),
                                              logger=None)

        self.model_meter = Meter(ptag='Model', stateful=True, csv_format=False)
        self.gossip_meter = Meter(ptag='Gossip', stateful=True, csv_format=False)
        self.gossip_read_flag.set()
        self.gossip_thread = None
        if self.engine is None:
            # portable data plane: the loop is a Python thread over isend / irecv
            self.gossip_thread = threading.Thread(target=self._gossip_target, daemon=True,
                                                  name='Gossip-Thread')
            self.gossip_thread.start()
        self.__register_hooks()

    # ------------------------------------------------------------------ #
    # public API
    # ------------------------------------------------------------------ #
    def update_lr(self, lr):
        if self._lr == lr:
            return
        self._lr = float(lr)
        self.gossip_update_flag.set()

    def forward(self, *inputs, **kwargs):
        if self.device_ids:
            from torch.nn.parallel.scatter_gather import scatter_kwargs
            inputs, kwargs = scatter_kwargs(inputs, kwargs, self.device_ids, dim=0)
            if self._replicas is not None and len(inputs) > 1:
                return self._replicas.forward(inputs, kwargs, self.output_device)
            return self.module(*inputs[0], **kwargs[0])
        return self.module(*inputs, **kwargs)

    def train(self, mode=True):
        super(BilatGossipDataParallel, self).train(mode)
        if self._replicas is not None:
            self._replicas.train(mode)
        return self

    def eval(self):
        super(BilatGossipDataParallel, self).eval()
        self._pull_model()
        return self

    def enable_gossip(self):
        self.gossip_enable = True
        self.gossip_enable_flag.set()
        if self.engine is not None:
            with self._locked_gossip_stream():
                self.engine.ctx.bilat_ctl(self._budget, 1)

    def disable_gossip(self):
        self.gossip_enable = False
        self.gossip_enable_flag.clear()
        if self.engine is not None:
            with self._locked_gossip_stream():
                self.engine.ctx.bilat_ctl(-1, 0)       # a round whose snapshot is out still completes

    def block(self):
        return          # the reference's barrier is unreachable too (ad_psgd.py:212-215)

    # the ranks never stop at the same point, so a consensus snapshot is not defined
    consensus_distance = average_model = averaged = consensus_unsupported('BilatGossipDataParallel (AD-PSGD)')

    def sync_comms(self):
        self._pull_model()

    def communicator_warmup(self):
        if dist.is_initialized():
            dist.barrier()
            time.sleep(0.1)
            dist.barrier()

    def shutdown(self):
        self._stop.set()
        self.gossip_enable_flag.set()
        if self.gossip_thread is not None:
            self.gossip_thread.join(timeout=10)
        if self.engine is not None:
            self.daemon.stop()

    @property
    def rounds_completed(self):
        """bilateral averaging rounds this rank has completed"""
        if self.engine is not None:
            return int(self.daemon.rounds_completed())
        return self._rounds_completed

    @rounds_completed.setter
    def rounds_completed(self, v):
        self._rounds_completed = v

    # ------------------------------------------------------------------ #
    # kernel data plane: everything the training thread does to the gossip copy is enqueued on
    # the daemon's stream while holding the daemon's mutex (== the reference's gossip_lock)
    # ------------------------------------------------------------------ #
    def _locked_gossip_stream(self):
        import contextlib

        @contextlib.contextmanager
        def cm():
            self.daemon.lock()                     # (blocks without the GIL)
            try:
                with torch.cuda.stream(self.gossip_stream):
                    yield
            finally:
                self.daemon.unlock()
        return cm()

    def _apply_on_gossip_stream(self, grad_is_train_buffer=False):
        """fused SGD-momentum step of the gossip copy with the pending gradients (+ budget refill)"""
        e = self.engine
        lr = self._lr
        if self._hyper[0] != lr:
            self._hyper = (lr,) + self._hyper[1:]
        e.set_hyper(*self._hyper)
        C = e.C
        e.ctx.step(C.F_PHASE1 | C.F_NO_ROTATE | C.F_SGD | C.F_ZERO_GRAD, self._apply_grid)
        e.ctx.bilat_ctl(self._budget, -1)
        self.grads_applied += 1

    def handoff(self):
        """Fast path of one training iteration (what the backward hook + ``optimizer.step()`` of
        the reference loop amount to): apply this step's gradients to the gossip copy with the
        fused SGD kernel, then pull the result into the training copy -- one enqueue under the
        daemon lock, the training stream waits only for those two local kernels."""
        self._check()
        dev = self.arena.flat.device
        main = torch.cuda.current_stream(dev)
        self.gossip_grad_flat.copy_(self.grad_flat, non_blocking=True)
        self._ev_main.record(main)
        with self._locked_gossip_stream():
            self.gossip_stream.wait_event(self._ev_main)
            self._apply_on_gossip_stream()
            self.arena.flat.copy_(self.gossip_flat, non_blocking=True)
            self._ev_pulled.record(self.gossip_stream)
        main.wait_event(self._ev_pulled)

    # ------------------------------------------------------------------ #
    # train-thread <-> gossip-thread hand-offs
    # ------------------------------------------------------------------ #
    def _check(self):
        if self._error is not None:
            raise RuntimeError('gossip thread died: %r' % (self._error,))
        if self.engine is not None:
            err = self.daemon.error()
            if err:
                raise RuntimeError('gossip daemon died: %s' % err)
            if self.daemon.last_status() != 0:
                raise NameError('Gossip flag timeout (device status %d)' % self.daemon.last_status())

    def _pull_model(self):
        """train copy <- gossip copy (one flat copy under the gossip lock)."""
        self._check()
        if self.engine is not None:
            # pull first, then apply the gradients handed over by _transfer_grads(): the caller's
            # own optimizer.step() applies them to the training copy (reference loop order,
            # gossip_sgd_adpsgd.py:366-370); the training stream waits for the pull only
            dev = self.arena.flat.device
            main = torch.cuda.current_stream(dev)
            self._ev_main.record(main)
            with self._locked_gossip_stream():
                self.gossip_stream.wait_event(self._ev_main)
                self.arena.flat.copy_(self.gossip_flat, non_blocking=True)
                self._ev_pulled.record(self.gossip_stream)
                if self._grads_pending:
                    self._apply_on_gossip_stream()
                    self._grads_pending = False
            main.wait_event(self._ev_pulled)
            return True
        with self.gossip_lock:
            self.arena.flat.copy_(self.gossip_flat, non_blocking=False)
        return True

    def _transfer_grads(self):
        """gossip-side gradient buffer <- this step's gradients."""
        self._check()
        if self.engine is None and not self.gossip_read_flag.wait(timeout=self._timeout_s):
            raise RuntimeError('gossip thread did not consume the previous gradients')
        params = list(self.module.parameters())
        g0 = params[0].grad
        if g0 is not None and g0.data_ptr() == self.grad_flat.data_ptr():
            self.gossip_grad_flat.copy_(self.grad_flat, non_blocking=False)   # one flat copy
        else:
            # an optimizer replaced / dropped the flat views (zero_grad(set_to_none=True)):
            # per-tensor copies, then re-bind the views for the next iteration
            for p, g in zip(params, self.gossip_grads):
                if p.requires_grad and p.grad is not None:
                    g.copy_(p.grad)
                else:
                    g.zero_()
        if self.engine is not None:
            self._grads_pending = True      # applied (stream-ordered) by the next _pull_model()
            return True
        self.gossip_read_flag.clear()
        self.train_write_flag.set()
        return True

    # ------------------------------------------------------------------ #
    # gossip thread
    # ------------------------------------------------------------------ #
    def _gossip_target(self):
        try:
            if self.gossip_flat.is_cuda:         # a new thread starts on device 0
                torch.cuda.set_device(self.gossip_flat.device)
            with torch.no_grad():
                self._loop_c10d()
        except Exception as e:           # surfaced to the train thread
            self._error = e
            self.gossip_read_flag.set()

    def _apply_pending(self, cfg):
        """learning-rate updates and fresh gradients -> gossip-side SGD step"""
        if self.gossip_update_flag.is_set():
            cfg['lr'] = self._lr
            self.gossip_update_flag.clear()
        if self.train_write_flag.is_set():
            bt = time.time()
            with self.gossip_lock:
                x, m = oracle.sgd_momentum(self.gossip_flat, self.gossip_grad_flat,
                                           self.momentum_flat, cfg['lr'], cfg['momentum'],
                                           cfg['weight_decay'], cfg['nesterov'])
                self.gossip_flat.copy_(x)
                self.momentum_flat.copy_(m)
            self.grads_applied += 1
            self._rounds_since_update = 0
            self.train_write_flag.clear()
            self.gossip_read_flag.set()
            self.model_meter.update(time.time() - bt)

    @staticmethod
    def _bilateral_update(x_now, own_snapshot, partner):
        """``x <- 1/2 (own_snapshot + partner) + (x_now - own_snapshot)``, in place.  The reference's
        gossip process cannot apply a gradient between building its message and averaging
        (one loop iteration, ``gossip/ad_psgd.py:332-361``), so it averages exactly what it sent;
        here gradients keep landing while a round is in flight, and whatever was applied since the
        snapshot (``x_now - own_snapshot``) is kept in full instead of being halved."""
        dev = x_now.device
        x_now.add_(partner.to(dev) - own_snapshot.to(dev), alpha=0.5)
        return x_now

    def _throttled(self, round_in_flight):
        """True when this rank has done enough rounds since its last gradient and
        is not in the middle of one (a round in flight is always completed)."""
        k = self.max_rounds_per_update
        return (k is not None) and (not round_in_flight) and (self._rounds_since_update >= k) \
            and self.training

    def _loop_c10d(self):
        """Same protocol over isend/irecv.  "Has my partner published?" is a key in
        the c10d store (the analogue of the probe kernel): a receive is only posted
        once the matching send exists, so no rank ever blocks on -- or exits with --
        a dangling receive, whatever its partner is doing (finished, validating,
        slow).  The reference's active rank blocks inside ``mix`` here
        (``gossip/gossiper.py:290-299``)."""
        cfg = dict(self.dist_config)
        alone = self.gossiper is None
        g = self.gossiper
        tr = g.transport if g is not None else None
        passive = self.graph.is_passive()
        store = None
        if not alone:
            from torch.distributed.distributed_c10d import _get_default_store
            store = _get_default_store()
        rnd = 0
        sent = None
        inflight = []
        wait = self._poll
        t_round = time.time()

        def key(r, src, dst):
            return 'adpsgd/%d/%d>%d' % (r, src, dst)

        def publish():
            with self.gossip_lock:
                snap = self.gossip_flat.to(g.device, copy=True)      # (comm device: see __init__)
            out = g.out_edges[0]
            req = tr.post_sends([snap], [out])[0]
            store.set(key(rnd, out.src, out.dest), '1')
            return (req, snap)

        while not self._stop.is_set():
            if not self.gossip_enable_flag.wait(timeout=0.05):
                continue
            self._apply_pending(cfg)
            if alone or self._throttled(sent is not None):
                time.sleep(self._poll)
                continue
            if sent is None:
                t_round = time.time()
                if not passive:
                    sent = publish()
            in_edge = g.in_edges[0]
            in_key = key(rnd, in_edge.src, in_edge.dest)
            if not store.check([in_key]):
                # back off exponentially (x1.5 up to 20 ms): a quiet partner must not cost the
                # store on rank 0 a constant 5 kHz of polls from every rank
                time.sleep(wait)
                wait = min(wait * 1.5, 0.02)
                continue
            wait = self._poll
            try:
                store.delete_key(in_key)       # consumed: the store does not grow with the run
            except Exception:                  # (a store without delete support keeps the key)
                pass
            if sent is None:          # passive: answer now that the partner showed up
                sent = publish()
            tr.post_recvs([g.in_msg_buffer], [in_edge])[0].wait()
            with self.gossip_lock:
                self._bilateral_update(self.gossip_flat, sent[1], g.in_msg_buffer)
            # never block on OUR send: the partner may have gone quiet before
            # posting its receive.  A send is certainly complete once the partner
            # has answered two later rounds, so only those are reaped.
            inflight.append(sent)
            while len(inflight) > 2:
                inflight.pop(0)[0].wait()
            sent = None
            g.refresh_peers_()
            rnd += 1
            self.rounds_completed += 1
            self._rounds_since_update += 1
            self.gossip_meter.update(time.time() - t_round)

    # ------------------------------------------------------------------ #
    def __register_hooks(self):
        self.register_full_backward_pre_hook(self.__make_backward_hook())

    def __make_backward_hook(self):
        def hook(*unused):
            if self._replicas is not None:          # sum the local replicas' gradients first
                self._replicas.reduce_grads(self.grad_flat)
            self._transfer_grads()
            self._pull_model()

        def queue_hook(*unused):
            Variable._execution_engine.queue_callback(hook)
        return queue_hook


# --------------------------------------------------------------------------- #
# graph-captured AD-PSGD training step
# --------------------------------------------------------------------------- #
class _BilatEngineShim(object):
    """The slice of GossipEngine that GossipTrainer touches, for the bilateral model."""

    def __init__(self, model: BilatGossipDataParallel):
        self.model = model
        self.device = model.arena.flat.device
        self.C = model.engine.C
        self.steps = 0

    def set_hyper(self, lr, momentum, weight_decay, nesterov, do_sgd=True, grad_scale=1.0):
        self.model.update_lr(lr)

    def check(self):
        self.model._check()


def make_bilat_trainer(model: BilatGossipDataParallel, lr, criterion=None, amp_dtype=None,
                       use_cuda_graph=True, warmup_iters=3, channels_last=True, lars=False, batch_mix=None,
                       ema=None):
    """AD-PSGD counterpart of :class:`~.trainer.GossipTrainer`: forward + fused loss/accuracy +
    backward are captured ONCE as a CUDA graph; after every replay the gradients are handed to
    the gossip side with :meth:`BilatGossipDataParallel.handoff` (fused SGD on the gossip copy +
    model pull, enqueued on the daemon's stream under its lock).  The bilateral averaging itself
    runs asynchronously on the native daemon's low-priority stream the whole time.  ``batch_mix``:
    mixup / CutMix as in ``GossipTrainer``.  ``ema`` must be None: a weight EMA is not supported,
    the gossip daemon rewrites the parameters concurrently on its own stream."""
    if ema is not None:
        raise ValueError('ModelEma is not supported with AD-PSGD: its gossip daemon rewrites the parameters '
                         'concurrently on another stream, so no launch sees a settled model')
    if lars:
        raise ValueError('LARS is not supported with AD-PSGD: its SGD runs on the gossip daemon\'s '
                         'copy, outside FusedGossipSGD')
    from .trainer import GossipTrainer

    class BilatTrainer(GossipTrainer):

        def __init__(self):
            assert model.engine is not None, 'BilatTrainer drives the nvlink kernel transport'
            self.model = model

            class _Opt(object):
                param_groups = [dict(lr=lr, momentum=model.dist_config['momentum'],
                                     weight_decay=model.dist_config['weight_decay'],
                                     nesterov=model.dist_config['nesterov'])]
                grad_scale = 1.0
            self.opt = _Opt()
            self.engine = _BilatEngineShim(model)
            self.k = None
            self.overlap = False
            self.gossip = False
            self._init_runtime(self.engine.device, criterion, amp_dtype, use_cuda_graph, warmup_iters,
                               channels_last, batch_mix)

        def _one_step(self, first=False):
            self._fwd_bwd()                      # the captured part

        def _run_on_stream(self):
            c0 = self.engine.C.launch_count()
            super(BilatTrainer, self)._run_on_stream()
            self.model.handoff()                 # eager: apply gradients + pull, under the daemon lock
            if self.graph is None or self.own_launches_per_step is None:
                self.own_launches_per_step = self.engine.C.launch_count() - c0
            else:
                self.own_launches_per_step = max(self.own_launches_per_step, 0)

        def _after_replay(self):
            pass

        def finish(self):
            torch.cuda.synchronize(self.device)
            self.model._check()

        def evaluate(self, batches):
            raise ValueError('evaluate() is not supported with AD-PSGD: its gossip daemon rewrites the '
                             'parameters asynchronously, so a captured evaluation would not see one model')

        def update_bn(self, batches):
            raise ValueError('update_bn() is not supported with AD-PSGD: its gossip daemon rewrites the '
                             'parameters asynchronously, so the statistics would not be those of one model')

        def check(self):
            self.model._check()

    return BilatTrainer()
