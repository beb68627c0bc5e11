"""
GossipEngine: drives the sm_90a gossip kernels for ONE rank.

It owns the peer-visible signal pad + double-buffered outbox (symmetric
memory), the device-side schedule tables emitted from a ``GraphManager`` /
``MixingManager`` pair, the device-resident hyper-parameters and kernel state,
and exposes the four launches the algorithms are built from:

    mix(sgd)            SGP / D-PSGD step: [SGD] + publish + pull + mix + de-bias
    publish(sgd, fold)  Overlap-SGP, main stream: [SGD] + fold residual + publish
    gather()            Overlap-SGP, side stream: residual = sum of P2P loads
    local(sgd, fold)    no communication: [SGD] / fold only (flush, world==1)

``msg_dtype=torch.bfloat16`` sends bf16 messages (half the bytes per in-neighbour) with exact
push-sum mass conservation: the outbox holds Q(x) = bf16(x), the sender keeps
x - (1 - self_w) Q(x), and the receivers add in_w * Q(x_j).  Only :meth:`mix` (SGP / D-PSGD)
supports it.

All launches go to the *current* CUDA stream and are CUDA-graph capturable:
nothing that changes per step (phase, parity, lr, push-sum weight) is a kernel
argument -- it all lives in device memory.
"""

from __future__ import annotations

from typing import Optional

import torch

from . import native


def build_tables(graph, mixing, device):
    """(table int32 [period, TABLE_ROW], wtable fp32 [period, WTABLE_ROW]).

    ``wtable[t] = [self_w, in_w_0..]`` where ``in_w_k`` is the weight the k-th
    in-neighbour assigns to its edge towards this rank at phase t, i.e. the
    receiver evaluates the sender's column of the mixing matrix (the senders
    never scale a message; reference K6 disappears)."""
    from ..topology.graph_manager import MAX_PEERS_PER_ITR as MP
    table = graph.device_table(device=None)
    period = table.shape[0]
    sched = graph._schedule
    k = graph.nprocs_per_node
    rows = []
    phases_self = graph.phases()
    per_rank_phases = {}
    for t in range(period):
        outs, ins = phases_self[t]
        self_w, _ = mixing.scalar_weights([p * k for p in outs], rank=graph.rank)
        row = [float(self_w)]
        for j in ins:
            if j not in per_rank_phases:
                ph = sched.phases(rank=j)
                per_rank_phases[j] = ph if graph.is_dynamic_graph() else ph[:1]
            outs_j = per_rank_phases[j][t][0]
            _, edge_w = mixing.scalar_weights([p * k for p in outs_j], rank=j)
            row.append(float(edge_w[graph.rank * k]))
        row += [0.0] * (1 + MP - len(row))
        rows.append(row)
    wtable = torch.tensor(rows, dtype=torch.float32)
    return table.to(device), wtable.to(device)


class GossipEngine(object):

    def __init__(self, world, params_flat: torch.Tensor, graph, mixing, *,
                 grad: Optional[torch.Tensor] = None,
                 momentum: Optional[torch.Tensor] = None,
                 shadow: Optional[torch.Tensor] = None,
                 with_residual: bool = False,
                 grid: Optional[int] = None, gather_grid: Optional[int] = None,
                 timeout_s: float = 30.0, name: str = 'sgp', segments: int = 4,
                 gather_tma: bool = True, soft_timeout_s: Optional[float] = None,
                 gather_dma: Optional[bool] = None, msg_dtype: Optional[torch.dtype] = None):
        C = native.load()
        if msg_dtype not in (None, torch.float32, torch.bfloat16):
            raise ValueError('gossip message dtype must be torch.float32 or torch.bfloat16, got %s'
                             % (msg_dtype,))
        self.msg_bf16 = msg_dtype == torch.bfloat16
        self.C = C
        self.world = world
        self.rank = world.rank
        self.nranks = world.world
        self.device = params_flat.device
        self.n = params_flat.numel()
        assert params_flat.dtype == torch.float32 and self.n % C.CHUNK == 0
        self.z = params_flat
        self.grad = grad
        self.momentum = momentum
        self.shadow = shadow
        self.residual = (torch.zeros(self.n, dtype=torch.float32, device=self.device)
                         if with_residual else None)
        self.graph = graph
        self.mixing = mixing
        assert graph.world_size == self.nranks, \
            'graph spans %d ranks, symmetric world has %d' % (graph.world_size, self.nranks)

        # symmetric allocations (collective across the world)
        self._name = name
        self.pad = world.alloc(name + '.pad', C.PAD_BYTES)
        elem = 2 if self.msg_bf16 else 4
        self.outbox = world.alloc(name + '.outbox', 2 * self.n * elem)

        # local kernel state / hyper-parameters
        self.state = torch.zeros(C.STATE_BYTES, dtype=torch.uint8, device=self.device)
        self._state_f32 = self.state.view(torch.float32)
        self._state_i32 = self.state.view(torch.int32)
        self._state_f32[C.STATE_OFF_PSW // 4: C.STATE_OFF_PSW // 4 + 2] = 1.0
        # soft heartbeat (default: a tenth of the hard one): waits that exceed it are counted and
        # reported by poll() as "delayed, still waiting" -- see SgpState::soft_timeouts
        soft = timeout_s / 10.0 if soft_timeout_s is None else soft_timeout_s
        self._state_i32[C.STATE_OFF_SOFT_TIMEOUT_US // 4] = int(min(max(soft, 0.0) * 1e6, 2 ** 31 - 1))
        self._soft_seen = 0
        self._state_f32[C.STATE_OFF_RES_SCALE // 4] = 1.0
        self._phase_base = 0            # host mirror of SgpState::phase_base
        self._gather_dma_pref = gather_dma
        # row 0: the hyper-parameters every SGD launch reads; rows 1..G: per-parameter-group rows
        # (set_param_groups), all in one buffer so that one H2D copy updates them together
        self._hyper_rows = torch.zeros(1 + C.MAX_GROUPS, C.HYPER_FLOATS, dtype=torch.float32,
                                       device=self.device)
        self.hyper = self._hyper_rows[0]
        self.groups = 0
        # ring of pinned staging slots: an lr change must not rewrite host memory that an earlier,
        # still-queued async H2D copy is going to read
        self._hyper_host = torch.zeros(8, 1 + C.MAX_GROUPS, C.HYPER_FLOATS, dtype=torch.float32).pin_memory()
        self._hyper_slot = 0
        self._hyper_events = [None] * 8
        self._hyper_cache = None
        self._status_host = None

        table, wtable = build_tables(graph, mixing, self.device)
        self.ctx = C.GossipContext(
            z=self.z, g=grad, m=momentum, shadow=shadow, residual=self.residual,
            pad_ptrs=self.pad.table, outbox_ptrs=self.outbox.table,
            table=table, wtable=wtable, rank=self.rank, world=self.nranks,
            state=self.state, hyper=self.hyper, timeout_s=float(timeout_s),
            msg_bf16=self.msg_bf16, outbox_bytes=int(self.outbox.nbytes))
        self.period = table.shape[0]
        # phase-1 / phase-2 interleave granularity; must be identical on all ranks
        self.ctx.set_segments(int(segments))
        self.max_grid = self.ctx.max_grid()
        sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        nchunks = self.n // C.CHUNK
        if grid is None:
            grid = min(self.max_grid, 2 * sms, C.MAX_CTAS)
        # every rank must use the same grid: per-CTA publish flags are matched by index
        self.grid = int(max(1, min(grid, nchunks, C.MAX_CTAS)))
        if gather_grid is None:
            gather_grid = min(32, self.grid)
        self.gather_grid = int(max(1, min(gather_grid, nchunks)))
        self.gather_tma = bool(gather_tma)
        self.steps = 0               # host mirror of SgpState.step
        self._graph_synced = 0       # rotations applied to the python graph object
        self._refresh_in_peers()
        self.set_hyper(0.0, 0.0, 0.0, False, do_sgd=False)
        torch.cuda.synchronize(self.device)
        world.barrier()

    # -- configuration ------------------------------------------------------ #
    def set_hyper(self, lr, momentum, weight_decay, nesterov, do_sgd=True, grad_scale=1.0, groups=None,
                  max_grad_norm=None):
        """Stage the SGD hyper-parameters for the next launches (device resident: a captured graph
        reads the new values).  ``groups``: with :meth:`set_param_groups`, one
        ``(lr, momentum, weight_decay, nesterov)`` per parameter group; ``do_sgd`` and
        ``grad_scale`` apply to every group.  ``max_grad_norm``: the clipping threshold of
        :meth:`set_grad_clip` (ignored while clipping is off)."""
        key = (float(lr), float(momentum), float(weight_decay), bool(nesterov),
               bool(do_sgd), float(grad_scale), 0.0 if max_grad_norm is None else float(max_grad_norm))
        if groups is not None:
            if len(groups) != self.groups:
                raise ValueError('set_hyper got %d group rows, set_param_groups configured %d'
                                 % (len(groups), self.groups))
            key += tuple((float(a), float(b), float(c), bool(d)) for a, b, c, d in groups)
        if key == self._hyper_cache:
            return
        self._hyper_cache = key
        slot = self._hyper_slot
        self._hyper_slot = (slot + 1) % self._hyper_host.shape[0]
        ev = self._hyper_events[slot]
        if ev is not None:
            ev.synchronize()                 # the copy that last used this slot has executed
        h = self._hyper_host[slot][0]
        h[0], h[1], h[2] = key[0], key[1], key[2]
        h[3] = 1.0 if key[3] else 0.0
        h[4] = 1.0 if key[4] else 0.0
        h[5] = key[5]
        h[6] = key[6]
        if groups is None:
            self.hyper.copy_(h, non_blocking=True)
        else:
            rows = self._hyper_host[slot][:1 + len(groups)]
            for r, (g_lr, g_mu, g_wd, g_nest) in zip(rows[1:], key[7:]):
                r[0], r[1], r[2], r[3] = g_lr, g_mu, g_wd, 1.0 if g_nest else 0.0
            self._hyper_rows[:1 + len(groups)].copy_(rows, non_blocking=True)
        ev = self._hyper_events[slot] = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))

    def set_param_groups(self, block_group: Optional[torch.Tensor], groups: int):
        """Per-parameter-group SGD: ``block_group`` (uint8, one entry per 64 elements of the arena)
        names the group of each 64-element block; every SGD launch then takes lr / momentum /
        weight_decay / nesterov from that group's row, staged by ``set_hyper(..., groups=rows)``.
        ``block_group=None`` returns to the single set of hyper-parameters."""
        if block_group is None:
            self.ctx.set_param_groups(None, None)
            self.groups = 0
        else:
            if not 1 <= groups <= self.C.MAX_GROUPS:
                raise ValueError('1 to %d parameter groups, got %d' % (self.C.MAX_GROUPS, groups))
            self.ctx.set_param_groups(block_group, self._hyper_rows[1:1 + groups])
            self.groups = int(groups)
        self._hyper_cache = None

    def set_lars(self, offsets=None, numels=None, enabled=None, trust_coefficient=0.001, eps=1e-8):
        """LARS on every SGD launch (needs :meth:`set_param_groups`): the arena holds tensors at
        ``offsets`` (64-element aligned, ascending) of ``numels`` elements; ``enabled[t]`` turns the
        trust ratio of tensor t on.  Each SGD launch then runs the norm and trust kernels first and
        scales d = g + wd*x of tensor t by ``lars_trust[t]``.  ``offsets=None`` turns LARS off."""
        if offsets is None:
            self.ctx.set_lars(None, None, None)
            return
        as_t = lambda v, dt: torch.as_tensor(v, dtype=dt, device='cpu')
        self.ctx.set_lars(as_t(offsets, torch.int64), as_t(numels, torch.int64), as_t(enabled, torch.uint8),
                          float(trust_coefficient), float(eps))

    @property
    def lars(self) -> bool:
        return self.ctx.lars()

    @property
    def lars_trust(self) -> Optional[torch.Tensor]:
        """fp32 [tensors] trust ratios of the last SGD launch (device tensor, rewritten by the next)"""
        return self.ctx.lars_trust() if self.ctx.lars() else None

    @property
    def lars_sumsq(self) -> Optional[torch.Tensor]:
        """fp64 [tensors, 2]: sum x^2 and sum g^2 per tensor as the last SGD launch saw them"""
        return self.ctx.lars_sumsq() if self.ctx.lars() else None

    def set_grad_clip(self, offsets=None, numels=None, enabled=True, skip_nonfinite=False):
        """Gradient-norm clipping and non-finite step skipping on every SGD launch.  The arena holds
        tensors at ``offsets`` (64-element aligned, ascending) of ``numels`` elements -- the layout
        :meth:`set_lars` takes; both share one norm plan.  Each SGD launch then first computes, in
        fp64, ``total = |g^|_2`` over those tensors with ``g^ = grad_scale * (g [+ g2])``:

        * ``enabled``: phase 1 applies ``coef * g^`` with ``coef = min(max_grad_norm / (total + 1e-6),
          1)`` (``torch.nn.utils.clip_grad_norm_``; a NaN total gives a NaN coef), ``max_grad_norm``
          staged by :meth:`set_hyper`;
        * ``skip_nonfinite``: a launch whose total is inf or NaN leaves x and the momentum alone (the
          gradient is still cleared, the publish and mix run as usual) and counts in
          :attr:`nonfinite_steps`.

        ``offsets=None`` turns both off.  Turning them on or off changes the launch sequence: a
        captured CUDA graph has to be captured again.  The skip count survives reconfiguration."""
        if offsets is None or not (enabled or skip_nonfinite):
            self.ctx.set_grad_clip(None, None, None, False, False)
            return
        as_t = lambda v: torch.as_tensor(v, dtype=torch.int64, device='cpu')
        self.ctx.set_grad_clip(as_t(offsets), as_t(numels), self._ensure_clip_state(), bool(enabled),
                               bool(skip_nonfinite))

    def _ensure_clip_state(self):
        if getattr(self, '_clip_state', None) is None:
            C = self.C
            self._clip_state = torch.zeros(C.CLIP_STATE_BYTES // 4, dtype=torch.float32, device=self.device)
            self._clip_state[C.CLIP_OFF_COEF // 4] = 1.0
        return self._clip_state

    @property
    def grad_clip(self) -> bool:
        return self.ctx.grad_clip()

    def _clip_word(self, off, dtype=torch.float32):
        if not self.ctx.grad_clip():
            return None
        return self._clip_state.view(dtype)[off // dtype.itemsize]

    @property
    def grad_norm(self) -> Optional[torch.Tensor]:
        """0-dim fp32 device tensor: the gradient norm (before clipping) of the last SGD launch,
        rewritten by the next one; None while clipping and skipping are off.  No synchronisation"""
        return self._clip_word(self.C.CLIP_OFF_TOTAL)

    @property
    def clip_coef(self) -> Optional[torch.Tensor]:
        """0-dim fp32 device tensor: the clip coefficient of the last SGD launch (1 when not clipped)"""
        return self._clip_word(self.C.CLIP_OFF_COEF)

    @property
    def grad_sumsq(self) -> Optional[torch.Tensor]:
        """0-dim fp64 device tensor: sum of g^2 of the last SGD launch"""
        return self._clip_word(self.C.CLIP_OFF_SUMSQ, torch.float64)

    @property
    def nonfinite_steps(self) -> int:
        """SGD launches skipped for a non-finite gradient norm so far (synchronises)"""
        if getattr(self, '_clip_state', None) is None:
            return 0
        return int(self._clip_state.view(torch.int32)[self.C.CLIP_OFF_SKIPPED // 4].item())

    @nonfinite_steps.setter
    def nonfinite_steps(self, v: int):
        self._ensure_clip_state().view(torch.int32)[self.C.CLIP_OFF_SKIPPED // 4] = int(v)

    def clip_update(self):
        """the norm and clip kernels alone, as the next SGD launch would run them (tests, benchmarks)"""
        self.ctx.clip_update()

    def set_schedule(self, graph=None, mixing=None):
        """Re-emit the device tables (e.g. after ``peers_per_itr`` changed).
        Collective in effect: callers drain their streams and barrier first."""
        C = self.C
        self.graph = graph or self.graph
        self.mixing = mixing or self.mixing
        table, wtable = build_tables(self.graph, self.mixing, self.device)
        self.ctx.set_schedule(table, wtable)
        self.period = table.shape[0]
        want = self.graph.phase_index()
        base = (want - self.steps) % self.period
        self._phase_base = int(base)
        self._refresh_in_peers()
        self._state_i32[C.STATE_OFF_PHASE_BASE // 4] = int(base)
        self._state_i32[C.STATE_OFF_ACK_FROM // 4] = int(self.steps)
        self._graph_synced = self.steps

    def set_grad(self, grad: torch.Tensor):
        self.grad = grad
        self.ctx.set_grad(grad)

    def set_sgd_buffers(self, grad: torch.Tensor, momentum: torch.Tensor, grad2=None):
        """``grad2``: optional fp32 buffer (same layout) that is ADDED to ``grad``:
        with bf16 compute weights the convolution/linear gradients arrive in the bf16
        buffer and the BatchNorm gradients in the fp32 one (each zero elsewhere)."""
        self.grad, self.momentum, self.grad2 = grad, momentum, grad2
        self.ctx.set_sgd_buffers(grad, momentum)
        self.ctx.set_grad2(grad2)

    # -- launches ------------------------------------------------------------ #
    def _common(self, sgd, zero_grad, in_numerator=False):
        C = self.C
        f = C.F_IN_NUMER if in_numerator else 0
        if sgd:
            f |= C.F_SGD
            if zero_grad:
                f |= C.F_ZERO_GRAD
        if self.shadow is not None:
            f |= C.F_SHADOW
        return f

    def _check_fp32_messages(self, what):
        if self.msg_bf16:
            raise RuntimeError('GossipEngine.%s is not implemented for bf16 messages (only mix() is)' % what)

    def mix(self, sgd=False, zero_grad=True, in_numerator=False):
        C = self.C
        f = self._common(sgd, zero_grad, in_numerator) | C.F_PHASE1 | C.F_PUBLISH | C.F_PHASE2
        self.ctx.step(f, self.grid)
        self.steps += 1

    def publish(self, sgd=False, fold=False, zero_grad=True, in_numerator=False):
        C = self.C
        self._check_fp32_messages('publish')
        f = self._common(sgd, zero_grad, in_numerator) | C.F_PHASE1 | C.F_PUBLISH
        if fold:
            f |= C.F_FOLD_RES
        self.ctx.step(f, self.grid)
        self.steps += 1

    def _refresh_in_peers(self):
        """in-neighbour per phase (host side) and whether the Overlap-SGP gather can run on the
        copy engines: that needs exactly one in-neighbour in every phase (then the residual is a
        plain copy of its outbox; the edge weight is applied when the residual is folded)."""
        phases = self.graph.phases()
        if not self.graph.is_dynamic_graph():
            phases = phases[:1] * max(1, self.period)
        self._in_peers = [list(ins) for _, ins in phases]
        eligible = self.nranks > 1 and all(len(ins) == 1 for ins in self._in_peers) \
            and len(self._in_peers) == self.period
        pref = self._gather_dma_pref
        if pref is None:
            import os
            pref = os.environ.get('SGP_B200_GATHER_DMA', '1') != '0'     # A/B switch
        self.gather_dma = bool(pref and eligible)

    def dma_key(self):
        """(schedule row, outbox parity) of the NEXT overlap step: what a captured CUDA graph with a
        DMA gather is specific to (the copy's source address is baked into the graph)"""
        return ((self.steps + self._phase_base) % self.period, self.steps & 1)

    def gather(self, tma=None, dma=None):
        """residual <- sum_k in_w[k] * outbox_k (Overlap-SGP side stream).  With one in-neighbour
        per step (the default schedules) this is a COPY-ENGINE transfer of the peer's outbox bracketed
        by a 1-CTA flag wait and a 1-thread ack kernel -- no SM is taken away from the forward pass;
        otherwise a gather kernel (TMA bulk copies by default, register-staged with ``tma=False``)."""
        self._check_fp32_messages('gather')
        use_dma = self.gather_dma if dma is None else (bool(dma) and self.gather_dma)
        if use_dma:
            s = self.steps - 1                       # publish() of this step already advanced the mirror
            j = self._in_peers[(s + self._phase_base) % self.period][0]
            src = self.outbox.peers[j].data_ptr() + (s & 1) * self.n * 4
            self.ctx.gather_dma(self.grid, int(src))
            return
        self.ctx.gather(self.gather_grid, self.grid, self.gather_tma if tma is None else bool(tma))

    def local(self, sgd=False, fold=False, zero_grad=True, in_numerator=False):
        C = self.C
        f = self._common(sgd, zero_grad, in_numerator) | C.F_PHASE1 | C.F_NO_ROTATE
        if fold:
            f |= C.F_FOLD_RES
        self.ctx.step(f, self.grid)

    # -- AD-PSGD building blocks (no kernel ever spins for long) -------------- #
    def publish_only(self):
        """Snapshot z into the outbox and release the flags; nothing else."""
        C = self.C
        self._check_fp32_messages('publish_only')
        self.ctx.step(C.F_PHASE1 | C.F_PUBLISH | C.F_NO_ROTATE | C.F_KEEP_Z, self.grid)

    def pull_only(self):
        """z <- self_w * z_now + sum_k in_w[k] * outbox_k ; ack ; advance the round.
        Call after :meth:`probe` reported the partner's snapshot is visible."""
        C = self.C
        self._check_fp32_messages('pull_only')
        f = C.F_PHASE2 | C.F_PUBLISH | C.F_SELF_FROM_Z
        if self.shadow is not None:
            f |= C.F_SHADOW
        self.ctx.step(f, self.grid)
        self.steps += 1

    def probe(self, host_flag=None):
        self._check_fp32_messages('probe')
        self.ctx.probe(self.grid, host_flag)

    def barrier(self):
        self.ctx.barrier()

    def consensus(self, out: Optional[torch.Tensor] = None, full: bool = False) -> torch.Tensor:
        """Consensus distance of the de-biased parameters z_i over every rank (collective: every
        rank of the world calls it, between gossip steps).  With the push-sum weights w_i,
        zbar = sum_i w_i z_i / sum_i w_i; returns an fp64 device tensor ``[2 + world]``:
        ``[distance_sq = (1/n) sum_i |z_i - zbar|^2, |zbar|^2, |z_0 - zbar|^2, ...]`` (the per-rank
        terms only with ``full=True``; zeros otherwise), bit-identical on every rank.  The tensor is
        this engine's result buffer: the next call rewrites it.

        ``full=False``: each rank reduces a 1/world slice of the elements (NVLink ingress about one
        model per rank).  ``full=True``: every rank computes the whole zbar into ``out`` (fp32,
        length n, required).

        Stream-ordered on the current stream, without a host synchronisation and without
        allocating after the first call (loop-back
        tests enqueue every virtual rank before synchronising).  The outbox is borrowed between
        device barriers; the gossip sequence numbers are untouched, so the next step runs as if
        this call had not happened.  A timed-out barrier yields NaN and raises at :meth:`poll`."""
        if full and out is None:
            raise ValueError('GossipEngine.consensus(full=True) writes the average model into `out`')
        self.prepare_consensus()
        return self.ctx.consensus(out if full else None, bool(full))

    def prepare_consensus(self):
        """Allocate what :meth:`consensus` needs (collective, once; consensus() calls it on first
        use).  A process that drives several virtual ranks from several threads calls it on every
        rank first: an allocation implicitly synchronises the device, which must not happen while
        another virtual rank's barrier kernel waits for this one."""
        if getattr(self, '_cons_slots', None) is not None:
            return
        C = self.C
        # 4 doubles per rank, symmetric: every rank reads every rank's partial sums
        self._cons_slots = self.world.alloc(self._name + '.consensus', 4 * 8)
        self._cons_scratch = torch.zeros(C.MAX_CTAS * 4 + 1, dtype=torch.float64, device=self.device)
        self._cons_result = torch.zeros(2 + self.nranks, dtype=torch.float64, device=self.device)
        sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        nchunks = self.n // C.CHUNK
        self.ctx.set_consensus_buffers(self._cons_slots.table, self._cons_scratch, self._cons_result,
                                       int(max(1, min(2 * sms, nchunks, C.MAX_CTAS))))

    def slowmo(self, u: torch.Tensor, x_prev: torch.Tensor, lr: float, alpha: float, beta: float,
               init: bool):
        """SlowMo step (collective: every rank of the world calls it, between gossip steps).  With
        zbar = sum_i w_i z_i / sum_i w_i, the same bits on every rank:

            init:  x_prev <- zbar ; u <- 0 ; z <- zbar
            else:  u <- beta u + (x_prev - zbar) / lr ; x_prev <- x_prev - alpha lr u ; z <- x_prev

        ``u`` / ``x_prev`` are fp32 tensors of the arena's length, identical on every rank; the
        bf16 shadow follows z, and both push-sum weights become 1.  Stream-ordered on the current
        stream, without a host synchronisation or an allocation; the step counter and the gossip
        sequence numbers are untouched.  A timed-out barrier leaves z, u, x_prev and the weights as
        they were and raises at :meth:`poll`."""
        C = self.C
        sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        grid = int(max(1, min(2 * sms, self.n // C.CHUNK, C.MAX_CTAS)))
        self.ctx.slowmo(u, x_prev, float(lr), float(alpha), float(beta), bool(init), grid)

    # -- host-visible state (each of these synchronises) -------------------- #
    def sync_graph(self):
        """Advance the python GraphManager to the device's phase."""
        if self.graph.is_dynamic_graph():
            for _ in range(self.steps - self._graph_synced):
                self.graph.get_peers(rotate=True)
        self._graph_synced = self.steps

    @property
    def status(self) -> int:
        return int(self._state_i32[self.C.STATE_OFF_STATUS // 4].item())

    def poll(self, blocking: bool = False):
        """Heartbeat poll of the kernels' sticky status word.  Non-blocking: enqueue a 4-byte
        async copy of the word into pinned host memory on the current stream and look at the
        value the PREVIOUS poll delivered (no host synchronisation; a failure is reported one
        poll late).  ``blocking=True`` synchronises the stream first.  Raises
        ``NameError('Gossip flag timeout')`` -- the reference's heartbeat error
        (``gossip/distributed.py:349-352``)."""
        if self._status_host is None:
            self._status_host = torch.zeros(1, dtype=torch.int32).pin_memory()
            self._status_dev = self._state_i32[self.C.STATE_OFF_STATUS // 4:
                                               self.C.STATE_OFF_STATUS // 4 + 1]
            self._soft_host = torch.zeros(1, dtype=torch.int32).pin_memory()
            self._soft_dev = self._state_i32[self.C.STATE_OFF_SOFT_TIMEOUTS // 4:
                                             self.C.STATE_OFF_SOFT_TIMEOUTS // 4 + 1]
        if torch.cuda.is_current_stream_capturing():
            return
        st = int(self._status_host[0])
        soft = int(self._soft_host[0])
        if soft > self._soft_seen:           # a peer was slower than the soft heartbeat; we kept waiting
            import logging
            logging.getLogger('sgp_b200').warning(
                'rank %d: %d gossip wait(s) exceeded the soft heartbeat and were retried (kept '
                'waiting for the peer)', self.rank, soft - self._soft_seen)
            self._soft_seen = soft
        if st == 0:
            self._status_host.copy_(self._status_dev, non_blocking=True)
            self._soft_host.copy_(self._soft_dev, non_blocking=True)
            if blocking:
                torch.cuda.current_stream(self.device).synchronize()
                st = int(self._status_host[0])
        if st != 0:
            raise NameError('Gossip flag timeout (rank %d: %s)' % (self.rank, self._status_name(st)))

    @staticmethod
    def _status_name(st):
        return {1: 'in-neighbour never published (heartbeat timeout)',
                2: 'out-neighbour never released the outbox (ack timeout)',
                3: 'device barrier timeout'}.get(st, 'code %d' % st)

    def check(self):
        st = self.status
        if st != 0:
            names = {1: 'in-neighbour never published (heartbeat timeout)',
                     2: 'out-neighbour never released the outbox (ack timeout)',
                     3: 'device barrier timeout'}
            raise RuntimeError('gossip kernel error on rank %d: %s'
                               % (self.rank, names.get(st, 'code %d' % st)))

    @property
    def soft_timeouts(self) -> int:
        """waits that exceeded the soft heartbeat so far (synchronises)"""
        return int(self._state_i32[self.C.STATE_OFF_SOFT_TIMEOUTS // 4].item())

    def clear_status(self):
        """forget a reported heartbeat failure (after the application decided to carry on)"""
        self._state_i32[self.C.STATE_OFF_STATUS // 4] = 0
        if self._status_host is not None:
            self._status_host.zero_()

    @property
    def device_step(self) -> int:
        return int(self._state_i32[self.C.STATE_OFF_STEP // 4].item())

    @property
    def ps_weight(self) -> float:
        off = self.C.STATE_OFF_PSW // 4
        step = self.device_step
        return float(self._state_f32[off + (step & 1)].item())

    @ps_weight.setter
    def ps_weight(self, v: float):
        off = self.C.STATE_OFF_PSW // 4
        self._state_f32[off: off + 2] = float(v)

    def ps_weight_tensor(self) -> torch.Tensor:
        """1-element device tensor view of the CURRENT push-sum weight (no sync
        of the value itself, but reads the step counter)."""
        off = self.C.STATE_OFF_PSW // 4
        return self._state_f32[off + (self.device_step & 1): off + (self.device_step & 1) + 1]

    @property
    def res_scale(self) -> float:
        """factor the pending residual buffer is multiplied with when folded (1 after a gather
        kernel; the in-neighbour's edge weight after a copy-engine gather)"""
        return float(self._state_f32[self.C.STATE_OFF_RES_SCALE // 4].item())

    @property
    def res_weight(self) -> float:
        return float(self._state_f32[self.C.STATE_OFF_RESW // 4].item())
