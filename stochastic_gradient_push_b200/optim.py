"""
FusedGossipSGD: SGD-with-momentum whose update runs INSIDE the gossip kernel.

The reference calls ``torch.optim.SGD.step()`` (P x 3..5 elementwise launches
in torch 1.x, ``gossip_sgd.py:200-205, 389``) and then ``transfer_params()``.
Here ``optimizer.step()`` only records the hyper-parameters (device-resident,
so a captured CUDA graph picks up learning-rate changes) and marks the update
pending; the next gossip launch of the wrapped
:class:`~.parallel.distributed.GossipDataParallel` -- ``transfer_params()`` in
sync mode, the forward pre-hook in overlap mode -- applies

    d = g + wd*x ; m = mu*m + d ; x -= lr*(nesterov ? d + mu*m : m)

to the push-sum *numerator* in the same pass that publishes / mixes it (the
reference also steps the numerator: its backward hook re-biases before
``optimizer.step``, ``gossip/distributed.py:564-565``).  Gradients live in one
flat buffer (``p.grad`` are views, autograd accumulates in place) that the
kernel zeroes after consuming, so ``zero_grad()`` is free.

On the c10d transport (CPU / gloo) the same update runs as plain torch ops on
the flat arena -- that path is the oracle for the kernel.

``param_groups`` (torch.optim style) gives groups of parameters their own lr,
momentum, weight_decay and nesterov -- e.g. :func:`no_bias_decay_groups`.  Every
arena tensor starts on a 64-element boundary, so a uint8 map with one entry per
64-element block names each element's group exactly; the kernels read it next
to a device table of the groups' values (DESIGN.md 2.0.3).

``lars=True`` (per group, or for all) adds layer-wise adaptive rate scaling (LARS; You, Gitman,
Ginsburg, 2017) as apex ``LARC(clip=False)`` puts it in front of SGD: every parameter tensor p of
such a group takes

    t_p = eta |x_p| / (|g_p| + wd |x_p| + eps)   (1 if |x_p| or |g_p| is 0) ;  d = t_p * (g + wd*x)

with x the push-sum numerator the step acts on.  The kernels compute the norms and t on the device
before every SGD launch (DESIGN.md 2.0.4); :func:`lars_groups` is the MLPerf ResNet-50 recipe.

``max_grad_norm`` clips the gradient the update consumes, g^ = grad_scale * g, as
``torch.nn.utils.clip_grad_norm_(params, max_grad_norm)`` would (norm type 2, over every parameter
of every group, in fp64); LARS then sees the clipped gradient.  ``skip_nonfinite=True`` skips the
SGD of a step whose gradient norm is inf or NaN: x and the momentum keep their bits, the gradient is
still cleared, and the rank keeps gossiping (DESIGN.md 2.0.6).
"""

from __future__ import annotations

import torch

from .ops import oracle

MAX_GROUPS = 16           # == SGP_MAX_GROUPS (sgp_common.cuh)
GROUP_BLOCK = 64          # == SGP_GROUP_BLOCK: elements per block-map entry
_HYPER_KEYS = ('lr', 'momentum', 'weight_decay', 'nesterov')
LARS_MAX_TENSORS = 65535  # == SGP_LARS_MAX_TENSORS: the block -> tensor map is uint16


def no_bias_decay_groups(module, weight_decay):
    """Two parameter groups for "no bias decay" (He et al., Bag of Tricks, CVPR 2019): every
    parameter with ``ndim <= 1`` (BatchNorm weight and bias, all biases) with ``weight_decay=0``,
    then everything else with ``weight_decay``.  For :class:`FusedGossipSGD` and torch.optim alike."""
    params = list(module.parameters())
    return [dict(params=[p for p in params if p.dim() <= 1], weight_decay=0.0),
            dict(params=[p for p in params if p.dim() > 1], weight_decay=weight_decay)]


def lars_groups(module, weight_decay):
    """The MLPerf ResNet-50 LARS recipe as two parameter groups: every parameter with ``ndim <= 1``
    (BatchNorm weight and bias, all biases) with ``weight_decay=0`` and ``lars=False``, then
    everything else with ``weight_decay`` and ``lars=True``."""
    params = list(module.parameters())
    return [dict(params=[p for p in params if p.dim() <= 1], weight_decay=0.0, lars=False),
            dict(params=[p for p in params if p.dim() > 1], weight_decay=weight_decay, lars=True)]


class FusedGossipSGD(object):

    def __init__(self, model, lr=0.1, momentum=0.0, weight_decay=0.0, nesterov=False,
                 grad_scale=1.0, param_groups=None, lars=False, trust_coefficient=0.001, lars_eps=1e-8,
                 max_grad_norm=None, skip_nonfinite=False):
        """``max_grad_norm``: a float > 0 clips the gradient of every step to that global 2-norm
        (``torch.nn.utils.clip_grad_norm_`` semantics); None: off.  ``skip_nonfinite``: a step whose
        gradient norm is inf or NaN leaves the parameters and the momentum unchanged, clears the
        gradient and counts in :attr:`nonfinite_steps`; without it such a norm propagates into the
        update as in torch (a NaN coefficient, or 0 for an infinite norm).

        Both act per rank, on the gradient the update consumes: gossip has no global gradient, and
        in hierarchical mode (``nprocs_per_node > 1``) the backward hook has already averaged it over
        the node, so every rank of a node clips the same node gradient.  BatchNorm running statistics
        are not protected: a NaN that the forward pass produces reaches them before any check.

        Turning either option on or off changes the kernel launches of a step, so a captured CUDA
        graph (GossipTrainer) has to be captured again; ``max_grad_norm`` itself lives in device
        memory, and a new value reaches a captured graph."""
        from .parallel.distributed import GossipDataParallel
        assert isinstance(model, GossipDataParallel)
        if nesterov and momentum <= 0:
            raise ValueError('Nesterov momentum requires a momentum')
        if not trust_coefficient > 0 or not lars_eps >= 0:
            raise ValueError('LARS needs trust_coefficient > 0 and lars_eps >= 0')
        self._max_grad_norm = self._check_max_grad_norm(max_grad_norm)
        self.skip_nonfinite = bool(skip_nonfinite)
        self.model = model
        self.defaults = dict(lr=lr, momentum=momentum, weight_decay=weight_decay,
                             nesterov=nesterov, dampening=0, lars=bool(lars))
        self.trust_coefficient = float(trust_coefficient)
        self.lars_eps = float(lars_eps)
        if param_groups is None:
            self.param_groups = [dict(self.defaults, params=[p for p in model.module.parameters()])]
        else:
            self.param_groups = self._partition(model, param_groups, self.defaults)
        # one group runs exactly the ungrouped path; several, or LARS, get the block map
        # (_setup_groups)
        self._lars_flags = None
        self._grouped = len(self.param_groups) > 1 or self._lars_on()
        self.grad_scale = grad_scale
        self._arenas = model._arenas
        self.grad_flat, self.momentum_flat = {}, {}
        for dtype, arena in self._arenas.items():
            hier = getattr(model, '_hier_grad', None)
            # hierarchical mode on the kernel plane: keep accumulating into the symmetric
            # (multicast-bound) flat gradient so the local-node average stays one NVLS kernel
            self.grad_flat[dtype] = hier if (hier is not None and dtype == torch.float32) \
                else arena.new_buffer()
            self.momentum_flat[dtype] = arena.new_buffer(dtype=torch.float32
                                                         if dtype != torch.float64 else dtype)
            arena.bind_grads(model._params_by_dtype[dtype], self.grad_flat[dtype])
        self.grad_lo = None
        if model._kernel is not None and model._twin:
            # bf16 compute twin: its conv/linear gradients accumulate into a bf16 flat
            # buffer, the normalisation gradients (and anything computed through the fp32
            # master module) into the fp32 one; the kernel adds the two
            arena = self._arenas[torch.float32]
            self.grad_lo = arena.new_buffer(dtype=torch.bfloat16)
            lo_views = arena.views_of(self.grad_lo)
            hi_views = arena.views_of(self.grad_flat[torch.float32])
            for p, lo, hi in zip(model._twin[0].parameters(), lo_views, hi_views):
                if p.requires_grad:
                    p.grad = lo if p.dtype == torch.bfloat16 else hi
            model._kernel.attach_sgd(self.grad_lo, self.momentum_flat[torch.float32],
                                     grad2=self.grad_flat[torch.float32])
        elif model._kernel is not None:
            model._kernel.attach_sgd(self.grad_flat[torch.float32],
                                     self.momentum_flat[torch.float32])
        model._fused_optimizer = self
        self._steps = 0
        if self._grouped:
            self._setup_groups()
        self._clip_flags = None
        self._setup_clip()

    @staticmethod
    def _partition(model, param_groups, defaults):
        """torch.optim-style group dicts -> groups that partition ``model.module.parameters()``
        (parameters not listed go into one trailing group with the constructor's values)"""
        index = {id(p): i for i, p in enumerate(model.module.parameters())}
        seen = set()
        groups = []
        for spec in param_groups:
            if not isinstance(spec, dict) or 'params' not in spec:
                raise ValueError('each parameter group is a dict with a "params" entry')
            params = spec['params']
            params = [params] if isinstance(params, torch.Tensor) else list(params)
            for p in params:
                if id(p) not in index:
                    raise ValueError('a parameter group holds a tensor that is not a parameter of '
                                     'the wrapped model')
                if id(p) in seen:
                    raise ValueError('a parameter appears in more than one parameter group')
                seen.add(id(p))
            groups.append(dict(spec, params=params))
        rest = [p for p in model.module.parameters() if id(p) not in seen]
        if rest:
            groups.append(dict(params=rest))
        if len(groups) > MAX_GROUPS:
            raise ValueError('FusedGossipSGD supports at most %d parameter groups, got %d'
                             % (MAX_GROUPS, len(groups)))
        groups = [dict(defaults, **g) for g in groups]
        for g in groups:
            if g['nesterov'] and g['momentum'] <= 0:
                raise ValueError('Nesterov momentum requires a momentum (parameter group with '
                                 'momentum=%r)' % (g['momentum'],))
        return groups

    def _setup_groups(self):
        """block map (uint8, one entry per 64 elements) of every dtype arena; the kernel plane
        hands the fp32 one to the engine, the c10d plane expands it to per-element indices"""
        m = self.model
        group_of = {}
        for gi, g in enumerate(self.param_groups):
            for p in g['params']:
                group_of[id(p)] = gi
        self._block_group, self._elem_group = {}, {}
        self._hyper_vectors, self._hyper_vectors_key = {}, None
        for dtype, arena in self._arenas.items():
            bmap = torch.zeros(arena.total // GROUP_BLOCK, dtype=torch.uint8)
            for p, off, n in zip(m._params_by_dtype[dtype], arena.offsets, arena.numels):
                if off % GROUP_BLOCK:
                    raise ValueError('per-group SGD needs every arena tensor on a %d-element '
                                     'boundary' % GROUP_BLOCK)
                bmap[off // GROUP_BLOCK: (off + n + GROUP_BLOCK - 1) // GROUP_BLOCK] = group_of[id(p)]
            self._block_group[dtype] = bmap.to(arena.device)
        k = m._kernel
        if k is not None:
            k.engine.set_param_groups(self._block_group[torch.float32], len(self.param_groups))
        else:
            for dtype, bmap in self._block_group.items():
                self._elem_group[dtype] = bmap.long().repeat_interleave(GROUP_BLOCK)
        self._setup_lars()

    def _lars_on(self):
        return any(g['lars'] for g in self.param_groups)

    def _setup_lars(self):
        """per-tensor LARS flags of every arena (fixed until load_state_dict changes them); the
        kernel plane hands the fp32 arena's layout to the engine, which builds its maps and tiles"""
        m = self.model
        lars_of = {}
        for g in self.param_groups:
            for p in g['params']:
                lars_of[id(p)] = bool(g['lars'])
        self._lars_flags = tuple(bool(g['lars']) for g in self.param_groups)
        self._tensor_lars, self._elem_tensor, self._tensor_group = {}, {}, {}
        if not self._lars_on():
            if m._kernel is not None:
                m._kernel.engine.set_lars(None)
            return
        for dtype, arena in self._arenas.items():
            params = m._params_by_dtype[dtype]
            if len(params) > LARS_MAX_TENSORS:
                raise ValueError('LARS supports at most %d tensors per arena, the %s arena holds %d'
                                 % (LARS_MAX_TENSORS, dtype, len(params)))
            self._tensor_lars[dtype] = [lars_of[id(p)] for p in params]
        k = m._kernel
        if k is not None:
            arena = self._arenas[torch.float32]
            k.engine.set_lars(arena.offsets, arena.numels, self._tensor_lars[torch.float32],
                              self.trust_coefficient, self.lars_eps)
        else:
            for dtype, arena in self._arenas.items():
                idx = torch.full((arena.total,), len(arena.offsets), dtype=torch.long)   # padding: own bin
                for t, (off, n) in enumerate(zip(arena.offsets, arena.numels)):
                    idx[off:off + n] = t
                self._elem_tensor[dtype] = idx
                bmap = self._block_group[dtype]
                self._tensor_group[dtype] = [int(bmap[off // GROUP_BLOCK]) for off in arena.offsets]

    def _c10d_trust(self, dtype, x, g):
        """per-element LARS trust ratios of one arena: fp64 norms of the numerator and of the scaled
        gradient per tensor, t = eta |x| / (|g| + wd |x| + eps) where the tensor's group has lars=True
        and both norms are > 0, else 1"""
        idx = self._elem_tensor[dtype].to(x.device)
        T = len(self._tensor_lars[dtype])
        sx = torch.zeros(T + 1, dtype=torch.float64, device=x.device).index_add_(0, idx, x.double() ** 2)
        sg = torch.zeros(T + 1, dtype=torch.float64, device=x.device).index_add_(0, idx, g.double() ** 2)
        nx, ng = sx[:T].sqrt(), sg[:T].sqrt()
        wd = torch.tensor([float(self.param_groups[gi]['weight_decay']) for gi in self._tensor_group[dtype]],
                          dtype=torch.float64, device=x.device)
        on = torch.tensor(self._tensor_lars[dtype], device=x.device) & (nx > 0) & (ng > 0)
        t = torch.where(on, self.trust_coefficient * nx / (ng + wd * nx + self.lars_eps),
                        torch.ones_like(nx))
        return torch.cat([t, t.new_ones(1)]).to(x.dtype)[idx]

    @staticmethod
    def _check_max_grad_norm(v):
        if v is None:
            return None
        try:
            v = float(v)
        except (TypeError, ValueError):
            raise ValueError('max_grad_norm must be a finite number > 0 or None, got %r' % (v,))
        if not (v > 0 and v != float('inf')):
            raise ValueError('max_grad_norm must be a finite number > 0 or None, got %r' % (v,))
        return v

    @property
    def max_grad_norm(self):
        """the clipping threshold (None: off).  A new value reaches the next step, a captured CUDA graph
        included; switching between None and a number re-plans the launches (re-capture needed)"""
        return self._max_grad_norm

    @max_grad_norm.setter
    def max_grad_norm(self, v):
        self._max_grad_norm = self._check_max_grad_norm(v)
        if self._clip_flags is not None and (self._max_grad_norm is not None, self.skip_nonfinite) != self._clip_flags:
            self._setup_clip()

    def _clip_on(self):
        return self.max_grad_norm is not None or self.skip_nonfinite

    def _setup_clip(self):
        """hand the fp32 arena's layout to the engine (kernel plane; it shares the LARS norm plan),
        or mark each arena's tensor elements, padding excluded (c10d plane)"""
        m = self.model
        self._clip_flags = (self.max_grad_norm is not None, self.skip_nonfinite)
        self._elem_valid = {}
        if not hasattr(self, '_nonfinite'):
            dev = self._arenas[next(iter(self._arenas))].device
            self._nonfinite = torch.zeros((), dtype=torch.int64, device=dev)     # c10d plane
            self._grad_norm = torch.zeros((), dtype=torch.float32, device=dev)
        k = m._kernel
        if k is not None:
            if not self._clip_on():
                k.engine.set_grad_clip(None)
                return
            arena = self._arenas[torch.float32]
            k.engine.set_grad_clip(arena.offsets, arena.numels, enabled=self.max_grad_norm is not None,
                                   skip_nonfinite=self.skip_nonfinite)
            return
        if self._clip_on():
            for dtype, arena in self._arenas.items():
                valid = torch.zeros(arena.total, dtype=torch.bool)
                for off, n in zip(arena.offsets, arena.numels):
                    valid[off:off + n] = True
                self._elem_valid[dtype] = valid.to(arena.device)

    def _c10d_clip(self, grads):
        """(coef or None, skip) of the c10d plane: the fp64 2-norm of every arena's scaled gradient,
        coef = max_grad_norm / (total + 1e-6) clamped at 1 (torch.clamp keeps a NaN), and whether
        skip_nonfinite skips this step (a 0-dim bool tensor, so no synchronisation)"""
        sumsq = None
        for dtype, g in grads.items():
            s = g.double()[self._elem_valid[dtype].to(g.device)].square().sum()
            sumsq = s if sumsq is None else sumsq + s.to(sumsq.device)
        total = sumsq.sqrt()
        self._grad_norm.copy_(total)
        coef = None
        if self.max_grad_norm is not None:
            coef = torch.clamp(self.max_grad_norm / (total + 1e-6), max=1.0).float()
        skip = None
        if self.skip_nonfinite:
            skip = ~torch.isfinite(total)
            self._nonfinite += skip.to(self._nonfinite.device)
        return coef, skip

    @property
    def grad_norm(self):
        """0-dim fp32 device tensor: the gradient norm before clipping of the last SGD step, rewritten
        by the next (None while clipping and skipping are off).  Reading it does not synchronise."""
        if not self._clip_on():
            return None
        k = self.model._kernel
        return k.engine.grad_norm if k is not None else self._grad_norm

    @property
    def nonfinite_steps(self) -> int:
        """steps skipped for a non-finite gradient norm so far (synchronises)"""
        k = self.model._kernel
        if k is not None:
            return k.engine.nonfinite_steps
        return int(self._nonfinite.item())

    def _set_nonfinite_steps(self, n):
        k = self.model._kernel
        if k is not None:
            k.engine.nonfinite_steps = n
        else:
            self._nonfinite.fill_(int(n))

    # -- torch.optim-like surface -------------------------------------------- #
    def _hyper(self):
        g = self.param_groups[0]
        return g['lr'], g['momentum'], g['weight_decay'], g['nesterov']

    def _group_rows(self):
        for g in self.param_groups:
            if g['nesterov'] and g['momentum'] <= 0:
                raise ValueError('Nesterov momentum requires a momentum')
        return [tuple(g[k] for k in _HYPER_KEYS) for g in self.param_groups]

    def set_engine_hyper(self, engine, do_sgd=True):
        """Stage every group's current values into the engine's device table (GossipTrainer calls
        this before each replay, so per-group lr changes reach a captured graph)"""
        lr, mu, wd, nest = self._hyper()
        engine.set_hyper(lr, mu, wd, nest, do_sgd=do_sgd, grad_scale=self.grad_scale,
                         groups=self._group_rows() if self._grouped else None,
                         max_grad_norm=self.max_grad_norm)

    def _c10d_vectors(self, dtype, rows):
        """per-element (lr, momentum, weight_decay, nesterov) of one arena, rebuilt only when a
        group's values changed"""
        if rows != self._hyper_vectors_key:
            self._hyper_vectors, self._hyper_vectors_key = {}, rows
        vec = self._hyper_vectors.get(dtype)
        if vec is None:
            idx = self._elem_group[dtype]
            arena = self._arenas[dtype]
            table = torch.tensor([r[:3] for r in rows], dtype=dtype)
            nest = torch.tensor([bool(r[3]) for r in rows])
            vec = self._hyper_vectors[dtype] = tuple(
                t.to(arena.device) for t in (table[:, 0][idx], table[:, 1][idx], table[:, 2][idx], nest[idx]))
        return vec

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        lr, mu, wd, nest = self._hyper()
        k = self.model._kernel
        if k is not None:
            self.set_engine_hyper(k.engine)
            k.sgd_pending = True
        else:
            m = self.model
            m.ps_numerator()                       # step the numerator (reference :564)
            rows = self._group_rows() if self._grouped else None
            grads = {}
            for dtype in self._arenas:
                g = self.grad_flat[dtype]
                grads[dtype] = g * self.grad_scale if self.grad_scale != 1.0 else g
            coef, skip = self._c10d_clip(grads) if self._clip_on() else (None, None)
            for dtype, arena in self._arenas.items():
                g = grads[dtype] if coef is None else grads[dtype] * coef.to(grads[dtype].device)
                if rows is not None:
                    lr, mu, wd, nest = self._c10d_vectors(dtype, rows)
                trust = self._c10d_trust(dtype, arena.flat, g) if self._lars_flags and any(self._lars_flags) \
                    else None
                x, mom = oracle.sgd_momentum(arena.flat, g, self.momentum_flat[dtype],
                                             lr, mu, wd, nest, trust=trust)
                if skip is not None:              # a skipped step keeps the numerator and momentum bits
                    keep = skip.to(x.device)
                    x = torch.where(keep, arena.flat, x)
                    mom = torch.where(keep, self.momentum_flat[dtype], mom)
                arena.flat.copy_(x)
                self.momentum_flat[dtype].copy_(mom)
        self._steps += 1
        return loss

    def zero_grad(self, set_to_none=False):
        """Free on the kernel path (the fused kernel clears the flat gradient
        right after reading it); explicit memset otherwise."""
        k = self.model._kernel
        if k is not None and k.sgd_pending:
            return
        for g in self.grad_flat.values():
            g.zero_()
        if self.grad_lo is not None:
            self.grad_lo.zero_()

    def state_dict(self):
        self.model._flush_pending()
        groups = [{k: v for k, v in g.items() if k != 'params'} for g in self.param_groups]
        return {'param_groups': groups, 'steps': self._steps,
                'lars': {'trust_coefficient': self.trust_coefficient, 'eps': self.lars_eps},
                'grad_clip': {'max_grad_norm': self.max_grad_norm, 'skip_nonfinite': self.skip_nonfinite,
                              'nonfinite_steps': self.nonfinite_steps},
                'momentum': {str(dt): m.detach().cpu().clone()
                             for dt, m in self.momentum_flat.items()}}

    def load_state_dict(self, sd):
        """Restores every group's hyper-parameters.  A checkpoint of a one-group optimizer also
        loads into a grouped one: its lr (the schedule's state) goes to every group, and each group
        keeps its own momentum, weight decay and nesterov.  The groups' ``lars`` flags, the trust
        coefficient and eps are restored too; if they change, the LARS maps are rebuilt (a CUDA graph
        captured before then has to be captured again).  So are ``max_grad_norm``, ``skip_nonfinite``
        and the count of skipped steps; a checkpoint without them keeps the constructor's values."""
        saved = sd['param_groups']
        before = (tuple(bool(g['lars']) for g in self.param_groups), self.trust_coefficient, self.lars_eps)
        if 'lars' in sd:
            self.trust_coefficient = float(sd['lars']['trust_coefficient'])
            self.lars_eps = float(sd['lars']['eps'])
        if len(saved) == len(self.param_groups):
            for g, s in zip(self.param_groups, saved):
                g.update({k: v for k, v in s.items() if k != 'params'})
                g['lars'] = bool(g.get('lars', False))
        elif len(saved) == 1:
            for g in self.param_groups:
                g['lr'] = saved[0]['lr']
        else:
            raise ValueError('checkpoint has %d parameter groups, this optimizer %d'
                             % (len(saved), len(self.param_groups)))
        after = (tuple(bool(g['lars']) for g in self.param_groups), self.trust_coefficient, self.lars_eps)
        if after != before:
            if self._grouped:
                self._setup_lars()
            else:
                self._grouped = True
                self._setup_groups()
        clip = sd.get('grad_clip')
        if clip is not None:
            self._max_grad_norm = self._check_max_grad_norm(clip['max_grad_norm'])
            self.skip_nonfinite = bool(clip['skip_nonfinite'])
            if (self._max_grad_norm is not None, self.skip_nonfinite) != self._clip_flags:
                self._setup_clip()
            self._set_nonfinite_steps(int(clip.get('nonfinite_steps', 0)))
        self._steps = sd.get('steps', 0)
        for dt, m in self.momentum_flat.items():
            m.copy_(sd['momentum'][str(dt)])
