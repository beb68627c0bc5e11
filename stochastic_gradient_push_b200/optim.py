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
"""

from __future__ import annotations

import torch

from .ops import oracle

MAX_GROUPS = 16           # == SGP_MAX_GROUPS (sgp_common.cuh)
GROUP_BLOCK = 64          # == SGP_GROUP_BLOCK: elements per block-map entry
_HYPER_KEYS = ('lr', 'momentum', 'weight_decay', 'nesterov')


def no_bias_decay_groups(module, weight_decay):
    """Two parameter groups for "no bias decay" (He et al., Bag of Tricks, CVPR 2019): every
    parameter with ``ndim <= 1`` (BatchNorm weight and bias, all biases) with ``weight_decay=0``,
    then everything else with ``weight_decay``.  For :class:`FusedGossipSGD` and torch.optim alike."""
    params = list(module.parameters())
    return [dict(params=[p for p in params if p.dim() <= 1], weight_decay=0.0),
            dict(params=[p for p in params if p.dim() > 1], weight_decay=weight_decay)]


class FusedGossipSGD(object):

    def __init__(self, model, lr=0.1, momentum=0.0, weight_decay=0.0, nesterov=False,
                 grad_scale=1.0, param_groups=None):
        from .parallel.distributed import GossipDataParallel
        assert isinstance(model, GossipDataParallel)
        if nesterov and momentum <= 0:
            raise ValueError('Nesterov momentum requires a momentum')
        self.model = model
        self.defaults = dict(lr=lr, momentum=momentum, weight_decay=weight_decay,
                             nesterov=nesterov, dampening=0)
        if param_groups is None:
            self.param_groups = [dict(self.defaults, params=[p for p in model.module.parameters()])]
        else:
            self.param_groups = self._partition(model, param_groups, self.defaults)
        # one group runs exactly the ungrouped path; several get the block map (_setup_groups)
        self._grouped = len(self.param_groups) > 1
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
                         groups=self._group_rows() if self._grouped else None)

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
            for dtype, arena in self._arenas.items():
                g = self.grad_flat[dtype]
                if self.grad_scale != 1.0:
                    g = g * self.grad_scale
                if rows is not None:
                    lr, mu, wd, nest = self._c10d_vectors(dtype, rows)
                x, mom = oracle.sgd_momentum(arena.flat, g, self.momentum_flat[dtype],
                                             lr, mu, wd, nest)
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
                'momentum': {str(dt): m.detach().cpu().clone()
                             for dt, m in self.momentum_flat.items()}}

    def load_state_dict(self, sd):
        """Restores every group's hyper-parameters.  A checkpoint of a one-group optimizer also
        loads into a grouped one: its lr (the schedule's state) goes to every group, and each group
        keeps its own momentum, weight decay and nesterov."""
        saved = sd['param_groups']
        if len(saved) == len(self.param_groups):
            for g, s in zip(self.param_groups, saved):
                g.update({k: v for k, v in s.items() if k != 'params'})
        elif len(saved) == 1:
            for g in self.param_groups:
                g['lr'] = saved[0]['lr']
        else:
            raise ValueError('checkpoint has %d parameter groups, this optimizer %d'
                             % (len(saved), len(self.param_groups)))
        self._steps = sd.get('steps', 0)
        for dt, m in self.momentum_flat.items():
            m.copy_(sd['momentum'][str(dt)])
