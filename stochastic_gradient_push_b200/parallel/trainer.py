"""
GossipTrainer: the flagship training step, captured ONCE as a CUDA graph.

One replay = forward (bf16 autocast, NHWC) + loss + backward + ONE fused
gossip kernel (SGD-momentum + publish + P2P pull + mix + de-bias), i.e. the
reference's whole hot loop (``gossip_sgd.py:369-393`` + the pre-forward /
backward hooks + the gossip thread) with zero Python on the critical path:

* the time-varying graph is a device table the kernel indexes with its own
  device-side step counter; the learning rate lives in device memory -- so the
  captured graph never needs re-capturing;
* Overlap-SGP forks the gather kernel onto ``gossip_stream`` INSIDE the graph:
  it pulls the peers' parameters over NVLink while forward/backward run;
* inputs arrive from pinned host memory through a prefetch stream (H2D of step
  k+1 overlaps compute of step k); the loss is read back through a pinned ring
  without a per-step host synchronisation.

Modes: ``'sgp'`` (push-sum, directed graph), ``'dpsgd'`` (push-pull, symmetric
graph) -- same kernel, the graph/mixing differ --, ``'osgp'`` (overlap), and
``'local'`` (world size 1 / gossip disabled).

Mixup / CutMix (``batch_mix=ops.batch_mix.BatchMix(...)``): the stage -> static input copy becomes
one launch of the batch-mix kernel (same bytes read and written), after an H2D copy of the step's
draw into the device mix state; the captured fused cross-entropy reads ``lam`` from that state.

Weight EMA (``ema=ops.model_ema.ModelEma(model, ...)``): ``ema.update()`` is the LAST launch of every
step, eager warm-up steps and captured graph alike, on the trainer's stream after the forward pass
(which updated the BatchNorm running statistics) and after the gossip / SGD launch -- under
Overlap-SGP after ``publish`` and the join with the gossip stream.  The EMA therefore follows the
parameters exactly as the next forward pass sees them: under Overlap-SGP the residual gathered during
step k is folded in at the next publish, so it reaches the EMA one step later, and a SlowMo step
(enqueued after the replay) reaches it at the next step.

Gradient accumulation (``accumulation_steps=k``): ``step()`` still takes the whole step batch of B
rows (one H2D copy); the step runs k forward/backward passes on the row slices
``static_in[j m:(j+1) m]``, m = B / k, then ONE gossip / SGD launch and one EMA update.  Micro-batch 0
writes its gradients into the arena as a k = 1 step does; each later one adds its fresh gradients with
one ``grad_accumulate`` launch (fp32 sums; with the bf16 twin into the fp32 ``g2`` buffer, which the
step kernel adds to the bf16 one).  The kernel scales the sum by ``fp32(grad_scale / k)``: the gradient
of the mean loss over the B rows, with BatchNorm statistics taken per micro-batch as in torch.  So
BatchNorm running statistics are updated k times per step (momentum applied each time) and
``num_batches_tracked`` grows by k; the metrics row is the mean of the k micro-batches' ``[loss,
prec@1, prec@5]``; ``static_out`` holds the LAST micro-batch's logits.  With ``batch_mix`` one draw
serves the step and each micro-batch is mixed with its own flipped micro-batch.

Evaluation (``evaluate(batches)``): the same network and precision as the step (the bf16 twin, else the
module under the trainer's autocast) in eval mode, one captured graph per batch shape: the forward, with
every 1x1 / stride-1 convolution and its BatchNorm (+ residual) (+ ReLU) as one GEMM launch
(``ops.fused_bn.eval_bn_gemm``), and one ``xent_eval_accumulate`` launch that adds the batch's loss sum
and top-1 / top-5 / row counts to a device accumulator, read back once at the end.  Nothing the
training step owns is touched.

Precise BatchNorm statistics (``update_bn(batches)``): the same network and precision in train mode
under ``torch.no_grad()``, over K batches, staged and captured per batch shape as in ``evaluate``.
Inside ``ops.fused_bn.precise_bn_stats`` every BatchNorm finalize launch adds its batch's mean and
unbiased variance to an fp64 accumulator instead of its running buffers; one ``bn_stats_commit``
launch then sets every running buffer to ``fp32(sum / K)``.  The first batch of a shape runs eagerly
(and is counted) before its graph is captured; a capture does not execute, so every batch is counted
once.

Stochastic depth (a ResNet built with ``drop_path_rate > 0``) lives in the model: each training forward
draws its masks with one ``drop_path_draw`` launch, so ``own_launches_per_step`` grows by one per forward
(k with ``accumulation_steps=k``: each micro-batch has its own masks), and every replay draws fresh
ones.  ``update_bn`` (inside ``precise_bn_stats``) and ``evaluate`` (eval mode) draw nothing and scale
nothing: precise statistics describe the network that evaluation runs.
"""

from __future__ import annotations

import contextlib
import math
import numbers
import os
from typing import Callable, NamedTuple, Optional

import torch

from ..ops.fused_bn import BNStatsAccumulator, eval_bn_gemm, precise_bn_stats
from ..ops.fused_loss import FusedCrossEntropyWithAccuracy, eval_accumulate, eval_accumulator
from ..optim import FusedGossipSGD
from .distributed import GossipDataParallel


def check_accumulation_steps(k) -> int:
    """``k`` as an int; ValueError unless it is an integer >= 1 (not a bool)."""
    if isinstance(k, bool) or not isinstance(k, numbers.Integral) or k < 1:
        raise ValueError('accumulation_steps must be an integer >= 1, got %r' % (k,))
    return int(k)


class EvalResult(NamedTuple):
    """What :meth:`GossipTrainer.evaluate` measured over the rows whose target is in ``[0, classes)``:
    the mean plain cross-entropy, prec@1 and prec@5 in percent, and the number of such rows."""
    loss: float
    prec1: float
    prec5: float
    count: int

    @classmethod
    def from_sums(cls, loss_sum: float, top1: int, top5: int, count: int) -> 'EvalResult':
        """from the accumulated sums; NaN means (and a count of 0) when no row was counted"""
        count = int(count)
        if count <= 0:
            return cls(math.nan, math.nan, math.nan, 0)
        return cls(float(loss_sum) / count, 100.0 * int(top1) / count, 100.0 * int(top5) / count, count)


class _EvalSlot(object):
    """per evaluation batch shape: staging and static buffers, and the captured graphs of
    ``evaluate`` (``graph``) and ``update_bn`` (``bn_graph``)"""
    __slots__ = ('stage', 'stage_tgt', 'static_in', 'static_tgt', 'ready', 'free', 'graph', 'out', 'bn_graph')


class GossipTrainer(object):

    def __init__(self, model: GossipDataParallel, optimizer: FusedGossipSGD,
                 criterion: Optional[Callable] = None, amp_dtype=torch.bfloat16,
                 use_cuda_graph: bool = True, warmup_iters: int = 3,
                 channels_last: bool = True, batch_mix=None, ema=None, accumulation_steps: int = 1):
        """``batch_mix``: an ``ops.batch_mix.BatchMix`` to train with mixup / CutMix (needs the
        fused criterion; the draw of each step comes from ``batch_mix.iteration``), or None.
        ``ema``: an ``ops.model_ema.ModelEma`` of ``model`` updated at the end of every step, or None.
        ``accumulation_steps``: k >= 1 forward/backward passes per step over equal row slices of the
        step batch, whose size must be divisible by k (see the module docstring); not with
        ``nprocs_per_node > 1``."""
        accumulation_steps = check_accumulation_steps(accumulation_steps)
        if accumulation_steps > 1 and getattr(model, 'nprocs_per_node', 1) > 1:
            raise ValueError('accumulation_steps > 1 is not supported with nprocs_per_node > 1 (hierarchical '
                             'mode averages the gradient inside the node at every backward pass)')
        assert model._kernel is not None, 'GossipTrainer drives the nvlink kernel transport'
        self.model = model
        self.opt = optimizer
        self.engine = model._kernel.engine
        self.k = model._kernel
        self.overlap = model.overlap
        self.gossip = model.dist_config['world_size'] > 1
        self._init_runtime(self.engine.device, criterion, amp_dtype, use_cuda_graph, warmup_iters,
                           channels_last, batch_mix, ema)
        self._slowmo_on = model.slowmo_frequency > 0      # step() runs the SlowMo step itself
        self.accumulation_steps = accumulation_steps
        if accumulation_steps > 1 and not self.batched_grad_copy and getattr(model, '_twin', None):
            raise ValueError('accumulation_steps > 1 with the bf16 compute twin needs the batched gradient '
                             'copy (SGP_B200_BATCHED_GRAD_COPY=0 would sum its gradients in bf16)')

    def _init_runtime(self, device, criterion, amp_dtype, use_cuda_graph, warmup_iters, channels_last,
                      batch_mix=None, ema=None):
        """state shared by every trainer flavour (gossip / all-reduce / bilateral)"""
        # default: fused softmax cross-entropy that also yields prec@1 / prec@5 (the reference loop
        # measures both every iteration, gossip_sgd.py:394-399) in the same launch
        self.criterion = criterion or FusedCrossEntropyWithAccuracy()
        self._fused_loss = isinstance(self.criterion, FusedCrossEntropyWithAccuracy)
        if batch_mix is not None and not batch_mix.enabled:
            batch_mix = None                     # both alphas 0: the plain copy and loss
        if batch_mix is not None and not self._fused_loss:
            raise ValueError('batch_mix needs the fused criterion (FusedCrossEntropyWithAccuracy): it '
                             'carries the mixed targets into the loss')
        self.batch_mix = batch_mix
        self.amp_dtype = amp_dtype
        self.use_graph = use_cuda_graph
        self.warmup_iters = warmup_iters
        self.channels_last = channels_last
        self.device = device
        self.graph = None
        self.static_in = None
        self.static_tgt = None
        self.static_loss = None
        self.static_metrics = None
        self.static_out = None
        self._eager_steps = 0
        # see _backward(); SGP_B200_BATCHED_GRAD_COPY=0 restores per-parameter accumulation
        self.batched_grad_copy = os.environ.get('SGP_B200_BATCHED_GRAD_COPY', '1') != '0'
        self._grad_slots = None
        self.accumulation_steps = 1          # (GossipTrainer(accumulation_steps=k) sets k)
        self._accum_dst = None               # per grad slot: the fp32 view micro-batches 1..k-1 add into
        self._micro = None                   # [(input slice, target slice)] of the k micro-batches
        self._micro_metrics = None           # [k, 3]: [loss, prec@1, prec@5] of each micro-batch
        # slots whose fresh gradient had a foreign dtype, shape or strides and were added with add_()
        self.accum_fallbacks = 0
        # every launch of the step runs on ONE dedicated side stream: autograd's
        # AccumulateGrad nodes are then created on the stream the graph is captured on
        self.stream = torch.cuda.Stream(device=self.device)
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        self.ema = ema
        if ema is not None:
            ema._stream = self.stream          # set_decay() / the counter read order with the step
        self._copy_stream = torch.cuda.Stream(device=self.device)
        self._stage = None
        self._stage_tgt = None
        self._stage_ready = torch.cuda.Event()
        self._stage_free = torch.cuda.Event()
        self._prefetched = False
        self._loss_ring = None
        self._loss_slot = 0
        self._skip_next_sgd = False
        self._slowmo_on = False
        # kernels of OUR extension in one training step (counted over the graph capture, or over
        # the last eager step): what bench.py reports as gpu_launches / step
        self.own_launches_per_step = None
        self._graphs = {}               # overlap + DMA gather: one captured graph per (row, parity)
        self._pool = None
        self._eval_slots = {}           # evaluate(): one _EvalSlot (and graph) per batch shape
        self._eval_acc = None
        self.eval_out = None            # logits of the last batch of the last evaluate()
        self.eval_launches_per_batch = None
        self._bn_acc = None             # update_bn(): the fp64 BatchNorm statistics accumulator
        self.update_bn_launches_per_batch = None

    # ------------------------------------------------------------------ #
    def _autocast(self):
        if self.amp_dtype is None or self.amp_dtype == torch.float32:
            return contextlib.nullcontext()
        return torch.autocast('cuda', dtype=self.amp_dtype)

    def _fwd_bwd(self):
        if self.accumulation_steps == 1:
            out = self._fwd_bwd_one(self.static_in, self.static_tgt, self.static_metrics, accumulate=False)
        else:
            for j, (x, t) in enumerate(self._micro):
                out = self._fwd_bwd_one(x, t, self._micro_metrics[j], accumulate=j > 0)
            torch.mean(self._micro_metrics, 0, out=self.static_metrics)
        self.static_out = out.detach()

    def _fwd_bwd_one(self, x, tgt, metrics_out, accumulate):
        """forward + loss + backward of one (micro-)batch; its ``[loss, prec@1 %, prec@5 %]`` go to
        ``metrics_out``.  ``accumulate``: add the gradients to the arena instead of writing them."""
        twin = getattr(self.model, '_twin', None)
        net = None
        if twin:
            # bf16 twin: weights already live in bf16 (shadow arena), input buffer is bf16
            net = twin[0]
            net.train(self.model.module.training)
            out = net(x)
            loss = self._loss(out, tgt)
        else:
            with self._autocast():
                out = self.model.module(x)
                loss = self._loss(out, tgt)
        self._backward(loss, net if twin else self.model.module, accumulate)
        metrics = getattr(self.criterion, 'metrics', None)
        if metrics is not None:
            metrics_out.copy_(metrics)                  # [loss, prec@1 %, prec@5 %]
        else:
            metrics_out[0].copy_(loss.detach())
        return out

    def _loss(self, out, tgt):
        if self.batch_mix is not None:            # two targets per row, lam from the device mix state
            return self.criterion(out, tgt, mix=self.batch_mix.state)
        return self.criterion(out if self._fused_loss else out.float(), tgt)

    def _backward(self, loss, net, accumulate=False):
        """``loss.backward()`` without ~160 per-parameter accumulate kernels: the flat gradient
        buffers are zero at this point (the fused SGD kernel clears them), so instead of letting
        autograd run ``p.grad += g`` once per parameter, the ``.grad`` views are detached for
        the backward pass (autograd then just keeps each fresh gradient) and the results are
        written into the arena with one multi-tensor copy per dtype.

        ``accumulate`` (micro-batches 1 .. k-1 of gradient accumulation): the fresh gradients are
        added in fp32 to :meth:`_accum_views` by one ``grad_accumulate`` launch instead."""
        if not self.batched_grad_copy:
            loss.backward()                                # (autograd accumulates into the views)
            return
        if self._grad_slots is None:
            self._grad_slots = [(p, p.grad) for p in net.parameters()
                                if p.requires_grad and p.grad is not None]
        for p, _ in self._grad_slots:
            p.grad = None
        loss.backward()
        if accumulate:
            self._accumulate_grads(net)
            return
        by_dtype = {}
        for p, view in self._grad_slots:
            g = p.grad
            p.grad = view
            if g is None:
                continue                                   # no gradient this step: slot stays zero
            if g.dtype != view.dtype or g.shape != view.shape:
                view.copy_(g)                              # foreign layout / dtype: plain copy
                continue
            dst, src = by_dtype.setdefault(view.dtype, ([], []))
            dst.append(view)
            src.append(g)
        for dst, src in by_dtype.values():
            torch._foreach_copy_(dst, src)

    def _accum_views(self, net):
        """per grad slot, the fp32 view the later micro-batches add into: the slot's own view for an
        fp32 model; with the bf16 twin the parameter's view in the fp32 ``g2`` buffer (``lo`` keeps
        micro-batch 0 in bf16, the step kernel reads ``g + g2`` and clears both)"""
        if self._accum_dst is None:
            if getattr(self.model, '_twin', None):
                hi = self.opt._arenas[torch.float32].views_of(self.opt.grad_flat[torch.float32])
                by_param = {id(p): v for p, v in zip(net.parameters(), hi)}
                self._accum_dst = [by_param[id(p)] for p, _ in self._grad_slots]
            else:
                self._accum_dst = [view for _, view in self._grad_slots]
        return self._accum_dst

    def _accumulate_grads(self, net):
        dst, src = [], []
        for (p, view), acc in zip(self._grad_slots, self._accum_views(net)):
            g = p.grad
            p.grad = view
            if g is None:
                continue
            # (a size-1 dim's stride addresses nothing: a 1x1 conv's fresh gradient may come
            # channels_last-strided while its arena view is contiguous, with the same memory order)
            if (acc.dtype == torch.float32 and g.dtype in (torch.float32, torch.bfloat16)
                    and g.shape == acc.shape
                    and all(n == 1 or a == b for n, a, b in zip(g.shape, g.stride(), acc.stride()))):
                dst.append(acc)
                src.append(g)
            else:
                acc.add_(g)                                # foreign layout / dtype: plain add
                self.accum_fallbacks += 1
        if dst:
            self.engine.C.grad_accumulate(dst, src)

    def _step_sync(self):
        """forward/backward, then ONE kernel: SGD + publish + pull + mix + de-bias
        (SGD only when there is nobody to gossip with)."""
        self._fwd_bwd()
        if self.gossip and self.model.gossip_enable:
            self.engine.mix(sgd=True)
        else:
            self.engine.local(sgd=True)

    def _step_overlap(self, first: bool):
        """publish(k) -> [gather(k) on gossip_stream || fwd/bwd(k)] ; the SGD of
        step k is fused into publish(k+1)."""
        e, k = self.engine, self.k
        main = torch.cuda.current_stream(self.device)
        side = self.model.gossip_stream
        e.publish(sgd=not first, fold=not first)
        fork = torch.cuda.Event()
        fork.record(main)
        side.wait_event(fork)
        with torch.cuda.stream(side):
            e.gather()
            join = torch.cuda.Event()
            join.record(side)
        self._fwd_bwd()
        main.wait_event(join)

    def _full_step(self, first=False):
        """the step of every trainer flavour (its ``_one_step``), then the EMA update as its last launch"""
        self._one_step(first)
        if self.ema is not None:
            self.ema.update()

    def _one_step(self, first=False):
        if self.overlap and self.gossip and self.model.gossip_enable:
            self._step_overlap(first)
        else:
            self._step_sync()

    # ------------------------------------------------------------------ #
    def _ensure_static(self, batch, target):
        if self.static_in is not None:
            return
        k = self.accumulation_steps
        if batch.shape[0] % k:
            raise ValueError('the step batch of %d rows is not divisible by accumulation_steps=%d'
                             % (batch.shape[0], k))
        fmt = torch.channels_last if (self.channels_last and batch.dim() == 4) \
            else torch.contiguous_format
        in_dtype = torch.bfloat16 if getattr(self.model, '_twin', None) else batch.dtype
        self.static_in = torch.empty(batch.shape, dtype=in_dtype, device=self.device
                                     ).contiguous(memory_format=fmt)
        self.static_tgt = torch.empty(target.shape, dtype=target.dtype, device=self.device)
        # staging keeps the HOST layout (plain pinned memcpy); the device-side
        # stage -> static copy performs the NCHW -> NHWC permute
        self._stage = torch.empty(batch.shape, dtype=batch.dtype, device=self.device)
        self._stage_tgt = torch.empty_like(self.static_tgt)
        self.static_metrics = torch.full((3,), float('nan'), dtype=torch.float32, device=self.device)
        self.static_loss = self.static_metrics[0]
        if k > 1:
            # dim-0 slices: an NHWC slice is itself channels_last-contiguous, so no copy
            m = batch.shape[0] // k
            self._micro = [(self.static_in[j * m:(j + 1) * m], self.static_tgt[j * m:(j + 1) * m])
                           for j in range(k)]
            self._micro_metrics = torch.full((k, 3), float('nan'), dtype=torch.float32, device=self.device)
        self._metrics_ring = torch.zeros(1024, 3, dtype=torch.float32).pin_memory()
        self._loss_ring = self._metrics_ring[:, 0]
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        self._stage_free.record(self.stream)

    def _set_lr(self):
        # overlap: the SGD of step k runs inside publish(k+1).  After finish() applied it early
        # (end of epoch / checkpoint) the next replay's publish must not apply it again: the
        # captured kernel reads `do_sgd` from device memory.  Every parameter group's values go
        # to the device table too, so a per-group lr change needs no re-capture
        do_sgd = not self._skip_next_sgd
        self._skip_next_sgd = False
        if isinstance(self.opt, FusedGossipSGD):
            self.opt.set_engine_hyper(self.engine, do_sgd=do_sgd, micro_batches=self.accumulation_steps)
            return
        g = self.opt.param_groups[0]          # (the all-reduce / AD-PSGD trainers' one-group facades)
        self.engine.set_hyper(g['lr'], g['momentum'], g['weight_decay'], g['nesterov'],
                              do_sgd=do_sgd, grad_scale=self.opt.grad_scale)

    def prefetch(self, batch_cpu, target_cpu):
        """Start the H2D copy of the NEXT step's inputs on the copy stream."""
        self._ensure_static(batch_cpu, target_cpu)
        cs = self._copy_stream
        cs.wait_event(self._stage_free)
        on_device = [t for t in (batch_cpu, target_cpu) if t.is_cuda]
        if on_device:
            # inputs produced on the GPU (e.g. data.GpuAugment output, a target moved by the caller):
            # order the copy after the stream that produced them and keep their memory alive
            cs.wait_stream(torch.cuda.current_stream(self.device))
            for t in on_device:
                t.record_stream(cs)
        with torch.cuda.stream(cs):
            self._stage.copy_(batch_cpu, non_blocking=True)
            self._stage_tgt.copy_(target_cpu, non_blocking=True)
            self._stage_ready.record(cs)
        self._prefetched = True

    def _load_inputs(self, batch, target):
        main = self.stream
        if batch is not None and not self._prefetched:
            self.prefetch(batch, target)
        main.wait_event(self._stage_ready)
        with torch.cuda.stream(main):
            if self.batch_mix is not None:
                # the same read and write of the batch, mixed with its flipped batch on the way
                # (with accumulation: each micro-batch with its own flipped micro-batch, one draw)
                self.batch_mix.apply(self._stage, self.static_in, micro_batches=self.accumulation_steps)
            else:
                self.static_in.copy_(self._stage, non_blocking=True)
            self.static_tgt.copy_(self._stage_tgt, non_blocking=True)
            self._stage_free.record(main)
        self._prefetched = False

    def step(self, batch=None, target=None, next_batch=None, next_target=None,
             read_loss: bool = True):
        """One training iteration through the public path.

        ``batch``/``target``: (pinned) host or device tensors for THIS step;
        pass ``None`` if a previous call already staged them via
        ``next_batch``/``prefetch``.  ``next_batch``/``next_target``: inputs of
        the FOLLOWING step; their H2D copy is started on the prefetch stream as
        soon as this step's inputs have left the staging buffer, so it overlaps
        this step's compute.  Returns the slot of :attr:`loss_ring` that holds
        this step's loss -- and of :attr:`metrics_ring` that holds ``[loss, prec@1 %, prec@5 %]``
        -- once the stream has drained (no host sync here)."""
        if batch is not None:
            self._ensure_static(batch, target)
        self._load_inputs(batch, target)
        if next_batch is not None:
            self.prefetch(next_batch, next_target)
        self._run()
        if self._slowmo_on:
            gamma = self.model._slowmo_tick(self.opt)
            if gamma is not None:
                self._slowmo(gamma)
        slot = self._loss_slot
        if read_loss:
            with torch.cuda.stream(self.stream):
                self._metrics_ring[slot].copy_(self.static_metrics, non_blocking=True)   # 12 bytes D2H
            self._loss_slot = (slot + 1) % self._metrics_ring.shape[0]
        return slot

    def step_resident(self):
        """Replay the step on whatever is resident in the static input buffers
        (no H2D, no loss read-back): the device-only number of bench.py."""
        assert self.static_in is not None
        self._run()

    def _run(self):
        with torch.cuda.stream(self.stream):
            self._run_on_stream()

    def _graph_key(self):
        """Overlap-SGP with the copy-engine gather: the source address of the DMA copy (which
        in-neighbour, which outbox half) is baked into a captured graph, so there is one graph per
        (schedule row, parity) -- lcm(period, 2) of them, sharing one memory pool."""
        if self.overlap and self.gossip and self.model.gossip_enable \
                and getattr(self.engine, 'gather_dma', False):
            return self.engine.dma_key()
        return None

    def _run_on_stream(self):
        self._set_lr()
        key = self._graph_key()
        if key is not None and self._graphs:
            if key not in self._graphs:           # first visit of this (row, parity): capture it
                self.graph = None
                self._capture()
            self.graph = self._graphs[key]
        if self.graph is not None:
            self.graph.replay()
            self._after_replay()
        elif self.use_graph and self._eager_steps >= self.warmup_iters:
            self._capture()
            self.graph.replay()
            self._after_replay()
        else:
            c0 = self.engine.C.launch_count()
            self._full_step(first=(self._eager_steps == 0))
            self.own_launches_per_step = self.engine.C.launch_count() - c0
            self._eager_steps += 1

    def _after_replay(self):
        if self.gossip and self.model.gossip_enable:
            self.engine.steps += 1

    @property
    def loss_ring(self):
        return self._loss_ring

    @property
    def metrics_ring(self):
        """pinned ``[1024, 3]`` ring: row ``slot`` = ``[loss, prec@1 %, prec@5 %]`` of that step"""
        return self._metrics_ring

    def _capture(self):
        torch.cuda.synchronize(self.device)
        steps_before = self.engine.steps
        self.graph = torch.cuda.CUDAGraph()
        if self._pool is None:
            self._pool = torch.cuda.graph_pool_handle()      # shared by the per-(row, parity) graphs
        key = self._graph_key()
        c0 = self.engine.C.launch_count()
        with torch.cuda.graph(self.graph, stream=self.stream, capture_error_mode='thread_local',
                              pool=self._pool):
            self._full_step(first=False)
        self.own_launches_per_step = self.engine.C.launch_count() - c0
        if key is not None:
            self._graphs[key] = self.graph
        # capture does not execute: undo the host-side step mirror advance
        self.engine.steps = steps_before
        torch.cuda.synchronize(self.device)

    def _slowmo(self, gamma):
        """The SlowMo step of ``model.slowmo_frequency > 0`` (see ``GossipDataParallel.perform_slowmo``,
        which users of the trainer do not call): enqueued on the trainer's stream after the step,
        with no host synchronisation; a heartbeat failure surfaces at the next check() / poll().
        Overlap-SGP first lands the deferred SGD and the gathered residual as finish() does.  The
        engine's step counter does not advance, so the captured graphs stay valid."""
        with torch.cuda.stream(self.stream):
            if self.overlap and self.gossip and self.model.gossip_enable:
                self.stream.wait_stream(self.model.gossip_stream)
                self._set_lr()
                self.engine.local(sgd=True, fold=True)
                self.engine.residual.zero_()       # already folded: the next publish adds 0
                self._skip_next_sgd = True
            self.model._slowmo_launch(gamma)

    def finish(self):
        """Drain: apply the last deferred SGD / residual (overlap), sync, and poll the kernels'
        health word.  Call at the end of an epoch, before validation / ``state_dict()``: the
        parameters then hold every update and all the push-sum mass received so far.  Training
        may simply continue afterwards (the next step skips the SGD that was applied here)."""
        if self.overlap and self.gossip and self._eager_steps + (self.graph is not None) > 0:
            with torch.cuda.stream(self.stream):
                self.stream.wait_stream(self.model.gossip_stream)
                self._set_lr()
                self.engine.local(sgd=True, fold=True)
                self.engine.residual.zero_()       # already folded: the next publish adds 0
            self._skip_next_sgd = True
        torch.cuda.synchronize(self.device)
        self.engine.check()

    def check(self):
        """Raise if a gossip kernel reported a heartbeat / ack timeout (reads one word)."""
        self.engine.check()

    # ------------------------------------------------------------------ #
    def evaluate(self, batches) -> EvalResult:
        """Validation of the current model over ``batches`` (an iterable of ``(input, target)``, (pinned)
        host or device tensors; a loader).  Drains the trainer first (:meth:`finish`), then runs the step's
        network in eval mode -- BatchNorm with its running statistics -- and restores the previous mode.
        Loss is the plain cross-entropy (no smoothing, no mixing); rows whose target is outside
        ``[0, classes)`` are not counted.  The H2D copy of batch i+1 overlaps batch i; each batch shape
        is captured once (in the trainer's graph pool) and replayed on later calls, so this works inside
        ``ModelEma.applied()`` and ``GossipDataParallel.averaged()``, which swap values in place.
        Parameters, momentum, BatchNorm statistics, the engine's step counter, the metrics ring, the
        training buffers and graphs, the EMA and the batch-mix iteration are left as they were.
        ``eval_out``: the last batch's logits; ``eval_launches_per_batch``: our kernels per batch."""
        self.finish()
        twin = getattr(self.model, '_twin', None)
        net = twin[0] if twin else self.model.module
        modules = [self.model.module] + ([net] if twin else [])
        modes = [m.training for m in modules]
        main = torch.cuda.current_stream(self.device)
        if self._eval_acc is None:
            self._eval_acc = eval_accumulator(self.device)
        self.stream.wait_stream(main)            # (in-place swaps by ema.applied() / averaged() on main)
        with torch.cuda.stream(self.stream):
            self._eval_acc.zero_()
        try:
            for m in modules:
                m.eval()
            with torch.no_grad():
                _, out = self._staged_pass(batches, lambda slot: self._eval_run(slot, net))
        finally:
            for m, mode in zip(modules, modes):
                m.train(mode)
        with torch.cuda.stream(self.stream):
            if out is not None:
                self.eval_out = out.clone()
            acc = self._eval_acc.cpu()           # the one read-back (synchronises the stream)
        main.wait_stream(self.stream)
        return EvalResult.from_sums(float(acc[:1].view(torch.float64)), int(acc[1]), int(acc[2]), int(acc[3]))

    def _staged_pass(self, batches, run):
        """``run(slot)`` for every ``(input, target)`` of ``batches`` in order, each staged through its
        shape's :class:`_EvalSlot`; the H2D copy of batch i+1 overlaps batch i.  Returns (number of
        batches, what the last ``run`` returned)."""
        n, out = 0, None
        it = iter(batches)
        nxt = next(it, None)
        slot = self._eval_prefetch(*nxt) if nxt is not None else None
        while slot is not None:
            self._eval_load(slot)
            nxt = next(it, None)
            cur, slot = slot, (self._eval_prefetch(*nxt) if nxt is not None else None)
            out = run(cur)
            n += 1
        return n, out

    def _eval_prefetch(self, batch, target) -> _EvalSlot:
        """start the H2D copy of an evaluation batch into its shape's staging buffers (copy stream)"""
        key = (tuple(batch.shape), batch.dtype, tuple(target.shape), target.dtype)
        slot = self._eval_slots.get(key)
        if slot is None:
            slot = self._eval_slots[key] = _EvalSlot()
            fmt = torch.channels_last if (self.channels_last and batch.dim() == 4) else torch.contiguous_format
            in_dtype = torch.bfloat16 if getattr(self.model, '_twin', None) else batch.dtype
            slot.static_in = torch.empty(batch.shape, dtype=in_dtype, device=self.device
                                         ).contiguous(memory_format=fmt)
            slot.static_tgt = torch.empty(target.shape, dtype=target.dtype, device=self.device)
            slot.stage = torch.empty(batch.shape, dtype=batch.dtype, device=self.device)
            slot.stage_tgt = torch.empty_like(slot.static_tgt)
            slot.ready, slot.free = torch.cuda.Event(), torch.cuda.Event()
            slot.graph = slot.out = slot.bn_graph = None
            slot.free.record(self.stream)
        cs = self._copy_stream
        cs.wait_event(slot.free)
        on_device = [t for t in (batch, target) if t.is_cuda]
        if on_device:
            cs.wait_stream(torch.cuda.current_stream(self.device))
            for t in on_device:
                t.record_stream(cs)
        with torch.cuda.stream(cs):
            slot.stage.copy_(batch, non_blocking=True)
            slot.stage_tgt.copy_(target, non_blocking=True)
            slot.ready.record(cs)
        return slot

    def _eval_load(self, slot: _EvalSlot):
        self.stream.wait_event(slot.ready)
        with torch.cuda.stream(self.stream):
            slot.static_in.copy_(slot.stage, non_blocking=True)
            slot.static_tgt.copy_(slot.stage_tgt, non_blocking=True)
            slot.free.record(self.stream)

    def _eval_autocast(self):
        """the step's precision: the bf16 twin runs without autocast, the module under the trainer's"""
        return contextlib.nullcontext() if getattr(self.model, '_twin', None) else self._autocast()

    def _eval_forward(self, slot: _EvalSlot, net):
        """forward + accumulate of one batch on the trainer's stream (captured or eager)"""
        with eval_bn_gemm(), self._eval_autocast():
            out = net(slot.static_in)
        eval_accumulate(out, slot.static_tgt, self._eval_acc)
        return out

    def _eval_run(self, slot: _EvalSlot, net):
        C = self.engine.C
        with torch.cuda.stream(self.stream):
            if not self.use_graph:
                c0 = C.launch_count()
                out = self._eval_forward(slot, net)
                self.eval_launches_per_batch = C.launch_count() - c0
                return out
            if slot.graph is None:
                # warm-up forward outside the capture (library algorithm choice, lazy initialisation);
                # eval mode writes no state, and the accumulator is not touched
                with eval_bn_gemm(), self._eval_autocast():
                    net(slot.static_in)
                torch.cuda.synchronize(self.device)
                if self._pool is None:
                    self._pool = torch.cuda.graph_pool_handle()
                graph = torch.cuda.CUDAGraph()
                c0 = C.launch_count()
                with torch.cuda.graph(graph, stream=self.stream, capture_error_mode='thread_local',
                                      pool=self._pool):
                    slot.out = self._eval_forward(slot, net)
                self.eval_launches_per_batch = C.launch_count() - c0
                slot.graph = graph
            slot.graph.replay()
            return slot.out

    # ------------------------------------------------------------------ #
    def update_bn(self, batches) -> int:
        """Precise BatchNorm statistics: set every BatchNorm layer's running mean and variance to the
        average over ``batches`` (an iterable of ``(input, target)`` as for :meth:`evaluate`; targets are
        ignored) of the batch mean and unbiased variance that the training forward computes for each batch,
        ``running = fp32(sum_k stat_k / K)`` with the sum in fp64 in batch order.  Every batch weighs the
        same, a partial one included (as ``torch.optim.swa_utils.update_bn``).  Drains the trainer first
        (:meth:`finish`), then runs the step's network and precision in train mode under ``no_grad``, each
        batch normalised by its own statistics; restores the previous mode.  Each batch shape is captured
        once (in the trainer's graph pool) and replayed on later calls, so this works inside
        ``ModelEma.applied()`` and ``GossipDataParallel.averaged()``.  Only the running statistics change:
        ``num_batches_tracked``, parameters, momentum, the engine's step counter, the metrics ring, the
        training buffers and graphs, the EMA and the batch-mix iteration are left as they were.  Returns K;
        with K = 0 nothing changes.  ``update_bn_launches_per_batch``: our kernels per batch."""
        self.finish()
        twin = getattr(self.model, '_twin', None)
        net = twin[0] if twin else self.model.module
        modules = [self.model.module] + ([net] if twin else [])
        modes = [m.training for m in modules]
        if self._bn_acc is None:
            self._bn_acc = BNStatsAccumulator(net)
        main = torch.cuda.current_stream(self.device)
        self.stream.wait_stream(main)            # (in-place swaps by ema.applied() / averaged() on main)
        with torch.cuda.stream(self.stream):
            self._bn_acc.zero_()
        try:
            for m in modules:
                m.train()
            with torch.no_grad(), precise_bn_stats(self._bn_acc):
                k, _ = self._staged_pass(batches, lambda slot: self._bn_run(slot, net))
        finally:
            for m, mode in zip(modules, modes):
                m.train(mode)
        if k > 0:
            with torch.cuda.stream(self.stream):
                self._bn_acc.commit(k)
        main.wait_stream(self.stream)
        return k

    def _bn_forward(self, slot: _EvalSlot, net):
        with self._eval_autocast():
            net(slot.static_in)

    def _bn_run(self, slot: _EvalSlot, net):
        """one batch of :meth:`update_bn` on the trainer's stream: its statistics go to the accumulator"""
        C = self.engine.C
        with torch.cuda.stream(self.stream):
            if slot.bn_graph is not None:
                slot.bn_graph.replay()
                return
            # eager: every batch; graphs: the first batch of a shape (library algorithm choice, lazy
            # initialisation) -- it is counted here, so the capture below is not replayed for it
            c0 = C.launch_count()
            self._bn_forward(slot, net)
            self.update_bn_launches_per_batch = C.launch_count() - c0
            if not self.use_graph:
                return
            torch.cuda.synchronize(self.device)
            if self._pool is None:
                self._pool = torch.cuda.graph_pool_handle()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=self.stream, capture_error_mode='thread_local', pool=self._pool):
                self._bn_forward(slot, net)
            slot.bn_graph = graph
