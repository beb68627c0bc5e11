"""
ResNet / ImageNet trainer for AR-SGD, SGP, Overlap-SGP and D-PSGD.

Functional parity with the reference's ``gossip_sgd.py`` (``main`` :163,
``train`` :346, ``validate`` :440, ``accuracy`` :474, ``update_state`` :491,
``update_peers_per_itr`` :497, ``update_learning_rate`` :508,
``make_dataloader`` :539, ``parse_args`` :586, ``init_model`` :693): same flags,
same LR / peers-per-itr schedules, same per-rank CSV, same checkpoint layout.

Launch (one rank per GPU):
    torchrun --nproc-per-node 8 gossip_sgd.py --batch_size 256 --lr 0.1 \
        --num_epochs 90 --nesterov True --warmup True --push_sum True --graph_type 0 \
        --schedule 30 0.1 60 0.1 80 0.1 --checkpoint_dir ./ckpt/ [--dataset_dir /imagenet]
or under SLURM with the scripts in ``job_scripts/`` (SLURM_PROCID / SLURM_NTASKS).

H100-native execution: parameters in a flat arena, SGD fused into the gossip
kernel (``--fused True``), bf16 NHWC compute (``--amp/--channels_last``),
device-side metrics read out once per ``--print_freq`` instead of three host
syncs per iteration, optional whole-step CUDA graph (``--cuda_graph True``).
"""

from __future__ import annotations

import itertools
import os
import socket
import time

import torch
import torch.distributed as dist
import torch.nn as nn

from . import common
from .common import (CSVLog, ConsensusLog, Meter, accuracy, build_parser, finalize_args,
                     fresh_state, init_model, make_dataloader, update_learning_rate,
                     update_peers_per_itr, update_state)
from ..experiment import ClusterManager, make_logger
from ..utils import tracing
from ..utils.helpers import communicate


def parse_args(argv=None):
    parser = build_parser(adpsgd=False)
    parser.add_argument('--cuda_graph', default=False, type=common.str2bool, nargs='?', const=True,
                        help='capture forward+backward+gossip once and replay (fused path only)')
    parser.add_argument('--accumulation_steps', default=1, type=int,
                        help='gradient accumulation: K forward/backward passes of batch_size / K rows each per '
                             'step, their gradients summed in fp32 before the one gossip / SGD step '
                             '(GossipTrainer(accumulation_steps=K)); --batch_size stays the per-rank step batch '
                             'and must be divisible by K.  BatchNorm statistics are per micro-batch.  SGP / OSGP '
                             '/ D-PSGD with --cuda_graph True --fused True and --nprocs_per_node 1')
    parser.add_argument('--eval_graph', default=False, type=common.str2bool, nargs='?', const=True,
                        help='validate (and --model_ema_decay / --validate_average validation) through '
                             'GossipTrainer.evaluate: one captured eval graph per batch shape, BatchNorm in the '
                             '1x1-conv GEMM epilogue, loss and top-1 / top-5 counted on the device and read back '
                             'once per pass.  Needs the captured trainer (--cuda_graph True --fused True on '
                             'the CUDA kernel transport, not --all_reduce)')
    parser.add_argument('--precise_bn_batches', default=0, type=int,
                        help='precise BatchNorm statistics: before each validation (the rank model, the '
                             '--model_ema_decay EMA and the --validate_average average model) set every running '
                             'mean / variance to the average of the batch statistics of the next N training '
                             'batches (augmented, never mixed), through GossipTrainer.update_bn.  0 = off.  '
                             'Needs the captured trainer (--cuda_graph True --fused True on the CUDA kernel '
                             'transport, not --all_reduce)')
    args = parser.parse_args(argv)
    common.check_accumulation_flags(args)
    common.check_eval_graph_flags(args)
    common.check_precise_bn_flags(args)
    return finalize_args(args, adpsgd=False)


def build_model_and_optimizer(args, log):
    from ..optim import FusedGossipSGD, lars_groups, no_bias_decay_groups
    from ..parallel.distributed import GossipDataParallel
    net = init_model(args)
    if args.all_reduce:
        if args.device == 'cuda' and args.transport != 'c10d':
            from ..parallel.allreduce import AllReduceDataParallel
            model = AllReduceDataParallel(net, rank=args.rank, world_size=args.world_size)
            optimizer = _AROptimizer(model, args)
        else:
            model = torch.nn.parallel.DistributedDataParallel(net) if args.world_size > 1 else net
            optimizer = torch.optim.SGD(model.parameters(), lr=args.lr, momentum=args.momentum,
                                        weight_decay=args.weight_decay, nesterov=args.nesterov)
        return model, optimizer
    model = GossipDataParallel(
        net, graph=args.graph, mixing=args.mixing, comm_device=args.comm_device,
        push_sum=args.push_sum, overlap=args.overlap, synch_freq=args.synch_freq,
        verbose=args.verbose, use_streams=not args.no_cuda_streams, rank=args.rank,
        world_size=args.world_size, transport=args.transport, nprocs_per_node=args.nprocs_per_node,
        gossip_dtype=torch.bfloat16 if args.gossip_dtype == 'bf16' else None,
        slowmo_frequency=args.slowmo_frequency, slowmo_lr=args.slowmo_lr,
        slowmo_momentum=args.slowmo_momentum,
        # the captured fast path trains through the bf16 shadow-weight twin (no autocast casts)
        compute_dtype=(torch.bfloat16 if (args.cuda_graph and args.amp and args.fused
                                          and args.device == 'cuda' and args.transport != 'c10d')
                       else None))
    groups = None
    if args.no_bias_decay:
        groups = (lars_groups if args.lars else no_bias_decay_groups)(net, args.weight_decay)
    if args.fused:
        optimizer = FusedGossipSGD(model, lr=args.lr, momentum=args.momentum,
                                   weight_decay=args.weight_decay, nesterov=args.nesterov,
                                   param_groups=groups, lars=args.lars, trust_coefficient=args.lars_trust,
                                   max_grad_norm=args.clip_grad_norm if args.clip_grad_norm > 0 else None,
                                   skip_nonfinite=args.skip_nonfinite)
    else:
        optimizer = torch.optim.SGD(groups if groups is not None else model.parameters(), lr=args.lr,
                                    momentum=args.momentum, weight_decay=args.weight_decay,
                                    nesterov=args.nesterov)
    log.info('transport: %s, fused optimizer: %s' % (model.transport, args.fused))
    return model, optimizer


class _AROptimizer(object):
    """optimizer facade over AllReduceDataParallel's fused all-reduce+SGD kernel"""

    def __init__(self, model, args):
        self.model = model
        self.param_groups = [dict(lr=args.lr, momentum=args.momentum,
                                  weight_decay=args.weight_decay, nesterov=args.nesterov)]

    def step(self):
        g = self.param_groups[0]
        self.model.set_hyper(g['lr'], g['momentum'], g['weight_decay'], g['nesterov'])
        self.model.allreduce_step()

    def zero_grad(self, set_to_none=False):
        pass          # the step clears the (symmetric) gradient buffer

    def state_dict(self):
        return {'param_groups': self.param_groups, 'momentum': self.model.momentum.cpu()}

    def load_state_dict(self, sd):
        self.param_groups[0].update(sd['param_groups'][0])
        self.model.momentum.copy_(sd['momentum'])


def main(argv=None):
    args = parse_args(argv)
    log = make_logger(args.rank, args.verbose)
    log.info('args: {}'.format({k: v for k, v in vars(args).items()
                                if k not in ('graph', 'mixing')}))
    log.info(socket.gethostname())
    torch.manual_seed(args.seed)
    if args.device == 'cuda':
        torch.cuda.manual_seed(args.seed)
        torch.backends.cudnn.benchmark = True

    if args.trace_file:
        tracing.enable(args.trace_file, rank=args.rank)
    model, optimizer = build_model_and_optimizer(args, log)
    criterion = nn.CrossEntropyLoss()      # == KLDiv(log_softmax, one_hot) of the reference
    # the training loss carries --label_smoothing; validation keeps the plain cross-entropy so that
    # validation losses stay comparable across runs
    train_criterion = nn.CrossEntropyLoss(label_smoothing=args.label_smoothing)
    optimizer.zero_grad()
    # --mixup_alpha / --cutmix_alpha: training batches only (validate() never mixes)
    args._batch_mix = common.make_batch_mix(args)
    # --model_ema_decay: weight EMA, updated after every step (the last launch of the captured step)
    args._ema = common.make_model_ema(args, model)
    args._ema_due = False
    args._trainer = None
    if args.cuda_graph and not args.all_reduce and args.fused and getattr(model, '_kernel', None):
        from ..ops.fused_loss import FusedCrossEntropyWithAccuracy
        from ..parallel.trainer import GossipTrainer
        # the fused softmax-xent + prec@1/5 kernel, captured in the graph (same value as
        # nn.CrossEntropyLoss(label_smoothing=...); tests/test_fused_loss_gpu.py)
        args._trainer = GossipTrainer(model, optimizer,
                                      FusedCrossEntropyWithAccuracy(label_smoothing=args.label_smoothing),
                                      amp_dtype=torch.bfloat16 if args.amp else None,
                                      batch_mix=args._batch_mix, ema=args._ema,
                                      accumulation_steps=args.accumulation_steps)
    if args.eval_graph and args._trainer is None:
        raise ValueError('--eval_graph is not supported with transport %s: the captured evaluation is '
                         'GossipTrainer.evaluate, which runs on the CUDA kernel transport only'
                         % getattr(model, 'transport', 'c10d'))
    if args.precise_bn_batches > 0 and args._trainer is None:
        raise ValueError('--precise_bn_batches is not supported with transport %s: the statistics are recomputed '
                         'by GossipTrainer.update_bn, which runs on the CUDA kernel transport only'
                         % getattr(model, 'transport', 'c10d'))
    if args.accumulation_steps > 1 and args._trainer is None:
        raise ValueError('--accumulation_steps > 1 needs the captured GossipTrainer step, which runs on the '
                         'CUDA kernel transport only (got device %s, transport %s)' % (args.device, model.transport))

    state = fresh_state(model.state_dict(), optimizer.state_dict())
    if args._ema is not None:
        state['model_ema'] = args._ema.state_dict()
    common.save_stochastic_depth(state, model)
    cmanager = ClusterManager(rank=args.rank, world_size=args.world_size, model_tag=args.tag,
                              state=state, all_workers=args.checkpoint_all)
    if args.resume and os.path.isfile(cmanager.checkpoint_fpath):
        log.info("=> loading checkpoint '{}'".format(cmanager.checkpoint_fpath))
        ckpt = torch.load(cmanager.checkpoint_fpath, map_location='cpu', weights_only=False)
        update_state(state, {k: ckpt[k] for k in (
            'epoch', 'itr', 'best_prec1', 'state_dict', 'optimizer', 'elapsed_time',
            'batch_meter', 'data_meter', 'nn_meter')})
        state['is_best'] = False
        model.load_state_dict(ckpt['state_dict'])
        optimizer.load_state_dict(ckpt['optimizer'])
        if args._ema is not None:
            if 'model_ema' in ckpt:
                args._ema.load_state_dict(ckpt['model_ema'])
                state['model_ema'] = ckpt['model_ema']
            else:
                log.warning('checkpoint has no model_ema: the EMA starts again from the loaded model')
                args._ema.reset()
        common.load_stochastic_depth(ckpt, state, model, log)
        log.info("=> loaded checkpoint (epoch {}; itr {})".format(ckpt['epoch'], ckpt['itr']))
    elif args.resume:
        log.info("=> no checkpoint found at '{}'".format(cmanager.checkpoint_fpath))

    batch_meter = Meter(state['batch_meter'])
    data_meter = Meter(state['data_meter'])
    nn_meter = Meter(state['nn_meter'])
    csv = CSVLog(args.out_fname, args.world_size, args.num_dataloader_workers, args.batch_size)
    args._consensus_log = (ConsensusLog(args.consensus_fname)
                           if args.consensus_freq > 0 or args.validate_average else None)
    args._ema_log = common.EmaLog(args.ema_fname) if args._ema is not None else None

    loader, sampler = make_dataloader(args, train=True)
    val_loader = None if args.train_fast else make_dataloader(args, train=False)

    start_itr, start_epoch = state['itr'], state['epoch']
    elapsed_time = state['elapsed_time']
    begin_time = time.time() - elapsed_time
    best_val_prec1 = state.get('best_prec1', 0)
    for epoch in range(start_epoch, args.num_epochs):
        sampler.set_epoch(epoch + args.seed * 90)
        if not args.all_reduce:
            update_peers_per_itr(args, model, epoch)
            model.block()
        train(args, model, train_criterion, optimizer, batch_meter, data_meter, nn_meter, loader,
              epoch, start_itr, csv, log)
        start_itr = 0
        if not args.train_fast:
            precise_bn(args, loader, log)          # (before the state is taken: checkpointed that way)
            elapsed_time = time.time() - begin_time
            update_state(state, {
                'epoch': epoch + 1, 'itr': 0, 'is_best': False,
                'state_dict': model.state_dict(), 'optimizer': optimizer.state_dict(),
                'elapsed_time': elapsed_time, 'batch_meter': batch_meter.__dict__,
                'data_meter': data_meter.__dict__, 'nn_meter': nn_meter.__dict__})
            if args._ema is not None:
                state['model_ema'] = args._ema.state_dict()
            common.save_stochastic_depth(state, model)
            prec1 = validate(args, val_loader, model, criterion, log)
            csv.val_row(epoch, batch_meter, nn_meter, data_meter, prec1)
            if args._ema is not None:
                validate_ema(args, val_loader, model, criterion, log, epoch, loader)
            if prec1 > best_val_prec1:
                update_state(state, {'is_best': True, 'best_prec1': prec1})
                best_val_prec1 = prec1
        if args._consensus_log is not None:
            epoch_end_consensus(args, model, criterion, val_loader, epoch, log, loader)
        if not args.train_fast:
            epoch_id = None if args.overwrite_checkpoints else epoch
            cmanager.save_checkpoint(epoch_id, requeue_on_signal=(epoch != args.num_epochs - 1))

    if args.train_fast:
        val_loader = make_dataloader(args, train=False)
        precise_bn(args, loader, log)
        prec1 = validate(args, val_loader, model, criterion, log)
        log.info('Test accuracy: {}'.format(prec1))
        if args._ema is not None:
            validate_ema(args, val_loader, model, criterion, log, args.num_epochs - 1, loader)
    log.info('elapsed_time {0}'.format(time.time() - begin_time))
    if tracing.get_tracer().enabled:            # shorter run than --trace_iters
        log.info('trace written to %s' % tracing.disable().dump())
    if dist.is_initialized():
        dist.barrier()
    return state


def _autocast(args):
    return torch.autocast('cuda', dtype=torch.bfloat16, enabled=bool(args.amp and args.device == 'cuda'))


def _drain_metrics(trainer, pending):
    """[loss, prec@1, prec@5] of every pending iteration with one synchronisation.  Graph path:
    the rows already sit in the trainer's pinned ring (slots); eager path: device tensors.
    Also the place where the gossip kernels' health word is polled (a peer that stopped
    publishing raises here, like the reference's 'Gossip flag timeout')."""
    if trainer is not None:
        trainer.stream.synchronize()
        trainer.check()
        return [trainer.metrics_ring[slot].tolist() for slot, _ in pending]
    return torch.stack([v for v, _ in pending]).cpu().tolist()


def train(args, model, criterion, optimizer, batch_meter, data_meter, nn_meter, loader, epoch,
          itr, csv, log):
    losses, top1, top5 = Meter(ptag='Loss'), Meter(ptag='Prec@1'), Meter(ptag='Prec@5')
    model.train()
    dev = args.device
    ignore = getattr(args, 'num_itr_ignore', 0) if epoch == 0 else 0
    limit = getattr(args, 'num_iterations_per_training_epoch', None)
    # device-side metric accumulators: [loss, prec1, prec5] per iteration, read
    # back once per print interval (the reference syncs 3x per iteration)
    pending = []
    trainer = getattr(args, '_trainer', None)
    batch_mix = getattr(args, '_batch_mix', None)
    ema = getattr(args, '_ema', None) if trainer is None else None    # (the trainer updates its own)
    it = iter(loader)
    for _ in range(itr):            # resume mid-epoch: skip what was already consumed
        next(it, None)
    t_batch = time.time()
    traced = 0
    for i, (batch, target) in enumerate(it, start=itr):
        if tracing.get_tracer().enabled:
            traced += 1
            if traced > args.trace_iters:       # bounded trace: dump once, then stop recording
                log.info('trace written to %s' % tracing.disable().dump())
        target = target.to(dev, non_blocking=True)
        batch = common.device_batch(args, batch, train=True)       # (uint8 shard batches only)
        if dev == 'cuda' and not batch.is_cuda and args.all_reduce:
            batch = batch.to(dev, non_blocking=True)
        t_data = time.time() - t_batch
        tracing.counter('data_ms', t_data * 1e3)
        t_nn = time.time()
        # the step policy changes the rate at most every 100 iterations (as the reference sets it);
        # poly decays it every iteration (a device-resident value: no graph re-capture)
        if i % 100 == 0 or args.lr_policy == 'poly':
            update_learning_rate(args, optimizer, epoch, itr=i, itr_per_epoch=len(loader))
        mix = None
        if batch_mix is not None:               # this iteration's draw: resumes reproduce it
            if trainer is not None:
                batch_mix.iteration = epoch * len(loader) + i
            else:
                batch, mix = common.mix_train_batch(args, batch_mix, batch, epoch * len(loader) + i)
        if trainer is not None:
            # whole step = one CUDA-graph replay (forward+backward+fused gossip kernel);
            # the metrics are computed on the trainer's stream, before the next replay
            # can overwrite the static output buffers
            # (loss, prec@1, prec@5 come out of the fused loss kernel inside the graph and land
            # in the trainer's pinned metrics ring: 12 bytes per step, no host sync)
            with tracing.span('step[graph]', itr=i):
                slot = trainer.step(batch, target)
            pending.append((slot, batch.size(0)))
        else:
            with tracing.span('forward', itr=i), _autocast(args):
                output = model(batch)
                loss = common.train_loss(criterion, output, target, mix, args.label_smoothing)
            if ema is not None and args._ema_due:
                # c10d plane: the previous step's gossip was received and de-biased by the forward
                # pre-hook just now; the EMA takes those parameters (and this forward's BN statistics)
                ema.update()
                args._ema_due = False
            with tracing.span('backward'):
                loss.backward()
            with tracing.span('optimizer'):
                optimizer.step()
                optimizer.zero_grad()
            if not args.overlap and not args.all_reduce:
                model.transfer_params()
            if getattr(args, 'slowmo_frequency', 0):
                model.perform_slowmo(optimizer)        # (the trainer path runs it inside step())
            if ema is not None:
                if getattr(model, 'is_ps_numerator', False):
                    args._ema_due = True               # gossip in flight: after the next forward pre-hook
                else:
                    ema.update()
            with torch.no_grad():
                p1, p5 = accuracy(output, target, topk=(1, 5))
                pending.append((torch.stack([loss.detach().float().reshape(()), p1[0], p5[0]]),
                                batch.size(0)))
        t_nn = time.time() - t_nn
        if ignore == 0:
            data_meter.update(t_data)
            nn_meter.update(t_nn)
            batch_meter.update(time.time() - t_batch)
        else:
            ignore -= 1
        t_batch = time.time()

        last = (limit not in (None, -1) and i + 1 == limit)
        if i % args.print_freq == 0 or last or len(pending) >= 512:
            vals = _drain_metrics(trainer, pending)                # ONE sync per interval
            for (l, a1, a5), (_, n) in zip(vals, pending):
                losses.update(l, n)
                top1.update(a1, n)
                top5.update(a5, n)
            pending = []
            csv.train_row(epoch, i, batch_meter, nn_meter, data_meter, losses, top1, top5)
        if getattr(args, '_consensus_log', None) is not None and args.consensus_freq > 0 \
                and (i + 1) % args.consensus_freq == 0:
            if trainer is not None:
                trainer.finish()            # (Overlap-SGP: the trainer holds the pending residual)
            log_consensus(args, model.consensus_distance(), epoch, i, log)
            t_batch = time.time()           # (not charged to the next iteration's data time)
        if last:
            break
    if trainer is not None:
        # end of epoch: land the deferred SGD / gathered residual (overlap) so that validation
        # and state_dict() see every update; eval / checkpointing run on the default stream
        trainer.finish()
    if pending:
        vals = _drain_metrics(trainer, pending)
        for (l, a1, a5), (_, n) in zip(vals, pending):
            losses.update(l, n)
            top1.update(a1, n)
            top5.update(a5, n)
    csv.train_row(epoch, i, batch_meter, nn_meter, data_meter, losses, top1, top5)
    k = getattr(args, 'accumulation_steps', 1)
    if k > 1:
        log.info('epoch {} gradient accumulation: {} micro-batches of {} rows per step of {} rows'.format(
            epoch, k, args.batch_size // k, args.batch_size))
    grad_norm = getattr(optimizer, 'grad_norm', None)       # (--clip_grad_norm / --skip_nonfinite)
    if grad_norm is not None:
        log.info('epoch {} last gradient norm {:.6e} non-finite steps skipped {}'.format(
            epoch, float(grad_norm), optimizer.nonfinite_steps))
    return losses.avg


def log_consensus(args, stats, epoch, itr, log, avg_prec1=None):
    log.info('consensus epoch {} itr {}: distance_sq {:.6e} average_norm_sq {:.6e} relative {:.6e}{}'.format(
        epoch, itr, stats.distance_sq, stats.average_norm_sq, stats.relative,
        '' if avg_prec1 is None else ' average-model Prec@1 {:.3f}'.format(avg_prec1)))
    args._consensus_log.row(epoch, itr, stats, avg_prec1)


def precise_bn(args, loader, log, label=''):
    """--precise_bn_batches N > 0: recompute the BatchNorm running statistics of the model the trainer
    runs now from the next N training batches (``GossipTrainer.update_bn``).  The batches come from a
    fresh iterator over ``loader``, closed afterwards (a shard loader's gather thread ends), and carry
    the training augmentation but are never mixed; they consume draws of the augmentation generator."""
    n = getattr(args, 'precise_bn_batches', 0)
    if n <= 0 or loader is None:
        return
    it = iter(loader)
    try:
        k = args._trainer.update_bn((common.device_batch(args, features, train=True), target)
                                    for features, target in itertools.islice(it, n))
    finally:
        close = getattr(it, 'close', None)
        if close is not None:
            close()
    log.info('precise BN: {}statistics from {} training batches'.format(label, k))


def epoch_end_consensus(args, model, criterion, val_loader, epoch, log, loader=None):
    """Consensus distance at the end of an epoch; with ``--validate_average`` also the validation
    accuracy of the push-sum average model.  BatchNorm running statistics are not gossiped: for
    that validation they are averaged over the ranks, and restored afterwards.  With
    --precise_bn_batches each rank first recomputes them for the average model from ``loader``."""
    trainer = getattr(args, '_trainer', None)
    if trainer is not None:
        trainer.finish()
    if not (args.validate_average and val_loader is not None):
        log_consensus(args, model.consensus_distance(), epoch, -1, log)
        return
    bufs = [b for b in model.module.buffers() if b.is_floating_point()]
    saved = [b.detach().clone() for b in bufs]

    def average_buffers():
        if args.world_size > 1 and bufs:
            with torch.no_grad():
                communicate(bufs, dist.all_reduce)
                for b in bufs:
                    b.div_(args.world_size)

    precise = getattr(args, 'precise_bn_batches', 0) > 0 and loader is not None
    if not precise:
        average_buffers()
    try:
        with model.averaged() as stats:
            if precise:
                precise_bn(args, loader, log, label='average-model ')
                average_buffers()
            prec1 = validate(args, val_loader, model, criterion, log)
    finally:
        with torch.no_grad():
            for b, s in zip(bufs, saved):
                b.copy_(s)
    log_consensus(args, stats, epoch, -1, log, avg_prec1=prec1)


def validate_ema(args, val_loader, model, criterion, log, epoch, loader=None):
    """Validate the EMA weights and BatchNorm statistics (``ModelEma.applied``, restored afterwards)
    and log their prec@1 / prec@5 to stdout and the EMA CSV.  With --precise_bn_batches the
    statistics are first recomputed for the EMA weights from ``loader``."""
    ema = args._ema
    with ema.applied():
        precise_bn(args, loader, log, label='EMA ')
        prec1, prec5 = evaluate(args, val_loader, model, criterion, log, label='EMA ')
    args._ema_log.row(epoch, ema.num_updates, prec1, prec5)
    return prec1


def validate(args, val_loader, model, criterion, log):
    return evaluate(args, val_loader, model, criterion, log)[0]


def evaluate(args, val_loader, model, criterion, log, label=''):
    """(prec@1, prec@5) over the validation set, logged as `` * <label>Prec@1 .. Prec@5 ..``;
    with --eval_graph through the trainer's captured evaluation"""
    trainer = getattr(args, '_trainer', None)
    if getattr(args, 'eval_graph', False) and trainer is not None:
        r = trainer.evaluate((common.device_batch(args, features, train=False), target)
                             for features, target in val_loader)
        log.info(' * {label}Prec@1 {p1:.3f} Prec@5 {p5:.3f}'.format(label=label, p1=r.prec1, p5=r.prec5))
        return r.prec1, r.prec5
    losses, top1, top5 = Meter(ptag='Loss'), Meter(ptag='Prec@1'), Meter(ptag='Prec@5')
    model.eval()
    dev = args.device
    with torch.no_grad():
        for features, target in val_loader:
            target = target.to(dev, non_blocking=True)
            features = common.device_batch(args, features, train=False).to(dev, non_blocking=True)
            if args.channels_last and dev == 'cuda':
                features = features.contiguous(memory_format=torch.channels_last)
            with _autocast(args):
                output = model(features)
                loss = criterion(output.float(), target)
            p1, p5 = accuracy(output, target, topk=(1, 5))
            n = features.size(0)
            losses.update(loss.item(), n)
            top1.update(p1.item(), n)
            top5.update(p5.item(), n)
    log.info(' * {label}Prec@1 {top1.avg:.3f} Prec@5 {top5.avg:.3f}'.format(label=label, top1=top1, top5=top5))
    return top1.avg, top5.avg


if __name__ == '__main__':
    main()
