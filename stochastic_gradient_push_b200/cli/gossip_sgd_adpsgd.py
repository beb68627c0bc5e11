"""
ResNet / ImageNet trainer for AD-PSGD (asynchronous bilateral gossip).

Functional parity with the reference's ``gossip_sgd_adpsgd.py``: wraps the
model in ``BilatGossipDataParallel`` (:166-177), trains with a *global*
iteration counter shared through a file on a common filesystem (every rank
appends one byte per iteration and reads the file size,
``update_global_iteration_counter`` :509-523), derives the epoch and the
learning rate of BOTH optimizers (the train-side one and the gossip-side one,
``update_bilat_learning_rate`` :478-506) from it, and stops when the global
epoch reaches ``--num_epochs`` (:267-309).

Differences: one control-plane process group is enough (the reference needs
``master_port`` and ``master_port+1`` because its gossip *process* owns a second
world); on the kernel data plane the gossip loop is a native (GIL-free) daemon thread
enqueueing a device-side round state machine on a lowest-priority stream of the same
GPU, on the c10d data plane a Python thread over isend / irecv (see
``parallel/ad_psgd.py``).
"""

from __future__ import annotations

import os
import socket
import time

import torch
import torch.distributed as dist
import torch.nn as nn

from .common import (CSVLog, Meter, accuracy, build_parser, finalize_args, fresh_state,
                     init_model, learning_rate_at, load_stochastic_depth, make_dataloader,
                     save_stochastic_depth, update_state)
from ..experiment import ClusterManager, make_logger
from ..utils import tracing
from .common import device_batch, make_batch_mix, mix_train_batch, train_loss


def parse_args(argv=None):
    parser = build_parser(adpsgd=True)
    parser.set_defaults(graph_type=1)       # shipped job script: bipartite exponential
    args = parser.parse_args(argv)
    args = finalize_args(args, adpsgd=True)
    if not args.shared_fpath:
        args.shared_fpath = os.path.join(args.checkpoint_dir, args.tag + 'global_itr.txt')
    return args


def update_global_iteration_counter(args, itr):
    """Append ``itr`` bytes to the shared file and return the global iteration
    count (= file size) -- a lock-free counter on any POSIX shared FS."""
    with open(args.shared_fpath, 'ab') as f:
        f.write(b'-' * int(itr))
        f.flush()
    return os.stat(args.shared_fpath).st_size


def global_epoch_of(args, global_itr, itr_per_epoch):
    return global_itr // (itr_per_epoch * args.world_size), \
        (global_itr // args.world_size) % itr_per_epoch


def update_bilat_learning_rate(args, model, optimizer, global_itr, itr_per_epoch):
    """One LR for the local optimizer and the gossip-side fused SGD."""
    epoch, itr = global_epoch_of(args, global_itr, itr_per_epoch)
    lr = learning_rate_at(args, epoch, itr, itr_per_epoch)
    for g in optimizer.param_groups:
        g['lr'] = lr
    model.update_lr(lr)
    return lr


def main(argv=None):
    from ..parallel.ad_psgd import BilatGossipDataParallel
    args = parse_args(argv)
    log = make_logger(args.rank, args.verbose)
    log.info(socket.gethostname())
    torch.manual_seed(args.seed)
    if args.device == 'cuda':
        torch.cuda.manual_seed(args.seed)
        torch.backends.cudnn.benchmark = True

    if args.trace_file:
        tracing.enable(args.trace_file, rank=args.rank)
    net = init_model(args)
    model = BilatGossipDataParallel(
        net, master_addr=args.master_addr, master_port=str(args.master_port),
        backend=args.backend, world_size=args.world_size, rank=args.rank,
        graph_class=args.graph_class, mixing_class=args.mixing_class,
        num_peers=args.ppi_schedule[0], comm_device=args.comm_device, lr=args.lr,
        momentum=args.momentum, weight_decay=args.weight_decay, nesterov=args.nesterov,
        verbose=args.verbose, network_interface_type=args.network_interface_type,
        transport=args.transport)
    criterion = nn.CrossEntropyLoss()
    # --label_smoothing applies to the training loss; validation keeps the plain cross-entropy
    train_criterion = nn.CrossEntropyLoss(label_smoothing=args.label_smoothing)
    optimizer = torch.optim.SGD(model.parameters(), lr=args.lr, momentum=args.momentum,
                                weight_decay=args.weight_decay, nesterov=args.nesterov)
    optimizer.zero_grad(set_to_none=False)
    # --mixup_alpha / --cutmix_alpha: training batches only (validate() never mixes)
    args._batch_mix = make_batch_mix(args)

    state = fresh_state(model.state_dict(), optimizer.state_dict())
    save_stochastic_depth(state, model)
    cmanager = ClusterManager(rank=args.rank, world_size=args.world_size, model_tag=args.tag,
                              state=state, all_workers=args.checkpoint_all)
    if args.resume and os.path.isfile(cmanager.checkpoint_fpath):
        ckpt = torch.load(cmanager.checkpoint_fpath, map_location='cpu', weights_only=False)
        update_state(state, {k: ckpt[k] for k in ckpt})
        model.load_state_dict(ckpt['state_dict'])
        optimizer.load_state_dict(ckpt['optimizer'])
        model.gossip_flat.copy_(model.arena.flat)
        load_stochastic_depth(ckpt, state, model, log)
    if args.rank == 0 and not args.resume and os.path.exists(args.shared_fpath):
        os.remove(args.shared_fpath)
    if dist.is_initialized():
        dist.barrier()

    batch_meter, data_meter, nn_meter = (Meter(state['batch_meter']), Meter(state['data_meter']),
                                         Meter(state['nn_meter']))
    csv = CSVLog(args.out_fname, args.world_size, args.num_dataloader_workers, args.batch_size)
    loader, sampler = make_dataloader(args, train=True)
    val_loader = None if args.train_fast else make_dataloader(args, train=False)
    itr_per_epoch = len(loader)
    begin_time = time.time() - state['elapsed_time']
    global_itr = update_global_iteration_counter(args, 0)
    global_epoch, _ = global_epoch_of(args, global_itr, itr_per_epoch)
    local_epoch = 0
    best = 0
    while global_epoch < args.num_epochs:
        sampler.set_epoch(local_epoch + args.seed * 90)
        global_itr = train(args, model, train_criterion, optimizer, batch_meter, data_meter, nn_meter,
                           loader, local_epoch, csv, log, itr_per_epoch)
        global_epoch, _ = global_epoch_of(args, global_itr, itr_per_epoch)
        local_epoch += 1
        if not args.train_fast:
            update_state(state, {
                'epoch': local_epoch, 'itr': 0, 'is_best': False,
                'state_dict': model.state_dict(), 'optimizer': optimizer.state_dict(),
                'elapsed_time': time.time() - begin_time, 'batch_meter': batch_meter.__dict__,
                'data_meter': data_meter.__dict__, 'nn_meter': nn_meter.__dict__})
            save_stochastic_depth(state, model)
            prec1 = validate(args, val_loader, model, criterion, log)
            csv.val_row(local_epoch - 1, batch_meter, nn_meter, data_meter, prec1)
            if prec1 > best:
                update_state(state, {'is_best': True, 'best_prec1': prec1})
                best = prec1
            cmanager.save_checkpoint(None, requeue_on_signal=(global_epoch < args.num_epochs))
    if args.train_fast:
        prec1 = validate(args, make_dataloader(args, train=False), model, criterion, log)
        log.info('Test accuracy: {}'.format(prec1))
    model.disable_gossip()
    log.info('elapsed_time {0}'.format(time.time() - begin_time))
    if tracing.get_tracer().enabled:
        log.info('trace written to %s' % tracing.disable().dump())
    if dist.is_initialized():
        dist.barrier()
    model.shutdown()
    return state


def train(args, model, criterion, optimizer, batch_meter, data_meter, nn_meter, loader, epoch,
          csv, log, itr_per_epoch):
    losses, top1, top5 = Meter(ptag='Loss'), Meter(ptag='Prec@1'), Meter(ptag='Prec@5')
    model.train()
    model.enable_gossip()
    dev = args.device
    amp = bool(args.amp and dev == 'cuda')
    batch_mix = getattr(args, '_batch_mix', None)
    global_itr = update_global_iteration_counter(args, 0)
    since_sync = 0
    t_batch = time.time()
    i = 0
    for i, (batch, target) in enumerate(loader):
        target = target.to(dev, non_blocking=True)
        batch = device_batch(args, batch, train=True)              # (uint8 shard batches only)
        t_data = time.time() - t_batch
        t_nn = time.time()
        if tracing.get_tracer().enabled and i >= args.trace_iters:
            log.info('trace written to %s' % tracing.disable().dump())
        mix = None
        if batch_mix is not None:            # keyed by this rank's own iteration count
            batch, mix = mix_train_batch(args, batch_mix, batch, epoch * itr_per_epoch + i)
        with tracing.span('forward', itr=i), torch.autocast('cuda', dtype=torch.bfloat16, enabled=amp):
            output = model(batch)
            loss = train_loss(criterion, output, target, mix, args.label_smoothing)
        with tracing.span('backward+exchange'):
            loss.backward()      # end-of-backward hook: push grads, pull the gossip model
        with tracing.span('optimizer'):
            optimizer.step()     # local step on the train copy (overwritten by the next pull)
            optimizer.zero_grad(set_to_none=False)
        since_sync += 1
        # every 100 iterations, staggered by rank, publish progress and refresh the LR
        if (i + args.rank) % 100 == 0:
            global_itr = update_global_iteration_counter(args, since_sync)
            since_sync = 0
            update_bilat_learning_rate(args, model, optimizer, global_itr, itr_per_epoch)
        t_nn = time.time() - t_nn
        data_meter.update(t_data)
        nn_meter.update(t_nn)
        batch_meter.update(time.time() - t_batch)
        t_batch = time.time()
        if i % args.print_freq == 0:
            p1, p5 = accuracy(output, target, topk=(1, 5))
            n = batch.size(0)
            losses.update(loss.item(), n)
            top1.update(p1.item(), n)
            top5.update(p5.item(), n)
            csv.train_row(epoch, i, batch_meter, nn_meter, data_meter, losses, top1, top5)
        g_epoch, _ = global_epoch_of(args, global_itr, itr_per_epoch)
        if g_epoch >= args.num_epochs:
            break
    global_itr = update_global_iteration_counter(args, since_sync)
    csv.train_row(epoch, i, batch_meter, nn_meter, data_meter, losses, top1, top5)
    return global_itr


def validate(args, val_loader, model, criterion, log):
    losses, top1, top5 = Meter(ptag='Loss'), Meter(ptag='Prec@1'), Meter(ptag='Prec@5')
    model.eval()                 # pulls the latest gossip model
    model.disable_gossip()
    dev = args.device
    with torch.no_grad():
        for features, target in val_loader:
            target = target.to(dev, non_blocking=True)
            features = device_batch(args, features, train=False)
            with torch.autocast('cuda', dtype=torch.bfloat16,
                                enabled=bool(args.amp and dev == 'cuda')):
                output = model(features)
                loss = criterion(output.float(), target)
            p1, p5 = accuracy(output, target, topk=(1, 5))
            n = features.size(0)
            losses.update(loss.item(), n)
            top1.update(p1.item(), n)
            top5.update(p5.item(), n)
    log.info(' * Prec@1 {top1.avg:.3f} Prec@5 {top5.avg:.3f}'.format(top1=top1, top5=top5))
    return top1.avg


if __name__ == '__main__':
    main()
