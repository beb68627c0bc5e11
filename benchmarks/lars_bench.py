"""LARS vs the same parameter groups without it (``FusedGossipSGD(lars=True)``, ``SGP_F_LARS``):
time of the fused SGD + gossip kernels at ResNet-50 size, N virtual ranks on ONE GPU (``LocalWorld``
loop-back), one host thread per rank.

    python benchmarks/lars_bench.py [--ranks 4] [--launches 200] [--block 25] [--out F.json]

Three measurements:
  (a) the norm + trust kernels alone (``GossipContext.lars_update``) on one rank, in ms and in GB/s
      of the bytes they must move, computed from the shapes;
  (b) the full synchronous step (``GossipEngine.mix(sgd=True)``) with ``lars_groups`` -- LARS on the
      weights, neither decay nor LARS on BatchNorm parameters and biases -- against the same two
      groups without LARS;
  (c) the Overlap-SGP pair ``publish(sgd=True, fold=True)`` + ``gather()``, the same two arms.
Device-timed with CUDA events per rank stream (max over ranks); the arms alternate in blocks of
``--block`` launches until each has ``--launches``.  Loop-back reads the peers' outboxes from local
HBM, so this measures the kernels' own cost, not NVLink.
"""
import argparse
import functools
import json
import os
import subprocess
import sys
import threading

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stochastic_gradient_push_b200 as sgp                                # noqa: E402
from stochastic_gradient_push_b200.models import resnet50                  # noqa: E402
from stochastic_gradient_push_b200.ops.peer_mix import GossipEngine        # noqa: E402
from stochastic_gradient_push_b200.optim import lars_groups                # noqa: E402
from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld    # noqa: E402
from stochastic_gradient_push_b200.utils.arena import ALIGN_ELEMS          # noqa: E402

HYPER = (0.1, 0.9, 1e-4, True)
GROUP_ROWS = [(0.1, 0.9, 0.0, True), (0.1, 0.9, 1e-4, True)]


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader',
                              '-i', '0'], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30)
        power = out.stdout.strip()
    except Exception as e:                          # noqa
        power = 'unknown (%s)' % e
    return name, power


def _in_threads(fns):
    errors = []

    def run(fn):
        try:
            fn()
        except BaseException as e:                  # noqa
            errors.append(e)
    threads = [threading.Thread(target=run, args=(fn,)) for fn in fns]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if errors:
        raise errors[0]


def _resnet50_layout(chunk):
    """arena length, block map, tensor offsets / numels and LARS flags of ResNet-50's lars_groups
    (the FlatArena layout)"""
    net = resnet50()
    small = set(id(p) for p in lars_groups(net, 1e-4)[0]['params'])
    offs, numels, groups, off = [], [], [], 0
    for p in net.parameters():
        offs.append(off)
        numels.append(p.numel())
        groups.append(0 if id(p) in small else 1)
        off = (off + p.numel() + ALIGN_ELEMS - 1) // ALIGN_ELEMS * ALIGN_ELEMS
    numel = (off + chunk - 1) // chunk * chunk
    bmap = torch.zeros(numel // 64, dtype=torch.uint8)
    for o, n, g in zip(offs, numels, groups):
        bmap[o // 64: (o + n + 63) // 64] = g
    return dict(numel=numel, bmap=bmap, offsets=offs, numels=numels, lars=[g == 1 for g in groups])


def _arm(n_ranks, layout, lars, overlap, name):
    dev = torch.device('cuda', 0)
    lw = LocalWorld(n_ranks)
    numel = layout['numel']
    ranks = []
    for r in range(n_ranks):
        g = sgp.NPeerDynamicDirectedExponentialGraph(r, n_ranks, peers_per_itr=1)
        e = GossipEngine(lw.view(r), torch.randn(numel, device=dev) * 0.05, g, sgp.UniformMixing(g, dev),
                         grad=torch.randn(numel, device=dev) * 1e-3, momentum=torch.zeros(numel, device=dev),
                         timeout_s=60.0, name=name, with_residual=overlap)
        e.set_param_groups(layout['bmap'].to(dev), len(GROUP_ROWS))
        if lars:
            e.set_lars(layout['offsets'], layout['numels'], layout['lars'])
        e.set_hyper(*HYPER, groups=GROUP_ROWS)
        ranks.append((e, torch.cuda.Stream(device=dev)))
    return ranks


def _norms_alone(layout, launches, warmup):
    """(a): the two LARS kernels on one engine; bytes from the shapes: x and g (fp32) of every tensor
    element, the fp64 tile partials written and read back, and the per-tensor outputs"""
    ranks = _arm(1, layout, True, False, 'lars_alone')
    e, s = ranks[0]
    ntiles, T = e.ctx.lars_tiles(), len(layout['numels'])
    nbytes = 8 * sum(layout['numels']) + 2 * 16 * ntiles + 16 * ntiles + T * (8 + 4 + 1 + 16 + 4)
    with torch.cuda.stream(s):
        for _ in range(warmup):
            e.ctx.lars_update()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        for _ in range(launches):
            e.ctx.lars_update()
        b.record(s)
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / launches
    return {'ms': round(ms, 4), 'bytes': nbytes, 'GB_per_s': round(nbytes / ms / 1e6, 1),
            'tiles': ntiles, 'tensors': T, 'norm_grid': e.ctx.lars_grid()}


def _launch(e, overlap):
    if overlap:
        e.publish(sgd=True, fold=True, zero_grad=False)
        e.gather()
    else:
        e.mix(sgd=True, zero_grad=False)


def _block(ranks, k, overlap):
    """k steps per rank, each rank from its own thread on its own stream -> ms per step"""
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in ranks]

    def run(i):
        e, s = ranks[i]
        with torch.cuda.stream(s):
            evs[i][0].record(s)
            for _ in range(k):
                _launch(e, overlap)
            evs[i][1].record(s)
    _in_threads([functools.partial(run, i) for i in range(len(ranks))])
    torch.cuda.synchronize()
    for e, _ in ranks:
        e.check()
    return max(a.elapsed_time(b) for a, b in evs) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ranks', type=int, default=4)
    ap.add_argument('--launches', type=int, default=200, help='timed steps per arm and workload')
    ap.add_argument('--block', type=int, default=25)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'

    from stochastic_gradient_push_b200.ops import native
    C = native.load()
    layout = _resnet50_layout(C.CHUNK)
    card, power = _card()
    result = {'card': card, 'power_limit,max_sm_clock': power, 'ranks': args.ranks,
              'params': sum(layout['numels']), 'numel': layout['numel'],
              'lars_tensors': sum(layout['lars']), 'launches_per_arm': args.launches,
              'note': 'loop-back on one GPU: in-neighbour messages are read from local HBM, not NVLink'}
    result['norms_and_trust_alone'] = _norms_alone(layout, args.launches, args.warmup)
    torch.cuda.synchronize()
    for workload, overlap in (('full_step', False), ('overlap_publish_gather', True)):
        arms = {'groups': _arm(args.ranks, layout, False, overlap, 'lars0_' + workload),
                'lars': _arm(args.ranks, layout, True, overlap, 'lars1_' + workload)}
        # all ranks' step kernels must be co-resident on the one GPU: split the grid between them
        grid = max(1, arms['groups'][0][0].max_grid // args.ranks)
        for label in arms:
            for e, _ in arms[label]:
                e.grid = grid
                e.gather_grid = min(e.gather_grid, grid)
            _block(arms[label], args.warmup, overlap)
        times = {label: [] for label in arms}
        done = 0
        while done < args.launches:
            k = min(args.block, args.launches - done)
            for label in arms:                      # alternate the arms
                times[label].append((_block(arms[label], k, overlap), k))
            done += k
        res = {'grid_per_rank': grid}
        for label in arms:
            ms = sum(t * k for t, k in times[label]) / sum(k for _, k in times[label])
            blocks = sorted(t for t, _ in times[label])
            res[label] = {'ms_per_step': round(ms, 4), 'block_ms_min': round(blocks[0], 4),
                          'block_ms_max': round(blocks[-1], 4)}
        res['lars_over_groups_time'] = round(res['lars']['ms_per_step'] / res['groups']['ms_per_step'], 4)
        result[workload] = res
        del arms
        torch.cuda.synchronize()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
