"""fp32 vs bf16 gossip messages: time of the fused SGP step (``GossipEngine.mix(sgd=True)``) at
ResNet-50 size, N virtual ranks on ONE GPU (``LocalWorld`` loop-back), one host thread per rank.

    python benchmarks/gossip_dtype_bench.py [--ranks 4] [--launches 200] [--block 25] [--out F.json]

Loop-back pulls read the peers' outboxes from local HBM, not over NVLink, so this is a
kernel-efficiency check of the bf16 path; the gain on NVLink or on a network between hosts is
NOT measured here.  Device-timed with CUDA events per rank stream (max over ranks); the two arms
alternate in blocks of ``--block`` launches until each has ``--launches``.
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
from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld    # noqa: E402


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


def _arm(n_ranks, numel, msg_dtype, grid, name):
    dev = torch.device('cuda', 0)
    lw = LocalWorld(n_ranks)
    ranks = []
    for r in range(n_ranks):
        g = sgp.NPeerDynamicDirectedExponentialGraph(r, n_ranks, peers_per_itr=1)
        e = GossipEngine(lw.view(r), torch.randn(numel, device=dev) * 0.05, g, sgp.UniformMixing(g, dev),
                         grad=torch.randn(numel, device=dev) * 1e-3, momentum=torch.zeros(numel, device=dev),
                         grid=grid, timeout_s=60.0, name=name, msg_dtype=msg_dtype)
        e.set_hyper(0.1, 0.9, 1e-4, True)
        ranks.append((e, torch.cuda.Stream(device=dev)))
    return ranks


def _block(ranks, k):
    """k launches per rank, each rank from its own thread on its own stream -> ms per launch"""
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in ranks]

    def run(i):
        e, s = ranks[i]
        with torch.cuda.stream(s):
            evs[i][0].record(s)
            for _ in range(k):
                e.mix(sgd=True, zero_grad=False)
            evs[i][1].record(s)
    _in_threads([functools.partial(run, i) for i in range(len(ranks))])
    torch.cuda.synchronize()
    for e, _ in ranks:
        e.check()
    return max(a.elapsed_time(b) for a, b in evs) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ranks', type=int, default=4)
    ap.add_argument('--launches', type=int, default=200, help='timed launches per arm (>= 200)')
    ap.add_argument('--block', type=int, default=25)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'

    from stochastic_gradient_push_b200.ops import native
    C = native.load()
    n_params = sum(p.numel() for p in resnet50().parameters())
    numel = (n_params + C.CHUNK - 1) // C.CHUNK * C.CHUNK
    card, power = _card()
    arms = {}
    for label, dt in (('fp32', None), ('bf16', torch.bfloat16)):
        arms[label] = _arm(args.ranks, numel, dt, None, 'bench_' + label)
    # all ranks' step kernels must be co-resident on the one GPU: split the grid between them
    grid = max(1, arms['fp32'][0][0].max_grid // args.ranks)
    for label in arms:
        for e, _ in arms[label]:
            e.grid = grid
    for label in arms:
        _block(arms[label], args.warmup)
    times = {label: [] for label in arms}
    done = 0
    while done < args.launches:
        k = min(args.block, args.launches - done)
        for label in arms:                          # alternate the arms
            times[label].append((_block(arms[label], k), k))
        done += k

    n_in = 1
    result = {'card': card, 'power_limit,max_sm_clock': power, 'ranks': args.ranks, 'grid_per_rank': grid,
              'params': n_params, 'numel': numel, 'launches_per_arm': args.launches,
              'note': 'loop-back on one GPU: in-neighbour messages are read from local HBM, not NVLink; '
                      'a kernel-efficiency check, not the multi-GPU gain (not measured)'}
    for label, elem in (('fp32', 4), ('bf16', 2)):
        ms = sum(t * k for t, k in times[label]) / sum(k for _, k in times[label])
        blocks = sorted(t for t, _ in times[label])
        msg_bytes = n_in * numel * elem
        result[label] = {'ms_per_step': round(ms, 4), 'block_ms_min': round(blocks[0], 4),
                         'block_ms_max': round(blocks[-1], 4),
                         'message_bytes_per_in_neighbour': msg_bytes,
                         'message_bytes_per_step_per_rank': msg_bytes}
    result['bf16_over_fp32_time'] = round(result['bf16']['ms_per_step'] / result['fp32']['ms_per_step'], 4)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
