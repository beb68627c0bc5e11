"""Consensus distance (slice mode) and push-sum average model (full mode) at ResNet-50 size:
``GossipEngine.consensus(full=False / True)``, N virtual ranks on ONE GPU (``LocalWorld``
loop-back), one host thread per rank.

    python benchmarks/consensus_bench.py [--ranks 4] [--calls 60] [--block 10] [--out F.json]

Loop-back reads every rank's snapshot from local HBM, not over NVLink, so this is a
kernel-efficiency number; the NVLink time is NOT measured here.  Device-timed with CUDA events
per rank stream (max over ranks); the two arms alternate in blocks of ``--block`` calls until each
has ``--calls``.  Bytes are computed from shapes, per rank and call:
  snapshot     read z + write the snapshot          2 * 4n
  slice        read every rank's snapshot of 1/N     4n
  full         read every rank's snapshot           4nN, + write zbar 4n
"""
import argparse
import functools
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stochastic_gradient_push_b200 as sgp                                # noqa: E402
from stochastic_gradient_push_b200.models import resnet50                  # noqa: E402
from stochastic_gradient_push_b200.ops.peer_mix import GossipEngine        # noqa: E402
from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld    # noqa: E402
from gossip_dtype_bench import _card, _in_threads                          # noqa: E402


def _world(n_ranks, numel):
    dev = torch.device('cuda', 0)
    lw = LocalWorld(n_ranks)
    base = torch.randn(numel, device=dev) * 0.05
    ranks = []
    for r in range(n_ranks):
        g = sgp.NPeerDynamicDirectedExponentialGraph(r, n_ranks, peers_per_itr=1)
        e = GossipEngine(lw.view(r), base + 1e-3 * torch.randn(numel, device=dev), g, sgp.UniformMixing(g, dev),
                         timeout_s=60.0, name='cons_bench')
        e.prepare_consensus()
        ranks.append((e, torch.cuda.Stream(device=dev), torch.empty(numel, device=dev)))
    torch.cuda.synchronize()
    return ranks


def _block(ranks, k, full):
    """k calls per rank, each rank from its own thread on its own stream -> ms per call"""
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in ranks]

    def run(i):
        e, s, out = ranks[i]
        with torch.cuda.stream(s):
            evs[i][0].record(s)
            for _ in range(k):
                e.consensus(out, full=full)
            evs[i][1].record(s)
    _in_threads([functools.partial(run, i) for i in range(len(ranks))])
    torch.cuda.synchronize()
    for e, _, _ in ranks:
        e.check()
    return max(a.elapsed_time(b) for a, b in evs) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ranks', type=int, default=4)
    ap.add_argument('--calls', type=int, default=60, help='timed calls per arm (>= 50)')
    ap.add_argument('--block', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'

    from stochastic_gradient_push_b200.ops import native
    C = native.load()
    n_params = sum(p.numel() for p in resnet50().parameters())
    numel = (n_params + C.CHUNK - 1) // C.CHUNK * C.CHUNK
    card, power = _card()
    ranks = _world(args.ranks, numel)
    # the result tensors come from the caching allocator: warm it (and the kernels) up first,
    # sequentially per rank would deadlock on the barriers, so one warm-up block per arm
    for full in (False, True):
        _block(ranks, args.warmup, full)
    times = {'slice': [], 'full': []}
    done = 0
    while done < args.calls:
        k = min(args.block, args.calls - done)
        for label in times:                          # alternate the arms
            times[label].append((_block(ranks, k, label == 'full'), k))
        done += k

    N, b = args.ranks, 4 * numel
    moved = {'slice': 2 * b + b, 'full': 2 * b + N * b + b}
    result = {'card': card, 'power_limit,max_sm_clock': power, 'ranks': N, 'params': n_params, 'numel': numel,
              'calls_per_arm': args.calls,
              'note': 'loop-back on one GPU: snapshots are read from local HBM, not NVLink; a kernel-efficiency '
                      'number, the NVLink time is not measured'}
    for label in times:
        ms = sum(t * k for t, k in times[label]) / sum(k for _, k in times[label])
        blocks = sorted(t for t, _ in times[label])
        result[label] = {'ms_per_call': round(ms, 4), 'block_ms_min': round(blocks[0], 4),
                         'block_ms_max': round(blocks[-1], 4), 'bytes_per_rank': moved[label],
                         'bytes_all_ranks': N * moved[label],
                         'GB_per_s_all_ranks': round(N * moved[label] / (ms * 1e-3) / 1e9, 1)}
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
