"""SlowMo step at ResNet-50 size: the fused ``GossipEngine.slowmo`` against the same step built
from ``GossipEngine.consensus(out, full=True)`` plus torch elementwise ops, N virtual ranks on ONE
GPU (``LocalWorld`` loop-back), one host thread per rank.

    python benchmarks/slowmo_bench.py [--ranks 4] [--calls 60] [--block 10] [--tau 48]
                                      [--step-ms MS] [--out F.json]

Loop-back reads every rank's snapshot from local HBM, not over NVLink, so these are
kernel-efficiency numbers; the NVLink time is NOT measured here.  Device-timed with CUDA events per
rank stream (max over ranks); the two arms alternate in blocks of ``--block`` calls until each has
``--calls``.  ``--step-ms``: a measured training step time (``bench.py``'s ms_per_step) to express
the cost amortised over ``--tau`` steps as a fraction of it.  Bytes from shapes, per rank and call
(n fp32 parameters, N ranks):
  fused   snapshot 2 * 4n + every snapshot 4nN + u, x_prev in 8n + u, x_prev, z out 12n
  torch   snapshot 2 * 4n + every snapshot 4nN + zbar out 4n
          + t = x_prev - zbar 12n, t /= lr 8n, u *= beta 8n, u += t 12n, x_prev -= a lr u 12n, z = x_prev 8n
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

LR, ALPHA, BETA = 0.1, 1.0, 0.5


def _world(n_ranks, numel):
    dev = torch.device('cuda', 0)
    lw = LocalWorld(n_ranks)
    base = torch.randn(numel, device=dev) * 0.05
    ranks = []
    for r in range(n_ranks):
        g = sgp.NPeerDynamicDirectedExponentialGraph(r, n_ranks, peers_per_itr=1)
        e = GossipEngine(lw.view(r), base + 1e-3 * torch.randn(numel, device=dev), g, sgp.UniformMixing(g, dev),
                         timeout_s=60.0, name='slowmo_bench')
        e.prepare_consensus()
        ranks.append(dict(e=e, s=torch.cuda.Stream(device=dev), u=torch.zeros(numel, device=dev),
                          xp=base.clone(), zbar=torch.empty(numel, device=dev), t=torch.empty(numel, device=dev)))
    # load the torch arm's elementwise kernels now: under lazy module loading a first launch can
    # wait for the whole device, where the other ranks' barrier kernels wait for this rank
    for rk in ranks:
        t = rk['t'].zero_()
        torch.sub(t, t, out=t)
        t.div_(LR)
        t.mul_(BETA).add_(t)
        t.sub_(t, alpha=ALPHA * LR)
        t.copy_(rk['xp'])
        rk['e'].ps_weight = 1.0
    torch.cuda.synchronize()
    return ranks


def _fused(rk):
    rk['e'].slowmo(rk['u'], rk['xp'], LR, ALPHA, BETA, False)


def _unfused(rk):
    e, u, xp, zbar, t = rk['e'], rk['u'], rk['xp'], rk['zbar'], rk['t']
    e.consensus(zbar, full=True)
    torch.sub(xp, zbar, out=t)
    t.div_(LR)
    u.mul_(BETA).add_(t)
    xp.sub_(u, alpha=ALPHA * LR)
    e.z.copy_(xp)
    e.ps_weight = 1.0


def _block(ranks, k, step):
    """k calls per rank, each rank from its own thread on its own stream -> ms per call"""
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in ranks]

    def run(i):
        rk = ranks[i]
        with torch.cuda.stream(rk['s']):
            evs[i][0].record(rk['s'])
            for _ in range(k):
                step(rk)
            evs[i][1].record(rk['s'])
    _in_threads([functools.partial(run, i) for i in range(len(ranks))])
    torch.cuda.synchronize()
    for rk in ranks:
        rk['e'].check()
    return max(a.elapsed_time(b) for a, b in evs) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ranks', type=int, default=4)
    ap.add_argument('--calls', type=int, default=60, help='timed calls per arm (>= 60)')
    ap.add_argument('--block', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--tau', type=int, default=48, help='SlowMo period the cost is amortised over')
    ap.add_argument('--step-ms', type=float, default=None, help='measured training step time (bench.py)')
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'

    from stochastic_gradient_push_b200.ops import native
    C = native.load()
    n_params = sum(p.numel() for p in resnet50().parameters())
    numel = (n_params + C.CHUNK - 1) // C.CHUNK * C.CHUNK
    card, power = _card()
    ranks = _world(args.ranks, numel)
    arms = {'fused': _fused, 'consensus+torch': _unfused}
    for step in arms.values():                   # kernels, allocator and library loaded once
        _block(ranks, args.warmup, step)
    times = {label: [] for label in arms}
    done = 0
    while done < args.calls:
        k = min(args.block, args.calls - done)
        for label, step in arms.items():         # alternate the arms
            times[label].append((_block(ranks, k, step), k))
        done += k

    N, b = args.ranks, 4 * numel
    moved = {'fused': 2 * b + N * b + 2 * b + 3 * b,
             'consensus+torch': 2 * b + N * b + b + 3 * b + 2 * b + 2 * b + 3 * b + 3 * b + 2 * b}
    result = {'card': card, 'power_limit,max_sm_clock': power, 'ranks': N, 'params': n_params, 'numel': numel,
              'calls_per_arm': args.calls, 'tau': args.tau, 'step_ms': args.step_ms,
              'note': 'loop-back on one GPU: snapshots are read from local HBM, not NVLink; kernel-efficiency '
                      'numbers, the NVLink time is not measured'}
    for label in times:
        ms = sum(t * k for t, k in times[label]) / sum(k for _, k in times[label])
        blocks = sorted(t for t, _ in times[label])
        r = {'ms_per_call': round(ms, 4), 'block_ms_min': round(blocks[0], 4),
             'block_ms_max': round(blocks[-1], 4), 'bytes_per_rank': moved[label],
             'GB_per_s_all_ranks': round(N * moved[label] / (ms * 1e-3) / 1e9, 1),
             'ms_per_step_amortised': round(ms / args.tau, 4)}
        if args.step_ms:
            r['fraction_of_step'] = round(ms / args.tau / args.step_ms, 5)
        result[label] = r
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
