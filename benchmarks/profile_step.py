#!/usr/bin/env python
"""
Per-kernel-class GPU time of the bench.py headline step (ResNet-50 SGP, one GPU).

    python benchmarks/profile_step.py [--dtype fp32|bf16] [--batch-size 256] [--steps 5]
                                      [--warmup 10] [--eager] [--out DIR]

Builds the same trainer as bench.py (``bench._build``), warms up and captures as bench does,
then records ``--steps`` replays under torch.profiler (CUDA activity only) and prints ms per
step per kernel class, plus the card name and power limit.  If the replays of the captured
graph carry no kernel records, the step is re-built and profiled eagerly (``--eager`` forces
that).  DIR/profile_<dtype>.json holds the same table.  Timing numbers come from a traced run:
compare them with each other, and take end-to-end step times from bench.py.
"""

from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

C1_MODE = {'0': 'c1_gemm MODE 0 (plain)', '1': 'c1_gemm MODE 1 (fwd + BN stats)',
           '2': 'c1_gemm MODE 2 (conv1 dgrad + skip grad)', '3': 'c1_gemm MODE 3 (+ bn3 bwd reduce)'}


def classify(name: str) -> str:
    m = re.search(r'c1_gemm_kernel<\s*\d+\s*,\s*(\d)', name)
    if m:
        return C1_MODE[m.group(1)]
    for key, cls in (('bn_bwd_reduce_kernel', 'BN bwd reduce'), ('bn_bwd_dx_kernel', 'BN bwd dx'),
                     ('bn_bwd_finalize', 'BN finalize'), ('stats_finalize', 'BN finalize'),
                     ('bn_eval_coeff', 'BN finalize'), ('bn_stats_kernel', 'BN stats'),
                     ('bn_apply_kernel', 'BN apply'), ('stem_', 'stem'), ('pool', 'pool'),
                     ('xent', 'loss'), ('sgp_', 'gossip / SGD'), ('gossip', 'gossip / SGD')):
        if key in name:
            return cls
    low = name.lower()
    if 'wgrad' in low:
        return 'cuDNN wgrad'
    if 'dgrad' in low:
        return 'cuDNN dgrad'
    if 'fprop' in low or 'conv' in low or 'xmma' in low or 'implicit' in low:
        return 'cuDNN fprop / other conv'
    return 'other'


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=20).stdout
        return out.strip().splitlines()[0]
    except Exception as e:          # pragma: no cover
        return 'nvidia-smi unavailable: %r' % e


def profile(args, eager):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    import bench

    ns = argparse.Namespace(model='resnet50', algo='sgp', ppi=1, no_graph=eager, autocast=False,
                            ar_transport='auto', adpsgd_rounds=4)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    torch.backends.cudnn.benchmark = True
    torch.backends.cudnn.allow_tf32 = True
    net, model, trainer, _ = bench._build(ns, args.dtype, args.batch_size, 0, 1, dev)
    g = torch.Generator().manual_seed(1234)
    batch = (torch.randn(args.batch_size, 3, 224, 224, generator=g).pin_memory(),
             torch.randint(0, 1000, (args.batch_size,), generator=g).pin_memory())
    for _ in range(max(args.warmup, 5)):
        trainer.step(*batch)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            trainer.step_resident()
        torch.cuda.synchronize()
    per_cls = defaultdict(float)
    launches = defaultdict(int)
    n = 0
    for evt in prof.events():
        if evt.device_type != torch.autograd.DeviceType.CUDA:
            continue
        cls = classify(evt.name)
        per_cls[cls] += evt.time_range.elapsed_us() / 1e3
        launches[cls] += 1
        n += 1
    trainer.finish()
    del trainer, model, net
    torch.cuda.empty_cache()
    return per_cls, launches, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--dtype', default='fp32', choices=['fp32', 'bf16'])
    ap.add_argument('--batch-size', type=int, default=256)
    ap.add_argument('--steps', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--eager', action='store_true')
    ap.add_argument('--out', default='profile_out')
    args = ap.parse_args()

    mode = 'eager' if args.eager else 'graph replay'
    per_cls, launches, n = profile(args, args.eager)
    if n < 50 * args.steps and not args.eager:          # replayed kernels not attributed
        mode = 'eager (graph replays carried no kernel records)'
        per_cls, launches, n = profile(args, True)
    total = sum(per_cls.values())
    rows = sorted(per_cls.items(), key=lambda kv: -kv[1])
    res = {'card': card(), 'dtype': args.dtype, 'batch': args.batch_size, 'steps': args.steps, 'mode': mode,
           'switches': {k: v for k, v in os.environ.items() if k.startswith('SGP_B200_')},
           'ms_per_step': {k: round(v / args.steps, 3) for k, v in rows},
           'launches_per_step': {k: launches[k] // args.steps for k, _ in rows},
           'kernel_ms_per_step_total': round(total / args.steps, 3)}
    print('card (name, power limit, max SM clock): %s' % res['card'])
    print('%s, batch %d, %s, %d steps' % (args.dtype, args.batch_size, mode, args.steps))
    for k, v in rows:
        print('  %-44s %8.3f ms  %5d launches' % (k, v / args.steps, launches[k] // args.steps))
    print('  %-44s %8.3f ms' % ('sum of kernel time', total / args.steps))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'profile_%s.json' % args.dtype), 'w') as f:
        json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
