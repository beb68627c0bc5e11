"""Cost of stochastic depth (``resnet50(drop_path_rate=p)``) in the captured training step, in one process:

ResNet-50 at ``--batch`` synthetic 224 x 224 images resident on the device, fp32 (TF32) and bf16 (the
compute twin), at rate 0 (today's step, no draw) against ``--rate`` (one draw launch per forward and the
scaled BatchNorm / MODE 3 kernels).  Each arm is a GossipTrainer warmed up and captured, then
``--steps`` replays timed with CUDA events around them and a final synchronise; the two arms of a dtype
are alternated ``--repeats`` times and the median ms/step is printed, with the own-kernel launches per
step of each.

    python benchmarks/drop_path_bench.py [--batch 256] [--rate 0.05] [--steps 20] [--repeats 5]

Prints the card name, power limit and max SM clock with the numbers, and one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stochastic_gradient_push_b200 as sgp                       # noqa: E402
from stochastic_gradient_push_b200 import models                 # noqa: E402


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader',
                              '-i', '0'], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30)
        power = out.stdout.strip()
    except Exception as e:                          # noqa
        power = 'unknown (%s)' % e
    return name, power


def _trainer(twin, rate):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    torch.manual_seed(0)
    dev = torch.device('cuda', 0)
    net = models.resnet50(drop_path_rate=rate).to(dev).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                               heartbeat_timeout=60, compute_dtype=torch.bfloat16 if twin else None)
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, weight_decay=1e-4)
    return GossipTrainer(model, opt, amp_dtype=torch.bfloat16 if twin else None)


def _timed(tr, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record(tr.stream)
    for _ in range(steps):
        tr.step_resident()
    b.record(tr.stream)
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def bench(args, twin, x, y):
    arms = {}
    for rate in (0.0, args.rate):
        tr = _trainer(twin, rate)
        for _ in range(5):                           # eager warm-up steps, then the capture
            tr.step(x, y)
        tr.finish()
        arms[rate] = tr
    times = {r: [] for r in arms}
    for _ in range(args.repeats):
        for r, tr in arms.items():
            times[r].append(_timed(tr, args.steps))
    out = {}
    for r, tr in arms.items():
        out['rate_%g' % r] = dict(ms_per_step=statistics.median(times[r]), spread_ms=max(times[r]) - min(times[r]),
                                  launches_per_step=tr.own_launches_per_step)
    del arms
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--rate', type=float, default=0.05)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=5)
    args = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    name, power = _card()
    print('card: %s, power limit / max SM clock: %s' % (name, power))
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(args.batch, 3, 224, 224, generator=gen).pin_memory()
    y = torch.randint(0, 1000, (args.batch,), generator=gen).pin_memory()
    out = dict(card=name, power=power, batch=args.batch, rate=args.rate)
    for label, twin in (('fp32', False), ('bf16', True)):
        r = bench(args, twin, x, y)
        out[label] = r
        a, b = r['rate_0'], r['rate_%g' % args.rate]
        print('%s ResNet-50, batch %d: rate 0 %.2f ms/step (spread %.2f, %d launches), rate %g %.2f ms/step '
              '(spread %.2f, %d launches)' % (label, args.batch, a['ms_per_step'], a['spread_ms'],
                                                a['launches_per_step'], args.rate, b['ms_per_step'], b['spread_ms'],
                                                b['launches_per_step']))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
