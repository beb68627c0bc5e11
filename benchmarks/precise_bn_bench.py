"""Cost of precise BatchNorm statistics (``GossipTrainer.update_bn``) per batch, next to the captured
evaluation (``GossipTrainer.evaluate``) and a captured training step, in one process:

ResNet-50 at ``--batch`` synthetic 224 x 224 images per batch in pinned host memory, fp32 (TF32) and bf16
(the compute twin).  ``update_bn`` and ``evaluate`` each run over ``--batches`` batches, H2D copies included;
the training step is ``--batches`` ``step()`` calls fed the same way.  Each arm's time is the whole pass,
CUDA events around it and a final synchronise, divided by the number of batches.  Every arm is warmed up
once (captures, library algorithm choice), then the three run ``--repeats`` times alternated; the median is
printed, with the own-kernel launches per batch of each.

    python benchmarks/precise_bn_bench.py [--batch 256] [--batches 20] [--repeats 5]

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


def _trainer(twin):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    torch.manual_seed(0)
    dev = torch.device('cuda', 0)
    net = models.resnet50().to(dev).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                               heartbeat_timeout=60, compute_dtype=torch.bfloat16 if twin else None)
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, weight_decay=1e-4)
    return GossipTrainer(model, opt, amp_dtype=torch.bfloat16 if twin else None)


def _timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def _train(tr, data):
    for x, y in data:
        tr.step(x, y)
    tr.finish()


def bench(args, twin, data):
    tr = _trainer(twin)
    arms = {'update_bn': lambda: tr.update_bn(data), 'evaluate': lambda: tr.evaluate(data),
            'train_step': lambda: _train(tr, data)}
    _train(tr, data[:4])                             # eager warm-up steps, then the captured step
    for fn in arms.values():                         # warm-up: captures, algorithm choice
        fn()
    times = {k: [] for k in arms}
    for _ in range(args.repeats):
        for k, fn in arms.items():
            times[k].append(_timed(fn) / len(data))
    out = {k + '_ms': statistics.median(v) for k, v in times.items()}
    out.update(update_bn_launches=tr.update_bn_launches_per_batch, evaluate_launches=tr.eval_launches_per_batch,
               train_step_launches=tr.own_launches_per_step)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--batches', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=5)
    args = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    name, power = _card()
    print('card: %s, power limit / max SM clock: %s' % (name, power))
    gen = torch.Generator().manual_seed(0)
    full = [(torch.randn(args.batch, 3, 224, 224, generator=gen).pin_memory(),
             torch.randint(0, 1000, (args.batch,), generator=gen).pin_memory()) for _ in range(4)]
    data = [full[i % 4] for i in range(args.batches)]
    out = dict(card=name, power=power, batch=args.batch, batches=args.batches)
    for label, twin in (('fp32', False), ('bf16', True)):
        r = bench(args, twin, data)
        out[label] = r
        print('%s ResNet-50, batch %d, ms per batch: update_bn %.2f, evaluate %.2f, training step %.2f; own launches '
              'per batch %d / %d / %d' % (label, args.batch, r['update_bn_ms'], r['evaluate_ms'], r['train_step_ms'],
                                          r['update_bn_launches'], r['evaluate_launches'], r['train_step_launches']))
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
