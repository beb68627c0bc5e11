"""Cost of setting the learning rate every iteration (``--lr_policy poly``) on the captured
training step: GossipTrainer on one GPU (ResNet-50, fp32, synthetic pinned batches), the learning
rate left unchanged (``set_hyper`` skips it) against a new value every step (one pinned staging
slot and one async 64-byte H2D copy per step; the 8-slot ring makes the host wait for the copy
issued 8 steps earlier).  The host drains the metrics ring every ``--drain`` steps, as the
training loop does every ``--print_freq`` iterations.

    python benchmarks/lr_cadence_bench.py [--batch 256 32] [--steps 200] [--block 20] [--drain 10]

Each block of ``--block`` steps is timed on the host from a synchronised start to a synchronised
end; the two arms alternate block by block.
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stochastic_gradient_push_b200 as sgp                                  # noqa: E402
from stochastic_gradient_push_b200 import models                             # noqa: E402
from stochastic_gradient_push_b200.optim import FusedGossipSGD               # noqa: E402
from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel  # noqa: E402
from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer     # noqa: E402

from xent_bench import _card                                                 # noqa: E402


def _block(trainer, opt, pool, k, drain, lr_of):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(k):
        for g in opt.param_groups:
            g['lr'] = lr_of(i)
        trainer.step(*pool[i % len(pool)])
        if (i + 1) % drain == 0:
            trainer.stream.synchronize()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / k


def measure(bs, steps, block, drain, warmup):
    dev = torch.device('cuda', 0)
    torch.manual_seed(1)
    net = models.init_imagenet_in_1hr(models.resnet50()).to(dev).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                               verbose=False, heartbeat_timeout=60)
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, weight_decay=1e-4, nesterov=True)
    trainer = GossipTrainer(model, opt, amp_dtype=None)
    g = torch.Generator().manual_seed(1234)
    pool = [(torch.randn(bs, 3, 224, 224, generator=g).pin_memory(),
             torch.randint(0, 1000, (bs,), generator=g).pin_memory()) for _ in range(4)]
    base = 0.1
    arms = {'fixed_lr': lambda i: base,
            'lr_every_step': lambda i: base * (1.0 - 1e-4 * ((i % block) + 1))}
    for lr_of in arms.values():
        _block(trainer, opt, pool, warmup, drain, lr_of)
    times = {k: [] for k in arms}
    done = 0
    while done < steps:
        for k, lr_of in arms.items():
            times[k].append(_block(trainer, opt, pool, block, drain, lr_of))
        done += block
    trainer.finish()
    res = {'per_gpu_batch': bs, 'graphed': trainer.graph is not None}
    for k, ts in times.items():
        ts = sorted(ts)
        res[k] = {'ms_per_step_median': round(ts[len(ts) // 2], 3), 'ms_min': round(ts[0], 3),
                  'ms_max': round(ts[-1], 3), 'blocks': len(ts)}
    res['every_step_minus_fixed_ms'] = round(res['lr_every_step']['ms_per_step_median'] -
                                             res['fixed_lr']['ms_per_step_median'], 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, nargs='+', default=[256, 32])
    ap.add_argument('--steps', type=int, default=200, help='timed steps per arm')
    ap.add_argument('--block', type=int, default=20)
    ap.add_argument('--drain', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'
    card, power = _card()
    result = {'card': card, 'power_limit,max_sm_clock': power, 'block': args.block, 'drain_every': args.drain}
    for bs in args.batch:
        result['batch%d' % bs] = measure(bs, args.steps, args.block, args.drain, args.warmup)
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
