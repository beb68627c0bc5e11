"""Validation pass cost: the eager CLI ``evaluate`` (``cli/gossip_sgd.py``) against the captured
``GossipTrainer.evaluate``, in one process:

1. pass: ResNet-50, ``--batches`` batches of ``--batch`` synthetic 224 x 224 images in pinned host memory
   (the last one partial when ``--tail`` > 0), fp32 (TF32) and bf16 (the compute twin).  Each arm's time
   is the whole pass, H2D copies included: CUDA events around it and a final synchronise.  Both arms are
   warmed up once (captures, library algorithm choice), then run ``--repeats`` times alternated; the
   median is printed;
2. GEMM: every ResNet-50 1x1 shape at batch 256 on ``C.conv1x1_bn_eval`` (BatchNorm (+ residual) + ReLU in
   the epilogue) against the library convolution + eval ``F.batch_norm`` (+ add) + ReLU, NHWC, CUDA events
   over ``--launches`` launches.

    python benchmarks/eval_bench.py [--batch 256] [--batches 196] [--repeats 3] [--launches 50]

Prints the card name and power limit with the numbers, and one JSON line.
"""
import argparse
import json
import logging
import os
import statistics
import subprocess
import sys
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stochastic_gradient_push_b200 as sgp                       # noqa: E402
from stochastic_gradient_push_b200 import models                 # noqa: E402
from stochastic_gradient_push_b200.cli import gossip_sgd         # noqa: E402
from stochastic_gradient_push_b200.ops import native             # noqa: E402

RESNET50_1X1 = [  # (H = W, N, K) at stride 1
    (56, 64, 64), (56, 256, 64), (56, 64, 256), (56, 128, 256),
    (28, 512, 128), (28, 128, 512), (28, 256, 512),
    (14, 1024, 256), (14, 256, 1024), (14, 512, 1024),
    (7, 2048, 512), (7, 512, 2048),
]


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
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def bench_pass(args, twin, data):
    tr = _trainer(twin)
    for i in range(3):                               # running statistics, and the training graph exists
        tr.step(*data[i])
    tr.finish()
    cli = types.SimpleNamespace(device='cuda', channels_last=True, amp=twin)
    log = logging.getLogger('eval_bench')
    crit = nn.CrossEntropyLoss()
    arms = {'eager': lambda: gossip_sgd.evaluate(cli, data, tr.model, crit, log),
            'graph': lambda: tr.evaluate(data)}
    for fn in arms.values():                         # warm-up: captures, algorithm choice
        fn()
    times = {k: [] for k in arms}
    res = {}
    for _ in range(args.repeats):
        for k, fn in arms.items():
            t, res[k] = _timed(fn)
            times[k].append(t)
    eager_p1, eager_p5 = res['eager']
    r = res['graph']
    return dict(eager_ms=statistics.median(times['eager']), graph_ms=statistics.median(times['graph']),
                eager_prec1=eager_p1, graph_prec1=r.prec1, eager_prec5=eager_p5, graph_prec5=r.prec5,
                launches_per_batch=tr.eval_launches_per_batch, images=r.count)


def bench_gemm(args, dtype):
    C = native.load()
    dev = torch.device('cuda', 0)
    g = torch.Generator(device=dev).manual_seed(1)
    rows = []
    for hw, N, K in RESNET50_1X1:
        x = torch.randn(args.batch, K, hw, hw, device=dev, generator=g).to(dtype).contiguous(
            memory_format=torch.channels_last)
        w = (torch.randn(N, K, 1, 1, device=dev, generator=g) / K ** 0.5).to(dtype).contiguous(
            memory_format=torch.channels_last)
        r = torch.randn(args.batch, N, hw, hw, device=dev, generator=g).to(dtype).contiguous(
            memory_format=torch.channels_last)
        gamma, beta = torch.rand(N, device=dev) + 0.5, torch.randn(N, device=dev) * 0.1
        mean, var = torch.randn(N, device=dev) * 0.1, torch.rand(N, device=dev) + 0.5
        res = {}
        for name, fn in (
                ('ours', lambda: C.conv1x1_bn_eval(x, w, gamma, beta, mean, var, 1e-5, True, r)),
                ('library', lambda: torch.relu(F.batch_norm(F.conv2d(x, w), mean, var, gamma, beta, False, 0.1,
                                                            1e-5) + r))):
            with torch.no_grad():
                for _ in range(3):
                    fn()
                t, _ = _timed(lambda: [fn() for _ in range(args.launches)])
            res[name] = t / args.launches
        rows.append(dict(shape=[args.batch, hw, hw, K, N], ours_ms=res['ours'], library_ms=res['library']))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--batches', type=int, default=196)
    ap.add_argument('--tail', type=int, default=80, help='rows of a final partial batch (0: none)')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--launches', type=int, default=50)
    args = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    name, power = _card()
    print('card: %s, power limit / max SM clock: %s' % (name, power))
    gen = torch.Generator().manual_seed(0)
    sizes = [args.batch] * args.batches + ([args.tail] if args.tail else [])
    # four distinct pinned full batches, cycled (every batch is still copied H2D): 196 distinct ones
    # would pin 30 GB of host memory
    full = [(torch.randn(args.batch, 3, 224, 224, generator=gen).pin_memory(),
             torch.randint(0, 1000, (args.batch,), generator=gen).pin_memory()) for _ in range(4)]
    data = [full[i % 4] for i in range(args.batches)]
    if args.tail:
        data.append((full[0][0][:args.tail].clone().pin_memory(), full[0][1][:args.tail].clone().pin_memory()))
    out = dict(card=name, power=power, batch=args.batch, images=sum(sizes))
    for label, twin in (('fp32', False), ('bf16', True)):
        p = bench_pass(args, twin, data)
        out['pass_' + label] = p
        print('%s pass over %d images: eager %.1f ms, evaluate %.1f ms (x%.2f); prec@1 %.3f / %.3f, prec@5 '
              '%.3f / %.3f; %d own launches per batch' % (
                  label, p['images'], p['eager_ms'], p['graph_ms'], p['eager_ms'] / p['graph_ms'],
                  p['eager_prec1'], p['graph_prec1'], p['eager_prec5'], p['graph_prec5'], p['launches_per_batch']))
        torch.cuda.empty_cache()
    for label, dtype in (('fp32', torch.float32), ('bf16', torch.bfloat16)):
        rows = bench_gemm(args, dtype)
        out['gemm_' + label] = rows
        for row in rows:
            print('%s 1x1 %s: conv+BN+add+ReLU %.3f ms, library %.3f ms' % (
                label, 'x'.join(map(str, row['shape'])), row['ours_ms'], row['library_ms']))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
