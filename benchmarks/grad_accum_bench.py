"""Cost of gradient accumulation (``GossipTrainer(accumulation_steps=k)``, ``grad_accumulate_kernel``), in
one process:

1. kernel: one ``grad_accumulate`` call over ResNet-50's gradient list (every parameter's fp32 arena
   view as dst; fresh sources with the same layout, fp32 and bf16).  CUDA events around ``--launches``
   calls after warm-up, median over ``--rounds`` rounds with the two source dtypes alternated.  The
   working set (about 300 MB) is larger than L2, so no flush is needed.  Achieved bytes/s counts the
   bytes the operation needs (read src, read dst, write dst: 12 B per element for fp32 sources, 10 B for
   bf16) against the H100 SXM data-sheet 3.35 TB/s;
2. step: the captured one-rank ResNet-50 step (fp32 / TF32) at (B, k) = (256, 1), (512, 2) and
   (1024, 4), i.e. 256-image micro-batches.  Each configuration runs in a process of its own (eager
   step, capture, replay, a warm-up block, then ``--steps`` timed replays), the processes alternated
   ``--repeats`` times: ms / step, images / s, own launches / step and peak ``max_memory_allocated``.

    python benchmarks/grad_accum_bench.py [--launches 200] [--rounds 5] [--steps 10] [--repeats 3]

Prints the card name and power limit with the numbers, and one JSON line.
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
from stochastic_gradient_push_b200.ops import native             # noqa: E402

from ema_bench import HBM_BYTES_PER_S, _card, _time              # noqa: E402

CONFIGS = ((256, 1), (512, 2), (1024, 4))


def _model(dev):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    torch.manual_seed(0)
    net = models.resnet50().to(dev).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                               heartbeat_timeout=60)
    assert model.transport == 'nvlink'
    opt = FusedGossipSGD(model, lr=0.01, momentum=0.9, weight_decay=1e-4, nesterov=True)
    return net, model, opt


def _trainer(model, opt, k):
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    return GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=True, warmup_iters=1, accumulation_steps=k)


def _batch(rows):
    g = torch.Generator().manual_seed(rows)
    return torch.randn(rows, 3, 224, 224, generator=g).pin_memory(), torch.randint(0, 1000, (rows,), generator=g).pin_memory()


def _run_config(B, k, steps):
    """one configuration: eager step, capture + replay, a warm-up block, then ``steps`` timed replays;
    prints ms / step, own launches / step and the peak max_memory_allocated as one JSON line"""
    dev = torch.device('cuda', 0)
    torch.backends.cudnn.benchmark = True
    _, model, opt = _model(dev)
    tr = _trainer(model, opt, k)
    x, y = _batch(B)
    for _ in range(3):
        tr.step(x, y)
    tr.finish()
    assert tr.graph is not None
    _time(tr.step_resident, steps, tr.stream)
    ms = _time(tr.step_resident, steps, tr.stream)
    tr.finish()
    print(json.dumps({'ms_per_step': ms, 'own_launches_per_step': tr.own_launches_per_step,
                      'peak_bytes': torch.cuda.max_memory_allocated()}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default=None, help='B,k: measure that configuration alone (one JSON line)')
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('grad_accum_bench.py measures on the GPU; no CUDA device found')
    if args.config:
        return _run_config(*(int(v) for v in args.config.split(',')), steps=args.steps)
    torch.backends.cudnn.benchmark = True
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    card, power = _card()
    C = native.load()
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())

    # ---- 1. kernel ---------------------------------------------------------------------------- #
    net, model, opt = _model(dev)
    dst = [p.grad for p in net.parameters()]
    numel = sum(d.numel() for d in dst)
    srcs = {'fp32': [torch.randn_like(d) for d in dst],
            'bf16': [torch.randn_like(d).to(torch.bfloat16) for d in dst]}
    bytes_per_el = {'fp32': 12, 'bf16': 10}
    c0 = C.launch_count()
    C.grad_accumulate(dst, srcs['fp32'])
    launches_per_call = C.launch_count() - c0
    for s in srcs.values():
        _time(lambda s=s: C.grad_accumulate(dst, s), 20, stream)          # warm-up
    ms = {k: [] for k in srcs}
    for _ in range(args.rounds):
        for k, s in srcs.items():
            ms[k].append(_time(lambda s=s: C.grad_accumulate(dst, s), args.launches, stream))
    kernel = {}
    for k, v in ms.items():
        med = statistics.median(v)
        nbytes = bytes_per_el[k] * numel
        rate = nbytes / (med * 1e-3)
        kernel[k] = {'us_per_call_median': round(med * 1e3, 2), 'us_min': round(min(v) * 1e3, 2),
                     'us_max': round(max(v) * 1e3, 2), 'tensors': len(dst), 'elements': numel,
                     'MB_per_call': round(nbytes / 1e6, 1), 'GB_per_s': round(rate / 1e9, 1),
                     'share_of_3.35TB/s': round(rate / HBM_BYTES_PER_S, 3), 'launches_per_call': launches_per_call}
        print('%s sources: %8.2f us / call (min %.2f, max %.2f), %d tensors, %.1f MB, %.0f GB/s = %.1f%% of '
              '3.35 TB/s, %d launch' % (k, med * 1e3, min(v) * 1e3, max(v) * 1e3, len(dst), nbytes / 1e6,
                                        rate / 1e9, 100 * rate / HBM_BYTES_PER_S, launches_per_call))
    for d in dst:
        d.zero_()
    del srcs

    # ---- 2. captured steps: each configuration in a process of its own, the processes alternated ---- #
    del net, model, opt
    runs = {c: [] for c in CONFIGS}
    for rep in range(args.repeats):
        for B, k in CONFIGS:
            out = subprocess.run([sys.executable, os.path.abspath(__file__), '--config', '%d,%d' % (B, k),
                                  '--steps', str(args.steps)],
                                 stdout=subprocess.PIPE, text=True, check=True).stdout
            runs[(B, k)].append(json.loads(out.strip().splitlines()[-1]))
    step = {}
    for (B, k), v in runs.items():
        ms = [r['ms_per_step'] for r in v]
        mean = statistics.mean(ms)
        key = 'B%d_k%d' % (B, k)
        step[key] = {'ms_per_step': [round(t, 3) for t in ms], 'mean': round(mean, 3),
                     'images_per_s': round(B / (mean * 1e-3), 1),
                     'own_launches_per_step': v[0]['own_launches_per_step'],
                     'peak_GiB': round(max(r['peak_bytes'] for r in v) / 2 ** 30, 2)}
        print('step B=%4d k=%d: %s ms (mean %.3f), %.0f images/s, %d own launches / step, peak %.2f GiB'
              % (B, k, step[key]['ms_per_step'], mean, step[key]['images_per_s'],
                 step[key]['own_launches_per_step'], step[key]['peak_GiB']))
    print('card: %s, power limit / max SM clock: %s' % (card, power))
    print(json.dumps({'card': card, 'power_limit,max_sm_clock': power, 'kernel': kernel, 'step': step}))


if __name__ == '__main__':
    main()
