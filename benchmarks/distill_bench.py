"""Cost of knowledge distillation (``GossipTrainer(teacher=...)``, ``--distill_alpha``), in one process:

(a) the distillation loss alone, forward + backward, at ``--batch`` x 1000 classes in fp32 and bf16: the fused
    DISTILL kernels (``fused_cross_entropy(teacher_logits=...)``) against the torch composition
    (``F.cross_entropy`` + ``F.kl_div`` + ``topk`` accuracies), and today's fused cross-entropy without a
    teacher.  CUDA events around ``--loss_iters`` calls, median of ``--repeats``.
(b) the captured ResNet-50 step at ``--batch`` synthetic 224 x 224 images resident on the device, fp32 (TF32)
    and bf16 (the compute twin), with no teacher, a ResNet-50 teacher and a ResNet-152 teacher.  Each arm is a
    GossipTrainer warmed up and captured, then ``--steps`` replays timed with CUDA events; the arms of a dtype
    are alternated ``--repeats`` times and the median ms/step is printed with the own-kernel launches per
    step and the arm's own peak device memory: the most it allocated, above what was allocated before it, while
    it was built, warmed up and captured.  A throwaway arm runs first, so that the library's algorithm search
    is in no measured arm's peak.

    python benchmarks/distill_bench.py [--batch 256] [--steps 20] [--repeats 5]

Prints the card name, power limit and max SM clock with the numbers, and one JSON line.
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stochastic_gradient_push_b200 as sgp                       # noqa: E402
from stochastic_gradient_push_b200 import models                 # noqa: E402
from stochastic_gradient_push_b200.ops.fused_loss import (FusedCrossEntropyWithAccuracy,  # noqa: E402
                                                          fused_cross_entropy)

DEV = torch.device('cuda', 0)


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader',
                              '-i', '0'], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30)
        power = out.stdout.strip()
    except Exception as e:                          # noqa
        power = 'unknown (%s)' % e
    return name, power


def _events_ms(fn, iters, repeats):
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) / iters)
    return statistics.median(times)


def _torch_composition(z, t, u, alpha, temp):
    loss = (1 - alpha) * F.cross_entropy(z.float(), t) + alpha * temp * temp * F.kl_div(
        F.log_softmax(z.float() / temp, 1), F.log_softmax(u.float() / temp, 1), reduction='batchmean',
        log_target=True)
    with torch.no_grad():
        _, pred = z.float().topk(5, 1, True, True)
        hit = pred.eq(t.view(-1, 1))
        metrics = torch.stack([loss.detach(), hit[:, :1].float().sum() * (100.0 / z.shape[0]),
                               hit.float().sum() * (100.0 / z.shape[0])])
    return loss, metrics


def loss_bench(args):
    out = {}
    for dtype in (torch.float32, torch.bfloat16):
        g = torch.Generator(device='cuda').manual_seed(0)
        z = (torch.randn(args.batch, 1000, device=DEV, generator=g) * 3).to(dtype).requires_grad_(True)
        u = (torch.randn(args.batch, 1000, device=DEV, generator=g) * 3).to(dtype)
        t = torch.randint(0, 1000, (args.batch,), device=DEV, generator=g)

        def fused():
            loss, _ = fused_cross_entropy(z, t, teacher_logits=u, distill_alpha=0.5, distill_temperature=2.0)
            loss.backward()

        def plain():
            loss, _ = fused_cross_entropy(z, t)
            loss.backward()

        def composed():
            loss, _ = _torch_composition(z, t, u, 0.5, 2.0)
            loss.backward()
        r = {name: _events_ms(fn, args.loss_iters, args.repeats)
             for name, fn in (('fused_distill', fused), ('torch_composition', composed), ('fused_xent', plain))}
        out[str(dtype).replace('torch.', '')] = r
        print('loss fwd+bwd %s, %d x 1000: fused distillation %.4f ms, torch composition %.4f ms, fused '
              'cross-entropy without a teacher %.4f ms' % (dtype, args.batch, r['fused_distill'],
                                                          r['torch_composition'], r['fused_xent']))
    return out


def _trainer(twin, teacher_name):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    torch.manual_seed(0)
    net = models.resnet50().to(DEV).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                               heartbeat_timeout=60, compute_dtype=torch.bfloat16 if twin else None)
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, weight_decay=1e-4)
    teacher, crit = None, FusedCrossEntropyWithAccuracy()
    if teacher_name is not None:
        teacher = models.MODEL_ZOO[teacher_name]().to(DEV).to(memory_format=torch.channels_last)
        crit = FusedCrossEntropyWithAccuracy(distill_alpha=0.5, distill_temperature=2.0)
    return GossipTrainer(model, opt, crit, amp_dtype=torch.bfloat16 if twin else None, teacher=teacher)


def _timed(tr, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record(tr.stream)
    for _ in range(steps):
        tr.step_resident()
    b.record(tr.stream)
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def _warmed(twin, teacher, x, y):
    tr = _trainer(twin, teacher)
    for _ in range(5):                               # eager warm-up steps, then the capture
        tr.step(x, y)
    tr.finish()
    return tr


def step_bench(args, twin, x, y):
    # a throwaway arm first: the library's algorithm search (and its workspace) happens there, so that no
    # measured arm's peak includes it
    _warmed(twin, None, x, y)
    gc.collect()
    torch.cuda.empty_cache()
    arms, peak = {}, {}
    for teacher in (None, 'resnet50', 'resnet152'):
        # each arm's own peak: the most it allocated above what the earlier (live) arms hold
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        arms[teacher or 'none'] = _warmed(twin, teacher, x, y)
        peak[teacher or 'none'] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    times = {k: [] for k in arms}
    for _ in range(args.repeats):
        for k, tr in arms.items():
            times[k].append(_timed(tr, args.steps))
    out = {}
    for k, tr in arms.items():
        out[k] = dict(ms_per_step=statistics.median(times[k]), spread_ms=max(times[k]) - min(times[k]),
                      launches_per_step=tr.own_launches_per_step, peak_gib=peak[k])
    del arms, tr
    gc.collect()
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--loss_iters', type=int, default=200)
    args = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    name, power = _card()
    print('card: %s, power limit / max SM clock: %s' % (name, power))
    out = dict(card=name, power=power, batch=args.batch, loss=loss_bench(args))
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(args.batch, 3, 224, 224, generator=gen).pin_memory()
    y = torch.randint(0, 1000, (args.batch,), generator=gen).pin_memory()
    for label, twin in (('fp32', False), ('bf16', True)):
        r = step_bench(args, twin, x, y)
        out[label] = r
        for k, v in r.items():
            print('%s ResNet-50 step, batch %d, teacher %s: %.2f ms/step (spread %.2f), %d launches, peak %.1f GiB'
                  % (label, args.batch, k, v['ms_per_step'], v['spread_ms'], v['launches_per_step'], v['peak_gib']))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
