"""Cost of the weight EMA (``ops/model_ema.py``, ``ema_update_kernel``), in one process:

1. kernel: one ``ModelEma.update()`` over ResNet-50's tracked set (the fp32 parameter arena of a
   one-rank ``GossipDataParallel`` as one segment, plus every BatchNorm running statistic) against
   ``torch._foreach_lerp_`` over the same tensors.  CUDA events around ``--launches`` launches after
   warm-up, median over ``--rounds`` rounds with the arms alternated.  The working set (about 300 MB)
   is larger than L2, so no flush is needed.  Achieved bytes/s counts 12 B per tracked element (read s,
   read e, write e) against the H100 SXM data-sheet 3.35 TB/s;
2. step: the captured one-rank ``GossipTrainer`` ResNet-50 step at ``--batch`` fp32 (TF32) without
   and with ``ema=``: both graphs are captured by one trainer (one memory pool) and replayed in
   alternating blocks of ``--steps`` steps, ``--repeats`` blocks each.

    python benchmarks/ema_bench.py [--launches 200] [--rounds 5] [--batch 256] [--steps 30] [--repeats 3]

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
from stochastic_gradient_push_b200.ops.model_ema import ModelEma  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader',
                              '-i', '0'], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30)
        power = out.stdout.strip()
    except Exception as e:                          # noqa
        power = 'unknown (%s)' % e
    return name, power


def _time(fn, n, stream):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(stream):
        a.record(stream)
        for _ in range(n):
            fn()
        b.record(stream)
    b.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('ema_bench.py measures on the GPU; no CUDA device found')
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    torch.backends.cudnn.benchmark = True
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    card, power = _card()
    torch.manual_seed(0)
    net = models.resnet50().to(dev).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                               heartbeat_timeout=60)
    assert model.transport == 'nvlink'
    ema = ModelEma(model, decay=0.9999)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())

    # ---- 1. kernel ---------------------------------------------------------------------------- #
    srcs = {k: v for k, v in net.state_dict(keep_vars=True).items() if v.is_floating_point()}
    e_list = [ema._entry_view(*ema._entries[k]) for k in srcs]
    s_list = [v.detach() for v in srcs.values()]
    payload = sum(v.numel() for v in s_list)
    w = 1.0 - 0.9999
    arms = {'ema_kernel': ema.update, 'foreach_lerp': lambda: torch._foreach_lerp_(e_list, s_list, w)}
    for fn in arms.values():
        _time(fn, 20, stream)                          # warm-up
    ms = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, fn in arms.items():
            ms[k].append(_time(fn, args.launches, stream))
    kernel = {}
    for k, v in ms.items():
        med = statistics.median(v)
        n_el = ema.numel if k == 'ema_kernel' else payload
        rate = 12.0 * n_el / (med * 1e-3)
        kernel[k] = {'us_per_launch_median': round(med * 1e3, 2), 'us_min': round(min(v) * 1e3, 2),
                     'us_max': round(max(v) * 1e3, 2), 'tracked_elements': n_el,
                     'GB_per_s': round(rate / 1e9, 1), 'share_of_3.35TB/s': round(rate / HBM_BYTES_PER_S, 3)}
        print('%-13s %8.2f us / update (min %.2f, max %.2f), %d elements, %.0f GB/s = %.1f%% of 3.35 TB/s'
              % (k, med * 1e3, min(v) * 1e3, max(v) * 1e3, n_el, rate / 1e9, 100 * rate / HBM_BYTES_PER_S))

    # ---- 2. captured training step without / with the EMA ---------------------------------------- #
    opt = FusedGossipSGD(model, lr=0.01, momentum=0.9, weight_decay=1e-4, nesterov=True)
    tr = GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=True, warmup_iters=3)
    x = torch.randn(args.batch, 3, 224, 224).pin_memory()
    y = torch.randint(0, 1000, (args.batch,)).pin_memory()
    for _ in range(4):                                  # 3 eager steps, then the capture without EMA
        tr.step(x, y)
    tr.finish()
    graphs = {'no_ema': (tr.graph, None, tr.own_launches_per_step)}
    tr.ema = ema
    ema._stream = tr.stream
    with torch.cuda.stream(tr.stream):
        tr._capture()
    graphs['ema'] = (tr.graph, ema, tr.own_launches_per_step)
    step_ms = {k: [] for k in graphs}
    for rep in range(args.repeats + 1):                 # the first block of each arm is warm-up
        for k, (g, e, _) in graphs.items():
            tr.graph, tr.ema = g, e
            t = _time(tr.step_resident, args.steps, tr.stream)
            if rep:
                step_ms[k].append(t)
    tr.finish()
    step = {k: {'ms_per_step': [round(t, 3) for t in v], 'mean': round(statistics.mean(v), 3),
                'own_launches_per_step': graphs[k][2]} for k, v in step_ms.items()}
    delta = step['ema']['mean'] - step['no_ema']['mean']
    for k, v in step.items():
        print('step %-7s %s ms (mean %.3f), %d own launches / step'
              % (k, v['ms_per_step'], v['mean'], v['own_launches_per_step']))
    print('EMA cost per step: %.3f ms (%.2f%%)' % (delta, 100 * delta / step['no_ema']['mean']))
    print('card: %s, power limit / max SM clock: %s' % (card, power))
    print(json.dumps({'card': card, 'power_limit,max_sm_clock': power, 'kernel': kernel, 'batch': args.batch,
                      'step': step, 'ema_ms_per_step': round(delta, 3)}))


if __name__ == '__main__':
    main()
