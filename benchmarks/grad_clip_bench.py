"""Cost of gradient-norm clipping in FusedGossipSGD (``max_grad_norm=``, ``SGP_F_CLIP``) at ResNet-50
size on one GPU.

    python benchmarks/grad_clip_bench.py [--launches 200] [--rounds 5] [--batch 256] [--steps 30]

Two measurements:
  (a) the norm + clip-finalize kernels alone (``GossipEngine.clip_update``) on the ResNet-50 arena,
      fp32 gradients and the bf16 compute twin (bf16 gradient + fp32 g2), in us and in GB/s of the
      gradient bytes they must read (4 B per element, 6 B with the twin), computed from the shapes;
  (b) the captured one-rank training step (fp32, batch ``--batch``) without clipping and with
      ``max_grad_norm`` on, two captured graphs of one trainer replayed in alternated blocks.
Device-timed with CUDA events.  Prints the card name and power limit with the numbers, and one
JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import stochastic_gradient_push_b200 as sgp                                # noqa: E402
from stochastic_gradient_push_b200 import models                           # noqa: E402

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


def _model(dev, twin):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    torch.manual_seed(0)
    net = models.resnet50().to(dev).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                               heartbeat_timeout=60, compute_dtype=torch.bfloat16 if twin else None)
    assert model.transport == 'nvlink'
    opt = FusedGossipSGD(model, lr=0.01, momentum=0.9, weight_decay=1e-4, nesterov=True, max_grad_norm=1.0)
    return net, model, opt


def kernels(args, dev, stream):
    out = {}
    for twin in (False, True):
        net, model, opt = _model(dev, twin)
        e = model.engine
        arena = model._arenas[torch.float32]
        elements = sum(arena.numels)
        opt.grad_flat[torch.float32].normal_()
        if opt.grad_lo is not None:
            opt.grad_lo.normal_()
        opt.set_engine_hyper(e)
        fn = e.clip_update
        _time(fn, 20, stream)                          # warm-up
        ms = [_time(fn, args.launches, stream) for _ in range(args.rounds)]
        med = statistics.median(ms)
        nbytes = elements * (6 if twin else 4)
        rate = nbytes / (med * 1e-3)
        key = 'bf16_twin' if twin else 'fp32'
        out[key] = {'us_median': round(med * 1e3, 2), 'us_min': round(min(ms) * 1e3, 2),
                    'us_max': round(max(ms) * 1e3, 2), 'elements': elements, 'tiles': e.ctx.lars_tiles(),
                    'bytes': nbytes, 'GB_per_s': round(rate / 1e9, 1),
                    'share_of_3.35TB/s': round(rate / HBM_BYTES_PER_S, 3)}
        print('norm + finalize %-9s %7.2f us (min %.2f, max %.2f), %d elements, %.0f GB/s = %.1f%% of 3.35 TB/s'
              % (key, med * 1e3, min(ms) * 1e3, max(ms) * 1e3, elements, rate / 1e9, 100 * rate / HBM_BYTES_PER_S))
        del net, model, opt, e
        torch.cuda.empty_cache()
    return out


def step(args, dev):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    torch.manual_seed(0)
    net = models.resnet50().to(dev).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                               heartbeat_timeout=60)
    opt = FusedGossipSGD(model, lr=0.01, momentum=0.9, weight_decay=1e-4, nesterov=True)
    tr = GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=True, warmup_iters=3)
    x = torch.randn(args.batch, 3, 224, 224).pin_memory()
    y = torch.randint(0, 1000, (args.batch,)).pin_memory()
    for _ in range(4):                                  # 3 eager steps, then the capture without clipping
        tr.step(x, y)
    tr.finish()
    graphs = {'off': (tr.graph, tr.own_launches_per_step)}
    # a threshold far above the norm: the clip kernels run every step, the update is unchanged
    opt.max_grad_norm = 1e6
    tr._set_lr()
    with torch.cuda.stream(tr.stream):
        tr._capture()
    graphs['clip'] = (tr.graph, tr.own_launches_per_step)
    step_ms = {k: [] for k in graphs}
    for rep in range(args.repeats + 1):                 # the first block of each arm is warm-up
        for k, (g, _) in graphs.items():
            tr.graph = g
            t = _time(tr.step_resident, args.steps, tr.stream)
            if rep:
                step_ms[k].append(t)
    tr.finish()
    out = {k: {'ms_per_step': [round(t, 3) for t in v], 'mean': round(statistics.mean(v), 3),
               'own_launches_per_step': graphs[k][1]} for k, v in step_ms.items()}
    for k, v in out.items():
        print('step %-5s %s ms (mean %.3f), %d own launches / step'
              % (k, v['ms_per_step'], v['mean'], v['own_launches_per_step']))
    delta = out['clip']['mean'] - out['off']['mean']
    print('clipping cost per step: %.3f ms (%.2f%%)' % (delta, 100 * delta / out['off']['mean']))
    return out, delta


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('grad_clip_bench.py measures on the GPU; no CUDA device found')
    torch.backends.cudnn.benchmark = True
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    card, power = _card()
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    kern = kernels(args, dev, stream)
    st, delta = step(args, dev)
    print('card: %s, power limit / max SM clock: %s' % (card, power))
    print(json.dumps({'card': card, 'power_limit,max_sm_clock': power, 'kernels': kern, 'batch': args.batch,
                      'step': st, 'clip_ms_per_step': round(delta, 3)}))


if __name__ == '__main__':
    main()
