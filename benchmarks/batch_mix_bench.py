"""Cost of mixup / CutMix on the training step (``ops/batch_mix.py``), three comparisons, each with
its arms alternated in one process:

1. input staging at B = 256, 3 x 224 x 224, fp32 NCHW source: the trainer's plain copy
   (``static_in.copy_(stage)``) against the batch-mix kernel (mixup and CutMix states), to an NHWC
   fp32 destination and to an NHWC bf16 one (the compute twin's input);
2. the fused cross-entropy forward + backward pair (B = 256, C = 1000) without and with ``MIX``;
3. the captured ResNet-50 training step (``GossipTrainer.step``, inputs from pinned host memory,
   one rank) with mixing off and on (mixup alpha 0.2 + CutMix alpha 1.0, ``--step-dtype`` compute).

    python benchmarks/batch_mix_bench.py [--batch 256] [--rounds 20] [--steps 30] [--out FILE]

Every arm is warmed up first; a round times each arm once with CUDA events, and the median over the
rounds is reported with its min / max.  Bytes are computed from the shapes: the staging copy reads
the batch once and writes it once, which is what the mixing kernel moves too.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stochastic_gradient_push_b200.ops import batch_mix as bm    # noqa: E402
from stochastic_gradient_push_b200.ops import native             # noqa: E402


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader',
                              '-i', '0'], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30)
        power = out.stdout.strip()
    except Exception as e:                          # noqa
        power = 'unknown (%s)' % e
    return name, power


def _alternate(arms, rounds, reps, stream=None):
    """arms: name -> callable enqueuing one unit of work; returns name -> sorted us per unit"""
    stream = stream or torch.cuda.current_stream()
    for fn in arms.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            for _ in range(reps):
                fn()
            b.record(stream)
            b.synchronize()
            times[k].append(a.elapsed_time(b) * 1e3 / reps)
    return {k: sorted(v) for k, v in times.items()}


def _summary(ts, nbytes=None):
    med = ts[len(ts) // 2]
    r = {'us_median': round(med, 2), 'us_min': round(ts[0], 2), 'us_max': round(ts[-1], 2)}
    if nbytes:
        r['GB_per_s_median'] = round(nbytes / med / 1e3, 1)
    return r


def staging(args):
    C_ = native.load()
    B, H, W = args.batch, args.image, args.image
    g = torch.Generator(device='cuda').manual_seed(0)
    src = torch.randn(B, 3, H, W, device='cuda', generator=g)
    mixup = bm.BatchMix(mixup_alpha=0.2)
    cutmix = bm.BatchMix(cutmix_alpha=1.0)
    mixup.stage(bm.MixParams(0.37, bm.MIXUP, 0, 0, 0, 0), src.device)
    cutmix.stage(bm.BatchMix(cutmix_alpha=1.0, seed=1).sample(H, W), src.device)
    res = {}
    for label, dtype in (('nhwc_fp32', torch.float32), ('nhwc_bf16', torch.bfloat16)):
        out = torch.empty(B, 3, H, W, device='cuda', dtype=dtype).contiguous(memory_format=torch.channels_last)
        arms = {'copy': lambda: out.copy_(src, non_blocking=True),
                'mixup_kernel': lambda: C_.batch_mix(src, out, mixup.state),
                'cutmix_kernel': lambda: C_.batch_mix(src, out, cutmix.state)}
        times = _alternate(arms, args.rounds, 10)
        nbytes = src.numel() * 4 + out.numel() * out.element_size()
        r = {'bytes': nbytes}
        r.update({k: _summary(v, nbytes) for k, v in times.items()})
        r['mixup_over_copy_time'] = round(r['mixup_kernel']['us_median'] / r['copy']['us_median'], 4)
        r['cutmix_over_copy_time'] = round(r['cutmix_kernel']['us_median'] / r['copy']['us_median'], 4)
        res[label] = r
    return res


def xent(args):
    C_ = native.load()
    B, C = args.batch, 1000
    state = torch.tensor([0.37, 1, 0, 0, 0, 0, 0, 0], device='cuda')
    gr = torch.ones(1, device='cuda')
    gen = torch.Generator(device='cuda').manual_seed(0)
    res = {}
    for label, dtype in (('fp32', torch.float32), ('bf16', torch.bfloat16)):
        logits = (torch.randn(B, C, device='cuda', generator=gen) * 3).to(dtype)
        target = torch.randint(0, C, (B,), device='cuda', generator=gen)

        def graph_of(mix, pairs=200):
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(3):
                    _, lse = C_.xent_forward(logits, target, 0.0, mix)
                    C_.xent_backward(logits, target, lse, gr, 0.0, mix)
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(pairs):
                    _, lse = C_.xent_forward(logits, target, 0.0, mix)
                    C_.xent_backward(logits, target, lse, gr, 0.0, mix)
            return graph
        g0, g1 = graph_of(None), graph_of(state)
        times = _alternate({'one_target': g0.replay, 'mix': g1.replay}, args.rounds, 1)
        r = {k: _summary([t / 200 for t in v]) for k, v in times.items()}
        r['mix_over_one_target_time'] = round(r['mix']['us_median'] / r['one_target']['us_median'], 4)
        res[label] = r
        del g0, g1
    return res


def step(args):
    import stochastic_gradient_push_b200 as sgp
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    dev = torch.device('cuda', 0)
    bf16 = args.step_dtype == 'bf16'
    B = args.batch
    trainers = {}
    for name, mix in (('mix_off', None), ('mix_on', bm.BatchMix(mixup_alpha=0.2, cutmix_alpha=1.0, seed=0))):
        torch.manual_seed(1)
        net = models.resnet50()
        models.init_imagenet_in_1hr(net)
        net = net.to(dev).to(memory_format=torch.channels_last)
        model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                                   verbose=False, heartbeat_timeout=60,
                                   compute_dtype=torch.bfloat16 if bf16 else None)
        opt = FusedGossipSGD(model, lr=0.1 * B / 256, momentum=0.9, weight_decay=1e-4, nesterov=True)
        trainers[name] = GossipTrainer(model, opt, amp_dtype=torch.bfloat16 if bf16 else None, batch_mix=mix)
    g = torch.Generator().manual_seed(1234)
    pool = [(torch.randn(B, 3, args.image, args.image, generator=g).pin_memory(),
             torch.randint(0, 1000, (B,), generator=g).pin_memory()) for _ in range(4)]
    for tr in trainers.values():
        for i in range(6):                       # eager warm-up, capture, replays
            tr.step(*pool[i % len(pool)])
        tr.finish()
    times = {k: [] for k in trainers}
    for _ in range(args.step_rounds):
        for k, tr in trainers.items():
            tr.prefetch(*pool[0])
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(tr.stream)
            for i in range(args.steps):
                nxt = pool[(i + 1) % len(pool)]
                tr.step(None, None, nxt[0], nxt[1])
            b.record(tr.stream)
            b.synchronize()
            times[k].append(a.elapsed_time(b) / args.steps)          # ms per step
    res = {'compute': args.step_dtype, 'steps_per_window': args.steps, 'windows': args.step_rounds}
    for k, ts in times.items():
        ts = sorted(ts)
        res[k] = {'ms_per_step_median': round(ts[len(ts) // 2], 3), 'ms_min': round(ts[0], 3),
                  'ms_max': round(ts[-1], 3), 'all': [round(t, 3) for t in ts]}
    res['on_over_off_time'] = round(res['mix_on']['ms_per_step_median'] / res['mix_off']['ms_per_step_median'], 4)
    for tr in trainers.values():
        tr.finish()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--image', type=int, default=224)
    ap.add_argument('--rounds', type=int, default=20, help='alternating rounds of the kernel comparisons')
    ap.add_argument('--steps', type=int, default=30, help='training steps per timed window')
    ap.add_argument('--step-rounds', type=int, default=6, help='alternating windows per step arm')
    ap.add_argument('--step-dtype', default='bf16', choices=['bf16', 'fp32'],
                    help='compute precision of the training-step comparison (bf16: the compute twin, whose '
                         'input the mixing kernel writes in bf16)')
    ap.add_argument('--skip-step', action='store_true')
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'
    card, power = _card()
    result = {'card': card, 'power_limit,max_sm_clock': power, 'B': args.batch, 'image': args.image,
              'staging': staging(args), 'xent_pair': xent(args)}
    if not args.skip_step:
        result['train_step'] = step(args)
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
