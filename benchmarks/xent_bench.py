"""Fused softmax cross-entropy + prec@1/5 (``csrc/loss_kernels.cu``) with and without label
smoothing: forward + backward at the training step's shape (B = 256 images, C = 1000 classes), for
fp32 and bf16 logits, eps = 0 (the unsmoothed kernels) against eps = 0.1.

    python benchmarks/xent_bench.py [--batch 256] [--classes 1000] [--pairs 200] [--rounds 20]

Each arm is one captured CUDA graph of ``--pairs`` forward + backward pairs (the loss runs inside
the captured training step, so launch gaps are not part of its cost).  After a warm-up the arms'
graphs replay alternately for ``--rounds`` rounds, each replay timed with CUDA events.  Bytes per
pair come from the shapes: the logits read by the forward and the backward, the gradient written,
the targets read twice, the log-sum-exp written and read, and the 3-float metrics.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stochastic_gradient_push_b200.ops import native        # noqa: E402


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader',
                              '-i', '0'], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30)
        power = out.stdout.strip()
    except Exception as e:                          # noqa
        power = 'unknown (%s)' % e
    return name, power


def _bytes_per_pair(B, C, elem):
    return 3 * B * C * elem + 2 * B * 8 + 2 * B * 4 + 3 * 4 + 4


def _graph(C_, logits, target, eps, pairs):
    g = torch.ones(1, device='cuda')
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            _, lse = C_.xent_forward(logits, target, eps)
            C_.xent_backward(logits, target, lse, g, eps)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(pairs):
            _, lse = C_.xent_forward(logits, target, eps)
            C_.xent_backward(logits, target, lse, g, eps)
    return graph


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--classes', type=int, default=1000)
    ap.add_argument('--pairs', type=int, default=200, help='forward + backward pairs per graph replay')
    ap.add_argument('--rounds', type=int, default=20, help='timed replays per arm, alternating')
    ap.add_argument('--eps', type=float, default=0.1)
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark needs a GPU'
    C_ = native.load()
    card, power = _card()
    B, C = args.batch, args.classes
    result = {'card': card, 'power_limit,max_sm_clock': power, 'B': B, 'C': C, 'pairs_per_replay': args.pairs,
              'rounds': args.rounds}
    gen = torch.Generator(device='cuda').manual_seed(0)
    for dtype, label, elem in ((torch.float32, 'fp32', 4), (torch.bfloat16, 'bf16', 2)):
        logits = (torch.randn(B, C, device='cuda', generator=gen) * 3).to(dtype)
        target = torch.randint(0, C, (B,), device='cuda', generator=gen)
        arms = {'eps0': _graph(C_, logits, target, 0.0, args.pairs),
                'eps%g' % args.eps: _graph(C_, logits, target, args.eps, args.pairs)}
        for graph in arms.values():               # warm-up replays
            for _ in range(3):
                graph.replay()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, graph in arms.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                graph.replay()
                b.record()
                b.synchronize()
                times[k].append(a.elapsed_time(b) * 1e3 / args.pairs)      # us per pair
        nbytes = _bytes_per_pair(B, C, elem)
        res = {'bytes_per_pair': nbytes}
        for k, ts in times.items():
            ts = sorted(ts)
            med = ts[len(ts) // 2]
            res[k] = {'us_per_pair_median': round(med, 3), 'us_min': round(ts[0], 3), 'us_max': round(ts[-1], 3),
                      'GB_per_s_median': round(nbytes / med / 1e3, 1)}
        keys = list(arms)
        res['smoothed_over_plain_time'] = round(res[keys[1]]['us_per_pair_median'] /
                                                res[keys[0]]['us_per_pair_median'], 4)
        result[label] = res
        del arms
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
