#!/usr/bin/env python
"""
HBM rate of every distinct fp32 BatchNorm streaming launch of the headline step
(ResNet-50, batch 256), against a same-size ``dst.copy_(src)``.

    python benchmarks/bn_bandwidth.py [--batch-size 256] [--iters 20] [--maps 0,1]
                                      [--sweep] [--out DIR]

The launch list comes from the model: a forward hook on every BatchNorm records its input
shape, and the block structure says which kernels its forward and backward run (a BN after
a 1x1 / stride-1 convolution gets its statistics from the GEMM epilogue; a bottleneck's bn3
backward reduction runs in the next block's conv1 dgrad, except for the network's last
block).  Each kernel is timed alone with CUDA events, the L2 flushed before every launch;
``--maps 0,1`` alternates the consecutive (0) and split (1) fp32 channel maps launch by
launch.  Bytes are computed from the shapes.  ``--sweep`` also times the split map at other
grid sizes (CTAs per SM).  Prints the card name and power limit; DIR/bn_bandwidth.json
holds every number.
"""

from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from collections import OrderedDict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SM_COUNT = 132


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=20).stdout
        return out.strip().splitlines()[0]
    except Exception as e:          # pragma: no cover
        return 'nvidia-smi unavailable: %r' % e


def bn_layers(batch):
    """[(name, C, M, kind)] for every BatchNorm of ResNet-50 at ``batch``; kind is 'stem',
    'bn1', 'bn2', 'bn3', 'bn3_last' or 'ds' / 'ds_s1' (downsample after a stride-2 / stride-1
    convolution)."""
    import torch
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.ops.fused_bn import FusedBatchNormAct2d
    net = models.resnet50().eval()
    shapes = {}
    hooks = [m.register_forward_hook(lambda m, i, o, n=n: shapes.__setitem__(n, tuple(i[0].shape)))
             for n, m in net.named_modules() if isinstance(m, FusedBatchNormAct2d)]
    with torch.no_grad():
        net(torch.zeros(1, 3, 224, 224))
    for h in hooks:
        h.remove()
    mods = dict(net.named_modules())
    last_bn3 = [n for n in shapes if n.endswith('.bn3')][-1]
    out = []
    for n, (_, C, H, W) in shapes.items():
        leaf = n.split('.')[-1]
        if n == 'bn1':
            kind = 'stem'
        elif n.endswith('downsample.1'):
            kind = 'ds' if mods[n[:-1] + '0'].stride != (1, 1) else 'ds_s1'
        elif leaf == 'bn3':
            kind = 'bn3_last' if n == last_bn3 else 'bn3'
        else:
            kind = leaf
        out.append((n, C, batch * H * W, kind))
    return out


def launches(layers):
    """distinct (kernel, variant, M, C) -> number of launches per step"""
    cnt = OrderedDict()

    def add(*key):
        cnt[key] = cnt.get(key, 0) + 1
    for _, C, M, kind in layers:
        relu = kind in ('stem', 'bn1', 'bn2')
        if kind in ('stem', 'bn2', 'ds'):                   # statistics not from a GEMM epilogue
            add('stats', '', M, C)
        add('apply', 'relu' if relu else ('add+relu+mask' if kind.startswith('bn3') else 'plain'), M, C)
        if relu:
            add('reduce', 'mode 1', M, C)
        elif kind in ('ds', 'ds_s1'):
            add('reduce', 'mode 0', M, C)
        elif kind == 'bn3_last':
            add('reduce', 'mode 2', M, C)
        add('dx', 'mode 1' if relu else 'mode 0', M, C)
    return cnt


def nbytes(kernel, variant, M, C):
    t = M * C * 4
    if kernel == 'stats':
        return t
    if kernel == 'apply':
        return (3 if 'add' in variant else 2) * t + (M * C // 8 if 'mask' in variant else 0)
    if kernel == 'reduce':
        return 4 * t if variant == 'mode 2' else 2 * t
    return 3 * t                                           # dx


def default_grid(kernel, variant, M, C):
    """the grid the launchers pick (bn_grid in csrc/bn_kernels.cu)"""
    per_sm = {'stats': 4, 'reduce': 3, 'dx': 6}.get(kernel, 6 if 'add' in variant else 8)
    tpr = C // 8
    rpi = 256 // tpr
    g = -(-(-(-M // rpi)) // 4)
    return max(1, min(g, SM_COUNT * per_sm))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch-size', type=int, default=256)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--maps', default='0,1')
    ap.add_argument('--sweep', action='store_true')
    ap.add_argument('--list', action='store_true', help='print the launch list and exit (no GPU)')
    ap.add_argument('--out', default='bn_bandwidth_out')
    args = ap.parse_args()

    layers = bn_layers(args.batch_size)
    todo = launches(layers)
    if args.list:
        for (k, v, M, C), n in todo.items():
            print('%-7s %-14s M=%-8d C=%-5d x%-2d %6.1f MB' % (k, v, M, C, n, nbytes(k, v, M, C) / 1e6))
        print('%d BN layers, %d distinct launches, %d launches per step'
              % (len(layers), len(todo), sum(todo.values())))
        return

    import torch
    from stochastic_gradient_push_b200.ops import native
    assert torch.cuda.is_available(), 'bn_bandwidth.py measures on a GPU'
    Cx = native.load()
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    maps = [int(m) for m in args.maps.split(',')]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    g = torch.Generator(device=dev).manual_seed(0)

    def timed(fn, n):
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]
        for e0, e1 in ev:
            flush.zero_()
            e0.record()
            fn()
            e1.record()
        torch.cuda.synchronize()
        ts = sorted(e0.elapsed_time(e1) for e0, e1 in ev)
        return ts[len(ts) // 2]

    print('card (name, power limit, max SM clock): %s' % card())
    rows = []
    prev_map = Cx.bn_f32_map()
    cache = {}
    for (kern, var, M, C), count in todo.items():
        if (M, C) not in cache:
            cache.clear()
            torch.cuda.empty_cache()
            mk = lambda: torch.randn(M, C, device=dev, generator=g)       # noqa: E731
            x, r, dy = mk(), mk(), mk()
            coef = torch.stack([x.mean(0), x.var(0).add(1e-5).rsqrt(), torch.rand(C, device=dev) + 0.5,
                                torch.randn(C, device=dev) * 0.1]).contiguous()
            c23 = (torch.randn(2, C, device=dev) * 0.1).contiguous()
            mask = torch.empty(M, C // 8, dtype=torch.uint8, device=dev)
            cache[(M, C)] = (x, r, dy, coef, c23, mask)
        x, r, dy, coef, c23, mask = cache[(M, C)]

        def fn_for(G):
            if kern == 'stats':
                return lambda: Cx.bn_kernel_stats(x, G)
            if kern == 'apply':
                add = 'add' in var
                return lambda: Cx.bn_kernel_apply(x, r if add else None, coef, var != 'plain',
                                                  mask if 'mask' in var else None, G)
            if kern == 'reduce':
                mode = int(var[-1])
                return lambda: Cx.bn_kernel_reduce(mode, dy, x, r if mode == 2 else None, coef, G)
            return lambda: Cx.bn_kernel_dx(int(var[-1]), dy, x, coef, c23, G)

        b = nbytes(kern, var, M, C)
        dst = torch.empty(M * C, device=dev)
        src = x.view(-1)
        row = {'kernel': kern, 'variant': var, 'M': M, 'C': C, 'launches_per_step': count, 'bytes': b,
               'grid': default_grid(kern, var, M, C)}
        for m in maps:                      # warm-up of every arm
            Cx.bn_f32_map(m)
            fn_for(0)()
        dst.copy_(src)
        ms = {m: [] for m in maps}
        copy_ms = []
        for _ in range(3):                  # arms alternated
            for m in maps:
                Cx.bn_f32_map(m)
                ms[m].append(timed(fn_for(0), args.iters))
            copy_ms.append(timed(lambda: dst.copy_(src), args.iters))
        for m in maps:
            t = sorted(ms[m])[1]
            row['map%d_ms' % m] = round(t, 4)
            row['map%d_TBps' % m] = round(b / t / 1e9, 3)
        tc = sorted(copy_ms)[1]
        row['copy_TBps'] = round(2 * M * C * 4 / tc / 1e9, 3)
        if args.sweep and 1 in maps:
            Cx.bn_f32_map(1)
            sw = {}
            for per_sm in (2, 3, 4, 6, 8, 12, 16):
                G = SM_COUNT * per_sm
                fn = fn_for(G)
                fn()
                sw[per_sm] = round(b / timed(fn, args.iters) / 1e9, 3)
            row['map1_sweep_TBps_by_ctas_per_sm'] = sw
        rows.append(row)
        print('%-7s %-14s M=%-8d C=%-5d x%-2d %s copy %.2f TB/s%s' % (
            kern, var, M, C, count,
            '  '.join('map%d %.3f ms %.2f TB/s' % (m, row['map%d_ms' % m], row['map%d_TBps' % m]) for m in maps),
            row['copy_TBps'], ('  sweep ' + str(row['map1_sweep_TBps_by_ctas_per_sm'])) if 'map1_sweep_TBps_by_ctas_per_sm' in row else ''),
            flush=True)
        del dst
    Cx.bn_f32_map(prev_map)

    summary = {}
    for kern in ('stats', 'apply', 'reduce', 'dx'):
        sel = [r for r in rows if r['kernel'] == kern]
        s = {'bytes_per_step': sum(r['bytes'] * r['launches_per_step'] for r in sel)}
        for m in maps:
            s['map%d_ms_per_step' % m] = round(sum(r['map%d_ms' % m] * r['launches_per_step'] for r in sel), 3)
            s['map%d_TBps' % m] = round(s['bytes_per_step'] / s['map%d_ms_per_step' % m] / 1e9, 3)
        summary[kern] = s
        print('%-7s per step: %s' % (kern, '  '.join('map%d %.3f ms (%.2f TB/s)' % (
            m, s['map%d_ms_per_step' % m], s['map%d_TBps' % m]) for m in maps)))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'bn_bandwidth.json'), 'w') as f:
        json.dump({'card': card(), 'batch': args.batch_size, 'rows': rows, 'per_step': summary}, f, indent=1)


if __name__ == '__main__':
    main()
