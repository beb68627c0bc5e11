"""Cost of the GPU input augmentation (``data.GpuAugment``) per 256-image batch, stored at S = 256 and
cropped to 224, fp32 and bf16 output, arms alternated in one process:

* ``grid_sample``: today's default path (``GpuAugment()``: RandomResizedCrop + flip + normalisation as
  one batched ``grid_sample``);
* ``kernel_identity``: the augment kernel with every op forced to Identity and no erasing;
* ``kernel_ta_erase``: ``GpuAugment(auto_augment='ta_wide', random_erase=0.1)`` -- host draws, one
  pinned H2D copy of the per-image rows and the kernel;
* ``kernel_ra``: ``GpuAugment(auto_augment='ra', ra_num_ops=2, ra_magnitude=9, random_erase=0.1)``, the
  same steps with RandAugment's two-op chain rows;
* ``kernel_imagenet``: ``GpuAugment(auto_augment='imagenet', random_erase=0.1)``, AutoAugment's
  ImageNet policy.

Each arm is timed with CUDA events around ``--reps`` calls, the median of ``--rounds`` rounds reported
with its min / max (ms per batch, host work included, as the training loop sees it).  The kernel alone
(``kernel_only``: the rows staged once, then launches back to back) is timed the same way for the
identity, TrivialAugment, RandAugment and AutoAugment rows, and reported with the bytes it must move,
computed from the shapes (uint8 input read once, output written once), over its time.  A chain op that
reads other pixels (geometric, Sharpness) before the last op also writes and reads back 3 out^2 bytes
per image through the output buffer; ``staging_bytes`` counts them for the drawn rows.  The input batch (50 MB) and the
output (154 MB fp32) do not fit in the 50 MB L2, so no flush is needed.

    python benchmarks/gpu_augment_bench.py [--batch 256] [--store 256] [--out 224] [--rounds 15] [--reps 10]

The host's share of a call, ``sample_params`` + ``kernel_rows`` per policy, is timed on the CPU clock.
Prints one JSON line with the card name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stochastic_gradient_push_b200.data.shards import (AUGMENT_OPS, GEOMETRIC_OPS, AugmentParams,  # noqa: E402
                                                       GpuAugment)
from stochastic_gradient_push_b200.ops import native                              # noqa: E402


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader',
                              '-i', '0'], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30)
        power = out.stdout.strip()
    except Exception as e:                          # noqa
        power = 'unknown (%s)' % e
    return name, power


def _alternate(arms, rounds, reps):
    """arms: name -> callable enqueuing one unit of work; returns name -> sorted ms per unit"""
    for fn in arms.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    stream = torch.cuda.current_stream()
    for _ in range(rounds):
        for k, fn in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            for _ in range(reps):
                fn()
            b.record(stream)
            b.synchronize()
            times[k].append(a.elapsed_time(b) / reps)
    return {k: sorted(v) for k, v in times.items()}


def _staging_bytes(op, out):
    """bytes the kernel stages through the output buffer for chain ops ``op`` [n, K]: 2 x 3 out^2 for each
    geometric / Sharpness op before the last non-Identity op of its row"""
    n = 0
    for ops in op.tolist():
        last = max([k for k, o in enumerate(ops) if o != 0], default=0)
        n += sum(AUGMENT_OPS[o] in GEOMETRIC_OPS or AUGMENT_OPS[o] == 'Sharpness' for o in ops[:last])
    return n * 2 * 3 * out * out


def _summary(v):
    return {'median_ms': round(v[len(v) // 2], 4), 'min_ms': round(v[0], 4), 'max_ms': round(v[-1], 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--store', type=int, default=256)
    ap.add_argument('--out', type=int, default=224)
    ap.add_argument('--rounds', type=int, default=15)
    ap.add_argument('--reps', type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('gpu_augment_bench.py needs a CUDA device')
    dev = torch.device('cuda', 0)
    C = native.load()
    B, S, O = args.batch, args.store, args.out
    x = torch.randint(0, 256, (B, S, S, 3), dtype=torch.uint8, device=dev)
    name, power = _card()
    result = {'bench': 'gpu_augment', 'gpu': name, 'power_limit_max_sm_clock': power, 'batch': B, 'store': S,
              'out': O, 'rounds': args.rounds, 'reps': args.reps}
    for dtype, tag in ((torch.float32, 'fp32'), (torch.bfloat16, 'bf16')):
        plain = GpuAugment(out_size=O, dtype=dtype, seed=1)
        ident = GpuAugment(out_size=O, dtype=dtype, seed=1, auto_augment='ta_wide')
        ta = GpuAugment(out_size=O, dtype=dtype, seed=1, auto_augment='ta_wide', random_erase=0.1)
        ra = GpuAugment(out_size=O, dtype=dtype, seed=1, auto_augment='ra', ra_num_ops=2, ra_magnitude=9,
                        random_erase=0.1)
        aa = GpuAugment(out_size=O, dtype=dtype, seed=1, auto_augment='imagenet', random_erase=0.1)
        cx, cy, w, h, flip = ident.sample_boxes(B)
        zeros = torch.zeros(B, dtype=torch.int64)
        p_ident = AugmentParams(cx, cy, w, h, flip, zeros, zeros.double(), torch.zeros(B, 4, dtype=torch.int64))
        arms = {
            'grid_sample': lambda: plain(x),
            'kernel_identity': lambda: ident.apply(x, p_ident),
            'kernel_ta_erase': lambda: ta(x),
            'kernel_ra': lambda: ra(x),
            'kernel_imagenet': lambda: aa(x),
        }
        y = torch.empty(B, 3, O, O, dtype=dtype, device=dev, memory_format=torch.channels_last)
        mean, inv = ident._norm('cpu')
        mean, inv = mean.view(-1).tolist(), inv.view(-1).tolist()
        rows_ident = ident._stage_rows(ident.kernel_rows(p_ident, S), dev)
        rows_ta = ta._stage_rows(ta.kernel_rows(ta.sample_params(B), S), dev)
        arms['kernel_only_identity'] = lambda: C.gpu_augment(x, rows_ident, y, mean, inv)
        p_ra, p_aa = ra.sample_params(B), aa.sample_params(B)
        rows_ra = ra._stage_rows(ra.kernel_rows(p_ra, S), dev)
        rows_aa = aa._stage_rows(aa.kernel_rows(p_aa, S), dev)
        arms['kernel_only_ta_erase'] = lambda: C.gpu_augment(x, rows_ta, y, mean, inv)
        arms['kernel_only_ra'] = lambda: C.gpu_augment(x, rows_ra, y, mean, inv)
        arms['kernel_only_imagenet'] = lambda: C.gpu_augment(x, rows_aa, y, mean, inv)
        times = _alternate(arms, args.rounds, args.reps)
        nbytes = B * S * S * 3 + B * O * O * 3 * y.element_size()
        res = {k: _summary(v) for k, v in times.items()}
        for k in ('kernel_only_identity', 'kernel_only_ta_erase', 'kernel_only_ra', 'kernel_only_imagenet'):
            res[k]['GBps'] = round(nbytes / (res[k]['median_ms'] * 1e-3) / 1e9, 1)
        res['kernel_only_ra']['staging_bytes'] = _staging_bytes(p_ra.op, O)
        res['kernel_only_imagenet']['staging_bytes'] = _staging_bytes(p_aa.op, O)
        res['bytes_per_batch'] = nbytes
        result[tag] = res
    # the host's share of a call: the draws and the rows (median of 50 calls, CPU clock)
    host = {}
    for policy in ('ta_wide', 'ra', 'imagenet'):
        aug = GpuAugment(out_size=O, seed=1, auto_augment=policy, random_erase=0.1)
        ts = []
        for _ in range(50):
            t0 = time.perf_counter()
            aug.kernel_rows(aug.sample_params(B), S)
            ts.append((time.perf_counter() - t0) * 1e3)
        host[policy] = round(sorted(ts)[len(ts) // 2], 4)
    result['host_draws_and_rows_ms'] = host
    print(json.dumps(result))


if __name__ == '__main__':
    main()
