"""Per-layer A/B of the ResNet-50 1x1 convolutions (forward, training mode):

    library conv  + fused-BN (stats pass + finalize + apply)      <- default path
    wgmma GEMM with the statistics in its epilogue + finalize + apply

and of the conv1 dgrad of every bottleneck (library dgrad + gradient-accumulation add vs the
same GEMM with the skip gradient added in its epilogue).

CUDA-event timing, L2 flushed between iterations, median of ``--iters`` runs.

    python benchmarks/conv1x1_bench.py --batch 256 --out gpurun_out/conv1x1_bench.json
"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from stochastic_gradient_push_b200.ops import fused_bn, native          # noqa: E402
from stochastic_gradient_push_b200.ops.fused_bn import FusedBatchNormAct2d, conv_bn_act   # noqa: E402

# (H=W, C_in, C_out, residual) of every stride-1 1x1 convolution in ResNet-50, with multiplicity
LAYERS = [
    (56, 64, 64, False, 1), (56, 64, 256, False, 1), (56, 64, 256, True, 3), (56, 256, 64, False, 2),
    (56, 256, 128, False, 1), (28, 128, 512, True, 4), (28, 512, 128, False, 3),
    (28, 512, 256, False, 1), (14, 256, 1024, True, 6), (14, 1024, 256, False, 5),
    (14, 1024, 512, False, 1), (7, 512, 2048, True, 3), (7, 2048, 512, False, 2),
]


# (H=W, width = C_out of conv1, C_in = block input channels) of conv1 in the 16 bottlenecks
DGRAD_LAYERS = [
    (56, 64, 64, 1), (56, 64, 256, 2), (56, 128, 256, 1), (28, 128, 512, 3),
    (28, 256, 512, 1), (14, 256, 1024, 5), (14, 512, 1024, 1), (7, 512, 2048, 2),
]


def timed(fn, iters, flush):
    ts = []
    for _ in range(iters):
        flush.add_(1.0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=256)
    ap.add_argument('--iters', type=int, default=15)
    ap.add_argument('--out', default='')
    ap.add_argument('--dtype', default='bf16', choices=['bf16', 'fp32'],
                    help='fp32: fp32 operands, TF32 tensor-core math (kind::tf32) vs cuDNN TF32')
    args = ap.parse_args()
    DT = torch.float32 if args.dtype == 'fp32' else torch.bfloat16
    esz = 4.0 if args.dtype == 'fp32' else 2.0
    native.load()
    flush = torch.zeros(64 * 1024 * 1024, device='cuda')          # 256 MB > L2
    rows, tot_lib, tot_tc = [], 0.0, 0.0
    for hw, cin, cout, add, mult in LAYERS:
        conv = nn.Conv2d(cin, cout, 1, bias=False).cuda().to(DT).to(memory_format=torch.channels_last)
        bn = FusedBatchNormAct2d(cout).cuda()
        x = torch.randn(args.batch, cin, hw, hw, device='cuda').to(DT) \
            .contiguous(memory_format=torch.channels_last)
        res = torch.randn(args.batch, cout, hw, hw, device='cuda').to(DT) \
            .contiguous(memory_format=torch.channels_last) if add else None
        w = conv.weight.detach()
        C = native.load()
        out = {}
        with torch.no_grad():
            for name, use in (('library', False), ('wgmma', True)):
                fused_bn.USE_TCGEN05_CONV1X1 = use
                fn = lambda: conv_bn_act(conv, bn, x, residual=res, relu=True)   # noqa: E731
                for _ in range(3):
                    fn()
                out[name] = timed(fn, args.iters, flush)
            out['lib_conv_only'] = timed(lambda: conv(x), args.iters, flush)
            out['tc_gemm_only'] = timed(lambda: C.conv1x1_forward(x, w), args.iters, flush)
            out['tc_gemm_stats'] = timed(lambda: C.conv1x1_forward(x, w, True), args.iters, flush)
        M = args.batch * hw * hw
        gemm_bytes = esz * (M * cin + M * cout + cin * cout)
        rows.append(dict(hw=hw, cin=cin, cout=cout, add=add, mult=mult, M=M,
                         gemm_tbps=gemm_bytes / out['tc_gemm_only'] / 1e9,
                         lib_conv_tbps=gemm_bytes / out['lib_conv_only'] / 1e9, **out))
        tot_lib += mult * out['library']
        tot_tc += mult * out['wgmma']
        print('%3dx%-3d %4d->%-4d add=%d x%d | conv+bn: lib %.3f ms  wgmma %.3f ms | conv only: lib %.3f '
              '(%.2f TB/s)  wgmma %.3f (%.2f TB/s), +stats %.3f' % (
                  hw, hw, cin, cout, add, mult, out['library'], out['wgmma'], out['lib_conv_only'],
                  rows[-1]['lib_conv_tbps'], out['tc_gemm_only'], rows[-1]['gemm_tbps'], out['tc_gemm_stats']), flush=True)
    print('ResNet-50 fwd 1x1 conv+BN total: library %.3f ms, wgmma %.3f ms' % (tot_lib, tot_tc))

    # backward of the first 1x1 convolution of every bottleneck: dX = dY . W (+ skip gradient)
    drows, d_lib, d_tc, d_m2, d_m3 = [], 0.0, 0.0, 0.0, 0.0
    for hw, width, cin, mult in DGRAD_LAYERS:
        dy = torch.randn(args.batch, width, hw, hw, device='cuda').to(DT) \
            .contiguous(memory_format=torch.channels_last)
        skip = torch.randn(args.batch, cin, hw, hw, device='cuda').to(DT) \
            .contiguous(memory_format=torch.channels_last)
        xin = torch.empty_like(skip)
        w = (torch.randn(width, cin, 1, 1, device='cuda') * cin ** -0.5).to(DT)
        C = native.load()

        def lib():
            dx = torch.ops.aten.convolution_backward(dy, xin, w, None, [1, 1], [0, 0], [1, 1], False, [0, 0], 1,
                                                     [True, False, False])[0]
            return dx.add_(skip)

        def fused():
            wt = w.reshape(width, cin).t().contiguous()
            return C.conv1x1_forward(dy, wt, False, skip)

        # the previous block's bn3 backward reduction: stand-alone (MODE 2 dgrad + mode-2 reduce
        # pass over dy / yraw3 / out3) vs folded into the dgrad epilogue (MODE 3)
        yraw3 = torch.randn_like(skip)
        out3 = torch.relu(yraw3)
        mask = torch.randint(0, 256, (skip.numel() // cin, cin // 8), dtype=torch.uint8, device='cuda')
        coef = torch.stack([yraw3.float().mean((0, 2, 3)), torch.ones(cin, device='cuda'),
                            torch.ones(cin, device='cuda'), torch.zeros(cin, device='cuda')])
        wt_ = w.reshape(width, cin).t().contiguous()

        def mode2_reduce():
            return C.bn_backward(C.conv1x1_forward(dy, wt_, False, skip), yraw3, out3, coef, True, True)

        def mode3():
            dz, partial = C.conv1x1_dgrad_bn_reduce(dy, wt_, skip, yraw3, coef, mask)
            return C.bn_backward_from_partials(dz, yraw3, coef, partial)

        with torch.no_grad():
            for _ in range(3):
                lib(); fused(); mode2_reduce(); mode3()
            t_lib, t_tc = timed(lib, args.iters, flush), timed(fused, args.iters, flush)
            t_m2, t_m3 = timed(mode2_reduce, args.iters, flush), timed(mode3, args.iters, flush)
        drows.append(dict(hw=hw, width=width, cin=cin, mult=mult, library=t_lib, wgmma=t_tc,
                          mode2_plus_bn_bwd=t_m2, mode3_plus_bn_bwd=t_m3))
        d_lib += mult * t_lib
        d_tc += mult * t_tc
        d_m2 += mult * t_m2
        d_m3 += mult * t_m3
        print('dgrad %3dx%-3d %4d->%-4d x%d | lib dgrad + add %.3f ms | wgmma dgrad(+skip) %.3f ms | '
              'bn3 bwd + dgrad: MODE 2 + reduce %.3f ms, MODE 3 %.3f ms' % (
                  hw, hw, width, cin, mult, t_lib, t_tc, t_m2, t_m3), flush=True)
    print('ResNet-50 conv1 dgrad + skip-gradient accumulation total: library %.3f ms, wgmma %.3f ms' % (d_lib, d_tc))
    print('with the previous bn3 backward (reduce + finalize + dx): MODE 2 + reduce %.3f ms, MODE 3 %.3f ms' % (
        d_m2, d_m3))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or '.', exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(dict(batch=args.batch, dtype=args.dtype, total_library_ms=tot_lib, total_wgmma_ms=tot_tc, layers=rows,
                           dgrad_library_ms=d_lib, dgrad_wgmma_ms=d_tc, dgrad_mode2_reduce_ms=d_m2,
                           dgrad_mode3_ms=d_m3, dgrad_layers=drows), f, indent=1)


if __name__ == '__main__':
    main()
