"""Blind-debug aid for the wgmma 1x1-conv GEMM: prints error maps (which row groups /
column chunks / k-blocks are wrong) instead of a bare pass/fail."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from stochastic_gradient_push_b200.ops import native   # noqa: E402


def report(M, K, N, mode):
    C = native.load()
    g = torch.Generator(device='cuda').manual_seed(1)
    if mode == 'rand':
        x = torch.randn(M, K, device='cuda', generator=g)
        w = torch.randn(N, K, device='cuda', generator=g) * K ** -0.5
    elif mode == 'rowid':      # y[m, n] = m (first k column is the row id / 64, W picks column 0)
        x = torch.zeros(M, K, device='cuda'); x[:, 0] = torch.arange(M, device='cuda') % 128
        w = torch.zeros(N, K, device='cuda'); w[:, 0] = 1
    else:                      # 'kid': y[m, n] = sum_k x[m,k] w[n,k] with x = one-hot(k = m % K), w[n,k] = k + n/1024
        x = torch.zeros(M, K, device='cuda'); x[torch.arange(M), torch.arange(M) % K] = 1
        w = (torch.arange(K, device='cuda')[None, :] % 64 + torch.zeros(N, 1, device='cuda')).float()
    x, w = x.to(torch.bfloat16), w.to(torch.bfloat16)
    y = C.conv1x1_forward(x, w).float()
    torch.cuda.synchronize()
    want = x.float() @ w.float().t()
    err = (y - want).abs()
    tol = 1e-2 + 1e-2 * want.abs()
    bad = err > tol
    print('[%s] M=%d K=%d N=%d: max err %.4g, bad fraction %.4g' % (mode, M, K, N, err.max().item(),
                                                                    bad.float().mean().item()))
    if bad.any():
        rows = bad.any(1).nonzero().flatten()
        cols = bad.any(0).nonzero().flatten()
        print('   bad rows: %d (first %s) rows%%8 hist %s' % (
            rows.numel(), rows[:12].tolist(), torch.bincount(rows % 8, minlength=8).tolist()))
        print('   bad cols: %d (first %s) col//8 hist %s' % (
            cols.numel(), cols[:12].tolist(), torch.bincount((cols // 8) % 8, minlength=8).tolist()))
        r, c = rows[0].item(), cols[0].item()
        print('   sample y[%d, %d:%d] = %s\n          want        = %s' % (
            r, c, c + 8, y[r, c:c + 8].tolist(), want[r, c:c + 8].tolist()))
    return not bad.any().item()


if __name__ == '__main__':
    ok = True
    for mode in ('rowid', 'kid', 'rand'):
        for M, K, N in ((128, 64, 64), (256, 128, 128), (384, 64, 256), (1000, 256, 512)):
            ok &= report(M, K, N, mode)
    print('ALL OK' if ok else 'FAILURES')
