"""The sm_90a augment kernel (csrc/augment_kernels.cu) behind data.GpuAugment's auto_augment='ta_wide' and
random_erase: each TrivialAugmentWide op against torchvision.transforms.v2.functional on uint8 images, the
crop stage against grid_sample, erasing, the unchanged default path, no host synchronisation, and one
training run of the CLI from shards."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from stochastic_gradient_push_b200.data.shards import (TA_WIDE_OPS, TA_WIDE_SIGNED, AugmentParams, GpuAugment,
                                                       ta_wide_magnitudes, ta_wide_matrix, write_shards_from_arrays)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TF = pytest.importorskip('torchvision.transforms.v2.functional')
DEV = torch.device('cuda', 0)
MEAN = torch.tensor((0.485, 0.456, 0.406)).view(3, 1, 1) * 255.0
INV = 1.0 / (torch.tensor((0.229, 0.224, 0.225)).view(3, 1, 1) * 255.0)
BIT_EXACT = ('Identity', 'Brightness', 'Color', 'Posterize', 'Solarize', 'AutoContrast', 'Equalize')
GEOMETRIC = ('ShearX', 'ShearY', 'TranslateX', 'TranslateY', 'Rotate')


def _normalise(u8):
    return (u8.float() - MEAN) * INV


def _test_images(n=8, size=64, seed=0):
    """uint8 [n, size, size, 3]: full-range noise, narrower ranges (AutoContrast / Equalize have work
    to do), a smooth gradient and a constant channel (AutoContrast's max == min, Equalize's step 0)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (n, size, size, 3), dtype=torch.uint8, generator=g)
    for i in range(1, 5):
        lo, hi = 12 * i, 255 - 20 * i
        x[i] = torch.randint(lo, hi, (size, size, 3), dtype=torch.uint8, generator=g)
    ramp = torch.arange(size).view(1, size, 1) + torch.arange(size).view(size, 1, 1)
    x[5] = (40 + ramp * 60 // (2 * size)).expand(size, size, 3).to(torch.uint8)
    x[6, :, :, 0] = 77
    return x


def _identity_params(n, op, magnitude, erase=None):
    one = torch.ones(n)
    return AugmentParams(one * 0.5, one * 0.5, one, one, one, torch.full((n,), op, dtype=torch.int64),
                         torch.full((n,), float(magnitude), dtype=torch.float64),
                         torch.zeros(n, 4, dtype=torch.int64) if erase is None else erase)


def _to_u8(y):
    """kernel fp32 output -> the uint8 values it normalised (exact: one step is ~0.017)"""
    return (y.float().cpu() / INV + MEAN).round().clamp(0, 255).to(torch.uint8)


def _cases():
    tables = ta_wide_magnitudes()
    for op in TA_WIDE_OPS:
        bins = (0, 1, 15, 20, 30) if op == 'Rotate' else (0, 1, 15, 30)
        for b in bins:
            for sign in ((1, -1) if op in TA_WIDE_SIGNED else (1,)):
                if tables[op] is None and (b or sign < 0):
                    continue
                yield op, (0.0 if tables[op] is None else sign * float(tables[op][b]))


@pytest.mark.parametrize('op,mag', list(_cases()))
def test_each_op_matches_torchvision(op, mag):
    x = _test_images()
    n, S = x.shape[0], x.shape[1]
    aug = GpuAugment(out_size=S, auto_augment='ta_wide')
    y = aug.apply(x.to(DEV), _identity_params(n, TA_WIDE_OPS.index(op), mag)).cpu()
    assert y.dtype == torch.float32 and y.is_contiguous(memory_format=torch.channels_last)
    from stochastic_gradient_push_b200.ops.oracle import ta_wide_op
    imgs = x.permute(0, 3, 1, 2)
    ref_u8 = torch.stack([ta_wide_op(imgs[i].contiguous(), op, mag) for i in range(n)])
    ref = _normalise(ref_u8)
    if op in BIT_EXACT:
        assert torch.equal(y, ref), (op, mag, (y != ref).sum().item())
        return
    got = _to_u8(y)
    assert torch.equal(_normalise(got), y)                       # the kernel wrote normalised uint8 values
    diff = got != ref_u8
    frac = diff.float().mean().item()
    assert frac <= 1e-3, (op, mag, frac)
    if op in ('Contrast', 'Sharpness'):
        assert (got.int() - ref_u8.int()).abs().max().item() <= 1
        return
    # nearest-neighbour ties: a differing pixel holds one of the source pixels around the exact
    # (fp64) source coordinate, or the fill where that lies outside
    m = ta_wide_matrix(op, mag, S)
    c0 = (S - 1) / 2.0
    for i, c, yy, xx in diff.nonzero().tolist():
        sx = m[0] * (xx - c0) + m[1] * (yy - c0) + m[2] + c0
        sy = m[3] * (xx - c0) + m[4] * (yy - c0) + m[5] + c0
        cands = set()
        for px in (math.floor(sx), math.floor(sx) + 1):
            for py in (math.floor(sy), math.floor(sy) + 1):
                cands.add(int(imgs[i, c, py, px]) if (0 <= px < S and 0 <= py < S) else 0)
        assert int(got[i, c, yy, xx]) in cands, (op, mag, i, c, yy, xx)


@pytest.mark.parametrize('out', [224, 176, 160])
@pytest.mark.parametrize('batch', [1, 7, 256])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_crop_stage_matches_grid_sample(out, batch, dtype):
    S = 256
    g = torch.Generator().manual_seed(out * 1000 + batch)
    x = torch.randint(0, 256, (batch, S, S, 3), dtype=torch.uint8, generator=g).to(DEV)
    aug = GpuAugment(out_size=out, seed=batch, auto_augment='ta_wide', dtype=dtype)
    cx, cy, w, h, flip = aug.sample_boxes(batch)
    zeros = torch.zeros(batch, dtype=torch.int64)
    p = AugmentParams(cx, cy, w, h, flip, zeros, zeros.double(), torch.zeros(batch, 4, dtype=torch.int64))
    y = aug.apply(x, p)
    assert y.dtype == dtype and y.shape == (batch, 3, out, out)
    theta = GpuAugment.crop_theta(cx, cy, w, h, flip).to(DEV)
    grid = F.affine_grid(theta, (batch, 3, out, out), align_corners=False)
    ref_u8 = F.grid_sample(x.permute(0, 3, 1, 2).float(), grid, mode='bilinear', padding_mode='border',
                           align_corners=False).round()
    mean, inv = MEAN.to(DEV), INV.to(DEV)
    norm = lambda u: ((u - mean) * inv).to(dtype)  # noqa: E731
    ref = norm(ref_u8)
    diff = y != ref
    assert diff.float().mean().item() <= 1e-3
    one_step = (y == norm(ref_u8 - 1)) | (y == norm(ref_u8 + 1))
    assert bool((~diff | one_step).all())


def test_erase_zeroes_exactly_the_box():
    x = _test_images(8, 96, seed=3).to(DEV)
    aug = GpuAugment(out_size=80, seed=5, auto_augment='ta_wide', random_erase=1.0)
    p = aug.sample_params(8)
    assert (p.erase[:, 2] > 0).all()
    y = aug.apply(x, p)
    y0 = aug.apply(x, p._replace(erase=torch.zeros_like(p.erase)))
    inside = torch.zeros(8, 1, 80, 80, dtype=torch.bool)
    for i, (top, left, h, w) in enumerate(p.erase.tolist()):
        inside[i, :, top:top + h, left:left + w] = True
    inside = inside.expand(8, 3, 80, 80).to(DEV)
    assert bool((y[inside] == 0).all())
    assert torch.equal(y[~inside], y0[~inside])
    bf = GpuAugment(out_size=80, seed=5, auto_augment='ta_wide', random_erase=1.0, dtype=torch.bfloat16)
    yb = bf.apply(x, p)
    assert bool((yb[inside] == 0).all()) and torch.equal(yb[~inside], y0[~inside].to(torch.bfloat16))


def test_default_path_is_unchanged():
    x = torch.randint(0, 256, (16, 256, 256, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
    x = x.to(DEV)
    for dtype in (torch.float32, torch.bfloat16):
        aug, ref = GpuAugment(seed=9, dtype=dtype), GpuAugment(seed=9, dtype=dtype)
        for train in (True, False):
            y = aug(x, train=train)
            # the grid_sample composition GpuAugment has always run
            n = x.shape[0]
            if train:
                cx, cy, w, h, flip = ref.sample_boxes(n)
            else:
                cx = cy = torch.full((n,), 0.5)
                w = h = torch.full((n,), ref.eval_ratio)
                flip = torch.ones(n)
            theta = torch.zeros(n, 2, 3)
            theta[:, 0, 0] = w * flip
            theta[:, 0, 2] = 2 * cx - 1
            theta[:, 1, 1] = h
            theta[:, 1, 2] = 2 * cy - 1
            grid = F.affine_grid(theta.to(DEV), (n, 3, 224, 224), align_corners=False)
            z = F.grid_sample(x.permute(0, 3, 1, 2).float(), grid, mode='bilinear', padding_mode='border',
                              align_corners=False)
            mean = torch.tensor(ref.mean, device=DEV).view(1, 3, 1, 1) * 255.0
            inv = 1.0 / (torch.tensor(ref.std, device=DEV).view(1, 3, 1, 1) * 255.0)
            z = ((z - mean) * inv).contiguous(memory_format=torch.channels_last).to(dtype)
            assert torch.equal(y, z) and y.stride() == z.stride()
    # evaluation with the options on is the same centre crop
    ta = GpuAugment(seed=9, auto_augment='ta_wide', random_erase=0.5)
    assert torch.equal(ta(x, train=False), GpuAugment(seed=9)(x, train=False))


def test_no_host_sync_and_deterministic():
    x = torch.randint(0, 256, (64, 256, 256, 3), dtype=torch.uint8).pin_memory()
    outs = []
    for _ in range(2):
        aug = GpuAugment(seed=4, auto_augment='ta_wide', random_erase=0.25, dtype=torch.bfloat16)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode('error')
        try:
            xs = [x.to(DEV, non_blocking=True) for _ in range(3)]
            ys = [aug(b) for b in xs]
        finally:
            torch.cuda.set_sync_debug_mode(0)
        outs.append(torch.stack(ys))
    assert torch.equal(outs[0], outs[1])
    assert not torch.equal(outs[0][0], outs[0][1])                 # each call draws anew


def test_many_calls_recycle_the_ring_and_match_the_draws():
    aug = GpuAugment(out_size=64, seed=2, auto_augment='ta_wide', random_erase=0.5)
    twin = GpuAugment(out_size=64, seed=2, auto_augment='ta_wide', random_erase=0.5)
    x = _test_images(12, 72, seed=8).to(DEV)
    ys = [aug(x) for _ in range(20)]                                # 20 calls through 8 ring slots
    for y in ys:
        assert torch.equal(y, twin.apply(x, twin.sample_params(12)))


def test_cli_trains_from_shards_with_trivial_augment(tmp_path, master_port):
    rng = np.random.default_rng(0)
    for split, n in (('train', 96), ('val', 32)):
        imgs = rng.integers(0, 256, (n, 40, 40, 3), dtype=np.uint8)
        write_shards_from_arrays(str(tmp_path / 'data' / split), imgs, rng.integers(0, 10, n), shard_size=64)
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '1',
           '--master-addr', '127.0.0.1', '--master-port', str(master_port), os.path.join(ROOT, 'gossip_sgd.py'),
           '--model', 'tiny', '--num_classes', '10', '--image_size', '32', '--dataset_dir', str(tmp_path / 'data'),
           '--data_format', 'shards', '--auto_augment', 'ta_wide', '--random_erase', '0.25', '--cuda_graph', 'True',
           '--batch_size', '16', '--verbose', 'False', '--print_freq', '2', '--num_dataloader_workers', '0',
           '--lr', '0.05', '--push_sum', 'True', '--graph_type', '5', '--num_epochs', '2',
           '--checkpoint_dir', str(tmp_path / 'ckpt') + '/', '--num_itr_ignore', '0']
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:]
    rows = open(str(tmp_path / 'ckpt' / 'out_r0_n1.csv')).read().splitlines()[5:]
    train_rows = [r.split(',') for r in rows if r.split(',')[1] != '-1']
    assert len(train_rows) >= 6
    assert all(math.isfinite(float(r[12])) for r in train_rows)
    assert any(r.split(',')[1] == '-1' for r in rows)                                       # validation ran
