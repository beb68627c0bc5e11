"""The augment kernel's op chains (csrc/augment_kernels.cu) behind GpuAugment(auto_augment='ra' / 'imagenet'):
every ordered pair of ops and sampled longer chains decompose into single-op launches bit for bit, Invert
against torchvision, full policy batches against the CPU composition, TrivialAugment + erase rows against
the previous kernel's recorded output, no host synchronisation, and CLI training runs from shards."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from stochastic_gradient_push_b200.data.shards import (AUGMENT_OPS, RA_BINS, TA_WIDE_SIGNED, AugmentParams,
                                                       GpuAugment, policy_magnitudes, write_shards_from_arrays)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TF = pytest.importorskip('torchvision.transforms.v2.functional')
DEV = torch.device('cuda', 0)
MEAN = torch.tensor((0.485, 0.456, 0.406)).view(3, 1, 1) * 255.0
INV = 1.0 / (torch.tensor((0.229, 0.224, 0.225)).view(3, 1, 1) * 255.0)
BIT_EXACT = ('Identity', 'Brightness', 'Color', 'Posterize', 'Solarize', 'AutoContrast', 'Equalize', 'Invert')


def _test_images(n, size, seed=0):
    """uint8 [n, size, size, 3]: noise, narrower ranges, a gradient and a constant channel"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (n, size, size, 3), dtype=torch.uint8, generator=g)
    for i in range(1, min(n, 4)):
        x[i] = torch.randint(12 * i, 255 - 20 * i, (size, size, 3), dtype=torch.uint8, generator=g)
    if n > 4:
        ramp = torch.arange(size).view(1, size, 1) + torch.arange(size).view(size, 1, 1)
        x[4] = (40 + ramp * 60 // (2 * size)).expand(size, size, 3).to(torch.uint8)
    if n > 5:
        x[5, :, :, 0] = 77
    return x


def _identity_params(ops, mags):
    """identity crop (out = S): the kernel's stage-1 image is the input itself"""
    ops = torch.as_tensor(ops, dtype=torch.int64)
    n = ops.shape[0]
    one = torch.ones(n)
    return AugmentParams(one * 0.5, one * 0.5, one, one, one, ops, torch.as_tensor(mags, dtype=torch.float64),
                         torch.zeros(n, 4, dtype=torch.int64))


def _to_u8(y):
    """kernel fp32 output -> the uint8 values it normalised (exact: one step is ~0.017)"""
    return (y.float().cpu() / INV + MEAN).round().clamp(0, 255).to(torch.uint8)


def _mag(name, size, sign):
    t = policy_magnitudes(RA_BINS, size)[name]
    return 0.0 if t is None else (sign if name in TA_WIDE_SIGNED else 1) * float(t[15])


def _decomposed(x, ops, mags, size):
    """the kernel's chain as single-op launches: each op's fp32 output read back as uint8 and fed to the next"""
    aug = GpuAugment(out_size=size, auto_augment='ra')
    cur = x
    for k in range(ops.shape[1]):
        y = aug.apply(cur.to(DEV), _identity_params(ops[:, k], mags[:, k]))
        cur = _to_u8(y).permute(0, 2, 3, 1).contiguous()
    return y


def _check_chain(x, ops, mags, size):
    ref = _decomposed(x, ops, mags, size)
    for dtype in (torch.float32, torch.bfloat16):
        aug = GpuAugment(out_size=size, auto_augment='ra', dtype=dtype)
        y = aug.apply(x.to(DEV), _identity_params(ops, mags))
        assert y.dtype == dtype
        assert torch.equal(y, ref.to(dtype)), (dtype, (y != ref.to(dtype)).sum().item())


@pytest.mark.parametrize('first', AUGMENT_OPS)
def test_every_pair_decomposes_into_single_ops(first):
    size = 64
    x = _test_images(6, size, seed=AUGMENT_OPS.index(first))
    ops, mags = [], []
    for second in AUGMENT_OPS:
        for sa in (1, -1):
            for sb in (1, -1):
                if (sa < 0 and first not in TA_WIDE_SIGNED) or (sb < 0 and second not in TA_WIDE_SIGNED):
                    continue
                ops.append([AUGMENT_OPS.index(first), AUGMENT_OPS.index(second)])
                mags.append([_mag(first, size, sa), _mag(second, size, sb)])
    ops = torch.tensor(ops).repeat_interleave(6, 0)
    mags = torch.tensor(mags, dtype=torch.float64).repeat_interleave(6, 0)
    _check_chain(x.repeat(len(ops) // 6, 1, 1, 1), ops, mags, size)


@pytest.mark.parametrize('k', [3, 4])
@pytest.mark.parametrize('size', [64, 63])           # 63: byte-wise staging (3 size^2 is not a multiple of 4)
def test_sampled_chains_decompose_into_single_ops(k, size):
    n = 96
    g = torch.Generator().manual_seed(100 * k + size)
    x = _test_images(n, size, seed=k)
    ops = torch.randint(len(AUGMENT_OPS), (n, k), generator=g)
    ops[: n // 4, 1] = 0                                                   # Identity inside a chain
    ops[n // 4: n // 2, -1] = 0                                            # trailing Identity
    signs = torch.where(torch.rand(n, k, generator=g) < 0.5, -1, 1)
    mags = torch.tensor([[_mag(AUGMENT_OPS[o], size, s) for o, s in zip(r, t)]
                         for r, t in zip(ops.tolist(), signs.tolist())], dtype=torch.float64)
    _check_chain(x, ops, mags, size)


def test_invert_matches_torchvision():
    x = _test_images(8, 64, seed=3)
    y = GpuAugment(out_size=64, auto_augment='ra').apply(x.to(DEV), _identity_params(torch.full((8,), 14),
                                                                                      torch.zeros(8)))
    ref = (TF.invert(x.permute(0, 3, 1, 2)).float() - MEAN) * INV
    assert torch.equal(y.cpu(), ref)


@pytest.mark.parametrize('policy', ['ra', 'imagenet'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_full_batches_equal_the_cpu_composition(policy, dtype):
    """B = 256 stored at 256 and cropped to 224, with erasing: every row whose ops are all bit-exact equals
    the CPU composition of the same draws on the kernel's own rounded crop"""
    from stochastic_gradient_push_b200.ops.oracle import ta_wide_op
    B, S, O = 256, 256, 224
    x = _test_images(B, S, seed=17)
    aug = GpuAugment(out_size=O, seed=23, auto_augment=policy, random_erase=0.25, dtype=dtype)
    p = aug.sample_params(B)
    y = aug.apply(x.to(DEV), p).cpu()
    zeros = torch.zeros(B, 0, dtype=torch.int64)
    crop = _to_u8(GpuAugment(out_size=O, auto_augment='ra').apply(
        x.to(DEV), p._replace(op=zeros, magnitude=zeros.double(), erase=torch.zeros_like(p.erase))))
    exact = [i for i in range(B) if all(AUGMENT_OPS[k] in BIT_EXACT for k in p.op[i].tolist())]
    assert len(exact) > 40
    for i in exact:
        img = crop[i]
        for op, mag in zip(p.op[i].tolist(), p.magnitude[i].tolist()):
            img = ta_wide_op(img, AUGMENT_OPS[op], mag)
        ref = (img.float() - MEAN) * INV
        top, left, h, w = p.erase[i].tolist()
        ref[:, top:top + h, left:left + w] = 0.0
        assert torch.equal(y[i], ref.to(dtype)), (i, p.op[i].tolist())


def test_ta_wide_rows_keep_the_previous_kernels_bits():
    """TrivialAugment + erase rows give the bits the one-op kernel gave (tests/golden/augment_parent_kernel.pt:
    the previous commit's kernel on an H100 for 16 images stored at 72, cropped to 40)"""
    rec = torch.load(os.path.join(ROOT, 'tests', 'golden', 'augment_parent_kernel.pt'))
    B, S, O, seed = rec['B'], rec['S'], rec['out'], rec['seed']
    x = torch.randint(0, 256, (B, S, S, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed))
    aug = GpuAugment(out_size=O, seed=seed, auto_augment='ta_wide', random_erase=0.5)
    p = aug.sample_params(B)
    for k, v in rec['params'].items():                                      # the draws are unchanged too
        assert torch.equal(getattr(p, k), v), k
    assert len(set(p.op.tolist())) >= 12 and int((p.erase[:, 2] > 0).sum()) >= 5
    for name, dt in (('fp32', torch.float32), ('bf16', torch.bfloat16)):
        y = GpuAugment(out_size=O, seed=seed, auto_augment='ta_wide', random_erase=0.5, dtype=dt).apply(x.to(DEV), p)
        assert torch.equal(y.cpu(), rec[name]), name


@pytest.mark.parametrize('policy', ['ra', 'imagenet'])
def test_no_host_sync_and_the_ring_is_reused(policy):
    x = torch.randint(0, 256, (64, 256, 256, 3), dtype=torch.uint8).pin_memory()
    outs = []
    for _ in range(2):
        aug = GpuAugment(seed=4, auto_augment=policy, random_erase=0.25, dtype=torch.bfloat16)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode('error')
        try:
            xs = [x.to(DEV, non_blocking=True) for _ in range(3)]
            ys = [aug(b) for b in xs]
        finally:
            torch.cuda.set_sync_debug_mode(0)
        outs.append(torch.stack(ys))
    assert torch.equal(outs[0], outs[1])
    assert not torch.equal(outs[0][0], outs[0][1])
    # 20 calls through the 8 pinned slots, then a one-op call through the same ring
    aug = GpuAugment(out_size=64, seed=2, auto_augment=policy, random_erase=0.5, ra_num_ops=4)
    twin = GpuAugment(out_size=64, seed=2, auto_augment=policy, random_erase=0.5, ra_num_ops=4)
    xs = _test_images(12, 72, seed=8).to(DEV)
    ys = [aug(xs) for _ in range(20)]
    for y in ys:
        assert torch.equal(y, twin.apply(xs, twin.sample_params(12)))
    p = twin.sample_params(12)
    one = p._replace(op=p.op[:, 0], magnitude=p.magnitude[:, 0])
    assert torch.equal(aug.apply(xs, one), twin.apply(xs, one))


@pytest.mark.parametrize('policy', ['ra', 'imagenet'])
def test_cli_trains_from_shards_with_the_policy(tmp_path, master_port, policy):
    rng = np.random.default_rng(0)
    for split, n in (('train', 96), ('val', 32)):
        imgs = rng.integers(0, 256, (n, 40, 40, 3), dtype=np.uint8)
        write_shards_from_arrays(str(tmp_path / 'data' / split), imgs, rng.integers(0, 10, n), shard_size=64)
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '1',
           '--master-addr', '127.0.0.1', '--master-port', str(master_port), os.path.join(ROOT, 'gossip_sgd.py'),
           '--model', 'tiny', '--num_classes', '10', '--image_size', '32', '--dataset_dir', str(tmp_path / 'data'),
           '--data_format', 'shards', '--auto_augment', policy, '--ra_num_ops', '3', '--random_erase', '0.25',
           '--cuda_graph', 'True', '--batch_size', '16', '--verbose', 'False', '--print_freq', '2',
           '--num_dataloader_workers', '0', '--lr', '0.05', '--push_sum', 'True', '--graph_type', '5',
           '--num_epochs', '2', '--checkpoint_dir', str(tmp_path / 'ckpt') + '/', '--num_itr_ignore', '0']
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:]
    rows = open(str(tmp_path / 'ckpt' / 'out_r0_n1.csv')).read().splitlines()[5:]
    train_rows = [r.split(',') for r in rows if r.split(',')[1] != '-1']
    assert len(train_rows) >= 6
    assert all(math.isfinite(float(r[12])) for r in train_rows)
    assert any(r.split(',')[1] == '-1' for r in rows)
