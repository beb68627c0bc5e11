"""RandAugment and AutoAugment (ImageNet policy) in data.GpuAugment, on the CPU: the magnitude tables and
sub-policies against torchvision v2, the draw laws, determinism, the op-chain composition against
torchvision, the kernel's chain rows, validation and the CLI flags."""
import itertools

import numpy as np
import pytest
import torch

from stochastic_gradient_push_b200.data.shards import (AA_BINS, AUGMENT_CHAIN_COL, AUGMENT_OPS, AUGMENT_ROW,
                                                       AUGMENT_ROW_ONE_OP, AUTO_AUGMENT_IMAGENET, RA_BINS,
                                                       TA_WIDE_OPS, TA_WIDE_SIGNED, AugmentParams, GpuAugment,
                                                       augment_smem_bytes, policy_magnitudes)

tv2 = pytest.importorskip('torchvision.transforms.v2')
import torchvision.transforms.v2.functional as TF  # noqa: E402


def _images(n, size, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (n, size, size, 3), dtype=torch.uint8, generator=g)
    if n > 1:                                        # a narrow range: AutoContrast / Equalize have work to do
        x[1] = torch.randint(40, 170, (size, size, 3), dtype=torch.uint8, generator=g)
    return x


def _normalise(img):
    mean = torch.tensor((0.485, 0.456, 0.406)).view(3, 1, 1) * 255.0
    inv = 1.0 / (torch.tensor((0.229, 0.224, 0.225)).view(3, 1, 1) * 255.0)
    return (img.float() - mean) * inv


def _rounded_crops(x, aug, p):
    theta = GpuAugment.crop_theta(p.cx, p.cy, p.w, p.h, p.flip)
    grid = torch.nn.functional.affine_grid(theta, (x.shape[0], 3, aug.out, aug.out), align_corners=False)
    y = torch.nn.functional.grid_sample(x.permute(0, 3, 1, 2).float(), grid, mode='bilinear',
                                        padding_mode='border', align_corners=False)
    return y.round().clamp(0, 255).to(torch.uint8)


def _torchvision_chain(img, names, mags):
    aa = tv2.AutoAugment()
    for name, mag in zip(names, mags):
        img = aa._apply_image_or_video_transform(img, name, float(mag), interpolation=aa.interpolation,
                                                 fill=aa._fill)
    return img


def _expected(x, aug, p):
    """torchvision's composition of params p: rounded crop, the ops left to right, normalise, erase"""
    crops = _rounded_crops(x, aug, p)
    ops = p.op if p.op.dim() == 2 else p.op[:, None]
    mags = p.magnitude if p.magnitude.dim() == 2 else p.magnitude[:, None]
    out = []
    for i in range(x.shape[0]):
        img = _normalise(_torchvision_chain(crops[i], [AUGMENT_OPS[k] for k in ops[i].tolist()], mags[i].tolist()))
        top, left, h, w = p.erase[i].tolist()
        if h:
            img = TF.erase(img, top, left, h, w, torch.zeros(1))
        out.append(img)
    return torch.stack(out)


def _chain_params(aug, n, ops, mags):
    cx, cy, w, h, flip = aug.sample_boxes(n)
    return AugmentParams(cx, cy, w, h, flip, torch.as_tensor(ops, dtype=torch.int64),
                         torch.as_tensor(mags, dtype=torch.float64), torch.zeros(n, 4, dtype=torch.int64))


def _mid(name, size, sign=1):
    """bin 15 of RandAugment's space, signed for the signed ops"""
    t = policy_magnitudes(RA_BINS, size)[name]
    return 0.0 if t is None else (sign if name in TA_WIDE_SIGNED else 1) * float(t[15])


# -- tables and draws ---------------------------------------------------------------------------------- #
@pytest.mark.parametrize('size', [224, 64, 277, 33])
def test_policy_tables_equal_torchvision(size):
    for cls, bins in ((tv2.RandAugment, RA_BINS), (tv2.AutoAugment, AA_BINS)):
        mine = policy_magnitudes(bins, size)
        for name, (fn, signed) in cls._AUGMENTATION_SPACE.items():
            assert name in AUGMENT_OPS and (name in TA_WIDE_SIGNED) == signed, name
            ref = fn(bins, size, size)
            if ref is None:
                assert mine[name] is None, name
            else:
                assert mine[name].dtype == ref.dtype and torch.equal(mine[name], ref), (cls, name)
    assert tuple(tv2.RandAugment._AUGMENTATION_SPACE) == TA_WIDE_OPS
    assert set(tv2.AutoAugment._AUGMENTATION_SPACE) == set(AUGMENT_OPS) - {'Identity'}
    assert AUGMENT_OPS == TA_WIDE_OPS + ('Invert',)


def test_sub_policies_equal_torchvision():
    assert [tuple(map(tuple, sub)) for sub in tv2.AutoAugment()._policies] == list(AUTO_AUGMENT_IMAGENET)
    assert len(AUTO_AUGMENT_IMAGENET) == 25


@pytest.mark.parametrize('num_ops,magnitude', [(2, 9), (3, 30), (1, 0)])
def test_rand_augment_draw_law(num_ops, magnitude):
    from scipy.stats import chisquare
    aug = GpuAugment(out_size=64, seed=5, auto_augment='ra', ra_num_ops=num_ops, ra_magnitude=magnitude)
    p = [aug.sample_params(2000) for _ in range(10)]
    ops, mags = torch.cat([q.op for q in p]), torch.cat([q.magnitude for q in p])
    assert ops.shape == (20000, num_ops) and mags.shape == ops.shape
    assert chisquare(torch.bincount(ops.flatten(), minlength=14).numpy()).pvalue > 1e-4
    assert int(ops.max()) < len(TA_WIDE_OPS)                                  # never Invert
    space = policy_magnitudes(RA_BINS, 64)
    for k, name in enumerate(TA_WIDE_OPS):
        sel = mags[ops == k]
        want = 0.0 if space[name] is None else float(space[name][magnitude])
        assert (sel.abs() == want).all(), name                                 # the bin is fixed
        if name in TA_WIDE_SIGNED and want != 0:
            assert abs((sel < 0).double().mean().item() - 0.5) < 0.05, name
        else:
            assert (sel >= 0).all(), name


def test_auto_augment_draw_law():
    """the joint law of (op, |magnitude|) in both slots equals the mixture over the 25 sub-policies
    with each op applied at its probability"""
    from scipy.stats import chisquare
    aug = GpuAugment(out_size=96, seed=6, auto_augment='imagenet')
    p = [aug.sample_params(5000) for _ in range(8)]
    ops, mags = torch.cat([q.op for q in p]), torch.cat([q.magnitude for q in p])
    assert ops.shape == (40000, 2)
    space = policy_magnitudes(AA_BINS, 96)
    law = {}
    for sub in AUTO_AUGMENT_IMAGENET:
        for on in itertools.product((0, 1), repeat=2):
            pr = 1.0 / 25
            key = []
            for (name, prob, b), o in zip(sub, on):
                pr *= prob if o else 1 - prob
                key += [AUGMENT_OPS.index(name), 0.0 if b is None else float(space[name][b])] if o else [0, 0.0]
            law[tuple(key)] = law.get(tuple(key), 0.0) + pr
    obs = {}
    for (a, b), (ma, mb) in zip(ops.tolist(), mags.abs().tolist()):
        obs[(a, ma, b, mb)] = obs.get((a, ma, b, mb), 0) + 1
    assert set(obs) <= {k for k, v in law.items() if v > 0}
    keys = [k for k, v in law.items() if v > 0]
    exp = np.array([law[k] for k in keys]) * len(ops)
    got = np.array([obs.get(k, 0) for k in keys])
    assert chisquare(got, exp / exp.sum() * got.sum()).pvalue > 1e-4
    signed = torch.tensor([AUGMENT_OPS[k] in TA_WIDE_SIGNED for k in ops.flatten().tolist()]).view_as(ops)
    sel = mags[signed & (mags != 0)]
    assert abs((sel < 0).double().mean().item() - 0.5) < 0.03
    assert (mags[~signed] >= 0).all()


def test_seeds_are_deterministic_and_crops_do_not_depend_on_the_policy():
    def draw(**kw):
        aug = GpuAugment(out_size=48, seed=11, **kw)
        return [aug.sample_params(64) for _ in range(3)]
    plain = GpuAugment(out_size=48, seed=11)
    boxes = [plain.sample_boxes(64) for _ in range(3)]
    for kw in (dict(auto_augment='ra'), dict(auto_augment='ra', ra_num_ops=4, random_erase=0.5),
               dict(auto_augment='imagenet', random_erase=0.3)):
        a, b = draw(**kw), draw(**kw)
        for pa, pb in zip(a, b):
            for x, y in zip(pa, pb):
                assert torch.equal(x, y)
        for p, bx in zip(a, boxes):
            for x, y in zip(p[:5], bx):
                assert torch.equal(x, y)


# -- the CPU composition ------------------------------------------------------------------------------- #
@pytest.mark.parametrize('first', AUGMENT_OPS)
def test_every_ordered_pair_equals_torchvision(first):
    size = 40
    aug = GpuAugment(out_size=size, seed=3, auto_augment='ra')
    x = _images(2, 52, seed=AUGMENT_OPS.index(first))
    for second in AUGMENT_OPS:
        for sa, sb in ((1, 1), (-1, -1)):
            mags = [_mid(first, size, sa), _mid(second, size, sb)]
            p = _chain_params(aug, 2, [[AUGMENT_OPS.index(first), AUGMENT_OPS.index(second)]] * 2, [mags] * 2)
            assert torch.equal(aug.apply(x, p), _expected(x, aug, p)), (first, second, sa)


@pytest.mark.parametrize('k', [3, 4])
def test_sampled_long_chains_equal_torchvision(k):
    size = 36
    aug = GpuAugment(out_size=size, seed=k, auto_augment='ra', ra_num_ops=k)
    g = torch.Generator().manual_seed(k)
    x = _images(12, 44, seed=k)
    ops = torch.randint(len(AUGMENT_OPS), (12, k), generator=g)
    signs = torch.where(torch.rand(12, k, generator=g) < 0.5, -1, 1)
    mags = [[_mid(AUGMENT_OPS[o], size, s) for o, s in zip(r, t)] for r, t in zip(ops.tolist(), signs.tolist())]
    p = _chain_params(aug, 12, ops, mags)
    assert torch.equal(aug.apply(x, p), _expected(x, aug, p))


@pytest.mark.parametrize('policy', ['ra', 'imagenet'])
def test_full_policy_draws_equal_torchvision(policy):
    aug = GpuAugment(out_size=40, seed=8, auto_augment=policy, random_erase=0.5)
    x = _images(24, 48, seed=4)
    p = aug.sample_params(24)
    y = aug.apply(x, p)
    assert y.dtype == torch.float32 and y.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(y, _expected(x, aug, p))
    assert torch.equal(GpuAugment(out_size=40, seed=8, auto_augment=policy, random_erase=0.5)(x), y)


def test_zero_ops_is_the_plain_rounded_crop():
    aug = GpuAugment(out_size=32, seed=1, auto_augment='ra', ra_num_ops=0)
    x = _images(4, 40)
    p = aug.sample_params(4)
    assert p.op.shape == (4, 0)
    assert torch.equal(aug.apply(x, p), _normalise(_rounded_crops(x, aug, p)))


# -- kernel rows --------------------------------------------------------------------------------------- #
def test_chain_rows_hold_each_op_at_its_columns():
    aug = GpuAugment(out_size=48, seed=2, auto_augment='ra', random_erase=1.0, ra_num_ops=4)
    p = aug.sample_params(64)
    rows = aug.kernel_rows(p, 56)
    assert rows.dtype == np.float32 and rows.shape == (64, AUGMENT_ROW) and AUGMENT_ROW % 4 == 0
    for k in range(4):
        one = aug.kernel_rows(p._replace(op=p.op[:, k], magnitude=p.magnitude[:, k]), 56)
        assert one.shape == (64, AUGMENT_ROW_ONE_OP)
        assert (one[:, :6] == rows[:, :6]).all() and (one[:, 15:19] == rows[:, 15:19]).all()
        col = 6 if k == 0 else AUGMENT_CHAIN_COL + 9 * (k - 1)
        assert (rows[:, col:col + 9] == one[:, 6:15]).all(), k
    # two ops: op 1 keeps the one-op columns, ops 3 and 4 are Identity (all zero)
    two = aug.kernel_rows(p._replace(op=p.op[:, :2], magnitude=p.magnitude[:, :2]), 56)
    assert (two[:, :AUGMENT_CHAIN_COL + 9] == rows[:, :AUGMENT_CHAIN_COL + 9]).all()
    assert (two[:, AUGMENT_CHAIN_COL + 9:] == 0).all()
    # an Invert op writes only its id
    inv = aug.kernel_rows(p._replace(op=torch.full((64, 1), 14), magnitude=torch.zeros(64, 1)), 56)
    assert (inv[:, 6] == 14).all() and (inv[:, 7:15] == 0).all() and (inv[:, 19:] == 0).all()
    with pytest.raises(ValueError, match='at most 4'):
        aug.kernel_rows(p._replace(op=torch.zeros(64, 5, dtype=torch.int64),
                                   magnitude=torch.zeros(64, 5, dtype=torch.float64)), 56)


def test_ta_wide_rows_keep_the_one_op_layout():
    aug = GpuAugment(out_size=48, seed=2, auto_augment='ta_wide', random_erase=0.5)
    p = aug.sample_params(32)
    assert p.op.shape == (32,)
    assert aug.kernel_rows(p, 56).shape == (32, AUGMENT_ROW_ONE_OP)


# -- validation and the command line ------------------------------------------------------------------- #
def test_options_are_validated():
    for bad in ('rand', 'rand_augment', 'autoaugment'):
        with pytest.raises(ValueError, match='auto_augment'):
            GpuAugment(auto_augment=bad)
    for v in (-1, 5, 2.0, True, '2'):
        with pytest.raises(ValueError, match='ra_num_ops'):
            GpuAugment(auto_augment='ra', ra_num_ops=v)
    for v in (-1, 31, 9.0, None):
        with pytest.raises(ValueError, match='ra_magnitude'):
            GpuAugment(auto_augment='ra', ra_magnitude=v)
    for v in (0, 4):
        GpuAugment(auto_augment='ra', ra_num_ops=v)
    GpuAugment(auto_augment='ra', ra_magnitude=30)
    # the chain allocates no shared memory: the policies accept every output size TrivialAugment does
    big = next(o for o in range(200, 400) if augment_smem_bytes(o) > 232448)
    for policy in ('ta_wide', 'ra', 'imagenet'):
        GpuAugment(out_size=big - 1, auto_augment=policy, ra_num_ops=4)
        with pytest.raises(ValueError, match='shared memory'):
            GpuAugment(out_size=big, auto_augment=policy)


def _parse(argv, tmp_path, adpsgd=False):
    if adpsgd:
        from stochastic_gradient_push_b200.cli import gossip_sgd_adpsgd as m
    else:
        from stochastic_gradient_push_b200.cli import gossip_sgd as m
    return m.parse_args(argv + ['--checkpoint_dir', str(tmp_path) + '/', '--device', 'cpu'])


@pytest.mark.parametrize('adpsgd', [False, True])
def test_flags_parse(tmp_path, adpsgd):
    args = _parse(['--dataset_dir', str(tmp_path)], tmp_path, adpsgd)
    assert args.auto_augment == 'none' and args.ra_num_ops == 2 and args.ra_magnitude == 9
    args = _parse(['--dataset_dir', str(tmp_path), '--auto_augment', 'ra', '--ra_num_ops', '3',
                   '--ra_magnitude', '15'], tmp_path, adpsgd)
    assert args.auto_augment == 'ra' and args.ra_num_ops == 3 and args.ra_magnitude == 15
    assert _parse(['--dataset_dir', str(tmp_path), '--auto_augment', 'imagenet'], tmp_path,
                  adpsgd).auto_augment == 'imagenet'
    for flag, v in (('--ra_num_ops', '5'), ('--ra_num_ops', '-1'), ('--ra_magnitude', '31')):
        with pytest.raises(ValueError, match=flag):
            _parse(['--dataset_dir', str(tmp_path), '--auto_augment', 'ra', flag, v], tmp_path, adpsgd)


@pytest.mark.parametrize('bad', ['rand', 'rand_augment'])
def test_unknown_policies_stay_refused(tmp_path, capsys, bad):
    with pytest.raises(SystemExit):
        _parse(['--auto_augment', bad], tmp_path)
    assert 'invalid choice' in capsys.readouterr().err


@pytest.mark.parametrize('policy', ['ra', 'imagenet'])
def test_synthetic_data_refuses_the_policies(tmp_path, policy):
    with pytest.raises(ValueError, match='synthetic data'):
        _parse(['--auto_augment', policy], tmp_path)


def test_folder_transforms_put_the_policy_after_the_flip(tmp_path):
    import torchvision.transforms as T
    from stochastic_gradient_push_b200.cli.common import folder_transforms
    base = ['--dataset_dir', str(tmp_path)]
    kinds = lambda c: [type(t) for t in c.transforms]  # noqa: E731
    c = folder_transforms(_parse(base + ['--auto_augment', 'ra', '--ra_num_ops', '3', '--ra_magnitude', '12',
                                         '--random_erase', '0.25'], tmp_path))
    assert kinds(c) == [T.RandomResizedCrop, T.RandomHorizontalFlip, T.RandAugment, T.ToTensor, T.Normalize,
                        T.RandomErasing]
    assert c.transforms[2].num_ops == 3 and c.transforms[2].magnitude == 12
    c = folder_transforms(_parse(base + ['--auto_augment', 'imagenet'], tmp_path))
    assert kinds(c) == [T.RandomResizedCrop, T.RandomHorizontalFlip, T.AutoAugment, T.ToTensor, T.Normalize]
    assert c.transforms[2].policy == T.AutoAugmentPolicy.IMAGENET
    v = folder_transforms(_parse(base + ['--auto_augment', 'ra'], tmp_path), train=False)
    assert kinds(v) == [T.Resize, T.CenterCrop, T.ToTensor, T.Normalize]


def test_shard_batches_take_the_policy(tmp_path):
    from stochastic_gradient_push_b200.cli import common
    args = _parse(['--dataset_dir', str(tmp_path), '--data_format', 'shards', '--auto_augment', 'ra',
                   '--ra_num_ops', '3', '--ra_magnitude', '20', '--image_size', '24'], tmp_path)
    x = _images(5, 32, seed=2)
    train = common.device_batch(args, x, train=True)
    aug = args._gpu_augment
    assert aug.auto_augment == 'ra' and aug.ra_num_ops == 3 and aug.ra_magnitude == 20
    twin = GpuAugment(out_size=24, seed=args.seed * 7919 + args.rank, auto_augment='ra', ra_num_ops=3,
                      ra_magnitude=20)
    assert torch.equal(train, twin.apply(x, twin.sample_params(5)))
    assert torch.equal(common.device_batch(args, x, train=False), GpuAugment(out_size=24)(x, train=False))
