"""TrivialAugmentWide and random erasing in data.GpuAugment, on the CPU: the host magnitude tables and
draws, determinism, the reference composition against torchvision, and the CLI flags."""
import numpy as np
import pytest
import torch

from stochastic_gradient_push_b200.data.shards import (TA_WIDE_BINS, TA_WIDE_OPS, TA_WIDE_SIGNED, AugmentParams,
                                                       GpuAugment, augment_smem_bytes, ta_wide_magnitudes)

tv2 = pytest.importorskip('torchvision.transforms.v2')
import torchvision.transforms.v2.functional as TF  # noqa: E402


def _images(n, size, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (n, size, size, 3), dtype=torch.uint8, generator=g)


# -- tables and draws ---------------------------------------------------------------------------------- #
def test_magnitude_tables_equal_torchvision():
    space = tv2.TrivialAugmentWide()._AUGMENTATION_SPACE
    assert tuple(space) == TA_WIDE_OPS
    mine = ta_wide_magnitudes()
    for name, (fn, signed) in space.items():
        ref = fn(TA_WIDE_BINS, 224, 224)
        assert (name in TA_WIDE_SIGNED) == signed, name
        if ref is None:
            assert mine[name] is None, name
        else:
            assert mine[name].dtype == ref.dtype and torch.equal(mine[name], ref), name


def test_op_bin_and_sign_frequencies_are_uniform():
    from scipy.stats import chisquare
    aug = GpuAugment(out_size=32, seed=5, auto_augment='ta_wide')
    tables = ta_wide_magnitudes()
    ops, mags = [], []
    for _ in range(40):
        p = aug.sample_params(1000)
        ops.append(p.op)
        mags.append(p.magnitude)
    ops, mags = torch.cat(ops), torch.cat(mags)
    assert chisquare(torch.bincount(ops, minlength=14).numpy()).pvalue > 1e-4
    bins = []
    for k, name in enumerate(TA_WIDE_OPS):
        sel = mags[ops == k]
        if tables[name] is None:
            assert (sel == 0).all()
            continue
        table = tables[name].double()
        idx = (sel.abs().view(-1, 1) - table.view(1, -1)).abs().argmin(1)
        assert torch.equal(table[idx], sel.abs()), name               # every magnitude is a table entry
        if len(table.unique()) == TA_WIDE_BINS:                        # (Posterize's bins share values)
            bins.append(idx)
        if name in TA_WIDE_SIGNED:
            neg = (sel < 0).sum().item()
            nonzero = (sel != 0).sum().item()
            assert abs(neg / nonzero - 0.5) < 0.05, name
        else:
            assert (sel >= 0).all(), name
    assert chisquare(torch.bincount(torch.cat(bins), minlength=31).numpy()).pvalue > 1e-4


@pytest.mark.parametrize('size', [224, 64])
def test_erase_boxes_obey_the_rules(size):
    aug = GpuAugment(out_size=size, seed=1, random_erase=0.5)
    e = torch.cat([aug.sample_params(2000).erase for _ in range(5)])
    on = e[:, 2] > 0
    assert abs(on.float().mean().item() - 0.5) < 0.03
    top, left, h, w = e[on].unbind(1)
    assert (h < size).all() and (w < size).all() and (h >= 1).all() and (w >= 1).all()
    assert (top >= 0).all() and (left >= 0).all() and (top + h <= size).all() and (left + w <= size).all()
    area = (h * w).double() / (size * size)
    # the rounded sides keep the drawn area and ratio up to half a pixel on each side
    slack = lambda x: (x + 0.5) / (x - 0.5).clamp(min=0.5)  # noqa: E731
    assert (area <= 0.33 * slack(h) * slack(w)).all() and (area >= 0.02 / (slack(h) * slack(w))).all()
    ratio = h.double() / w.double()
    assert (ratio <= 3.3 * slack(h) * slack(w)).all() and (ratio >= 0.3 / (slack(h) * slack(w))).all()
    assert (e[~on] == 0).all()
    # positions are uniform over the free range
    free = (size - h + 1).double()
    u = (top.double() + 0.5) / free
    assert abs(u.mean().item() - 0.5) < 0.03


def test_erase_probability_zero_and_one():
    assert (GpuAugment(out_size=32, seed=2, random_erase=1e-9).sample_params(5000).erase == 0).all()
    e = GpuAugment(out_size=224, seed=2, random_erase=1.0).sample_params(5000).erase
    # with p = 1 only draws whose 10 attempts all miss leave an image unerased: rare at 224
    assert (e[:, 2] > 0).float().mean().item() > 0.99


def test_same_seed_same_params_and_crops_do_not_depend_on_the_options():
    def draw(**kw):
        aug = GpuAugment(out_size=48, seed=11, **kw)
        return [aug.sample_params(64) for _ in range(3)]
    a, b = draw(auto_augment='ta_wide', random_erase=0.3), draw(auto_augment='ta_wide', random_erase=0.3)
    for pa, pb in zip(a, b):
        for x, y in zip(pa, pb):
            assert torch.equal(x, y)
    plain = GpuAugment(out_size=48, seed=11)
    boxes = [plain.sample_boxes(64) for _ in range(3)]
    for other in (a, draw(auto_augment='ta_wide'), draw(random_erase=1.0)):
        for p, bx in zip(other, boxes):
            for x, y in zip(p[:5], bx):
                assert torch.equal(x, y)


def test_options_are_validated():
    with pytest.raises(ValueError, match='auto_augment'):
        GpuAugment(auto_augment='rand')
    for p in (-0.1, 1.5, float('nan')):
        with pytest.raises(ValueError, match='random_erase'):
            GpuAugment(random_erase=p)
    big = next(o for o in range(200, 400) if augment_smem_bytes(o) > 232448)
    assert big > 256
    with pytest.raises(ValueError, match='shared memory'):
        GpuAugment(out_size=big, auto_augment='ta_wide')
    GpuAugment(out_size=big - 1, random_erase=0.5)
    GpuAugment(out_size=big)                                          # the default path has no such limit


# -- the reference composition ------------------------------------------------------------------------- #
def _params(aug, n, op, magnitude, erase=None):
    cx, cy, w, h, flip = aug.sample_boxes(n)
    return AugmentParams(cx, cy, w, h, flip, torch.full((n,), op, dtype=torch.int64),
                         torch.full((n,), float(magnitude), dtype=torch.float64),
                         torch.zeros(n, 4, dtype=torch.int64) if erase is None else erase)


def _rounded_crops(x, aug, p):
    theta = GpuAugment.crop_theta(p.cx, p.cy, p.w, p.h, p.flip)
    grid = torch.nn.functional.affine_grid(theta, (x.shape[0], 3, aug.out, aug.out), align_corners=False)
    y = torch.nn.functional.grid_sample(x.permute(0, 3, 1, 2).float(), grid, mode='bilinear',
                                        padding_mode='border', align_corners=False)
    return y.round().clamp(0, 255).to(torch.uint8)


def _normalise(img):
    mean = torch.tensor((0.485, 0.456, 0.406)).view(3, 1, 1) * 255.0
    inv = 1.0 / (torch.tensor((0.229, 0.224, 0.225)).view(3, 1, 1) * 255.0)
    return (img.float() - mean) * inv


@pytest.mark.parametrize('op', TA_WIDE_OPS)
def test_cpu_composition_equals_torchvision_trivial_augment(op):
    aug = GpuAugment(out_size=40, seed=3, auto_augment='ta_wide')
    x = _images(4, 56, seed=TA_WIDE_OPS.index(op))
    ta = tv2.TrivialAugmentWide()
    table = ta_wide_magnitudes()[op]
    for b in (0, 1, 15, 30):
        for sign in ((1, -1) if op in TA_WIDE_SIGNED else (1,)):
            mag = 0.0 if table is None else sign * float(table[b])
            p = _params(aug, 4, TA_WIDE_OPS.index(op), mag)
            y = aug.apply(x, p)
            crops = _rounded_crops(x, aug, p)
            for i in range(4):
                ref = ta._apply_image_or_video_transform(crops[i], op, mag, interpolation=ta.interpolation,
                                                         fill=ta._fill)
                assert torch.equal(y[i], _normalise(ref)), (op, b, sign)


def test_cpu_composition_erases_as_torchvision():
    aug = GpuAugment(out_size=40, seed=4, auto_augment='ta_wide', random_erase=1.0)
    x = _images(16, 48, seed=9)
    p = aug.sample_params(16)
    assert (p.erase[:, 2] > 0).sum() >= 12
    y = aug.apply(x, p)
    crops = _rounded_crops(x, aug, p)
    ta = tv2.TrivialAugmentWide()
    for i in range(16):
        name = TA_WIDE_OPS[int(p.op[i])]
        img = _normalise(ta._apply_image_or_video_transform(crops[i], name, float(p.magnitude[i]),
                                                            interpolation=ta.interpolation, fill=ta._fill))
        top, left, h, w = p.erase[i].tolist()
        if h:
            img = TF.erase(img, top, left, h, w, torch.zeros(1))
        assert torch.equal(y[i], img)
    assert y.is_contiguous(memory_format=torch.channels_last) and y.dtype == torch.float32


def test_call_uses_the_draws_and_evaluation_never_augments():
    x = _images(6, 40, seed=1)
    a = GpuAugment(out_size=32, seed=7, auto_augment='ta_wide', random_erase=0.5)
    b = GpuAugment(out_size=32, seed=7, auto_augment='ta_wide', random_erase=0.5)
    assert torch.equal(a(x), b.apply(x, b.sample_params(6)))
    assert torch.equal(a(x, train=False), GpuAugment(out_size=32, seed=7)(x, train=False))
    bf = GpuAugment(out_size=32, seed=7, auto_augment='ta_wide', dtype=torch.bfloat16)(x)
    assert bf.dtype == torch.bfloat16
    plain = GpuAugment(out_size=32, seed=7, random_erase=0.5, channels_last=False)(x)
    assert plain.is_contiguous()


def test_kernel_rows_hold_the_op_scalars_in_fp32():
    aug = GpuAugment(out_size=32, seed=0)
    n = len(TA_WIDE_OPS)
    cx, cy, w, h, flip = aug.sample_boxes(n)
    mags = torch.tensor([0.0, 0.33, -0.33, 12.8, -3.2, 94.5, -0.5, 0.627, -0.264, 0.99, 4.0, 0.4, 0.0, 0.0],
                        dtype=torch.float64)
    erase = torch.zeros(n, 4, dtype=torch.int64)
    erase[3] = torch.tensor([2, 5, 7, 9])
    p = AugmentParams(cx, cy, w, h, flip, torch.arange(n), mags, erase)
    rows = aug.kernel_rows(p, 40)
    assert rows.dtype == np.float32 and rows.shape == (n, 24)
    assert rows[:, 6].tolist() == list(range(n))
    assert rows[6, 7] == np.float32(1.0 - 0.5)
    assert rows[7, 7] == np.float32(1.627) and rows[7, 8] == np.float32(1.0 - 1.627)
    assert rows[9, 8] == np.float32(1.0 - 1.99)
    assert rows[10, 7] == 0xF0 and rows[11, 7] == np.float32(255 * 0.4)
    assert rows[3, 15:19].tolist() == [2, 9, 5, 14]
    # TranslateX by int(12.8) = 12 pixels: the inverse map shifts the source 12 px left
    assert rows[3, 9:15].tolist() == [np.float32(1 / 16), 0.0, np.float32(-12 / 16), 0.0, np.float32(1 / 16), 0.0]
    theta = GpuAugment.crop_theta(cx, cy, w, h, flip).reshape(n, 6).numpy()
    assert (rows[:, :6] == theta).all()


# -- command line -------------------------------------------------------------------------------------- #
def _parse(argv, tmp_path):
    from stochastic_gradient_push_b200.cli import gossip_sgd
    return gossip_sgd.parse_args(argv + ['--checkpoint_dir', str(tmp_path) + '/', '--device', 'cpu'])


def test_flags_parse_and_default_off(tmp_path):
    args = _parse([], tmp_path)
    assert args.auto_augment == 'none' and args.random_erase == 0.0
    args = _parse(['--dataset_dir', str(tmp_path), '--auto_augment', 'ta_wide', '--random_erase', '0.25'], tmp_path)
    assert args.auto_augment == 'ta_wide' and args.random_erase == 0.25
    from stochastic_gradient_push_b200.cli.common import build_parser
    assert build_parser(adpsgd=True).parse_args(['--auto_augment', 'ta_wide']).auto_augment == 'ta_wide'


@pytest.mark.parametrize('p', ['-0.1', '1.01', 'nan'])
def test_random_erase_must_lie_in_the_unit_interval(tmp_path, p):
    with pytest.raises(ValueError, match='--random_erase must be in'):
        _parse(['--dataset_dir', str(tmp_path), '--random_erase', p], tmp_path)


def test_unknown_policy_is_refused(tmp_path, capsys):
    with pytest.raises(SystemExit):
        _parse(['--auto_augment', 'rand_augment'], tmp_path)
    assert 'invalid choice' in capsys.readouterr().err


@pytest.mark.parametrize('extra', [['--auto_augment', 'ta_wide'], ['--random_erase', '0.1']])
def test_synthetic_data_refuses_the_flags(tmp_path, extra):
    with pytest.raises(ValueError, match='synthetic data'):
        _parse(extra, tmp_path)
    with pytest.raises(ValueError, match='synthetic data'):
        _parse(extra + ['--dataset_dir', str(tmp_path), '--synthetic', 'True'], tmp_path)


def test_folder_transforms_follow_the_recipe_order(tmp_path):
    import torchvision.transforms as T
    from stochastic_gradient_push_b200.cli.common import folder_transforms
    base = ['--dataset_dir', str(tmp_path)]
    kinds = lambda c: [type(t) for t in c.transforms]  # noqa: E731
    plain = [T.RandomResizedCrop, T.RandomHorizontalFlip, T.ToTensor, T.Normalize]
    assert kinds(folder_transforms(_parse(base, tmp_path))) == plain
    args = _parse(base + ['--auto_augment', 'ta_wide', '--random_erase', '0.25'], tmp_path)
    c = folder_transforms(args)
    assert kinds(c) == [T.RandomResizedCrop, T.RandomHorizontalFlip, T.TrivialAugmentWide, T.ToTensor,
                        T.Normalize, T.RandomErasing]
    assert c.transforms[-1].p == 0.25 and c.transforms[-1].value == 0
    assert kinds(folder_transforms(_parse(base + ['--random_erase', '0.5'], tmp_path))) == plain + [T.RandomErasing]
    # validation: unchanged by the flags
    val = [T.Resize, T.CenterCrop, T.ToTensor, T.Normalize]
    for a in (_parse(base, tmp_path), args):
        v = folder_transforms(a, train=False)
        assert kinds(v) == val and v.transforms[0].size == int(a.image_size * 256 / 224)


def test_shard_validation_batches_are_not_augmented(tmp_path):
    from stochastic_gradient_push_b200.cli import common
    args = _parse(['--dataset_dir', str(tmp_path), '--data_format', 'shards', '--auto_augment', 'ta_wide',
                   '--random_erase', '1.0', '--image_size', '24'], tmp_path)
    x = _images(5, 32, seed=2)
    val = common.device_batch(args, x, train=False)
    assert args._gpu_augment.auto_augment == 'ta_wide' and args._gpu_augment.random_erase == 1.0
    assert torch.equal(val, GpuAugment(out_size=24)(x, train=False))
    train = common.device_batch(args, x, train=True)
    assert train.shape == val.shape and (train == 0).any()
