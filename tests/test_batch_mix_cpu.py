"""Batch mixup / CutMix (ops/batch_mix.py) without a GPU: the host sampler, the plain torch composition
of the mixed batch and of the two-target loss against hand-written formulas, argument checks, the CLI
flags, and a two-rank gloo run of the CLI with mixing on."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from stochastic_gradient_push_b200.cli import common
from stochastic_gradient_push_b200.ops import batch_mix as bm
from stochastic_gradient_push_b200.ops import fused_loss


# --------------------------------------------------------------------------- #
# sampler
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize('alpha', [0.2, 1.0, 2.0])
def test_mixup_lam_has_beta_moments(alpha):
    mix = bm.BatchMix(mixup_alpha=alpha, seed=5)
    lam = np.array([mix.sample(32, 32).lam for _ in range(20000)])
    var = 1.0 / (4.0 * (2.0 * alpha + 1.0))                  # Beta(a, a): mean 1/2, var 1/(4(2a+1))
    assert abs(lam.mean() - 0.5) < 4 * math.sqrt(var / lam.size)
    assert abs(lam.var() - var) < 0.1 * var
    assert lam.min() >= 0.0 and lam.max() <= 1.0


def test_draw_is_a_pure_function_of_seed_rank_and_iteration():
    a = bm.BatchMix(0.2, 1.0, seed=11, rank=3)
    first = [a.sample(224, 224) for _ in range(50)]
    b = bm.BatchMix(0.2, 1.0, seed=11, rank=3)
    assert [b.sample(224, 224, itr=i) for i in range(50)] == first
    b.iteration = 17                                           # a resumed run
    assert b.sample(224, 224) == first[17] and b.iteration == 18
    other_rank = bm.BatchMix(0.2, 1.0, seed=11, rank=4)
    other_seed = bm.BatchMix(0.2, 1.0, seed=12, rank=3)
    assert [other_rank.sample(224, 224, itr=i) for i in range(50)] != first
    assert [other_seed.sample(224, 224, itr=i) for i in range(50)] != first
    assert len(set(p.lam for p in first)) > 40                 # the iterations differ from each other


@pytest.mark.parametrize('H,W', [(224, 224), (17, 31), (1, 5)])
def test_cutmix_box_is_inside_the_image_and_sets_lam(H, W):
    mix = bm.BatchMix(cutmix_alpha=1.0, seed=2)
    areas = 0
    for i in range(2000):
        p = mix.sample(H, W)
        assert p.mode == bm.CUTMIX
        assert 0 <= p.y0 <= p.y1 <= H and 0 <= p.x0 <= p.x1 <= W
        area = (p.y1 - p.y0) * (p.x1 - p.x0)
        assert p.lam == float(np.float32(1.0 - area / float(H * W)))
        areas += area > 0
    if H * W > 100:
        assert areas > 1000


def test_switch_prob_and_mix_prob():
    both = bm.BatchMix(0.2, 1.0, switch_prob=0.5, seed=1)
    modes = [both.sample(8, 8).mode for _ in range(4000)]
    assert abs(modes.count(bm.CUTMIX) / 4000.0 - 0.5) < 0.05 and bm.NO_MIX not in modes
    assert {bm.BatchMix(0.2, 1.0, switch_prob=1.0).sample(8, 8).mode for _ in range(50)} == {bm.CUTMIX}
    assert {bm.BatchMix(0.2, 1.0, switch_prob=0.0).sample(8, 8).mode for _ in range(50)} == {bm.MIXUP}
    never = bm.BatchMix(0.2, 1.0, mix_prob=0.0, seed=4)
    assert all(never.sample(8, 8) == bm.MixParams(1.0, bm.NO_MIX, 0, 0, 0, 0) for _ in range(500))
    half = bm.BatchMix(mixup_alpha=0.2, mix_prob=0.3, seed=4)
    mixed = sum(half.sample(8, 8).mode != bm.NO_MIX for _ in range(4000))
    assert abs(mixed / 4000.0 - 0.3) < 0.05
    assert not bm.BatchMix().enabled and bm.BatchMix().sample(8, 8).mode == bm.NO_MIX


@pytest.mark.parametrize('kw', [
    dict(mixup_alpha=-0.1), dict(cutmix_alpha=-1), dict(mixup_alpha=float('nan')),
    dict(cutmix_alpha=float('inf')), dict(mix_prob=1.5), dict(mix_prob=-0.1), dict(switch_prob=2.0),
    dict(switch_prob=float('nan')),
])
def test_bad_arguments_raise(kw):
    with pytest.raises(ValueError):
        bm.BatchMix(**kw)


# --------------------------------------------------------------------------- #
# the torch composition
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize('B', [1, 6, 7])
@pytest.mark.parametrize('channels_last', [False, True])
def test_cpu_apply_mixup_and_cutmix(B, channels_last):
    x = torch.randn(B, 3, 5, 9)
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    mix = bm.BatchMix(0.2, 1.0)
    p = bm.MixParams(0.375, bm.MIXUP, 0, 0, 0, 0)
    out = mix.apply(x, params=p)
    want = 0.375 * x + 0.625 * x.flip(0)
    torch.testing.assert_close(out, want, rtol=1e-6, atol=1e-6)
    if B % 2:
        mid = B // 2
        torch.testing.assert_close(out[mid], x[mid], rtol=1e-6, atol=1e-7)
    assert torch.equal(mix.state[:6], torch.tensor([0.375, 1, 0, 0, 0, 0]))
    p = bm.MixParams(0.5, bm.CUTMIX, 1, 4, 2, 7)
    out = mix.apply(x, params=p)
    want = x.clone()
    want[:, :, 1:4, 2:7] = x.flip(0)[:, :, 1:4, 2:7]
    assert torch.equal(out, want)
    if B % 2:
        assert torch.equal(out[B // 2], x[B // 2])
    assert torch.equal(mix.apply(x, params=bm.MixParams(1.0, bm.NO_MIX, 0, 0, 0, 0)), x)


def _two_ce(logits, target, lam, eps):
    """hand-written: lam CE_eps(z, t) + (1 - lam) CE_eps(z, t flipped), rows with an out-of-range
    target on either side dropped, mean over all B rows"""
    B, C = logits.shape
    tb = target.flip(0)
    ok = (target >= 0) & (target < C) & (tb >= 0) & (tb < C)
    total = logits.new_zeros(())
    for i in range(B):
        if ok[i]:
            total = total + lam * F.cross_entropy(logits[i:i + 1], target[i:i + 1], label_smoothing=eps) \
                + (1 - lam) * F.cross_entropy(logits[i:i + 1], tb[i:i + 1], label_smoothing=eps)
    return total / B


@pytest.mark.parametrize('eps', [0.0, 0.1])
@pytest.mark.parametrize('lam', [0.0, 0.37, 1.0])
@pytest.mark.parametrize('B', [1, 8, 9])
def test_mixed_loss_matches_two_cross_entropies(B, lam, eps):
    C = 11
    g = torch.Generator().manual_seed(B * 7 + int(lam * 100))
    logits = (torch.randn(B, C, generator=g) * 2).requires_grad_(True)
    target = torch.randint(0, C, (B,), generator=g)
    if B > 1:
        target[0] = target[-1]                           # an a == b row pair
    if B > 3:
        target[2] = C + 4                                # out of range: rows 2 and B-3 drop out
    state = torch.tensor([lam, 1, 0, 0, 0, 0, 0, 0])
    loss, metrics = fused_loss.fused_cross_entropy(logits, target, eps, mix=state)
    ref_logits = logits.detach().clone().requires_grad_(True)
    want = _two_ce(ref_logits, target, lam, eps)
    torch.testing.assert_close(loss, want, rtol=1e-5, atol=1e-6)
    loss.backward()
    want.backward()
    torch.testing.assert_close(logits.grad, ref_logits.grad, rtol=1e-5, atol=1e-6)
    if B > 3:
        assert torch.all(logits.grad[2] == 0) and torch.all(logits.grad[B - 3] == 0)
    # accuracies count against the row's own target
    pred = logits.detach().topk(5, 1).indices
    p1 = (pred[:, 0] == target).sum().item() * 100.0 / B
    p5 = (pred == target[:, None]).any(1).sum().item() * 100.0 / B
    torch.testing.assert_close(metrics[1].item(), p1)
    torch.testing.assert_close(metrics[2].item(), p5)


def test_criterion_without_mix_is_unchanged():
    logits = torch.randn(6, 10)
    target = torch.randint(0, 10, (6,))
    crit = fused_loss.FusedCrossEntropyWithAccuracy(0.1)
    a = crit(logits, target)
    b = crit(logits, target, mix=None)
    assert torch.equal(a, b) and torch.equal(a, F.cross_entropy(logits, target, label_smoothing=0.1))


# --------------------------------------------------------------------------- #
# CLI
# --------------------------------------------------------------------------- #
def _parse(tmp_path, extra, adpsgd=False):
    args = common.build_parser(adpsgd=adpsgd).parse_args(
        ['--device', 'cpu', '--backend', 'gloo', '--checkpoint_dir', str(tmp_path) + '/'] + extra)
    return common.finalize_args(args, adpsgd=adpsgd)


@pytest.mark.parametrize('adpsgd', [False, True])
def test_mix_flags_parse(tmp_path, adpsgd):
    d = common.build_parser(adpsgd=adpsgd).parse_args([])
    assert (d.mixup_alpha, d.cutmix_alpha, d.mix_prob, d.mix_switch_prob) == (0.0, 0.0, 1.0, 0.5)
    a = _parse(tmp_path, ['--mixup_alpha', '0.2', '--cutmix_alpha', '1.0', '--mix_prob', '0.8',
                          '--mix_switch_prob', '0.25', '--label_smoothing', '0.1'], adpsgd)
    m = common.make_batch_mix(a)
    assert (m.mixup_alpha, m.cutmix_alpha, m.mix_prob, m.switch_prob) == (0.2, 1.0, 0.8, 0.25)
    assert (m.seed, m.rank) == (a.seed, a.rank)
    assert common.make_batch_mix(_parse(tmp_path, [], adpsgd)) is None


@pytest.mark.parametrize('adpsgd', [False, True])
@pytest.mark.parametrize('extra,what', [
    (['--mixup_alpha', '-0.2'], '--mixup_alpha'),
    (['--cutmix_alpha', '-1'], '--cutmix_alpha'),
    (['--cutmix_alpha', 'inf'], '--cutmix_alpha'),
    (['--mix_prob', '1.5'], '--mix_prob'),
    (['--mix_switch_prob', '-0.5'], '--mix_switch_prob'),
    (['--mix_prob', 'nan'], '--mix_prob'),
])
def test_mix_flags_are_validated(tmp_path, adpsgd, extra, what):
    with pytest.raises(ValueError, match=what):
        _parse(tmp_path, extra, adpsgd)


def test_gossip_sgd_cli_mixup_cutmix_two_ranks_cpu(tmp_path, master_port):
    from test_cli_and_experiment import COMMON, _torchrun
    out = _torchrun(2, 'gossip_sgd.py', COMMON + [
        '--push_sum', 'True', '--graph_type', '5', '--mixup_alpha', '0.2', '--cutmix_alpha', '1.0',
        '--label_smoothing', '0.1', '--num_epochs', '2', '--checkpoint_dir', str(tmp_path) + '/',
        '--num_itr_ignore', '0'], master_port)
    assert out.returncode == 0, out.stdout[-3000:]
    for r in range(2):
        lines = open(str(tmp_path / ('out_r%d_n2.csv' % r))).read().splitlines()
        rows = [l.split(',') for l in lines[5:]]
        assert rows and all(len(row) == 18 for row in rows)
        assert any(row[1] == '-1' for row in rows)             # validation ran (unmixed)
        train = [row for row in rows if row[1] != '-1']
        assert train and all(float(row[11]) == float(row[11]) for row in train)
