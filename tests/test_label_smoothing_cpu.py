"""Label smoothing of the fused loss module's CPU fallback, the polynomial learning-rate policy
(``--lr_policy poly``, ``--warmup_epochs``) and the flag checks of both additions."""
import types

import pytest
import torch
import torch.nn.functional as F

from stochastic_gradient_push_b200.cli import common
from stochastic_gradient_push_b200.ops import fused_loss


# --------------------------------------------------------------------------- #
# loss
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize('eps', [0.0, 0.1, 0.5, 1.0])
def test_cpu_fallback_matches_torch_label_smoothing(eps):
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(40, 17, generator=g) * 3).requires_grad_(True)
    target = torch.randint(0, 17, (40,), generator=g)
    crit = fused_loss.FusedCrossEntropyWithAccuracy(label_smoothing=eps)
    loss = crit(logits, target)
    loss.backward()
    ref = logits.detach().clone().requires_grad_(True)
    want = F.cross_entropy(ref, target, label_smoothing=eps)
    want.backward()
    torch.testing.assert_close(loss, want)
    torch.testing.assert_close(crit.metrics[0], want.detach())
    torch.testing.assert_close(logits.grad, ref.grad)
    pred = logits.detach().topk(5, 1)[1]
    torch.testing.assert_close(crit.metrics[1], (pred[:, 0] == target).float().mean() * 100)
    torch.testing.assert_close(crit.metrics[2], (pred == target[:, None]).any(1).float().mean() * 100)
    loss2, m2 = fused_loss.fused_cross_entropy(logits.detach(), target, label_smoothing=eps)
    torch.testing.assert_close(loss2, want.detach())


@pytest.mark.parametrize('eps', [-0.1, 1.5, float('nan'), float('inf')])
def test_invalid_label_smoothing_raises(eps):
    with pytest.raises(ValueError, match='label_smoothing'):
        fused_loss.FusedCrossEntropyWithAccuracy(label_smoothing=eps)
    with pytest.raises(ValueError, match='label_smoothing'):
        fused_loss.fused_cross_entropy(torch.randn(4, 5), torch.zeros(4, dtype=torch.long), eps)
    with pytest.raises(ValueError, match='label_smoothing'):
        fused_loss.reference_loss_and_accuracy(torch.randn(4, 5), torch.zeros(4, dtype=torch.long), eps)


def test_default_criterion_is_unsmoothed():
    assert fused_loss.FusedCrossEntropyWithAccuracy().label_smoothing == 0.0


# --------------------------------------------------------------------------- #
# learning-rate policy
# --------------------------------------------------------------------------- #
def _args(**kw):
    base = dict(lr=0.1, batch_size=256, world_size=8, warmup=True, num_epochs=10, warmup_epochs=2,
                lr_policy='poly', poly_power=2.0, end_lr=1e-4, lr_schedule={30: 0.1, 60: 0.1, 80: 0.1})
    base.update(kw)
    return types.SimpleNamespace(**base)


TARGET = 0.1 * 256 * 8 / 256
IPE = 50


def _all_rates(a):
    return [common.learning_rate_at(a, e, i, IPE) for e in range(a.num_epochs) for i in range(IPE)]


def test_poly_warmup_endpoints():
    a = _args()
    assert common.learning_rate_at(a, 0, 0, IPE) == pytest.approx(0.1 + (TARGET - 0.1) / (2 * IPE), abs=1e-12)
    assert common.learning_rate_at(a, 1, IPE - 1, IPE) == pytest.approx(TARGET, abs=1e-12)


def test_poly_first_post_warmup_iteration_is_target():
    a = _args()
    assert common.learning_rate_at(a, 2, 0, IPE) == pytest.approx(TARGET, abs=1e-12)


@pytest.mark.parametrize('power', [2.0, 1.0, 0.5])
def test_poly_last_iteration(power):
    a = _args(poly_power=power)
    T, W = 10 * IPE, 2 * IPE
    want = 1e-4 + (TARGET - 1e-4) * (1.0 / (T - W)) ** power
    assert common.learning_rate_at(a, 9, IPE - 1, IPE) == pytest.approx(want, rel=1e-9, abs=1e-15)


def test_poly_never_increases_after_warmup():
    a = _args()
    rates = _all_rates(a)[2 * IPE:]
    assert all(y <= x for x, y in zip(rates, rates[1:]))
    assert rates[0] == pytest.approx(TARGET) and rates[-1] > a.end_lr


def test_poly_power_one_is_linear():
    a = _args(poly_power=1.0)
    rates = _all_rates(a)[2 * IPE:]
    steps = [x - y for x, y in zip(rates, rates[1:])]
    want = (TARGET - a.end_lr) / (8 * IPE)
    assert all(s == pytest.approx(want, rel=1e-6) for s in steps)


def test_poly_without_warmup_decays_from_the_first_iteration():
    a = _args(warmup=False)
    rates = _all_rates(a)
    assert rates[0] == pytest.approx(TARGET, abs=1e-12)
    assert rates[1] < rates[0]
    assert rates[-1] == pytest.approx(1e-4 + (TARGET - 1e-4) * (1.0 / (10 * IPE)) ** 2, rel=1e-9)


def test_poly_whole_epochs_without_itr():
    a = _args()
    assert common.learning_rate_at(a, 2) == pytest.approx(TARGET)
    assert common.learning_rate_at(a, 6) == pytest.approx(1e-4 + (TARGET - 1e-4) * 0.5 ** 2)
    assert common.learning_rate_at(a, 10) == pytest.approx(1e-4)


def test_small_target_skips_the_ramp_under_poly():
    a = _args(batch_size=32, world_size=2)
    small = 0.1 * 32 * 2 / 256
    assert common.learning_rate_at(a, 0, 0, IPE) == small
    assert common.learning_rate_at(a, 2, 0, IPE) == pytest.approx(small)


def test_warmup_epochs_only_changes_the_step_ramp_length():
    base = types.SimpleNamespace(lr=0.1, batch_size=256, world_size=8, warmup=True,
                                 lr_schedule={30: 0.1, 60: 0.1, 80: 0.1})
    five = types.SimpleNamespace(**dict(vars(base), warmup_epochs=5, lr_policy='step'))
    # the defaults reproduce the fields-absent policy bit for bit
    for e in (0, 3, 4, 5, 29, 30, 85):
        for i in (0, 17, IPE - 1):
            assert common.learning_rate_at(five, e, i, IPE) == common.learning_rate_at(base, e, i, IPE)
    for w in (1, 3, 8):
        a = types.SimpleNamespace(**dict(vars(base), warmup_epochs=w, lr_policy='step'))
        for e in range(w):
            for i in range(IPE):
                frac = (e * IPE + i + 1) / (w * IPE)
                assert common.learning_rate_at(a, e, i, IPE) == pytest.approx(0.1 + (TARGET - 0.1) * frac)
        assert common.learning_rate_at(a, w, 0, IPE) == TARGET
        assert common.learning_rate_at(a, 30, 0, IPE) == common.learning_rate_at(base, 30, 0, IPE)
    zero = types.SimpleNamespace(**dict(vars(base), warmup_epochs=0))
    assert common.learning_rate_at(zero, 0, 0, IPE) == TARGET


# --------------------------------------------------------------------------- #
# flag checks
# --------------------------------------------------------------------------- #
def _parse(tmp_path, extra, adpsgd=False):
    args = common.build_parser(adpsgd=adpsgd).parse_args(
        ['--device', 'cpu', '--backend', 'gloo', '--checkpoint_dir', str(tmp_path) + '/'] + extra)
    return common.finalize_args(args, adpsgd=adpsgd)


def test_new_flag_defaults():
    d = common.build_parser().parse_args([])
    assert (d.lr_policy, d.poly_power, d.end_lr, d.warmup_epochs, d.label_smoothing) == \
        ('step', 2.0, 0.0001, 5, 0.0)
    ad = common.build_parser(adpsgd=True).parse_args(['--lr_policy', 'poly', '--label_smoothing', '0.1'])
    assert ad.lr_policy == 'poly' and ad.label_smoothing == 0.1
    with pytest.raises(SystemExit):
        common.build_parser().parse_args(['--lr_policy', 'cosine'])


@pytest.mark.parametrize('adpsgd', [False, True])
@pytest.mark.parametrize('extra,what', [
    (['--lr_policy', 'poly', '--schedule', '30', '0.1'], '--schedule'),
    (['--lr_policy', 'poly', '--poly_power', '0'], '--poly_power'),
    (['--lr_policy', 'poly', '--poly_power', '-1'], '--poly_power'),
    (['--lr_policy', 'poly', '--end_lr', '-0.001'], '--end_lr'),
    (['--warmup_epochs', '-1'], '--warmup_epochs'),
    (['--lr_policy', 'poly', '--warmup', 'True', '--warmup_epochs', '5', '--num_epochs', '5'], 'warm-up'),
    (['--label_smoothing', '-0.1'], '--label_smoothing'),
    (['--label_smoothing', '1.01'], '--label_smoothing'),
    (['--label_smoothing', 'nan'], '--label_smoothing'),
])
def test_finalize_args_rejects(tmp_path, adpsgd, extra, what):
    with pytest.raises(ValueError, match=what):
        _parse(tmp_path, extra, adpsgd)


def test_finalize_args_accepts_the_recipe(tmp_path):
    a = _parse(tmp_path, ['--lr_policy', 'poly', '--warmup', 'True', '--warmup_epochs', '2',
                          '--num_epochs', '3', '--label_smoothing', '0.1'])
    assert a.lr_policy == 'poly' and a.label_smoothing == 0.1
    # without --warmup the warm-up length does not constrain num_epochs
    _parse(tmp_path, ['--lr_policy', 'poly', '--warmup_epochs', '5', '--num_epochs', '2'])
    _parse(tmp_path, ['--label_smoothing', '1.0', '--warmup_epochs', '0'])


def test_gossip_sgd_cli_label_smoothing_poly_two_ranks_cpu(tmp_path, master_port):
    from test_cli_and_experiment import COMMON, _torchrun
    out = _torchrun(2, 'gossip_sgd.py', COMMON + [
        '--push_sum', 'True', '--graph_type', '5', '--label_smoothing', '0.1', '--lr_policy', 'poly',
        '--warmup', 'True', '--warmup_epochs', '1', '--num_epochs', '2',
        '--checkpoint_dir', str(tmp_path) + '/', '--num_itr_ignore', '0'], master_port)
    assert out.returncode == 0, out.stdout[-3000:]
    for r in range(2):
        lines = open(str(tmp_path / ('out_r%d_n2.csv' % r))).read().splitlines()
        rows = [l.split(',') for l in lines[5:]]
        assert rows and all(len(row) == 18 for row in rows)
        train = [row for row in rows if row[1] != '-1']
        assert train and all(float(row[11]) == float(row[11]) for row in train)
