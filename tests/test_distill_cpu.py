"""Knowledge distillation without a GPU: the torch reference of the distillation loss against a
hand-written fp64 formula and its autograd gradient, the argument checks of the op, the trainer and the
command line, teacher checkpoint loading, and a 2-rank gloo command-line run."""
import argparse
import logging
import math
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from stochastic_gradient_push_b200 import models
from stochastic_gradient_push_b200.cli import common
from stochastic_gradient_push_b200.ops.fused_loss import (FusedCrossEntropyWithAccuracy, check_distill_args,
                                                          fused_cross_entropy, reference_distillation_loss)
from stochastic_gradient_push_b200.parallel.trainer import (GossipTrainer, check_distill_teacher,
                                                            teacher_compute_twin)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _formula(z, u, t, alpha, temp, eps=0.0, lam=None):
    """the objective row by row in fp64 numpy, straight from its definition"""
    z, u, t = z.double().numpy(), u.double().numpy(), t.numpy()
    B, C = z.shape
    total = 0.0
    for i in range(B):
        ts = [(t[i], 1.0)] if lam is None else [(t[i], lam), (t[B - 1 - i], 1.0 - lam)]
        if any(not 0 <= tt < C for tt, _ in ts):
            continue
        logq = z[i] - np.log(np.sum(np.exp(z[i])))
        ce = 0.0
        for tt, w in ts:
            y = np.full(C, eps / C)
            y[tt] += 1.0 - eps
            ce += w * -np.sum(y * logq)
        p = np.exp(u[i] / temp) / np.sum(np.exp(u[i] / temp))
        qt = np.exp(z[i] / temp) / np.sum(np.exp(z[i] / temp))
        kl = np.sum(p * (np.log(p) - np.log(qt)))
        total += (1.0 - alpha) * ce + alpha * temp * temp * kl
    return total / B


CASES = [(alpha, temp, eps, lam) for alpha in (0.25, 0.5, 1.0) for temp in (1.0, 2.0, 4.0)
         for eps, lam in ((0.0, None), (0.1, None), (0.0, 0.3), (0.1, 0.7))]


@pytest.mark.parametrize('alpha,temp,eps,lam', CASES)
def test_reference_matches_the_fp64_formula(alpha, temp, eps, lam):
    g = torch.Generator().manual_seed(1)
    z = torch.randn(7, 13, generator=g, dtype=torch.float64) * 3
    u = torch.randn(7, 13, generator=g, dtype=torch.float64) * 3
    t = torch.randint(0, 13, (7,), generator=g)
    t[2] = -1                                        # an invalid row (and, mixed, its partner row 4)
    loss, p1, p5 = reference_distillation_loss(z, t, u, alpha, temp, eps, lam=lam)
    assert loss.dtype == torch.float64
    assert loss.item() == pytest.approx(_formula(z, u, t, alpha, temp, eps, lam), rel=1e-12, abs=1e-12)
    assert 0.0 <= p1.item() <= p5.item() <= 100.0


def test_reference_is_the_torch_composition():
    """every target valid: (1 - a) F.cross_entropy + a T^2 F.kl_div(batchmean, log_target)"""
    g = torch.Generator().manual_seed(2)
    z, u = torch.randn(16, 10, generator=g), torch.randn(16, 10, generator=g)
    t = torch.randint(0, 10, (16,), generator=g)
    a, T, eps = 0.4, 3.0, 0.1
    want = (1 - a) * F.cross_entropy(z, t, label_smoothing=eps) + a * T * T * F.kl_div(
        F.log_softmax(z / T, 1), F.log_softmax(u / T, 1), reduction='batchmean', log_target=True)
    got = reference_distillation_loss(z, t, u, a, T, eps)[0]
    torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-6)
    # accuracies are the student's, as reference_loss_and_accuracy counts them
    from stochastic_gradient_push_b200.ops.fused_loss import reference_loss_and_accuracy
    _, p1, p5 = reference_distillation_loss(z, t, u, a, T)
    _, q1, q5 = reference_loss_and_accuracy(z, t)
    assert (p1.item(), p5.item()) == (q1.item(), q5.item())


@pytest.mark.parametrize('eps,lam', [(0.0, None), (0.1, None), (0.1, 0.25)])
@pytest.mark.parametrize('temp', [1.0, 2.5])
def test_reference_gradcheck(eps, lam, temp):
    g = torch.Generator().manual_seed(3)
    z = torch.randn(5, 6, generator=g, dtype=torch.float64, requires_grad=True)
    u = torch.randn(5, 6, generator=g, dtype=torch.float64)
    t = torch.tensor([0, 5, 2, 7, 3])                # row 3 is out of range
    assert torch.autograd.gradcheck(
        lambda zz: reference_distillation_loss(zz, t, u, 0.6, temp, eps, lam=lam)[0], (z,))
    # the invalid row (and, mixed, its partner) gets a zero gradient; the teacher gets none
    (dz,) = torch.autograd.grad(reference_distillation_loss(z, t, u.requires_grad_(), 0.6, temp, eps, lam=lam)[0],
                                (z,))
    assert torch.all(dz[3] == 0)
    if lam is not None:
        assert torch.all(dz[1] == 0)


def test_cpu_fallback_of_the_op_and_criterion():
    g = torch.Generator().manual_seed(4)
    z, u = torch.randn(8, 10, generator=g), torch.randn(8, 10, generator=g)
    t = torch.randint(0, 10, (8,), generator=g)
    loss, metrics = fused_cross_entropy(z, t, 0.1, teacher_logits=u, distill_alpha=0.5, distill_temperature=2.0)
    want = reference_distillation_loss(z, t, u, 0.5, 2.0, 0.1)
    assert loss.item() == want[0].item() and metrics.tolist() == [x.item() for x in want]
    crit = FusedCrossEntropyWithAccuracy(label_smoothing=0.1, distill_alpha=0.5, distill_temperature=2.0)
    assert crit(z, t, teacher_logits=u).item() == want[0].item()
    assert 'distill_alpha=0.5' in repr(crit)
    mix = torch.tensor([0.3, 1, 0, 0, 0, 0, 0, 0])
    loss, _ = fused_cross_entropy(z, t, teacher_logits=u, distill_alpha=0.5, mix=mix)
    assert loss.item() == reference_distillation_loss(z, t, u, 0.5, 1.0, lam=mix[0])[0].item()
    # alpha = 0 without a teacher is the plain loss
    assert FusedCrossEntropyWithAccuracy()(z, t).item() == F.cross_entropy(z, t).item()


def test_op_argument_rejections():
    z, u, t = torch.randn(4, 5), torch.randn(4, 5), torch.tensor([0, 1, 2, 3])
    for a in (-0.1, 1.1, float('nan')):
        with pytest.raises(ValueError, match='distill_alpha'):
            fused_cross_entropy(z, t, teacher_logits=u, distill_alpha=a)
        with pytest.raises(ValueError, match='distill_alpha'):
            FusedCrossEntropyWithAccuracy(distill_alpha=a)
    for T in (0.0, -1.0, float('inf'), float('nan')):
        with pytest.raises(ValueError, match='distill_temperature'):
            fused_cross_entropy(z, t, teacher_logits=u, distill_alpha=0.5, distill_temperature=T)
        with pytest.raises(ValueError, match='distill_temperature'):
            check_distill_args(0.5, T)
    with pytest.raises(ValueError, match='needs teacher_logits'):
        fused_cross_entropy(z, t, distill_alpha=0.5)
    with pytest.raises(ValueError, match='needs teacher_logits'):
        FusedCrossEntropyWithAccuracy(distill_alpha=0.5)(z, t)
    with pytest.raises(ValueError, match='distill_alpha = 0'):
        fused_cross_entropy(z, t, teacher_logits=u)
    with pytest.raises(ValueError, match='shape and dtype'):
        fused_cross_entropy(z, t, teacher_logits=torch.randn(4, 6), distill_alpha=0.5)
    with pytest.raises(ValueError, match='shape and dtype'):
        fused_cross_entropy(z, t, teacher_logits=u.double(), distill_alpha=0.5)
    with pytest.raises(ValueError, match='shape and dtype'):
        reference_distillation_loss(z, t, u[:3], 0.5)


class _Crit(nn.Module):
    def forward(self, out, tgt):
        return out.sum()


def test_trainer_teacher_rejections():
    teacher = nn.Linear(4, 3)
    kd = FusedCrossEntropyWithAccuracy(distill_alpha=0.5)
    check_distill_teacher(None, FusedCrossEntropyWithAccuracy(), 'cpu')
    check_distill_teacher(None, _Crit(), 'cpu')
    check_distill_teacher(teacher, kd, 'cpu')
    with pytest.raises(ValueError, match='no teacher'):
        check_distill_teacher(None, kd, 'cpu')
    with pytest.raises(ValueError, match='distill_alpha > 0'):
        check_distill_teacher(teacher, FusedCrossEntropyWithAccuracy(), 'cpu')
    with pytest.raises(ValueError, match='distill_alpha > 0'):
        check_distill_teacher(teacher, _Crit(), 'cpu')
    with pytest.raises(ValueError, match='nn.Module'):
        check_distill_teacher(lambda x: x, kd, 'cpu')
    with pytest.raises(ValueError, match='device'):
        check_distill_teacher(teacher, kd, torch.device('cuda', 0))
    # the constructor's step (a bare trainer: no GPU here)
    t = GossipTrainer.__new__(GossipTrainer)
    t.criterion, t.device, t.model = kd, torch.device('cpu'), types.SimpleNamespace(_twin=[])
    teacher.train()
    t._attach_teacher(teacher)
    assert t.teacher is teacher and t._teacher_net is teacher
    assert not teacher.training and not any(p.requires_grad for p in teacher.parameters())
    t.criterion = FusedCrossEntropyWithAccuracy()
    with pytest.raises(ValueError):
        t._attach_teacher(teacher)


def test_adpsgd_trainer_rejects_a_teacher():
    from stochastic_gradient_push_b200.parallel.ad_psgd import make_bilat_trainer
    with pytest.raises(ValueError, match='AD-PSGD'):
        make_bilat_trainer(None, 0.1, teacher=nn.Linear(2, 2))
    with pytest.raises(ValueError, match='AD-PSGD'):
        make_bilat_trainer(None, 0.1, criterion=FusedCrossEntropyWithAccuracy(distill_alpha=0.5))


def test_teacher_compute_twin_dtypes():
    net = models.TinyConvNet()
    twin = teacher_compute_twin(net)
    for (name, p), (_, q) in zip(net.named_parameters(), twin.named_parameters()):
        norm = name.startswith('features.1') or name.startswith('features.4')
        assert q.dtype == (torch.float32 if norm else torch.bfloat16), name
        assert torch.equal(q.float(), p.to(q.dtype).float())
    assert all(b.dtype == a.dtype for a, b in zip(net.buffers(), twin.buffers()))
    assert not twin.training and not any(p.requires_grad for p in twin.parameters())
    assert all(p.dtype == torch.float32 for p in net.parameters())        # the teacher itself is untouched


def _args(**kw):
    base = dict(distill_alpha=0.0, distill_temperature=1.0, teacher_model=None, teacher_checkpoint=None,
                model='resnet50', num_classes=1000)
    base.update(kw)
    return argparse.Namespace(**base)


def test_check_distill_flags():
    ok = dict(distill_alpha=0.5, teacher_model='resnet18', teacher_checkpoint='t.pth')
    common.check_distill_flags(_args())
    common.check_distill_flags(_args(**ok))
    common.check_distill_flags(_args(**dict(ok, distill_alpha=1.0, distill_temperature=4.0)))
    common.check_distill_flags(_args(**dict(ok, teacher_model='tiny'), model='tiny'))
    common.check_distill_flags(_args(**dict(ok, teacher_model='tiny'), num_classes=10))
    for a in (-0.5, 1.5):
        with pytest.raises(ValueError, match='--distill_alpha must be'):
            common.check_distill_flags(_args(**dict(ok, distill_alpha=a)))
    for T in (0.0, -2.0, float('inf')):
        with pytest.raises(ValueError, match='--distill_temperature'):
            common.check_distill_flags(_args(**dict(ok, distill_temperature=T)))
    with pytest.raises(ValueError, match='--teacher_model and --teacher_checkpoint'):
        common.check_distill_flags(_args(distill_alpha=0.5, teacher_model='resnet18'))
    with pytest.raises(ValueError, match='--teacher_model and --teacher_checkpoint'):
        common.check_distill_flags(_args(distill_alpha=0.5, teacher_checkpoint='t.pth'))
    with pytest.raises(ValueError, match='one of'):
        common.check_distill_flags(_args(**dict(ok, teacher_model='vgg')))
    with pytest.raises(ValueError, match='classes'):
        common.check_distill_flags(_args(**dict(ok, teacher_model='tiny')))
    with pytest.raises(ValueError, match='classes'):
        common.check_distill_flags(_args(**ok, model='tiny'))
    with pytest.raises(ValueError, match='AD-PSGD'):
        common.check_distill_flags(_args(**ok), adpsgd=True)
    common.check_distill_flags(_args(), adpsgd=True)
    p = common.build_parser()
    a = p.parse_args([])
    assert (a.distill_alpha, a.distill_temperature, a.teacher_model, a.teacher_checkpoint) == (0.0, 1.0, None, None)
    a = p.parse_args(['--distill_alpha', '0.5', '--distill_temperature', '2', '--teacher_model', 'resnet50',
                      '--teacher_checkpoint', 'x.pth'])
    assert (a.distill_alpha, a.distill_temperature, a.teacher_model, a.teacher_checkpoint) == \
        (0.5, 2.0, 'resnet50', 'x.pth')


def _load_args(path):
    return argparse.Namespace(distill_alpha=0.5, teacher_model='tiny', teacher_checkpoint=str(path),
                              num_classes=10, device='cpu', channels_last=False)


def _same(a, b):
    sa, sb = a.state_dict(), b.state_dict()
    return sa.keys() == sb.keys() and all(torch.equal(sa[k], sb[k]) for k in sa)


def test_teacher_loading_from_a_bare_state_dict(tmp_path):
    torch.manual_seed(5)
    net = models.TinyConvNet()
    torch.save(net.state_dict(), tmp_path / 'teacher.pth')
    t = common.load_teacher(_load_args(tmp_path / 'teacher.pth'))
    assert _same(t, net) and not t.training and not any(p.requires_grad for p in t.parameters())
    assert common.load_teacher(argparse.Namespace(distill_alpha=0.0)) is None
    # strict: a file of another architecture does not load
    torch.save(models.TinyConvNet(width=8).state_dict(), tmp_path / 'other.pth')
    with pytest.raises(RuntimeError):
        common.load_teacher(_load_args(tmp_path / 'other.pth'))


def test_teacher_loading_from_a_cli_checkpoint(tmp_path):
    """the layout gossip_sgd.py writes: state['state_dict'] = GossipDataParallel.state_dict() =
    {'state_dict': {'module.<key>': ..., <wrapper entries>}, 'ps_weight': ..., 'is_ps_numerator': ...}"""
    torch.manual_seed(6)
    net = models.TinyConvNet()
    inner = {'module.' + k: v for k, v in net.state_dict().items()}
    inner['gossip_ps_factor'] = torch.ones(1)                      # a wrapper's own entry
    state = common.fresh_state({'state_dict': inner, 'ps_weight': torch.ones(1), 'is_ps_numerator': False}, {})
    torch.save(state, tmp_path / 'checkpoint.pth.tar')
    t = common.load_teacher(_load_args(tmp_path / 'checkpoint.pth.tar'))
    assert _same(t, net)
    # an all-reduce checkpoint: the module's state_dict with the DDP prefix, no inner level
    torch.save(common.fresh_state({'module.' + k: v for k, v in net.state_dict().items()}, {}),
               tmp_path / 'ar.pth.tar')
    assert _same(common.load_teacher(_load_args(tmp_path / 'ar.pth.tar')), net)


def _torchrun(nproc, args, port, timeout=600):
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(nproc),
           '--master-addr', '127.0.0.1', '--master-port', str(port), os.path.join(ROOT, 'gossip_sgd.py')] + args
    env = dict(os.environ, OMP_NUM_THREADS='1')
    return subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout,
                          env=env)


COMMON = ['--device', 'cpu', '--backend', 'gloo', '--model', 'tiny', '--num_classes', '10',
          '--image_size', '16', '--synthetic', 'True', '--synthetic_len', '64', '--batch_size', '4',
          '--verbose', 'False', '--print_freq', '2', '--amp', 'False',
          '--num_dataloader_workers', '0', '--lr', '0.05']


@pytest.mark.parametrize('extra', [['--push_sum', 'True', '--graph_type', '5'],
                                   ['--all_reduce', 'True', '--graph_type', '-1']])
def test_cli_two_ranks_distill_cpu(tmp_path, master_port, extra):
    torch.manual_seed(7)
    torch.save(models.TinyConvNet().state_dict(), tmp_path / 'teacher.pth')
    out = _torchrun(2, COMMON + extra + [
        '--num_epochs', '1', '--checkpoint_dir', str(tmp_path) + '/', '--num_itr_ignore', '0',
        '--distill_alpha', '0.5', '--distill_temperature', '2', '--teacher_model', 'tiny',
        '--teacher_checkpoint', str(tmp_path / 'teacher.pth')], master_port)
    assert out.returncode == 0, out.stdout[-3000:]
    assert out.stdout.count(' * Teacher Prec@1') == 2, out.stdout[-3000:]        # once per rank
    for r in range(2):
        rows = [l.split(',') for l in open(str(tmp_path / ('out_r%d_n2.csv' % r))).read().splitlines()[5:]]
        assert rows and all(math.isfinite(float(row[11])) for row in rows if row[1] != '-1')
        ck = torch.load(str(tmp_path / ('checkpoint_r%d_n2.pth.tar' % r)), map_location='cpu', weights_only=False)
        assert not any('teacher' in k for k in ck)


def test_adpsgd_cli_rejects_distillation(tmp_path):
    from stochastic_gradient_push_b200.cli import gossip_sgd_adpsgd
    with pytest.raises(ValueError, match='AD-PSGD'):
        gossip_sgd_adpsgd.parse_args(COMMON + ['--checkpoint_dir', str(tmp_path) + '/', '--distill_alpha', '0.5',
                                               '--teacher_model', 'tiny', '--teacher_checkpoint', 'x.pth'])
