"""Knowledge distillation on the GPU: the DISTILL instantiations of the fused cross-entropy kernels
(csrc/loss_kernels.cu) against ``reference_distillation_loss``, their edge rows, the unchanged kernels
without a teacher, graph capture, and ``GossipTrainer(teacher=...)`` on two loop-back ranks."""
import copy
import functools
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200 import models
from stochastic_gradient_push_b200.ops import batch_mix as bm
from stochastic_gradient_push_b200.ops import native
from stochastic_gradient_push_b200.ops.fused_loss import (FusedCrossEntropyWithAccuracy, fused_cross_entropy,
                                                          reference_distillation_loss)

from test_gdp_loopback_gpu import _in_threads

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
BF16 = torch.bfloat16
SHAPES = [(256, 1000), (32, 1000), (7, 10), (1, 5), (64, 33), (16, 4099)]


def _mix_state(lam):
    return torch.tensor([lam, 1, 0, 0, 0, 0, 0, 0], dtype=torch.float32, device=DEV)


def _inputs(B, C, dtype, seed=0, scale=3.0):
    g = torch.Generator(device='cuda').manual_seed(B * 31 + C + seed)
    z = (torch.randn(B, C, device='cuda', generator=g) * scale).to(dtype)
    u = (torch.randn(B, C, device='cuda', generator=g) * scale).to(dtype)
    t = torch.randint(0, C, (B,), device='cuda', generator=g)
    return z, u, t


def _ranked_accuracy(z, t):
    """prec@1 / prec@5 as the kernels count them: rank = #{j : z_j > z_t}, so a logit tied with the target's
    counts as ranked below it (bf16 logits tie); rows with an out-of-range target count as misses"""
    B, C = z.shape
    valid = (t >= 0) & (t < C)
    zt = z.float().gather(1, torch.where(valid, t, 0).view(-1, 1))
    rank = (z.float() > zt).sum(1)
    return ((rank < 1) & valid).sum().float() * (100.0 / B), ((rank < 5) & valid).sum().float() * (100.0 / B)


def _check(z, u, t, alpha, temp, eps, lam, grad_scale=1.7):
    """fused loss, metrics and gradient against the torch oracle on the same (rounded) values"""
    dtype = z.dtype
    zz = z.clone().requires_grad_(True)
    mix = None if lam is None else _mix_state(lam)
    crit = FusedCrossEntropyWithAccuracy(label_smoothing=eps, distill_alpha=alpha, distill_temperature=temp)
    loss = crit(zz, t, mix=mix, teacher_logits=u)
    (loss * grad_scale).backward()
    torch.cuda.synchronize()
    ref = z.detach().float().requires_grad_(True)
    want, p1, p5 = reference_distillation_loss(ref, t, u.float(), alpha, temp, eps, lam=lam)
    (want * grad_scale).backward()
    B = z.shape[0]
    tl = 1e-5 * max(1.0, temp * temp)
    torch.testing.assert_close(loss.detach(), want.detach(), rtol=1e-5, atol=tl)
    torch.testing.assert_close(crit.metrics[0], want.detach(), rtol=1e-5, atol=tl)
    p1, p5 = _ranked_accuracy(z, t)
    torch.testing.assert_close(crit.metrics[1], p1, rtol=0, atol=1e-3)
    torch.testing.assert_close(crit.metrics[2], p5, rtol=0, atol=1e-3)
    tol = (1e-6 if dtype == torch.float32 else 4e-3 / B) * temp
    torch.testing.assert_close(zz.grad.float(), ref.grad, rtol=1e-4 if dtype == torch.float32 else 1e-2, atol=tol)
    return zz.grad


@pytest.mark.parametrize('eps,lam', [(0.0, None), (0.1, None), (0.0, 0.3), (0.1, 0.8), (0.0, 1.0)])
@pytest.mark.parametrize('temp', [1.0, 2.0, 4.0])
@pytest.mark.parametrize('alpha', [0.25, 0.5, 1.0])
@pytest.mark.parametrize('B,C', SHAPES)
@pytest.mark.parametrize('dtype', [torch.float32, BF16], ids=['fp32', 'bf16'])
def test_kernel_matches_the_oracle(dtype, B, C, alpha, temp, eps, lam):
    z, u, t = _inputs(B, C, dtype)
    assert native.load().xent_can_fuse(z, t)
    _check(z, u, t, alpha, temp, eps, lam)


@pytest.mark.parametrize('lam', [None, 0.4])
@pytest.mark.parametrize('dtype', [torch.float32, BF16], ids=['fp32', 'bf16'])
def test_out_of_range_targets_add_nothing(dtype, lam):
    B, C = 32, 1000
    z, u, t = _inputs(B, C, dtype, seed=5)
    t[3], t[10], t[20] = -1, C, -100
    grad = _check(z, u, t, 0.5, 2.0, 0.1, lam)
    bad = [3, 10, 20] + ([] if lam is None else [B - 1 - 3, B - 1 - 10, B - 1 - 20])
    assert torch.all(grad[bad] == 0)
    good = [i for i in range(B) if i not in bad]
    assert torch.all(grad[good].abs().sum(1) > 0)


@pytest.mark.parametrize('temp', [1.0, 4.0])
@pytest.mark.parametrize('dtype', [torch.float32, BF16], ids=['fp32', 'bf16'])
def test_large_logits_stay_finite(dtype, temp):
    B, C = 64, 1000
    z, u, t = _inputs(B, C, torch.float32, seed=9)
    z = (torch.sign(z) * 1e4 + z).to(dtype)
    u = (torch.sign(u) * 1e4 - u).to(dtype)
    zz = z.clone().requires_grad_(True)
    crit = FusedCrossEntropyWithAccuracy(distill_alpha=0.5, distill_temperature=temp)
    loss = crit(zz, t, teacher_logits=u)
    loss.backward()
    ref = z.float().requires_grad_(True)
    want = reference_distillation_loss(ref, t, u.float(), 0.5, temp)[0]
    want.backward()
    assert torch.isfinite(loss) and torch.isfinite(zz.grad).all()
    torch.testing.assert_close(loss.detach(), want.detach(), rtol=1e-4, atol=1e-2)
    torch.testing.assert_close(zz.grad.float(), ref.grad, rtol=1e-2, atol=1e-5 * temp)


@pytest.mark.parametrize('eps,lam', [(0.0, None), (0.1, None), (0.1, 0.3)])
@pytest.mark.parametrize('dtype', [torch.float32, BF16], ids=['fp32', 'bf16'])
def test_teacher_equal_to_student_is_scaled_cross_entropy(dtype, eps, lam):
    B, C = 64, 1000
    z, _, t = _inputs(B, C, dtype, seed=3)
    mix = None if lam is None else _mix_state(lam)
    for temp in (1.0, 3.0):
        alpha = 0.3
        zz = z.clone().requires_grad_(True)
        loss, metrics = fused_cross_entropy(zz, t, eps, mix=mix, teacher_logits=z, distill_alpha=alpha,
                                            distill_temperature=temp)
        loss.backward()
        z0 = z.clone().requires_grad_(True)
        ce, m0 = fused_cross_entropy(z0, t, eps, mix=mix)
        ce.backward()
        torch.testing.assert_close(loss, (1 - alpha) * ce.detach(), rtol=1e-6, atol=2e-6)
        assert torch.equal(metrics[1:], m0[1:])
        tol = 1e-7 if dtype == torch.float32 else 4e-3 / B
        torch.testing.assert_close(zz.grad.float(), (1 - alpha) * z0.grad.float(), rtol=1e-2, atol=tol)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'xent_parent_kernels.pt')


def test_no_teacher_matches_the_parent_kernels_bit_for_bit():
    """``tests/golden/xent_parent_kernels.pt`` holds logits ([16, 257], fp32 and bf16, two rows with an
    out-of-range target), targets, the per-row lse, metrics and gradient (grad_out 1.3) that the commit before
    knowledge distillation computed with ``xent_forward`` / ``xent_backward`` on an H100, for label smoothing 0
    and 0.1, each without mixing and with a mix state at lam 0.6.  Without a teacher the kernels must give the
    same per-row lse and gradient, bit for bit, through the binding and through the op at alpha = 0."""
    C = native.load()
    gold = torch.load(GOLDEN, weights_only=True)
    t = gold['target'].to(DEV)
    g = gold['grad_out'].to(DEV)
    assert len(gold['cases']) == 8
    for case in gold['cases']:
        z = gold['logits_' + case['dtype']].to(DEV)
        eps, lam = case['eps'], case['lam']
        mix = None if lam is None else _mix_state(lam)
        metrics, lse = C.xent_forward(z, t, eps, mix)
        assert torch.equal(lse.cpu(), case['lse']), case
        assert torch.equal(C.xent_backward(z, t, lse, g, eps, mix).cpu(), case['grad']), case
        torch.testing.assert_close(metrics.cpu(), case['metrics'], rtol=1e-6, atol=1e-6)
        zz = z.clone().requires_grad_(True)
        loss, _ = fused_cross_entropy(zz, t, eps, mix=mix, distill_alpha=0.0)
        (loss * float(g)).backward()
        assert torch.equal(zz.grad.cpu(), case['grad']), case
        # with a teacher, the first of the three lse rows is the same per-row lse
        _, lse3 = C.xent_forward(z, t, eps, mix, torch.randn_like(z), 0.5, 2.0)
        assert lse3.shape == (3, z.shape[0]) and torch.equal(lse3[0].cpu(), case['lse'])


def test_binding_rejects_bad_teacher_arguments():
    C = native.load()
    z, u, t = _inputs(8, 10, torch.float32)
    for bad in (u[:4], u.to(BF16), u.t().contiguous().t(), u.cpu()):
        with pytest.raises(RuntimeError, match='teacher_logits'):
            C.xent_forward(z, t, 0.0, None, bad, 0.5, 1.0)
    for a, T in ((0.0, 1.0), (1.5, 1.0), (0.5, 0.0), (0.5, float('inf'))):
        with pytest.raises(RuntimeError, match='distill'):
            C.xent_forward(z, t, 0.0, None, u, a, T)
    m, lse = C.xent_forward(z, t, 0.0, None, u, 0.5, 1.0)
    with pytest.raises(RuntimeError, match='lse'):
        C.xent_backward(z, t, lse[0].contiguous(), torch.ones(1, device=DEV), 0.0, None, u, 0.5, 1.0)
    with pytest.raises(ValueError, match='device'):
        fused_cross_entropy(z, t, teacher_logits=u.cpu(), distill_alpha=0.5)


def test_captured_loss_follows_new_teacher_logits():
    C = native.load()
    B, Cn = 64, 1000
    z, u, t = _inputs(B, Cn, torch.float32, seed=21)
    g = torch.ones(1, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            C.xent_forward(z, t, 0.1, None, u, 0.5, 2.0)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            metrics, lse = C.xent_forward(z, t, 0.1, None, u, 0.5, 2.0)
            dz = C.xent_backward(z, t, lse, g, 0.1, None, u, 0.5, 2.0)
    torch.cuda.current_stream().wait_stream(s)
    for seed in (22, 23):
        u.copy_(_inputs(B, Cn, torch.float32, seed=seed)[1])
        graph.replay()
        torch.cuda.synchronize()
        ref = z.clone().requires_grad_(True)
        want = reference_distillation_loss(ref, t, u, 0.5, 2.0, 0.1)[0]
        want.backward()
        torch.testing.assert_close(metrics[0], want.detach(), rtol=1e-5, atol=4e-5)
        torch.testing.assert_close(dz, ref.grad, rtol=1e-4, atol=2e-6)


# ---------------------------------------------------------------------------------------------------- #
# the trainer
# ---------------------------------------------------------------------------------------------------- #
class _Mlp(nn.Module):
    """Linear -> BatchNorm1d -> ReLU -> Linear: torch's own kernels, reproducible run to run"""

    def __init__(self):
        super().__init__()
        self.fc1 = nn.Linear(48, 32)
        self.bn = nn.BatchNorm1d(32)
        self.fc2 = nn.Linear(32, 10)

    def forward(self, x):
        return self.fc2(torch.relu(self.bn(self.fc1(x))))


def _teacher(net_fn, seed=23):
    torch.manual_seed(seed)
    net = net_fn().to(DEV).to(memory_format=torch.channels_last)
    with torch.no_grad():                               # non-trivial running statistics
        for m in net.modules():
            if isinstance(m, nn.modules.batchnorm._BatchNorm):
                m.running_mean.uniform_(-0.2, 0.2)
                m.running_var.uniform_(0.5, 1.5)
    return net


def _trainer(net_fn, teacher=None, alpha=0.5, temp=2.0, k=1, use_graph=False, twin=False, world=None, rank=0,
             seed=11, name='', batch_mix=None, ema_decay=None):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    torch.manual_seed(seed)
    net = net_fn().to(DEV).to(memory_format=torch.channels_last)
    n = 1 if world is None else 2
    kw = dict(symmetric_world=world.view(rank), transport='nvlink', grid=4, symmetric_name=name) if world else {}
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(rank, n), rank=rank,
                               world_size=n, heartbeat_timeout=20, compute_dtype=BF16 if twin else None, **kw)
    opt = FusedGossipSGD(model, lr=0.0, momentum=0.0, weight_decay=0.0)
    ema = None
    if ema_decay is not None:
        from stochastic_gradient_push_b200.ops.model_ema import ModelEma
        ema = ModelEma(model, decay=ema_decay)
    crit = FusedCrossEntropyWithAccuracy(label_smoothing=0.1, distill_alpha=alpha if teacher is not None else 0.0,
                                         distill_temperature=temp)
    return GossipTrainer(model, opt, crit, amp_dtype=None, use_cuda_graph=use_graph,
                         warmup_iters=1 if world is None else 10 ** 6, accumulation_steps=k,
                         batch_mix=batch_mix, ema=ema, teacher=teacher)


def _data(rows, seed, shape=(48,), classes=10):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((rows,) + shape, generator=g).pin_memory(),
            torch.randint(0, classes, (rows,), generator=g).pin_memory())


def _state(module):
    return [t.detach().clone() for t in list(module.parameters()) + list(module.buffers())]


def test_trainer_rejects_mismatched_teacher_and_criterion():
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    with pytest.raises(ValueError, match='no teacher'):
        tr = _trainer(_Mlp)
        GossipTrainer(tr.model, tr.opt, FusedCrossEntropyWithAccuracy(distill_alpha=0.5))
    with pytest.raises(ValueError, match='distill_alpha > 0'):
        GossipTrainer(tr.model, tr.opt, FusedCrossEntropyWithAccuracy(), teacher=_teacher(_Mlp))
    with pytest.raises(ValueError, match='device'):
        GossipTrainer(tr.model, tr.opt, FusedCrossEntropyWithAccuracy(distill_alpha=0.5), teacher=_Mlp())


@pytest.mark.parametrize('twin', [False, True], ids=['fp32', 'bf16-twin'])
def test_loopback_graphed_steps_equal_eager_steps_bit_for_bit(twin):
    """two ranks (identical start, lr = 0): g^ of each graphed step equals the eager run's, bit for bit;
    the teacher is untouched and the arena does not grow"""
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    steps = 4
    batches = [[_data(16, 100 * r + s) for s in range(steps)] for r in range(2)]
    teachers = [_teacher(_Mlp) for _ in range(2)]
    before = [_state(t) for t in teachers]
    runs = []
    for use_graph in (False, True):
        lw = LocalWorld(2)
        trs = [_trainer(_Mlp, teachers[r], use_graph=use_graph, twin=twin, world=lw, rank=r,
                        name='kd_%d_%d' % (use_graph, twin)) for r in range(2)]
        plain = _trainer(_Mlp, twin=twin)
        assert trs[0].model.arena.flat.numel() == plain.model.arena.flat.numel()
        got = []
        for s in range(steps):
            if use_graph and s == 1:
                for tr in trs:
                    with torch.cuda.stream(tr.stream):
                        tr._capture()
            _in_threads([functools.partial(trs[r].step, *batches[r][s]) for r in range(2)])
            torch.cuda.synchronize()
            got.append([tr.opt.momentum_flat[torch.float32].clone() for tr in trs])
        for tr in trs:
            tr.finish()
            assert (tr.graph is not None) == use_graph
        runs.append(got)
    for s in range(steps):
        for r in range(2):
            assert torch.equal(runs[0][s][r], runs[1][s][r]), (s, r)
            assert runs[0][s][r].abs().max() > 0
    for t, b in zip(teachers, before):
        assert all(torch.equal(x, y) for x, y in zip(_state(t), b))
        assert not t.training


def _reference_grad(net, teacher, x, y, alpha, temp, eps=0.1, lam=None, autocast=False):
    """the torch step: the student forward in train mode plus reference_distillation_loss (two targets with
    ``lam``), both networks under bf16 autocast with ``autocast``; the flat gradient"""
    net = copy.deepcopy(net).train()
    for p in net.parameters():
        p.requires_grad_(True)
        p.grad = None
    with torch.autocast('cuda', dtype=BF16, enabled=autocast):
        with torch.no_grad():
            u = teacher(x)
        out = net(x)
    loss = reference_distillation_loss(out.float(), y, u.float(), alpha, temp, eps, lam=lam)[0]
    loss.backward()
    return torch.cat([p.grad.reshape(-1) for p in net.parameters()])


def _rel_err(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


def _resnet():
    return models.resnet18(num_classes=10)


@pytest.mark.parametrize('variant', ['plain', 'accum2', 'batch_mix', 'ema', 'bf16-twin'])
def test_resnet_step_matches_torch_and_counts_the_teacher(variant):
    twin = variant == 'bf16-twin'
    k = 2 if variant == 'accum2' else 1
    mix = bm.BatchMix(0.4, 0.0, seed=5) if variant == 'batch_mix' else None
    ema = 0.9 if variant == 'ema' else None
    teacher = _teacher(lambda: models.resnet18(num_classes=10))
    before = _state(teacher)
    x, y = _data(16, 7, shape=(3, 64, 64))
    tr = _trainer(_resnet, teacher, alpha=0.5, temp=2.0, k=k, use_graph=True, twin=twin, batch_mix=mix,
                  ema_decay=ema)
    plain = _trainer(_resnet, k=k, use_graph=True, twin=twin, batch_mix=bm.BatchMix(0.4, 0.0, seed=5) if mix
                     else None, ema_decay=ema)
    assert tr.model.arena.flat.numel() == plain.model.arena.flat.numel()
    assert set(tr.model.state_dict()['state_dict']) == set(plain.model.state_dict()['state_dict'])
    net0 = copy.deepcopy(tr.model.module)
    tr.step(x, y)                                                   # eager warm-up step
    tr.finish()
    g_eager = tr.opt.momentum_flat[torch.float32].clone()
    flat = torch.cat([v.reshape(-1) for v in tr.opt._arenas[torch.float32].views_of(g_eager)])
    xs = x.to(DEV).contiguous(memory_format=torch.channels_last)
    ys = y.to(DEV)
    if mix is not None:
        # the batch the step trained on (mixed with its flipped batch) and the lam its loss kernels read
        assert mix.last.mode == bm.MIXUP
        xs, lam = tr.static_in.clone(), float(mix.state[0])
        assert 0.0 < lam < 1.0
        want = _reference_grad(net0, teacher, xs, ys, 0.5, 2.0, lam=lam)
    else:
        m = 16 // k
        want = sum(_reference_grad(net0, teacher, xs[j * m:(j + 1) * m], ys[j * m:(j + 1) * m], 0.5, 2.0,
                                   autocast=twin) for j in range(k)) / k
    if twin:
        # bf16 twin (bf16 weights, activations and teacher copy) against bf16 autocast of the fp32 networks
        assert _rel_err(flat, want) < 5e-2
        with torch.no_grad(), torch.autocast('cuda', dtype=BF16):
            u_ref = teacher(xs)
        u = tr._teacher_forward(tr.static_in)
        assert u.dtype == BF16 and u.shape == u_ref.shape
        assert _rel_err(u.float(), u_ref.float()) < 3e-2
        assert _rel_err(u.float(), teacher(xs).float()) < 3e-2          # (fp32 eval forward)
    else:
        scale = float(want.abs().max())
        torch.testing.assert_close(flat, want, rtol=1e-3, atol=2e-3 * scale)
    for _ in range(2):                                              # captured, replayed
        tr.step(x, y)
        plain.step(x, y)
    tr.finish()
    plain.finish()
    assert tr.graph is not None and plain.graph is not None
    g = tr.opt.momentum_flat[torch.float32]
    assert torch.isfinite(g).all()
    if mix is None:                                                 # (a mixed step draws a new lam)
        torch.testing.assert_close(g, g_eager, rtol=1e-3, atol=1e-3 * float(g_eager.abs().max()))
    # the teacher's launches, counted on an eager teacher forward of one micro-batch
    C = native.load()
    with torch.cuda.stream(tr.stream):
        c0 = C.launch_count()
        tr._teacher_forward(tr._micro[0][0] if k > 1 else tr.static_in)
        teacher_launches = C.launch_count() - c0
    assert teacher_launches > 0
    assert tr.own_launches_per_step == plain.own_launches_per_step + k * teacher_launches
    assert all(torch.equal(a, b) for a, b in zip(_state(teacher), before))
    assert not teacher.training and not any(p.requires_grad for p in teacher.parameters())
    metrics = tr.metrics_ring[(tr._loss_slot - 1) % 1024]
    assert torch.isfinite(metrics).all() and 0 <= float(metrics[1]) <= float(metrics[2]) <= 100


@pytest.mark.parametrize('twin', [False, True], ids=['fp32', 'bf16-twin'])
def test_evaluate_and_update_bn_do_not_run_the_teacher(twin):
    teacher = _teacher(lambda: models.resnet18(num_classes=10))
    batches = [_data(8, 50 + i, shape=(3, 64, 64)) for i in range(2)]
    results = []
    for t in (teacher, None):
        tr = _trainer(_resnet, t, use_graph=True, twin=twin)
        r = tr.evaluate(batches)
        eval_launches = tr.eval_launches_per_batch
        k = tr.update_bn(batches)
        bn = [b.clone() for b in tr.model.module.buffers()]
        results.append((r, eval_launches, k, tr.update_bn_launches_per_batch, bn))
    (r1, e1, k1, u1, bn1), (r0, e0, k0, u0, bn0) = results
    assert (r1.prec1, r1.prec5, r1.count) == (r0.prec1, r0.prec5, r0.count)
    assert r1.loss == pytest.approx(r0.loss, rel=1e-6)
    assert e1 == e0 and k1 == k0 == 2 and u1 == u0
    for a, b in zip(bn1, bn0):
        torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-6)


# ---------------------------------------------------------------------------------------------------- #
# the command line, one rank on one GPU
# ---------------------------------------------------------------------------------------------------- #
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLI = ['--model', 'tiny', '--num_classes', '10', '--image_size', '32', '--synthetic', 'True', '--synthetic_len', '64',
       '--batch_size', '16', '--verbose', 'False', '--print_freq', '2', '--num_dataloader_workers', '0', '--lr',
       '0.05', '--num_epochs', '1', '--num_itr_ignore', '0', '--distill_alpha', '0.5', '--distill_temperature', '2',
       '--teacher_model', 'tiny']


@pytest.mark.parametrize('extra', [
    ['--cuda_graph', 'False'],                                   # the eager loop: host batches, fused SGD
    ['--cuda_graph', 'False', '--fused', 'False'],
    ['--cuda_graph', 'False', '--amp', 'False'],
    ['--cuda_graph', 'True'],                                    # the captured trainer (bf16 twin)
    ['--all_reduce', 'True', '--graph_type', '-1'],
], ids=['eager', 'unfused', 'eager-fp32', 'graph', 'all-reduce'])
def test_cli_distills_on_the_gpu(tmp_path, master_port, extra):
    torch.manual_seed(3)
    torch.save(models.TinyConvNet().state_dict(), str(tmp_path / 'teacher.pth'))
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '1', '--master-addr',
           '127.0.0.1', '--master-port', str(master_port), os.path.join(ROOT, 'gossip_sgd.py')] + CLI + extra + [
           '--teacher_checkpoint', str(tmp_path / 'teacher.pth'), '--checkpoint_dir', str(tmp_path) + '/']
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:]
    assert out.stdout.count(' * Teacher Prec@1') == 1, out.stdout[-3000:]
    rows = [r.split(',') for r in open(str(tmp_path / 'out_r0_n1.csv')).read().splitlines()[5:]]
    losses = [float(r[12]) for r in rows if r[1] != '-1']
    assert losses and all(l == l and 0 < l < float('inf') for l in losses)
