"""Label smoothing in the fused cross-entropy kernel (csrc/loss_kernels.cu) against
``F.cross_entropy(label_smoothing=eps)``, its eps = 0 path against the unsmoothed call, graph capture,
and a two-rank loop-back trainer that trains on the smoothed fused loss."""
import functools

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops import fused_loss, native

from test_gdp_loopback_gpu import _in_threads

pytestmark = pytest.mark.gpu

SHAPES = [(256, 1000), (32, 1000), (7, 10), (1, 5), (64, 33), (16, 4099)]


def _inputs(B, C, dtype):
    g = torch.Generator(device='cuda').manual_seed(B * 31 + C)
    logits = (torch.randn(B, C, device='cuda', generator=g) * 3).to(dtype).requires_grad_(True)
    target = torch.randint(0, C, (B,), device='cuda', generator=g)
    return logits, target


@pytest.mark.parametrize('eps', [0.1, 0.5, 1.0])
@pytest.mark.parametrize('B,C', SHAPES)
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_smoothed_loss_metrics_and_gradient(B, C, dtype, eps):
    logits, target = _inputs(B, C, dtype)
    crit = fused_loss.FusedCrossEntropyWithAccuracy(label_smoothing=eps)
    loss = crit(logits, target)
    assert native.load().xent_can_fuse(logits.detach(), target)
    (loss * 1.7).backward()
    torch.cuda.synchronize()

    ref_logits = logits.detach().float().requires_grad_(True)
    want = F.cross_entropy(ref_logits, target, label_smoothing=eps)
    (want * 1.7).backward()
    _, p1, p5 = fused_loss.reference_loss_and_accuracy(ref_logits.detach(), target)
    torch.testing.assert_close(loss.detach(), want.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(crit.metrics[0], want.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(crit.metrics[1], p1, rtol=0, atol=1e-3)
    torch.testing.assert_close(crit.metrics[2], p5, rtol=0, atol=1e-3)
    tol = 1e-6 if dtype == torch.float32 else 4e-3 / B
    torch.testing.assert_close(logits.grad.float(), ref_logits.grad, rtol=1e-2 if dtype != torch.float32 else 1e-4,
                               atol=tol)


@pytest.mark.parametrize('B,C', SHAPES)
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_zero_smoothing_is_the_unsmoothed_kernel(B, C, dtype):
    """eps = 0 through the new argument runs the unsmoothed kernels: the per-row log-sum-exp, the
    gradient and the accuracies are bit-identical.  The mean loss is summed with float atomics
    across rows, whose order is not fixed, so it is bit-identical for one row and equal to within
    that reordering otherwise."""
    C_ = native.load()
    logits, target = _inputs(B, C, dtype)
    lg = logits.detach()
    m0, lse0 = C_.xent_forward(lg, target)
    m1, lse1 = C_.xent_forward(lg, target, 0.0)
    m2, lse2 = C_.xent_forward(lg, target, label_smoothing=0.0)
    g = torch.tensor([1.7], device='cuda')
    d0 = C_.xent_backward(lg, target, lse0, g)
    d1 = C_.xent_backward(lg, target, lse0, g, 0.0)
    torch.cuda.synchronize()
    assert torch.equal(lse0, lse1) and torch.equal(lse0, lse2)
    assert torch.equal(d0.view(torch.int16 if dtype == torch.bfloat16 else torch.int32),
                       d1.view(torch.int16 if dtype == torch.bfloat16 else torch.int32))
    # B non-negative fp32 terms summed in another order differ by at most (B - 1) ulp of the sum
    reorder = B * 2.0 ** -23
    exact_prec = (100.0 / B) * (1 << 20) == round((100.0 / B) * (1 << 20))     # 100/B a short binary fraction
    for m in (m1, m2):
        if B == 1:
            assert torch.equal(m, m0)
        else:
            torch.testing.assert_close(m[0], m0[0], rtol=reorder, atol=0)
        if exact_prec:
            assert torch.equal(m[1:], m0[1:])
        else:
            torch.testing.assert_close(m[1:], m0[1:], rtol=reorder, atol=0)

    # and through the module: the same loss value, gradient bits and metrics
    a = logits.detach().clone().requires_grad_(True)
    b = logits.detach().clone().requires_grad_(True)
    la, ma = fused_loss.fused_cross_entropy(a, target)
    lb, mb = fused_loss.fused_cross_entropy(b, target, label_smoothing=0.0)
    la.backward()
    lb.backward()
    torch.cuda.synchronize()
    assert torch.equal(a.grad, b.grad)
    torch.testing.assert_close(lb, la, rtol=reorder, atol=0)


@pytest.mark.parametrize('eps', [-0.01, 1.01, float('nan')])
def test_binding_rejects_invalid_smoothing(eps):
    C_ = native.load()
    logits, target = _inputs(8, 10, torch.float32)
    with pytest.raises(RuntimeError, match='label_smoothing'):
        C_.xent_forward(logits.detach(), target, eps)
    _, lse = C_.xent_forward(logits.detach(), target)
    with pytest.raises(RuntimeError, match='label_smoothing'):
        C_.xent_backward(logits.detach(), target, lse, torch.ones(1, device='cuda'), eps)
    with pytest.raises(ValueError, match='label_smoothing'):
        fused_loss.fused_cross_entropy(logits, target, eps)


def test_out_of_range_target_adds_no_loss_and_no_gradient():
    B, C, eps = 16, 50, 0.2
    logits, target = _inputs(B, C, torch.float32)
    target = target.clone()
    target[3], target[9] = -1, C
    loss, m = fused_loss.fused_cross_entropy(logits, target, label_smoothing=eps)
    loss.backward()
    torch.cuda.synchronize()
    keep = torch.ones(B, dtype=torch.bool, device='cuda')
    keep[3] = keep[9] = False
    ref = logits.detach().requires_grad_(True)
    per_row = F.cross_entropy(ref[keep], target[keep], label_smoothing=eps, reduction='none')
    want = per_row.sum() / B
    want.backward()
    torch.testing.assert_close(loss.detach(), want.detach(), rtol=1e-5, atol=1e-5)
    assert (logits.grad[3] == 0).all() and (logits.grad[9] == 0).all()
    torch.testing.assert_close(logits.grad, ref.grad, rtol=1e-4, atol=1e-6)


def test_cuda_graph_capture_with_smoothing():
    eps = 0.1
    logits = torch.randn(32, 100, device='cuda', requires_grad=True)
    target = torch.randint(0, 100, (32,), device='cuda')
    out = torch.zeros(3, device='cuda')
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            loss, m = fused_loss.fused_cross_entropy(logits, target, label_smoothing=eps)
            loss.backward()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    logits.grad = None
    with torch.cuda.graph(graph):
        loss, m = fused_loss.fused_cross_entropy(logits, target, label_smoothing=eps)
        loss.backward()
        out.copy_(m)
    with torch.no_grad():
        logits.copy_(torch.randn(32, 100, device='cuda'))
    logits.grad.zero_()
    graph.replay()
    torch.cuda.synchronize()
    ref = logits.detach().clone().requires_grad_(True)
    want = F.cross_entropy(ref, target, label_smoothing=eps)
    want.backward()
    torch.testing.assert_close(out[0], want.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(logits.grad, ref.grad, rtol=1e-4, atol=1e-6)
    _, p1, p5 = fused_loss.reference_loss_and_accuracy(ref.detach(), target)
    torch.testing.assert_close(out[1], p1, rtol=0, atol=1e-3)
    torch.testing.assert_close(out[2], p5, rtol=0, atol=1e-3)


def _loopback_run(make_criterion, use_graph, n=2, steps=6, make_net=None):
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    dev = torch.device('cuda', 0)
    lw = LocalWorld(n)
    trainers = []
    for r in range(n):
        torch.manual_seed(7 + r)
        net = (make_net or models.TinyConvNet)().to(dev).to(memory_format=torch.channels_last)
        model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(r, n),
                                   rank=r, world_size=n, heartbeat_timeout=20, symmetric_world=lw.view(r),
                                   transport='nvlink', grid=4, symmetric_name='loopback_smooth')
        opt = FusedGossipSGD(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True)
        trainers.append(GossipTrainer(model, opt, make_criterion(), amp_dtype=None, use_cuda_graph=use_graph,
                                      warmup_iters=10 ** 6))
    gens = [torch.Generator().manual_seed(100 + r) for r in range(n)]
    slots = [[] for _ in range(n)]
    for s in range(steps):
        if use_graph and s == 2:
            for tr in trainers:          # every capture before any replay (see test_gdp_loopback_gpu)
                with torch.cuda.stream(tr.stream):
                    tr._capture()

        def rank_step(r):
            x = torch.randn(8, 3, 32, 32, generator=gens[r]).pin_memory()
            y = torch.randint(0, 10, (8,), generator=gens[r]).pin_memory()
            slots[r].append(trainers[r].step(x, y))
        _in_threads([functools.partial(rank_step, r) for r in range(n)])
        torch.cuda.synchronize()
    for tr in trainers:
        tr.finish()
    assert all((tr.graph is not None) == use_graph for tr in trainers)
    return [(tr.model.arena.flat.cpu().clone(), tr.metrics_ring[slots[r]].clone())
            for r, tr in enumerate(trainers)]


def test_loopback_trainer_with_smoothed_fused_loss():
    """FusedCrossEntropyWithAccuracy(0.1) in GossipTrainer: the graphed and eager runs agree, both
    match a run with nn.CrossEntropyLoss(label_smoothing=0.1), and the metrics ring carries the
    smoothed loss with finite prec@1 / prec@5."""
    eps = 0.1
    fused = functools.partial(fused_loss.FusedCrossEntropyWithAccuracy, label_smoothing=eps)
    eager = _loopback_run(fused, use_graph=False)
    graphed = _loopback_run(fused, use_graph=True)
    torch_ce = _loopback_run(lambda: nn.CrossEntropyLoss(label_smoothing=eps), use_graph=False)
    for r in range(2):
        assert torch.isfinite(eager[r][0]).all()
        torch.testing.assert_close(graphed[r][0], eager[r][0], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(eager[r][0], torch_ce[r][0], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(graphed[r][0], torch_ce[r][0], rtol=1e-4, atol=1e-5)
        for run in (eager, graphed):
            ring = run[r][1]
            assert torch.isfinite(ring).all()
            assert ((ring[:, 1] >= 0) & (ring[:, 1] <= ring[:, 2]) & (ring[:, 2] <= 100)).all()
            # the smoothed training loss, as nn.CrossEntropyLoss(label_smoothing=eps) computes it
            torch.testing.assert_close(ring[:, 0], torch_ce[r][1][:, 0], rtol=1e-4, atol=1e-5)
        assert torch.isnan(torch_ce[r][1][:, 1:]).all()       # an unfused criterion measures no accuracy
