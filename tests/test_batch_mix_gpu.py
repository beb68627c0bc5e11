"""Batch mixup / CutMix on the GPU: the batch-mix kernel (csrc/mix_kernels.cu) against
``reference_batch_mix``, the two-target fused cross-entropy (csrc/loss_kernels.cu, MIX = true) against
``reference_mixed_loss_and_accuracy``, ``mix=None`` against the one-target kernels, and a two-rank
loop-back GossipTrainer with ``batch_mix``: graph-captured equals eager, and mixing off is today's step."""
import functools

import pytest
import torch

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops import batch_mix as bm
from stochastic_gradient_push_b200.ops import fused_loss, native

from test_gdp_loopback_gpu import _in_threads

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


# --------------------------------------------------------------------------- #
# batch-mix kernel
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize('B,H,W', [(1, 7, 5), (7, 13, 21), (256, 16, 24)])
@pytest.mark.parametrize('src_nhwc', [False, True])
@pytest.mark.parametrize('out_dtype,out_nhwc', [(torch.float32, True), (torch.bfloat16, True),
                                                (torch.float32, False)])
def test_mix_kernel_matches_reference(B, H, W, src_nhwc, out_dtype, out_nhwc):
    g = torch.Generator(device='cuda').manual_seed(B * 131 + H)
    x = torch.randn(B, 3, H, W, device='cuda', generator=g) * 4
    if src_nhwc:
        x = x.contiguous(memory_format=torch.channels_last)
    fmt = torch.channels_last if out_nhwc else torch.contiguous_format
    out = torch.empty(B, 3, H, W, device='cuda', dtype=out_dtype).contiguous(memory_format=fmt)
    mix = bm.BatchMix(0.2, 1.0)
    cases = [bm.MixParams(0.37, bm.MIXUP, 0, 0, 0, 0), bm.MixParams(0.0, bm.MIXUP, 0, 0, 0, 0),
             bm.MixParams(float(torch.tensor(0.8125).item()), bm.CUTMIX, 1, H - 2, 2, W - 1),
             bm.MixParams(1.0, bm.CUTMIX, 0, 0, 0, W), bm.MixParams(1.0, bm.NO_MIX, 0, 0, 0, 0)]
    cases += [mix.sample(H, W, itr=i) for i in range(4)]
    for p in cases:
        out.fill_(float('nan'))
        mix.apply(x, out, params=p)
        torch.cuda.synchronize()
        want = bm.reference_batch_mix(x, p).to(out_dtype)
        # mixup: the documented fp32 formula, bit for bit; CutMix and the plain copy: a select
        assert torch.equal(_bits(out.contiguous()), _bits(want.contiguous())), p
        if B % 2 and p.mode != bm.MIXUP:
            assert torch.equal(out[B // 2].float(), x[B // 2].to(out_dtype).float())
    if B % 2:
        mix.apply(x, out, params=bm.MixParams(0.37, bm.MIXUP, 0, 0, 0, 0))
        torch.testing.assert_close(out[B // 2].float(), x[B // 2].to(out_dtype).float(),
                                   rtol=1e-6 if out_dtype == torch.float32 else 1e-2, atol=1e-6)


def test_mix_kernel_follows_the_staged_state_under_graph_capture():
    """the kernel reads lam and the box from the device state: a captured launch replays every
    step's draw without re-capture"""
    x = torch.randn(6, 3, 10, 12, device='cuda')
    out = torch.empty(6, 3, 10, 12, device='cuda').contiguous(memory_format=torch.channels_last)
    mix = bm.BatchMix(0.4, 1.0, seed=9)
    mix.apply(x, out, params=bm.MixParams(1.0, bm.NO_MIX, 0, 0, 0, 0))
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        native.load().batch_mix(x, out, mix.state)
    for i in range(12):
        p = mix.sample(10, 12, itr=i)
        mix.stage(p, x.device)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, bm.reference_batch_mix(x, p)), p


def test_mix_kernel_rejects_bad_tensors():
    C = native.load()
    x = torch.randn(4, 3, 8, 8, device='cuda')
    state = torch.zeros(8, device='cuda')
    with pytest.raises(RuntimeError):
        C.batch_mix(x, x, state)                                   # in place
    with pytest.raises(RuntimeError):
        C.batch_mix(x.half(), torch.empty_like(x), state)          # fp16 source
    with pytest.raises(RuntimeError):
        C.batch_mix(x, torch.empty(4, 3, 8, 9, device='cuda'), state)
    with pytest.raises(RuntimeError):
        C.batch_mix(x, torch.empty_like(x), torch.zeros(3, device='cuda'))
    with pytest.raises(RuntimeError):
        C.batch_mix(x[:, :, :, :4], torch.empty(4, 3, 8, 4, device='cuda'), state)   # not dense


# --------------------------------------------------------------------------- #
# two-target fused cross-entropy
# --------------------------------------------------------------------------- #
SHAPES = [(256, 1000), (7, 10), (1, 5), (64, 33)]


@pytest.mark.parametrize('lam', [0.0, 0.37, 1.0])
@pytest.mark.parametrize('eps', [0.0, 0.1])
@pytest.mark.parametrize('B,C', SHAPES)
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_mixed_loss_metrics_and_gradient(B, C, dtype, eps, lam):
    g = torch.Generator(device='cuda').manual_seed(B * 31 + C)
    logits = (torch.randn(B, C, device='cuda', generator=g) * 3).to(dtype).requires_grad_(True)
    target = torch.randint(0, C, (B,), device='cuda', generator=g)
    if B >= 4:
        target[1] = target[B - 2]                    # a == b rows
        target[0] = C + 3                            # out of range: rows 0 and B-1 add nothing
    state = torch.tensor([lam, 1, 0, 0, 0, 0, 0, 0], device='cuda')
    crit = fused_loss.FusedCrossEntropyWithAccuracy(label_smoothing=eps)
    loss = crit(logits, target, mix=state)
    assert native.load().xent_can_fuse(logits.detach(), target)
    (loss * 1.7).backward()
    torch.cuda.synchronize()

    ref_logits = logits.detach().float().requires_grad_(True)
    want, p1, p5 = bm.reference_mixed_loss_and_accuracy(ref_logits, target, lam, eps)
    (want * 1.7).backward()
    torch.testing.assert_close(loss.detach(), want.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(crit.metrics[0], want.detach(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(crit.metrics[1], p1, rtol=0, atol=1e-3)
    torch.testing.assert_close(crit.metrics[2], p5, rtol=0, atol=1e-3)
    tol = 1e-6 if dtype == torch.float32 else 4e-3 / B
    torch.testing.assert_close(logits.grad.float(), ref_logits.grad,
                               rtol=1e-4 if dtype == torch.float32 else 1e-2, atol=tol)
    if B >= 4:
        assert torch.all(logits.grad[0] == 0) and torch.all(logits.grad[B - 1] == 0)


@pytest.mark.parametrize('eps', [0.0, 0.1])
@pytest.mark.parametrize('B,C', SHAPES)
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_no_mix_is_the_one_target_kernel(B, C, dtype, eps):
    """mix=None runs the MIX = false kernels: per-row log-sum-exp, gradient and accuracies are
    bit-identical to the call without the argument"""
    C_ = native.load()
    g = torch.Generator(device='cuda').manual_seed(B + C)
    lg = (torch.randn(B, C, device='cuda', generator=g) * 3).to(dtype)
    target = torch.randint(0, C, (B,), device='cuda', generator=g)
    m0, lse0 = C_.xent_forward(lg, target, eps)
    m1, lse1 = C_.xent_forward(lg, target, eps, None)
    m2, lse2 = C_.xent_forward(lg, target, label_smoothing=eps, mix=None)
    gr = torch.tensor([1.3], device='cuda')
    d0 = C_.xent_backward(lg, target, lse0, gr, eps)
    d1 = C_.xent_backward(lg, target, lse0, gr, eps, None)
    crit = fused_loss.FusedCrossEntropyWithAccuracy(eps)
    lgr = lg.clone().requires_grad_(True)
    crit(lgr, target, mix=None).backward(torch.tensor(1.3, device='cuda'))
    torch.cuda.synchronize()
    assert torch.equal(lse0, lse1) and torch.equal(lse0, lse2)
    assert torch.equal(_bits(d0), _bits(d1)) and torch.equal(_bits(d0), _bits(lgr.grad))
    for m in (m1, m2, crit.metrics):
        torch.testing.assert_close(m[0], m0[0], rtol=B * 2.0 ** -23, atol=0)
        torch.testing.assert_close(m[1:], m0[1:], rtol=0, atol=1e-3)


def test_unmixed_state_gives_the_one_target_gradient():
    """mode 0 (a step the draw left unmixed) has lam = 1: the MIX kernels then subtract exactly the
    one-target mass, so the gradient is bit-identical"""
    C_ = native.load()
    lg = torch.randn(32, 100, device='cuda') * 3
    target = torch.randint(0, 100, (32,), device='cuda')
    state = torch.tensor([1.0, 0, 0, 0, 0, 0, 0, 0], device='cuda')
    gr = torch.tensor([0.7], device='cuda')
    m0, lse0 = C_.xent_forward(lg, target)
    m1, lse1 = C_.xent_forward(lg, target, 0.0, state)
    d0 = C_.xent_backward(lg, target, lse0, gr)
    d1 = C_.xent_backward(lg, target, lse1, gr, 0.0, state)
    torch.cuda.synchronize()
    assert torch.equal(lse0, lse1) and torch.equal(d0, d1)
    torch.testing.assert_close(m1, m0, rtol=32 * 2.0 ** -23, atol=1e-3)


# --------------------------------------------------------------------------- #
# loop-back trainer
# --------------------------------------------------------------------------- #
def _train(n, steps, use_graph, make_mix, tag):
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
        net = models.TinyConvNet().to(dev).to(memory_format=torch.channels_last)
        model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(r, n),
                                   rank=r, world_size=n, heartbeat_timeout=20, symmetric_world=lw.view(r),
                                   transport='nvlink', grid=4, symmetric_name='loopback_mix_' + tag)
        opt = FusedGossipSGD(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True)
        trainers.append(GossipTrainer(model, opt, fused_loss.FusedCrossEntropyWithAccuracy(0.1), amp_dtype=None,
                                      use_cuda_graph=use_graph, warmup_iters=10 ** 6, batch_mix=make_mix(r)))
    gens = [torch.Generator().manual_seed(100 + r) for r in range(n)]
    inputs, metrics = [], []
    for s in range(steps):
        if use_graph and s == 2:
            for tr in trainers:              # every capture before any replay (see test_gdp_loopback_gpu)
                with torch.cuda.stream(tr.stream):
                    tr._capture()

        def rank_step(r):
            x = torch.randn(9, 3, 20, 28, generator=gens[r]).pin_memory()
            y = torch.randint(0, 10, (9,), generator=gens[r]).pin_memory()
            slot = trainers[r].step(x, y)
            trainers[r].stream.synchronize()
            metrics.append((s, r, trainers[r].metrics_ring[slot].clone()))
            inputs.append((s, r, trainers[r].static_in.clone()))
        _in_threads([functools.partial(rank_step, r) for r in range(n)])
        torch.cuda.synchronize()
    for tr in trainers:
        tr.finish()
        assert (tr.graph is not None) == use_graph
    return ([tr.model.arena.flat.cpu().clone() for tr in trainers], sorted(inputs, key=lambda t: t[:2]),
            sorted(metrics, key=lambda t: t[:2]), trainers)


def test_loopback_trainer_with_batch_mix_graphed_equals_eager():
    n, steps = 2, 8

    def mix(r):
        return bm.BatchMix(mixup_alpha=0.4, cutmix_alpha=1.0, seed=3, rank=r)
    eager, eager_in, eager_m, trainers = _train(n, steps, False, mix, 'e')
    graphed, graphed_in, graphed_m, _ = _train(n, steps, True, mix, 'g')
    assert {tr.batch_mix.last.mode for tr in trainers} <= {bm.MIXUP, bm.CUTMIX}
    for (s, r, a), (_, _, b) in zip(eager_in, graphed_in):
        assert torch.equal(a, b), (s, r)                  # same draw, same mixed batch
    for (s, r, a), (_, _, b) in zip(eager_m, graphed_m):
        torch.testing.assert_close(b, a, rtol=1e-4, atol=1e-4)
    for r in range(n):
        assert torch.isfinite(eager[r]).all()
        torch.testing.assert_close(graphed[r], eager[r], rtol=1e-4, atol=1e-5)


def test_loopback_trainer_with_mixing_off_is_todays_step():
    n, steps = 2, 5
    base, base_in, base_m, _ = _train(n, steps, True, lambda r: None, 'base')
    off, off_in, off_m, trainers = _train(n, steps, True, lambda r: bm.BatchMix(seed=3, rank=r), 'off')
    assert all(tr.batch_mix is None for tr in trainers)        # both alphas 0: the plain copy and loss
    # every step drawn unmixed: the mix kernel copies, the two-target loss has lam = 1
    never, never_in, never_m, _ = _train(
        n, steps, True, lambda r: bm.BatchMix(0.4, 1.0, mix_prob=0.0, seed=3, rank=r), 'never')
    # the inputs are bit-identical; parameters and metrics are compared to within the float-atomic
    # reorderings two runs of the same step may differ by
    for (s, r, a), (_, _, b), (_, _, c) in zip(base_in, off_in, never_in):
        assert torch.equal(a, b) and torch.equal(a, c), (s, r)
    for (s, r, a), (_, _, b), (_, _, c) in zip(base_m, off_m, never_m):
        torch.testing.assert_close(b, a, rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(c, a, rtol=1e-5, atol=1e-5)
    for r in range(n):
        torch.testing.assert_close(off[r], base[r], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(never[r], base[r], rtol=1e-5, atol=1e-6)
