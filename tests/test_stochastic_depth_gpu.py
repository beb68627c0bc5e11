"""Stochastic depth on the GPU: the draw kernel against its oracle and its device counter under graph
capture; the scaled fused BatchNorm kernels (bf16, fp32 split and consecutive maps) and the conv1x1 path,
including the MODE 3 hand-off, against the reference composition's autograd; and the model under
GossipTrainer (captured replays against eager steps, gradient accumulation, update_bn and evaluate)."""
import pytest
import torch
import torch.nn.functional as F

from stochastic_gradient_push_b200 import models
from stochastic_gradient_push_b200.ops import fused_bn, native, oracle
from stochastic_gradient_push_b200.ops.fused_bn import (FusedBatchNormAct2d, bn_f32_map, conv_bn_act,
                                                        fused_bn_act, reference_bn_act)
from stochastic_gradient_push_b200.ops.stochastic_depth import StochasticDepth

from test_fused_bn_gpu import assert_mostly_close
from test_trainer_evaluate_gpu import _data, _same_metrics, _trainer

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
BF16 = torch.bfloat16


@pytest.fixture
def deterministic_cudnn():
    prev = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = prev


# ---------------------------------------------------------------------------------------------------- #
# the draw kernel
# ---------------------------------------------------------------------------------------------------- #
@pytest.mark.parametrize('seed,rank,start,n,L,p', [(47, 0, 0, 256, 16, 0.05), (-3, 5, 123456789, 7, 8, 0.5),
                                                   (2 ** 40, 1, 2 ** 33, 1000, 50, 0.9), (0, 0, 0, 1, 1, 0.3)])
def test_draw_kernel_matches_the_oracle(seed, rank, start, n, L, p):
    sd = StochasticDepth(L, p, seed=seed, rank=rank)
    sd.set_draws(start)
    for d in range(3):
        got = sd.draw(n, DEV)
        assert got.shape == (L, n) and got.dtype == torch.float32 and got.device == DEV
        want = oracle.drop_path_scales(seed, rank, start + d, sd.thresholds, sd.keep_scales, n)
        assert torch.equal(got.cpu(), want)
    assert sd.draws == start + 3


def test_counter_advances_per_replay_not_at_capture():
    sd = StochasticDepth(16, 0.2, seed=1, rank=0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        sd.draw(32, DEV)                                      # eager: draw 0
    torch.cuda.synchronize()
    assert sd.draws == 1
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out = sd.draw(32, DEV)
    torch.cuda.synchronize()
    assert sd.draws == 1                                      # a capture does not execute
    for d in (1, 2, 3):
        g.replay()
        torch.cuda.synchronize()
        assert sd.draws == d + 1
        assert torch.equal(out.cpu(), oracle.drop_path_scales(1, 0, d, sd.thresholds, sd.keep_scales, 32))


# ---------------------------------------------------------------------------------------------------- #
# op level
# ---------------------------------------------------------------------------------------------------- #
def _scales(N, g, drop=0.3, keep=1.25):
    u = torch.rand(N, generator=g)
    s = torch.where(u < drop, torch.zeros(N), torch.full((N,), keep))
    s[0], s[-1] = 0.0, keep                                   # at least one of each
    return s.to(DEV)


def _run_bn(fn, x, res, w, b, s, dtype, dy):
    x = x.detach().clone().to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    r = res.detach().clone().to(dtype).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    w = w.detach().clone().requires_grad_(True)
    b = b.detach().clone().requires_grad_(True)
    C = w.numel()
    rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    y = fn(x, w, b, rm, rv, None, residual=r, relu=True, training=True, branch_scale=s)
    y.backward(dy.to(dtype).contiguous(memory_format=torch.channels_last))
    return dict(y=y.detach().float(), dx=x.grad.float(), dres=r.grad.float(), dw=w.grad, db=b.grad, rm=rm, rv=rv)


MAPS = [(torch.bfloat16, True), (torch.float32, True), (torch.float32, False)]
MAP_IDS = ['bf16', 'f32-split', 'f32-consecutive']


@pytest.mark.parametrize('shape', [(8, 64, 14, 14), (4, 256, 7, 9), (6, 2048, 2, 2), (32, 64, 56, 56)])
@pytest.mark.parametrize('dtype,split', MAPS, ids=MAP_IDS)
def test_scaled_bn_matches_the_reference(shape, dtype, split):
    g = torch.Generator().manual_seed(1)
    N, C, H, W = shape
    x = (torch.randn(shape, generator=g) * 2 + 0.5).to(DEV)
    res = torch.randn(shape, generator=g).to(DEV)
    w = (torch.rand(C, generator=g) + 0.5).to(DEV)
    b = (torch.randn(C, generator=g) * 0.1).to(DEV)
    dy = torch.randn(shape, generator=g).to(DEV)
    s = _scales(N, g)
    with bn_f32_map(split):
        got = _run_bn(fused_bn_act, x, res, w, b, s, dtype, dy)
        ones = _run_bn(fused_bn_act, x, res, w, b, torch.ones(N, device=DEV), dtype, dy)
        plain = _run_bn(fused_bn_act, x, res, w, b, None, dtype, dy)
    want = _run_bn(reference_bn_act, x.to(dtype).float(), res.to(dtype).float(), w, b, s, torch.float32,
                   dy.to(dtype).float())
    tol = dict(rtol=1e-4, atol=1e-4) if dtype == torch.float32 else dict(rtol=2e-2, atol=2e-2)
    for k in ('y', 'dx', 'dres'):
        assert_mostly_close(got[k], want[k], **tol)
    for k in ('dw', 'db'):
        torch.testing.assert_close(got[k], want[k], rtol=1e-3 if dtype == torch.float32 else 2e-2,
                                   atol=1e-3 if dtype == torch.float32 else 5e-1)
    torch.testing.assert_close(got['rm'], want['rm'], rtol=1e-4, atol=1e-4)
    for k in plain:                                           # s = 1: the unscaled kernels, bit for bit
        assert torch.equal(ones[k], plain[k]), k
    dropped = (s == 0).nonzero().flatten()
    r = res.to(dtype)
    for n in dropped.tolist():                                # a dropped sample's output is relu(residual)
        assert torch.equal(got['y'][n], F.relu(r[n]).float())


def _conv_bn(C_in=64, C_out=256, seed=0):
    torch.manual_seed(seed)
    conv = torch.nn.Conv2d(C_in, C_out, 1, bias=False).to(DEV).to(memory_format=torch.channels_last)
    bn = FusedBatchNormAct2d(C_out).to(DEV)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_(0, 0.1)
    return conv, bn


def _rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-12)).item()


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_scaled_conv_bn_act_matches_the_unfused_path(dtype, monkeypatch):
    """the wgmma conv + scaled BN op against the library convolution + the scaled stand-alone BN op (checked
    against the reference above), as test_conv1x1_gpu compares the unscaled ones: TF32 / bf16 rounding
    flips ReLU masks of near-zero activations, so the two are compared in norm"""
    g = torch.Generator().manual_seed(2)
    N, H, W = 8, 14, 14
    conv, bn = _conv_bn()
    conv = conv.to(dtype)
    x = torch.randn(N, 64, H, W, generator=g).to(DEV).to(dtype).contiguous(memory_format=torch.channels_last)
    res = torch.randn(N, 256, H, W, generator=g).to(DEV).to(dtype).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(N, 256, H, W, generator=g).to(DEV).to(dtype).contiguous(memory_format=torch.channels_last)
    s = _scales(N, g)

    def run(gemm, s):
        monkeypatch.setattr(fused_bn, 'USE_TCGEN05_CONV1X1', gemm)
        xi, ri = x.clone().requires_grad_(True), res.clone().requires_grad_(True)
        conv.weight.grad = bn.weight.grad = bn.bias.grad = None
        y = conv_bn_act(conv, bn, xi, residual=ri, relu=True, branch_scale=s)
        y.backward(dy)
        return dict(y=y.detach().float(), dx=xi.grad.float(), dres=ri.grad.float(),
                    dw=conv.weight.grad.float(), dg=bn.weight.grad.clone(), db=bn.bias.grad.clone())
    got, want = run(True, s), run(False, s)
    for k in got:
        assert _rel(got[k], want[k]) < 3e-2, k
    ones, plain = run(True, torch.ones(N, device=DEV)), run(True, None)
    for k in plain:                                           # s = 1: the unscaled kernels, bit for bit
        assert torch.equal(ones[k], plain[k]), k
    for n in (s == 0).nonzero().flatten().tolist():           # a dropped sample's output is relu(residual)
        assert torch.equal(got['y'][n], F.relu(res[n]).float())


def _bottlenecks(dtype, rate):
    torch.manual_seed(3)
    net = models.ResNet(models.Bottleneck, [2, 1, 1, 1], num_classes=10, drop_path_rate=rate)
    net = net.to(DEV).to(memory_format=torch.channels_last)
    for m in net.modules():                                   # compute-dtype convolutions, fp32 BatchNorm
        if isinstance(m, torch.nn.Conv2d):
            m.to(dtype)
    return net


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
def test_mode3_handoff_with_scales(dtype, monkeypatch):
    """two consecutive bottlenecks (layer1's), the first scaled: MODE 3 engaged gives the gradients of
    the stand-alone reduction (SGP_B200_BN_BWD_FUSE=0)"""
    g = torch.Generator().manual_seed(4)
    x = torch.randn(4, 64, 16, 16, generator=g).to(DEV).to(dtype).contiguous(memory_format=torch.channels_last)
    dy = torch.randn(4, 256, 16, 16, generator=g).to(DEV).to(dtype).contiguous(memory_format=torch.channels_last)
    s = _scales(4, g, drop=0.4, keep=1.5)
    C = native.load()
    calls = []
    real = C.conv1x1_dgrad_bn_reduce

    def spy(*a, **kw):
        calls.append(kw.get('branch_scale'))
        return real(*a, **kw)
    monkeypatch.setattr(C, 'conv1x1_dgrad_bn_reduce', spy)
    net = _bottlenecks(dtype, 0.0)
    blk0, blk1 = net.layer1[0], net.layer1[1]

    def run(fuse):
        monkeypatch.setattr(fused_bn, 'USE_BN_BWD_FUSE', fuse)
        net.zero_grad(set_to_none=True)
        xi = x.clone().requires_grad_(True)
        h = blk0(xi, s)
        y = blk1(h)
        y.backward(dy)
        return [xi.grad.float()] + [p.grad.float() for p in list(blk0.parameters()) + list(blk1.parameters())]
    plain = run(False)
    assert not calls
    fused = run(True)
    assert len(calls) == 1 and calls[0] is not None and torch.equal(calls[0], s)   # the hand-off was used
    tol = dict(rtol=2e-3, atol=2e-3) if dtype == torch.float32 else dict(rtol=3e-2, atol=3e-2)
    assert_mostly_close(fused[0], plain[0], **tol)
    for a, b in zip(fused[1:], plain[1:]):
        torch.testing.assert_close(a, b, rtol=2e-2, atol=2e-2 if dtype == torch.float32 else 2e-1)


# ---------------------------------------------------------------------------------------------------- #
# the model
# ---------------------------------------------------------------------------------------------------- #
@pytest.mark.parametrize('arch', ['resnet18', 'resnet50'])
def test_model_matches_the_reference_with_the_same_scales(arch, monkeypatch):
    """loss and gradients of a training step at rate 0.1 through the fused kernels, through the library path
    (FORCE_REFERENCE, fp32 / TF32) and in fp64 (the truth), all with the same draws: ours is as close to the
    truth as the library path is (the pattern of test_conv1x1_gpu's fp32 bottleneck test)"""
    import copy
    torch.manual_seed(5)
    net0 = getattr(models, arch)(num_classes=10, drop_path_rate=0.1).to(DEV).to(memory_format=torch.channels_last)
    sd = net0.stochastic_depth
    x, t = _data(8, 6, hw=64)
    x, t = x.to(DEV).contiguous(memory_format=torch.channels_last), t.to(DEV)

    def run(mode):
        net, xi = copy.deepcopy(net0), x
        monkeypatch.setattr(fused_bn, 'FORCE_REFERENCE', mode != 'ours')
        if mode == 'fp64':
            net, xi = net.double(), x.double()
        sd.set_draws(7)
        loss = F.cross_entropy(net(xi), t)
        loss.backward()
        torch.cuda.synchronize()
        return [loss.detach().double().view(1)] + [p.grad.double() for p in net.parameters()]
    truth, ours, lib = run('fp64'), run('ours'), run('lib')
    assert sd.draws == 8
    for i, (a, b, c) in enumerate(zip(ours, lib, truth)):
        e_ours, e_lib = _rel(a, c), _rel(b, c)
        assert e_ours < max(3.0 * e_lib, 2e-3), (i, e_ours, e_lib)


def _sd_trainer(arch, twin, use_graph, rate=0.1):
    def net_fn():
        return getattr(models, arch)(num_classes=10, drop_path_rate=rate)
    return _trainer(twin=twin, use_graph=use_graph, net_fn=net_fn, lr=0.02)


@pytest.mark.parametrize('arch', ['resnet18', 'resnet50'])
@pytest.mark.parametrize('twin', [False, True], ids=['fp32', 'bf16-twin'])
def test_captured_replays_equal_eager_steps(arch, twin, deterministic_cudnn):
    """the same draws, eager or replayed, and (lr 0: the same weights at every step) the same logits, bit for
    bit, at every step; the loss rows agree to the rounding of the loss kernel's float atomics"""
    batches = [_data(16, 30 + s) for s in range(4)]
    runs = []
    for use_graph in (False, True):
        tr = _trainer(twin=twin, use_graph=use_graph, lr=0.0,
                      net_fn=lambda: getattr(models, arch)(num_classes=10, drop_path_rate=0.1))
        sd = tr.model.module.stochastic_depth
        if twin:
            assert tr.model._twin[0].stochastic_depth is sd
        seen = []
        real = sd.draw

        def spy(n, device):
            out = real(n, device)
            seen.append(out)
            return out
        sd.draw = spy
        draws, logits, metrics = [], [], []
        for b in batches:
            slot = tr.step(*b)
            torch.cuda.synchronize()
            draws.append(seen[-1].cpu().clone())
            logits.append(tr.static_out.cpu().clone())
            metrics.append(tr.metrics_ring[slot].clone())
        tr.finish()
        assert sd.draws == len(batches)                       # one draw per forward, replays included
        assert (tr.graph is not None) == use_graph
        for d, o in enumerate(draws):
            assert torch.equal(o, oracle.drop_path_scales(sd.seed, sd.rank, d, sd.thresholds, sd.keep_scales, 16))
        runs.append((logits, metrics))
    (l0, m0), (l1, m1) = runs
    for a, b in zip(l0, l1):
        assert torch.equal(a, b)
    for a, b in zip(m0, m1):
        _same_metrics(a, b)


def test_accumulation_draws_per_micro_batch(deterministic_cudnn):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    import stochastic_gradient_push_b200 as sgp
    torch.manual_seed(11)
    net = models.resnet18(num_classes=10, drop_path_rate=0.3).to(DEV).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                               heartbeat_timeout=20)
    opt = FusedGossipSGD(model, lr=0.02, momentum=0.9, weight_decay=1e-4)
    tr = GossipTrainer(model, opt, amp_dtype=None, warmup_iters=1, accumulation_steps=2)
    seen = []
    real = net.stochastic_depth.draw

    def spy(n, device):
        out = real(n, device)
        seen.append(out)
        return out
    net.stochastic_depth.draw = spy
    for s in range(3):
        tr.step(*_data(16, 50 + s))
    tr.finish()
    sd = net.stochastic_depth
    assert sd.draws == 6                                      # two micro-batches per step, replays included
    # eager step: two draws of 8 rows with consecutive draw indices (their own masks)
    assert len(seen) >= 4 and seen[0].shape == (8, 8)
    assert not torch.equal(seen[0].cpu(), seen[1].cpu())


@pytest.mark.parametrize('twin', [False, True], ids=['fp32', 'bf16-twin'])
def test_update_bn_and_evaluate_do_not_drop(twin, deterministic_cudnn):
    results = []
    for rate in (0.0, 0.2):
        tr = _sd_trainer('resnet18', twin, True, rate=rate)      # (the same seed: the same weights)
        sd = tr.model.module.stochastic_depth
        batches = [_data(16, 60), _data(16, 61)]
        assert tr.update_bn(batches) == 2
        stats = [b.clone() for b in tr.model.module.buffers()]
        r = tr.evaluate([_data(16, 62), _data(7, 63)])
        if sd is not None:
            assert sd.draws == 0
        results.append((stats, r, tr.model.arena.flat.clone()))
    (s0, r0, w0), (s1, r1, w1) = results
    assert torch.equal(w0, w1)
    assert all(torch.equal(a, b) for a, b in zip(s0, s1))
    assert r0[1:] == r1[1:]
    assert abs(r0.loss - r1.loss) <= 1e-6 * abs(r0.loss)     # (the loss sum uses float atomics)
