"""GossipTrainer.evaluate on the GPU:

* the eval-BN epilogue of the 1x1-conv GEMM (MODES 4 / 5, ``C.conv1x1_bn_eval``) against conv ->
  eval batch_norm -> (+R) -> ReLU in fp64 on the same (TF32-truncated / bf16) operands, on every ResNet-50
  1x1 shape at batch 8 and 256 and on forced small grids (many row tiles per CTA);
* the accumulate kernel (``xent_eval_accumulate``): hit and row counts equal torch's topk exactly on
  tie-free logits, over batches with a partial one and invalid targets; the loss sum to 1e-6;
* end to end on ResNet-50: ``eval_out`` against an eager eval forward, counts against topk;
* no side effects on training (local, loop-back SGP and OSGP), and parameter swaps by ``ema.applied()``
  without a new capture."""
import functools

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops import fused_loss, native
from stochastic_gradient_push_b200.ops.fused_bn import FusedBatchNormAct2d, conv_bn_act

from test_conv1x1_scale_gpu import GRID_SHAPES, RESNET50_SHAPES, ROWS, _tf32
from test_gdp_loopback_gpu import _in_threads

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
BF16 = torch.bfloat16
DTYPES = {'f32': torch.float32, 'bf16': BF16}


# ---------------------------------------------------------------------------------------------------- #
# the GEMM
# ---------------------------------------------------------------------------------------------------- #
def _bn_params(N, g):
    gamma = torch.rand(N, device=DEV, generator=g) + 0.5
    beta = torch.randn(N, device=DEV, generator=g) * 0.2
    mean = torch.randn(N, device=DEV, generator=g) * 0.3
    var = torch.rand(N, device=DEV, generator=g) + 0.5
    return gamma, beta, mean, var


def _check_eval_gemm(C, M, N, K, dtype, relu, res, num_sms=0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, K, device=DEV, generator=g).to(dtype)
    w = (torch.randn(N, K, device=DEV, generator=g) / K ** 0.5).to(dtype)
    r = torch.randn(M, N, device=DEV, generator=g).to(dtype) if res else None
    gamma, beta, mean, var = _bn_params(N, g)
    y = C.conv1x1_bn_eval(x, w, gamma, beta, mean, var, 1e-5, relu, r, num_sms=num_sms)
    assert y.shape == (M, N) and y.dtype == dtype
    f32 = dtype == torch.float32
    xo, wo = (_tf32(x), _tf32(w)) if f32 else (x, w)
    # conv -> F.batch_norm(training=False) -> (+R) -> ReLU, in fp64 on the operands the tensor cores see
    rtol, atol = (1e-3, 1e-3) if f32 else (2.0 ** -7, 1e-2)
    wd = wo.double().t()
    for i in range(0, M, ROWS):
        z = xo[i:i + ROWS].double() @ wd
        want = F.batch_norm(z, mean.double(), var.double(), gamma.double(), beta.double(), False, 0.1, 1e-5)
        if res:
            want = want + r[i:i + ROWS].double()
        if relu:
            want = torch.relu(want)
        err = (y[i:i + ROWS].double() - want).abs()
        assert bool((err <= atol + rtol * want.abs()).all()), (M, N, K, dtype, relu, res, i, err.max().item())
    return y


@pytest.mark.parametrize('dtype', ['f32', 'bf16'])
@pytest.mark.parametrize('batch', [8, 256])
def test_eval_gemm_matches_conv_bn_on_resnet50_shapes(dtype, batch):
    C = native.load()
    for (M, N, K) in RESNET50_SHAPES:
        M = M // 256 * batch
        for relu, res in ((True, False), (False, False), (True, True)):
            _check_eval_gemm(C, M, N, K, DTYPES[dtype], relu, res, seed=M + N + K)


@pytest.mark.parametrize('dtype', ['f32', 'bf16'])
@pytest.mark.parametrize('sms', [1, 3, 8])
def test_eval_gemm_on_small_grids(dtype, sms):
    """a few CTAs: every CTA walks dozens of row tiles (ring wrap-around, recycled slabs, R prefetch)"""
    C = native.load()
    for (M, N, K) in GRID_SHAPES + [(8 * 56 * 56, 256, 64), (8 * 7 * 7, 2048, 512)]:
        for relu, res in ((True, False), (True, True)):
            y = _check_eval_gemm(C, M, N, K, DTYPES[dtype], relu, res, num_sms=sms, seed=3)
            y0 = _check_eval_gemm(C, M, N, K, DTYPES[dtype], relu, res, num_sms=0, seed=3)
            p, p0 = (C.conv1x1_plan(M, N, K, s or torch.cuda.get_device_properties(0).multi_processor_count,
                                    res, dtype == 'f32') for s in (sms, 0))
            if p['block_n'] == p0['block_n']:
                assert torch.equal(y, y0)                  # the grid does not change a single output


def test_eval_gemm_follows_in_place_parameter_changes_in_a_graph():
    C = native.load()
    M, N, K = 4096, 256, 64
    g = torch.Generator(device=DEV).manual_seed(5)
    x = torch.randn(M, K, device=DEV, generator=g)
    w = torch.randn(N, K, device=DEV, generator=g) / 8
    gamma, beta, mean, var = _bn_params(N, g)
    C.conv1x1_bn_eval(x, w, gamma, beta, mean, var, 1e-5, True)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = C.conv1x1_bn_eval(x, w, gamma, beta, mean, var, 1e-5, True)
    for t in (gamma, beta, mean, var):
        t.mul_(1.5)
    graph.replay()
    want = C.conv1x1_bn_eval(x, w, gamma, beta, mean, var, 1e-5, True)
    assert torch.equal(y, want)


# ---------------------------------------------------------------------------------------------------- #
# the accumulate kernel
# ---------------------------------------------------------------------------------------------------- #
def _tie_free_logits(B, Cn, dtype, g):
    """each row a permutation of k / 8, k < Cn: distinct and exact in bf16 for Cn <= 256"""
    vals = torch.argsort(torch.rand(B, Cn, device=DEV, generator=g), dim=1).float() / 8 - Cn / 16
    return vals.to(dtype)


@pytest.mark.parametrize('dtype,classes', [('f32', 1000), ('bf16', 200), ('f32', 3)])
def test_accumulate_counts_equal_topk_over_batches(dtype, classes):
    g = torch.Generator(device=DEV).manual_seed(9)
    acc = fused_loss.eval_accumulator(DEV)
    loss_sum, hits1, hits5, rows = 0.0, 0, 0, 0
    for B in (256, 256, 77):
        z = _tie_free_logits(B, classes, DTYPES[dtype], g)
        t = torch.randint(0, classes, (B,), device=DEV, generator=g)
        t[::11] = -1
        t[5::13] = classes
        t[7::29] = -100
        fused_loss.eval_accumulate(z, t, acc)
        ok = (t >= 0) & (t < classes)
        zf, tv = z[ok].double(), t[ok]
        k = min(5, classes)
        top = zf.topk(k, 1, True, True).indices
        hits1 += int((top[:, 0] == tv).sum())
        hits5 += int((top == tv[:, None]).any(1).sum())
        rows += int(ok.sum())
        loss_sum += float(F.cross_entropy(zf, tv, reduction='sum'))
    a = acc.cpu()
    assert (int(a[1]), int(a[2]), int(a[3])) == (hits1, hits5, rows)
    assert float(a[:1].view(torch.float64)) == pytest.approx(loss_sum, rel=1e-6)


# ---------------------------------------------------------------------------------------------------- #
# the trainer
# ---------------------------------------------------------------------------------------------------- #
class _Block(nn.Module):
    """two 1x1 conv + BatchNorm layers, the second with the block input as residual, and a classifier:
    both eval GEMM modes, and a training step that is reproducible run to run (no float atomics in our
    kernels here; cuDNN is asked for deterministic algorithms)"""

    def __init__(self, C=64, classes=10):
        super().__init__()
        self.conv1, self.bn1 = nn.Conv2d(C, C, 1, bias=False), FusedBatchNormAct2d(C)
        self.conv2, self.bn2 = nn.Conv2d(C, C, 1, bias=False), FusedBatchNormAct2d(C)
        self.fc = nn.Linear(C, classes)

    def forward(self, x):
        y = conv_bn_act(self.conv1, self.bn1, x, relu=True)
        y = conv_bn_act(self.conv2, self.bn2, y, residual=x, relu=True)
        return self.fc(y.mean((2, 3)))


def _resnet50(classes=10):
    from stochastic_gradient_push_b200 import models
    return models.resnet50(num_classes=classes)


def _trainer(twin=False, world=None, rank=0, overlap=False, use_graph=True, warmup=1, name='', ema_decay=None,
             seed=11, lr=0.05, net_fn=_resnet50):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    torch.manual_seed(seed)
    net = net_fn().to(DEV).to(memory_format=torch.channels_last)
    n = 1 if world is None else 2
    kw = dict(symmetric_world=world.view(rank), transport='nvlink', grid=4, symmetric_name=name) if world else {}
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(rank, n), rank=rank,
                               world_size=n, overlap=overlap, heartbeat_timeout=20,
                               compute_dtype=BF16 if twin else None, **kw)
    if overlap:
        model.engine._gather_dma_pref = False               # the TMA gather (see test_gdp_loopback_gpu)
        model.engine._refresh_in_peers()
    opt = FusedGossipSGD(model, lr=lr, momentum=0.9, weight_decay=1e-4)
    ema = None
    if ema_decay is not None:
        from stochastic_gradient_push_b200.ops.model_ema import ModelEma
        ema = ModelEma(model, decay=ema_decay)
    return GossipTrainer(model, opt, amp_dtype=BF16 if twin else None, use_cuda_graph=use_graph,
                         warmup_iters=warmup, ema=ema)


def _data(rows, seed, hw=32, classes=10, channels=3):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(rows, channels, hw, hw, generator=g).pin_memory(),
            torch.randint(0, classes, (rows,), generator=g).pin_memory())


def _state(tr):
    net = tr.model.module
    bufs = [b.clone() for b in net.buffers()]
    return [tr.model.arena.flat.clone(), tr.opt.momentum_flat[torch.float32].clone()] + bufs


def _equal_states(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), i


@pytest.mark.parametrize('twin', [False, True], ids=['fp32', 'bf16-twin'])
def test_evaluate_matches_an_eager_eval_forward(twin):
    tr = _trainer(twin=twin, lr=0.0)
    for s in range(3):                                  # running statistics from real batches
        tr.step(*_data(16, s))
    tr.finish()
    val = [_data(16, 10), _data(16, 11), _data(5, 12)]
    r = tr.evaluate(val)
    assert r.count == 37 and 0 <= r.prec1 <= r.prec5 <= 100 and r.loss > 0
    assert tr.model.module.training                     # the previous mode is back
    net = tr.model._twin[0] if twin else tr.model.module
    net.eval()
    with torch.no_grad():
        x = val[-1][0].to(DEV).to(BF16 if twin else torch.float32).contiguous(memory_format=torch.channels_last)
        want = net(x).float()
    net.train()
    got = tr.eval_out.float()
    assert got.shape == want.shape
    scale = float(want.abs().max())
    tol = (5e-2 if twin else 1e-2) * max(scale, 1.0)
    torch.testing.assert_close(got, want, rtol=0, atol=tol)
    assert tr.eval_launches_per_batch is not None and tr.eval_launches_per_batch > 10
    # one batch: the counts are torch's topk on eval_out (the kernel ranks ties below the target)
    one = tr.evaluate([val[0]])
    z, t = tr.eval_out.double(), val[0][1].to(DEV)
    top = z.topk(5, 1, True, True).indices
    zt = z.gather(1, t[:, None])
    if not bool(((z == zt).sum(1) > 1).any()):
        assert round(one.prec1 * 16 / 100) == int((top[:, 0] == t).sum())
        assert round(one.prec5 * 16 / 100) == int((top == t[:, None]).any(1).sum())
    assert one.loss == pytest.approx(float(F.cross_entropy(z, t)), rel=1e-5)


def _same_metrics(a, b):
    """[loss, prec@1, prec@5] rows: the loss kernel sums its rows with shared-memory float atomics, so
    the rows agree to rounding, not bit for bit, even between two runs of the same training"""
    torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-4)


@pytest.fixture
def deterministic_cudnn():
    prev = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = prev


def _block_data(rows, seed):
    return _data(rows, seed, hw=8, channels=64)


def test_evaluate_has_no_side_effects_local(deterministic_cudnn):
    """train k -> evaluate -> train k equals 2k steps, bit for bit (captured training and evaluation
    graphs in one pool)"""
    k = 3
    batches = [_block_data(16, 20 + s) for s in range(2 * k)]
    val = [_block_data(16, 40), _block_data(7, 41)]
    refs = []
    for _ in range(2):                                  # the premise: training is reproducible
        ref = _trainer(net_fn=_Block)
        for b in batches:
            ref.step(*b)
        ref.finish()
        refs.append(ref)
    _equal_states(_state(refs[0]), _state(refs[1]))
    ref = refs[0]
    tr = _trainer(net_fn=_Block)
    for b in batches[:k]:
        tr.step(*b)
    assert tr.graph is not None
    torch.cuda.synchronize()                            # (the step ran on the trainer's stream)
    before = tr.static_out.clone()
    r = tr.evaluate(val)
    assert r.count == 23 and tr.eval_launches_per_batch >= 3
    assert torch.equal(tr.static_out, before)
    for b in batches[k:]:
        tr.step(*b)
    tr.finish()
    assert tr.engine.steps == ref.engine.steps
    _equal_states(_state(tr), _state(ref))
    _same_metrics(tr.metrics_ring[:2 * k], ref.metrics_ring[:2 * k])


@pytest.mark.parametrize('algo', ['sgp', 'osgp'])
def test_evaluate_has_no_side_effects_loopback(algo, deterministic_cudnn):
    """2 loop-back ranks, eager steps, captured evaluation; OSGP against a finish()-only run"""
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    overlap = algo == 'osgp'
    k = 2
    data = [[_block_data(8, 60 + 10 * r + s) for s in range(2 * k)] for r in range(2)]
    val = [_block_data(8, 90), _block_data(3, 91)]

    def run(evaluate, tag):
        lw = LocalWorld(2)
        trs = [_trainer(world=lw, rank=r, overlap=overlap, warmup=10 ** 6, name='ev_%s_%s' % (algo, tag),
                        net_fn=_Block) for r in range(2)]
        for s in range(2 * k):
            if s == k:
                torch.cuda.synchronize()
                for tr in trs:
                    tr.evaluate(val) if evaluate else tr.finish()
            _in_threads([functools.partial(trs[r].step, *data[r][s]) for r in range(2)])
            torch.cuda.synchronize()
        for tr in trs:
            tr.finish()
        return [(_state(tr), tr.metrics_ring[:2 * k].clone(), tr.engine.steps) for tr in trs]

    plain = run(False, 'b')
    for (sa, ma, na), (sb, mb, nb) in zip(run(False, 'c'), plain):      # the premise: reproducible
        _equal_states(sa, sb)
        _same_metrics(ma, mb)
        assert na == nb
    for (sa, ma, na), (sb, mb, nb) in zip(run(True, 'a'), plain):
        _equal_states(sa, sb)
        _same_metrics(ma, mb)
        assert na == nb


def test_evaluate_inside_ema_applied_follows_the_swap_without_recapture():
    tr = _trainer(ema_decay=0.5)
    for s in range(4):
        tr.step(*_data(16, 70 + s))
    val = [_data(16, 80), _data(16, 81), _data(5, 82)]
    plain = tr.evaluate(val)
    graphs = {k: s.graph for k, s in tr._eval_slots.items()}
    assert len(graphs) == 2 and all(g is not None for g in graphs.values())
    with tr.ema.applied():
        swapped = tr.evaluate(val)
    assert {k: s.graph for k, s in tr._eval_slots.items()} == graphs      # nothing captured again
    again = tr.evaluate(val)
    assert again.count == plain.count and (again.prec1, again.prec5) == (plain.prec1, plain.prec5)
    assert again.loss == pytest.approx(plain.loss, rel=1e-12)
    # a model loaded with the EMA state, evaluated by a trainer of its own
    ref = _trainer(lr=0.0, seed=12)
    ref.model.module.load_state_dict(tr.ema.state_dict()['state_dict'], strict=False)
    want = ref.evaluate(val)
    assert (swapped.count, swapped.prec1, swapped.prec5) == (want.count, want.prec1, want.prec5)
    assert swapped.loss == pytest.approx(want.loss, rel=1e-6)
    assert swapped != plain

