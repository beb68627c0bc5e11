"""Gradient accumulation on the GPU: the ``grad_accumulate`` kernel (csrc/accum_kernels.cu) bit for bit
against ``dst.add_(src.float())``, and ``GossipTrainer(accumulation_steps=k)``:

* exact: with ``lr = momentum = weight_decay = 0`` the step leaves ``momentum_flat == g^`` exactly
  (``fmaf(0, x, gv)`` and ``fmaf(0, m, d)`` are exact), so k = 2 on [A; B] must give
  ``fp32(fp32(m_A + m_B) * 0.5)`` bit for bit, m_A and m_B from k = 1 steps on A and on B -- on a small
  model whose forward/backward the test first shows to be reproducible run to run;
* a small ResNet within a stated fp32 / TF32 tolerance, and no foreign-layout fallback on ResNet-50;
* loop-back gossip (SGP, Overlap-SGP with the TMA and the copy-engine gather) against world 1;
* BatchMix and the metrics row; the launch count and the peak memory."""
import functools
import gc
import math

import pytest
import torch
import torch.nn as nn

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops import batch_mix as bm
from stochastic_gradient_push_b200.ops import native

from test_gdp_loopback_gpu import _in_threads

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)
BF16 = torch.bfloat16


def _C():
    return native.load()


# ---------------------------------------------------------------------------------------------------- #
# the kernel
# ---------------------------------------------------------------------------------------------------- #
def _pairs(dtype, gen):
    """(dst, src) pairs: numels 1, 3, 64, 4099 and 1 << 20, a 16-byte-misaligned src view, a misaligned
    dst view, a channels_last pair, a 1x1 weight pair and 60 tiny segments"""
    def rnd(n, dt):
        return (torch.randn(n, generator=gen, device=DEV) * 3).to(dt)
    pairs = [(rnd(n, torch.float32), rnd(n, dtype)) for n in (1, 3, 64, 4099, 1 << 20)]
    big = rnd(5000, dtype)
    pairs.append((rnd(4097, torch.float32), big[1:4098]))                   # src 2 or 4 bytes off
    dbig = rnd(5000, torch.float32)
    pairs.append((dbig[3:4099], rnd(4096, dtype)))                         # dst 12 bytes off
    cl = rnd(2 * 16 * 5 * 7, torch.float32).view(2, 16, 5, 7).contiguous(memory_format=torch.channels_last)
    pairs.append((cl, rnd(cl.numel(), dtype).view(2, 16, 5, 7).contiguous(memory_format=torch.channels_last)))
    # a 1x1 conv weight: contiguous dst, channels_last-strided src -- only the size-1 dims' strides differ
    w = rnd(64 * 32, torch.float32).view(64, 32, 1, 1)
    pairs.append((w, rnd(w.numel(), dtype).as_strided((64, 32, 1, 1), (32, 1, 2048, 2048))))
    assert pairs[-1][0].stride() != pairs[-1][1].stride()
    for i in range(60):
        n = 1 + (i * 7) % 45
        pairs.append((rnd(n, torch.float32), rnd(n, dtype)))
    return pairs


@pytest.mark.parametrize('dtype', [torch.float32, BF16], ids=['fp32', 'bf16'])
def test_kernel_is_bit_identical_to_add(dtype):
    pairs = _pairs(dtype, torch.Generator(device=DEV).manual_seed(1))
    assert pairs[5][1].data_ptr() % 16 != 0 and pairs[6][0].data_ptr() % 16 != 0
    want = [d.clone().add_(s.float()) for d, s in pairs]
    c0 = _C().launch_count()
    _C().grad_accumulate([d for d, _ in pairs], [s for _, s in pairs])
    assert _C().launch_count() - c0 == 1
    torch.cuda.synchronize()
    for i, ((d, _), w) in enumerate(zip(pairs, want)):
        assert torch.equal(d.view(torch.int32), w.view(torch.int32)), i
    # a zero dst receives exactly the (widened) source
    for d, s in pairs[:5]:
        d.zero_()
    _C().grad_accumulate([d for d, _ in pairs[:5]], [s for _, s in pairs[:5]])
    torch.cuda.synchronize()
    for d, s in pairs[:5]:
        assert torch.equal(d, s.float())


def test_bytes_around_views_are_untouched():
    g = torch.Generator(device=DEV).manual_seed(4)
    for dtype in (torch.float32, BF16):
        dbig = torch.randn(5000, generator=g, device=DEV)
        sbig = torch.randn(5000, generator=g, device=DEV).to(dtype)
        before = dbig.clone()
        _C().grad_accumulate([dbig[3:4102]], [sbig[1:4100]])
        torch.cuda.synchronize()
        assert torch.equal(dbig[:3], before[:3]) and torch.equal(dbig[4102:], before[4102:])
        assert torch.equal(dbig[3:4102], before[3:4102] + sbig[1:4100].float())


def test_a_list_longer_than_one_table_is_split():
    per = _C().ACCUM_MAX_SEGS
    n = 2 * per + 5
    g = torch.Generator(device=DEV).manual_seed(2)
    dst = [torch.randn(1 + i % 9, generator=g, device=DEV) for i in range(n)]
    src = [torch.randn(d.numel(), generator=g, device=DEV).to(BF16 if i % 2 else torch.float32)
           for i, d in enumerate(dst)]
    want = [d.clone().add_(s.float()) for d, s in zip(dst, src)]
    c0 = _C().launch_count()
    _C().grad_accumulate(dst, src)
    assert _C().launch_count() - c0 == 3
    torch.cuda.synchronize()
    assert all(torch.equal(d, w) for d, w in zip(dst, want))


def test_an_empty_list_launches_nothing():
    c0 = _C().launch_count()
    _C().grad_accumulate([], [])
    empty = torch.empty(0, device=DEV)
    _C().grad_accumulate([empty], [empty.clone()])           # nothing to add either
    assert _C().launch_count() == c0


def test_inputs_are_validated():
    a = torch.zeros(8, device=DEV)
    bad = [
        ([a], [a.clone(), a.clone()]),                                   # list lengths
        ([a.half()], [a.clone()]),                                       # dst dtype
        ([a], [a.clone().half()]),                                       # src dtype
        ([a], [torch.zeros(9, device=DEV)]),                             # numel
        ([a], [torch.zeros(8)]),                                         # device
        ([torch.zeros(4, 2, device=DEV)], [torch.zeros(2, 4, device=DEV).t()]),   # strides
        ([torch.zeros(16, device=DEV)[::2]], [a.clone()]),              # not dense
        ([a], [a]),                                                      # overlap
    ]
    for dst, src in bad:
        with pytest.raises(RuntimeError, match='grad_accumulate'):
            _C().grad_accumulate(dst, src)


def test_captured_launch_replays_on_new_data():
    g = torch.Generator(device=DEV).manual_seed(3)
    dst = [torch.zeros(n, device=DEV) for n in (5, 4099, 70000)]
    src = [torch.zeros(n, device=DEV, dtype=BF16 if n == 4099 else torch.float32) for n in (5, 4099, 70000)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        _C().grad_accumulate(dst, src)
    for _ in range(3):
        for d, x in zip(dst, src):
            d.copy_(torch.randn(d.shape, generator=g, device=DEV))
            x.copy_(torch.randn(x.shape, generator=g, device=DEV))
        want = [d.clone().add_(x.float()) for d, x in zip(dst, src)]
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(d, w) for d, w in zip(dst, want))


# ---------------------------------------------------------------------------------------------------- #
# trainer, exact
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


def _trainer(net_fn, k, use_graph=False, twin=False, world=None, rank=0, seed=11, overlap=False, dma=True,
             name='', batch_mix=None, ema_decay=None, **opt_kw):
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
    if overlap and not dma:
        model.engine._gather_dma_pref = False               # the TMA gather (see test_gdp_loopback_gpu)
        model.engine._refresh_in_peers()
    opt_kw = dict(dict(lr=0.0, momentum=0.0, weight_decay=0.0), **opt_kw)
    opt = FusedGossipSGD(model, **opt_kw)
    ema = None
    if ema_decay is not None:
        from stochastic_gradient_push_b200.ops.model_ema import ModelEma
        ema = ModelEma(model, decay=ema_decay)
    return GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=use_graph,
                         warmup_iters=1 if world is None else 10 ** 6, accumulation_steps=k,
                         batch_mix=batch_mix, ema=ema)


def _data(rows, seed, shape=(48,), classes=10):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((rows,) + shape, generator=g).pin_memory(),
            torch.randint(0, classes, (rows,), generator=g).pin_memory())


def _cat(*batches):
    return torch.cat([b[0] for b in batches]).pin_memory(), torch.cat([b[1] for b in batches]).pin_memory()


def _step(tr, x, y):
    """one step; returns g^ (= momentum_flat with lr = momentum = weight_decay = 0)"""
    tr.step(x, y)
    tr.finish()
    return tr.opt.momentum_flat[torch.float32].clone()


def _bn(tr):
    bn = tr.model.module.bn
    return [bn.running_mean.clone(), bn.running_var.clone(), bn.num_batches_tracked.clone()]


@pytest.mark.parametrize('twin', [False, True], ids=['fp32', 'bf16-twin'])
def test_two_micro_batches_equal_two_single_steps_bit_for_bit(twin):
    A, B = _data(8, 1), _data(8, 2)
    runs = []
    for _ in range(2):                      # the model's forward/backward is reproducible run to run
        tr = _trainer(_Mlp, 1, twin=twin)
        runs.append((_step(tr, *A), _step(tr, *B), _bn(tr), tr))
    (mA, mB, bn_ref, ref), (mA2, mB2, bn2, _) = runs
    assert torch.equal(mA, mA2) and torch.equal(mB, mB2)
    assert all(torch.equal(a, b) for a, b in zip(bn_ref, bn2))
    assert not torch.equal(mA, mB) and mA.abs().max() > 0
    want = (mA + mB) * 0.5
    _step(ref, *A)
    _step(ref, *B)
    bn_ref2 = _bn(ref)                                   # after A, B, A, B
    for use_graph in (False, True):
        tr = _trainer(_Mlp, 2, use_graph=use_graph, twin=twin)
        assert torch.equal(_step(tr, *_cat(A, B)), want)                # the eager (warm-up) step
        got = _bn(tr)
        assert torch.equal(got[0], bn_ref[0]) and torch.equal(got[1], bn_ref[1])
        assert int(got[2]) == 2                                          # k forward passes
        if use_graph:
            assert torch.equal(_step(tr, *_cat(A, B)), want)            # captured and replayed
            assert tr.graph is not None
            got = _bn(tr)
            assert all(torch.equal(a, b) for a, b in zip(got, bn_ref2))
            assert int(got[2]) == 4
        assert tr.accum_fallbacks == 0
        assert float(tr.opt.grad_scale) == 1.0


# ---------------------------------------------------------------------------------------------------- #
# trainer, ResNet
# ---------------------------------------------------------------------------------------------------- #
def _resnet18():
    from stochastic_gradient_push_b200 import models
    return models.resnet18(num_classes=10)


@pytest.mark.parametrize('k', [2, 4])
def test_resnet_micro_batches_match_single_steps(k):
    m = 8
    micro = [_data(m, 40 + j, shape=(3, 64, 64)) for j in range(k)]
    ref = _trainer(_resnet18, 1)
    want = torch.stack([_step(ref, *b).double() for b in micro]).mean(0)
    tr = _trainer(_resnet18, k, use_graph=True)
    for _ in range(2):                                  # eager, then captured and replayed
        got = _step(tr, *_cat(*micro)).double()
        # the two differ only in the order of the float atomics inside the BatchNorm and weight-gradient
        # reductions: an fp32 / TF32 tolerance relative to the largest gradient element
        scale = float(want.abs().max())
        torch.testing.assert_close(got, want, rtol=1e-3, atol=1e-4 * scale)
    assert tr.graph is not None
    assert tr.accum_fallbacks == 0


class _CountAccum(object):
    """engine.C with grad_accumulate calls counted"""

    def __init__(self, C):
        self._C = C
        self.calls = 0

    def __getattr__(self, name):
        return getattr(self._C, name)

    def grad_accumulate(self, dst, src):
        self.calls += 1
        return self._C.grad_accumulate(dst, src)


@pytest.mark.parametrize('twin', [False, True], ids=['fp32', 'bf16-twin'])
def test_resnet50_has_no_foreign_layout_fallback_and_launches_are_linear_in_k(twin):
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.ops.fused_loss import FusedCrossEntropyWithAccuracy
    m, launches, per_pass = 4, {}, None
    for k in (1, 2, 4):
        tr = _trainer(lambda: models.resnet50(num_classes=10), k, use_graph=True, twin=twin)
        tr.engine.C = counter = _CountAccum(tr.engine.C)
        x, y = _data(m * k, 7, shape=(3, 64, 64))
        for _ in range(3):                              # eager, capture + replay, replay
            tr.step(x, y)
        tr.finish()
        assert tr.graph is not None
        assert counter.calls == 2 * (k - 1)            # the eager step and the capture; replays call nothing
        assert tr.accum_fallbacks == 0
        assert torch.isfinite(tr.opt.momentum_flat[torch.float32]).all()
        launches[k] = tr.own_launches_per_step
        if k == 1:
            # own launches of one plain forward / loss / backward of the module the step runs, at the
            # micro-batch shape (the trainer is not stepped again)
            net, crit = tr.model.compute_module, FusedCrossEntropyWithAccuracy()
            xd = tr.static_in.clone()
            yd = y.to(DEV)
            crit(net(xd), yd).backward()               # warm-up
            torch.cuda.synchronize()
            c0 = _C().launch_count()
            crit(net(xd), yd).backward()
            per_pass = _C().launch_count() - c0
        del tr
    print('own launches per step (k: count):', launches, 'per forward/backward:', per_pass)
    for k in (2, 4):
        assert launches[k] == launches[1] + (k - 1) * (per_pass + 1)      # one accumulation launch each


def test_resnet50_batch256_k1_launch_count_is_unchanged():
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    torch.manual_seed(1)
    net = models.resnet50()
    models.init_imagenet_in_1hr(net)
    net = net.to(DEV).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                               verbose=False, heartbeat_timeout=60)
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, weight_decay=1e-4, nesterov=True)
    trainer = GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=True, warmup_iters=1, accumulation_steps=1)
    x, y = _data(256, 1234, shape=(3, 224, 224), classes=1000)
    for _ in range(3):
        trainer.step(x, y)
    torch.cuda.synchronize()
    assert trainer.graph is not None and trainer._micro is None and trainer._micro_metrics is None
    assert trainer.own_launches_per_step == 326
    assert torch.isfinite(model.arena.flat).all()


def test_peak_memory_grows_less_with_accumulation():
    """ResNet-18 at 112 px, m = 32: doubling the step batch by k = 2 costs less than half of what
    doubling the micro-batch costs (the activations of one micro-batch at a time)"""
    from stochastic_gradient_push_b200 import models

    def peak(rows, k):
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        tr = _trainer(models.resnet18, k, use_graph=True)
        x, y = _data(rows, 3, shape=(3, 112, 112), classes=1000)
        for _ in range(2):
            tr.step(x, y)
        tr.finish()
        assert tr.graph is not None
        out = torch.cuda.max_memory_allocated() - base
        del tr
        return out
    m = 32
    p11, p21, p22 = peak(m, 1), peak(2 * m, 1), peak(2 * m, 2)
    print('peak MiB: (m, 1) %.1f, (2m, 1) %.1f, (2m, 2) %.1f' % (p11 / 2 ** 20, p21 / 2 ** 20, p22 / 2 ** 20))
    assert p21 > p11
    assert p22 - p11 < 0.5 * (p21 - p11)


# ---------------------------------------------------------------------------------------------------- #
# gossip
# ---------------------------------------------------------------------------------------------------- #
@pytest.mark.parametrize('algo', ['sgp', 'osgp-tma', 'osgp-dma'])
def test_loopback_ranks_match_their_world1_reference(algo):
    """identical parameters on both ranks and lr = 0: mixing keeps them identical, so each rank's g^
    equals the one world 1 computes on the same step batch; clipping on (a threshold it never reaches)
    gives optimizer.grad_norm = |g^|"""
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    overlap, dma = algo.startswith('osgp'), algo.endswith('dma')
    use_graph = algo != 'osgp-dma'                      # the copy-engine gather runs eager here
    k, steps = 2, 2
    batches = [_data(16, 60 + r) for r in range(2)]
    refs = [_step(_trainer(_Mlp, k), *b) for b in batches]
    lw = LocalWorld(2)
    trainers = [_trainer(_Mlp, k, use_graph=use_graph, world=lw, rank=r, overlap=overlap, dma=dma,
                         name='accum_' + algo.replace('-', '_'), max_grad_norm=1e6) for r in range(2)]
    x0 = trainers[0].model.arena.flat.clone()
    assert torch.equal(x0, trainers[1].model.arena.flat)
    for s in range(steps):
        if use_graph and s == 1:
            for tr in trainers:                         # every capture before any replay
                with torch.cuda.stream(tr.stream):
                    tr._capture()
        _in_threads([functools.partial(trainers[r].step, *batches[r]) for r in range(2)])
        torch.cuda.synchronize()
        if not overlap:                                 # (Overlap-SGP defers the SGD to the next publish)
            for r, tr in enumerate(trainers):
                assert torch.equal(tr.opt.momentum_flat[torch.float32], refs[r]), (s, r)
    for tr in trainers:
        tr.finish()
        assert (tr.graph is not None) == use_graph
        assert torch.equal(tr.model.arena.flat, x0)     # the premise: lr = 0 and exact mixing
    for r, tr in enumerate(trainers):
        ghat = tr.opt.momentum_flat[torch.float32]
        assert torch.equal(ghat, refs[r]), r
        norm = math.sqrt(float(ghat.double().square().sum()))
        assert float(tr.opt.grad_norm) == pytest.approx(norm, rel=2.0 ** -23)     # (an fp32 value)
        assert tr.accum_fallbacks == 0


# ---------------------------------------------------------------------------------------------------- #
# mixing and metrics
# ---------------------------------------------------------------------------------------------------- #
@pytest.mark.parametrize('alphas', [(0.4, 0.0), (0.0, 1.0)], ids=['mixup', 'cutmix'])
@pytest.mark.parametrize('use_graph', [False, True], ids=['eager', 'graph'])
def test_batch_mix_slices_and_metrics_row(alphas, use_graph):
    from stochastic_gradient_push_b200 import models
    k, m = 4, 6
    mix = bm.BatchMix(*alphas, seed=5)
    tr = _trainer(models.TinyConvNet, k, use_graph=use_graph, batch_mix=mix, ema_decay=0.9,
                  lr=0.05, momentum=0.9)
    for s in range(3):
        mix.iteration = 100 + s
        x, y = _data(k * m, 20 + s, shape=(3, 16, 16))
        slot = tr.step(x, y)
        tr.stream.synchronize()
        assert mix.iteration == 101 + s                 # one draw per step
        p = mix.sample(16, 16, itr=100 + s)
        assert mix.last == p and p.mode != bm.NO_MIX
        for j in range(k):
            sl = slice(j * m, (j + 1) * m)
            assert torch.equal(tr.static_in[sl], bm.reference_batch_mix(x[sl].to(DEV), p)), (s, j)
        micro = tr._micro_metrics.clone()
        assert torch.equal(tr.static_metrics, micro.mean(0))
        assert torch.equal(tr.metrics_ring[slot], micro.mean(0).cpu())
        # the last micro-batch's logits are static_out, its metrics the last row: the two-target loss of
        # that micro-batch alone, each row paired with its flip inside the micro-batch
        loss, p1, p5 = bm.reference_mixed_loss_and_accuracy(tr.static_out, y[-m:].to(DEV), p.lam)
        assert tr.static_out.shape[0] == m
        torch.testing.assert_close(micro[-1, 0], loss.float(), rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(micro[-1, 1:], torch.stack([p1, p5]).float(), rtol=0, atol=1e-3)
    tr.finish()
    assert (tr.graph is not None) == use_graph
    assert tr.ema.num_updates == 3                      # once per step, not per micro-batch
