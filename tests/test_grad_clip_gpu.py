"""Gradient-norm clipping and non-finite step skipping on the kernel plane (``SGP_F_CLIP``): N virtual
ranks on one GPU (``LocalWorld`` loop-back) against a simulation that takes the global norm in fp64
and then follows the kernels' fmaf order -- the full step (pipe and register-staged, fp32 and bf16
messages), the overlap publish / gather (DMA and TMA) / local flush --, the norm against
``torch.linalg.vector_norm`` and bit-identical across grids and runs, ``coef == 1`` bit-identical to
an engine without clipping, LARS on the clipped gradient, the bf16 gradient + fp32 g2 of the compute
twin, the skip of a NaN gradient, a graph-captured trainer against eager (a threshold change after
capture, a NaN loss step) and the launch counts of a ResNet-50 step."""
import functools
import math

import pytest
import torch

import stochastic_gradient_push_b200 as sgp

from test_gdp_loopback_gpu import _in_threads
from test_lars_gpu import NUMELS, ROWS, _configure, _lars_step, _layout, _trust
from test_param_groups_gpu import _fma, _mk_world

pytestmark = pytest.mark.gpu

CHUNK = 4096
BF16 = torch.bfloat16
HYPER = (0.1, 0.9, 1e-3, True)            # lr, momentum, weight_decay, nesterov (ungrouped)


def _clip_on(engines, norm=True, skip=False):
    offs, _ = _layout()
    for e in engines:
        e.set_grad_clip(offs, NUMELS, enabled=norm, skip_nonfinite=skip)


def _set(engines, max_norm, grad_scale=1.0):
    for e in engines:
        e.set_hyper(*HYPER, grad_scale=grad_scale, max_grad_norm=max_norm)


def _norm(g):
    """fp64 2-norm of g^ over the tensors of the layout (padding excluded)"""
    offs, _ = _layout()
    return math.sqrt(sum(float(g[o:o + n].double().square().sum()) for o, n in zip(offs, NUMELS)))


def _coef(total, max_norm):
    c = max_norm / (total + 1e-6)
    return torch.tensor(1.0 if c > 1.0 else c, dtype=torch.float32)


def _sgd(x, g, m, gscale):
    """the kernels' fp32 chain: gv = g * gscale ; d = fmaf(wd, x, gv) ; m = fmaf(mu, m, d) ; x -= ..."""
    lr, mu, wd = (torch.tensor(v, dtype=torch.float32) for v in HYPER[:3])
    nest = HYPER[3]
    x, m = x.float(), m.float()
    gv = g.float() * gscale
    d = _fma(wd, x, gv)
    m = _fma(mu, m, d)
    upd = _fma(mu, m, d) if nest else m
    return _fma(-lr, upd, x).double(), m.double()


@pytest.mark.parametrize('pipe', [True, False], ids=['pipe', 'regs'])
@pytest.mark.parametrize('msg_dtype', [None, BF16], ids=['fp32', 'bf16'])
def test_mix_matches_clip_simulation(msg_dtype, pipe):
    n, numel = 4, 3 * CHUNK
    engines, tables, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, pipe, msg_dtype,
                                         name='clip_mix')
    _clip_on(engines)
    for step, max_norm in enumerate((20.0, 1e4, 5.0, 1e4)):        # clipping on steps 0 and 2
        _set(engines, max_norm)
        for e in engines:
            e.grad.normal_()
        torch.cuda.synchronize()
        zs = [e.z.double().cpu() for e in engines]
        ms = [e.momentum.double().cpu() for e in engines]
        gs = [e.grad.float().cpu() for e in engines]
        ws = [e.ps_weight for e in engines]
        for e, s in zip(engines, streams):
            with torch.cuda.stream(s):
                e.mix(sgd=True)
        torch.cuda.synchronize()
        xs, new_m = [], []
        for i, e in enumerate(engines):
            total = _norm(gs[i])
            assert float(e.grad_sumsq) == pytest.approx(total ** 2, rel=1e-12)
            assert float(e.grad_norm) == pytest.approx(total, rel=1e-6)
            coef = _coef(total, max_norm)
            assert float(e.clip_coef) == pytest.approx(float(coef), rel=1e-6)
            assert (float(e.clip_coef) < 1) == (max_norm < 100)
            x0 = zs[i].float() * torch.tensor(ws[i], dtype=torch.float32)
            x, m = _sgd(x0, gs[i], ms[i], e.clip_coef.cpu())
            xs.append(x)
            new_m.append(m)
        sent = [x.to(BF16).double() if msg_dtype is not None else x for x in xs]
        for i, e in enumerate(engines):
            t, wt = tables[i]
            row = step % t.shape[0]
            sw = float(wt[row, 0])
            acc = xs[i] - (1 - sw) * sent[i]
            wn = sw * ws[i]
            for k in range(int(t[row, 0])):
                j = int(t[row, 2 + k])
                acc = acc + float(wt[row, 1 + k]) * sent[j]
                wn += float(wt[row, 1 + k]) * ws[j]
            e.check()
            torch.testing.assert_close(e.z.double().cpu(), acc / wn, rtol=1e-4, atol=1e-5)
            torch.testing.assert_close(e.momentum.double().cpu(), new_m[i], rtol=1e-4, atol=1e-5)
            assert torch.all(e.grad == 0)
            assert abs(e.ps_weight - wn) < 1e-6


@pytest.mark.parametrize('dma', [True, False], ids=['dma', 'tma'])
def test_overlap_publish_gather_local_match_clip_simulation(dma):
    n, numel = 2, 3 * CHUNK
    engines, tables, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, True,
                                         residual=True, name='clip_osgp%d' % dma)
    _clip_on(engines)
    ms = [e.momentum.double().cpu() for e in engines]
    res, wres = [torch.zeros(numel, dtype=torch.float64) for _ in range(n)], [0.0] * n
    zs = [e.z.double().cpu() for e in engines]
    ws = [1.0] * n
    for step, max_norm in enumerate((20.0, 1e4, 10.0)):
        _set(engines, max_norm)
        for e in engines:
            e.grad.normal_()
        torch.cuda.synchronize()
        gs = [e.grad.float().cpu() for e in engines]
        for e, s in zip(engines, streams):
            with torch.cuda.stream(s):
                e.publish(sgd=True, fold=step > 0)
                e.gather(tma=True, dma=dma)
        torch.cuda.synchronize()
        xs = []
        for i, e in enumerate(engines):
            coef = _coef(_norm(gs[i]), max_norm)
            assert float(e.clip_coef) == pytest.approx(float(coef), rel=1e-6)
            x, ms[i] = _sgd((zs[i] * ws[i]).float(), gs[i], ms[i], e.clip_coef.cpu())
            xs.append((x + res[i], ws[i] + wres[i]))
        for i in range(n):
            t, wt = tables[i]
            row = step % t.shape[0]
            sw = float(wt[row, 0])
            x, w1 = xs[i]
            zs[i], ws[i] = x / w1, sw * w1
            res[i] = sum(float(wt[row, 1 + k]) * xs[int(t[row, 2 + k])][0] for k in range(int(t[row, 0])))
            wres[i] = sum(float(wt[row, 1 + k]) * xs[int(t[row, 2 + k])][1] for k in range(int(t[row, 0])))
        for i, e in enumerate(engines):
            e.check()
            torch.testing.assert_close(e.z.double().cpu(), zs[i], rtol=1e-4, atol=1e-5)
            zs[i] = e.z.double().cpu()
            ws[i] = e.ps_weight
    _set(engines, 15.0)
    for e in engines:
        e.grad.normal_()
    torch.cuda.synchronize()
    gs = [e.grad.float().cpu() for e in engines]
    for e in engines:
        e.local(sgd=True, fold=True)
    torch.cuda.synchronize()
    for i, e in enumerate(engines):
        e.check()
        coef = _coef(_norm(gs[i]), 15.0)
        assert float(coef) < 1 and float(e.clip_coef) == pytest.approx(float(coef), rel=1e-6)
        x, ms[i] = _sgd((zs[i] * ws[i]).float(), gs[i], ms[i], e.clip_coef.cpu())
        torch.testing.assert_close(e.z.double().cpu(), (x + res[i]) / (ws[i] + wres[i]), rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(e.momentum.double().cpu(), ms[i], rtol=1e-4, atol=1e-5)


def test_norm_is_exact_and_bit_identical_across_grids_and_runs():
    numel = 3 * CHUNK
    engines, _, _ = _mk_world(1, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, True, name='clip_det')
    e = engines[0]
    _clip_on(engines)
    _set(engines, 30.0, grad_scale=0.75)
    g = e.grad.clone()
    want = torch.linalg.vector_norm(torch.cat([(g[o:o + n].double() * 0.75) for o, n in zip(_layout()[0], NUMELS)]))
    seen = []
    for grid in (e.ctx.lars_grid(), e.ctx.lars_grid(), 1, 3, 7):
        e.ctx.set_lars_grid(grid)
        e.clip_update()
        torch.cuda.synchronize()
        seen.append((e.grad_sumsq.clone(), e.grad_norm.clone(), e.clip_coef.clone()))
    for s in seen[1:]:
        assert all(torch.equal(a, b) for a, b in zip(s, seen[0]))
    torch.testing.assert_close(seen[0][1].double().cpu(), want.cpu(), rtol=1e-6, atol=0)
    assert float(seen[0][2]) < 1
    assert e.ctx.lars_tiles() == sum((n + CHUNK - 1) // CHUNK for n in NUMELS)
    assert not e.lars                                   # the norm plan serves clipping alone


@pytest.mark.parametrize('pipe', [True, False], ids=['pipe', 'regs'])
@pytest.mark.parametrize('msg_dtype', [None, BF16], ids=['fp32', 'bf16'])
def test_coef_one_is_bit_identical_to_no_clipping(msg_dtype, pipe):
    n, numel = 2, 3 * CHUNK
    worlds = []
    for clip in (False, True):
        engines, _, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, pipe, msg_dtype,
                                        name='clip_one%d' % clip)
        if clip:
            _clip_on(engines, skip=True)
        _set(engines, 1e9, grad_scale=0.5)
        worlds.append((engines, streams))
    for step in range(3):
        g = [torch.randn(numel, device='cuda') for _ in range(n)]
        for engines, streams in worlds:
            for e, gr in zip(engines, g):
                e.grad.copy_(gr)
            torch.cuda.synchronize()
            for e, s in zip(engines, streams):
                with torch.cuda.stream(s):
                    e.mix(sgd=True)
            torch.cuda.synchronize()
    for a, b in zip(*(w[0] for w in worlds)):
        a.check()
        b.check()
        assert not a.grad_clip and b.grad_clip and float(b.clip_coef) == 1.0
        assert torch.equal(a.z, b.z) and torch.equal(a.momentum, b.momentum)


@pytest.mark.parametrize('max_norm', [5.0, 1e4], ids=['clipping', 'not-clipping'])
def test_lars_trust_sees_the_clipped_gradient(max_norm):
    n, numel = 2, 3 * CHUNK
    engines, tables, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, True,
                                         name='clip_lars')
    _configure(engines, numel)
    _clip_on(engines)
    for e in engines:
        e.set_hyper(0.5, 0.5, 0.5, True, groups=ROWS, max_grad_norm=max_norm)
    zs = [e.z.double().cpu() for e in engines]
    ms = [e.momentum.double().cpu() for e in engines]
    gs = [e.grad.float().cpu() for e in engines]
    for e, s in zip(engines, streams):
        with torch.cuda.stream(s):
            e.mix(sgd=True)
    torch.cuda.synchronize()
    xs = []
    for i, e in enumerate(engines):
        e.check()
        coef = _coef(_norm(gs[i]), max_norm)
        assert float(e.clip_coef) == pytest.approx(float(coef), rel=1e-6)
        x0 = zs[i].float()
        trust = _trust(x0, gs[i].double() * float(e.clip_coef), numel)
        torch.testing.assert_close(e.lars_trust.double().cpu(), trust, rtol=1e-6, atol=0)
        x, m = _lars_step(x0, gs[i] * e.clip_coef.cpu(), ms[i], numel, e.lars_trust.cpu())
        xs.append(x)
        torch.testing.assert_close(e.momentum.double().cpu(), m, rtol=1e-4, atol=1e-5)
    for i, e in enumerate(engines):
        t, wt = tables[i]
        acc = float(wt[0, 0]) * xs[i]
        for k in range(int(t[0, 0])):
            acc = acc + float(wt[0, 1 + k]) * xs[int(t[0, 2 + k])]
        torch.testing.assert_close(e.z.double().cpu(), acc, rtol=1e-4, atol=1e-5)


def test_bf16_gradient_plus_fp32_g2_norm():
    n, numel = 2, 3 * CHUNK
    engines, _, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, True, name='clip_twin')
    dev = engines[0].device
    lo = [torch.randn(numel, device=dev).to(BF16) for _ in range(n)]
    hi = [torch.randn(numel, device=dev) for _ in range(n)]
    for e, a, b in zip(engines, lo, hi):
        e.set_sgd_buffers(a, e.momentum, grad2=b)
    _clip_on(engines)
    _set(engines, 10.0, grad_scale=0.25)
    gs = [((a.float() + b) * 0.25).cpu() for a, b in zip(lo, hi)]     # g^ as phase 1 forms it
    for e, s in zip(engines, streams):
        with torch.cuda.stream(s):
            e.mix(sgd=True, zero_grad=False)
    torch.cuda.synchronize()
    for i, e in enumerate(engines):
        e.check()
        assert float(e.grad_norm) == pytest.approx(_norm(gs[i]), rel=1e-6)
        assert float(e.clip_coef) == pytest.approx(float(_coef(_norm(gs[i]), 10.0)), rel=1e-6)


def test_skip_nonfinite_on_the_engine():
    n, numel, bad = 4, 3 * CHUNK, 1
    engines, tables, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, True,
                                         name='clip_skip')
    _clip_on(engines, skip=True)
    _set(engines, 20.0)
    for e in engines:
        e.momentum.normal_()
    engines[bad].grad[100] = float('nan')                   # (inside tensor 0, not padding)
    torch.cuda.synchronize()
    zs = [e.z.double().cpu() for e in engines]
    ms = [e.momentum.clone() for e in engines]
    gs = [e.grad.float().cpu() for e in engines]
    for e, s in zip(engines, streams):
        with torch.cuda.stream(s):
            e.mix(sgd=True)
    torch.cuda.synchronize()
    xs = []
    for i, e in enumerate(engines):
        e.check()
        assert e.nonfinite_steps == (1 if i == bad else 0)
        assert torch.all(e.grad == 0)
        if i == bad:
            assert math.isnan(float(e.grad_norm))
            assert torch.equal(e.momentum, ms[i])
            xs.append(zs[i])                                  # x untouched (w == 1)
        else:
            x, _ = _sgd(zs[i].float(), gs[i], ms[i].double().cpu(), e.clip_coef.cpu())
            xs.append(x)
    for i, e in enumerate(engines):
        t, wt = tables[i]
        acc = float(wt[0, 0]) * xs[i]
        for k in range(int(t[0, 0])):
            acc = acc + float(wt[0, 1 + k]) * xs[int(t[0, 2 + k])]
        assert torch.isfinite(e.z).all()
        torch.testing.assert_close(e.z.double().cpu(), acc, rtol=1e-4, atol=1e-5)
    assert sum(e.ps_weight for e in engines) == pytest.approx(n, abs=1e-5)
    # the next step runs normally and does not count
    for e in engines:
        e.grad.normal_()
    for e, s in zip(engines, streams):
        with torch.cuda.stream(s):
            e.mix(sgd=True)
    torch.cuda.synchronize()
    assert [e.nonfinite_steps for e in engines] == [1 if i == bad else 0 for i in range(n)]
    assert all(torch.isfinite(e.z).all() for e in engines)


class _ScaledLoss(object):
    """cross-entropy times a device scalar: setting it to NaN makes one step's gradient NaN while the
    forward pass (and so BatchNorm's running statistics) stays finite"""

    def __init__(self, dev):
        self.scale = torch.ones((), device=dev)

    def __call__(self, out, tgt):
        return torch.nn.functional.cross_entropy(out, tgt) * self.scale


def _trainers(n, use_graph, name):
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    dev = torch.device('cuda', 0)
    lw = LocalWorld(n) if n > 1 else None
    out = []
    for r in range(n):
        torch.manual_seed(7 + r)
        net = models.TinyConvNet().to(dev).to(memory_format=torch.channels_last)
        kw = dict(symmetric_world=lw.view(r), transport='nvlink', grid=4, symmetric_name=name) if n > 1 else {}
        model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(r, n), rank=r,
                                   world_size=n, heartbeat_timeout=20, **kw)
        opt = FusedGossipSGD(model, lr=0.5, momentum=0.9, nesterov=True, weight_decay=1e-4,
                             max_grad_norm=1e-3, skip_nonfinite=True)
        assert model.engine.grad_clip
        out.append(GossipTrainer(model, opt, criterion=_ScaledLoss(dev), amp_dtype=None,
                                 use_cuda_graph=use_graph, warmup_iters=10 ** 6))
    return out


@pytest.mark.parametrize('n', [1, 2], ids=['one-rank', 'loopback'])
def test_graphed_trainer_matches_eager_threshold_change_and_nan_step(n):
    steps, nan_step = 7, 5
    results = []
    for use_graph in (False, True):
        trainers = _trainers(n, use_graph, 'loopback_clip%d_%d' % (n, use_graph))
        gens = [torch.Generator().manual_seed(100 + r) for r in range(n)]
        coefs = []
        for s in range(steps):
            if use_graph and s == 2:
                for tr in trainers:
                    with torch.cuda.stream(tr.stream):
                        tr._capture()
            for r, tr in enumerate(trainers):  # the threshold changes after capture; rank 0's loss is NaN once
                tr.opt.max_grad_norm = 1e-3 if s < 4 else 1e6
                tr.criterion.scale.fill_(float('nan') if (s == nan_step and r == 0) else 1.0)
            torch.cuda.synchronize()

            def rank_step(r):
                x = torch.randn(8, 3, 32, 32, generator=gens[r]).pin_memory()
                y = torch.randint(0, 10, (8,), generator=gens[r]).pin_memory()
                trainers[r].step(x, y)
            _in_threads([functools.partial(rank_step, r) for r in range(n)])
            torch.cuda.synchronize()
            coefs.append([float(tr.model.engine.clip_coef) for tr in trainers])
        for tr in trainers:
            tr.finish()
            tr.criterion.scale.fill_(1.0)
        results.append(([tr.model.arena.flat.cpu().clone() for tr in trainers], coefs,
                        [tr.opt.nonfinite_steps for tr in trainers],
                        [torch.cat([b.reshape(-1).float() for b in tr.model.module.buffers()]).cpu()
                         for tr in trainers]))
        assert all((tr.graph is not None) == use_graph for tr in trainers)
    (eager, c_eager, k_eager, bn_eager), (graphed, c_graphed, k_graphed, bn_graphed) = results
    assert k_eager == k_graphed == [1] + [0] * (n - 1)
    for r in range(n):
        assert torch.isfinite(eager[r]).all() and torch.isfinite(graphed[r]).all()
        assert torch.isfinite(bn_graphed[r]).all()
        torch.testing.assert_close(graphed[r], eager[r], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(bn_graphed[r], bn_eager[r], rtol=1e-4, atol=1e-5)
    # the threshold reached the captured graph: clipping before step 4, none after
    for c in (c_eager, c_graphed):
        assert all(v < 1 for v in c[3]) and all(v == 1 for v in c[6])


def _resnet50_launches(**opt_kw):
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD, lars_groups
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    dev = torch.device('cuda', 0)
    torch.manual_seed(1)
    net = models.resnet50()
    models.init_imagenet_in_1hr(net)
    net = net.to(dev).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                               verbose=False, heartbeat_timeout=60)
    if opt_kw.pop('lars', False):
        opt_kw.update(param_groups=lars_groups(net, 1e-4), lars=True)
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, weight_decay=1e-4, nesterov=True, **opt_kw)
    trainer = GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=True, warmup_iters=1)
    g = torch.Generator().manual_seed(1234)
    x = torch.randn(256, 3, 224, 224, generator=g).pin_memory()
    y = torch.randint(0, 1000, (256,), generator=g).pin_memory()
    for _ in range(3):                   # eager, capture + replay, replay
        trainer.step(x, y)
    torch.cuda.synchronize()
    assert trainer.graph is not None
    out = trainer.own_launches_per_step, torch.isfinite(model.arena.flat).all().item()
    del trainer, opt, model, net
    torch.cuda.empty_cache()
    return out


def test_resnet50_launch_counts():
    off, ok0 = _resnet50_launches()
    clip, ok1 = _resnet50_launches(max_grad_norm=1.0, skip_nonfinite=True)
    skip, ok2 = _resnet50_launches(skip_nonfinite=True)
    lars, ok3 = _resnet50_launches(lars=True)
    lars_clip, ok4 = _resnet50_launches(lars=True, max_grad_norm=1.0)
    assert ok0 and ok1 and ok2 and ok3 and ok4
    print('launches per step: off %d, clip %d, skip %d, lars %d, lars+clip %d' % (off, clip, skip, lars, lars_clip))
    assert off == 326
    assert clip == skip == off + 2            # norms + finalize
    assert lars_clip == lars + 1              # the finalize; the norm kernel is LARS's
