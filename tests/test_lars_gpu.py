"""LARS on the kernel plane (``SGP_F_LARS``): N virtual ranks on one GPU (``LocalWorld`` loop-back)
against a simulation that takes each tensor's trust ratio from fp64 norms and then follows the
kernels' fmaf order -- the full step (pipe and register-staged, fp32 and bf16 messages), the overlap
publish / gather (DMA and TMA) / local flush --, deterministic trust ratios, groups without LARS
bit-identical to the grouped kernels, the norms of a ResNet-50 arena against ``torch._foreach_norm``,
a graph-captured trainer against eager with a weight-decay change after capture, and the bf16
gradient + fp32 g2 of the compute twin."""
import functools

import pytest
import torch

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops.peer_mix import build_tables

from test_gdp_loopback_gpu import _in_threads
from test_param_groups_gpu import _fma, _mk_world

pytestmark = pytest.mark.gpu

CHUNK = 4096
BF16 = torch.bfloat16
# group 0: no LARS, no decay (the "ndim <= 1" group); group 1: LARS with decay
ROWS = [(0.1, 0.9, 0.0, True), (0.2, 0.9, 1e-3, False)]
ENABLED_GROUPS = (False, True)
ETA, EPS = 0.02, 1e-8
NUMELS = [5000, 37, 4200, 900, 1, 1500]        # 64-aligned offsets, tail padding up to 3 chunks
GROUP_OF = [1, 0, 1, 0, 0, 1]


def _layout(numels=NUMELS):
    offs, off = [], 0
    for n in numels:
        offs.append(off)
        off = (off + n + 63) // 64 * 64
    return offs, off


def _maps(numel, numels=NUMELS, group_of=GROUP_OF):
    """(block -> group uint8, block -> tensor long) as the optimizer and the engine build them
    (blocks no tensor covers: group 0, tensor 0)"""
    offs, _ = _layout(numels)
    bgroup = torch.zeros(numel // 64, dtype=torch.uint8)
    btensor = torch.zeros(numel // 64, dtype=torch.long)
    for t, (o, n) in enumerate(zip(offs, numels)):
        bgroup[o // 64:(o + n + 63) // 64] = group_of[t]
        btensor[o // 64:(o + n + 63) // 64] = t
    return bgroup, btensor


def _configure(engines, numel, enabled_groups=ENABLED_GROUPS):
    offs, _ = _layout()
    bgroup, _ = _maps(numel)
    for e in engines:
        e.set_param_groups(bgroup.to(e.device), len(ROWS))
        e.set_hyper(0.5, 0.5, 0.5, True, groups=ROWS)
        e.set_lars(offs, NUMELS, [enabled_groups[g] for g in GROUP_OF], ETA, EPS)


def _trust(x, g, numel, enabled_groups=ENABLED_GROUPS):
    """fp32 x and g^ -> the per-tensor fp32 trust ratios, from fp64 norms"""
    offs, _ = _layout()
    out = []
    for o, n, gi in zip(offs, NUMELS, GROUP_OF):
        nx, ng = x[o:o + n].double().norm().item(), g[o:o + n].double().norm().item()
        wd = torch.tensor(ROWS[gi][2], dtype=torch.float32).double().item()
        eta = torch.tensor(ETA, dtype=torch.float32).double().item()
        eps = torch.tensor(EPS, dtype=torch.float32).double().item()
        t = eta * nx / (ng + wd * nx + eps) if (enabled_groups[gi] and nx > 0 and ng > 0) else 1.0
        out.append(t)
    return torch.tensor(out, dtype=torch.float64)


def _lars_step(x, g, m, numel, trust):
    """the kernels' fp32 chain: d = t * fmaf(wd, x, g) ; m = fmaf(mu, m, d) ; x = fmaf(-lr, upd, x)"""
    bgroup, btensor = _maps(numel)
    idx = bgroup.long().repeat_interleave(64)
    t = trust.float()[btensor.repeat_interleave(64)]
    rows = torch.tensor([r[:3] for r in ROWS], dtype=torch.float32)
    lr, mu, wd = rows[:, 0][idx], rows[:, 1][idx], rows[:, 2][idx]
    nest = torch.tensor([bool(r[3]) for r in ROWS])[idx]
    x, g, m = x.float(), g.float(), m.float()
    d = t * _fma(wd, x, g)
    m = _fma(mu, m, d)
    x = _fma(-lr, torch.where(nest, _fma(mu, m, d), m), x)
    return x.double(), m.double()


@pytest.mark.parametrize('pipe', [True, False], ids=['pipe', 'regs'])
@pytest.mark.parametrize('msg_dtype', [None, BF16], ids=['fp32', 'bf16'])
def test_mix_matches_lars_simulation(msg_dtype, pipe):
    n, numel, steps = 4, 3 * CHUNK, 4
    graph_cls = sgp.NPeerDynamicDirectedExponentialGraph
    engines, tables, streams = _mk_world(n, numel, graph_cls, 1, pipe, msg_dtype, name='lars_mix')
    _configure(engines, numel)
    for step in range(steps):
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
            x0 = zs[i].float() * torch.tensor(ws[i], dtype=torch.float32)
            trust = _trust(x0, gs[i], numel)
            torch.testing.assert_close(e.lars_trust.double().cpu(), trust, rtol=1e-6, atol=0)
            assert (trust != 1).sum() == 3            # the three LARS tensors
            x, m = _lars_step(x0, gs[i], ms[i], numel, e.lars_trust.cpu())
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
            assert abs(e.ps_weight - wn) < 1e-6


@pytest.mark.parametrize('dma', [True, False], ids=['dma', 'tma'])
def test_overlap_publish_gather_local_match_lars_simulation(dma):
    n, numel = 2, 3 * CHUNK
    engines, tables, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, True,
                                         residual=True, name='lars_osgp%d' % dma)
    _configure(engines, numel)
    ms = [e.momentum.double().cpu() for e in engines]
    res, wres = [torch.zeros(numel, dtype=torch.float64) for _ in range(n)], [0.0] * n
    zs = [e.z.double().cpu() for e in engines]
    ws = [1.0] * n
    for step in range(3):
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
            x0 = (zs[i] * ws[i]).float()
            trust = _trust(x0, gs[i], numel)          # the norms are of x BEFORE the residual fold
            torch.testing.assert_close(e.lars_trust.double().cpu(), trust, rtol=1e-6, atol=0)
            x, ms[i] = _lars_step(x0, gs[i], ms[i], numel, e.lars_trust.cpu())
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
    for e in engines:
        e.grad.normal_()
    torch.cuda.synchronize()
    gs = [e.grad.float().cpu() for e in engines]
    for e in engines:
        e.local(sgd=True, fold=True)
    torch.cuda.synchronize()
    for i, e in enumerate(engines):
        e.check()
        x0 = (zs[i] * ws[i]).float()
        x, ms[i] = _lars_step(x0, gs[i], ms[i], numel, _trust(x0, gs[i], numel))
        want = (x + res[i]) / (ws[i] + wres[i])
        torch.testing.assert_close(e.z.double().cpu(), want, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(e.momentum.double().cpu(), ms[i], rtol=1e-4, atol=1e-5)


def test_trust_is_bit_identical_across_launches_and_grids():
    numel = 3 * CHUNK
    engines, _, _ = _mk_world(1, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, True, name='lars_det')
    e = engines[0]
    _configure(engines, numel)
    z0, m0 = e.z.clone(), e.momentum.clone()
    seen = []
    for grid in (e.ctx.lars_grid(), e.ctx.lars_grid(), 1, 3):
        e.ctx.set_lars_grid(grid)
        e.z.copy_(z0)
        e.momentum.copy_(m0)
        e.local(sgd=True, zero_grad=False)
        torch.cuda.synchronize()
        e.check()
        seen.append((e.lars_trust.clone(), e.lars_sumsq.clone(), e.z.clone()))
    for t, s, z in seen[1:]:
        assert torch.equal(t, seen[0][0]) and torch.equal(s, seen[0][1]) and torch.equal(z, seen[0][2])
    assert e.ctx.lars_tiles() == sum((n + CHUNK - 1) // CHUNK for n in NUMELS)


@pytest.mark.parametrize('pipe', [True, False], ids=['pipe', 'regs'])
@pytest.mark.parametrize('msg_dtype', [None, BF16], ids=['fp32', 'bf16'])
def test_all_groups_excluded_is_bit_identical_to_grouped_kernels(msg_dtype, pipe):
    n, numel = 2, 3 * CHUNK
    worlds = []
    for lars in (False, True):
        engines, _, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, pipe,
                                        msg_dtype, name='lars_off%d' % lars)
        _configure(engines, numel, enabled_groups=(False, False))
        if not lars:
            for e in engines:
                e.set_lars(None)
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
        assert not a.lars and b.lars and torch.all(b.lars_trust == 1)
        assert torch.equal(a.z, b.z) and torch.equal(a.momentum, b.momentum)


def test_resnet50_arena_norms_match_foreach_norm():
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD, lars_groups
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    dev = torch.device('cuda', 0)
    torch.manual_seed(1)
    net = models.resnet50().to(dev)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0,
                               world_size=1, heartbeat_timeout=20)
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, nesterov=True,
                         param_groups=lars_groups(model.module, 5e-5), lars=True)
    e = model.engine
    arena = model.arena
    g = opt.grad_flat[torch.float32]
    for v in arena.views_of(g):
        v.normal_()
    x = (arena.flat * e.ps_weight).clone()
    gv = [v.double() for v in arena.views_of(g.clone())]
    opt.set_engine_hyper(e)
    e.local(sgd=True)
    torch.cuda.synchronize()
    e.check()
    xv = [v.double() for v in arena.views_of(x)]
    sumsq = e.lars_sumsq.cpu()
    want_x = torch.stack(torch._foreach_norm(xv)).cpu()
    want_g = torch.stack(torch._foreach_norm(gv)).cpu()
    assert max(arena.numels) > 2_000_000
    torch.testing.assert_close(sumsq[:, 0].sqrt(), want_x, rtol=1e-9, atol=0)
    torch.testing.assert_close(sumsq[:, 1].sqrt(), want_g, rtol=1e-9, atol=0)
    on = torch.tensor([p.dim() > 1 for p in model.module.parameters()])
    want_t = torch.where(on, 0.001 * want_x / (want_g + torch.tensor(5e-5).double() * want_x + 1e-8),
                         torch.ones_like(want_x))
    torch.testing.assert_close(e.lars_trust.double().cpu(), want_t, rtol=1e-6, atol=0)


def _loopback_trainers(n, use_graph, name):
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD, lars_groups
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    dev = torch.device('cuda', 0)
    lw = LocalWorld(n)
    trainers = []
    for r in range(n):
        torch.manual_seed(7 + r)
        net = models.TinyConvNet().to(dev).to(memory_format=torch.channels_last)
        model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(r, n), rank=r,
                                   world_size=n, heartbeat_timeout=20, symmetric_world=lw.view(r),
                                   transport='nvlink', grid=4, symmetric_name=name)
        opt = FusedGossipSGD(model, lr=0.5, momentum=0.9, nesterov=True, trust_coefficient=0.02,
                             param_groups=lars_groups(model.module, 1e-4), lars=True)
        assert model.engine.groups == 2 and model.engine.lars
        trainers.append(GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=use_graph,
                                      warmup_iters=10 ** 6))
    return trainers


def test_graphed_trainer_matches_eager_and_reads_weight_decay_from_device_memory():
    n, steps = 2, 7
    results = []
    for use_graph in (False, True):
        trainers = _loopback_trainers(n, use_graph, 'loopback_lars%d' % use_graph)
        gens = [torch.Generator().manual_seed(100 + r) for r in range(n)]
        for s in range(steps):
            if use_graph and s == 2:
                for tr in trainers:
                    with torch.cuda.stream(tr.stream):
                        tr._capture()
            for tr in trainers:              # the LARS group's weight decay changes after capture
                tr.opt.param_groups[1]['weight_decay'] = 1e-4 if s < 4 else 0.5

            def rank_step(r):
                x = torch.randn(8, 3, 32, 32, generator=gens[r]).pin_memory()
                y = torch.randint(0, 10, (8,), generator=gens[r]).pin_memory()
                trainers[r].step(x, y)
            _in_threads([functools.partial(rank_step, r) for r in range(n)])
            torch.cuda.synchronize()
        for tr in trainers:
            tr.finish()
        results.append(([tr.model.arena.flat.cpu().clone() for tr in trainers],
                        [tr.model.engine.lars_trust.cpu().clone() for tr in trainers]))
        assert all((tr.graph is not None) == use_graph for tr in trainers)
    (eager, t_eager), (graphed, t_graphed) = results
    for r in range(n):
        assert torch.isfinite(eager[r]).all()
        torch.testing.assert_close(graphed[r], eager[r], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(t_graphed[r], t_eager[r], rtol=1e-4, atol=0)
        assert (t_eager[r] != 1).any() and (t_eager[r] == 1).any()
    # the weight decay reached the captured trust kernel: with wd = 0.5, t < eta / wd
    assert all(float(t[t != 1].max()) < 0.02 / 0.5 for t in t_graphed)


def test_bf16_gradient_plus_fp32_g2_matches_simulation():
    n, numel = 2, 3 * CHUNK
    engines, tables, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, True,
                                         name='lars_twin')
    dev = engines[0].device
    lo = [torch.randn(numel, device=dev).to(BF16) for _ in range(n)]
    hi = [torch.randn(numel, device=dev) for _ in range(n)]
    for e, a, b in zip(engines, lo, hi):
        e.set_sgd_buffers(a, e.momentum, grad2=b)
    _configure(engines, numel)
    for e in engines:
        e.set_hyper(0.5, 0.5, 0.5, True, grad_scale=0.25, groups=ROWS)
    zs = [e.z.double().cpu() for e in engines]
    ms = [e.momentum.double().cpu() for e in engines]
    gs = [((a.float() + b) * 0.25).cpu() for a, b in zip(lo, hi)]     # g^ as phase 1 forms it
    for e, s in zip(engines, streams):
        with torch.cuda.stream(s):
            e.mix(sgd=True, zero_grad=False)
    torch.cuda.synchronize()
    xs = []
    for i, e in enumerate(engines):
        e.check()
        x0 = zs[i].float()
        trust = _trust(x0, gs[i], numel)
        torch.testing.assert_close(e.lars_trust.double().cpu(), trust, rtol=1e-6, atol=0)
        x, m = _lars_step(x0, gs[i], ms[i], numel, e.lars_trust.cpu())
        xs.append(x)
        torch.testing.assert_close(e.momentum.double().cpu(), m, rtol=1e-4, atol=1e-5)
    for i, e in enumerate(engines):
        t, wt = tables[i]
        sw = float(wt[0, 0])
        acc = sw * xs[i]
        for k in range(int(t[0, 0])):
            acc = acc + float(wt[0, 1 + k]) * xs[int(t[0, 2 + k])]
        torch.testing.assert_close(e.z.double().cpu(), acc, rtol=1e-4, atol=1e-5)
