"""Per-parameter-group SGD on the kernel plane (``SGP_F_GROUPS``): N virtual ranks on one GPU
(``LocalWorld`` loop-back) against a simulation that applies each 64-element block's group values
and mixes in table order -- the full step (pipe and register-staged, fp32 and bf16 messages), the
overlap publish / gather / local flush --, default-valued groups bit-identical to the ungrouped
kernels, exact no-decay on a zero-gradient parameter, a graph-captured trainer that sees a per-group
lr change without re-capture, and the bf16 compute twin."""
import functools

import pytest
import torch

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops.peer_mix import build_tables

from test_gdp_loopback_gpu import _in_threads

pytestmark = pytest.mark.gpu

CHUNK = 4096
BF16 = torch.bfloat16
ROWS = [(0.1, 0.9, 1e-4, True), (0.02, 0.5, 0.0, False), (0.3, 0.0, 3e-3, False)]


def _mk_world(n, numel, graph_cls, ppi, pipe, msg_dtype=None, residual=False, grid=8, name='pgroups'):
    from stochastic_gradient_push_b200.ops.peer_mix import GossipEngine
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    dev = torch.device('cuda', 0)
    torch.manual_seed(0)
    lw = LocalWorld(n)
    engines, tables, streams = [], [], []
    for r in range(n):
        g = graph_cls(r, n, peers_per_itr=ppi)
        e = GossipEngine(lw.view(r), torch.randn(numel, device=dev), g, sgp.UniformMixing(g, dev),
                         grad=torch.randn(numel, device=dev), momentum=torch.zeros(numel, device=dev),
                         grid=grid, timeout_s=10.0, name=name, msg_dtype=msg_dtype, with_residual=residual)
        e.ctx.set_pipe(pipe)
        engines.append(e)
        gc = graph_cls(r, n, peers_per_itr=ppi)
        tables.append(build_tables(gc, sgp.UniformMixing(gc, 'cpu'), 'cpu'))
        streams.append(torch.cuda.Stream(device=dev))
    return engines, tables, streams


def _block_map(numel, groups, seed=5):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, groups, (numel // 64,), generator=g, dtype=torch.uint8)


def _vectors(bmap, rows):
    idx = bmap.long().repeat_interleave(64)
    t = torch.tensor([r[:3] for r in rows], dtype=torch.float64)
    nest = torch.tensor([bool(r[3]) for r in rows])
    return t[:, 0][idx], t[:, 1][idx], t[:, 2][idx], nest[idx]


def _fma(a, b, c):
    """fp32 fmaf: the product of two fp32 values is exact in fp64"""
    return (a.double() * b.double() + c.double()).float()


def _sgd(x, g, m, vec):
    """the kernels' fp32 fmaf chain (sgd1), so that the bf16 rounding of the result matches too"""
    lr, mu, wd, nest = (v if v.dtype == torch.bool else v.float() for v in vec)
    x, g, m = x.float(), g.float(), m.float()
    d = _fma(wd, x, g)
    m = _fma(mu, m, d)
    x = _fma(-lr, torch.where(nest, _fma(mu, m, d), m), x)
    return x.double(), m.double()


def _set_groups(engines, bmap, rows):
    for e in engines:
        e.set_param_groups(bmap.to(e.device), len(rows))
        e.set_hyper(0.5, 0.5, 0.5, True, groups=rows)     # row 0 values must not be used


@pytest.mark.parametrize('pipe', [True, False], ids=['pipe', 'regs'])
@pytest.mark.parametrize('msg_dtype', [None, BF16], ids=['fp32', 'bf16'])
@pytest.mark.parametrize('graph_cls,ppi', [(sgp.NPeerDynamicDirectedExponentialGraph, 1),
                                           (sgp.DynamicDirectedExponentialGraph, 2)])
def test_mix_matches_group_simulation(graph_cls, ppi, msg_dtype, pipe):
    n, numel, steps = 4, 3 * CHUNK, 4
    engines, tables, streams = _mk_world(n, numel, graph_cls, ppi, pipe, msg_dtype)
    bmap = _block_map(numel, len(ROWS))
    _set_groups(engines, bmap, ROWS)
    vec = _vectors(bmap, ROWS)
    zs = [e.z.double().cpu() for e in engines]
    ms = [e.momentum.double().cpu() for e in engines]
    ws = [1.0] * n
    for step in range(steps):
        gs = []
        for e in engines:
            e.grad.normal_()
            gs.append(e.grad.double().cpu())
        torch.cuda.synchronize()
        for e, s in zip(engines, streams):
            with torch.cuda.stream(s):
                e.mix(sgd=True)
        torch.cuda.synchronize()
        xs = []
        for i in range(n):
            x, ms[i] = _sgd(zs[i].float() * torch.tensor(ws[i], dtype=torch.float32), gs[i], ms[i], vec)
            xs.append(x)
        sent = [x.to(BF16).double() if msg_dtype is not None else x for x in xs]
        new_z, new_w = [], []
        for i in range(n):
            t, wt = tables[i]
            row = step % t.shape[0]
            sw = float(wt[row, 0])
            acc = xs[i] - (1 - sw) * sent[i]
            wn = sw * ws[i]
            for k in range(int(t[row, 0])):
                j = int(t[row, 2 + k])
                acc = acc + float(wt[row, 1 + k]) * sent[j]
                wn += float(wt[row, 1 + k]) * ws[j]
            new_z.append(acc / wn)
            new_w.append(wn)
        zs, ws = new_z, new_w
        for i, e in enumerate(engines):
            e.check()
            torch.testing.assert_close(e.z.double().cpu(), zs[i], rtol=1e-4, atol=1e-5)
            torch.testing.assert_close(e.momentum.double().cpu(), ms[i], rtol=1e-4, atol=1e-5)
            assert abs(e.ps_weight - ws[i]) < 1e-6
            # each step starts from the kernel's fp32 state, so that the bf16 rounding of x = z * w
            # sees the same operands
            zs[i] = e.z.double().cpu()
            ms[i] = e.momentum.double().cpu()
            ws[i] = e.ps_weight


def test_overlap_publish_gather_local_match_group_simulation():
    n, numel = 2, 2 * CHUNK
    engines, tables, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, True,
                                         residual=True, name='pgroups_osgp')
    bmap = _block_map(numel, len(ROWS), seed=9)
    _set_groups(engines, bmap, ROWS)
    vec = _vectors(bmap, ROWS)
    zs = [e.z.double().cpu() for e in engines]
    ms = [e.momentum.double().cpu() for e in engines]
    ws = [1.0] * n
    res, wres = [torch.zeros(numel, dtype=torch.float64) for _ in range(n)], [0.0] * n
    for step in range(3):
        gs = []
        for e in engines:
            e.grad.normal_()
            gs.append(e.grad.double().cpu())
        torch.cuda.synchronize()
        for e, s in zip(engines, streams):
            with torch.cuda.stream(s):
                e.publish(sgd=True, fold=step > 0)
                e.gather()
        torch.cuda.synchronize()
        xs = []
        for i in range(n):
            x, ms[i] = _sgd(zs[i] * ws[i], gs[i], ms[i], vec)
            x = x + res[i]
            w1 = ws[i] + wres[i]
            xs.append((x, w1))
        for i in range(n):
            t, wt = tables[i]
            row = step % t.shape[0]
            sw = float(wt[row, 0])
            x, w1 = xs[i]
            zs[i], ws[i] = x / w1, sw * w1
            res[i] = sum(float(wt[row, 1 + k]) * xs[int(t[row, 2 + k])][0] for k in range(int(t[row, 0])))
            wres[i] = sum(float(wt[row, 1 + k]) * xs[int(t[row, 2 + k])][1] for k in range(int(t[row, 0])))
    # flush: the last gradient and the residual, no communication
    for e in engines:
        e.grad.normal_()
    gs = [e.grad.double().cpu() for e in engines]
    for e in engines:
        e.local(sgd=True, fold=True)
    torch.cuda.synchronize()
    for i, e in enumerate(engines):
        e.check()
        x, ms[i] = _sgd(zs[i] * ws[i], gs[i], ms[i], vec)
        want = (x + res[i]) / (ws[i] + wres[i])
        torch.testing.assert_close(e.z.double().cpu(), want, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(e.momentum.double().cpu(), ms[i], rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize('pipe', [True, False], ids=['pipe', 'regs'])
@pytest.mark.parametrize('msg_dtype', [None, BF16], ids=['fp32', 'bf16'])
def test_default_valued_groups_are_bit_identical(msg_dtype, pipe):
    n, numel = 2, 2 * CHUNK
    hyper = (0.1, 0.9, 1e-4, True)
    worlds = []
    for grouped in (False, True):
        engines, _, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, pipe,
                                        msg_dtype, name='pgroups_eq%d' % grouped)
        if grouped:
            for e in engines:
                e.set_param_groups(_block_map(numel, 2).to(e.device), 2)
        worlds.append((engines, streams))
    for step in range(3):
        g = [torch.randn(numel, device='cuda') for _ in range(n)]
        for (engines, streams), grouped in zip(worlds, (False, True)):
            for e, gr in zip(engines, g):
                e.grad.copy_(gr)
                e.set_hyper(*hyper, groups=[hyper, hyper] if grouped else None)
            torch.cuda.synchronize()
            for e, s in zip(engines, streams):
                with torch.cuda.stream(s):
                    e.mix(sgd=True)
            torch.cuda.synchronize()
    for a, b in zip(*(w[0] for w in worlds)):
        a.check()
        b.check()
        assert b.ctx.param_groups() == 2 and a.ctx.param_groups() == 0
        assert torch.equal(a.z, b.z) and torch.equal(a.momentum, b.momentum)


def test_zero_gradient_parameter_without_decay_stays_exact():
    n, numel = 2, 2 * CHUNK
    engines, _, _ = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, True, name='pgroups_wd')
    e = engines[0]
    bmap = torch.zeros(numel // 64, dtype=torch.uint8)
    bmap[: numel // 128] = 1                       # first half: wd = 0 ; second half: wd > 0
    e.set_param_groups(bmap.to(e.device), 2)
    e.grad.zero_()
    z0 = e.z.clone()
    for _ in range(5):
        e.set_hyper(0.1, 0.9, 0.0, False, groups=[(0.1, 0.9, 1e-2, False), (0.1, 0.9, 0.0, True)])
        e.local(sgd=True)
    torch.cuda.synchronize()
    e.check()
    half = numel // 2
    assert torch.equal(e.z[:half], z0[:half])
    assert torch.equal(e.momentum[:half], torch.zeros_like(e.momentum[:half]))
    assert (e.z[half:].abs() < z0[half:].abs()).float().mean().item() > 0.99


def _loopback_trainers(n, use_graph, name, compute_dtype=None):
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD, no_bias_decay_groups
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
                                   transport='nvlink', grid=4, symmetric_name=name, compute_dtype=compute_dtype)
        opt = FusedGossipSGD(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True,
                             param_groups=no_bias_decay_groups(model.module, 1e-4))
        assert model.engine.groups == 2
        trainers.append(GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=use_graph,
                                      warmup_iters=10 ** 6))
    return trainers


def test_graphed_trainer_reads_group_lr_from_device_memory():
    n, steps = 2, 7
    results = []
    for use_graph in (False, True):
        trainers = _loopback_trainers(n, use_graph, 'loopback_pgroups%d' % use_graph)
        gens = [torch.Generator().manual_seed(100 + r) for r in range(n)]
        for s in range(steps):
            if use_graph and s == 2:
                for tr in trainers:          # every capture before any replay (see test_gdp_loopback_gpu)
                    with torch.cuda.stream(tr.stream):
                        tr._capture()
            for tr in trainers:              # only group 1's lr changes between replays
                tr.opt.param_groups[1]['lr'] = 0.05 * (1 + 0.3 * s)

            def rank_step(r):
                x = torch.randn(8, 3, 32, 32, generator=gens[r]).pin_memory()
                y = torch.randint(0, 10, (8,), generator=gens[r]).pin_memory()
                trainers[r].step(x, y)
            _in_threads([functools.partial(rank_step, r) for r in range(n)])
            torch.cuda.synchronize()
        for tr in trainers:
            tr.finish()
        results.append([tr.model.arena.flat.cpu().clone() for tr in trainers])
        assert all((tr.graph is not None) == use_graph for tr in trainers)
    eager, graphed = results
    for r in range(n):
        assert torch.isfinite(eager[r]).all()
        torch.testing.assert_close(graphed[r], eager[r], rtol=1e-4, atol=1e-5)


def test_bf16_compute_twin_trains_with_two_groups():
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD, no_bias_decay_groups
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    dev = torch.device('cuda', 0)
    torch.manual_seed(3)
    net = models.TinyConvNet(width=32).to(dev).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0,
                               world_size=1, heartbeat_timeout=20, compute_dtype=torch.bfloat16)
    groups = no_bias_decay_groups(model.module, 0.05)
    opt = FusedGossipSGD(model, lr=0.05, momentum=0.9, weight_decay=0.05, nesterov=True, param_groups=groups)
    assert model.engine.groups == 2 and model.compute_module is not model.module
    tr = GossipTrainer(model, opt, amp_dtype=torch.bfloat16, use_cuda_graph=True, warmup_iters=2)
    g = torch.Generator().manual_seed(11)
    x = torch.randn(32, 3, 32, 32, generator=g).pin_memory()
    y = torch.randint(0, 10, (32,), generator=g).pin_memory()
    slots = [tr.step(x, y) for _ in range(8)]
    tr.finish()
    losses = [float(tr.loss_ring[s]) for s in slots]
    assert all(l == l for l in losses) and losses[-1] < losses[0]
    torch.testing.assert_close(model.compute_shadow.float(), model.arena.flat.bfloat16().float(), rtol=0, atol=0)
