"""bf16 gossip messages on the kernel plane (``GossipEngine(msg_dtype=torch.bfloat16)``,
``GossipDataParallel(gossip_dtype=torch.bfloat16)``): N virtual ranks on one GPU (``LocalWorld``
loop-back) against a simulation that performs the kernels' fp32 operations in the same order and
rounds the messages the same way, push-sum mass conservation, a graph-captured trainer step, and
the heartbeat fallback."""
import functools

import pytest
import torch

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops.peer_mix import build_tables

from test_gdp_loopback_gpu import _in_threads

pytestmark = pytest.mark.gpu

CHUNK = 4096
BF16 = torch.bfloat16


def _mk_world(n, numel, graph_cls, ppi, pipe, mixing=None, with_sgd=True, grid=8, seed=0):
    from stochastic_gradient_push_b200.ops.peer_mix import GossipEngine
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    dev = torch.device('cuda', 0)
    torch.manual_seed(seed)
    lw = LocalWorld(n)
    engines, graphs, streams = [], [], []
    for r in range(n):
        g = graph_cls(r, n, peers_per_itr=ppi)
        m = mixing(g, dev) if mixing else sgp.UniformMixing(g, dev)
        z = torch.randn(numel, device=dev)
        kw = dict(grad=torch.randn(numel, device=dev), momentum=torch.zeros(numel, device=dev)) \
            if with_sgd else {}
        e = GossipEngine(lw.view(r), z, g, m, grid=grid, timeout_s=10.0, name='bf16', msg_dtype=BF16, **kw)
        e.ctx.set_pipe(pipe)
        engines.append(e)
        graphs.append(g)
        streams.append(torch.cuda.Stream(device=dev))
    return engines, graphs, streams


def _f32(v):
    return torch.tensor(v, dtype=torch.float32)


def _fma(a, b, c):
    """fp32 fmaf: the product of two fp32 (or bf16 x fp32) values is exact in fp64"""
    return (a.double() * b.double() + c.double()).float()


def _kernel_step_sim(zs, ws, gs, ms, tables, step, hyper):
    """One full bf16 gossip step of every rank, operation for operation as the kernels do it:
    phase 1 x = z*w ; SGD (fmaf chain) ; publish q = bf16(x) ; keep c = fmaf(q, self_w - 1, x);
    phase 2 acc = c ; acc = fmaf(q_k, in_w[k], acc) over the in-neighbours in table order ;
    w' = fmaf(in_w[k], w_k, self_w * w) ; z = acc * (1 / w')."""
    n = len(zs)
    xs, qs, cs = [], [], []
    for i in range(n):
        t, wt = tables[i]
        row = step % t.shape[0]
        sw = wt[row, 0]
        x = zs[i] * _f32(ws[i])
        if hyper is not None:
            lr, mu, wd, nest = hyper
            d = _fma(_f32(wd), x, gs[i])
            ms[i] = _fma(_f32(mu), ms[i], d)
            upd = _fma(_f32(mu), ms[i], d) if nest else ms[i]
            x = _fma(_f32(-lr), upd, x)
        q = x.to(BF16)
        xs.append(x)
        qs.append(q)
        cs.append(_fma(q, sw - 1.0, x))
    new_z, new_w = [], []
    for i in range(n):
        t, wt = tables[i]
        row = step % t.shape[0]
        sw = wt[row, 0]
        acc = cs[i]
        wn = sw * _f32(ws[i])
        for k in range(int(t[row, 0])):
            j = int(t[row, 2 + k])
            if j < 0:
                continue
            acc = _fma(qs[j], wt[row, 1 + k], acc)
            wn = _fma(wt[row, 1 + k], _f32(ws[j]), wn)
        new_z.append(acc * (_f32(1.0) / wn))
        new_w.append(float(wn))
    return new_z, new_w


@pytest.mark.parametrize('pipe', [True, False], ids=['pipe', 'regs'])
@pytest.mark.parametrize('graph_cls,ppi', [
    (sgp.NPeerDynamicDirectedExponentialGraph, 1),
    (sgp.DynamicDirectedExponentialGraph, 2),
    (sgp.RingGraph, 1),
])
def test_kernel_plane_matches_bf16_simulation(graph_cls, ppi, pipe):
    n, numel, steps = 4, 3 * CHUNK, 5
    hyper = (0.1, 0.9, 1e-4, True)
    engines, graphs, streams = _mk_world(n, numel, graph_cls, ppi, pipe)
    tables = []
    for r in range(n):
        g = graph_cls(r, n, peers_per_itr=ppi)
        t, wt = build_tables(g, sgp.UniformMixing(g, 'cpu'), 'cpu')
        tables.append((t, wt))
    zs = [e.z.cpu().clone() for e in engines]
    ms = [e.momentum.cpu().clone() for e in engines]
    ws = [1.0] * n
    for step in range(steps):
        gs = []
        for e in engines:
            e.grad.normal_()
            gs.append(e.grad.cpu().clone())
            e.set_hyper(*hyper)
        torch.cuda.synchronize()
        for e, s in zip(engines, streams):
            with torch.cuda.stream(s):
                e.mix(sgd=True)
        torch.cuda.synchronize()
        zs, ws = _kernel_step_sim(zs, ws, gs, ms, tables, step, hyper)
        for i, e in enumerate(engines):
            e.check()
            torch.testing.assert_close(e.z.cpu(), zs[i], rtol=1e-4, atol=1e-5)
            torch.testing.assert_close(e.momentum.cpu(), ms[i], rtol=1e-4, atol=1e-5)
            assert abs(e.ps_weight - ws[i]) < 1e-6


@pytest.mark.parametrize('mixing', ['uniform', 'self_weighted'])
def test_mass_is_conserved_and_consensus_reaches_bf16_resolution(mixing):
    n, numel, steps = 4, 2 * CHUNK, 50
    mix = None if mixing == 'uniform' else functools.partial(sgp.SelfWeightedMixing,
                                                             self_weight=[0.3, 0.5, 0.6, 0.45])
    engines, _, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, True,
                                    mixing=mix, with_sgd=False)
    z0 = torch.stack([e.z.double().cpu() for e in engines])
    mass0 = z0.sum(0)
    spread0 = (z0 - z0.mean(0)).abs().max().item()
    for _ in range(steps):
        for e, s in zip(engines, streams):
            with torch.cuda.stream(s):
                e.mix(sgd=False)
        torch.cuda.synchronize()
    for e in engines:
        e.check()
    zw = torch.stack([e.z.double().cpu() * e.ps_weight for e in engines])
    torch.testing.assert_close(zw.sum(0), mass0, rtol=0, atol=1e-4)
    assert abs(sum(e.ps_weight for e in engines) - n) < 1e-5
    zs = torch.stack([e.z.double().cpu() for e in engines])
    spread = (zs - zs.mean(0)).abs().max().item()
    # the messages are bf16 (8 significant bits): consensus stops at a few bf16 ulps of the average
    assert spread < 2 ** -6 * zs.mean(0).abs().max().item() and spread < 0.01 * spread0


@pytest.mark.parametrize('pipe', [True, False], ids=['pipe', 'regs'])
def test_dead_peer_leaves_the_documented_fallback(pipe):
    """an in-neighbour that never publishes: the heartbeat trips, and z is what the rank still
    holds after sending, c = x - (1 - self_w) Q(x), de-biased over the weight it kept, self_w * w"""
    n, numel = 2, 2 * CHUNK
    engines, graphs, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1, pipe,
                                         with_sgd=False)
    e = engines[0]
    e.ctx.set_timeout(0.3)
    sw = float(build_tables(graphs[0], sgp.UniformMixing(graphs[0], 'cpu'), 'cpu')[1][0, 0])
    x = e.z.cpu().clone()
    with torch.cuda.stream(streams[0]):
        e.mix(sgd=False)                             # rank 1 never launches
    torch.cuda.synchronize()
    with pytest.raises(NameError, match='Gossip flag timeout'):
        e.poll(blocking=True)
    c = _fma(x.to(BF16), _f32(sw) - 1.0, x)
    z = e.z.cpu()
    assert torch.isfinite(z).all()
    torch.testing.assert_close(z, c * (_f32(1.0) / (_f32(sw) * _f32(1.0))), rtol=1e-6, atol=1e-7)
    if pipe:
        assert abs(e.ps_weight - sw) < 1e-7
    e.clear_status()
    e.poll(blocking=True)


def test_bf16_engine_rejects_operations_it_does_not_implement():
    engines, _, _ = _mk_world(2, CHUNK, sgp.NPeerDynamicDirectedExponentialGraph, 1, True, with_sgd=False)
    e = engines[0]
    for op in (lambda: e.publish(), lambda: e.gather(), lambda: e.publish_only(), lambda: e.pull_only(),
               lambda: e.probe()):
        with pytest.raises(RuntimeError, match='bf16'):
            op()
    assert e.outbox.nbytes == 2 * CHUNK * 2


def test_loopback_graphed_trainer_with_bf16_messages_equals_eager():
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    dev = torch.device('cuda', 0)
    n, steps = 2, 7
    results = []
    for use_graph in (False, True):
        lw = LocalWorld(n)
        trainers = []
        for r in range(n):
            torch.manual_seed(7 + r)
            net = models.TinyConvNet().to(dev).to(memory_format=torch.channels_last)
            model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(r, n),
                                       rank=r, world_size=n, heartbeat_timeout=20, symmetric_world=lw.view(r),
                                       transport='nvlink', grid=4, symmetric_name='loopback_bf16',
                                       gossip_dtype=BF16)
            assert model.engine.msg_bf16
            opt = FusedGossipSGD(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True)
            trainers.append(GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=use_graph, warmup_iters=10 ** 6))
        gens = [torch.Generator().manual_seed(100 + r) for r in range(n)]
        for s in range(steps):
            if use_graph and s == 2:
                for tr in trainers:          # every capture before any replay (see test_gdp_loopback_gpu)
                    with torch.cuda.stream(tr.stream):
                        tr._capture()

            def rank_step(r):
                x = torch.randn(8, 3, 32, 32, generator=gens[r]).pin_memory()
                y = torch.randint(0, 10, (8,), generator=gens[r]).pin_memory()
                trainers[r].step(x, y)
            _in_threads([functools.partial(rank_step, r) for r in range(n)])
            torch.cuda.synchronize()
        for tr in trainers:
            tr.finish()
        results.append([(tr.model.arena.flat.cpu().clone(), tr.engine.device_step) for tr in trainers])
        assert all((tr.graph is not None) == use_graph for tr in trainers)
    eager, graphed = results
    for r in range(n):
        assert torch.isfinite(eager[r][0]).all()
        torch.testing.assert_close(graphed[r][0], eager[r][0], rtol=1e-4, atol=1e-5)
        assert graphed[r][1] == eager[r][1] == steps
