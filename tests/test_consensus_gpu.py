"""Consensus distance and the push-sum average model on the kernel plane
(``GossipEngine.consensus``, ``GossipDataParallel.consensus_distance`` / ``average_model``):
N virtual ranks on one GPU (``LocalWorld`` loop-back) against fp64 references, agreement of the
slice and full modes, bit-identical results on every rank, and gossip that continues exactly as if
the call had not happened."""
import functools

import pytest
import torch

import stochastic_gradient_push_b200 as sgp

from test_gdp_loopback_gpu import _in_threads

pytestmark = pytest.mark.gpu

CHUNK = 4096
BF16 = torch.bfloat16


def _mk_world(n, numel, msg_dtype=None, pipe=True, mixing=None, name='cons', seed=0, spread=1e-3):
    """n engines whose parameters are a common random vector plus a small per-rank deviation"""
    from stochastic_gradient_push_b200.ops.peer_mix import GossipEngine
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    dev = torch.device('cuda', 0)
    gen = torch.Generator().manual_seed(seed)
    base = torch.randn(numel, generator=gen)
    lw = LocalWorld(n)
    engines, streams = [], []
    for r in range(n):
        g = sgp.NPeerDynamicDirectedExponentialGraph(r, n)
        m = mixing(g, dev) if mixing else sgp.UniformMixing(g, dev)
        z = (base + spread * torch.randn(numel, generator=gen)).to(dev)
        e = GossipEngine(lw.view(r), z, g, m, grid=8, timeout_s=10.0, name=name, msg_dtype=msg_dtype)
        e.ctx.set_pipe(pipe)
        engines.append(e)
        streams.append(torch.cuda.Stream(device=dev))
    return engines, streams


def _run_consensus(engines, streams, full):
    """enqueue every rank's call on its own stream, then synchronise"""
    outs = [torch.full_like(e.z, float('nan')) if full else None for e in engines]
    torch.cuda.synchronize()                         # (weights / outputs written on the default stream)
    res = []
    for e, s, o in zip(engines, streams, outs):
        with torch.cuda.stream(s):
            res.append(e.consensus(o, full=full))
    torch.cuda.synchronize()
    for e in engines:
        e.check()
    return [r.cpu() for r in res], outs


def _reference(engines):
    zs = torch.stack([e.z.double().cpu() for e in engines])
    ws = torch.tensor([e.ps_weight for e in engines], dtype=torch.float64)
    zbar = (ws[:, None] * zs).sum(0) / ws.sum()
    per_rank = ((zs - zbar) ** 2).sum(1)
    return zbar, per_rank.mean().item(), (zbar ** 2).sum().item(), per_rank


@pytest.mark.parametrize('msg', ['fp32', 'bf16'])
@pytest.mark.parametrize('n', [3, 4])
def test_slice_and_full_match_fp64(n, msg):
    # 7 chunks: the slices of the ranks have different lengths
    engines, streams = _mk_world(n, 7 * CHUNK, msg_dtype=BF16 if msg == 'bf16' else None)
    for r, e in enumerate(engines):
        e.ps_weight = 0.55 + 0.3 * r                 # irregular mixing: w != 1
    zbar, dsq, nrm, per_rank = _reference(engines)

    sl, _ = _run_consensus(engines, streams, full=False)
    fu, outs = _run_consensus(engines, streams, full=True)
    for r in range(n):
        assert torch.equal(sl[r], sl[0]) and torch.equal(fu[r], fu[0]), 'results differ between ranks'
        assert torch.equal(outs[r], outs[0]), 'average models differ between ranks'
    for res in (sl[0], fu[0]):
        assert abs(res[0].item() - dsq) <= 1e-4 * dsq
        assert abs(res[1].item() - nrm) <= 1e-5 * nrm
    torch.testing.assert_close(fu[0][2:], per_rank, rtol=1e-4, atol=0)
    assert (sl[0][2:] == 0).all()
    assert abs(sl[0][0].item() - fu[0][0].item()) <= 1e-4 * dsq
    zmax = zbar.abs().max().item()
    torch.testing.assert_close(outs[0].double().cpu(), zbar, rtol=1e-5, atol=1e-6 * zmax)
    # the plain mean is a different point when w != 1: the test would notice the unweighted average
    plain = torch.stack([e.z.double().cpu() for e in engines]).mean(0)
    assert (plain - zbar).abs().max().item() > 10 * 1e-6 * zmax


@pytest.mark.parametrize('msg', ['fp32', 'bf16'])
def test_identical_replicas_have_zero_distance(msg):
    engines, streams = _mk_world(4, 3 * CHUNK, msg_dtype=BF16 if msg == 'bf16' else None, spread=0.0)
    for full in (False, True):
        res, outs = _run_consensus(engines, streams, full=full)
        for r in range(4):
            assert res[r][0].item() == 0.0
            if full:
                assert torch.equal(outs[r], engines[0].z)
                assert (res[r][2:] == 0).all()


@pytest.mark.parametrize('msg', ['fp32', 'bf16'])
@pytest.mark.parametrize('pipe', [True, False], ids=['pipe', 'regs'])
def test_gossip_after_consensus_is_unchanged(pipe, msg):
    """the snapshot borrows the outbox between barriers and leaves the sequence numbers alone: the
    following steps (same step numbers, same flags) give the bits of a world that never called it"""
    dt = BF16 if msg == 'bf16' else None
    mix = functools.partial(sgp.SelfWeightedMixing, self_weight=[0.3, 0.5, 0.6, 0.45])
    worlds = [_mk_world(4, 5 * CHUNK, msg_dtype=dt, pipe=pipe, mixing=mix, name='cons_w%d' % k)
              for k in range(2)]
    for k, (engines, streams) in enumerate(worlds):
        for step in range(6):
            if k == 1 and step in (2, 4):
                _run_consensus(engines, streams, full=(step == 4))
            for e, s in zip(engines, streams):
                with torch.cuda.stream(s):
                    e.mix(sgd=False)
            torch.cuda.synchronize()
        for e in engines:
            e.check()
    for a, b in zip(worlds[0][0], worlds[1][0]):
        assert torch.equal(a.z, b.z)
        assert a.ps_weight == b.ps_weight and a.device_step == b.device_step == 6


def test_bf16_consensus_falls_to_a_floor():
    """gossip-only steps: fp32 messages contract to fp32 rounding, bf16 messages stop at a floor
    of a few bf16 ulps, which the consensus distance makes visible"""
    curves = {}
    for msg in ('fp32', 'bf16'):
        engines, streams = _mk_world(4, 4 * CHUNK, msg_dtype=BF16 if msg == 'bf16' else None,
                                     spread=1.0, name='floor_' + msg)
        curve = []
        for step in range(41):
            if step % 4 == 0:
                res, _ = _run_consensus(engines, streams, full=False)
                curve.append((res[0][0].item(), res[0][1].item()))
            for e, s in zip(engines, streams):
                with torch.cuda.stream(s):
                    e.mix(sgd=False)
            torch.cuda.synchronize()
        curves[msg] = curve
    bf = [d for d, _ in curves['bf16']]
    fp = [d for d, _ in curves['fp32']]
    nrm = curves['bf16'][-1][1]
    assert bf[0] > 1e3 * max(bf[3:])                 # it falls ...
    assert min(bf[3:]) > 0 and max(bf[3:]) < 20 * min(bf[3:])      # ... and flattens
    assert (bf[-1] / nrm) ** 0.5 < 2 ** -8          # at bf16 resolution
    assert bf[-1] > 100 * fp[-1]                    # which fp32 messages do not have


@pytest.mark.parametrize('algo', ['sgp', 'osgp'])
def test_graphed_trainer_average_model(algo):
    """captured GossipTrainer steps, finish(), then average_model() on every rank: zbar is the
    weighted average of the ranks' arenas, and replays continue without a heartbeat error"""
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    dev = torch.device('cuda', 0)
    n = 3
    lw = LocalWorld(n)
    trainers, streams = [], []
    for r in range(n):
        torch.manual_seed(7 + r)
        net = models.TinyConvNet().to(dev).to(memory_format=torch.channels_last)
        graph = sgp.NPeerDynamicDirectedExponentialGraph(r, n)
        model = GossipDataParallel(net, graph=graph, mixing=sgp.SelfWeightedMixing(graph, dev, self_weight=[0.4, 0.5, 0.6]),
                                   overlap=(algo == 'osgp'), rank=r, world_size=n, heartbeat_timeout=20,
                                   symmetric_world=lw.view(r), transport='nvlink', grid=4,
                                   symmetric_name='cons_trainer')
        model.engine._gather_dma_pref = False        # see test_loopback_graphed_trainer_equals_eager
        model.engine._refresh_in_peers()
        opt = FusedGossipSGD(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True)
        trainers.append(GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=True, warmup_iters=10 ** 6))
        streams.append(torch.cuda.Stream(device=dev))
    gens = [torch.Generator().manual_seed(100 + r) for r in range(n)]

    def steps(k):
        for _ in range(k):
            def rank_step(r):
                x = torch.randn(8, 3, 32, 32, generator=gens[r]).pin_memory()
                y = torch.randint(0, 10, (8,), generator=gens[r]).pin_memory()
                trainers[r].step(x, y)
            _in_threads([functools.partial(rank_step, r) for r in range(n)])
            torch.cuda.synchronize()
        for tr in trainers:
            tr.finish()

    steps(2)
    for tr in trainers:                              # every capture before any replay
        with torch.cuda.stream(tr.stream):
            tr._capture()
    # every virtual rank allocates before any of them enters the collective (an allocation
    # synchronises the shared device, see GossipEngine.prepare_consensus)
    avgs = []
    for tr in trainers:
        tr.model.prepare_consensus()
        avgs.append(torch.empty_like(tr.model.arena.flat))
    torch.cuda.synchronize()
    for rnd in range(2):
        steps(4)

        def rank_avg(r):
            with torch.cuda.stream(streams[r]):
                trainers[r].model.average_model(out=avgs[r])
                torch.cuda.current_stream().synchronize()
        _in_threads([functools.partial(rank_avg, r) for r in range(n)])
        zs = torch.stack([tr.model.arena.flat.double().cpu() for tr in trainers])
        ws = torch.tensor([tr.engine.ps_weight for tr in trainers], dtype=torch.float64)
        assert (ws - 1).abs().max() > 1e-3            # the weighted average is not the plain mean
        zbar = (ws[:, None] * zs).sum(0) / ws.sum()
        for r in range(n):
            assert torch.equal(avgs[r], avgs[0])
            torch.testing.assert_close(avgs[r].double().cpu(), zbar, rtol=1e-5,
                                       atol=1e-6 * zbar.abs().max().item())
            st = trainers[r].model.last_consensus
            assert st == trainers[0].model.last_consensus
            per = ((zs - zbar) ** 2).sum(1)
            assert abs(st.distance_sq - per.mean().item()) <= 1e-4 * per.mean().item()
            torch.testing.assert_close(torch.tensor(st.rank_distance_sq, dtype=torch.float64), per,
                                       rtol=1e-4, atol=0)
    for tr in trainers:
        assert tr.graph is not None
        tr.check()
        assert tr.engine.device_step == 10
