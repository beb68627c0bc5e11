"""SlowMo on the kernel plane (``GossipEngine.slowmo``, ``GossipTrainer`` with
``slowmo_frequency > 0``): N virtual ranks on one GPU (``LocalWorld`` loop-back) against fp64
references, bit-identical results on every rank, gossip that continues as if the parameters had been
set by hand, the captured trainer against the eager one, and the heartbeat path."""
import functools

import pytest
import torch

import stochastic_gradient_push_b200 as sgp

from test_gdp_loopback_gpu import _in_threads

pytestmark = pytest.mark.gpu

CHUNK = 4096
BF16 = torch.bfloat16


def _mk_world(n, numel, msg_dtype=None, mixing=None, shadow=True, name='slowmo', seed=0, timeout_s=10.0):
    """n engines (with a bf16 shadow) and their SlowMo buffers u, x_prev"""
    from stochastic_gradient_push_b200.ops.peer_mix import GossipEngine
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    dev = torch.device('cuda', 0)
    gen = torch.Generator().manual_seed(seed)
    base = torch.randn(numel, generator=gen)
    lw = LocalWorld(n)
    ranks = []
    for r in range(n):
        g = sgp.NPeerDynamicDirectedExponentialGraph(r, n)
        m = mixing(g, dev) if mixing else sgp.UniformMixing(g, dev)
        z = (base + 0.5 * torch.randn(numel, generator=gen)).to(dev)
        sh = z.to(BF16) if shadow else None
        e = GossipEngine(lw.view(r), z, g, m, shadow=sh, grid=8, timeout_s=timeout_s, name=name,
                         msg_dtype=msg_dtype)
        ranks.append(dict(e=e, s=torch.cuda.Stream(device=dev), u=torch.zeros_like(z), xp=torch.zeros_like(z)))
    return ranks


def _slowmo(ranks, lr, alpha, beta, init):
    """enqueue every rank's call on its own stream, then synchronise"""
    torch.cuda.synchronize()
    for rk in ranks:
        with torch.cuda.stream(rk['s']):
            rk['e'].slowmo(rk['u'], rk['xp'], lr, alpha, beta, init)
    torch.cuda.synchronize()
    for rk in ranks:
        rk['e'].check()


def _close(got, ref):
    """1e-6 relative to the tensor's largest element"""
    err = (got.double().cpu() - ref).abs().max().item()
    assert err <= 1e-6 * ref.abs().max().item(), err


@pytest.mark.parametrize('msg', ['fp32', 'bf16'])
@pytest.mark.parametrize('n', [3, 4])
@pytest.mark.parametrize('chunks', ['7', 'grid+7'])
def test_slowmo_matches_fp64(n, msg, chunks):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    # 7 chunks: a chunk per CTA; 2 * SMs + 7: seven CTAs take a second chunk
    nchunks = 7 if chunks == '7' else 2 * sms + 7
    ranks = _mk_world(n, nchunks * CHUNK, msg_dtype=BF16 if msg == 'bf16' else None)
    gen = torch.Generator().manual_seed(1)
    lr, alpha, beta = 0.05, 0.8, 0.6
    u = xp = None
    for call in range(3):
        if call:
            for rk in ranks:                     # the ranks drift apart again between calls
                rk['e'].z.add_((2.0 * torch.randn(rk['e'].n, generator=gen)).cuda())
        for r, rk in enumerate(ranks):
            rk['e'].ps_weight = 0.55 + 0.3 * r + 0.1 * call      # irregular mixing: w != 1
        zs = torch.stack([rk['e'].z.double().cpu() for rk in ranks])
        ws = torch.tensor([rk['e'].ps_weight for rk in ranks], dtype=torch.float64)
        zbar = (ws[:, None] * zs).sum(0) / ws.sum()
        if call == 0:
            u, xp = torch.zeros_like(zbar), zbar
        else:
            u = beta * u + (xp - zbar) / lr
            xp = xp - alpha * lr * u
        _slowmo(ranks, lr, alpha, beta, init=(call == 0))
        r0 = ranks[0]
        for rk in ranks:
            e = rk['e']
            assert torch.equal(e.z, r0['e'].z) and torch.equal(rk['u'], r0['u']) and \
                torch.equal(rk['xp'], r0['xp']), 'ranks differ'
            assert torch.equal(e.z, rk['xp'])
            assert torch.equal(e.shadow, e.z.to(BF16))
            off = e.C.STATE_OFF_PSW // 4
            assert e._state_f32[off: off + 2].tolist() == [1.0, 1.0]
            assert e.device_step == 0
        if call == 0:
            assert (r0['u'] == 0).all()
        _close(r0['xp'], xp)
        _close(r0['u'], u)
        _close(r0['e'].z, xp)


@pytest.mark.parametrize('msg', ['fp32', 'bf16'])
def test_gossip_after_slowmo_is_unchanged(msg):
    """the call leaves the step counter and the sequence numbers alone: five gossip steps after it
    give the bits of a world whose z and w were set to the same values by hand"""
    dt = BF16 if msg == 'bf16' else None
    mix = functools.partial(sgp.SelfWeightedMixing, self_weight=[0.3, 0.5, 0.6, 0.45])
    worlds = [_mk_world(4, 5 * CHUNK, msg_dtype=dt, mixing=mix, shadow=False, name='slowmo_w%d' % k)
              for k in range(2)]

    def mix_steps(ranks, k):
        for _ in range(k):
            for rk in ranks:
                with torch.cuda.stream(rk['s']):
                    rk['e'].mix(sgd=False)
            torch.cuda.synchronize()
    for ranks in worlds:
        mix_steps(ranks, 3)
    called, by_hand = worlds
    assert called[0]['e'].ps_weight != 1.0
    _slowmo(called, 0.1, 1.0, 0.5, init=True)
    for rk in called:
        rk['e'].z.add_(0.01 * rk['e'].rank)          # an update call needs x_prev != zbar
    _slowmo(called, 0.1, 1.0, 0.5, init=False)
    for a, b in zip(called, by_hand):
        b['e'].z.copy_(a['e'].z)
        b['e'].ps_weight = 1.0
    for ranks in worlds:
        mix_steps(ranks, 5)
    for a, b in zip(called, by_hand):
        a['e'].check()
        b['e'].check()
        assert torch.equal(a['e'].z, b['e'].z)
        assert a['e'].ps_weight == b['e'].ps_weight and a['e'].device_step == b['e'].device_step == 8


def _trainers(n, algo, use_graph, tau):
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
        graph = sgp.NPeerDynamicDirectedExponentialGraph(r, n)
        model = GossipDataParallel(net, graph=graph, mixing=sgp.SelfWeightedMixing(graph, dev, self_weight=[0.4, 0.6]),
                                   overlap=(algo == 'osgp'), rank=r, world_size=n, heartbeat_timeout=20,
                                   symmetric_world=lw.view(r), transport='nvlink', grid=4,
                                   symmetric_name='slowmo_trainer', slowmo_frequency=tau, slowmo_lr=0.9,
                                   slowmo_momentum=0.5)
        if algo == 'osgp':
            assert model.engine.gather_dma, 'the copy-engine gather is expected on this schedule'
        opt = FusedGossipSGD(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True)
        trainers.append(GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=use_graph, warmup_iters=10 ** 6))
    return trainers


@pytest.mark.parametrize('algo', ['sgp', 'osgp'])
def test_graphed_trainer_with_slowmo_equals_eager(algo):
    n, steps, tau = 2, 7, 2
    results = []
    for use_graph in (False, True):
        trainers = _trainers(n, algo, use_graph, tau)
        gens = [torch.Generator().manual_seed(100 + r) for r in range(n)]

        def run(s):
            def rank_step(r):
                x = torch.randn(8, 3, 32, 32, generator=gens[r]).pin_memory()
                y = torch.randint(0, 10, (8,), generator=gens[r]).pin_memory()
                trainers[r].step(x, y)
            _in_threads([functools.partial(rank_step, r) for r in range(n)])
            torch.cuda.synchronize()
        for s in range(steps):
            if use_graph and s == 2:
                # every rank's graphs before any replay (a capture synchronises the device, which
                # must not happen while another virtual rank's replay waits for our flags); with
                # the copy-engine gather one graph per (schedule row, parity)
                for tr in trainers:
                    e = tr.engine
                    keys = 2 * e.period if tr._graph_key() is not None else 1
                    with torch.cuda.stream(tr.stream):
                        for d in range(keys):
                            e.steps += d
                            tr._capture()
                            e.steps -= d
            run(s)
        assert all(tr.model._slowmo_calls == steps for tr in trainers)
        for tr in trainers:
            tr.finish()
        results.append([(tr.model.arena.flat.cpu().clone(), tr.engine.device_step) for tr in trainers])
        assert all((tr.graph is not None) == use_graph for tr in trainers)
        if use_graph:
            # one more step makes a SlowMo step: the ranks agree exactly, and finish() after it
            # does not apply the drained update a second time
            run(steps)
            for tr in trainers:
                tr.model.prepare_consensus()
            torch.cuda.synchronize()
            before = [tr.model.arena.flat.clone() for tr in trainers]
            for tr in trainers:
                tr.finish()
            assert all(torch.equal(b, tr.model.arena.flat) for b, tr in zip(before, trainers))
            assert torch.equal(before[0], before[1])
            dsq = [None] * n

            def rank_cons(r):
                with torch.cuda.stream(trainers[r].stream):
                    dsq[r] = trainers[r].model.consensus_distance().distance_sq
            _in_threads([functools.partial(rank_cons, r) for r in range(n)])
            assert dsq == [0.0] * n
            for tr in trainers:
                assert tr.engine.ps_weight == 1.0 and tr.engine.device_step == steps + 1
                tr.check()
    eager, graphed = results
    for r in range(n):
        torch.testing.assert_close(graphed[r][0], eager[r][0], rtol=1e-4, atol=1e-5)
        assert graphed[r][1] == eager[r][1] == steps


def test_heartbeat_timeout_leaves_the_state_untouched():
    """one virtual rank never enters the collective: the bounded barrier wait trips the heartbeat,
    poll() raises, and z, u, x_prev and w are what they were"""
    ranks = _mk_world(2, 2 * CHUNK, name='slowmo_dead')
    rk = ranks[0]
    e = rk['e']
    e.ctx.set_timeout(0.3)
    e.ps_weight = 0.75
    rk['u'].normal_()
    rk['xp'].normal_()
    torch.cuda.synchronize()
    before = [t.clone() for t in (e.z, rk['u'], rk['xp'], e.shadow)]
    with torch.cuda.stream(rk['s']):
        e.slowmo(rk['u'], rk['xp'], 0.1, 1.0, 0.5, False)        # rank 1 never calls it
        with pytest.raises(NameError, match='Gossip flag timeout'):
            e.poll(blocking=True)
    for b, t in zip(before, (e.z, rk['u'], rk['xp'], e.shadow)):
        assert torch.equal(b, t) and torch.isfinite(t.float()).all()
    off = e.C.STATE_OFF_PSW // 4
    assert e._state_f32[off: off + 2].tolist() == [0.75, 0.75]
    e.clear_status()
