"""sm_90a kernels vs plain PyTorch fp32/fp64 oracles.

Loop-back layout: N virtual ranks on ONE GPU (``LocalWorld``), each with its
own stream and a small grid so that all kernels are co-resident and really spin
on each other's flags.  Multi-GPU tests spawn one process per GPU and go
through the IPC rendezvous.
"""
import pytest
import torch

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops import oracle

pytestmark = pytest.mark.gpu

CHUNK = 4096
PIPE = [True]


@pytest.fixture(autouse=True, params=[True, False], ids=['pipe', 'regs'])
def _step_kernel_variant(request):
    """every test runs with both implementations of the full gossip step: the warp-specialised
    TMA kernel (sgp_step_pipe_kernel, default) and the register-staged one (sgp_step_kernel)"""
    PIPE[0] = request.param
    yield


def _mk_world(n, numel, graph_cls, ppi, mixing_cls=None, with_sgd=True, bf16=False,
              overlap=False, grid=8, seed=0, **graph_kw):
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    from stochastic_gradient_push_b200.ops.peer_mix import GossipEngine
    dev = torch.device('cuda', 0)
    torch.manual_seed(seed)
    lw = LocalWorld(n)
    engines, graphs, mixings, streams = [], [], [], []
    for r in range(n):
        g = graph_cls(r, n, peers_per_itr=ppi, **graph_kw)
        m = (mixing_cls or sgp.UniformMixing)(g, dev)
        z = torch.randn(numel, device=dev)
        grad = torch.randn(numel, device=dev)
        if bf16:
            grad = grad.bfloat16()
        mom = torch.zeros(numel, device=dev)
        shadow = torch.zeros(numel, device=dev, dtype=torch.bfloat16) if bf16 else None
        e = GossipEngine(lw.view(r), z, g, m, grad=grad if with_sgd else None,
                         momentum=mom if with_sgd else None, shadow=shadow,
                         with_residual=overlap, grid=grid, gather_grid=4, timeout_s=10.0,
                         name='t')
        e.ctx.set_pipe(PIPE[0])
        engines.append(e)
        graphs.append(g)
        mixings.append(m)
        streams.append(torch.cuda.Stream(device=dev))
    return engines, graphs, mixings, streams


def _oracle_graphs(graphs, mixing_cls=None):
    n = len(graphs)
    gs = [type(g)(g.rank, n, peers_per_itr=g.peers_per_itr, dedupe=g.dedupe) for g in graphs]
    ms = [(mixing_cls or sgp.UniformMixing)(g, 'cpu') for g in gs]
    return gs, ms


@pytest.mark.parametrize('graph_cls,ppi', [
    (sgp.NPeerDynamicDirectedExponentialGraph, 1),
    (sgp.NPeerDynamicDirectedExponentialGraph, 2),
    (sgp.DynamicDirectedExponentialGraph, 1),
    (sgp.DynamicBipartiteExponentialGraph, 1),
    (sgp.RingGraph, 1),
])
def test_fused_sgd_mix_matches_oracle(graph_cls, ppi):
    n, numel, steps = 4, 3 * CHUNK, 7
    engines, graphs, _, streams = _mk_world(n, numel, graph_cls, ppi)
    ogs, oms = _oracle_graphs(graphs)
    lr, mu, wd, nest = 0.1, 0.9, 1e-4, True
    zs = [e.z.double().clone() for e in engines]
    ms = [e.momentum.double().clone() for e in engines]
    ws = [1.0] * n
    for step in range(steps):
        gs = []
        for e in engines:
            e.grad.normal_()
            gs.append(e.grad.double().clone())
            e.set_hyper(lr, mu, wd, nest)
        torch.cuda.synchronize()
        for e, s in zip(engines, streams):
            with torch.cuda.stream(s):
                e.mix(sgd=True)
        torch.cuda.synchronize()
        xs = []
        for i in range(n):
            x, ms[i] = oracle.sgd_momentum(zs[i] * ws[i], gs[i], ms[i], lr, mu, wd, nest)
            xs.append(x)
        xs, ws = oracle.mix_columns(xs, ws, ogs, oms)
        oracle.rotate_all(ogs)
        zs = [x / w for x, w in zip(xs, ws)]
        for i, e in enumerate(engines):
            e.check()
            assert e.device_step == step + 1
            torch.testing.assert_close(e.z.double(), zs[i], rtol=1e-5, atol=1e-5)
            torch.testing.assert_close(e.momentum.double(), ms[i], rtol=1e-5, atol=1e-5)
            assert e.grad.abs().sum().item() == 0.0           # fused zero_grad
            assert abs(e.ps_weight - ws[i]) < 1e-5


def test_mix_reaches_exact_mean_npdde8():
    """SURVEY 4.4: x0 = 10*r on 8 ranks -> 35 everywhere after 3 mixes."""
    n, numel = 8, CHUNK
    engines, graphs, _, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph,
                                            1, with_sgd=False, grid=1)
    want = {0: [35, 45, 35], 1: [5, 35, 35], 2: [15, 25, 35], 3: [25, 15, 35],
            4: [35, 25, 35], 5: [45, 35, 35], 6: [55, 45, 35], 7: [65, 55, 35]}
    for r, e in enumerate(engines):
        e.z.fill_(10.0 * r)
    for step in range(3):
        torch.cuda.synchronize()
        for e, s in zip(engines, streams):
            with torch.cuda.stream(s):
                e.mix(sgd=False)
        torch.cuda.synchronize()
        for r, e in enumerate(engines):
            e.check()
            assert abs(e.z[0].item() - want[r][step]) < 1e-4
            assert abs(e.z[-1].item() - want[r][step]) < 1e-4


def test_irregular_mixing_tracks_push_sum_weight():
    n, numel, steps = 4, 2 * CHUNK, 9
    import functools
    mix_cls = functools.partial(sgp.SelfWeightedMixing, self_weight=[0.3, 0.5, 0.6, 0.45])
    engines, graphs, _, streams = _mk_world(
        n, numel, sgp.DynamicDirectedExponentialGraph, 1,
        mixing_cls=mix_cls, with_sgd=False)
    ogs, oms = _oracle_graphs(graphs, mix_cls)
    xs = [e.z.double().clone() for e in engines]
    total = sum(xs)
    ws = [1.0] * n
    for _ in range(steps):
        for e, s in zip(engines, streams):
            with torch.cuda.stream(s):
                e.mix(sgd=False)
        torch.cuda.synchronize()
        xs, ws = oracle.mix_columns(xs, ws, ogs, oms)
        oracle.rotate_all(ogs)
    wsum = 0.0
    for i, e in enumerate(engines):
        e.check()
        torch.testing.assert_close(e.z.double(), xs[i] / ws[i], rtol=1e-4, atol=1e-4)
        assert abs(e.ps_weight - ws[i]) < 1e-5
        wsum += e.ps_weight
    assert abs(wsum - n) < 1e-4                     # column stochastic: mass conserved
    assert any(abs(w - 1.0) > 1e-3 for w in ws)     # ... and genuinely irregular
    mass = sum(e.z.double() * e.ps_weight for e in engines)
    torch.testing.assert_close(mass, total, rtol=1e-4, atol=1e-4)


def test_bf16_grads_and_shadow():
    n, numel = 2, 2 * CHUNK
    engines, graphs, _, streams = _mk_world(n, numel, sgp.RingGraph, 1, bf16=True)
    ogs, oms = _oracle_graphs(graphs)
    lr, mu, wd = 0.05, 0.9, 5e-4
    zs = [e.z.double().clone() for e in engines]
    gs = [e.grad.double().clone() for e in engines]        # bf16 values, exactly
    for e in engines:
        e.set_hyper(lr, mu, wd, False)
    torch.cuda.synchronize()
    for e, s in zip(engines, streams):
        with torch.cuda.stream(s):
            e.mix(sgd=True)
    torch.cuda.synchronize()
    xs = [oracle.sgd_momentum(zs[i], gs[i], torch.zeros_like(zs[i]), lr, mu, wd, False)[0]
          for i in range(n)]
    xs, ws = oracle.mix_columns(xs, [1.0] * n, ogs, oms)
    for i, e in enumerate(engines):
        e.check()
        torch.testing.assert_close(e.z.double(), xs[i], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(e.shadow.float(), e.z.bfloat16().float(), rtol=0, atol=0)
        assert e.grad.float().abs().sum().item() == 0.0


@pytest.mark.parametrize('dma', [True, False], ids=['copy-engine-gather', 'kernel-gather'])
def test_overlap_publish_gather_fold_matches_oracle(dma):
    """OSGP arithmetic: x <- x - lr*dir ; x += residual ; publish ; residual of
    step k is folded at step k+1 (1-step stale).  The gather runs either on the copy engines
    (flag-wait kernel + cudaMemcpyAsync of the in-neighbour's outbox + ack kernel; the edge weight
    is applied at fold time) or as the TMA gather kernel."""
    n, numel, steps = 4, 2 * CHUNK, 6
    engines, graphs, _, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph,
                                            1, overlap=True)
    for e in engines:
        assert e.gather_dma                     # one in-neighbour per phase: eligible
        e._gather_dma_pref = dma
        e._refresh_in_peers()
        assert e.gather_dma == dma
    side = [torch.cuda.Stream() for _ in range(n)]
    ogs, oms = _oracle_graphs(graphs)
    lr, mu, wd, nest = 0.1, 0.9, 1e-4, False
    zs = [e.z.double().clone() for e in engines]
    ms = [torch.zeros_like(z) for z in zs]
    ws = [1.0] * n
    res = [torch.zeros_like(z) for z in zs]
    wres = [0.0] * n
    for step in range(steps):
        gs = []
        for e in engines:
            e.grad.normal_()
            gs.append(e.grad.double().clone())
            e.set_hyper(lr, mu, wd, nest, do_sgd=(step > 0))
        torch.cuda.synchronize()
        for e, s in zip(engines, streams):
            with torch.cuda.stream(s):
                e.publish(sgd=True, fold=True)
        torch.cuda.synchronize()
        for e, s in zip(engines, side):
            with torch.cuda.stream(s):
                e.gather()
        torch.cuda.synchronize()
        # oracle
        pub, pubw = [], []
        for i in range(n):
            x = zs[i] * ws[i]
            if step > 0:
                x, ms[i] = oracle.sgd_momentum(x, gs[i], ms[i], lr, mu, wd, nest)
            x = x + res[i]
            w1 = ws[i] + wres[i]
            pub.append(x)
            pubw.append(w1)
        cols = [oms[j].scalar_weights(ogs[j].get_peers()[0]) for j in range(n)]
        for i in range(n):
            self_w = cols[i][0]
            zs[i] = pub[i] / pubw[i]
            ws[i] = self_w * pubw[i]
            _, ins = ogs[i].get_peers()
            res[i] = sum(cols[j][1][i] * pub[j] for j in ins)
            wres[i] = sum(cols[j][1][i] * pubw[j] for j in ins)
        oracle.rotate_all(ogs)
        for i, e in enumerate(engines):
            e.check()
            torch.testing.assert_close(e.z.double(), zs[i], rtol=1e-5, atol=1e-5)
            torch.testing.assert_close(e.residual.double() * e.res_scale, res[i], rtol=1e-5, atol=1e-5)
            assert abs(e.ps_weight - ws[i]) < 1e-6
            assert abs(e.res_weight - wres[i]) < 1e-6
    # flush: fold the last residual without publishing
    for e in engines:
        e.set_hyper(lr, mu, wd, nest, do_sgd=False)
        e.local(sgd=False, fold=True)
    torch.cuda.synchronize()
    for i, e in enumerate(engines):
        x = zs[i] * ws[i] + res[i]
        w = ws[i] + wres[i]
        torch.testing.assert_close(e.z.double(), x / w, rtol=1e-5, atol=1e-5)
        assert abs(e.ps_weight - w) < 1e-6


def test_timeout_sets_status_instead_of_hanging():
    """A peer that never shows up must trip the heartbeat, not hang the GPU."""
    n, numel = 2, CHUNK
    engines, _, _, streams = _mk_world(n, numel, sgp.RingGraph, 1, with_sgd=False, grid=1)
    engines[0].ctx.set_timeout(0.2)
    with torch.cuda.stream(streams[0]):
        engines[0].mix(sgd=False)            # rank 1 never launches
    torch.cuda.synchronize()
    assert engines[0].status == 1
    with pytest.raises(RuntimeError):
        engines[0].check()


def test_sgd_only_world1_matches_torch_optim():
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    from stochastic_gradient_push_b200.ops.peer_mix import GossipEngine
    dev = torch.device('cuda', 0)
    numel = 2 * CHUNK
    g = sgp.NPeerDynamicDirectedExponentialGraph(0, 1)
    z = torch.randn(numel, device=dev)
    p = torch.nn.Parameter(z.clone())
    opt = torch.optim.SGD([p], lr=0.1, momentum=0.9, weight_decay=1e-4, nesterov=True)
    grad = torch.zeros(numel, device=dev)
    e = GossipEngine(LocalWorld(1).view(0), z, g, sgp.UniformMixing(g, dev), grad=grad,
                     momentum=torch.zeros(numel, device=dev), timeout_s=5.0, name='w1')
    e.set_hyper(0.1, 0.9, 1e-4, True)
    for _ in range(4):
        gr = torch.randn(numel, device=dev)
        grad.copy_(gr)
        p.grad = gr.clone()
        opt.step()
        e.mix(sgd=True)
        torch.cuda.synchronize()
        torch.testing.assert_close(e.z, p.data, rtol=1e-5, atol=1e-6)


def test_scale_kernel():
    from stochastic_gradient_push_b200.ops import native
    C = native.load()
    x = torch.randn(CHUNK, device='cuda')
    ref = x.clone()
    s = torch.tensor([0.75], device='cuda')
    sh = torch.zeros(CHUNK, device='cuda', dtype=torch.bfloat16)
    C.scale_(x, s, False, sh)
    torch.testing.assert_close(x, ref * 0.75)
    torch.testing.assert_close(sh, x.bfloat16())
    C.scale_(x, s, True, None)
    torch.testing.assert_close(x, ref, rtol=1e-6, atol=1e-6)


# --------------------------------------------------------------------------- #
# failure handling (SURVEY 5.3): soft heartbeat = counted + retried wait, hard heartbeat = sticky
# status + a VALID parameter state
# --------------------------------------------------------------------------- #
def test_slow_peer_is_waited_for_counted_and_mass_is_conserved():
    import time
    n, numel = 2, 2 * CHUNK
    engines, graphs, _, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1)
    ogs, oms = _oracle_graphs(graphs)
    C = engines[0].C
    for e in engines:
        e._state_i32[C.STATE_OFF_SOFT_TIMEOUT_US // 4] = 50_000        # 50 ms soft, 10 s hard
        e.set_hyper(0.1, 0.9, 0.0, False)
    zs = [e.z.double().clone() for e in engines]
    gs = [e.grad.double().clone() for e in engines]
    torch.cuda.synchronize()
    with torch.cuda.stream(streams[0]):
        engines[0].mix(sgd=True)
    time.sleep(0.4)                                  # rank 1 is 0.4 s late: past the soft heartbeat
    with torch.cuda.stream(streams[1]):
        engines[1].mix(sgd=True)
    torch.cuda.synchronize()
    for e in engines:
        e.check()                                    # no hard failure
    assert engines[0].soft_timeouts >= 1             # ... but the delay was noticed
    engines[0].poll(blocking=True)
    engines[0].poll(blocking=True)                   # (logs the retried wait; must not raise)
    xs = []
    for i in range(n):
        x, _ = oracle.sgd_momentum(zs[i], gs[i], torch.zeros_like(zs[i]), 0.1, 0.9, 0.0, False)
        xs.append(x)
    xs, ws = oracle.mix_columns(xs, [1.0] * n, ogs, oms)
    for i, e in enumerate(engines):
        torch.testing.assert_close(e.z.double(), xs[i] / ws[i], rtol=1e-5, atol=1e-6)
    assert abs(sum(e.ps_weight for e in engines) - n) < 1e-5          # push-sum mass conserved


def test_dead_peer_trips_the_heartbeat_and_leaves_valid_parameters():
    n, numel = 2, 2 * CHUNK
    engines, graphs, _, streams = _mk_world(n, numel, sgp.NPeerDynamicDirectedExponentialGraph, 1)
    e = engines[0]
    e.ctx.set_timeout(0.3)
    e.set_hyper(0.1, 0.0, 0.0, False)
    z0, g0 = e.z.double().clone(), e.grad.double().clone()
    with torch.cuda.stream(streams[0]):
        e.mix(sgd=True)                              # rank 1 never launches
    torch.cuda.synchronize()
    with pytest.raises(NameError, match='Gossip flag timeout'):
        e.poll(blocking=True)
    with pytest.raises(RuntimeError):
        e.check()
    # every in-message was lost, nothing stale: z is the de-biased SGD result of this step
    torch.testing.assert_close(e.z.double(), z0 - 0.1 * g0, rtol=1e-6, atol=1e-7)
    assert e.device_step == 1
    e.clear_status()
    e.poll(blocking=True)                            # healthy again after the application cleared it
