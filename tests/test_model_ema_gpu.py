"""ModelEma on the GPU: ``ema_update_kernel`` against an fp64 emulation of its fmaf sequence (fp32
and bf16 sources, heads, tails, many small segments), the warm-up decay and the device counter,
CUDA-graph replay with decay changes, the loop-back GossipTrainer with ``ema=`` (graphed and eager,
SGP / OSGP / world 1) against an EMA rebuilt from per-step snapshots, ``applied()`` with the bf16
compute shadow, and state_dict round trips."""
import functools

import numpy as np
import pytest
import torch
import torch.nn as nn

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops.model_ema import ModelEma, decay_at

from test_gdp_loopback_gpu import _in_threads

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda', 0)


def _emulate(e, s, d_t):
    """fmaf(1 - d_t, s - e, e): fp32 w and s - e, the exact product and the sum in fp64"""
    w = float(np.float32(1.0) - np.float32(d_t))
    return ((s.float() - e).double() * w + e.double()).float()


def _ulps(a, b):
    """largest distance in fp32 units in the last place (same-sign values)"""
    ia = a.contiguous().view(torch.int32).long()
    ib = b.contiguous().view(torch.int32).long()
    return int((ia - ib).abs().max().item()) if a.numel() else 0


class _Bag(nn.Module):
    """parameters of numel 1, 3, 64, 4099 and 1 << 20, a misaligned view and 60 tiny buffers"""

    def __init__(self, dtype):
        super().__init__()
        g = torch.Generator().manual_seed(5)

        def make(n):                       # created on the device: Module.to() would re-align a view
            return torch.randn(n, generator=g).to(device=DEV, dtype=dtype)
        for i, n in enumerate((1, 3, 64, 4099, 1 << 20)):
            setattr(self, 'p%d' % i, nn.Parameter(make(n)))
        self.register_buffer('odd', make(8200)[3:3 + 4101])     # source 16-byte misaligned: scalar head
        for i in range(60):
            self.register_buffer('t%d' % i, make(1 + i % 7))

    def srcs(self):
        return {k: v for k, v in self.state_dict(keep_vars=True).items()}


def _perturb(bag, g):
    with torch.no_grad():
        for v in bag.srcs().values():
            v.add_(torch.randn(v.shape, generator=g).to(v.dtype).to(v.device))


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('decay,warmup', [(0.9, False), (0.99, True)])
def test_kernel_matches_fp64_emulation_and_lerp(dtype, decay, warmup):
    bag = _Bag(dtype)
    assert bag.odd.data_ptr() % 16 != 0
    ema = ModelEma(bag, decay=decay, warmup=warmup)
    assert len(ema._segs) == 5 + 1 + 60
    ref = {k: v.detach().float().clone() for k, v in bag.srcs().items()}
    g = torch.Generator().manual_seed(11)
    for t in range(5):
        _perturb(bag, g)
        ema.update()
        d = decay_at(decay, warmup, t)
        w = float(np.float32(1.0) - d)
        got = ema.state_dict()['state_dict']
        for k, s in bag.srcs().items():
            s = s.detach()
            lerp = torch.lerp(ref[k], s.float(), w)
            ref[k] = _emulate(ref[k], s, d)
            out = got[k].to(DEV)
            assert _ulps(out, ref[k]) <= 1, (t, k)
            torch.testing.assert_close(out, lerp, rtol=1e-6, atol=1e-6 * float(lerp.abs().max()))
            ref[k] = out                       # continue from the kernel's bits
    assert ema.num_updates == 5


@pytest.mark.parametrize('decay', [0.9999, 0.5])
def test_warmup_decay_and_counter(decay):
    bag = _Bag(torch.float32)
    ema = ModelEma(bag, decay=decay, warmup=True)
    e = {k: v.detach().clone() for k, v in bag.srcs().items()}
    g = torch.Generator().manual_seed(2)
    for t in range(21):
        assert ema.num_updates == t
        _perturb(bag, g)
        ema.update()
        got = ema.state_dict()['state_dict']
        d = decay_at(decay, True, t)
        assert d == min(np.float32(decay), np.float32(np.float32(1 + t) / np.float32(10 + t)))
        for k, s in bag.srcs().items():
            e[k] = _emulate(e[k], s.detach(), d)
            assert _ulps(got[k].to(DEV), e[k]) <= 1, (t, k)
            e[k] = got[k].to(DEV)
    assert ema.num_updates == 21


def test_graph_replay_with_decay_changes_matches_eager():
    torch.manual_seed(0)
    bag_g, bag_e = _Bag(torch.float32), _Bag(torch.float32)
    ema_g = ModelEma(bag_g, decay=0.9, warmup=True)
    ema_e = ModelEma(bag_e, decay=0.9, warmup=True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        ema_g.update()
    torch.cuda.synchronize()
    assert ema_g.num_updates == 0                     # capture does not execute
    gg, ge = torch.Generator().manual_seed(4), torch.Generator().manual_seed(4)
    for i in range(30):
        if i % 7 == 3:
            ema_g.set_decay(0.5 + 0.01 * i)
            ema_e.set_decay(0.5 + 0.01 * i)
        _perturb(bag_g, gg)
        _perturb(bag_e, ge)
        graph.replay()
        ema_e.update()
    torch.cuda.synchronize()
    assert torch.equal(ema_g.ema, ema_e.ema)
    assert ema_g.num_updates == 30 and ema_e.num_updates == 30


# --------------------------------------------------------------------------- #
# loop-back trainer
# --------------------------------------------------------------------------- #
def _snap(net):
    return {k: v.detach().float().cpu().clone() for k, v in net.state_dict().items() if v.is_floating_point()}


def _train(n, algo, steps, use_graph, with_ema, tag):
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    from stochastic_gradient_push_b200.parallel.trainer import GossipTrainer
    lw = LocalWorld(n)
    trainers, emas, snaps = [], [], [[] for _ in range(n)]
    for r in range(n):
        torch.manual_seed(7 + r)
        net = models.TinyConvNet().to(DEV).to(memory_format=torch.channels_last)
        model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(r, n),
                                   overlap=(algo == 'osgp'), rank=r, world_size=n, heartbeat_timeout=20,
                                   symmetric_world=lw.view(r), transport='nvlink', grid=4,
                                   symmetric_name='loopback_ema_' + tag)
        if use_graph and algo == 'osgp':
            model.engine._gather_dma_pref = False         # (see test_gdp_loopback_gpu)
            model.engine._refresh_in_peers()
        opt = FusedGossipSGD(model, lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=True)
        ema = ModelEma(model, decay=0.7, warmup=True) if with_ema else None
        emas.append(ema)
        snaps[r].append(_snap(net))
        trainers.append(GossipTrainer(model, opt, amp_dtype=None, use_cuda_graph=use_graph,
                                      warmup_iters=10 ** 6, ema=ema))
    gens = [torch.Generator().manual_seed(100 + r) for r in range(n)]
    for s in range(steps):
        if use_graph and s == 2:
            for tr in trainers:              # every capture before any replay
                with torch.cuda.stream(tr.stream):
                    tr._capture()

        def rank_step(r):
            x = torch.randn(8, 3, 32, 32, generator=gens[r]).pin_memory()
            y = torch.randint(0, 10, (8,), generator=gens[r]).pin_memory()
            trainers[r].step(x, y)
        _in_threads([functools.partial(rank_step, r) for r in range(n)])
        torch.cuda.synchronize()
        for r in range(n):                   # what the EMA of step s saw: nothing runs after it
            snaps[r].append(_snap(trainers[r].model.module))
    launches = [tr.own_launches_per_step for tr in trainers]
    for tr in trainers:
        tr.finish()
        assert (tr.graph is not None) == use_graph
    return trainers, emas, snaps, launches


@pytest.mark.parametrize('n,algo', [(2, 'sgp'), (2, 'osgp'), (1, 'local')])
def test_loopback_trainer_ema_graphed_equals_eager_and_snapshots(n, algo):
    steps = 8
    runs = {}
    for name, graph, ema in (('base', True, False), ('eager', False, True), ('graph', True, True)):
        runs[name] = _train(n, algo, steps, graph, ema, '%s_%s' % (algo, name))
    _, _, _, base_launches = runs['base']
    _, _, _, ema_launches = runs['graph']
    assert [b + 1 for b in base_launches] == ema_launches
    for name in ('eager', 'graph'):
        _, emas, snaps, _ = runs[name]
        for r in range(n):
            assert emas[r].num_updates == steps
            got = emas[r].state_dict()['state_dict']
            ref = dict(snaps[r][0])
            assert set(got) == set(ref)
            for t in range(steps):
                d = decay_at(0.7, True, t)
                ref = {k: _emulate(ref[k], snaps[r][t + 1][k], d) for k in ref}
            for k in ref:
                assert _ulps(got[k], ref[k]) <= steps, (name, r, k)     # <= 1 ulp per step
                torch.testing.assert_close(got[k], ref[k], rtol=1e-6, atol=1e-7)
    for r in range(n):
        e = runs['eager'][1][r].state_dict()['state_dict']
        g = runs['graph'][1][r].state_dict()['state_dict']
        for k in e:
            # the two runs' parameters agree to within the float-atomic reorderings of two runs of a step
            torch.testing.assert_close(g[k], e[k], rtol=1e-4, atol=1e-5)


def test_applied_swaps_ema_in_with_the_bf16_shadow_and_restores_bits():
    from stochastic_gradient_push_b200 import models
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    torch.manual_seed(3)
    net = models.TinyConvNet().to(DEV).to(memory_format=torch.channels_last)
    model = GossipDataParallel(net, graph=sgp.NPeerDynamicDirectedExponentialGraph(0, 1), rank=0, world_size=1,
                               heartbeat_timeout=20, compute_dtype=torch.bfloat16)
    assert model.compute_shadow is not None
    ema = ModelEma(model, decay=0.6)
    g = torch.Generator(device=DEV).manual_seed(1)
    for _ in range(3):
        with torch.no_grad():
            model.arena.flat.add_(torch.randn(model.arena.flat.shape, generator=g, device=DEV))
            model.compute_shadow.copy_(model.arena.flat)
            net.train()
            net(torch.randn(4, 3, 32, 32, device=DEV).contiguous(memory_format=torch.channels_last))
        ema.update()
    flat, shadow = model.arena.flat.clone(), model.compute_shadow.clone()
    bufs = {k: v.clone() for k, v in net.state_dict().items()}
    fresh = models.TinyConvNet().to(DEV).to(memory_format=torch.channels_last)
    fresh.load_state_dict(ema.state_dict()['state_dict'], strict=False)
    fresh.eval()
    x = torch.randn(6, 3, 32, 32, device=DEV).contiguous(memory_format=torch.channels_last)
    net.eval()
    with torch.no_grad(), ema.applied():
        inside = net(x)
        assert torch.equal(model.compute_shadow, model.arena.flat.to(torch.bfloat16))
        for k, v in ema.state_dict()['state_dict'].items():
            assert torch.equal(net.state_dict()[k].cpu(), v), k
        expect = fresh(x)
    torch.testing.assert_close(inside, expect, rtol=1e-6, atol=1e-6)
    assert torch.equal(model.arena.flat, flat) and torch.equal(model.compute_shadow, shadow)
    for k, v in net.state_dict().items():
        assert torch.equal(v, bufs[k]), k


def test_state_dict_round_trip_continues_with_the_same_bits():
    bag = _Bag(torch.float32)
    a = ModelEma(bag, decay=0.8, warmup=True)
    g = torch.Generator().manual_seed(9)
    for _ in range(3):
        _perturb(bag, g)
        a.update()
    b = ModelEma(bag, decay=0.1)
    b.load_state_dict(a.state_dict())
    assert (b.decay, b.warmup, b.num_updates) == (0.8, True, 3)
    for _ in range(4):
        _perturb(bag, g)
        a.update()
        b.update()
    assert torch.equal(a.ema, b.ema) and b.num_updates == 7
