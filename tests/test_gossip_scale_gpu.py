"""The gossip kernels at the sizes where a CTA handles many chunks: N virtual ranks on one GPU
(``LocalWorld`` loop-back) against fp64 oracles, and bit-for-bit invariance under the work split.

A real ResNet-50 arena is 6240 chunks of 4096 floats, about 24 per CTA and step.  At that size the
step kernels cut a CTA's chunks into several multi-chunk publish segments, the 4-stage ring of
``sgp_step_pipe_kernel`` wraps many times, and the 6-stage ``TmaRing`` of the TMA gather, the
consensus kernels and SlowMo refills.  Each test states which of those paths its shape reaches,
computed in Python the way ``cta_chunks`` / ``clamped_segments`` compute it, so that the claim
cannot silently stop being true.

  A  the full synchronous step (``mix(sgd=True)``), both kernels, all six <MSG_BF16, GROUPS, LARS>
     variants, against fp64; and identical bits for any grid, segment count and kernel mix
  B  Overlap-SGP: publish with fold, then the TMA, register and copy-engine gathers
  C  consensus and SlowMo over a ResNet-50-sized arena
  D  one ResNet-50-sized synchronous step, both kernels, fp32 and bf16 + groups + LARS
"""
import functools
import gc
import itertools

import pytest
import torch

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops import oracle

pytestmark = pytest.mark.gpu

CHUNK = 4096
BF16 = torch.bfloat16
PIPE_STAGES = 4              # ring of sgp_step_pipe_kernel
RING_STAGES = 6              # TmaRing: TMA gather, consensus, SlowMo
RESNET50_CHUNKS = -(-25_557_032 // CHUNK)        # 6240

# id: (chunks, step grid, segments)
SHAPES = {
    'S1': (37, 8, 4),        # 5 or 4 chunks per CTA; segments 1,1,1,2 and 1,1,1,1
    'S2': (213, 16, 4),      # 14 or 13 chunks per CTA
    'S3': (40, 1, 15),       # one CTA, 15 segments of 2-3 chunks
    'S4': (9, 8, 15),        # empty segments between non-empty ones
    'S5': (213, 16, 1),      # one segment: one flag wait, then the whole ring
}
# id: (graph class, ranks, peers per iteration)
TOPOS = {
    'npdde4x1': (sgp.NPeerDynamicDirectedExponentialGraph, 4, 1),
    'npdde4x2': (sgp.NPeerDynamicDirectedExponentialGraph, 4, 2),
    'ring4': (sgp.RingGraph, 4, 1),
    'npdde8x3': (sgp.NPeerDynamicDirectedExponentialGraph, 8, 3),
    'npdde2x1': (sgp.NPeerDynamicDirectedExponentialGraph, 2, 1),
}
A_TOPOS = ['npdde4x1', 'npdde4x2', 'ring4', 'npdde8x3']      # (D runs two ranks)
# id: (message dtype, parameter groups, LARS)
VARIANTS = {
    'fp32': (None, False, False),
    'fp32-groups': (None, True, False),
    'fp32-groups-lars': (None, True, True),
    'bf16': (BF16, False, False),
    'bf16-groups': (BF16, True, False),
    'bf16-groups-lars': (BF16, True, True),
}
HYPER = (0.1, 0.9, 1e-4, True)
GROUP_ROWS = [(0.1, 0.9, 1e-4, True), (0.02, 0.5, 0.0, False), (0.3, 0.0, 3e-3, False)]
# LARS: group 0 without LARS or decay, group 1 with both
LARS_ROWS = [(0.1, 0.9, 0.0, True), (0.2, 0.9, 1e-3, False)]
LARS_ENABLED = (False, True)
ETA, EPS = 0.02, 1e-8
# tensor sizes, repeated over the arena: many chunks, less than a chunk, boundaries inside chunks
LARS_PATTERN = [int(2.6 * CHUNK), 37, 4200, 900, 1, 1500, 9 * CHUNK + 123]
LARS_GROUP_OF = [1, 0, 1, 0, 0, 1, 1]

_names = itertools.count()


# --------------------------------------------------------------------------------------------- #
# work decomposition, as the kernels compute it
# --------------------------------------------------------------------------------------------- #
def _cta_chunks(nchunks, grid, b):
    """cta_chunks: CTA b of `grid` owns chunks b, b + grid, ..."""
    return (nchunks - 1 - b) // grid + 1 if nchunks > b else 0


def _segment_sizes(chunks, segments):
    """the it_lo / it_hi split of one CTA's chunks into publish segments"""
    return [chunks * (s + 1) // segments - chunks * s // segments for s in range(segments)]


def _split(nchunks, grid, segments):
    per_cta = [_cta_chunks(nchunks, grid, b) for b in range(grid)]
    return per_cta, [_segment_sizes(c, segments) for c in per_cta]


def _check_shape(sid, e, n_in):
    """what shape `sid` exercises in the step kernels, for the grid and segments `e` launches with"""
    per_cta, segs = _split(e.n // CHUNK, e.grid, e.ctx.segments())
    claims = {
        'S1': set(per_cta) == {4, 5} and segs[0] == [1, 1, 1, 2] and segs[-1] == [1, 1, 1, 1],
        'S2': set(per_cta) == {13, 14} and max(max(s) for s in segs) > 1,
        'S3': per_cta == [40] and len(segs[0]) == 15 and set(segs[0]) == {2, 3},
        'S4': per_cta[0] == 2 and set(per_cta[1:]) == {1} and segs[0].index(1) > 0
              and 0 in segs[0][segs[0].index(1):],
        'S5': len(segs[0]) == 1 and segs[0][0] == per_cta[0] > PIPE_STAGES,
    }
    assert claims[sid], (sid, per_cta, segs)
    if sid != 'S4':          # (S4 is about empty segments; its CTAs pull at most 2 x n_in items)
        assert max(per_cta) * n_in > PIPE_STAGES, 'the pipe ring does not wrap'
    return per_cta


# --------------------------------------------------------------------------------------------- #
# harness
# --------------------------------------------------------------------------------------------- #
@functools.lru_cache(maxsize=None)
def _max_grid():
    """co-resident CTAs of the step kernels on this device"""
    from stochastic_gradient_push_b200.ops.peer_mix import GossipEngine
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    g = sgp.NPeerDynamicDirectedExponentialGraph(0, 1)
    z = torch.zeros(CHUNK, device='cuda')
    return GossipEngine(LocalWorld(1).view(0), z, g, sgp.UniformMixing(g, z.device), timeout_s=10.0,
                        name='scale_probe').max_grid


def _in_degree(topo):
    graph_cls, n, ppi = TOPOS[topo]
    return max(len(ins) for _, ins in graph_cls(0, n, peers_per_itr=ppi).phases())


def _world(topo, nchunks, *, grid, segments=4, gather_grid=None, msg_dtype=None, with_residual=False,
           pipe=True, shadow=True, seed=0):
    """one engine and one stream per virtual rank; `pipe`: one bool for every rank or one per rank"""
    from stochastic_gradient_push_b200.ops.peer_mix import GossipEngine
    from stochastic_gradient_push_b200.parallel.symmetric import LocalWorld
    graph_cls, n, ppi = TOPOS[topo]
    dev = torch.device('cuda', 0)
    gen = torch.Generator(device=dev).manual_seed(seed)
    numel = nchunks * CHUNK
    lw = LocalWorld(n)
    name = 'scale%d' % next(_names)
    pipes = list(pipe) if isinstance(pipe, (list, tuple)) else [pipe] * n
    engines, streams = [], []
    for r in range(n):
        g = graph_cls(r, n, peers_per_itr=ppi)
        if topo == 'npdde8x3':
            assert all(len(ins) == 3 for _, ins in g.phases())
        e = GossipEngine(lw.view(r), torch.randn(numel, device=dev, generator=gen), g,
                         sgp.UniformMixing(g, dev), grad=torch.zeros(numel, device=dev),
                         momentum=0.1 * torch.randn(numel, device=dev, generator=gen),
                         shadow=torch.zeros(numel, device=dev, dtype=BF16) if shadow else None,
                         with_residual=with_residual, grid=grid, gather_grid=gather_grid, timeout_s=10.0,
                         name=name, segments=segments, msg_dtype=msg_dtype)
        e.ctx.set_pipe(pipes[r])
        engines.append(e)
        streams.append(torch.cuda.Stream(device=dev))
    # the virtual ranks spin on each other's flags: all their CTAs must be resident at once
    assert n * engines[0].grid <= engines[0].max_grid, (n, engines[0].grid, engines[0].max_grid)
    return engines, streams


def _oracle_graphs(topo):
    graph_cls, n, ppi = TOPOS[topo]
    gs = [graph_cls(r, n, peers_per_itr=ppi) for r in range(n)]
    return gs, [sgp.UniformMixing(g, 'cpu') for g in gs]


def _set_grads(engines, seed, step):
    gen = torch.Generator(device=engines[0].device).manual_seed(1000 * seed + step)
    for e in engines:
        e.grad.copy_(torch.randn(e.n, device=e.device, generator=gen))


def _mix_all(engines, streams):
    torch.cuda.synchronize()
    for e, s in zip(engines, streams):
        with torch.cuda.stream(s):
            e.mix(sgd=True)
    torch.cuda.synchronize()
    for e in engines:
        e.check()


def _free():
    gc.collect()
    torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------------- #
# parameter groups and LARS
# --------------------------------------------------------------------------------------------- #
def _f32(v):
    return torch.tensor(v, dtype=torch.float32)


def _lars_layout(numel):
    """(offsets, numels, group of each tensor): LARS_PATTERN over the arena, 64-aligned offsets, the
    last tensor running to the end"""
    offs, nums, groups, off, k = [], [], [], 0, 0
    while off < numel:
        n = min(LARS_PATTERN[k % len(LARS_PATTERN)], numel - off)
        offs.append(off)
        nums.append(n)
        groups.append(LARS_GROUP_OF[k % len(LARS_GROUP_OF)])
        off = (off + n + 63) // 64 * 64
        k += 1
    return offs, nums, groups


class _Setup(object):
    """the hyper-parameters of one variant as the kernels see them, per element (fp32), and the
    LARS layout"""

    def __init__(self, variant, numel, dev, seed=5):
        _, groups, lars = VARIANTS[variant]
        self.lars = lars
        self.rows = None
        if lars:
            self.offs, self.nums, tgroup = _lars_layout(numel)
            bgroup = torch.zeros(numel // 64, dtype=torch.uint8)
            btensor = torch.zeros(numel // 64, dtype=torch.long)
            for t, (o, n, gi) in enumerate(zip(self.offs, self.nums, tgroup)):
                bgroup[o // 64:(o + n + 63) // 64] = gi
                btensor[o // 64:(o + n + 63) // 64] = t
            self.rows = LARS_ROWS
            self.enabled = [LARS_ENABLED[gi] for gi in tgroup]
            self.bmap = bgroup.to(dev)
            self.elem_tensor = btensor.to(dev).repeat_interleave(64)
            # tensor of each element inside a tensor (not its 64-alignment padding), -1 elsewhere
            owner = torch.full((numel,), -1, dtype=torch.long)
            for t, (o, n) in enumerate(zip(self.offs, self.nums)):
                owner[o:o + n] = t
            self.owner = owner.to(dev)
            wd = torch.tensor([LARS_ROWS[gi][2] for gi in tgroup], dtype=torch.float32)
            self.tensor_wd = wd.double().to(dev)
            self.tensor_on = torch.tensor(self.enabled, device=dev)
        elif groups:
            g = torch.Generator().manual_seed(seed)
            self.bmap = torch.randint(0, len(GROUP_ROWS), (numel // 64,), generator=g, dtype=torch.uint8).to(dev)
            self.rows = GROUP_ROWS
        if self.rows is None:
            lr, mu, wd, nest = HYPER
            self.lr, self.mu, self.wd = (_f32(v).to(dev) for v in (lr, mu, wd))
            self.nest = torch.tensor(nest, device=dev)
        else:
            idx = self.bmap.long().repeat_interleave(64)
            t = torch.tensor([r[:3] for r in self.rows], dtype=torch.float32, device=dev)
            self.lr, self.mu, self.wd = t[:, 0][idx], t[:, 1][idx], t[:, 2][idx]
            self.nest = torch.tensor([bool(r[3]) for r in self.rows], device=dev)[idx]

    def configure(self, engines):
        for e in engines:
            if self.rows is None:
                e.set_hyper(*HYPER)
                continue
            e.set_param_groups(self.bmap, len(self.rows))
            e.set_hyper(0.5, 0.5, 0.5, True, groups=self.rows)       # row 0 must not be used
            if self.lars:
                e.set_lars(self.offs, self.nums, self.enabled, ETA, EPS)
            assert e.groups == len(self.rows) and e.lars == self.lars

    def trust(self, x, g):
        """per-tensor trust ratios of fp32 x and g, from fp64 norms"""
        T = len(self.offs)
        inside = self.owner >= 0
        own = self.owner[inside]
        sx = torch.zeros(T, dtype=torch.float64, device=x.device).index_add_(0, own, x[inside].double() ** 2)
        sg = torch.zeros(T, dtype=torch.float64, device=x.device).index_add_(0, own, g[inside].double() ** 2)
        nx, ng = sx.sqrt(), sg.sqrt()
        eta, eps = _f32(ETA).item(), _f32(EPS).item()
        t = eta * nx / (ng + self.tensor_wd * nx + eps)
        return torch.where(self.tensor_on & (sx > 0) & (sg > 0), t, torch.ones_like(t))

    def phase1(self, z, w, g, m, trust):
        """phase 1 of the step kernels in their fp32 operation order: x = z * w ;
        d = [t *] fmaf(wd, x, g) ; m = fmaf(mu, m, d) ; x = fmaf(-lr, nesterov ? fmaf(mu, m, d) : m, x)"""
        def fma(a, b, c):                  # the product of two fp32 values is exact in fp64
            return (a.double() * b.double() + c.double()).float()
        x = z * _f32(w).to(z.device)
        d = fma(self.wd, x, g)
        if trust is not None:
            d = trust * d
        m = fma(self.mu, m, d)
        x = fma(-self.lr, torch.where(self.nest, fma(self.mu, m, d), m), x)
        return x, m

    def sgd64(self, z, w, g, m, trust):
        """the same update in fp64 (torch.optim.SGD semantics)"""
        return oracle.sgd_momentum(z.double() * w, g.double(), m.double(), self.lr.double(), self.mu.double(),
                                   self.wd.double(), self.nest,
                                   trust=None if trust is None else trust.double())


def _run_and_check(engines, streams, setup, topo, steps, seed):
    """`steps` full synchronous steps, each checked against fp64: the SGD update of every rank (in
    the kernels' fp32 operation order, itself checked against oracle.sgd_momentum), then the column
    mix of mix_columns; with bf16 messages every rank sends Q(x) = bf16(x) and keeps
    x - (1 - self_w) Q(x), so z = (x - Q(x) + mix of the Q) / w'.  Each step starts from the
    kernels' fp32 state, so that the bf16 rounding of x sees the same operands"""
    bf16 = engines[0].msg_bf16
    ogs, oms = _oracle_graphs(topo)
    for step in range(steps):
        _set_grads(engines, seed, step)
        torch.cuda.synchronize()
        zs = [e.z.clone() for e in engines]
        ms = [e.momentum.clone() for e in engines]
        gs = [e.grad.clone() for e in engines]
        ws = [e.ps_weight for e in engines]
        _mix_all(engines, streams)
        xs = []
        for i, e in enumerate(engines):
            trust = None
            if setup.lars:
                torch.testing.assert_close(e.lars_trust.double(), setup.trust(zs[i] * _f32(ws[i]).cuda(), gs[i]),
                                           rtol=1e-6, atol=0)
                trust = e.lars_trust[setup.elem_tensor]
            x, m = setup.phase1(zs[i], ws[i], gs[i], ms[i], trust)
            x64, m64 = setup.sgd64(zs[i], ws[i], gs[i], ms[i], trust)
            torch.testing.assert_close(x.double(), x64, rtol=1e-5, atol=1e-5)
            torch.testing.assert_close(e.momentum.double(), m64, rtol=1e-5, atol=1e-5)
            torch.testing.assert_close(e.momentum, m, rtol=1e-5, atol=1e-6)
            xs.append(x)
        sent = [x.to(BF16).double() if bf16 else x.double() for x in xs]
        mixed, new_w = oracle.mix_columns(sent, ws, ogs, oms)
        oracle.rotate_all(ogs)
        for i, e in enumerate(engines):
            acc = mixed[i] + (xs[i].double() - sent[i]) if bf16 else mixed[i]
            torch.testing.assert_close(e.z.double(), acc / new_w[i], rtol=1e-5, atol=1e-5)
            assert abs(e.ps_weight - new_w[i]) < 1e-6
            assert torch.equal(e.shadow, e.z.to(BF16))
            assert torch.count_nonzero(e.grad).item() == 0          # fused zero_grad reached every chunk
            assert e.device_step == step + 1


# --------------------------------------------------------------------------------------------- #
# A. the full synchronous step
# --------------------------------------------------------------------------------------------- #
# every shape with every variant; the topology rotates with them, so that every shape and every
# variant meets every topology
A_CASES = [(sid, var, A_TOPOS[(si + vi) % len(A_TOPOS)])
           for si, sid in enumerate(SHAPES) for vi, var in enumerate(VARIANTS)]


@pytest.mark.parametrize('pipe', [True, False], ids=['pipe', 'regs'])
@pytest.mark.parametrize('sid,variant,topo', A_CASES, ids=['-'.join(c) for c in A_CASES])
def test_step_matches_fp64(sid, variant, topo, pipe):
    nchunks, grid, segments = SHAPES[sid]
    msg_dtype = VARIANTS[variant][0]
    engines, streams = _world(topo, nchunks, grid=grid, segments=segments, msg_dtype=msg_dtype, pipe=pipe,
                              seed=sum(map(ord, sid + variant)))
    _check_shape(sid, engines[0], _in_degree(topo))
    setup = _Setup(variant, engines[0].n, engines[0].device)
    setup.configure(engines)
    _run_and_check(engines, streams, setup, topo, steps=5, seed=7)


def _final_state(engines):
    return [(e.z.clone(), e.momentum.clone(), e.shadow.clone(), e.ps_weight) for e in engines]


def _assert_same_bits(want, got, what):
    for r, (a, b) in enumerate(zip(want, got)):
        for name, x, y in zip(('z', 'momentum', 'shadow'), a[:3], b[:3]):
            assert torch.equal(x, y), '%s of rank %d differs: %s' % (name, r, what)
        assert a[3] == b[3], 'push-sum weight of rank %d differs: %s' % (r, what)


@pytest.mark.parametrize('variant,topo', [('fp32', 'npdde4x2'), ('bf16-groups-lars', 'npdde8x3')])
def test_bits_do_not_depend_on_grid_segments_or_kernel(variant, topo):
    """phase 1 is per element, phase 2 is own * self_w followed by fmaf over the in-neighbours in
    table order in both kernels, and the LARS trust comes from the fixed-order norm kernel: which
    CTA owns a chunk, which segment it lands in and which kernel a rank runs change no bit"""
    nchunks, n = 213, TOPOS[topo][1]
    kernels = {'pipe': True, 'regs': False, 'mixed': [r % 2 == 0 for r in range(n)]}
    # from one CTA pulling 213 x n_in ring items down to 13-14 chunks per CTA at grid 16
    assert min(_cta_chunks(nchunks, 16, b) for b in range(16)) * _in_degree(topo) > PIPE_STAGES
    want = None
    for kernel, grid, segments in itertools.product(kernels, (1, 3, 8, 16), (1, 4, 15)):
        engines, streams = _world(topo, nchunks, grid=grid, segments=segments, msg_dtype=VARIANTS[variant][0],
                                  pipe=kernels[kernel], seed=11)
        setup = _Setup(variant, engines[0].n, engines[0].device)
        setup.configure(engines)
        for step in range(5):
            _set_grads(engines, 3, step)
            _mix_all(engines, streams)
        got = _final_state(engines)
        if want is None:
            want = got
        else:
            _assert_same_bits(want, got, 'kernel %s, grid %d, %d segments' % (kernel, grid, segments))
        del engines, streams
        _free()


# --------------------------------------------------------------------------------------------- #
# B. Overlap-SGP: publish with fold, then gather
# --------------------------------------------------------------------------------------------- #
GATHER_GRIDS = (1, 3, 16)        # step s gathers with GATHER_GRIDS[s % 3]


def _gather(e, method):
    if method == 'dma':
        e.gather(dma=True)
    else:
        e.gather(tma=(method == 'tma'), dma=False)


@pytest.mark.parametrize('topo', A_TOPOS)
@pytest.mark.parametrize('sid', ['S1', 'S2'])
def test_overlap_publish_gather_fold_matches_fp64(sid, topo):
    """x <- x - lr*dir ; x += residual ; publish ; the residual of step k is folded at step k+1.
    The TMA gather and the register gather agree bit for bit (as values: -0 == +0); the copy-engine
    gather (single in-neighbour only) brings the raw outbox and applies the edge weight at fold time"""
    nchunks, grid, segments = SHAPES[sid]
    n, n_in = TOPOS[topo][1], _in_degree(topo)
    worlds = {}
    for method in ['tma', 'regs'] + (['dma'] if n_in == 1 else []):
        engines, streams = _world(topo, nchunks, grid=grid, segments=segments, with_residual=True, shadow=False,
                                  seed=21)
        for e in engines:
            e._gather_dma_pref = method == 'dma'
            e._refresh_in_peers()
            assert e.gather_dma == (method == 'dma')
        worlds[method] = (engines, streams, [torch.cuda.Stream() for _ in engines])
    ref = worlds['tma'][0]
    _check_shape(sid, ref[0], n_in)
    # the TMA gather's (chunk, in-neighbour) ring wraps; at gather grid 1 one CTA pulls every chunk
    # while its flag wait covers every publishing CTA
    assert _cta_chunks(nchunks, GATHER_GRIDS[0], 0) == nchunks and nchunks * n_in > RING_STAGES
    assert _cta_chunks(nchunks, GATHER_GRIDS[1], 0) * n_in > RING_STAGES

    ogs, oms = _oracle_graphs(topo)
    lr, mu, wd, nest = 0.1, 0.9, 1e-4, False
    zs = [e.z.double() for e in ref]
    ms = [e.momentum.double() for e in ref]
    ws = [1.0] * n
    res = [torch.zeros_like(z) for z in zs]
    wres = [0.0] * n
    for step in range(6):
        for engines, _, _ in worlds.values():
            _set_grads(engines, 5, step)
            for e in engines:
                e.set_hyper(lr, mu, wd, nest, do_sgd=(step > 0))
                e.gather_grid = GATHER_GRIDS[step % len(GATHER_GRIDS)]
        torch.cuda.synchronize()
        gs = [e.grad.double() for e in ref]
        torch.cuda.synchronize()                     # (publish clears the gradients the oracle reads)
        for method, (engines, streams, side) in worlds.items():
            for e, s in zip(engines, streams):
                with torch.cuda.stream(s):
                    e.publish(sgd=True, fold=True)
            torch.cuda.synchronize()
            for e, s in zip(engines, side):
                with torch.cuda.stream(s):
                    _gather(e, method)
            torch.cuda.synchronize()
        pub, pubw = [], []
        for i in range(n):
            x = zs[i] * ws[i]
            if step > 0:
                x, ms[i] = oracle.sgd_momentum(x, gs[i], ms[i], lr, mu, wd, nest)
            pub.append(x + res[i])
            pubw.append(ws[i] + wres[i])
        cols = [oms[j].scalar_weights(ogs[j].get_peers()[0]) for j in range(n)]
        for i in range(n):
            zs[i] = pub[i] / pubw[i]
            ws[i] = cols[i][0] * pubw[i]
            _, ins = ogs[i].get_peers()
            res[i] = sum(cols[j][1][i] * pub[j] for j in ins)
            wres[i] = sum(cols[j][1][i] * pubw[j] for j in ins)
        oracle.rotate_all(ogs)
        for method, (engines, _, _) in worlds.items():
            for i, e in enumerate(engines):
                e.check()
                torch.testing.assert_close(e.z.double(), zs[i], rtol=1e-5, atol=1e-5)
                torch.testing.assert_close(e.momentum.double(), ms[i], rtol=1e-5, atol=1e-5)
                torch.testing.assert_close(e.residual.double() * e.res_scale, res[i], rtol=1e-5, atol=1e-5)
                assert abs(e.ps_weight - ws[i]) < 1e-6
                assert abs(e.res_weight - wres[i]) < 1e-6
        for a, b in zip(worlds['tma'][0], worlds['regs'][0]):
            assert a.res_scale == b.res_scale == 1.0
            assert (a.residual == b.residual).all(), 'TMA and register gathers differ at step %d' % step
            assert torch.equal(a.z, b.z)


# --------------------------------------------------------------------------------------------- #
# C. consensus and SlowMo over a ResNet-50-sized arena
# --------------------------------------------------------------------------------------------- #
def _snapshot_grid(nchunks):
    """the grid of the consensus and SlowMo kernels (GossipEngine.prepare_consensus / slowmo)"""
    return min(2 * torch.cuda.get_device_properties(0).multi_processor_count, nchunks)


def _zbar(engines):
    """push-sum average sum_i w_i z_i / sum_i w_i, in fp64 on the device"""
    ws = [e.ps_weight for e in engines]
    acc = torch.zeros(engines[0].n, dtype=torch.float64, device=engines[0].device)
    for w, e in zip(ws, engines):
        acc.add_(e.z.double(), alpha=w)
    return acc.div_(sum(ws))


@pytest.mark.parametrize('msg', ['fp32', 'bf16'])
def test_consensus_over_a_resnet50_arena_matches_fp64(msg):
    n, nchunks = 4, RESNET50_CHUNKS
    engines, streams = _world('npdde4x1', nchunks, grid=8, msg_dtype=BF16 if msg == 'bf16' else None,
                              shadow=False, seed=31)
    grid = _snapshot_grid(nchunks)
    # slice mode: each CTA takes 5-6 chunks of its rank's slice, (chunk, rank) items: 20-24;
    # full mode: 23-24 chunks, 92-96 items.  Every CTA refills the 6-stage ring
    slices = [nchunks * (r + 1) // n - nchunks * r // n for r in range(n)]
    assert min(_cta_chunks(c, grid, b) for c in slices for b in range(grid)) * n > 3 * RING_STAGES
    assert min(_cta_chunks(nchunks, grid, b) for b in range(grid)) * n > 15 * RING_STAGES
    gen = torch.Generator(device=engines[0].device).manual_seed(32)
    base = torch.randn(engines[0].n, device=engines[0].device, generator=gen)
    for r, e in enumerate(engines):
        e.z.copy_(base + 1e-3 * torch.randn(e.n, device=e.device, generator=gen))
        e.ps_weight = 0.55 + 0.3 * r                    # irregular mixing: w != 1
        e.prepare_consensus()                           # every rank allocates before the collective
    torch.cuda.synchronize()
    zbar = _zbar(engines)
    per_rank = torch.stack([((e.z.double() - zbar) ** 2).sum() for e in engines]).cpu()
    dsq, nrm = per_rank.mean().item(), (zbar ** 2).sum().item()

    def run(full):
        outs = [torch.full_like(e.z, float('nan')) if full else None for e in engines]
        torch.cuda.synchronize()
        res = []
        for e, s, o in zip(engines, streams, outs):
            with torch.cuda.stream(s):
                res.append(e.consensus(o, full=full))
        torch.cuda.synchronize()
        for e in engines:
            e.check()
        return [r.cpu() for r in res], outs

    sl, _ = run(False)
    fu, outs = run(True)
    for r in range(n):
        assert torch.equal(sl[r], sl[0]) and torch.equal(fu[r], fu[0]), 'results differ between ranks'
        assert torch.equal(outs[r], outs[0]), 'average models differ between ranks'
    for res in (sl[0], fu[0]):
        assert abs(res[0].item() - dsq) <= 1e-4 * dsq
        assert abs(res[1].item() - nrm) <= 1e-5 * nrm
    torch.testing.assert_close(fu[0][2:], per_rank, rtol=1e-4, atol=0)
    assert (sl[0][2:] == 0).all()
    zmax = zbar.abs().max().item()
    torch.testing.assert_close(outs[0].double(), zbar, rtol=1e-5, atol=1e-6 * zmax)


def _close(got, ref):
    """1e-6 relative to the tensor's largest element"""
    err = (got.double() - ref).abs().max().item()
    assert err <= 1e-6 * ref.abs().max().item(), err


@pytest.mark.parametrize('msg', ['fp32', 'bf16'])
def test_slowmo_over_a_resnet50_arena_matches_fp64(msg):
    n, nchunks = 4, RESNET50_CHUNKS
    engines, streams = _world('npdde4x1', nchunks, grid=8, msg_dtype=BF16 if msg == 'bf16' else None, seed=41)
    grid = _snapshot_grid(nchunks)
    assert min(_cta_chunks(nchunks, grid, b) for b in range(grid)) * n > 15 * RING_STAGES     # 92-96 items
    dev = engines[0].device
    gen = torch.Generator(device=dev).manual_seed(42)
    base = torch.randn(engines[0].n, device=dev, generator=gen)
    for e in engines:
        e.z.copy_(base + 0.5 * torch.randn(e.n, device=dev, generator=gen))
    us = [torch.zeros_like(e.z) for e in engines]
    xps = [torch.zeros_like(e.z) for e in engines]
    lr, alpha, beta = 0.05, 0.8, 0.6
    u = xp = None
    for call in range(3):
        if call:
            for e in engines:                            # the ranks drift apart again between calls
                e.z.add_(2.0 * torch.randn(e.n, device=dev, generator=gen))
        for r, e in enumerate(engines):
            e.ps_weight = 0.55 + 0.3 * r + 0.1 * call    # irregular mixing: w != 1
        torch.cuda.synchronize()
        zbar = _zbar(engines)
        if call == 0:
            u, xp = torch.zeros_like(zbar), zbar
        else:
            u = beta * u + (xp - zbar) / lr
            xp = xp - alpha * lr * u
        torch.cuda.synchronize()                         # (the kernels overwrite the z the oracle reads)
        for e, s, uu, xx in zip(engines, streams, us, xps):
            with torch.cuda.stream(s):
                e.slowmo(uu, xx, lr, alpha, beta, call == 0)
        torch.cuda.synchronize()
        for r, e in enumerate(engines):
            e.check()
            assert torch.equal(e.z, engines[0].z) and torch.equal(us[r], us[0]) and torch.equal(xps[r], xps[0]), \
                'ranks differ'
            assert torch.equal(e.z, xps[r])
            assert torch.equal(e.shadow, e.z.to(BF16))
            off = e.C.STATE_OFF_PSW // 4
            assert e._state_f32[off: off + 2].tolist() == [1.0, 1.0]
        _close(xps[0], xp)
        _close(us[0], u)
        _close(engines[0].z, xp)


# --------------------------------------------------------------------------------------------- #
# D. one ResNet-50-sized synchronous step
# --------------------------------------------------------------------------------------------- #
@pytest.mark.parametrize('variant', ['fp32', 'bf16-groups-lars'])
def test_resnet50_sized_step_matches_fp64_with_both_kernels(variant):
    """two ranks sharing the GPU's co-resident CTAs: about 47 chunks per CTA in 4 segments of 11-12"""
    nchunks = RESNET50_CHUNKS
    grid = _max_grid() // 2
    finals = {}
    for pipe in (True, False):
        engines, streams = _world('npdde2x1', nchunks, grid=grid, msg_dtype=VARIANTS[variant][0], pipe=pipe,
                                  seed=51)
        per_cta, segs = _split(nchunks, engines[0].grid, engines[0].ctx.segments())
        assert min(per_cta) > 10 * PIPE_STAGES and min(min(s) for s in segs) > 1
        setup = _Setup(variant, engines[0].n, engines[0].device)
        setup.configure(engines)
        _run_and_check(engines, streams, setup, 'npdde2x1', steps=3, seed=9)
        finals[pipe] = _final_state(engines)
        del engines, streams, setup
        _free()
    _assert_same_bits(finals[True], finals[False], 'pipelined vs register-staged kernel')
