"""LARS in FusedGossipSGD (``lars=True``) on the c10d plane (gloo, CPU): SGP, OSGP and D-PSGD with
``lars_groups`` (one group without LARS) under self-weighted mixing (w != 1, so the numerator's norm
matters) against a per-tensor torch LARS + mixing simulation in fp64, the trust rule's edge cases,
``lars_groups``, the checkpoint round trip, the command line's ``--lars`` and its rejections, and
what ptxas reports for the new sm_90a kernels."""

import os
import re

import pytest
import torch

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops import oracle

import test_distributed_c10d as sim
from dist_utils import run_distributed

SELF_W = [0.3, 0.5, 0.6, 0.45]
HYPER = dict(lr=0.4, momentum=0.9, weight_decay=5e-3, nesterov=True)
WD, ETA, EPS = 2e-2, 0.05, 1e-8


def _gdp(rank, world, graph_name, push_sum, overlap):
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    graph = getattr(sgp, graph_name)(rank, world, peers_per_itr=1)
    mix = sgp.SelfWeightedMixing(graph, 'cpu', self_weight=SELF_W)
    model = GossipDataParallel(sim._model(rank), graph=graph, mixing=mix, push_sum=push_sum,
                               overlap=overlap, rank=rank, world_size=world, verbose=False)
    assert model.transport == 'c10d'
    return model


def _worker(rank, world, graph_name, push_sum, overlap, lars, steps):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD, lars_groups
    model = _gdp(rank, world, graph_name, push_sum, overlap)
    groups = lars_groups(model.module, WD)
    for g in groups:
        g['lars'] = g['lars'] and lars
    opt = FusedGossipSGD(model, param_groups=groups, lars=lars, trust_coefficient=ETA, lars_eps=EPS, **HYPER)
    model.train()
    for step in range(steps):
        x, y = sim._batch(rank, step)
        ((model(x) - y) ** 2).mean().backward()
        opt.step()
        opt.zero_grad()
        if not overlap:
            model.transfer_params()
    model.sync_comms()
    model.unbias()
    return sim._flat(model.module).tolist(), float(model.ps_weight)


def _lars_sgd(x, g, m, params, lars):
    """torch.optim.SGD with LARC(clip=False) in front, tensor by tensor over sim._flat's layout:
    [W1, b1, W2, b2]; the weights (ndim > 1) take WD and LARS, the biases neither"""
    xs, ms, off = [], [], 0
    for p in params:
        n = p.numel()
        xp, gp, mp = x[off:off + n], g[off:off + n], m[off:off + n]
        wd = WD if p.dim() > 1 else 0.0
        d = gp + wd * xp
        if lars and p.dim() > 1:
            nx, ng = xp.norm().item(), gp.norm().item()
            if nx > 0 and ng > 0:
                d = d * (ETA * nx / (ng + wd * nx + EPS))
        mp = HYPER['momentum'] * mp + d
        xs.append(xp - HYPER['lr'] * (d + HYPER['momentum'] * mp))      # nesterov
        ms.append(mp)
        off += n
    return torch.cat(xs), torch.cat(ms)


def _simulate(world, graph_name, overlap, steps, lars=True):
    models = [sim._model(r).double() for r in range(world)]
    graphs = [getattr(sgp, graph_name)(r, world, peers_per_itr=1) for r in range(world)]
    mix = [sgp.SelfWeightedMixing(g, 'cpu', self_weight=SELF_W) for g in graphs]
    ws = [1.0] * world
    xs = [sim._flat(m).clone() for m in models]
    moms = [torch.zeros_like(x) for x in xs]
    res = [torch.zeros_like(x) for x in xs]
    wres = [0.0] * world

    def load(m, flat):
        off = 0
        for p in m.parameters():
            p.data.copy_(flat[off:off + p.numel()].view_as(p))
            off += p.numel()

    for step in range(steps):
        if overlap:
            xs = [x + r for x, r in zip(xs, res)]
            ws = [w + wr for w, wr in zip(ws, wres)]
            cols = [mix[j].scalar_weights(graphs[j].get_peers()[0], rank=j) for j in range(world)]
            snap, snapw = [x.clone() for x in xs], list(ws)
            for i in range(world):
                _, ins = graphs[i].get_peers()
                res[i] = sum(cols[j][1][i] * snap[j] for j in ins)
                wres[i] = sum(cols[j][1][i] * snapw[j] for j in ins)
                xs[i] = cols[i][0] * xs[i]
                ws[i] = cols[i][0] * ws[i]
            oracle.rotate_all(graphs)
        grads = []
        for i, m in enumerate(models):
            load(m, xs[i] / ws[i])
            m.zero_grad()
            x, y = sim._batch(i, step)
            ((m(x.double()) - y.double()) ** 2).mean().backward()
            grads.append(torch.cat([p.grad.reshape(-1) for p in m.parameters()]))
        for i in range(world):
            xs[i], moms[i] = _lars_sgd(xs[i], grads[i], moms[i], list(models[i].parameters()), lars)
        if not overlap:
            xs, ws = oracle.mix_columns(xs, ws, graphs, mix)
            oracle.rotate_all(graphs)
    if overlap:
        xs = [x + r for x, r in zip(xs, res)]
        ws = [w + wr for w, wr in zip(ws, wres)]
    return [x / w for x, w in zip(xs, ws)], ws


@pytest.mark.parametrize('graph_name,push_sum,overlap', [
    ('NPeerDynamicDirectedExponentialGraph', True, False),     # SGP
    ('NPeerDynamicDirectedExponentialGraph', True, True),      # OSGP
    ('RingGraph', False, False),                               # D-PSGD
], ids=['sgp', 'osgp', 'dpsgd'])
def test_lars_matches_per_tensor_torch_simulation(graph_name, push_sum, overlap):
    world, steps = 4, 5
    out = run_distributed(_worker, world, graph_name, push_sum, overlap, True, steps)
    want, ws = _simulate(world, graph_name, overlap, steps)
    for r in range(world):
        got, w = out[r]
        torch.testing.assert_close(torch.tensor(got, dtype=torch.float64), want[r], rtol=1e-5, atol=1e-6)
        assert abs(w - ws[r]) < 1e-5
    if push_sum:
        assert any(abs(w - 1) > 1e-3 for _, w in out)
    # LARS matters: the same groups without it end elsewhere
    plain = run_distributed(_worker, world, graph_name, push_sum, overlap, False, steps)
    assert max(abs(a - b) for a, b in zip(plain[0][0], out[0][0])) > 1e-3


def _single():
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    return GossipDataParallel(sim._model(0), graph=sgp.RingGraph(0, 1), rank=0, world_size=1)


def test_trust_is_one_for_zero_norms_and_excluded_groups():
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    model = _single()
    w1, b1, w2, b2 = list(model.module.parameters())
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, weight_decay=1e-3, trust_coefficient=0.01,
                         param_groups=[dict(params=[w1, w2, b2], lars=True), dict(params=[b1], lars=False)])
    assert opt._grouped and opt._lars_flags == (True, False)
    arena = model._arenas[torch.float32]
    x = arena.flat.clone()
    g = torch.randn_like(x)
    views = arena.views_of(x)
    views[2].zero_()                                  # W2: |x| = 0
    gviews = arena.views_of(g)
    gviews[3].zero_()                                 # b2: |g| = 0
    t = arena.views_of(opt._c10d_trust(torch.float32, x, g))
    assert torch.all(t[1] == 1) and torch.all(t[2] == 1) and torch.all(t[3] == 1)   # b1 excluded
    nx, ng = views[0].double().norm(), gviews[0].double().norm()
    want = 0.01 * nx / (ng + 1e-3 * nx + 1e-8)
    assert torch.all(t[0] == want.float())
    # lars=False everywhere: no trust at all, the plain grouped step
    other = _single()
    plain = FusedGossipSGD(other, lr=0.1, param_groups=[dict(params=[next(other.module.parameters())], lars=False)])
    assert not plain._lars_on() and plain._lars_flags == (False, False)


def test_one_group_with_lars_installs_the_block_map():
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    opt = FusedGossipSGD(_single(), lr=0.1, momentum=0.9, lars=True)
    assert len(opt.param_groups) == 1 and opt._grouped and opt.param_groups[0]['lars'] is True
    assert FusedGossipSGD(_single(), lr=0.1).param_groups[0]['lars'] is False
    with pytest.raises(ValueError, match='LARS'):
        FusedGossipSGD(_single(), lars=True, trust_coefficient=0.0)


def test_lars_groups_resnet50():
    from stochastic_gradient_push_b200.models import resnet50
    from stochastic_gradient_push_b200.optim import lars_groups
    net = resnet50()
    g0, g1 = lars_groups(net, 5e-5)
    assert (g0['weight_decay'], g0['lars']) == (0.0, False) and (g1['weight_decay'], g1['lars']) == (5e-5, True)
    assert [id(p) for p in g0['params']] == [id(p) for p in net.parameters() if p.dim() <= 1]
    assert [id(p) for p in g1['params']] == [id(p) for p in net.parameters() if p.dim() > 1]
    assert len(g0['params']) == 2 * 53 + 1 and len(g1['params']) == 53 + 1


def test_state_dict_round_trips_lars_settings():
    from stochastic_gradient_push_b200.optim import FusedGossipSGD, lars_groups
    model = _single()
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, param_groups=lars_groups(model.module, 1e-4),
                         lars=True, trust_coefficient=0.02, lars_eps=1e-6)
    sd = opt.state_dict()
    assert [g['lars'] for g in sd['param_groups']] == [False, True]
    assert sd['lars'] == {'trust_coefficient': 0.02, 'eps': 1e-6}
    other = FusedGossipSGD(model, lr=0.1, momentum=0.9, param_groups=[dict(params=list(model.module.parameters())[:2]),
                                                                      dict(params=list(model.module.parameters())[2:])])
    assert not other._lars_on()
    other.load_state_dict(sd)
    assert [g['lars'] for g in other.param_groups] == [False, True]
    assert (other.trust_coefficient, other.lars_eps) == (0.02, 1e-6)
    assert other._lars_flags == (False, True)
    assert other.state_dict()['lars'] == sd['lars']


def test_too_many_tensors_is_refused():
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    import stochastic_gradient_push_b200.optim as optim
    model = GossipDataParallel(sim._model(0), graph=sgp.RingGraph(0, 1), rank=0, world_size=1)
    old = optim.LARS_MAX_TENSORS
    optim.LARS_MAX_TENSORS = 3                       # sim._model has 4 tensors
    try:
        with pytest.raises(ValueError, match='LARS supports at most 3 tensors'):
            FusedGossipSGD(model, lars=True)
    finally:
        optim.LARS_MAX_TENSORS = old


def test_cli_parses_lars_and_rejects_unsupported_modes(tmp_path):
    from stochastic_gradient_push_b200.cli.common import build_parser, finalize_args
    base = ['--device', 'cpu', '--checkpoint_dir', str(tmp_path) + '/']
    args = build_parser().parse_args(['--lars', 'True', '--lars_trust', '0.02'] + base)
    assert args.lars is True and args.lars_trust == 0.02
    finalize_args(args)
    defaults = build_parser().parse_args([])
    assert defaults.lars is False and defaults.lars_trust == 0.001
    for adpsgd, extra, what in ((False, ['--all_reduce', 'True', '--graph_type', '-1'], '--all_reduce'),
                                (False, ['--fused', 'False'], '--fused False'),
                                (True, [], 'AD-PSGD')):
        args = build_parser(adpsgd=adpsgd).parse_args(['--lars', 'True'] + base + extra)
        with pytest.raises(ValueError, match='--lars is not supported with %s' % re.escape(what)):
            finalize_args(args, adpsgd=adpsgd)


def test_all_reduce_and_adpsgd_trainers_reject_lars():
    from stochastic_gradient_push_b200.parallel.ad_psgd import make_bilat_trainer
    from stochastic_gradient_push_b200.parallel.allreduce import ARTrainer
    with pytest.raises(ValueError, match='LARS'):
        ARTrainer(None, lr=0.1, lars=True)
    with pytest.raises(ValueError, match='LARS'):
        make_bilat_trainer(None, lr=0.1, lars=True)


def test_gossip_sgd_cli_with_lars_two_ranks_cpu(tmp_path, master_port):
    from test_cli_and_experiment import COMMON, _torchrun
    args = COMMON + ['--push_sum', 'True', '--graph_type', '5', '--num_epochs', '1', '--num_itr_ignore', '0',
                     '--seed', '47', '--lars', 'True', '--lars_trust', '0.01', '--no_bias_decay', 'True',
                     '--checkpoint_dir', str(tmp_path) + '/']
    out = _torchrun(2, 'gossip_sgd.py', args, master_port)
    assert out.returncode == 0, out.stdout[-3000:]
    for r in range(2):
        assert len(open(str(tmp_path / ('out_r%d_n2.csv' % r))).read().splitlines()) > 2


def _ptxas_entries():
    """{demangled-ish kernel name: (registers, spill store bytes)} from the build's ptxas log"""
    from stochastic_gradient_push_b200.ops import build
    build.build()
    log = open(os.path.join(build.OBJ_DIR, 'ptxas.log')).read()
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r'(\d+) bytes spill stores', line)
        if cur and m:
            out.setdefault(cur, {})['spill'] = int(m.group(1))
        m = re.search(r'Used (\d+) registers', line)
        if cur and m:
            out.setdefault(cur, {})['regs'] = int(m.group(1))
    return out


def test_ptxas_lists_the_lars_kernels_and_the_pipe_variants_fit_two_ctas():
    entries = _ptxas_entries()
    norms = [v for k, v in entries.items() if 'sgp_lars_norms_kernel' in k]
    trust = [v for k, v in entries.items() if 'sgp_lars_trust_kernel' in k]
    assert len(norms) == 1 and len(trust) == 1
    assert norms[0]['spill'] == 0 and trust[0]['spill'] == 0
    # Itanium mangling of sgp_step_pipe_kernel<MSG_BF16, true, true>: template args Lb0/Lb1, Lb1, Lb1
    pipe = [v for k, v in entries.items() if 'sgp_step_pipe_kernel' in k and k.endswith('ELb1ELb1EEv7SgpArgs')]
    regs = [v for k, v in entries.items() if 'sgp_step_kernel' in k and k.endswith('ELb1ELb1EEv7SgpArgs')]
    assert len(pipe) == 2 and len(regs) == 2
    # 9 warps x 2 CTAs per SM fit at <= 102 registers per thread; 8 warps x 2 at <= 128
    assert all(v['regs'] <= 102 for v in pipe), pipe
    assert all(v['regs'] <= 128 and v['spill'] == 0 for v in regs), regs
