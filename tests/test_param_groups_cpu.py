"""Per-parameter-group hyper-parameters of FusedGossipSGD (``param_groups=``) on the c10d plane
(gloo, CPU): SGP, OSGP and D-PSGD with two and three groups against an fp64 whole-world
simulation, one explicit group bit-identical to ``param_groups=None``, the validation errors, the
checkpoint round trip, ``no_bias_decay_groups`` and the command line's ``--no_bias_decay``."""

import pytest
import torch

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.ops import oracle

import test_distributed_c10d as sim
from dist_utils import run_distributed

SELF_W = [0.3, 0.5, 0.6, 0.45]
DEFAULTS = dict(lr=0.08, momentum=0.0, weight_decay=5e-3, nesterov=False)


def _groups(model, kind):
    """parameters of sim._model: [W1 (5x6), b1 (5), W2 (3x5), b2 (3)]"""
    w1, b1, w2, b2 = list(model.parameters())
    if kind == 'two':          # no-bias-decay style: the weights take the defaults
        return [dict(params=[b1, b2], weight_decay=0.0, lr=0.03)]
    return [dict(params=[w1], lr=0.05, momentum=0.9, weight_decay=1e-3, nesterov=True),
            dict(params=[b2, b1], lr=0.02, momentum=0.5, weight_decay=0.0)]      # W2: trailing default group


def _gdp(rank, world, graph_name, ppi, push_sum, overlap, mixing):
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    graph = getattr(sgp, graph_name)(rank, world, peers_per_itr=ppi)
    mix = sgp.UniformMixing(graph, 'cpu') if mixing == 'uniform' else \
        sgp.SelfWeightedMixing(graph, 'cpu', self_weight=SELF_W)
    model = GossipDataParallel(sim._model(rank), graph=graph, mixing=mix, push_sum=push_sum,
                               overlap=overlap, rank=rank, world_size=world, verbose=False)
    assert model.transport == 'c10d'
    return model


def _worker(rank, world, graph_name, ppi, push_sum, overlap, mixing, kind, steps):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    model = _gdp(rank, world, graph_name, ppi, push_sum, overlap, mixing)
    groups = None if kind is None else _groups(model.module, kind)
    opt = FusedGossipSGD(model, param_groups=groups, **DEFAULTS)
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


def _hyper_vectors(kind):
    """per-element (lr, momentum, weight_decay, nesterov) over sim._flat's layout"""
    m = sim._model(0).double()
    group_of = {}
    rows = []
    for gi, g in enumerate(_groups(m, kind)):
        for p in g['params']:
            group_of[id(p)] = gi
        rows.append(dict(DEFAULTS, **{k: v for k, v in g.items() if k != 'params'}))
    rows.append(dict(DEFAULTS))
    per = [rows[group_of.get(id(p), len(rows) - 1)] for p in m.parameters()]
    numels = [p.numel() for p in m.parameters()]

    def vec(key, dtype):
        return torch.cat([torch.full((n,), r[key], dtype=dtype) for r, n in zip(per, numels)])
    return (vec('lr', torch.float64), vec('momentum', torch.float64), vec('weight_decay', torch.float64),
            vec('nesterov', torch.bool))


def _simulate(world, graph_name, ppi, overlap, mixing, kind, steps):
    """the whole world in one process, fp64, each element with its group's hyper-parameters"""
    models = [sim._model(r).double() for r in range(world)]
    graphs = [getattr(sgp, graph_name)(r, world, peers_per_itr=ppi) for r in range(world)]
    mix = [sgp.UniformMixing(g, 'cpu') if mixing == 'uniform' else
           sgp.SelfWeightedMixing(g, 'cpu', self_weight=SELF_W) for g in graphs]
    lr, mu, wd, nest = _hyper_vectors(kind)
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
            xs[i], moms[i] = oracle.sgd_momentum(xs[i], grads[i], moms[i], lr, mu, wd, nest)
        if not overlap:
            xs, ws = oracle.mix_columns(xs, ws, graphs, mix)
            oracle.rotate_all(graphs)
    if overlap:
        xs = [x + r for x, r in zip(xs, res)]
        ws = [w + wr for w, wr in zip(ws, wres)]
    return [x / w for x, w in zip(xs, ws)], ws


@pytest.mark.parametrize('graph_name,ppi,push_sum,overlap', [
    ('NPeerDynamicDirectedExponentialGraph', 1, True, False),     # SGP
    ('NPeerDynamicDirectedExponentialGraph', 1, True, True),      # OSGP
    ('RingGraph', 1, False, False),                               # D-PSGD
], ids=['sgp', 'osgp', 'dpsgd'])
@pytest.mark.parametrize('mixing,kind', [('uniform', 'three'), ('self_weighted', 'two'),
                                         ('self_weighted', 'three')])
def test_groups_match_fp64_simulation(graph_name, ppi, push_sum, overlap, mixing, kind):
    world, steps = 4, 6
    out = run_distributed(_worker, world, graph_name, ppi, push_sum, overlap, mixing, kind, steps)
    want, ws = _simulate(world, graph_name, ppi, overlap, mixing, kind, steps)
    for r in range(world):
        got, w = out[r]
        torch.testing.assert_close(torch.tensor(got, dtype=torch.float64), want[r], rtol=1e-5, atol=1e-6)
        assert abs(w - ws[r]) < 1e-5
    if mixing == 'self_weighted' and push_sum:
        assert any(abs(w - 1) > 1e-3 for _, w in out)
    # the groups matter: the single-group run ends elsewhere
    plain = run_distributed(_worker, world, graph_name, ppi, push_sum, overlap, mixing, None, steps)
    assert max(abs(a - b) for a, b in zip(plain[0][0], out[0][0])) > 1e-4


def _one_group_worker(rank, world):
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    finals = []
    for explicit in (False, True):
        model = _gdp(rank, world, 'DynamicDirectedExponentialGraph', 2, True, False, 'self_weighted')
        groups = [dict(params=list(model.module.parameters()))] if explicit else None
        opt = FusedGossipSGD(model, lr=0.05, momentum=0.9, weight_decay=1e-3, nesterov=True,
                             param_groups=groups)
        assert len(opt.param_groups) == 1 and not opt._grouped
        model.train()
        for step in range(4):
            x, y = sim._batch(rank, step)
            ((model(x) - y) ** 2).mean().backward()
            opt.step()
            opt.zero_grad()
            model.transfer_params()
        model.sync_comms()
        finals.append(model.arena.flat.clone())
    return torch.equal(*finals)


def test_one_explicit_group_is_bit_identical_to_none():
    assert all(run_distributed(_one_group_worker, 2))


def _single():
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    model = GossipDataParallel(sim._model(0), graph=sgp.RingGraph(0, 1), rank=0, world_size=1)
    return model


def test_validation_errors():
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    model = _single()
    w1, b1, w2, b2 = list(model.module.parameters())
    with pytest.raises(ValueError, match='more than one'):
        FusedGossipSGD(model, param_groups=[dict(params=[w1, b1]), dict(params=[b1])])
    with pytest.raises(ValueError, match='not a parameter'):
        FusedGossipSGD(model, param_groups=[dict(params=[torch.nn.Parameter(torch.zeros(3))])])
    with pytest.raises(ValueError, match='at most 16'):
        big = _single()
        FusedGossipSGD(big, param_groups=[dict(params=[]) for _ in range(17)])
    with pytest.raises(ValueError, match='Nesterov'):
        FusedGossipSGD(model, momentum=0.9, param_groups=[dict(params=[w1], momentum=0.0, nesterov=True)])
    # 16 groups (the trailing default one included) are fine
    FusedGossipSGD(_single(), param_groups=[dict(params=[]) for _ in range(15)])


def test_slowmo_rejects_unequal_learning_rates():
    from stochastic_gradient_push_b200.optim import FusedGossipSGD
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    model = GossipDataParallel(sim._model(0), graph=sgp.RingGraph(0, 1), rank=0, world_size=1,
                               slowmo_frequency=1)
    w1, b1, w2, b2 = list(model.module.parameters())
    opt = FusedGossipSGD(model, lr=0.1, param_groups=[dict(params=[b1, b2], weight_decay=0.0)])
    assert model.perform_slowmo(opt)                       # equal lr, different weight decay: fine
    opt.param_groups[0]['lr'] = 0.05
    with pytest.raises(ValueError, match='one base learning rate'):
        model.perform_slowmo(opt)


def test_state_dict_round_trip_and_one_group_checkpoint():
    from stochastic_gradient_push_b200.optim import FusedGossipSGD, no_bias_decay_groups
    model = _single()
    opt = FusedGossipSGD(model, lr=0.1, momentum=0.9, weight_decay=1e-4,
                         param_groups=no_bias_decay_groups(model.module, 1e-4))
    opt.param_groups[0]['lr'] = 0.02
    opt.param_groups[1]['momentum'] = 0.8
    sd = opt.state_dict()
    assert [g['weight_decay'] for g in sd['param_groups']] == [0.0, 1e-4]
    other = FusedGossipSGD(model, lr=0.1, momentum=0.9, weight_decay=1e-4,
                           param_groups=no_bias_decay_groups(model.module, 1e-4))
    other.load_state_dict(sd)
    keys = ('lr', 'momentum', 'weight_decay', 'nesterov')
    assert [[g[k] for k in keys] for g in other.param_groups] == [[g[k] for k in keys] for g in opt.param_groups]
    # a checkpoint of the one-group optimizer: its lr goes to every group, the rest stays per group
    plain = FusedGossipSGD(_single(), lr=0.003, momentum=0.5, weight_decay=1e-4).state_dict()
    other.load_state_dict(plain)
    assert [g['lr'] for g in other.param_groups] == [0.003, 0.003]
    assert [g['weight_decay'] for g in other.param_groups] == [0.0, 1e-4]
    with pytest.raises(ValueError, match='parameter groups'):
        other.load_state_dict(dict(plain, param_groups=[plain['param_groups'][0]] * 3))


def test_no_bias_decay_groups_resnet50():
    from stochastic_gradient_push_b200.models import resnet50
    from stochastic_gradient_push_b200.optim import no_bias_decay_groups
    net = resnet50()
    g0, g1 = no_bias_decay_groups(net, 1e-4)
    assert g0['weight_decay'] == 0.0 and g1['weight_decay'] == 1e-4
    small = [p for p in net.parameters() if p.dim() <= 1]
    assert [id(p) for p in g0['params']] == [id(p) for p in small]
    assert [id(p) for p in g1['params']] == [id(p) for p in net.parameters() if p.dim() > 1]
    assert len(small) == 2 * 53 + 1       # 53 BatchNorms x (weight, bias) + the fc bias


def test_cli_rejects_no_bias_decay_where_unsupported(tmp_path):
    from stochastic_gradient_push_b200.cli.common import build_parser, finalize_args
    for adpsgd, extra, what in ((False, ['--all_reduce', 'True', '--graph_type', '-1'], '--all_reduce'),
                                (True, [], 'AD-PSGD')):
        args = build_parser(adpsgd=adpsgd).parse_args(
            ['--no_bias_decay', 'True', '--device', 'cpu', '--checkpoint_dir', str(tmp_path) + '/'] + extra)
        with pytest.raises(ValueError, match=what):
            finalize_args(args, adpsgd=adpsgd)
    assert build_parser().parse_args([]).no_bias_decay is False


@pytest.mark.parametrize('fused', ['True', 'False'])
def test_gossip_sgd_cli_with_no_bias_decay_two_ranks_cpu(tmp_path, master_port, fused):
    from test_cli_and_experiment import COMMON, _torchrun
    args = COMMON + ['--push_sum', 'True', '--graph_type', '5', '--num_epochs', '1', '--num_itr_ignore', '0',
                     '--seed', '47', '--no_bias_decay', 'True', '--fused', fused,
                     '--checkpoint_dir', str(tmp_path) + '/']
    out = _torchrun(2, 'gossip_sgd.py', args, master_port)
    assert out.returncode == 0, out.stdout[-3000:]
    for r in range(2):
        assert len(open(str(tmp_path / ('out_r%d_n2.csv' % r))).read().splitlines()) > 2
