"""SlowMo (``GossipDataParallel(slowmo_frequency=...)``, ``perform_slowmo``) on the c10d plane
(gloo, CPU): every SlowMo step against an fp64 simulation from the all-gathered parameters and
push-sum weights, rank-identical results, periodic exact averaging as the beta = 0, alpha = 1 case,
frequency 0 as a no-op, the checkpoint round trip, the configurations that reject it and the
command line's ``--slowmo_frequency``."""

import types

import pytest
import torch
import torch.distributed as dist

import stochastic_gradient_push_b200 as sgp

import test_distributed_c10d as sim
from dist_utils import run_distributed

SELF_W = [0.3, 0.5, 0.6, 0.45]


def _gdp(rank, world, graph_name, ppi, push_sum, overlap, mixing, **kw):
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    graph = getattr(sgp, graph_name)(rank, world, peers_per_itr=ppi)
    mix = sgp.UniformMixing(graph, 'cpu') if mixing == 'uniform' else \
        sgp.SelfWeightedMixing(graph, 'cpu', self_weight=SELF_W)
    model = GossipDataParallel(sim._model(rank), graph=graph, mixing=mix, push_sum=push_sum,
                               overlap=overlap, rank=rank, world_size=world, **kw)
    assert model.transport == 'c10d'
    return model


def _step(model, opt, rank, step, overlap):
    x, y = sim._batch(rank, step)
    ((model(x) - y) ** 2).mean().backward()
    opt.step()
    opt.zero_grad()
    if not overlap:
        model.transfer_params()


def _gather(t, world):
    ts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(ts, t)
    return ts


def _slowmo_worker(rank, world, graph_name, ppi, push_sum, overlap, mixing, freq, alpha, beta, steps):
    model = _gdp(rank, world, graph_name, ppi, push_sum, overlap, mixing,
                 slowmo_frequency=freq, slowmo_lr=alpha, slowmo_momentum=beta)
    opt = torch.optim.SGD(model.parameters(), lr=sim.LR, momentum=sim.MU, weight_decay=sim.WD)
    model.train()
    recs = []
    for step in range(steps):
        _step(model, opt, rank, step, overlap)
        due = (step + 1) % freq == 0
        rec = None
        if due:
            # the state perform_slowmo() starts from: in-flight gossip drained, parameters de-biased
            model.sync_comms()
            model.unbias()
            z = model.arena.flat.clone()
            w = torch.tensor([float(model.ps_weight)], dtype=torch.float32)
            rec = dict(zs=[t.tolist() for t in _gather(z, world)],
                       ws=[float(t) for t in _gather(w, world)],
                       init=not model._slowmo_initialized,
                       u0=model._slowmo_u.tolist(), xp0=model._slowmo_x_prev.tolist())
        ran = model.perform_slowmo(opt)
        assert ran == due
        if due:
            flat = model.arena.flat.clone()
            rec.update(flat=flat.tolist(), u=model._slowmo_u.tolist(), xp=model._slowmo_x_prev.tolist(),
                       w=float(model.ps_weight), all_equal=all(torch.equal(t, flat) for t in _gather(flat, world)),
                       dsq=model.consensus_distance().distance_sq,
                       views=all(torch.equal(p.detach().reshape(-1), v.reshape(-1))
                                 for p, v in zip(model.module.parameters(), model.arena.views_of(flat))))
            recs.append(rec)
    return recs


def _close(got, ref):
    """rtol 1e-6, with the tolerance of the tensor's largest element for elements near zero"""
    got = torch.tensor(got, dtype=torch.float64)
    torch.testing.assert_close(got, ref, rtol=1e-6, atol=1e-6 * ref.abs().max().item() + 1e-12)


@pytest.mark.parametrize('graph_name,ppi,push_sum,overlap', [
    ('NPeerDynamicDirectedExponentialGraph', 1, True, False),     # SGP
    ('NPeerDynamicDirectedExponentialGraph', 1, True, True),      # OSGP
    ('RingGraph', 1, False, False),                               # D-PSGD
], ids=['sgp', 'osgp', 'dpsgd'])
@pytest.mark.parametrize('mixing', ['uniform', 'self_weighted'])
def test_slowmo_matches_fp64_simulation(graph_name, ppi, push_sum, overlap, mixing):
    world, freq, alpha, beta = 4, 3, 0.8, 0.6
    out = run_distributed(_slowmo_worker, world, graph_name, ppi, push_sum, overlap, mixing,
                          freq, alpha, beta, 10)
    assert len(out[0]) == 3
    saw_w = False
    for call in range(3):
        recs = [out[r][call] for r in range(world)]
        ref = recs[0]
        zs = torch.tensor(ref['zs'], dtype=torch.float64)
        ws = torch.tensor(ref['ws'], dtype=torch.float64)
        saw_w = saw_w or (ws - 1).abs().max().item() > 1e-3
        zbar = (ws[:, None] * zs).sum(0) / ws.sum()
        # the plane holds zbar in fp32 (then updates in fp32): round it once, as it does
        zbar = zbar.float().double()
        u0 = torch.tensor(ref['u0'], dtype=torch.float64)
        xp0 = torch.tensor(ref['xp0'], dtype=torch.float64)
        assert ref['init'] == (call == 0)
        if ref['init']:
            u, xp = torch.zeros_like(zbar), zbar
        else:
            u = beta * u0 + (xp0 - zbar) / sim.LR
            xp = xp0 - alpha * sim.LR * u
            assert (xp - zbar).abs().max().item() > 1e-4      # not just the average
        for rec in recs:
            assert rec['zs'] == ref['zs'] and rec['ws'] == ref['ws']
            assert rec['flat'] == ref['flat'] and rec['u'] == ref['u'] and rec['xp'] == ref['xp']
            assert rec['all_equal'] and rec['views']
            assert rec['w'] == 1.0
            assert rec['dsq'] == 0.0
            assert rec['flat'] == rec['xp']
            if rec['init']:
                assert all(v == 0.0 for v in rec['u'])
            _close(rec['u'], u)
            _close(rec['xp'], xp)
    if mixing == 'self_weighted':
        assert saw_w


def _averaging_worker(rank, world):
    model = _gdp(rank, world, 'DynamicDirectedExponentialGraph', 2, True, False, 'self_weighted',
                 slowmo_frequency=2, slowmo_lr=1.0, slowmo_momentum=0.0)
    opt = torch.optim.SGD(model.parameters(), lr=sim.LR, momentum=sim.MU, weight_decay=sim.WD)
    model.train()
    recs = []
    for step in range(6):
        _step(model, opt, rank, step, False)
        avg = model.average_model() if (step + 1) % 2 == 0 else None
        w = float(model.ps_weight)
        if model.perform_slowmo(opt):
            recs.append(dict(avg=avg.tolist(), flat=model.arena.flat.tolist(), u=model._slowmo_u.tolist(), w=w))
    return recs


def test_zero_momentum_unit_lr_is_periodic_exact_averaging():
    out = run_distributed(_averaging_worker, 4)
    for recs in out:
        assert len(recs) == 3
        assert any(abs(r['w'] - 1) > 1e-3 for r in recs)         # the average is weighted
        assert all(v == 0.0 for v in recs[0]['u'])               # the first call only averages
        for r in recs:
            avg = torch.tensor(r['avg'])
            torch.testing.assert_close(torch.tensor(r['flat']), avg, rtol=1e-6,
                                       atol=1e-6 * avg.abs().max().item())


def _off_worker(rank, world):
    finals = []
    for call in (False, True):
        model = _gdp(rank, world, 'NPeerDynamicDirectedExponentialGraph', 1, True, False, 'self_weighted')
        opt = torch.optim.SGD(model.parameters(), lr=sim.LR, momentum=sim.MU, weight_decay=sim.WD)
        model.train()
        ran = []
        for step in range(5):
            _step(model, opt, rank, step, False)
            if call:
                ran.append(model.perform_slowmo(opt))
        keys = sorted(model.state_dict())
        model.sync_comms()
        model.unbias()
        finals.append((sim._flat(model.module).tolist(), float(model.ps_weight), ran, keys))
    return finals


def test_frequency_zero_is_a_no_op():
    for without, with_calls in run_distributed(_off_worker, 4):
        assert with_calls[2] == [False] * 5
        assert without[:2] == with_calls[:2]
        assert without[3] == with_calls[3] == ['is_ps_numerator', 'ps_weight', 'state_dict']


def _checkpoint_worker(rank, world):
    kw = dict(slowmo_frequency=3, slowmo_lr=0.7, slowmo_momentum=0.5)
    args = (rank, world, 'DynamicDirectedExponentialGraph', 2, True, False, 'self_weighted')
    model = _gdp(*args, **kw)
    opt = torch.optim.SGD(model.parameters(), lr=sim.LR, momentum=sim.MU, weight_decay=sim.WD)
    model.train()
    for step in range(6):
        _step(model, opt, rank, step, False)
        model.perform_slowmo(opt)
    sd = model.state_dict()
    assert set(sd) == {'state_dict', 'ps_weight', 'is_ps_numerator', 'slowmo'}
    restored = _gdp(*args, **kw)
    restored.load_state_dict(sd)
    same = (torch.equal(restored._slowmo_u, model._slowmo_u) and
            torch.equal(restored._slowmo_x_prev, model._slowmo_x_prev) and
            restored._slowmo_initialized is True and restored._slowmo_calls == model._slowmo_calls == 6 and
            torch.equal(restored.arena.flat, model.arena.flat))
    assert model._slowmo_u.abs().max().item() > 0
    # the same step from the same parameters on both: nothing else decides the result
    lr = types.SimpleNamespace(param_groups=[{'lr': 0.02}])
    for m in (model, restored):
        with torch.no_grad():
            m.arena.flat.add_(0.01 * (rank + 1))
        assert [m.perform_slowmo(lr) for _ in range(3)] == [False, False, True]
    after = (torch.equal(restored.arena.flat, model.arena.flat) and
             torch.equal(restored._slowmo_u, model._slowmo_u) and
             torch.equal(restored._slowmo_x_prev, model._slowmo_x_prev))
    return same, after


def test_checkpoint_round_trip():
    for same, after in run_distributed(_checkpoint_worker, 4):
        assert same and after


def test_world_of_one_applies_the_update():
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    model = GossipDataParallel(sim._model(0), graph=sgp.RingGraph(0, 1), rank=0, world_size=1,
                               slowmo_frequency=1, slowmo_lr=0.5, slowmo_momentum=0.9)
    opt = types.SimpleNamespace(param_groups=[{'lr': 0.1}])
    x0 = model.arena.flat.clone()
    assert model.perform_slowmo(opt)
    assert torch.equal(model.arena.flat, x0) and torch.equal(model._slowmo_x_prev, x0)
    with torch.no_grad():
        model.arena.flat.add_(0.25)
    z = model.arena.flat.clone()
    assert model.perform_slowmo(opt)
    u = (x0 - z) / 0.1
    torch.testing.assert_close(model._slowmo_u, u, rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(model.arena.flat, x0 - 0.5 * 0.1 * u, rtol=1e-6, atol=1e-6)
    with pytest.raises(ValueError, match='learning rate'):
        model.perform_slowmo(types.SimpleNamespace(param_groups=[{'lr': 0.0}]))


@pytest.mark.parametrize('kw', [
    dict(slowmo_frequency=-1), dict(slowmo_frequency=1.5), dict(slowmo_frequency=True),
    dict(slowmo_frequency=2, slowmo_lr=0.0), dict(slowmo_frequency=2, slowmo_lr=float('nan')),
    dict(slowmo_frequency=2, slowmo_momentum=1.0), dict(slowmo_frequency=2, slowmo_momentum=-0.1),
])
def test_invalid_arguments_raise(kw):
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    with pytest.raises(ValueError, match='slowmo'):
        GossipDataParallel(sim._model(0), graph=sgp.RingGraph(0, 1), rank=0, world_size=1, **kw)


def test_unsupported_configurations_raise():
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    with pytest.raises(ValueError, match='nprocs_per_node'):
        GossipDataParallel(sim._model(0), nprocs_per_node=2, rank=0, world_size=2, slowmo_frequency=3)
    with pytest.raises(ValueError, match='fp32'):
        GossipDataParallel(sim._model(0).double(), graph=sgp.RingGraph(0, 1), rank=0, world_size=1,
                           slowmo_frequency=3)


def test_cli_rejects_slowmo_where_unsupported(tmp_path):
    from stochastic_gradient_push_b200.cli.common import build_parser, finalize_args
    for adpsgd, extra, what in ((False, ['--all_reduce', 'True', '--graph_type', '-1'], '--all_reduce'),
                                (True, [], 'AD-PSGD'),
                                (False, ['--nprocs_per_node', '2'], 'nprocs_per_node'),
                                (False, ['--slowmo_momentum', '1.5'], 'slowmo_momentum')):
        args = build_parser(adpsgd=adpsgd).parse_args(
            ['--slowmo_frequency', '4', '--device', 'cpu', '--checkpoint_dir', str(tmp_path) + '/'] + extra)
        with pytest.raises(ValueError, match=what):
            finalize_args(args, adpsgd=adpsgd)
    args = build_parser().parse_args([])
    assert (args.slowmo_frequency, args.slowmo_lr, args.slowmo_momentum) == (0, 1.0, 0.5)


def test_gossip_sgd_cli_with_slowmo_two_ranks_cpu(tmp_path, master_port):
    from test_cli_and_experiment import COMMON, _torchrun
    args = COMMON + ['--push_sum', 'True', '--graph_type', '5', '--num_epochs', '1', '--num_itr_ignore', '0',
                     '--seed', '47', '--slowmo_frequency', '2', '--slowmo_momentum', '0.7',
                     '--checkpoint_dir', str(tmp_path) + '/']
    out = _torchrun(2, 'gossip_sgd.py', args, master_port)
    assert out.returncode == 0, out.stdout[-3000:]
    for r in range(2):
        assert len(open(str(tmp_path / ('out_r%d_n2.csv' % r))).read().splitlines()) > 2
