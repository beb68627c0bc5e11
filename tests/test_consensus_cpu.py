"""Consensus distance and the push-sum average model on the c10d plane (gloo, CPU):
``GossipDataParallel.consensus_distance`` / ``average_model`` / ``averaged`` against an fp64
computation from all-gathered parameters and weights, training that continues bit for bit, the
configurations that reject them, and the command line's ``--consensus_freq`` /
``--validate_average``."""

import pytest
import torch
import torch.distributed as dist

import stochastic_gradient_push_b200 as sgp

import test_distributed_c10d as sim
from dist_utils import run_distributed


def _gdp(rank, world, graph_name, ppi, push_sum, overlap, mixing):
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    graph = getattr(sgp, graph_name)(rank, world, peers_per_itr=ppi)
    mix = sgp.UniformMixing(graph, 'cpu') if mixing == 'uniform' else \
        sgp.SelfWeightedMixing(graph, 'cpu', self_weight=[0.3, 0.5, 0.6, 0.45])
    model = GossipDataParallel(sim._model(rank), graph=graph, mixing=mix, push_sum=push_sum,
                               overlap=overlap, rank=rank, world_size=world)
    assert model.transport == 'c10d'
    return model


def _train(model, rank, steps, overlap, call_at=(), record=None):
    opt = torch.optim.SGD(model.parameters(), lr=sim.LR, momentum=sim.MU, weight_decay=sim.WD)
    model.train()
    for step in range(steps):
        x, y = sim._batch(rank, step)
        ((model(x) - y) ** 2).mean().backward()
        opt.step()
        opt.zero_grad()
        if not overlap:
            model.transfer_params()
        if step in call_at:
            record(model)


def _check_worker(rank, world, graph_name, ppi, push_sum, overlap, mixing):
    model = _gdp(rank, world, graph_name, ppi, push_sum, overlap, mixing)
    out = []

    def record(m):
        sl = m.consensus_distance()
        avg = m.average_model()
        full = m.last_consensus
        z = m.arena.flat.clone()
        w = torch.tensor([float(m.ps_weight)], dtype=torch.float64)     # (fp32, as the kernel plane keeps it)
        zs = [torch.empty_like(z) for _ in range(world)]
        ws = [torch.empty_like(w) for _ in range(world)]
        dist.all_gather(zs, z)
        dist.all_gather(ws, w)
        with m.averaged() as st:
            inside = m.arena.flat.clone()
            inside_module = [v.detach().clone() for v in m.module.parameters()]
            assert st == full
        views_ok = all(torch.equal(p, v) for p, v in zip(inside_module, m.arena.views_of(inside)))
        restored = torch.equal(m.arena.flat, z) and views_ok and \
            all(torch.equal(p, v) for p, v in zip(m.module.parameters(), m.arena.views_of(z)))
        out.append(dict(slice=tuple(sl), relative=sl.relative, full=tuple(full), avg=avg.tolist(),
                        inside=inside.tolist(), restored=restored,
                        zs=[t.tolist() for t in zs], ws=[float(t) for t in ws]))
    _train(model, rank, 4, overlap, call_at=(1, 3), record=record)
    return out


@pytest.mark.parametrize('graph_name,ppi,push_sum,overlap,mixing', [
    ('NPeerDynamicDirectedExponentialGraph', 1, True, False, 'uniform'),      # SGP, regular
    ('DynamicDirectedExponentialGraph', 2, True, False, 'self_weighted'),    # SGP, w != 1
    ('RingGraph', 1, False, False, 'uniform'),                                # D-PSGD
    ('NPeerDynamicDirectedExponentialGraph', 1, True, True, 'self_weighted'),  # OSGP, w != 1
])
def test_matches_fp64_of_all_gathered_models(graph_name, ppi, push_sum, overlap, mixing):
    world = 4
    out = run_distributed(_check_worker, world, graph_name, ppi, push_sum, overlap, mixing)
    for call in range(2):
        recs = [out[r][call] for r in range(world)]
        ref = recs[0]
        zs = torch.tensor(ref['zs'], dtype=torch.float64)
        ws = torch.tensor(ref['ws'], dtype=torch.float64)
        zbar = (ws[:, None] * zs).sum(0) / ws.sum()
        per = ((zs - zbar) ** 2).sum(1)
        if mixing == 'self_weighted':
            assert (ws - 1).abs().max() > 1e-3
            plain = zs.mean(0)
            assert (plain - zbar).abs().max() > 1e-3 * zbar.abs().max()
        for r, rec in enumerate(recs):
            assert rec['zs'] == ref['zs'] and rec['ws'] == ref['ws']
            assert rec['slice'] == ref['slice'] and rec['full'] == ref['full'] and rec['avg'] == ref['avg']
            d, nrm, ranks = rec['slice']
            assert ranks is None
            assert abs(d - per.mean().item()) <= 1e-6 * per.mean().item()
            assert abs(nrm - (zbar ** 2).sum().item()) <= 1e-6 * nrm
            assert abs(rec['relative'] - (d / nrm) ** 0.5) <= 1e-12
            d_f, nrm_f, ranks_f = rec['full']
            assert d_f == d and nrm_f == nrm
            torch.testing.assert_close(torch.tensor(ranks_f, dtype=torch.float64), per, rtol=1e-6, atol=0)
            torch.testing.assert_close(torch.tensor(rec['avg'], dtype=torch.float64), zbar,
                                       rtol=1e-6, atol=1e-7)
            assert rec['inside'] == rec['avg'] and rec['restored']
            assert torch.equal(torch.tensor(rec['zs'][r]), torch.tensor(ref['zs'][r]))
        assert d > 0


def _continue_worker(rank, world):
    finals = []
    for call_at in ((), (0, 2, 3)):
        model = _gdp(rank, world, 'NPeerDynamicDirectedExponentialGraph', 1, True, False, 'uniform')

        def record(m):
            m.consensus_distance()
            with m.averaged():
                pass
            m.average_model()
        _train(model, rank, 6, False, call_at=call_at, record=record)
        model.sync_comms()
        model.unbias()
        finals.append((sim._flat(model.module).tolist(), float(model.ps_weight)))
    return finals


def test_training_after_a_call_is_bit_identical():
    out = run_distributed(_continue_worker, 4)
    for without, with_calls in out:
        assert without == with_calls


def _hier_reject_worker(rank, world):
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    model = GossipDataParallel(sim._model(rank), nprocs_per_node=2, rank=rank, world_size=world)
    msgs = []
    for fn in (model.consensus_distance, model.average_model, model.averaged().__enter__):
        try:
            fn()
        except ValueError as e:
            msgs.append(str(e))
    return msgs


def test_unsupported_configurations_raise():
    from stochastic_gradient_push_b200.parallel.ad_psgd import BilatGossipDataParallel
    from stochastic_gradient_push_b200.parallel.allreduce import AllReduceDataParallel
    for cls, what in ((BilatGossipDataParallel, 'AD-PSGD'), (AllReduceDataParallel, 'AllReduceDataParallel')):
        for name in ('consensus_distance', 'average_model', 'averaged'):
            with pytest.raises(ValueError, match=what):
                getattr(cls, name)(object())
    for msgs in run_distributed(_hier_reject_worker, 4):
        assert len(msgs) == 3 and all('nprocs_per_node' in m for m in msgs)


def test_world_of_one():
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    model = GossipDataParallel(sim._model(0), graph=sgp.RingGraph(0, 1), rank=0, world_size=1)
    st = model.consensus_distance()
    z = model.arena.flat.clone()
    assert st.distance_sq == 0.0 and st.relative == 0.0 and st.rank_distance_sq is None
    assert abs(st.average_norm_sq - z.double().pow(2).sum().item()) <= 1e-12
    assert torch.equal(model.average_model(), z)
    assert model.last_consensus.rank_distance_sq == [0.0]


def test_cli_rejects_consensus_flags_where_unsupported(tmp_path):
    from stochastic_gradient_push_b200.cli.common import build_parser, finalize_args
    for adpsgd, extra, what in ((False, ['--all_reduce', 'True', '--graph_type', '-1'], '--all_reduce'),
                                (True, [], 'AD-PSGD')):
        for flag in (['--consensus_freq', '5'], ['--validate_average', 'True']):
            args = build_parser(adpsgd=adpsgd).parse_args(
                flag + ['--device', 'cpu', '--checkpoint_dir', str(tmp_path) + '/'] + extra)
            with pytest.raises(ValueError, match=what):
                finalize_args(args, adpsgd=adpsgd)
    args = build_parser().parse_args([])
    assert args.consensus_freq == 0 and args.validate_average is False


def test_gossip_sgd_cli_logs_consensus_two_ranks_cpu(tmp_path, master_port):
    from test_cli_and_experiment import COMMON, _torchrun
    base = COMMON + ['--push_sum', 'True', '--graph_type', '5', '--num_epochs', '1',
                     '--num_itr_ignore', '0', '--seed', '47']
    runs = {}
    for tag, extra in (('plain', []), ('cons', ['--consensus_freq', '2', '--validate_average', 'True'])):
        d = tmp_path / tag
        d.mkdir()
        out = _torchrun(2, 'gossip_sgd.py', base + ['--checkpoint_dir', str(d) + '/'] + extra, master_port)
        assert out.returncode == 0, out.stdout[-3000:]
        runs[tag] = (d, out.stdout)
    d, stdout = runs['cons']
    assert 'consensus' in stdout
    for r in range(2):
        lines = open(str(d / ('consensus_r%d_n2.csv' % r))).read().splitlines()
        header = lines[0].split(',')
        assert header == ['epoch', 'itr', 'distance_sq', 'average_norm_sq', 'relative', 'avg_prec1']
        rows = [l.split(',') for l in lines[1:]]
        assert len(rows) >= 3
        assert all(float(row[2]) >= 0 and float(row[3]) > 0 for row in rows)
        assert any(row[5] != '' for row in rows)          # the epoch-end row validates the average
        # the per-iteration log keeps its format (timings differ between runs, not the columns)
        plain = open(str(runs['plain'][0] / ('out_r%d_n2.csv' % r))).read().splitlines()
        cons = open(str(d / ('out_r%d_n2.csv' % r))).read().splitlines()
        assert len(plain) == len(cons)
        assert [len(l.split(',')) for l in plain] == [len(l.split(',')) for l in cons]
