"""bf16 gossip messages (``GossipDataParallel(gossip_dtype=torch.bfloat16)``) on the c10d plane
(gloo, CPU) vs a whole-world simulation that rounds the messages the same way, push-sum mass
conservation, the wire size of a message, and the configurations that reject bf16 messages."""

import pytest
import torch

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.gossiper import (bf16_message_numel, bf16_message_weight,
                                                    pack_bf16_message)
from stochastic_gradient_push_b200.ops import oracle

import test_distributed_c10d as sim
from dist_utils import run_distributed

SELF_W = [0.3, 0.5, 0.6, 0.45]


def _mixing(kind, graph, device='cpu'):
    if kind == 'uniform':
        return sgp.UniformMixing(graph, device)
    return sgp.SelfWeightedMixing(graph, device, self_weight=SELF_W)


def _simulate_bf16(world, graph_name, ppi, steps, mixing, naive=False):
    """``test_distributed_c10d._simulate`` (synchronous, SGD on the numerators) with the c10d
    plane's bf16 messages: rank j sends m = Q(a_ij * x_j) to each out-neighbour i and keeps
    x_j - sum of what it sent; weights travel in fp32.  ``naive``: the sender keeps a_jj * x_j
    instead (the mass-drifting variant).  Returns (z, w, mass): ``mass`` is sum_i x_i(0) plus every
    SGD update of the run, i.e. what sum_i z_i * w_i would be with no gossip at all."""
    models = [sim._model(r) for r in range(world)]
    graphs = [getattr(sgp, graph_name)(r, world, peers_per_itr=ppi) for r in range(world)]
    mix = [_mixing(mixing, g) for g in graphs]
    ws = [1.0] * world
    moms = [torch.zeros_like(sim._flat(m)) for m in models]
    xs = [sim._flat(m).clone() for m in models]
    mass = sum(x.double() for x in xs)

    def load(m, flat):
        off = 0
        for p in m.parameters():
            p.data.copy_(flat[off:off + p.numel()].view_as(p))
            off += p.numel()

    for step in range(steps):
        grads = []
        for i, m in enumerate(models):
            load(m, xs[i] / ws[i])
            m.zero_grad()
            x, y = sim._batch(i, step)
            ((m(x) - y) ** 2).mean().backward()
            grads.append(torch.cat([p.grad.reshape(-1) for p in m.parameters()]))
        for i in range(world):
            new, moms[i] = oracle.sgd_momentum(xs[i], grads[i], moms[i], sim.LR, sim.MU, sim.WD, False)
            mass = mass + (new.double() - xs[i].double())
            xs[i] = new
        # exchange, in the data plane's order: the sender subtracts its messages (one per
        # out-edge), the receiver adds the remote in-messages, then its self-edge messages
        edges = [g.get_edges() for g in graphs]
        sent, wsent, kept, wkept = [], [], [], []
        for j in range(world):
            outs, _ = edges[j]
            self_w, edge_w = mix[j].scalar_weights([e.dest for e in outs], rank=j)
            q = {e.dest: (xs[j] * float(edge_w[e.dest])).to(torch.bfloat16) for e in outs}
            wq = {e.dest: float(torch.tensor(ws[j] * float(edge_w[e.dest]), dtype=torch.float32))
                  for e in outs}
            loc = xs[j].clone()
            if naive:
                loc = loc * self_w
            else:
                for e in outs:
                    loc = loc - q[e.dest].float()
            sent.append(q)
            wsent.append(wq)
            kept.append(loc)
            wkept.append(ws[j] * self_w)
        for i in range(world):
            outs, ins = edges[i]
            acc, w = kept[i], wkept[i]
            for e in [e for e in ins if e.src != e.dest] + [e for e in outs if e.src == e.dest]:
                acc = acc + sent[e.src][i].float()
                w = w + wsent[e.src][i]
            xs[i], ws[i] = acc, w
        oracle.rotate_all(graphs)
    return [x / w for x, w in zip(xs, ws)], ws, mass


def _worker(rank, world, graph_name, ppi, steps, push_sum, mixing):
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    graph = getattr(sgp, graph_name)(rank, world, peers_per_itr=ppi)
    model = GossipDataParallel(sim._model(rank), graph=graph, mixing=_mixing(mixing, graph),
                               push_sum=push_sum, rank=rank, world_size=world,
                               gossip_dtype=torch.bfloat16)
    assert model.transport == 'c10d' and model.gossip_dtype == torch.bfloat16
    opt = torch.optim.SGD(model.parameters(), lr=sim.LR, momentum=sim.MU, weight_decay=sim.WD)
    model.train()
    for step in range(steps):
        x, y = sim._batch(rank, step)
        ((model(x) - y) ** 2).mean().backward()
        opt.step()
        opt.zero_grad()
        model.transfer_params()
    model.sync_comms()
    model.unbias()
    sd = model.state_dict()
    wire = {k: (b.numel() * b.element_size(), model.arena.total) for k, b in model._c10d.send_bufs.items()}
    return sim._flat(model.module).tolist(), float(sd['ps_weight']), sd.get('gossip_dtype'), wire


@pytest.mark.parametrize('graph_name,ppi,push_sum,mixing', [
    ('NPeerDynamicDirectedExponentialGraph', 1, True, 'uniform'),        # SGP, regular
    ('DynamicDirectedExponentialGraph', 2, True, 'self_weighted'),      # SGP, irregular weights
    ('RingGraph', 1, False, 'uniform'),                                  # D-PSGD
    ('DynamicBipartiteExponentialGraph', 1, False, 'self_weighted'),    # D-PSGD, irregular weights
])
def test_bf16_messages_match_simulation_and_conserve_mass(graph_name, ppi, push_sum, mixing):
    world, steps = 4, 5
    out = run_distributed(_worker, world, graph_name, ppi, steps, push_sum, mixing)
    want, ws, mass = _simulate_bf16(world, graph_name, ppi, steps, mixing)
    got_mass = torch.zeros_like(mass)
    for r in range(world):
        got, w, dtype_rec, _ = out[r]
        torch.testing.assert_close(torch.tensor(got), want[r], rtol=1e-4, atol=1e-5)
        assert abs(w - ws[r]) < 1e-5
        assert dtype_rec == 'bfloat16'
        got_mass += torch.tensor(got, dtype=torch.float64) * w
    # sum_i x_i after gossip == the same SGD updates with no gossip, to fp32 rounding
    torch.testing.assert_close(got_mass, mass, rtol=0, atol=1e-5)
    # ... and the check sees the bug: keeping a_jj * x_j while sending Q(a_ij * x_j) drifts
    zn, wn, mass_n = _simulate_bf16(world, graph_name, ppi, steps, mixing, naive=True)
    drift = sum(z.double() * w for z, w in zip(zn, wn)) - mass_n
    assert drift.abs().max().item() > 1e-4


def test_message_is_half_the_bytes_on_the_wire():
    for n in (53, 54, 25_557_032):
        assert bf16_message_numel(n) * 2 == 2 * n + (2 if n & 1 else 0) + 4
    x = torch.randn(53)
    msg = torch.empty(bf16_message_numel(53), dtype=torch.bfloat16)
    q = pack_bf16_message(msg, x, 0.25, 0.123456789)
    assert torch.equal(msg[:53], (x * 0.25).to(torch.bfloat16)) and torch.equal(q, msg[:53])
    # the push-sum weight is not rounded to bf16
    assert bf16_message_weight(msg, 53) == float(torch.tensor(0.123456789, dtype=torch.float32))
    # what a rank really sends: one message per out-edge of n * 2 + a constant bytes
    out = run_distributed(_worker, 2, 'RingGraph', 1, 1, True, 'uniform')
    for _, _, _, wire in out:
        assert wire
        for nbytes, n in wire.values():        # (n: the parameter arena's length)
            assert nbytes == n * 2 + (2 if n & 1 else 0) + 4
            assert nbytes < (n + 1) * 4 * 0.51


def test_unsupported_combinations_raise():
    from stochastic_gradient_push_b200.parallel.ad_psgd import BilatGossipDataParallel
    from stochastic_gradient_push_b200.parallel.allreduce import AllReduceDataParallel
    from stochastic_gradient_push_b200.parallel.distributed import GossipDataParallel
    bf16 = torch.bfloat16
    graph = sgp.RingGraph(0, 2)
    with pytest.raises(ValueError, match='overlap=True'):
        GossipDataParallel(sim._model(0), graph=graph, overlap=True, rank=0, world_size=2, gossip_dtype=bf16)
    with pytest.raises(ValueError, match='nprocs_per_node'):
        GossipDataParallel(sim._model(0), graph=graph, nprocs_per_node=2, rank=0, world_size=4, gossip_dtype=bf16)
    with pytest.raises(ValueError, match='gossip_dtype must be'):
        GossipDataParallel(sim._model(0), graph=graph, rank=0, world_size=2, gossip_dtype=torch.float16)
    with pytest.raises(ValueError, match='BilatGossipDataParallel'):
        BilatGossipDataParallel(sim._model(0), rank=0, world_size=2, gossip_dtype=bf16)
    with pytest.raises(ValueError, match='AllReduceDataParallel'):
        AllReduceDataParallel(sim._model(0), rank=0, world_size=1, gossip_dtype=bf16)


@pytest.mark.parametrize('adpsgd,extra,what', [
    (False, ['--overlap', 'True'], '--overlap'),
    (False, ['--all_reduce', 'True', '--graph_type', '-1'], '--all_reduce'),
    (False, ['--nprocs_per_node', '2'], '--nprocs_per_node'),
    (True, [], 'AD-PSGD'),
])
def test_cli_rejects_bf16_messages_where_unsupported(tmp_path, adpsgd, extra, what):
    from stochastic_gradient_push_b200.cli.common import build_parser, finalize_args
    args = build_parser(adpsgd=adpsgd).parse_args(
        ['--gossip_dtype', 'bf16', '--device', 'cpu', '--checkpoint_dir', str(tmp_path) + '/'] + extra)
    with pytest.raises(ValueError, match=what):
        finalize_args(args, adpsgd=adpsgd)


def test_cli_parses_gossip_dtype():
    from stochastic_gradient_push_b200.cli.common import build_parser
    assert build_parser().parse_args([]).gossip_dtype == 'fp32'
    assert build_parser().parse_args(['--gossip_dtype', 'bf16']).gossip_dtype == 'bf16'
    with pytest.raises(SystemExit):
        build_parser().parse_args(['--gossip_dtype', 'fp16'])


def test_gossip_sgd_cli_bf16_messages_two_ranks_cpu(tmp_path, master_port):
    from test_cli_and_experiment import COMMON, _torchrun
    out = _torchrun(2, 'gossip_sgd.py', COMMON + [
        '--push_sum', 'True', '--graph_type', '5', '--gossip_dtype', 'bf16',
        '--num_epochs', '1', '--checkpoint_dir', str(tmp_path) + '/', '--num_itr_ignore', '0'],
        master_port)
    assert out.returncode == 0, out.stdout[-3000:]
    for r in range(2):
        lines = open(str(tmp_path / ('out_r%d_n2.csv' % r))).read().splitlines()
        rows = [l.split(',') for l in lines[5:]]
        assert rows and all(len(row) == 18 for row in rows)
