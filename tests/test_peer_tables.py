"""Device schedule tables (ops/peer_mix.build_tables): the receiver-side edge weights the sm_90a
gossip kernel multiplies its P2P loads with.  Host logic only -- no GPU.

Push-sum needs a COLUMN-stochastic mixing matrix every step: whatever rank j keeps for itself plus
whatever each of its out-neighbours takes from it must sum to 1 -- otherwise mass leaks and the
de-biased average drifts.  Because the kernel lets the *receiver* apply the sender's weight, that
property lives in these tables."""
import pytest
import torch

import stochastic_gradient_push_b200 as sgp
from stochastic_gradient_push_b200.mixing_manager import SelfWeightedMixing, UniformMixing
from stochastic_gradient_push_b200.ops.peer_mix import build_tables
from stochastic_gradient_push_b200.topology.graph_manager import MAX_PEERS_PER_ITR as MP

GRAPHS = ['DynamicDirectedExponentialGraph', 'NPeerDynamicDirectedExponentialGraph',
          'DynamicBipartiteExponentialGraph', 'DynamicDirectedLinearGraph',
          'DynamicBipartiteLinearGraph', 'RingGraph']


def _world_tables(name, world, ppi, mixing_factory):
    tabs = []
    for r in range(world):
        g = getattr(sgp, name)(r, world, peers_per_itr=ppi)
        tabs.append(build_tables(g, mixing_factory(g, r), 'cpu'))
    return tabs


def _column_sums(tabs, world):
    """sums[t][j] = self weight of j + everything j's out-neighbours take from j at phase t."""
    period = tabs[0][0].shape[0]
    sums = torch.zeros(period, world, dtype=torch.float64)
    for i, (table, wtable) in enumerate(tabs):
        assert table.shape[0] == wtable.shape[0] == period
        for t in range(period):
            n_in = int(table[t, 0])
            sums[t, i] += float(wtable[t, 0])                     # self loop
            for k in range(n_in):
                j = int(table[t, 2 + k])
                sums[t, j] += float(wtable[t, 1 + k])             # i pulls w from j
            assert torch.all(wtable[t, 1 + n_in:] == 0)           # padding carries no weight
    return sums


@pytest.mark.parametrize('name', GRAPHS)
@pytest.mark.parametrize('world,ppi', [(2, 1), (4, 1), (8, 1), (8, 2), (6, 1)])
def test_uniform_mixing_tables_are_column_stochastic(name, world, ppi):
    tabs = _world_tables(name, world, ppi, lambda g, r: UniformMixing(g, 'cpu'))
    sums = _column_sums(tabs, world)
    torch.testing.assert_close(sums, torch.ones_like(sums), rtol=0, atol=1e-6)


@pytest.mark.parametrize('name', ['NPeerDynamicDirectedExponentialGraph', 'RingGraph',
                                  'DynamicDirectedExponentialGraph'])
def test_rank_dependent_mixing_stays_column_stochastic(name):
    """Irregular weights (every rank keeps a different share): the receiver must look up the SENDER's
    weights, which is exactly what build_tables encodes."""
    world = 8
    shares = [0.2 + 0.08 * r for r in range(world)]
    tabs = _world_tables(name, world, 1, lambda g, r: SelfWeightedMixing(g, 'cpu', self_weight=shares))
    sums = _column_sums(tabs, world)
    torch.testing.assert_close(sums, torch.ones_like(sums), rtol=0, atol=1e-6)
    for r, (_, wtable) in enumerate(tabs):
        assert abs(float(wtable[0, 0]) - shares[r]) < 1e-6        # self weight is the rank's own share


def test_table_shapes_and_in_neighbour_order():
    g = sgp.NPeerDynamicDirectedExponentialGraph(3, 8, peers_per_itr=2)
    table, wtable = build_tables(g, UniformMixing(g, 'cpu'), 'cpu')
    assert table.dtype == torch.int32 and wtable.dtype == torch.float32
    assert table.shape == (g.period, 2 + 2 * MP) and wtable.shape == (g.period, 1 + MP)
    for t, (outs, ins) in enumerate(g.phases()):
        assert table[t, 2:2 + len(ins)].tolist() == ins           # weights are listed in this order
        assert table[t, 2 + MP:2 + MP + len(outs)].tolist() == outs
        assert abs(float(wtable[t, 0]) - 1.0 / (len(outs) + 1)) < 1e-7
