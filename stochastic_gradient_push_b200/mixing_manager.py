"""
Mixing managers: the weights of one gossip step.

API parity with ``gossip/mixing_manager.py:19-56`` (``MixingManager``,
``UniformMixing``; ``get_mixing_weights`` returns a dict with ``'lo'``,
``'uniform'`` and one entry per out-peer rank).  In addition every manager can
answer :meth:`scalar_weights` -- plain Python floats ``(self_weight,
{out_peer: weight})`` -- which is what the fused sm_90a kernels consume: the
sender publishes its per-edge weight next to its outbox and the *receiver*
applies it while it accumulates the P2P loads, so no "scale the message"
kernel (reference K6, ``gossip/gossiper.py:139-147``) ever runs.
"""

import torch


class MixingManager(object):

    def __init__(self, graph, device=None):
        self.graph_manager = graph
        self.device = device

    def is_regular(self):
        """True iff the stationary distribution is uniform, i.e. the push-sum
        weight stays at 1 and need not be communicated."""
        return self.graph_manager.is_regular_graph() and self.is_uniform()

    def is_uniform(self):
        raise NotImplementedError

    def scalar_weights(self, out_peers=None, rank=None):
        """(self_weight, {out_peer_rank: edge_weight}) as floats: the column of
        the mixing matrix owned by ``rank`` (default: this rank) when it pushes
        to ``out_peers`` (default: the graph's current out-peers).  Columns sum
        to 1.  Receivers evaluate their in-neighbours' columns with this."""
        raise NotImplementedError

    def get_mixing_weights(self, residual_adjusted=True):
        """Reference-shaped dict of 1-element tensors.  ``residual_adjusted``
        divides the edge weights by the self weight (the caller has already
        scaled, or will lazily scale, its message by ``lo``)."""
        out_peers, _ = self.graph_manager.get_peers()
        lo, edge = self.scalar_weights(out_peers)
        mk = lambda v: torch.tensor([v], device=self.device)   # noqa: E731
        weights = {'lo': mk(lo)}
        scale = lo if residual_adjusted else 1.0
        if self.is_uniform():
            uni = next(iter(edge.values())) if edge else lo
            weights['uniform'] = mk(uni / scale)
        for peer, w in edge.items():
            weights[peer] = mk(w / scale)
        return weights


class UniformMixing(MixingManager):
    """Every out-edge and the self-loop get 1/(out_degree+1)."""

    def is_uniform(self):
        return True

    def scalar_weights(self, out_peers=None, rank=None):
        if out_peers is None:
            out_peers, _ = self.graph_manager.get_peers()
        w = 1.0 / (len(out_peers) + 1.0)
        return w, {p: w for p in out_peers}


class SelfWeightedMixing(MixingManager):
    """Non-uniform column-stochastic mixing: keep ``self_weight`` locally and
    split the remainder evenly over the out-peers.  Not regular, so the
    push-sum weight drifts from 1 and is carried through the gossip -- this
    exercises the "irregular" half of the API that is dead code in the
    reference tree (``gossip/gossiper.py:83-85, 131-132, 163-164``)."""

    def __init__(self, graph, device=None, self_weight=0.5):
        """``self_weight``: float, or a callable / sequence indexed by
        (node-level) rank for a genuinely non-doubly-stochastic matrix."""
        super().__init__(graph, device)
        self.self_weight = self_weight

    def _sw(self, rank):
        rank = self.graph_manager.rank if rank is None else rank
        sw = self.self_weight
        if callable(sw):
            sw = sw(rank)
        elif isinstance(sw, (list, tuple)):
            sw = sw[rank % len(sw)]
        sw = float(sw)
        assert 0.0 < sw < 1.0
        return sw

    def is_uniform(self):
        return False

    def is_regular(self):
        return False

    def scalar_weights(self, out_peers=None, rank=None):
        if out_peers is None:
            out_peers, _ = self.graph_manager.get_peers()
        if not out_peers:
            return 1.0, {}
        sw = self._sw(rank)
        w = (1.0 - sw) / len(out_peers)
        return sw, {p: w for p in out_peers}


MIXING_STRATEGIES = {
    0: UniformMixing,
    1: SelfWeightedMixing,
    -1: None,
}
