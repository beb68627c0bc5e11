"""
Graph managers: the six gossip topologies behind the reference's
``GraphManager`` API (``gossip/graph_manager.py:35-279``), rebuilt on top of the
pure-math :class:`~.schedule.PeerSchedule`.

Differences from the reference that are deliberate:

* **No process groups are needed.**  The reference creates one 2-rank NCCL
  group per phone-book entry (``gossip/graph_manager.py:27``) to emulate
  point-to-point sends with broadcasts.  Here the data plane is one-sided P2P
  loads over NVSwitch peer memory, so a graph is plain integers and can be
  built on a CPU-only host, inside unit tests, with no ``torch.distributed``.
  ``Edge.process_group`` is ``None`` unless :meth:`materialize_process_groups`
  is called (collective; only useful for reference-style broadcast transports).
* **The graph emits a device table** (:meth:`device_table`): per phase the in-
  and out-neighbours of this rank as an int32 tensor that the sm_90a kernels
  index with ``step % period`` -- the per-step neighbour list never touches
  Python on the hot path.
* ``world_size == 1`` is a valid (peer-less) graph instead of a math domain
  error.
"""

from __future__ import annotations

from typing import List, Optional, Tuple

from .schedule import PeerSchedule, make_schedule

MAX_PEERS_PER_ITR = 8   # compile-time bound shared with ops/csrc/sgp_kernels.cuh


class Edge(object):
    """Directed edge ``src -> dest`` (process-level ranks)."""

    __slots__ = ('src', 'dest', 'process_group')

    def __init__(self, src: int, dest: int, process_group=None):
        self.src = src
        self.dest = dest
        self.process_group = process_group

    def __repr__(self):
        return 'Edge(%d->%d)' % (self.src, self.dest)

    def __eq__(self, other):
        return isinstance(other, Edge) and (self.src, self.dest) == (other.src, other.dest)

    def __hash__(self):
        return hash((self.src, self.dest))


class GraphManager(object):
    """Base class; subclasses set ``KIND`` and the four predicates."""

    KIND: str = None
    _REGULAR = True
    _BIPARTITE = False
    _DYNAMIC = True

    def __init__(self, rank, world_size, nprocs_per_node=1, local_rank=0,
                 peers_per_itr=1, dedupe=False):
        assert int(peers_per_itr) >= 1
        assert int(peers_per_itr) <= MAX_PEERS_PER_ITR
        self.rank = rank
        self.world_size = world_size
        self.nprocs_per_node = nprocs_per_node
        self.local_rank = local_rank
        self.dedupe = dedupe
        self._peers_per_itr = int(peers_per_itr)
        self._schedule = self._make_graph()
        k = nprocs_per_node
        self.phone_book: List[List[Edge]] = [
            [Edge(r * k, p * k) for p in book]
            for r, book in enumerate(self._schedule.books)]

    # -- construction ------------------------------------------------------ #
    def _make_graph(self) -> PeerSchedule:
        if self.KIND is None:
            raise NotImplementedError
        return make_schedule(self.KIND, self.rank, self.world_size,
                             self._peers_per_itr, self.dedupe)

    def materialize_process_groups(self):
        """Collectively create a 2-rank group per edge (reference behaviour,
        ``gossip/graph_manager.py:27``).  Every rank must call this."""
        import torch.distributed as dist
        for book in self.phone_book:
            for e in book:
                if e.process_group is None and e.src != e.dest:
                    e.process_group = dist.new_group([e.src, e.dest])

    # -- peers-per-iteration ------------------------------------------------ #
    @property
    def peers_per_itr(self):
        return self._peers_per_itr

    @peers_per_itr.setter
    def peers_per_itr(self, v):
        # reference: the phone book is NOT rebuilt, only the window is reset
        # (gossip/graph_manager.py:52-56)
        self._peers_per_itr = int(v)
        self._schedule.peers_per_itr = int(v)
        self._schedule.reset()

    @property
    def _group_indices(self):
        return self._schedule.slots

    @_group_indices.setter
    def _group_indices(self, v):
        self._schedule.slots = list(v)

    # -- predicates --------------------------------------------------------- #
    def is_regular_graph(self):
        return self._REGULAR

    def is_bipartite_graph(self):
        return self._BIPARTITE

    def is_passive(self, rank=None):
        if not self._BIPARTITE:
            return False
        rank = self.rank if rank is None else rank
        return (rank % 2) == 0

    def is_dynamic_graph(self, graph_type=None):
        return self._DYNAMIC

    # -- queries ------------------------------------------------------------ #
    def _rotate_group_indices(self):
        self._schedule.rotate()

    def get_peers(self, rotate=False) -> Tuple[List[int], List[int]]:
        """(out_peers, in_peers) as process-level ranks for ``self.rank``."""
        if rotate:
            self._rotate_group_indices()
        k = self.nprocs_per_node
        outs, ins = self._schedule.current()
        return [p * k for p in outs], [p * k for p in ins]

    def get_edges(self, rotate=False) -> Tuple[List[Edge], List[Edge]]:
        if rotate:
            self._rotate_group_indices()
        out_edges, in_edges = [], []
        for s in self._schedule.slots:
            if s < len(self.phone_book[self.rank]):
                out_edges.append(self.phone_book[self.rank][s])
            for r, book in enumerate(self.phone_book):
                if s >= len(book):
                    continue
                if book[s].dest == self.rank * self.nprocs_per_node:
                    in_edges.append(book[s])
        return out_edges, in_edges

    def _rotate_forward(self, r, p):
        return (r + p) % self.world_size

    def _rotate_backward(self, r, p):
        return (r - p) % self.world_size

    # -- device-side neighbour table --------------------------------------- #
    @property
    def period(self) -> int:
        return self._schedule.period if self._DYNAMIC else 1

    def phase_index(self) -> int:
        return self._schedule.phase_index() if self._DYNAMIC else 0

    def phases(self):
        """[(out_peers, in_peers)] for one period (node-level ranks)."""
        ph = self._schedule.phases()
        return ph if self._DYNAMIC else ph[:1]

    def device_table(self, device=None):
        """int32 tensor ``[period, 2 + 2*MAX_PEERS_PER_ITR]``; row t is
        ``[n_in, n_out, in_0..in_7, out_0..out_7]`` (-1 padded) for the window
        a freshly reset graph uses at its t-th iteration.  Ranks are
        node-level indices into the symmetric peer table."""
        import torch
        rows = []
        for outs, ins in self.phases():
            assert len(ins) <= MAX_PEERS_PER_ITR and len(outs) <= MAX_PEERS_PER_ITR
            row = [len(ins), len(outs)]
            row += ins + [-1] * (MAX_PEERS_PER_ITR - len(ins))
            row += outs + [-1] * (MAX_PEERS_PER_ITR - len(outs))
            rows.append(row)
        return torch.tensor(rows, dtype=torch.int32, device=device)


class DynamicDirectedExponentialGraph(GraphManager):
    KIND = 'dde'


class NPeerDynamicDirectedExponentialGraph(GraphManager):
    KIND = 'npdde'


class DynamicBipartiteExponentialGraph(GraphManager):
    KIND = 'dbe'
    _BIPARTITE = True


class DynamicDirectedLinearGraph(GraphManager):
    KIND = 'ddl'


class DynamicBipartiteLinearGraph(GraphManager):
    KIND = 'dbl'
    _BIPARTITE = True


class RingGraph(GraphManager):
    KIND = 'ring'
    _DYNAMIC = False


GRAPH_TOPOLOGIES = {
    0: DynamicDirectedExponentialGraph,
    1: DynamicBipartiteExponentialGraph,
    2: DynamicDirectedLinearGraph,
    3: DynamicBipartiteLinearGraph,
    4: RingGraph,
    5: NPeerDynamicDirectedExponentialGraph,
    -1: None,
}
