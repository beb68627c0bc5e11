"""
Pure-math peer schedules for gossip topologies.

This module knows nothing about process groups, CUDA or torch.distributed: a
topology is a *phone book* -- for every rank the ordered list of ranks it may
push to -- plus a window of ``peers_per_itr`` consecutive phone-book slots that
is active in a given iteration and slides by ``peers_per_itr`` every time the
graph is rotated.  Everything the transports need (the c10d fallback, the
device-side neighbour table indexed by the sm_90a mix kernels) is derived from
this one structure.

Parity notes (reference = facebookresearch/stochastic_gradient_push):

* slot layout and rotation follow ``gossip/graph_manager.py:91-133`` (out-peers
  are the active slots of this rank's book, in-peers are every *other* rank
  whose book points at this rank in the same slot; rotation advances each slot
  index by ``peers_per_itr`` modulo the length of this rank's book);
* the reference's ``_add_peers`` de-duplication never fires
  (``gossip/graph_manager.py:66-73`` compares an int with ``Edge`` objects), so
  books keep repeated peers, e.g. n=8 directed-exponential is ``[1,7,2,6,4,4]``.
  ``dedupe=False`` (default) reproduces that sequence; ``dedupe=True`` gives the
  schedule the reference *intended*.
"""

from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Sequence, Tuple


def _ilog(x: float, base: float) -> int:
    """``int(log_base(x))`` exactly as the reference evaluates it with floats."""
    return int(math.log(x, base))


def fwd(rank: int, hops: int, n: int) -> int:
    return (rank + hops) % n


def bwd(rank: int, hops: int, n: int) -> int:
    return (rank - hops) % n


# --------------------------------------------------------------------------- #
# phone-book builders: rank -> ordered list of destination ranks
# --------------------------------------------------------------------------- #
def _exp_levels(n: int, base: int) -> range:
    if n < 2:
        return range(0)
    return range(0, _ilog(n - 1, base) + 1)


def book_directed_exponential(n: int, ppi: int = 1) -> List[List[int]]:
    """+-2^i for i in [0, floor(log2(n-1))]  (gossip/graph_manager.py:149-164)."""
    books = []
    for r in range(n):
        peers = []
        for i in _exp_levels(n, 2):
            peers += [fwd(r, 2 ** i, n), bwd(r, 2 ** i, n)]
        books.append(peers)
    return books


def book_npeer_directed_exponential(n: int, ppi: int = 1) -> List[List[int]]:
    """forward hops j*(ppi+1)^i, j in [1,ppi]  (gossip/graph_manager.py:167-184)."""
    books = []
    for r in range(n):
        peers = []
        for i in _exp_levels(n, ppi + 1):
            for j in range(1, ppi + 1):
                peers.append(fwd(r, j * (ppi + 1) ** i, n))
        books.append(peers)
    return books


def _passive(rank: int) -> bool:
    return rank % 2 == 0


def _bipartite_filter(r: int, f: int, b: int) -> bool:
    """Keep the pair only if it crosses the even/odd partition on both sides."""
    if not _passive(r):
        return _passive(f) and _passive(b)
    return not (_passive(f) or _passive(b))


def book_bipartite_exponential(n: int, ppi: int = 1) -> List[List[int]]:
    """+-1, +-(1+2^i); even ranks passive  (gossip/graph_manager.py:187-215)."""
    books = []
    for r in range(n):
        peers = []
        for i in _exp_levels(n, 2):
            hop = 1 if i == 0 else 1 + 2 ** i
            f, b = fwd(r, hop, n), bwd(r, hop, n)
            if _bipartite_filter(r, f, b):
                peers += [f, b]
        books.append(peers)
    return books


def book_directed_linear(n: int, ppi: int = 1) -> List[List[int]]:
    """+-i for odd i < n  (gossip/graph_manager.py:218-235)."""
    books = []
    for r in range(n):
        peers = []
        for i in range(1, n, 2):
            peers += [fwd(r, i, n), bwd(r, i, n)]
        books.append(peers)
    return books


def book_bipartite_linear(n: int, ppi: int = 1) -> List[List[int]]:
    """+-i for all i < n crossing the partition  (gossip/graph_manager.py:238-262)."""
    books = []
    for r in range(n):
        peers = []
        for i in range(1, n):
            f, b = fwd(r, i, n), bwd(r, i, n)
            if _bipartite_filter(r, f, b):
                peers += [f, b]
        books.append(peers)
    return books


def book_ring(n: int, ppi: int = 1) -> List[List[int]]:
    """+1, -1, static  (gossip/graph_manager.py:265-279)."""
    return [[fwd(r, 1, n), bwd(r, 1, n)] for r in range(n)]


def _dedupe(book: Sequence[int]) -> List[int]:
    seen, out = set(), []
    for p in book:
        if p not in seen:
            seen.add(p)
            out.append(p)
    return out


# --------------------------------------------------------------------------- #
# Schedule
# --------------------------------------------------------------------------- #
@dataclass
class PeerSchedule:
    """Phone books of all ranks + the sliding active-slot window of one rank."""

    world_size: int
    books: List[List[int]]
    rank: int
    peers_per_itr: int = 1
    slots: List[int] = field(default_factory=list)

    def __post_init__(self):
        if not self.slots:
            self.reset()

    # -- window ------------------------------------------------------------ #
    def reset(self):
        self.slots = list(range(self.peers_per_itr))

    def rotate(self):
        period = len(self.books[self.rank])
        if period == 0:
            return
        self.slots = [(s + self.peers_per_itr) % period for s in self.slots]

    # -- queries ----------------------------------------------------------- #
    def peers_at(self, slots: Sequence[int], rank: int = None
                 ) -> Tuple[List[int], List[int]]:
        """(out_peers, in_peers) of ``rank`` for the given active slots."""
        rank = self.rank if rank is None else rank
        outs, ins = [], []
        my_book = self.books[rank]
        for s in slots:
            if s < len(my_book):
                outs.append(my_book[s])
            for other, book in enumerate(self.books):
                # a self-edge (e.g. n=2, ppi=2 -> book [1, 0]) is delivered
                # locally so the mixing stays column-stochastic; the reference
                # skips it (gossip/graph_manager.py:101-102) and loses the mass
                if s < len(book) and book[s] == rank:
                    ins.append(other)
        return outs, ins

    def current(self) -> Tuple[List[int], List[int]]:
        return self.peers_at(self.slots)

    @property
    def period(self) -> int:
        """Number of distinct window positions before the schedule repeats."""
        length = len(self.books[self.rank])
        if length == 0:
            return 1
        return length // math.gcd(length, self.peers_per_itr)

    def phases(self, rank: int = None) -> List[Tuple[List[int], List[int]]]:
        """(out, in) for every phase of one full period starting at the reset
        window; phase ``t`` is what a freshly reset graph uses at iteration t."""
        length = max(len(self.books[self.rank]), 1)
        slots = list(range(self.peers_per_itr))
        out = []
        for _ in range(self.period):
            out.append(self.peers_at(slots, rank))
            slots = [(s + self.peers_per_itr) % length for s in slots]
        return out

    def phase_index(self) -> int:
        """Index into :meth:`phases` of the current window."""
        length = max(len(self.books[self.rank]), 1)
        slots = list(range(self.peers_per_itr))
        for t in range(self.period):
            if slots == self.slots:
                return t
            slots = [(s + self.peers_per_itr) % length for s in slots]
        raise RuntimeError('window %r is not on the rotation orbit' % (self.slots,))


BOOK_BUILDERS: Dict[str, Callable[[int, int], List[List[int]]]] = {
    'dde': book_directed_exponential,
    'npdde': book_npeer_directed_exponential,
    'dbe': book_bipartite_exponential,
    'ddl': book_directed_linear,
    'dbl': book_bipartite_linear,
    'ring': book_ring,
}


def make_schedule(kind: str, rank: int, world_size: int, peers_per_itr: int = 1,
                  dedupe: bool = False) -> PeerSchedule:
    books = BOOK_BUILDERS[kind](world_size, peers_per_itr)
    if dedupe:
        books = [_dedupe(b) for b in books]
    return PeerSchedule(world_size, books, rank, peers_per_itr)
