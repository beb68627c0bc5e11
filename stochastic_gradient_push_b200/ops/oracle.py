"""
Plain PyTorch oracles for the fused kernels (used by the numerics tests and by
the CPU fallback paths).  All functions are functional: they return new
tensors and never touch symmetric memory.
"""

from __future__ import annotations

from typing import List, Sequence, Tuple

import torch


def sgd_momentum(x, g, m, lr, momentum, weight_decay, nesterov, trust=None):
    """torch.optim.SGD (dampening 0) on the push-sum numerator; returns (x, m).  The
    hyper-parameters are scalars or per-element tensors (``nesterov`` then a bool tensor).
    ``trust``: per-element LARS trust ratios, d = trust * (g + wd * x)."""
    d = g + weight_decay * x
    if trust is not None:
        d = trust * d
    m = momentum * m + d
    if isinstance(nesterov, torch.Tensor):
        upd = torch.where(nesterov, d + momentum * m, m)
    else:
        upd = d + momentum * m if nesterov else m
    return x - lr * upd, m


def mix_columns(xs: Sequence[torch.Tensor], ws: Sequence[float], graphs, mixings
                ) -> Tuple[List[torch.Tensor], List[float]]:
    """One synchronous gossip step over all ranks:
    x_i <- a_ii x_i + sum_{j in in(i)} a_ji x_j  (same for the weights), where
    column j of A is what ``mixings[j]`` assigns to j's current out-edges."""
    n = len(xs)
    new_x = [None] * n
    new_w = [0.0] * n
    cols = []
    for j in range(n):
        outs, _ = graphs[j].get_peers()
        cols.append(mixings[j].scalar_weights(outs, rank=j))
    k = graphs[0].nprocs_per_node
    for i in range(n):
        self_w, _ = cols[i]
        acc = xs[i] * self_w
        w = ws[i] * self_w
        _, ins = graphs[i].get_peers()
        for j in ins:
            jj = j // k
            a = cols[jj][1][i * k]
            acc = acc + a * xs[jj]
            w = w + a * ws[jj]
        new_x[i], new_w[i] = acc, w
    return new_x, new_w


def rotate_all(graphs):
    for g in graphs:
        if g.is_dynamic_graph():
            g.get_peers(rotate=True)
