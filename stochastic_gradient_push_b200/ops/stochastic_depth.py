"""
Stochastic depth (Huang et al., ECCV 2016) for the residual blocks: timm's ``DropPath(scale_by_keep=True)``
/ torchvision's ``stochastic_depth(mode='row')`` on the residual branch, with timm's linear rate rule.

In a training forward, block ``l`` of ``L`` drops with ``p_l = p * l / (L - 1)`` (block 0 never drops, the
last drops with ``p``): sample ``n`` gets the branch scale ``s_n = 0`` with probability ``p_l``, otherwise
``1 / (1 - p_l)``, and the block computes ``relu(s_n * bn(conv(x)) + identity)``.  The scale enters the
fused BatchNorm kernels and the conv1x1 dgrad epilogue (``ops.fused_bn``: ``branch_scale``), so the fused
hot path stays intact.

:meth:`StochasticDepth.draw` writes all ``L x N`` scales of one forward in ONE launch
(``csrc/drop_path_kernels.cu``) from a counter-based hash of ``(seed, rank, draw index, block, sample)``.
The draw index lives in device memory and the same launch increments it, so every replay of a captured
graph draws fresh masks and a capture draws none.  :func:`ops.oracle.drop_path_scales` reproduces every
bit on the CPU, and is what a CPU forward uses.
"""

from __future__ import annotations

import torch

from . import native, oracle

MAX_BLOCKS = 256            # DP_MAX_BLOCKS of csrc/drop_path_kernels.cu


def block_rates(num_blocks: int, drop_path_rate: float):
    """timm's linear rule: ``p_l = p * l / (L - 1)`` for ``l = 0 .. L-1`` (``[0.0]`` for one block)"""
    if num_blocks == 1:
        return [0.0]
    return [drop_path_rate * l / (num_blocks - 1) for l in range(num_blocks)]


def keep_threshold(rate: float) -> int:
    """the kernel keeps a sample iff its 24-bit uniform is below ``round((1 - rate) 2^24)``"""
    return min(1 << 24, int((1.0 - rate) * (1 << 24) + 0.5))


class StochasticDepth(object):
    """The per-block drop rates, the ``(seed, rank)`` of the draws and the draw counter of one model.

    Not a module: it has no parameters or buffers, so ``state_dict`` keys, the parameter arena and the
    buffer broadcasts of the model are those of the model without it.  The counter lives in device memory,
    one per device the model runs on; a deep copy of the model (the bf16 compute twin, an EMA copy) shares
    this object and so the same draw sequence.  :attr:`draws` / :meth:`state_dict` read it back (a host
    synchronisation), for checkpoints."""

    def __init__(self, num_blocks: int, drop_path_rate: float, seed: int = 0, rank: int = 0):
        p = float(drop_path_rate)
        if not 0.0 <= p < 1.0:
            raise ValueError('drop_path_rate must be in [0, 1), got %r' % (drop_path_rate,))
        if not 1 <= num_blocks <= MAX_BLOCKS:
            raise ValueError('stochastic depth covers 1 to %d residual blocks, got %d' % (MAX_BLOCKS, num_blocks))
        self.drop_path_rate = p
        self.rates = block_rates(num_blocks, p)
        self.thresholds = [keep_threshold(r) for r in self.rates]
        # fp32(1 / (1 - p_l)), as the kernel stores it
        self.keep_scales = [float(torch.tensor(1.0 / (1.0 - r), dtype=torch.float32)) for r in self.rates]
        self.seed, self.rank = int(seed), int(rank)
        self._counters = {}           # device -> int64 [1] draw counter

    @property
    def num_blocks(self) -> int:
        return len(self.rates)

    def reseed(self, seed: int, rank: int):
        """draw from ``(seed, rank)`` from now on (the counter is kept)"""
        self.seed, self.rank = int(seed), int(rank)

    def __deepcopy__(self, memo):
        return self

    def _counter(self, device: torch.device) -> torch.Tensor:
        c = self._counters.get(device)
        if c is None:
            c = self._counters[device] = torch.full((1,), self.draws, dtype=torch.int64, device=device)
        return c

    @property
    def draws(self) -> int:
        """the number of draws so far (the largest counter over the devices)"""
        return max([int(c.item()) for c in self._counters.values()] or [0])

    def set_draws(self, n: int):
        n = int(n)
        if n < 0:
            raise ValueError('the draw counter must be >= 0, got %r' % (n,))
        if not self._counters:
            self._counters[torch.device('cpu')] = torch.zeros(1, dtype=torch.int64)
        for c in self._counters.values():
            c.fill_(n)

    def state_dict(self) -> dict:
        return {'draws': self.draws}

    def load_state_dict(self, state: dict):
        self.set_draws(state['draws'])

    def draw(self, n: int, device) -> torch.Tensor:
        """the ``[L, n]`` fp32 branch scales of one training forward of ``n`` samples, and advance the counter:
        one ``drop_path_draw`` launch on CUDA, :func:`ops.oracle.drop_path_scales` on the CPU"""
        device = torch.device(device)
        if device.type == 'cuda' and device.index is None:
            device = torch.device('cuda', torch.cuda.current_device())
        counter = self._counter(device)
        if device.type == 'cuda':
            return native.load().drop_path_draw(counter, self.seed, self.rank, self.thresholds, self.keep_scales,
                                                int(n))
        s = oracle.drop_path_scales(self.seed, self.rank, int(counter.item()), self.thresholds, self.keep_scales,
                                    int(n))
        counter.add_(1)
        return s.to(device)
