"""
ModelEma: an exponential moving average of a model's weights and BatchNorm statistics.

    e <- fmaf(w_t, s - e, e),   w_t = 1 - d_t

with d_t = ``decay`` or, with ``warmup=True``, d_t = min(decay, (1 + t) / (10 + t)) where t is the
number of updates already applied (TensorFlow's ``ExponentialMovingAverage(num_updates)`` rule).
The EMA is initialised with a copy of the model (as timm's ``ModelEmaV2``), and evaluated with
:meth:`ModelEma.applied`.

On CUDA one :meth:`update` is ONE launch of ``ema_update_kernel`` (``csrc/ema_kernels.cu``) over
every tracked tensor, stream-ordered and graph-capturable: ``GossipTrainer(..., ema=ema)`` runs it
as the last launch of the captured step.  The tracked tensors are described by a segment table built
at construction (source address, numel, offset in the flat fp32 EMA buffer, source dtype):

* the floating-point parameters of a ``GossipDataParallel`` / ``AllReduceDataParallel`` live in a
  :class:`~..utils.arena.FlatArena`: each arena is ONE segment;
* every floating-point buffer (BatchNorm ``running_mean`` / ``running_var``) is a small segment of
  its own; integer buffers (``num_batches_tracked``) are not tracked;
* a plain ``nn.Module``'s parameters are one segment each.

Sources are fp32 or bf16; the EMA is fp32, every segment 64-element (256-byte) aligned.  The decay
row ``[decay, warmup, count]`` lives on the device: :meth:`set_decay` is a host-to-device write, so
a captured graph never needs re-capturing, and the kernel advances the counter once per launch.

The segment table holds addresses.  If a parameter or buffer tensor is *replaced* after the
``ModelEma`` was built (rather than updated in place, e.g. ``module.bn.running_mean = t``), build a
new ``ModelEma``.  On CPU tensors :meth:`update` is a plain-torch computation of the same formula.
"""

from __future__ import annotations

import contextlib
from collections import OrderedDict
from typing import List, Optional

import numpy as np
import torch

from ..utils.arena import ALIGN_ELEMS

EMA_CHUNK = 8192          # elements per work item of ema_update_kernel (csrc/ema_kernels.cu)
_SRC_DTYPES = {torch.float32: 0, torch.bfloat16: 1}


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def check_decay(decay) -> float:
    d = float(decay)
    if not 0.0 <= d < 1.0:
        raise ValueError('ModelEma decay must be in [0, 1), got %r' % (decay,))
    return d


def decay_at(decay: float, warmup: bool, t: int) -> np.float32:
    """d_t as the kernel computes it, in fp32: ``decay`` or min(decay, (1 + t) / (10 + t))"""
    d = np.float32(decay)
    if not warmup:
        return d
    r = np.float32(np.float32(1.0) + np.float32(t)) / np.float32(np.float32(10.0) + np.float32(t))
    return np.float32(min(d, r))


def reference_update(e: torch.Tensor, s: torch.Tensor, d_t) -> torch.Tensor:
    """fmaf(1 - d_t, s - e, e) with fp32 e and s - e, the product and sum in fp64 (exact product,
    so at most one fp32 ulp from a true fused multiply-add).  Returns a new fp32 tensor."""
    w = float(np.float32(1.0) - np.float32(d_t))
    diff = s.float() - e                                    # fp32, as the kernel
    return (diff.double() * w + e.double()).float()


def _dense_flat(t: torch.Tensor) -> torch.Tensor:
    """The 1-D memory-order view of a dense tensor (contiguous or channels-last)."""
    if not (t.is_contiguous() or (t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last))):
        raise ValueError('ModelEma tracks dense tensors (contiguous or channels-last), got strides %s'
                         % (tuple(t.stride()),))
    return t.detach().as_strided((t.numel(),), (1,))


class ModelEma(object):

    def __init__(self, module, decay: float = 0.9999, warmup: bool = False):
        """``module``: a plain ``nn.Module``, a ``GossipDataParallel`` or an ``AllReduceDataParallel``
        (the EMA tracks the wrapped module; with a bf16 compute twin its buffers are the wrapped
        module's buffers, and :meth:`applied` also refreshes the bf16 shadow weights)."""
        from ..parallel.distributed import GossipDataParallel
        self.decay = check_decay(decay)
        self.warmup = bool(warmup)
        self._gdp = module if isinstance(module, GossipDataParallel) else None
        self.module = getattr(module, 'module', module)       # the wrapped network
        arenas = []
        if self._gdp is not None:
            arenas = list(self._gdp._arenas.values())
        elif hasattr(module, 'arena') and hasattr(module, 'module'):   # AllReduceDataParallel
            arenas = [module.arena]
        self._shadow = self._gdp.compute_shadow if self._gdp is not None else None

        # -- segments: arenas whole, then every other floating tensor on its own ---------------- #
        segs = []                 # (flat source view, offset in the EMA buffer)
        where = {}                # data_ptr of an arena -> (arena flat, EMA offset)
        off = 0
        for a in arenas:
            src = a.flat[:a.used]
            segs.append((src, off))
            where[id(a)] = (a, off)
            off = _round_up(off + a.used, ALIGN_ELEMS)
        self._entries = OrderedDict()        # state_dict name -> (source tensor, EMA storage offset)
        seen = {}
        for name, t in self.module.state_dict(keep_vars=True).items():
            if not t.is_floating_point():
                continue
            if t.dtype not in _SRC_DTYPES:
                raise ValueError('ModelEma tracks fp32 and bf16 tensors; %s is %s' % (name, t.dtype))
            ptr = t.data_ptr()
            if ptr in seen:                          # tied tensors share one EMA slot
                self._entries[name] = (t, seen[ptr])
                continue
            base = None
            for a, a_off in where.values():
                lo = a.flat.data_ptr()
                if a.flat.dtype == t.dtype and lo <= ptr < lo + a.used * a.flat.element_size():
                    base = a_off + (ptr - lo) // a.flat.element_size()
                    break
            if base is None:
                segs.append((_dense_flat(t), off))
                base = off
                off = _round_up(off + t.numel(), ALIGN_ELEMS)
            seen[ptr] = base
            self._entries[name] = (t, base)
        if not segs:
            raise ValueError('ModelEma: the module has no floating-point parameters or buffers')
        devices = set(s.device for s, _ in segs)
        if len(devices) != 1:
            raise ValueError('ModelEma needs every tracked tensor on one device, got %s' % sorted(map(str, devices)))
        self.device = devices.pop()
        self._segs = segs
        self.numel = sum(s.numel() for s, _ in segs)     # tracked elements per update
        self.ema = torch.zeros(max(off, 1), dtype=torch.float32, device=self.device)
        # device row [decay, warmup, count (uint32 bits), done_ctas (uint32 bits)]
        self._state = torch.zeros(4, dtype=torch.float32, device=self.device)
        self._stream = None          # GossipTrainer: decay writes go on the trainer's stream
        self._C = None
        if self.device.type == 'cuda':
            from . import native
            self._C = native.load()
            assert self._C.EMA_CHUNK == EMA_CHUNK
            table, items = [], []
            for i, (src, o) in enumerate(segs):
                table.append([src.data_ptr(), src.numel(), o, _SRC_DTYPES[src.dtype]])
                items.extend([i, c] for c in range((src.numel() + EMA_CHUNK - 1) // EMA_CHUNK))
            self._table = torch.tensor(table, dtype=torch.int64).to(self.device)
            self._items = torch.tensor(items, dtype=torch.int32).reshape(-1, 2).to(self.device)
        self.reset()

    # ------------------------------------------------------------------ #
    def _ema_views(self):
        for src, o in self._segs:
            yield src, self.ema.narrow(0, o, src.numel())

    def _row_stream(self):
        if self._stream is not None and self.device.type == 'cuda':
            return torch.cuda.stream(self._stream)
        return contextlib.nullcontext()

    def _write_row(self, count: int):
        row = torch.tensor([self.decay, 1.0 if self.warmup else 0.0, 0.0, 0.0], dtype=torch.float32)
        row.view(torch.int32)[2] = int(count)
        with self._row_stream():
            self._state.copy_(row)

    def _check_debiased(self):
        if self._gdp is not None and self._gdp.is_ps_numerator:
            raise RuntimeError('ModelEma: the GossipDataParallel holds push-sum numerators; the EMA averages '
                               'de-biased parameters (update after the gossip step has de-biased them)')

    @torch.no_grad()
    def reset(self):
        """Copy the module's current parameters and buffers into the EMA and zero the counter."""
        for src, e in self._ema_views():
            e.copy_(src)
        self._write_row(0)

    # ------------------------------------------------------------------ #
    def update(self):
        """One EMA step over every tracked tensor: one kernel launch on the current stream (no host
        synchronisation, graph-capturable); the device counter advances by one."""
        self._check_debiased()
        if self._C is not None:
            self._C.ema_update(self.ema, self._table, self._items, self._state)
            return
        if self.device.type != 'cpu':
            raise RuntimeError('ModelEma: no EMA kernel for device %s' % self.device)
        t = self.num_updates
        d = decay_at(self.decay, self.warmup, t)
        with torch.no_grad():
            for src, e in self._ema_views():
                e.copy_(reference_update(e, src, d))
        self._state.view(torch.int32)[2] = t + 1

    def set_decay(self, decay: float):
        """Stage a new decay on the device (a host-to-device write of the decay row; a captured graph
        needs no re-capture).  Ordered on the current stream, or on the trainer's stream once a
        ``GossipTrainer`` drives this EMA."""
        self.decay = check_decay(decay)
        with self._row_stream():
            self._state[0:1].copy_(torch.tensor([self.decay], dtype=torch.float32))

    @property
    def num_updates(self) -> int:
        """Updates applied so far (reads the device counter: synchronises)."""
        if self._stream is not None and self.device.type == 'cuda':
            self._stream.synchronize()
        return int(self._state.view(torch.int32)[2].item())

    # ------------------------------------------------------------------ #
    @contextlib.contextmanager
    def applied(self):
        """Context manager: inside the block the module's parameters, its floating-point buffers
        (BatchNorm running statistics) and, where the wrapper has one, the bf16 compute shadow hold
        the EMA; on exit they are restored bit for bit.  Runs on the current stream."""
        self._check_debiased()
        with torch.no_grad():
            saved = [src.clone() for src, _ in self._segs]
            saved_shadow = self._shadow.clone() if self._shadow is not None else None
            for src, e in self._ema_views():
                src.copy_(e)
            if self._shadow is not None:
                self._shadow.copy_(self._gdp.arena.flat)
        try:
            yield self
        finally:
            with torch.no_grad():
                for (src, _), s in zip(self._segs, saved):
                    src.copy_(s)
                if self._shadow is not None:
                    self._shadow.copy_(saved_shadow)

    def _entry_view(self, t: torch.Tensor, base: int) -> torch.Tensor:
        return self.ema.as_strided(t.shape, t.stride(), base)

    def state_dict(self) -> dict:
        """``{'state_dict': {name: fp32 EMA tensor}, 'decay', 'warmup', 'num_updates'}``; the names
        are those of the wrapped module's ``state_dict`` (floating-point entries only), so
        ``net.load_state_dict(sd['state_dict'], strict=False)`` loads the EMA weights into a model."""
        entries = OrderedDict((name, self._entry_view(t, base).detach().cpu().clone())
                              for name, (t, base) in self._entries.items())
        return {'state_dict': entries, 'decay': self.decay, 'warmup': self.warmup,
                'num_updates': self.num_updates}

    @torch.no_grad()
    def load_state_dict(self, sd: dict):
        missing = [n for n in self._entries if n not in sd['state_dict']]
        if missing:
            raise KeyError('ModelEma.load_state_dict: missing entries %s' % missing[:8])
        for name, (t, base) in self._entries.items():
            self._entry_view(t, base).copy_(sd['state_dict'][name])
        self.decay = check_decay(sd['decay'])
        self.warmup = bool(sd['warmup'])
        self._write_row(int(sd['num_updates']))
