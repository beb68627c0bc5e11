"""
BatchMix: mixup (Zhang et al., ICLR 2018) and CutMix (Yun et al., ICCV 2019) in batch mode, fused
into the training step's input staging copy and its fused cross-entropy.

Every step draws, on the host, one set of parameters for the whole batch:

* with probability ``mix_prob`` the step is mixed; if both alphas are > 0, CutMix is chosen with
  probability ``switch_prob``, otherwise mixup;
* row ``i`` is mixed with row ``B-1-i`` (the flipped batch: no permutation tensor);
* mixup: ``lam ~ Beta(a, a)`` and ``x_i <- fmaf(lam, x_i, (1 - lam) * x_j)`` in fp32 ((1 - lam)
  and the product rounded to fp32, then one fused multiply-add);
* CutMix: ``lam ~ Beta(a, a)``; a box of area fraction ``1 - lam`` at a uniform centre, clipped
  to the image, takes the partner's pixels (a bit-exact copy); ``lam`` is then recomputed from the
  clipped box: ``lam = 1 - box_area / (H W)``;
* odd ``B``: the middle row is its own partner.

The draw is a pure function of ``(seed, rank, iteration)`` (a counter-based Philox stream keyed by
seed and rank, the iteration in the counter), so a resumed run draws the same values once
:attr:`BatchMix.iteration` is set to the global iteration; there is no state to checkpoint.

The parameters go to a small device-resident mix state ``[lam, mode, y0, y1, x0, x1]`` (mode 0 =
not mixed, 1 = mixup, 2 = CutMix) through an H2D copy from an 8-slot pinned ring, on the stream
that launches the mixing; a slot is reused only after its previous copy has executed.  Because the
kernels read ``lam`` and the box from that state, a captured training graph stays valid:

* ``csrc/mix_kernels.cu`` replaces the trainer's stage -> static input copy (NCHW or NHWC fp32
  source, NCHW or NHWC fp32 / bf16 destination; one CTA column per row pair, so every source
  element is read once and every destination element written once);
* the fused cross-entropy (``fused_loss.fused_cross_entropy(..., mix=state)``) computes
  ``lam CE_eps(z_i, t_i) + (1 - lam) CE_eps(z_i, t_{B-1-i})`` and its gradient in the same single
  launches.  prec@1 / prec@5 count against each row's own (un-flipped) target.
"""

from __future__ import annotations

import math
from collections import namedtuple

import numpy as np
import torch

from . import native
from .fused_loss import check_label_smoothing

MixParams = namedtuple('MixParams', 'lam mode y0 y1 x0 x1')
NO_MIX, MIXUP, CUTMIX = 0, 1, 2
RING_SLOTS = 8
STATE_LEN = 8                   # [lam, mode, y0, y1, x0, x1] + 2 floats of padding


def check_mix_args(mixup_alpha, cutmix_alpha, mix_prob, switch_prob):
    """ValueError unless both alphas are >= 0 and both probabilities lie in [0, 1]."""
    for name, v in (('mixup_alpha', mixup_alpha), ('cutmix_alpha', cutmix_alpha)):
        if not float(v) >= 0.0 or math.isinf(float(v)):
            raise ValueError('%s must be a finite value >= 0, got %r' % (name, v))
    for name, v in (('mix_prob', mix_prob), ('switch_prob', switch_prob)):
        if not 0.0 <= float(v) <= 1.0:
            raise ValueError('%s must be in [0, 1], got %r' % (name, v))


def cutmix_box(lam: float, H: int, W: int, cy: int, cx: int):
    """Box of area fraction ``1 - lam`` centred at ``(cy, cx)``, clipped to the ``H x W`` image:
    ``(y0, y1, x0, x1)``, half-open."""
    cut = math.sqrt(1.0 - lam)
    ch, cw = int(H * cut), int(W * cut)
    y0, y1 = min(max(cy - ch // 2, 0), H), min(max(cy + ch // 2, 0), H)
    x0, x1 = min(max(cx - cw // 2, 0), W), min(max(cx + cw // 2, 0), W)
    return y0, y1, x0, x1


def _unpack(params):
    if isinstance(params, torch.Tensor):
        params = params.detach().float().cpu().tolist()
    lam, mode, y0, y1, x0, x1 = (float(v) for v in list(params)[:6])
    return lam, int(mode), int(y0), int(y1), int(x0), int(x1)


def reference_batch_mix(x: torch.Tensor, params) -> torch.Tensor:
    """The mixed batch (fp32, ``x``'s shape) for ``params`` = :class:`MixParams` or a mix state:
    mixup as ``fmaf(lam, x_i, (1 - lam) * x_j)`` with every fp32 rounding the kernel makes, CutMix
    as a copy of the partner's box."""
    lam, mode, y0, y1, x0, x1 = _unpack(params)
    xf = x.float()
    xj = xf.flip(0)
    if mode == MIXUP:
        lam32 = torch.tensor(lam, dtype=torch.float32)
        om = (torch.tensor(1.0, dtype=torch.float32) - lam32).to(x.device)
        t = om * xj                                        # fp32 product, rounded
        # lam * x_i is exact in fp64 (24 + 24 bits); the sum is rounded once more to fp32
        return (lam32.double().to(x.device) * xf.double() + t.double()).float()
    out = xf.clone()
    if mode == CUTMIX:
        out[:, :, y0:y1, x0:x1] = xj[:, :, y0:y1, x0:x1]
    return out


def reference_mixed_loss_and_accuracy(logits: torch.Tensor, target: torch.Tensor, lam,
                                      label_smoothing: float = 0.0):
    """(loss, prec@1 %, prec@5 %) of the two-target loss
    ``mean_i [lam CE_eps(z_i, t_i) + (1 - lam) CE_eps(z_i, t_{B-1-i})]``, in plain PyTorch.  A row
    whose target or partner target is out of range adds no loss (the mean still divides by B);
    the accuracies count against each row's own target."""
    eps = check_label_smoothing(label_smoothing)
    lf = logits.float()
    B, C = lf.shape
    lam = torch.as_tensor(lam, dtype=torch.float32).to(lf.device)
    tb = target.flip(0)
    va = (target >= 0) & (target < C)
    vb = (tb >= 0) & (tb < C)
    za = lf.gather(1, torch.where(va, target, 0).view(-1, 1)).view(-1)
    zb = lf.gather(1, torch.where(vb, tb, 0).view(-1, 1)).view(-1)
    lse = torch.logsumexp(lf, 1)
    loss_i = lse - (1.0 - eps) * (lam * za + (1.0 - lam) * zb)
    if eps:
        loss_i = loss_i - eps * lf.mean(1)
    loss = torch.where(va & vb, loss_i, torch.zeros_like(loss_i)).sum() / B
    with torch.no_grad():
        k = min(5, C)
        _, pred = lf.topk(k, 1, True, True)
        hit = pred.eq(target.view(-1, 1))
        scale = 100.0 / B
        p1 = hit[:, :1].reshape(-1).float().sum() * scale
        p5 = hit.reshape(-1).float().sum() * scale
    return loss, p1, p5


class BatchMix(object):
    """Batch-mode mixup / CutMix for the training step (see the module docstring).

    ``apply(src, out)`` draws the next step's parameters, stages them in :attr:`state` and writes
    the mixed batch to ``out``; pass ``mix=batch_mix.state`` to the fused cross-entropy of that
    step.  ``GossipTrainer(..., batch_mix=...)`` does both inside its input staging."""

    def __init__(self, mixup_alpha: float = 0.0, cutmix_alpha: float = 0.0, mix_prob: float = 1.0,
                 switch_prob: float = 0.5, seed: int = 0, rank: int = 0):
        check_mix_args(mixup_alpha, cutmix_alpha, mix_prob, switch_prob)
        self.mixup_alpha = float(mixup_alpha)
        self.cutmix_alpha = float(cutmix_alpha)
        self.mix_prob = float(mix_prob)
        self.switch_prob = float(switch_prob)
        self.seed = int(seed)
        self.rank = int(rank)
        self.iteration = 0              # global iteration of the next draw
        self.last = None                # MixParams of the last apply()
        self.state = None               # device (or CPU) fp32 [lam, mode, y0, y1, x0, x1, 0, 0]
        self._host = None
        self._host_np = None
        self._events = [None] * RING_SLOTS
        self._slot = 0

    @property
    def enabled(self) -> bool:
        return self.mixup_alpha > 0 or self.cutmix_alpha > 0

    def __repr__(self):
        return ('BatchMix(mixup_alpha=%g, cutmix_alpha=%g, mix_prob=%g, switch_prob=%g, seed=%d, rank=%d)'
                % (self.mixup_alpha, self.cutmix_alpha, self.mix_prob, self.switch_prob, self.seed, self.rank))

    # -- host sampler ------------------------------------------------------------------------- #
    def sample(self, H: int, W: int, itr=None) -> MixParams:
        """Parameters of global iteration ``itr`` (default :attr:`iteration`, which then advances)
        for ``H x W`` images: a pure function of ``(seed, rank, itr)``."""
        if itr is None:
            itr = self.iteration
            self.iteration += 1
        itr = int(itr)
        if itr < 0:
            raise ValueError('iteration must be >= 0, got %d' % itr)
        key = np.array([self.seed % (1 << 64), self.rank % (1 << 64)], dtype=np.uint64)
        rng = np.random.Generator(np.random.Philox(key=key, counter=np.array([0, 0, itr, 0], dtype=np.uint64)))
        if not self.enabled or rng.random() >= self.mix_prob:
            return MixParams(1.0, NO_MIX, 0, 0, 0, 0)
        if self.mixup_alpha > 0 and self.cutmix_alpha > 0:
            cutmix = rng.random() < self.switch_prob
        else:
            cutmix = self.cutmix_alpha > 0
        a = self.cutmix_alpha if cutmix else self.mixup_alpha
        lam = float(rng.beta(a, a))
        if not cutmix:
            return MixParams(float(np.float32(lam)), MIXUP, 0, 0, 0, 0)
        cy, cx = int(rng.integers(H)), int(rng.integers(W))
        y0, y1, x0, x1 = cutmix_box(lam, H, W, cy, cx)
        lam = 1.0 - (y1 - y0) * (x1 - x0) / float(H * W)
        return MixParams(float(np.float32(lam)), CUTMIX, y0, y1, x0, x1)

    # -- device mix state --------------------------------------------------------------------- #
    def stage(self, params: MixParams, device) -> torch.Tensor:
        """Write ``params`` into :attr:`state` on ``device``: an H2D copy from the pinned ring on
        the current stream (CUDA), or a plain write (CPU).  Returns :attr:`state`, whose address
        never changes."""
        device = torch.device(device)
        if device.type == 'cuda' and device.index is None:
            device = torch.device('cuda', torch.cuda.current_device())
        if self.state is None:
            self.state = torch.zeros(STATE_LEN, dtype=torch.float32, device=device)
            self._host = torch.zeros(RING_SLOTS, STATE_LEN, dtype=torch.float32)
            if device.type == 'cuda':
                self._host = self._host.pin_memory()
            self._host_np = self._host.numpy()
        elif self.state.device != device:
            raise ValueError('BatchMix state lives on %s, got inputs on %s' % (self.state.device, device))
        slot = self._slot
        self._slot = (slot + 1) % RING_SLOTS
        ev = self._events[slot]
        if ev is not None:
            ev.synchronize()                 # the copy that last read this slot has executed
        self._host_np[slot, :6] = params
        if self.state.is_cuda:
            self.state.copy_(self._host[slot], non_blocking=True)
            ev = self._events[slot] = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self.state.device))
        else:
            self.state.copy_(self._host[slot])
        return self.state

    # -- mixing ------------------------------------------------------------------------------- #
    def apply(self, src: torch.Tensor, out: torch.Tensor = None, params: MixParams = None,
              micro_batches: int = 1) -> torch.Tensor:
        """``out`` <- ``src`` mixed with its flipped batch.  ``params`` default: the next draw
        (:meth:`sample`).  CUDA: one launch of the sm_90a kernel (``src`` fp32, NCHW or NHWC;
        ``out`` NCHW or NHWC, fp32 or bf16; a missing extension is an error).  CPU: the plain torch
        composition :func:`reference_batch_mix`.

        ``micro_batches = k > 1`` (gradient accumulation): the batch is k equal row slices, each mixed
        with its own flipped slice -- row i of slice j pairs with row m-1-i of that slice, as the fused
        two-target loss of that micro-batch pairs them --, under ONE draw staged once: k launches that
        move the same bytes as one."""
        if src.dim() != 4:
            raise ValueError('BatchMix.apply takes a 4-d image batch, got shape %s' % (tuple(src.shape),))
        k = int(micro_batches)
        if k < 1 or src.shape[0] % k:
            raise ValueError('micro_batches must be >= 1 and divide the batch of %d rows, got %r'
                             % (src.shape[0], micro_batches))
        if params is None:
            params = self.sample(src.shape[2], src.shape[3])
        if out is None:
            fmt = torch.channels_last if (src.is_contiguous(memory_format=torch.channels_last)
                                          and not src.is_contiguous()) else torch.contiguous_format
            out = torch.empty(src.shape, dtype=torch.float32, device=src.device).contiguous(memory_format=fmt)
        state = self.stage(params, src.device)
        m = src.shape[0] // k
        for j in range(k):
            s, o = (src, out) if k == 1 else (src[j * m:(j + 1) * m], out[j * m:(j + 1) * m])
            if src.is_cuda:
                native.load().batch_mix(s, o, state)
            else:
                o.copy_(reference_batch_mix(s, params))
        self.last = params
        return out
