"""
FusedCrossEntropyWithAccuracy: softmax cross-entropy + prec@1 / prec@5 in ONE launch.

The reference computes ``nn.CrossEntropyLoss`` and then, every iteration,
``accuracy(output, target, topk=(1, 5))`` followed by three ``.item()`` host
synchronisations (``/root/reference/gossip_sgd.py:372-373, 394-399, 192-198``).
Here one sm_90a kernel (``csrc/loss_kernels.cu``) emits the mean loss and both
accuracies into a 3-float device tensor and keeps the per-row log-sum-exp for
the backward kernel; the training step copies those 12 bytes into a pinned ring
without ever blocking the host (``parallel/trainer.py``).

``criterion(logits, target)`` returns the scalar loss (autograd-connected) and
leaves ``criterion.metrics`` = device tensor ``[loss, prec@1 %, prec@5 %]``.
CPU tensors / unsupported dtypes run the plain PyTorch composition, which is
also the oracle in ``tests/test_fused_loss_gpu.py``.

Label smoothing (``label_smoothing=eps``, in [0, 1]) follows
``torch.nn.functional.cross_entropy(label_smoothing=eps)``:
``loss_i = lse_i - (1 - eps) z_{i,t} - (eps / C) sum_j z_{i,j}``, averaged over the batch, and
``metrics[0]`` is that smoothed loss (the one training minimises); prec@1 / prec@5 do not depend
on eps.  The reference's KL divergence against the smoothed one-hot target would be lower by the
constant entropy of that target, with the same gradient.  ``eps = 0`` runs exactly the
unsmoothed kernels.

Mixup / CutMix (``mix=state``, the device mix state of ``batch_mix.BatchMix``): row ``i`` has two
targets, its own ``t_i`` and its partner's ``t_{B-1-i}``, weighted ``lam`` and ``1 - lam`` (``lam``
read by the kernels from ``state[0]``, so a captured graph follows each step's draw):
``loss_i = lam CE_eps(z_i, t_i) + (1 - lam) CE_eps(z_i, t_{B-1-i})``.  prec@1 / prec@5 still count
against each row's own target.  ``mix=None`` runs exactly the one-target kernels.
"""

from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import native


def check_label_smoothing(label_smoothing) -> float:
    eps = float(label_smoothing)
    if not 0.0 <= eps <= 1.0:
        raise ValueError('label_smoothing must be in [0, 1], got %r' % (label_smoothing,))
    return eps


def reference_loss_and_accuracy(logits: torch.Tensor, target: torch.Tensor, label_smoothing: float = 0.0):
    """(loss, prec@1 %, prec@5 %) the way the reference's loop computes them (loss with
    ``F.cross_entropy(label_smoothing=...)``)."""
    eps = check_label_smoothing(label_smoothing)
    loss = F.cross_entropy(logits.float(), target, label_smoothing=eps)
    with torch.no_grad():
        k = min(5, logits.shape[1])
        _, pred = logits.float().topk(k, 1, True, True)
        hit = pred.eq(target.view(-1, 1))
        scale = 100.0 / logits.shape[0]
        p1 = hit[:, :1].reshape(-1).float().sum() * scale
        p5 = hit.reshape(-1).float().sum() * scale
    return loss, p1, p5


class _FusedXent(torch.autograd.Function):

    @staticmethod
    def forward(ctx, logits, target, label_smoothing, mix):
        C = native.load()
        metrics, lse = C.xent_forward(logits, target, label_smoothing, mix)
        ctx.save_for_backward(logits, target, lse)
        ctx.label_smoothing = label_smoothing
        ctx.mix = mix
        ctx.mark_non_differentiable(metrics)
        return metrics[0], metrics

    @staticmethod
    def backward(ctx, g_loss, _g_metrics):
        C = native.load()
        logits, target, lse = ctx.saved_tensors
        g = g_loss.reshape(1).to(torch.float32)
        return C.xent_backward(logits, target, lse, g, ctx.label_smoothing, ctx.mix), None, None, None


def fused_cross_entropy(logits: torch.Tensor, target: torch.Tensor, label_smoothing: float = 0.0,
                        mix: torch.Tensor = None):
    """Returns ``(loss, metrics)``; ``metrics = [loss, prec@1 %, prec@5 %]`` (fp32, detached).
    ``label_smoothing`` in [0, 1], as in ``F.cross_entropy``.  ``mix``: the mix state of
    ``batch_mix.BatchMix`` (two targets per row, see the module docstring), or None."""
    eps = check_label_smoothing(label_smoothing)
    if logits.is_cuda and native.available():
        lg = logits if logits.is_contiguous() else logits.contiguous()
        if native.load().xent_can_fuse(lg, target):
            loss, metrics = _FusedXent.apply(lg, target, eps, mix)
            return loss, metrics
    if mix is None:
        loss, p1, p5 = reference_loss_and_accuracy(logits, target, eps)
    else:
        from .batch_mix import reference_mixed_loss_and_accuracy
        loss, p1, p5 = reference_mixed_loss_and_accuracy(logits, target, mix[0], eps)
    return loss, torch.stack([loss.detach().float(), p1, p5])


def eval_accumulator(device) -> torch.Tensor:
    """a zeroed evaluation accumulator for :func:`eval_accumulate`: int64 ``[4]`` on ``device`` =
    ``[loss sum (fp64 bits: acc[:1].view(torch.float64)), top-1 hits, top-5 hits, counted rows]``"""
    return torch.zeros(4, dtype=torch.int64, device=device)


def eval_accumulate(logits: torch.Tensor, target: torch.Tensor, acc: torch.Tensor) -> None:
    """Adds this batch's plain cross-entropy sum (fp64) and top-1 / top-5 / row counts to ``acc``
    (:func:`eval_accumulator`) in one launch of the forward kernel's row scan: no per-row loss is
    stored and nothing is read back.  Rows whose target is outside ``[0, C)`` are not counted.  A logit
    tied with the target's counts as ranked below it.  CUDA fp32 / bf16 logits only."""
    lg = logits if logits.is_contiguous() else logits.contiguous()
    C = native.load()
    if not C.xent_can_fuse(lg, target):
        raise ValueError('eval_accumulate needs 2-d fp32 / bf16 CUDA logits and int64 CUDA targets, got %s %s '
                         'and %s %s' % (tuple(logits.shape), logits.dtype, tuple(target.shape), target.dtype))
    C.xent_eval_accumulate(lg, target, acc)


class FusedCrossEntropyWithAccuracy(nn.Module):
    """Drop-in for ``nn.CrossEntropyLoss(label_smoothing=label_smoothing)`` (mean reduction) that
    also measures accuracy."""

    def __init__(self, label_smoothing: float = 0.0):
        super().__init__()
        self.label_smoothing = check_label_smoothing(label_smoothing)
        self.metrics = None

    def forward(self, logits, target, mix=None):
        """``mix``: the device mix state of ``batch_mix.BatchMix`` for mixup / CutMix targets
        (prec@1 / prec@5 then count against each row's own target), or None."""
        loss, self.metrics = fused_cross_entropy(logits, target, self.label_smoothing, mix=mix)
        return loss

    def extra_repr(self):
        return 'label_smoothing=%g' % self.label_smoothing if self.label_smoothing else ''
