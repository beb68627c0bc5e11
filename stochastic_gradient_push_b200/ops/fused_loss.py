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
"""

from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import native


def reference_loss_and_accuracy(logits: torch.Tensor, target: torch.Tensor):
    """(loss, prec@1 %, prec@5 %) the way the reference's loop computes them."""
    loss = F.cross_entropy(logits.float(), target)
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
    def forward(ctx, logits, target):
        C = native.load()
        metrics, lse = C.xent_forward(logits, target)
        ctx.save_for_backward(logits, target, lse)
        ctx.mark_non_differentiable(metrics)
        return metrics[0], metrics

    @staticmethod
    def backward(ctx, g_loss, _g_metrics):
        C = native.load()
        logits, target, lse = ctx.saved_tensors
        g = g_loss.reshape(1).to(torch.float32)
        return C.xent_backward(logits, target, lse, g), None


def fused_cross_entropy(logits: torch.Tensor, target: torch.Tensor):
    """Returns ``(loss, metrics)``; ``metrics = [loss, prec@1 %, prec@5 %]`` (fp32, detached)."""
    if logits.is_cuda and native.available():
        lg = logits if logits.is_contiguous() else logits.contiguous()
        if native.load().xent_can_fuse(lg, target):
            loss, metrics = _FusedXent.apply(lg, target)
            return loss, metrics
    loss, p1, p5 = reference_loss_and_accuracy(logits, target)
    return loss, torch.stack([loss.detach().float(), p1, p5])


class FusedCrossEntropyWithAccuracy(nn.Module):
    """Drop-in for ``nn.CrossEntropyLoss()`` (mean reduction) that also measures accuracy."""

    def __init__(self):
        super().__init__()
        self.metrics = None

    def forward(self, logits, target):
        loss, self.metrics = fused_cross_entropy(logits, target)
        return loss
