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

Knowledge distillation (``teacher_logits=u``, ``distill_alpha`` = alpha in (0, 1], ``distill_temperature`` =
T > 0; Hinton et al. 2015): ``loss_i = (1 - alpha) CE_eps(z_i, .) + alpha T^2 KL(softmax(u_i / T) ||
softmax(z_i / T))`` with ``CE_eps`` the (smoothed, mixed) cross-entropy above, averaged over the batch:
``(1 - alpha) F.cross_entropy(z, y, label_smoothing=eps) + alpha T^2 F.kl_div(F.log_softmax(z / T),
F.log_softmax(u / T), reduction='batchmean', log_target=True)`` when every target is valid.  The same two
launches compute it, reading ``u`` once in each; ``metrics[0]`` is that combined objective and prec@1 /
prec@5 are the student's.  The teacher logits get no gradient.  A row whose target (or partner target) is
out of range adds neither term.  ``distill_alpha = 0`` without teacher logits runs exactly the kernels above.
"""

from __future__ import annotations

import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import native


def check_label_smoothing(label_smoothing) -> float:
    eps = float(label_smoothing)
    if not 0.0 <= eps <= 1.0:
        raise ValueError('label_smoothing must be in [0, 1], got %r' % (label_smoothing,))
    return eps


def check_distill_args(distill_alpha, distill_temperature) -> tuple:
    """``(alpha, T)`` as floats; ValueError unless alpha is in [0, 1] and T is finite and > 0."""
    alpha, temp = float(distill_alpha), float(distill_temperature)
    if not 0.0 <= alpha <= 1.0:
        raise ValueError('distill_alpha must be in [0, 1], got %r' % (distill_alpha,))
    if not (math.isfinite(temp) and temp > 0.0):
        raise ValueError('distill_temperature must be finite and > 0, got %r' % (distill_temperature,))
    return alpha, temp


def _check_teacher_logits(logits, teacher_logits, alpha):
    if alpha > 0.0 and teacher_logits is None:
        raise ValueError('distill_alpha > 0 needs teacher_logits')
    if teacher_logits is None:
        return
    if alpha == 0.0:
        raise ValueError('teacher_logits were given with distill_alpha = 0')
    if teacher_logits.shape != logits.shape or teacher_logits.dtype != logits.dtype:
        raise ValueError('teacher_logits must have the logits\' shape and dtype: got %s %s for logits %s %s'
                         % (tuple(teacher_logits.shape), teacher_logits.dtype, tuple(logits.shape), logits.dtype))
    if teacher_logits.device != logits.device:
        raise ValueError('teacher_logits must be on the logits\' device: got %s for %s'
                         % (teacher_logits.device, logits.device))


def reference_distillation_loss(logits: torch.Tensor, target: torch.Tensor, teacher_logits: torch.Tensor,
                                distill_alpha: float, distill_temperature: float = 1.0,
                                label_smoothing: float = 0.0, lam=None):
    """(loss, prec@1 %, prec@5 %) of the distillation objective in plain PyTorch (fp32, fp64 for fp64
    logits): ``mean_i [(1 - alpha) CE_eps(z_i, .) + alpha T^2 KL(softmax(u_i / T) || softmax(z_i / T))]``
    with ``CE_eps`` the label-smoothed cross-entropy, or with ``lam`` (a float or 0-d tensor) the two-target
    ``lam CE_eps(z_i, t_i) + (1 - lam) CE_eps(z_i, t_{B-1-i})``.  A row whose target (or partner target) is
    out of range adds no loss (the mean still divides by B).  The teacher logits are detached; the
    accuracies are the student's against each row's own target."""
    eps = check_label_smoothing(label_smoothing)
    alpha, temp = check_distill_args(distill_alpha, distill_temperature)
    _check_teacher_logits(logits, teacher_logits, alpha)
    ct = torch.float64 if logits.dtype == torch.float64 else torch.float32
    lf = logits.to(ct)
    B, C = lf.shape
    valid = (target >= 0) & (target < C)
    za = lf.gather(1, torch.where(valid, target, 0).view(-1, 1)).view(-1)
    if lam is None:
        zy = za
    else:
        lam = torch.as_tensor(lam, dtype=ct, device=lf.device)
        tb = target.flip(0)
        vb = (tb >= 0) & (tb < C)
        valid = valid & vb
        zb = lf.gather(1, torch.where(vb, tb, 0).view(-1, 1)).view(-1)
        zy = lam * za + (1.0 - lam) * zb
    ce = torch.logsumexp(lf, 1) - (1.0 - eps) * zy
    if eps:
        ce = ce - eps * lf.mean(1)
    loss_i = (1.0 - alpha) * ce
    if alpha > 0.0:
        uf = teacher_logits.detach().to(ct)
        kl = F.kl_div(F.log_softmax(lf / temp, 1), F.log_softmax(uf / temp, 1), reduction='none',
                      log_target=True).sum(1)
        loss_i = loss_i + (alpha * temp * temp) * kl
    loss = torch.where(valid, loss_i, torch.zeros_like(loss_i)).sum() / B
    with torch.no_grad():
        k = min(5, C)
        _, pred = lf.topk(k, 1, True, True)
        hit = pred.eq(target.view(-1, 1))
        scale = 100.0 / B
        p1 = hit[:, :1].reshape(-1).float().sum() * scale
        p5 = hit.reshape(-1).float().sum() * scale
    return loss, p1, p5


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
    def forward(ctx, logits, target, label_smoothing, mix, teacher, alpha, temperature):
        C = native.load()
        metrics, lse = C.xent_forward(logits, target, label_smoothing, mix, teacher, alpha, temperature)
        ctx.save_for_backward(logits, target, lse)
        ctx.label_smoothing = label_smoothing
        ctx.mix = mix
        ctx.distill = (teacher, alpha, temperature)
        ctx.mark_non_differentiable(metrics)
        return metrics[0], metrics

    @staticmethod
    def backward(ctx, g_loss, _g_metrics):
        C = native.load()
        logits, target, lse = ctx.saved_tensors
        g = g_loss.reshape(1).to(torch.float32)
        dz = C.xent_backward(logits, target, lse, g, ctx.label_smoothing, ctx.mix, *ctx.distill)
        return dz, None, None, None, None, None, None


def fused_cross_entropy(logits: torch.Tensor, target: torch.Tensor, label_smoothing: float = 0.0,
                        mix: torch.Tensor = None, teacher_logits: torch.Tensor = None,
                        distill_alpha: float = 0.0, distill_temperature: float = 1.0):
    """Returns ``(loss, metrics)``; ``metrics = [loss, prec@1 %, prec@5 %]`` (fp32, detached).
    ``label_smoothing`` in [0, 1], as in ``F.cross_entropy``.  ``mix``: the mix state of
    ``batch_mix.BatchMix`` (two targets per row, see the module docstring), or None.
    ``teacher_logits``: the teacher's logits (the logits' shape and dtype; no gradient), given exactly when
    ``distill_alpha`` in [0, 1] is > 0; ``distill_temperature`` > 0 (see the module docstring)."""
    eps = check_label_smoothing(label_smoothing)
    alpha, temp = check_distill_args(distill_alpha, distill_temperature)
    _check_teacher_logits(logits, teacher_logits, alpha)
    if logits.is_cuda and native.available():
        lg = logits if logits.is_contiguous() else logits.contiguous()
        if native.load().xent_can_fuse(lg, target):
            u = None
            if teacher_logits is not None:
                u = teacher_logits.detach()
                u = u if u.is_contiguous() else u.contiguous()
            loss, metrics = _FusedXent.apply(lg, target, eps, mix, u, alpha, temp)
            return loss, metrics
    if teacher_logits is not None:
        loss, p1, p5 = reference_distillation_loss(logits, target, teacher_logits, alpha, temp, eps,
                                                   lam=None if mix is None else mix[0])
    elif mix is None:
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
    also measures accuracy.  With ``distill_alpha`` > 0 it is the distillation objective (module
    docstring) and every call takes the teacher's logits."""

    def __init__(self, label_smoothing: float = 0.0, distill_alpha: float = 0.0, distill_temperature: float = 1.0):
        super().__init__()
        self.label_smoothing = check_label_smoothing(label_smoothing)
        self.distill_alpha, self.distill_temperature = check_distill_args(distill_alpha, distill_temperature)
        self.metrics = None

    def forward(self, logits, target, mix=None, teacher_logits=None):
        """``mix``: the device mix state of ``batch_mix.BatchMix`` for mixup / CutMix targets
        (prec@1 / prec@5 then count against each row's own target), or None.  ``teacher_logits``:
        the teacher's logits, given exactly when ``distill_alpha`` > 0."""
        loss, self.metrics = fused_cross_entropy(logits, target, self.label_smoothing, mix=mix,
                                                 teacher_logits=teacher_logits, distill_alpha=self.distill_alpha,
                                                 distill_temperature=self.distill_temperature)
        return loss

    def extra_repr(self):
        parts = ['label_smoothing=%g' % self.label_smoothing] if self.label_smoothing else []
        if self.distill_alpha:
            parts.append('distill_alpha=%g, distill_temperature=%g' % (self.distill_alpha, self.distill_temperature))
        return ', '.join(parts)
