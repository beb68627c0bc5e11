"""
FusedBatchNormAct2d: BatchNorm2d (+ residual add) (+ ReLU) as ONE op, backed by
the sm_90a NHWC kernels in ``csrc/bn_kernels.cu``.

Why it exists: in the ResNet-50 training step at batch 256 the launch list
attributes most of the
GPU time to the framework's channels-last BatchNorm kernels and ~13 % to
stand-alone ReLU / add / cast kernels, versus ~15 % for the tensor-core
convolutions.  All of that work is memory-bound, so it is rewritten as the
minimum number of 16-byte-vectorised passes over HBM (forward 2 reads + 1
write instead of 5 reads + 3 writes; backward recomputes the ReLU mask from the
saved input instead of reading a mask/output tensor).

The module is a drop-in ``nn.BatchNorm2d`` subclass (same parameters, buffers
and ``state_dict`` keys); ``forward(x, residual=None, relu=False)``.  Anything
the kernels do not cover (CPU tensors, NCHW layout, C % 8 != 0, fp16/fp64)
runs the reference composition ``relu(batch_norm(x) + residual)``, which is
also the oracle in the numerics tests.

``conv_bn_act`` / ``conv_bn_act_split`` go one step further for 1x1 / stride-1
convolutions: the convolution itself runs as the hand-written wgmma GEMM of
``csrc/conv1x1_kernels.cu`` (TMA operand ring, register accumulators), whose
epilogue produces the BatchNorm statistics (no separate statistics pass) and,
in backward, adds the skip-branch gradient of a residual block inside the
dgrad GEMM (no autograd accumulation pass).  Also here: the NHWC max-pool and
the tensor-core stem convolution wrappers.
"""

from __future__ import annotations

import contextlib
import os
import threading

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import native


FORCE_REFERENCE = False      # debugging / A-B switch: route everything to the PyTorch composition

# 1x1 convolutions feeding a training-mode BatchNorm run as the wgmma GEMM with the
# statistics fused into its epilogue (csrc/conv1x1_kernels.cu).  SGP_B200_CONV1X1=0 routes
# them back to the library convolution + stand-alone statistics pass.
USE_TCGEN05_CONV1X1 = os.environ.get('SGP_B200_CONV1X1', '1') != '0'


# the tensor-core stem kernels (csrc/stem_kernels.cu); SGP_B200_STEM=0 -> library convolution
USE_STEM_KERNELS = os.environ.get('SGP_B200_STEM', '1') != '0'

# A residual block's last BN backward reduction runs inside the next block's conv1 dgrad GEMM
# (MODE 3 of csrc/conv1x1_kernels.cu); SGP_B200_BN_BWD_FUSE=0 keeps the stand-alone reduce pass.
USE_BN_BWD_FUSE = os.environ.get('SGP_B200_BN_BWD_FUSE', '1') != '0'


@contextlib.contextmanager
def bn_f32_map(split: bool):
    """Run the fp32 BatchNorm kernels launched inside the block with the split channel map (the
    default; coalesced 16-byte accesses) or, ``split=False``, with 8 consecutive channels per thread
    (the bf16 map; ``SGP_B200_BN_F32_MAP=0`` selects it for the whole process).  Both give
    bit-identical results."""
    C = native.load()
    prev = C.bn_f32_map(1 if split else 0)
    try:
        yield
    finally:
        C.bn_f32_map(prev)


class _ThreadFlag(threading.local):
    on = False


# set by eval_bn_gemm(): eval-mode conv_bn_act calls the GEMM with BatchNorm in its epilogue.  Per thread: a
# distilling training step runs its teacher inside the block while ranks driven from other threads of the
# process may be in their train-mode forward
_EVAL_GEMM = _ThreadFlag()


@contextlib.contextmanager
def eval_bn_gemm():
    """Inside the block, ``conv_bn_act`` with an eval-mode BatchNorm and gradients disabled runs every
    1x1 / stride-1 convolution the GEMM covers as ONE launch: the GEMM with the BatchNorm affine map of
    the running statistics, the residual add and the ReLU in its epilogue (``C.conv1x1_bn_eval``)
    instead of the library convolution and a separate BatchNorm pass.  Outside it an eval forward runs
    as before, bit for bit.  ``GossipTrainer.evaluate`` uses it."""
    prev = _EVAL_GEMM.on
    _EVAL_GEMM.on = True
    try:
        yield
    finally:
        _EVAL_GEMM.on = prev


# set by precise_bn_stats(): the BNStatsAccumulator train-mode BatchNorm layers add their batch statistics to
_PRECISE_BN = [None]


class BNStatsAccumulator(object):
    """fp64 sums of the per-batch statistics of every BatchNorm layer of ``module``, for precise BatchNorm
    statistics (``GossipTrainer.update_bn``).  One flat fp64 buffer (:attr:`flat`), allocated once, so its
    addresses are stable under graph capture; layer l's view (:attr:`views`) is ``[2 C_l]``: the sum of its
    batch means, then the sum of its unbiased batch variances -- the fp32 values the training forward would
    blend into the running buffers.  Every BatchNorm layer that tracks running statistics must be a
    :class:`FusedBatchNormAct2d` (ValueError otherwise)."""

    def __init__(self, module: nn.Module):
        from torch.nn.modules.batchnorm import _BatchNorm
        layers = [m for m in module.modules() if isinstance(m, _BatchNorm) and m.track_running_stats]
        other = sorted(set(type(m).__name__ for m in layers if not isinstance(m, FusedBatchNormAct2d)))
        if other:
            raise ValueError('precise BatchNorm statistics need every BatchNorm layer to be a FusedBatchNormAct2d; '
                             'found %s' % ', '.join(other))
        sizes = [2 * m.num_features for m in layers]
        device = layers[0].running_mean.device if layers else torch.device('cpu')
        self.layers = layers
        self.flat = torch.zeros(sum(sizes), dtype=torch.float64, device=device)
        self.views = list(self.flat.split(sizes))
        self._view_of = {m: v for m, v in zip(layers, self.views)}

    def view_of(self, bn) -> torch.Tensor:
        v = self._view_of.get(bn)
        if v is None:
            raise ValueError('precise_bn_stats: a train-mode BatchNorm layer (%s) is not one of the '
                             "accumulator's layers" % bn)
        return v

    def zero_(self):
        self.flat.zero_()

    @torch.no_grad()
    def commit(self, k: int):
        """``running_mean = fp32(sum of means / k)``, ``running_var = fp32(sum of variances / k)`` for every
        layer, k >= 1: one ``bn_stats_commit`` launch on CUDA, torch ops on the reference path."""
        if k < 1:
            raise ValueError('commit needs k >= 1, got %r' % (k,))
        if not self.layers:
            return
        if FORCE_REFERENCE or not self.flat.is_cuda:
            for m, v in zip(self.layers, self.views):
                c = m.num_features
                m.running_mean.copy_((v[:c] / k).float())
                m.running_var.copy_((v[c:] / k).float())
            return
        native.load().bn_stats_commit(self.views, [m.running_mean for m in self.layers],
                                      [m.running_var for m in self.layers], int(k))


@contextlib.contextmanager
def precise_bn_stats(acc: BNStatsAccumulator):
    """Inside the block every train-mode ``FusedBatchNormAct2d``, ``conv_bn_act`` and ``conv_bn_act_split``
    of ``acc``'s layers normalises with its batch statistics as in training, but adds those statistics
    (the batch mean and unbiased variance, as fp32 values) to its view of ``acc`` in fp64 instead of
    updating its running buffers; ``num_batches_tracked`` is not advanced.  The forward's outputs are those
    of a training forward, bit for bit.  Outside it a forward runs as before.
    ``GossipTrainer.update_bn`` uses it, then ``acc.commit(K)``."""
    prev = _PRECISE_BN[0]
    _PRECISE_BN[0] = acc
    try:
        yield acc
    finally:
        _PRECISE_BN[0] = prev


def precise_bn_active() -> bool:
    """True inside :func:`precise_bn_stats` (the forward then describes the network evaluation runs: no
    stochastic depth)"""
    return _PRECISE_BN[0] is not None


def _acc_of(bn, training: bool):
    """the accumulator view of a train-mode BatchNorm inside :func:`precise_bn_stats`, else None"""
    acc = _PRECISE_BN[0]
    if acc is None or not training or not bn.track_running_stats:
        return None
    return acc.view_of(bn)


def _can_fuse(x: torch.Tensor) -> bool:
    if FORCE_REFERENCE or not x.is_cuda or not native.available():
        return False
    return bool(native.load().bn_can_fuse(x))


class _FusedBNAct(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, residual, weight, bias, running_mean, running_var, nbt,
                training, momentum, eps, relu, acc, branch_scale):
        C = native.load()
        y, coef = C.bn_forward(x, residual, weight, bias, running_mean, running_var, nbt,
                               training, momentum, eps, relu, acc, **_scale_kw(branch_scale))
        ctx.branch_scale = branch_scale
        ctx.relu = relu
        ctx.add = residual is not None
        ctx.training = training
        if ctx.add:
            ctx.save_for_backward(x, y, coef, weight)
        else:
            ctx.save_for_backward(x, coef, weight)
        return y

    @staticmethod
    def backward(ctx, dy):
        C = native.load()
        if ctx.add:
            x, y, coef, weight = ctx.saved_tensors
        else:
            x, coef, weight = ctx.saved_tensors
            y = None
        if not ctx.training:
            # eval-mode BN is an affine map: dx = scale * dz
            scale = coef[2].to(dy.dtype).view(1, -1, 1, 1)
            dz = dy
            if ctx.relu:
                out = y if ctx.add else torch.relu(F.batch_norm(x, None, None, training=False))
                dz = dy * (out > 0)
            return dz * scale, (dz if ctx.add else None), None, None, None, None, None, \
                None, None, None, None, None, None
        dx, dz, ggamma, gbeta = C.bn_backward(dy, x, y, coef, ctx.relu, ctx.add, **_scale_kw(ctx.branch_scale))
        return dx, (dz if ctx.add else None), ggamma, gbeta, None, None, None, None, None, None, None, None, None


def _scale_kw(branch_scale):
    """the ``branch_scale`` keyword of the native calls: none at all without a scale (today's calls)"""
    return {} if branch_scale is None else {'branch_scale': branch_scale}


def _check_branch_scale(branch_scale, x, residual):
    if branch_scale is None:
        return
    if residual is None:
        raise ValueError('branch_scale scales a residual branch: it needs a residual')
    if branch_scale.dim() != 1 or branch_scale.shape[0] != x.shape[0] or branch_scale.dtype != torch.float32:
        raise ValueError('branch_scale must be an fp32 [N] tensor, one value per sample, got %s %s'
                         % (tuple(branch_scale.shape), branch_scale.dtype))


def fused_bn_act(x, weight, bias, running_mean, running_var, num_batches_tracked=None,
                 residual=None, relu=False, training=True, momentum=0.1, eps=1e-5, acc=None, branch_scale=None):
    """Functional form; falls back to plain PyTorch when the kernels cannot run.  ``acc`` (training
    only): an fp64 ``[2C]`` accumulator that receives the batch statistics instead of the running
    buffers (see :func:`precise_bn_stats`).  ``branch_scale`` (with a residual; stochastic depth, see
    ``ops.stochastic_depth``): an fp32 ``[N]`` per-sample scale of the BN output before the residual add,
    ``relu?(bn(x) * s[n] + residual)``; the fused kernels apply it in training mode."""
    _check_branch_scale(branch_scale, x, residual)
    fusable = _can_fuse(x) and weight is not None and weight.dtype == torch.float32 \
        and (residual is None or (relu and residual.dtype == x.dtype
                                  and residual.stride() == x.stride())) \
        and (branch_scale is None or (training and branch_scale.device == x.device))
    if fusable and (training or not torch.is_grad_enabled() or not x.requires_grad):
        return _FusedBNAct.apply(x, residual, weight, bias, running_mean, running_var,
                                 num_batches_tracked, training, momentum, eps, relu, acc,
                                 None if branch_scale is None else branch_scale.contiguous())
    return reference_bn_act(x, weight, bias, running_mean, running_var, num_batches_tracked,
                            residual, relu, training, momentum, eps, acc, branch_scale)


def reference_bn_act(x, weight, bias, running_mean, running_var, num_batches_tracked=None,
                     residual=None, relu=False, training=True, momentum=0.1, eps=1e-5, acc=None,
                     branch_scale=None):
    if acc is not None:
        # the batch statistics exactly as a momentum-1 update of zeroed running buffers writes them
        stats = torch.zeros(2, x.shape[1], dtype=running_mean.dtype, device=x.device)
        y = F.batch_norm(x, stats[0], stats[1], weight, bias, True, 1.0, eps)
        acc.add_(stats.view(-1))
    else:
        if training and num_batches_tracked is not None:
            num_batches_tracked.add_(1)
        y = F.batch_norm(x, running_mean, running_var, weight, bias, training, momentum, eps)
    if branch_scale is not None:
        # in (at least) fp32, rounded once, as the kernels do
        ct = torch.promote_types(y.dtype, torch.float32)
        y = (y.to(ct) * branch_scale.view(-1, 1, 1, 1).to(ct) + residual.to(ct)).to(y.dtype)
    elif residual is not None:
        y = y + residual
    return F.relu(y) if relu else y


class FusedBatchNormAct2d(nn.BatchNorm2d):
    """``y = relu?(bn(x) (+ residual)?)`` -- see module docstring."""

    def forward(self, x, residual=None, relu=False, branch_scale=None):
        training = self.training or (self.running_mean is None)
        momentum = 0.1 if self.momentum is None else self.momentum
        return fused_bn_act(
            x, self.weight, self.bias,
            self.running_mean if self.track_running_stats else None,
            self.running_var if self.track_running_stats else None,
            self.num_batches_tracked if (self.track_running_stats and training) else None,
            residual=residual, relu=relu, training=training, momentum=momentum, eps=self.eps,
            acc=_acc_of(self, training), branch_scale=branch_scale)


# --------------------------------------------------------------------------- #
# 1x1 convolution + BatchNorm (+ residual) (+ ReLU)
# --------------------------------------------------------------------------- #
class _BNBackwardHandoff:
    """What a residual block's last BN (``_Conv1x1BNAct`` with a residual) leaves on its output
    so that the next block's conv1 dgrad (``_Conv1x1BNActSplit``) can do that BN's backward
    reduction in its epilogue: the BN input ``yraw``, its ``coef``, the output's 1-bit ReLU
    ``mask`` and its stochastic-depth ``branch_scale`` (or None).  The dgrad records which tensor it produced (``dz_key``: data pointer and version)
    and the reduction ``partial``; the BN backward uses them only if its incoming gradient is
    that very tensor, unmodified."""
    __slots__ = ('yraw', 'coef', 'mask', 'branch_scale', 'dz_key', 'partial')

    def __init__(self, yraw, coef, mask, branch_scale=None):
        self.yraw, self.coef, self.mask, self.branch_scale = yraw, coef, mask, branch_scale
        self.dz_key = self.partial = None


class _Conv1x1BNAct(torch.autograd.Function):
    """``act(bn(conv1x1(x, w)) [+ residual])`` in training mode.  Forward: wgmma GEMM
    whose epilogue also produces the BatchNorm statistics, finalize, apply.  Backward: the
    fused BN backward, then the library's dgrad / wgrad for the convolution."""

    @staticmethod
    def forward(ctx, x, w, residual, gamma, beta, running_mean, running_var, nbt, momentum, eps, relu, acc,
                branch_scale):
        C = native.load()
        w16 = w if w.dtype == x.dtype else w.detach().to(x.dtype)      # compute-dtype weights
        mask = None
        if residual is not None and relu and USE_BN_BWD_FUSE:
            M, N = x.numel() // x.shape[1], w.shape[0]
            mask = torch.empty((M, N // 8), dtype=torch.uint8, device=x.device)
        yraw, out, coef = C.conv1x1_bn_forward(x, w16, residual, gamma, beta, running_mean, running_var,
                                               nbt, momentum, eps, relu, mask, acc=acc, **_scale_kw(branch_scale))
        ctx.relu = relu
        ctx.add = residual is not None
        ctx.w_dtype = w.dtype
        ctx.branch_scale = branch_scale
        ctx.handoff = None
        if mask is not None:
            ctx.handoff = out._sgp_bn_handoff = _BNBackwardHandoff(yraw, coef, mask, branch_scale)
        if ctx.add:
            ctx.save_for_backward(x, w16, yraw, coef, out)
        else:
            ctx.save_for_backward(x, w16, yraw, coef)
        return out

    @staticmethod
    def backward(ctx, dy):
        C = native.load()
        x, w16, yraw, coef = ctx.saved_tensors[:4]
        out = ctx.saved_tensors[4] if ctx.add else None
        h = ctx.handoff
        if h is not None and h.dz_key == (dy.data_ptr(), dy._version) and dy.stride() == yraw.stride():
            # dy is the next block's MODE 3 dgrad output: already masked (it is this BN's dz and the
            # residual branch's gradient), its reduction already done
            dyraw, ggamma, gbeta = C.bn_backward_from_partials(dy, yraw, coef, h.partial,
                                                               **_scale_kw(ctx.branch_scale))
            dz = dy
        else:
            dyraw, dz, ggamma, gbeta = C.bn_backward(dy, yraw, out, coef, ctx.relu, ctx.add,
                                                     **_scale_kw(ctx.branch_scale))
        if h is not None:
            h.dz_key = h.partial = None
        dx, dw, _ = torch.ops.aten.convolution_backward(
            dyraw, x, w16, None, [1, 1], [0, 0], [1, 1], False, [0, 0], 1,
            [ctx.needs_input_grad[0], ctx.needs_input_grad[1], False])
        if dw is not None and dw.dtype != ctx.w_dtype:
            dw = dw.to(ctx.w_dtype)
        return dx, dw, (dz if ctx.add else None), ggamma, gbeta, None, None, None, None, None, None, None, None


class _Conv1x1BNActSplit(torch.autograd.Function):
    """``(act(bn(conv1x1(x, w))), x)`` for a block input that also feeds the skip connection.
    Returning ``x`` through the op routes the skip-branch gradient into ``backward``, where the
    dgrad GEMM adds it in its epilogue (fp32, before rounding) instead of autograd running a
    separate read-read-write accumulation pass over the widest activation of the block."""

    @staticmethod
    def forward(ctx, x, w, gamma, beta, running_mean, running_var, nbt, momentum, eps, relu, handoff, acc):
        C = native.load()
        w16 = w if w.dtype == x.dtype else w.detach().to(x.dtype)
        yraw, out, coef = C.conv1x1_bn_forward(x, w16, None, gamma, beta, running_mean, running_var,
                                               nbt, momentum, eps, relu, acc=acc)
        ctx.relu = relu
        ctx.w_dtype = w.dtype
        ctx.handoff = handoff
        ctx.save_for_backward(x, w16, yraw, coef)
        ctx.set_materialize_grads(False)
        return out, x.view_as(x)

    @staticmethod
    def backward(ctx, d_out, d_skip):
        C = native.load()
        x, w16, yraw, coef = ctx.saved_tensors
        if d_out is None:
            d_out = torch.zeros_like(yraw)
        dyraw, _, ggamma, gbeta = C.bn_backward(d_out, yraw, None, coef, ctx.relu, False)
        dx = dw = None
        if ctx.needs_input_grad[0]:
            # dX = dY . W: the same GEMM with the transposed weight as its K-major B operand
            wt = w16.reshape(w16.shape[0], w16.shape[1]).t().contiguous()
            res = d_skip
            if res is not None and (res.dtype != dyraw.dtype
                                    or not res.is_contiguous(memory_format=torch.channels_last)):
                res = res.to(dyraw.dtype).contiguous(memory_format=torch.channels_last)
            h = ctx.handoff
            if (h is not None and res is not None and h.yraw.dtype == dyraw.dtype
                    and h.yraw.stride() == res.stride() and C.conv1x1_can_fuse(dyraw, wt)):
                # + the previous block's last BN backward reduction (MODE 3): dx is that BN's dz
                dx, h.partial = C.conv1x1_dgrad_bn_reduce(dyraw, wt, res, h.yraw, h.coef, h.mask,
                                                          **_scale_kw(h.branch_scale))
                h.dz_key = (dx.data_ptr(), dx._version)
            elif C.conv1x1_can_fuse(dyraw, wt):
                dx = C.conv1x1_forward(dyraw, wt, False, res)
            else:
                dx = torch.ops.aten.convolution_backward(
                    dyraw, x, w16, None, [1, 1], [0, 0], [1, 1], False, [0, 0], 1, [True, False, False])[0]
                if res is not None:
                    dx = dx + res
        if ctx.needs_input_grad[1]:
            dw = torch.ops.aten.convolution_backward(
                dyraw, x, w16, None, [1, 1], [0, 0], [1, 1], False, [0, 0], 1, [False, True, False])[1]
            if dw.dtype != ctx.w_dtype:
                dw = dw.to(ctx.w_dtype)
        return dx, dw, ggamma, gbeta, None, None, None, None, None, None, None, None


def _conv1x1_operands(conv, bn, x, residual, relu):
    """(x, fusable): x possibly cast the way autocast would; fusable says whether the wgmma
    conv + BN path covers this call."""
    train_or_eval = bn.training or (_EVAL_GEMM.on and not torch.is_grad_enabled())
    if not (USE_TCGEN05_CONV1X1 and not FORCE_REFERENCE and train_or_eval and bn.track_running_stats
            and x.is_cuda and native.available() and x.dim() == 4
            and conv.kernel_size == (1, 1) and conv.stride == (1, 1) and conv.padding == (0, 0)
            and conv.groups == 1 and conv.bias is None and bn.weight is not None
            and bn.weight.dtype == torch.float32 and (residual is None or relu)):
        return x, False
    w = conv.weight
    if x.dtype == torch.float32 and torch.is_autocast_enabled():
        x = x.to(torch.bfloat16)
    if x.dtype == torch.float32:
        # fp32 activations: the GEMM multiplies in TF32 (what the library convolution does by
        # default); honour a user who switched TF32 off
        dtype_ok = w.dtype == torch.float32 and torch.backends.cudnn.allow_tf32
    else:
        dtype_ok = x.dtype == torch.bfloat16 and (w.dtype == torch.bfloat16 or torch.is_autocast_enabled())
    if not (dtype_ok and x.is_contiguous(memory_format=torch.channels_last)
            and (residual is None or (residual.dtype == x.dtype
                                      and residual.is_contiguous(memory_format=torch.channels_last)))):
        return x, False
    wk = w if w.dtype == x.dtype else w.detach().to(x.dtype)
    return x, bool(native.load().conv1x1_can_fuse(x, wk)) and conv.out_channels % 8 == 0


def conv_bn_act(conv: nn.Conv2d, bn: 'FusedBatchNormAct2d', x, residual=None, relu=False, branch_scale=None):
    """``bn(conv(x), residual=residual, relu=relu, branch_scale=branch_scale)``; 1x1 / stride-1 convolutions
    of NHWC bf16 activations in training mode take the fused wgmma path, and so do eval-mode ones inside
    :func:`eval_bn_gemm`."""
    _check_branch_scale(branch_scale, x, residual)
    xk, ok = _conv1x1_operands(conv, bn, x, residual, relu)
    if branch_scale is not None and not (bn.training and branch_scale.device == x.device):
        ok = False
    if ok and not bn.training:
        w = conv.weight if conv.weight.dtype == xk.dtype else conv.weight.detach().to(xk.dtype)
        return native.load().conv1x1_bn_eval(xk, w, bn.weight, bn.bias, bn.running_mean, bn.running_var,
                                             bn.eps, relu, residual)
    if ok:
        momentum = 0.1 if bn.momentum is None else bn.momentum
        return _Conv1x1BNAct.apply(xk, conv.weight, residual, bn.weight, bn.bias, bn.running_mean,
                                   bn.running_var, bn.num_batches_tracked, momentum, bn.eps, relu,
                                   _acc_of(bn, True), None if branch_scale is None else branch_scale.contiguous())
    if branch_scale is None:
        return bn(conv(x), residual=residual, relu=relu)
    return bn(conv(x), residual=residual, relu=relu, branch_scale=branch_scale)


def conv_bn_act_split(conv: nn.Conv2d, bn: 'FusedBatchNormAct2d', x, relu=False):
    """``(bn(conv(x), relu=relu), x)`` for an ``x`` that is also consumed by a skip connection:
    use the returned ``x`` for the skip branch and its gradient is added inside the dgrad GEMM
    of ``conv`` (see :class:`_Conv1x1BNActSplit`).  Falls back to ``(conv_bn_act(...), x)``.

    When ``x`` is the output of the previous block's fused last BN, that BN's backward reduction
    also moves into the dgrad; the gradient ``x`` then receives is the post-ReLU-mask one, so this
    is skipped when anyone can observe it (a hook on ``x`` or ``x.retain_grad()``)."""
    if x.requires_grad and torch.is_grad_enabled():
        xk, ok = _conv1x1_operands(conv, bn, x, None, relu)
        if ok and xk is x:
            momentum = 0.1 if bn.momentum is None else bn.momentum
            handoff = getattr(x, '_sgp_bn_handoff', None)
            if handoff is not None and (not USE_BN_BWD_FUSE or x._backward_hooks or x.retains_grad
                                        or handoff.yraw.shape != x.shape):
                handoff = None
            return _Conv1x1BNActSplit.apply(x, conv.weight, bn.weight, bn.bias, bn.running_mean,
                                            bn.running_var, bn.num_batches_tracked, momentum, bn.eps, relu,
                                            handoff, _acc_of(bn, True))
    return conv_bn_act(conv, bn, x, relu=relu), x


# --------------------------------------------------------------------------- #
# NHWC max-pool
# --------------------------------------------------------------------------- #
class _MaxPoolNHWC(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, k, s, p):
        C = native.load()
        y, code = C.maxpool_forward(x, k, s, p)
        ctx.save_for_backward(code)
        ctx.geom = (x.shape[2], x.shape[3], k, s, p)
        return y

    @staticmethod
    def backward(ctx, dy):
        C = native.load()
        (code,) = ctx.saved_tensors
        H, W, k, s, p = ctx.geom
        return C.maxpool_backward(dy, code, H, W, k, s, p), None, None, None


class MaxPool2dNHWC(nn.MaxPool2d):
    """``nn.MaxPool2d`` whose channels-last CUDA path is the sm_90a gather
    kernel pair in ``csrc/pool_kernels.cu`` (1-byte argmax codes instead of
    int64 indices, atomic-free backward).  Other inputs use the stock op."""

    def forward(self, x):
        k, s, p = self.kernel_size, self.stride, self.padding
        simple = all(isinstance(v, int) for v in (k, s, p)) and self.dilation == 1 \
            and not self.ceil_mode and not self.return_indices
        if simple and not FORCE_REFERENCE and x.is_cuda and native.available() \
                and native.load().pool_can_fuse(x, k, s, p):
            return _MaxPoolNHWC.apply(x, k, s, p)
        return super().forward(x)


# --------------------------------------------------------------------------- #
# ResNet stem convolution
# --------------------------------------------------------------------------- #
class _StemConv(torch.autograd.Function):

    @staticmethod
    def forward(ctx, x, weight):
        C = native.load()
        w16 = weight                   # compute-dtype weights: bf16, or fp32 (TF32 tensor-core math)
        if w16.dtype != x.dtype or not w16.is_contiguous(memory_format=torch.channels_last):
            w16 = weight.detach().to(x.dtype).contiguous(memory_format=torch.channels_last)
        ctx.save_for_backward(x)
        ctx.w_dtype = weight.dtype
        return C.stem_forward(x, w16)

    @staticmethod
    def backward(ctx, dy):
        C = native.load()
        (x,) = ctx.saved_tensors
        dw = C.stem_wgrad(x, dy)
        return None, dw.to(ctx.w_dtype)


def stem_conv(conv: nn.Conv2d, x: torch.Tensor) -> torch.Tensor:
    """``conv(x)`` for the ResNet stem (3 -> 64 channels, 7x7, stride 2, pad 3, no bias).
    NHWC bf16 CUDA inputs run the tensor-core implicit-GEMM kernels in
    ``csrc/stem_kernels.cu`` (the library needs 1.48 ms + 0.77 ms for this layer at batch
    256; its HBM traffic is worth ~0.1 ms); anything else runs ``conv`` unchanged."""
    ok = (USE_STEM_KERNELS and not FORCE_REFERENCE and x.is_cuda and native.available() and not x.requires_grad
          and conv.in_channels == 3 and conv.out_channels == 64 and conv.kernel_size == (7, 7)
          and conv.stride == (2, 2) and conv.padding == (3, 3) and conv.dilation == (1, 1)
          and conv.groups == 1 and conv.bias is None)
    if ok and x.dtype == torch.float32 and torch.is_autocast_enabled():
        x = x.to(torch.bfloat16)          # what autocast would do inside the convolution
    dtype_ok = x.dtype == torch.bfloat16 or (x.dtype == torch.float32 and conv.weight.dtype == torch.float32
                                             and torch.backends.cudnn.allow_tf32)
    if ok and dtype_ok and x.dim() == 4 \
            and x.is_contiguous(memory_format=torch.channels_last) and x.shape[2] >= 7 and x.shape[3] >= 7:
        return _StemConv.apply(x, conv.weight)
    return conv(x)
