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


def ta_wide_op(img: torch.Tensor, op: str, magnitude: float) -> torch.Tensor:
    """The augmentation op ``op`` (any of ``data.shards.AUGMENT_OPS``) at the signed ``magnitude`` on a
    uint8 ``[3, H, W]`` image, through ``torchvision.transforms.v2.functional`` with the arguments
    TrivialAugmentWide, RandAugment and AutoAugment pass (nearest interpolation, fill 0)."""
    import math
    import torchvision.transforms.v2.functional as TF
    from torchvision.transforms import InterpolationMode
    nearest = InterpolationMode.NEAREST
    if op == 'Identity':
        return img
    if op in ('ShearX', 'ShearY'):
        deg = math.degrees(math.atan(magnitude))
        return TF.affine(img, angle=0.0, translate=[0, 0], scale=1.0,
                         shear=[deg, 0.0] if op == 'ShearX' else [0.0, deg], interpolation=nearest,
                         fill=None, center=[0, 0])
    if op in ('TranslateX', 'TranslateY'):
        t = [int(magnitude), 0] if op == 'TranslateX' else [0, int(magnitude)]
        return TF.affine(img, angle=0.0, translate=t, scale=1.0, shear=[0.0, 0.0], interpolation=nearest,
                         fill=None)
    if op == 'Rotate':
        return TF.rotate(img, angle=magnitude, interpolation=nearest, fill=None)
    if op == 'Brightness':
        return TF.adjust_brightness(img, 1.0 + magnitude)
    if op == 'Color':
        return TF.adjust_saturation(img, 1.0 + magnitude)
    if op == 'Contrast':
        return TF.adjust_contrast(img, 1.0 + magnitude)
    if op == 'Sharpness':
        return TF.adjust_sharpness(img, 1.0 + magnitude)
    if op == 'Posterize':
        return TF.posterize(img, int(magnitude))
    if op == 'Solarize':
        return TF.solarize(img, 255 * magnitude)
    if op == 'AutoContrast':
        return TF.autocontrast(img)
    if op == 'Equalize':
        return TF.equalize(img)
    if op == 'Invert':
        return TF.invert(img)
    raise ValueError('unknown augmentation op %r' % (op,))


def reference_augment(batch_u8: torch.Tensor, theta: torch.Tensor, ops, magnitudes, erase, out_size: int,
                      mean: torch.Tensor, inv: torch.Tensor) -> torch.Tensor:
    """What the augment kernel computes, in plain PyTorch + torchvision: ``grid_sample`` of the
    uint8 NHWC batch with the crop maps ``theta`` (bilinear, border, align_corners=False), rounded
    to uint8; per sample the op ``data.shards.AUGMENT_OPS[ops[i]]`` at ``magnitudes[i]``, or with
    ``[n, K]`` ops and magnitudes the ops ``ops[i, 0]``, ..., ``ops[i, K - 1]`` left to right, each on
    the uint8 result of the one before; ``(v - mean) * inv`` in fp32; 0 inside each
    ``erase[i] = (top, left, h, w)`` box.  Returns fp32 ``[n, 3, out, out]`` in channels-last memory
    format."""
    import torch.nn.functional as F
    from ..data.shards import AUGMENT_OPS
    n = batch_u8.shape[0]
    x = batch_u8.permute(0, 3, 1, 2).float()
    grid = F.affine_grid(theta.to(x.device), (n, 3, out_size, out_size), align_corners=False)
    crop = F.grid_sample(x, grid, mode='bilinear', padding_mode='border', align_corners=False)
    crop = crop.round().clamp(0, 255).to(torch.uint8)
    y = torch.empty(n, 3, out_size, out_size)
    ops, magnitudes = torch.as_tensor(ops), torch.as_tensor(magnitudes)
    if ops.dim() == 1:
        ops, magnitudes = ops[:, None], magnitudes[:, None]
    for i in range(n):
        img = crop[i]
        for op, magnitude in zip(ops[i].tolist(), magnitudes[i].tolist()):
            img = ta_wide_op(img, AUGMENT_OPS[int(op)], float(magnitude))
        y[i] = (img.float() - mean[0]) * inv[0]
        top, left, h, w = (int(v) for v in erase[i])
        y[i, :, top:top + h, left:left + w] = 0.0
    return y.contiguous(memory_format=torch.channels_last)


_MASK64 = (1 << 64) - 1


def _mix64(z):
    """splitmix64's finaliser on uint64 numpy arrays (wrapping arithmetic)"""
    import numpy as np
    z = (z + np.uint64(0x9E3779B97F4A7C15)) & np.uint64(_MASK64)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def drop_path_scales(seed: int, rank: int, draw: int, thresholds, keep_scales, n: int) -> torch.Tensor:
    """What ``drop_path_draw_kernel`` writes for draw index ``draw``: the fp32 ``[L, n]`` stochastic-depth
    branch scales, ``out[l][i] = keep_scales[l]`` if the top 24 bits of
    ``mix(mix(mix(mix(seed) ^ rank) ^ draw) ^ (l << 32 | i))`` are below ``thresholds[l]``, else 0
    (``mix`` = splitmix64's finaliser, seed / rank / draw as uint64)."""
    import numpy as np
    L = len(thresholds)
    with np.errstate(over='ignore'):
        base = _mix64(np.array([int(seed) & _MASK64], dtype=np.uint64))
        base = _mix64(base ^ np.uint64(int(rank) & _MASK64))
        base = _mix64(base ^ np.uint64(int(draw) & _MASK64))
        key = (np.arange(L, dtype=np.uint64)[:, None] << np.uint64(32)) | np.arange(n, dtype=np.uint64)[None, :]
        u = _mix64(base ^ key) >> np.uint64(40)
    keep = u < np.array(thresholds, dtype=np.uint64)[:, None]
    out = np.where(keep, np.array(keep_scales, dtype=np.float32)[:, None], np.float32(0.0))
    return torch.from_numpy(out.astype(np.float32))


def rotate_all(graphs):
    for g in graphs:
        if g.is_dynamic_graph():
            g.get_peers(rotate=True)
