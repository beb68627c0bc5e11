"""
Pre-decoded image shards + GPU-side augmentation: the input pipeline that keeps up with an H100.

The reference feeds its trainer with ``torchvision.datasets.ImageFolder`` + ``DataLoader`` workers
(``gossip_sgd.py:539-583``): JPEG decode, ``RandomResizedCrop``, flip, ``ToTensor``, ``Normalize`` on
the CPU, 602 KB of fp32 per image over PCIe.  That is ~1-2 k images/s per process; one H100 trains
ResNet-50 at 2.8 k images/s (fp32/TF32) to 5.8 k (bf16) at batch 256 (measured at a 400 W power
limit), i.e. the stock pipeline would leave the GPU idle much of the time.  (The stock pipeline stays available: ``--data_format folder``.)

Here the dataset is decoded ONCE into uint8 shards (``write_shards``: short side resized to
``store_size``, centre crop, raw RGB, ``.npy`` files that are memory-mapped at training time):

* the loader (:class:`ShardLoader`) only gathers rows of the maps into a pinned uint8 batch --
  a background thread keeps ``prefetch`` batches ahead; 196 KB per 256x256 image, 3x less PCIe
  traffic than fp32 crops;
* crop / scale / flip / normalisation run on the GPU as ONE batched ``grid_sample``
  (:class:`GpuAugment`: per-sample random-resized-crop boxes expressed as affine grids, bilinear,
  flip = negated x scale), producing the channels-last fp32 / bf16 batch the model consumes.
  The same code runs on the CPU (tests).

Sharding over ranks and epochs follows ``DistributedSampler``: one seeded permutation per epoch,
rank r takes ``perm[r::world]``, the tail is dropped (``drop_last=True`` as in the reference's
training loader).
"""

from __future__ import annotations

import functools
import json
import math
import os
import queue
import threading
from typing import List, NamedTuple, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)
RING_SLOTS = 8                  # pinned staging slots of the augment kernel's per-image rows


# --------------------------------------------------------------------------- #
# writing
# --------------------------------------------------------------------------- #
def write_shards_from_arrays(out_dir: str, images: np.ndarray, labels: Sequence[int],
                             classes: Optional[List[str]] = None, shard_size: int = 4096) -> dict:
    """``images``: uint8 [N, S, S, 3]; writes ``images_%05d.npy`` / ``labels_%05d.npy`` + ``index.json``."""
    images = np.asarray(images)
    labels = np.asarray(labels, dtype=np.int64)
    assert images.dtype == np.uint8 and images.ndim == 4 and images.shape[3] == 3
    assert images.shape[1] == images.shape[2] and len(images) == len(labels)
    os.makedirs(out_dir, exist_ok=True)
    counts = []
    for s, lo in enumerate(range(0, len(images), shard_size)):
        hi = min(lo + shard_size, len(images))
        np.save(os.path.join(out_dir, 'images_%05d.npy' % s), images[lo:hi])
        np.save(os.path.join(out_dir, 'labels_%05d.npy' % s), labels[lo:hi])
        counts.append(hi - lo)
    index = {'format': 'sgp_b200_shards_v1', 'size': int(images.shape[1]), 'counts': counts,
             'classes': list(classes) if classes is not None else None}
    with open(os.path.join(out_dir, 'index.json'), 'w') as f:
        json.dump(index, f)
    return index


def write_shards(image_folder: str, out_dir: str, store_size: int = 256, shard_size: int = 4096,
                 limit: Optional[int] = None) -> dict:
    """Decode an ``ImageFolder`` tree (``root/class_x/*.jpg``) once: resize the short side to
    ``store_size`` (bilinear), centre-crop to ``store_size x store_size``, store raw RGB."""
    from PIL import Image
    classes = sorted(d for d in os.listdir(image_folder) if os.path.isdir(os.path.join(image_folder, d)))
    files = []
    for ci, c in enumerate(classes):
        for name in sorted(os.listdir(os.path.join(image_folder, c))):
            if name.lower().endswith(('.jpg', '.jpeg', '.png', '.bmp', '.webp', '.ppm')):
                files.append((os.path.join(image_folder, c, name), ci))
    if limit is not None:
        files = files[:limit]
    os.makedirs(out_dir, exist_ok=True)
    counts = []
    for s, lo in enumerate(range(0, len(files), shard_size)):
        chunk = files[lo:lo + shard_size]
        arr = np.empty((len(chunk), store_size, store_size, 3), dtype=np.uint8)
        for i, (path, _) in enumerate(chunk):
            with Image.open(path) as im:
                im = im.convert('RGB')
                w, h = im.size
                scale = store_size / min(w, h)
                nw, nh = max(store_size, round(w * scale)), max(store_size, round(h * scale))
                im = im.resize((nw, nh), Image.BILINEAR)
                left, top = (nw - store_size) // 2, (nh - store_size) // 2
                arr[i] = np.asarray(im.crop((left, top, left + store_size, top + store_size)))
        np.save(os.path.join(out_dir, 'images_%05d.npy' % s), arr)
        np.save(os.path.join(out_dir, 'labels_%05d.npy' % s), np.asarray([c for _, c in chunk], dtype=np.int64))
        counts.append(len(chunk))
    index = {'format': 'sgp_b200_shards_v1', 'size': store_size, 'counts': counts, 'classes': classes}
    with open(os.path.join(out_dir, 'index.json'), 'w') as f:
        json.dump(index, f)
    return index


# --------------------------------------------------------------------------- #
# reading
# --------------------------------------------------------------------------- #
class ShardLoader(object):
    """Iterates ``(uint8 [B, S, S, 3] pinned-host batch, int64 [B] labels)`` over this rank's share
    of the shards.  ``set_epoch`` reseeds the permutation (it is its own sampler, like the CLI's
    synthetic loader)."""

    def __init__(self, root: str, batch_size: int, world_size: int = 1, rank: int = 0, shuffle: bool = True,
                 drop_last: bool = True, seed: int = 0, prefetch: int = 3, pin: Optional[bool] = None):
        with open(os.path.join(root, 'index.json')) as f:
            self.index = json.load(f)
        assert self.index.get('format') == 'sgp_b200_shards_v1', 'not a shard directory: %s' % root
        self.size = int(self.index['size'])
        self.counts = [int(c) for c in self.index['counts']]
        self.images = [np.load(os.path.join(root, 'images_%05d.npy' % s), mmap_mode='r')
                       for s in range(len(self.counts))]
        self.labels = np.concatenate([np.load(os.path.join(root, 'labels_%05d.npy' % s))
                                      for s in range(len(self.counts))]) if self.counts else np.zeros(0, np.int64)
        self.offsets = np.concatenate([[0], np.cumsum(self.counts)]).astype(np.int64)
        self.total = int(self.offsets[-1])
        self.batch_size, self.world_size, self.rank = int(batch_size), int(world_size), int(rank)
        self.shuffle, self.drop_last, self.seed = shuffle, drop_last, int(seed)
        self.prefetch = max(1, int(prefetch))
        self.pin = torch.cuda.is_available() if pin is None else bool(pin)
        self.use_native = True
        self.gather_threads = int(os.environ.get('SGP_B200_LOADER_THREADS', 8))   # memcpy threads per batch
        self.sampler = self
        self._epoch = 0
        per_rank = self.total // self.world_size if drop_last else -(-self.total // self.world_size)
        self.n_batches = per_rank // self.batch_size if drop_last else -(-per_rank // self.batch_size)
        self.per_rank = per_rank

    def set_epoch(self, epoch: int):
        self._epoch = int(epoch)

    def __len__(self):
        return self.n_batches

    def indices(self, epoch: Optional[int] = None) -> np.ndarray:
        """this rank's sample indices for ``epoch`` (DistributedSampler arithmetic)"""
        epoch = self._epoch if epoch is None else epoch
        if self.shuffle:
            g = torch.Generator().manual_seed(self.seed * 1000003 + epoch)
            perm = torch.randperm(self.total, generator=g).numpy()
        else:
            perm = np.arange(self.total)
        if self.drop_last:
            perm = perm[:self.per_rank * self.world_size]
        else:                              # pad by wrapping, like DistributedSampler
            need = self.per_rank * self.world_size - len(perm)
            if need > 0:
                perm = np.concatenate([perm, perm[:need]])
        return perm[self.rank::self.world_size]

    def _native(self):
        """the extension's multi-threaded row gather (``csrc/data_loader.cpp``), or None"""
        if getattr(self, '_gather_fn', False) is False:
            self._gather_fn = None
            try:
                from ..ops import native
                if native.available():
                    self._gather_fn = native.load().gather_rows_u8
                    self._ptrs = [int(a.ctypes.data) for a in self.images]
                    self._row_bytes = self.size * self.size * 3
            except Exception:
                self._gather_fn = None
        return self._gather_fn

    def _gather(self, idx: np.ndarray, out: torch.Tensor):
        """rows ``idx`` of the concatenated shards -> ``out``: a multi-threaded memcpy in the native
        extension (GIL released), else one numpy fancy-index copy per shard"""
        shard = np.searchsorted(self.offsets, idx, side='right') - 1
        fn = self._native() if self.use_native else None
        if fn is not None:
            fn(self._ptrs, self.counts, self._row_bytes, torch.from_numpy(shard.astype(np.int64)),
               torch.from_numpy((idx - self.offsets[shard]).astype(np.int64)), out, self.gather_threads)
            return
        dst = out.numpy()
        for s in np.unique(shard):
            sel = np.nonzero(shard == s)[0]
            local = idx[sel] - self.offsets[s]
            order = np.argsort(local, kind='stable')          # ascending file offsets: sequential reads
            dst[sel[order]] = self.images[s][local[order]]

    def __iter__(self):
        idx = self.indices()
        B = self.batch_size
        nb = self.n_batches
        S = self.size
        q: 'queue.Queue' = queue.Queue(maxsize=self.prefetch)
        stop = threading.Event()
        pin = self.pin
        # pinned allocations are made against the calling thread's current device; a new thread
        # starts on device 0, which would create a stray context there from every rank
        device = torch.cuda.current_device() if (pin and torch.cuda.is_available()) else None

        def work():
            try:
                if device is not None:
                    torch.cuda.set_device(device)
                for b in range(nb):
                    if stop.is_set():
                        return
                    sel = idx[b * B:(b + 1) * B]
                    # a fresh pinned tensor per batch: the consumer's non-blocking H2D copy may still
                    # be queued when later batches are produced; torch's caching host allocator only
                    # recycles a pinned block once the copies that read it have completed
                    buf = torch.empty(len(sel), S, S, 3, dtype=torch.uint8, pin_memory=pin)
                    self._gather(sel, buf)
                    q.put((buf, torch.from_numpy(self.labels[sel])))
                q.put(None)
            except Exception as e:                          # surfaced to the consumer
                q.put(e)

        t = threading.Thread(target=work, name='shard-loader', daemon=True)
        t.start()
        try:
            while True:
                item = q.get()
                if item is None:
                    break
                if isinstance(item, Exception):
                    raise item
                yield item
        finally:
            stop.set()
            while not q.empty():                            # unblock a producer stuck in put()
                try:
                    q.get_nowait()
                except queue.Empty:
                    break
            t.join()                    # it puts at most one more batch into the drained queue, then sees stop

# --------------------------------------------------------------------------- #
# GPU-side augmentation
# --------------------------------------------------------------------------- #
# TrivialAugmentWide (Mueller & Hutter 2021) as torchvision.transforms.v2.TrivialAugmentWide draws it:
# one op uniform over these 14, one of 31 magnitude bins, a random sign for the signed ops
TA_WIDE_OPS = ('Identity', 'ShearX', 'ShearY', 'TranslateX', 'TranslateY', 'Rotate', 'Brightness', 'Color',
               'Contrast', 'Sharpness', 'Posterize', 'Solarize', 'AutoContrast', 'Equalize')
TA_WIDE_SIGNED = frozenset(TA_WIDE_OPS[1:10])
TA_WIDE_BINS = 31
GEOMETRIC_OPS = frozenset(TA_WIDE_OPS[1:6])
# every op the augment kernel applies (its op ids): AutoAugment's ImageNet policy adds Invert
AUGMENT_OPS = TA_WIDE_OPS + ('Invert',)
# RandAugment (Cubuk et al. 2020) as torchvision.transforms.v2.RandAugment draws it: num_ops ops, each
# uniform over TA_WIDE_OPS, at bin `magnitude` of 31, a random sign for the signed ops
RA_BINS = 31
RA_MAX_OPS = 4
# AutoAugment's ImageNet policy (Cubuk et al. 2019) as torchvision.transforms.v2.AutoAugment holds it:
# one of these 25 sub-policies uniformly, each (op, probability, bin of 10) applied with its probability
AA_BINS = 10
AUTO_AUGMENT_IMAGENET = (
    (('Posterize', 0.4, 8), ('Rotate', 0.6, 9)),
    (('Solarize', 0.6, 5), ('AutoContrast', 0.6, None)),
    (('Equalize', 0.8, None), ('Equalize', 0.6, None)),
    (('Posterize', 0.6, 7), ('Posterize', 0.6, 6)),
    (('Equalize', 0.4, None), ('Solarize', 0.2, 4)),
    (('Equalize', 0.4, None), ('Rotate', 0.8, 8)),
    (('Solarize', 0.6, 3), ('Equalize', 0.6, None)),
    (('Posterize', 0.8, 5), ('Equalize', 1.0, None)),
    (('Rotate', 0.2, 3), ('Solarize', 0.6, 8)),
    (('Equalize', 0.6, None), ('Posterize', 0.4, 6)),
    (('Rotate', 0.8, 8), ('Color', 0.4, 0)),
    (('Rotate', 0.4, 9), ('Equalize', 0.6, None)),
    (('Equalize', 0.0, None), ('Equalize', 0.8, None)),
    (('Invert', 0.6, None), ('Equalize', 1.0, None)),
    (('Color', 0.6, 4), ('Contrast', 1.0, 8)),
    (('Rotate', 0.8, 8), ('Color', 1.0, 2)),
    (('Color', 0.8, 8), ('Solarize', 0.8, 7)),
    (('Sharpness', 0.4, 7), ('Invert', 0.6, None)),
    (('ShearX', 0.6, 5), ('Equalize', 1.0, None)),
    (('Color', 0.4, 0), ('Equalize', 0.6, None)),
    (('Equalize', 0.4, None), ('Solarize', 0.2, 4)),
    (('Solarize', 0.6, 5), ('AutoContrast', 0.6, None)),
    (('Invert', 0.6, None), ('Equalize', 1.0, None)),
    (('Color', 0.6, 4), ('Contrast', 1.0, 8)),
    (('Equalize', 0.8, None), ('Equalize', 0.6, None)),
)
ERASE_SCALE = (0.02, 0.33)
ERASE_RATIO = (0.3, 3.3)
ERASE_ATTEMPTS = 10
# dynamic shared memory one CTA may use on sm_90 (227 KB); the augment kernel keeps the whole
# out x out x 3 uint8 crop there plus its per-op tables
SM90_SMEM_PER_CTA = 232448
# the augment kernel's per-image rows: one op (TrivialAugment, erasing only), or a chain of up to
# AUGMENT_MAX_OPS ops (RandAugment, AutoAugment); op k >= 2 at AUGMENT_CHAIN_COL + 9 (k - 2)
AUGMENT_ROW_ONE_OP = 24
AUGMENT_ROW = 48
AUGMENT_MAX_OPS = 4
AUGMENT_CHAIN_COL = 19


def ta_wide_magnitudes(num_bins: int = TA_WIDE_BINS) -> dict:
    """op name -> magnitude per bin (fp32 values as torchvision's v2 tables hold them; None for
    the ops without a magnitude)."""
    lin = lambda hi: torch.linspace(0.0, hi, num_bins)  # noqa: E731
    return {
        'Identity': None, 'ShearX': lin(0.99), 'ShearY': lin(0.99), 'TranslateX': lin(32.0),
        'TranslateY': lin(32.0), 'Rotate': lin(135.0), 'Brightness': lin(0.99), 'Color': lin(0.99),
        'Contrast': lin(0.99), 'Sharpness': lin(0.99),
        'Posterize': (8 - (torch.arange(num_bins) / ((num_bins - 1) / 6))).round().int(),
        'Solarize': torch.linspace(1.0, 0.0, num_bins), 'AutoContrast': None, 'Equalize': None,
    }


def policy_magnitudes(num_bins: int, size: int) -> dict:
    """op name (every op of :data:`AUGMENT_OPS`) -> magnitude per bin of RandAugment's and
    AutoAugment's shared space for ``size x size`` images (fp32 values as torchvision's v2 tables
    hold them; None for the ops without a magnitude).  RandAugment takes 31 bins, AutoAugment 10."""
    lin = lambda hi: torch.linspace(0.0, hi, num_bins)  # noqa: E731
    return {
        'Identity': None, 'ShearX': lin(0.3), 'ShearY': lin(0.3), 'TranslateX': lin(150.0 / 331.0 * size),
        'TranslateY': lin(150.0 / 331.0 * size), 'Rotate': lin(30.0), 'Brightness': lin(0.9), 'Color': lin(0.9),
        'Contrast': lin(0.9), 'Sharpness': lin(0.9),
        'Posterize': (8 - (torch.arange(num_bins) / ((num_bins - 1) / 4))).round().int(),
        'Solarize': torch.linspace(1.0, 0.0, num_bins), 'AutoContrast': None, 'Equalize': None, 'Invert': None,
    }


def augment_smem_bytes(out: int) -> int:
    """Shared memory of one augment-kernel CTA for ``out x out`` output images (the kernel's
    ``aug_smem_bytes``)."""
    return (3 * out * out + 15) // 16 * 16 + (3 * 256 + 16) * 4


class AugmentParams(NamedTuple):
    """Per-sample parameters of one training batch (CPU tensors, ``n`` rows each).

    ``cx, cy, w, h, flip``: the RandomResizedCrop box as fractions of the stored image and the flip
    sign (fp32, :meth:`GpuAugment.sample_boxes`); ``op``: int64 index into :data:`AUGMENT_OPS`,
    ``[n]`` for one op per sample or ``[n, K]`` for a chain of ``K <= 4`` ops applied left to right;
    ``magnitude``: float64, shaped as ``op``, the signed magnitude torchvision would pass to the op (0
    for the ops without one); ``erase``: int64 ``[n, 4]`` box ``(top, left, height, width)`` in output
    pixels, height 0 = no box."""
    cx: torch.Tensor
    cy: torch.Tensor
    w: torch.Tensor
    h: torch.Tensor
    flip: torch.Tensor
    op: torch.Tensor
    magnitude: torch.Tensor
    erase: torch.Tensor


def inverse_affine_matrix(center, angle: float, translate, shear) -> List[float]:
    """Inverse of ``T C R(angle) Sh(shear) C^-1`` (scale 1) as the 2 x 3 row-major list that maps
    output pixels to input pixels, in coordinates relative to the image centre: the matrix
    torchvision's ``affine`` / ``rotate`` sample through.  Angles in degrees."""
    rot = math.radians(angle)
    sx, sy = math.radians(shear[0]), math.radians(shear[1])
    cx, cy = center
    tx, ty = translate
    # R S the forward rotation-shear block [[a, b], [c, d]] (determinant 1)
    a = math.cos(rot - sy) / math.cos(sy)
    b = -(a * math.tan(sx) + math.sin(rot))
    c = math.sin(rot - sy) / math.cos(sy)
    d = math.cos(rot) - c * math.tan(sx)
    m = [d, -b, 0.0, -c, a, 0.0]
    m[2] += cx - m[0] * (cx + tx) - m[1] * (cy + ty)
    m[5] += cy - m[3] * (cx + tx) - m[4] * (cy + ty)
    return m


def ta_wide_matrix(op: str, magnitude: float, size: int) -> List[float]:
    """The inverse affine matrix of geometric op ``op`` at ``magnitude`` on a ``size x size``
    image, with the arguments TrivialAugmentWide passes (shears about the top-left corner,
    translations truncated to whole pixels, rotations about the centre)."""
    if op in ('ShearX', 'ShearY'):
        deg = math.degrees(math.atan(magnitude))
        shear = [deg, 0.0] if op == 'ShearX' else [0.0, deg]
        return inverse_affine_matrix([-size * 0.5, -size * 0.5], 0.0, [0.0, 0.0], shear)
    if op in ('TranslateX', 'TranslateY'):
        t = [float(int(magnitude)), 0.0] if op == 'TranslateX' else [0.0, float(int(magnitude))]
        return inverse_affine_matrix([0.0, 0.0], 0.0, t, [0.0, 0.0])
    if op == 'Rotate':
        return inverse_affine_matrix([0.0, 0.0], -(magnitude % 360), [0.0, 0.0], [0.0, 0.0])
    raise ValueError('%s is not a geometric op' % op)


@functools.lru_cache(maxsize=4096)
def _geometric_columns(op: str, magnitude: float, size: int) -> np.ndarray:
    """a geometric op's six row entries: torchvision's _affine_grid rescaling theta^T / [w / 2, h / 2]
    of :func:`ta_wide_matrix`, in fp32.  Cached: a policy draws few distinct (op, magnitude) pairs."""
    m = np.asarray(ta_wide_matrix(op, magnitude, size), dtype=np.float32)
    return m / np.float32(0.5 * size)


class GpuAugment(object):
    """uint8 ``[B, S, S, 3]`` -> normalised ``[B, 3, out, out]`` (channels-last memory format).

    training: ``RandomResizedCrop(out, scale, ratio)`` + horizontal flip, all samples in ONE
    ``grid_sample`` (the crop box of sample i is the affine map ``theta_i``; flip negates its x
    scale); evaluation: centre crop of ``out / eval_ratio`` resized to ``out`` (the reference's
    ``Resize(256) + CenterCrop(224)`` when the shards were stored at 256).

    ``auto_augment`` adds an augmentation policy on the uint8 crop: ``'ta_wide'`` TrivialAugmentWide,
    ``'ra'`` RandAugment (``ra_num_ops`` ops at bin ``ra_magnitude`` of 31, torchvision v2 semantics),
    ``'imagenet'`` AutoAugment with the ImageNet policy; ``random_erase=p`` adds
    ``RandomErasing(p, value=0)`` after the normalisation, in torchvision's recipe order.  With
    either on, a training batch on the GPU is ONE launch of the sm_90a augment kernel
    (``csrc/augment_kernels.cu``): the crop rounded to uint8 as torchvision's uint8 pipeline
    rounds it, the op or chain of ops (each on the uint8 result of the one before), the
    normalisation and the erase box.  Their draws come from a second
    generator, so the crop boxes and flips of a seed do not depend on these options.  CPU batches
    take the reference composition (``ops.oracle.reference_augment``); evaluation never augments."""

    def __init__(self, out_size: int = 224, scale=(0.08, 1.0), ratio=(3.0 / 4.0, 4.0 / 3.0),
                 mean=IMAGENET_MEAN, std=IMAGENET_STD, dtype=torch.float32, eval_ratio: float = 0.875,
                 seed: int = 0, channels_last: bool = True, auto_augment: Optional[str] = None,
                 random_erase: float = 0.0, ra_num_ops: int = 2, ra_magnitude: int = 9):
        self.out = int(out_size)
        self.scale, self.ratio = scale, ratio
        self.mean, self.std = tuple(mean), tuple(std)
        self.dtype = dtype
        self.eval_ratio = float(eval_ratio)
        self.channels_last = channels_last
        self._gen = torch.Generator().manual_seed(int(seed))
        self._consts = {}
        if auto_augment not in (None, 'ta_wide', 'ra', 'imagenet'):
            raise ValueError("auto_augment must be None, 'ta_wide', 'ra' or 'imagenet', got %r" % (auto_augment,))
        if not 0.0 <= float(random_erase) <= 1.0:
            raise ValueError('random_erase must be in [0, 1], got %r' % (random_erase,))
        for name, v, hi in (('ra_num_ops', ra_num_ops, RA_MAX_OPS), ('ra_magnitude', ra_magnitude, RA_BINS - 1)):
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or not 0 <= v <= hi:
                raise ValueError('%s must be an integer in [0, %d], got %r' % (name, hi, v))
        self.auto_augment = auto_augment
        self.random_erase = float(random_erase)
        self.ra_num_ops, self.ra_magnitude = int(ra_num_ops), int(ra_magnitude)
        if self.augments and augment_smem_bytes(self.out) > SM90_SMEM_PER_CTA:
            raise ValueError('out_size %d needs %d bytes of shared memory per image with auto_augment / '
                             'random_erase; an sm_90 CTA has %d' % (self.out, augment_smem_bytes(self.out),
                                                                   SM90_SMEM_PER_CTA))
        self._aug_gen = torch.Generator().manual_seed(int(seed) * 1000003 + 0x7A5)
        tables = ta_wide_magnitudes()
        self._table = torch.stack([torch.zeros(TA_WIDE_BINS, dtype=torch.float64) if tables[k] is None
                                   else tables[k].double() for k in TA_WIDE_OPS])
        self._signed = torch.tensor([k in TA_WIDE_SIGNED for k in AUGMENT_OPS])
        # RandAugment: each op's magnitude at the fixed bin; AutoAugment: per sub-policy and slot the
        # op id, its probability (fp32, as torchvision compares it) and its magnitude
        space = policy_magnitudes(RA_BINS, self.out)
        self._ra_mag = torch.tensor([0.0 if space[k] is None else float(space[k][self.ra_magnitude])
                                     for k in AUGMENT_OPS], dtype=torch.float64)
        space = policy_magnitudes(AA_BINS, self.out)
        self._aa_op = torch.tensor([[AUGMENT_OPS.index(o) for o, _, _ in sub] for sub in AUTO_AUGMENT_IMAGENET])
        self._aa_prob = torch.tensor([[p for _, p, _ in sub] for sub in AUTO_AUGMENT_IMAGENET], dtype=torch.float32)
        self._aa_mag = torch.tensor([[0.0 if b is None else float(space[o][b]) for o, _, b in sub]
                                     for sub in AUTO_AUGMENT_IMAGENET], dtype=torch.float64)
        self._ring = None
        self._events = [None] * RING_SLOTS
        self._slot = 0

    @property
    def augments(self) -> bool:
        """True when training batches take the augment kernel (a policy or erasing on)."""
        return self.auto_augment is not None or self.random_erase > 0

    def _norm(self, device):
        key = str(device)
        if key not in self._consts:
            mean = torch.tensor(self.mean, dtype=torch.float32, device=device).view(1, 3, 1, 1) * 255.0
            inv = 1.0 / (torch.tensor(self.std, dtype=torch.float32, device=device).view(1, 3, 1, 1) * 255.0)
            self._consts[key] = (mean, inv)
        return self._consts[key]

    def sample_boxes(self, n: int):
        """RandomResizedCrop parameters as fractions of the stored square image:
        (cx, cy, w, h) in [0, 1], flip in {-1, +1} (host-side RNG: a few hundred bytes per batch).
        Area ~ U(scale), log-ratio ~ U(log ratio) as in torchvision; a box that does not fit is
        clamped to the image instead of being re-drawn (torchvision retries 10 times, then falls back
        to a centre crop), and the crops come from the stored centre square, not the full frame."""
        g = self._gen
        area = torch.empty(n).uniform_(self.scale[0], self.scale[1], generator=g)
        logr = torch.empty(n).uniform_(math.log(self.ratio[0]), math.log(self.ratio[1]), generator=g)
        r = torch.exp(logr)
        w = torch.sqrt(area * r).clamp(max=1.0)
        h = torch.sqrt(area / r).clamp(max=1.0)
        cx = w / 2 + torch.rand(n, generator=g) * (1.0 - w)
        cy = h / 2 + torch.rand(n, generator=g) * (1.0 - h)
        flip = torch.where(torch.rand(n, generator=g) < 0.5, -torch.ones(n), torch.ones(n))
        return cx, cy, w, h, flip

    @staticmethod
    def crop_theta(cx, cy, w, h, flip) -> torch.Tensor:
        """fp32 ``[n, 2, 3]`` affine maps of the crop boxes (``F.affine_grid`` convention)."""
        theta = torch.zeros(len(cx), 2, 3)
        theta[:, 0, 0] = w * flip          # output x in [-1, 1] -> input x: centre + half-width * x
        theta[:, 0, 2] = 2 * cx - 1
        theta[:, 1, 1] = h
        theta[:, 1, 2] = 2 * cy - 1
        return theta

    def sample_params(self, n: int) -> AugmentParams:
        """The next training batch's :class:`AugmentParams`: crop boxes and flips from
        :meth:`sample_boxes`, then, from the second generator, per sample, the policy's ops and
        RandomErasing's box.  TrivialAugmentWide (``op`` ``[n]``): the op (uniform over
        :data:`TA_WIDE_OPS`), bin (uniform over 31) and sign (negative with probability 1/2, signed
        ops only).  RandAugment (``op`` ``[n, ra_num_ops]``): each op uniform over :data:`TA_WIDE_OPS`
        at bin ``ra_magnitude``, then each sign.  AutoAugment (``op`` ``[n, 2]``): the sub-policy
        (uniform over 25), whether each of its ops applies (Identity otherwise), then each sign.
        RandomErasing: with probability ``p``, up to
        10 attempts of area fraction U(0.02, 0.33) and log aspect ratio U(log 0.3, log 3.3),
        ``h = round(sqrt(area r))``, ``w = round(sqrt(area / r))``; the first box strictly inside
        the image is placed at a uniform integer position, none if no attempt fits."""
        cx, cy, w, h, flip = self.sample_boxes(n)
        g = self._aug_gen
        op = torch.zeros(n, dtype=torch.int64)
        magnitude = torch.zeros(n, dtype=torch.float64)
        if self.auto_augment == 'ta_wide':
            op = torch.randint(len(TA_WIDE_OPS), (n,), generator=g)
            bins = torch.randint(TA_WIDE_BINS, (n,), generator=g)
            negate = torch.rand(n, generator=g) <= 0.5
            sign = torch.where(negate & self._signed[op], -1.0, 1.0).double()
            magnitude = self._table[op, bins] * sign
        elif self.auto_augment == 'ra':
            k = self.ra_num_ops
            op = torch.randint(len(TA_WIDE_OPS), (n, k), generator=g)
            negate = torch.rand(n, k, generator=g) <= 0.5
            sign = torch.where(negate & self._signed[op], -1.0, 1.0).double()
            magnitude = self._ra_mag[op] * sign
        elif self.auto_augment == 'imagenet':
            sub = torch.randint(len(AUTO_AUGMENT_IMAGENET), (n,), generator=g)
            on = torch.rand(n, 2, generator=g) <= self._aa_prob[sub]
            negate = torch.rand(n, 2, generator=g) <= 0.5
            op = torch.where(on, self._aa_op[sub], 0)
            sign = torch.where(negate & self._signed[op], -1.0, 1.0).double()
            magnitude = torch.where(on, self._aa_mag[sub], 0.0) * sign
        erase = torch.zeros(n, 4, dtype=torch.int64)
        if self.random_erase > 0:
            size = self.out
            hit = torch.rand(n, generator=g) < self.random_erase
            area = size * size * torch.empty(n, ERASE_ATTEMPTS, dtype=torch.float64).uniform_(
                ERASE_SCALE[0], ERASE_SCALE[1], generator=g)
            logr = torch.empty(n, ERASE_ATTEMPTS, dtype=torch.float64).uniform_(
                math.log(ERASE_RATIO[0]), math.log(ERASE_RATIO[1]), generator=g)
            pos = torch.rand(n, 2, dtype=torch.float64, generator=g).numpy()
            # (numpy for the elementwise math: torch's intra-op pool costs more than these few
            # thousand elements)
            r = np.exp(logr.numpy())
            area = area.numpy()
            eh = np.round(np.sqrt(area * r)).astype(np.int64)
            ew = np.round(np.sqrt(area / r)).astype(np.int64)
            fits = (eh < size) & (ew < size)
            first = fits.argmax(1)[:, None]                               # first attempt that fits
            bh, bw = np.take_along_axis(eh, first, 1)[:, 0], np.take_along_axis(ew, first, 1)[:, 0]
            on = hit.numpy() & fits.any(1)
            top = np.minimum((pos[:, 0] * (size - bh + 1)).astype(np.int64), size - bh)
            left = np.minimum((pos[:, 1] * (size - bw + 1)).astype(np.int64), size - bw)
            erase = torch.from_numpy(np.where(on[:, None], np.stack([top, left, bh, bw], 1), 0))
        return AugmentParams(cx, cy, w, h, flip, op, magnitude, erase)

    def kernel_rows(self, params: AugmentParams, S: int) -> np.ndarray:
        """fp32 ``[n, AUGMENT_ROW_ONE_OP]`` for one op per sample (``params.op`` ``[n]``), else
        ``[n, AUGMENT_ROW]`` with op k of the chain at its columns and Identity after the last: the
        augment kernel's per-image rows for ``params`` (layout in ``csrc/augment_kernels.cu``).  Every
        op scalar is rounded to fp32 the way torch rounds a Python scalar against an fp32 tensor."""
        op, mag = params.op.numpy(), params.magnitude.numpy()
        chain = op.ndim == 2
        if not chain:
            op, mag = op[:, None], mag[:, None]
        n, k = op.shape
        if k > AUGMENT_MAX_OPS:
            raise ValueError('the augment kernel applies at most %d ops per image, got %d' % (AUGMENT_MAX_OPS, k))
        rows = np.zeros((n, AUGMENT_ROW if chain else AUGMENT_ROW_ONE_OP), dtype=np.float32)
        rows[:, 0:6] = self.crop_theta(params.cx, params.cy, params.w, params.h, params.flip).reshape(n, 6).numpy()
        for j in range(k):
            col = 6 if j == 0 else AUGMENT_CHAIN_COL + 9 * (j - 1)
            self._op_columns(rows[:, col:col + 9], op[:, j], mag[:, j])
        e = params.erase.numpy()
        rows[:, 15], rows[:, 16], rows[:, 17], rows[:, 18] = e[:, 0], e[:, 0] + e[:, 2], e[:, 1], e[:, 1] + e[:, 3]
        return rows

    def _op_columns(self, cols: np.ndarray, op: np.ndarray, mag: np.ndarray):
        """one op's 9 row columns: id, two scalars, the geometric ops' six matrix entries"""
        out = self.out
        cols[:, 0] = op
        is_op = lambda *names: np.isin(op, [AUGMENT_OPS.index(k) for k in names])  # noqa: E731
        sel = is_op('Brightness', 'Color', 'Contrast')
        cols[sel, 1] = 1.0 + mag[sel]
        sel = is_op('Color', 'Contrast', 'Sharpness')
        cols[sel, 2] = 1.0 - (1.0 + mag[sel])
        sel = is_op('Posterize')
        bits = mag[sel].astype(np.int64)
        cols[sel, 1] = np.where(bits >= 8, 255, ((1 << bits) - 1) << np.maximum(8 - bits, 0))
        sel = is_op('Solarize')
        cols[sel, 1] = 255.0 * mag[sel]
        for i in np.nonzero(is_op(*GEOMETRIC_OPS))[0]:
            cols[i, 3:9] = _geometric_columns(AUGMENT_OPS[op[i]], float(mag[i]), out)

    def _stage_rows(self, rows: np.ndarray, device) -> torch.Tensor:
        """``rows`` -> a fresh device tensor through ONE non-blocking H2D copy from a slot of a
        pinned ring; a slot is rewritten only after the copy that last read it has executed."""
        n, width = rows.shape
        if self._ring is None or self._ring.shape[1] < n * width:
            for ev in self._events:
                if ev is not None:
                    ev.synchronize()
            self._ring = torch.empty(RING_SLOTS, n * width, dtype=torch.float32, pin_memory=True)
            self._events = [None] * RING_SLOTS
        slot = self._slot
        self._slot = (slot + 1) % RING_SLOTS
        if self._events[slot] is not None:
            self._events[slot].synchronize()
        host = self._ring[slot, :n * width].view(n, width)
        host.numpy()[:] = rows
        dev_rows = torch.empty(n, width, dtype=torch.float32, device=device)
        dev_rows.copy_(host, non_blocking=True)
        ev = self._events[slot] = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(device))
        return dev_rows

    def apply(self, batch_u8: torch.Tensor, params: AugmentParams) -> torch.Tensor:
        """The training output of ``batch_u8`` for explicit per-sample ``params``: crop, round to
        uint8, the op or chain of ops, normalise, erase.  CUDA: one launch of the sm_90a augment
        kernel (a missing extension is an error) and no host synchronisation; CPU: the reference
        composition ``ops.oracle.reference_augment``."""
        assert batch_u8.dtype == torch.uint8 and batch_u8.dim() == 4 and batch_u8.shape[-1] == 3
        n, S = batch_u8.shape[0], batch_u8.shape[1]
        if augment_smem_bytes(self.out) > SM90_SMEM_PER_CTA:
            raise ValueError('out_size %d is too large for the augment kernel' % self.out)
        mean, inv = self._norm('cpu')
        if not batch_u8.is_cuda:
            from ..ops.oracle import reference_augment
            theta = self.crop_theta(params.cx, params.cy, params.w, params.h, params.flip)
            y = reference_augment(batch_u8, theta, params.op, params.magnitude, params.erase, self.out, mean, inv)
        else:
            from ..ops import native
            C = native.load()
            y = torch.empty(n, 3, self.out, self.out, dtype=self.dtype, device=batch_u8.device,
                            memory_format=torch.channels_last)
            rows = self._stage_rows(self.kernel_rows(params, S), batch_u8.device)
            C.gpu_augment(batch_u8.contiguous(), rows, y, mean.view(-1).tolist(), inv.view(-1).tolist())
        if not self.channels_last:
            y = y.contiguous()
        return y.to(self.dtype)

    def __call__(self, batch_u8: torch.Tensor, train: bool = True) -> torch.Tensor:
        assert batch_u8.dtype == torch.uint8 and batch_u8.dim() == 4 and batch_u8.shape[-1] == 3
        if train and self.augments:
            return self.apply(batch_u8, self.sample_params(batch_u8.shape[0]))
        dev = batch_u8.device
        n = batch_u8.shape[0]
        x = batch_u8.permute(0, 3, 1, 2).float()            # NCHW view of the NHWC bytes (= channels-last)
        if train:
            cx, cy, w, h, flip = self.sample_boxes(n)
        else:
            cx = cy = torch.full((n,), 0.5)
            w = h = torch.full((n,), self.eval_ratio)
            flip = torch.ones(n)
        theta = self.crop_theta(cx, cy, w, h, flip)
        theta = theta.to(dev, non_blocking=True)
        grid = F.affine_grid(theta, (n, 3, self.out, self.out), align_corners=False)
        y = F.grid_sample(x, grid, mode='bilinear', padding_mode='border', align_corners=False)
        mean, inv = self._norm(dev)
        y = (y - mean) * inv
        if self.channels_last:
            y = y.contiguous(memory_format=torch.channels_last)
        return y.to(self.dtype)
