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

import json
import math
import os
import queue
import threading
from typing import List, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


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


# --------------------------------------------------------------------------- #
# GPU-side augmentation
# --------------------------------------------------------------------------- #
class GpuAugment(object):
    """uint8 ``[B, S, S, 3]`` -> normalised ``[B, 3, out, out]`` (channels-last memory format).

    training: ``RandomResizedCrop(out, scale, ratio)`` + horizontal flip, all samples in ONE
    ``grid_sample`` (the crop box of sample i is the affine map ``theta_i``; flip negates its x
    scale); evaluation: centre crop of ``out / eval_ratio`` resized to ``out`` (the reference's
    ``Resize(256) + CenterCrop(224)`` when the shards were stored at 256)."""

    def __init__(self, out_size: int = 224, scale=(0.08, 1.0), ratio=(3.0 / 4.0, 4.0 / 3.0),
                 mean=IMAGENET_MEAN, std=IMAGENET_STD, dtype=torch.float32, eval_ratio: float = 0.875,
                 seed: int = 0, channels_last: bool = True):
        self.out = int(out_size)
        self.scale, self.ratio = scale, ratio
        self.mean, self.std = tuple(mean), tuple(std)
        self.dtype = dtype
        self.eval_ratio = float(eval_ratio)
        self.channels_last = channels_last
        self._gen = torch.Generator().manual_seed(int(seed))
        self._consts = {}

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

    def __call__(self, batch_u8: torch.Tensor, train: bool = True) -> torch.Tensor:
        assert batch_u8.dtype == torch.uint8 and batch_u8.dim() == 4 and batch_u8.shape[-1] == 3
        dev = batch_u8.device
        n = batch_u8.shape[0]
        x = batch_u8.permute(0, 3, 1, 2).float()            # NCHW view of the NHWC bytes (= channels-last)
        if train:
            cx, cy, w, h, flip = self.sample_boxes(n)
        else:
            cx = cy = torch.full((n,), 0.5)
            w = h = torch.full((n,), self.eval_ratio)
            flip = torch.ones(n)
        theta = torch.zeros(n, 2, 3)
        theta[:, 0, 0] = w * flip          # output x in [-1, 1] -> input x: centre + half-width * x
        theta[:, 0, 2] = 2 * cx - 1
        theta[:, 1, 1] = h
        theta[:, 1, 2] = 2 * cy - 1
        theta = theta.to(dev, non_blocking=True)
        grid = F.affine_grid(theta, (n, 3, self.out, self.out), align_corners=False)
        y = F.grid_sample(x, grid, mode='bilinear', padding_mode='border', align_corners=False)
        mean, inv = self._norm(dev)
        y = (y - mean) * inv
        if self.channels_last:
            y = y.contiguous(memory_format=torch.channels_last)
        return y.to(self.dtype)
