"""Synthetic stand-in for the reference's TFRecord queues (source_segmenter.py:331-355,
adversarial.py:607-631): 256x256x3 z-scored slices + a 256x256 integer label map per sample
(README.md:49-64 schema).  The real MMWHS records are not available offline (SURVEY 2.1 row 10);
the TFRecord reader itself is a "next" row (SURVEY 8f #2).

Batches are produced in pinned host memory, like a feed_dict, so the host->device copy is part of the
step exactly as in the reference (source_segmenter.py:484).
"""
import numpy as np
import torch


def label_maps(B, seed, size=256, num_cls=5):
    """nested ellipses: classes 1..num_cls-1 on background 0, centres / radii jittered by `seed`"""
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:size, 0:size].astype(np.float32)
    out = np.zeros((B, size, size), np.int64)
    radii = np.linspace(0.39 * size, 0.1 * size, num_cls - 1)
    for b in range(B):
        cy, cx = size / 2 + rng.uniform(-20, 20), size / 2 + rng.uniform(-20, 20)
        for c, rad in zip(range(1, num_cls), radii):
            ry, rx = rad * rng.uniform(0.8, 1.0), rad * rng.uniform(0.8, 1.0)
            out[b][((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1.0] = c
    return out


class SyntheticSource:
    """yields (images [B,256,256,3] fp32, labels [B,256,256] int64) as pinned host tensors"""

    def __init__(self, batch_size, seed=1234, shift=0.0, scale=1.0, size=256, num_cls=5, pool=4, contrast=0.0):
        """contrast > 0 adds a per-class intensity ((class - (num_cls-1)/2) * contrast / 2) to the noise, so that the labels can be
        learned from the images (the held-out Dice gate trains on this); 0 = pure z-scored noise (the throughput workloads)"""
        self.B, self.size, self.num_cls = batch_size, size, num_cls
        g = torch.Generator().manual_seed(seed)
        self.pool = []
        for i in range(pool):
            x = torch.randn(batch_size, size, size, 3, generator=g) * scale + shift
            y = torch.from_numpy(label_maps(batch_size, seed + 99 + i, size, num_cls))
            if contrast:
                x = x + ((y.to(torch.float32) - (num_cls - 1) / 2.0) * (contrast / 2.0)).unsqueeze(-1)
            if torch.cuda.is_available():
                x, y = x.pin_memory(), y.pin_memory()
            self.pool.append((x, y))
        self.i = 0

    def next(self):
        item = self.pool[self.i % len(self.pool)]
        self.i += 1
        return item


class VolumeSource:
    """Augmented training slices drawn straight from MMWHS volumes on the device (preprocess.py): next() returns (images
    [B,256,256,3] fp32, labels [B,256,256] int64) like TFRecordSource.next(), but already on the device, so the trainers'
    to_device is a no-op.  Every subject of `pairs` ((image_path, label_path) NIfTI pairs) is prepared once and its sub-volume
    uploaded; each next() draws per sample a subject, a slice and (augment=True) an augmentation from
    np.random.RandomState(seed), and resamples the whole batch in one pnp_resample_planes launch.  A batch stays valid until
    the next-but-one call (two alternating output buffers, like TFRecordSource's)."""

    def __init__(self, pairs, batch_size, seed, augment=True):
        from . import preprocess
        from . import runtime as rt
        pairs = list(pairs)
        if not pairs:
            raise ValueError("empty volume list")
        self.B, self.augment = batch_size, augment
        self.subjects = [preprocess.Subject(im, lb) for im, lb in pairs]
        vol, cls, self.offsets = preprocess.stack(self.subjects)
        dev = rt.device()
        self.vol, self.cls = torch.from_numpy(vol).to(dev), torch.from_numpy(cls).to(dev)
        self.rng = np.random.RandomState(seed)
        S = preprocess.SIZE
        self._out = [(torch.empty(batch_size, S, S, 3, dtype=torch.float32, device=dev),
                      torch.empty(batch_size, S, S, dtype=torch.int64, device=dev)) for _ in range(2)]
        self._mats = [torch.empty(batch_size, 3, 3, 3, dtype=torch.float32, device=dev) for _ in range(2)]
        # the matrices go up from pinned memory without stalling the stream; an event says when a host buffer is free again
        self._host = [torch.empty(batch_size, 3, 3, 3, dtype=torch.float32, pin_memory=True) for _ in range(2)]
        self._copied = [None, None]
        self._flip = 0

    def draw_matrices(self):
        """fp32 [B, 3, 3, 3]: the matrices of the channels j - 1, j, j + 1 of B samples drawn from the generator"""
        mats = []
        for _ in range(self.B):
            s = int(self.rng.randint(len(self.subjects)))
            j, T = self.subjects[s].draw(self.rng, self.augment)
            mats.append(self.subjects[s].matrices((j - 1, j, j + 1), T, self.offsets[s]))
        return np.stack(mats)

    def next(self):
        from .functional import resample_planes
        i = self._flip
        self._flip ^= 1
        x, y = self._out[i]
        if self._copied[i] is not None:
            self._copied[i].synchronize()
        self._host[i].numpy()[...] = self.draw_matrices()
        self._mats[i].copy_(self._host[i], non_blocking=True)
        self._copied[i] = torch.cuda.Event()
        self._copied[i].record()
        resample_planes(self.vol, self.cls, self._mats[i], x.shape[1], x.shape[2], True, 1, x, y)
        return x, y


def pick_source(given, files, batch_size, seed, num_cls, shift=0.0, scale=1.0):
    """a trainer's input stream: `given` if there is one, else a TFRecordSource over `files` (the reference's lists/*_list of
    single-example TFRecord files, README.md:49-64), else a SyntheticSource with this shift / scale / num_cls"""
    if given is not None:
        return given
    if files:
        from .tfrecord import TFRecordSource
        return TFRecordSource(files, batch_size, seed=seed)
    return SyntheticSource(batch_size, seed=seed, shift=shift, scale=scale, num_cls=num_cls)


def to_device(x, dev):
    return x.to(dev, non_blocking=True)
