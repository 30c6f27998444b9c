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
    the next-but-one call (two alternating output buffers, like TFRecordSource's).

    Opt-in augmentations on the device (preprocess.py; both need augment=True):
    * elastic=True: a displacement field [B, 2, 256, 256] per batch (pnp_smooth_noise_field, Philox stream
      field_stream(ELASTIC_STREAM_TAG, t)); the subjects are prepared with the reach ELASTIC_REACH_PX;
    * intensity=True: a bias field [B, 256, 256] (stream field_stream(BIAS_STREAM_TAG, t)) and per sample a contrast and an
      offset drawn from the generator after that sample's slice and transform.
    t counts the batches drawn (from 0), so the fields are a function of `seed` alone.  Each field and (a, b) live in buffers of their own
    for each of the two output buffers; the batch is one pnp_resample_planes_aug launch after the field calls.  With both off
    nothing extra is drawn or launched, and the batches are those of a source built without the flags."""

    def __init__(self, pairs, batch_size, seed, augment=True, elastic=False, intensity=False):
        from . import preprocess
        from . import runtime as rt
        pairs = list(pairs)
        if not pairs:
            raise ValueError("empty volume list")
        if (elastic or intensity) and not augment:
            raise ValueError("elastic / intensity augmentation needs augment=True")
        self.B, self.augment, self.elastic, self.intensity = batch_size, augment, bool(elastic), bool(intensity)
        reach = preprocess.ELASTIC_REACH_PX if elastic else preprocess.REACH_PX
        self.subjects = [preprocess.Subject(im, lb, reach_px=reach) for im, lb in pairs]
        vol, cls, self.offsets = preprocess.stack(self.subjects)
        dev = rt.device()
        self.vol, self.cls = torch.from_numpy(vol).to(dev), torch.from_numpy(cls).to(dev)
        self.seed, self.draws = seed, 0
        self.rng = np.random.RandomState(seed)
        S = preprocess.SIZE
        self._out = [(torch.empty(batch_size, S, S, 3, dtype=torch.float32, device=dev),
                      torch.empty(batch_size, S, S, dtype=torch.int64, device=dev)) for _ in range(2)]
        self._mats = [torch.empty(batch_size, 3, 3, 3, dtype=torch.float32, device=dev) for _ in range(2)]
        # the matrices go up from pinned memory without stalling the stream; an event says when a host buffer is free again
        self._host = [torch.empty(batch_size, 3, 3, 3, dtype=torch.float32, pin_memory=True) for _ in range(2)]
        self._copied = [None, None]
        self._flip = 0
        self._fields = [{} for _ in range(2)]
        if elastic or intensity:
            self._tmp = torch.empty(batch_size * (2 if elastic else 1) * S * S, dtype=torch.float32, device=dev)
        if elastic:
            self._elastic_taps = torch.from_numpy(preprocess.gaussian_taps(preprocess.ELASTIC_SIGMA)).to(dev)
            for f in self._fields:
                f["disp"] = torch.empty(batch_size, 2, S, S, dtype=torch.float32, device=dev)
        if intensity:
            self._bias_taps = torch.from_numpy(preprocess.gaussian_taps(preprocess.BIAS_SIGMA)).to(dev)
            for f in self._fields:
                f["gain"] = torch.empty(batch_size, S, S, dtype=torch.float32, device=dev)
                f["ab"] = torch.empty(batch_size, 2, dtype=torch.float32, device=dev)
                f["ab_host"] = torch.empty(batch_size, 2, dtype=torch.float32, pin_memory=True)

    def draw_samples(self):
        """(fp32 [B, 3, 3, 3] matrices of the channels j - 1, j, j + 1, fp32 [B, 2] (contrast, offset) or None) of B samples
        drawn from the generator: per sample the subject, (j, T), then (a, b) when intensity augmentation is on"""
        from . import preprocess
        mats, ab = [], []
        for _ in range(self.B):
            s = int(self.rng.randint(len(self.subjects)))
            j, T = self.subjects[s].draw(self.rng, self.augment)
            mats.append(self.subjects[s].matrices((j - 1, j, j + 1), T, self.offsets[s]))
            if self.intensity:
                ab.append(preprocess.intensity_draw(self.rng))
        return np.stack(mats), (np.asarray(ab, np.float64).astype(np.float32) if self.intensity else None)

    def draw_matrices(self):
        """fp32 [B, 3, 3, 3]: the matrices of the channels j - 1, j, j + 1 of B samples drawn from the generator"""
        return self.draw_samples()[0]

    def _field(self, tag, t, K, taps, amp, bound, out):
        from . import preprocess
        from .functional import smooth_noise_field
        S = preprocess.SIZE
        return smooth_noise_field(self.seed, preprocess.field_stream(tag, t), self.B, K, S, S, taps, amp, -bound, bound,
                                  out=out, tmp=self._tmp[:self.B * K * S * S].view(self.B, K, S, S))

    def next(self):
        from . import preprocess as pp
        from .functional import resample_planes
        i = self._flip
        self._flip ^= 1
        x, y = self._out[i]
        f = self._fields[i]
        if self._copied[i] is not None:
            self._copied[i].synchronize()
        mats, ab = self.draw_samples()
        t = self.draws
        self.draws += 1
        self._host[i].numpy()[...] = mats
        self._mats[i].copy_(self._host[i], non_blocking=True)
        if self.intensity:
            f["ab_host"].numpy()[...] = ab
            f["ab"].copy_(f["ab_host"], non_blocking=True)
        self._copied[i] = torch.cuda.Event()
        self._copied[i].record()
        if not (self.elastic or self.intensity):
            resample_planes(self.vol, self.cls, self._mats[i], x.shape[1], x.shape[2], True, 1, x, y)
            return x, y
        disp = gain = None
        if self.elastic:
            disp = self._field(pp.ELASTIC_STREAM_TAG, t, 2, self._elastic_taps, pp.ELASTIC_ALPHA, pp.ELASTIC_MAX_PX, f["disp"])
        if self.intensity:
            self._field(pp.BIAS_STREAM_TAG, t, 1, self._bias_taps, pp.BIAS_BETA, pp.BIAS_MAX, f["gain"].view(self.B, 1, *x.shape[1:3]))
            gain = f["gain"]
        resample_planes(self.vol, self.cls, self._mats[i], x.shape[1], x.shape[2], True, 1, x, y, disp=disp, gain=gain,
                        ab=f["ab"] if self.intensity else None)
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
