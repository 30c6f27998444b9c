"""Prepare MMWHS volumes as the reference's README step 1 describes (preprocess.py):

  python prepare_data.py --modality ct|mr --pairs LIST --split train|val|test --out DIR [--slices-per-volume 600] [--seed S]
                         [--no-augment] [--elastic] [--intensity]

LIST has one `image_path label_path` pair per line ({ct,mr}_train_10xx_{image,label}.nii.gz).
* train / val: one single-example TFRecord file per sample in the 8-feature schema (tfrecord.encode_example): image [256,256,3]
  fp32 (slices j - 1, j, j + 1), label [256,256,3] class ids as fp32.  --slices-per-volume samples per subject with augmentation;
  --no-augment writes every slice of the heart's range once, unaugmented.  Writes DIR/{mod}_{split}/*.tfrecords,
  DIR/lists/{mod}_{split}_list (what --train-list / --lists read) and DIR/lists/{mod}_{split}_volumes (the pairs, for
  train_gan.py --volumes).
  --elastic / --intensity (augmented training split only): the records also carry the elastic deformation and the intensity
  variation of preprocess.py, drawn as data.VolumeSource draws them: (a, b) after each sample's (j, T), and per launch of CHUNK
  samples the fields of draw t = 0, 1, .. (counted over the whole command) from Philox seed --seed.
* test: DIR/{mod}_test/<name>_{image,label}.nii.gz, every slice of the crop unaugmented, stored flipped along the first two axes
  (test_eval's default flip_correction puts them back in the training orientation), with their world affine; and
  DIR/lists/{mod}_test_nii_list / {mod}_test_label_list."""
import argparse
import logging
import os

import numpy as np
import torch

from . import nifti
from . import preprocess
from . import runtime as rt
from . import tfrecord
from .functional import resample_planes, smooth_noise_field

CHUNK = 64          # samples per launch when writing records


def _upload(subject):
    dev = rt.device()
    return torch.from_numpy(subject.vol).to(dev), torch.from_numpy(subject.cls).to(dev)


class FieldDraws(object):
    """the device fields of --elastic / --intensity: one per launch, draw t counted over the whole command"""

    def __init__(self, seed, elastic, intensity):
        self.seed, self.elastic, self.intensity, self.t = seed, elastic, intensity, 0
        dev = rt.device()
        self.taps_e = torch.from_numpy(preprocess.gaussian_taps(preprocess.ELASTIC_SIGMA)).to(dev) if elastic else None
        self.taps_b = torch.from_numpy(preprocess.gaussian_taps(preprocess.BIAS_SIGMA)).to(dev) if intensity else None

    def next(self, B):
        """-> (disp [B, 2, S, S] or None, gain [B, S, S] or None) of the next draw"""
        S, pp, t = preprocess.SIZE, preprocess, self.t
        self.t += 1
        disp = gain = None
        if self.elastic:
            disp = smooth_noise_field(self.seed, pp.field_stream(pp.ELASTIC_STREAM_TAG, t), B, 2, S, S, self.taps_e, pp.ELASTIC_ALPHA,
                                      -pp.ELASTIC_MAX_PX, pp.ELASTIC_MAX_PX)
        if self.intensity:
            gain = smooth_noise_field(self.seed, pp.field_stream(pp.BIAS_STREAM_TAG, t), B, 1, S, S, self.taps_b, pp.BIAS_BETA,
                                      -pp.BIAS_MAX, pp.BIAS_MAX)[:, 0]
        return disp, gain


def write_records(subject, out_dir, n, rng, augment=True, fields=None):
    """the subject's samples as single-example TFRecord files -> their paths; `fields` (a FieldDraws) adds the elastic and
    intensity augmentations"""
    vol, cls = _upload(subject)
    intensity = fields is not None and fields.intensity
    if augment:
        draws = []
        for _ in range(n):
            j, T = subject.draw(rng, True)
            draws.append((j, T, preprocess.intensity_draw(rng) if intensity else None))
    else:
        draws = [(j, None, None) for j in range(subject.j_lo, subject.j_hi + 1)]
    paths = []
    for at in range(0, len(draws), CHUNK):
        part = draws[at:at + CHUNK]
        mats = torch.from_numpy(np.stack([subject.matrices((j - 1, j, j + 1), T) for j, T, _ in part])).to(vol.device)
        if fields is None:
            img, lab = resample_planes(vol, cls, mats, preprocess.SIZE, preprocess.SIZE, True, 3)
        else:
            disp, gain = fields.next(len(part))
            ab = torch.from_numpy(np.asarray([d[2] for d in part], np.float64).astype(np.float32)).to(vol.device) if intensity else None
            img, lab = resample_planes(vol, cls, mats, preprocess.SIZE, preprocess.SIZE, True, 3, disp=disp, gain=gain, ab=ab)
        img, lab = img.cpu().numpy(), lab.cpu().numpy().astype(np.float32)
        for k in range(len(part)):
            p = os.path.join(out_dir, "%s_%04d.tfrecords" % (subject.name, at + k))
            tfrecord.write_record(p, [tfrecord.encode_example(img[k], lab[k])])
            paths.append(os.path.abspath(p))
    return paths


def test_volume(subject):
    """(image fp32 [256,256,D], labels uint8 [256,256,D]) in the training orientation: every slice, unaugmented, one launch"""
    vol, cls = _upload(subject)
    mats = subject.matrices(range(subject.D))[None]
    img, lab = resample_planes(vol, cls, torch.from_numpy(mats).to(vol.device), preprocess.SIZE, preprocess.SIZE, True, subject.D)
    return img[0].cpu().numpy(), lab[0].cpu().numpy().astype(np.uint8)


def write_test(subject, out_dir):
    """the stored test pair (flipped along axes 0 and 1) -> (image path, label path)"""
    img, lab = test_volume(subject)
    aff = subject.test_affine()
    ip = os.path.join(out_dir, subject.name + "_image.nii.gz")
    lp = os.path.join(out_dir, subject.name + "_label.nii.gz")
    nifti.save(np.ascontiguousarray(img[::-1, ::-1]), aff, ip)
    nifti.save(np.ascontiguousarray(lab[::-1, ::-1]), aff, lp)
    return os.path.abspath(ip), os.path.abspath(lp)


def _write_list(path, lines):
    with open(path, "w") as f:
        for ln in lines:
            f.write(ln + "\n")


def prepare(modality, pairs, split, out, slices_per_volume=600, seed=0, augment=True, elastic=False, intensity=False):
    """the command's work; returns the list files it wrote"""
    if (elastic or intensity) and (split != "train" or not augment):
        raise ValueError("elastic / intensity augmentation applies to the augmented training split only")
    fields = FieldDraws(seed, elastic, intensity) if (elastic or intensity) else None
    lists = os.path.join(out, "lists")
    os.makedirs(lists, exist_ok=True)
    data_dir = os.path.join(out, "%s_%s" % (modality, split))
    os.makedirs(data_dir, exist_ok=True)
    rng = np.random.RandomState(seed)
    written = []
    for im, lb in pairs:
        s = preprocess.Subject(im, lb, reach_px=preprocess.ELASTIC_REACH_PX if elastic else preprocess.REACH_PX)
        logging.info("%s: spacing %s mm, pixel %.4f mm, D = %d, heart slices %d..%d", s.name, np.round(s.spacing, 4), s.px, s.D,
                     s.j_lo, s.j_hi)
        if split == "test":
            written.append(write_test(s, data_dir))
        else:
            written.extend(write_records(s, data_dir, slices_per_volume, rng, augment, fields))
    if split == "test":
        out_lists = [os.path.join(lists, "%s_test_nii_list" % modality), os.path.join(lists, "%s_test_label_list" % modality)]
        _write_list(out_lists[0], [w[0] for w in written])
        _write_list(out_lists[1], [w[1] for w in written])
    else:
        out_lists = [os.path.join(lists, "%s_%s_list" % (modality, split)), os.path.join(lists, "%s_%s_volumes" % (modality, split))]
        _write_list(out_lists[0], written)
        _write_list(out_lists[1], ["%s %s" % (os.path.abspath(im), os.path.abspath(lb)) for im, lb in pairs])
    return out_lists


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--modality", required=True, choices=["ct", "mr"])
    ap.add_argument("--pairs", required=True, help="text file of `image_path label_path` lines")
    ap.add_argument("--split", required=True, choices=["train", "val", "test"])
    ap.add_argument("--out", required=True)
    ap.add_argument("--slices-per-volume", type=int, default=600)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--no-augment", action="store_true", help="every slice of the heart's range once, without augmentation")
    ap.add_argument("--elastic", action="store_true", help="augmented training split: add the elastic deformation (preprocess.py)")
    ap.add_argument("--intensity", action="store_true",
                    help="augmented training split: add the bias field, contrast and offset (preprocess.py)")
    a = ap.parse_args(argv)
    if (a.elastic or a.intensity) and (a.split != "train" or a.no_augment):
        ap.error("--elastic / --intensity apply to the augmented training split only (--split train without --no-augment)")
    logging.basicConfig(level=logging.INFO)
    for p in prepare(a.modality, preprocess.read_pairs(a.pairs), a.split, a.out, a.slices_per_volume, a.seed, not a.no_augment,
                     a.elastic, a.intensity):
        print(p)


if __name__ == "__main__":
    main()
