"""Prepare MMWHS volumes as the reference's README step 1 describes (preprocess.py):

  python prepare_data.py --modality ct|mr --pairs LIST --split train|val|test --out DIR [--slices-per-volume 600] [--seed S]
                         [--no-augment]

LIST has one `image_path label_path` pair per line ({ct,mr}_train_10xx_{image,label}.nii.gz).
* train / val: one single-example TFRecord file per sample in the 8-feature schema (tfrecord.encode_example): image [256,256,3]
  fp32 (slices j - 1, j, j + 1), label [256,256,3] class ids as fp32.  --slices-per-volume samples per subject with augmentation;
  --no-augment writes every slice of the heart's range once, unaugmented.  Writes DIR/{mod}_{split}/*.tfrecords,
  DIR/lists/{mod}_{split}_list (what --train-list / --lists read) and DIR/lists/{mod}_{split}_volumes (the pairs, for
  train_gan.py --volumes).
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
from .functional import resample_planes

CHUNK = 64          # samples per launch when writing records


def _upload(subject):
    dev = rt.device()
    return torch.from_numpy(subject.vol).to(dev), torch.from_numpy(subject.cls).to(dev)


def write_records(subject, out_dir, n, rng, augment=True):
    """the subject's samples as single-example TFRecord files -> their paths"""
    vol, cls = _upload(subject)
    if augment:
        draws = [subject.draw(rng, True) for _ in range(n)]
    else:
        draws = [(j, None) for j in range(subject.j_lo, subject.j_hi + 1)]
    paths = []
    for at in range(0, len(draws), CHUNK):
        part = draws[at:at + CHUNK]
        mats = np.stack([subject.matrices((j - 1, j, j + 1), T) for j, T in part])
        img, lab = resample_planes(vol, cls, torch.from_numpy(mats).to(vol.device), preprocess.SIZE, preprocess.SIZE, True, 3)
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


def prepare(modality, pairs, split, out, slices_per_volume=600, seed=0, augment=True):
    """the command's work; returns the list files it wrote"""
    lists = os.path.join(out, "lists")
    os.makedirs(lists, exist_ok=True)
    data_dir = os.path.join(out, "%s_%s" % (modality, split))
    os.makedirs(data_dir, exist_ok=True)
    rng = np.random.RandomState(seed)
    written = []
    for im, lb in pairs:
        s = preprocess.Subject(im, lb)
        logging.info("%s: spacing %s mm, pixel %.4f mm, D = %d, heart slices %d..%d", s.name, np.round(s.spacing, 4), s.px, s.D,
                     s.j_lo, s.j_hi)
        if split == "test":
            written.append(write_test(s, data_dir))
        else:
            written.extend(write_records(s, data_dir, slices_per_volume, rng, augment))
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
    a = ap.parse_args(argv)
    logging.basicConfig(level=logging.INFO)
    for p in prepare(a.modality, preprocess.read_pairs(a.pairs), a.split, a.out, a.slices_per_volume, a.seed, not a.no_augment):
        print(p)


if __name__ == "__main__":
    main()
