"""Locate the heart in an unlabelled scan with the segmentation network itself, so that the scan can be cropped as a labelled one
is (DESIGN 6.1, "heart localisation").

* Calibration, from labelled pairs of the source modality (the target's labels are never read): in the coronal frame, W is the
  whole-heart box (every MMWHS value, as preprocess.Subject crops) and F the box of classes 1-4 (what the network predicts; RV, RA
  and PA are background).  Per coronal axis a, in mm: extent_a = (W_hi - W_lo + 1) s_a, below_a = (F_lo - W_lo) s_a, above_a =
  (W_hi - F_hi) s_a.  The calibration is the np.median of each over the pairs.
* Located box of native labels L: fg = (1 <= L < C), its largest 26-connected component (pnp_largest_components at C = 2), that
  component's native box (pnp_label_boxes), mapped exactly to the coronal frame through Subject.frame (a signed permutation), and
  expanded to a whole-heart box: lo_a = max(0, F_lo - r(below_a / s_a)), hi_a = min(n_a - 1, F_hi + r(above_a / s_a)), r(x) =
  floor(x + 0.5).  No fg voxel: not located.
* Seed: windows of L_a = min(n_a, max(1, r(extent_a / s_a))) voxels per coronal axis, k_a = 1 if L_a = n_a else
  ceil(2 (n_a - L_a) / L_a) + 1 of them at starts r(i (n_a - L_a) / (k_a - 1)), rows-, columns-, then slices-major.  Each window is
  a subject cropped at that box (preprocess.Subject.from_box; a window of constant intensity is skipped and counted); their class
  probabilities are summed at every native voxel in window order (functional.NativeAccumulator, the rules of
  pnp_native_labels_ensemble) and the located box of those labels is box_0.
* Iteration k = 0, 1, ...: crop S_k at box_k, predict, native labels (pnp_native_labels), locate box_{k+1}.  Converged when every
  face of box_{k+1} is within LOCATE_TOL_MM of box_k's (the result is S_k); stopped, not converged, after LOCATE_MAX_ITER
  iterations (the last S_k) or when nothing is located (the last S_k, none if the seed found nothing)."""
import json
import logging
import math

import numpy as np
import torch

from . import functional as F
from . import nifti
from . import preprocess

LOCATE_TOL_MM = 2.0
LOCATE_MAX_ITER = 4
NETWORK_CLASSES = (1, 2, 3, 4)            # the structures the network predicts (preprocess.LABEL_TABLE)


def r(x):
    """floor(x + 0.5): the rounding of every mm -> voxel conversion here"""
    return int(math.floor(float(x) + 0.5))


class Calibration(object):
    """extent, below, above: fp64 [3] in mm per coronal axis (rows, columns, slices); subjects: the calibrating pairs' names"""

    def __init__(self, extent, below, above, subjects=()):
        self.extent = np.asarray(extent, np.float64).reshape(3)
        self.below = np.asarray(below, np.float64).reshape(3)
        self.above = np.asarray(above, np.float64).reshape(3)
        self.subjects = [str(s) for s in subjects]

    def to_dict(self):
        return {"extent_mm": self.extent.tolist(), "below_mm": self.below.tolist(), "above_mm": self.above.tolist(),
                "subjects": self.subjects, "count": len(self.subjects)}

    def save(self, path):
        with open(path, "w") as f:
            json.dump(self.to_dict(), f, indent=1)
        return path

    @classmethod
    def load(cls, path):
        with open(path) as f:
            d = json.load(f)
        return cls(d["extent_mm"], d["below_mm"], d["above_mm"], d.get("subjects", ()))


def as_calibration(c):
    """a Calibration, or the path of its JSON file"""
    return c if isinstance(c, Calibration) else Calibration.load(c)


def pair_geometry(image_path, label_path):
    """(W, F, spacing): the coronal whole-heart box, the class 1-4 box and the coronal spacing of one labelled pair"""
    im, lb = nifti.load(image_path), nifti.load(label_path)
    if tuple(im.shape) != tuple(lb.shape) or len(im.shape) != 3:
        raise ValueError("%s: image %s and label %s must be equal-shaped 3-D volumes" % (image_path, im.shape, lb.shape))
    cls, heart, _ = preprocess.map_labels(lb.get_data())
    heart, spacing = preprocess.to_coronal(heart, im.get_affine())[:2]
    cls = preprocess.to_coronal(cls, im.get_affine())[0]
    fg = np.isin(cls, NETWORK_CLASSES)
    if not fg.any():
        raise ValueError("%s: no voxel of classes 1-4 (LV myocardium, LA, LV blood, aorta): it cannot calibrate the localiser"
                         % label_path)
    return preprocess.heart_box(heart), preprocess.heart_box(fg), np.asarray(spacing, np.float64)


def pair_numbers(W, Fb, s):
    """(extent, below, above) in mm, each [3], of one pair's boxes"""
    extent = np.array([(W[a][1] - W[a][0] + 1) * s[a] for a in range(3)])
    below = np.array([(Fb[a][0] - W[a][0]) * s[a] for a in range(3)])
    above = np.array([(W[a][1] - Fb[a][1]) * s[a] for a in range(3)])
    return extent, below, above


def calibrate(pairs):
    """the Calibration of labelled (image, label) pairs: the median of each number over the pairs"""
    pairs = list(pairs)
    if not pairs:
        raise ValueError("calibrate: no pairs")
    nums = [pair_numbers(*pair_geometry(im, lb)) for im, lb in pairs]
    med = [np.median(np.stack([n[i] for n in nums]), axis=0) for i in range(3)]
    return Calibration(*med, subjects=[preprocess.subject_name(im) for im, _ in pairs])


def seed_windows(shape, spacing, calibration):
    """[box] of the seed pass over a coronal volume of `shape`: box = [(lo, hi)] * 3, rows-, columns-, then slices-major"""
    starts = []
    for a in range(3):
        n = int(shape[a])
        L = min(n, max(1, r(calibration.extent[a] / spacing[a])))
        k = 1 if L == n else int(math.ceil(2.0 * (n - L) / L)) + 1
        starts.append([(0 if k == 1 else r(i * (n - L) / (k - 1.0)), L) for i in range(k)])
    return [[(s0, s0 + L0 - 1), (s1, s1 + L1 - 1), (s2, s2 + L2 - 1)]
            for s0, L0 in starts[0] for s1, L1 in starts[1] for s2, L2 in starts[2]]


def coronal_box(native_box, frame):
    """the coronal box [(lo, hi)] * 3 of a native box [(lo, hi)] * 3 under Subject.frame (coronal voxel -> native voxel, a signed
    permutation): exact"""
    out = []
    for a in range(3):
        v = int(np.flatnonzero(frame[:3, a])[0])
        lo, hi = native_box[v]
        if frame[v, a] > 0:
            out.append((int(lo), int(hi)))
        else:
            t = int(round(frame[v, 3]))
            out.append((t - int(hi), t - int(lo)))
    return out


def expand_box(fbox, shape, spacing, calibration):
    """the whole-heart box around a class 1-4 box: below / above converted to voxels, clamped into the volume"""
    return [(max(0, fbox[a][0] - r(calibration.below[a] / spacing[a])),
             min(int(shape[a]) - 1, fbox[a][1] + r(calibration.above[a] / spacing[a]))) for a in range(3)]


def located_box(labels, num_cls, scan, calibration):
    """the located whole-heart box (coronal) of native labels (uint8 on the device), or None when no voxel is of class 1 ..
    num_cls - 1"""
    fg = ((labels >= 1) & (labels < num_cls)).to(torch.uint8)
    largest, _, _ = F.largest_components(fg, 2, 26, out=fg)
    b = F.label_boxes(largest, 2)[1]
    if b[0] == 0:
        return None
    native = [(int(b[1 + 2 * v]), int(b[2 + 2 * v])) for v in range(3)]
    return expand_box(coronal_box(native, scan.frame), scan.raw.shape, scan.spacing, calibration)


def face_distance_mm(a, b, spacing):
    """the largest distance in mm between corresponding faces of two coronal boxes"""
    return max(max(abs(a[i][0] - b[i][0]), abs(a[i][1] - b[i][1])) * float(spacing[i]) for i in range(3))


def box_iou(a, b):
    """intersection over union of two inclusive voxel boxes"""
    inter, va, vb = 1, 1, 1
    for (alo, ahi), (blo, bhi) in zip(a, b):
        inter *= max(0, min(ahi, bhi) - max(alo, blo) + 1)
        va *= ahi - alo + 1
        vb *= bhi - blo + 1
    return inter / float(va + vb - inter)


class Located(object):
    """what locate found: subject (the located preprocess.Subject, None if nothing was found), boxes (box_0, box_1, ...; coronal),
    iterations, converged, windows (seed windows predicted) and skipped (seed windows of constant intensity)"""

    def __init__(self, subject, boxes, iterations, converged, windows, skipped):
        self.subject, self.boxes, self.iterations, self.converged = subject, boxes, iterations, converged
        self.windows, self.skipped = windows, skipped


def locate(scan, predict, calibration, num_cls):
    """the seed pass and the re-cropping iteration on `scan` (preprocess.Scan or an image path) -> Located.  predict(subject) ->
    fp32 [D, 256, 256, num_cls] class probabilities on the device (native.predict_scores of the network; tests substitute an
    oracle)."""
    from .native import map32
    scan = scan if isinstance(scan, preprocess.Scan) else preprocess.Scan(scan)
    calibration = as_calibration(calibration)
    windows = seed_windows(scan.raw.shape, scan.spacing, calibration)
    acc = F.NativeAccumulator(scan.native_shape, num_cls)
    used = skipped = 0
    for box in windows:
        try:
            s = preprocess.Subject.from_box(scan, box)
        except preprocess.ConstantIntensity:
            skipped += 1
            continue
        acc.add(predict(s), torch.from_numpy(map32(s)).to(acc.sums.device))
        used += 1
    labels, _ = acc.labels()
    del acc
    box = located_box(labels, num_cls, scan, calibration)
    logging.info("%s: seed pass over %d windows (%d of constant intensity skipped) -> %s", scan.name, used, skipped, box)
    boxes = [box]
    subject, iterations, converged = None, 0, False
    while box is not None:
        subject = preprocess.Subject.from_box(scan, box)
        iterations += 1
        scores = predict(subject)
        labels, _ = F.native_labels(scores, torch.from_numpy(map32(subject)).to(scores.device), subject.native_shape)
        del scores
        nxt = located_box(labels, num_cls, scan, calibration)
        if nxt is None:
            break
        boxes.append(nxt)
        if face_distance_mm(nxt, box, scan.spacing) <= LOCATE_TOL_MM:
            converged = True
            break
        if iterations >= LOCATE_MAX_ITER:
            break
        box = nxt
    logging.info("%s: located box %s after %d iteration(s), %s", scan.name, None if subject is None else subject.box, iterations,
                 "converged" if converged else "not converged")
    return Located(subject, boxes, iterations, converged, used, skipped)


def truth_box(subject, label_path):
    """the coronal whole-heart box of a label volume, as Subject(image, label) crops it (for scoring a located box); `subject`:
    a preprocess.Scan or Subject of the label's image"""
    _, heart, _ = preprocess.map_labels(nifti.load(label_path).get_data())
    return preprocess.heart_box(preprocess.to_coronal(heart, subject.native_affine)[0])


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description="calibrate the heart localiser from labelled source-modality pairs")
    ap.add_argument("--pairs", required=True, help="text file of `image_path label_path` lines (source modality, e.g. MR)")
    ap.add_argument("--out", required=True, help="the calibration's JSON file")
    a = ap.parse_args(argv)
    logging.basicConfig(level=logging.INFO)
    cal = calibrate(preprocess.read_pairs(a.pairs))
    cal.save(a.out)
    print(a.out)
    return cal
