"""Data preparation of the MMWHS challenge volumes: step 1 of the reference's README (crop around the heart, cut the top 2 % of
each volume's intensity histogram, z-score each volume, sample 2-D coronal slices with data augmentation and 3 neighbouring
slices as channels).  The reference describes these steps but ships no code for them, so every choice below that its README does
not fix is this project's own: the coronal frame, the crop margin, the augmentation ranges and the label table (DESIGN 6.1).

Host side, in fp64 numpy:
* labels: MMWHS values 205 / 420 / 500 / 820 -> classes 1 / 2 / 3 / 4 of evaluation.contour_map (LV myocardium, LA blood, LV
  blood, ascending aorta); every other value -> 0.  Voxels holding a value outside the MMWHS set are counted and logged.
* orientation: the nearest signed axis permutation to RAS+ of the NIfTI affine (nifti.header_affine), as nibabel's
  io_orientation chooses it; spacing from the affine's column norms.  Coronal frame: rows run superior -> inferior, columns from the
  patient's right to left (radiological), slices anterior -> posterior.  The largest angle between a voxel axis and its world axis
  is logged: oblique volumes are resampled along the nearest permutation, not along their true axes.
* crop: the bounding box of every non-zero MMWHS label (the whole heart) in mm.  The in-plane square of side (1 + 2 margin) times
  the larger in-plane extent maps to 256 x 256 pixels; output voxels are isotropic at that pixel size, so the channels j - 1, j,
  j + 1 are one pixel apart, and D slices cover the box's anterior-posterior extent plus the margin.
* intensity: over the raw voxels inside the box, p98 = np.percentile(., 98) (linear), then mu and the population sigma of
  min(x, p98); the device volume is (min(x, p98) - mu) / sigma, computed in fp64 and rounded to fp32 once.  Only the box plus the
  largest displacement an augmentation can reach is uploaded, with the volume's edge voxels repeated beyond its border (what
  clamping the coordinate into the whole volume would read) and class 0 there.
* augmentation, per sample: slice j uniform over the heart's slice range, then a rotation U(-15, 15) degrees about the crop
  centre, a scale U(0.9, 1.1) per in-plane axis and a translation U(-10, 10) pixels per axis, from a seeded np.random.RandomState;
  output pixel p samples the un-augmented frame at centre + t + R(theta) S (p - centre).  Matrices are composed in fp64 and
  rounded to fp32 once.  augment=False: the identity at every slice.
* opt-in augmentations on the device (data.VolumeSource(elastic=, intensity=), prepare_data --elastic / --intensity), fields from
  functional.smooth_noise_field: uniforms of Philox (seed, field_stream(tag, t)) on [-1, 1) smoothed by gaussian_taps(sigma) along
  columns, then rows.
  - elastic: d = clamp(ELASTIC_ALPHA s, +-ELASTIC_MAX_PX) at ELASTIC_SIGMA, per sample, shared by the three channels and the label;
    output pixel (r, c) samples the matrix at (r + d_r, c + d_c).  Subjects of elastic sources reach ELASTIC_REACH_PX.
  - intensity: gain g = clamp(1 + BIAS_BETA s, 1 +- BIAS_MAX) at BIAS_SIGMA, then (a, b) = intensity_draw(rng) after the sample's
    (j, T); image out = a (g v) + b.
  With both off nothing extra is drawn or launched.

The device side is one pnp_resample_planes launch per batch (functional.resample_planes), plus one pnp_smooth_noise_field call per
field switched on."""
import logging
import math
import os

import numpy as np

from . import nifti

MMWHS_VALUES = (205, 420, 500, 550, 600, 820, 850)
LABEL_TABLE = {205: 1, 420: 2, 500: 3, 820: 4}       # MMWHS value -> evaluation.contour_map class
SIZE = 256                                           # output planes are SIZE x SIZE
MARGIN = 0.1
ROTATION_DEG = 15.0
SCALE_RANGE = (0.9, 1.1)
SHIFT_PX = 10.0
# RAS+ world axis and direction of the coronal frame's axes: rows S -> I (-z), columns R -> L (-x), slices A -> P (-y)
FRAME = ((2, -1), (0, -1), (1, -1))
CENTRE = (SIZE - 1) / 2.0
# the farthest an augmented pixel samples from the crop centre, in output pixels
REACH_PX = SCALE_RANGE[1] * math.hypot(CENTRE, CENTRE) + math.hypot(SHIFT_PX, SHIFT_PX)
# opt-in elastic deformation: displacement d = clamp(ALPHA s, +-D_MAX) px of a uniform field s smoothed at ELASTIC_SIGMA px
ELASTIC_SIGMA = 10.0
ELASTIC_ALPHA = 160.0
ELASTIC_MAX_PX = 16.0
# the reach of an elastic source: a displacement of at most D_MAX per axis, through the largest scale
ELASTIC_REACH_PX = REACH_PX + SCALE_RANGE[1] * math.sqrt(2.0) * ELASTIC_MAX_PX
# opt-in intensity variation: bias field g = clamp(1 + BIAS_BETA s, 1 +- BIAS_MAX) of a field smoothed at BIAS_SIGMA px, then a
# contrast a ~ U(CONTRAST_RANGE) and an offset b ~ U(OFFSET_RANGE) (z-score units) per sample
BIAS_SIGMA = 32.0
BIAS_BETA = 20.0
BIAS_MAX = 0.5
CONTRAST_RANGE = (0.75, 1.25)
OFFSET_RANGE = (-0.1, 0.1)
# Philox stream of draw t of a field: tag << 32 | t (dropout streams count up from 1 and stay far below 2^32)
ELASTIC_STREAM_TAG = 0xE1A5
BIAS_STREAM_TAG = 0xB1A5


def map_labels(raw):
    """MMWHS label values -> (uint8 class ids, boolean whole-heart mask, number of voxels outside {0} and the MMWHS set)"""
    raw = np.asarray(raw)
    out = np.zeros(raw.shape, np.uint8)
    for v, c in LABEL_TABLE.items():
        out[raw == v] = c
    heart = np.isin(raw, MMWHS_VALUES)
    unknown = int(raw.size - heart.sum() - (raw == 0).sum())
    return out, heart, unknown


def orientation(affine):
    """voxel axis v -> (RAS+ world axis, sign) of the nearest signed axis permutation, the voxel spacing and the largest angle
    (degrees) between a voxel axis and its world axis.  Like nibabel's io_orientation: the column-normalised rotation is replaced
    by its nearest orthogonal matrix (SVD), then the largest |entry| assigns one voxel axis to one world axis at a time."""
    rzs = np.asarray(affine, np.float64)[:3, :3]
    zooms = np.sqrt((rzs ** 2).sum(0))
    zooms = np.where(zooms == 0, 1.0, zooms)
    R = rzs / zooms
    P, _, Qt = np.linalg.svd(R)
    O = P @ Qt
    axis, sign = [0, 0, 0], [1, 1, 1]
    work = np.abs(O)
    for _ in range(3):
        w, v = np.unravel_index(np.argmax(work), work.shape)
        axis[v], sign[v] = int(w), (1 if O[w, v] >= 0 else -1)
        work[w, :] = -1.0
        work[:, v] = -1.0
    cos = [abs(R[axis[v], v]) for v in range(3)]
    angle = float(np.degrees(np.arccos(min(1.0, min(cos)))))
    return axis, sign, zooms, angle


def coronal_frame(affine, shape):
    """the coronal frame of a volume of `shape` stored with `affine` -> (perm, flip, F, zooms, angle): coronal axis a is voxel axis
    perm[a], reversed where flip[a]; F (4 x 4) maps coronal voxel to stored voxel; zooms and angle as orientation() returns them"""
    axis, sign, zooms, angle = orientation(affine)
    perm, flip = [], []
    for w, d in FRAME:
        v = axis.index(w)
        perm.append(v)
        flip.append(sign[v] != d)
    F = np.zeros((4, 4))
    F[3, 3] = 1.0
    for a, v in enumerate(perm):
        if flip[a]:
            F[v, a], F[v, 3] = -1.0, shape[v] - 1.0
        else:
            F[v, a] = 1.0
    return perm, flip, F, zooms, angle


def to_coronal(data, affine):
    """-> (array in the coronal frame (a view), its spacing [3] in mm, its voxel-to-world affine, largest axis angle in degrees)"""
    perm, flip, F, zooms, angle = coronal_frame(affine, np.shape(data))
    arr = np.transpose(np.asarray(data), perm)
    for a in range(3):
        if flip[a]:
            arr = np.flip(arr, a)
    return arr, zooms[perm], np.asarray(affine, np.float64) @ F, angle


def heart_box(heart):
    """inclusive voxel index bounds [(lo, hi)] * 3 of the non-zero voxels of a boolean mask"""
    box = []
    for a in range(3):
        nz = np.flatnonzero(np.any(heart, axis=tuple(b for b in range(3) if b != a)))
        if nz.size == 0:
            raise ValueError("no MMWHS heart label in the volume")
        box.append((int(nz[0]), int(nz[-1])))
    return box


class ConstantIntensity(ValueError):
    """intensity_stats of a box whose clipped intensities are constant"""


def intensity_stats(raw_box):
    """(p98, mu, sigma) of the raw voxels inside the heart box: linear 98th percentile, then the mean and population standard
    deviation of min(x, p98), in fp64"""
    x = np.asarray(raw_box, np.float64)
    p98 = float(np.percentile(x, 98))
    clipped = np.minimum(x, p98)
    mu, sigma = float(clipped.mean()), float(clipped.std())
    if not sigma > 0:
        raise ConstantIntensity("constant intensity inside the heart box: the volume cannot be z-scored")
    return p98, mu, sigma


def augment_transform(rng):
    """a 3 x 3 fp64 map from output pixel (r, c, 1) to the un-augmented frame: rotation, per-axis scale, translation (drawn in
    that order; tta_transform composes them)"""
    th = rng.uniform(-ROTATION_DEG, ROTATION_DEG)
    s = rng.uniform(SCALE_RANGE[0], SCALE_RANGE[1], 2)
    t = rng.uniform(-SHIFT_PX, SHIFT_PX, 2)
    return tta_transform(th, s, t)


def tta_transform(theta_deg, scale=(1.0, 1.0), shift=(0.0, 0.0)):
    """the deterministic form of augment_transform: a 3 x 3 fp64 map from output pixel (r, c, 1) to the un-augmented frame,
    centre + t + R(theta) diag(s) (p - centre), for a rotation of `theta_deg` degrees, per-axis scale (s_r, s_c) and translation
    (t_r, t_c) in pixels.  Values outside the training ranges (ROTATION_DEG, SCALE_RANGE, SHIFT_PX) raise ValueError: the network
    has not seen such transforms, and the uploaded sub-volume only reaches REACH_PX."""
    s, t = np.asarray(scale, np.float64).reshape(2), np.asarray(shift, np.float64).reshape(2)
    if not -ROTATION_DEG <= float(theta_deg) <= ROTATION_DEG:
        raise ValueError("rotation %r degrees outside the training range [-%g, %g]" % (theta_deg, ROTATION_DEG, ROTATION_DEG))
    if not all(SCALE_RANGE[0] <= float(x) <= SCALE_RANGE[1] for x in s):
        raise ValueError("scale %s outside the training range [%g, %g]" % (s.tolist(), SCALE_RANGE[0], SCALE_RANGE[1]))
    if not all(-SHIFT_PX <= float(x) <= SHIFT_PX for x in t):
        raise ValueError("shift %s px outside the training range [-%g, %g]" % (t.tolist(), SHIFT_PX, SHIFT_PX))
    th = np.deg2rad(theta_deg)
    A = np.array([[math.cos(th), -math.sin(th)], [math.sin(th), math.cos(th)]]) @ np.diag(s)
    T = np.eye(3)
    T[:2, :2] = A
    T[:2, 2] = CENTRE + t - A @ np.array([CENTRE, CENTRE])
    return T


def gaussian_taps(sigma):
    """fp32 [2R + 1]: the taps of scipy.ndimage.gaussian_filter1d(sigma) (truncate 4, R = int(4 sigma + 0.5)), exp(-t^2 / 2 sigma^2)
    normalised in fp64 and rounded to fp32 once"""
    R = int(4.0 * float(sigma) + 0.5)
    t = np.arange(-R, R + 1, dtype=np.float64)
    w = np.exp(-0.5 / (float(sigma) * float(sigma)) * t ** 2)
    return (w / w.sum()).astype(np.float32)


def field_stream(tag, t):
    """the Philox stream of draw t of the field kind `tag` (ELASTIC_STREAM_TAG, BIAS_STREAM_TAG)"""
    if not 0 <= int(t) < 1 << 32:
        raise ValueError("field draw index %d outside [0, 2^32)" % t)
    return (int(tag) << 32) | int(t)


def intensity_draw(rng):
    """one sample's (contrast a, offset b), drawn in that order; only called when intensity augmentation is on"""
    a = rng.uniform(CONTRAST_RANGE[0], CONTRAST_RANGE[1])
    b = rng.uniform(OFFSET_RANGE[0], OFFSET_RANGE[1])
    return a, b


def subject_name(image_path):
    b = os.path.basename(str(image_path))
    for ext in (".nii.gz", ".nii"):
        if b.endswith(ext):
            b = b[:-len(ext)]
    return b[:-len("_image")] if b.endswith("_image") else b


class Scan(object):
    """One loaded image in the coronal frame: `raw` (a view of the stored voxels), its `spacing` in mm, `coronal_affine`, and the
    native grid a prediction is written back onto (`native_shape`, `native_affine`, `frame`: coronal voxel -> native voxel).
    Loading is the slow part of a subject; the heart localisation (localise.py) crops many subjects out of one Scan."""

    def __init__(self, image_path):
        self.path = str(image_path)
        self.name = subject_name(image_path)
        self.image = im = nifti.load(image_path)
        if len(im.shape) != 3:
            raise ValueError("%s: image %s must be a 3-D volume" % (self.name, im.shape))
        self.raw, spacing, self.coronal_affine, angle = to_coronal(im.get_data(), im.get_affine())
        self.native_shape = tuple(int(n) for n in im.shape)
        self.native_affine = np.asarray(im.get_affine(), np.float64)
        self.frame = coronal_frame(self.native_affine, self.native_shape)[2]
        self.spacing = np.asarray(spacing, np.float64)
        self.angle = angle


class Subject(object):
    """One prepared (image, label) pair.  `vol` (fp32) and `cls` (uint8) are the uploaded sub-volume in slice-major order
    [slice, row, column] of the coronal frame, so a plane's gathers run along contiguous rows.  `D` slices of 256 x 256 pixels of
    `px` mm; the heart covers slices j_lo .. j_hi (each with both neighbours inside the D).  `box` is the coronal voxel box the
    crop was set from: the whole-heart label box for Subject(image, label), any box for Subject.from_box(scan, box) (no labels:
    `cls` is class 0 everywhere)."""

    def __init__(self, image_path, label_path, margin=MARGIN, reach_px=REACH_PX):
        scan = self._geometry(image_path)
        cls_all, box = self._labels(scan, label_path)
        self._crop(scan, cls_all, box, margin, reach_px)

    @classmethod
    def from_box(cls, scan, box, margin=MARGIN, reach_px=REACH_PX):
        """the subject of `scan` (a Scan or an image path) cropped at the coronal voxel box [(lo, hi)] * 3 exactly as a
        ground-truth box would crop it, without labels"""
        self = cls.__new__(cls)
        scan = self._geometry(scan)
        self._crop(scan, np.zeros(scan.raw.shape, np.uint8), [(int(lo), int(hi)) for lo, hi in box], margin, reach_px)
        return self

    def _geometry(self, image):
        """step 1: the image, its coronal frame and native grid"""
        scan = image if isinstance(image, Scan) else Scan(image)
        self.name = scan.name
        self.coronal_affine = scan.coronal_affine
        # the native grid, for predictions written back onto it (native.py): shape, affine, and coronal voxel -> native voxel
        self.native_shape = scan.native_shape
        self.native_affine = scan.native_affine
        self.frame = scan.frame
        return scan

    def _labels(self, scan, label_path):
        """step 2: class ids in the coronal frame and the whole-heart box of the label volume"""
        lb = nifti.load(label_path)
        if scan.native_shape != tuple(int(n) for n in lb.shape):
            raise ValueError("%s: image %s and label %s must be equal-shaped 3-D volumes" % (self.name, scan.native_shape, lb.shape))
        cls_all, heart, unknown = map_labels(lb.get_data())
        affine = scan.image.get_affine()
        cls_all = to_coronal(cls_all, affine)[0]
        heart = to_coronal(heart, affine)[0]
        if unknown:
            logging.warning("%s: %d label voxels hold values outside the MMWHS set (mapped to background)", self.name, unknown)
        return cls_all, heart_box(heart)

    def _crop(self, scan, cls_all, box, margin, reach_px):
        """step 3: the crop, intensity statistics and uploaded sub-volume set from the coronal voxel box"""
        raw = scan.raw
        logging.info("%s: largest angle between a voxel axis and its world axis %.3f degrees", self.name, scan.angle)
        self.spacing = s = scan.spacing
        self.box = box
        ext = np.array([(hi - lo + 1) * s[a] for a, (lo, hi) in enumerate(box)])
        self.centre = c = np.array([(lo + hi) / 2.0 for lo, hi in box])
        self.px = px = (1.0 + 2.0 * margin) * max(ext[0], ext[1]) / SIZE
        self.D = D = max(3, int(math.ceil((1.0 + 2.0 * margin) * ext[2] / px)))
        mid, half = (D - 1) / 2.0, ext[2] / (2.0 * px)
        self.j_lo, self.j_hi = max(1, int(math.ceil(mid - half))), min(D - 2, int(math.floor(mid + half)))
        if self.j_lo > self.j_hi:
            self.j_lo = self.j_hi = min(max(int(round(mid)), 1), D - 2)
        self.p98, self.mu, self.sigma = intensity_stats(raw[box[0][0]:box[0][1] + 1, box[1][0]:box[1][1] + 1,
                                                            box[2][0]:box[2][1] + 1])
        # the sub-volume every sample can reach: reach_px in plane (REACH_PX; ELASTIC_REACH_PX for elastic sources), slices
        # 0 .. D-1, one voxel more for the interpolation
        self.reach_px = reach_px
        reach = np.array([reach_px * px / s[0], reach_px * px / s[1], mid * px / s[2]])
        self.lo = lo = np.floor(c - reach).astype(np.int64) - 1
        hi = np.ceil(c + reach).astype(np.int64) + 1
        idx = [np.arange(lo[a], hi[a] + 1) for a in range(3)]
        inside = [(i >= 0) & (i < raw.shape[a]) for a, i in enumerate(idx)]
        clamped = [np.clip(i, 0, raw.shape[a] - 1) for a, i in enumerate(idx)]
        sub = np.asarray(raw[np.ix_(*clamped)], np.float64)
        self.vol = np.ascontiguousarray(((np.minimum(sub, self.p98) - self.mu) / self.sigma).astype(np.float32).transpose(2, 0, 1))
        inside = inside[0][:, None, None] & inside[1][None, :, None] & inside[2][None, None, :]
        self.cls = np.ascontiguousarray(np.where(inside, cls_all[np.ix_(*clamped)], 0).astype(np.uint8).transpose(2, 0, 1))

    def base(self, j):
        """3 x 3 fp64 map from un-augmented pixel (r, c, 1) of slice j to this sub-volume's (slice, row, column) coordinates"""
        s, c, px, lo = self.spacing, self.centre, self.px, self.lo
        return np.array([[0.0, 0.0, c[2] + (j - (self.D - 1) / 2.0) * px / s[2] - lo[2]],
                         [px / s[0], 0.0, c[0] - CENTRE * px / s[0] - lo[0]],
                         [0.0, px / s[1], c[1] - CENTRE * px / s[1] - lo[1]]])

    def matrices(self, slices, T=None, slice_offset=0):
        """fp32 [len(slices), 3, 3]: base(j) @ T for each slice j (T = None: the identity), composed in fp64 and rounded once;
        slice_offset shifts the slice coordinate (subjects stacked along the slice axis)"""
        out = []
        for j in slices:
            m = self.base(j) if T is None else self.base(j) @ T
            m[0, 2] += slice_offset
            out.append(m)
        return np.asarray(out, np.float64).astype(np.float32)

    def draw(self, rng, augment=True):
        """one sample: (slice j, in-plane transform or None); j first, then the augmentation"""
        j = int(rng.randint(self.j_lo, self.j_hi + 1))
        return j, (augment_transform(rng) if augment else None)

    def test_affine(self):
        """voxel-to-world affine of the stored test volume: stored voxel (i, j, k) is training pixel (255 - i, 255 - j) of slice k
        (the volume is stored flipped along its first two axes; test_eval's flip_correction undoes it)"""
        s, c, px = self.spacing, self.centre, self.px
        G = np.array([[px / s[0], 0, 0, c[0] - CENTRE * px / s[0]],
                      [0, px / s[1], 0, c[1] - CENTRE * px / s[1]],
                      [0, 0, px / s[2], c[2] - (self.D - 1) / 2.0 * px / s[2]],
                      [0, 0, 0, 1.0]])
        S = np.array([[-1.0, 0, 0, SIZE - 1], [0, -1.0, 0, SIZE - 1], [0, 0, 1.0, 0], [0, 0, 0, 1.0]])
        return self.coronal_affine @ G @ S


def stack(subjects):
    """subjects' sub-volumes stacked along the slice axis, padded to common rows / columns (repeated edge voxels, class 0) ->
    (vol fp32, cls uint8, slice offset of each subject)"""
    R = max(s.vol.shape[1] for s in subjects)
    Cc = max(s.vol.shape[2] for s in subjects)
    vols, clss, offs, off = [], [], [], 0
    for s in subjects:
        pad = ((0, 0), (0, R - s.vol.shape[1]), (0, Cc - s.vol.shape[2]))
        vols.append(np.pad(s.vol, pad, mode="edge"))
        clss.append(np.pad(s.cls, pad))
        offs.append(off)
        off += s.vol.shape[0]
    return np.concatenate(vols), np.concatenate(clss), offs


def read_pairs(path):
    """a text file of `image_path label_path` lines -> [(image, label)]; blank lines are skipped"""
    out = []
    with open(path) as f:
        for ln in f:
            parts = ln.split()
            if not parts:
                continue
            if len(parts) != 2:
                raise ValueError("%s: expected `image_path label_path`, got %r" % (path, ln.strip()))
            out.append((parts[0], parts[1]))
    return out
