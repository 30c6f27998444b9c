"""Segment test subjects on their original MMWHS grid and score them there, in millimetres.

A raw (image, label) pair goes in (preprocess.Subject: orientation, ground-truth heart crop, intensity cut and z-score, exactly as
for the prepared test split), and a label map of that same scan comes out:
* prediction: every frame 1 .. D - 2 of the prepared grid in ascending order, each batch's input frames (planes j - 1, j, j + 1,
  unaugmented) drawn on the device by one pnp_resample_planes launch; the last short batch is padded with copies of its last
  frame (the network needs its full static batch) and the padded outputs are discarded.  The trainer's inference forward gives
  the logits, pnp_pixel_softmax2 the class probabilities, written into a score volume [D, 256, 256, C]; frames 0 and D - 1 lie in
  the crop margin and hold background with probability 1.
* resampling: one pnp_native_labels launch samples the score volume at every native voxel (trilinear, the taps and lerp order of
  pnp_resample_planes) and labels it by the argmax; outside the prepared grid the voxel is background.  The native voxel ->
  prepared coordinate map is the inverse of Subject.base composed with to_coronal's permutation and flip, computed in fp64 from
  the subject's own geometry and rounded to fp32 once.
* scoring against preprocess.map_labels of the native label volume: per-class Dice / Jaccard from the kernel's confusion counts,
  ASSD / HD in mm from functional.surface_distances with the native voxel sizes (the column norms of the image's affine), and
  on request the q-th percentile HD in mm (HD95 at q = 95).
* optional post-processing (largest_component = 6 or 26): one pnp_largest_components call keeps the largest 3-D connected
  component of each class and sets the rest to background, in place on the device, before anything else sees the labels; it takes
  the native ground truth, so Dice / Jaccard come from its counts.  ASSD / HD and the written file are then those of the
  post-processed labels; the Dice before it (from pnp_native_labels' counts), the number of components and the voxels removed are
  kept too.
* optional ensembling (Ensemble: several checkpoints and / or test-time transforms): K members, ordered checkpoint-major and
  transform-minor, each predicted into its slice of one [K, D, 256, 256, C] score buffer -- a checkpoint is restored into the
  network before its members' frames are predicted, and a transform T (preprocess.tta_transform) draws the member's input frames
  with subject.matrices(.., T) --, then one pnp_native_labels_ensemble launch samples every member at every native voxel through
  its own map (member_map), sums the class scores of the members covering it and labels it by the argmax.  The written file, the
  metrics and the post-processing are those of the ensemble labels; the Dice of member 0 alone is kept too.  K = 1 is the path
  above.
* outputs under <out>/: native_pred/<name>_label.nii.gz (int16 MMWHS codes 205 / 420 / 500 / 820 for classes 1-4, 0 elsewhere,
  with the image's shape and affine) and native.csv (one row per subject; <organ>_hd<q>_mm columns when a percentile is asked,
  <organ>_dice_raw / _components / _removed after those with the post-processing, and `members` and <organ>_dice_first after
  all the others for an ensemble).

* optional heart localisation (run(locate=), segment; localise.py): the crop is the box the network itself locates in the scan,
  without its labels -- a sliding-window seed pass, then re-cropping around the predicted heart until the crop stops moving --,
  and the subject is predicted from that crop as above.  With labels, native.csv adds windows, iterations, converged, box_iou
  and box_err_mm (the located against the ground-truth whole-heart box) after all the others; segment writes located.csv.

Otherwise the crop is the ground-truth heart box, as for the prepared test split: a native-grid score is then that of a
prediction made inside a ground-truth region of interest."""
import contextlib
import logging
import os

import numpy as np
import torch

from . import evaluation
from . import functional as F
from . import nifti
from . import preprocess
from . import runtime as rt
from .lib import _dice, _jaccard
from .prepare_data import _upload

CSV_COLUMNS = ("dice", "assd_mm", "hd_mm", "border_pred", "border_gt")
COMPONENT_COLUMNS = ("dice_raw", "components", "removed")      # per organ, with the largest-component post-processing
ENSEMBLE_COLUMNS = ("dice_first",)                              # per organ, after `members`, for an ensemble of K > 1
LOCATE_COLUMNS = ("windows", "iterations", "converged", "box_iou", "box_err_mm")   # after all others, for located subjects
CONNECTIVITIES = (6, 26)
MAX_MEMBERS = 16                                                # PNP_NATIVE_MAX_MEMBERS
SLOT_KEYWORDS = ("Adam", "RMS")                                 # optimizer slot names: never needed by a prediction


def voxel_map(subject):
    """fp64 [3, 4]: native voxel (i, j, k, 1) -> prepared (slice, row, column) of the subject's score volume"""
    s, c, px, Fr = subject.spacing, subject.centre, subject.px, subject.frame
    to_coronal = np.eye(4)                         # the inverse of the signed permutation Fr: coronal voxel = R^T (native - t)
    to_coronal[:3, :3] = Fr[:3, :3].T
    to_coronal[:3, 3] = -Fr[:3, :3].T @ Fr[:3, 3]
    # coronal (row, column, slice) -> prepared (slice, row, column): the inverse of Subject.base
    to_prepared = np.zeros((3, 4))
    to_prepared[0, 2], to_prepared[0, 3] = s[2] / px, (subject.D - 1) / 2.0 - c[2] * s[2] / px
    to_prepared[1, 0], to_prepared[1, 3] = s[0] / px, preprocess.CENTRE - c[0] * s[0] / px
    to_prepared[2, 1], to_prepared[2, 3] = s[1] / px, preprocess.CENTRE - c[1] * s[1] / px
    return to_prepared @ to_coronal


def map32(subject):
    """voxel_map rounded to fp32 once: the 12 values pnp_native_labels reads"""
    return voxel_map(subject).astype(np.float32).reshape(-1)


def member_map(subject, T=None):
    """fp64 [3, 4]: native voxel -> (slice, row, column) of the score volume predicted from frames drawn through the in-plane
    transform T (3 x 3, member pixel -> un-augmented pixel; None: the identity).  Un-augmented pixel b is member pixel T^-1 b, so
    the row and column rows of voxel_map are mapped through T^-1; the slice row is voxel_map's.  T = None or the identity gives
    voxel_map itself, bit for bit."""
    M = voxel_map(subject)
    if T is None or np.array_equal(np.asarray(T, np.float64), np.eye(3)):
        return M
    H = np.vstack([M[1:3], [0.0, 0.0, 0.0, 1.0]])
    out = M.copy()
    out[1:3] = (np.linalg.inv(np.asarray(T, np.float64)) @ H)[:2]
    return out


def member_map32(subject, T=None):
    """member_map rounded to fp32 once, as map32"""
    return member_map(subject, T).astype(np.float32).reshape(-1)


def native_spacing(subject):
    """voxel sizes of the native grid in mm, in native axis order: the column norms of the image's affine"""
    return np.sqrt((subject.native_affine[:3, :3] ** 2).sum(0))


def label_codes(num_cls):
    """int16 [num_cls]: class -> MMWHS label value (0 for background and classes outside preprocess.LABEL_TABLE)"""
    codes = np.zeros(num_cls, np.int16)
    for v, c in preprocess.LABEL_TABLE.items():
        if c < num_cls:
            codes[c] = v
    return codes


def input_frames(subject, vol, frames, T=None):
    """fp32 [len(frames), 256, 256, 3] on the device: the planes (j - 1, j, j + 1) of each frame j, drawn through the in-plane
    transform T (None: unaugmented), one launch"""
    mats = np.stack([subject.matrices((j - 1, j, j + 1), T) for j in frames])
    img, _ = F.resample_planes(vol, None, torch.from_numpy(mats).to(vol.device), preprocess.SIZE, preprocess.SIZE, True, 0)
    return img


def frame_batches(D, batch_size):
    """frames 1 .. D - 2 in ascending order, cut into batches of `batch_size`; the last may be short"""
    frames = list(range(1, D - 1))
    return [frames[at:at + batch_size] for at in range(0, len(frames), batch_size)]


def predict_scores(subject, logits_fn, batch_size, num_cls, T=None, out=None):
    """fp32 [D, 256, 256, num_cls] on the device: pixel_softmax2 of `logits_fn` (x [B, 256, 256, 3] -> logits [B, 256, 256, C])
    at every frame 1 .. D - 2, its input frames drawn through the in-plane transform T (None: unaugmented); frames 0 and D - 1
    are background with probability 1.  `out` (contiguous fp32 [D, 256, 256, num_cls] on the device, e.g. one member's slice of
    an ensemble's score buffer) may be given to write into."""
    vol, _ = _upload(subject)
    shape = (subject.D, preprocess.SIZE, preprocess.SIZE, num_cls)
    if out is None:
        scores = torch.zeros(shape, dtype=torch.float32, device=vol.device)
    else:
        if tuple(out.shape) != shape or out.dtype != torch.float32 or not out.is_contiguous():
            raise ValueError("predict_scores: out must be contiguous fp32 %s, got %s %s" % (shape, tuple(out.shape), out.dtype))
        scores = out
        scores[0].zero_()
        scores[subject.D - 1].zero_()
    scores[0, ..., 0] = 1.0
    scores[subject.D - 1, ..., 0] = 1.0
    with torch.no_grad():
        for part in frame_batches(subject.D, batch_size):
            x = input_frames(subject, vol, part + [part[-1]] * (batch_size - len(part)), T)
            prob = F.pixel_softmax2(logits_fn(x))
            scores[part[0]:part[-1] + 1] = prob[:len(part)]
    return scores


def ground_truth(label_path):
    """uint8 class ids of the native label volume (preprocess.map_labels), on the device"""
    cls, _, _ = preprocess.map_labels(nifti.load(label_path).get_data())
    return torch.from_numpy(np.ascontiguousarray(cls)).to(rt.device())


def native_prediction(subject, scores, gt, T=None):
    """(labels uint8 [native shape] on the device, confusion counts int64 [C, C] on the host, None without gt): one
    pnp_native_labels launch.  T: the in-plane transform the score volume was predicted through (None: unaugmented)."""
    vmap = torch.from_numpy(member_map32(subject, T)).to(scores.device)
    labels, cm = F.native_labels(scores, vmap, subject.native_shape, gt)
    return labels, (None if cm is None else cm.cpu().numpy())


def check_members(K):
    """K ensemble members must be 1 .. MAX_MEMBERS (ValueError otherwise)"""
    if not 1 <= K <= MAX_MEMBERS:
        raise ValueError("an ensemble holds 1 to %d members, got %d" % (MAX_MEMBERS, K))
    return K


def tta_transforms(tta):
    """[(theta_deg, scale_r, scale_c, shift_r, shift_c)] -> [3 x 3 preprocess.tta_transform, None for the identity]; values
    outside the training ranges raise ValueError"""
    out = []
    for t in tta:
        if len(t) != 5:
            raise ValueError("a test-time transform is (theta_deg, scale_r, scale_c, shift_r, shift_c), got %r" % (t,))
        T = preprocess.tta_transform(t[0], (t[1], t[2]), (t[3], t[4]))
        out.append(None if np.array_equal(T, np.eye(3)) else T)
    return out


def checkpoint_missing(path, skip_keywords, strip_suffix=False):
    """the graph variables (runtime.graph) a .npz checkpoint lacks, leaving out names that contain one of `skip_keywords`.
    `strip_suffix`: a key 'x:0' stores variable x -- only for a trainer whose `restore` loads such keys (the GAN trainer's does,
    the segmenter trainer's loads exact names only), so that the check counts exactly what `restore` will load"""
    with np.load(path) as z:
        stored = {k[:-2] if strip_suffix and k.endswith(":0") else k for k in z.files}
    return [n for n in rt.graph.order if n not in stored and not any(kw in n for kw in skip_keywords)]


class Ensemble(object):
    """The members of a native-grid ensemble: `checkpoints` (.npz paths; None: the network as it stands) times in-plane
    `transforms` (3 x 3 from preprocess.tta_transform, None for the identity; None: the identity only), ordered checkpoint-major,
    transform-minor.  Every checkpoint must hold every graph variable whose name contains none of `skip_keywords` (the optimizer
    slots, and the critics for the GAN trainer), under the key names the network's `restore` loads (`strip_suffix`:
    checkpoint_missing), else ValueError: `restore` would otherwise leave the previous member's value in place.  All checks run
    here, before any prediction."""

    def __init__(self, net, checkpoints=None, transforms=None, skip_keywords=(), strip_suffix=False):
        self.net = net
        self.checkpoints = [None] if checkpoints is None else [str(c) for c in checkpoints]
        self.transforms = [None] if not transforms else list(transforms)
        if not self.checkpoints:
            raise ValueError("an ensemble needs at least one checkpoint")
        self.K = check_members(len(self.checkpoints) * len(self.transforms))
        for path in self.checkpoints:
            if path is not None:
                missing = checkpoint_missing(path, tuple(skip_keywords), strip_suffix)
                if missing:
                    raise ValueError("checkpoint %s lacks %d variable(s) the prediction needs: %s" % (
                        path, len(missing), ", ".join(missing[:8]) + (" ..." if len(missing) > 8 else "")))
        self.loaded = None

    def members(self):
        """[(checkpoint or None, transform or None)] in member order"""
        return [(c, T) for c in self.checkpoints for T in self.transforms]

    def load(self, path):
        """restore `path` into the network (runtime.load_state_dict bumps every variable's version, so cached operand planes and
        folded batch-norm epilogues are re-derived); a no-op for None or the checkpoint already loaded"""
        if path is not None and path != self.loaded:
            self.net.restore(path)
            self.loaded = path

    @contextlib.contextmanager
    def preserved(self):
        """every graph variable (and the network's last_restored) put back bit for bit on exit when checkpoints are swapped"""
        if self.checkpoints == [None]:
            yield
            return
        state = rt.state_dict()
        had, last = hasattr(self.net, "last_restored"), getattr(self.net, "last_restored", None)
        try:
            yield
        finally:
            rt.load_state_dict(state, strict=True)
            if had:
                self.net.last_restored = last
            elif hasattr(self.net, "last_restored"):
                del self.net.last_restored
            self.loaded = None


def workspace_bytes(subject, K, num_cls):
    """bytes of an ensemble's score buffer: K x D x 256 x 256 x C fp32"""
    return K * subject.D * preprocess.SIZE * preprocess.SIZE * num_cls * 4


def ensemble_scores(subject, logits_fn, batch_size, num_cls, ensemble):
    """(scores fp32 [K, D, 256, 256, num_cls] on the device, maps fp32 [K, 12] on the device): member k's predict_scores through
    its transform, written into its slice of one buffer after its checkpoint is loaded, and its member_map32"""
    scores = torch.empty((ensemble.K, subject.D, preprocess.SIZE, preprocess.SIZE, num_cls), dtype=torch.float32,
                         device=rt.device())
    maps = []
    for k, (path, T) in enumerate(ensemble.members()):
        ensemble.load(path)
        predict_scores(subject, logits_fn, batch_size, num_cls, T, out=scores[k])
        maps.append(member_map32(subject, T))
    return scores, torch.from_numpy(np.stack(maps)).to(scores.device)


def surface_mm(subject, labels, gt, num_cls, hd_percentile=None):
    """functional.surface_distances of the native prediction against the native ground truth, in mm"""
    return F.surface_distances(labels, gt, num_cls, spacing=native_spacing(subject), hd_percentile=hd_percentile)


def write_prediction(subject, labels, out_dir, num_cls):
    """native_pred/<name>_label.nii.gz: MMWHS codes of the host labels with the image's shape and affine -> its path"""
    path = os.path.join(out_dir, subject.name + "_label.nii.gz")
    nifti.save(label_codes(num_cls)[labels], subject.native_affine, path)
    return path


def check_connectivity(largest_component):
    """None, or the connectivity 6 or 26 of the largest-component post-processing (ValueError otherwise)"""
    if largest_component is not None and (isinstance(largest_component, bool) or largest_component not in CONNECTIVITIES):
        raise ValueError("largest_component must be None, 6 or 26, got %r" % (largest_component,))
    return None if largest_component is None else int(largest_component)


def evaluate_subject(logits_fn, subject, label_path, out_dir, batch_size, num_cls, hd_percentile=None, largest_component=None,
                     ensemble=None):
    """one subject end to end -> dict: subject, dice, jaccard, cm, the surface_distances fields, the prediction's path.
    `subject` is an image path (cropped at its ground-truth heart box: preprocess.Subject(subject, label_path)) or an already built
    preprocess.Subject (e.g. one located by localise.locate).  `label_path` None: nothing is scored, and the dict holds subject,
    path and counts (voxels per class of the written labels) only.
    `largest_component` 6 or 26 keeps only the largest connected component of each class of the native labels (in place, before
    they are scored or written) and adds largest_component, dice_raw (before it), components (in the raw labels), kept and
    removed (voxels), each [num_cls].  `ensemble` (an Ensemble) predicts through its members; with K > 1 the labels are those of
    pnp_native_labels_ensemble and members (K) and dice_first (member 0 alone, without post-processing) are added."""
    largest_component = check_connectivity(largest_component)
    s = subject if isinstance(subject, preprocess.Subject) else preprocess.Subject(subject, label_path)
    scored = label_path is not None
    gt = None
    ens = {}
    if ensemble is None or ensemble.K == 1:
        path, T = (None, None) if ensemble is None else ensemble.members()[0]
        if ensemble is not None:
            ensemble.load(path)
        scores = predict_scores(s, logits_fn, batch_size, num_cls, T)
        gt = ground_truth(label_path) if scored else None
        labels, cm = native_prediction(s, scores, gt, T)
    else:
        logging.info("%s: %d ensemble members, score buffer %.1f MB", s.name, ensemble.K,
                     workspace_bytes(s, ensemble.K, num_cls) / 1e6)
        scores, vmap = ensemble_scores(s, logits_fn, batch_size, num_cls, ensemble)
        gt = ground_truth(label_path) if scored else None
        labels, cm = F.native_labels(scores, vmap, s.native_shape, gt)
        ens = {"members": ensemble.K}
        if scored:
            _, cm_first = F.native_labels(scores[0], vmap[0], s.native_shape, gt)
            cm = cm.cpu().numpy()
            ens["dice_first"] = _dice(cm_first.cpu().numpy())
    del scores
    post = {}
    if largest_component is not None:
        if scored:
            post["dice_raw"] = _dice(cm)
        labels, stats, cm = F.largest_components(labels, num_cls, largest_component, gt=gt, out=labels)
        post.update(stats, largest_component=largest_component)
    if not scored:
        counts = F.label_boxes(labels, num_cls)[:, 0]
        labels = labels.cpu().numpy()
        res = dict(subject=s.name, counts=counts, path=write_prediction(s, labels, out_dir, num_cls))
        res.update(post)
        res.update(ens)
        logging.info("%s: native grid %s, %d prepared frames, voxels per class %s (not scored)", s.name, s.native_shape, s.D,
                     counts.tolist())
        return res
    labels, gt = labels.cpu().numpy(), gt.cpu().numpy()
    res = surface_mm(s, labels, gt, num_cls, hd_percentile)
    res.update(subject=s.name, dice=_dice(cm), jaccard=_jaccard(cm), cm=cm, path=write_prediction(s, labels, out_dir, num_cls))
    res.update(post)
    res.update(ens)
    if largest_component is None:
        logging.info("%s: native grid %s, %d prepared frames, Dice %s", s.name, s.native_shape, s.D, np.round(res["dice"], 4))
    else:
        logging.info("%s: native grid %s, %d prepared frames, Dice %s (largest %d-connected component; raw Dice %s, %s voxels "
                     "removed)", s.name, s.native_shape, s.D, np.round(res["dice"], 4), largest_component,
                     np.round(res["dice_raw"], 4), res["removed"][1:].tolist())
    if ens:
        logging.info("%s: Dice of member 0 alone %s", s.name, np.round(res["dice_first"], 4))
    return res


def locate_subject(logits_fn, image_path, batch_size, num_cls, calibration, ensemble=None):
    """localise.locate on one image with the network as restored (an ensemble's first checkpoint, no transform) -> Located"""
    from . import localise
    if ensemble is not None:
        ensemble.load(ensemble.checkpoints[0])
    return localise.locate(image_path, lambda s: predict_scores(s, logits_fn, batch_size, num_cls), calibration, num_cls)


def located_fields(found, scan_spacing, truth=None):
    """the LOCATE_COLUMNS of a Located (and, with the ground-truth whole-heart box, box_iou and box_err_mm)"""
    from . import localise
    out = {"windows": found.windows, "iterations": found.iterations, "converged": found.converged}
    if truth is not None:
        out["box_iou"] = localise.box_iou(found.subject.box, truth)
        out["box_err_mm"] = localise.face_distance_mm(found.subject.box, truth, scan_spacing)
    return out


def _largest_component(results):
    """the connectivity the subjects' dicts carry (None: none); every subject must carry the same"""
    ks = {r.get("largest_component") for r in results}
    if len(ks) > 1:
        raise ValueError("subjects post-processed with different connectivities: %s" % sorted(ks, key=str))
    return ks.pop() if ks else None


def _members(results):
    """the ensemble size the subjects' dicts carry (None: one member); every subject must carry the same"""
    ks = {r.get("members") for r in results}
    if len(ks) > 1:
        raise ValueError("subjects predicted by ensembles of different sizes: %s" % sorted(ks, key=str))
    return ks.pop() if ks else None


def _located(results):
    """whether the subjects' dicts carry the localisation's fields; every subject must agree"""
    ks = {"windows" in r for r in results}
    if len(ks) > 1:
        raise ValueError("some subjects were located and some were not")
    return ks.pop() if ks else False


def write_csv(path, results, num_cls):
    """one row per subject: subject, then <organ>_<column> for every organ and CSV_COLUMNS entry (NaN: organ absent),
    <organ>_hd<q>_mm when the subjects were scored with a percentile, after all of those <organ>_<column> for every organ and
    COMPONENT_COLUMNS entry when the labels were post-processed to their largest components, and after everything else, for an
    ensemble of K > 1 members, `members` and <organ>_<column> for every organ and ENSEMBLE_COLUMNS entry, then LOCATE_COLUMNS for
    subjects cropped at a located box"""
    names = evaluation._organ_names(num_cls)
    q = evaluation._hd_percentile(results)
    cols = CSV_COLUMNS if q is None else CSV_COLUMNS + (evaluation.pct_name(q) + "_mm",)
    post = _largest_component(results) is not None
    extra = ["%s_%s" % (names[c], k) for c in range(1, num_cls) for k in COMPONENT_COLUMNS] if post else []
    members = _members(results)
    if members is not None:
        extra += ["members"] + ["%s_%s" % (names[c], k) for c in range(1, num_cls) for k in ENSEMBLE_COLUMNS]
    located = _located(results)
    if located:
        extra += list(LOCATE_COLUMNS)
    with open(path, "w") as f:
        f.write(",".join(["subject"] + ["%s_%s" % (names[c], k) for c in range(1, num_cls) for k in cols] + extra) + "\n")
        for r in results:
            row = [str(r["subject"])]
            for c in range(1, num_cls):
                row += [repr(float(r["dice"][c])), repr(float(r["assd"][c])), repr(float(r["hd"][c])), str(int(r["border_pred"][c])),
                        str(int(r["border_gt"][c]))]
                if q is not None:
                    row.append(repr(float(r["hd_pct"][c])))
            if post:
                for c in range(1, num_cls):
                    row += [repr(float(r["dice_raw"][c])), str(int(r["components"][c])), str(int(r["removed"][c]))]
            if members is not None:
                row.append(str(int(r["members"])))
                row += [repr(float(r["dice_first"][c])) for c in range(1, num_cls)]
            if located:
                row += [str(int(r["windows"])), str(int(r["iterations"])), str(bool(r["converged"])), repr(float(r["box_iou"])),
                        repr(float(r["box_err_mm"]))]
            f.write(",".join(row) + "\n")
    return path


def run(logits_fn, pairs, output_path, batch_size, num_cls, hd_percentile=None, largest_component=None, ensemble=None,
        locate=None):
    """every (image, label) pair through evaluate_subject; writes <output_path>/native_pred/*.nii.gz and native.csv, prints the
    per-organ mean and spread of Dice / Jaccard and of ASSD / HD (and the `hd_percentile`-th percentile HD) in mm -> the
    per-subject results.  `largest_component` 6 or 26: every prediction is first reduced to the largest connected component of
    each class (evaluate_subject); the files and printed figures are then those of the post-processed labels.  `ensemble` (an
    Ensemble): every subject is predicted by its members, and every graph variable holds its value from before the call again
    when it returns.  `locate` (a localise.Calibration or its JSON path): every subject is cropped at the box localise.locate finds
    without its labels, which are read only afterwards, to score the prediction and the box (native.csv adds LOCATE_COLUMNS); a
    subject in which nothing is located is logged and left out."""
    largest_component = check_connectivity(largest_component)
    pred_dir = os.path.join(output_path, "native_pred")
    os.makedirs(pred_dir, exist_ok=True)
    if locate is not None:
        from . import localise
        locate = localise.as_calibration(locate)
    if ensemble is not None:
        logging.info("native-grid ensemble: %d checkpoint(s) x %d transform(s) = %d members", len(ensemble.checkpoints),
                     len(ensemble.transforms), ensemble.K)
    results = []
    with (ensemble.preserved() if ensemble is not None else contextlib.nullcontext()):
        for im, lb in pairs:
            if locate is None:
                results.append(evaluate_subject(logits_fn, im, lb, pred_dir, batch_size, num_cls, hd_percentile, largest_component,
                                                ensemble))
                continue
            found = locate_subject(logits_fn, im, batch_size, num_cls, locate, ensemble)
            if found.subject is None:
                logging.error("%s: no heart located; the subject is left out of native.csv", preprocess.subject_name(im))
                continue
            truth = localise.truth_box(found.subject, lb)
            res = evaluate_subject(logits_fn, found.subject, lb, pred_dir, batch_size, num_cls, hd_percentile, largest_component,
                                   ensemble)
            res.update(located_fields(found, found.subject.spacing, truth))
            results.append(res)
    write_csv(os.path.join(output_path, "native.csv"), results, num_cls)
    evaluation.sample_metric_stddev([(r["dice"], r["jaccard"]) for r in results], num_cls)
    evaluation.surface_metric_stddev(results, num_cls, units="mm")
    return results


def write_located_csv(path, results, num_cls):
    """located.csv: subject, windows, iterations, converged, the located coronal box (voxels, then its extent in mm per axis), px,
    D, and per organ the predicted volume in mL (voxels x native voxel volume); a subject in which nothing was located has empty
    box, px, D and volume fields"""
    names = evaluation._organ_names(num_cls)
    axes = ("row", "col", "slice")
    head = (["subject", "windows", "iterations", "converged"] + ["box_%s_%s" % (a, e) for a in axes for e in ("lo", "hi")] +
            ["box_%s_mm" % a for a in axes] + ["px_mm", "D"] + ["%s_ml" % names[c] for c in range(1, num_cls)])
    with open(path, "w") as f:
        f.write(",".join(head) + "\n")
        for r in results:
            row = [str(r["subject"]), str(int(r["windows"])), str(int(r["iterations"])), str(bool(r["converged"]))]
            if r.get("box") is None:
                row += [""] * (len(head) - len(row))
            else:
                row += [str(int(v)) for lohi in r["box"] for v in lohi]
                row += [repr(float(x)) for x in r["box_mm"]]
                row += [repr(float(r["px"])), str(int(r["D"]))]
                row += [repr(float(r["volume_ml"][c])) for c in range(1, num_cls)]
            f.write(",".join(row) + "\n")
    return path


def segment(logits_fn, images, output_path, batch_size, num_cls, calibration, largest_component=None, ensemble=None):
    """unlabelled scans segmented on their own grid: each image is located (localise.locate with `calibration`, a
    localise.Calibration or its JSON path), cropped at the located box and predicted as evaluate_subject predicts a labelled one
    (`largest_component`, `ensemble` as there).  Writes <output_path>/native_pred/<name>_label.nii.gz and located.csv
    (write_located_csv) -> the per-subject dicts.  No label is read."""
    from . import localise
    largest_component = check_connectivity(largest_component)
    calibration = localise.as_calibration(calibration)
    pred_dir = os.path.join(output_path, "native_pred")
    os.makedirs(pred_dir, exist_ok=True)
    results = []
    with (ensemble.preserved() if ensemble is not None else contextlib.nullcontext()):
        for im in images:
            found = locate_subject(logits_fn, im, batch_size, num_cls, calibration, ensemble)
            res = {"subject": preprocess.subject_name(im), "box": None}
            if found.subject is None:
                logging.error("%s: no heart located; nothing written", res["subject"])
            else:
                s = found.subject
                res = evaluate_subject(logits_fn, s, None, pred_dir, batch_size, num_cls, None, largest_component, ensemble)
                res.update(box=s.box, box_mm=[(hi - lo + 1) * s.spacing[a] for a, (lo, hi) in enumerate(s.box)], px=s.px, D=s.D,
                           volume_ml=res["counts"] * float(np.prod(native_spacing(s))) / 1000.0)
            res.update(located_fields(found, None))
            results.append(res)
    write_located_csv(os.path.join(output_path, "located.csv"), results, num_cls)
    return results


def read_images(path):
    """a text file of one image path per line -> [path]; blank lines are skipped"""
    out = []
    with open(path) as f:
        for ln in f:
            parts = ln.split()
            if not parts:
                continue
            if len(parts) != 1:
                raise ValueError("%s: expected one image path per line, got %r" % (path, ln.strip()))
            out.append(parts[0])
    return out


def trainer_ensemble(net, checkpoints, tta, skip_keywords, strip_suffix):
    """the Ensemble of a trainer's test_native(checkpoints=, tta=), or None when both are None (today's single prediction)"""
    if checkpoints is None and tta is None:
        return None
    return Ensemble(net, checkpoints, tta_transforms(tta) if tta is not None else None, skip_keywords, strip_suffix)


def build_trainer(kind, checkpoint, batch_size):
    """the GAN trainer (train_gan.configure("train-gan")) or the segmenter trainer (train_segmenter's configuration), restored
    from `checkpoint` (None: the network keeps its initialisation)"""
    num_cls = 5
    if kind == "gan":
        from . import adversarial as adv
        from . import train_gan
        ck, nc, tc = train_gan.configure("train-gan")
        net = adv.Full_DRN(channels=3, batch_size=batch_size, n_class=num_cls, cost_kwargs=ck, network_config=nc)
        trainer = adv.Trainer(net, num_cls=num_cls, batch_size=batch_size, opt_kwargs=dict(train_gan.opt_kwargs), train_config=tc)
    elif kind == "segmenter":
        from . import source_segmenter as seg
        from . import train_segmenter as ts
        net = seg.Full_DRN(channels=3, n_class=num_cls, batch_size=batch_size, cost_kwargs=dict(ts.cost_kwargs))
        trainer = seg.Trainer(net, None, None, num_cls=num_cls, batch_size=batch_size, optimizer=ts.optimizer,
                              opt_kwargs=dict(ts.opt_kwargs))
    else:
        raise ValueError("trainer must be 'gan' or 'segmenter', got %r" % (kind,))
    if checkpoint is not None:
        net.restore(checkpoint)
    return trainer


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description="segment raw MMWHS subjects on their own voxel grid and score them there in mm")
    ap.add_argument("--trainer", required=True, choices=["gan", "segmenter"])
    ap.add_argument("--checkpoint", required=True, nargs="+", metavar="CKPT",
                    help=".npz checkpoint(s) of that trainer; several are ensembled (their class probabilities summed at every "
                         "native voxel before the argmax; native.csv columns members and <organ>_dice_first)")
    ap.add_argument("--pairs", default=None, help="text file of `image_path label_path` lines (as prepare_data.py reads)")
    ap.add_argument("--images", default=None, metavar="LIST",
                    help="text file of one unlabelled image path per line: segmented without scoring (needs --locate; writes "
                         "located.csv)")
    ap.add_argument("--locate", default=None, metavar="CALIBRATION",
                    help="crop each scan at the heart box the network itself locates (localiser JSON of calibrate_localiser.py) "
                         "instead of the ground-truth box; with --pairs native.csv adds windows, iterations, converged, box_iou "
                         "and box_err_mm")
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch-size", type=int, default=8, help="frames per forward call")
    ap.add_argument("--hd-percentile", type=float, default=None, metavar="Q",
                    help="also score the Q-th percentile Hausdorff distance in mm (95: HD95; native.csv column <organ>_hd<Q>_mm)")
    ap.add_argument("--largest-component", type=int, default=None, choices=CONNECTIVITIES, metavar="{6,26}",
                    help="keep only the largest 6- or 26-connected component of each organ before scoring and writing the "
                         "prediction (native.csv columns <organ>_dice_raw, _components, _removed)")
    ap.add_argument("--tta-rotations", type=float, nargs="+", default=[0.0], metavar="DEG",
                    help="test-time augmentation: in-plane rotations in degrees (within +-%g), combined rotation-major with "
                         "--tta-scales into ensemble members" % preprocess.ROTATION_DEG)
    ap.add_argument("--tta-scales", type=float, nargs="+", default=[1.0], metavar="S",
                    help="test-time augmentation: isotropic in-plane scales (within [%g, %g])" % preprocess.SCALE_RANGE)
    a = ap.parse_args(argv)
    if (a.pairs is None) == (a.images is None):
        ap.error("give exactly one of --pairs and --images")
    if a.images is not None and a.locate is None:
        ap.error("--images needs --locate: an unlabelled scan has no ground-truth box to crop at")
    if a.images is not None and a.hd_percentile is not None:
        ap.error("--hd-percentile scores against labels; --images has none")
    logging.basicConfig(level=logging.INFO)
    tta = [(r, sc, sc, 0.0, 0.0) for r in a.tta_rotations for sc in a.tta_scales]
    check_members(len(a.checkpoint) * len(tta))       # before any work
    transforms = tta_transforms(tta)
    tta = None if len(transforms) == 1 and transforms[0] is None else tta      # the identity alone: today's single prediction
    checkpoints = None if len(a.checkpoint) == 1 else a.checkpoint
    if a.locate is not None:
        from . import localise
        calibration = localise.Calibration.load(a.locate)          # before any work
    trainer = build_trainer(a.trainer, a.checkpoint[0] if checkpoints is None else None, a.batch_size)
    os.makedirs(a.out, exist_ok=True)
    post = {} if a.largest_component is None else {"largest_component": a.largest_component}
    if checkpoints is not None or tta is not None:
        post.update(checkpoints=checkpoints, tta=tta)
    if a.images is not None:
        results = trainer.segment_native(read_images(a.images), a.out, calibration, **post)
        print(os.path.join(a.out, "located.csv"))
        return results
    if a.locate is not None:
        post["locate"] = calibration
    results = trainer.test_native(preprocess.read_pairs(a.pairs), a.out, a.hd_percentile, **post)
    print(os.path.join(a.out, "native.csv"))
    return results
