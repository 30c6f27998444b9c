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
* outputs under <out>/: native_pred/<name>_label.nii.gz (int16 MMWHS codes 205 / 420 / 500 / 820 for classes 1-4, 0 elsewhere,
  with the image's shape and affine) and native.csv (one row per subject; <organ>_hd<q>_mm columns when a percentile is asked,
  and <organ>_dice_raw / _components / _removed after all the others with the post-processing).

The crop is the ground-truth heart box, as for the prepared test split: a native-grid score is that of a prediction made inside a
ground-truth region of interest."""
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
CONNECTIVITIES = (6, 26)


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


def input_frames(subject, vol, frames):
    """fp32 [len(frames), 256, 256, 3] on the device: the unaugmented planes (j - 1, j, j + 1) of each frame j, one launch"""
    mats = np.stack([subject.matrices((j - 1, j, j + 1)) for j in frames])
    img, _ = F.resample_planes(vol, None, torch.from_numpy(mats).to(vol.device), preprocess.SIZE, preprocess.SIZE, True, 0)
    return img


def frame_batches(D, batch_size):
    """frames 1 .. D - 2 in ascending order, cut into batches of `batch_size`; the last may be short"""
    frames = list(range(1, D - 1))
    return [frames[at:at + batch_size] for at in range(0, len(frames), batch_size)]


def predict_scores(subject, logits_fn, batch_size, num_cls):
    """fp32 [D, 256, 256, num_cls] on the device: pixel_softmax2 of `logits_fn` (x [B, 256, 256, 3] -> logits [B, 256, 256, C])
    at every frame 1 .. D - 2; frames 0 and D - 1 are background with probability 1"""
    vol, _ = _upload(subject)
    scores = torch.zeros(subject.D, preprocess.SIZE, preprocess.SIZE, num_cls, dtype=torch.float32, device=vol.device)
    scores[0, ..., 0] = 1.0
    scores[subject.D - 1, ..., 0] = 1.0
    with torch.no_grad():
        for part in frame_batches(subject.D, batch_size):
            x = input_frames(subject, vol, part + [part[-1]] * (batch_size - len(part)))
            prob = F.pixel_softmax2(logits_fn(x))
            scores[part[0]:part[-1] + 1] = prob[:len(part)]
    return scores


def ground_truth(label_path):
    """uint8 class ids of the native label volume (preprocess.map_labels), on the device"""
    cls, _, _ = preprocess.map_labels(nifti.load(label_path).get_data())
    return torch.from_numpy(np.ascontiguousarray(cls)).to(rt.device())


def native_prediction(subject, scores, gt):
    """(labels uint8 [native shape] on the device, confusion counts int64 [C, C] on the host): one pnp_native_labels launch"""
    vmap = torch.from_numpy(map32(subject)).to(scores.device)
    labels, cm = F.native_labels(scores, vmap, subject.native_shape, gt)
    return labels, cm.cpu().numpy()


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


def evaluate_subject(logits_fn, image_path, label_path, out_dir, batch_size, num_cls, hd_percentile=None, largest_component=None):
    """one subject end to end -> dict: subject, dice, jaccard, cm, the surface_distances fields, the prediction's path.
    `largest_component` 6 or 26 keeps only the largest connected component of each class of the native labels (in place, before
    they are scored or written) and adds largest_component, dice_raw (before it), components (in the raw labels), kept and
    removed (voxels), each [num_cls]."""
    largest_component = check_connectivity(largest_component)
    s = preprocess.Subject(image_path, label_path)
    scores = predict_scores(s, logits_fn, batch_size, num_cls)
    gt = ground_truth(label_path)
    labels, cm = native_prediction(s, scores, gt)
    del scores
    post = {}
    if largest_component is not None:
        post["dice_raw"] = _dice(cm)
        labels, stats, cm = F.largest_components(labels, num_cls, largest_component, gt=gt, out=labels)
        post.update(stats, largest_component=largest_component)
    labels, gt = labels.cpu().numpy(), gt.cpu().numpy()
    res = surface_mm(s, labels, gt, num_cls, hd_percentile)
    res.update(subject=s.name, dice=_dice(cm), jaccard=_jaccard(cm), cm=cm, path=write_prediction(s, labels, out_dir, num_cls))
    res.update(post)
    if largest_component is None:
        logging.info("%s: native grid %s, %d prepared frames, Dice %s", s.name, s.native_shape, s.D, np.round(res["dice"], 4))
    else:
        logging.info("%s: native grid %s, %d prepared frames, Dice %s (largest %d-connected component; raw Dice %s, %s voxels "
                     "removed)", s.name, s.native_shape, s.D, np.round(res["dice"], 4), largest_component,
                     np.round(res["dice_raw"], 4), res["removed"][1:].tolist())
    return res


def _largest_component(results):
    """the connectivity the subjects' dicts carry (None: none); every subject must carry the same"""
    ks = {r.get("largest_component") for r in results}
    if len(ks) > 1:
        raise ValueError("subjects post-processed with different connectivities: %s" % sorted(ks, key=str))
    return ks.pop() if ks else None


def write_csv(path, results, num_cls):
    """one row per subject: subject, then <organ>_<column> for every organ and CSV_COLUMNS entry (NaN: organ absent),
    <organ>_hd<q>_mm when the subjects were scored with a percentile, and after all of those <organ>_<column> for every organ and
    COMPONENT_COLUMNS entry when the labels were post-processed to their largest components"""
    names = evaluation._organ_names(num_cls)
    q = evaluation._hd_percentile(results)
    cols = CSV_COLUMNS if q is None else CSV_COLUMNS + (evaluation.pct_name(q) + "_mm",)
    post = _largest_component(results) is not None
    extra = ["%s_%s" % (names[c], k) for c in range(1, num_cls) for k in COMPONENT_COLUMNS] if post else []
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
            f.write(",".join(row) + "\n")
    return path


def run(logits_fn, pairs, output_path, batch_size, num_cls, hd_percentile=None, largest_component=None):
    """every (image, label) pair through evaluate_subject; writes <output_path>/native_pred/*.nii.gz and native.csv, prints the
    per-organ mean and spread of Dice / Jaccard and of ASSD / HD (and the `hd_percentile`-th percentile HD) in mm -> the
    per-subject results.  `largest_component` 6 or 26: every prediction is first reduced to the largest connected component of
    each class (evaluate_subject); the files and printed figures are then those of the post-processed labels."""
    largest_component = check_connectivity(largest_component)
    pred_dir = os.path.join(output_path, "native_pred")
    os.makedirs(pred_dir, exist_ok=True)
    results = [evaluate_subject(logits_fn, im, lb, pred_dir, batch_size, num_cls, hd_percentile, largest_component)
               for im, lb in pairs]
    write_csv(os.path.join(output_path, "native.csv"), results, num_cls)
    evaluation.sample_metric_stddev([(r["dice"], r["jaccard"]) for r in results], num_cls)
    evaluation.surface_metric_stddev(results, num_cls, units="mm")
    return results


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
    ap.add_argument("--checkpoint", required=True, help=".npz checkpoint of that trainer")
    ap.add_argument("--pairs", required=True, help="text file of `image_path label_path` lines (as prepare_data.py reads)")
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch-size", type=int, default=8, help="frames per forward call")
    ap.add_argument("--hd-percentile", type=float, default=None, metavar="Q",
                    help="also score the Q-th percentile Hausdorff distance in mm (95: HD95; native.csv column <organ>_hd<Q>_mm)")
    ap.add_argument("--largest-component", type=int, default=None, choices=CONNECTIVITIES, metavar="{6,26}",
                    help="keep only the largest 6- or 26-connected component of each organ before scoring and writing the "
                         "prediction (native.csv columns <organ>_dice_raw, _components, _removed)")
    a = ap.parse_args(argv)
    logging.basicConfig(level=logging.INFO)
    trainer = build_trainer(a.trainer, a.checkpoint, a.batch_size)
    os.makedirs(a.out, exist_ok=True)
    post = {} if a.largest_component is None else {"largest_component": a.largest_component}
    results = trainer.test_native(preprocess.read_pairs(a.pairs), a.out, a.hd_percentile, **post)
    print(os.path.join(a.out, "native.csv"))
    return results
