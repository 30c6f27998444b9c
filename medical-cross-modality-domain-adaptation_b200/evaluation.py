"""The per-subject test protocol both reference trainers share (`test_eval` / `sample_metric_stddev`: adversarial.py:993-1084,
source_segmenter.py:572-664): NIfTI subjects in, per-organ Dice / Jaccard mean and spread over subjects out.

The network forward is the caller's (`predict(x[B,256,256,3] on the device, one-hot y) -> (argmax labels, confusion counts)`), so the
adversarial trainer evaluates its adapted CT stream and the segmenter trainer its own graph through the same loop.  Host side only."""
import logging
import os

import numpy as np

from .lib import _dice, _jaccard, _save_nii_prediction, read_nii_image

# label value -> organ name of the console tables (adversarial.py:19-25, source_segmenter.py:20-26)
contour_map = {"bg": 0, "la_myo": 1, "la_blood": 2, "lv_blood": 3, "aa": 4}


def subject_batches(depth, batch_size, shuffle, rng=None):
    """Frame indices of each forward call for one subject of `depth` frames.

    adversarial.py:1021-1030: frames 1 .. depth-2 (each is fed with its two neighbours as channels) in shuffled order, cut into
    floor(depth / batch_size) batches; what does not fill a batch is dropped, and because the list holds depth - 2 frames the last
    batch can come up short (its unused rows stay zero in the reference's feed and are counted in its confusion matrix as
    background-vs-whatever-the-network-says-about-a-zero-image; we do the same).  source_segmenter.py:608-612 walks the frames in order
    (its `range(a : b)` is a syntax error and frame 0 has no left neighbour; the adversarial trainer's frame list is the working form
    of the same loop, so the unshuffled variant of it is used)."""
    frames = list(range(1, depth - 1))
    if shuffle:
        (np.random if rng is None else rng).shuffle(frames)
    return [frames[ii * batch_size:(ii + 1) * batch_size] for ii in range(depth // batch_size)]


def sample_metric_stddev(sample_eval_list, num_cls):
    """adversarial.py:1054-1084 == source_segmenter.py:634-664: per-organ spread and mean over subjects, printed like the reference;
    returns (per-class mean Dice [num_cls], `subject_level_list[:1]`) -- the second value is the reference's slip (row 0 of the
    [num_cls, 2] mean table, i.e. background (Dice, Jaccard), where the per-class Jaccard column `[:, 1]` was meant).  The intended
    column is returned by `subject_level_means`."""
    metric_mat = _metric_mat(sample_eval_list, num_cls)
    print("------- inside the sample_metric_stddev file ---- ")
    for organ, ind in contour_map.items():
        print("organ: %s" % organ)
        print("dice_stddev: %s" % np.std(metric_mat[:, int(ind), 0]))
        print("jaccard_stddev: %s" % np.std(metric_mat[:, int(ind), 1]))
    print("------- inside the sample_metric_stddev file ----  ")
    for organ, ind in contour_map.items():
        print("organ: %s" % organ)
        print("dice_mean: %s" % np.mean(metric_mat[:, int(ind), 0]))
        print("jaccard_mean %s" % np.mean(metric_mat[:, int(ind), 1]))
    print("-------")
    print("all_dice_mean: %s" % np.mean(metric_mat[:, 1:, 0]))
    print("all_jaccard_mean: %s" % np.mean(metric_mat[:, 1:, 1]))
    subject_level_list = np.mean(metric_mat, axis=0)
    return subject_level_list[:, 0], subject_level_list[:1]


def _metric_mat(sample_eval_list, num_cls):
    metric_mat = np.zeros([len(sample_eval_list), num_cls, 2])
    for ii, (dice, jac) in enumerate(sample_eval_list):
        for ind in contour_map.values():
            if int(ind) < num_cls:
                metric_mat[ii, int(ind), 0] = dice[int(ind)]
                metric_mat[ii, int(ind), 1] = jac[int(ind)]
    return metric_mat


def subject_level_means(sample_eval_list, num_cls):
    """(mean Dice per class, mean Jaccard per class) over subjects -- what sample_metric_stddev's return value was meant to be"""
    m = np.mean(_metric_mat(sample_eval_list, num_cls), axis=0)
    return m[:, 0], m[:, 1]


def eval_volume(predict, raw, raw_y, batch_size, num_cls, flip_correction=True, shuffle=True, rng=None, to_device=None):
    """One subject: `raw` [H, W, D] intensities, `raw_y` [H, W, D] integer labels (what read_nii_image returns).
    Returns (per-class Dice, per-class Jaccard, confusion matrix [label, prediction], predicted label volume in the evaluated --
    i.e. flipped, when flip_correction -- orientation)."""
    raw = np.asarray(raw, np.float32)
    raw_y = np.asarray(raw_y)
    if raw.ndim != 3 or raw_y.shape != raw.shape:
        raise ValueError("test subject: image %s and label %s must be equal-shaped 3-D volumes" % (raw.shape, raw_y.shape))
    if flip_correction:
        raw, raw_y = np.flip(np.flip(raw, 0), 1), np.flip(np.flip(raw_y, 0), 1)
    cm = np.zeros([num_cls, num_cls])
    pred_vol = np.zeros(raw_y.shape, np.int64)
    for idx in subject_batches(raw.shape[2], batch_size, shuffle, rng):
        vol = np.zeros((batch_size,) + raw.shape[:2] + (3,), np.float32)
        sl = np.zeros((batch_size,) + raw.shape[:2], np.int64)
        for k, jj in enumerate(idx):
            vol[k] = raw[..., jj - 1:jj + 2]
            sl[k] = raw_y[..., jj]
        pred, counts = predict(vol, sl)
        cm += np.asarray(counts, np.float64)
        for k, jj in enumerate(idx):
            pred_vol[..., jj] = pred[k]
    return _dice(cm), _jaccard(cm), cm, pred_vol


SURFACE_COLUMNS = ("assd", "hd", "asd_pred_gt", "asd_gt_pred", "border_pred", "border_gt")


def surface_distances(pred_vol, gt_vol, num_cls, spacing=None):
    """Per-organ surface distances of one subject on the GPU (functional.surface_distances): a dict of [num_cls] arrays `assd`,
    `hd`, `asd_pred_gt`, `asd_gt_pred` (background and organs absent from either volume: NaN) and the border voxel counts
    `border_pred`, `border_gt`.  Distances are in voxel units unless `spacing` (three voxel sizes) is given, like SIFA's
    evaluation.

    `pred_vol` as `eval_volume` / `Trainer.test_eval_volume` return it is in the evaluated orientation: flipped along both
    in-plane axes when flip_correction is on.  Flip the ground truth the same way before calling, e.g.
    `surface_distances(pred_vol, np.flip(np.flip(raw_y, 0), 1), num_cls)`.  Frames the protocol never predicts (the first and
    last, and any a short batch drops) are background in `pred_vol` and are scored as such."""
    from .functional import surface_distances as _sd
    return _sd(pred_vol, gt_vol, num_cls, spacing)


def _organ_names(num_cls):
    names = {int(v): k for k, v in contour_map.items()}
    return [names.get(c, "class_%d" % c) for c in range(num_cls)]


def surface_metric_stddev(sample_surface_list, num_cls):
    """Per-organ spread and mean of ASSD and HD over subjects, printed in the form of sample_metric_stddev's lines.  Subjects where
    the organ is absent from the prediction or the ground truth (NaN) are left out and counted.  Returns (mean ASSD [num_cls],
    mean HD [num_cls]), NaN where no subject has the organ in both volumes."""
    names = _organ_names(num_cls)
    stats = {}
    for key in ("assd", "hd"):
        mat = np.array([s[key] for s in sample_surface_list], np.float64).reshape(len(sample_surface_list), num_cls)
        stats[key] = [mat[~np.isnan(mat[:, c]), c] for c in range(num_cls)]
    print("------- surface distances over subjects (voxel units) ---- ")
    for c in range(1, num_cls):
        print("organ: %s" % names[c])
        print("assd_stddev: %s" % (np.std(stats["assd"][c]) if len(stats["assd"][c]) else np.nan))
        print("hd_stddev: %s" % (np.std(stats["hd"][c]) if len(stats["hd"][c]) else np.nan))
    print("------- surface distances over subjects (voxel units) ----  ")
    mean = {k: np.full(num_cls, np.nan) for k in ("assd", "hd")}
    for c in range(1, num_cls):
        print("organ: %s" % names[c])
        for key in ("assd", "hd"):
            if len(stats[key][c]):
                mean[key][c] = np.mean(stats[key][c])
        print("assd_mean: %s" % mean["assd"][c])
        print("hd_mean: %s" % mean["hd"][c])
        print("skipped subjects (organ absent from prediction or ground truth): %d" % (len(sample_surface_list) - len(stats["assd"][c])))
    print("-------")
    return mean["assd"], mean["hd"]


def write_surface_csv(path, sample_surface_list, num_cls):
    """one row per subject: subject, then <organ>_<column> for every organ and SURFACE_COLUMNS entry (NaN: organ absent)"""
    names = _organ_names(num_cls)
    with open(path, "w") as f:
        f.write(",".join(["subject"] + ["%s_%s" % (names[c], k) for c in range(1, num_cls) for k in SURFACE_COLUMNS]) + "\n")
        for s in sample_surface_list:
            row = [str(s["subject"])]
            for c in range(1, num_cls):
                row += [str(int(s[k][c])) if k.startswith("border") else repr(float(s[k][c])) for k in SURFACE_COLUMNS]
            f.write(",".join(row) + "\n")
    return path


def run_test_eval(predict, test_label_list, test_nii_list, batch_size, num_cls, output_path, pred_subdir, flip_correction=True,
                  save_result=False, shuffle=True, write_cm=False, rng=None, surface_metrics=False):
    """The subject loop of both `test_eval`s.  Returns (sample_eval_list, summed confusion matrix), and with `surface_metrics`
    a third value: per subject the dict of `surface_distances` plus its "subject" (the image file's name), computed on the
    volumes `save_result` writes -- `pred_vol` against the ground truth in the same orientation, labels above the class range
    as background."""
    pred_folder = os.path.join(output_path, pred_subdir)
    try:
        os.makedirs(pred_folder)
    except OSError:
        logging.info("prediction folder exists")
    if test_label_list is None or test_nii_list is None:
        raise ValueError("test_eval needs test_label_list and test_nii_list (paths of the label / image .nii files)")
    all_cm = np.zeros([num_cls, num_cls])
    sample_eval_list = []
    sample_surface_list = []
    for idx_file, (label_fid, nii_fid) in enumerate(zip(test_label_list, test_nii_list)):
        if not os.path.isfile(nii_fid):
            raise Exception("cannot find sample %s" % str(nii_fid))
        raw = read_nii_image(nii_fid)
        raw_y = read_nii_image(label_fid)
        dice, jac, cm, pred_vol = eval_volume(predict, raw, raw_y, batch_size, num_cls, flip_correction, shuffle, rng)
        logging.info("sample %d (%s): %d frames processed" % (idx_file, os.path.basename(str(nii_fid)), raw.shape[2]))
        all_cm += cm
        sample_eval_list.append((dice, jac))
        gth = np.flip(np.flip(np.asarray(raw_y), 0), 1) if flip_correction else np.asarray(raw_y)
        if save_result:
            _save_nii_prediction(gth.astype(np.int16), pred_vol.astype(np.int16), nii_fid, pred_folder,
                                 out_bname="dense_pred_" + os.path.basename(str(nii_fid)), num_cls=num_cls)
        if surface_metrics:
            sd = surface_distances(pred_vol.astype(np.int16), gth.astype(np.int16), num_cls)
            sd["subject"] = os.path.basename(str(nii_fid))
            sample_surface_list.append(sd)
    if write_cm:
        np.savetxt(os.path.join(output_path, "cm.csv"), all_cm)
    if surface_metrics:
        return sample_eval_list, all_cm, sample_surface_list
    return sample_eval_list, all_cm
