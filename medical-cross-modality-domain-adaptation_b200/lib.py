"""The reference's lib.py: the helpers that sit on the hot path (one-hot feed, Dice evaluation), the confusion-matrix Dice / Jaccard
of the per-subject evaluation, and the NIfTI I/O of the test protocol (lib.py:31-72) on the in-tree NIfTI-1 reader / writer
(`nifti.py`; `nibabel` is absent from this image)."""
import os

import numpy as np
import torch

from . import functional as F
from . import nifti


def _read_lists(fid):
    """lib.py:7-20: read a text file of paths, one per line (lines shorter than 3 chars skipped); None when the file is absent."""
    if not os.path.isfile(fid):
        return None
    with open(fid, 'r') as fd:
        lines = fd.readlines()
    return [ln.split('\n')[0] for ln in lines if len(ln) >= 3]


def _label_decomp(num_cls, label_vol):
    """lib.py:75-92: one-hot of an integer label map.  Accepts numpy (host, like the reference) or a torch
    tensor (stays on its device).  Returns float32 [..., num_cls]."""
    if isinstance(label_vol, np.ndarray):
        return np.stack([(label_vol == i) for i in range(num_cls)], axis=-1).astype(np.float32)
    return F.one_hot(label_vol, num_cls)


def _dice_eval(logits_or_pred, labels, n_class):
    """lib.py:96-110: hard Dice of argmax prediction vs one-hot labels, background included.
    Takes the logits (or the softmax map -- same argmax) [B,H,W,C]; returns (mean dice, per-class list)
    as device tensors computed from the confusion matrix kernel."""
    cm = F.confusion_counts(logits_or_pred, labels).to(torch.float64)
    inse = torch.diagonal(cm)
    union = cm.sum(0) + cm.sum(1)
    arr = 2.0 * inse / (union + 1e-7)
    return arr.mean(), [arr[i] for i in range(n_class)]


def _jaccard(conf_matrix):
    """lib.py:121-135"""
    cm = np.asarray(conf_matrix, dtype=np.float64)
    pp, gp, hit = cm.sum(0), cm.sum(1), np.diag(cm)
    den = pp + gp - hit
    return np.where(den == 0, 0.0, hit / np.where(den == 0, 1.0, den))


def _dice(conf_matrix):
    """lib.py:138-152"""
    cm = np.asarray(conf_matrix, dtype=np.float64)
    pp, gp, hit = cm.sum(0), cm.sum(1), np.diag(cm)
    den = pp + gp
    return np.where(den == 0, 0.0, 2.0 * hit / np.where(den == 0, 1.0, den))


def _indicator_eval(cm):
    """lib.py:155-175: print per-organ Dice / Jaccard from a confusion matrix."""
    contour_map = {"bg": 0, "la_myo": 1, "la_blood": 2, "lv_blood": 3, "aa": 4}
    dice, jaccard = _dice(cm), _jaccard(cm)
    print(cm)
    for organ, ind in contour_map.items():
        print("organ: %s" % organ)
        print("dice: %s" % dice[int(ind)])
        print("jaccard: %s" % jaccard[int(ind)])
    return dice, jaccard


def _inverse_lookup(my_dict, _value):
    """lib.py:113-118: first key whose value equals `_value`, else None"""
    for key, dic_value in list(my_dict.items()):
        if dic_value == _value:
            return key
    return None


def read_nii_image(input_fid):
    """lib.py:64-67: the voxel array of a .nii / .nii.gz file (what `nib.load(fid).get_data()` returns)"""
    return nifti.load(input_fid).get_data()


def read_nii_object(input_fid):
    """lib.py:69-72: the loaded volume object (get_data(), get_affine(), header)"""
    return nifti.load(input_fid)


def write_nii(array_data, filename, path="", affine=None):
    """lib.py:47-62: write an array as NIfTI-1; without an affine the identity is used (and said so, like the reference)"""
    if affine is None:
        print("No information about the global coordinate system")
        affine = np.diag([1, 1, 1, 1])
    save_fid = os.path.join(path, filename)
    try:
        nifti.save(array_data, affine, save_fid)
        print("Nii object %s has been saved!" % save_fid)
    except Exception:
        raise Exception("file %s cannot be saved!" % save_fid)
    return save_fid


def _save_nii_prediction(gth, comp_pred, ref_fid, out_folder, out_bname, debug=False, num_cls=5):
    """lib.py:31-45: prediction and ground truth of one subject as .nii.gz next to each other, in the reference volume's world
    coordinates.  The reference's body reads `self.num_cls` inside this free function (a NameError, lib.py:43); the intent --
    labels above the class range count as background in the saved ground truth -- is kept with an explicit `num_cls`."""
    ref_affine = read_nii_object(ref_fid).get_affine()
    out_bname = out_bname.split(".")[0] + ".nii.gz"
    pred_fid = write_nii(comp_pred, out_bname, out_folder, affine=ref_affine)
    _local_gth = np.array(gth, copy=True)
    _local_gth[_local_gth > num_cls - 1] = 0
    gth_fid = write_nii(_local_gth, "gth_" + out_bname, out_folder, affine=ref_affine)
    return pred_fid, gth_fid


def _save(state, model_path, global_step=None):
    """lib.py:23-29 analogue: variables keyed by TF names in one .npz (the checkpoint naming contract)."""
    path = model_path if global_step is None else "%s-%d" % (model_path, int(global_step))
    tmp = "%s.tmp.%d.npz" % (path, os.getpid())
    np.savez(tmp, **state)            # a reader (or a second writer) never sees a half-written checkpoint
    os.replace(tmp, path + ".npz")
    return path + ".npz"


def save_checkpoint(trainer, save_path, output_path):
    """both trainers' save: trainer.checkpoint_state() as <save_path>-<global_step>.npz and <output_path>/latest.npz, written by
    rank 0 while every rank waits.  A trainer with a weights' moving average (trainer.ema) also gets the averaged-weights
    checkpoints <save_path>-<global_step>_ema.npz and <output_path>/latest_ema.npz (ema.averaged_weights), which every
    consumer of a checkpoint reads as it reads the others"""
    from . import runtime as rt
    from .ema import averaged_weights
    st = trainer.checkpoint_state()
    avg = averaged_weights(st, rt.graph.order) if getattr(trainer, "ema", None) is not None else None

    def write():
        _save(st, save_path, global_step=trainer.global_step)
        _save(st, os.path.join(output_path, "latest"))
        if avg is not None:
            _save(avg, "%s-%d_ema" % (save_path, int(trainer.global_step)))
            _save(avg, os.path.join(output_path, "latest_ema"))
    trainer.dp.save_checkpoint(write)
