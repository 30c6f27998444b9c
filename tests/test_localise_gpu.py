"""The heart localisation on the GPU (the kernels' own C-ABI tests are tests/test_native_accumulate_exact_gpu.py):
* localise.locate with an oracle predictor (the ground-truth one-hot labels resampled through each subject's own matrices) on a
  phantom heart embedded off-centre in a larger scan: it converges in <= 3 iterations to the ground-truth whole-heart box within
  one voxel per face, its final labels equal the ground-truth-crop path's where the boxes agree, and the box is the same whether
  the label file is present, absent or swapped;
* end to end with both trainers (seeded weights, output filter scaled): segment_native and test_native(locate=) with a
  two-checkpoint ensemble and the largest-component clean-up, and the command line: native shape and affine, CSV columns, the
  final labels against a fresh prediction at the located box, and every variable restored."""
import csv
import os
import shutil

import numpy as np
import pytest
import torch

from tests import mmwhs_phantom as ph
from tests.models import bn_noise

pytestmark = pytest.mark.gpu


# ---- localisation with an oracle predictor --------------------------------------------------------------------------------
def _embedded_pair(directory, seed, perm, name, body_shape=(56, 48, 34), at=(18, 4, 10)):
    """a phantom heart (tests/mmwhs_phantom.py) embedded off-centre at `at` in a larger body of soft-tissue noise, stored under
    `perm`"""
    from pnp_b200 import nifti
    img, lab, aff = ph.ras_subject(seed, shape=(34, 30, 22), spacing=(0.8, 1.1, 1.7))
    rng = np.random.RandomState(seed + 100)
    body = rng.normal(-30.0, 30.0, body_shape)
    body_lab = np.zeros(body_shape, np.int16)
    sl = tuple(slice(a, a + s) for a, s in zip(at, img.shape))
    body[sl] = img
    body_lab[sl] = lab
    ri, A_ = ph.permuted(body.astype(np.int16), aff, *perm)
    rl, _ = ph.permuted(body_lab, aff, *perm)
    ip, lp = os.path.join(directory, name + "_image.nii.gz"), os.path.join(directory, name + "_label.nii.gz")
    nifti.save(ri, A_, ip)
    nifti.save(rl, A_, lp)
    return ip, lp


def _oracle_predict(scan, label_path, C):
    """predict(subject) -> one-hot fp32 [D, 256, 256, C] of the ground-truth classes resampled through the subject's own matrices
    (the labelled crop of the same box: vol, px, D and the matrices equal the subject's)"""
    from pnp_b200 import functional as F
    from pnp_b200 import preprocess
    probe = preprocess.Subject.__new__(preprocess.Subject)
    probe._geometry(scan)
    cls_all, _ = probe._labels(scan, label_path)

    def predict(s):
        lab = preprocess.Subject.__new__(preprocess.Subject)
        lab._geometry(scan)
        lab._crop(scan, cls_all, s.box, preprocess.MARGIN, s.reach_px)
        assert np.array_equal(lab.vol, s.vol)
        mats = torch.from_numpy(np.stack([lab.matrices((j,)) for j in range(s.D)])).cuda()
        _, l = F.resample_planes(None, torch.from_numpy(lab.cls).cuda(), mats, preprocess.SIZE, preprocess.SIZE, False, 1)
        return torch.nn.functional.one_hot(l, C).float().contiguous()
    return predict


@pytest.mark.parametrize("perm_index", [5, 27, 44])
def test_locate_with_an_oracle_predictor(tmp_path, perm_index):
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F
    from pnp_b200 import localise, native, preprocess
    C = 5
    ip, lp = _embedded_pair(str(tmp_path), 81, ph.SIGNED_PERMUTATIONS[perm_index], "ct_train_1001")
    cal = localise.calibrate([(ip, lp)])
    scan = preprocess.Scan(ip)
    truth = preprocess.Subject(ip, lp)
    found = localise.locate(scan, _oracle_predict(scan, lp, C), cal, C)
    print("  perm %d: located" % perm_index, flush=True)
    assert found.subject is not None and found.converged and found.iterations <= 3, (found.boxes, found.iterations)
    assert found.windows > 1
    box = found.subject.box
    assert all(abs(box[a][e] - truth.box[a][e]) <= 1 for a in range(3) for e in range(2)), (box, truth.box)
    print("  perm %d: %d windows, %d iterations, boxes %s, truth %s" % (perm_index, found.windows, found.iterations, found.boxes,
                                                                        truth.box))
    # at the truth box the final labels are the ground-truth-crop path's, bit for bit
    at_truth = preprocess.Subject.from_box(scan, truth.box)
    pred = _oracle_predict(scan, lp, C)
    a, _ = F.native_labels(pred(at_truth), torch.from_numpy(native.map32(at_truth)).cuda(), at_truth.native_shape)
    b, _ = F.native_labels(pred(truth), torch.from_numpy(native.map32(truth)).cuda(), truth.native_shape)
    assert torch.equal(a, b)
    if [tuple(x) for x in box] == [tuple(x) for x in truth.box]:
        c, _ = F.native_labels(pred(found.subject), torch.from_numpy(native.map32(found.subject)).cuda(), truth.native_shape)
        assert torch.equal(c, b)
    # the label file is never read: absent (the image alone in another directory) or swapped, the box is the same
    alone = tmp_path / "alone"
    alone.mkdir()
    shutil.copy(ip, str(alone / os.path.basename(ip)))
    again = localise.locate(str(alone / os.path.basename(ip)), _oracle_predict(scan, lp, C), cal, C)
    assert again.boxes == found.boxes
    os.replace(lp, str(tmp_path / "moved.nii.gz"))
    _, other = _embedded_pair(str(tmp_path / "alone"), 82, ph.SIGNED_PERMUTATIONS[perm_index], "other")
    os.replace(other, lp)
    third = localise.locate(scan, _oracle_predict(preprocess.Scan(ip), str(tmp_path / "moved.nii.gz"), C), cal, C)
    assert third.boxes == found.boxes


# ---- end to end ----------------------------------------------------------------------------------------------------------
B = 3
NUM_CLS = 5
CODES = {0: 0, 205: 1, 420: 2, 500: 3, 820: 4}


def _logits_fn(trainer, kind):
    return trainer._ct_logits if kind == "gan" else trainer._logits


def _scaled_checkpoint(kind, P, pair, path):
    """P with its output filter scaled so that the largest |logit| on a few frames of `pair` is 20, saved to `path`"""
    from pnp_b200 import native, preprocess, prepare_data
    np.savez(path, **P)
    trainer = native.build_trainer(kind, path, B)
    s = preprocess.Subject(*pair)
    vol, _ = prepare_data._upload(s)
    with torch.no_grad():
        big = max(float(_logits_fn(trainer, kind)(native.input_frames(s, vol, [j, j + 1, j + 2])).abs().max())
                  for j in (1, s.D // 3, s.D // 2, s.D - 4))
    P = dict(P)
    P["output/Variable"] = (P["output/Variable"] * np.float32(20.0 / big)).astype(np.float32)
    np.savez(path, **P)
    return path


@pytest.mark.parametrize("kind", ["gan", "segmenter"])
def test_end_to_end(tmp_path, kind):
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F
    from pnp_b200 import localise, native, nifti, preprocess
    from pnp_b200 import runtime as rt
    from oracle.pnp_graphs import OracleAdversarial, OracleSegmenter, init_numpy_params
    rt.set_conv_backend("auto")
    pairs = [_embedded_pair(str(tmp_path), 91, ph.SIGNED_PERMUTATIONS[12 if kind == "gan" else 33], "ct_train_1001",
                            body_shape=(42, 38, 28), at=(8, 1, 5))]
    cal_path = localise.calibrate(pairs).save(str(tmp_path / "localiser.json"))
    oracle = OracleAdversarial if kind == "gan" else OracleSegmenter
    ws, bns = oracle.layout()
    ckpts = []
    for seed in (3, 4):
        P = init_numpy_params(ws, bns, seed, 0.05)
        bn_noise(P, bns, seed + 10)
        ckpts.append(_scaled_checkpoint(kind, P, pairs[0], str(tmp_path / ("%s_%d.npz" % (kind, seed)))))
    trainer = native.build_trainer(kind, ckpts[0], B)
    before = rt.state_dict()
    seg_dir, run_dir = str(tmp_path / "seg"), str(tmp_path / "run")
    print("  %s: segment_native" % kind, flush=True)
    seg = trainer.segment_native([p[0] for p in pairs], seg_dir, cal_path, largest_component=26, checkpoints=ckpts)
    print("  %s: windows %s, iterations %s; test_native(locate=)" % (kind, [r["windows"] for r in seg],
                                                                     [r["iterations"] for r in seg]), flush=True)
    res = trainer.test_native(pairs, run_dir, largest_component=26, checkpoints=ckpts, locate=cal_path)
    after = rt.state_dict()
    assert before.keys() == after.keys() and all(np.array_equal(before[k].view(np.uint8), after[k].view(np.uint8)) for k in before), \
        "variables not restored"
    with open(os.path.join(seg_dir, "located.csv")) as f:
        rows = list(csv.DictReader(f))
    assert [r["subject"] for r in rows] == ["ct_train_1001"]
    assert list(rows[0])[:4] == ["subject", "windows", "iterations", "converged"] and list(rows[0])[-4:] == [
        "la_myo_ml", "la_blood_ml", "lv_blood_ml", "aa_ml"]
    with open(os.path.join(run_dir, "native.csv")) as f:
        head = f.readline().strip().split(",")
    assert head[-5:] == list(native.LOCATE_COLUMNS) and "members" in head
    assert len(res) == len(seg)
    fresh = native.build_trainer(kind, ckpts[0], B)
    for (ip, lp), r, row in zip(pairs, seg, rows):
        assert r.get("box") is not None, "nothing located in %s" % ip
        img = nifti.load(ip)
        out = nifti.load(r["path"])
        assert tuple(out.shape) == tuple(img.shape) and np.array_equal(out.get_affine(), img.get_affine())
        got = np.vectorize(CODES.get)(np.asarray(out.get_data())).astype(np.uint8)
        assert int(row["box_row_lo"]) == r["box"][0][0] and int(row["D"]) == r["D"]
        counts = np.bincount(got.reshape(-1), minlength=NUM_CLS)
        vox_ml = float(np.prod(native.native_spacing(preprocess.Subject.from_box(ip, r["box"])))) / 1000.0
        assert np.allclose([float(row[k]) for k in ("la_myo_ml", "la_blood_ml", "lv_blood_ml", "aa_ml")], counts[1:] * vox_ml)
        # a fresh ensemble prediction at the located box, through the same path, agrees on >= 99.99 % of voxels
        s = preprocess.Subject.from_box(ip, r["box"])
        ens = native.Ensemble(fresh.net, ckpts, None, native.SLOT_KEYWORDS + (("cls",) if kind == "gan" else ()), kind == "gan")
        with ens.preserved():
            scores, vmap = native.ensemble_scores(s, _logits_fn(fresh, kind), B, NUM_CLS, ens)
        labels, _ = F.native_labels(scores, vmap, s.native_shape)
        labels, _, _ = F.largest_components(labels, NUM_CLS, 26, out=labels)
        agree = float((labels.cpu().numpy() == got).mean())
        assert agree >= 0.9999, (ip, agree)
    print("  %s: fresh prediction agrees; command line" % kind, flush=True)
    # the command line: --images (unscored) and --pairs --locate (scored)
    img_list = str(tmp_path / "images")
    with open(img_list, "w") as f:
        f.write("".join(p[0] + "\n" for p in pairs))
    cli_dir = str(tmp_path / "cli")
    native.main(["--trainer", kind, "--checkpoint", ckpts[0], "--images", img_list, "--locate", cal_path, "--out", cli_dir,
                 "--batch-size", str(B), "--largest-component", "26"])
    assert os.path.exists(os.path.join(cli_dir, "located.csv"))
    assert sorted(os.listdir(os.path.join(cli_dir, "native_pred"))) == ["ct_train_1001_label.nii.gz"]
