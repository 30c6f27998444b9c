"""Native-grid segmentation and scoring (native.py, evaluate_native.py) end to end on seeded phantom subjects (tests/mmwhs_phantom.py)
stored under three signed axis permutations with anisotropic spacing, with both trainers restored from small seeded checkpoints:
* the device input frames equal the planes of prepare_data.test_volume bit for bit;
* the native labels equal oracle/native_exact.py applied to the pipeline's own score volume and fp32 map, bit for bit, and the
  kernel's confusion counts are np.bincount's;
* the kernel's Dice equals numpy Dice of the written NIfTI against the native ground truth exactly; ASSD / HD equal
  oracle/surface_exact.py with the native spacing to 1e-13 relative; the file has the image's shape and affine bit for bit and
  only MMWHS codes;
* on the frames test_eval_volume predicts, the argmax of the new path agrees with the reference protocol on >= 99.99 % of pixels
  (not bit-equal: batch composition changes the order of the wgmma split-K atomics), with the output filter scaled so that no
  logit overflows the reference's softmax;
* one-hot prepared ground truth fed as scores: every native voxel whose eight trilinear taps carry one class gets that class."""
import csv
import os

import numpy as np
import pytest
import torch

from tests import mmwhs_phantom as ph
from tests.models import bn_noise

pytestmark = pytest.mark.gpu
B = 3
NUM_CLS = 5
CODES = {0, 205, 420, 500, 820}


@pytest.fixture(scope="module")
def phantoms(tmp_path_factory):
    import pnp_b200  # noqa: F401
    from oracle.pnp_graphs import OracleAdversarial, OracleSegmenter, init_numpy_params
    d = tmp_path_factory.mktemp("native")
    perms = [ph.SIGNED_PERMUTATIONS[i] for i in (5, 22, 41)]
    pairs = ph.write_pairs(str(d), "ct", [41, 42, 43], perms=perms, shape=(40, 36, 30), spacing=(0.8, 1.1, 1.7))
    pair_file = str(d / "pairs")
    with open(pair_file, "w") as f:
        f.write("".join("%s %s\n" % p for p in pairs))
    ckpt = {}
    for kind, oracle in (("gan", OracleAdversarial), ("segmenter", OracleSegmenter)):
        ws, bns = oracle.layout()
        P = init_numpy_params(ws, bns, 0, 0.05)
        bn_noise(P, bns, 6)
        ckpt[kind] = str(d / ("%s.npz" % kind))
        np.savez(ckpt[kind], **P)
    return {"dir": d, "pairs": pairs, "pair_file": pair_file, "ckpt": ckpt}


def test_input_frames_equal_the_test_volume(phantoms):
    from pnp_b200 import native, preprocess, prepare_data
    for pair in phantoms["pairs"]:
        s = preprocess.Subject(*pair)
        vol, _ = prepare_data._upload(s)
        frames = [1, 2, s.D // 2, s.D - 2]
        x = native.input_frames(s, vol, frames).cpu().numpy()
        img, _ = prepare_data.test_volume(s)
        for i, j in enumerate(frames):
            assert np.array_equal(x[i].view(np.int32), np.ascontiguousarray(img[:, :, j - 1:j + 2]).view(np.int32)), (s.name, j)


def _classes(codes_vol):
    lut = {v: c for c, v in enumerate(native_codes())}
    out = np.zeros(codes_vol.shape, np.uint8)
    for v, c in lut.items():
        out[codes_vol == v] = c
    return out


def native_codes():
    from pnp_b200 import native
    return native.label_codes(NUM_CLS).tolist()


def _logits_fn(trainer, kind):
    return trainer._ct_logits if kind == "gan" else trainer._logits


def _moderate_checkpoint(kind, path, pair, out_path):
    """the checkpoint with its output filter scaled so that the largest |logit| on a few frames of `pair` is 20: the reference's
    pixel_wise_softmax_2 does not subtract the maximum, so a logit above ~88 overflows exp() and its clipped NaN moves the
    argmax -- seeded random weights reach that, trained ones do not; the output layer has no bias, so the logits scale with it"""
    from pnp_b200 import native, preprocess, prepare_data
    trainer = native.build_trainer(kind, path, B)
    s = preprocess.Subject(*pair)
    vol, _ = prepare_data._upload(s)
    with torch.no_grad():
        big = max(float(_logits_fn(trainer, kind)(native.input_frames(s, vol, [j, j + 1, j + 2])).abs().max())
                  for j in (1, s.D // 3, s.D // 2, s.D - 4))
    P = dict(np.load(path))
    P["output/Variable"] = (P["output/Variable"] * np.float32(20.0 / big)).astype(np.float32)
    np.savez(out_path, **P)
    print("  %s: largest |logit| %.3g on the seeded weights, output filter scaled by %.3g" % (kind, big, 20.0 / big))
    return out_path


@pytest.mark.parametrize("kind", ["gan", "segmenter"])
def test_native_evaluation(phantoms, kind, tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import evaluation, native, nifti, preprocess, prepare_data, runtime as rt
    from oracle import native_exact as N
    from oracle import surface_exact as se
    rt.set_conv_backend("auto")
    ckpt = _moderate_checkpoint(kind, phantoms["ckpt"][kind], phantoms["pairs"][0], str(tmp_path / "moderate.npz"))
    # ---- the command line: native_pred/*.nii.gz and native.csv ------------------------------------------------------------
    cli = str(tmp_path / "cli")
    native.main(["--trainer", kind, "--checkpoint", ckpt, "--pairs", phantoms["pair_file"], "--out", cli,
                 "--batch-size", str(B)])
    with open(os.path.join(cli, "native.csv")) as f:
        rows = list(csv.reader(f))
    names = [preprocess.subject_name(im) for im, _ in phantoms["pairs"]]
    assert rows[0] == ["subject"] + ["%s_%s" % (o, k) for o in ("la_myo", "la_blood", "lv_blood", "aa") for k in native.CSV_COLUMNS]
    assert [r[0] for r in rows[1:]] == names
    assert sorted(os.listdir(os.path.join(cli, "native_pred"))) == sorted(n + "_label.nii.gz" for n in names)
    # ---- the trainer's entry point, checked piece by piece -------------------------------------------------------------------
    trainer = native.build_trainer(kind, ckpt, B)
    out = str(tmp_path / "out")
    results = trainer.test_native(phantoms["pairs"], out)
    logits_fn = _logits_fn(trainer, kind)
    agree_total = [0, 0]
    for (im, lb), res in zip(phantoms["pairs"], results):
        s = preprocess.Subject(im, lb)
        image = nifti.load(im)
        gt = preprocess.map_labels(nifti.load(lb).get_data())[0]
        # the written file: the image's shape and affine bit for bit, MMWHS codes only
        written = nifti.load(res["path"])
        assert written.shape == image.shape and written.get_data().dtype == np.int16
        assert np.array_equal(written.get_affine().view(np.int64), image.get_affine().view(np.int64))
        assert set(np.unique(written.get_data()).tolist()) <= CODES
        pred = _classes(written.get_data())
        # Dice of the kernel's counts == numpy Dice of the written file, exactly
        want_dice = np.array([2.0 * ((pred == c) & (gt == c)).sum() / max(1, (pred == c).sum() + (gt == c).sum())
                              if ((pred == c).sum() + (gt == c).sum()) else 0.0 for c in range(NUM_CLS)])
        assert np.array_equal(res["dice"], want_dice), (res["dice"], want_dice)
        assert res["cm"].sum() == gt.size
        # ASSD / HD in mm against the scipy oracle with the native spacing
        sp = native.native_spacing(s)
        ref = se.surface_metrics(pred, gt, NUM_CLS, sp)
        for key in ("assd", "hd"):
            np.testing.assert_allclose(res[key], ref[key], rtol=1e-13, atol=0, equal_nan=True)
        assert np.array_equal(res["border_pred"], ref["border_pred"]) and np.array_equal(res["border_gt"], ref["border_gt"])
        print("  %s %s: native %s, D %d, Dice %s, ASSD mm %s" % (kind, s.name, s.native_shape, s.D, np.round(res["dice"][1:], 4),
                                                            np.round(res["assd"][1:], 3)))
        # the kernel on the pipeline's own score volume and map == the oracle, bit for bit
        scores = native.predict_scores(s, logits_fn, B, NUM_CLS)
        gt_dev = native.ground_truth(lb)
        labels, cm = native.native_prediction(s, scores, gt_dev)
        sc = scores.cpu().numpy()
        want = N.labels_ref(sc, native.map32(s), s.native_shape)
        assert np.array_equal(labels.cpu().numpy(), want), "%s: %d labels differ" % (s.name, int((labels.cpu().numpy() != want).sum()))
        assert np.array_equal(cm, N.confusion_ref(want, gt, NUM_CLS))
        assert (sc[0, ..., 0] == 1).all() and (sc[-1, ..., 0] == 1).all() and not sc[[0, -1], ..., 1:].any()
        # the reference protocol's frames: its argmax against the new path's
        img, lab = prepare_data.test_volume(s)
        stored_img, stored_lab = img[::-1, ::-1], lab[::-1, ::-1]
        if kind == "gan":
            seed = 5
            _, _, _, pv = trainer.test_eval_volume(stored_img, stored_lab, flip_correction=True, shuffle_seed=seed)
            batches = evaluation.subject_batches(s.D, B, True, np.random.RandomState(seed))
        else:
            _, _, _, pv = trainer.test_eval_volume(stored_img, stored_lab, flip_correction=True)
            batches = evaluation.subject_batches(s.D, B, False)
        assert np.isfinite(sc).all() and sc.min() >= 0
        top = sc.argmax(3)
        for j in sum(batches, []):
            agree_total[0] += int((pv[:, :, j] == top[j]).sum())
            agree_total[1] += top[j].size
        # the ground-truth round trip: one-hot prepared labels as scores
        onehot = np.eye(NUM_CLS, dtype=np.float32)[np.transpose(lab, (2, 0, 1))]
        rt_labels, _ = native.native_prediction(s, torch.from_numpy(onehot).cuda(), gt_dev)
        rt_labels = rt_labels.cpu().numpy()
        u = N.coords(native.map32(s), s.native_shape)
        ok = N.inside(u, onehot.shape[:3])
        taps = []
        for a in range(3):
            n = onehot.shape[a]
            x = np.fmin(np.fmax(u[a], np.float32(0)), np.float32(n - 1))
            i0 = np.floor(x).astype(np.int64)
            taps.append((i0, np.minimum(i0 + 1, n - 1)))
        cls = np.transpose(lab, (2, 0, 1))
        corners = np.stack([cls[taps[0][a], taps[1][b], taps[2][c]] for a in (0, 1) for b in (0, 1) for c in (0, 1)])
        single = ok & (corners == corners[0]).all(0)
        assert np.array_equal(rt_labels[single], corners[0][single]) and not rt_labels[~ok].any()
        print("    round trip: %d of %d native voxels have one class on all eight taps; agreement with the native ground truth %.4f"
              % (int(single.sum()), single.size, float((rt_labels == gt).mean())))
    agree = agree_total[0] / agree_total[1]
    print("  %s: the native path's argmax agrees with test_eval_volume on %d of %d pixels (%.6f)" % (
        kind, agree_total[0], agree_total[1], agree))
    assert agree >= 0.9999
