"""Native-grid ensembles (native.Ensemble, Trainer.test_native(checkpoints=, tta=), evaluate_native.py --checkpoint A B
--tta-rotations ...) end to end on seeded phantom subjects (tests/mmwhs_phantom.py) under two signed axis permutations, with both
trainers and two seeded checkpoints each (their output filter scaled so that no logit overflows the softmax):
* the test-time input frames equal pnp_resample_planes of subject.matrices(.., T) bit for bit;
* the native labels equal oracle/ensemble_exact.py applied to the pipeline's own [K] score buffer and fp32 maps, bit for bit, and
  the written file holds exactly those labels; the kernel's Dice equals numpy Dice of the written file exactly; dice_first equals
  the Dice of native_labels(scores[0]) of the same run;
* each member's score slice agrees with a fresh trainer restored from that checkpoint alone and predicting through that
  transform on >= 99.99 % of argmax pixels (not bit for bit: the split-K atomics) -- stale cached operands after a checkpoint
  swap would break this;
* every trainer variable is bit-identical before and after test_native(checkpoints=..);
* a checkpoint lacking an inference variable, an out-of-range transform and K > 16 each raise before any prediction;
* the command line writes the added columns and only MMWHS codes, composed with --largest-component 26 --hd-percentile 95."""
import csv
import os

import numpy as np
import pytest
import torch

from oracle import ensemble_exact as E
from oracle import native_exact as N
from tests import mmwhs_phantom as ph
from tests.models import bn_noise

pytestmark = pytest.mark.gpu
B = 3
NUM_CLS = 5
CODES = {0, 205, 420, 500, 820}
TTA = [(-10.0, 1.0, 1.0, 0.0, 0.0), (0.0, 1.0, 1.0, 0.0, 0.0), (7.5, 1.05, 0.95, 2.0, -3.0)]
ORGANS = ("la_myo", "la_blood", "lv_blood", "aa")


def _logits_fn(trainer, kind):
    return trainer._ct_logits if kind == "gan" else trainer._logits


def _scaled_checkpoint(kind, P, pair, path):
    """P with its output filter scaled so that the largest |logit| on a few frames of `pair` is 20 (the softmax does not subtract
    the maximum; the output layer has no bias, so the logits scale with it), saved to `path`"""
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


@pytest.fixture(scope="module")
def phantoms(tmp_path_factory):
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt
    from oracle.pnp_graphs import OracleAdversarial, OracleSegmenter, init_numpy_params
    rt.set_conv_backend("auto")
    d = tmp_path_factory.mktemp("ensemble")
    perms = [ph.SIGNED_PERMUTATIONS[i] for i in (9, 30)]
    pairs = ph.write_pairs(str(d), "ct", [51, 52], perms=perms, shape=(40, 36, 30), spacing=(0.8, 1.1, 1.7))
    pair_file = str(d / "pairs")
    with open(pair_file, "w") as f:
        f.write("".join("%s %s\n" % p for p in pairs))
    ckpt = {}
    for kind, oracle in (("gan", OracleAdversarial), ("segmenter", OracleSegmenter)):
        ws, bns = oracle.layout()
        ckpt[kind] = []
        for seed in (3, 4):
            P = init_numpy_params(ws, bns, seed, 0.05)
            bn_noise(P, bns, seed + 10)
            ckpt[kind].append(_scaled_checkpoint(kind, P, pairs[0], str(d / ("%s_%d.npz" % (kind, seed)))))
    return {"dir": d, "pairs": pairs, "pair_file": pair_file, "ckpt": ckpt}


def _classes(codes_vol):
    from pnp_b200 import native
    out = np.zeros(codes_vol.shape, np.uint8)
    for c, v in enumerate(native.label_codes(NUM_CLS).tolist()):
        if c:
            out[codes_vol == v] = c
    return out


def _dice(pred, gt):
    return np.array([2.0 * ((pred == c) & (gt == c)).sum() / ((pred == c).sum() + (gt == c).sum())
                     if ((pred == c).sum() + (gt == c).sum()) else 0.0 for c in range(NUM_CLS)])


def test_tta_input_frames_equal_resample_planes_of_the_transformed_matrices(phantoms):
    from pnp_b200 import functional as F, native, preprocess, prepare_data
    s = preprocess.Subject(*phantoms["pairs"][0])
    vol, _ = prepare_data._upload(s)
    frames = [1, s.D // 2, s.D - 2]
    assert torch.equal(native.input_frames(s, vol, frames, None), native.input_frames(s, vol, frames))
    for T in native.tta_transforms(TTA):
        x = native.input_frames(s, vol, frames, T)
        mats = torch.from_numpy(np.stack([s.matrices((j - 1, j, j + 1), T) for j in frames])).cuda()
        want, _ = F.resample_planes(vol, None, mats, preprocess.SIZE, preprocess.SIZE, True, 0)
        assert torch.equal(x.view(torch.int32), want.view(torch.int32))


@pytest.mark.parametrize("kind", ["gan", "segmenter"])
def test_ensemble_end_to_end(phantoms, kind, tmp_path, monkeypatch):
    from pnp_b200 import functional as F, native, nifti, preprocess, runtime as rt
    from pnp_b200.lib import _dice as kernel_dice
    A, Bk = phantoms["ckpt"][kind]
    trainer = native.build_trainer(kind, A, B)
    before = rt.state_dict()
    # ---- record the pipeline's own native_labels calls (the [K] score buffer, the maps, scores[0]) -----------------------
    calls = []
    real = F.native_labels

    def recording(scores, vmap, shape, gt=None, out=None):
        labels, cm = real(scores, vmap, shape, gt, out)
        calls.append((scores.cpu().numpy(), vmap.cpu().numpy(), tuple(shape), labels.cpu().numpy(),
                      None if cm is None else cm.cpu().numpy()))
        return labels, cm

    monkeypatch.setattr(F, "native_labels", recording)
    out = str(tmp_path / "out")
    results = trainer.test_native(phantoms["pairs"], out, checkpoints=[A, Bk], tta=TTA)
    monkeypatch.setattr(F, "native_labels", real)
    K = 2 * len(TTA)
    # ---- every variable is back, bit for bit -------------------------------------------------------------------------------
    after = rt.state_dict()
    assert sorted(after) == sorted(before)
    for k in before:
        assert np.array_equal(after[k].view(np.uint8), before[k].view(np.uint8)), k
    assert len(calls) == 2 * len(phantoms["pairs"])
    for i, ((im, lb), res) in enumerate(zip(phantoms["pairs"], results)):
        s = preprocess.Subject(im, lb)
        gt = preprocess.map_labels(nifti.load(lb).get_data())[0]
        (sc, vm, shape, labels, cm), (sc0, vm0, _, _, cm0) = calls[2 * i], calls[2 * i + 1]
        assert sc.shape == (K, s.D, 256, 256, NUM_CLS) and vm.shape == (K, 12) and res["members"] == K
        # the maps are the members' fp32 maps, checkpoint-major and transform-minor
        Ts = native.tta_transforms(TTA) * 2
        assert np.array_equal(vm, np.stack([native.member_map32(s, T) for T in Ts]))
        # the labels are the oracle's on the pipeline's own buffer, and the written file holds them
        want = E.ensemble_ref(sc, vm, shape)
        assert np.array_equal(labels, want), "%s: %d labels differ" % (s.name, int((labels != want).sum()))
        assert np.array_equal(cm, N.confusion_ref(want, gt, NUM_CLS))
        written = nifti.load(res["path"])
        assert set(np.unique(written.get_data()).tolist()) <= CODES
        pred = _classes(written.get_data())
        assert np.array_equal(pred, labels)
        assert np.array_equal(res["dice"], _dice(pred, gt))
        # dice_first: member 0 alone, from the same run's scores[0]
        assert np.array_equal(sc0, sc[0]) and np.array_equal(vm0, vm[0])
        first = N.labels_ref(sc[0], vm[0], shape)
        assert np.array_equal(res["dice_first"], kernel_dice(N.confusion_ref(first, gt, NUM_CLS)))
        print("  %s %s: K %d, Dice %s, member 0 alone %s" % (kind, s.name, K, np.round(res["dice"][1:], 4),
                                                            np.round(res["dice_first"][1:], 4)))
    with open(os.path.join(out, "native.csv")) as f:
        header = next(csv.reader(f))
    assert header[-5:] == ["members"] + ["%s_dice_first" % o for o in ORGANS]
    # ---- each member against a fresh trainer restored from its checkpoint alone -------------------------------------------------
    sc = calls[0][0]
    s = preprocess.Subject(*phantoms["pairs"][0])
    agree = [0, 0]
    Ts = native.tta_transforms(TTA)
    for c, path in enumerate((A, Bk)):
        fresh = native.build_trainer(kind, path, B)
        for t, T in enumerate(Ts):
            mine = native.predict_scores(s, _logits_fn(fresh, kind), B, NUM_CLS, T).cpu().numpy()
            agree[0] += int((mine.argmax(3) == sc[c * len(Ts) + t].argmax(3)).sum())
            agree[1] += mine[..., 0].size
    print("  %s: member scores agree with fresh trainers on %d of %d pixels" % (kind, agree[0], agree[1]))
    assert agree[0] >= 0.9999 * agree[1]


@pytest.mark.parametrize("kind", ["gan", "segmenter"])
def test_bad_members_raise_before_any_prediction(phantoms, kind, tmp_path):
    from pnp_b200 import native, runtime as rt
    A, Bk = phantoms["ckpt"][kind]
    trainer = native.build_trainer(kind, A, B)
    P = dict(np.load(A))
    victim = next(n for n in rt.graph.order if "cls" not in n and n in P)
    del P[victim]
    lacking = str(tmp_path / "lacking.npz")
    np.savez(lacking, **P)
    out = tmp_path / "out"
    with pytest.raises(ValueError, match=victim):
        trainer.test_native(phantoms["pairs"], str(out), checkpoints=[A, lacking])
    with pytest.raises(ValueError, match="training range"):
        trainer.test_native(phantoms["pairs"], str(out), tta=[(0.0, 1.0, 1.0, 0.0, 0.0), (20.0, 1.0, 1.0, 0.0, 0.0)])
    with pytest.raises(ValueError, match="1 to 16 members"):
        trainer.test_native(phantoms["pairs"], str(out), checkpoints=[A, Bk, A], tta=[(float(t), 1.0, 1.0, 0.0, 0.0)
                                                                                    for t in range(-12, 13, 4)])
    assert not out.exists()
    if kind == "gan":       # the critics are not needed for a prediction
        P = {k: v for k, v in np.load(A).items() if "cls" not in k}
        no_critics = str(tmp_path / "no_critics.npz")
        np.savez(no_critics, **P)
        native.Ensemble(trainer.net, [A, no_critics], None, native.SLOT_KEYWORDS + ("cls",))
    # TF-style keys 'x:0': the GAN trainer's restore loads them as x (through its relaxed branch, which leaves the critics
    # alone -- a prediction does not read them), the segmenter trainer's loads nothing from them, so only the GAN trainer may
    # take such a checkpoint as a member
    suffixed = str(tmp_path / "suffixed.npz")
    np.savez(suffixed, **{k + ":0": v for k, v in np.load(A).items()})
    if kind == "gan":
        trainer.net.restore(A)
        want = rt.state_dict()
        trainer.net.restore(Bk)
        trainer.net.restore(suffixed)
        got = rt.state_dict()
        assert all(np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)) for k in want if "cls" not in k)
        assert native.trainer_ensemble(trainer.net, [Bk, suffixed], None, native.SLOT_KEYWORDS + ("cls",), True).K == 2
    else:
        with pytest.raises(ValueError, match="lacks"):
            trainer.test_native(phantoms["pairs"], str(out), checkpoints=[A, suffixed])
        assert not out.exists()


@pytest.mark.parametrize("kind", ["gan", "segmenter"])
def test_command_line_ensemble(phantoms, kind, tmp_path):
    from pnp_b200 import native, preprocess
    A, Bk = phantoms["ckpt"][kind]
    cli = str(tmp_path / "cli")
    native.main(["--trainer", kind, "--checkpoint", A, Bk, "--pairs", phantoms["pair_file"], "--out", cli, "--batch-size", str(B),
                 "--tta-rotations", "-10", "0", "10", "--largest-component", "26", "--hd-percentile", "95"])
    with open(os.path.join(cli, "native.csv")) as f:
        rows = list(csv.reader(f))
    cols = native.CSV_COLUMNS + ("hd95_mm",)
    want = (["subject"] + ["%s_%s" % (o, k) for o in ORGANS for k in cols] +
            ["%s_%s" % (o, k) for o in ORGANS for k in native.COMPONENT_COLUMNS] + ["members"] +
            ["%s_dice_first" % o for o in ORGANS])
    assert rows[0] == want
    assert [r[0] for r in rows[1:]] == [preprocess.subject_name(im) for im, _ in phantoms["pairs"]]
    assert all(r[rows[0].index("members")] == "6" for r in rows[1:])
    for name in os.listdir(os.path.join(cli, "native_pred")):
        from pnp_b200 import nifti
        assert set(np.unique(nifti.load(os.path.join(cli, "native_pred", name)).get_data()).tolist()) <= CODES
