"""The checks of the heart localisation (localise.py, preprocess.Subject.from_box, pnp_native_accumulate) that need no GPU:
* Subject.from_box at the ground-truth whole-heart box equals Subject(image, label) bit for bit in every attribute but the labels,
  on phantoms stored under several signed axis permutations;
* the calibration equals a direct numpy computation of the definition and round-trips through JSON; a pair without classes 1-4
  raises;
* the seed windows cover every coronal voxel, L_a = n_a included, in the documented order;
* coronal_box maps a native box to heart_box of the coronal mask for all 48 signed permutations; expand_box expands and clamps;
* oracle/accumulate_exact.py equals oracle/ensemble_exact.py for K <= 16 at every case of the ensemble table, and each plausible
  kernel bug (adding the first covering prediction to +0, launching in descending order) changes some output;
* the command line refuses --images without --locate and --hd-percentile with --images before any work."""
import itertools
import json

import numpy as np
import pytest

from oracle import accumulate_exact as A
from oracle import ensemble_exact as E
from tests import mmwhs_phantom as ph

ENS_CASES = [
    ("acc_random_k3_c5", 3, (9, 11, 8), 5, (12, 10, 11), "random", "random"),
    ("acc_full_k2_c2", 2, (8, 9, 7), 2, (11, 12, 10), "random", "full"),
    ("acc_disjoint_k3_c8", 3, (7, 8, 9), 8, (12, 9, 10), "random", "disjoint"),
    ("acc_mixed_k3_c5", 3, (8, 9, 10), 5, (10, 11, 12), "random", ["full", "random", "negative"]),
    ("acc_near_ties_k16_c2", 16, (6, 7, 8), 2, (14, 13, 12), "near_ties", "full"),
    ("acc_nan_k3_c5", 3, (6, 7, 8), 5, (9, 8, 7), "random", ["full", "nan", "random"]),
    ("acc_edges_k2_c5", 2, (6, 7, 5), 5, (7, 8, 11), "random", "edges"),
    ("acc_ties_k2_c5", 2, (8, 9, 10), 5, (12, 13, 11), "ties", "full"),
    ("acc_k1_permuted_c8", 1, (10, 12, 8), 8, (14, 9, 12), "random", "permuted"),
]


@pytest.mark.parametrize("case", ENS_CASES, ids=lambda c: c[0])
def test_accumulator_oracle_equals_the_ensemble_oracle(case):
    tag, K, n, C, m, sk, mk = case
    scores, maps, _ = E.operands(tag, K, n, C, m, sk, mk)
    sums, covered = A.accumulate_ref(scores, maps, m)
    assert np.array_equal(A.labels_ref(sums, covered), E.ensemble_ref(scores, maps, m))


def _signed_zero_case():
    """one prediction sampled at the even voxels of its grid (f = 0 on every axis): class 0 is -0 there and negative at the odd
    neighbours, so every lerp a + 0 (b - a) keeps -0 (0 times a negative difference is -0), and storing the first prediction keeps
    the sign that adding it to the zeroed sums (+0 + -0 = +0) loses"""
    rng = np.random.RandomState(7)
    m, C = (4, 5, 3), 3
    n = tuple(2 * x + 1 for x in m)
    scores = -np.abs(rng.standard_normal((1,) + n + (C,))).astype(np.float32) - np.float32(0.5)
    scores[0, ::2, ::2, ::2, 0] = np.float32(-0.0)
    vmap = np.zeros((1, 3, 4), np.float32)
    for a in range(3):
        vmap[0, a, a] = 2.0
    return scores, vmap.reshape(1, 12), m


def test_mutations_change_some_output():
    scores, maps, m = _signed_zero_case()
    s_ok, c_ok = A.accumulate_ref(scores, maps, m)
    s_bug, _ = A.accumulate_ref(scores, maps, m, add_to_zero=True)
    assert c_ok.all() and np.signbit(s_ok[..., 0]).all() and not np.signbit(s_bug[..., 0]).any()
    changed = 0
    for case in ENS_CASES:
        tag, K, n, C, mm, sk, mk = case
        if K < 2:
            continue
        sc, mp, _ = E.operands(tag, K, n, C, mm, sk, mk)
        s1, c1 = A.accumulate_ref(sc, mp, mm)
        s2, c2 = A.accumulate_ref(sc, mp, mm, descending=True)
        changed += int((s1.view(np.uint32) != s2.view(np.uint32)).sum())
    assert changed > 0


def test_label_boxes_oracle_matches_heart_box():
    from pnp_b200 import preprocess
    rng = np.random.RandomState(3)
    lab = np.zeros((9, 10, 11), np.uint8)
    lab[2:5, 3:9, 1:2] = 2
    lab[7, 0, 10] = 1
    lab[0, 0, 0] = 9                       # >= C: background
    b = A.boxes_ref(lab, 4)
    assert b[3].tolist() == [0, 9, -1, 10, -1, 11, -1]
    assert b[2].tolist() == [18, 2, 4, 3, 8, 1, 1]
    assert b[1].tolist() == [1, 7, 7, 0, 0, 10, 10]
    assert b[0, 0] == lab.size - 19
    box = preprocess.heart_box(lab == 2)
    assert [tuple(b[2, 1 + 2 * a:3 + 2 * a]) for a in range(3)] == box
    del rng


# ---- preprocess.Subject.from_box ------------------------------------------------------------------------------------------
ATTRS = ("name", "coronal_affine", "native_shape", "native_affine", "frame", "spacing", "centre", "px", "D", "j_lo", "j_hi", "p98",
         "mu", "sigma", "reach_px", "lo", "vol", "box")


def _same(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))
    return type(a) == type(b) and a == b


@pytest.mark.parametrize("perm_index", [0, 9, 21, 30, 47])
def test_from_box_at_the_truth_box_equals_the_labelled_subject(tmp_path, perm_index):
    from pnp_b200 import preprocess
    pairs = ph.write_pairs(str(tmp_path), "ct", [61], perms=[ph.SIGNED_PERMUTATIONS[perm_index]], shape=(30, 28, 20),
                           spacing=(0.8, 1.1, 1.7))
    lab = preprocess.Subject(*pairs[0])
    scan = preprocess.Scan(pairs[0][0])
    for got in (preprocess.Subject.from_box(scan, lab.box), preprocess.Subject.from_box(pairs[0][0], lab.box)):
        for k in ATTRS:
            assert _same(getattr(got, k), getattr(lab, k)), k
        assert got.cls.shape == lab.cls.shape and not got.cls.any()
        for j in (1, lab.D // 2):
            assert np.array_equal(got.matrices((j - 1, j, j + 1)), lab.matrices((j - 1, j, j + 1)))
        assert np.array_equal(got.test_affine(), lab.test_affine())


# ---- calibration ---------------------------------------------------------------------------------------------------------
def _numpy_calibration(pairs):
    from pnp_b200 import nifti, preprocess
    rows = []
    for im, lb in pairs:
        img, lab = nifti.load(im), nifti.load(lb)
        raw = np.asarray(lab.get_data())
        perm, flip, _, zooms, _ = preprocess.coronal_frame(img.get_affine(), img.shape)
        s = zooms[perm]
        cor = np.transpose(raw, perm)
        for a in range(3):
            if flip[a]:
                cor = np.flip(cor, a)
        boxes = []
        for mask in (np.isin(cor, preprocess.MMWHS_VALUES), np.isin(cor, list(preprocess.LABEL_TABLE))):
            idx = np.argwhere(mask)
            boxes.append((idx.min(0), idx.max(0)))
        (wl, wh), (fl, fh) = boxes
        rows.append(np.concatenate([(wh - wl + 1) * s, (fl - wl) * s, (wh - fh) * s]))
    return np.median(np.stack(rows), axis=0)


def test_calibration_equals_numpy_and_round_trips(tmp_path):
    from pnp_b200 import localise
    perms = [ph.SIGNED_PERMUTATIONS[i] for i in (3, 17, 40)]
    pairs = ph.write_pairs(str(tmp_path), "mr", [71, 72, 73], perms=perms, shape=(30, 28, 20), spacing=(0.9, 1.0, 1.5))
    cal = localise.calibrate(pairs)
    want = _numpy_calibration(pairs)
    assert np.array_equal(np.concatenate([cal.extent, cal.below, cal.above]), want)
    assert cal.subjects == ["mr_train_1001", "mr_train_1002", "mr_train_1003"]
    path = cal.save(str(tmp_path / "cal.json"))
    with open(path) as f:
        d = json.load(f)
    assert d["count"] == 3
    back = localise.Calibration.load(path)
    for k in ("extent", "below", "above"):
        assert np.array_equal(getattr(back, k), getattr(cal, k))
    assert back.subjects == cal.subjects


def test_calibration_rejects_a_pair_without_the_predicted_structures(tmp_path):
    from pnp_b200 import localise, nifti
    img, lab, aff = ph.ras_subject(5, shape=(20, 18, 12))
    lab[np.isin(lab, list((205, 420, 500, 820)))] = 550
    nifti.save(img, aff, str(tmp_path / "a_image.nii.gz"))
    nifti.save(lab, aff, str(tmp_path / "a_label.nii.gz"))
    with pytest.raises(ValueError, match="classes 1-4"):
        localise.calibrate([(str(tmp_path / "a_image.nii.gz"), str(tmp_path / "a_label.nii.gz"))])


# ---- seed windows, box mapping -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape,spacing,extent", [((40, 36, 30), (0.8, 1.1, 1.7), (20.0, 15.0, 30.0)),
                                                  ((17, 50, 9), (1.0, 0.5, 2.0), (40.0, 7.3, 3.0)),
                                                  ((5, 6, 7), (1.0, 1.0, 1.0), (0.1, 100.0, 3.5))])
def test_seed_windows_cover_every_voxel(shape, spacing, extent):
    from pnp_b200 import localise
    cal = localise.Calibration(extent, (0, 0, 0), (0, 0, 0))
    wins = localise.seed_windows(shape, np.array(spacing), cal)
    cover = np.zeros(shape, np.int64)
    for (a0, b0), (a1, b1), (a2, b2) in wins:
        cover[a0:b0 + 1, a1:b1 + 1, a2:b2 + 1] += 1
    assert cover.min() >= 1
    L = [min(n, max(1, localise.r(e / s))) for n, e, s in zip(shape, extent, spacing)]
    k = [1 if l == n else int(np.ceil(2.0 * (n - l) / l)) + 1 for n, l in zip(shape, L)]
    assert len(wins) == k[0] * k[1] * k[2]
    assert all(w[a][1] - w[a][0] + 1 == L[a] for w in wins for a in range(3))
    starts = [[0] if k[a] == 1 else [localise.r(i * (shape[a] - L[a]) / (k[a] - 1.0)) for i in range(k[a])] for a in range(3)]
    want = [[(s, s + L[a] - 1) for a, s in enumerate(t)] for t in itertools.product(*starts)]    # rows-, columns-, slices-major
    assert wins == want
    if extent[1] == 100.0:
        assert all(w[1] == (0, shape[1] - 1) for w in wins)        # L_a = n_a: one window spanning the axis


def test_coronal_box_of_every_signed_permutation():
    from pnp_b200 import localise, preprocess
    rng = np.random.RandomState(11)
    ras = np.zeros((13, 11, 9), bool)
    ras[3:8, 2:4, 5:9] = True
    ras[rng.randint(3, 8), 6, 1] = True
    aff = np.diag([0.8, 1.1, 1.7, 1.0])
    for perm, signs in ph.SIGNED_PERMUTATIONS:
        stored, A_ = ph.permuted(ras, aff, perm, signs)
        native = [(int(np.flatnonzero(np.any(stored, axis=tuple(b for b in range(3) if b != v)))[0]),
                   int(np.flatnonzero(np.any(stored, axis=tuple(b for b in range(3) if b != v)))[-1])) for v in range(3)]
        frame = preprocess.coronal_frame(A_, stored.shape)[2]
        cor = preprocess.to_coronal(stored, A_)[0]
        assert localise.coronal_box(native, frame) == preprocess.heart_box(cor), (perm, signs)


def test_expand_box_expands_and_clamps():
    from pnp_b200 import localise
    cal = localise.Calibration((0, 0, 0), (2.0, 0.74, 3.4), (1.6, 5.0, 0.0))
    s = np.array([0.8, 1.0, 1.7])
    # r(2.0 / 0.8) = r(2.5) = 3, r(0.74) = 1, r(2.0) = 2; above: r(2.0) = 2, 5, 0
    assert localise.expand_box([(10, 20), (5, 8), (4, 6)], (40, 30, 20), s, cal) == [(7, 22), (4, 13), (2, 6)]
    assert localise.expand_box([(1, 38), (0, 27), (1, 19)], (40, 30, 20), s, cal) == [(0, 39), (0, 29), (0, 19)]


def test_box_iou_and_face_distance():
    from pnp_b200 import localise
    a, b = [(0, 9), (0, 9), (0, 9)], [(5, 14), (0, 9), (0, 9)]
    assert localise.box_iou(a, a) == 1.0 and localise.box_iou(a, b) == 500 / 1500.0
    assert localise.face_distance_mm(a, b, (0.5, 1.0, 1.0)) == 2.5


# ---- command line --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("argv,msg", [
    (["--images", "x"], "--images needs --locate"),
    (["--images", "x", "--locate", "c.json", "--hd-percentile", "95"], "--hd-percentile"),
    (["--pairs", "p", "--images", "x", "--locate", "c.json"], "exactly one of"),
    ([], "exactly one of"),
])
def test_cli_refusals(argv, msg, capsys):
    from pnp_b200 import native
    with pytest.raises(SystemExit):
        native.main(["--trainer", "gan", "--checkpoint", "nothing.npz", "--out", "nowhere"] + argv)
    assert msg in capsys.readouterr().err
