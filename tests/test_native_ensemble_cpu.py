"""The checks of native-grid ensembling (pnp_native_labels_ensemble, native.Ensemble, preprocess.tta_transform) that need no GPU:
* oracle/ensemble_exact.py: each plausible kernel bug (members summed in descending k, sums divided by the cover count, coverage
  decided by member 0 alone, FMA-contracted coordinates) changes some output of the case table; at K = 1 it is
  oracle/native_exact.py's labels_ref on every score and map kind; two identical members label as one member, bit for bit
  (2 v is exact);
* native.member_map: the identity gives voxel_map bit for bit; for all 48 signed axis permutations of a phantom and several
  in-range transforms T, the member map followed by T takes every native voxel to voxel_map's un-augmented coordinate to 1e-9;
* preprocess.tta_transform reproduces augment_transform's matrices from the same draws bit for bit and rejects values outside
  the training ranges; the ensemble's host checks (member count, transform tuples, CSV columns)."""
import csv
import math

import numpy as np
import pytest

from oracle import ensemble_exact as E
from oracle import native_exact as N
from tests import mmwhs_phantom as ph

F32 = np.float32

# (tag, K, score grid n, C, native grid m, score kind, map kind(s))
CASES = [
    ("random_k3_c5", 3, (9, 11, 8), 5, (12, 10, 11), "random", "random"),
    ("full_k2_c2", 2, (8, 9, 7), 2, (11, 12, 10), "random", "full"),
    ("disjoint_k3_c8", 3, (7, 8, 9), 8, (12, 9, 10), "random", "disjoint"),
    ("mixed_k3_c5", 3, (8, 9, 10), 5, (10, 11, 12), "random", ["full", "random", "negative"]),
    ("near_ties_k3_c2", 3, (10, 12, 9), 2, (24, 22, 20), "near_ties", "full"),
    ("near_ties_random_k2_c2", 2, (12, 14, 10), 2, (30, 28, 26), "near_ties", "random"),
    ("near_ties_k16_c2", 16, (6, 7, 8), 2, (14, 13, 12), "near_ties", "full"),
    ("nan_member_k3_c5", 3, (6, 7, 8), 5, (9, 8, 7), "random", ["full", "nan", "random"]),
    ("edges_k2_c5", 2, (6, 7, 5), 5, (7, 8, 11), "random", "edges"),
    ("ties_k2_c5", 2, (8, 9, 10), 5, (12, 13, 11), "ties", "full"),
]
SINGLE_KINDS = [("random", "random"), ("random", "permuted"), ("random", "negative"), ("ties", "random"),
                ("near_ties", "random"), ("random", "edges"), ("random", "nan"), ("random", "full")]


def _case(tag):
    return next(c for c in CASES if c[0] == tag)


def _operands(case):
    tag, K, n, C, m, sk, mk = case
    return E.operands(tag, K, n, C, m, sk, mk)


MUTATIONS = {
    "members summed in descending k": dict(reverse=True),
    "sums divided by the cover count": dict(divide=True),
    "coverage of member 0 alone": dict(first_cover=True),
    "FMA-contracted coordinates": dict(fma=True),
}


@pytest.mark.parametrize("bug", list(MUTATIONS), ids=[k.replace(" ", "_") for k in MUTATIONS])
def test_each_mutation_changes_some_output(bug):
    d = 0
    for case in CASES:
        scores, maps, _ = _operands(case)
        d += int((E.ensemble_ref(scores, maps, case[4]) != E.ensemble_ref(scores, maps, case[4], **MUTATIONS[bug])).sum())
    print("  MUTATION %-34s %d differing labels" % (bug, d))
    assert d >= 1


@pytest.mark.parametrize("kinds", SINGLE_KINDS, ids=lambda k: "%s_%s" % k)
@pytest.mark.parametrize("C", [2, 5, 8])
def test_one_member_is_labels_ref(kinds, C):
    sk, mk = kinds
    scores, maps, _ = E.operands("one_%s_%s_%d" % (sk, mk, C), 1, (7, 9, 8), C, (10, 9, 11), sk if C >= 5 or sk != "ties" else
                                 "random", mk)
    want = N.labels_ref(scores[0], maps[0], (10, 9, 11))
    assert np.array_equal(E.ensemble_ref(scores, maps, (10, 9, 11)), want)


@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_two_identical_members_label_as_one(case):
    scores, maps, _ = _operands(case)
    m = case[4]
    for k in range(case[1]):
        one = E.ensemble_ref(scores[k:k + 1], maps[k:k + 1], m)
        two = E.ensemble_ref(np.stack([scores[k], scores[k]]), np.stack([maps[k], maps[k]]), m)
        assert np.array_equal(one, two), (case[0], k)


def test_coverage_and_known_answers():
    """disjoint members: each voxel takes the label of the one member covering it; a member that covers nothing (NaN map) does
    not change the labels of the others"""
    case = _case("disjoint_k3_c8")
    scores, maps, _ = _operands(case)
    m = case[4]
    got = E.ensemble_ref(scores, maps, m)
    cover = [N.inside(N.coords(maps[k], m), scores.shape[1:4]) for k in range(3)]
    assert not (cover[0] & cover[1]).any() and not (cover[1] & cover[2]).any() and not (cover[0] & cover[2]).any()
    assert all(c.any() for c in cover)
    for k in range(3):
        alone = N.labels_ref(scores[k], maps[k], m)
        assert np.array_equal(got[cover[k]], alone[cover[k]])
    assert not got[~(cover[0] | cover[1] | cover[2])].any()
    case = _case("nan_member_k3_c5")
    scores, maps, _ = _operands(case)
    m = case[4]
    assert not N.inside(N.coords(maps[1], m), scores.shape[1:4]).any()
    keep = [0, 2]
    assert np.array_equal(E.ensemble_ref(scores, maps, m), E.ensemble_ref(scores[keep], maps[keep], m))


# ------------------------------------------------------------------------------------------------
# the host side: member maps, test-time transforms, checks and columns
# ------------------------------------------------------------------------------------------------
def _subjects(tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import preprocess
    for i, (perm, signs) in enumerate(ph.SIGNED_PERMUTATIONS):
        d = tmp_path / ("p%02d" % i)
        d.mkdir()
        (pair,) = ph.write_pairs(str(d), "ct", [37], perms=[(perm, signs)], shape=(28, 25, 17), spacing=(0.8, 0.95, 1.5))
        yield preprocess.Subject(*pair)


def test_member_maps_compose_with_their_transform_for_all_48_signed_permutations(tmp_path):
    from pnp_b200 import native, preprocess
    transforms = [preprocess.tta_transform(10.0), preprocess.tta_transform(-15.0, (0.9, 1.1), (3.0, -10.0)),
                  preprocess.tta_transform(4.5, (1.05, 0.95)), preprocess.tta_transform(0.0, (1.1, 1.1), (-2.5, 0.0))]
    count = 0
    for s in _subjects(tmp_path):
        V = native.voxel_map(s)
        assert np.array_equal(native.member_map(s).view(np.int64), V.view(np.int64))
        assert np.array_equal(native.member_map(s, np.eye(3)).view(np.int64), V.view(np.int64))
        assert np.array_equal(native.member_map32(s, None).view(np.int32), native.map32(s).view(np.int32))
        vox = np.array([[i, j, k, 1.0] for i in range(0, s.native_shape[0], 3) for j in range(0, s.native_shape[1], 4)
                        for k in range(0, s.native_shape[2], 2)]).T
        base = V @ vox
        for T in transforms:
            Mk = native.member_map(s, T)
            assert np.array_equal(Mk[0], V[0])                  # the slice coordinate does not move
            p = Mk @ vox                                        # member (slice, row, column)
            back = T @ np.vstack([p[1:3], np.ones(p.shape[1])])  # the member's pixel through T: the un-augmented pixel
            assert np.abs(back[:2] - base[1:3]).max() <= 1e-9, s.name
            assert native.member_map32(s, T).dtype == np.float32
            assert np.array_equal(native.member_map32(s, T), Mk.astype(F32).reshape(-1))
        count += 1
    assert count == 48


def test_tta_transform_is_augment_transform_of_the_same_draws():
    import pnp_b200  # noqa: F401
    from pnp_b200 import preprocess as P
    for seed in range(20):
        a, b = np.random.RandomState(seed), np.random.RandomState(seed)
        got = P.augment_transform(a)
        th = b.uniform(-P.ROTATION_DEG, P.ROTATION_DEG)
        s = b.uniform(P.SCALE_RANGE[0], P.SCALE_RANGE[1], 2)
        t = b.uniform(-P.SHIFT_PX, P.SHIFT_PX, 2)
        assert np.array_equal(got.view(np.int64), P.tta_transform(th, s, t).view(np.int64))
        # the composition augment_transform has always used, written out
        r = np.deg2rad(th)
        A = np.array([[math.cos(r), -math.sin(r)], [math.sin(r), math.cos(r)]]) @ np.diag(s)
        want = np.eye(3)
        want[:2, :2] = A
        want[:2, 2] = P.CENTRE + t - A @ np.array([P.CENTRE, P.CENTRE])
        assert np.array_equal(got.view(np.int64), want.view(np.int64))
        assert np.array_equal(got.view(np.int64), P.tta_transform(th, tuple(s), tuple(t)).view(np.int64))
        assert a.uniform() == b.uniform()                       # the same number of draws
    assert np.array_equal(P.tta_transform(0.0), np.eye(3))
    for bounds in ((15.0, (1.1, 0.9), (10.0, -10.0)), (-15.0, (0.9, 1.1), (-10.0, 10.0))):
        P.tta_transform(*bounds)
    for bad in ((15.5,), (-16.0,), (float("nan"),), (0.0, (0.89, 1.0)), (0.0, (1.0, 1.11)), (0.0, (1.0, 1.0), (10.5, 0.0)),
                (0.0, (1.0, 1.0), (0.0, -11.0)), (0.0, (float("nan"), 1.0))):
        with pytest.raises(ValueError):
            P.tta_transform(*bad)


def test_member_count_and_transform_checks():
    import pnp_b200  # noqa: F401
    from pnp_b200 import native
    assert native.MAX_MEMBERS == 16
    assert native.check_members(1) == 1 and native.check_members(16) == 16
    for K in (0, 17):
        with pytest.raises(ValueError):
            native.check_members(K)
    Ts = native.tta_transforms([(0, 1, 1, 0, 0), (10, 1, 1, 0, 0), (0, 1.1, 1.1, 0, 0)])
    assert Ts[0] is None and Ts[1].shape == (3, 3) and Ts[2].shape == (3, 3)
    with pytest.raises(ValueError):
        native.tta_transforms([(20, 1, 1, 0, 0)])
    with pytest.raises(ValueError):
        native.tta_transforms([(0, 1, 1)])


def test_cli_rejects_too_many_members_before_any_work(tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import native
    # 2 checkpoints x 3 rotations x 3 scales = 18 members: refused before the checkpoints or the pairs are read
    with pytest.raises(ValueError, match="1 to 16 members"):
        native.main(["--trainer", "gan", "--checkpoint", "a.npz", "b.npz", "--pairs", str(tmp_path / "none"), "--out",
                     str(tmp_path / "o"), "--tta-rotations", "-5", "0", "5", "--tta-scales", "0.95", "1", "1.05"])
    with pytest.raises(ValueError, match="training range"):
        native.main(["--trainer", "gan", "--checkpoint", "a.npz", "--pairs", str(tmp_path / "none"), "--out",
                     str(tmp_path / "o"), "--tta-rotations", "30"])
    assert not (tmp_path / "o").exists()


def test_csv_columns_of_an_ensemble(tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import native
    C = 5
    r = dict(subject="s1", dice=np.linspace(0, 1, C), assd=np.ones(C), hd=np.ones(C), border_pred=np.arange(C),
             border_gt=np.arange(C), largest_component=26, dice_raw=np.ones(C) * 0.5,
             components=np.arange(C), removed=np.arange(C), members=8, dice_first=np.ones(C) * 0.25)
    path = native.write_csv(str(tmp_path / "native.csv"), [r], C)
    with open(path) as f:
        rows = list(csv.reader(f))
    organs = ("la_myo", "la_blood", "lv_blood", "aa")
    base = ["subject"] + ["%s_%s" % (o, k) for o in organs for k in native.CSV_COLUMNS]
    post = ["%s_%s" % (o, k) for o in organs for k in native.COMPONENT_COLUMNS]
    assert rows[0] == base + post + ["members"] + ["%s_dice_first" % o for o in organs]
    assert rows[1][len(base) + len(post)] == "8" and [float(x) for x in rows[1][-4:]] == [0.25] * 4
    plain = {k: v for k, v in r.items() if k not in ("members", "dice_first")}
    with open(native.write_csv(str(tmp_path / "plain.csv"), [plain], C)) as f:
        assert next(csv.reader(f)) == base + post


class _Recorder(object):
    """stands in for a trainer: records the arguments test_native is called with"""

    def __init__(self, log, kind, checkpoint, batch_size):
        log.append(("build", kind, checkpoint, batch_size))
        self.log = log

    def test_native(self, pairs, out, hd_percentile=None, **kw):
        self.log.append(("test_native", pairs, hd_percentile, kw))
        return []


@pytest.mark.parametrize("args, built_from, want", [
    (["--checkpoint", "A.npz", "--tta-rotations", "10"], "A.npz", dict(checkpoints=None, tta=[(10.0, 1.0, 1.0, 0.0, 0.0)])),
    (["--checkpoint", "A.npz", "--tta-scales", "0.95"], "A.npz", dict(checkpoints=None, tta=[(0.0, 0.95, 0.95, 0.0, 0.0)])),
    (["--checkpoint", "A.npz", "B.npz", "--tta-rotations", "5"], None,
     dict(checkpoints=["A.npz", "B.npz"], tta=[(5.0, 1.0, 1.0, 0.0, 0.0)])),
    (["--checkpoint", "A.npz", "B.npz"], None, dict(checkpoints=["A.npz", "B.npz"], tta=None)),
    (["--checkpoint", "A.npz", "--tta-rotations", "0", "0"], "A.npz",
     dict(checkpoints=None, tta=[(0.0, 1.0, 1.0, 0.0, 0.0)] * 2)),
    (["--checkpoint", "A.npz", "--tta-rotations", "-10", "10", "--tta-scales", "0.9", "1"], "A.npz",
     dict(checkpoints=None, tta=[(-10.0, 0.9, 0.9, 0.0, 0.0), (-10.0, 1.0, 1.0, 0.0, 0.0), (10.0, 0.9, 0.9, 0.0, 0.0),
                                 (10.0, 1.0, 1.0, 0.0, 0.0)])),
    (["--checkpoint", "A.npz"], "A.npz", {}),
    (["--checkpoint", "A.npz", "--tta-rotations", "0", "--tta-scales", "1"], "A.npz", {}),
], ids=["one_rotation", "one_scale", "two_checkpoints_one_rotation", "two_checkpoints", "identity_twice", "product", "plain",
        "explicit_identity"])
def test_cli_members_reach_the_trainer(tmp_path, monkeypatch, args, built_from, want):
    """every valid combination of --checkpoint, --tta-rotations and --tta-scales reaches test_native with its members (a single
    non-identity transform included); one checkpoint and the identity alone is today's call"""
    import pnp_b200  # noqa: F401
    from pnp_b200 import native
    log = []
    monkeypatch.setattr(native, "build_trainer", lambda kind, ck, bs: _Recorder(log, kind, ck, bs))
    pairs = tmp_path / "pairs"
    pairs.write_text("")
    native.main(["--trainer", "segmenter", "--pairs", str(pairs), "--out", str(tmp_path / "o"), "--batch-size", "4"] + args)
    assert log == [("build", "segmenter", built_from, 4), ("test_native", [], None, want)]


def test_checkpoint_check_counts_what_restore_loads(tmp_path):
    """a key 'x:0' stores variable x only where the trainer's restore strips the suffix (the GAN trainer's); for the segmenter
    trainer, whose restore loads exact names only, such a checkpoint lacks x"""
    import torch
    import pnp_b200  # noqa: F401
    from pnp_b200 import native, runtime as rt
    saved = dict(rt.graph.__dict__)
    try:
        rt.reset_default_graph()
        with rt.variable_scope("group_1"):
            for name in ("w", "bn/gamma", "Adam_state"):
                rt.get_variable(name, lambda: torch.zeros(2))
        with rt.variable_scope("cls_1"):
            rt.get_variable("w", lambda: torch.zeros(2))
        plain, suffixed = str(tmp_path / "plain.npz"), str(tmp_path / "suffixed.npz")
        np.savez(plain, **{"group_1/w": np.zeros(2), "group_1/bn/gamma": np.zeros(2)})
        np.savez(suffixed, **{"group_1/w:0": np.zeros(2), "group_1/bn/gamma": np.zeros(2)})
        assert native.checkpoint_missing(plain, native.SLOT_KEYWORDS) == ["cls_1/w"]
        assert native.checkpoint_missing(plain, native.SLOT_KEYWORDS + ("cls",)) == []
        assert native.checkpoint_missing(suffixed, native.SLOT_KEYWORDS + ("cls",), strip_suffix=True) == []
        assert native.checkpoint_missing(suffixed, native.SLOT_KEYWORDS + ("cls",), strip_suffix=False) == ["group_1/w"]
        with pytest.raises(ValueError, match="group_1/w"):
            native.Ensemble(None, [plain, suffixed], None, native.SLOT_KEYWORDS + ("cls",), strip_suffix=False)
        assert native.Ensemble(None, [plain, suffixed], None, native.SLOT_KEYWORDS + ("cls",), strip_suffix=True).K == 2
    finally:
        rt.graph.__dict__.clear()
        rt.graph.__dict__.update(saved)
