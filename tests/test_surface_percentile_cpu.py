"""The percentile Hausdorff distance (HD95 at q = 95) on the host: the pooled-percentile oracle of oracle/surface_percentile.py in its
scipy and brute-force forms against each other and against known answers, the plain restatement of numpy's `linear` percentile
that pnp_surface_distance_pct implements against np.percentile itself, the argument checks of the C-ABI entry point (which
return before any launch) and of the host layer, and the hd<q> columns of the test protocol's tables.  The kernels are tested
on the GPU in tests/test_surface_percentile_exact_gpu.py."""
import ctypes
import math
import os

import numpy as np
import pytest

from oracle import surface_exact as se
from oracle import surface_percentile as spc

QS = (0.0, 12.5, 50.0, 95.0, 99.0, 100.0)


def _ellipsoids(rng, shape, num_cls):
    g = np.ogrid[:shape[0], :shape[1], :shape[2]]
    v = np.zeros(shape, np.int64)
    for c in range(1, num_cls):
        centre = rng.uniform(-0.2, 1.2, 3) * shape
        radii = rng.uniform(0.15, 0.8, 3) * np.array(shape) + 0.5
        v[sum(((g[a] - centre[a]) / radii[a]) ** 2 for a in range(3)) < 1] = c
    return v


def test_scipy_and_brute_force_percentiles_agree_bit_for_bit_at_unit_spacing():
    rng = np.random.default_rng(95)
    for it in range(60):
        shape = tuple(int(x) for x in rng.integers(1, 12, 3))
        C = int(rng.integers(2, 7))
        if it % 2:
            p = rng.integers(0, C + 2, shape) * (rng.random(shape) < rng.random())
            g = rng.integers(0, C + 2, shape) * (rng.random(shape) < rng.random())
        else:
            p, g = _ellipsoids(rng, shape, C), _ellipsoids(rng, shape, C)
        for q in QS:
            a, b = spc.hd_percentile(p, g, C, q), spc.hd_percentile(p, g, C, q, form="brute")
            assert a.tobytes() == b.tobytes(), (it, q, a, b)
        sd, bp, bg = spc.scipy_distances(p, g, C)
        bd = spc.brute_distances(p, g, C)[0]
        for c in range(1, C):
            if sd[c][0] is None:
                assert bd[c] == (None, None) and not (bp[c].any() and bg[c].any())
                continue
            for x, y in zip(sd[c], bd[c]):
                assert x.tobytes() == y.tobytes()
            m = se.metrics(se.scipy_raw(p, g, C))
            assert spc.hd_percentile(p, g, C, 100.0)[c] == m["hd"][c]


def test_distance_arrays_are_the_ones_the_raw_tables_sum_and_maximise():
    rng = np.random.default_rng(14)
    for it in range(40):
        shape = tuple(int(x) for x in rng.integers(1, 11, 3))
        C = int(rng.integers(2, 7))
        p = rng.integers(0, C + 2, shape) * (rng.random(shape) < rng.random())
        g = _ellipsoids(rng, shape, C) if it % 2 else rng.integers(0, C + 2, shape) * (rng.random(shape) < rng.random())
        sp = None if it % 3 == 0 else tuple(float(x) for x in rng.uniform(0.3, 3.0, 3))
        for dist_fn, raw_fn in ((spc.scipy_distances, se.scipy_raw), (spc.brute_distances, se.brute_raw)):
            dist, bp, bg = dist_fn(p, g, C, sp)
            raw = raw_fn(p, g, C, sp)
            for c in range(1, C):
                da, db = dist[c]
                assert raw[c - 1, 1] == bp[c].sum() and raw[c - 1, 4] == bg[c].sum()
                if da is None:
                    assert np.isnan(raw[c - 1, [0, 2, 3, 5]]).all()
                    continue
                assert len(da) == raw[c - 1, 1] and len(db) == raw[c - 1, 4]
                want = [math.fsum(da), float(da.max()), math.fsum(db), float(db.max())]
                assert np.array(want).tobytes() == raw[c - 1, [0, 2, 3, 5]].tobytes()


def test_two_single_voxels():
    p, g = np.zeros((7, 8, 9), np.int64), np.zeros((7, 8, 9), np.int64)
    p[1, 2, 3] = 2
    g[5, 7, 4] = 2
    want = math.sqrt(16.0 + 25.0 + 1.0)
    for q in QS:
        for form in ("scipy", "brute"):
            got = spc.hd_percentile(p, g, 3, q, form=form)
            assert got[2] == want and np.isnan(got[1]) and np.isnan(got[0])


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_parallel_slabs_k_apart_give_k_at_every_percentile(axis):
    for k in (1, 3, 6):
        shape = [9, 10, 11]
        shape[axis] = 12
        p, g = np.zeros(shape, np.int64), np.zeros(shape, np.int64)
        sl = [slice(None)] * 3
        sl[axis] = 2
        p[tuple(sl)] = 1
        sl[axis] = 2 + k
        g[tuple(sl)] = 1
        for q in QS + (37.25, 99.9):
            for spacing, s in ((None, 1.0), ((2.0, 2.0, 2.0), 2.0)):
                assert spc.hd_percentile(p, g, 2, q, spacing)[1] == k * s
                assert spc.hd_percentile(p, g, 2, q, spacing, form="brute")[1] == k * s


def test_small_case_worked_by_hand_on_both_sides_of_gamma_one_half():
    # pred: the single voxel (0, 0, 0) of a 1 x 1 x 4 volume; ground truth: all four voxels, every one of them a border voxel.
    # d(pred -> gt) = [0], d(gt -> pred) = [0, 1, 2, 3]: pooled D = [0, 0, 1, 2, 3], n = 5, v = 4 q / 100.
    p, g = np.zeros((1, 1, 4), np.int64), np.zeros((1, 1, 4), np.int64)
    p[0, 0, 0] = 1
    g[:] = 1
    cases = {
        30.0: 0.0 + 1.0 * (4 * 0.3 - 1),           # v = 1.2: a = D(1) = 0, b = D(2) = 1, gamma 0.2 < 0.5: a + delta gamma
        65.0: 2.0 - 1.0 * (1.0 - (4 * 0.65 - 2)),  # v = 2.6: a = D(2) = 1, b = D(3) = 2, gamma 0.6 >= 0.5: b - delta (1 - gamma)
        50.0: 1.0,                                 # v = 2: gamma 0, D(2)
        87.5: 3.0 - 1.0 * 0.5,                     # v = 3.5: gamma 0.5 takes the b - delta (1 - gamma) branch
        100.0: 3.0,                                # v = n - 1: D(4)
    }
    d = np.hstack(spc.scipy_distances(p, g, 2)[0][1])
    assert sorted(d.tolist()) == [0.0, 0.0, 1.0, 2.0, 3.0]
    for q, want in cases.items():
        assert spc.percentile_linear(d, q) == want == np.percentile(d, q), q
        assert spc.hd_percentile(p, g, 2, q)[1] == want and spc.hd_percentile(p, g, 2, q, form="brute")[1] == want
    assert cases[30.0] != 0.2 and abs(cases[30.0] - 0.2) < 1e-15     # the rounding of 4 * 0.3 shows through, as in numpy


def test_linear_restatement_equals_numpy_percentile():
    rng = np.random.default_rng(12)
    qs = QS + (0.1, 1.0, 5.0, 25.0, 33.3, 66.7, 75.0, 90.0, 97.5, 99.9, 100.0 / 3.0, 1e-9, 100 - 1e-9)
    for n in range(1, 3001):
        d = np.sqrt(rng.integers(0, 400, n).astype(np.float64)) * (1.0 if n % 3 else rng.uniform(0.3, 3.0))
        for q in (qs if n < 200 or n % 7 == 0 else (95.0, 50.0)):
            assert spc.percentile_linear(d, q) == np.percentile(d, q), (n, q)
    for it in range(200):
        d = rng.random(int(rng.integers(2, 50000 if it < 10 else 500))) * rng.uniform(0.1, 1e3)
        q = float(rng.uniform(0, 100)) if it % 2 else float(rng.choice(qs))
        assert spc.percentile_linear(d, q) == np.percentile(d, q), (it, q)


# ---- the C-ABI and host layer argument checks ----------------------------------------------------------------------------
def _A(x):
    return (x + 255) // 256 * 256


def test_c_abi_rejects_bad_arguments_and_sizes_the_workspace():
    import pnp_b200  # noqa: F401
    from pnp_b200 import _C
    lib = _C.lib
    nb, nb0 = ctypes.c_longlong(-7), ctypes.c_longlong(-7)
    for n0, n1, n2 in [(1, 1, 1), (256, 256, 256), (256, 256, 131), (37, 29, 23), (1024, 1, 3), (3, 1024, 1024)]:
        for C in (2, 5, 8):
            assert lib.pnp_surface_distance_pct_workspace(n0, n1, n2, C, ctypes.byref(nb)) == 0
            assert lib.pnp_surface_distance_workspace(n0, n1, n2, C, ctypes.byref(nb0)) == 0
            N, L = n0 * n1 * n2, n1 * n2
            assert nb.value == nb0.value + _A(16 * N) + _A(8 * L) + _A(8 * ((2 * L + 255) // 256)) + _A(16584)
    nb.value = -7
    for args, rc in [((0, 4, 4, 5), 100001), ((4, -1, 4, 5), 100001), ((4, 4, 4, 9), 100002), ((4, 4, 4, 1), 100002),
                     ((4, 4, 1025, 2), 100002)]:
        assert lib.pnp_surface_distance_pct_workspace(*args, ctypes.byref(nb)) == rc
        assert nb.value == -7
    assert lib.pnp_surface_distance_pct_workspace(4, 4, 4, 5, None) == 100001
    assert lib.pnp_surface_distance_pct_workspace(4, 4, 4, 5, ctypes.byref(nb)) == 0
    need = nb.value
    # every check comes before the device is touched: these return without a launch on any machine
    fake = ctypes.c_void_p(0x1000)
    sp = (ctypes.c_double * 3)(1.0, 1.0, 1.0)
    bad_q = [float("nan"), float("inf"), -float("inf"), -1e-300, -0.5, 100.0000001, 101.0, 1e308]
    for q in bad_q:
        assert lib.pnp_surface_distance_pct(fake, fake, 4, 4, 4, 5, sp, q, fake, need, fake, None) == 100001, q
    for args, rc in [((fake, fake, 4, 4, 4, 9, sp, 95.0, fake, 1 << 30, fake), 100002),
                     ((fake, fake, 4, 4, 4, 5, sp, 95.0, fake, need - 1, fake), 100001),
                     ((fake, fake, 4, 4, 4, 5, (ctypes.c_double * 3)(1.0, -1.0, 1.0), 95.0, fake, need, fake), 100001),
                     ((None, fake, 4, 4, 4, 5, sp, 95.0, fake, need, fake), 100001),
                     ((fake, None, 4, 4, 4, 5, sp, 95.0, fake, need, fake), 100001),
                     ((fake, fake, 4, 4, 4, 5, sp, 95.0, None, need, fake), 100001),
                     ((fake, fake, 4, 4, 4, 5, sp, 95.0, fake, need, None), 100001),
                     ((fake, fake, 0, 4, 4, 5, sp, 95.0, fake, need, fake), 100001),
                     ((fake, fake, 2000, 4, 4, 5, sp, 95.0, fake, 1 << 40, fake), 100002)]:
        assert lib.pnp_surface_distance_pct(*args, None) == rc, args
    # the workspace of the entry without a percentile is too short for this one
    nb0.value = 0
    assert lib.pnp_surface_distance_workspace(4, 4, 4, 5, ctypes.byref(nb0)) == 0 and nb0.value < need
    assert lib.pnp_surface_distance_pct(fake, fake, 4, 4, 4, 5, sp, 95.0, fake, nb0.value, fake, None) == 100001


def test_surface_distances_rejects_bad_percentiles_before_any_launch():
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F
    v = np.zeros((4, 5, 6), np.uint8)
    for q in (float("nan"), float("inf"), -1.0, 100.5, "x"):
        with pytest.raises(ValueError):
            F.surface_distances(v, v, 5, hd_percentile=q)


def test_surface_from_raw_reads_both_tables():
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F
    nan = math.nan
    raw6 = np.array([[6.0, 3.0, 4.0, 10.0, 5.0, 7.0], [nan, 2.0, nan, nan, 0.0, nan]])
    raw7 = np.hstack([raw6, [[5.5], [nan]]])
    a, b = F.surface_from_raw(raw6), F.surface_from_raw(raw7)
    assert sorted(a) == sorted(F.SURFACE_KEYS + ("border_pred", "border_gt"))
    assert sorted(b) == sorted(list(a) + ["hd_pct"])
    for k in a:
        np.testing.assert_array_equal(a[k], b[k])
    np.testing.assert_array_equal(b["hd_pct"], [nan, 5.5, nan])


# ---- the per-subject table and CSV of the test protocol -------------------------------------------------------------------
def _subjects(q):
    nan = math.nan
    subjects = []
    for i, (assd, hd, hdq) in enumerate([([nan, 1.0, 2.0, nan, 4.0], [nan, 3.0, 5.0, nan, 8.0], [nan, 2.5, 4.0, nan, 6.0]),
                                         ([nan, 3.0, nan, nan, 6.0], [nan, 7.0, nan, nan, 9.0], [nan, 6.5, nan, nan, 8.0])]):
        s = {k: np.array(v) for k, v in (("assd", assd), ("hd", hd), ("asd_pred_gt", assd), ("asd_gt_pred", assd))}
        s["border_pred"] = np.array([0, 10, 11 * (1 - i), 0, 13])
        s["border_gt"] = np.array([0, 20, 21, 0, 23])
        s["subject"] = "ct_%d_image.nii.gz" % i
        if q is not None:
            s["hd_pct"] = np.array(hdq)
            s["hd_percentile"] = q
        subjects.append(s)
    return subjects


def test_surface_table_and_csv_gain_the_percentile_only_when_asked(tmp_path, capsys):
    import pnp_b200  # noqa: F401
    from pnp_b200 import evaluation as ev
    plain = ev.surface_metric_stddev(_subjects(None), 5)
    out_plain = capsys.readouterr().out
    with_q = ev.surface_metric_stddev(_subjects(95.0), 5)
    out_q = capsys.readouterr().out
    for a, b in zip(plain, with_q):
        np.testing.assert_array_equal(a, b)
    assert "hd95" not in out_plain
    assert [ln for ln in out_q.splitlines() if "hd95" not in ln] == out_plain.splitlines()
    assert "hd95_mean: 4.5" in out_q and "hd95_stddev: 2.0" in out_q and "hd95_mean: 7.0" in out_q
    p0 = ev.write_surface_csv(str(tmp_path / "plain.csv"), _subjects(None), 5)
    p1 = ev.write_surface_csv(str(tmp_path / "q.csv"), _subjects(95.0), 5)
    l0, l1 = open(p0).read().splitlines(), open(p1).read().splitlines()
    h0, h1 = l0[0].split(","), l1[0].split(",")
    assert len(h0) == 1 + 4 * 6 and len(h1) == 1 + 4 * 7 and not any("hd95" in h for h in h0)
    assert h1[1:8] == ["la_myo_" + k for k in ev.SURFACE_COLUMNS] + ["la_myo_hd95"]
    r0, r1 = dict(zip(h0, l0[1].split(","))), dict(zip(h1, l1[1].split(",")))
    assert all(r1[k] == v for k, v in r0.items())
    assert float(r1["la_myo_hd95"]) == 2.5 and r1["lv_blood_hd95"] == "nan" and float(r1["aa_hd95"]) == 6.0
    assert ev.pct_name(95.0) == "hd95" and ev.pct_name(99.5) == "hd99.5" and ev.pct_name(100) == "hd100"
    mixed = _subjects(95.0)[:1] + _subjects(99.0)[1:]
    with pytest.raises(ValueError):
        ev.write_surface_csv(str(tmp_path / "mixed.csv"), mixed, 5)


def test_native_csv_gains_the_mm_column_only_when_asked(tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import native
    rows = {}
    for q in (None, 95.0):
        results = _subjects(q)
        for r in results:
            r["dice"] = np.array([0.9, 0.8, 0.7, 0.0, 0.6])
        path = native.write_csv(str(tmp_path / ("native_%s.csv" % q)), results, 5)
        rows[q] = open(path).read().splitlines()
    h0, h1 = rows[None][0].split(","), rows[95.0][0].split(",")
    assert h0 == ["subject"] + ["%s_%s" % (o, k) for o in ("la_myo", "la_blood", "lv_blood", "aa") for k in native.CSV_COLUMNS]
    assert h1 == ["subject"] + ["%s_%s" % (o, k) for o in ("la_myo", "la_blood", "lv_blood", "aa")
                                for k in native.CSV_COLUMNS + ("hd95_mm",)]
    r0, r1 = dict(zip(h0, rows[None][1].split(","))), dict(zip(h1, rows[95.0][1].split(",")))
    assert all(r1[k] == v for k, v in r0.items()) and float(r1["la_myo_hd95_mm"]) == 2.5


def test_run_test_eval_refuses_a_percentile_without_surface_metrics(tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import evaluation as ev
    with pytest.raises(ValueError):
        ev.run_test_eval(None, [], [], 2, 5, str(tmp_path), "x", surface_metrics=False, hd_percentile=95)
    assert not os.path.exists(str(tmp_path / "x"))


def test_evaluate_native_takes_the_percentile_flag(monkeypatch, tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import native
    seen = {}

    class T:
        def test_native(self, pairs, out, hd_percentile=None):
            seen["q"] = hd_percentile
            return []

    monkeypatch.setattr(native, "build_trainer", lambda kind, ckpt, b: T())
    monkeypatch.setattr(native.preprocess, "read_pairs", lambda path: [])
    base = ["--trainer", "gan", "--checkpoint", "c.npz", "--pairs", "p", "--out", str(tmp_path / "o")]
    native.main(base)
    assert seen["q"] is None
    native.main(base + ["--hd-percentile", "95"])
    assert seen["q"] == 95.0
