"""Per-class surface distances (ASSD / HD) on the host: the two forms of oracle/surface_exact.py against each other and against
known answers, the argument checks of `functional.surface_distances` and of the C-ABI entry points (which return before any
launch), and the per-subject table and CSV of the test protocol.  The kernels themselves are tested on the GPU in
tests/test_surface_distance_gpu.py."""
import ctypes
import math
import os

import numpy as np
import pytest

from oracle import surface_exact as se


def _ellipsoids(rng, shape, num_cls):
    g = np.ogrid[:shape[0], :shape[1], :shape[2]]
    v = np.zeros(shape, np.int64)
    for c in range(1, num_cls):
        centre = rng.uniform(-0.2, 1.2, 3) * shape
        radii = rng.uniform(0.15, 0.8, 3) * np.array(shape) + 0.5
        v[sum(((g[a] - centre[a]) / radii[a]) ** 2 for a in range(3)) < 1] = c
    return v


def _random_pair(rng, it):
    shape = tuple(int(x) for x in rng.integers(1, 12, 3))
    C = int(rng.integers(2, 9))
    kind = it % 4
    if kind == 0:                                   # salt and pepper, labels above the range included
        p = rng.integers(0, C + 2, shape) * (rng.random(shape) < rng.random())
        g = rng.integers(0, C + 2, shape) * (rng.random(shape) < rng.random())
    elif kind == 1:                                 # blobs, often touching the faces
        p, g = _ellipsoids(rng, shape, C), _ellipsoids(rng, shape, C)
    elif kind == 2:                                 # whole-volume and single-voxel objects
        p = np.full(shape, int(rng.integers(1, C)), np.int64)
        g = np.zeros(shape, np.int64)
        g[tuple(int(rng.integers(0, n)) for n in shape)] = int(p.flat[0])
    else:                                           # 1-voxel-thick sheets and rods
        p, g = np.zeros(shape, np.int64), np.zeros(shape, np.int64)
        a = int(rng.integers(0, 3))
        sl = [slice(None)] * 3
        sl[a] = int(rng.integers(0, shape[a]))
        p[tuple(sl)] = 1
        g[int(rng.integers(0, shape[0])), int(rng.integers(0, shape[1])), :] = 1
    sp = None if it % 3 == 0 else tuple(float(x) for x in rng.uniform(0.3, 3.0, 3))
    return p, g, C, sp


def _close(a, b, rtol):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert np.array_equal(np.isnan(a), np.isnan(b)), (a, b)
    m = ~np.isnan(b)
    assert np.all(np.abs(a[m] - b[m]) <= rtol * np.abs(b[m])), (a, b)


def test_scipy_form_equals_brute_force_on_random_small_volumes():
    rng = np.random.default_rng(2024)
    for it in range(120):
        p, g, C, sp = _random_pair(rng, it)
        for a, b in zip(se.scipy_borders(p, C)[1:], se.brute_borders(p, C)[1:]):
            assert np.array_equal(a, b)
        _close(se.scipy_raw(p, g, C, sp), se.brute_raw(p, g, C, sp), 1e-12)


def test_identical_volumes_give_zero():
    rng = np.random.default_rng(5)
    v = _ellipsoids(rng, (13, 17, 11), 5)
    m = se.surface_metrics(v, v, 5)
    present = [c for c in range(1, 5) if (v == c).any()]
    assert present
    for c in present:
        assert m["assd"][c] == 0.0 and m["hd"][c] == 0.0 and m["border_pred"][c] == m["border_gt"][c] > 0


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("k", [1, 3, 6])
def test_parallel_slabs_k_apart_give_exactly_k(axis, k):
    shape = [9, 10, 11]
    shape[axis] = 12
    p, g = np.zeros(shape, np.int64), np.zeros(shape, np.int64)
    sl = [slice(None)] * 3
    sl[axis] = 2
    p[tuple(sl)] = 1
    sl[axis] = 2 + k
    g[tuple(sl)] = 1
    for spacing, s in ((None, 1.0), ((0.5, 0.5, 0.5), 0.5), ((2.0, 2.0, 2.0), 2.0)):
        for raw in (se.scipy_raw(p, g, 2, spacing), se.brute_raw(p, g, 2, spacing)):
            m = se.metrics(raw)
            assert m["assd"][1] == k * s and m["hd"][1] == k * s
            assert m["asd_pred_gt"][1] == m["asd_gt_pred"][1] == k * s
            assert m["border_pred"][1] == p.sum() and m["border_gt"][1] == g.sum()    # one-voxel slabs are all border


def test_two_single_voxels_give_their_euclidean_distance():
    p, g = np.zeros((7, 8, 9), np.int64), np.zeros((7, 8, 9), np.int64)
    p[1, 2, 3] = 2
    g[5, 7, 4] = 2
    for sp in (None, (0.7, 1.3, 2.5)):
        s = (1.0, 1.0, 1.0) if sp is None else sp
        want = math.sqrt(((4 * s[0]) ** 2 + (5 * s[1]) ** 2) + (1 * s[2]) ** 2)
        for raw in (se.scipy_raw(p, g, 3, sp), se.brute_raw(p, g, 3, sp)):
            m = se.metrics(raw)
            assert m["assd"][2] == m["hd"][2] == want
            assert np.isnan(m["assd"][1]) and m["border_pred"][1] == m["border_gt"][1] == 0


def test_full_volume_class_has_exactly_its_face_voxels_as_border():
    for shape in [(1, 1, 1), (1, 5, 7), (2, 2, 2), (4, 5, 6)]:
        v = np.full(shape, 3, np.int64)
        face = np.ones(shape, bool)
        if min(shape) > 2:
            face[1:-1, 1:-1, 1:-1] = False
        for b in (se.scipy_borders(v, 4)[3], se.brute_borders(v, 4)[3]):
            assert np.array_equal(b, face)


def test_absent_classes_and_out_of_range_labels():
    p, g = np.zeros((6, 6, 6), np.int64), np.zeros((6, 6, 6), np.int64)
    p[1:3, 1:3, 1:3] = 1
    g[2:4, 2:4, 2:4] = 1
    p[4, 4, 4] = 2                 # class 2 only in the prediction
    g[0, 5, 0] = 7                 # labels >= num_cls and < 0 are background
    p[5, 0, 5] = -3
    raw = se.scipy_raw(p, g, 4)
    np.testing.assert_array_equal(raw, se.brute_raw(p, g, 4))
    m = se.metrics(raw)
    assert np.isfinite(m["assd"][1])
    assert np.isnan(m["assd"][2]) and m["border_pred"][2] == 1 and m["border_gt"][2] == 0
    assert np.isnan(m["hd"][3]) and m["border_pred"][3] == m["border_gt"][3] == 0
    assert np.isnan(m["assd"][0])


# ---- host argument checks ------------------------------------------------------------------------------------------------------
def test_surface_distances_rejects_bad_arguments_before_any_launch():
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F
    v = np.zeros((4, 5, 6), np.uint8)
    bad = [((v, v[:, :, :5], 5), {}), ((v[0], v[0], 5), {}), ((v, v, 9), {}), ((v, v, 1), {}),
           ((np.zeros((1025, 1, 1)), np.zeros((1025, 1, 1)), 2), {}), ((np.zeros((0, 3, 3)), np.zeros((0, 3, 3)), 2), {}),
           ((v, v, 5), {"spacing": (1.0, 0.0, 1.0)}), ((v, v, 5), {"spacing": (1.0, 1.0)}),
           ((v, v, 5), {"spacing": (1.0, float("nan"), 1.0)}), ((v.astype(np.float32), v, 5), {})]
    for args, kw in bad:
        with pytest.raises(ValueError):
            F.surface_distances(*args, **kw)


def test_c_abi_rejects_bad_arguments_and_sizes_the_workspace():
    import pnp_b200  # noqa: F401
    from pnp_b200 import _C
    lib = _C.lib
    nb = ctypes.c_longlong(-7)
    A = lambda x: (x + 255) // 256 * 256
    for n0, n1, n2 in [(1, 1, 1), (256, 256, 256), (37, 29, 23), (1024, 1, 3)]:
        assert lib.pnp_surface_distance_workspace(n0, n1, n2, 5, ctypes.byref(nb)) == 0
        N, L = n0 * n1 * n2, n1 * n2
        assert nb.value == A(2 * N) + A(4 * N) + A(8 * N) + 2 * A(16 * L) + A(8 * L)
    assert lib.pnp_surface_distance_workspace(256, 256, 256, 5, ctypes.byref(nb)) == 0 and nb.value < 2 ** 30
    nb.value = -7
    for args, rc in [((0, 4, 4, 5), 100001), ((4, -1, 4, 5), 100001), ((4, 4, 4, 9), 100002), ((4, 4, 4, 1), 100002),
                     ((4, 4, 1025, 2), 100002)]:
        assert lib.pnp_surface_distance_workspace(*args, ctypes.byref(nb)) == rc
        assert nb.value == -7
    assert lib.pnp_surface_distance_workspace(4, 4, 4, 5, None) == 100001
    # the launcher checks everything before it touches the device: these return without a launch on any machine
    fake = ctypes.c_void_p(0x1000)
    sp = (ctypes.c_double * 3)(1.0, 1.0, 1.0)
    for args, rc in [((fake, fake, 4, 4, 4, 9, sp, fake, 1 << 20, fake), 100002),
                     ((fake, fake, 4, 4, 4, 5, sp, fake, 10, fake), 100001),
                     ((fake, fake, 4, 4, 4, 5, (ctypes.c_double * 3)(1.0, -1.0, 1.0), fake, 1 << 20, fake), 100001),
                     ((None, fake, 4, 4, 4, 5, sp, fake, 1 << 20, fake), 100001),
                     ((fake, fake, 2000, 4, 4, 5, sp, fake, 1 << 40, fake), 100002)]:
        assert lib.pnp_surface_distance(*args, None) == rc


# ---- the per-subject table and CSV of the test protocol -------------------------------------------------------------------
def test_surface_table_and_csv(tmp_path, capsys):
    import pnp_b200  # noqa: F401
    from pnp_b200 import evaluation as ev
    nan = math.nan
    subjects = []
    for i, (assd, hd) in enumerate([([nan, 1.0, 2.0, nan, 4.0], [nan, 3.0, 5.0, nan, 8.0]),
                                    ([nan, 3.0, nan, nan, 6.0], [nan, 7.0, nan, nan, 9.0])]):
        s = {k: np.array(v) for k, v in (("assd", assd), ("hd", hd), ("asd_pred_gt", assd), ("asd_gt_pred", assd))}
        s["border_pred"] = np.array([0, 10, 11 * (1 - i), 0, 13])
        s["border_gt"] = np.array([0, 20, 21, 0, 23])
        s["subject"] = "ct_%d_image.nii.gz" % i
        subjects.append(s)
    mean_assd, mean_hd = ev.surface_metric_stddev(subjects, 5)
    np.testing.assert_array_equal(mean_assd, [nan, 2.0, 2.0, nan, 5.0])
    np.testing.assert_array_equal(mean_hd, [nan, 5.0, 5.0, nan, 8.5])
    out = capsys.readouterr().out
    assert "organ: la_myo" in out and "assd_mean: 2.0" in out and "hd_stddev: 2.0" in out and "organ: bg" not in out
    assert out.count("skipped subjects (organ absent from prediction or ground truth): 1") == 1
    assert out.count("skipped subjects (organ absent from prediction or ground truth): 2") == 1
    path = ev.write_surface_csv(str(tmp_path / "surface.csv"), subjects, 5)
    lines = open(path).read().splitlines()
    head = lines[0].split(",")
    assert head[0] == "subject" and head[1:7] == ["la_myo_" + k for k in ev.SURFACE_COLUMNS] and len(head) == 1 + 4 * 6
    row = dict(zip(head, lines[1].split(",")))
    assert row["subject"] == "ct_0_image.nii.gz" and float(row["la_blood_assd"]) == 2.0 and row["lv_blood_hd"] == "nan"
    assert row["aa_border_gt"] == "23" and len(lines) == 3
