"""The largest-component references of oracle/components_exact.py against each other, the C-ABI's argument checks and workspace
formula, and the host layer's argument checks, table columns and command-line flag; no GPU needed."""
import ctypes
import math

import numpy as np
import pytest

from oracle import components_exact as ce

FAKE = ctypes.c_void_p(0x1000)


def _A(x):
    return (x + 255) // 256 * 256


def _equal(a, b, tag):
    for x, y, what in zip(a, b, ("out", "stats", "cm")):
        if x is None or y is None:
            assert x is None and y is None, (tag, what)
        else:
            assert x.dtype == y.dtype and np.array_equal(x, y), (tag, what)


def _random_cases():
    rng = np.random.RandomState(7)
    for shape in [(5, 6, 7), (1, 9, 11), (8, 1, 1), (1, 1, 1), (1, 1, 13), (6, 1, 8), (4, 4, 4)]:
        for C in (2, 5, 8):
            for density in (0.2, 0.5, 0.9):
                fg = rng.rand(*shape) < density
                lab = np.where(fg, rng.randint(1, C + 2, size=shape), 0).astype(np.uint8)   # labels up to C + 1
                yield shape, C, lab, rng.randint(0, C + 2, size=shape).astype(np.uint8)


@pytest.mark.parametrize("connectivity", [6, 26])
def test_scipy_and_flood_fill_agree_on_random_volumes(connectivity):
    n = 0
    for shape, C, lab, gt in _random_cases():
        a = ce.scipy_lcc(lab, C, connectivity, gt)
        b = ce.bfs_lcc(lab, C, connectivity, gt)
        _equal(a, b, (shape, C))
        assert a[2].sum() == lab.size
        assert a[1][0, 2] == (lab >= C).sum()
        fg = (lab > 0) & (lab < C)
        assert (a[1][1:, 1] + a[1][1:, 2]).sum() == fg.sum()
        _equal(ce.scipy_lcc(lab, C, connectivity), ce.bfs_lcc(lab, C, connectivity), (shape, C, "no gt"))
        n += 1
    assert n == 63


def test_tie_break_keeps_the_component_whose_first_voxel_comes_first():
    # two 2-voxel components of class 1; the later-starting one is reached first by a scan from the end
    lab = np.zeros((3, 4, 5), np.uint8)
    lab[2, 3, 3:5] = 1            # starts at linear index 58
    lab[0, 0, 1:3] = 1            # starts at linear index 1
    for conn in (6, 26):
        out, st, _ = ce.scipy_lcc(lab, 2, conn)
        assert out[0, 0, 1] == 1 and out[0, 0, 2] == 1 and out[2, 3].sum() == 0
        assert st[1].tolist() == [2, 2, 2]
        _equal((out, st, None), ce.bfs_lcc(lab, 2, conn), conn)
    # a diagonal pair: two components at 6-connectivity, one at 26
    lab = np.zeros((2, 2, 2), np.uint8)
    lab[0, 0, 0] = lab[1, 1, 1] = 3
    for conn, comps, kept in ((6, 2, 1), (26, 1, 2)):
        out, st, _ = ce.scipy_lcc(lab, 5, conn)
        assert st[3].tolist() == [comps, kept, 2 - kept] and out[0, 0, 0] == 3
        _equal((out, st, None), ce.bfs_lcc(lab, 5, conn), conn)


def test_checkerboard_empty_classes_and_out_of_range_labels():
    i, j, k = np.indices((4, 5, 6))
    lab = ((i + j + k) % 2).astype(np.uint8)
    for conn in (6, 26):
        out, st, _ = ce.scipy_lcc(lab, 2, conn)
        _equal((out, st, None), ce.bfs_lcc(lab, 2, conn), conn)
        if conn == 6:
            assert st[1].tolist() == [60, 1, 59] and out.sum() == 1 and out[0, 0, 1] == 1
        else:
            assert st[1].tolist() == [1, 60, 0] and np.array_equal(out, lab)
    lab = np.full((3, 3, 3), 9, np.uint8)
    out, st, cm = ce.scipy_lcc(lab, 8, 26, lab)
    assert not out.any() and st.tolist() == [[0, 0, 27]] + [[0, 0, 0]] * 7 and cm[0, 0] == 27
    _equal((out, st, cm), ce.bfs_lcc(lab, 8, 26, lab), "all out of range")


def test_c_abi_rejects_bad_arguments_and_sizes_the_workspace():
    import pnp_b200  # noqa: F401
    from pnp_b200 import _C
    lib = _C.lib
    nb = ctypes.c_longlong(-7)
    for n0, n1, n2 in [(1, 1, 1), (512, 512, 300), (256, 256, 256), (37, 29, 23), (1, 1, 2 ** 30), (2 ** 15, 2 ** 15, 1)]:
        for C in (2, 5, 8):
            for conn in (6, 26):
                nb.value = -7
                assert lib.pnp_largest_components_workspace(n0, n1, n2, C, conn, ctypes.byref(nb)) == 0
                assert nb.value == 2 * _A(4 * n0 * n1 * n2) + 256
    nb.value = -7
    for args, rc in [((0, 4, 4, 5, 6), 100001), ((4, -1, 4, 5, 6), 100001), ((4, 4, 4, 9, 6), 100002), ((4, 4, 4, 1, 26), 100002),
                     ((4, 4, 4, 5, 18), 100002), ((4, 4, 4, 5, 0), 100002), ((2 ** 11, 2 ** 10, 2 ** 10, 5, 6), 100002),
                     ((2 ** 15, 2 ** 15, 2, 5, 26), 100002)]:
        assert lib.pnp_largest_components_workspace(*args, ctypes.byref(nb)) == rc, args
        assert nb.value == -7
    assert lib.pnp_largest_components_workspace(4, 4, 4, 5, 6, None) == 100001
    assert lib.pnp_largest_components_workspace(4, 4, 4, 5, 6, ctypes.byref(nb)) == 0
    need = nb.value
    assert need == 2 * 256 + 256
    # every check comes before the device is touched: these return without a launch on any machine
    f = FAKE
    for args, rc in [((None, 4, 4, 4, 5, 6, f, None, None, f, f, need), 100001),
                     ((f, 4, 4, 4, 5, 6, None, None, None, f, f, need), 100001),
                     ((f, 4, 4, 4, 5, 6, f, f, None, f, f, need), 100001),
                     ((f, 4, 4, 4, 5, 6, f, None, f, f, f, need), 100001),
                     ((f, 4, 4, 4, 5, 6, f, None, None, None, f, need), 100001),
                     ((f, 4, 4, 4, 5, 6, f, None, None, f, None, need), 100001),
                     ((f, 4, 4, 4, 5, 6, f, None, None, f, f, need - 1), 100001),
                     ((f, 4, 0, 4, 5, 6, f, None, None, f, f, need), 100001),
                     ((f, 4, 4, -3, 5, 6, f, None, None, f, f, need), 100001),
                     ((f, 4, 4, 4, 9, 6, f, None, None, f, f, need), 100002),
                     ((f, 4, 4, 4, 1, 6, f, None, None, f, f, need), 100002),
                     ((f, 4, 4, 4, 5, 18, f, None, None, f, f, need), 100002),
                     ((f, 4, 4, 4, 5, 8, f, f, f, f, f, need), 100002),
                     ((f, 2 ** 11, 2 ** 10, 2 ** 10, 5, 6, f, None, None, f, f, 1 << 40), 100002)]:
        assert lib.pnp_largest_components(*args, None) == rc, args


def test_largest_components_checks_its_arguments_on_the_host():
    import pnp_b200  # noqa: F401
    import torch
    from pnp_b200 import functional as F
    v = torch.zeros(4, 5, 6, dtype=torch.uint8)
    for num_cls, conn in [(1, 6), (9, 6), (5, 18), (5, 0), (5, True), (5, "6"), (5, None)]:
        with pytest.raises(ValueError):
            F.largest_components(v, num_cls, conn)
    for bad in (v, np.zeros((4, 5, 6), np.uint8), torch.zeros(4, 5, dtype=torch.uint8), torch.zeros(4, 5, 6, dtype=torch.int64)):
        with pytest.raises(ValueError, match="labels must be a uint8 3-D tensor on the device"):
            F.largest_components(bad, 5, 6)


def _result(post):
    nan = math.nan
    r = {"subject": "ct_1_image.nii.gz", "dice": np.array([0.9, 0.8, 0.7, 0.0, 0.6]),
         "assd": np.array([nan, 1.0, 2.0, nan, 4.0]), "hd": np.array([nan, 3.0, 5.0, nan, 8.0]),
         "border_pred": np.array([0, 10, 11, 0, 13]), "border_gt": np.array([0, 20, 21, 0, 23])}
    if post:
        r.update(largest_component=26, dice_raw=np.array([0.0, 0.75, 0.5, 0.0, 0.25]), components=np.array([0, 3, 1, 0, 7]),
                 kept=np.array([0, 5, 6, 0, 7]), removed=np.array([4, 2, 0, 0, 9]))
    return r


def test_native_csv_gains_the_component_columns_after_all_others_only_when_asked(tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import native
    organs = ("la_myo", "la_blood", "lv_blood", "aa")
    lines = {}
    for post in (False, True):
        path = native.write_csv(str(tmp_path / ("n%d.csv" % post)), [_result(post)], 5)
        lines[post] = open(path).read().splitlines()
    h0, h1 = lines[False][0].split(","), lines[True][0].split(",")
    assert h0 == ["subject"] + ["%s_%s" % (o, k) for o in organs for k in native.CSV_COLUMNS]
    assert h1 == h0 + ["%s_%s" % (o, k) for o in organs for k in ("dice_raw", "components", "removed")]
    r0, r1 = lines[False][1].split(","), lines[True][1].split(",")
    assert r1[:len(r0)] == r0
    extra = dict(zip(h1[len(h0):], r1[len(r0):]))
    assert float(extra["la_myo_dice_raw"]) == 0.75 and extra["la_myo_components"] == "3" and extra["aa_removed"] == "9"
    assert extra["lv_blood_components"] == "0"
    mixed = [_result(True), dict(_result(True), largest_component=6)]
    with pytest.raises(ValueError):
        native.write_csv(str(tmp_path / "mixed.csv"), mixed, 5)


def test_native_run_refuses_a_bad_connectivity_before_any_work(tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import native
    for bad in (0, 8, 18, True, "26", 6.5):
        with pytest.raises(ValueError):
            native.run(None, [("a", "b")], str(tmp_path / "o"), 2, 5, largest_component=bad)
    assert not (tmp_path / "o").exists()
    assert native.check_connectivity(None) is None and native.check_connectivity(6) == 6 and native.check_connectivity(26) == 26


def test_evaluate_native_takes_the_largest_component_flag(monkeypatch, tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import native
    seen = []

    class T:
        def test_native(self, pairs, out, hd_percentile=None, **kw):
            seen.append((hd_percentile, kw))
            return []

    monkeypatch.setattr(native, "build_trainer", lambda kind, ckpt, b: T())
    monkeypatch.setattr(native.preprocess, "read_pairs", lambda path: [])
    base = ["--trainer", "gan", "--checkpoint", "c.npz", "--pairs", "p", "--out", str(tmp_path / "o")]
    native.main(base)
    native.main(base + ["--largest-component", "6"])
    native.main(base + ["--largest-component", "26", "--hd-percentile", "95"])
    assert seen == [(None, {}), (None, {"largest_component": 6}), (95.0, {"largest_component": 26})]
    for bad in ("18", "0", "x", "6.0"):
        with pytest.raises(SystemExit):
            native.main(base + ["--largest-component", bad])
    assert len(seen) == 3
