"""pnp_surface_distance_pct (csrc/metrics3d.cu) and its host layer on the device, against oracle/surface_percentile.py:
* unit spacing: HD_q bit for bit np.percentile(np.hstack((da, db)), q) of the oracle's distance arrays, for q in QS, on the
  shapes of tests/test_surface_distance_gpu.py, on a 256 x 256 x 131 subject, on a sweep of pooled counts n built from
  one-voxel-thick lines (integer v, gamma < 0.5 and gamma >= 0.5 all occur), on tie-heavy volumes and on a class whose pooled
  list takes the select kernels several grid-stride sweeps; the brute-force oracle on small volumes;
* the first six columns bit-identical to pnp_surface_distance on the same inputs; q = 100 is HD and q = 0 the smallest distance;
* anisotropic spacing to 1e-13 relative; absent classes and labels >= C give NaN with the border counts set; repeated calls
  bit-identical; rejected calls leave `out` untouched;
* both trainers' test_eval(..., surface_metrics=True, hd_percentile=95) against the oracle applied to the volumes it saved, with
  every other output equal to a run without the percentile; test_native(..., hd_percentile=95) and the command line against the
  oracle applied to the written native prediction and the native ground truth at native spacing."""
import csv
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import surface_percentile as spc
from tests import mmwhs_phantom as ph

pytestmark = pytest.mark.gpu
QS = (0.0, 12.5, 50.0, 95.0, 99.0, 100.0)
SHAPES = [(1, 1, 1), (1, 1, 40), (1, 33, 1), (47, 1, 1), (1, 9, 14), (37, 29, 23), (16, 64, 5), (8, 3, 200)]
SEL_SWEEP = 132 * 2 * 256          # keys one sweep of the select kernels' grid covers


def _u8(v, C):
    return np.ascontiguousarray(np.where((v >= 0) & (v < C), v, 0), np.uint8)


def _dev(pred, gt, C):
    from pnp_b200 import _C, runtime as rt
    return torch.from_numpy(_u8(pred, C)).cuda(), torch.from_numpy(_u8(gt, C)).cuda(), _C, rt


def _raw6(pred, gt, C, spacing=None):
    dp, dg, _C, rt = _dev(pred, gt, C)
    nb = ctypes.c_longlong(0)
    _C.call("pnp_surface_distance_workspace", *dp.shape, C, ctypes.byref(nb))
    ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    out = torch.empty((C - 1) * 6, dtype=torch.float64, device="cuda")
    sp = None if spacing is None else (ctypes.c_double * 3)(*spacing)
    _C.call("pnp_surface_distance", dp.data_ptr(), dg.data_ptr(), *dp.shape, C, sp, ws.data_ptr(), nb.value, out.data_ptr(),
            rt.stream())
    return out.cpu().numpy().reshape(C - 1, 6)


def _raw7(pred, gt, C, qs, spacing=None):
    """[len(qs), C - 1, 7]: one workspace, one call per q"""
    dp, dg, _C, rt = _dev(pred, gt, C)
    nb = ctypes.c_longlong(0)
    _C.call("pnp_surface_distance_pct_workspace", *dp.shape, C, ctypes.byref(nb))
    ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    sp = None if spacing is None else (ctypes.c_double * 3)(*spacing)
    res = []
    for q in qs:
        out = torch.empty((C - 1) * 7, dtype=torch.float64, device="cuda")
        _C.call("pnp_surface_distance_pct", dp.data_ptr(), dg.data_ptr(), *dp.shape, C, sp, float(q), ws.data_ptr(), nb.value,
                out.data_ptr(), rt.stream())
        res.append(out.cpu().numpy().reshape(C - 1, 7))
    return np.stack(res)


def _pooled(pred, gt, C, spacing=None, form="scipy"):
    dist = (spc.scipy_distances if form == "scipy" else spc.brute_distances)(pred, gt, C, spacing)[0]
    return [None] + [None if dist[c][0] is None else np.hstack(dist[c]) for c in range(1, C)]


def _check(pred, gt, C, qs=QS, form="scipy"):
    """HD_q bit for bit the oracle's np.percentile, columns 0-5 bit for bit pnp_surface_distance's -> the pooled lists"""
    got = _raw7(pred, gt, C, qs)
    six = _raw6(pred, gt, C)
    pooled = _pooled(pred, gt, C, form=form)
    for i, q in enumerate(qs):
        assert got[i, :, :6].tobytes() == six.tobytes(), q
        for c in range(1, C):
            if pooled[c] is None:
                assert np.isnan(got[i, c - 1, 6]), (q, c)
            else:
                want = np.percentile(pooled[c], q)
                assert got[i, c - 1, 6] == want, (q, c, got[i, c - 1, 6], want, len(pooled[c]))
                if q == 100.0:
                    assert want == max(six[c - 1, 2], six[c - 1, 5])
                if q == 0.0:
                    assert want == pooled[c].min()
    return pooled


def _ellipsoids(rng, shape, num_cls, lo=0.1, hi=0.45):
    g = np.ogrid[:shape[0], :shape[1], :shape[2]]
    v = np.zeros(shape, np.int64)
    for c in range(1, num_cls):
        centre = rng.uniform(0.1, 0.9, 3) * shape
        radii = rng.uniform(lo, hi, 3) * np.array(shape) + 0.5
        v[sum(((g[a] - centre[a]) / radii[a]) ** 2 for a in range(3)) < 1] = c
    return v


@pytest.mark.parametrize("shape", SHAPES)
def test_matches_numpy_percentile_of_the_oracle_unit_spacing(shape):
    import pnp_b200  # noqa: F401
    rng = np.random.default_rng(sum(shape) + 95)
    for it in range(6):
        C = int(rng.integers(2, 9))
        if it % 2:
            p = rng.integers(0, C + 3, shape) * (rng.random(shape) < rng.uniform(0.02, 0.6))
            g = rng.integers(0, C + 3, shape) * (rng.random(shape) < rng.uniform(0.02, 0.6))
        else:
            p, g = _ellipsoids(rng, shape, C), _ellipsoids(rng, shape, C)
        _check(p, g, C)


def test_matches_brute_force_on_small_volumes():
    import pnp_b200  # noqa: F401
    rng = np.random.default_rng(77)
    for it in range(20):
        shape = tuple(int(x) for x in rng.integers(1, 14, 3))
        C = int(rng.integers(2, 9))
        p = rng.integers(0, C + 1, shape) * (rng.random(shape) < rng.random())
        g = _ellipsoids(rng, shape, C)
        _check(p, g, C, form="brute")


def test_256x256x131_subject():
    import pnp_b200  # noqa: F401
    rng = np.random.default_rng(131)
    shape = (256, 256, 131)
    g = _ellipsoids(rng, shape, 5, 0.1, 0.3)
    p = np.where(rng.random(shape) < 1e-3, rng.integers(0, 7, shape), np.roll(g, (2, -3, 1), (0, 1, 2)))
    pooled = _check(p, g, 5)
    assert all(x is not None for x in pooled[1:])


def test_sweep_of_pooled_counts_covers_every_interpolation_branch():
    """pred: a line of a voxels along axis 2, gt: a line of b voxels two rows over and shifted -- one voxel thick, so every
    voxel is a border voxel and n = a + b.  Several hundred n from 2 up."""
    import pnp_b200  # noqa: F401
    qs = (12.5, 50.0, 95.0, 99.0, 37.3, 100.0 / 3.0)
    branches = {"integer v": 0, "gamma < 0.5": 0, "gamma >= 0.5": 0}
    shape = (3, 4, 260)
    pairs = [(1, 1)] + [(a, 1 + a % 3) for a in range(1, 255)] + [(a, 200 + a % 50) for a in range(100, 250, 2)]
    for a, b in pairs:
        p, g = np.zeros(shape, np.int64), np.zeros(shape, np.int64)
        p[0, 0, :a] = 1
        g[2, 3, 5:5 + b] = 1
        got = _raw7(p, g, 2, qs)
        d = _pooled(p, g, 2)[1]
        n = a + b
        assert len(d) == n and got[0, 0, 1] == a and got[0, 0, 4] == b
        for i, q in enumerate(qs):
            assert got[i, 0, 6] == np.percentile(d, q), (a, b, q)
            v = (n - 1) * (q / 100.0)
            gam = v - np.floor(v)
            branches["integer v" if gam == 0 else ("gamma < 0.5" if gam < 0.5 else "gamma >= 0.5")] += 1
    assert len({a + b for a, b in pairs}) >= 200
    assert all(k > 50 for k in branches.values()), branches


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_tie_heavy_slabs(axis):
    import pnp_b200  # noqa: F401
    shape = [40, 50, 60]
    for k in (1, 4, 17):
        p, g = np.zeros(shape, np.int64), np.zeros(shape, np.int64)
        sl = [slice(None)] * 3
        sl[axis] = 3
        p[tuple(sl)] = 2
        sl[axis] = 3 + k
        g[tuple(sl)] = 2
        _check(p, g, 3, QS + (37.25,))
        got = _raw7(p, g, 3, QS)
        assert (got[:, 1, 6] == k).all()


def test_small_integer_distances_and_several_grid_sweeps():
    """labels drawn voxel by voxel: nearly every voxel is a border voxel, the distances are square roots of small integers
    with heavy ties, and the pooled list of each class spans several sweeps of the select kernels' grid"""
    import pnp_b200  # noqa: F401
    rng = np.random.default_rng(5)
    shape = (96, 96, 80)
    p = rng.integers(0, 3, shape) * (rng.random(shape) < 0.7)
    g = rng.integers(0, 3, shape) * (rng.random(shape) < 0.7)
    pooled = _check(p, g, 3, QS + (0.01, 99.99, 63.7))
    assert min(len(x) for x in pooled[1:]) > 3 * SEL_SWEEP
    assert len(np.unique(pooled[1])) < 10


@pytest.mark.parametrize("shape", [(37, 29, 23), (64, 48, 40), (1, 30, 30)])
def test_anisotropic_spacing(shape):
    import pnp_b200  # noqa: F401
    rng = np.random.default_rng(11)
    for spacing in [(0.7, 1.3, 2.5), (2.5, 0.7, 1.3), (1.0, 1.0, 3.0)]:
        C = 5
        p, g = _ellipsoids(rng, shape, C), _ellipsoids(rng, shape, C)
        got = _raw7(p, g, C, QS, spacing)
        six = _raw6(p, g, C, spacing)
        for i, q in enumerate(QS):
            assert got[i, :, :6].tobytes() == six.tobytes()
            ref = spc.hd_percentile(p, g, C, q, spacing)[1:]
            assert np.array_equal(np.isnan(got[i, :, 6]), np.isnan(ref))
            m = ~np.isnan(ref)
            assert np.all(np.abs(got[i, m, 6] - ref[m]) <= 1e-13 * np.abs(ref[m])), (q, got[i, :, 6], ref)


def test_absent_classes_and_labels_out_of_range():
    import pnp_b200  # noqa: F401
    p, g = np.zeros((9, 10, 11), np.int64), np.zeros((9, 10, 11), np.int64)
    p[1, 2, 3], g[7, 9, 0] = 1, 1
    p[4, 4, 4] = 2                   # only in the prediction
    g[5, 5, 5] = 3                   # only in the ground truth
    p[0, 0, 0], g[8, 9, 10] = 200, 6  # >= C: background
    got = _raw7(p, g, 5, QS)
    d = np.sqrt(36.0 + 49.0 + 9.0)
    assert (got[:, 0, 6] == d).all()
    assert np.isnan(got[:, 1:, 6]).all()
    assert tuple(got[0, 1, [1, 4]]) == (1, 0) and tuple(got[0, 2, [1, 4]]) == (0, 1) and tuple(got[0, 3, [1, 4]]) == (0, 0)
    _check(p, g, 5)


def test_repeated_calls_are_bit_identical():
    import pnp_b200  # noqa: F401
    rng = np.random.default_rng(3)
    shape = (96, 80, 71)
    p, g = _ellipsoids(rng, shape, 6), _ellipsoids(rng, shape, 6)
    p = np.where(rng.random(shape) < 0.01, rng.integers(0, 6, shape), p)
    a = _raw7(p, g, 6, (95.0, 95.0, 50.0, 50.0), (0.7, 1.3, 2.5))
    assert a[0].tobytes() == a[1].tobytes() and a[2].tobytes() == a[3].tobytes()
    b = _raw7(p, g, 6, (95.0, 50.0), (0.7, 1.3, 2.5))
    assert b[0].tobytes() == a[0].tobytes() and b[1].tobytes() == a[2].tobytes()


def test_rejected_arguments_leave_out_untouched():
    import pnp_b200  # noqa: F401
    from pnp_b200 import _C, runtime as rt
    v = torch.zeros(4 * 5 * 6, dtype=torch.uint8, device="cuda")
    nb = ctypes.c_longlong(0)
    _C.call("pnp_surface_distance_pct_workspace", 4, 5, 6, 5, ctypes.byref(nb))
    ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    out = torch.full((8 * 7,), 1234.5, dtype=torch.float64, device="cuda")
    sp = (ctypes.c_double * 3)(1.0, 1.0, 1.0)
    P = v.data_ptr()
    for args, rc in [((4, 5, 6, 5, sp, float("nan"), nb.value), 100001), ((4, 5, 6, 5, sp, float("inf"), nb.value), 100001),
                     ((4, 5, 6, 5, sp, -0.1, nb.value), 100001), ((4, 5, 6, 5, sp, 100.5, nb.value), 100001),
                     ((4, 5, 6, 9, sp, 95.0, nb.value), 100002), ((4, 0, 6, 5, sp, 95.0, nb.value), 100001),
                     ((4, 5, 6, 5, (ctypes.c_double * 3)(1.0, 0.0, 1.0), 95.0, nb.value), 100001),
                     ((4, 5, 6, 5, sp, 95.0, nb.value - 1), 100001)]:
        n0, n1, n2, C, s, q, nbytes = args
        assert _C.lib.pnp_surface_distance_pct(P, P, n0, n1, n2, C, s, q, ws.data_ptr(), nbytes, out.data_ptr(), rt.stream()) == rc
    torch.cuda.synchronize()
    assert bool((out == 1234.5).all())


def test_functional_surface_distances_with_and_without_the_percentile():
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F
    rng = np.random.default_rng(17)
    shape = (50, 41, 33)
    g = _ellipsoids(rng, shape, 5)
    p = np.roll(g, 2, axis=1).astype(np.int32)
    p[p == 3] = 0
    for spacing in (None, (0.7, 1.3, 2.5)):
        plain = F.surface_distances(p, g, 5, spacing)
        got = F.surface_distances(p, g, 5, spacing, hd_percentile=95)
        assert sorted(got) == sorted(list(plain) + ["hd_pct", "hd_percentile"]) and got["hd_percentile"] == 95.0
        for k in plain:
            assert np.asarray(plain[k]).tobytes() == np.asarray(got[k]).tobytes(), k
        ref = spc.hd_percentile(p, g, 5, 95, spacing)
        np.testing.assert_allclose(got["hd_pct"], ref, rtol=1e-13 if spacing else 0, atol=0, equal_nan=True)
        assert np.array_equal(np.isnan(got["hd_pct"]), np.isnan(plain["hd"])) and np.isnan(got["hd_pct"][3])


# ---- the test protocol of both trainers ----------------------------------------------------------------------------------
def _stddev_block(text):
    lines = text.splitlines()
    a = next(i for i, ln in enumerate(lines) if "inside the sample_metric_stddev" in ln)
    b = next(i for i, ln in enumerate(lines) if ln.startswith("all_jaccard_mean"))
    return lines[a:b + 1]


def _surface_block(text):
    lines = text.splitlines()
    return lines[next(i for i, ln in enumerate(lines) if ln.startswith("------- surface distances")):]


def _check_hd95(surface_list, pred_dir, nii, num_cls):
    from pnp_b200.lib import read_nii_image
    finite = 0
    for s, f in zip(surface_list, nii):
        b = os.path.basename(f).split(".")[0] + ".nii.gz"
        p = read_nii_image(os.path.join(pred_dir, "dense_pred_" + b))
        g = read_nii_image(os.path.join(pred_dir, "gth_dense_pred_" + b))
        ref = spc.hd_percentile(p, g, num_cls, 95)
        assert s["hd_percentile"] == 95.0 and np.array_equal(np.isnan(s["hd_pct"]), np.isnan(ref))
        m = ~np.isnan(ref)
        assert s["hd_pct"][m].tobytes() == ref[m].tobytes(), (s["hd_pct"], ref)
        finite += int(m.sum())
    assert finite > 0


def _csv(path):
    with open(path) as f:
        return list(csv.DictReader(f))


def _same_but_hd95(rows0, rows1, suffix=""):
    assert len(rows0) == len(rows1)
    for r0, r1 in zip(rows0, rows1):
        assert {k: v for k, v in r1.items() if not k.endswith("_hd95" + suffix)} == r0
        assert sum(k.endswith("_hd95" + suffix) for k in r1) == 4


def test_test_eval_hd95_both_trainers(tmp_path, capsys):
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv, source_segmenter as seg
    from pnp_b200.data import label_maps
    from pnp_b200.lib import write_nii
    from pnp_b200.train_gan import configure
    from oracle.pnp_graphs import OracleAdversarial, OracleSegmenter, init_numpy_params
    from tests.models import bn_noise
    rt.set_conv_backend("auto")
    B = 2
    rng = np.random.RandomState(33)
    nii, lab = [], []
    for i, D in enumerate([5, 7]):
        raw = rng.randn(256, 256, D).astype(np.float32)
        raw_y = np.transpose(label_maps(D, 90 + i), (1, 2, 0)).astype(np.int16)
        raw_y[0, 0, 0] = 9
        nii.append(write_nii(raw, "ct_%d_image.nii.gz" % i, str(tmp_path)))
        lab.append(write_nii(raw_y, "ct_%d_label.nii.gz" % i, str(tmp_path)))

    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 6)
    ck, nc, tc = configure("train-gan")
    net = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc)
    rt.load_state_dict(P)
    tr = adv.Trainer(net, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": 3e-4}, train_config=tc, test_label_list=lab,
                     test_nii_list=nii)
    with pytest.raises(ValueError):
        tr.test_eval(str(tmp_path), surface_metrics=False, hd_percentile=95)
    runs = {}
    for q in (None, 95):
        out = str(tmp_path / ("adv_%s" % q))
        os.makedirs(out)
        capsys.readouterr()
        np.random.seed(5)
        res = tr.test_eval(out, flip_correction=True, save_result=True, surface_metrics=True, hd_percentile=q)
        runs[q] = (res, list(tr.sample_eval_list), open(os.path.join(out, "cm.csv")).read(), capsys.readouterr().out, out,
                   list(tr.sample_surface_list))
    (r0, l0, cm0, t0, o0, s0), (r1, l1, cm1, t1, o1, s1) = runs[None], runs[95]
    np.testing.assert_array_equal(r0[0], r1[0])
    np.testing.assert_array_equal(r0[1], r1[1])
    for (d0, j0), (d1, j1) in zip(l0, l1):
        np.testing.assert_array_equal(d0, d1)
        np.testing.assert_array_equal(j0, j1)
    assert cm0 == cm1 and _stddev_block(t0) == _stddev_block(t1)
    assert [ln for ln in _surface_block(t1) if not ln.startswith("hd95_")] == _surface_block(t0) and "hd95_mean" in t1
    _same_but_hd95(_csv(os.path.join(o0, "surface.csv")), _csv(os.path.join(o1, "surface.csv")))
    _check_hd95(s1, os.path.join(o1, "dense_pred"), nii, 5)

    ws, bns = OracleSegmenter.layout()
    Ps = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(Ps, bns, 6)
    snet = seg.Full_DRN(channels=3, n_class=5, batch_size=B,
                        cost_kwargs={"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0})
    rt.load_state_dict(Ps)
    st = seg.Trainer(snet, None, None, num_cls=5, batch_size=B, test_nii_list=nii, test_label_list=lab, optimizer="adam",
                     opt_kwargs={"learning_rate": 1e-3})
    with pytest.raises(ValueError):
        st.test_eval(str(tmp_path), surface_metrics=False, hd_percentile=95)
    runs = {}
    for q in (None, 95):
        out = str(tmp_path / ("seg_%s" % q))
        os.makedirs(out)
        capsys.readouterr()
        res = st.test_eval(out, flip_correction=False, save_result=True, surface_metrics=True, hd_percentile=q)
        runs[q] = (res, list(st.sample_eval_list), capsys.readouterr().out, out, list(st.sample_surface_list))
    np.testing.assert_array_equal(runs[None][0][0], runs[95][0][0])
    np.testing.assert_array_equal(runs[None][0][1], runs[95][0][1])
    assert _stddev_block(runs[None][2]) == _stddev_block(runs[95][2])
    assert [ln for ln in _surface_block(runs[95][2]) if not ln.startswith("hd95_")] == _surface_block(runs[None][2])
    for (d0, j0), (d1, j1) in zip(runs[None][1], runs[95][1]):
        np.testing.assert_array_equal(d0, d1)
        np.testing.assert_array_equal(j0, j1)
    _same_but_hd95(_csv(os.path.join(runs[None][3], "surface.csv")), _csv(os.path.join(runs[95][3], "surface.csv")))
    _check_hd95(runs[95][4], os.path.join(runs[95][3], "test_pred"), nii, 5)


@pytest.mark.parametrize("kind", ["gan", "segmenter"])
def test_native_hd95_mm(kind, tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import native, nifti, preprocess, runtime as rt
    from oracle.pnp_graphs import OracleAdversarial, OracleSegmenter, init_numpy_params
    from tests.models import bn_noise
    rt.set_conv_backend("auto")
    perms = [ph.SIGNED_PERMUTATIONS[i] for i in (5, 41)]
    pairs = ph.write_pairs(str(tmp_path), "ct", [41, 43], perms=perms, shape=(40, 36, 30), spacing=(0.8, 1.1, 1.7))
    ws, bns = (OracleAdversarial if kind == "gan" else OracleSegmenter).layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 6)
    ckpt = str(tmp_path / "ckpt.npz")
    np.savez(ckpt, **P)
    trainer = native.build_trainer(kind, ckpt, 3)
    results = trainer.test_native(pairs, str(tmp_path / "q"), hd_percentile=95)
    organs = ("la_myo", "la_blood", "lv_blood", "aa")
    head = ["subject"] + ["%s_%s" % (o, k) for o in organs for k in native.CSV_COLUMNS + ("hd95_mm",)]
    rows = _csv(str(tmp_path / "q" / "native.csv"))
    assert list(rows[0]) == head and len(rows) == len(pairs)
    lut = {int(v): c for c, v in enumerate(native.label_codes(5).tolist()) if c == 0 or v}
    finite = 0
    for (im, lb), r, row in zip(pairs, results, rows):
        assert [float(row["%s_hd95_mm" % o]) for o in organs] == pytest.approx(list(r["hd_pct"][1:]), rel=0, abs=0, nan_ok=True)
        s = preprocess.Subject(im, lb)
        codes = nifti.load(r["path"]).get_data()
        pred = np.zeros(codes.shape, np.uint8)
        for v, c in lut.items():
            pred[codes == v] = c
        gt = preprocess.map_labels(nifti.load(lb).get_data())[0]
        ref = spc.hd_percentile(pred, gt, 5, 95, native.native_spacing(s))
        np.testing.assert_allclose(r["hd_pct"], ref, rtol=1e-13, atol=0, equal_nan=True)
        finite += int(np.isfinite(ref).sum())
    assert finite > 0
    if kind == "gan":                                  # the command line
        pair_file = str(tmp_path / "pairs")
        with open(pair_file, "w") as f:
            f.write("".join("%s %s\n" % p for p in pairs))
        cli = str(tmp_path / "cli")
        native.main(["--trainer", kind, "--checkpoint", ckpt, "--pairs", pair_file, "--out", cli, "--batch-size", "3",
                     "--hd-percentile", "95"])
        assert list(_csv(os.path.join(cli, "native.csv"))[0]) == head
