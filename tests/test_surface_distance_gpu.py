"""pnp_surface_distance (csrc/metrics3d.cu) and its host layer on the device, against oracle/surface_exact.py:
* unit spacing: border counts equal, maxima bit for bit, sums to 1e-12 relative (bit for bit where every distance is an integer);
* anisotropic spacing: sums and maxima to 1e-13 relative;
* shapes from 1 x 1 x 1 through lines and odd sizes to 256 x 256 x 131; classes absent from either volume; labels >= C;
* repeated calls bit-identical; rejected arguments leave `out` untouched;
* both trainers' test_eval(..., surface_metrics=True) on NIfTI subjects against the oracle applied to the saved volumes, with
  Dice / Jaccard, the return values and cm.csv identical to a run without it."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import surface_exact as se

pytestmark = pytest.mark.gpu


def _raw_gpu(pred, gt, C, spacing=None, out=None):
    import pnp_b200  # noqa: F401
    from pnp_b200 import _C, runtime as rt
    p = np.ascontiguousarray(np.where((pred >= 0) & (pred < C), pred, 0), np.uint8)
    g = np.ascontiguousarray(np.where((gt >= 0) & (gt < C), gt, 0), np.uint8)
    nb = ctypes.c_longlong(0)
    _C.call("pnp_surface_distance_workspace", *p.shape, C, ctypes.byref(nb))
    dp, dg = torch.from_numpy(p).cuda(), torch.from_numpy(g).cuda()
    ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    out = torch.empty((C - 1) * 6, dtype=torch.float64, device="cuda") if out is None else out
    sp = None if spacing is None else (ctypes.c_double * 3)(*spacing)
    _C.call("pnp_surface_distance", dp.data_ptr(), dg.data_ptr(), *p.shape, C, sp, ws.data_ptr(), nb.value, out.data_ptr(),
            rt.stream())
    return out.cpu().numpy().reshape(C - 1, 6)


def _check_unit(got, ref):
    """counts and maxima bit for bit, sums to 1e-12 relative, NaN where the oracle has NaN"""
    assert np.array_equal(np.isnan(got), np.isnan(ref)), (got, ref)
    np.testing.assert_array_equal(got[:, [1, 4]], ref[:, [1, 4]])
    np.testing.assert_array_equal(got[:, [2, 5]], ref[:, [2, 5]])
    m = ~np.isnan(ref[:, [0, 3]])
    s, r = got[:, [0, 3]][m], ref[:, [0, 3]][m]
    assert np.all(np.abs(s - r) <= 1e-12 * np.abs(r)), (s, r)


def _ellipsoids(rng, shape, num_cls, lo=0.1, hi=0.45):
    g = np.ogrid[:shape[0], :shape[1], :shape[2]]
    v = np.zeros(shape, np.int64)
    for c in range(1, num_cls):
        centre = rng.uniform(0.1, 0.9, 3) * shape
        radii = rng.uniform(lo, hi, 3) * np.array(shape) + 0.5
        v[sum(((g[a] - centre[a]) / radii[a]) ** 2 for a in range(3)) < 1] = c
    return v


SHAPES = [(1, 1, 1), (1, 1, 40), (1, 33, 1), (47, 1, 1), (1, 9, 14), (37, 29, 23), (16, 64, 5), (8, 3, 200)]


@pytest.mark.parametrize("shape", SHAPES)
def test_matches_oracle_unit_spacing(shape):
    rng = np.random.default_rng(sum(shape))
    for it in range(6):
        C = int(rng.integers(2, 9))
        if it % 2:
            p = rng.integers(0, C + 3, shape) * (rng.random(shape) < rng.uniform(0.02, 0.6))
            g = rng.integers(0, C + 3, shape) * (rng.random(shape) < rng.uniform(0.02, 0.6))
        else:
            p, g = _ellipsoids(rng, shape, C), _ellipsoids(rng, shape, C)
        _check_unit(_raw_gpu(p, g, C), se.scipy_raw(p, g, C))


def test_matches_brute_force_on_small_volumes():
    rng = np.random.default_rng(7)
    for it in range(20):
        shape = tuple(int(x) for x in rng.integers(1, 14, 3))
        C = int(rng.integers(2, 9))
        p = rng.integers(0, C + 1, shape) * (rng.random(shape) < rng.random())
        g = _ellipsoids(rng, shape, C)
        _check_unit(_raw_gpu(p, g, C), se.brute_raw(p, g, C))


def test_256x256x131_subject():
    rng = np.random.default_rng(131)
    shape = (256, 256, 131)
    g = _ellipsoids(rng, shape, 5, 0.1, 0.3)
    p = np.where(rng.random(shape) < 1e-3, rng.integers(0, 7, shape), np.roll(g, (2, -3, 1), (0, 1, 2)))
    got, ref = _raw_gpu(p, g, 5), se.scipy_raw(p, g, 5)
    assert np.all(got[:, 1] > 0) and np.all(got[:, 4] > 0)
    _check_unit(got, ref)


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_parallel_slabs_bit_for_bit(axis):
    shape = [40, 50, 60]
    for k in (1, 4, 17):
        p, g = np.zeros(shape, np.int64), np.zeros(shape, np.int64)
        sl = [slice(None)] * 3
        sl[axis] = 3
        p[tuple(sl)] = 2
        sl[axis] = 3 + k
        g[tuple(sl)] = 2
        got = _raw_gpu(p, g, 3)
        ref = se.scipy_raw(p, g, 3)
        np.testing.assert_array_equal(got, ref)
        n = p.sum() // 2
        assert got[1, 0] == k * n and got[1, 2] == k and got[1, 3] == k * n
        got = _raw_gpu(p, g, 3, spacing=(2.0, 2.0, 2.0))
        assert got[1, 0] == 2 * k * n and got[1, 5] == 2 * k


def test_single_voxels_absent_classes_and_labels_out_of_range():
    p, g = np.zeros((9, 10, 11), np.int64), np.zeros((9, 10, 11), np.int64)
    p[1, 2, 3], g[7, 9, 0] = 1, 1
    p[4, 4, 4] = 2                   # only in the prediction
    g[5, 5, 5] = 3                   # only in the ground truth
    p[0, 0, 0], g[8, 9, 10] = 200, 6  # >= C: background
    got = _raw_gpu(p, g, 5)
    ref = se.scipy_raw(p, g, 5)
    _check_unit(got, ref)
    d = np.sqrt(36.0 + 49.0 + 9.0)
    assert got[0, 0] == got[0, 2] == got[0, 3] == got[0, 5] == d
    assert np.isnan(got[1, [0, 2, 3, 5]]).all() and tuple(got[1, [1, 4]]) == (1, 0)
    assert np.isnan(got[2, [0, 2, 3, 5]]).all() and tuple(got[2, [1, 4]]) == (0, 1)
    assert np.isnan(got[3, [0, 2, 3, 5]]).all() and tuple(got[3, [1, 4]]) == (0, 0)


@pytest.mark.parametrize("shape", [(37, 29, 23), (64, 48, 40), (1, 30, 30)])
def test_anisotropic_spacing(shape):
    rng = np.random.default_rng(11)
    for spacing in [(0.7, 1.3, 2.5), (2.5, 0.7, 1.3), (1.0, 1.0, 3.0)]:
        C = 5
        p, g = _ellipsoids(rng, shape, C), _ellipsoids(rng, shape, C)
        got, ref = _raw_gpu(p, g, C, spacing), se.scipy_raw(p, g, C, spacing)
        assert np.array_equal(np.isnan(got), np.isnan(ref))
        np.testing.assert_array_equal(got[:, [1, 4]], ref[:, [1, 4]])
        m = ~np.isnan(ref)
        assert np.all(np.abs(got[m] - ref[m]) <= 1e-13 * np.abs(ref[m])), (got, ref)


def test_repeated_calls_are_bit_identical():
    rng = np.random.default_rng(3)
    shape = (96, 80, 71)
    p, g = _ellipsoids(rng, shape, 6), _ellipsoids(rng, shape, 6)
    a = _raw_gpu(p, g, 6, (0.7, 1.3, 2.5))
    b = _raw_gpu(p, g, 6, (0.7, 1.3, 2.5))
    assert a.tobytes() == b.tobytes()


def test_rejected_arguments_leave_out_untouched():
    import pnp_b200  # noqa: F401
    from pnp_b200 import _C, runtime as rt
    v = torch.zeros(4 * 5 * 6, dtype=torch.uint8, device="cuda")
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    out = torch.full((8 * 6,), 1234.5, dtype=torch.float64, device="cuda")
    sp = (ctypes.c_double * 3)(1.0, 1.0, 1.0)
    P = v.data_ptr()
    for args, rc in [((4, 5, 6, 9, sp, 1 << 20), 100002), ((4, 5, 6, 1, sp, 1 << 20), 100002),
                     ((4, 0, 6, 5, sp, 1 << 20), 100001), ((4, 5, 1025, 5, sp, 1 << 20), 100002),
                     ((4, 5, 6, 5, (ctypes.c_double * 3)(1.0, 0.0, 1.0), 1 << 20), 100001), ((4, 5, 6, 5, sp, 64), 100001)]:
        n0, n1, n2, C, s, nb = args
        assert _C.lib.pnp_surface_distance(P, P, n0, n1, n2, C, s, ws.data_ptr(), nb, out.data_ptr(), rt.stream()) == rc
    torch.cuda.synchronize()
    assert bool((out == 1234.5).all())


def test_functional_surface_distances_matches_oracle():
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F
    rng = np.random.default_rng(17)
    shape = (50, 41, 33)
    g = _ellipsoids(rng, shape, 5)
    p = np.roll(g, 2, axis=1).astype(np.int32)
    p[p == 3] = 0                                   # organ 3 missing from the prediction
    p[0, 0, :5] = -1                                # negative labels are background too
    for spacing in (None, (0.7, 1.3, 2.5)):
        got, ref = F.surface_distances(p, g, 5, spacing), se.surface_metrics(p, g, 5, spacing)
        for k in ("border_pred", "border_gt"):
            np.testing.assert_array_equal(got[k], ref[k])
        for k in ("asd_pred_gt", "asd_gt_pred", "assd", "hd"):
            assert np.array_equal(np.isnan(got[k]), np.isnan(ref[k])), k
            m = ~np.isnan(ref[k])
            assert np.all(np.abs(got[k][m] - ref[k][m]) <= 1e-12 * np.abs(ref[k][m])), (k, got[k], ref[k])
        assert np.isnan(got["assd"][0]) and np.isnan(got["assd"][3]) and got["border_pred"][3] == 0
        u8 = F.surface_distances(np.where(p < 0, 200, p).astype(np.uint8), g, 5, spacing)    # uint8 goes up unmapped
        for k in got:
            np.testing.assert_array_equal(u8[k], got[k])


# ---- the test protocol of both trainers ----------------------------------------------------------------------------------
def _stddev_block(text):
    lines = text.splitlines()
    a = next(i for i, ln in enumerate(lines) if "inside the sample_metric_stddev" in ln)
    b = next(i for i, ln in enumerate(lines) if ln.startswith("all_jaccard_mean"))
    return lines[a:b + 1]


def _check_subjects(surface_list, pred_dir, nii, num_cls):
    from pnp_b200.lib import read_nii_image
    assert [s["subject"] for s in surface_list] == [os.path.basename(f) for f in nii]
    for s, f in zip(surface_list, nii):
        b = os.path.basename(f).split(".")[0] + ".nii.gz"
        p = read_nii_image(os.path.join(pred_dir, "dense_pred_" + b))
        g = read_nii_image(os.path.join(pred_dir, "gth_dense_pred_" + b))
        ref = se.surface_metrics(p, g, num_cls)
        for k in ("border_pred", "border_gt"):
            np.testing.assert_array_equal(s[k], ref[k])
        for k in ("assd", "hd", "asd_pred_gt", "asd_gt_pred"):
            assert np.array_equal(np.isnan(s[k]), np.isnan(ref[k])), k
            m = ~np.isnan(ref[k])
            assert np.all(np.abs(s[k][m] - ref[k][m]) <= 1e-12 * np.abs(ref[k][m])), (k, s[k], ref[k])
        assert np.isfinite(s["assd"][1:]).any()


def test_test_eval_surface_metrics_both_trainers(tmp_path, capsys):
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv, source_segmenter as seg
    from pnp_b200.data import label_maps
    from pnp_b200.lib import write_nii
    from pnp_b200.train_gan import configure
    from oracle.pnp_graphs import OracleAdversarial, OracleSegmenter, init_numpy_params
    from tests.test_parity_configs_gpu import _bn_noise
    rt.set_conv_backend("auto")
    B = 2
    rng = np.random.RandomState(33)
    nii, lab = [], []
    for i, D in enumerate([5, 7]):
        raw = rng.randn(256, 256, D).astype(np.float32)
        raw_y = np.transpose(label_maps(D, 90 + i), (1, 2, 0)).astype(np.int16)
        raw_y[0, 0, 0] = 9                                              # above the class range: background in the saved truth
        nii.append(write_nii(raw, "ct_%d_image.nii.gz" % i, str(tmp_path)))
        lab.append(write_nii(raw_y, "ct_%d_label.nii.gz" % i, str(tmp_path)))

    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    _bn_noise(P, bns, 6)
    ck, nc, tc = configure("train-gan")
    net = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc)
    rt.load_state_dict(P)
    tr = adv.Trainer(net, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": 3e-4}, train_config=tc, test_label_list=lab,
                     test_nii_list=nii)
    runs = {}
    for on in (False, True):
        out = str(tmp_path / ("adv_%d" % on))
        os.makedirs(out)
        capsys.readouterr()
        np.random.seed(5)
        res = tr.test_eval(out, flip_correction=True, save_result=True, surface_metrics=on)
        runs[on] = (res, list(tr.sample_eval_list), open(os.path.join(out, "cm.csv")).read(), _stddev_block(capsys.readouterr().out), out)
    (r0, l0, cm0, t0, _), (r1, l1, cm1, t1, out1) = runs[False], runs[True]
    np.testing.assert_array_equal(r0[0], r1[0])
    np.testing.assert_array_equal(r0[1], r1[1])
    for (d0, j0), (d1, j1) in zip(l0, l1):
        np.testing.assert_array_equal(d0, d1)
        np.testing.assert_array_equal(j0, j1)
    assert cm0 == cm1 and t0 == t1
    assert not os.path.exists(os.path.join(runs[False][4], "surface.csv"))
    _check_subjects(tr.sample_surface_list, os.path.join(out1, "dense_pred"), nii, 5)
    rows = open(os.path.join(out1, "surface.csv")).read().splitlines()
    assert len(rows) == 3 and rows[1].startswith("ct_0_image.nii.gz,")

    ws, bns = OracleSegmenter.layout()
    Ps = init_numpy_params(ws, bns, 0, 0.05)
    _bn_noise(Ps, bns, 6)
    snet = seg.Full_DRN(channels=3, n_class=5, batch_size=B,
                        cost_kwargs={"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0})
    rt.load_state_dict(Ps)
    st = seg.Trainer(snet, None, None, num_cls=5, batch_size=B, test_nii_list=nii, test_label_list=lab, optimizer="adam",
                     opt_kwargs={"learning_rate": 1e-3})
    runs = {}
    for on in (False, True):
        out = str(tmp_path / ("seg_%d" % on))
        os.makedirs(out)
        capsys.readouterr()
        res = st.test_eval(out, flip_correction=False, save_result=True, surface_metrics=on)
        runs[on] = (res, list(st.sample_eval_list), _stddev_block(capsys.readouterr().out), out)
    np.testing.assert_array_equal(runs[False][0][0], runs[True][0][0])
    np.testing.assert_array_equal(runs[False][0][1], runs[True][0][1])
    assert runs[False][2] == runs[True][2]
    for (d0, j0), (d1, j1) in zip(runs[False][1], runs[True][1]):
        np.testing.assert_array_equal(d0, d1)
        np.testing.assert_array_equal(j0, j1)
    _check_subjects(st.sample_surface_list, os.path.join(runs[True][3], "test_pred"), nii, 5)
    assert os.path.exists(os.path.join(runs[True][3], "surface.csv"))
