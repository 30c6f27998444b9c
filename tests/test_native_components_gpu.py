"""The largest-component post-processing of the native-grid path (native.run / Trainer.test_native(…, largest_component=6 | 26),
evaluate_native.py --largest-component) end to end on seeded phantom subjects (tests/mmwhs_phantom.py) under three signed axis
permutations with anisotropic spacing, with both trainers restored from small seeded checkpoints whose random-weight predictions
are heavily fragmented:
* the written NIfTI equals oracle/components_exact.scipy_lcc of the labels a run without the option writes, bit for bit;
* <organ>_dice equals numpy Dice of the written file against the native ground truth exactly, <organ>_dice_raw the option-free
  run's <organ>_dice, and the component and removed-voxel counts the oracle's;
* ASSD / HD / HD95 equal oracle/surface_exact.py and oracle/surface_percentile.py on the post-processed volume at native spacing
  to 1e-13 relative;
* a run without the option writes exactly the existing native.csv columns and makes no pnp_largest_components call."""
import csv
import os

import numpy as np
import pytest

from oracle import components_exact as ce
from oracle import surface_exact as se
from oracle import surface_percentile as spc
from tests import mmwhs_phantom as ph
from tests.models import bn_noise

pytestmark = pytest.mark.gpu
B = 3
NUM_CLS = 5
ORGANS = ("la_myo", "la_blood", "lv_blood", "aa")


@pytest.fixture(scope="module")
def phantoms(tmp_path_factory):
    import pnp_b200  # noqa: F401
    from oracle.pnp_graphs import OracleAdversarial, OracleSegmenter, init_numpy_params
    d = tmp_path_factory.mktemp("native_lcc")
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
    return {"dir": d, "pairs": pairs, "pair_file": pair_file, "ckpt": ckpt, "plain": {}}


def _csv(path):
    with open(path) as f:
        rows = list(csv.reader(f))
    return rows[0], [dict(zip(rows[0], r)) for r in rows[1:]]


def _classes(path):
    from pnp_b200 import native, nifti
    codes = nifti.load(path).get_data()
    out = np.zeros(codes.shape, np.uint8)
    for c, v in enumerate(native.label_codes(NUM_CLS).tolist()):
        if c and v:
            out[codes == v] = c
    return out


def _dice(pred, gt):
    return np.array([2.0 * ((pred == c) & (gt == c)).sum() / max(1, (pred == c).sum() + (gt == c).sum())
                     if ((pred == c).sum() + (gt == c).sum()) else 0.0 for c in range(NUM_CLS)])


def _run_logged(monkeypatch, fn):
    """fn() with every C-ABI call the functional layer makes recorded -> (its result, the called names)"""
    from pnp_b200 import functional as F
    names = []
    real = F.call

    def logged(name, *args):
        names.append(name)
        return real(name, *args)

    monkeypatch.setattr(F, "call", logged)
    try:
        return fn(), names
    finally:
        monkeypatch.setattr(F, "call", real)


def _plain(phantoms, kind, monkeypatch):
    """the option-free run of this trainer (once per module): results, csv rows, the raw class volumes it wrote"""
    if kind not in phantoms["plain"]:
        from pnp_b200 import native, runtime as rt
        rt.set_conv_backend("auto")
        trainer = native.build_trainer(kind, phantoms["ckpt"][kind], B)
        out = str(phantoms["dir"] / ("plain_" + kind))
        results, names = _run_logged(monkeypatch, lambda: trainer.test_native(phantoms["pairs"], out))
        assert "pnp_native_labels" in names and "pnp_largest_components" not in names
        assert "pnp_largest_components_workspace" not in names
        head, rows = _csv(os.path.join(out, "native.csv"))
        assert head == ["subject"] + ["%s_%s" % (o, k) for o in ORGANS for k in native.CSV_COLUMNS]
        assert all("largest_component" not in r and "dice_raw" not in r for r in results)
        phantoms["plain"][kind] = (results, rows, [_classes(r["path"]) for r in results])
    return phantoms["plain"][kind]


@pytest.mark.parametrize("conn", [6, 26])
@pytest.mark.parametrize("kind", ["gan", "segmenter"])
def test_native_largest_component(phantoms, kind, conn, tmp_path, monkeypatch):
    import pnp_b200  # noqa: F401
    from pnp_b200 import native, preprocess, nifti
    plain_results, plain_rows, raws = _plain(phantoms, kind, monkeypatch)
    trainer = native.build_trainer(kind, phantoms["ckpt"][kind], B)
    out = str(tmp_path / "lcc")
    results, names = _run_logged(monkeypatch, lambda: trainer.test_native(phantoms["pairs"], out, hd_percentile=95,
                                                                          largest_component=conn))
    assert names.count("pnp_largest_components") == len(phantoms["pairs"])
    head, rows = _csv(os.path.join(out, "native.csv"))
    assert head == (["subject"] + ["%s_%s" % (o, k) for o in ORGANS for k in native.CSV_COLUMNS + ("hd95_mm",)]
                    + ["%s_%s" % (o, k) for o in ORGANS for k in ("dice_raw", "components", "removed")])
    removed_total = 0
    for (im, lb), res, row, prow, pres, raw in zip(phantoms["pairs"], results, rows, plain_rows, plain_results, raws):
        s = preprocess.Subject(im, lb)
        gt = preprocess.map_labels(nifti.load(lb).get_data())[0]
        assert res["largest_component"] == conn
        # the written file: scipy's largest components of the option-free prediction, bit for bit
        written = _classes(res["path"])
        want, st, cm = ce.scipy_lcc(raw, NUM_CLS, conn, gt)
        assert np.array_equal(written, want), "%s: %d voxels differ" % (s.name, int((written != want).sum()))
        assert np.array_equal(res["cm"], cm)
        assert np.array_equal(res["components"], st[:, 0]) and np.array_equal(res["kept"], st[:, 1])
        assert np.array_equal(res["removed"], st[:, 2])
        # Dice: post-processed from the call's counts, raw from pnp_native_labels' counts
        assert np.array_equal(res["dice"], _dice(written, gt))
        assert np.array_equal(res["dice_raw"], pres["dice"]) and np.array_equal(res["dice_raw"], _dice(raw, gt))
        for c, o in enumerate(ORGANS, 1):
            assert row["%s_dice" % o] == repr(float(res["dice"][c]))
            assert row["%s_dice_raw" % o] == prow["%s_dice" % o]
            assert int(row["%s_components" % o]) == st[c, 0] and int(row["%s_removed" % o]) == st[c, 2]
        # surface distances of the post-processed labels at native spacing
        sp = native.native_spacing(s)
        ref = se.surface_metrics(written, gt, NUM_CLS, sp)
        for key in ("assd", "hd"):
            np.testing.assert_allclose(res[key], ref[key], rtol=1e-13, atol=0, equal_nan=True)
        assert np.array_equal(res["border_pred"], ref["border_pred"]) and np.array_equal(res["border_gt"], ref["border_gt"])
        np.testing.assert_allclose(res["hd_pct"], spc.hd_percentile(written, gt, NUM_CLS, 95, sp), rtol=1e-13, atol=0,
                                   equal_nan=True)
        removed_total += int(st[1:, 2].sum())
        print("  %s %d-conn %s: components %s, removed %s, Dice raw %s -> %s" % (
            kind, conn, s.name, st[1:, 0].tolist(), st[1:, 2].tolist(), np.round(res["dice_raw"][1:], 4),
            np.round(res["dice"][1:], 4)))
    assert removed_total > 0, "the phantom predictions should carry islands to remove"


def test_evaluate_native_with_largest_component_end_to_end(phantoms, tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import native, preprocess
    cli = str(tmp_path / "cli")
    native.main(["--trainer", "gan", "--checkpoint", phantoms["ckpt"]["gan"], "--pairs", phantoms["pair_file"], "--out", cli,
                 "--batch-size", str(B), "--largest-component", "26"])
    head, rows = _csv(os.path.join(cli, "native.csv"))
    assert head == (["subject"] + ["%s_%s" % (o, k) for o in ORGANS for k in native.CSV_COLUMNS]
                    + ["%s_%s" % (o, k) for o in ORGANS for k in ("dice_raw", "components", "removed")])
    names = [preprocess.subject_name(im) for im, _ in phantoms["pairs"]]
    assert [r["subject"] for r in rows] == names
    assert sorted(os.listdir(os.path.join(cli, "native_pred"))) == sorted(n + "_label.nii.gz" for n in names)
