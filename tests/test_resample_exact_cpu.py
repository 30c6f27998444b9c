"""The checks of tests/test_resample_exact_gpu.py and tests/test_preprocess_gpu.py that need no GPU:
* oracle/resample_exact.py (the numpy restatement of pnp_resample_planes) against independent fp64 forms -- images against
  scipy.ndimage.map_coordinates(order=1, mode='nearest') within a bound from the count of fp32 roundings, labels against an
  explicit nearest-voxel loop -- and against known answers; each plausible kernel bug changes some output;
* the GPU file's case table reaches the grid-stride cap with two or more iterations and a single partial CTA;
* the host side of preprocess.py against direct numpy: the label table, the orientation of all 48 signed axis permutations of
  one phantom, the heart box, p98 / mu / sigma and the matrix composition."""
import math

import numpy as np
import pytest
from scipy import ndimage

from oracle import resample_exact as R
from tests import mmwhs_phantom as ph
from tests import test_resample_exact_gpu as G

F32 = np.float32
U = 2.0 ** -24


# ------------------------------------------------------------------------------------------------
# the restatement against independent forms
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in G.CASES if "cap" not in c[0]], ids=lambda c: c[0])
def test_image_matches_map_coordinates_within_the_rounding_bound(case):
    """same fp32 coordinates, fp64 interpolation: each lerp level costs at most 3 roundings of values bounded by max|vol| (the
    difference b - a by 2 max|vol|), so |fp32 - fp64| <= 3 levels * 5 u max|vol| (first order) -- 16 u max|vol| covers it"""
    vol, cls, mats = G.operands(case)
    tag, shape, B, H, W, C, image, lp = case
    u = R.coords(mats, B, H, W, C)
    got = R.image_ref(vol, u)
    want = ndimage.map_coordinates(vol.astype(np.float64), [np.nan_to_num(u[a].astype(np.float64)).reshape(-1) for a in range(3)],
                                   order=1, mode="nearest").reshape(got.shape)
    bound = 16 * U * float(np.abs(vol).max())
    err = float(np.abs(got.astype(np.float64) - want).max())
    print("  %s: max |fp32 - fp64| = %.3e (bound %.3e)" % (tag, err, bound))
    assert err <= bound


def _labels_loop(cls, u):
    out = np.zeros(u.shape[1:], np.int64)
    n = cls.shape
    for idx in np.ndindex(*u.shape[1:]):
        v = [float(u[(a,) + idx]) for a in range(3)]
        if all(-0.5 <= v[a] < n[a] - 0.5 for a in range(3)):
            out[idx] = cls[tuple(int(math.floor(v[a] + 0.5)) for a in range(3))]
    return out


@pytest.mark.parametrize("case", [c for c in G.CASES if c[2] * c[3] * c[4] * c[5] <= 20000], ids=lambda c: c[0])
def test_labels_match_an_explicit_nearest_voxel_loop(case):
    vol, cls, mats = G.operands(case)
    tag, shape, B, H, W, C, image, lp = case
    u = R.coords(mats, B, H, W, C)
    assert np.array_equal(R.label_ref(cls, u), _labels_loop(cls, u))


def _planes(mats_list, B, C):
    return np.asarray(mats_list, F32).reshape(B, C, 3, 3)


def test_known_answers():
    rng = np.random.RandomState(5)
    vol = rng.standard_normal((6, 7, 5)).astype(F32)
    cls = rng.randint(0, 9, (6, 7, 5)).astype(np.uint8)
    # identity: plane k samples (r, c, k) -> an exact copy of vol[:, :, k]
    ident = _planes([[[1, 0, 0], [0, 1, 0], [0, 0, k]] for k in range(5)], 1, 5)
    img, lab = R.resample_ref(vol, cls, ident, 1, 6, 7, 5, 5)
    assert np.array_equal(img[0], vol) and np.array_equal(lab[0], cls.astype(np.int64))
    # an integer shift is an exact shift; what falls outside clamps (image) or is class 0 (labels)
    sh = _planes([[[1, 0, 2], [0, 1, -1], [0, 0, 3]]], 1, 1)
    img, lab = R.resample_ref(vol, cls, sh, 1, 6, 7, 1, 1)
    r, c = np.arange(6)[:, None], np.arange(7)[None, :]
    assert np.array_equal(img[0, :, :, 0], vol[np.minimum(r + 2, 5), np.clip(c - 1, 0, 6), 3])
    want = np.where((r + 2 <= 5) & (c - 1 >= 0), cls[np.minimum(r + 2, 5), np.clip(c - 1, 0, 6), 3], 0)
    assert np.array_equal(lab[0], want)
    # 90 degree rotations are exact permutations (np.rot90 of a square slice)
    sq = rng.standard_normal((7, 7, 2)).astype(F32)
    sqc = rng.randint(0, 9, (7, 7, 2)).astype(np.uint8)
    rot = _planes([[[0, 1, 0], [-1, 0, 6], [0, 0, 1]]], 1, 1)          # out[r, c] = in[c, 6 - r]
    img, lab = R.resample_ref(sq, sqc, rot, 1, 7, 7, 1, 1)
    assert np.array_equal(img[0, :, :, 0], np.rot90(sq[:, :, 1])) and np.array_equal(lab[0], np.rot90(sqc[:, :, 1]))
    rot180 = _planes([[[-1, 0, 6], [0, -1, 6], [0, 0, 0]]], 1, 1)
    img, _ = R.resample_ref(sq, sqc, rot180, 1, 7, 7, 1, 0)
    assert np.array_equal(img[0, :, :, 0], np.rot90(sq[:, :, 0], 2))
    # label ties round up: u = k + 0.5 -> voxel k + 1; u = -0.5 -> voxel 0; u = n - 0.5 -> outside
    line = np.arange(1, 6, dtype=np.uint8).reshape(5, 1, 1)
    half = _planes([[[1, 0, -0.5], [0, 0, 0], [0, 0, 0]]], 1, 1)        # u0 = r - 0.5, r = 0 .. 5
    _, lab = R.resample_ref(np.zeros((5, 1, 1), F32), line, half, 1, 6, 1, 1, 1)
    assert lab.reshape(-1).tolist() == [1, 2, 3, 4, 5, 0]
    # an axis of length 1: every coordinate along it clamps to 0 (image) and only [-0.5, 0.5) is inside (labels)
    flat = rng.standard_normal((1, 4, 3)).astype(F32)
    m = _planes([[[0, 0, 0.49], [0, 1, 0], [0, 0, 2]], [[0, 0, -7.0], [0, 1, 0], [0, 0, 2]], [[0, 0, 0.5], [0, 1, 0], [0, 0, 2]]],
                1, 3)
    img, lab = R.resample_ref(flat, np.full((1, 4, 3), 3, np.uint8), m, 1, 1, 4, 3, 3)
    assert all(np.array_equal(img[0, 0, :, k], flat[0, :, 2]) for k in range(3))
    assert lab[0, 0, :, 0].tolist() == [3] * 4 and lab[0, 0, :, 1].tolist() == [0] * 4 and lab[0, 0, :, 2].tolist() == [0] * 4
    # far outside: the image is the clamped corner, labels 0; NaN coordinates clamp to 0 and are class 0
    far = _planes([[[0, 0, -1e6], [0, 0, 1e6], [0, 0, np.nan]]], 1, 1)
    img, lab = R.resample_ref(vol, cls + 1, far, 1, 2, 2, 1, 1)
    assert bool((img == vol[0, 6, 0]).all()) and bool((lab == 0).all())


def test_launch_regimes_of_the_gpu_cases():
    launches = [R.launch(B, H, W, C, image, lp) for _, _, B, H, W, C, image, lp in G.CASES]
    assert any(l.capped and l.iters >= 2 for l in launches)
    assert any(l.single_partial for l in launches)
    assert {c[7] for c in G.CASES} >= {0, 1} and any(c[7] == c[5] > 1 for c in G.CASES)
    assert any(not c[6] and c[7] == 1 for c in G.CASES) and any(not c[6] and c[7] == c[5] for c in G.CASES)
    assert R.launch(2, 256, 256, 70) == R.Launch(8448, True, 5, False)
    assert R.launch(1, 5, 7, 3) == R.Launch(1, False, 1, True)
    assert R.launch(4, 256, 256, 3, False, 1) == R.Launch(256, False, 4, False)


# ------------------------------------------------------------------------------------------------
# negative controls: each plausible kernel bug changes some output of the GPU file's cases
# ------------------------------------------------------------------------------------------------
def _ndiff(**bug):
    d = 0
    for case in G.CASES:
        if "cap" in case[0]:
            continue
        vol, cls, mats = G.operands(case)
        tag, shape, B, H, W, C, image, lp = case
        a = R.resample_ref(vol, cls, mats, B, H, W, C, lp or 1, True)
        b = R.resample_ref(vol, cls, mats, B, H, W, C, lp or 1, True, **bug)
        d += int((a[0].view(np.int32) != b[0].view(np.int32)).sum()) + int((a[1] != b[1]).sum())
    return d


NEGATIVE_CONTROLS = {
    "axes interpolated 0, 1, 2": dict(axis_order=(0, 1, 2)),
    "FMA contraction": dict(fma=True),
    "labels round half to even": dict(half_even=True),
    "coordinates not clamped": dict(no_clamp=True),
}


@pytest.mark.parametrize("bug", list(NEGATIVE_CONTROLS), ids=[k.replace(" ", "_") for k in NEGATIVE_CONTROLS])
def test_negative_control(bug):
    n = _ndiff(**NEGATIVE_CONTROLS[bug])
    print("  NEGATIVE CONTROL %-30s %d differing elements" % (bug, n))
    assert n >= 1


# ------------------------------------------------------------------------------------------------
# host side of the preparation
# ------------------------------------------------------------------------------------------------
def _pp():
    import pnp_b200  # noqa: F401
    from pnp_b200 import preprocess
    return preprocess


def test_label_table():
    pp = _pp()
    from pnp_b200 import evaluation
    cm = evaluation.contour_map
    assert pp.LABEL_TABLE == {205: cm["la_myo"], 420: cm["la_blood"], 500: cm["lv_blood"], 820: cm["aa"]}
    raw = np.array([0, 205, 420, 500, 550, 600, 820, 850, 7, 421, 205.0, 3])
    cls, heart, unknown = pp.map_labels(raw)
    assert cls.tolist() == [0, 1, 2, 3, 0, 0, 4, 0, 0, 0, 1, 0] and cls.dtype == np.uint8
    assert heart.tolist() == [False] + [True] * 7 + [False, False, True, False]
    assert unknown == 3


def test_orientation_of_all_48_signed_permutations():
    """every storage of one phantom gives the same coronal array, spacing and world affine; the array equals the RAS grid
    re-indexed directly: rows along -z, columns along -x, slices along -y"""
    pp = _pp()
    img, lab, aff = ph.ras_subject(3)
    want = np.flip(np.transpose(img, (2, 0, 1)), (0, 1, 2))
    ref_aff = None
    for perm, signs in ph.SIGNED_PERMUTATIONS:
        ri, A = ph.permuted(img, aff, perm, signs)
        axis, sign, zooms, angle = pp.orientation(A)
        assert axis == list(perm) and sign == list(signs) and angle == 0.0
        arr, sp, caff, _ = pp.to_coronal(ri, A)
        assert np.array_equal(arr, want), (perm, signs)
        assert np.allclose(sp, [aff[2, 2], aff[0, 0], aff[1, 1]], rtol=0, atol=1e-12)
        ref_aff = caff if ref_aff is None else ref_aff
        assert np.allclose(caff, ref_aff, rtol=0, atol=1e-9)
    # the coronal affine maps coronal voxel (0, 0, 0) to the superior, right, anterior corner of the RAS grid
    corner = aff @ np.array([img.shape[0] - 1, img.shape[1] - 1, img.shape[2] - 1, 1.0])
    assert np.allclose(ref_aff @ np.array([0, 0, 0, 1.0]), corner)
    # a slightly oblique affine keeps the permutation and reports its angle
    th = np.deg2rad(4.0)
    rot = np.eye(4)
    rot[:2, :2] = [[math.cos(th), -math.sin(th)], [math.sin(th), math.cos(th)]]
    axis, sign, zooms, angle = pp.orientation(rot @ aff)
    assert axis == [0, 1, 2] and sign == [1, 1, 1] and abs(angle - 4.0) < 1e-9
    assert np.allclose(zooms, np.diag(aff)[:3])


def test_heart_box_and_intensity_statistics():
    pp = _pp()
    img, lab, aff = ph.ras_subject(11, unknown=5)
    _, heart, unknown = pp.map_labels(lab)
    assert unknown == 5
    box = pp.heart_box(heart)
    nz = np.argwhere(np.isin(lab, pp.MMWHS_VALUES))
    assert box == [(int(nz[:, a].min()), int(nz[:, a].max())) for a in range(3)]
    raw = img[box[0][0]:box[0][1] + 1, box[1][0]:box[1][1] + 1, box[2][0]:box[2][1] + 1].astype(np.float64)
    p98, mu, sigma = pp.intensity_stats(raw)
    s = np.sort(raw.reshape(-1))
    pos = 0.98 * (s.size - 1)
    lo = int(math.floor(pos))
    assert p98 == pytest.approx(s[lo] + (pos - lo) * (s[min(lo + 1, s.size - 1)] - s[lo]), rel=1e-15)
    c = np.minimum(raw, p98).reshape(-1)
    assert mu == pytest.approx(math.fsum(c) / c.size, rel=1e-13)
    assert sigma == pytest.approx(math.sqrt(math.fsum((c - math.fsum(c) / c.size) ** 2) / c.size), rel=1e-12)
    assert p98 < 3000.0 and (raw >= 3000).any()
    with pytest.raises(ValueError):
        pp.heart_box(np.zeros((3, 3, 3), bool))
    with pytest.raises(ValueError):
        pp.intensity_stats(np.ones((2, 2, 2)))


def test_matrix_composition(tmp_path):
    """base(j) @ T in fp64, rounded once; T maps output pixels to the un-augmented frame about the crop centre"""
    pp = _pp()
    pairs = ph.write_pairs(str(tmp_path), "mr", [4])
    s = pp.Subject(*pairs[0])
    rng = np.random.RandomState(9)
    j, T = s.draw(rng, True)
    r2 = np.random.RandomState(9)
    assert j == r2.randint(s.j_lo, s.j_hi + 1)
    th, sc, t = np.deg2rad(r2.uniform(-15, 15)), r2.uniform(0.9, 1.1, 2), r2.uniform(-10, 10, 2)
    p = np.array([3.0, 250.0])
    q = T[:2, :2] @ p + T[:2, 2]
    rot = np.array([[math.cos(th), -math.sin(th)], [math.sin(th), math.cos(th)]])
    assert np.allclose(q, 127.5 + t + rot @ (sc * (p - 127.5)), rtol=0, atol=1e-12)
    m = s.matrices((j - 1, j, j + 1), T, slice_offset=40)
    assert m.dtype == np.float32 and m.shape == (3, 3, 3)
    for k, jj in enumerate((j - 1, j, j + 1)):
        want = s.base(jj) @ T
        want[0, 2] += 40
        assert np.array_equal(m[k], want.astype(np.float32))
    # neighbouring channels are one output pixel apart along the slice axis: px / spacing source voxels
    assert np.allclose(np.diff(m[:, 0, 2].astype(np.float64)), s.px / s.spacing[2], rtol=0, atol=1e-5)
    # the identity: base alone, and the pixel (r, c) of slice j lands at the crop centre plus the pixel offset in mm
    b = s.matrices((j,))[0].astype(np.float64)
    r, c = 100.0, 31.0
    u = b @ np.array([r, c, 1.0])
    assert np.allclose(u[1] + s.lo[0], s.centre[0] + (r - 127.5) * s.px / s.spacing[0], atol=1e-4)
    assert np.allclose(u[2] + s.lo[1], s.centre[1] + (c - 127.5) * s.px / s.spacing[1], atol=1e-4)
    # every sample an augmentation can draw stays inside the uploaded sub-volume (no clamping at its edge)
    for _ in range(200):
        j, T = s.draw(rng, True)
        for mm in s.matrices((j - 1, j, j + 1), T).astype(np.float64):
            for rr, cc in ((0, 0), (0, 255), (255, 0), (255, 255)):
                uu = mm @ np.array([rr, cc, 1.0])
                assert np.all(uu >= 0) and np.all(uu <= np.array(s.vol.shape) - 1)
