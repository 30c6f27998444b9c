"""The nearest-neighbour reference of the surface distances (oracle/surface_kdtree.py) against the two older ones of
oracle/surface_exact.py and oracle/surface_percentile.py, on the case tables of the GPU tests of pnp_surface_distance(_pct):
* unit spacing: border voxels, the per-class distance arrays (da, db) and the raw [C-1, 6] table bit for bit scipy's, and
  hd_percentile(form="kdtree") bit for bit form="scipy", on the SHAPES table, slabs, absent classes, labels >= C and a
  160 x 150 x 140 phantom;
* the all-pairs search on small volumes, at unit and anisotropic spacing bit for bit (both take the exact minimum of the
  header's expression);
* the phantoms of the native-size GPU tests, and the power of these checks: a 26-neighbour border and a distance with s0 and s2
  swapped both fail them."""
import numpy as np
import pytest
from scipy import ndimage

from oracle import surface_exact as se
from oracle import surface_kdtree as sk
from oracle import surface_percentile as spc

QS = (0.0, 12.5, 50.0, 95.0, 99.0, 100.0)
SHAPES = [(1, 1, 1), (1, 1, 40), (1, 33, 1), (47, 1, 1), (1, 9, 14), (37, 29, 23), (16, 64, 5), (8, 3, 200)]
SPACINGS = [(0.7, 1.3, 2.5), (2.5, 0.7, 1.3), (1.0, 1.0, 3.0), (0.36, 0.36, 0.62)]


def _ellipsoids(rng, shape, num_cls, lo=0.1, hi=0.45):
    g = np.ogrid[:shape[0], :shape[1], :shape[2]]
    v = np.zeros(shape, np.int64)
    for c in range(1, num_cls):
        centre = rng.uniform(0.1, 0.9, 3) * shape
        radii = rng.uniform(lo, hi, 3) * np.array(shape) + 0.5
        v[sum(((g[a] - centre[a]) / radii[a]) ** 2 for a in range(3)) < 1] = c
    return v


def _same_arrays(kd, ref, C):
    """(dist, borders of pred, borders of gt) of kdtree_distances against scipy_distances' or brute_distances', bit for bit"""
    (dk, ka, kb), (dr, ra, rb) = kd, ref
    for c in range(1, C):
        assert np.array_equal(ka[c], np.argwhere(ra[c])) and np.array_equal(kb[c], np.argwhere(rb[c])), c
        if dr[c][0] is None:
            assert dk[c] == (None, None), c
            continue
        for x, y in zip(dk[c], dr[c]):
            assert x.tobytes() == y.tobytes(), (c, x, y)


def _check_scipy(p, g, C, qs=()):
    """kdtree against scipy at unit spacing: borders, distance arrays and raw table bit for bit, and hd_percentile at qs"""
    kd = sk.kdtree_distances(p, g, C)
    _same_arrays(kd, spc.scipy_distances(p, g, C), C)
    got, ref = sk.raw_table(*kd), se.scipy_raw(p, g, C)
    assert got.tobytes() == ref.tobytes(), (got, ref)
    for q in qs:
        a, b = spc.hd_percentile(p, g, C, q, form="kdtree"), spc.hd_percentile(p, g, C, q)
        assert a.tobytes() == b.tobytes(), (q, a, b)
    return got


def _check_brute(p, g, C, spacing=None):
    kd = sk.kdtree_distances(p, g, C, spacing)
    _same_arrays(kd, spc.brute_distances(p, g, C, spacing), C)
    got, ref = sk.raw_table(*kd), se.brute_raw(p, g, C, spacing)
    assert got.tobytes() == ref.tobytes(), (spacing, got, ref)
    return got


@pytest.mark.parametrize("shape", SHAPES)
def test_equals_scipy_bit_for_bit_on_the_gpu_shape_table(shape):
    rng = np.random.default_rng(sum(shape))
    for it in range(6):
        C = int(rng.integers(2, 9))
        if it % 2:
            p = rng.integers(0, C + 3, shape) * (rng.random(shape) < rng.uniform(0.02, 0.6))
            g = rng.integers(0, C + 3, shape) * (rng.random(shape) < rng.uniform(0.02, 0.6))
        else:
            p, g = _ellipsoids(rng, shape, C), _ellipsoids(rng, shape, C)
        _check_scipy(p, g, C, QS)


def test_equals_brute_force_on_small_volumes_at_unit_and_anisotropic_spacing():
    for seed in (7, 77):
        rng = np.random.default_rng(seed)
        for it in range(20):
            shape = tuple(int(x) for x in rng.integers(1, 14, 3))
            C = int(rng.integers(2, 9))
            p = rng.integers(0, C + 1, shape) * (rng.random(shape) < rng.random())
            g = _ellipsoids(rng, shape, C)
            _check_brute(p, g, C)
            _check_brute(p, g, C, SPACINGS[it % len(SPACINGS)])
            _check_brute(p, g, C, tuple(float(x) for x in rng.uniform(0.3, 3.0, 3)))


@pytest.mark.parametrize("shape", [(37, 29, 23), (64, 48, 40), (1, 30, 30)])
def test_equals_brute_force_at_anisotropic_spacing(shape):
    rng = np.random.default_rng(11)
    for spacing in SPACINGS:
        p, g = _ellipsoids(rng, shape, 5), _ellipsoids(rng, shape, 5)
        got = _check_brute(p, g, 5, spacing)
        ref = se.scipy_raw(p, g, 5, spacing)
        m = ~np.isnan(ref)
        assert np.all(np.abs(got[m] - ref[m]) <= 1e-13 * np.abs(ref[m]))


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_slabs_bit_for_bit(axis):
    shape = [40, 50, 60]
    for k in (1, 4, 17):
        p, g = np.zeros(shape, np.int64), np.zeros(shape, np.int64)
        sl = [slice(None)] * 3
        sl[axis] = 3
        p[tuple(sl)] = 2
        sl[axis] = 3 + k
        g[tuple(sl)] = 2
        got = _check_scipy(p, g, 3, QS + (37.25,))
        assert got[1, 2] == got[1, 5] == k
        assert sk.kdtree_raw(p, g, 3, (2.0, 2.0, 2.0))[1, 2] == 2 * k


def test_absent_classes_and_labels_out_of_range():
    p, g = np.zeros((9, 10, 11), np.int64), np.zeros((9, 10, 11), np.int64)
    p[1, 2, 3], g[7, 9, 0] = 1, 1
    p[4, 4, 4] = 2                   # only in the prediction
    g[5, 5, 5] = 3                   # only in the ground truth
    p[0, 0, 0], g[8, 9, 10] = 200, 6  # >= C: background
    p[8, 0, 0] = -4                  # negative: background
    got = _check_scipy(p, g, 5, QS)
    assert got[0, 0] == got[0, 2] == np.sqrt(36.0 + 49.0 + 9.0)
    assert np.isnan(got[1:, [0, 2, 3, 5]]).all() and got[1:, [1, 4]].tolist() == [[1, 0], [0, 1], [0, 0]]
    _check_brute(p, g, 5, (0.7, 1.3, 2.5))
    assert sk.kdtree_raw(p.astype(np.uint8), g.astype(np.uint8), 5).tobytes() == got.tobytes()


def test_160x150x140_phantom_equals_scipy():
    p, g = sk.native_ct_subject(5, (160, 150, 140), 8)
    got = _check_scipy(p, g, 8)
    assert np.all(got[:, [1, 4]] > 0)


# ---- the phantoms of the native-size GPU tests ---------------------------------------------------------------------------------
def test_native_ct_subject_has_what_its_docstring_promises():
    shape, C = (96, 90, 60), 8
    p, g = sk.native_ct_subject(3, shape, C)
    q, h = sk.native_ct_subject(3, shape, C)
    assert p.dtype == g.dtype == np.uint8 and p.shape == g.shape == shape
    assert np.array_equal(p, q) and np.array_equal(g, h)
    assert set(np.unique(g).tolist()) == set(range(C))
    assert (g[0] == 1).any() and (g[:, :, -1] == 2).any()
    touch = [(g[tuple(slice(1, None) if b == a else slice(None) for b in range(3))] *
              g[tuple(slice(None, -1) if b == a else slice(None) for b in range(3))] == 12).any() for a in range(3)]
    assert any(touch)                                               # a 3 next to a 4
    assert (p >= C).any() and 0.5e-3 < np.mean(p != np.roll(g, (3, -2, 2), (0, 1, 2))) < 0.3
    _check_scipy(p, g, C, (95.0,))


@pytest.mark.parametrize("shape,axis", [((1024, 5, 6), 0), ((4, 1024, 3), 1), ((3, 4, 1024), 2), ((40, 5, 6), 0)])
def test_line_features_reach_n_minus_1(shape, axis):
    p, g = sk.line_features(shape, axis)
    n = shape[axis]
    got = _check_brute(p, g, 4)
    assert got[0, 2] == got[0, 5] == n - 1 and got[0, 1] == got[0, 4] == 1
    assert got[1, 4] == n and got[2, 1] == 2
    for spacing in SPACINGS[:2]:
        _check_brute(p, g, 4, spacing)


# ---- the checks above have power ----------------------------------------------------------------------------------------------
def test_a_26_neighbour_border_is_caught(monkeypatch):
    def border26(x):
        return x & ~ndimage.binary_erosion(x, structure=np.ones((3, 3, 3), bool), border_value=0)
    rng = np.random.default_rng(sum(SHAPES[5]))
    p, g = _ellipsoids(rng, SHAPES[5], 5), _ellipsoids(rng, SHAPES[5], 5)
    _check_scipy(p, g, 5)
    monkeypatch.setattr(sk, "_border", border26)
    with pytest.raises(AssertionError):
        _check_scipy(p, g, 5)
    with pytest.raises(AssertionError):
        _check_brute(p, g, 5)


def test_a_distance_with_s0_and_s2_swapped_is_caught(monkeypatch):
    d2 = sk._d2
    rng = np.random.default_rng(11)
    p, g = _ellipsoids(rng, (37, 29, 23), 5), _ellipsoids(rng, (37, 29, 23), 5)
    _check_brute(p, g, 5, SPACINGS[0])
    monkeypatch.setattr(sk, "_d2", lambda src, dst, sp: d2(src, dst, (sp[2], sp[1], sp[0])))
    _check_scipy(p, g, 5)                                  # invisible at unit spacing ...
    with pytest.raises(AssertionError):
        _check_brute(p, g, 5, SPACINGS[0])                 # ... caught at anisotropic spacing
