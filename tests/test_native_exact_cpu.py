"""The checks of tests/test_native_exact_gpu.py and tests/test_native_eval_gpu.py that need no GPU:
* oracle/native_exact.py (the numpy restatement of pnp_native_labels) against scipy.ndimage.map_coordinates(order=1,
  mode='nearest') per class followed by a first-max argmax, wherever the top two fp64 scores are further apart than the fp32
  rounding bound; each plausible kernel bug changes some output;
* the GPU file's case table reaches the grid-stride cap with two or more iterations and a single partial CTA;
* the host map of native.py: for all 48 signed axis permutations of one phantom, the fp64 native voxel -> prepared coordinate map
  composed with Subject.base (and the coronal frame) is the identity, and the native-to-world path agrees with
  Subject.test_affine()."""
import numpy as np
import pytest
from scipy import ndimage

from oracle import native_exact as N
from tests import mmwhs_phantom as ph
from tests import test_native_exact_gpu as G

F32 = np.float32
U = 2.0 ** -24
CPU_CASES = [c for c in G.CASES if "cap" not in c[0]]


# ------------------------------------------------------------------------------------------------
# the restatement against an independent form
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CPU_CASES, ids=lambda c: c[0])
def test_labels_match_map_coordinates_outside_the_rounding_bound(case):
    """same fp32 coordinates, fp64 interpolation per class (scipy), first maximum: each fp32 score is within 16 u max|scores| of
    its fp64 value (tests/test_resample_exact_cpu.py derives the bound), so where the fp64 top two differ by more than twice that
    the argmax cannot differ"""
    tag, n, C, m, _, _ = case
    scores, vmap, _ = G.operands(case)
    got = N.labels_ref(scores, vmap, m)
    u = N.coords(vmap, m)
    ok = N.inside(u, n)
    assert not got[~ok].any()
    pts = [u[a][ok].astype(np.float64) for a in range(3)]
    v = np.stack([ndimage.map_coordinates(scores[..., c].astype(np.float64), pts, order=1, mode="nearest") for c in range(C)])
    want = np.argmax(v, axis=0)             # numpy's argmax returns the first maximum
    top2 = np.sort(v, axis=0)[-2:]
    bound = 2 * 16 * U * float(np.abs(scores).max())
    clear = (top2[1] - top2[0]) > bound
    agree = got[ok][clear] == want[clear]
    print("  %s: %d inside voxels, %d within the bound %.2e of a tie, %d disagreements elsewhere" % (
        tag, int(ok.sum()), int((~clear).sum()), bound, int((~agree).sum())))
    assert agree.all()
    assert ok.sum() > 0 or tag.startswith("nan")          # the NaN case's coordinates are NaN or infinite everywhere


def test_known_answers():
    """identity map: the argmax of the score volume itself; a constant class wins exactly where the others are lower; ties go to
    the lowest index; the confusion counts are np.bincount's"""
    rng = np.random.RandomState(4)
    n = (5, 6, 7)
    s = rng.standard_normal(n + (4,)).astype(F32)
    ident = np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0], F32)
    assert np.array_equal(N.labels_ref(s, ident, n), np.argmax(s, axis=3).astype(np.uint8))
    tie = np.repeat(s[..., :1], 4, axis=3)
    assert not N.labels_ref(tie, ident, n).any()
    assert (N.labels_ref(tie, ident, n, ge=True) == 3).all()
    shifted = ident.copy()
    shifted[3] = -1.0                       # u0 = i - 1: the first native slice is outside
    lab = N.labels_ref(s, shifted, n)
    assert not lab[0].any() and np.array_equal(lab[1:], np.argmax(s[:-1], axis=3).astype(np.uint8))
    gt = rng.randint(0, 6, n).astype(np.uint8)
    cm = N.confusion_ref(lab, gt, 4)
    g = np.where(gt < 4, gt, 0)
    assert all(cm[a, b] == int(((g == a) & (lab == b)).sum()) for a in range(4) for b in range(4))


def test_launch_regimes_of_the_gpu_cases():
    launches = [N.launch(*c[3]) for c in G.CASES]
    assert any(l.capped and l.iters >= 2 for l in launches)
    assert any(l.single_partial for l in launches)
    assert {c[2] for c in G.CASES} >= {2, 5, 8}
    assert N.launch(220, 205, 200) == N.Launch(8448, True, 5, False)
    assert N.launch(5, 7, 9) == N.Launch(1, False, 2, True)


# ------------------------------------------------------------------------------------------------
# negative controls: each plausible kernel bug changes some output of the GPU file's cases
# ------------------------------------------------------------------------------------------------
NEGATIVE_CONTROLS = {
    "FMA-contracted coordinates": dict(fma=True),
    "axes interpolated 0, 1, 2": dict(axis_order=(0, 1, 2)),
    "argmax with >=": dict(ge=True),
    "upper bound n - 0.5 inclusive": dict(inclusive=True),
    "no NaN guard": dict(no_nan_guard=True),
}


@pytest.mark.parametrize("bug", list(NEGATIVE_CONTROLS), ids=[k.replace(" ", "_") for k in NEGATIVE_CONTROLS])
def test_negative_control(bug):
    d = 0
    for case in CPU_CASES:
        scores, vmap, _ = G.operands(case)
        m = case[3]
        d += int((N.labels_ref(scores, vmap, m) != N.labels_ref(scores, vmap, m, **NEGATIVE_CONTROLS[bug])).sum())
    print("  NEGATIVE CONTROL %-32s %d differing labels" % (bug, d))
    assert d >= 1


# ------------------------------------------------------------------------------------------------
# the host map of native.py
# ------------------------------------------------------------------------------------------------
def _subjects(tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import preprocess
    for i, (perm, signs) in enumerate(ph.SIGNED_PERMUTATIONS):
        d = tmp_path / ("p%02d" % i)
        d.mkdir()
        (pair,) = ph.write_pairs(str(d), "ct", [31], perms=[(perm, signs)], shape=(30, 27, 18), spacing=(0.7, 0.9, 1.6))
        yield preprocess.Subject(*pair)


def test_voxel_map_inverts_the_preparation_for_all_48_signed_permutations(tmp_path):
    from pnp_b200 import native, preprocess
    S = preprocess.SIZE - 1
    count = 0
    for s in _subjects(tmp_path):
        M = native.voxel_map(s)
        A = s.native_affine
        corners = np.array([[i, j, k, 1.0] for i in (0, s.native_shape[0] - 1) for j in (0, s.native_shape[1] - 1)
                            for k in (0, s.native_shape[2] - 1)] + [[3.0, 7.0, 2.0, 1.0]])
        for v in corners:
            sl, r, c = M @ v
            # Subject.base: prepared pixel (r, c) of slice sl -> sub-volume (slice, row, column); + lo -> coronal (row, column,
            # slice); the coronal frame -> native voxel
            sub = s.base(sl) @ np.array([r, c, 1.0])
            coronal = np.array([sub[1] + s.lo[0], sub[2] + s.lo[1], sub[0] + s.lo[2], 1.0])
            assert np.abs(s.frame @ coronal - v).max() <= 1e-9, (s.name, v)
            # native -> world equals the stored test volume's affine at the same point: test voxel (255 - r, 255 - c, sl)
            world = s.test_affine() @ np.array([S - r, S - c, sl, 1.0])
            assert np.abs(world - A @ v).max() <= 1e-9, (s.name, v)
        assert np.allclose(native.native_spacing(s)[list(s.frame[:3, :3].nonzero()[0])], s.spacing[list(s.frame[:3, :3].nonzero()[1])],
                           rtol=0, atol=1e-6)
        assert native.map32(s).dtype == np.float32 and np.array_equal(native.map32(s), M.astype(np.float32).reshape(-1))
        count += 1
    assert count == 48


def test_label_codes_and_frame_batches():
    import pnp_b200  # noqa: F401
    from pnp_b200 import native
    assert native.label_codes(5).tolist() == [0, 205, 420, 500, 820] and native.label_codes(5).dtype == np.int16
    assert native.label_codes(3).tolist() == [0, 205, 420]
    assert native.frame_batches(9, 3) == [[1, 2, 3], [4, 5, 6], [7]]
    assert native.frame_batches(8, 3) == [[1, 2, 3], [4, 5, 6]]
    assert sum(native.frame_batches(40, 8), []) == list(range(1, 39))
