"""pnp_surface_distance and pnp_surface_distance_pct (csrc/metrics3d.cu) at the sizes the native-grid evaluation runs them at,
against the nearest-neighbour reference oracle/surface_kdtree.py, at the C-ABI and through functional.surface_distances:
* every axis at PNP_SD_MAX_DIM = 1024 and on both sides of the size at which a transform pass needs more than 48 KB of dynamic
  shared memory (n2 764 / 765 for the axis-2 pass, n1 and n0 768 / 769 for the envelope passes), with one-voxel features at
  the two ends of a line (distance 1023, envelopes of up to 1024 parabolas) and C = 8 ellipsoids;
* the percentile's chunked scan of the per-block query counts (1024 block totals per chunk): L = n1 n2 past 131072 at
  8 x 512 x 300 (two chunks) and 4 x 1024 x 1024 (eight), with classes whose lines cover every chunk, lie in the last chunk
  only, or have dA in chunk 0 and dB in the last chunk only (|dA| = off(L) is then read across chunks);
* a 512 x 512 x 300 CT phantom with C = 8 at unit spacing and at CT spacing, repeated calls bit-identical, and native.surface_mm
  of a subject stored with a permuted, flipped affine equal to the call given that spacing explicitly;
* at every shape the workspace sizes are the header's formulas, a call one byte short is refused with out left at its NaN
  sentinel, and a call on exactly that many bytes writes every slot of out.
Unit spacing: counts, maxima and HD_q bit for bit, sums to 1e-12 relative; other spacings: everything to 1e-13 relative;
columns 0-5 of the percentile call bit-identical to pnp_surface_distance.  With -s every case prints which passes take more
than 48 KB of shared memory, how many scan chunks run, and the oracle's and the kernels' wall times."""
import ctypes
import time

import numpy as np
import pytest
import torch

from oracle import surface_kdtree as sk
from tests import cabi

pytestmark = pytest.mark.gpu
QS = (0.0, 5.0, 50.0, 95.0, 99.5, 100.0)
ANISO = (0.7, 1.3, 2.5)
CT_SPACING = (0.3515625, 0.3515625, 0.625)   # 180 mm / 512 in plane, 0.625 mm slices: exact in the fp32 of a NIfTI header
SENTINEL = 0x7FF80000DEADBEEF                 # a quiet NaN no kernel writes

# launch geometry of csrc/metrics3d.cu
ROWS = LINES = 32          # lines per block of the axis-2 pass / of the envelope passes (int16 per entry)
SCAN = 256                 # axis-0 lines per block total of sd_count_kernel
SCAN_CHUNK = 1024          # block totals sd_scan_kernel scans per iteration
SMEM_DEFAULT = 48 * 1024   # above this a kernel needs cudaFuncAttributeMaxDynamicSharedMemorySize
PASSES = ("pass2", "pass1", "pass0")

AXIS_CASES = [((768, 6, 5), 0), ((769, 6, 5), 0), ((1024, 6, 5), 0), ((5, 768, 6), 1), ((6, 769, 5), 1), ((5, 1024, 6), 1),
              ((6, 5, 764), 2), ((5, 6, 765), 2), ((6, 5, 1024), 2)]
CHUNK_SHAPES = [(8, 512, 300), (4, 1024, 1024)]
NATIVE_SHAPE = (512, 512, 300)
ALL_SHAPES = [s for s, _ in AXIS_CASES] + CHUNK_SHAPES + [NATIVE_SHAPE]


def smem_bytes(shape):
    n0, n1, n2 = shape
    return {"pass2": ROWS * (((n2 + 3) & ~3) + 2) * 2, "pass1": n1 * LINES * 2, "pass0": n0 * LINES * 2}


def scan_chunks(shape):
    return cabi.cdiv(cabi.cdiv(2 * shape[1] * shape[2], SCAN), SCAN_CHUNK)


def line_chunks(idx, t, shape):
    """the scan chunks of the axis-0 lines g = t L + l that hold the border voxels idx [n, 3] (t = 0: dA, 1: dB)"""
    L = shape[1] * shape[2]
    return set(((t * L + idx[:, 1] * shape[2] + idx[:, 2]) // (SCAN * SCAN_CHUNK)).tolist())


def workspace_bytes(shape, pct):
    """the workspace formulas of include/pnp_b200.h"""
    A = lambda x: (x + 255) // 256 * 256
    n0, n1, n2 = shape
    N, L = n0 * n1 * n2, n1 * n2
    b = A(2 * N) + A(4 * N) + A(8 * N) + 2 * A(16 * L) + A(8 * L)
    return b + (A(16 * N) + A(8 * L) + A(8 * cabi.cdiv(2 * L, 256)) + A(16584) if pct else 0)


def _describe(tag, shape):
    s = smem_bytes(shape)
    big = [p for p in PASSES if s[p] > SMEM_DEFAULT]
    print("\n  %s %s: passes over 48 KB of shared memory: %s; scan chunks: %d" % (
        tag, shape, ", ".join("%s (%d B)" % (p, s[p]) for p in big) or "none", scan_chunks(shape)))


def _sentinel(n):
    return torch.full((n,), SENTINEL, dtype=torch.int64, device="cuda").view(torch.float64)


def _kernel(pred, gt, C, spacing=None, qs=QS):
    """-> (out of pnp_surface_distance [C-1, 6], outs of pnp_surface_distance_pct [len(qs), C-1, 7], kernel wall seconds).
    pred and gt go up as they are (labels >= C included).  Per entry point: the workspace size is the header's formula, a call
    one byte short returns PNP_ERR_BAD_ARG and leaves out at its sentinel, the calls on exactly that many bytes write every
    slot.  Each workspace is freed before the next."""
    _C, rt = cabi.lib()
    shape = tuple(pred.shape)
    dp = torch.from_numpy(np.ascontiguousarray(pred, np.uint8)).cuda()
    dg = torch.from_numpy(np.ascontiguousarray(gt, np.uint8)).cuda()
    sp = None if spacing is None else (ctypes.c_double * 3)(*spacing)
    res, wall = {}, 0.0
    for pct in (False, True):
        name = "pnp_surface_distance_pct" if pct else "pnp_surface_distance"
        nb = ctypes.c_longlong(-1)
        _C.call(name + "_workspace", *shape, C, ctypes.byref(nb))
        assert nb.value == workspace_bytes(shape, pct), (name, shape, nb.value)
        ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
        cols = 7 if pct else 6

        def run(q, nbytes, out):
            extra = (float(q),) if pct else ()
            return getattr(_C.lib, name)(dp.data_ptr(), dg.data_ptr(), *shape, C, sp, *extra, ws.data_ptr(), nbytes,
                                         out.data_ptr(), rt.stream())
        out = _sentinel((C - 1) * cols)
        assert run(qs[0], nb.value - 1, out) == cabi.BAD_ARG
        cabi.sync()
        assert bool((out.view(torch.int64) == SENTINEL).all()), (name, "wrote out on a refused call")
        outs = [_sentinel((C - 1) * cols) for _ in (qs if pct else (None,))]
        cabi.sync()
        t0 = time.perf_counter()
        for q, o in zip(qs, outs):
            assert run(q, nb.value, o) == 0
        cabi.sync()
        wall += time.perf_counter() - t0
        for o in outs:
            assert not bool((o.view(torch.int64) == SENTINEL).any()), (name, "left a slot of out unwritten")
        res[pct] = np.stack([o.cpu().numpy().reshape(C - 1, cols) for o in outs])
        del ws, out, outs
        torch.cuda.empty_cache()
    return res[False][0], res[True], wall


def _check(pred, gt, C, spacing=None, qs=QS, tag=""):
    """both entry points against the kdtree reference -> (six, seven, kdtree_distances' result)"""
    t0 = time.perf_counter()
    kd = sk.kdtree_distances(pred, gt, C, spacing)
    ref = sk.raw_table(*kd)
    t_oracle = time.perf_counter() - t0
    six, seven, t_kernel = _kernel(pred, gt, C, spacing, qs)
    print("    %s, spacing %s: oracle %.2f s, kernels %.3f s (%d calls)" % (tag, spacing or "unit", t_oracle, t_kernel,
                                                                           1 + len(qs)))
    for i, q in enumerate(qs):
        assert seven[i, :, :6].tobytes() == six.tobytes(), (tag, q)
    assert np.array_equal(np.isnan(six), np.isnan(ref)), (tag, six, ref)
    np.testing.assert_array_equal(six[:, [1, 4]], ref[:, [1, 4]], err_msg=tag)
    m = ~np.isnan(ref)
    if spacing is None:
        np.testing.assert_array_equal(six[:, [2, 5]], ref[:, [2, 5]], err_msg=tag)
        s, r = six[:, [0, 3]][m[:, [0, 3]]], ref[:, [0, 3]][m[:, [0, 3]]]
        assert np.all(np.abs(s - r) <= 1e-12 * np.abs(r)), (tag, s, r)
    else:
        assert np.all(np.abs(six[m] - ref[m]) <= 1e-13 * np.abs(ref[m])), (tag, six, ref)
    dist = kd[0]
    for c in range(1, C):
        if dist[c][0] is None:
            assert np.isnan(seven[:, c - 1, 6]).all(), (tag, c)
            continue
        pooled = np.hstack(dist[c])
        for i, q in enumerate(qs):
            got, want = seven[i, c - 1, 6], np.percentile(pooled, q)
            ok = got == want if spacing is None else abs(got - want) <= 1e-13 * abs(want)
            assert ok, "%s: class %d, q %g: HD_q %r, reference %r (pooled n %d, |dA| %d)" % (tag, c, q, got, want, len(pooled),
                                                                                          len(dist[c][0]))
            if q == 100.0:
                assert got == max(six[c - 1, 2], six[c - 1, 5]), (tag, c)
    return six, seven, kd


def _ellipsoids(rng, shape, C):
    """C - 1 random ellipsoids (pred: a second draw, with a 1% speckle of labels up to C + 2)"""
    vols = []
    for _ in range(2):
        v = np.zeros(shape, np.uint8)
        for c in range(1, C):
            sk.ellipsoid(v, c, rng.uniform(0.1, 0.9, 3) * shape, rng.uniform(0.1, 0.45, 3) * np.array(shape) + 0.5)
        vols.append(v)
    p, g = vols
    speckle = rng.random(shape) < 0.01
    p[speckle] = rng.integers(0, C + 3, int(speckle.sum()))
    return p, g


def test_case_table_covers_each_pass_on_both_sides_of_48_kb_and_1_2_8_scan_chunks():
    for shape in ALL_SHAPES:
        _describe("case", shape)
    for p in PASSES:
        assert {smem_bytes(s)[p] > SMEM_DEFAULT for s in ALL_SHAPES} == {False, True}, p
    for p, a, b in (("pass2", (6, 5, 764), (5, 6, 765)), ("pass1", (5, 768, 6), (6, 769, 5)), ("pass0", (768, 6, 5), (769, 6, 5))):
        assert smem_bytes(a)[p] <= SMEM_DEFAULT < smem_bytes(b)[p] and a in ALL_SHAPES and b in ALL_SHAPES, p
    assert {1, 2, 8} <= {scan_chunks(s) for s in ALL_SHAPES}
    assert max(max(s) for s in ALL_SHAPES) == 1024 and all(max(s[a] for s in ALL_SHAPES) == 1024 for a in range(3))


@pytest.mark.parametrize("shape,axis", AXIS_CASES)
def test_each_axis_at_and_across_the_shared_memory_limit(shape, axis):
    _describe("axis %d" % axis, shape)
    n = shape[axis]
    p, g = sk.line_features(shape, axis)
    for spacing in (None, ANISO):
        six, _, _ = _check(p, g, 4, spacing, tag="line features")
        s = 1.0 if spacing is None else spacing[axis]
        assert six[0, 2] == six[0, 5] == (n - 1) * s and six[1, 4] == n
    p, g = _ellipsoids(np.random.default_rng(sum(shape)), shape, 8)
    for spacing in (None, ANISO):
        _check(p, g, 8, spacing, tag="C = 8 ellipsoids")


def _chunk_phantom(shape, seed):
    """(pred, gt), C = 6, laid out over the rows i1 of the axis-0 lines (line l = i1 n2 + i2; the chunk of line g = t L + l is
    g // 262144):
      class 1: two large ellipsoids across every row: lines in every chunk;
      class 2: pred in the first rows only, gt in the last rows only: dA in chunk 0 only, dB in the last chunk only;
      class 3: pred and gt both in the last rows: every line in the last chunk of its side;
      class 4: gt only, in the last rows (NaN, its counts set);
      class 5: a 1e-3 speckle in the background of both volumes, classes 2-4 drawn over it;
    and 500 voxels of labels >= C in pred."""
    rng = np.random.default_rng(seed)
    n0, n1, n2 = shape
    pred, gt = np.zeros(shape, np.uint8), np.zeros(shape, np.uint8)
    sk.ellipsoid(gt, 1, (n0 / 2, n1 / 2, n2 / 2), (0.7 * n0, 0.52 * n1, 0.12 * n2))
    sk.ellipsoid(pred, 1, (n0 / 2 + 1, n1 / 2 - 3, n2 / 2 + 2), (0.6 * n0, 0.5 * n1, 0.1 * n2))
    for v in (pred, gt):
        k = int(v.size * 1e-3)
        at = rng.integers(0, v.size, k)
        v.reshape(-1)[at] = np.where(v.reshape(-1)[at] == 0, 5, v.reshape(-1)[at])
    pred.reshape(-1)[rng.integers(0, pred.size, 500)] = rng.integers(6, 256, 500)
    r = (0.5 * n0, 0.04 * n1, 0.1 * n2)
    sk.ellipsoid(pred, 2, (n0 / 2, 0.06 * n1, 0.2 * n2), r)
    sk.ellipsoid(gt, 2, (n0 / 2, 0.94 * n1, 0.8 * n2), r)
    sk.ellipsoid(pred, 3, (n0 / 2, 0.95 * n1, 0.3 * n2), r)
    sk.ellipsoid(gt, 3, (n0 / 2 - 1, 0.93 * n1, 0.35 * n2), r)
    sk.ellipsoid(gt, 4, (n0 / 2, 0.95 * n1, 0.6 * n2), r)
    return pred, gt


@pytest.mark.parametrize("shape", CHUNK_SHAPES)
def test_chunked_scan_of_the_percentile(shape):
    _describe("chunked scan", shape)
    p, g = _chunk_phantom(shape, sum(shape))
    ba, bb = sk.borders(p, 6), sk.borders(g, 6)
    chunks, L = scan_chunks(shape), shape[1] * shape[2]
    last, last_a = chunks - 1, (L - 1) // (SCAN * SCAN_CHUNK)
    for c in range(1, 6):
        print("    class %d: dA lines in chunks %s, dB lines in chunks %s" % (
            c, sorted(line_chunks(ba[c], 0, shape)), sorted(line_chunks(bb[c], 1, shape))))
    assert line_chunks(ba[1], 0, shape) | line_chunks(bb[1], 1, shape) == set(range(chunks))
    assert line_chunks(ba[2], 0, shape) == {0} and line_chunks(bb[2], 1, shape) == {last}
    assert line_chunks(ba[3], 0, shape) == {last_a} and line_chunks(bb[3], 1, shape) == {last}
    assert len(ba[4]) == 0 and line_chunks(bb[4], 1, shape) == {last}
    for spacing in (None, ANISO):
        _, seven, _ = _check(p, g, 6, spacing, tag="chunked scan")
        assert np.isfinite(seven[:, :3, 6]).all() and np.isnan(seven[:, 3, 6]).all()


CODES = np.array([0, 205, 420, 500, 550, 600, 820, 850], np.int16)   # class -> MMWHS label value


def _subject(directory, gt):
    """a preprocess.Subject of the native volume gt (its classes stored as MMWHS label values, the image a function of them)
    whose affine runs stored axis v along world axis (2, 0, 1)[v], in direction (-1, +1, -1)[v], CT_SPACING[v] mm apart: a
    permuted and flipped affine whose row norms are not its column norms"""
    from pnp_b200 import nifti, preprocess
    A = np.zeros((4, 4))
    A[3, 3] = 1.0
    for v, (w, sign) in enumerate(zip((2, 0, 1), (-1.0, 1.0, -1.0))):
        A[w, v] = sign * CT_SPACING[v]
    A[:3, 3] = (90.0, -60.0, 45.0)
    assert tuple(np.sqrt((A[:3, :3] ** 2).sum(1))) != CT_SPACING
    ip, lp = str(directory / "ct_native_image.nii"), str(directory / "ct_native_label.nii")
    nifti.save((gt.astype(np.int16) * 40 - 300), A, ip)
    nifti.save(CODES[gt], A, lp)
    return preprocess.Subject(ip, lp)


def test_native_ct_subject(tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F, native
    _describe("native CT", NATIVE_SHAPE)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    p, g = sk.native_ct_subject(2026, NATIVE_SHAPE, 8)
    print("    phantom %.2f s" % (time.perf_counter() - t0))
    six, _, (_, ba, bb) = _check(p, g, 8, None, tag="native CT")
    assert np.all(six[:, [1, 4]] > 0)
    assert any(1 in line_chunks(bb[c], 1, NATIVE_SHAPE) for c in range(1, 8))   # pooled slots past the first chunk's lines
    six, seven, _ = _check(p, g, 8, CT_SPACING, tag="native CT")
    six2, seven2, _ = _kernel(p, g, 8, CT_SPACING, (95.0, 95.0))
    assert six2.tobytes() == six.tobytes()
    assert seven2[0].tobytes() == seven2[1].tobytes() == seven[QS.index(95.0)].tobytes()
    t0 = time.perf_counter()
    s = _subject(tmp_path, g)
    print("    subject written and loaded %.2f s" % (time.perf_counter() - t0))
    assert s.native_shape == NATIVE_SHAPE and tuple(native.native_spacing(s)) == CT_SPACING
    got = native.surface_mm(s, p, g, 8, hd_percentile=95)
    want = F.surface_from_raw(seven[QS.index(95.0)])
    want["hd_percentile"] = 95.0
    assert sorted(got) == sorted(want)
    for k in want:
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), k
    print("    peak device memory %.2f GB" % (torch.cuda.max_memory_allocated() / 1e9))
