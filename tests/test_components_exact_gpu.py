"""pnp_largest_components against oracle/components_exact.scipy_lcc, bit for bit: the output volume, stats and cm (np.bincount), at
6- and 26-connectivity, on random labels (labels up to C + 1), shapes with partial CTAs and grid-stride sweeps, degenerate shapes,
checkerboards, a serpentine component next to one a voxel smaller, equal-size ties, a volume of one class and a native-size
volume of >= 2^26 voxels; in place, repeated calls, and rejected arguments leaving every output untouched."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import components_exact as ce
from tests import cabi

pytestmark = pytest.mark.gpu
CONNS = (6, 26)


def _check(lab, C, conn, gt=None, tag=""):
    from pnp_b200 import functional as F
    dl = torch.from_numpy(np.ascontiguousarray(lab)).cuda()
    dg = None if gt is None else torch.from_numpy(np.ascontiguousarray(gt)).cuda()
    out, st, cm = F.largest_components(dl, C, conn, gt=dg)
    want, wst, wcm = ce.scipy_lcc(lab, C, conn, gt)
    got = out.cpu().numpy()
    assert np.array_equal(got, want), "%s conn %d: %d voxels differ" % (tag, conn, int((got != want).sum()))
    for i, k in enumerate(("components", "kept", "removed")):
        assert st[k].dtype == np.int64 and np.array_equal(st[k], wst[:, i]), (tag, conn, k, st[k], wst[:, i])
    if gt is None:
        assert cm is None
    else:
        assert cm.dtype == np.int64 and np.array_equal(cm, wcm), (tag, conn)
    return got, wst


@pytest.mark.parametrize("conn", CONNS)
def test_random_labels_at_several_densities(conn):
    cabi.lib()
    rng = np.random.RandomState(11)
    for C in (2, 5, 8):
        for density in (0.05, 0.31, 0.6, 0.95):
            shape = (23, 31, 37)
            fg = rng.rand(*shape) < density
            lab = np.where(fg, rng.randint(1, C + 2, size=shape), 0).astype(np.uint8)
            gt = rng.randint(0, C + 2, size=shape).astype(np.uint8)
            _, st = _check(lab, C, conn, gt, "C %d density %.2f" % (C, density))
    # binary site percolation near the 6-connected threshold: the largest, most tangled components
    lab = (rng.rand(64, 64, 64) < 0.31).astype(np.uint8)
    _check(lab, 2, conn, lab, "percolation")


@pytest.mark.parametrize("conn", CONNS)
def test_partial_blocks_and_degenerate_shapes(conn):
    cabi.lib()
    rng = np.random.RandomState(5)
    for shape in [(1, 1, 1), (1, 1, 300), (300, 1, 1), (1, 300, 1), (1, 17, 19), (19, 1, 17), (17, 19, 1), (2, 2, 2), (3, 257, 5),
                  (33, 7, 129), (1, 1023, 1025)]:
        for C in (2, 5):
            lab = np.where(rng.rand(*shape) < 0.5, rng.randint(1, C + 2, size=shape), 0).astype(np.uint8)
            _check(lab, C, conn, lab[::-1].copy(), "shape %s C %d" % (shape, C))
    # more voxels than one sweep of the capped grid covers (132 * 64 CTAs of 1024 voxels): several grid-stride iterations
    lab = np.where(rng.rand(97, 211, 509) < 0.4, rng.randint(1, 6, size=(97, 211, 509)), 0).astype(np.uint8)
    _check(lab, 5, conn, None, "grid-stride")


def test_checkerboard():
    cabi.lib()
    i, j, k = np.indices((9, 10, 11))
    lab = (1 + (i + j + k) % 2).astype(np.uint8)          # classes 1 and 2 interleaved
    out6, st6 = _check(lab, 3, 6, None, "checkerboard")
    n1, n2 = int((lab == 1).sum()), int((lab == 2).sum())
    assert st6[1].tolist() == [n1, 1, n1 - 1] and st6[2].tolist() == [n2, 1, n2 - 1]
    assert out6[0, 0, 0] == 1 and out6[0, 0, 1] == 2 and int((out6 > 0).sum()) == 2      # the first voxel of each class
    out26, st26 = _check(lab, 3, 26, None, "checkerboard")
    assert st26[1].tolist() == [1, n1, 0] and st26[2].tolist() == [1, n2, 0] and np.array_equal(out26, lab)


def _serpentine(n0, n1, n2, h):
    """class 1: a snake in columns >= h + 1 of every even plane (even rows full, odd rows one connector voxel at alternating ends),
    the even planes joined by one voxel in the odd planes between them; and in columns < h, a raster-order prefix of that box
    one voxel smaller than the snake (its first voxel comes first)"""
    lab = np.zeros((n0, n1, n2), np.uint8)
    for i in range(0, n0, 2):
        for j in range(n1):
            if j % 2 == 0:
                lab[i, j, h + 1:] = 1
            else:
                lab[i, j, n2 - 1 if (j // 2) % 2 == 0 else h + 1] = 1
        if i + 1 < n0 - 1:
            lab[i + 1, 0, h + 1] = 1
    size = int(lab.sum())
    box = np.zeros((n0, n1, h), np.uint8).reshape(-1)
    assert size - 1 <= box.size
    box[:size - 1] = 1
    lab[:, :, :h] = box.reshape(n0, n1, h)
    return lab, size


@pytest.mark.parametrize("conn", CONNS)
def test_serpentine_beats_a_component_one_voxel_smaller(conn):
    cabi.lib()
    lab, size = _serpentine(9, 301, 260, 100)
    out, st = _check(lab, 2, conn, None, "serpentine")
    assert st[1].tolist() == [2, size, size - 1]
    assert not out[:, :, :100].any() and np.array_equal(out[:, :, 101:], lab[:, :, 101:])
    # the snake one voxel shorter (the free end of its last row): now the box (first in C order) wins the tie
    lab[8, 300, 259] = 0
    _, st = _check(lab, 2, conn, None, "serpentine tie")
    assert st[1].tolist() == [2, size - 1, size - 1]


@pytest.mark.parametrize("conn", CONNS)
def test_equal_sizes_keep_the_component_with_the_smallest_first_index(conn):
    cabi.lib()
    n0, n1, n2 = 40, 6, 50
    # A: a bar down axis 0 in the last column (first voxel at index 49, but it reaches the end of the volume); B: a row of the
    # same length in the last plane starting at column 0 (first voxel near the end): A is kept
    lab = np.zeros((n0, n1, n2), np.uint8)
    lab[:, 0, n2 - 1] = 3
    lab[n0 - 1, n1 - 1, :n0] = 3
    out, st = _check(lab, 5, conn, None, "bar and row")
    assert st[3].tolist() == [2, n0, n0] and out[:, 0, n2 - 1].all() and not out[n0 - 1, n1 - 1, :n0].any()
    # many equal 2-voxel pieces of several classes in a scrambled order
    rng = np.random.RandomState(3)
    lab = np.zeros((20, 20, 20), np.uint8)
    cells = rng.permutation(np.array([(a, b, c) for a in range(0, 20, 3) for b in range(0, 20, 3) for c in range(0, 19, 3)]))
    for t, (a, b, c) in enumerate(cells):
        lab[a, b, c:c + 2] = 1 + t % 4
    _check(lab, 5, conn, lab, "pieces")


@pytest.mark.parametrize("conn", CONNS)
def test_one_class_everywhere_and_nothing_at_all(conn):
    cabi.lib()
    lab = np.full((30, 40, 50), 4, np.uint8)
    out, st = _check(lab, 5, conn, lab, "all class 4")
    assert np.array_equal(out, lab) and st[4].tolist() == [1, lab.size, 0] and not st[:4].any()
    lab = np.zeros((30, 40, 50), np.uint8)
    _, st = _check(lab, 8, conn, lab, "empty")
    assert not st.any()
    lab = np.full((30, 40, 50), 200, np.uint8)
    out, st = _check(lab, 8, conn, lab, "out of range")
    assert not out.any() and st[0].tolist() == [0, 0, lab.size]


def _phantom(shape, seed):
    """four ellipsoid organs in a native-size volume, with salt-and-pepper islands of every class"""
    rng = np.random.RandomState(seed)
    n0, n1, n2 = shape
    i, j, k = np.ogrid[:n0, :n1, :n2]
    lab = np.zeros(shape, np.uint8)
    for c, (ci, cj, ck, r) in enumerate([(0.5, 0.45, 0.5, 0.18), (0.45, 0.6, 0.4, 0.12), (0.6, 0.4, 0.6, 0.14),
                                         (0.35, 0.5, 0.65, 0.08)], 1):
        lab[((i - ci * n0) / (r * n0)) ** 2 + ((j - cj * n1) / (r * n1)) ** 2 + ((k - ck * n2) / (r * n2)) ** 2 <= 1] = c
    salt = rng.rand(*shape) < 0.002
    lab[salt] = rng.randint(1, 7, size=int(salt.sum()))
    return lab


@pytest.mark.parametrize("conn", CONNS)
def test_native_size_volume(conn):
    cabi.lib()
    shape = (260, 512, 512)                          # 68.2 M voxels >= 2^26
    assert np.prod(shape) >= 1 << 26
    lab = _phantom(shape, 17)
    gt = _phantom(shape, 18)
    _, st = _check(lab, 5, conn, gt, "native size")
    assert st[1:, 0].min() > 1 and st[0, 2] > 0


def test_in_place_and_repeated_calls_are_bit_identical():
    cabi.lib()
    from pnp_b200 import functional as F
    rng = np.random.RandomState(9)
    lab = np.where(rng.rand(45, 67, 89) < 0.45, rng.randint(1, 7, size=(45, 67, 89)), 0).astype(np.uint8)
    gt = rng.randint(0, 7, size=lab.shape).astype(np.uint8)
    dg = torch.from_numpy(gt).cuda()
    for conn in CONNS:
        want, wst, wcm = ce.scipy_lcc(lab, 5, conn, gt)
        runs = []
        for _ in range(3):
            dl = torch.from_numpy(lab).cuda()
            out, st, cm = F.largest_components(dl, 5, conn, gt=dg)
            runs.append((out.cpu().numpy(), np.stack([st[k] for k in F.COMPONENT_STATS], 1), cm))
        for o, s, c in runs:
            assert np.array_equal(o, want) and np.array_equal(s, wst) and np.array_equal(c, wcm)
        dl = torch.from_numpy(lab).cuda()
        out, st, cm = F.largest_components(dl, 5, conn, gt=dg, out=dl)
        assert out.data_ptr() == dl.data_ptr()
        assert np.array_equal(dl.cpu().numpy(), want) and np.array_equal(cm, wcm)
        assert np.array_equal(np.stack([st[k] for k in F.COMPONENT_STATS], 1), wst)


def test_rejected_arguments_leave_every_output_untouched():
    _C, rt = cabi.lib()
    lib = _C.lib
    shape = (6, 7, 8)
    C = 5
    lab = torch.randint(0, 7, shape, dtype=torch.uint8, device="cuda")
    gt = torch.randint(0, 7, shape, dtype=torch.uint8, device="cuda")
    nb = ctypes.c_longlong(0)
    assert lib.pnp_largest_components_workspace(*shape, C, 6, ctypes.byref(nb)) == 0
    ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    out = torch.full(shape, 0xAB, dtype=torch.uint8, device="cuda")
    stats = torch.full((8, 3), 0x7FC0BEEF, dtype=torch.int64, device="cuda")
    cm = torch.full((8, 8), 0x7FC0BEEF, dtype=torch.int64, device="cuda")
    bufs = {"out": out, "stats": stats, "cm": cm, "labels": lab}
    before = cabi.snapshot(bufs)
    p = cabi.ptr
    good = [p(lab), *shape, C, 6, p(out), p(gt), p(cm), p(stats), p(ws), nb.value]
    cases = [("labels NULL", 0, None, cabi.BAD_ARG), ("out NULL", 6, None, cabi.BAD_ARG), ("gt only", 8, None, cabi.BAD_ARG),
             ("cm only", 7, None, cabi.BAD_ARG), ("stats NULL", 9, None, cabi.BAD_ARG), ("ws NULL", 10, None, cabi.BAD_ARG),
             ("ws short", 11, nb.value - 1, cabi.BAD_ARG), ("n0 0", 1, 0, cabi.BAD_ARG), ("n2 -1", 3, -1, cabi.BAD_ARG),
             ("C 1", 4, 1, cabi.UNSUPPORTED), ("C 9", 4, 9, cabi.UNSUPPORTED), ("conn 18", 5, 18, cabi.UNSUPPORTED),
             ("conn 8", 5, 8, cabi.UNSUPPORTED), ("2^31 voxels", 1, (1 << 31) // (7 * 8) + 1, cabi.UNSUPPORTED)]
    for tag, at, value, rc in cases:
        args = list(good)
        args[at] = value
        assert lib.pnp_largest_components(*args, rt.stream()) == rc, tag
        cabi.assert_untouched(tag, "pnp_largest_components", bufs, before)
    # the good call then writes them
    assert lib.pnp_largest_components(*good, rt.stream()) == 0
    cabi.sync()
    want, wst, wcm = ce.scipy_lcc(lab.cpu().numpy(), C, 6, gt.cpu().numpy())
    assert np.array_equal(out.cpu().numpy(), want)
    assert np.array_equal(stats[:C].cpu().numpy(), wst) and np.array_equal(cm.view(-1)[:C * C].view(C, C).cpu().numpy(), wcm)
    assert (stats[C:] == 0x7FC0BEEF).all() and (cm.view(-1)[C * C:] == 0x7FC0BEEF).all()
