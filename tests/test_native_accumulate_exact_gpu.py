"""The localisation kernels at the C-ABI (csrc/resample.cu, csrc/components3d.cu):
* pnp_native_accumulate + pnp_native_accumulated_labels bit for bit against oracle/accumulate_exact.py (sums, coverage, labels,
  counts), and against pnp_native_labels_ensemble (K <= 16) and pnp_native_labels (K = 1): K = 1, 2, 3, 16, 40 at C = 2, 5, 8;
  disjoint, partial and full coverage; NaN maps; edge coordinates; a partial CTA; a grid-stride sweep past the cap; a sums buffer
  of m0 m1 m2 C >= 2^31 floats;
* pnp_label_boxes against numpy: empty classes, a single voxel, a full volume, labels >= C, 260 x 512 x 512;
* rejected arguments leave the outputs untouched."""
import numpy as np
import pytest
import torch

from oracle import accumulate_exact as A
from oracle import ensemble_exact as E
from oracle import native_exact as N
from tests.cabi import BAD_ARG, UNSUPPORTED, assert_untouched, lib, snapshot, sync

pytestmark = pytest.mark.gpu
OUT_SENTINEL = 0xAB
CM_SENTINEL = -0x5EED

CASES = [
    ("acc_k1_random_c5", 1, (12, 9, 10), 5, (13, 8, 11), "random", "random"),
    ("acc_k2_full_c2", 2, (9, 13, 7), 2, (11, 10, 12), "random", "full"),
    ("acc_k3_disjoint_c5", 3, (8, 9, 10), 5, (15, 11, 12), "random", "disjoint"),
    ("acc_k3_partial_c8", 3, (7, 11, 9), 8, (10, 12, 9), "random", "random"),
    ("acc_k3_nan_c8", 3, (6, 7, 8), 8, (9, 8, 7), "random", ["full", "nan", "random"]),
    ("acc_k2_edges_c5", 2, (6, 7, 5), 5, (7, 8, 11), "random", "edges"),
    ("acc_k16_near_ties_c2", 16, (6, 7, 8), 2, (14, 13, 12), "near_ties", "full"),
    ("acc_k16_mixed_c5", 16, (7, 8, 6), 5, (12, 11, 10), "random", ["full", "random", "negative", "disjoint"] * 4),
    ("acc_k16_partial_cta_c8", 16, (5, 6, 7), 8, (5, 7, 9), "random", "random"),
    ("acc_k40_mixed_c5", 40, (6, 7, 5), 5, (11, 10, 9), "near_ties", ["full", "random", "negative", "nan", "edges"] * 8),
    ("acc_k2_cap_c2", 2, (40, 64, 64), 2, (220, 205, 200), "random", "full"),
]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _p(t):
    return None if t is None else t.data_ptr()


def _accumulate(_C, rt, scores, maps, n, C, m):
    sums = torch.zeros(tuple(m) + (C,), dtype=torch.float32, device="cuda")
    covered = torch.zeros(tuple(m), dtype=torch.uint8, device="cuda")
    for k in range(scores.shape[0]):
        assert _C.lib.pnp_native_accumulate(_p(scores[k]), *n, C, _p(maps[k]), *m, _p(sums), _p(covered), rt.stream()) == 0
    return sums, covered


def _labels(_C, rt, sums, covered, m, C, gt):
    out = torch.full(tuple(m), OUT_SENTINEL, dtype=torch.uint8, device="cuda")
    cm = torch.full((C, C), CM_SENTINEL, dtype=torch.int64, device="cuda")
    assert _C.lib.pnp_native_accumulated_labels(_p(sums), _p(covered), *m, C, _p(out), _p(gt), _p(cm), rt.stream()) == 0
    return out, cm


def test_case_table_reaches_every_launch_regime():
    launches = [N.launch(*c[4]) for c in CASES]
    assert any(l.capped and l.iters >= 2 for l in launches) and any(l.single_partial for l in launches)
    assert {c[1] for c in CASES} >= {1, 2, 3, 16, 40} and {c[3] for c in CASES} >= {2, 5, 8}


@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_accumulate_bit_exact(case):
    _C, rt = lib()
    tag, K, n, C, m, sk, mk = case
    scores, maps, gt = E.operands(tag, K, n, C, m, sk, mk)
    ds, dm, dg = _dev(scores), _dev(maps), _dev(gt)
    sums, covered = _accumulate(_C, rt, ds, dm, n, C, m)
    out, cm = _labels(_C, rt, sums, covered, m, C, dg)
    sync()
    want_sums, want_cov = A.accumulate_ref(scores, maps, m)
    assert np.array_equal(covered.cpu().numpy(), want_cov), tag + " coverage"
    assert np.array_equal(sums.cpu().numpy().view(np.uint32), want_sums.view(np.uint32)), tag + " sums"
    want = A.labels_ref(want_sums, want_cov)
    assert np.array_equal(out.cpu().numpy(), want), tag + " labels"
    assert np.array_equal(cm.cpu().numpy(), N.confusion_ref(want, gt, C)), tag + " counts"
    if K <= 16:
        ens = torch.empty(tuple(m), dtype=torch.uint8, device="cuda")
        ecm = torch.empty((C, C), dtype=torch.int64, device="cuda")
        assert _C.lib.pnp_native_labels_ensemble(_p(ds), K, *n, C, _p(dm), *m, _p(ens), _p(dg), _p(ecm), rt.stream()) == 0
        sync()
        assert torch.equal(ens, out) and torch.equal(ecm, cm), tag + " vs pnp_native_labels_ensemble"
    if K == 1:
        one = torch.empty(tuple(m), dtype=torch.uint8, device="cuda")
        ocm = torch.empty((C, C), dtype=torch.int64, device="cuda")
        assert _C.lib.pnp_native_labels(_p(ds), *n, C, _p(dm), *m, _p(one), _p(dg), _p(ocm), rt.stream()) == 0
        sync()
        assert torch.equal(one, out) and torch.equal(ocm, cm), tag + " vs pnp_native_labels"
    # without gt only the labels are written; a repeated sequence is bit-identical
    out2 = torch.full(tuple(m), OUT_SENTINEL, dtype=torch.uint8, device="cuda")
    assert _C.lib.pnp_native_accumulated_labels(_p(sums), _p(covered), *m, C, _p(out2), None, None, rt.stream()) == 0
    sums2, covered2 = _accumulate(_C, rt, ds, dm, n, C, m)
    sync()
    assert torch.equal(out2, out) and torch.equal(sums2.view(torch.int32), sums.view(torch.int32)) and torch.equal(covered2, covered)


def test_functional_accumulator_equals_the_ensemble_wrapper():
    _C, rt = lib()
    from pnp_b200 import functional as F
    tag, K, n, C, m, sk, mk = CASES[7]
    scores, maps, gt = E.operands(tag, K, n, C, m, sk, mk)
    acc = F.NativeAccumulator(m, C)
    for k in range(K):
        acc.add(_dev(scores[k]), _dev(maps[k]))
    labels, cm = acc.labels(_dev(gt))
    want, wcm = F.native_labels(_dev(scores), _dev(maps), m, _dev(gt))
    assert acc.count == K and torch.equal(labels, want) and torch.equal(cm, wcm)
    with pytest.raises(ValueError):
        acc.add(_dev(scores[0][..., :2]), _dev(maps[0]))


def test_sums_beyond_2_31_floats():
    """m = 1024 x 1024 x 1025 voxels at C = 2: 2^31 + 2 M floats of sums.  The scores vary along the score grid's axis 0 only and
    the maps read axis 0 from native axis 0 alone, so every native plane i holds one label and one sum pair: the oracle runs on
    an m0 x 1 x 1 line and is broadcast"""
    _C, rt = lib()
    C, m, n = 2, (1024, 1024, 1025), (64, 2, 2)
    assert m[0] * m[1] * m[2] * C >= 2 ** 31 and m[0] * m[1] * m[2] < 2 ** 31
    rng = np.random.RandomState(231)
    K = 3
    line = rng.standard_normal((K, n[0], 1, 1, C)).astype(np.float32)
    scores = np.ascontiguousarray(np.repeat(np.repeat(line, 2, 2), 2, 3))
    maps = np.zeros((K, 3, 4), np.float32)
    for k in range(K):
        maps[k, 0, 0] = np.float32(rng.uniform(0.04, 0.06))
        maps[k, 0, 3] = np.float32(rng.uniform(-0.5, 20.0))
    maps = maps.reshape(K, 12)
    sums, covered = _accumulate(_C, rt, _dev(scores), _dev(maps), n, C, m)
    out, cm = _labels(_C, rt, sums, covered, m, C, torch.zeros(m, dtype=torch.uint8, device="cuda"))
    sync()
    ws, wc = A.accumulate_ref(scores, maps, (m[0], 1, 1))
    want = A.labels_ref(ws, wc)[:, 0, 0]
    got = out.cpu().numpy()
    assert np.array_equal(got, np.broadcast_to(want[:, None, None], m))
    tail = sums[-1, -1].cpu().numpy()                                # the last row: beyond 2^31 floats
    assert np.array_equal(tail.view(np.uint32), np.broadcast_to(ws[-1, 0], tail.shape).view(np.uint32))
    assert int(cm.sum()) == m[0] * m[1] * m[2]
    del sums, covered, out
    torch.cuda.empty_cache()


def _box_cases():
    rng = np.random.RandomState(5)
    full = np.full((7, 9, 11), 3, np.uint8)
    single = np.zeros((6, 5, 4), np.uint8)
    single[4, 0, 3] = 2
    over = rng.randint(0, 12, (13, 17, 19)).astype(np.uint8)
    big = np.zeros((260, 512, 512), np.uint8)
    big[40:200, 100:460, 7:300] = rng.randint(0, 5, (160, 360, 293)).astype(np.uint8)
    big[259, 511, 511] = 4
    return [("full", full, 5), ("single_voxel", single, 8), ("labels_over_C", over, 6), ("empty_classes", single, 4),
            ("ct_size", big, 5), ("c2", over, 2)]


@pytest.mark.parametrize("case", _box_cases(), ids=lambda c: c[0])
def test_label_boxes_equal_numpy(case):
    _C, rt = lib()
    tag, lab, C = case
    out = torch.full((C, 7), CM_SENTINEL, dtype=torch.int64, device="cuda")
    assert _C.lib.pnp_label_boxes(_p(_dev(lab)), *lab.shape, C, _p(out), rt.stream()) == 0
    sync()
    assert np.array_equal(out.cpu().numpy(), A.boxes_ref(lab, C)), tag


def test_rejected_arguments_leave_the_outputs_untouched():
    _C, rt = lib()
    n, C, m = (4, 5, 6), 3, (3, 4, 5)
    scores = torch.randn(n + (C,), device="cuda")
    vmap = torch.randn(12, device="cuda")
    sums = torch.full(m + (C,), 7.0, device="cuda")
    covered = torch.full(m, 3, dtype=torch.uint8, device="cuda")
    out = torch.full(m, OUT_SENTINEL, dtype=torch.uint8, device="cuda")
    cm = torch.full((C, C), CM_SENTINEL, dtype=torch.int64, device="cuda")
    gt = torch.zeros(m, dtype=torch.uint8, device="cuda")
    boxes = torch.full((C, 7), CM_SENTINEL, dtype=torch.int64, device="cuda")
    bufs = {"sums": sums, "covered": covered, "out": out, "cm": cm, "boxes": boxes}
    before = snapshot(bufs)
    big = (1 << 23) + 1
    acc = lambda sc, nn, c, mp, mm, s, cv: _C.lib.pnp_native_accumulate(_p(sc), *nn, c, _p(mp), *mm, _p(s), _p(cv), rt.stream())
    lab = lambda s, cv, mm, c, o, g, k: _C.lib.pnp_native_accumulated_labels(_p(s), _p(cv), *mm, c, _p(o), _p(g), _p(k), rt.stream())
    box = lambda l, nn, c, o: _C.lib.pnp_label_boxes(_p(l), *nn, c, _p(o), rt.stream())
    bad = [
        ("accumulate: NULL sums", BAD_ARG, acc, (scores, n, C, vmap, m, None, covered)),
        ("accumulate: NULL covered", BAD_ARG, acc, (scores, n, C, vmap, m, sums, None)),
        ("accumulate: NULL scores", BAD_ARG, acc, (None, n, C, vmap, m, sums, covered)),
        ("accumulate: NULL map", BAD_ARG, acc, (scores, n, C, None, m, sums, covered)),
        ("accumulate: n1 = 0", BAD_ARG, acc, (scores, (4, 0, 6), C, vmap, m, sums, covered)),
        ("accumulate: m2 < 0", BAD_ARG, acc, (scores, n, C, vmap, (3, 4, -5), sums, covered)),
        ("accumulate: C = 1", UNSUPPORTED, acc, (scores, n, 1, vmap, m, sums, covered)),
        ("accumulate: C = 9", UNSUPPORTED, acc, (scores, n, 9, vmap, m, sums, covered)),
        ("accumulate: n0 above PNP_RS_MAX_DIM", UNSUPPORTED, acc, (scores, (big, 1, 1), C, vmap, m, sums, covered)),
        ("accumulate: m0 m1 m2 = 2^31", UNSUPPORTED, acc, (scores, n, C, vmap, (1 << 11, 1 << 10, 1 << 10), sums, covered)),
        ("labels: NULL sums", BAD_ARG, lab, (None, covered, m, C, out, gt, cm)),
        ("labels: NULL covered", BAD_ARG, lab, (sums, None, m, C, out, gt, cm)),
        ("labels: NULL out", BAD_ARG, lab, (sums, covered, m, C, None, gt, cm)),
        ("labels: gt without cm", BAD_ARG, lab, (sums, covered, m, C, out, gt, None)),
        ("labels: cm without gt", BAD_ARG, lab, (sums, covered, m, C, out, None, cm)),
        ("labels: m1 = 0", BAD_ARG, lab, (sums, covered, (3, 0, 5), C, out, gt, cm)),
        ("labels: C = 9", UNSUPPORTED, lab, (sums, covered, m, 9, out, gt, cm)),
        ("labels: m2 above PNP_RS_MAX_DIM", UNSUPPORTED, lab, (sums, covered, (1, 1, big), C, out, gt, cm)),
        ("labels: m0 m1 m2 = 2^31", UNSUPPORTED, lab, (sums, covered, (1 << 11, 1 << 10, 1 << 10), C, out, gt, cm)),
        ("boxes: NULL labels", BAD_ARG, box, (None, m, C, boxes)),
        ("boxes: NULL out", BAD_ARG, box, (gt, m, C, None)),
        ("boxes: n0 = 0", BAD_ARG, box, (gt, (0, 4, 5), C, boxes)),
        ("boxes: C = 1", UNSUPPORTED, box, (gt, m, 1, boxes)),
        ("boxes: C = 9", UNSUPPORTED, box, (gt, m, 9, boxes)),
        ("boxes: n0 n1 n2 = 2^31", UNSUPPORTED, box, (gt, (1 << 11, 1 << 10, 1 << 10), C, boxes)),
    ]
    for what, rc_want, fn, args in bad:
        rc = fn(*args)
        assert rc == rc_want, (what, rc)
        assert_untouched(what, "localisation kernels", bufs, before)
