"""pnp_native_labels_ensemble (csrc/resample.cu) bit for bit against its numpy restatement oracle/ensemble_exact.py, at the C-ABI:
K = 1, 2, 3 and 16 members at C = 2, 5 and 8; disjoint, partial and full coverage; near-tie sums that turn on the last bit of an
addition; a member with a NaN map; edge coordinates; a single partial CTA and a grid-stride sweep past the cap; member offsets
beyond 2^31 floats in total.  At K = 1 labels and counts equal pnp_native_labels'; the counts equal np.bincount; repeated calls
are bit-identical; every rejected argument leaves its sentinel-filled outputs untouched; the functional wrapper equals the
C-ABI."""
import numpy as np
import pytest
import torch

from oracle import ensemble_exact as E
from oracle import native_exact as N
from tests.cabi import BAD_ARG, UNSUPPORTED, assert_untouched, lib, snapshot, sync

pytestmark = pytest.mark.gpu
OUT_SENTINEL = 0xAB
CM_SENTINEL = -0x5EED

# (tag, K, score grid n, C, native grid m, score kind, map kind(s))
CASES = [
    ("k1_random_c5", 1, (12, 9, 10), 5, (13, 8, 11), "random", "random"),
    ("k1_permuted_c8", 1, (10, 12, 8), 8, (14, 9, 12), "random", "permuted"),
    ("k2_full_c2", 2, (9, 13, 7), 2, (11, 10, 12), "random", "full"),
    ("k2_partial_c8", 2, (7, 11, 9), 8, (10, 12, 9), "random", "random"),
    ("k3_disjoint_c5", 3, (8, 9, 10), 5, (15, 11, 12), "random", "disjoint"),
    ("k3_mixed_c5", 3, (8, 9, 10), 5, (10, 11, 12), "random", ["full", "random", "negative"]),
    ("k3_near_ties_c2", 3, (10, 12, 9), 2, (30, 28, 26), "near_ties", "full"),
    ("k3_nan_member_c8", 3, (6, 7, 8), 8, (9, 8, 7), "random", ["full", "nan", "random"]),
    ("k2_edges_c5", 2, (6, 7, 5), 5, (7, 8, 11), "random", "edges"),
    ("k2_ties_c5", 2, (8, 9, 10), 5, (12, 13, 11), "ties", "full"),
    ("k16_near_ties_c2", 16, (6, 7, 8), 2, (14, 13, 12), "near_ties", "full"),
    ("k16_mixed_c5", 16, (7, 8, 6), 5, (12, 11, 10), "random", ["full", "random", "negative", "disjoint"] * 4),
    ("k16_partial_cta_c8", 16, (5, 6, 7), 8, (5, 7, 9), "random", "random"),
    ("k2_cap_c2", 2, (40, 64, 64), 2, (220, 205, 200), "random", "full"),
]


def _call(_C, rt, scores, K, n, C, maps, m, out, gt, cm):
    p = lambda t: None if t is None else t.data_ptr()
    return _C.lib.pnp_native_labels_ensemble(p(scores), K, *n, C, p(maps), *m, p(out), p(gt), p(cm), rt.stream())


def _buffers(C, m):
    out = torch.full(tuple(m), OUT_SENTINEL, dtype=torch.uint8, device="cuda")
    cm = torch.full((C, C), CM_SENTINEL, dtype=torch.int64, device="cuda")
    return out, cm


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def test_case_table_reaches_every_launch_regime():
    launches = [N.launch(*c[4]) for c in CASES]
    assert any(l.capped and l.iters >= 2 for l in launches) and any(l.single_partial for l in launches)
    assert {c[1] for c in CASES} >= {1, 2, 3, 16} and {c[3] for c in CASES} >= {2, 5, 8}


@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_pnp_native_labels_ensemble_bit_exact(case):
    _C, rt = lib()
    tag, K, n, C, m, sk, mk = case
    scores, maps, gt = E.operands(tag, K, n, C, m, sk, mk)
    ds, dm, dg = _dev(scores), _dev(maps), _dev(gt)
    out, cm = _buffers(C, m)
    assert _call(_C, rt, ds, K, n, C, dm, m, out, dg, cm) == 0
    sync()
    want = E.ensemble_ref(scores, maps, m)
    got = out.cpu().numpy()
    bad = np.argwhere(got != want)
    assert bad.size == 0, "%s: %d of %d labels differ; first at %s: got %d, ref %d" % (
        tag, len(bad), got.size, tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])])
    assert np.array_equal(cm.cpu().numpy(), N.confusion_ref(want, gt, C)), tag + " confusion counts"
    assert int(cm.sum()) == int(np.prod(m))
    cover = sum(N.inside(N.coords(maps[k], m), n).astype(np.int64) for k in range(K))
    print("  %s: %d native voxels, covered by 0 / 1 / >1 members: %d / %d / %d, classes %s" % (
        tag, got.size, int((cover == 0).sum()), int((cover == 1).sum()), int((cover > 1).sum()),
        np.bincount(got.reshape(-1), minlength=C).tolist()))
    # repeated calls are bit-identical; without gt only the labels are written
    first_out, first_cm = out.clone(), cm.clone()
    assert _call(_C, rt, ds, K, n, C, dm, m, out, dg, cm) == 0
    sync()
    assert torch.equal(first_out, out) and torch.equal(first_cm, cm)
    out2, cm2 = _buffers(C, m)
    assert _call(_C, rt, ds, K, n, C, dm, m, out2, None, None) == 0
    sync()
    assert torch.equal(out2, out) and bool((cm2 == CM_SENTINEL).all())
    if K == 1:      # the single-member call is pnp_native_labels, bit for bit
        out1, cm1 = _buffers(C, m)
        assert _C.lib.pnp_native_labels(ds.data_ptr(), *n, C, dm.data_ptr(), *m, out1.data_ptr(), dg.data_ptr(), cm1.data_ptr(),
                                        rt.stream()) == 0
        sync()
        assert torch.equal(out1, out) and torch.equal(cm1, cm)


def test_member_offsets_beyond_2_31_floats():
    """16 members of 64 x 1024 x 1200 x 2 fp32 (157 M floats, 629 MB each): member 15 starts at 2.36 G floats.  The scores
    vary along axis 0 only, and the maps keep axes 1 and 2 inside [0, 1], so a 64 x 2 x 2 copy of every member gives the oracle
    the same trilinear values (a lerp between equal values is exact)"""
    _C, rt = lib()
    K, C, big, m = 16, 2, (64, 1024, 1200), (70, 3, 3)
    assert (K - 1) * big[0] * big[1] * big[2] * C > 2 ** 31
    rng = np.random.RandomState(231)
    line = rng.standard_normal((K, big[0], 1, 1, C)).astype(np.float32)
    line[..., 1] = line[..., 0] + line[..., 0] * np.float32(2.0 ** -22) * rng.randint(-2, 3, (K, big[0], 1, 1)).astype(np.float32)
    small = np.repeat(np.repeat(line, 2, 2), 2, 3)
    maps = np.zeros((K, 3, 4), np.float32)
    for k in range(K):
        maps[k, 0, 0] = np.float32(rng.uniform(0.8, 0.95))
        maps[k, 0, 3] = np.float32(rng.uniform(-0.5, 2.0))
        maps[k, 1, 1] = maps[k, 2, 2] = np.float32(0.5)
    maps = maps.reshape(K, 12)
    gt = rng.randint(0, C, m).astype(np.uint8)
    scores = torch.empty((K,) + big + (C,), dtype=torch.float32, device="cuda")
    for k in range(K):
        scores[k].copy_(_dev(line[k]).expand(big[0], big[1], big[2], C))
    out, cm = _buffers(C, m)
    assert _call(_C, rt, scores, K, big, C, _dev(maps), m, out, _dev(gt), cm) == 0
    sync()
    want = E.ensemble_ref(small, maps, m)
    assert np.array_equal(out.cpu().numpy(), want)
    assert np.array_equal(cm.cpu().numpy(), N.confusion_ref(want, gt, C))
    # the last member alone is sampled from beyond 2^31 floats: its labels equal its own small copy's
    last, _ = _buffers(C, m)
    assert _call(_C, rt, scores[K - 1:], 1, big, C, _dev(maps[K - 1:]), m, last, None, None) == 0
    sync()
    assert np.array_equal(last.cpu().numpy(), N.labels_ref(small[K - 1], maps[K - 1], m))
    del scores
    torch.cuda.empty_cache()


def test_functional_wrapper_equals_the_c_abi():
    _C, rt = lib()
    from pnp_b200 import functional as F
    tag, K, n, C, m, sk, mk = CASES[5]
    scores, maps, gt = E.operands(tag, K, n, C, m, sk, mk)
    labels, cm = F.native_labels(_dev(scores), _dev(maps), m, _dev(gt))
    want = E.ensemble_ref(scores, maps, m)
    assert labels.dtype == torch.uint8 and tuple(labels.shape) == m
    assert np.array_equal(labels.cpu().numpy(), want) and np.array_equal(cm.cpu().numpy(), N.confusion_ref(want, gt, C))
    alone, none = F.native_labels(_dev(scores), _dev(maps), m)
    assert none is None and torch.equal(alone, labels)
    one, cm1 = F.native_labels(_dev(scores[:1]), _dev(maps[:1]), m, _dev(gt))
    four, cm4 = F.native_labels(_dev(scores[0]), _dev(maps[0]), m, _dev(gt))
    assert torch.equal(one, four) and torch.equal(cm1, cm4)
    with pytest.raises(ValueError):
        F.native_labels(_dev(scores), _dev(maps[:2]), m)


def test_rejected_arguments_leave_the_outputs_untouched():
    _C, rt = lib()
    n, C, m, K = (4, 5, 6), 3, (3, 4, 5), 2
    scores = torch.randn((K,) + n + (C,), device="cuda")
    maps = torch.randn(K, 12, device="cuda")
    big_maps = torch.randn(17, 12, device="cuda")
    gt = torch.randint(0, C, m, dtype=torch.uint8, device="cuda")
    out, cm = _buffers(C, m)
    bufs = {"out": out, "cm": cm}
    before = snapshot(bufs)
    big = (1 << 23) + 1
    bad = [
        ("K = 0", BAD_ARG, (scores, 0, n, C, maps, m, out, gt, cm)),
        ("K < 0", BAD_ARG, (scores, -1, n, C, maps, m, out, gt, cm)),
        ("K = 17", UNSUPPORTED, (scores, 17, n, C, big_maps, m, out, gt, cm)),
        ("NULL maps", BAD_ARG, (scores, K, n, C, None, m, out, gt, cm)),
        ("NULL maps, K = 17", BAD_ARG, (scores, 17, n, C, None, m, out, gt, cm)),
        ("C = 1", UNSUPPORTED, (scores, K, n, 1, maps, m, out, gt, cm)),
        ("C = 9", UNSUPPORTED, (scores, K, n, 9, maps, m, out, gt, cm)),
        ("NULL scores", BAD_ARG, (None, K, n, C, maps, m, out, gt, cm)),
        ("NULL out", BAD_ARG, (scores, K, n, C, maps, m, None, gt, cm)),
        ("gt without cm", BAD_ARG, (scores, K, n, C, maps, m, out, gt, None)),
        ("cm without gt", BAD_ARG, (scores, K, n, C, maps, m, out, None, cm)),
        ("n1 = 0", BAD_ARG, (scores, K, (4, 0, 6), C, maps, m, out, gt, cm)),
        ("m2 < 0", BAD_ARG, (scores, K, n, C, maps, (3, 4, -5), out, gt, cm)),
        ("n0 above PNP_RS_MAX_DIM", UNSUPPORTED, (scores, K, (big, 1, 1), C, maps, m, out, gt, cm)),
        ("m1 above PNP_RS_MAX_DIM", UNSUPPORTED, (scores, K, n, C, maps, (1, big, 1), out, gt, cm)),
        ("member n0 n1 n2 C = 2^31", UNSUPPORTED, (scores, K, (1 << 10, 1 << 10, 1 << 8), 8, maps, m, out, gt, cm)),
        ("m0 m1 m2 = 2^31", UNSUPPORTED, (scores, K, n, C, maps, (1 << 11, 1 << 10, 1 << 10), out, gt, cm)),
    ]
    for what, rc_want, args in bad:
        rc = _call(_C, rt, *args)
        assert rc == rc_want, (what, rc)
        assert_untouched(what, "pnp_native_labels_ensemble", bufs, before)
