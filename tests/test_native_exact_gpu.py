"""pnp_native_labels (csrc/resample.cu) bit for bit against its numpy restatement oracle/native_exact.py, at the C-ABI: C = 2, 5
and 8, tie-heavy scores (constant planes, equal pairs), coordinates exactly at -0.5 and n - 0.5, NaN coordinates, permuted and
negative maps, the grid-stride cap with several iterations and a single partial CTA; the confusion counts equal np.bincount;
repeated calls are bit-identical; every rejected argument leaves its sentinel-filled outputs untouched.  The case table is shared
with tests/test_native_exact_cpu.py, which checks the restatement itself."""
import numpy as np
import pytest
import torch

from oracle import native_exact as N
from tests.cabi import BAD_ARG, UNSUPPORTED, assert_untouched, lib, snapshot, sync

F32 = np.float32
OUT_SENTINEL = 0xAB
CM_SENTINEL = -0x5EED

# (tag, score grid (n0, n1, n2), C, native grid (m0, m1, m2), score kind, map kind)
CASES = [
    ("random_c2", (9, 13, 7), 2, (11, 10, 12), "random", "random"),
    ("random_c5", (12, 9, 10), 5, (13, 8, 11), "random", "random"),
    ("random_c8", (7, 11, 9), 8, (10, 12, 9), "random", "random"),
    ("permuted_c5", (10, 12, 8), 5, (14, 9, 12), "random", "permuted"),
    ("negative_c8", (9, 10, 11), 8, (12, 11, 10), "random", "negative"),
    ("ties_c5", (8, 9, 10), 5, (12, 13, 11), "ties", "random"),
    ("near_ties_c2", (12, 14, 10), 2, (30, 28, 26), "near_ties", "random"),
    ("edges_c3", (6, 7, 5), 3, (7, 8, 11), "random", "edges"),
    ("nan_c4", (6, 5, 7), 4, (5, 6, 8), "random", "nan"),
    ("partial_cta_c3", (5, 6, 7), 3, (5, 7, 9), "random", "random"),
    ("cap_c2", (40, 64, 64), 2, (220, 205, 200), "random", "scaled"),
]


def _scores(kind, n, C, rng):
    if kind == "ties":          # constant planes and equal pairs: exact ties everywhere
        s = np.zeros(tuple(n) + (C,), F32)
        s[..., 0] = rng.randint(0, 3, n) * F32(0.5)
        s[..., 1] = s[..., 0]
        s[..., 2] = F32(0.5)
        s[..., 3] = rng.randint(0, 3, n) * F32(0.5)
        s[..., 4] = s[..., 3]
        s[n[0] // 2] = F32(0.25)                       # a constant plane: every class ties there
        return s
    s = rng.standard_normal(tuple(n) + (C,)).astype(F32)
    if kind == "near_ties":     # class 1 is class 0 moved by a few ulp: the argmax turns on the last bits
        s[..., 1] = s[..., 0] + s[..., 0] * F32(2.0 ** -22) * rng.randint(-2, 3, n).astype(F32)
    return s


def _map(kind, n, m, rng):
    n, m = np.array(n, np.float64), np.array(m, np.float64)
    M = np.zeros((3, 4))
    if kind == "edges":         # u_a = s_a * index - 0.5: the first voxel lands on -0.5 (inside), some on n - 0.5 (outside)
        for a in range(3):
            M[a, a] = (n[a]) / (m[a] - 1)
            M[a, 3] = -0.5
        M[2, 2] = 0.5           # n2 = 5, m2 = 11: u2 = 0.5 k - 0.5 reaches 4.5 = n2 - 0.5 at k = 10
    elif kind == "nan":         # an infinite coefficient: inf * 0 = NaN at k = 0, inf beyond
        M[0, 0], M[1, 1], M[2, 2] = 1.0, 1.0, np.inf
    elif kind == "permuted":    # u0 follows k, u1 follows i, u2 follows j
        M[0, 2], M[1, 0], M[2, 1] = n[0] / m[2], n[1] / m[0], n[2] / m[1]
        M[:, 3] = rng.uniform(-1.0, 0.5, 3)
    elif kind == "negative":    # every axis reversed
        for a in range(3):
            M[a, a] = -rng.uniform(0.8, 1.2) * n[a] / m[a]
            M[a, 3] = n[a] - 0.5 + rng.uniform(-0.5, 0.5)
    elif kind == "scaled":
        for a in range(3):
            M[a, a] = rng.uniform(0.9, 1.1) * n[a] / m[a]
            M[a, 3] = rng.uniform(-1.0, 1.0)
    else:
        M[:, :3] = rng.uniform(-1.5, 1.5, (3, 3)) * (n[:, None] / m[None, :])
        M[:, 3] = rng.uniform(-1, n + 1)
    return M.astype(F32).reshape(-1)


def operands(case):
    """(scores fp32 [n0, n1, n2, C], map fp32 [12], gt uint8 [m0, m1, m2]) of a case, drawn on the host from a seed of the case;
    gt holds labels up to C + 1 (those >= C count as background)"""
    tag, n, C, m, skind, mkind = case
    rng = np.random.RandomState(sum(map(ord, tag)))
    scores = _scores(skind, n, C, rng)
    vmap = _map(mkind, n, m, rng)
    gt = rng.randint(0, C + 2, m).astype(np.uint8)
    return scores, vmap, gt


def _call(_C, rt, scores, n, C, vmap, m, out, gt, cm):
    p = lambda t: None if t is None else t.data_ptr()
    return _C.lib.pnp_native_labels(p(scores), *n, C, p(vmap), *m, p(out), p(gt), p(cm), rt.stream())


def _buffers(C, m):
    out = torch.full(tuple(m), OUT_SENTINEL, dtype=torch.uint8, device="cuda")
    cm = torch.full((C, C), CM_SENTINEL, dtype=torch.int64, device="cuda")
    return out, cm


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_pnp_native_labels_bit_exact(case):
    _C, rt = lib()
    tag, n, C, m, _, _ = case
    scores, vmap, gt = operands(case)
    ds, dm, dg = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (scores, vmap, gt))
    out, cm = _buffers(C, m)
    assert _call(_C, rt, ds, n, C, dm, m, out, dg, cm) == 0
    sync()
    want = N.labels_ref(scores, vmap, m)
    got = out.cpu().numpy()
    bad = np.argwhere(got != want)
    assert bad.size == 0, "%s: %d of %d labels differ; first at %s: got %d, ref %d" % (
        tag, len(bad), got.size, tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])])
    assert np.array_equal(cm.cpu().numpy(), N.confusion_ref(want, gt, C)), tag + " confusion counts"
    assert int(cm.sum()) == int(np.prod(m))
    print("  %s: %s native voxels, classes %s" % (tag, got.size, np.bincount(got.reshape(-1), minlength=C).tolist()))
    # repeated calls are bit-identical; without gt only the labels are written
    first_out, first_cm = out.clone(), cm.clone()
    assert _call(_C, rt, ds, n, C, dm, m, out, dg, cm) == 0
    sync()
    assert torch.equal(first_out, out) and torch.equal(first_cm, cm)
    out2, cm2 = _buffers(C, m)
    assert _call(_C, rt, ds, n, C, dm, m, out2, None, None) == 0
    sync()
    assert torch.equal(out2, out) and bool((cm2 == CM_SENTINEL).all())


@pytest.mark.gpu
def test_functional_wrapper_equals_the_c_abi():
    lib()
    from pnp_b200 import functional as F
    case = CASES[3]
    tag, n, C, m, _, _ = case
    scores, vmap, gt = operands(case)
    labels, cm = F.native_labels(torch.from_numpy(scores).cuda(), torch.from_numpy(vmap).cuda(), m, torch.from_numpy(gt).cuda())
    want = N.labels_ref(scores, vmap, m)
    assert labels.dtype == torch.uint8 and tuple(labels.shape) == m
    assert np.array_equal(labels.cpu().numpy(), want) and np.array_equal(cm.cpu().numpy(), N.confusion_ref(want, gt, C))
    alone, none = F.native_labels(torch.from_numpy(scores).cuda(), torch.from_numpy(vmap).cuda(), m)
    assert none is None and torch.equal(alone, labels)


@pytest.mark.gpu
def test_rejected_arguments_leave_the_outputs_untouched():
    _C, rt = lib()
    n, C, m = (4, 5, 6), 3, (3, 4, 5)
    scores = torch.randn(n + (C,), device="cuda")
    vmap = torch.randn(12, device="cuda")
    gt = torch.randint(0, C, m, dtype=torch.uint8, device="cuda")
    out, cm = _buffers(C, m)
    bufs = {"out": out, "cm": cm}
    before = snapshot(bufs)
    big = (1 << 23) + 1
    bad = [
        ("C = 1", UNSUPPORTED, (scores, n, 1, vmap, m, out, gt, cm)),
        ("C = 9", UNSUPPORTED, (scores, n, 9, vmap, m, out, gt, cm)),
        ("NULL scores", BAD_ARG, (None, n, C, vmap, m, out, gt, cm)),
        ("NULL map", BAD_ARG, (scores, n, C, None, m, out, gt, cm)),
        ("NULL out", BAD_ARG, (scores, n, C, vmap, m, None, gt, cm)),
        ("gt without cm", BAD_ARG, (scores, n, C, vmap, m, out, gt, None)),
        ("cm without gt", BAD_ARG, (scores, n, C, vmap, m, out, None, cm)),
        ("n1 = 0", BAD_ARG, (scores, (4, 0, 6), C, vmap, m, out, gt, cm)),
        ("m2 < 0", BAD_ARG, (scores, n, C, vmap, (3, 4, -5), out, gt, cm)),
        ("n0 above PNP_RS_MAX_DIM", UNSUPPORTED, (scores, (big, 1, 1), C, vmap, m, out, gt, cm)),
        ("m1 above PNP_RS_MAX_DIM", UNSUPPORTED, (scores, n, C, vmap, (1, big, 1), out, gt, cm)),
        ("n0 n1 n2 C = 2^31", UNSUPPORTED, (scores, (1 << 10, 1 << 10, 1 << 8), 8, vmap, m, out, gt, cm)),
        ("m0 m1 m2 = 2^31", UNSUPPORTED, (scores, n, C, vmap, (1 << 11, 1 << 10, 1 << 10), out, gt, cm)),
    ]
    for what, rc_want, args in bad:
        rc = _call(_C, rt, *args)
        assert rc == rc_want, (what, rc)
        assert_untouched(what, "pnp_native_labels", bufs, before)
    assert _C.lib.pnp_version() >= 104
