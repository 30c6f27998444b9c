"""A numpy float32 restatement of pnp_native_accumulate and pnp_native_accumulated_labels (csrc/resample.cu, include/pnp_b200.h
"native-grid labels of any number of predictions") in the kernels' operation order, built from oracle/native_exact.py's pieces.
Test-only.

accumulate_ref runs one launch per prediction, in the given order: u = native_exact.coords of its map; where native_exact.inside
holds, its class scores (native_exact.class_scores) are stored as they are into a voxel not yet covered and added to the sums
(one float32 addition per class) of a covered one.  labels_ref is native_exact.first_max of the sums where covered, 0 elsewhere.
Each mutation flag restates one plausible kernel bug (add_to_zero, descending): tests/test_localise_cpu.py checks that each one
changes some output."""
import numpy as np

from oracle import native_exact as N

F32 = np.float32


def accumulate_ref(scores, maps, shape, add_to_zero=False, descending=False):
    """-> (sums fp32 [m0, m1, m2, C], covered uint8 [m0, m1, m2]) after one launch per prediction (scores fp32 [K, n0, n1, n2, C]
    or a list of [n_k, C] volumes of any shapes, maps fp32 [K, 12]).
    add_to_zero: the first covering prediction added to the zeroed sums instead of stored (+0 + -0 is +0);
    descending:  the predictions launched in descending k."""
    maps = np.asarray(maps, F32).reshape(-1, 12)
    K = len(scores)
    if maps.shape[0] != K:
        raise ValueError("%d score volumes but %d maps" % (K, maps.shape[0]))
    shape = tuple(int(s) for s in shape)
    C = np.asarray(scores[0]).shape[-1]
    sums = np.zeros(shape + (C,), F32)
    covered = np.zeros(shape, np.uint8)
    for k in (range(K - 1, -1, -1) if descending else range(K)):
        member = np.asarray(scores[k], F32)
        u = N.coords(maps[k], shape)
        ok = N.inside(u, member.shape[:3])
        if not ok.any():
            continue
        v = N.class_scores(member, u[:, ok]).T              # [voxels, C]
        first = covered[ok] == 0
        if add_to_zero:
            sums[ok] = sums[ok] + v
        else:
            sums[ok] = np.where(first[:, None], v, sums[ok] + v)
        covered[ok] = 1
    return sums, covered


def labels_ref(sums, covered):
    """-> uint8 [m0, m1, m2]: the first maximum of each covered voxel's sums, 0 elsewhere"""
    sums, covered = np.asarray(sums, F32), np.asarray(covered) != 0
    out = np.zeros(covered.shape, np.uint8)
    if covered.any():
        out[covered] = N.first_max(np.moveaxis(sums[covered], -1, 0)).astype(np.uint8)
    return out


def boxes_ref(labels, C):
    """int64 [C, 7]: per class (count, lo0, hi0, lo1, hi1, lo2, hi2) of `labels` (labels >= C count as class 0); an empty class is
    (0, n0, -1, n1, -1, n2, -1)"""
    labels = np.asarray(labels)
    cls = np.where(labels < C, labels, 0)
    n = labels.shape
    out = np.zeros((C, 7), np.int64)
    for c in range(C):
        m = cls == c
        out[c, 0] = int(m.sum())
        for a in range(3):
            nz = np.flatnonzero(np.any(m, axis=tuple(b for b in range(3) if b != a)))
            out[c, 1 + 2 * a], out[c, 2 + 2 * a] = (int(nz[0]), int(nz[-1])) if nz.size else (n[a], -1)
    return out
