"""References of pnp_surface_distance_pct's percentile column (include/pnp_b200.h): the pooled percentile of the surface distances
that medpy.metric.binary.hd95 computes, HD_q = np.percentile(np.hstack((da, db)), q), with da = d(v, dB) over v in dA and
db = d(v, dA) over v in dB, the border sets and distances of oracle/surface_exact.py.

* `scipy_distances` / `brute_distances` give the per-class arrays (da, db) of surface_exact's two forms -- the values its
  `scipy_raw` / `brute_raw` sum and maximise: scipy.ndimage's distance transform, and an all-pairs search for small volumes
  (oracle/surface_kdtree.py's `kdtree_distances`, a nearest-neighbour search fast at native CT size, is the third form);
* `hd_percentile` is medpy's line on them;
* `percentile_linear` restates numpy's default `linear` percentile operation by operation (the formula the kernel implements);
  the CPU tests hold it equal to np.percentile.

Labels outside [0, num_cls) count as background; a class whose border is empty in either volume has no arrays and a NaN
percentile.  Host numpy only."""
import math

import numpy as np
from scipy import ndimage

from oracle import surface_exact as se
from oracle import surface_kdtree as sk


def scipy_distances(pred, gt, num_cls, spacing=None):
    """(dist, borders of pred, borders of gt): dist is a [num_cls] list (entry 0 None) of (da, db), d(v, dB) for v in dA and
    d(v, dA) for v in dB, each in C order of the voxels, (None, None) when either border is empty -- scipy.ndimage's transform"""
    sp = (1.0, 1.0, 1.0) if spacing is None else tuple(float(s) for s in spacing)
    bp, bg = se.scipy_borders(pred, num_cls), se.scipy_borders(gt, num_cls)
    out = [None]
    for c in range(1, num_cls):
        a, b = bp[c], bg[c]
        if a.any() and b.any():
            out.append((ndimage.distance_transform_edt(~b, sampling=sp)[a], ndimage.distance_transform_edt(~a, sampling=sp)[b]))
        else:
            out.append((None, None))
    return out, bp, bg


def brute_distances(pred, gt, num_cls, spacing=None):
    """scipy_distances' result from surface_exact.brute_borders and an all-pairs search (d^2 in scipy's expression and order)"""
    sp = (1.0, 1.0, 1.0) if spacing is None else tuple(float(s) for s in spacing)
    bp, bg = se.brute_borders(pred, num_cls), se.brute_borders(gt, num_cls)
    out = [None]
    for c in range(1, num_cls):
        a, b = np.argwhere(bp[c]), np.argwhere(bg[c])
        out.append((se._nearest(a, b, sp), se._nearest(b, a, sp)) if len(a) and len(b) else (None, None))
    return out, bp, bg


def hd_percentile(pred, gt, num_cls, q, spacing=None, form="scipy"):
    """[num_cls]: medpy.metric.binary.hd95's pooled percentile, np.percentile(np.hstack((da, db)), q), per class (index 0 and
    classes with an empty border: NaN); `form` "scipy", "brute" or "kdtree" (oracle/surface_kdtree.py) picks the distance
    arrays"""
    forms = {"scipy": scipy_distances, "brute": brute_distances, "kdtree": sk.kdtree_distances}
    dist = forms[form](pred, gt, num_cls, spacing)[0]
    out = np.full(num_cls, math.nan)
    for c in range(1, num_cls):
        da, db = dist[c]
        if da is not None:
            out[c] = np.percentile(np.hstack((da, db)), q)
    return out


def percentile_linear(values, q):
    """numpy.percentile(values, q) (method `linear`) restated in plain Python floats, each operation rounded on its own:
    qf = q / 100, v = (n - 1) qf, lo = floor(v) and hi = lo + 1 (both n - 1 when v >= n - 1), gamma = v - lo, a and b the
    order statistics lo and hi, delta = b - a; b - delta (1 - gamma) when gamma >= 0.5, else a + delta gamma (numpy's _lerp)"""
    d = sorted(float(x) for x in values)
    n = len(d)
    qf = float(q) / 100.0
    v = float(n - 1) * qf
    if v >= n - 1:
        lo = hi = n - 1
    else:
        lo = math.floor(v)
        hi = lo + 1
    gamma = v - lo
    a, b = d[lo], d[hi]
    delta = b - a
    return b - delta * (1.0 - gamma) if gamma >= 0.5 else a + delta * gamma
