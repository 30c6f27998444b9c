"""Two independent references of pnp_surface_distance (include/pnp_b200.h, "evaluation: 3-D surface distances"): per-class
border sets of a predicted and a ground-truth label volume and the distances between them, in the C-ABI's output layout
out[C-1, 6] = [sum d(dA -> dB), |dA|, max d(dA -> dB), sum d(dB -> dA), |dB|, max d(dB -> dA)].

* `scipy_raw` restates the definition with scipy.ndimage: dX = X & ~binary_erosion(X, 6-neighbour cross, border_value=0) and
  d(., dB) = distance_transform_edt(~dB, sampling=spacing); sums are math.fsum (correctly rounded).
* `brute_raw` finds the borders by comparing every voxel with its six neighbours in a zero-padded copy and the distances by
  testing every pair of border voxels, with d^2 = ((s0 D0)^2 + (s1 D1)^2) + (s2 D2)^2 -- scipy's expression and order.  It is
  for small volumes.

Labels outside [0, num_cls) count as background.  A class whose border is empty in either volume gets NaN sums and maxima.
Host numpy only."""
import math

import numpy as np
from scipy import ndimage

CROSS = ndimage.generate_binary_structure(3, 1)


def _labels(vol, num_cls):
    v = np.asarray(vol)
    if v.ndim != 3:
        raise ValueError("expected a 3-D label volume, got shape %s" % (v.shape,))
    return np.where((v >= 0) & (v < num_cls), v, 0)


def _spacing(spacing):
    return (1.0, 1.0, 1.0) if spacing is None else tuple(float(s) for s in spacing)


def scipy_borders(vol, num_cls):
    """[num_cls] list of boolean border volumes (entry 0, background, is None)"""
    lab = _labels(vol, num_cls)
    out = [None]
    for c in range(1, num_cls):
        x = lab == c
        out.append(x & ~ndimage.binary_erosion(x, structure=CROSS, iterations=1, border_value=0))
    return out


def brute_borders(vol, num_cls):
    """the same border sets from an explicit six-neighbour comparison (voxels outside the volume are background)"""
    lab = _labels(vol, num_cls).astype(np.int64)
    p = np.pad(lab, 1, constant_values=-1)
    n0, n1, n2 = lab.shape
    core = p[1:-1, 1:-1, 1:-1]
    differs = np.zeros(lab.shape, bool)
    for a in range(3):
        for s in (-1, 1):
            sl = [slice(1, n0 + 1), slice(1, n1 + 1), slice(1, n2 + 1)]
            sl[a] = slice(1 + s, (n0, n1, n2)[a] + 1 + s)
            differs |= p[tuple(sl)] != core
    return [None] + [(lab == c) & differs for c in range(1, num_cls)]


def _row(sums_a, max_a, na, sums_b, max_b, nb):
    if na == 0 or nb == 0:
        return [math.nan, float(na), math.nan, math.nan, float(nb), math.nan]
    return [sums_a, float(na), max_a, sums_b, float(nb), max_b]


def scipy_raw(pred, gt, num_cls, spacing=None):
    sp = _spacing(spacing)
    bp, bg = scipy_borders(pred, num_cls), scipy_borders(gt, num_cls)
    out = np.zeros((num_cls - 1, 6))
    for c in range(1, num_cls):
        a, b = bp[c], bg[c]
        na, nb = int(a.sum()), int(b.sum())
        if na and nb:
            da = ndimage.distance_transform_edt(~b, sampling=sp)[a]
            db = ndimage.distance_transform_edt(~a, sampling=sp)[b]
            out[c - 1] = _row(math.fsum(da), float(da.max()), na, math.fsum(db), float(db.max()), nb)
        else:
            out[c - 1] = _row(0.0, 0.0, na, 0.0, 0.0, nb)
    return out


def _nearest(src, dst, sp, chunk=2048):
    """d(v, dst) for every v of src (integer coordinates [n, 3]), all pairs"""
    out = np.empty(len(src))
    for i in range(0, len(src), chunk):
        diff = (src[i:i + chunk, None, :] - dst[None, :, :]).astype(np.float64)
        d = [diff[..., k] * sp[k] for k in range(3)]
        d2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
        out[i:i + chunk] = np.sqrt(d2.min(axis=1))
    return out


def brute_raw(pred, gt, num_cls, spacing=None):
    sp = _spacing(spacing)
    bp, bg = brute_borders(pred, num_cls), brute_borders(gt, num_cls)
    out = np.zeros((num_cls - 1, 6))
    for c in range(1, num_cls):
        a, b = np.argwhere(bp[c]), np.argwhere(bg[c])
        if len(a) and len(b):
            da, db = _nearest(a, b, sp), _nearest(b, a, sp)
            out[c - 1] = _row(math.fsum(da), float(da.max()), len(a), math.fsum(db), float(db.max()), len(b))
        else:
            out[c - 1] = _row(0.0, 0.0, len(a), 0.0, 0.0, len(b))
    return out


def metrics(raw):
    """per-class arrays [num_cls] (index 0 and classes with an empty border: NaN) from a raw [num_cls - 1, 6] table"""
    raw = np.asarray(raw, np.float64)
    nan = np.full(raw.shape[0] + 1, math.nan)
    m = {k: nan.copy() for k in ("asd_pred_gt", "asd_gt_pred", "assd", "hd")}
    m["border_pred"] = np.zeros(raw.shape[0] + 1, np.int64)
    m["border_gt"] = np.zeros(raw.shape[0] + 1, np.int64)
    for c in range(1, raw.shape[0] + 1):
        s_a, n_a, x_a, s_b, n_b, x_b = raw[c - 1]
        m["border_pred"][c], m["border_gt"][c] = int(n_a), int(n_b)
        if n_a and n_b:
            m["asd_pred_gt"][c], m["asd_gt_pred"][c] = s_a / n_a, s_b / n_b
            m["assd"][c] = (s_a / n_a + s_b / n_b) / 2.0
            m["hd"][c] = max(x_a, x_b)
    return m


def surface_metrics(pred, gt, num_cls, spacing=None):
    """the scipy form, as per-class ASSD / HD arrays"""
    return metrics(scipy_raw(pred, gt, num_cls, spacing))
