"""A third reference of pnp_surface_distance and pnp_surface_distance_pct (include/pnp_b200.h), fast enough for native CT volumes
(512 x 512 x 300, ~80 M voxels), where surface_exact.scipy_raw takes minutes and brute_raw cannot run at all:

* borders: per class, the boolean volume X minus its erosion by the 6-neighbour cross (voxels outside the volume are not in X),
  from six shifted ANDs; labels outside [1, num_cls) are never equal to a class, so they count as background;
* distances: for every voxel v of dA the nearest voxels of dB by scipy.spatial.cKDTree over the scaled coordinates
  idx * spacing, then d(v, dB) re-derived from the integer index differences D in the header's expression and order, fp64:
  sqrt(((s0 D0)^2 + (s1 D1)^2) + (s2 D2)^2); likewise with dA and dB swapped.  At unit spacing every squared distance is an
  integer the tree computes exactly, so its nearest voxel gives the minimum bit for bit.  At other spacings every voxel within
  (1 + 1e-12) of the tree's minimum is a candidate and the smallest re-derived value wins: the header's definition, the minimum
  over dB of that expression, whatever order the tree rounds its own distances in.

`kdtree_raw` gives surface_exact's [C-1, 6] table (sums by math.fsum, the same NaN rules), `kdtree_distances` the per-class
pooled arrays (da, db) that surface_percentile.hd_percentile(form="kdtree") reads.  `native_ct_subject` and `line_features`
build the phantoms of the native-size tests.  Host numpy + scipy only."""
import math

import numpy as np
from scipy.spatial import cKDTree

from oracle import surface_exact as se

TIE = 1e-12            # relative width of the band of candidates around the tree's minimum at non-unit spacing
K = 8                  # candidates asked of the tree per query before the band is searched in full


def _border(x):
    """boolean x minus its erosion by the 6-neighbour cross, voxels outside the volume counting as not in x"""
    inner = x.copy()
    inner[0] = inner[-1] = False
    inner[:, 0] = inner[:, -1] = False
    inner[:, :, 0] = inner[:, :, -1] = False
    inner[1:] &= x[:-1]
    inner[:-1] &= x[1:]
    inner[:, 1:] &= x[:, :-1]
    inner[:, :-1] &= x[:, 1:]
    inner[:, :, 1:] &= x[:, :, :-1]
    inner[:, :, :-1] &= x[:, :, 1:]
    return x & ~inner


def borders(vol, num_cls):
    """[num_cls] list (entry 0 None) of int64 [n, 3] border voxel indices of each class, in C order"""
    v = np.asarray(vol)
    if v.ndim != 3:
        raise ValueError("expected a 3-D label volume, got shape %s" % (v.shape,))
    return [None] + [np.argwhere(_border(v == c)) for c in range(1, num_cls)]


def _d2(src, dst, sp):
    """squared distances ((s0 D0)^2 + (s1 D1)^2) + (s2 D2)^2 in fp64, D = src - dst exact in integers"""
    D = (src - dst).astype(np.float64)
    d0, d1, d2 = D[..., 0] * sp[0], D[..., 1] * sp[1], D[..., 2] * sp[2]
    return (d0 * d0 + d1 * d1) + d2 * d2


def _nearest(src, dst, sp):
    """d(v, dst) for every v of src (integer indices [n, 3]) -- the minimum over dst of the header's expression"""
    s = np.asarray(sp, np.float64)
    tree = cKDTree(dst * s)
    pts = src * s
    if sp == (1.0, 1.0, 1.0):
        _, i = tree.query(pts, k=1, workers=-1)
        return np.sqrt(_d2(src, dst[i], sp))
    k = min(K, len(dst))
    dist, idx = tree.query(pts, k=k, workers=-1)
    dist, idx = dist.reshape(len(src), k), idx.reshape(len(src), k)
    band = dist[:, 0] * (1.0 + TIE)
    d2 = np.where(dist <= band[:, None], _d2(src[:, None, :], dst[idx], sp), np.inf)
    best = d2.min(axis=1)
    if k < len(dst):
        for r in np.flatnonzero(dist[:, -1] <= band):     # more than k candidates in the band: all of them
            j = tree.query_ball_point(pts[r], band[r])
            best[r] = _d2(src[r], dst[j], sp).min()
    return np.sqrt(best)


def kdtree_distances(pred, gt, num_cls, spacing=None):
    """(dist, borders of pred, borders of gt): dist is a [num_cls] list (entry 0 None) of (da, db), d(v, dB) for v in dA and
    d(v, dA) for v in dB, each in C order of the voxels, (None, None) when either border is empty; the borders are
    `borders`' index arrays"""
    sp = se._spacing(spacing)
    ba, bb = borders(pred, num_cls), borders(gt, num_cls)
    out = [None]
    for c in range(1, num_cls):
        a, b = ba[c], bb[c]
        out.append((_nearest(a, b, sp), _nearest(b, a, sp)) if len(a) and len(b) else (None, None))
    return out, ba, bb


def raw_table(dist, ba, bb):
    """surface_exact's [C-1, 6] table from kdtree_distances' result"""
    out = np.zeros((len(dist) - 1, 6))
    for c in range(1, len(dist)):
        da, db = dist[c]
        na, nb = len(ba[c]), len(bb[c])
        if da is None:
            out[c - 1] = se._row(0.0, 0.0, na, 0.0, 0.0, nb)
        else:
            out[c - 1] = se._row(math.fsum(da), float(da.max()), na, math.fsum(db), float(db.max()), nb)
    return out


def kdtree_raw(pred, gt, num_cls, spacing=None):
    return raw_table(*kdtree_distances(pred, gt, num_cls, spacing))


# ---- phantoms ------------------------------------------------------------------------------------------------------------------
def ellipsoid(vol, c, centre, radii):
    """sets the voxels of `vol` strictly inside the ellipsoid (centre, radii), clipped to the volume, to c; touches only its box"""
    centre, radii = np.asarray(centre, np.float64), np.asarray(radii, np.float64)
    lo = np.maximum(np.floor(centre - radii).astype(np.int64), 0)
    hi = np.minimum(np.ceil(centre + radii).astype(np.int64) + 1, vol.shape)
    if (hi <= lo).any():
        return
    g = np.ogrid[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
    inside = sum(((g[a] - centre[a]) / radii[a]) ** 2 for a in range(3)) < 1.0
    vol[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]][inside] = c


def native_ct_subject(seed, shape=(512, 512, 300), num_cls=8):
    """(pred, gt) uint8 [shape]: a CT-sized phantom.  gt holds num_cls - 1 ellipsoid organs: organ 1 cut by the face i0 = 0,
    organ 2 by the face i2 = n2 - 1, organs 3 and 4 overlapping (touching along a shared surface), the rest anywhere.  pred is
    gt shifted by (3, -2, 2) voxels with zeros shifted in, a 1e-3 speckle of labels drawn from [0, num_cls + 2] (labels >= num_cls
    included) and a few detached fragments of random organs.  Vectorised: a 512 x 512 x 300 pair takes seconds."""
    rng = np.random.default_rng(seed)
    n = np.array(shape, np.float64)
    gt = np.zeros(shape, np.uint8)
    prev = None
    for c in range(1, num_cls):
        radii = rng.uniform(0.07, 0.2, 3) * n + 1.0
        centre = rng.uniform(0.2, 0.8, 3) * n
        if c == 1:
            centre[0] = 0.3 * radii[0]
        elif c == 2:
            centre[2] = n[2] - 1 - 0.4 * radii[2]
        elif c == 4:
            centre = prev[0] + 0.8 * (prev[1] + radii) * np.array([0.0, 1.0, 0.0])
        ellipsoid(gt, c, centre, radii)
        prev = (centre, radii)
    pred = np.zeros(shape, np.uint8)
    shift = (3, -2, 2)
    src = tuple(slice(max(0, -s), shape[a] - max(0, s)) for a, s in enumerate(shift))
    dst = tuple(slice(max(0, s), shape[a] - max(0, -s)) for a, s in enumerate(shift))
    pred[dst] = gt[src]
    for _ in range(5):
        ellipsoid(pred, int(rng.integers(1, num_cls)), rng.uniform(0.05, 0.95, 3) * n, rng.uniform(2.0, 7.0, 3))
    N = pred.size
    k = int(N * 1e-3)
    pred.reshape(-1)[rng.integers(0, N, k)] = rng.integers(0, num_cls + 3, k).astype(np.uint8)
    return pred, gt


def line_features(shape, axis):
    """(pred, gt) uint8 [shape], C = 4, of one-voxel features on lines along `axis` (n = shape[axis]; the other two sizes at
    least 3), so that distances along a line reach n - 1 and an envelope holds n parabolas:
      class 1: pred at position 0 and gt at position n - 1 of one line: d = n - 1 both ways;
      class 2: gt along a whole line (n features, g = 0 at each: n envelope entries in every pass along `axis`), pred along
               positions [n/3, 2n/3) of the neighbouring line;
      class 3: pred at both ends of a line, gt at its middle and one line over."""
    pred, gt = np.zeros(shape, np.uint8), np.zeros(shape, np.uint8)
    n = shape[axis]
    others = [a for a in range(3) if a != axis]

    def at(vol, pos, o, c):
        idx = [0, 0, 0]
        idx[axis] = pos
        idx[others[0]], idx[others[1]] = o
        vol[tuple(idx)] = c

    m0, m1 = shape[others[0]], shape[others[1]]
    at(pred, 0, (0, 0), 1)
    at(gt, n - 1, (0, 0), 1)
    at(gt, slice(None), (m0 - 1, m1 - 1), 2)
    at(pred, slice(n // 3, 2 * n // 3), (m0 - 2, m1 - 1), 2)
    at(pred, 0, (m0 // 2, m1 // 2), 3)
    at(pred, n - 1, (m0 // 2, m1 // 2), 3)
    at(gt, n // 2, (m0 // 2, m1 // 2 - 1), 3)
    return pred, gt
