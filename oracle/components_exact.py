"""Largest connected component per class of a 3-D label volume: two independent references for pnp_largest_components.

Definition (include/pnp_b200.h, "largest connected component per class"): labels >= C are background.  For each class c in
1 .. C-1 the components of {v : labels[v] == c} are taken under 6- or 26-connectivity; the kept one has the most voxels, and
among equal sizes the one whose smallest C-order linear index is smallest.  out[v] = c inside the kept component of c, else 0.
stats[c] = (components, voxels kept, voxels removed); row 0 = (0, 0, number of labels >= C).  cm[gt][out] over every voxel,
ground-truth labels >= C as background.

scipy_lcc: scipy.ndimage.label per class, sizes by np.bincount, np.argmax (scipy numbers components in raster order of their
first voxel, so the first maximum is the tie rule).  bfs_lcc: a plain Python flood fill for small volumes, written without
scipy, with the tie rule stated explicitly."""
from collections import deque

import numpy as np


def structure(connectivity):
    from scipy import ndimage
    if connectivity not in (6, 26):
        raise ValueError("connectivity must be 6 or 26, got %r" % (connectivity,))
    return ndimage.generate_binary_structure(3, 1 if connectivity == 6 else 3)


def confusion(gt, out, C):
    """cm[gt][out] with ground-truth labels >= C as background (np.bincount)"""
    g = np.asarray(gt).astype(np.int64).ravel()
    g = np.where(g < C, g, 0)
    return np.bincount(g * C + np.asarray(out).astype(np.int64).ravel(), minlength=C * C).reshape(C, C)


def scipy_lcc(labels, C, connectivity, gt=None):
    """-> (out uint8 like labels, stats int64 [C, 3], cm int64 [C, C] or None)"""
    from scipy import ndimage
    labels = np.asarray(labels)
    s = structure(connectivity)
    out = np.zeros(labels.shape, np.uint8)
    stats = np.zeros((C, 3), np.int64)
    stats[0, 2] = int((labels >= C).sum())
    for c in range(1, C):
        mask = labels == c
        lab, n = ndimage.label(mask, s)
        stats[c, 0] = n
        if n == 0:
            continue
        sizes = np.bincount(lab.ravel())[1:]
        keep = int(np.argmax(sizes)) + 1
        out[lab == keep] = c
        stats[c, 1] = int(sizes[keep - 1])
        stats[c, 2] = int(mask.sum()) - stats[c, 1]
    return out, stats, (None if gt is None else confusion(gt, out, C))


def neighbours(connectivity):
    """the offsets of the 6 face or 26 face / edge / corner neighbours"""
    offs = [(a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1) if (a, b, c) != (0, 0, 0)]
    if connectivity == 6:
        return [d for d in offs if sum(map(abs, d)) == 1]
    if connectivity == 26:
        return offs
    raise ValueError("connectivity must be 6 or 26, got %r" % (connectivity,))


def bfs_lcc(labels, C, connectivity, gt=None):
    """the same by breadth-first flood fill in plain Python (small volumes): components found in C order of their first voxel,
    and a later component replaces the kept one only if it is strictly larger -> (out, stats, cm or None)"""
    labels = np.asarray(labels)
    n0, n1, n2 = labels.shape
    lab = labels.tolist()
    offs = neighbours(connectivity)
    seen = [[[False] * n2 for _ in range(n1)] for _ in range(n0)]
    best = {}                               # class -> (size, voxels) of the kept component so far
    stats = np.zeros((C, 3), np.int64)
    for i in range(n0):
        for j in range(n1):
            for k in range(n2):
                c = lab[i][j][k]
                if c >= C:
                    stats[0, 2] += 1
                    continue
                if c == 0 or seen[i][j][k]:
                    continue
                seen[i][j][k] = True
                comp, todo = [], deque([(i, j, k)])
                while todo:
                    a, b, e = todo.popleft()
                    comp.append((a, b, e))
                    for d0, d1, d2 in offs:
                        x, y, z = a + d0, b + d1, e + d2
                        if 0 <= x < n0 and 0 <= y < n1 and 0 <= z < n2 and not seen[x][y][z] and lab[x][y][z] == c:
                            seen[x][y][z] = True
                            todo.append((x, y, z))
                stats[c, 0] += 1
                # (i, j, k) is this component's first voxel in C order, and components are met in that order: keeping the
                # earlier one on a tie keeps the one whose smallest linear index is smallest
                if c not in best or len(comp) > best[c][0]:
                    best[c] = (len(comp), comp)
    out = np.zeros(labels.shape, np.uint8)
    for c, (size, comp) in best.items():
        for v in comp:
            out[v] = c
        stats[c, 1] = size
        stats[c, 2] = int((labels == c).sum()) - size
    return out, stats, (None if gt is None else confusion(gt, out, C))
