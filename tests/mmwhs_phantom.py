"""Seeded phantom MMWHS subjects for the data-preparation tests: nested ellipsoids carrying all seven MMWHS label values in a
RAS-ordered voxel grid with anisotropic spacing, and the same subject re-stored under any signed axis permutation of its affine."""
import itertools
import os

import numpy as np

# MMWHS value -> (centre as a fraction of the grid, radii as a fraction of the grid, mean intensity); later entries overwrite
STRUCTURES = [(550, (0.45, 0.62, 0.50), (0.20, 0.16, 0.22), 260.0),     # RV blood
              (600, (0.38, 0.45, 0.66), (0.16, 0.14, 0.14), 250.0),     # RA blood
              (205, (0.58, 0.48, 0.46), (0.22, 0.20, 0.24), 120.0),     # LV myocardium
              (500, (0.58, 0.48, 0.46), (0.14, 0.12, 0.16), 300.0),     # LV blood
              (420, (0.60, 0.30, 0.62), (0.15, 0.10, 0.12), 280.0),     # LA blood
              (820, (0.50, 0.42, 0.72), (0.07, 0.07, 0.14), 320.0),     # ascending aorta
              (850, (0.42, 0.58, 0.74), (0.07, 0.07, 0.10), 310.0)]     # pulmonary artery


def ras_subject(seed, shape=(48, 44, 26), spacing=(0.8, 0.9, 1.6), unknown=0):
    """(image int16, label int16) in RAS voxel order (axis 0 +x, 1 +y, 2 +z) and the diagonal affine; `unknown` voxels carry a
    label value outside the MMWHS set"""
    rng = np.random.RandomState(seed)
    g = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij")
    lab = np.zeros(shape, np.int16)
    img = rng.normal(-50.0, 40.0, shape)
    for v, centre, radii, mean in STRUCTURES:
        c = (np.array(centre) + rng.uniform(-0.03, 0.03, 3)) * np.array(shape)
        r = np.array(radii) * np.array(shape)
        m = sum(((g[a] - c[a]) / r[a]) ** 2 for a in range(3)) <= 1.0
        lab[m] = v
        img[m] = rng.normal(mean, 25.0, int(m.sum()))
    img[rng.rand(*shape) < 0.003] = 3000.0                  # bright outliers: the 98th-percentile cut has work to do
    if unknown:
        flat = rng.choice(lab.size, unknown, replace=False)
        lab.reshape(-1)[flat] = 7
    aff = np.diag(list(spacing) + [1.0])
    aff[:3, 3] = (-40.0, 12.5, -7.0)
    return img.astype(np.int16), lab, aff


SIGNED_PERMUTATIONS = [(p, s) for p in itertools.permutations(range(3)) for s in itertools.product((1, -1), repeat=3)]


def permuted(arr, affine, perm, signs):
    """the RAS-ordered `arr` stored with voxel axis v along RAS axis perm[v] in direction signs[v], and that storage's affine"""
    out = np.transpose(arr, perm)
    A = np.zeros((4, 4))
    A[3, 3] = 1.0
    x0 = np.zeros(3)
    for v in range(3):
        w = perm[v]
        if signs[v] < 0:
            out = np.flip(out, v)
            x0[w] = arr.shape[w] - 1
        A[w, v] = signs[v] * affine[w, w]
    A[:3, 3] = affine[:3, :3] @ x0 + affine[:3, 3]
    return np.ascontiguousarray(out), A


def write_pairs(directory, modality, seeds, perms=None, **kw):
    """phantom subjects as {modality}_train_10xx_{image,label}.nii.gz under `directory` -> [(image path, label path)]"""
    from pnp_b200 import nifti
    pairs = []
    for i, seed in enumerate(seeds):
        img, lab, aff = ras_subject(seed, **kw)
        perm, signs = (perms or SIGNED_PERMUTATIONS)[(7 * i + 3) % len(perms or SIGNED_PERMUTATIONS)]
        ri, A = permuted(img, aff, perm, signs)
        rl, _ = permuted(lab, aff, perm, signs)
        ip = os.path.join(directory, "%s_train_%d_image.nii.gz" % (modality, 1001 + i))
        lp = os.path.join(directory, "%s_train_%d_label.nii.gz" % (modality, 1001 + i))
        nifti.save(ri, A, ip)
        nifti.save(rl, A, lp)
        pairs.append((ip, lp))
    return pairs
