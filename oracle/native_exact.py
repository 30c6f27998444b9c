"""A numpy float32 restatement of pnp_native_labels (csrc/resample.cu, include/pnp_b200.h "native-grid labels") in the kernel's
operation order, plus its launch configuration.  Test-only.

Every fp32 operation of the kernel is one numpy float32 operation here, rounded on its own: u_a = ((m_a0 i + m_a1 j) + m_a2 k) +
m_a3; class 0 outside [-0.5, n - 0.5) or at a NaN coordinate; otherwise each class score is oracle/resample_exact.py's trilinear
interpolation (the kernel shares pnp_resample_planes' taps and lerps), and the label is the first maximum over the classes.  Each
reference takes the flag of one plausible kernel bug (fma, axis_order, ge, inclusive, no_nan_guard): tests/test_native_exact_cpu.py
checks that each one changes some output."""
import numpy as np

from oracle.elementwise_exact import grid_for
from oracle.resample_exact import CAP, PER_BLOCK, THREADS, Launch, image_ref

F32 = np.float32


def launch(m0, m1, m2):
    """the launcher's grid_for(m0*m1*m2, 1024) grid-stride launch"""
    items = m0 * m1 * m2
    g = grid_for(items, PER_BLOCK)
    return Launch(g, -(-items // PER_BLOCK) > CAP, -(-items // (g * THREADS)), g == 1 and items < PER_BLOCK)


def coords(vmap, shape, fma=False):
    """u [3, m0, m1, m2] fp32: u_a = ((m_a0 i + m_a1 j) + m_a2 k) + m_a3 at native voxel (i, j, k)"""
    m = np.asarray(vmap, F32).reshape(3, 4)
    i = np.arange(shape[0], dtype=F32)[:, None, None]
    j = np.arange(shape[1], dtype=F32)[None, :, None]
    k = np.arange(shape[2], dtype=F32)[None, None, :]
    out = []
    with np.errstate(invalid="ignore"):
        for a in range(3):
            out.append(_coord(m[a], i, j, k, fma))
    return np.stack(out)


def _coord(m, i, j, k, fma):
    s = m[0] * i + m[1] * j
    if fma:      # fma(m_a2, k, s) + m_a3: the last product is not rounded on its own
        s = (s.astype(np.float64) + m[2].astype(np.float64) * k.astype(np.float64)).astype(F32)
    else:
        s = s + m[2] * k
    return s + m[3]


def inside(u, n, inclusive=False, no_nan_guard=False):
    """u [3, ...] inside [-0.5, n_a - 0.5) on every axis; a NaN coordinate is outside"""
    ok = np.ones(u.shape[1:], bool)
    with np.errstate(invalid="ignore"):
        for a in range(3):
            hi = F32(n[a]) - F32(0.5)
            if no_nan_guard:       # !(u < -0.5 || u >= hi): a NaN passes
                ok &= ~((u[a] < F32(-0.5)) | (u[a] >= hi))
            elif inclusive:
                ok &= (u[a] >= F32(-0.5)) & (u[a] <= hi)
            else:
                ok &= (u[a] >= F32(-0.5)) & (u[a] < hi)
    return ok


def class_scores(scores, u, axis_order=(2, 1, 0)):
    """fp32 [C, ...]: the trilinear score of every class at u [3, ...]"""
    scores = np.asarray(scores, F32)
    return np.stack([image_ref(scores[..., c], u, axis_order=axis_order) for c in range(scores.shape[3])])


def first_max(v, ge=False):
    """int64 argmax over axis 0 by the kernel's running comparison (v > top; `ge`: v >= top, the last index wins a tie)"""
    top, best = v[0].copy(), np.zeros(v.shape[1:], np.int64)
    with np.errstate(invalid="ignore"):
        for c in range(1, v.shape[0]):
            better = (v[c] >= top) if ge else (v[c] > top)
            top = np.where(better, v[c], top)
            best = np.where(better, c, best)
    return best


def labels_ref(scores, vmap, shape, axis_order=(2, 1, 0), fma=False, ge=False, inclusive=False, no_nan_guard=False):
    """-> uint8 [m0, m1, m2]: native-grid labels of the prepared-grid class scores (fp32 [n0, n1, n2, C])"""
    scores = np.asarray(scores, F32)
    u = coords(vmap, shape, fma)
    ok = inside(u, scores.shape[:3], inclusive, no_nan_guard)
    out = np.zeros(tuple(shape), np.uint8)
    if ok.any():
        out[ok] = first_max(class_scores(scores, u[:, ok], axis_order), ge).astype(np.uint8)
    return out


def confusion_ref(labels, gt, C):
    """int64 [C, C]: counts of (truth, prediction) pairs; truth labels >= C count as background"""
    g = np.asarray(gt).astype(np.int64).reshape(-1)
    g = np.where(g < C, g, 0)
    return np.bincount(g * C + np.asarray(labels).astype(np.int64).reshape(-1), minlength=C * C).reshape(C, C)
