"""A numpy float32 restatement of pnp_resample_planes (csrc/resample.cu, include/pnp_b200.h "data preparation") in the kernel's
operation order, plus its launch configuration.  Test-only.

Every fp32 operation of the kernel is one numpy float32 operation here, rounded on its own: u_i = (m_i0 r + m_i1 c) + m_i2, the
clamp, floor, f = x - i0 and the three lerp levels a + f (b - a) along axes 2, 1, 0; labels floor(u + 0.5) with class 0 outside
[-0.5, n - 0.5).  Each reference takes the flag of one plausible kernel bug (axis_order, fma, half_even, no_clamp):
tests/test_resample_exact_cpu.py checks that each one changes some output."""
from collections import namedtuple

import numpy as np

from oracle.elementwise_exact import NUM_SMS, grid_for

F32 = np.float32
CAP = NUM_SMS * 64
THREADS = 256
PER_BLOCK = 256 * 4
Launch = namedtuple("Launch", "grid capped iters single_partial")


def launch(B, H, W, C, img=True, label_planes=1):
    """the launcher's grid_for(B*H*W*Cw, 1024) grid-stride launch; Cw = 1 when only the middle label plane is written"""
    cw = C if (img or label_planes != 1) else 1
    items = B * H * W * cw
    g = grid_for(items, PER_BLOCK)
    return Launch(g, -(-items // PER_BLOCK) > CAP, -(-items // (g * THREADS)), g == 1 and items < PER_BLOCK)


def coords(mats, B, H, W, C, fma=False):
    """u [3, B, H, W, C] fp32: u_i = (m_i0 r + m_i1 c) + m_i2 of plane b*C + k at pixel (r, c)"""
    m = np.asarray(mats, F32).reshape(B, C, 3, 3)
    r = np.arange(H, dtype=F32)[None, :, None, None]
    c = np.arange(W, dtype=F32)[None, None, :, None]
    out = []
    for i in range(3):
        m0, m1, m2 = (m[:, :, i, j].reshape(B, 1, 1, C) for j in range(3))
        if fma:      # fma(m0, r, m1 c) + m2: the first product is not rounded on its own
            out.append((m0.astype(np.float64) * r + (m1 * c).astype(np.float64)).astype(F32) + m2)
        else:
            out.append((m0 * r + m1 * c) + m2)
    return np.stack(out)


def _lerp(a, b, f, fma=False):
    if fma:
        return (a.astype(np.float64) + f.astype(np.float64) * (b - a).astype(np.float64)).astype(F32)
    return a + f * (b - a)


def _taps(u, n, no_clamp=False):
    x = u if no_clamp else np.fmin(np.fmax(u, F32(0)), F32(n - 1))
    fl = np.floor(x)
    i0 = np.clip(fl, 0, n - 1).astype(np.int64)
    return i0, np.minimum(i0 + 1, n - 1), (x - fl).astype(F32)


def image_ref(vol, u, axis_order=(2, 1, 0), fma=False, no_clamp=False):
    """trilinear interpolation of vol (fp32 [n0, n1, n2]) at u [3, ...]: lerp along axis_order[0], then [1], then [2]"""
    vol = np.asarray(vol, F32)
    first, second, third = axis_order
    with np.errstate(invalid="ignore", over="ignore"):
        taps = [_taps(u[a], vol.shape[a], no_clamp) for a in range(3)]

        def corner(s1, s2, s3):
            """vol at tap s1 (0: i0, 1: i1) along `first`, s2 along `second`, s3 along `third`"""
            s = [0, 0, 0]
            s[first], s[second], s[third] = s1, s2, s3
            return vol[taps[0][s[0]], taps[1][s[1]], taps[2][s[2]]]

        lerp1 = {(s2, s3): _lerp(corner(0, s2, s3), corner(1, s2, s3), taps[first][2], fma) for s2 in (0, 1) for s3 in (0, 1)}
        lerp2 = [_lerp(lerp1[(0, s3)], lerp1[(1, s3)], taps[second][2], fma) for s3 in (0, 1)]
        return _lerp(lerp2[0], lerp2[1], taps[third][2], fma)


def label_ref(cls, u, half_even=False):
    """nearest voxel floor(u + 0.5) of cls (uint8 [n0, n1, n2]) at u [3, ...]; class 0 outside [-0.5, n - 0.5) or at NaN"""
    cls = np.asarray(cls)
    inside = np.ones(u.shape[1:], bool)
    idx = []
    with np.errstate(invalid="ignore"):
        for a in range(3):
            n = cls.shape[a]
            inside &= (u[a] >= F32(-0.5)) & (u[a] < F32(n) - F32(0.5))
            j = np.rint(u[a]) if half_even else np.floor(u[a] + F32(0.5))
            idx.append(np.clip(np.where(inside, j, 0), 0, n - 1).astype(np.int64))
    return np.where(inside, cls[idx[0], idx[1], idx[2]], 0).astype(np.int64)


def resample_ref(vol, cls, mats, B, H, W, C, label_planes, img=True, **bug):
    """-> (img fp32 [B, H, W, C] or None, lab int64 [B, H, W] (label_planes 1), [B, H, W, C] (label_planes C) or None)"""
    img_bug = {k: v for k, v in bug.items() if k in ("axis_order", "fma", "no_clamp")}
    u = coords(mats, B, H, W, C, fma=bug.get("fma", False))
    out_img = image_ref(vol, u, **img_bug) if img else None
    out_lab = None
    if label_planes:
        if label_planes == 1:
            out_lab = label_ref(cls, u[:, :, :, :, C // 2], bug.get("half_even", False))
        else:
            out_lab = label_ref(cls, u, bug.get("half_even", False))
    return out_img, out_lab
