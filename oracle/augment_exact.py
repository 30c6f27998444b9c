"""A numpy float32 restatement of the augmentation kernels of csrc/resample.cu (include/pnp_b200.h, "data augmentation"):
pnp_smooth_noise_field and pnp_resample_planes_aug, in the kernels' operation order.  Test-only.

* uniforms: element e = ((b K + k) H + r) W + c takes word e & 3 of Philox4x32-10 block e >> 2 of (seed, stream) (oracle/philox.py)
  and maps it to fl32(x >> 8) 2^-23 - 1, exact in fp32.
* smoothing: pass 1 along c, then pass 2 along r; s = sum_{t=-R..R} w_t x[i + t] with 0 outside the plane, from +0 in increasing t,
  every product and sum one fp32 numpy operation (rounded on its own); the output is min(max(amp s, lo), hi).
* resampling: the coordinates of oracle/resample_exact.py at the displaced pixel (r + d_r, c + d_c), then its trilinear image and
  nearest-voxel labels; the image becomes (a ((1 + gain) v)) + b.  A field given as None skips its operations, as in the kernel.

gaussian_taps is restated here from scipy's definition rather than imported from the package."""
import numpy as np

from oracle import philox
from oracle import resample_exact as R

F32 = np.float32
NF_MAX_R = 128                     # PNP_NF_MAX_R


def gaussian_taps(sigma):
    """scipy.ndimage's Gaussian kernel at truncate 4 (R = int(4 sigma + 0.5)), normalised in fp64, rounded to fp32 once"""
    r = int(4.0 * sigma + 0.5)
    x = np.arange(-r, r + 1, dtype=np.float64)
    phi = np.exp(-0.5 / (sigma * sigma) * x ** 2)
    return (phi / phi.sum()).astype(F32)


def uniforms(seed, stream, B, K, H, W):
    """fp32 [B, K, H, W] on [-1, 1)"""
    n = B * K * H * W
    words = philox.blocks(seed, stream, (n + 3) // 4).reshape(-1)[:n]        # word w of block b sits at 4 b + w = e
    return ((words >> np.uint32(8)).astype(F32) * F32(2.0 ** -23) - F32(1)).reshape(B, K, H, W)


def smooth_pass(x, taps, axis):
    """one pass along `axis` of x (fp32): s_i = sum_t taps[t + R] x[i + t], zero outside, from +0 in increasing t"""
    x = np.asarray(x, F32)
    taps = np.asarray(taps, F32)
    r = (len(taps) - 1) // 2
    n = x.shape[axis]
    pad = [(0, 0)] * x.ndim
    pad[axis] = (r, r)
    xp = np.pad(x, pad)
    s = np.zeros_like(x)
    for t in range(2 * r + 1):
        sl = [slice(None)] * x.ndim
        sl[axis] = slice(t, t + n)
        s = s + taps[t] * xp[tuple(sl)]
    return s


def smooth(x, taps):
    """pass 1 along c (the last axis), then pass 2 along r"""
    return smooth_pass(smooth_pass(x, taps, -1), taps, -2)


def noise_field(seed, stream, B, K, H, W, taps, amp, lo, hi):
    """pnp_smooth_noise_field: fp32 [B, K, H, W]"""
    s = smooth(uniforms(seed, stream, B, K, H, W), taps)
    return np.fmin(np.fmax(F32(amp) * s, F32(lo)), F32(hi))


def coords_aug(mats, B, H, W, C, disp=None):
    """u [3, B, H, W, C] fp32 at the displaced pixel: u_i = (m_i0 r' + m_i1 c') + m_i2, r' = r + d_r, c' = c + d_c"""
    m = np.asarray(mats, F32).reshape(B, C, 3, 3)
    r = np.broadcast_to(np.arange(H, dtype=F32)[None, :, None], (B, H, W))
    c = np.broadcast_to(np.arange(W, dtype=F32)[None, None, :], (B, H, W))
    if disp is not None:
        d = np.asarray(disp, F32)
        r, c = r + d[:, 0], c + d[:, 1]
    r, c = r[..., None], c[..., None]
    return np.stack([(m[:, :, i, 0].reshape(B, 1, 1, C) * r + m[:, :, i, 1].reshape(B, 1, 1, C) * c) + m[:, :, i, 2].reshape(B, 1, 1, C)
                     for i in range(3)])


def resample_aug_ref(vol, cls, mats, B, H, W, C, label_planes, img=True, disp=None, gain=None, ab=None):
    """pnp_resample_planes_aug -> (img fp32 [B, H, W, C] or None, lab int64 as resample_exact.resample_ref returns it or None)"""
    u = coords_aug(mats, B, H, W, C, disp)
    out_img = None
    if img:
        v = R.image_ref(vol, u)
        if gain is not None:
            v = (F32(1) + np.asarray(gain, F32))[..., None] * v
        if ab is not None:
            ab = np.asarray(ab, F32)
            v = ab[:, 0].reshape(B, 1, 1, 1) * v + ab[:, 1].reshape(B, 1, 1, 1)
        out_img = v.astype(F32)
    out_lab = None
    if label_planes == 1:
        out_lab = R.label_ref(cls, u[:, :, :, :, C // 2])
    elif label_planes:
        out_lab = R.label_ref(cls, u)
    return out_img, out_lab


def smooth_error_bound(taps):
    """a-priori bound on |two fp32 passes - the fp64 Gaussian of the same uniforms| (|x| <= 1, fp64 weights w summing to 1).
    A pass of n = 2R + 1 rounded products and n - 1 rounded sums of inputs with error e_in (exact values |x| <= 1, so the exact
    pass-1 values are <= 1 as well): |out - sum w x| <= e_in + (g_n (1 + u) + u)(1 + e_in), where u = 2^-24 and g_n = n u / (1 - n u):
    the recursive-sum bound g_n sum |w~ x^|, the fp32 weights' rounding u |w|, and sum |w~| <= 1 + u."""
    u = 2.0 ** -24
    n = len(taps)
    g = n * u / (1 - n * u)
    k = g * (1 + u) + u
    e1 = k
    return e1 + k * (1 + e1)
