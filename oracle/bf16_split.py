"""Split-aware fp64 reference of the tensor-core convolutions (conv_tc.cu).

The wgmma kernels multiply bf16 operand planes: every fp32 operand x is stored as hi = rn_bf16(x), lo = rn_bf16(x - hi) (the
fp32 subtraction is exact), and nterms = 3 issues hi*hi + hi*lo + lo*hi, nterms = 1 hi*hi.  Those products are exact in fp32,
so the only difference between a correct kernel and the fp64 value of exactly these terms is the order of its fp32
accumulation.  Checking |got - ref| <= tau * sum|a||b| per element, with ref and the conditioning sum|a||b| from here, needs
no allowance for the operand rounding: for nterms 1 it is two to four orders of magnitude tighter than a max-normalised bound
against the true convolution of the fp32 operands, and for every nterms it holds at each element, small ones included.

Everything here is plain torch in fp64 and works on any device; the operand layouts are those of include/pnp_b200.h:
activations NHWC, forward weight planes [tap][Cout][CinP], data-gradient weight planes [tap][Cin][Cout], HWIO fp32 weights.
The geometry is pnp_conv_geom (stride, dilation, pad_t / pad_l, zero padding; SYMMETRIC = already mirror-padded input)."""
from collections import namedtuple

import torch

Geom = namedtuple("Geom", "B H W Cin Ho Wo Cout kh kw stride dil pad_t pad_l")

# Per-element tolerance of the tensor-core launchers against the split reference: |got - ref| <= TAU * sum|a||b|, keyed by
# (launcher, nterms).  Each value is about 3x the worst ratio |got - ref| / sum|a||b| measured over every case of
# tests/test_tc_split_exact_gpu.py (default and alternative switches) on an H100 SXM (700 W); the worst case is always the
# deepest reduction, group_10 at real width (fwd K = 4608, dgrad K = 23040, wgrad K = 2048 pixels).  The ratio grows with K:
# the tensor cores' fp32 accumulation is not a sequence of round-to-nearest additions.
TAU = {
    ("fwd", 3): 6.7e-6,      # measured 2.26e-6
    ("fwd", 1): 2.1e-6,      # measured 7.72e-7
    ("dgrad", 3): 1.4e-5,    # measured 4.45e-6
    ("dgrad", 1): 4.4e-6,    # measured 1.45e-6
    ("wgrad", 3): 4.5e-6,    # measured 1.48e-6
    ("wgrad", 1): 1.5e-6,    # measured 5.01e-7
}


# ------------------------------------------------------------------------------------------------
# the split
# ------------------------------------------------------------------------------------------------
def split(x):
    """fp32 tensor -> (hi, lo) torch.bfloat16 tensors, bit for bit what the device's split1 / split_pair write: round to nearest
    even twice, denormals kept (torch's float32 -> bfloat16 conversion is RNE and does not flush)"""
    x = x.to(torch.float32)
    hi = x.to(torch.bfloat16)
    lo = (x - hi.to(torch.float32)).to(torch.bfloat16)
    return hi, lo


def bits(p):
    """bf16 tensor (or an int16 / uint16 view of one) -> int32 tensor of its 16-bit patterns"""
    if p.dtype == torch.bfloat16:
        p = p.view(torch.int16)
    return p.to(torch.int32) & 0xFFFF


def planes_equal(got, ref):
    """bf16 planes equal bit for bit, except that any NaN matches any NaN (the device and torch use different NaN payloads)"""
    g, r = bits(got), bits(ref)
    nan_g = ((g & 0x7F80) == 0x7F80) & ((g & 0x7F) != 0)
    nan_r = ((r & 0x7F80) == 0x7F80) & ((r & 0x7F) != 0)
    return bool(torch.all((g == r) | (nan_g & nan_r)))


def to64(p):
    return p.to(torch.float64)


def fwd_weight_planes(hi, lo, kh, kw, Cin, Cout, cin_pad=0):
    """[tap][Cout][CinP] forward weight planes -> fp64 HWIO (hi, lo) [kh, kw, Cin, Cout] (the zero channels >= Cin dropped)"""
    cp = max(Cin, cin_pad)

    def f(p):
        return None if p is None else to64(p).reshape(kh, kw, Cout, cp)[..., :Cin].permute(0, 1, 3, 2).contiguous()
    return f(hi), f(lo)


def dgrad_weight_planes(hi, lo, kh, kw, Cin, Cout):
    """[tap][Cin][Cout] data-gradient weight planes -> fp64 HWIO (hi, lo) [kh, kw, Cin, Cout]"""
    def f(p):
        return None if p is None else to64(p).reshape(kh, kw, Cin, Cout)
    return f(hi), f(lo)


# ------------------------------------------------------------------------------------------------
# the three bilinear maps, tap by tap (so a test can drop or move single taps)
# ------------------------------------------------------------------------------------------------
def _range(off, s, n_in, n_out):
    """output indices o in [lo, hi) with 0 <= o*s + off < n_in"""
    lo = max(0, -(off // s) if off < 0 else 0)
    while lo < n_out and lo * s + off < 0:
        lo += 1
    hi = lo
    while hi < n_out and hi * s + off < n_in:
        hi += 1
    return lo, hi


def tap_offsets(g, taps=None):
    """[(tap index, oy, ox)] input offsets of the forward taps: input pixel = output pixel * stride + (oy, ox)"""
    out = []
    for ky in range(g.kh):
        for kx in range(g.kw):
            t = ky * g.kw + kx
            if taps is None or t in taps:
                out.append((t, ky * g.dil - g.pad_t, kx * g.dil - g.pad_l))
    return out


def fwd_bilinear(x, w, g, taps=None, shift=None):
    """y[b,o,p,:] = sum_tap x[b, o*s + oy, p*s + ox, :] @ w[tap]; x NHWC fp64, w HWIO fp64.  shift = {tap: (dy, dx)} moves the
    input offset of single taps (negative controls)"""
    B, s = x.shape[0], g.stride
    y = torch.zeros(B, g.Ho, g.Wo, w.shape[3], dtype=torch.float64, device=x.device)
    wf = w.reshape(g.kh * g.kw, w.shape[2], w.shape[3])
    for t, oy, ox in tap_offsets(g, taps):
        if shift and t in shift:
            oy, ox = oy + shift[t][0], ox + shift[t][1]
        y0, y1 = _range(oy, s, x.shape[1], g.Ho)
        x0, x1 = _range(ox, s, x.shape[2], g.Wo)
        if y0 >= y1 or x0 >= x1:
            continue
        xs = x[:, y0 * s + oy:(y1 - 1) * s + oy + 1:s, x0 * s + ox:(x1 - 1) * s + ox + 1:s, :]
        y[:, y0:y1, x0:x1, :] += xs @ wf[t]
    return y


def dgrad_bilinear(dy, w, g, taps=None):
    """dx[b, o*s + oy, p*s + ox, :] += dy[b,o,p,:] @ w[tap]^T over the forward taps; dy NHWC fp64, w HWIO fp64"""
    B, s = dy.shape[0], g.stride
    dx = torch.zeros(B, g.H, g.W, w.shape[2], dtype=torch.float64, device=dy.device)
    wf = w.reshape(g.kh * g.kw, w.shape[2], w.shape[3])
    for t, oy, ox in tap_offsets(g, taps):
        y0, y1 = _range(oy, s, g.H, dy.shape[1])
        x0, x1 = _range(ox, s, g.W, dy.shape[2])
        if y0 >= y1 or x0 >= x1:
            continue
        dx[:, y0 * s + oy:(y1 - 1) * s + oy + 1:s, x0 * s + ox:(x1 - 1) * s + ox + 1:s, :] += dy[:, y0:y1, x0:x1, :] @ wf[t].T
    return dx


def wgrad_bilinear(x, dy, g, taps=None):
    """dw[tap] = sum_pixels x[b, o*s + oy, p*s + ox, :]^T dy[b,o,p,:]  -> HWIO fp64 [kh, kw, Cin, Cout]"""
    s = g.stride
    dw = torch.zeros(g.kh * g.kw, x.shape[3], dy.shape[3], dtype=torch.float64, device=x.device)
    for t, oy, ox in tap_offsets(g, taps):
        y0, y1 = _range(oy, s, x.shape[1], dy.shape[1])
        x0, x1 = _range(ox, s, x.shape[2], dy.shape[2])
        if y0 >= y1 or x0 >= x1:
            continue
        xs = x[:, y0 * s + oy:(y1 - 1) * s + oy + 1:s, x0 * s + ox:(x1 - 1) * s + ox + 1:s, :].reshape(-1, x.shape[3])
        dw[t] = xs.T @ dy[:, y0:y1, x0:x1, :].reshape(-1, dy.shape[3])
    return dw.reshape(g.kh, g.kw, x.shape[3], dy.shape[3])


# ------------------------------------------------------------------------------------------------
# split references: the fp64 value of exactly the terms the kernel multiplies, and sum|a||b|
# ------------------------------------------------------------------------------------------------
def split_terms(bil, a_hi, a_lo, b_hi, b_lo, nterms, cross=True):
    """-> (ref, cond).  nterms 3: hi*hi + hi*lo + lo*hi = bil(a_hi + a_lo, b_hi + b_lo) - bil(a_lo, b_lo); nterms 1: hi*hi.
    cross=False drops the a_lo*b_hi term (a negative control).  cond = bil(|a|, |b|) of the operands the kernel sees."""
    if nterms == 1:
        return bil(a_hi, b_hi), bil(a_hi.abs(), b_hi.abs())
    a, b = a_hi + a_lo, b_hi + b_lo
    ref = bil(a, b) - bil(a_lo, b_lo)
    if not cross:
        ref = ref - bil(a_lo, b_hi)
    return ref, bil(a.abs(), b.abs())


def fwd_ref(x_hi, x_lo, w_hi, w_lo, g, nterms, **kw):
    return split_terms(lambda a, b: fwd_bilinear(a, b, g, **kw), x_hi, x_lo, w_hi, w_lo, nterms)


def dgrad_ref(dy_hi, dy_lo, w_hi, w_lo, g, nterms, **kw):
    return split_terms(lambda a, b: dgrad_bilinear(a, b, g, **kw), dy_hi, dy_lo, w_hi, w_lo, nterms)


def wgrad_ref(x_hi, x_lo, dy_hi, dy_lo, g, nterms, **kw):
    return split_terms(lambda a, b: wgrad_bilinear(a, b, g, **kw), x_hi, x_lo, dy_hi, dy_lo, nterms)


def dgrad_phase_taps(g, py, px):
    """forward taps that feed the dx pixels (i, j) with i % s == py, j % s == px (one phase of a strided data gradient)"""
    s = g.stride
    return {t for t, oy, ox in tap_offsets(g) if (py - oy) % s == 0 and (px - ox) % s == 0}


def worst_ratio(got, ref, cond, slack=None):
    """max over elements of (|got - ref| - slack)+ / cond: the smallest tau that violations() accepts (inf if an element with
    cond == 0 misses by more than its slack, or got is not finite)"""
    got = got.to(torch.float64)
    if not bool(torch.isfinite(got).all()):
        return float("inf")
    err = (got - ref).abs()
    if slack is not None:
        err = (err - slack).clamp_min(0)
    if bool(((cond == 0) & (err != 0)).any()):
        return float("inf")
    return float((err / torch.where(cond > 0, cond, torch.ones_like(cond))).max())


def violations(got, ref, cond, tau, slack=None):
    """number of elements with |got - ref| > tau * cond + slack"""
    err = (got.to(torch.float64) - ref).abs()
    bound = tau * cond + (0 if slack is None else slack)
    return int((~(err <= bound)).sum())
