"""fp64 reference of the fused segmenter tail and a restatement of the SIMT launchers' kernel selection (conv_simt.cu).

The plain convolutions are checked against the bilinear maps of oracle/bf16_split.py (fwd_bilinear, dgrad_bilinear,
wgrad_bilinear: ABI layouts, pnp_conv_geom geometry).  This module adds
- the tail y = conv_{kh x kw}(mirror_pad(PS_r(X))) (pnp_ps_mirror_conv_fwd) and its gradient w.r.t. X (pnp_ps_mirror_conv_bwd),
  both in fp64 on any device.  The phase shift and the SYMMETRIC pad are index maps, so every coefficient of the composition is
  non-negative and the same map applied to |X| and |w| (or |dy| and |w|) is sum|a||b| per element;
- simt_instance(): which kernel instantiation (and, for the weight gradient, how many pixel splits) each launcher picks for a
  geometry, restating dispatch_gather, the few-output condition, launch_wgrad and tail5_mode;
- the per-element tolerances TAU of the real-valued checks and the rigorous bound gamma(n)."""
import os
import re
from collections import namedtuple

import torch

from . import bf16_split as S

TailGeom = namedtuple("TailGeom", "B a b G r kh kw Cout order_b1")

U = 2.0 ** -24        # unit roundoff of fp32
NUM_SMS = 132         # PNP_NUM_SMS of common.cuh: the launchers' grid-fill rules are compiled for an H100 SXM

# Per-element tolerance of the real-valued (randn operand) checks in tests/test_simt_exact_gpu.py: |got - ref| <= TAU *
# sum|a||b|, keyed by launcher.  Each value is about 3x the worst ratio |got - ref| / sum|a||b| measured over every real-valued
# case of that file, PNP_TAIL5 = 0..3 included, on an H100 SXM (700 W).  The fp32 SIMT kernels accumulate with one FMA chain per
# output element (the weight gradient: one chain per pixel split, then fp32 atomics), so these sit one to two orders of
# magnitude below the tensor-core TAU of bf16_split.py, and far below the rigorous gamma_n.
TAU = {
    "fwd": 1.1e-6,        # measured 3.60e-7 (c16_o128_192: the 128x128 tile)
    "dgrad": 9.3e-7,      # measured 3.11e-7 (o16_c128_192)
    "wgrad": 1.9e-7,      # measured 5.07e-8 and 6.30e-8 in two runs (c64_o70_s2; the atomics make it vary)
    "tail_fwd": 1.0e-6,   # measured 3.36e-7 (k5_r8_256, generic kernel under PNP_TAIL5 = 0 / 2)
    "tail_bwd": 1.1e-6,   # measured 3.67e-7 (k5_r8_256, register-tiled 5x5 kernel)
}


def gamma(n):
    """the rigorous bound gamma_n = n u / (1 - n u) of any fp32 evaluation of a sum of n products (Higham, Thm 3.4)"""
    return n * U / (1 - n * U)


# ------------------------------------------------------------------------------------------------
# the fused tail
# ------------------------------------------------------------------------------------------------
def ps(X, r, order_b1):
    """PS_r (ops.py:23-27) with an explicit sub-pixel order: X [B, a, b, G*r*r] -> [B, a*r, b*r, G]
       order_b1 = 0 (batch >= 2): out[n, i*r + q, j*r + p, g] = X[n, i, j, g*r*r + p*r + q]
       order_b1 = 1 (batch == 1): out[n, i*r + p, j*r + q, g] = X[n, i, j, g*r*r + p*r + q]"""
    B, a, b, C = X.shape
    G = C // (r * r)
    Xv = X.reshape(B, a, b, G, r, r)
    out = Xv.permute(0, 1, 4, 2, 5, 3) if order_b1 else Xv.permute(0, 1, 5, 2, 4, 3)
    return out.reshape(B, a * r, b * r, G)


def mirror_index(n, p):
    """source index of each of the n + 2p positions of a SYMMETRIC pad by p (edge included)"""
    idx = []
    for i in range(-p, n + p):
        idx.append(-i - 1 if i < 0 else (2 * n - 1 - i if i >= n else i))
    return idx


def mirror_pad(x, ph, pw):
    """tf.pad SYMMETRIC by ph rows and pw columns on NHWC"""
    iy = torch.tensor(mirror_index(x.shape[1], ph), device=x.device)
    ix = torch.tensor(mirror_index(x.shape[2], pw), device=x.device)
    return x.index_select(1, iy).index_select(2, ix)


def tail_conv_geom(t):
    """oracle Geom of the VALID convolution over the mirror-padded map"""
    H, W = t.a * t.r, t.b * t.r
    return S.Geom(t.B, H + 2 * (t.kh // 2), W + 2 * (t.kw // 2), t.G, H, W, t.Cout, t.kh, t.kw, 1, 1, 0, 0)


def tail_fwd(X, w, t):
    """y [B, a*r, b*r, Cout] = conv VALID(mirror_pad(PS_r(X)), w); X fp64 [B, a, b, G*r*r], w fp64 HWIO [kh, kw, G, Cout]"""
    return S.fwd_bilinear(mirror_pad(ps(X, t.r, t.order_b1), t.kh // 2, t.kw // 2), w, tail_conv_geom(t))


def tail_fwd_ref(X, w, t):
    """-> (ref, sum|a||b|) of the forward tail"""
    return tail_fwd(X, w, t), tail_fwd(X.abs(), w.abs(), t)


def _tail_bwd_autograd(dy, w, t):
    X = torch.zeros(t.B, t.a, t.b, t.G * t.r * t.r, dtype=torch.float64, device=dy.device, requires_grad=True)
    with torch.enable_grad():
        tail_fwd(X, w, t).backward(dy)
    return X.grad


def tail_bwd_ref(dy, w, t):
    """-> (ref, sum|a||b|) of dX = PS^T(mirror_pad^T(conv^T(dy, w))), by fp64 autograd of tail_fwd"""
    return _tail_bwd_autograd(dy, w, t), _tail_bwd_autograd(dy.abs(), w.abs(), t)


def tail_bwd_explicit(dy, w, t, drop_fold=None):
    """the same gradient written out: transposed convolution, fold of the padded border, inverse phase shift.  drop_fold =
    'top' / 'bottom' / 'left' / 'right' leaves the mirrored rows / columns of that edge unfolded (a negative control)"""
    g = tail_conv_geom(t)
    H, W, ph, pw = t.a * t.r, t.b * t.r, t.kh // 2, t.kw // 2
    dxp = S.dgrad_bilinear(dy, w, g)
    iy, ix = mirror_index(H, ph), mirror_index(W, pw)
    keep_y = [not ((drop_fold == "top" and i < ph) or (drop_fold == "bottom" and i >= H + ph)) for i in range(H + 2 * ph)]
    keep_x = [not ((drop_fold == "left" and i < pw) or (drop_fold == "right" and i >= W + pw)) for i in range(W + 2 * pw)]
    dxp = dxp * torch.tensor(keep_y, dtype=dxp.dtype, device=dxp.device).view(1, -1, 1, 1)
    dxp = dxp * torch.tensor(keep_x, dtype=dxp.dtype, device=dxp.device).view(1, 1, -1, 1)
    rows = torch.zeros(t.B, H, W + 2 * pw, t.G, dtype=dxp.dtype, device=dxp.device)
    rows.index_add_(1, torch.tensor(iy, device=dxp.device), dxp)
    dflat = torch.zeros(t.B, H, W, t.G, dtype=dxp.dtype, device=dxp.device)
    dflat.index_add_(2, torch.tensor(ix, device=dxp.device), rows)
    Xv = dflat.reshape(t.B, t.a, t.r, t.b, t.r, t.G)          # [n, i, row offset, j, col offset, g]
    if t.order_b1:
        out = Xv.permute(0, 1, 3, 5, 2, 4)                     # sub = (row offset) * r + (col offset)
    else:
        out = Xv.permute(0, 1, 3, 5, 4, 2)                     # sub = (col offset) * r + (row offset)
    return out.reshape(t.B, t.a, t.b, t.G * t.r * t.r)


# ------------------------------------------------------------------------------------------------
# kernel selection of conv_simt.cu
# ------------------------------------------------------------------------------------------------
_INST = re.compile(r"((?:conv_gather|conv_wgrad|conv_few_out|ps_mirror_conv5?(?:_bwd)?)_kernel)<([^<>]*)>")


def instances_in(text):
    """set of 'name<args>' (no blanks) of the SIMT kernel instantiations named in `text` (nm -C output, profiler names)"""
    return {"%s<%s>" % (m.group(1), m.group(2).replace(" ", "")) for m in _INST.finditer(text)}


def _cdiv(a, b):
    return -(-a // b)


def _gather(tile, tr):
    return "conv_gather_kernel<%s,%s>" % (",".join(str(v) for v in tile), "true" if tr else "false")


def _dispatch_gather(IC, OC, M, tr):
    """dispatch_gather<TR>: IC = channels gathered (fwd Cin, dgrad Cout), OC = channels produced, M = rows produced"""
    if IC % 4:
        if OC <= 8:
            return _gather((1024, 8, 8, 4, 8, 1), tr)
        if OC <= 16:
            return _gather((256, 16, 16, 4, 4, 1), tr)
        return _gather((128, 64, 16, 8, 4, 1), tr)
    k16 = IC % 16 == 0
    bk = 16 if k16 else 8
    if OC <= 8:
        return _gather((1024, 8, 8, 4, 8, 4), tr)
    if OC <= 16:
        return _gather((256, 16, bk, 4, 4, 4), tr)
    if OC <= 32:
        return _gather((256, 32, bk, 8, 4, 4), tr)
    if OC <= 64 or _cdiv(M, 128) * _cdiv(OC, 128) < 2 * NUM_SMS:
        return _gather((128, 64, bk, 8, 4, 4), tr)
    return _gather((128, 128, bk, 8, 8, 4), tr)


def gather_tile(kernel):
    """'conv_gather_kernel<BM,BN,BK,...>' -> (BM, BN, BK)"""
    v = kernel[kernel.index("<") + 1:-1].split(",")
    return int(v[0]), int(v[1]), int(v[2])


def dgrad_phase_rows(g, kernel):
    """rows per phase of the phase-major data-gradient row order launch_gather picks (0 = plain row order)"""
    BM, _, BK = gather_tile(kernel)
    s = g.stride
    if s > 1 and g.H % s == 0 and g.W % s == 0 and g.Cout % BK == 0:
        pr = g.B * (g.H // s) * (g.W // s)
        if pr % BM == 0:
            return pr
    return 0


def wgrad_splits(g, BKK, BN, BR):
    """launch_wgrad: pixel splits of the weight gradient (about 6 CTAs per SM, at least 4 reduction blocks per CTA)"""
    M, KK = g.B * g.Ho * g.Wo, g.kh * g.kw * g.Cin
    tiles = _cdiv(KK, BKK) * _cdiv(g.Cout, BN)
    want = (NUM_SMS * 6 + tiles - 1) // tiles
    splits = min(max(want, 1), _cdiv(M, BR * 4))
    splits = min(max(splits, 1), 65535)
    mps = _cdiv(_cdiv(M, splits), BR) * BR
    return _cdiv(M, mps)


def tail5_mode():
    """PNP_TAIL5 as tail5_mode() reads it (atoi, default 3)"""
    e = os.environ.get("PNP_TAIL5")
    if e is None:
        return 3
    m = re.match(r"\s*([+-]?\d+)", e)
    return int(m.group(1)) if m else 0


def simt_instance(launcher, g, drop=False, accumulate=0):
    """-> (kernel instantiation 'name<args>', pixel splits for the weight gradient else None) of one launch.
    launcher: 'fwd' / 'dgrad' / 'wgrad' with an oracle Geom (the FORWARD geometry), or 'tail_fwd' / 'tail_bwd' with a
    TailGeom; drop: the forward runs with dropout"""
    if launcher == "fwd":
        if (g.Cout in (5, 8) and g.Cin % 8 == 0 and g.stride == 1 and g.dil == 1 and g.kh <= 5 and g.kw <= 5 and not accumulate
                and not drop and g.B <= 65535):
            return "conv_few_out_kernel<%d>" % g.Cout, None
        return _dispatch_gather(g.Cin, g.Cout, g.B * g.Ho * g.Wo, False), None
    if launcher == "dgrad":
        return _dispatch_gather(g.Cout, g.Cin, g.B * g.H * g.W, True), None
    if launcher == "wgrad":
        if g.Cin % 4:
            cfg = (64, 16, 16, 4, 1, 1) if g.Cout <= 16 else (64, 64, 16, 4, 4, 1)
        elif g.Cout <= 8:
            cfg = (128, 8, 16, 4, 1, 4)
        elif g.Cout <= 16:
            cfg = (64, 16, 16, 4, 1, 4)
        elif g.Cout <= 32:
            cfg = (64, 32, 16, 4, 2, 4)
        elif g.Cout <= 64 or g.kh * g.kw * g.Cin < 128:
            cfg = (64, 64, 16, 4, 4, 4)
        else:
            cfg = (128, 128, 16, 8, 8, 4)
        return "conv_wgrad_kernel<%s>" % ",".join(str(v) for v in cfg), wgrad_splits(g, cfg[0], cfg[1], cfg[2])
    if launcher in ("tail_fwd", "tail_bwd"):
        bit = 1 if launcher == "tail_fwd" else 2
        suffix = "" if launcher == "tail_fwd" else "_bwd"
        if g.kh == 5 and g.kw == 5 and g.Cout in (5, 8) and tail5_mode() & bit:
            return "ps_mirror_conv5%s_kernel<%d>" % (suffix, g.Cout), None
        return "ps_mirror_conv%s_kernel<%d>" % (suffix, g.Cout), None
    raise ValueError(launcher)
