"""Host-side operators of the H100 hot path: thin torch.autograd.Function wrappers whose forward and
backward are sequences of launches into libpnp_b200.so (include/pnp_b200.h).  PyTorch supplies device
memory, the stream and the autograd tape; every arithmetic kernel is ours.  NHWC fp32 activations,
HWIO weights, exactly like the reference (layers.py / ops.py).

Trainable variables receive their gradients by direct accumulation into `var.grad` (normally a view
of a flat gradient arena, see optim.py); the Functions return None for them so autograd adds nothing.
"""
import ctypes
import math
import os

import numpy as np
import torch

from . import _C
from . import runtime as rt
from ._C import call, ptr, ConvGeom, DropCfg

ACT_NONE, ACT_RELU, ACT_LRELU = 0, 1, 2

# fuse BN batch statistics into the wgmma conv epilogue (otherwise a separate pnp_bn_stats pass)
FUSE_BN_STATS = True
# emit the bf16 operand planes from the BN-apply / BN-backward kernels instead of a separate split pass
FUSE_SPLIT = os.environ.get("PNP_FUSE_SPLIT", "1") != "0"
# bench.py sets this to a list to time every wgmma launch with CUDA events: (start, end, flops, tag)
PROFILE = None
# debugging aid: callable(sv, dy, g, dz, dx) invoked at the end of every layer_backward
DEBUG_HOOK = None


def _tc_launch(tag, flops, name, *args):
    if PROFILE is None:
        call(name, *args)
        return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    call(name, *args)
    e1.record()
    kern = "simt"
    if name in ("pnp_conv2d_tc_fwd", "pnp_conv2d_tc_fwd_fused", "pnp_conv2d_tc_dgrad"):
        n_, k_, s_ = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
        _C.lib.pnp_tc_last_config(ctypes.byref(n_), ctypes.byref(k_), ctypes.byref(s_))
        kern = "conv_tc_kernel<%d, %d, %d>" % (n_.value, 1 if _tc_mode() == 1 else 3, k_.value)
    elif name == "pnp_conv2d_tc_wgrad":
        kern = "conv_wgrad_tc_kernel"
    PROFILE.append((e0, e1, flops, tag, kern))


def same_pad(n, k, s, d=1):
    """TF 'SAME' (before, after) padding -- asymmetric for strided convs (SURVEY App. B.1)."""
    out = -(-n // s)
    total = max((out - 1) * s + (k - 1) * d + 1 - n, 0)
    return total // 2, total - total // 2


def _zeros_f64(n, dev):
    """zeroed fp64 accumulators: a slice of the per-step scratch pool (ONE memset per step, runtime.Scratch) when it has room,
    else an individual allocation + fill"""
    t = rt.scratch.take(n, dev)
    if t is not None:
        return t
    t = torch.empty(n, dtype=torch.float64, device=dev)
    call("pnp_fill", ptr(t), 0.0, 2 * n, rt.stream())
    return t


def _drop_cfg(keep_prob):
    """-> (ctypes DropCfg or None, (stream_id, keep) or None)"""
    if keep_prob is None or keep_prob >= 1.0:
        return None, None
    sid = rt.rng.next_stream()
    return DropCfg(rt.rng.seed_ptr(), sid, float(keep_prob)), (sid, float(keep_prob))


def _drop_from(info):
    if info is None:
        return None
    return DropCfg(rt.rng.seed_ptr(), info[0], info[1])


def _byref(x):
    return None if x is None else ctypes.byref(x)


# ------------------------------------------------------------------------------------------------
# low-level convolution launches
# ------------------------------------------------------------------------------------------------
def _tc_mode():
    b = rt.conv_backend()
    if b == "simt" or not rt.tc_available():
        return 0
    return 1 if b == "tc1" else 3


# wgmma wgrad can be switched off separately (PNP_TC_WGRAD=0) for A/B measurements
TC_WGRAD = os.environ.get("PNP_TC_WGRAD", "1") != "0"
TC_PAD32 = os.environ.get("PNP_TC_PAD32", "0") == "1"
_tc_declined = set()     # (kind, geometry) the wgmma launchers returned PNP_ERR_UNSUPPORTED for -> general SIMT kernel
_tc_proven = set()       # (kind, geometry) that HAVE run on the tensor-core path: only for those may a producer drop the fp32 copy


def _gkey(kind, g):
    return (kind, g.B, g.H, g.W, g.Cin, g.Ho, g.Wo, g.Cout, g.kh, g.kw, g.stride, g.dil, g.pad_t, g.pad_l)


def _cin_pad(g):
    """channel count of the (zero padded) operand planes: Cin = 32 layers (cls_1 res a) use the 64-channel K chunk"""
    if g.Cin % 64 == 0 or (g.Cin == 32 and TC_K32):
        return g.Cin
    return ((g.Cin + 63) // 64) * 64


def _tc_ch(c):
    """channel counts the wgmma kernels tile natively: multiples of 64 (128-byte swizzle rows), 32 (64-byte) or 16 (32-byte)"""
    return c % 64 == 0 or c == 32 or (c == 16 and TC_K16)


# the native 32-channel wgmma tiles (K block of 32 / N tile of 32); PNP_TC_K32=0 sends those layers back to the SIMT kernel
TC_K32 = os.environ.get("PNP_TC_K32", "1") != "0"
# 16-channel layers (g1/g2, mask critic): 16-wide K blocks (SWIZZLE_32B).  One TMA instruction moves only 4 KB there, so the
# kernel is TMA-issue bound and roughly at par with the SIMT kernel (r1p: fwd 256x256 16->16 144 us vs 131 us, dgrad 121 vs 141)
TC_K16 = os.environ.get("PNP_TC_K16", "1") != "0"


def _tc_candidate(kind, g):
    if g.kh * g.kw > 25 or _gkey(kind, g) in _tc_declined:
        return False
    if g.Cin % 64 == 0 and g.Cout % 64 == 0:
        # (measured r1e: even the tiny stride-4 data gradients -- cls_5_3, m_cls_4, s*s latency-bound phase launches -- are
        #  2.5x faster here than on the general kernel, whose transposed gather multiplies 15/16 zeros)
        return True
    if kind == "wgrad":
        # the weight-gradient GEMM has M = Cin: a 32-channel layer packs four taps into the 128-row MMA tile (native 32-channel
        # planes); the older zero-padded-plane variant measured slower than the SIMT kernel (r1e) and stays opt-in
        if g.Cout % 64 != 0:
            return False
        return (TC_K32 and g.Cin == 32) or (TC_PAD32 and g.Cin % 32 == 0 and g.Cin >= 32)
    return TC_K32 and _tc_ch(g.Cin) and _tc_ch(g.Cout)


def _new_planes(shape, dev, nterms):
    hi = torch.empty(shape, dtype=torch.bfloat16, device=dev)
    lo = torch.empty(shape, dtype=torch.bfloat16, device=dev) if nterms == 3 else None
    return hi, lo


class _PlanesOnly:
    """stand-in for a tensor whose fp32 copy was never written: it only carries the bf16 operand planes.  Any consumer that
    asks for its address (a SIMT kernel) fails loudly instead of reading garbage."""

    def __init__(self, shape, dev):
        self.shape, self.device = tuple(shape), dev

    def data_ptr(self):
        raise RuntimeError("this gradient exists only as bf16 operand planes; its fp32 copy was elided")

    def contiguous(self):
        return self

    def numel(self):
        n = 1
        for d in self.shape:
            n *= d
        return n


def _planes_of(x, nterms):
    """bf16 operand planes of x: emitted by the producing kernel when available, else one split pass"""
    p = getattr(x, "_pnp_planes", None)
    if p is not None and p[0] == nterms:
        return p[1], p[2]
    return split_bf16(x, nterms)


def _want_planes(C):
    """producers emit planes for tensors a wgmma convolution is likely to consume (64-multiple channel counts)"""
    nt = _tc_mode()
    return nt if (nt and FUSE_SPLIT and (C % 64 == 0 or (C == 32 and TC_K32) or (C == 16 and TC_K32 and TC_K16))) else 0


def split_bf16(x, nterms):
    hi = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    lo = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if nterms == 3 else None
    call("pnp_split_bf16", ptr(x), ptr(hi), ptr(lo), x.numel(), rt.stream())
    return hi, lo


def _weight_planes(W, for_dgrad, nterms, cin_pad=0):
    ver = getattr(W, "pnp_version", None)
    cache = W.__dict__.setdefault("_pnp_planes", {})
    key = (for_dgrad, nterms, cin_pad)
    hit = cache.get(key)
    if hit is not None and ver is not None and hit[0] == ver:
        return hit[1], hit[2]
    kh, kw, cin, cout = W.shape
    hi = torch.empty(kh * kw * max(cin, cin_pad) * cout, dtype=torch.bfloat16, device=W.device)
    lo = torch.empty_like(hi) if nterms == 3 else None
    call("pnp_split_weight_bf16", ptr(W), ptr(hi), ptr(lo), kh, kw, cin, cout, 1 if for_dgrad else 0, cin_pad, rt.stream())
    cache[key] = (ver, hi, lo)
    return hi, lo


def _padded_planes(x, nterms, cpad):
    """[.., C] fp32 -> [.., cpad] bf16 planes (zero channels beyond C)"""
    shape = tuple(x.shape[:-1]) + (cpad,)
    hi, lo = _new_planes(shape, x.device, nterms)
    call("pnp_split_bf16_pad", ptr(x), ptr(hi), ptr(lo), x.numel() // x.shape[-1], x.shape[-1], cpad, rt.stream())
    return hi, lo


def _weight_T(W):
    ver = getattr(W, "pnp_version", None)
    hit = W.__dict__.get("_pnp_wT")
    if hit is not None and ver is not None and hit[0] == ver:
        return hit[1]
    kh, kw, cin, cout = W.shape
    wT = torch.empty(kh, kw, cout, cin, dtype=W.dtype, device=W.device)
    call("pnp_weight_transpose", ptr(W), ptr(wT), kh * kw, cin, cout, rt.stream())
    W.__dict__["_pnp_wT"] = (ver, wT)
    return wT


def drop_operand_caches(variables):
    """forget the operands cached on these variables (bf16 weight planes, transposed SIMT weights, folded inference-mode batch-norm
    coefficients), so that their next use re-derives them from the live values"""
    for v in variables:
        for attr in ("_pnp_planes", "_pnp_wT", "_pnp_bncoef"):
            v.__dict__.pop(attr, None)


def _conv_flops(g):
    return 2.0 * g.B * g.Ho * g.Wo * g.Cout * g.kh * g.kw * g.Cin


class Epilogue:
    """what the wgmma forward convolution may apply to its accumulator before it leaves the SM (pnp_conv2d_tc_fwd_fused):
    y = act(z * scale + shift + skip), plus the bf16 operand planes of y"""
    __slots__ = ("scale", "shift", "skip", "skip_c", "skip_off", "act", "planes", "planes_only")

    def __init__(self, scale=None, shift=None, skip=None, skip_off=0, act=ACT_NONE, planes=0, planes_only=False):
        self.scale, self.shift, self.skip, self.skip_off, self.act, self.planes = scale, shift, skip, skip_off, act, planes
        self.planes_only = planes_only
        self.skip_c = skip.shape[-1] if skip is not None else 0


def conv_fwd_raw(xp, W, geom, drop=None, stats=None, keep_planes=False, ep=None):
    """z = conv(xp, W) [* dropout]; xp already mirror-padded if needed.  stats=(sum,sumsq) f64 buffers are filled only
    when the tensor-core path can fuse them.  ep (an Epilogue, tensor-core path only): the returned tensor is the layer's final y and
    carries its planes.  Returns (z or y, stats_done, (hi, lo) bf16 planes of xp or None, epilogue applied)."""
    z = torch.empty(geom.B, geom.Ho, geom.Wo, geom.Cout, dtype=torch.float32, device=xp.device)
    nt = _tc_mode()
    if nt and _tc_candidate("fwd", geom):
        planes = _planes_of(xp, nt)
        whi, wlo = _weight_planes(W, False, nt)
        g_tc = geom
        fuse = stats is not None and FUSE_BN_STATS
        try:
            tag = "fwd%dx%d.%d.%d" % (geom.Ho, geom.Cin, geom.Cout, geom.kh * geom.stride)
            if ep is None:
                _tc_launch(tag, _conv_flops(geom), "pnp_conv2d_tc_fwd", ptr(planes[0]), ptr(planes[1]), ptr(whi), ptr(wlo), ptr(z),
                           ctypes.byref(g_tc), nt, _byref(drop), 0, ptr(stats[0]) if fuse else None, ptr(stats[1]) if fuse else None,
                           rt.stream())
                _tc_proven.add(_gkey("fwd", geom))
                return z, fuse, (planes if keep_planes else None), False
            yh, yl = _new_planes(z.shape, xp.device, ep.planes) if ep.planes else (None, None)
            if ep.planes and ep.planes_only:
                z = _PlanesOnly(z.shape, xp.device)
            cep = _C.TcEpilogue(ptr(ep.scale), ptr(ep.shift), ptr(ep.skip), ep.skip_c, ep.skip_off, ep.act, ptr(yh), ptr(yl))
            _tc_launch(tag, _conv_flops(geom), "pnp_conv2d_tc_fwd_fused", ptr(planes[0]), ptr(planes[1]), ptr(whi), ptr(wlo),
                       None if isinstance(z, _PlanesOnly) else ptr(z),
                       ctypes.byref(g_tc), nt, _byref(drop), 0, None, None, ctypes.byref(cep), rt.stream())
            _tc_proven.add(_gkey("fwd", geom))
            if ep.planes:
                z._pnp_planes = (ep.planes, yh, yl)
            return z, False, (planes if keep_planes else None), True
        except _C.Unsupported:
            _tc_declined.add(_gkey("fwd", geom))
    _tc_launch("simt:fwd%dx%d.%d.%d" % (geom.Ho, geom.Cin, geom.Cout, geom.kh * geom.stride), _conv_flops(geom), "pnp_conv2d_fwd", ptr(xp), ptr(W), ptr(z), ctypes.byref(geom), _byref(drop), 0, rt.stream())
    return z, False, None, False


def _bn_infer_coef(bn):
    """[scale, shift, mean, invstd] of an inference-mode batch norm (moving statistics), cached per variable versions: a frozen
    sub-graph (the source segmenter inside every D step) pays for them once, not once per layer call"""
    key = tuple(getattr(t, "pnp_version", 0) for t in (bn.gamma, bn.beta, bn.moving_mean, bn.moving_var))
    hit = bn.gamma.__dict__.get("_pnp_bncoef")
    if hit is not None and hit[0] == key:
        return hit[1]
    C = bn.gamma.numel()
    vec = torch.empty(4, C, dtype=torch.float32, device=bn.gamma.device)
    call("pnp_bn_finalize", None, None, 1, C, ptr(bn.gamma), ptr(bn.beta), ptr(bn.moving_mean), ptr(bn.moving_var), 0, ptr(vec[0]),
         ptr(vec[1]), ptr(vec[2]), ptr(vec[3]), rt.stream())
    bn.gamma.__dict__["_pnp_bncoef"] = (key, vec)
    return vec


def conv_dgrad_raw(dz, W, geom, into=None, dz_planes=None):
    """dx[B,H,W,Cin] = conv^T(dz, W); if `into` is given the result is accumulated into it."""
    acc = 1 if into is not None else 0
    dx = into if into is not None else torch.empty(geom.B, geom.H, geom.W, geom.Cin, dtype=torch.float32, device=dz.device)
    nt = _tc_mode()
    if nt and _tc_candidate("dgrad", geom):
        hi, lo = dz_planes if dz_planes is not None else split_bf16(dz, nt)
        whi, wlo = _weight_planes(W, True, nt)
        try:
            _tc_launch("dgr%dx%d.%d.%d" % (geom.Ho, geom.Cin, geom.Cout, geom.kh * geom.stride), _conv_flops(geom), "pnp_conv2d_tc_dgrad", ptr(hi), ptr(lo), ptr(whi), ptr(wlo), ptr(dx),
                       ctypes.byref(geom), nt, acc, rt.stream())
            _tc_proven.add(_gkey("dgrad", geom))
            return dx
        except _C.Unsupported:
            _tc_declined.add(_gkey("dgrad", geom))
    _tc_launch("simt:dgr%dx%d.%d.%d" % (geom.Ho, geom.Cin, geom.Cout, geom.kh * geom.stride), _conv_flops(geom), "pnp_conv2d_dgrad", ptr(dz), ptr(_weight_T(W)), ptr(dx), ctypes.byref(geom), acc, rt.stream())
    return dx


def conv_wgrad_raw(xp, dz, W, geom, x_planes=None, dz_planes=None):
    if W.grad is None:
        W.grad = torch.empty_like(W)
        call("pnp_fill", ptr(W.grad), 0.0, W.numel(), rt.stream())
    nt = _tc_mode()
    if nt and TC_WGRAD and _tc_candidate("wgrad", geom):
        cp = _cin_pad(geom)
        if cp != geom.Cin:
            xh, xl = _padded_planes(xp, nt, cp)      # (the planes kept by the forward pass are the unpadded 32-channel ones)
        elif x_planes is not None:
            xh, xl = x_planes
        else:
            xh, xl = _planes_of(xp, nt)
        dh, dl = dz_planes if dz_planes is not None else split_bf16(dz, nt)
        try:
            _tc_launch("wgr%dx%d.%d.%d" % (geom.Ho, geom.Cin, geom.Cout, geom.kh * geom.stride), _conv_flops(geom), "pnp_conv2d_tc_wgrad", ptr(xh), ptr(xl), ptr(dh), ptr(dl), ptr(W.grad),
                       ctypes.byref(geom), nt, cp if cp != geom.Cin else 0, rt.stream())
            _grad_written(W)
            _tc_proven.add(_gkey("wgrad", geom))
            return
        except _C.Unsupported:
            _tc_declined.add(_gkey("wgrad", geom))
    _tc_launch("simt:wgr%dx%d.%d.%d" % (geom.Ho, geom.Cin, geom.Cout, geom.kh * geom.stride), _conv_flops(geom), "pnp_conv2d_wgrad", ptr(xp), ptr(dz), ptr(W.grad), ctypes.byref(geom), rt.stream())
    _grad_written(W)


def _tc_will_run(kind, geom):
    return bool(_tc_mode()) and _tc_candidate(kind, geom) and (kind != "wgrad" or TC_WGRAD)


# ------------------------------------------------------------------------------------------------
# one fused layer: [mirror pad] -> conv -> dropout -> [BN] -> [+skip] -> [act]
# ------------------------------------------------------------------------------------------------
class BNVars:
    """handles of one tf.contrib.layers.batch_norm scope (layers.py:95-100)"""
    __slots__ = ("gamma", "beta", "moving_mean", "moving_var")

    def __init__(self, gamma, beta, moving_mean, moving_var):
        self.gamma, self.beta, self.moving_mean, self.moving_var = gamma, beta, moving_mean, moving_var


class LayerCfg:
    __slots__ = ("stride", "dil", "padding", "keep_prob", "bn", "bn_training", "act", "skip_off", "grad_on")

    def __init__(self, stride=1, dil=1, padding="SAME", keep_prob=1.0, bn=None, bn_training=True, act=ACT_NONE, skip_off=0):
        self.stride, self.dil, self.padding, self.keep_prob = stride, dil, padding, keep_prob
        self.bn, self.bn_training, self.act, self.skip_off = bn, bool(bn_training), act, skip_off
        self.grad_on = True


def _geometry(x_shape, w_shape, cfg):
    B, H, Wd, C = x_shape
    kh, kw, cin, cout = w_shape
    if C != cin:
        raise ValueError("conv: input has %d channels, filter expects %d" % (C, cin))
    p = 0
    if cfg.padding == "SYMMETRIC":
        p = kh // 2
        H, Wd = H + 2 * p, Wd + 2 * p
        pt = pl = 0
        Ho = (H - ((kh - 1) * cfg.dil + 1)) // cfg.stride + 1
        Wo = (Wd - ((kw - 1) * cfg.dil + 1)) // cfg.stride + 1
    elif cfg.padding == "SAME":
        pt, _ = same_pad(H, kh, cfg.stride, cfg.dil)
        pl, _ = same_pad(Wd, kw, cfg.stride, cfg.dil)
        Ho, Wo = -(-H // cfg.stride), -(-Wd // cfg.stride)
    elif cfg.padding == "VALID":
        pt = pl = 0
        Ho = (H - ((kh - 1) * cfg.dil + 1)) // cfg.stride + 1
        Wo = (Wd - ((kw - 1) * cfg.dil + 1)) // cfg.stride + 1
    else:
        # the reference leaves conv_2d unbound for unknown strings (layers.py:17-25) -> UnboundLocalError
        raise UnboundLocalError("local variable 'conv_2d' referenced before assignment (padding=%r)" % (cfg.padding,))
    return p, ConvGeom(B, H, Wd, cin, Ho, Wo, cout, kh, kw, cfg.stride, cfg.dil, pt, pl)


# fold inference-mode batch norm + skip + activation into the wgmma epilogue (PNP_FUSE_EPILOGUE=0: separate apply kernel)
FUSE_EPILOGUE = os.environ.get("PNP_FUSE_EPILOGUE", "1") != "0"

# the active bnstats.Collector while batch-norm statistics are re-estimated (bnstats.collecting), else None
BN_COLLECTOR = None


def layer_forward(x, W, cfg, skip=None, save=True, planes_only=False):
    """returns (y, saved) -- `saved` is None when save is False (inference / frozen sub-graph).
    planes_only: the caller guarantees that y is consumed ONLY as bf16 operand planes (the hidden activation of a residual
    block whose second convolution runs on the tensor-core path): its fp32 copy is then never written, and the backward pass
    takes the activation's sign from the hi plane."""
    x = x.contiguous()
    dev = x.device
    p, geom = _geometry(x.shape, W.shape, cfg)
    if p:
        xp = torch.empty(geom.B, geom.H, geom.W, geom.Cin, dtype=torch.float32, device=dev)
        call("pnp_mirror_pad_fwd", ptr(x), ptr(xp), x.shape[0], x.shape[1], x.shape[2], x.shape[3], p, rt.stream())
    else:
        xp = x
    drop, drop_info = _drop_cfg(cfg.keep_prob)
    C = geom.Cout
    M = geom.B * geom.Ho * geom.Wo
    bn = cfg.bn
    keep_planes = save and W.requires_grad
    cs = skip.shape[-1] if skip is not None else 0
    mean = invstd = None
    # ---- (a) everything after the convolution folded into its epilogue: an inference-mode batch norm whose parameters take
    #          no gradient (the frozen segmenter inside the D / G steps, evaluation), or a plain activation / skip
    bn_frozen = bn is not None and not cfg.bn_training and not (save and (bn.gamma.requires_grad or bn.beta.requires_grad))
    foldable = FUSE_EPILOGUE and _tc_will_run("fwd", geom) and (bn_frozen or (bn is None and (cfg.act != ACT_NONE or skip is not None)))
    if foldable:
        coef = _bn_infer_coef(bn) if bn is not None else None
        ep = Epilogue(coef[0] if bn is not None else None, coef[1] if bn is not None else None, skip, cfg.skip_off, cfg.act,
                      _want_planes(C), planes_only and bool(_want_planes(C)))
        y, _, x_planes, applied = conv_fwd_raw(xp, W, geom, drop, None, keep_planes, ep)
        if applied:
            if not save:
                return y, None
            saved = {"cfg": cfg, "geom": geom, "p": p, "x_shape": tuple(x.shape), "xp": xp, "xs": x_planes, "W": W, "drop": drop_info,
                     "z": None, "y": y if cfg.act != ACT_NONE else None, "mean": coef[2] if bn is not None else None,
                     "invstd": coef[3] if bn is not None else None, "skip_c": cs}
            if isinstance(y, _PlanesOnly):
                saved["y"], saved["y_hi"] = None, y._pnp_planes[1]
            return y, saved
        z, stats_done = y, False            # the launcher declined the tensor-core path: z is the plain convolution
        stats = None
    else:
        stats = None
        if bn is not None and cfg.bn_training:
            s = _zeros_f64(2 * C, dev)
            stats = (s[:C], s[C:])
        z, stats_done, x_planes, _ = conv_fwd_raw(xp, W, geom, drop, stats, keep_planes)
    # ---- (b) batch norm (+ skip, activation) as one streaming pass over z; the per-channel finalize lives inside it
    if bn is not None:
        if cfg.bn_training and not stats_done:
            call("pnp_bn_stats", ptr(z), M, C, ptr(stats[0]), ptr(stats[1]), rt.stream())
        if cfg.bn_training and BN_COLLECTOR is not None:
            BN_COLLECTOR.add(bn, stats, M)
        vec = torch.empty(2, C, dtype=torch.float32, device=dev)
        mean, invstd = vec[0], vec[1]
        if cfg.bn_training:
            bn.moving_mean.pnp_version = getattr(bn.moving_mean, "pnp_version", 0) + 1
            bn.moving_var.pnp_version = getattr(bn.moving_var, "pnp_version", 0) + 1
        nt = _want_planes(C)
        y = _PlanesOnly(z.shape, dev) if (planes_only and nt) else torch.empty_like(z)
        yh, yl = _new_planes(z.shape, dev, nt) if nt else (None, None)
        call("pnp_bn_apply_fused", ptr(z), ptr(stats[0]) if stats else None, ptr(stats[1]) if stats else None, M, C, ptr(bn.gamma),
             ptr(bn.beta), ptr(bn.moving_mean), ptr(bn.moving_var), 1 if cfg.bn_training else 0, ptr(skip), cs, cfg.skip_off, cfg.act,
             None if isinstance(y, _PlanesOnly) else ptr(y), ptr(yh), ptr(yl), ptr(mean), ptr(invstd), rt.stream())
        if nt:
            y._pnp_planes = (nt, yh, yl)
    elif cfg.act != ACT_NONE or skip is not None:
        y = torch.empty_like(z)
        call("pnp_bn_act_apply", ptr(z), None, None, ptr(skip), cs, cfg.skip_off, cfg.act, ptr(y), None, None, M, C, rt.stream())
    else:
        y = z
    if not save:
        return y, None
    saved = {
        "cfg": cfg, "geom": geom, "p": p, "x_shape": tuple(x.shape), "xp": xp, "xs": x_planes, "W": W, "drop": drop_info,
        "z": z if (bn is not None) else None, "y": y if cfg.act != ACT_NONE else None,
        "mean": mean, "invstd": invstd, "skip_c": cs,
    }
    if isinstance(y, _PlanesOnly):
        saved["y"], saved["y_hi"] = None, y._pnp_planes[1]
    return y, saved


# PNP_BN_BWD_DIRECT=0: always materialise g = dy*act'(y) (the r1 data flow)
BN_BWD_DIRECT = os.environ.get("PNP_BN_BWD_DIRECT", "1") != "0"


def layer_backward(sv, dy, need_dx=True, dx_into=None, want_dskip=False):
    """returns (dx or None, dskip or None).  Parameter gradients are accumulated into var.grad."""
    cfg, geom, W = sv["cfg"], sv["geom"], sv["W"]
    dy = dy.contiguous()
    dev = dy.device
    C = geom.Cout
    M = geom.B * geom.Ho * geom.Wo
    bn = cfg.bn
    drop = _drop_from(sv["drop"])
    y = sv["y"]
    y_hi = sv.get("y_hi")             # the forward pass elided the fp32 activation: its sign lives in the bf16 hi plane
    g_owned = False
    if bn is not None:
        need_dparam = bn.gamma.requires_grad or bn.beta.requires_grad
        coef = None
        dgamma = dbeta = None
        nt = _tc_mode()
        use_w = W.requires_grad and _tc_will_run("wgrad", geom)
        use_d = need_dx and _tc_will_run("dgrad", geom)
        want = bool(nt and FUSE_SPLIT and (use_w or use_d))
        # fp32 dz is only read by the SIMT kernels: drop it when every consumer has already run on the tensor-core path
        consumers = [("wgrad", W.requires_grad), ("dgrad", need_dx)]
        need_f32 = not want or any(on and _gkey(kind, geom) not in _tc_proven for kind, on in consumers)
        need_g = bool(want_dskip and sv["skip_c"])          # the residual skip's gradient IS g: only then must it exist in HBM
        if (cfg.bn_training or need_dparam) and bn.gamma.requires_grad:
            dgamma = _grad_slot(bn.gamma)
        if (cfg.bn_training or need_dparam) and bn.beta.requires_grad:
            dbeta = _grad_slot(bn.beta)
        dz = torch.empty(dy.shape, dtype=torch.float32, device=dev) if need_f32 else None
        dzh, dzl = _new_planes(dy.shape, dev, nt) if want else (None, None)
        if y_hi is not None and not (BN_BWD_DIRECT and not need_g):
            raise RuntimeError("planes-only activation reached a backward path that needs its fp32 copy")
        if BN_BWD_DIRECT and not need_g:
            # two passes over (dy, y, z), no g: 24-28 bytes per element instead of 32
            if cfg.bn_training or need_dparam:
                coef = _zeros_f64(2 * C, dev)
                call("pnp_bn_bwd_reduce_sums", ptr(dy), ptr(y), ptr(y_hi), ptr(sv["z"]), ptr(sv["mean"]), ptr(sv["invstd"]), cfg.act,
                     ptr(coef[:C]), ptr(coef[C:]), M, C, rt.stream())
            call("pnp_bn_bwd_apply_direct", ptr(dy), ptr(y), ptr(y_hi), cfg.act, ptr(sv["z"]), ptr(sv["mean"]), ptr(sv["invstd"]),
                 ptr(bn.gamma), ptr(coef[:C]) if coef is not None else None, ptr(coef[C:]) if coef is not None else None, M, C,
                 1 if cfg.bn_training else 0, _byref(drop), ptr(dgamma), ptr(dbeta), ptr(dz), ptr(dzh), ptr(dzl), rt.stream())
            g = None
        else:
            if cfg.bn_training or need_dparam:
                g = torch.empty(dy.shape, dtype=torch.float32, device=dev)
                g_owned = True
                coef = _zeros_f64(2 * C, dev)
                call("pnp_bn_bwd_reduce", ptr(dy), ptr(y), ptr(sv["z"]), ptr(sv["mean"]), ptr(sv["invstd"]), cfg.act, ptr(g),
                     ptr(coef[:C]), ptr(coef[C:]), M, C, rt.stream())
            elif cfg.act != ACT_NONE:
                g = torch.empty(dy.shape, dtype=torch.float32, device=dev)
                g_owned = True
                call("pnp_act_bwd", ptr(dy), ptr(y), cfg.act, ptr(g), dy.numel(), rt.stream())
            else:
                g = dy
            call("pnp_bn_bwd_apply_direct", ptr(g), None, None, ACT_NONE, ptr(sv["z"]), ptr(sv["mean"]), ptr(sv["invstd"]), ptr(bn.gamma),
                 ptr(coef[:C]) if coef is not None else None, ptr(coef[C:]) if coef is not None else None, M, C,
                 1 if cfg.bn_training else 0, _byref(drop), ptr(dgamma), ptr(dbeta), ptr(dz), ptr(dzh), ptr(dzl), rt.stream())
        if dgamma is not None:
            _grad_written(bn.gamma)
        if dbeta is not None:
            _grad_written(bn.beta)
        if dz is None:
            dz = _PlanesOnly(dy.shape, dev)
        if want:
            dz._pnp_planes = (nt, dzh, dzl)
    else:
        if cfg.act != ACT_NONE:
            g = torch.empty(dy.shape, dtype=torch.float32, device=dev)
            g_owned = True
            call("pnp_act_bwd", ptr(dy), ptr(y), cfg.act, ptr(g), dy.numel(), rt.stream())
        else:
            g = dy
        if drop is not None:
            dz = torch.empty(dy.shape, dtype=torch.float32, device=dev)
            call("pnp_dropout_apply", ptr(g), ptr(dz), g.numel(), ctypes.byref(drop), rt.stream())
        else:
            dz = g
    dskip = None
    if want_dskip and sv["skip_c"]:
        cs = sv["skip_c"]
        if cs == C and g_owned:
            dskip = g            # safe to hand out / accumulate into: nothing reads g after this point
        else:
            dskip = torch.empty(dy.shape[:-1] + (cs,), dtype=torch.float32, device=dev)
            call("pnp_channel_slice", ptr(g), C, cfg.skip_off if cs != C else 0, cs, ptr(dskip), M, 0, rt.stream())
    dz_planes = None
    if (W.requires_grad and _tc_will_run("wgrad", geom)) or (need_dx and _tc_will_run("dgrad", geom)):
        dz_planes = _planes_of(dz, _tc_mode())
    if W.requires_grad:
        conv_wgrad_raw(sv["xp"], dz, W, geom, sv.get("xs"), dz_planes)
    dx = None
    if need_dx:
        if sv["p"]:
            dxp = conv_dgrad_raw(dz, W, geom, None, dz_planes)
            B, H, Wd, Cin = sv["x_shape"]
            dx = torch.empty(sv["x_shape"], dtype=torch.float32, device=dev)
            call("pnp_mirror_pad_bwd", ptr(dxp), ptr(dx), B, H, Wd, Cin, sv["p"], rt.stream())
            if dx_into is not None:
                raise NotImplementedError("accumulating dgrad through a SYMMETRIC pad is not used by the hot path")
        else:
            dx = conv_dgrad_raw(dz, W, geom, dx_into, dz_planes)
    if DEBUG_HOOK is not None:
        DEBUG_HOOK(sv, dy, g, dz, dx)
    return dx, dskip


def _grad_written(v):
    """a gradient contribution to `v` has been launched: data-parallel reducers start a bucket's all-reduce when its last
    contribution of the step is in (parallel.BucketedAllReduce)"""
    hook = getattr(v, "_pnp_grad_hook", None)
    if hook is not None:
        hook(v)


def _grad_slot(v):
    if v.grad is None:
        v.grad = torch.empty_like(v)
        call("pnp_fill", ptr(v.grad), 0.0, v.numel(), rt.stream())
    return v.grad


def _bn_params(cfg):
    return [] if cfg.bn is None else [cfg.bn.gamma, cfg.bn.beta]


class _ConvLayerFn(torch.autograd.Function):
    """conv2d / conv_bn_2d / conv_bn_relu2d / dilate_* of layers.py as ONE fused op (optionally + skip)."""

    @staticmethod
    def forward(ctx, x, skip, cfg, W, *bnp):
        # autograd.Function.forward always runs with grad mode off, and needs_input_grad reflects the inputs' requires_grad flags
        # whatever the caller's grad mode is (r2 ncu: a torch.no_grad() forward of a TRAINABLE network kept saving activations and
        # never folded its batch norms) -- the wrapper records the caller's grad mode on the LayerCfg
        save = any(ctx.needs_input_grad) and getattr(cfg, "grad_on", True)
        y, sv = layer_forward(x, W, cfg, skip, save)
        ctx.sv = sv
        ctx.has_skip = skip is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        sv = ctx.sv
        need_dx = ctx.needs_input_grad[0]
        want_ds = ctx.has_skip and ctx.needs_input_grad[1]
        dx, dskip = layer_backward(sv, dy, need_dx, None, want_ds)
        ctx.sv = None
        return (dx, dskip, None, None) + (None,) * (len(ctx.needs_input_grad) - 4)


def conv_layer(x, W, cfg, skip=None):
    cfg.grad_on = torch.is_grad_enabled()
    return _ConvLayerFn.apply(x, skip, cfg, W, *_bn_params(cfg))


class _ResBlockFn(torch.autograd.Function):
    """residual_block / DR_block of layers.py:145-189: act(x_s + BN(conv(act(BN(conv(x)))))) with the
    skip-gradient and the first conv's dgrad merged by the dgrad epilogue (no separate add kernel)."""

    @staticmethod
    def forward(ctx, x, cfg1, cfg2, W1, W2, *bnp):
        save = any(ctx.needs_input_grad) and getattr(cfg1, "grad_on", True)
        h, s1 = layer_forward(x, W1, cfg1, None, save, planes_only=_hidden_planes_only(x, W1, W2, cfg1, cfg2, save))
        y, s2 = layer_forward(h, W2, cfg2, x, save)
        ctx.s1, ctx.s2 = s1, s2
        return y

    @staticmethod
    def backward(ctx, dy):
        need_dx = ctx.needs_input_grad[0]
        dh, dskip = layer_backward(ctx.s2, dy, True, None, need_dx)
        dx, _ = layer_backward(ctx.s1, dh, need_dx, dskip if need_dx else None, False)
        ctx.s1 = ctx.s2 = None
        return (dx, None, None, None, None) + (None,) * (len(ctx.needs_input_grad) - 5)


# PNP_PLANES_ONLY=0: always write the fp32 hidden activation of a residual block
PLANES_ONLY = os.environ.get("PNP_PLANES_ONLY", "1") != "0"


def _hidden_planes_only(x, W1, W2, cfg1, cfg2, save):
    """may the hidden activation h = act(BN(conv1(x))) of a residual block exist as bf16 planes only?  Yes when its single
    consumer, conv2 (forward, and the weight gradient if W2 trains), has already run on the tensor-core path for this geometry, h
    has a batch norm (whose apply pass / epilogue emits the planes) and the backward pass is the g-less one."""
    if not (PLANES_ONLY and BN_BWD_DIRECT and FUSE_SPLIT and cfg1.bn is not None and cfg2.padding == "SAME" and _tc_mode()):
        return False
    try:
        _, g1 = _geometry(tuple(x.shape), W1.shape, cfg1)
        _, g2 = _geometry((g1.B, g1.Ho, g1.Wo, g1.Cout), W2.shape, cfg2)
    except Exception:      # noqa: BLE001 -- shape errors surface in layer_forward with their proper message
        return False
    if not _want_planes(g1.Cout) or _gkey("fwd", g2) not in _tc_proven:
        return False
    if save and W2.requires_grad and _gkey("wgrad", g2) not in _tc_proven:
        return False
    return True


def res_block(x, W1, W2, cfg1, cfg2):
    cfg1.grad_on = cfg2.grad_on = torch.is_grad_enabled()
    return _ResBlockFn.apply(x, cfg1, cfg2, W1, W2, *(_bn_params(cfg1) + _bn_params(cfg2)))


# ------------------------------------------------------------------------------------------------
# pooling / phase shift / discriminator input
# ------------------------------------------------------------------------------------------------
class _MaxPool2Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = x.contiguous()
        B, H, W, C = x.shape
        y = torch.empty(B, H // 2, W // 2, C, dtype=x.dtype, device=x.device)
        call("pnp_maxpool2_fwd", ptr(x), ptr(y), B, H, W, C, rt.stream())
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        B, H, W, C = x.shape
        dx = torch.empty_like(x)
        call("pnp_maxpool2_bwd", ptr(x), ptr(dy.contiguous()), ptr(dx), B, H, W, C, rt.stream())
        return dx


def max_pool2(x):
    return _MaxPool2Fn.apply(x)


class _AvgPool2Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = x.contiguous()
        B, H, W, C = x.shape
        y = torch.empty(B, H // 2, W // 2, C, dtype=x.dtype, device=x.device)
        call("pnp_avgpool2", ptr(x), ptr(y), B, H, W, C, 0, rt.stream())
        ctx.shape = (B, H, W, C)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, H, W, C = ctx.shape
        dx = torch.empty(ctx.shape, dtype=dy.dtype, device=dy.device)
        call("pnp_avgpool2", ptr(dy.contiguous()), ptr(dx), B, H, W, C, 1, rt.stream())
        return dx


def avg_pool2(x):
    return _AvgPool2Fn.apply(x)


class _PoolFn(torch.autograd.Function):
    """tf.nn.max_pool / avg_pool, ksize = strides = n, padding 'SAME', any n (layers.py:102-106)"""

    @staticmethod
    def forward(ctx, x, n, avg):
        x = x.contiguous()
        B, H, W, C = x.shape
        y = torch.empty(B, -(-H // n), -(-W // n), C, dtype=x.dtype, device=x.device)
        call("pnp_pool_fwd", ptr(x), ptr(y), B, H, W, C, n, 1 if avg else 0, rt.stream())
        ctx.meta = (B, H, W, C, n, avg)
        ctx.save_for_backward(*(() if avg else (x,)))
        return y

    @staticmethod
    def backward(ctx, dy):
        B, H, W, C, n, avg = ctx.meta
        x = None if avg else ctx.saved_tensors[0]
        dx = torch.empty(B, H, W, C, dtype=dy.dtype, device=dy.device)
        call("pnp_pool_bwd", ptr(x), ptr(dy.contiguous()), ptr(dx), B, H, W, C, n, 1 if avg else 0, rt.stream())
        return dx, None, None


def pool_same(x, n, avg=False):
    return _PoolFn.apply(x, int(n), bool(avg))


class _CropConcatFn(torch.autograd.Function):
    """crop_and_concat / simple_concat2d (layers.py:108-127): [centre crop of x1 to x2's height and width | x2] along channels"""

    @staticmethod
    def forward(ctx, x1, x2):
        x1, x2 = x1.contiguous(), x2.contiguous()
        B, H1, W1, C1 = x1.shape
        B2, H2, W2, C2 = x2.shape
        out = torch.empty(B, H2, W2, C1 + C2, dtype=x1.dtype, device=x1.device)
        call("pnp_crop_concat_fwd", ptr(x1), ptr(x2), ptr(out), B, H1, W1, C1, H2, W2, C2, rt.stream())
        ctx.meta = (B, H1, W1, C1, H2, W2, C2)
        return out

    @staticmethod
    def backward(ctx, dout):
        B, H1, W1, C1, H2, W2, C2 = ctx.meta
        n1, n2 = ctx.needs_input_grad
        dx1 = torch.empty(B, H1, W1, C1, dtype=dout.dtype, device=dout.device) if n1 else None
        dx2 = torch.empty(B, H2, W2, C2, dtype=dout.dtype, device=dout.device) if n2 else None
        if n1 or n2:
            call("pnp_crop_concat_bwd", ptr(dout.contiguous()), ptr(dx1), ptr(dx2), B, H1, W1, C1, H2, W2, C2, rt.stream())
        return dx1, dx2


def crop_concat(x1, x2):
    return _CropConcatFn.apply(x1, x2)


class _CrossEntropyFn(torch.autograd.Function):
    """layers.cross_entropy (layers.py:140-141): -mean(y_ * log(clip(output_map, 1e-10, 1)))"""

    @staticmethod
    def forward(ctx, y_, p):
        y_, p = y_.contiguous(), p.contiguous()
        acc = torch.zeros(1, dtype=torch.float64, device=p.device)
        out = torch.empty(1, dtype=torch.float32, device=p.device)
        call("pnp_cross_entropy_fwd", ptr(y_), ptr(p), p.numel(), ptr(acc), ptr(out), rt.stream())
        ctx.save_for_backward(y_, p)
        return out.reshape(())

    @staticmethod
    def backward(ctx, g):
        y_, p = ctx.saved_tensors
        ny, np_ = ctx.needs_input_grad
        dy = torch.empty_like(y_) if ny else None
        dp = torch.empty_like(p) if np_ else None
        if ny or np_:
            call("pnp_cross_entropy_bwd", ptr(y_), ptr(p), ptr(g.contiguous().reshape(1).float()), p.numel(), ptr(dy), ptr(dp), rt.stream())
        return dy, dp


def cross_entropy(y_, p):
    return _CrossEntropyFn.apply(y_, p)


class _PhaseShiftFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, X, r, G, order_b1):
        X = X.contiguous()
        B, a, b, C = X.shape
        if C != G * r * r:
            raise ValueError("PS: %d channels cannot be split into %d groups of %d" % (C, G, r * r))
        out = torch.empty(B, a * r, b * r, G, dtype=X.dtype, device=X.device)
        call("pnp_phase_shift_fwd", ptr(X), ptr(out), B, a, b, G, r, G, 0, 1, order_b1, rt.stream())
        ctx.meta = (B, a, b, G, r, order_b1)
        return out

    @staticmethod
    def backward(ctx, dout):
        B, a, b, G, r, o = ctx.meta
        dX = torch.empty(B, a, b, G * r * r, dtype=dout.dtype, device=dout.device)
        call("pnp_phase_shift_bwd", ptr(dout.contiguous()), ptr(dX), B, a, b, G, r, G, 0, 1, o, rt.stream())
        return dX, None, None, None


def phase_shift(X, r, n_channel, batch_size):
    return _PhaseShiftFn.apply(X, r, n_channel, 1 if batch_size == 1 else 0)


class _TailFn(torch.autograd.Function):
    """The segmenter tail PS(r) -> SYMMETRIC pad -> k x k convolution (source_segmenter.py:200-207) as ONE kernel: the phase
    shift and the mirror padding are index maps inside the convolution's tile loader (pnp_ps_mirror_conv_fwd).  Used when the
    output filter takes no gradient (every adversarial step, evaluation); the gradient w.r.t. X runs through the stand-alone
    kernels (transposed conv -> mirror-pad fold -> inverse phase shift)."""

    @staticmethod
    def forward(ctx, X, w, r, G, order_b1):
        X = X.contiguous()
        B, a, b, C = X.shape
        kh, kw, cin, cout = w.shape
        if C != G * r * r or cin != G:
            raise ValueError("tail: %d channels cannot be split into %d groups of %d (filter expects %d)" % (C, G, r * r, cin))
        y = torch.empty(B, a * r, b * r, cout, dtype=X.dtype, device=X.device)
        flops = 2.0 * B * a * r * b * r * cout * kh * kw * cin
        _tc_launch("simt:tail%dx%d.%d.%d" % (a * r, cin, cout, kh), flops, "pnp_ps_mirror_conv_fwd", ptr(X), ptr(w), ptr(y), B, a, b, G, r,
                   kh, kw, cout, order_b1, rt.stream())
        ctx.w = w
        ctx.meta = (B, a, b, G, r, order_b1)
        return y

    @staticmethod
    def backward(ctx, dy):
        B, a, b, G, r, o = ctx.meta
        w = ctx.w
        kh, kw, cin, cout = w.shape
        p = kh // 2
        H, W = a * r, b * r
        if FUSE_TAIL_BWD:
            dX = torch.empty(B, a, b, G * r * r, dtype=dy.dtype, device=dy.device)
            flops = 2.0 * B * H * W * cout * kh * kw * cin
            _tc_launch("simt:tailbwd%dx%d.%d.%d" % (H, cin, cout, kh), flops, "pnp_ps_mirror_conv_bwd", ptr(dy.contiguous()), ptr(w), ptr(dX),
                       B, a, b, G, r, kh, kw, cout, o, rt.stream())
            return dX, None, None, None, None
        geom = ConvGeom(B, H + 2 * p, W + 2 * p, cin, H, W, cout, kh, kw, 1, 1, 0, 0)
        dxp = conv_dgrad_raw(dy.contiguous(), w, geom)
        dflat = torch.empty(B, H, W, cin, dtype=dy.dtype, device=dy.device)
        call("pnp_mirror_pad_bwd", ptr(dxp), ptr(dflat), B, H, W, cin, p, rt.stream())
        dX = torch.empty(B, a, b, G * r * r, dtype=dy.dtype, device=dy.device)
        call("pnp_phase_shift_bwd", ptr(dflat), ptr(dX), B, a, b, G, r, G, 0, 1, o, rt.stream())
        return dX, None, None, None, None


# PNP_FUSE_TAIL=0: phase shift, mirror pad and output convolution as three kernels
FUSE_TAIL = os.environ.get("PNP_FUSE_TAIL", "1") != "0"
# PNP_FUSE_TAIL_BWD=0: its input gradient as transposed conv -> mirror-pad fold -> inverse phase shift (three kernels)
FUSE_TAIL_BWD = os.environ.get("PNP_FUSE_TAIL_BWD", "1") != "0"


def tail_ps_conv(X, w, r, n_channel, batch_size):
    return _TailFn.apply(X, w, r, n_channel, 1 if batch_size == 1 else 0)


class _DiscInputFn(torch.autograd.Function):
    """adversarial.py:325-335 in one gather: [PS(c4,2) x3 | PS(c6,4) | PS(b7,8) | PS(c9,8) | logits | argmax]"""

    @staticmethod
    def forward(ctx, c4, c6, b7, c9, logits, r, order_b1):
        srcs = [c4.contiguous(), c6.contiguous(), b7.contiguous(), c9.contiguous()]
        logits = logits.contiguous()
        B, H, W, NC = logits.shape
        plan = []
        off = 0
        for t, ntile in zip(srcs, (3, 1, 1, 1)):
            G = t.shape[-1] // (r * r)
            plan.append((t.shape[1], t.shape[2], G, off, ntile))
            off += G * ntile
        ctot = off + NC + 1
        out = torch.empty(B, H, W, ctot, dtype=logits.dtype, device=logits.device)
        if ctot % 4 == 0 and ctot <= 64:
            n = len(srcs)
            ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in srcs])
            ia = lambda k: (ctypes.c_int * n)(*[pl[k] for pl in plan])
            call("pnp_disc_input_fwd", ptrs, ia(0), ia(1), ia(2), ia(4), n, ptr(logits), NC, ptr(out), B, H, W, r, order_b1, rt.stream())
        else:
            for t, (a, b, G, coff, ntile) in zip(srcs, plan):
                call("pnp_phase_shift_fwd", ptr(t), ptr(out), B, a, b, G, r, ctot, coff, ntile, order_b1, rt.stream())
            call("pnp_logits_argmax_concat", ptr(logits), ptr(out), B * H * W, NC, ctot, off, rt.stream())
        ctx.meta = (B, H, W, NC, r, order_b1, plan, ctot, off)
        return out

    @staticmethod
    def backward(ctx, dout):
        B, H, W, NC, r, o, plan, ctot, off = ctx.meta
        dout = dout.contiguous()
        grads = []
        for i, (a, b, G, coff, ntile) in enumerate(plan):
            if ctx.needs_input_grad[i]:
                dX = torch.empty(B, a, b, G * r * r, dtype=dout.dtype, device=dout.device)
                call("pnp_phase_shift_bwd", ptr(dout), ptr(dX), B, a, b, G, r, ctot, coff, ntile, o, rt.stream())
                grads.append(dX)
            else:
                grads.append(None)
        dl = None
        if ctx.needs_input_grad[4]:
            dl = torch.empty(B, H, W, NC, dtype=dout.dtype, device=dout.device)
            call("pnp_channel_slice", ptr(dout), ctot, off, NC, ptr(dl), B * H * W, 0, rt.stream())
        return tuple(grads) + (dl, None, None)


def disc_input(c4, c6, b7, c9, logits, batch_size, r=8):
    return _DiscInputFn.apply(c4, c6, b7, c9, logits, r, 1 if batch_size == 1 else 0)


# ------------------------------------------------------------------------------------------------
# losses / metrics
# ------------------------------------------------------------------------------------------------
class _SegLossFn(torch.autograd.Function):
    """(weighted CE, soft Dice) of source_segmenter.py:241-273 from one reduction pass."""

    @staticmethod
    def forward(ctx, logits, y):
        logits, y = logits.contiguous(), y.contiguous()
        C = logits.shape[-1]
        P = logits.numel() // C
        acc = _zeros_f64(4 * C, logits.device)
        call("pnp_segloss_reduce", ptr(logits), ptr(y), P, C, ptr(acc), rt.stream())
        out = torch.empty(2, dtype=torch.float32, device=logits.device)
        coef = torch.empty(3 * C, dtype=torch.float32, device=logits.device)
        call("pnp_segloss_finalize", ptr(acc), P, C, ptr(out), ptr(coef), rt.stream())
        ctx.save_for_backward(logits, y, coef)
        return out[0], out[1]

    @staticmethod
    def backward(ctx, g_wce, g_dice):
        logits, y, coef = ctx.saved_tensors
        C = logits.shape[-1]
        P = logits.numel() // C
        dl = torch.empty_like(logits)
        call("pnp_segloss_bwd", ptr(logits), ptr(y), ptr(coef), ptr(g_wce.contiguous()), ptr(g_dice.contiguous()), ptr(dl), P, C,
             rt.stream())
        return dl, None


def seg_losses(logits, y):
    return _SegLossFn.apply(logits, y)


class _EntropyLossFn(torch.autograd.Function):
    """mean per-pixel softmax entropy of logits [..., C] (TENT's objective, pnp_entropy_*) and the mean class probability p-bar,
    which is a diagnostic and not differentiated"""

    @staticmethod
    def forward(ctx, logits):
        logits = logits.contiguous()
        C = logits.shape[-1]
        P = logits.numel() // C
        acc = _zeros_f64(1 + C, logits.device)
        call("pnp_entropy_reduce", ptr(logits), P, C, ptr(acc), rt.stream())
        out = torch.empty(1 + C, dtype=torch.float32, device=logits.device)
        call("pnp_entropy_finalize", ptr(acc), P, C, ptr(out), rt.stream())
        ctx.save_for_backward(logits)
        pbar = out[1:]
        ctx.mark_non_differentiable(pbar)
        return out[0], pbar

    @staticmethod
    def backward(ctx, g, _g_pbar):
        logits, = ctx.saved_tensors
        C = logits.shape[-1]
        P = logits.numel() // C
        dl = torch.empty_like(logits)
        call("pnp_entropy_bwd", ptr(logits), ptr(g.contiguous()), ptr(dl), P, C, rt.stream())
        return dl


def entropy_loss(logits):
    """-> (loss, pbar): the mean over pixels of -sum_c p_c log p_c of the softmax of `logits` [B, H, W, C], and the mean class
    probability [C]"""
    return _EntropyLossFn.apply(logits)


def pixel_softmax2(logits):
    logits = logits.contiguous()
    C = logits.shape[-1]
    out = torch.empty_like(logits)
    call("pnp_pixel_softmax2", ptr(logits), ptr(out), logits.numel() // C, C, rt.stream())
    return out


IMG_KINDS = {"channel": 0, "argmax": 1, "softmax2_argmax": 2}       # PNP_IMG_* of include/pnp_b200.h


def image_summary(sources, max_outputs=3):
    """The uint8 panels of tf.summary.image(name, tf.expand_dims(tf.cast(t, tf.float32), 3), max_outputs) for every source of
    one monitoring pass, in one launch and one device->host copy.  `sources`: list of (tensor fp32 [B,H,W,C] on the device, kind,
    channel) with kind "channel" (t = tensor[..., channel]), "argmax" (t = tf.argmax(tensor, 3)) or "softmax2_argmax"
    (t = tf.argmax(pixel_wise_softmax_2(tensor), 3)); every source has the same B, H, W.
    Returns a host numpy.uint8 array [nsrc, min(B, max_outputs), H, W]."""
    ts = [t.contiguous() for t, _, _ in sources]
    B, H, W = ts[0].shape[:3]
    for t in ts:
        if t.dim() != 4 or tuple(t.shape[:3]) != (B, H, W) or t.dtype != torch.float32:
            raise ValueError("image_summary: every source must be fp32 [%d, %d, %d, C], got %s %s" % (B, H, W, tuple(t.shape), t.dtype))
    n, ns = min(B, int(max_outputs)), len(ts)
    dev = torch.empty(ns, n, H, W, dtype=torch.uint8, device=ts[0].device)
    ia = lambda vals: (ctypes.c_int * ns)(*vals)
    call("pnp_image_summary_u8", (ctypes.c_void_p * ns)(*[t.data_ptr() for t in ts]), ia([IMG_KINDS[k] for _, k, _ in sources]),
         ia([t.shape[3] for t in ts]), ia([int(c) for _, _, c in sources]), ns, B, H, W, n, ptr(dev), rt.stream())
    host = torch.empty(dev.shape, dtype=torch.uint8, pin_memory=True)
    host.copy_(dev, non_blocking=True)
    torch.cuda.current_stream().synchronize()
    return host.numpy()


def one_hot(labels, num_cls):
    """device-side lib._label_decomp (lib.py:75-92): int64 [..] -> fp32 [.., num_cls]"""
    labels = labels.contiguous().to(torch.int64)
    out = torch.empty(labels.shape + (num_cls,), dtype=torch.float32, device=labels.device)
    call("pnp_one_hot", ptr(labels), ptr(out), labels.numel(), num_cls, rt.stream())
    return out


SD_MAX_DIM = 1024        # PNP_SD_MAX_DIM of include/pnp_b200.h
SURFACE_KEYS = ("asd_pred_gt", "asd_gt_pred", "assd", "hd")


def _surface_args(pred, gt, num_cls, spacing):
    """host-side checks of surface_distances: -> (pred, gt) as uint8 volumes with out-of-range labels mapped to 0, spacing"""
    num_cls = int(num_cls)
    if not 2 <= num_cls <= 8:
        raise ValueError("surface_distances: num_cls must be in [2, 8] (one border bit per class in a byte), got %d" % num_cls)
    pred, gt = np.asarray(pred), np.asarray(gt)
    if pred.ndim != 3 or pred.shape != gt.shape:
        raise ValueError("surface_distances: pred %s and gt %s must be equal-shaped 3-D label volumes" % (pred.shape, gt.shape))
    if min(pred.shape) < 1 or max(pred.shape) > SD_MAX_DIM:
        raise ValueError("surface_distances: every dimension must be in [1, %d], got %s" % (SD_MAX_DIM, pred.shape))
    for name, v in (("pred", pred), ("gt", gt)):
        if not (np.issubdtype(v.dtype, np.integer) or np.issubdtype(v.dtype, np.bool_)):
            raise ValueError("surface_distances: %s must hold integer labels, got %s" % (name, v.dtype))
    sp = (1.0, 1.0, 1.0) if spacing is None else tuple(float(s) for s in np.asarray(spacing, np.float64).reshape(-1))
    if len(sp) != 3 or not all(math.isfinite(s) and s > 0 for s in sp):
        raise ValueError("surface_distances: spacing must be 3 positive finite numbers, got %r" % (spacing,))
    def as_u8(v):
        if v.dtype == np.uint8:            # uploaded as it is: the kernels count labels >= num_cls as background
            return np.ascontiguousarray(v)
        return np.ascontiguousarray(np.where((v >= 0) & (v < num_cls), v, 0), dtype=np.uint8)
    return as_u8(pred), as_u8(gt), sp


def surface_distances(pred, gt, num_cls, spacing=None, hd_percentile=None):
    """Per-class surface distances of a predicted label volume against a ground truth (medpy.metric.binary.assd / hd / hd95,
    which the papers' evaluation calls without spacing), on the device.

    `pred`, `gt`: host integer arrays [n0, n1, n2] (each n <= 1024); labels outside [0, num_cls) count as background.
    `spacing`: voxel size along the three axes, default 1 (voxel units).  For each class c >= 1 with A = (pred == c) and
    B = (gt == c), the border dX is X minus its erosion by the 6-neighbour cross (voxels on the faces of the volume are border
    voxels) and d(v, S) is the Euclidean distance from v to the nearest voxel of S.  Returns a dict of host arrays [num_cls]:
      asd_pred_gt  mean of d(v, dB) over v in dA;   asd_gt_pred  mean of d(v, dA) over v in dB;
      assd         (asd_pred_gt + asd_gt_pred) / 2 (the mean of the two means, like medpy);
      hd           the larger of the two maxima;
      border_pred / border_gt  |dA| / |dB| (int64).
    Index 0 (background) and classes absent from pred or gt are NaN; the border counts say which side was empty.
    `hd_percentile` q in [0, 100] also gives `hd_pct`, numpy.percentile(q) of the pooled distances {d(v, dB) : v in dA} and
    {d(v, dA) : v in dB} (medpy's hd95 at q = 95; q = 100 is `hd`), and `hd_percentile` = q.
    One upload of each volume, one pnp_surface_distance (or pnp_surface_distance_pct) call, one copy back."""
    p, g, sp = _surface_args(pred, gt, num_cls, spacing)
    pct = hd_percentile is not None
    if pct:
        q = float(hd_percentile)
        if not (math.isfinite(q) and 0.0 <= q <= 100.0):
            raise ValueError("surface_distances: hd_percentile must be a number in [0, 100], got %r" % (hd_percentile,))
    n0, n1, n2 = p.shape
    nbytes = ctypes.c_longlong(0)
    call("pnp_surface_distance_pct_workspace" if pct else "pnp_surface_distance_workspace", n0, n1, n2, num_cls, ctypes.byref(nbytes))
    dev = rt.device()
    dp, dg = torch.from_numpy(p).to(dev), torch.from_numpy(g).to(dev)
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    cols = 7 if pct else 6
    out = torch.empty((num_cls - 1) * cols, dtype=torch.float64, device=dev)
    sp = (ctypes.c_double * 3)(*sp)
    if pct:
        call("pnp_surface_distance_pct", ptr(dp), ptr(dg), n0, n1, n2, num_cls, sp, q, ptr(ws), nbytes.value, ptr(out), rt.stream())
    else:
        call("pnp_surface_distance", ptr(dp), ptr(dg), n0, n1, n2, num_cls, sp, ptr(ws), nbytes.value, ptr(out), rt.stream())
    res = surface_from_raw(out.cpu().numpy().reshape(num_cls - 1, cols))
    if pct:
        res["hd_percentile"] = q
    return res


def surface_from_raw(raw):
    """surface_distances' per-class dict from pnp_surface_distance's out[C-1][6] table, or from pnp_surface_distance_pct's
    out[C-1][7] (which adds `hd_pct`)"""
    raw = np.asarray(raw, np.float64)
    C = raw.shape[0] + 1
    res = {k: np.full(C, np.nan) for k in SURFACE_KEYS}
    res["border_pred"] = np.zeros(C, np.int64)
    res["border_gt"] = np.zeros(C, np.int64)
    if raw.shape[1] == 7:
        res["hd_pct"] = np.full(C, np.nan)
    for c in range(1, C):
        s_pg, n_p, max_pg, s_gp, n_g, max_gp = raw[c - 1, :6]
        res["border_pred"][c], res["border_gt"][c] = int(n_p), int(n_g)
        if n_p > 0 and n_g > 0:
            res["asd_pred_gt"][c], res["asd_gt_pred"][c] = s_pg / n_p, s_gp / n_g
            res["assd"][c] = (res["asd_pred_gt"][c] + res["asd_gt_pred"][c]) / 2.0
            res["hd"][c] = max(max_pg, max_gp)
            if raw.shape[1] == 7:
                res["hd_pct"][c] = raw[c - 1, 6]
    return res


def _aug_field(name, t, shape):
    if t is None:
        return None
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32 or tuple(t.shape) != shape:
        raise ValueError("resample_planes: %s must be fp32 %s on the device, got %s" % (
            name, shape, (type(t).__name__ if not isinstance(t, torch.Tensor) else "%s %s on %s" % (t.dtype, tuple(t.shape), t.device))))
    return t.contiguous()


def resample_planes(vol, cls, mats, H, W, image=True, label_planes=1, img=None, lab=None, disp=None, gain=None, ab=None):
    """Planes resampled out of a device volume in one pnp_resample_planes launch (include/pnp_b200.h, "data preparation").
    `vol` fp32 and `cls` uint8 [n0, n1, n2] (either may be None when its output is not wanted), `mats` fp32 [B, C, 3, 3] on the
    device.  Returns (img fp32 [B, H, W, C] or None, lab int64 [B, H, W] (label_planes 1), [B, H, W, C] (label_planes C) or None);
    `img` / `lab` may be given to write into.
    Any of the augmentation fields (fp32 on the device, "data augmentation") makes it one pnp_resample_planes_aug launch: `disp`
    [B, 2, H, W] displaces each output pixel (r, c) by (d_r, d_c) before its matrix, `gain` [B, H, W] multiplies the image by
    1 + gain, `ab` [B, 2] then maps it to a * v + b."""
    B, C = mats.shape[0], mats.shape[1]
    ref = vol if vol is not None else cls
    n0, n1, n2 = ref.shape
    if image and img is None:
        img = torch.empty(B, H, W, C, dtype=torch.float32, device=ref.device)
    if label_planes and lab is None:
        lab = torch.empty((B, H, W) if label_planes == 1 else (B, H, W, C), dtype=torch.int64, device=ref.device)
    args = (ptr(vol), ptr(cls), n0, n1, n2, ptr(mats), B, H, W, C, ptr(img) if image else None, ptr(lab) if label_planes else None,
            label_planes)
    if disp is None and gain is None and ab is None:
        call("pnp_resample_planes", *args, rt.stream())
    else:
        disp, gain, ab = _aug_field("disp", disp, (B, 2, H, W)), _aug_field("gain", gain, (B, H, W)), _aug_field("ab", ab, (B, 2))
        call("pnp_resample_planes_aug", *args, ptr(disp), ptr(gain), ptr(ab), rt.stream())
    return (img if image else None), (lab if label_planes else None)


def smooth_noise_field(seed, stream_id, B, K, H, W, taps, amp, lo, hi, out=None, tmp=None):
    """A smoothed uniform noise field in one pnp_smooth_noise_field call (two launches; include/pnp_b200.h, "data augmentation"):
    out [B, K, H, W] = clamp(amp * s, lo, hi), s the Philox uniforms of (seed, stream_id) on [-1, 1) filtered along columns and
    then rows with `taps` (fp32 [2R + 1] on the device, preprocess.gaussian_taps).  `out` and `tmp` (the first pass, same shape)
    may be given to write into.  Returns out."""
    if not isinstance(taps, torch.Tensor) or not taps.is_cuda or taps.dtype != torch.float32 or taps.dim() != 1 or taps.numel() % 2 != 1:
        raise ValueError("smooth_noise_field: taps must be an odd-length fp32 vector on the device")
    shape = (B, K, H, W)
    for name, t in (("out", out), ("tmp", tmp)):
        if t is not None and (t.dtype != torch.float32 or tuple(t.shape) != shape or not t.is_contiguous()):
            raise ValueError("smooth_noise_field: %s must be contiguous fp32 %s" % (name, shape))
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=taps.device)
    if tmp is None:
        tmp = torch.empty(shape, dtype=torch.float32, device=taps.device)
    call("pnp_smooth_noise_field", int(seed) & 0xFFFFFFFFFFFFFFFF, int(stream_id) & 0xFFFFFFFFFFFFFFFF, B, K, H, W, ptr(taps),
         (taps.numel() - 1) // 2, float(amp), float(lo), float(hi), ptr(out), ptr(tmp), rt.stream())
    return out


def native_labels(scores, vmap, shape, gt=None, out=None):
    """A prepared-grid prediction sampled back onto a native grid in one pnp_native_labels launch (include/pnp_b200.h,
    "native-grid labels").  `scores` fp32 [n0, n1, n2, C] on the device, `vmap` fp32 [12] (device) from native voxel to prepared
    coordinate, `shape` the native (m0, m1, m2).  Returns (labels uint8 [m0, m1, m2], confusion counts int64 [C, C] (rows =
    truth) or None); `gt` uint8 [m0, m1, m2] on the device asks for the counts, `out` may be given to write into.
    An ensemble -- `scores` fp32 [K, n0, n1, n2, C] with `vmap` fp32 [K, 12], member k's scores and map -- is one
    pnp_native_labels_ensemble launch: the class scores of the members covering each native voxel are summed in ascending k
    before the argmax ("native-grid labels of an ensemble")."""
    scores, vmap = scores.contiguous(), vmap.contiguous()
    if scores.dim() == 5:
        K, n0, n1, n2, C = scores.shape
        if tuple(vmap.shape) != (K, 12):
            raise ValueError("native_labels: an ensemble of %d members needs vmap [%d, 12], got %s" % (K, K, tuple(vmap.shape)))
    else:
        K = None
        n0, n1, n2, C = scores.shape
    m0, m1, m2 = (int(s) for s in shape)
    if out is None:
        out = torch.empty(m0, m1, m2, dtype=torch.uint8, device=scores.device)
    cm = None
    if gt is not None:
        gt = gt.contiguous()
        if tuple(gt.shape) != (m0, m1, m2) or gt.dtype != torch.uint8:
            raise ValueError("native_labels: gt must be uint8 %s, got %s %s" % ((m0, m1, m2), tuple(gt.shape), gt.dtype))
        cm = torch.empty(C, C, dtype=torch.int64, device=scores.device)
    if K is None:
        call("pnp_native_labels", ptr(scores), n0, n1, n2, C, ptr(vmap), m0, m1, m2, ptr(out), ptr(gt), ptr(cm), rt.stream())
    else:
        call("pnp_native_labels_ensemble", ptr(scores), K, n0, n1, n2, C, ptr(vmap), m0, m1, m2, ptr(out), ptr(gt), ptr(cm),
             rt.stream())
    return out, cm


class NativeAccumulator(object):
    """Native-grid labels of any number of predictions (include/pnp_b200.h, "native-grid labels of any number of predictions"):
    fp32 sums [m0, m1, m2, C] and uint8 coverage flags [m0, m1, m2] on the device, zeroed once here.  `add(scores, vmap)` is one
    pnp_native_accumulate launch (scores fp32 [n0, n1, n2, C], vmap fp32 [12], both on the device); `labels(gt=None, out=None)` one
    pnp_native_accumulated_labels launch -> (labels uint8 [m0, m1, m2], confusion counts int64 [C, C] (rows = truth) or None), the
    labels pnp_native_labels_ensemble gives for the same predictions in the same order."""

    def __init__(self, shape, num_cls, device=None):
        self.shape = tuple(int(s) for s in shape)
        self.C = int(num_cls)
        device = rt.device() if device is None else device
        self.sums = torch.zeros(self.shape + (self.C,), dtype=torch.float32, device=device)
        self.covered = torch.zeros(self.shape, dtype=torch.uint8, device=device)
        self.count = 0

    def add(self, scores, vmap):
        scores, vmap = scores.contiguous(), vmap.contiguous()
        n0, n1, n2, C = scores.shape
        if C != self.C or tuple(vmap.shape) != (12,):
            raise ValueError("NativeAccumulator.add: scores [n0, n1, n2, %d] and vmap [12] expected, got %s and %s" % (
                self.C, tuple(scores.shape), tuple(vmap.shape)))
        m0, m1, m2 = self.shape
        call("pnp_native_accumulate", ptr(scores), n0, n1, n2, C, ptr(vmap), m0, m1, m2, ptr(self.sums), ptr(self.covered),
             rt.stream())
        self.count += 1

    def labels(self, gt=None, out=None):
        m0, m1, m2 = self.shape
        if out is None:
            out = torch.empty(self.shape, dtype=torch.uint8, device=self.sums.device)
        cm = None
        if gt is not None:
            gt = gt.contiguous()
            if tuple(gt.shape) != self.shape or gt.dtype != torch.uint8:
                raise ValueError("NativeAccumulator.labels: gt must be uint8 %s, got %s %s" % (self.shape, tuple(gt.shape), gt.dtype))
            cm = torch.empty(self.C, self.C, dtype=torch.int64, device=self.sums.device)
        call("pnp_native_accumulated_labels", ptr(self.sums), ptr(self.covered), m0, m1, m2, self.C, ptr(out), ptr(gt), ptr(cm),
             rt.stream())
        return out, cm


BOX_FIELDS = ("count", "lo0", "hi0", "lo1", "hi1", "lo2", "hi2")


def label_boxes(labels, num_cls):
    """host int64 [num_cls, 7]: per class (count, lo0, hi0, lo1, hi1, lo2, hi2) of `labels` (uint8 [n0, n1, n2] on the device;
    labels >= num_cls count as class 0), one pnp_label_boxes call; an empty class is (0, n0, -1, n1, -1, n2, -1)"""
    if not isinstance(labels, torch.Tensor) or not labels.is_cuda or labels.dtype != torch.uint8 or labels.dim() != 3:
        raise ValueError("label_boxes: labels must be a uint8 3-D tensor on the device")
    labels = labels.contiguous()
    out = torch.empty(int(num_cls), 7, dtype=torch.int64, device=labels.device)
    call("pnp_label_boxes", ptr(labels), *labels.shape, int(num_cls), ptr(out), rt.stream())
    return out.cpu().numpy()


COMPONENT_STATS = ("components", "kept", "removed")


def _u8_volume(name, v, shape=None):
    if not isinstance(v, torch.Tensor) or not v.is_cuda or v.dtype != torch.uint8 or v.dim() != 3:
        raise ValueError("largest_components: %s must be a uint8 3-D tensor on the device, got %s" % (
            name, (type(v).__name__ if not isinstance(v, torch.Tensor) else "%s %s on %s" % (v.dtype, tuple(v.shape), v.device))))
    if shape is not None and tuple(v.shape) != shape:
        raise ValueError("largest_components: %s must have the labels' shape %s, got %s" % (name, shape, tuple(v.shape)))


def largest_components(labels, num_cls, connectivity, gt=None, out=None):
    """The largest connected component of each class kept, everything else set to background, in one pnp_largest_components
    call (include/pnp_b200.h, "largest connected component per class").  `labels` uint8 [n0, n1, n2] on the device (labels
    >= num_cls count as background), `connectivity` 6 (face neighbours) or 26 (face, edge and corner neighbours).  Among
    components of equal size the one whose first voxel in C order comes first is kept.  Returns (out uint8 [n0, n1, n2] on the
    device, stats, cm): stats is a dict of host int64 arrays [num_cls] -- `components` (per class, in the input), `kept` and
    `removed` voxels (index 0: 0, 0 and the number of labels >= num_cls); `gt` uint8 [n0, n1, n2] on the device asks for the
    confusion counts cm[gt][out] (host int64 [num_cls, num_cls], rows = truth; else None).  `out` may be given to write into,
    `labels` itself included."""
    num_cls = int(num_cls)
    if not 2 <= num_cls <= 8:
        raise ValueError("largest_components: num_cls must be in [2, 8], got %d" % num_cls)
    if isinstance(connectivity, bool) or connectivity not in (6, 26):
        raise ValueError("largest_components: connectivity must be 6 or 26, got %r" % (connectivity,))
    _u8_volume("labels", labels)
    shape = tuple(labels.shape)
    if min(shape) < 1 or labels.numel() >= 1 << 31:
        raise ValueError("largest_components: every dimension must be >= 1 and the volume below 2^31 voxels, got %s" % (shape,))
    labels = labels.contiguous()
    if gt is not None:
        _u8_volume("gt", gt, shape)
        gt = gt.contiguous()
    if out is None:
        out = torch.empty(shape, dtype=torch.uint8, device=labels.device)
    else:
        _u8_volume("out", out, shape)
        if not out.is_contiguous():
            raise ValueError("largest_components: out must be contiguous")
    n0, n1, n2 = shape
    nbytes = ctypes.c_longlong(0)
    call("pnp_largest_components_workspace", n0, n1, n2, num_cls, int(connectivity), ctypes.byref(nbytes))
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=labels.device)
    stats = torch.empty(num_cls, 3, dtype=torch.int64, device=labels.device)
    cm = None if gt is None else torch.empty(num_cls, num_cls, dtype=torch.int64, device=labels.device)
    call("pnp_largest_components", ptr(labels), n0, n1, n2, num_cls, int(connectivity), ptr(out), ptr(gt), ptr(cm), ptr(stats),
         ptr(ws), nbytes.value, rt.stream())
    st = stats.cpu().numpy()
    return out, {k: st[:, i].copy() for i, k in enumerate(COMPONENT_STATS)}, (None if cm is None else cm.cpu().numpy())


def confusion_counts(logits, y):
    """[C,C] int64 confusion matrix (rows = truth) of argmax(logits) vs one-hot y (lib.py:96-110)."""
    logits, y = logits.contiguous(), y.contiguous()
    C = logits.shape[-1]
    cnt = torch.empty(C * C, dtype=torch.int64, device=logits.device)
    call("pnp_fill", ptr(cnt), 0.0, 2 * C * C, rt.stream())
    call("pnp_confusion", ptr(logits), ptr(y), logits.numel() // C, C, ptr(cnt), rt.stream())
    return cnt.view(C, C)


class _FCFn(torch.autograd.Function):
    """tf.matmul([B,F],[F,1]) (adversarial.py:397,440)"""

    @staticmethod
    def forward(ctx, x, w):
        x = x.contiguous()
        B, F = x.shape
        out = torch.empty(B, 1, dtype=x.dtype, device=x.device)
        call("pnp_fc_fwd", ptr(x), ptr(w), ptr(out), B, F, rt.stream())
        ctx.save_for_backward(x)
        ctx.w = w
        return out

    @staticmethod
    def backward(ctx, dout):
        (x,) = ctx.saved_tensors
        w = ctx.w
        B, F = x.shape
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw = _grad_slot(w) if w.requires_grad else None
        if dx is not None or dw is not None:
            call("pnp_fc_bwd", ptr(x), ptr(w), ptr(dout.contiguous()), ptr(dx), ptr(dw), B, F, rt.stream())
            if dw is not None:
                _grad_written(w)
        return dx, None


def fc(x, w):
    return _FCFn.apply(x, w)


class _MeanComboFn(torch.autograd.Function):
    """ca*mean(a) + cb*mean(b): the WGAN loss terms of adversarial.py:455-459"""

    @staticmethod
    def forward(ctx, a, ca, b, cb):
        a = a.contiguous()
        n = a.numel()
        out = torch.empty(1, dtype=a.dtype, device=a.device)
        call("pnp_mean_combo", ptr(a), float(ca), ptr(b.contiguous()) if b is not None else None, float(cb), n, ptr(out), rt.stream())
        ctx.meta = (ca, cb, n, a.shape, b is not None)
        return out[0]

    @staticmethod
    def backward(ctx, g):
        ca, cb, n, shape, has_b = ctx.meta
        def mk(c):
            t = torch.empty(shape, dtype=g.dtype, device=g.device)
            _bcast(t, g, float(c) / n)
            return t
        da = mk(ca) if ctx.needs_input_grad[0] else None
        db = mk(cb) if (has_b and ctx.needs_input_grad[2]) else None
        return da, None, db, None


def _bcast(t, g, c):
    """t[:] = c * g for a device scalar g: the FC backward kernel with B = 1 (dx[0, f] = dout[0] * w[f])."""
    F = t.numel()
    w = torch.empty(F, dtype=t.dtype, device=t.device)
    call("pnp_fill", ptr(w), float(c), F, rt.stream())
    call("pnp_fc_bwd", ptr(w), ptr(w), ptr(g.reshape(1).contiguous()), ptr(t), None, 1, F, rt.stream())


def mean_combo(a, ca, b=None, cb=0.0):
    return _MeanComboFn.apply(a, ca, b, cb)


def l2_loss_sum(tensors):
    """sum_i tf.nn.l2_loss(w_i) as a python float-on-device tensor (monitoring only)."""
    dev = tensors[0].device
    acc = _zeros_f64(1, dev)
    for t in tensors:
        call("pnp_l2_loss_acc", ptr(t), t.numel(), ptr(acc), rt.stream())
    return acc
