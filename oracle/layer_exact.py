"""fp64 references of ONE layer of the dispatcher (functional.layer_forward / layer_backward / _TailFn), stage by stage, each fed
the kernel's own inputs to that stage, with an a-priori per-element bound.

A layer is [mirror pad] -> conv -> dropout -> [BN] -> [+skip] -> [act].  Checking a real training step layer by layer, with each
stage's reference computed from what the kernels actually consumed (the bf16 operand planes, the kernel's z, mean, invstd, dy,
dz planes), keeps rounding from building up through depth: every bound below is per element and fixed before the run.

Every function returns (ref, bound) fp64 tensors, or a dict of them; a stage passes when |got - ref| <= bound at every element
(ratio() reports max |got - ref| / bound).  The bounds:
- wgmma convolutions: bf16_split.TAU[(launcher, nterms)] * sum|a||b| of the planes the kernel multiplies.  The weight gradient
  is the one launcher whose reduction grows with the batch: its bound follows the launch (tc_wgrad_split), TAU on each CTA's
  chain of pixels up to the longest chain TAU was measured at and a truncating-chain bound beyond it (tc_wgrad_tau), plus
  gamma_splits for the fp32 atomics that merge the CTAs;
- fp32 SIMT convolutions (conv_simt.cu) and the fused tail: gamma_n * sum|a||b|, with n the longest fp32 chain an output element
  goes through, whatever the order: the forward runs one FMA chain per element over kh*kw*Cin products, the data gradient over
  kh*kw*Cout, the tail forward over kh*kw*G; the tail's input gradient folds up to four mirrored positions per element,
  n = 4*kh*kw*Cout; the weight gradient runs a chain of m_per_split pixels per CTA and merges the splits with fp32 atomics
  (simt_wgrad_split restates launch_wgrad), n = m_per_split + splits.  gamma_n bounds every summation of that depth (Higham,
  Thm 3.4);
- a dropout multiplier fl32(1/keep) multiplies the fp32 result once more: + u |ref|;
- batch norm: the TAU of oracle/elementwise_exact.py (bn_finalize, bn_apply) on the magnitudes it defines, the inverse standard
  deviation conditioned by E[z^2] / (var + eps) (the one-pass variance cancels); the backward pass, which has no measured TAU,
  gamma_{PROMOTE_ROWS + 3} on the per-channel sums (fp32 partials of at most 64 rows before the fp64 promotion, three roundings
  in g * xhat) and 8u on the few fp32 operations of the apply;
- a result accumulated into an existing fp32 buffer (W.grad, gamma.grad, the merged skip gradient) adds u (|before| + |after|).
Everything is plain torch in fp64 and runs on any device."""
import torch

from . import bf16_split as S
from . import elementwise_exact as E
from . import simt_exact as X

U = 2.0 ** -24
NONE, RELU, LRELU = E.NONE, E.RELU, E.LRELU
# |x - (hi + lo)| <= SPLIT_REL * |x| of the operand split: bf16 keeps 8 significant bits, so hi is within 2^-8 |x| (nterms 1) and
# lo = rn(x - hi) within 2^-8 |x - hi| <= 2^-16 |x| (nterms 3)
SPLIT_REL = {3: 2.0 ** -16, 1: 2.0 ** -8}
TAU_BN_BWD_SUM = X.gamma(E.PROMOTE_ROWS + 3)
TAU_BN_BWD_APPLY = 8 * U
WGRAD_K_MEASURED = 2048      # the longest weight-gradient chain (pixels) bf16_split.TAU was measured at


def d(t):
    return None if t is None else t.to(torch.float64)


def gamma(n):
    return X.gamma(n)


# ------------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------------
def ratio(got, ref, bound):
    """max over elements of |got - ref| / bound (0 where they are equal; inf where got is not finite or bound is 0 and they
    differ)"""
    got = d(got)
    if not bool(torch.isfinite(got).all()):
        return float("inf")
    err = (got - ref).abs()
    if err.numel() == 0:
        return 0.0
    r = torch.where(err == 0, torch.zeros_like(err), err / bound)
    return float(r.max())


def with_mask(ref, bound, mask):
    """the dropout multiplier applied to an fp32 result: one more rounding"""
    if mask is None:
        return ref, bound
    m = d(mask)
    ref = ref * m
    return ref, bound * m.abs() + U * ref.abs()


def accumulated(ref, bound, before):
    """ref added onto an fp32 buffer holding `before`: one rounding of the sum"""
    if before is None:
        return ref, bound
    out = ref + d(before)
    return out, bound + U * (d(before).abs() + out.abs())


# ------------------------------------------------------------------------------------------------
# convolutions
# ------------------------------------------------------------------------------------------------
def geom(g):
    """functional's ConvGeom (ctypes) -> bf16_split.Geom"""
    return S.Geom(g.B, g.H, g.W, g.Cin, g.Ho, g.Wo, g.Cout, g.kh, g.kw, g.stride, g.dil, g.pad_t, g.pad_l)


def _planes64(hi, lo, nterms):
    return d(hi), (d(lo) if nterms == 3 else torch.zeros_like(d(hi)))


def _w_planes(W, nterms):
    hi, lo = S.split(W)
    return _planes64(hi, lo, nterms)


def fwd_tc(x_hi, x_lo, W, g, nterms, mask=None):
    """z of the wgmma forward from the x planes it consumed and split(W)"""
    xh, xl = _planes64(x_hi, x_lo, nterms)
    wh, wl = _w_planes(W, nterms)
    ref, cond = S.fwd_ref(xh, xl, wh, wl, g, nterms)
    return with_mask(ref, S.TAU[("fwd", nterms)] * cond, mask)


def fwd_simt(xp, W, g, mask=None):
    ref = S.fwd_bilinear(d(xp), d(W), g)
    cond = S.fwd_bilinear(d(xp).abs(), d(W).abs(), g)
    return with_mask(ref, gamma(g.kh * g.kw * g.Cin) * cond, mask)


def mirror_fold(dxp, p):
    """adjoint of the SYMMETRIC pad by p on NHWC: every padded position adds into its source"""
    B, Hp, Wp, C = dxp.shape
    H, W = Hp - 2 * p, Wp - 2 * p
    iy = torch.tensor(X.mirror_index(H, p), device=dxp.device)
    ix = torch.tensor(X.mirror_index(W, p), device=dxp.device)
    rows = torch.zeros(B, H, Wp, C, dtype=dxp.dtype, device=dxp.device).index_add_(1, iy, dxp)
    return torch.zeros(B, H, W, C, dtype=dxp.dtype, device=dxp.device).index_add_(2, ix, rows)


def _dgrad_finish(ref, bound, cond, p, into):
    if p:
        # the fold adds at most four fp32 values per element
        ref, bound = mirror_fold(ref, p), mirror_fold(bound, p) + gamma(3) * mirror_fold(cond, p)
    return accumulated(ref, bound, into)


def dgrad_tc(dz_hi, dz_lo, W, g, nterms, p=0, into=None):
    """dx of the wgmma data gradient from the kernel's dz planes and split(W); p: fold through a SYMMETRIC pad; into: dx_into
    as it was before the call"""
    dh, dl = _planes64(dz_hi, dz_lo, nterms)
    wh, wl = _w_planes(W, nterms)
    ref, cond = S.dgrad_ref(dh, dl, wh, wl, g, nterms)
    return _dgrad_finish(ref, S.TAU[("dgrad", nterms)] * cond, cond, p, into)


def dgrad_simt(dz, W, g, p=0, into=None):
    ref = S.dgrad_bilinear(d(dz), d(W), g)
    cond = S.dgrad_bilinear(d(dz).abs(), d(W).abs(), g)
    return _dgrad_finish(ref, gamma(g.kh * g.kw * g.Cout) * cond, cond, p, into)


def _cdiv(a, b):
    return -(-a // b)


def simt_wgrad_split(g):
    """(pixels per CTA chain, splits) of pnp_conv2d_wgrad: launch_wgrad of conv_simt.cu aims at ~6 CTAs per SM, keeps at least 4
    reduction blocks of BR pixels per CTA, rounds the pixels per split up to BR and merges the splits with fp32 atomics"""
    inst, _ = X.simt_instance("wgrad", g)
    BKK, BN, BR = (int(v) for v in inst[inst.index("<") + 1:-1].split(",")[:3])
    M, KK = g.B * g.Ho * g.Wo, g.kh * g.kw * g.Cin
    tiles = _cdiv(KK, BKK) * _cdiv(g.Cout, BN)
    splits = min(max((X.NUM_SMS * 6 + tiles - 1) // tiles, 1), _cdiv(M, BR * 4))
    splits = min(max(splits, 1), 65535)
    mps = _cdiv(_cdiv(M, splits), BR) * BR
    return mps, _cdiv(M, mps)


def tc_wgrad_split(g, sms=X.NUM_SMS, x_channels=0):
    """(pixels per CTA chain, splits) of pnp_conv2d_tc_wgrad (conv_tc.cu): blocks of 64 pixels (choose_tile, exact), tiles of
    packed taps x 128 input channels x 64 / 128 output channels, splits = 2 * SMs / tiles clamped to [1, blocks / 4], merged with
    fp32 atomics.  x_channels: channel count of the x planes the launcher was given (0: Cin)"""
    xc = x_channels or g.Cin
    rows = 64
    if g.Cout % 64:
        return g.B * g.Ho * g.Wo, 1       # a geometry the launcher declines: one chain over the whole reduction
    if g.Wo >= rows:
        tw, th, tn = rows, 1, 1
    else:
        tw, th = g.Wo, min(rows // g.Wo, g.Ho)
        tn = max(rows // (tw * th), 1) if th == g.Ho else 1
    num_pb = (g.Wo // tw) * (g.Ho // th) * _cdiv(g.B, tn)
    pack = 2 if (g.Cin == 64 and xc == 64) else (4 if (g.Cin == 32 and xc == 32) else 1)
    tiles = _cdiv(g.kh * g.kw, pack) * _cdiv(g.Cin, 128) * (g.Cout // (128 if g.Cout % 128 == 0 else 64))
    splits = min((2 * sms) // tiles, max(num_pb // 4, 1))
    splits = max(splits, 1)
    pb = _cdiv(num_pb, splits)
    return pb * rows, _cdiv(num_pb, pb)


def tc_wgrad_tau(chain, nterms):
    """per-CTA tolerance of the wgmma weight gradient over a chain of `chain` pixels: bf16_split.TAU[("wgrad", nterms)] up to the
    longest chain it was measured at; beyond it, the bound of nterms * chain / 16 fp32 additions into one accumulator (the kernel
    issues one wgmma of 16 products per split term and k-step: lo*hi, hi*lo, hi*hi) that each truncate rather than round, 2u each"""
    tau = S.TAU[("wgrad", nterms)]
    return tau if chain <= WGRAD_K_MEASURED else max(tau, 2 * U * (nterms * chain / 16 + 1))


def _split_sum(ref, cond, tau_chain, splits, before):
    """partial sums within tau_chain * cond each, merged by `splits` fp32 atomics onto `before`: every atomic rounds the running
    value once, so that stage adds gamma_splits * (|before| + sum|a||b|)"""
    bound = (tau_chain + gamma(splits)) * cond
    if before is None:
        return ref, bound
    return ref + d(before), bound + gamma(splits) * d(before).abs()


def wgrad_tc(x_hi, x_lo, dz_hi, dz_lo, g, nterms, before=None, sms=X.NUM_SMS, x_channels=0):
    xh, xl = _planes64(x_hi, x_lo, nterms)
    dh, dl = _planes64(dz_hi, dz_lo, nterms)
    ref, cond = S.wgrad_ref(xh, xl, dh, dl, g, nterms)
    chain, splits = tc_wgrad_split(g, sms, x_channels)
    return _split_sum(ref, cond, tc_wgrad_tau(chain, nterms), splits, before)


def wgrad_simt(xp, dz, g, before=None):
    """each CTA runs one fp32 FMA chain of m_per_split pixels per element, the splits are merged with fp32 atomics:
    gamma_{m_per_split} on the chains, gamma_splits on the atomics"""
    ref = S.wgrad_bilinear(d(xp), d(dz), g)
    cond = S.wgrad_bilinear(d(xp).abs(), d(dz).abs(), g)
    mps, splits = simt_wgrad_split(g)
    return _split_sum(ref, cond, gamma(mps), splits, before)


# ------------------------------------------------------------------------------------------------
# batch norm forward, activation, skip
# ------------------------------------------------------------------------------------------------
def bn_train_stats(z, gamma_, beta, mm0, mv0):
    """mean, invstd and the moving statistics after a training-mode BN over the kernel's z [.., C]; mm0 / mv0 are the moving
    statistics before the layer -> {name: (ref, bound)}"""
    C = z.shape[-1]
    zf = d(z).reshape(-1, C)
    M = zf.shape[0]
    s1, s2, sabs = E.bn_stats_ref(zf)
    r = E.bn_finalize_ref(s1, s2, M, gamma_, beta, mm0, mv0, 1, s_abs=sabs)
    tau = E.TAU["bn_finalize"]
    mean = s1 / M
    var = (s2 / M - mean * mean).clamp_min(0)
    out = {k: (r[k][0], tau * r[k][1]) for k in ("mean", "moving_mean", "moving_var")}
    inv = r["invstd"][0]
    out["invstd"] = (inv, tau * inv * (1 + (s2 / M) / (var + E.BN_EPS)))
    return out


LEAK32 = float(torch.tensor(E.LEAK, dtype=torch.float32))    # the kernels' 0.2f
FLUSH = 2.0 ** -126          # the producers flush positive subnormal activations to +0


def act64(v, act):
    """the activation in fp64 with the kernels' slope 0.2f"""
    if act == NONE:
        return v
    return torch.where(v > 0, v, torch.zeros_like(v) if act == RELU else LEAK32 * v)


def slope64(y, act):
    """act'(y) taken from the sign of the kernel's y (or of its bf16 hi plane)"""
    one = torch.ones(y.shape, dtype=torch.float64, device=y.device)
    if act == NONE:
        return one
    return torch.where(y > 0, one, torch.zeros_like(one) if act == RELU else torch.full_like(one, LEAK32))


def _epilogue(zs, shift, mag, skip, skip_off, act):
    """act(zs + shift + skip) on [M, C] rows -> (y, magnitude); skip has Cs channels placed at skip_off"""
    v = zs + shift
    if skip is not None:
        sk = d(skip).reshape(zs.shape[0], -1)
        Cs = sk.shape[1]
        v[:, skip_off:skip_off + Cs] += sk
        mag[:, skip_off:skip_off + Cs] += sk.abs()
    return act64(v, act), mag


def bn_apply(z, mean, invstd, gamma_, beta, skip=None, skip_off=0, act=NONE):
    """y = act(z * scale + shift + skip) from the kernel's z, mean and invstd (training mode), or the moving statistics' mean
    and invstd (inference mode) -> (ref, bound)"""
    C = z.shape[-1]
    scale = d(gamma_) * d(invstd)
    shift = d(beta) - d(mean) * scale
    zs = d(z).reshape(-1, C) * scale
    y, mag = _epilogue(zs, shift, zs.abs() + d(beta).abs() + (d(mean) * scale).abs(), skip, skip_off, act)
    bound = E.TAU["bn_apply"] * mag + (FLUSH if act != NONE else 0.0)
    return y.reshape(z.shape), bound.reshape(z.shape)


def act_apply(z, skip=None, skip_off=0, act=NONE):
    """y = act(z + skip) of a layer without batch norm (pnp_bn_act_apply)"""
    C = z.shape[-1]
    one = torch.ones(C, dtype=torch.float64, device=z.device)
    return bn_apply(z, torch.zeros_like(one), one, one, torch.zeros_like(one), skip, skip_off, act)


def moving_coef(gamma_, beta, mm, mv):
    """(scale, shift, magnitude of shift) of an inference-mode BN in fp64 from the moving statistics"""
    inv = 1.0 / torch.sqrt(d(mv) + E.BN_EPS)
    scale = d(gamma_) * inv
    return scale, d(beta) - d(mm) * scale, d(beta).abs() + (d(mm) * scale).abs()


def fused_epilogue(conv_ref, conv_bound, scale=None, shift=None, shift_mag=None, skip=None, skip_off=0, act=NONE):
    """y of the wgmma forward with the epilogue act(acc * scale + shift + skip): the convolution's bound carried through |scale|,
    plus TAU["bn_apply"] on the magnitude of the epilogue, whose fp32 shift = beta - mean * scale carries the rounding of both
    terms (shift_mag = |beta| + |mean * scale|; an element the dropout zeroed is the shift alone)"""
    C = conv_ref.shape[-1]
    if scale is None:
        scale = torch.ones(C, dtype=torch.float64, device=conv_ref.device)
        shift = shift_mag = torch.zeros_like(scale)
    zs = conv_ref.reshape(-1, C) * scale
    y, mag = _epilogue(zs, shift, zs.abs() + shift_mag, skip, skip_off, act)
    bound = E.TAU["bn_apply"] * mag + conv_bound.reshape(-1, C) * scale.abs() + (FLUSH if act != NONE else 0.0)
    return y.reshape(conv_ref.shape), bound.reshape(conv_ref.shape)


def planes_value(hi, lo, nterms):
    """(hi + lo) of a planes-only tensor and the split's own relative error"""
    v = d(hi) + (d(lo) if nterms == 3 and lo is not None else 0.0)
    return v, SPLIT_REL[nterms]


# ------------------------------------------------------------------------------------------------
# activation / batch norm backward
# ------------------------------------------------------------------------------------------------
def layer_bwd(dy, y_sign, act, z=None, mean=None, invstd=None, gamma_=None, training=False, mask=None):
    """the elementwise backward of one layer from the kernel's dy, the sign source of the activation (y, or its bf16 hi
    plane), z, mean, invstd and gamma (None without batch norm) and the dropout multipliers -> {"g", "dz", ["dgamma", "dbeta"]}
    as (ref, bound); dgamma / dbeta are this call's contributions"""
    C = dy.shape[-1]
    shape = dy.shape
    dyf = dy.reshape(-1, C)
    gd = d(dyf) * slope64(d(y_sign).reshape(-1, C), act) if act != NONE else d(dyf)
    out = {"g": (gd.reshape(shape), U * gd.abs().reshape(shape))}
    m = None if mask is None else mask.reshape(-1, C)
    if gamma_ is None:
        ref, bound = with_mask(gd, U * gd.abs(), m)
        out["dz"] = (ref.reshape(shape), bound.reshape(shape))
        return out
    M = dyf.shape[0]
    k = d(gamma_) * d(invstd)
    if not training:
        pre, bound = gd, k.abs() * TAU_BN_BWD_APPLY * gd.abs()
    if z is None:
        # an inference-mode layer folded into the convolution's epilogue keeps no z: its parameters take no gradient
        ref, bound = with_mask(k * pre, bound, m)
        out["dz"] = (ref.reshape(shape), bound.reshape(shape))
        return out
    # (the inference-mode parameter gradients use the moving statistics' mean and invstd the same way)
    xhat = (d(z).reshape(-1, C) - d(mean)) * d(invstd)
    gx = gd * xhat
    sg, sgx, sga, sgxa = gd.sum(0), gx.sum(0), gd.abs().sum(0), gx.abs().sum(0)
    c1, c2 = sg / M, sgx / M
    if training:
        pre = gd - c1 - xhat * c2
        bound = k.abs() * (TAU_BN_BWD_SUM * (sga / M + xhat.abs() * sgxa / M) + TAU_BN_BWD_APPLY * (gd.abs() + c1.abs() + (xhat * c2).abs()))
    ref, bound = with_mask(k * pre, bound, m)
    out["dz"] = (ref.reshape(shape), bound.reshape(shape))
    out["dgamma"] = (sgx, TAU_BN_BWD_SUM * sgxa)
    out["dbeta"] = (sg, TAU_BN_BWD_SUM * sga)
    return out


# ------------------------------------------------------------------------------------------------
# the fused segmenter tail
# ------------------------------------------------------------------------------------------------
def tail_fwd(X_, w, t):
    """y of pnp_ps_mirror_conv_fwd: one FMA chain of kh*kw*G products per element"""
    ref, cond = X.tail_fwd_ref(d(X_), d(w), t)
    return ref, gamma(t.kh * t.kw * t.G) * cond


def tail_bwd(dy, w, t):
    """dX of pnp_ps_mirror_conv_bwd: at most 4*kh*kw*Cout products per element (the mirror fold)"""
    ref, cond = X.tail_bwd_ref(d(dy), d(w), t)
    return ref, gamma(4 * t.kh * t.kw * t.Cout) * cond
