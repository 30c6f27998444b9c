"""fp64 references of the batch-norm, activation, loss and metric kernels of elementwise.cu, in their C-ABI layouts, and a
restatement of their launch configuration.

Layouts are those of include/pnp_b200.h: activations are [M, C] rows (NHWC flattened), a residual skip has Cs channels placed at
channel offset skip_off, BN sums are fp64 [C], the BN backward coef is [c1 (C) | c2 (C)], the seg-loss accumulator acc[4C] is
[sum y | sum p*y | sum p*p | sum -y*log(clip(p, .005, 1))] and its coef[3C] is [w/P | -(2/C)/D | (4/C)*inse/D^2].

Each reference returns, next to its value, the magnitude its error bound scales with: sum|terms| for a sum, E[z^2] for a
variance, and for a short expression the same expression evaluated on absolute values.  The real-valued checks of
tests/test_elementwise_exact_gpu.py require |got - ref| <= TAU[key] * magnitude at every element.

Everything is plain torch in fp64 and runs on any device."""
from collections import namedtuple

import torch

NUM_SMS = 132                 # PNP_NUM_SMS of common.cuh: the grid rules are compiled for an H100 SXM, whatever the device
BN_EPS = 1e-3
BN_DECAY = 0.9
LEAK = 0.2
NONE, RELU, LRELU = 0, 1, 2   # PNP_ACT_*
PROMOTE_ROWS = 64             # bn_reduce_kernel promotes its fp32 partial sums to fp64 every 32 two-row iterations
F32_EXACT = 2.0 ** 24         # integers below this are exact in fp32

# Per-element tolerances of the real-valued checks, |got - ref| <= TAU * magnitude.  Each is about 3x the worst ratio measured
# over every real-valued case of tests/test_elementwise_exact_gpu.py on an H100 SXM (80 GB HBM3, 400 W power limit).
TAU = {
    "bn_var": 1.5e-7,         # one-pass variance from pnp_bn_stats sums, magnitude E[z^2]: measured 4.96e-8 (M 32, mean/std 10)
    "bn_finalize": 8.2e-7,    # mean / invstd / scale / shift / moving averages: measured 2.72e-7, set by the moving mean, whose
                              # fp32 weights 0.9f and 1 - 0.9f = 0.10000002 differ from 0.9 / 0.1 by up to 2.4e-7
    "bn_apply": 5.0e-7,       # y of the training-mode pnp_bn_apply_fused: measured 1.66e-7 (M 8192)
    "seg_sums": 1.4e-8,       # sum y, sum p*y, sum p*p of pnp_segloss_reduce: measured 4.63e-9 (C 8, P 524288)
    "seg_ce": 2.0e-8,         # sum -y*log(clip p), magnitude sum |y|(|log clip p| + 1): measured 6.54e-9
    "seg_finalize": 1.7e-7,   # out[0..1] and coef of pnp_segloss_finalize from the kernel's own acc: measured 5.74e-8
    "seg_bwd": 1.6e-5,        # dlogits of pnp_segloss_bwd from the kernel's own coef: measured 5.48e-6 (C 8); it grows with C
                              # (1.2e-6 at C 2), as the spread of the randn * 3 logits does: p carries the fp32 rounding of l - max l
}
# pnp_bn_finalize's invstd (rsqrtf and one Newton step) is within this many fp32 ulps of the correctly rounded 1/sqrt(fl(var + eps))
# over 0, subnormals, the neighbourhood of eps and up to 1e30: measured on 2^20 variances, 84.1 % exact, 15.9 % at 1 ulp and 19
# values at 2 ulps (the sweep is deterministic, so the bound is the measured maximum).
INVSTD_ULP = 2


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------
# launch configuration
# ------------------------------------------------------------------------------------------------
ReduceCfg = namedtuple("ReduceCfg", "tpr rstep rpb grid capped rows_per_thread")


def reduce_launch_cfg(M, C):
    """reduce_launch_cfg of elementwise.cu (pnp_bn_stats, pnp_bn_bwd_reduce, pnp_bn_bwd_reduce_sums), or None where it declines:
    tpr threads per row (one per channel quad, rounded up to a power of two), rstep = 256 / tpr row lanes, rpb rows per CTA
    (8 per row lane, or M / (8 * 132) when the grid would exceed one wave of 8 CTAs per SM), the grid, whether that cap
    applied, and the most rows one thread sums"""
    if C <= 0 or M <= 0 or C % 4 or C > 1024:
        return None
    t = 1
    while t < C // 4:
        t <<= 1
    rstep = 256 // t
    rows = rstep * 8
    g = _cdiv(M, rows)
    cap = NUM_SMS * 8
    capped = g > cap
    if capped:
        rows = _cdiv(M, cap)
    return ReduceCfg(t, rstep, rows, _cdiv(M, rows), capped, _cdiv(min(rows, M), rstep))


def _lane_rows(n, rstep):
    return [max(0, _cdiv(n - l, rstep)) for l in range(rstep)]


def reduce_regimes(M, C):
    """the set of bn_reduce_kernel regimes a launch reaches"""
    cfg = reduce_launch_cfg(M, C)
    tags = {"tpr%d" % cfg.tpr}
    if C // 4 < cfg.tpr:
        tags.add("idle_lanes")
    last = M - (cfg.grid - 1) * cfg.rpb
    if last != cfg.rpb:
        tags.add("ragged")
    if any(r % 2 for n in (cfg.rpb, last) for r in _lane_rows(n, cfg.rstep)):
        tags.add("odd_rows")          # a thread's last iteration has no second row (hasB false)
    if M < cfg.rstep:
        tags.add("m_lt_rstep")
    if cfg.capped:
        tags.add("capped")
    if cfg.rows_per_thread > PROMOTE_ROWS:
        tags.add("promoted")
    return tags


def grid_for(work_items, per_block):
    """grid_for of elementwise.cu: one CTA per per_block items, at least 1, at most 64 per SM (the kernels grid-stride)"""
    return int(min(max(_cdiv(work_items, per_block), 1), NUM_SMS * 64))


# ------------------------------------------------------------------------------------------------
# activations
# ------------------------------------------------------------------------------------------------
def act_fwd(v, act):
    """the activation in fp32 as the kernels apply it: positive subnormals flush to +0, leaky ReLU multiplies by 0.2f"""
    v = v.to(torch.float32)
    if act == NONE:
        return v
    tiny = 2.0 ** -126
    if act == RELU:
        return torch.where(v >= tiny, v, torch.zeros_like(v))
    return torch.where(v >= tiny, v, torch.where(v > 0, torch.zeros_like(v), v * torch.tensor(LEAK, dtype=torch.float32)))


def act_slope(y, act, slope_at_zero=None):
    """act'(y) as fp32: 1 for y > 0, else 0 (ReLU) or 0.2f (leaky ReLU); slope_at_zero overrides y == 0 (a negative control)"""
    one = torch.ones_like(y, dtype=torch.float32)
    if act == NONE:
        return one
    low = torch.zeros_like(one) if act == RELU else torch.full_like(one, LEAK)
    s = torch.where(y > 0, one, low)
    if slope_at_zero is not None:
        s = torch.where(y == 0, torch.full_like(one, slope_at_zero), s)
    return s


# ------------------------------------------------------------------------------------------------
# batch norm forward
# ------------------------------------------------------------------------------------------------
def bn_stats_ref(z):
    """-> (sum, sumsq, sum|z|) per channel of z [M, C]"""
    z = z.double()
    return z.sum(0), (z * z).sum(0), z.abs().sum(0)


def bn_moments(z):
    """-> (mean, two-pass biased variance, E[z^2]) per channel"""
    z = z.double()
    m = z.mean(0)
    return m, ((z - m) ** 2).mean(0), (z * z).mean(0)


def bn_finalize_ref(s1, s2, M, gamma, beta, mm, mv, training, s_abs=None, unbiased=True):
    """pnp_bn_finalize from fp64 sums -> dict of (value, magnitude) for mean, invstd, scale, shift, moving_mean, moving_var.
    training == 0: the moving statistics.  s_abs = sum|z| (magnitude of the mean; default |sum|).  unbiased=False uses the
    biased variance in the moving average (a negative control)."""
    d = lambda t: t.double()  # noqa: E731
    gamma, beta, mm, mv = d(gamma), d(beta), d(mm), d(mv)
    if training:
        s1, s2 = d(s1), d(s2)
        mean = s1 / M
        var = (s2 / M - mean * mean).clamp_min(0)
        m_abs = (s1.abs() if s_abs is None else d(s_abs)) / M
        unb = var * (M / (M - 1)) if (M > 1 and unbiased) else var
        e2 = s2 / M
        new_mm = BN_DECAY * mm + (1 - BN_DECAY) * mean
        new_mv = BN_DECAY * mv + (1 - BN_DECAY) * unb
        mm_mag = BN_DECAY * mm.abs() + (1 - BN_DECAY) * m_abs
        mv_mag = BN_DECAY * mv.abs() + (1 - BN_DECAY) * e2 * (M / (M - 1) if M > 1 else 1.0)
    else:
        mean, var, m_abs = mm, mv, mm.abs()
        new_mm, new_mv, mm_mag, mv_mag = mm, mv, mm.abs(), mv.abs()
    invstd = 1.0 / torch.sqrt(var + BN_EPS)
    scale = gamma * invstd
    shift = beta - mean * scale
    return {"mean": (mean, m_abs), "invstd": (invstd, invstd), "scale": (scale, scale.abs()),
            "shift": (shift, beta.abs() + (m_abs * scale).abs()), "moving_mean": (new_mm, mm_mag),
            "moving_var": (new_mv, mv_mag)}


def bn_apply_ref(z, scale, shift, skip=None, skip_off=0, act=NONE, shift_mag=None):
    """y = act(z * scale + shift + skip) -> (y as fp32 via act_fwd, magnitude |z*scale| + |shift| + |skip|).  The pre-activation
    is formed in fp64; the activation is applied in fp32 (exact for ReLU, one rounding of 0.2f*v for leaky ReLU)"""
    z = z.double()
    v = z * scale.double() + shift.double()
    mag = (z * scale.double()).abs() + (shift.double().abs() if shift_mag is None else shift_mag.double())
    if skip is not None:
        Cs = skip.shape[1]
        v[:, skip_off:skip_off + Cs] += skip.double()
        mag[:, skip_off:skip_off + Cs] += skip.double().abs()
    return act_fwd(v, act), mag


# ------------------------------------------------------------------------------------------------
# batch norm backward
# ------------------------------------------------------------------------------------------------
def bn_bwd_reduce_ref(dy, y, z, mean, invstd, act, slope_at_zero=None):
    """g = dy * act'(y) (fp32), sum_g, sum_gx = sum g * (z - mean) * invstd -> (g, sum_g, sum_gx, sum|g|, sum|g xhat|)"""
    g = dy.float() * act_slope(y, act, slope_at_zero) if act != NONE else dy.float()
    xhat = (z.double() - mean.double()) * invstd.double()
    gx = g.double() * xhat
    return g, g.double().sum(0), gx.sum(0), g.double().abs().sum(0), gx.abs().sum(0)


def bn_bwd_finalize_ref(sum_g, sum_gx, M):
    """coef = [sum_g / M | sum_gx / M]"""
    return torch.cat([sum_g.double() / M, sum_gx.double() / M])


def bn_bwd_apply_ref(g, z, mean, invstd, gamma, c1, c2, training, mask=None, c2_invstd=True):
    """dz = gamma * invstd * (g - c1 - (z - mean) * invstd * c2) (training) or gamma * invstd * g, in fp64, then the dropout
    multiplier as the final fp32 multiply -> (dz fp32, magnitude).  c2_invstd=False drops the invstd of the c2 term (a negative
    control)."""
    d = lambda t: t.double()  # noqa: E731
    k = d(gamma) * d(invstd)
    if training:
        xs = (d(z) - d(mean)) * (d(invstd) if c2_invstd else 1.0)
        pre = d(g) - d(c1) - xs * d(c2)
        mag = k.abs() * (d(g).abs() + d(c1).abs() + (xs * d(c2)).abs())
    else:
        pre = d(g)
        mag = k.abs() * d(g).abs()
    dz = (k * pre).float()
    if mask is not None:
        dz = dz * mask.float()
        mag = mag * mask.double().abs()
    return dz, mag


# ------------------------------------------------------------------------------------------------
# losses and metrics
# ------------------------------------------------------------------------------------------------
CLIP = 0.005


def softmax64(logits):
    return torch.softmax(logits.double(), dim=-1)


def segloss_reduce_ref(logits, y, drop_pixel=None):
    """acc[4C] of pnp_segloss_reduce for logits, y [P, C] -> (acc, magnitude).  The CE magnitude is sum |y| (|log clip p| + 1):
    the log has an absolute, not a relative, error where p is near 1.  drop_pixel leaves one pixel out (a negative control)."""
    p, yd = softmax64(logits), y.double()
    if drop_pixel is not None:
        keep = torch.ones(p.shape[0], 1, dtype=torch.float64, device=p.device)
        keep[drop_pixel] = 0
        yd, p = yd * keep, p * keep
    lg = torch.log(p.clamp(CLIP, 1.0))
    acc = torch.cat([yd.sum(0), (p * yd).sum(0), (p * p).sum(0), (-yd * lg).sum(0)])
    mag = torch.cat([yd.abs().sum(0), (p * yd).abs().sum(0), (p * p).sum(0), (yd.abs() * (lg.abs() + 1)).sum(0)])
    return acc, mag


def segloss_finalize_ref(acc, P, C):
    """pnp_segloss_finalize from acc -> (out[2], out magnitude, coef[3C])"""
    acc = acc.double()
    sy, inse, l, ce = acc[:C], acc[C:2 * C], acc[2 * C:3 * C], acc[3 * C:]
    w = 1.0 - sy / sy.sum()
    D = l + sy + 1e-7
    out = torch.stack([(w * ce).sum() / P, -(2.0 * inse / D).sum() / C])
    mag = torch.stack([(w * ce).abs().sum() / P, (2.0 * inse / D).abs().sum() / C])
    coef = torch.cat([w / P, -(2.0 / C) / D, (4.0 / C) * inse / (D * D)])
    return out, mag, coef


def segloss_bwd_ref(logits, y, coef, g_wce, g_dice, clip_strict=False):
    """dlogits = p * (dp - sum_c dp_c p_c), dp = g_dice (coef1 y + coef2 p) + [p >= .005] g_wce (-coef0 y / p) -> (dlogits,
    magnitude).  clip_strict=True gates the CE term with p > .005 (a negative control)."""
    C = logits.shape[1]
    p, yd, cf = softmax64(logits), y.double(), coef.double()
    c0, c1, c2 = cf[:C], cf[C:2 * C], cf[2 * C:]
    gate = (p > CLIP) if clip_strict else (p >= CLIP)
    t_dice = g_dice * (c1 * yd + c2 * p)
    t_ce = torch.where(gate, g_wce * (-c0 * yd / p), torch.zeros_like(p))
    dp = t_dice + t_ce
    dp_abs = (g_dice * (c1 * yd).abs() + abs(g_dice) * (c2 * p).abs() + t_ce.abs()).abs()
    dot = (dp * p).sum(1, keepdim=True)
    dot_abs = (dp_abs * p).sum(1, keepdim=True)
    return p * (dp - dot), p * (dp_abs + dot_abs)


def confusion_ref(logits, y):
    """counts[C * C] (rows = truth), argmax resolving ties to the first maximum"""
    C = logits.shape[1]
    pa, ya = logits.argmax(1), y.argmax(1)
    return torch.bincount(ya * C + pa, minlength=C * C)


def l2_ref(w):
    return 0.5 * (w.double() ** 2).sum()


def fc_fwd_ref(x, w):
    return x.double() @ w.double()


def fc_bwd_ref(x, w, dout):
    """-> (dx [B, F], dw [F]) of out = x @ w"""
    return dout.double()[:, None] * w.double()[None, :], (dout.double()[:, None] * x.double()).sum(0)


def mean_combo_ref(a, ca, b, cb):
    """ca * mean(a) + cb * mean(b): the fp64 sum, rounded to fp32 and divided by n in fp32 (the kernel's final division)"""
    n = a.numel()
    s = ca * a.double().sum() + (cb * b.double().sum() if b is not None else 0.0)
    return s.float() / torch.tensor(float(n), dtype=torch.float32)


# ------------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------------
def worst_ratio(got, ref, mag):
    r = (got.double() - ref.double()).abs() / mag.double().clamp_min(1e-300)
    r = torch.where((got.double() == ref.double()), torch.zeros_like(r), r)
    return float(r.max()) if r.numel() else 0.0


def violations(got, ref, mag, tau):
    return int(((got.double() - ref.double()).abs() > tau * mag.double()).sum())


def f32_ulp_distance(a, b):
    """|a - b| in fp32 ulps, for finite non-negative fp32 tensors"""
    ia = a.float().contiguous().view(torch.int32).to(torch.int64)
    ib = b.float().contiguous().view(torch.int32).to(torch.int64)
    return (ia - ib).abs()


def rsqrt_f32_ref(var_f32):
    """1 / sqrt(fl32(var + 1e-3f)), rounded once from fp64 to fp32"""
    x = var_f32.float() + torch.tensor(BN_EPS, dtype=torch.float32)
    return (1.0 / torch.sqrt(x.double())).float()
