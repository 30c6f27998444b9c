"""fp64 references of the optimizer steps of elementwise.cu (pnp_adam_advance, pnp_adam_step, pnp_rmsprop_step,
pnp_momentum_step), restating the C-ABI contract of include/pnp_b200.h per element, and the dyadic operands on which the
kernels must agree with them bit for bit.

The contract, per element i of an arena of n = 1024 k elements (wd = seg_wd[chunk_seg[i / 1024]], s = grad_scale):
    gg = wd * theta + g * s
    Adam      m = b1 m + (1 - b1) gg ; v = b2 v + (1 - b2) gg^2 ; theta -= lr_t m / (sqrt(v) + eps), lr_t = fp32(state[3])
    RMSProp   ms = decay ms + (1 - decay) gg^2 ; mom = momentum mom + lr gg / sqrt(ms + eps) ; theta -= mom ;
              then theta = clamp(theta, -clip, clip) when clip = seg_clip[...] > 0 (no seg_clip: no clip)
    Momentum  accum = momentum accum + gg ; theta -= lr accum
    pnp_adam_advance: state = [b1^t, b2^t, lr, lr_t] in doubles; t += 1 multiplies the powers by the fp32 betas promoted to
              double, and lr_t = lr sqrt(1 - b2^t) / (1 - b1^t).
The hyper-parameters are taken as the kernel sees them: fp32 values (1 - b1 in fp32 is exact for b1 in [0.5, 1]).

Each step reference returns the new values in fp64, the magnitude each one's error scales with (the step evaluated on
absolute values, with the first-order sensitivity of the quotient to its denominator), and the list of intermediates; an
exact case asserts that every intermediate is an fp32 value, so that neither operation order nor FMA contraction can change
the result.  Everything is plain torch and runs on any device."""
import math

import torch

CHUNK = 1024
U32 = 2.0 ** -24        # unit roundoff of fp32

# Per-element tolerances of the real-valued checks, |got - ref| <= TAU * magnitude (tests/test_optim_exact_gpu.py).  Each is
# about 3x the worst ratio measured over those cases on an H100 SXM (80 GB HBM3, 700 W power limit).  GAMMA_K is the
# first-order rigorous bound gamma_k = k u / (1 - k u) with k the longest chain of fp32 roundings of the step (gg 2, m / ms 3,
# v 3 + 2 x gg, sqrt 1, eps 1, mul 1, div 1, theta 1).
TAU = {
    "adam": 6.2e-7,       # measured 2.06e-7 over 5 steps of the TF defaults (0.9 / 0.999 / 1e-8)
    "rmsprop": 6.5e-7,    # measured 2.14e-7 (momentum 0) and 2.16e-7 (momentum 0.9), decay 0.9, eps 1e-10
    "momentum": 3.4e-7,   # measured 1.12e-7 (lr 0.2, momentum 0.2)
}
GAMMA_K = 16


def gamma(k=GAMMA_K):
    return k * U32 / (1 - k * U32)


def f32(x):
    """a Python float rounded to fp32, as a double"""
    return float(torch.tensor(float(x), dtype=torch.float32))


def per_element(table, chunk_seg, n=None):
    """seg table [nseg] -> the per-element value table[chunk_seg[i // 1024]], fp64 [n]"""
    v = table.double()[chunk_seg.long()].repeat_interleave(CHUNK)
    return v if n is None else v[:n]


def fp32_exact(*ts):
    """every element of every fp64 tensor is an fp32 value (finite)"""
    return all(bool(torch.isfinite(t).all()) and torch.equal(t.float().double(), t) for t in ts)


def _d(t):
    return t.double()


# ------------------------------------------------------------------------------------------------
# references
# ------------------------------------------------------------------------------------------------
def adam_advance(state, b1, b2):
    """state = [b1^t, b2^t, lr, lr_t] (Python floats, i.e. doubles) -> the state after one pnp_adam_advance"""
    p1, p2 = state[0] * f32(b1), state[1] * f32(b2)
    return [p1, p2, state[2], state[2] * math.sqrt(1.0 - p2) / (1.0 - p1)]


def _gg(theta, grad, chunk_seg, seg_wd, grad_scale):
    wd = per_element(seg_wd, chunk_seg, theta.numel())
    wt, gs = wd * _d(theta), _d(grad) * f32(grad_scale)
    return wt + gs, wt.abs() + gs.abs(), [wt, gs, wt + gs]


def adam_step(theta, grad, m, v, chunk_seg, seg_wd, state, b1, b2, eps, grad_scale):
    """-> dict theta, m, v (fp64), mag_theta, mag_m, mag_v, inter (intermediates)"""
    b1, b2, eps, lr_t = f32(b1), f32(b2), f32(eps), f32(state[3])
    gg, mag_gg, inter = _gg(theta, grad, chunk_seg, seg_wd, grad_scale)
    m_new = b1 * _d(m) + (1 - b1) * gg
    v_new = b2 * _d(v) + (1 - b2) * gg * gg
    den = v_new.sqrt() + eps
    upd = lr_t * m_new / den
    inter += [b1 * _d(m), (1 - b1) * gg, m_new, gg * gg, (1 - b2) * gg * gg, b2 * _d(v), v_new, v_new.sqrt(), den, lr_t * m_new,
              upd, _d(theta) - upd]
    mag_m = b1 * _d(m).abs() + (1 - b1) * mag_gg
    mag_v = b2 * _d(v).abs() + (1 - b2) * mag_gg * mag_gg
    sens = 1 + mag_v / (2 * v_new.sqrt() * den)
    mag_t = _d(theta).abs() + lr_t * (mag_m + m_new.abs() * sens) / den
    return dict(theta=_d(theta) - upd, m=m_new, v=v_new, mag_theta=mag_t, mag_m=mag_m, mag_v=mag_v, inter=inter)


def rmsprop_step(theta, grad, ms, mom, chunk_seg, seg_wd, seg_clip, lr, decay, momentum, eps, grad_scale):
    """seg_clip may be None (no clip); lr is the fp32 value of the device scalar"""
    lr, decay, momentum, eps = f32(lr), f32(decay), f32(momentum), f32(eps)
    gg, mag_gg, inter = _gg(theta, grad, chunk_seg, seg_wd, grad_scale)
    ms_new = decay * _d(ms) + (1 - decay) * gg * gg
    root = (ms_new + eps).sqrt()
    q = lr * gg / root
    mom_new = momentum * _d(mom) + q
    t = _d(theta) - mom_new
    inter += [gg * gg, (1 - decay) * gg * gg, decay * _d(ms), ms_new, ms_new + eps, root, lr * gg, q, momentum * _d(mom), mom_new, t]
    if seg_clip is not None:
        clip = per_element(seg_clip, chunk_seg, t.numel())
        t = torch.where(clip > 0, torch.minimum(torch.maximum(t, -clip), clip), t)
    mag_ms = decay * _d(ms).abs() + (1 - decay) * mag_gg * mag_gg
    mag_q = lr * (mag_gg + gg.abs() * mag_ms / (2 * (ms_new + eps))) / root
    mag_mom = momentum * _d(mom).abs() + mag_q
    return dict(theta=t, ms=ms_new, mom=mom_new, mag_theta=_d(theta).abs() + mag_mom, mag_ms=mag_ms, mag_mom=mag_mom, inter=inter)


def momentum_step(theta, grad, accum, chunk_seg, seg_wd, lr, momentum, grad_scale):
    lr, momentum = f32(lr), f32(momentum)
    gg, mag_gg, inter = _gg(theta, grad, chunk_seg, seg_wd, grad_scale)
    ac = momentum * _d(accum) + gg
    inter += [momentum * _d(accum), ac, lr * ac, _d(theta) - lr * ac]
    mag_ac = momentum * _d(accum).abs() + mag_gg
    return dict(theta=_d(theta) - lr * ac, accum=ac, mag_theta=_d(theta).abs() + lr * mag_ac, mag_accum=mag_ac, inter=inter)


def worst_ratio(got, ref, mag):
    d = (got.double() - ref).abs()
    r = d / mag.clamp_min(1e-300)
    r = torch.where(d == 0, torch.zeros_like(r), r)
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------------------------------------
# dyadic operands: every intermediate of the step is an fp32 value
# ------------------------------------------------------------------------------------------------
WD_CHOICES = [0.0, 0.25, 0.5, 0.75]
CLIP_CHOICES = [0.0, 2.0, 1.5]


def segment_table(nchunks, nseg, gen, monotone=False):
    """chunk_seg [nchunks] int32: nseg segments, non-monotone with repeated ids unless monotone"""
    if monotone:
        return torch.div(torch.arange(nchunks) * nseg, nchunks, rounding_mode="floor").int()
    seg = torch.randint(0, nseg, (nchunks,), generator=gen).int()
    seg[: min(nseg, nchunks)] = torch.randperm(nseg, generator=gen)[: min(nseg, nchunks)].int()
    return seg


def _pick(values, shape, gen):
    v = torch.tensor(values, dtype=torch.float32)
    return v[torch.randint(0, len(values), shape, generator=gen)]


def _ints(lo, hi, shape, gen, scale=1.0):
    return torch.randint(lo, hi + 1, shape, generator=gen).float() * scale


def _square_fill(gg, k):
    """a second-moment state s with 0.5 s + 0.5 gg^2 = 4^k exactly: s = 2 * 4^k - gg^2"""
    return (2.0 * 4.0 ** k - gg.double() ** 2).float()


def dyadic_case(kind, n, nseg, grad_scale, seed, zero_g_segments=0, monotone=False):
    """operands of an exact case (CPU fp32 tensors).  theta in 2^-2 [-16, 16], g in [-8, 8] (0 on `zero_g_segments` segments),
    wd in {0, 1/4, 1/2, 3/4} (segment 0 has wd 0), the second-moment state chosen so that the new one is 4^k, k in {4, 5, 6},
    first moments in 2^-4 [-128, 128].  RMSProp: clip in {0, 2, 3/2} per segment, and a quarter of the elements of the wd = 0
    segments get g = 0 and theta exactly on +-clip or 1/4 beyond it."""
    gen = torch.Generator().manual_seed(seed)
    nch = n // CHUNK
    chunk_seg = segment_table(nch, nseg, gen, monotone)
    seg_wd = _pick(WD_CHOICES, (nseg,), gen)
    seg_wd[0] = 0.0
    theta = _ints(-16, 16, (n,), gen, 0.25)
    grad = _ints(-8, 8, (n,), gen)
    if zero_g_segments:
        dead = torch.randperm(nseg, generator=gen)[:zero_g_segments]
        grad[torch.isin(chunk_seg.long(), dead).repeat_interleave(CHUNK)] = 0.0
    c = dict(chunk_seg=chunk_seg, seg_wd=seg_wd, grad_scale=grad_scale, n=n)
    if kind == "rmsprop":
        seg_clip = _pick(CLIP_CHOICES, (nseg,), gen)
        seg_clip[0] = 2.0
        if nseg > 1:
            seg_clip[-1] = 0.0
        clip = per_element(seg_clip, chunk_seg).float()
        wd = per_element(seg_wd, chunk_seg).float()
        edge = (wd == 0) & (clip > 0) & (torch.rand(n, generator=gen) < 0.25)
        sign = torch.where(torch.rand(n, generator=gen) < 0.5, -1.0, 1.0)
        beyond = torch.where(torch.rand(n, generator=gen) < 0.5, 0.0, 0.25)
        theta = torch.where(edge, sign * (clip + beyond), theta)
        grad = torch.where(edge, torch.zeros_like(grad), grad)
        c["seg_clip"] = seg_clip
        c["edge"] = edge
    gg = per_element(seg_wd, chunk_seg) * theta.double() + grad.double() * grad_scale
    k = torch.randint(4, 7, (n,), generator=gen).double()
    first = _ints(-128, 128, (n,), gen, 1.0 / 16)
    c.update(theta=theta, grad=grad)
    if kind == "adam":
        c.update(m=first, v=_square_fill(gg, k), state=[0.5 ** 3, 0.5 ** 3, 0.25, 0.125], b1=0.5, b2=0.5, eps=0.0)
    elif kind == "rmsprop":
        c.update(ms=_square_fill(gg, k), mom=first, lr=0.125, decay=0.5, momentum=0.5, eps=0.0)
    else:
        c.update(accum=first, lr=0.125, momentum=0.5)
    return c


def reference(kind, c, **override):
    """the reference step on a case dict (CPU fp32 tensors), any argument overridden"""
    a = dict(c, **override)
    if kind == "adam":
        return adam_step(a["theta"], a["grad"], a["m"], a["v"], a["chunk_seg"], a["seg_wd"], a["state"], a["b1"], a["b2"], a["eps"],
                         a["grad_scale"])
    if kind == "rmsprop":
        return rmsprop_step(a["theta"], a["grad"], a["ms"], a["mom"], a["chunk_seg"], a["seg_wd"], a.get("seg_clip"), a["lr"],
                            a["decay"], a["momentum"], a["eps"], a["grad_scale"])
    return momentum_step(a["theta"], a["grad"], a["accum"], a["chunk_seg"], a["seg_wd"], a["lr"], a["momentum"], a["grad_scale"])


OUTPUTS = {"adam": ("theta", "m", "v"), "rmsprop": ("theta", "ms", "mom"), "momentum": ("theta", "accum")}
MAGS = {"theta": "mag_theta", "m": "mag_m", "v": "mag_v", "ms": "mag_ms", "mom": "mag_mom", "accum": "mag_accum"}
