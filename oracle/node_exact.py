"""fp64 references of the autograd nodes of the training steps that are not convolutions (functional._MaxPool2Fn, _DiscInputFn,
_FCFn, _MeanComboFn, _SegLossFn, the confusion counts and l2_loss_sum), each fed the kernels' own inputs, with an a-priori
per-element bound, and the bound of autograd's own summation of the gradients a tensor receives.

Every real-valued function returns (ref, bound) fp64 tensors; a stage passes when |got - ref| <= bound at every element
(layer_exact.ratio).  The exact ones return the value the kernel must produce bit for bit.  The bounds:
- max-pool forward / backward (first-max routing), the disc-input gather, the channel slice and the confusion counts move or count
  values: exact;
- the disc-input backward adds its ntile copies in fp32, in the order of phase_shift_bwd_kernel (0.f + tile 0 + tile 1 + ...):
  exact against that restatement;
- FC forward (fc_fwd_kernel: per-thread FMA chains, a warp tree, eight partials): any order of F products, gamma_F sum|x||w|;
  dx = dout * w is one rounding, u |dout w|;
- FC dw: fc_bwd_kernel runs an FMA chain of length B from 0 and adds it to the arena slot once (dw[f] += acc):
  gamma_{B+1} (|before| + sum_b |dout x|);
- mean combo forward: each term ca*a + cb*b rounds twice, the 256-thread tree adds at most n - 1 times, the division by n once:
  gamma_{n+2} (|ca| sum|a| + |cb| sum|b|) / n, with ca, cb the fp32 values the kernel receives; backward (functional._bcast:
  pnp_fill with fl32(c/n), then dout * w): gamma_2 |c g / n|;
- seg loss: the accumulator from the fp32 softmax's error, which grows with |l - max l| (segloss_acc); oracle/elementwise_exact.py's
  TAU on the magnitudes it defines for the two losses and coef from the kernel's accumulator (seg_finalize) and for dlogits from
  the kernel's coef (seg_bwd);
- l2_loss_sum: fp32 FMA partials of at most 64 squares per thread, promoted to fp64 and summed there:
  (gamma_64 + n 2^-53) * sum w^2 / 2 (every term is positive);
- the ledger: k gradients of one tensor summed by autograd in fp32, in whatever order, are within gamma_{k-1} sum_i |g_i| of
  their fp64 sum.
Everything is plain torch and runs on any device."""
import torch

from . import elementwise_exact as E
from . import movement_exact as M

U = M.U
U64 = 2.0 ** -53
DISC_NTILES = (3, 1, 1, 1)       # [PS(c4, 2) x3 | PS(c6, 4) | PS(b7, 8) | PS(c9, 8)] of adversarial.py:325-335
L2_CHAIN = 64                    # l2_loss_kernel promotes its fp32 partial to fp64 every 64 squares


def gamma(k):
    return M.gamma(max(int(k), 0))


def f32(x):
    """a Python float as the fp32 value a kernel argument receives, as a double"""
    return float(torch.tensor(float(x), dtype=torch.float32))


def _d(t):
    return t.to(torch.float64)


# ------------------------------------------------------------------------------------------------
# exact: max pool, disc input, channel slice, confusion counts
# ------------------------------------------------------------------------------------------------
def maxpool_fwd(x):
    return M.pool_max_ref(x, 2)


def maxpool_bwd(x, dy):
    """MaxPoolGrad with each window's gradient routed to its first maximum in row-major order"""
    return M.pool_max_bwd_ref(x, dy, 2, first=True)


def disc_plan(srcs, r):
    """-> (Gs, ntiles) of the four sources"""
    return [t.shape[-1] // (r * r) for t in srcs], list(DISC_NTILES)


def disc_input_fwd(srcs, logits, r, order_b1):
    Gs, nt = disc_plan(srcs, r)
    return M.disc_input_ref(srcs, Gs, nt, logits, r, order_b1)


def disc_input_bwd(dout, r, G, coff, ntile, order_b1, tiles=None):
    """the gradient of one source: its ntile copies added in dout's dtype in kernel order, then the inverse phase shift.
    tiles: how many copies to add (a negative control)"""
    s = torch.zeros_like(dout[..., coff:coff + G])
    for t in range(ntile if tiles is None else tiles):
        s = s + dout[..., coff + t * G:coff + (t + 1) * G]
    return M.phase_shift_inv(s, r, G, order_b1)


def channel_slice(g, C, off, Cs):
    return M.channel_slice_ref(g, C, off, Cs, None, False)


def confusion(logits, y):
    C = logits.shape[-1]
    return E.confusion_ref(logits.reshape(-1, C), y.reshape(-1, C))


# ------------------------------------------------------------------------------------------------
# FC
# ------------------------------------------------------------------------------------------------
def fc_fwd(x, w):
    """out [B, 1] = x [B, F] @ w [F, 1]"""
    x, w = _d(x), _d(w).reshape(-1, 1)
    return x @ w, gamma(x.shape[1]) * (x.abs() @ w.abs())


def fc_dx(dout, w):
    dout, w = _d(dout).reshape(-1, 1), _d(w).reshape(1, -1)
    ref = dout * w
    return ref, U * ref.abs()


def fc_dw(x, dout, before=None):
    """-> (before + sum_b dout[b] x[b], bound) as [F, 1]; before None is the zeroed slot"""
    x, dout = _d(x), _d(dout).reshape(-1, 1)
    s, mag = (dout * x).sum(0), (dout * x).abs().sum(0)
    if before is not None:
        b = _d(before).reshape(-1)
        s, mag = s + b, mag + b.abs()
    return s.reshape(-1, 1), (gamma(x.shape[0] + 1) * mag).reshape(-1, 1)


# ------------------------------------------------------------------------------------------------
# mean combo: ca * mean(a) + cb * mean(b)
# ------------------------------------------------------------------------------------------------
def mean_combo_fwd(a, ca, b=None, cb=0.0):
    n = a.numel()
    ca, cb = f32(ca), f32(cb)
    s, mag = ca * _d(a).sum(), abs(ca) * _d(a).abs().sum()
    if b is not None:
        s, mag = s + cb * _d(b).sum(), mag + abs(cb) * _d(b).abs().sum()
    return s / n, gamma(n + 2) * mag / n


def mean_combo_bwd(g, c, n, shape):
    """the gradient of one operand, c * g / n broadcast to `shape`"""
    ref = torch.full(shape, float(c) / n * float(g), dtype=torch.float64, device=getattr(g, "device", None))
    return ref, gamma(2) * ref.abs()


# ------------------------------------------------------------------------------------------------
# seg loss (weighted cross entropy, soft Dice)
# ------------------------------------------------------------------------------------------------
def segloss_acc(logits, y):
    """acc[4C] of pnp_segloss_reduce -> (acc, bound).  segloss_reduce_kernel forms p in fp32 (stable_softmax: l - max l rounded
    once, expf within 2 ulps, C - 1 additions, 1/s and the product each rounded once), so each p_c is within
    eps_c = (|t_c| + max_k |t_k| + C + 10) u of the exact softmax, t = l - max l; the four per-pixel terms (y, p y, p^2,
    -y log clip p, logf within 1 ulp) then run in fp32 chains of at most 32 pixels per thread before the fp64 promotion, and the
    fp64 sums add (P / 32 + 10^4) 2^-53.  Unlike elementwise_exact.TAU (measured on randn * 3 logits), this bound holds for
    any spread of the logits: eps_c grows with |l - max l|."""
    C = logits.shape[-1]
    l, yd = _d(logits.reshape(-1, C)), _d(y.reshape(-1, C))
    acc, _ = E.segloss_reduce_ref(logits.reshape(-1, C), y.reshape(-1, C))
    p = E.softmax64(l)
    t = (l - l.max(1, keepdim=True).values).abs()
    eps = 1.01 * U * (t + t.max(1, keepdim=True).values + C + 10)
    lg = torch.log(p.clamp(E.CLIP, 1.0)).abs()
    chain = gamma(32) + (l.shape[0] / 32 + 1e4) * U64
    py, pp = (p * yd).abs(), p * p
    bound = torch.cat([chain * yd.abs().sum(0), (py * (eps + chain)).sum(0), (pp * (2 * eps + U + chain)).sum(0),
                       (yd.abs() * (eps + (2 * U + chain) * lg)).sum(0)])
    return acc, bound


def segloss_out(acc, P, C):
    """(out[2], coef[3C]) of pnp_segloss_finalize from the kernel's acc -> ((out, bound), (coef, bound))"""
    out, mag, coef = E.segloss_finalize_ref(acc, P, C)
    t = E.TAU["seg_finalize"]
    return (out, t * mag), (coef, t * coef.abs())


def segloss_bwd(logits, y, coef, g_wce, g_dice):
    C = logits.shape[-1]
    ref, mag = E.segloss_bwd_ref(logits.reshape(-1, C), y.reshape(-1, C), coef, float(g_wce), float(g_dice))
    return ref.reshape(logits.shape), (E.TAU["seg_bwd"] * mag).reshape(logits.shape)


# ------------------------------------------------------------------------------------------------
# l2_loss_sum and the ledger
# ------------------------------------------------------------------------------------------------
def l2_sum(tensors, mults=None):
    """sum_i mult_i * tf.nn.l2_loss(w_i) -> (ref, bound); every term is positive, so the bound is relative"""
    mults = [1] * len(tensors) if mults is None else mults
    ref = sum(m * float(E.l2_ref(t)) for t, m in zip(tensors, mults))
    n = sum(t.numel() for t in tensors)
    return ref, (gamma(L2_CHAIN) + (n + 16) * U64) * ref


def ledger(grads):
    """k gradients of one tensor (each reshaped to it) -> (fp64 sum, gamma_{k-1} sum|g_i|)"""
    gs = [_d(g) for g in grads]
    ref = sum(gs[1:], gs[0].clone())
    return ref, gamma(len(gs) - 1) * sum(g.abs() for g in gs)


# ------------------------------------------------------------------------------------------------
# the regularisers of the reference graphs, from its recorded weight lists
# ------------------------------------------------------------------------------------------------
def multiplicities(names):
    """{name: how often the list holds it}: the reference appends the critics' weights on each of their two calls, and the
    back half of the segmenter to mr_front_weights twice"""
    out = {}
    for n in names:
        out[n] = out.get(n, 0) + 1
    return out


def regularisers(trace, ck, lam, l2):
    """the reference's L2 terms (adversarial.py:461-470) from l2(name) = tf.nn.l2_loss of that variable: every weight list summed
    with its multiplicities -> {dis_reg, gen_reg, fixed_coeff_reg}"""
    wl = trace["weight_lists"]
    s = lambda key: sum(l2(n) for n in wl[key])  # noqa: E731
    return {"dis_reg": ck["gan_regularizer"] * ck["miu_dis"] * (s("cls_weights") + lam * s("m_cls_weights")),
            "gen_reg": ck["gan_regularizer"] * ck["miu_gen"] * s("ct_front_weights"),
            "fixed_coeff_reg": ck["regularizer"] * (s("mr_front_weights") + s("joint_weights"))}


def segmenter_regulariser(trace, ck, l2):
    """regularizer_loss of source_segmenter.py:211-240 over its recorded conv_weights list"""
    return ck["regularizer"] * sum(l2(n) for n in trace["source_segmenter"]["conv_weights"])


def gan_weight_decay(trace, ck, lam, dis_sub_iter, gen_sub_iter):
    """per-variable coefficient wd of the gradient wd * w of dis_reg / dis_sub_iter (critic optimizer) and gen_reg / gen_sub_iter
    (generator optimizer) -> ({name: wd}, {name: wd}); names absent take none"""
    wl = trace["weight_lists"]
    base = ck["gan_regularizer"] * ck["miu_dis"] / dis_sub_iter
    d = {n: base * m for n, m in multiplicities(wl["cls_weights"]).items()}
    d.update({n: base * lam * m for n, m in multiplicities(wl["m_cls_weights"]).items()})
    gb = ck["gan_regularizer"] * ck["miu_gen"] / gen_sub_iter
    return d, {n: gb * m for n, m in multiplicities(wl["ct_front_weights"]).items()}


def segmenter_weight_decay(trace, ck):
    return {n: ck["regularizer"] * m for n, m in multiplicities(trace["source_segmenter"]["conv_weights"]).items()}


def critic_clip(trace):
    """{name: c}: clip_op clamps these critic variables to [-c, c] after every critic step"""
    out = {}
    for c in trace["optimizer"]["clip"]:
        assert c["lo"] == -c["hi"] and c["of_same_var"], c
        out[c["var"]] = c["hi"]
    return out
