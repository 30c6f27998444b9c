"""numpy fp64 restatement of the softmax-entropy objective of elementwise.cu (pnp_entropy_reduce / _finalize / _bwd), and the
a-priori bound on how far the kernels' fp32 evaluation may lie from it.

Per pixel p of logits [B, H, W, C] (fp32 values, evaluated in fp64):
    m = max_c l_c;  t_c = l_c - m;  s = sum_c exp(t_c);  log p_c = t_c - log s;  p_c = exp(t_c) / s
    H_p = -sum_c p_c log p_c;   L = (1/P) sum_p H_p;   pbar_c = (1/P) sum_p p_c;   dL/dl_j = -(1/P) p_j (log p_j + H_p)
with P = B * H * W.

The mutation flags restate plausible mistakes, for the tests that show each one changes some output:
  no_max=True     the exponentials taken of the raw logits in fp32, without subtracting the max (overflow above 88.7)
  per_batch=True  the sum over pixels divided by B instead of P
  drop_h=True     the gradient without its H_p term, -(1/P) p_j log p_j
  clamp=True      log p clamped at log(0.005), as the weighted cross-entropy of the segmentation loss does"""
import numpy as np

U = 2.0 ** -24            # fp32 unit roundoff
E_EXP = 4 * U             # expf: at most 2 ulp (CUDA C Programming Guide, single-precision maths functions)
E_LOG = 2 * U             # logf: at most 1 ulp
TINY = 2.0 ** -125        # twice the smallest normal fp32: what an underflowing (flushed or subnormal) term can lose


def _pieces(logits, no_max=False, clamp=False):
    """-> (t, lp, p, H) in fp64, per pixel, of fp32 logits [..., C]"""
    l = np.asarray(logits, np.float32)
    if no_max:
        with np.errstate(over="ignore", invalid="ignore"):
            e = np.exp(l).astype(np.float64)
            t = l.astype(np.float64)
            s = e.sum(-1, keepdims=True)
            lp = t - np.log(s)
            p = e / s
    else:
        l64 = l.astype(np.float64)
        t = l64 - l64.max(-1, keepdims=True)
        e = np.exp(t)
        s = e.sum(-1, keepdims=True)
        lp = t - np.log(s)
        p = e / s
    if clamp:
        lp = np.log(np.clip(p, 0.005, 1.0))
    H = -(p * lp).sum(-1)
    return t, lp, p, H


def entropy(logits, g=1.0, no_max=False, per_batch=False, drop_h=False, clamp=False):
    """-> (L, pbar [C], dlogits = g * dL/dlogits [..., C], H [...]) in fp64 of fp32 logits [B, H, W, C]"""
    logits = np.asarray(logits, np.float32)
    C = logits.shape[-1]
    P = logits.size // C
    n = logits.shape[0] if per_batch else P
    _, lp, p, H = _pieces(logits, no_max, clamp)
    L = H.sum() / n
    pbar = p.reshape(-1, C).sum(0) / n
    inner = lp if drop_h else lp + H[..., None]
    d = -(float(g) / n) * p * inner
    return L, pbar, d, H


def bounds(logits, g=1.0):
    """a-priori bounds (DESIGN 6.1) on |kernel - entropy()| for (L, pbar [C], dlogits [..., C]) of fp32 logits, from the exact
    values.  First-order error propagation through the kernel's expression, each fp32 operation rounded with relative error
    <= U, expf within E_EXP and logf within E_LOG; the first-order terms are doubled to cover the higher-order ones, and TINY
    covers exponentials that underflow the normal range.  Pixels with a non-finite logit get an infinite bound (they are
    checked for NaN instead)."""
    logits = np.asarray(logits, np.float32)
    C = logits.shape[-1]
    P = logits.size // C
    with np.errstate(invalid="ignore"):
        t, lp, p, H = _pieces(logits)
        a = np.log(np.exp(t).sum(-1))                                  # log s, in [0, log C]
        alp = np.abs(lp)
        rho = U * np.abs(t) + E_EXP                                    # relative error of e_c (t_c rounded, then expf)
        sigma = (p * rho).sum(-1) + (C - 1) * U                        # relative error of s
        alpha = sigma + E_LOG * a                                      # absolute error of logf(s)
        dlp = U * np.abs(t) + alpha[..., None] + U * alp               # absolute error of log p_c
        r = rho + sigma[..., None] + U                                 # relative error of p_c = e_c / s
        dH = 2 * ((p * (dlp + alp * r)).sum(-1) + C * U * H) + C * (1 + alp.max(-1)) * TINY
        bL = dH.mean() + 2 * U * abs(H.mean()) + P * 2.0 ** -52 * (H.mean() + dH.mean())
        bp = 2 * (p * r).reshape(-1, C).mean(0) + TINY + 2 * U * p.reshape(-1, C).mean(0)
        k = abs(float(g)) / P
        uk = 2 * U if P > 2 ** 24 else U                               # -g / (float)P: the division, and P's conversion
        x = np.abs(lp + H[..., None])
        bd = 2 * k * p * (dlp + dH[..., None] + x * (r + 2 * U + uk)) + k * (2 + alp + H[..., None]) * TINY + 2.0 ** -148
    bad = ~np.isfinite(logits).all(-1)
    dH = np.where(bad, np.inf, dH)
    bd = np.where(bad[..., None], np.inf, bd)
    if bad.any():
        bL = np.inf
        bp = np.full(C, np.inf)
    return float(bL), bp, bd
