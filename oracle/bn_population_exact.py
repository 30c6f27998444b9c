"""numpy fp64 restatement of the batch-norm population statistics of elementwise.cu (pnp_bn_accumulate, pnp_bn_population),
operation for operation, and an independent two-pass reference.

    A1 += S1_b;  A2 += S2_b                                      (accumulate: one call per pass, passes in order)
    m = A1 / n;  v = A2 / n - m * m;  v = 0 if v < 0             (population; a NaN passes)
    mean = (fp32) m;  var = (fp32) (n > 1 ? v * (n / (n - 1)) : v)

numpy evaluates fp64 array operations one at a time, each rounded to nearest, and never contracts a multiply and an add: that
is exactly what the kernels' __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn do, and astype(float32) rounds to nearest even as
the kernels' (float) conversion does.

The mutation flags restate common mistakes, for the tests that show each one changes some output:
  average_variances=True  the stored variance is the mean of the per-pass variances (fvcore's PreciseBN), not the pooled one
  biased=True             no Bessel factor
  fma=True                v = A2 / n - m * m with the product kept exact and one rounding at the end (FMA contraction)
  fp32=True               the sums accumulated in fp32
  reverse=True            the passes added last to first"""
from fractions import Fraction

import numpy as np


def accumulate(acc, s1, s2, fp32=False):
    """acc [2C] fp64 (fp32 with the mutation) += (s1, s2) of one pass -> the new accumulator"""
    t = np.float32 if fp32 else np.float64
    C = len(s1)
    out = np.asarray(acc, t).copy()
    out[:C] = out[:C] + np.asarray(s1).astype(t)
    out[C:] = out[C:] + np.asarray(s2).astype(t)
    return out


def _fma_neg(m, c):
    """c - m * m rounded once (exact product), elementwise, NaN / inf as the hardware gives them"""
    out = np.empty_like(c)
    for i, (a, b) in enumerate(zip(m, c)):
        if not (np.isfinite(a) and np.isfinite(b)):
            out[i] = b - a * a
        else:
            out[i] = float(Fraction(float(b)) - Fraction(float(a)) * Fraction(float(a)))
    return out


def moments(acc, count, fma=False):
    """-> (m, v) in fp64 before the Bessel factor and the fp32 rounding (v clamped at 0, a NaN passes)"""
    acc = np.asarray(acc, np.float64)
    C = len(acc) // 2
    n = np.float64(count)
    m = acc[:C] / n
    a2 = acc[C:] / n
    v = _fma_neg(m, a2) if fma else a2 - m * m
    v = np.where(v < 0.0, 0.0, v)
    return m, v


def stored(m, v, count, biased=False):
    """-> (moving_mean, moving_variance) fp32"""
    if count > 1 and not biased:
        v = v * (np.float64(count) / np.float64(count - 1))
    return m.astype(np.float32), v.astype(np.float32)


def population(acc, count, fma=False, biased=False):
    """pnp_bn_population of one entry: acc [2C] fp64, count n -> (moving_mean, moving_variance) fp32"""
    m, v = moments(acc, count, fma)
    return stored(m, v, count, biased)


def recalibrate(passes, average_variances=False, biased=False, fma=False, fp32=False, reverse=False):
    """passes: [(S1_b [C], S2_b [C], M_b)] in pass order -> (moving_mean, moving_variance) fp32 of the whole procedure"""
    C = len(passes[0][0])
    order = passes[::-1] if reverse else passes
    n = sum(int(M) for _, _, M in passes)
    if average_variances:
        vs, ms = [], []
        for s1, s2, M in passes:
            m_b, v_b = moments(np.concatenate([s1, s2]), M)
            ms.append(m_b)
            vs.append(v_b)
        m, v = np.mean(ms, axis=0), np.mean(vs, axis=0)
        return stored(m, v, n, biased)
    acc = np.zeros(2 * C, np.float32 if fp32 else np.float64)
    for s1, s2, _ in order:
        acc = accumulate(acc, s1, s2, fp32)
    return population(acc.astype(np.float64), n, fma, biased)


def batch_sums(z):
    """fp64 (sum, sumsq) per channel of one pass's values z [M, C] (what a layer's forward hands over)"""
    z = np.asarray(z, np.float64)
    return z.sum(axis=0), (z * z).sum(axis=0), z.shape[0]


def two_pass(values):
    """independent reference: the pooled mean and unbiased variance of every value seen, values [(M_b, C)] concatenated,
    in fp64 by the two-pass formula -> (mean, unbiased variance) fp64"""
    x = np.concatenate([np.asarray(v, np.float64) for v in values], axis=0)
    n = x.shape[0]
    m = x.mean(axis=0)
    v = ((x - m) ** 2).sum(axis=0) / n
    return m, (v * (n / (n - 1)) if n > 1 else v)
