"""numpy fp32 restatement of the weights' exponential moving average of elementwise.cu (pnp_ema_advance, pnp_ema_update,
pnp_ema_swap): tf.train.ExponentialMovingAverage(decay, num_updates=n) with every operation rounded on its own.

    nf = (float)n;  d = min(decay, (1 + nf) / (10 + nf));  c = 1 - d;  n += 1          (advance)
    s = s - (s - x) * c                                                                (update: assign_sub(s, (s - x) * (1 - d)))

numpy evaluates np.float32 scalar and array operations one at a time, each rounded to nearest fp32, and never contracts a
multiply and an add: that is exactly what the kernels' __fadd_rn / __fsub_rn / __fmul_rn / __fdiv_rn do.

The mutation flags restate common mistakes, for the tests that show each one changes some output:
  form="blend"     the update written as d * s + (1 - d) * x
  fma=True         s - (s - x) * c with the product kept exact and one rounding at the end (what FMA contraction does)
  decay_fp64=True  d and c computed in fp64 and rounded to fp32 once
  n_offset=k       the schedule read at n + k"""
import numpy as np

f32 = np.float32


def advance(n, decay, decay_fp64=False, n_offset=0):
    """-> (c, n + 1): the fp32 factor 1 - d of update number n (0-based) and the advanced count"""
    m = int(n) + int(n_offset)
    if decay_fp64:
        d = min(float(f32(decay)), (1.0 + m) / (10.0 + m))
        return f32(1.0 - d), int(n) + 1
    nf = f32(m)                          # int64 -> fp32, round to nearest even (__ll2float_rn)
    d = min(f32(decay), (f32(1.0) + nf) / (f32(10.0) + nf))
    return f32(f32(1.0) - d), int(n) + 1


def update(s, x, c, form="assign_sub", fma=False):
    """one update of the fp32 shadow s towards the live values x with factor c -> new shadow (s is not modified)"""
    s = np.asarray(s, dtype=np.float32)
    x = np.asarray(x, dtype=np.float32)
    c = f32(c)
    if form == "blend":
        d = f32(f32(1.0) - c)
        return (d * s + (f32(1.0) - d) * x).astype(np.float32)
    diff = s - x
    if fma:
        # the fp32 * fp32 product is exact in fp64; the fp64 difference is then rounded to fp32 (an FMA's single rounding, up to
        # a double rounding the designed inputs do not meet)
        return (s.astype(np.float64) - diff.astype(np.float64) * np.float64(c)).astype(np.float32)
    return (s - diff * c).astype(np.float32)


def steps(shadow, lives, n, decay, **mut):
    """the recurrence over `lives` (one fp32 array per averaged step, in order) from `shadow` at count n -> (shadow, n)"""
    s = np.asarray(shadow, dtype=np.float32).copy()
    adv = {k: v for k, v in mut.items() if k in ("decay_fp64", "n_offset")}
    upd = {k: v for k, v in mut.items() if k in ("form", "fma")}
    for x in lives:
        c, n = advance(n, decay, **adv)
        s = update(s, x, c, **upd)
    return s, n


def swap(shadow, live):
    """-> (new shadow, new live): the contents exchanged"""
    return np.array(live, dtype=np.float32, copy=True), np.array(shadow, dtype=np.float32, copy=True)
