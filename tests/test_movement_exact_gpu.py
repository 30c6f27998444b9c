"""The pooling, padding, phase-shift, gather, slice / concat, one-hot, fill, softmax and cross-entropy kernels against the
references of oracle/movement_exact.py, called at the C-ABI, at every dispatch path and launch regime.

a. data movement, bit for bit: every output starts as a NaN sentinel and is compared as int32 bit patterns with the reference,
   so an element written that should not be (a channel outside a phase shift's or a logits concat's range) or not written that
   should be is a failure.  The max poolings run on tie-heavy operands (small integers, constant planes, +-inf, +-FLT_MAX, windows
   of -inf) with a distinct gradient per window; integer operands make the average poolings and every backward sum exact.
   Each launcher runs at grid_for's 8448-CTA cap with at least two grid-stride iterations and as one partial CTA;
b. real-valued cases: randn operands of the sums against fp64 within gamma_k * sum|terms|, pixel_softmax2 and cross_entropy
   within a priori bounds from CUDA's documented expf / logf errors (each test prints its worst ratio next to the bound);
c. the functional fallback route of the discriminator input (a channel count that is not a multiple of 4), forward and backward;
d. rejected calls return PNP_ERR_BAD_ARG / PNP_ERR_UNSUPPORTED and leave every output untouched;
e. the exact cases again under PNP_PDL=1, in their own process."""
import ctypes

import pytest
import torch

from oracle import movement_exact as M
from tests.cabi import (BAD_ARG, DEV, SENTINEL, UNSUPPORTED, assert_bits, assert_untouched, cpu_gen, ints, lib, pick, ptr, rerun,
                        sentinel, snapshot, sync)

pytestmark = pytest.mark.gpu
INF = float("inf")

# ------------------------------------------------------------------------------------------------
# case tables (the CPU file checks that together they reach every regime of every launcher)
# ------------------------------------------------------------------------------------------------
# (id, B, H, W, C, operand kind)
MAXPOOL2_CASES = [
    ("C4_ints", 2, 6, 10, 4, "ints"), ("C16_const", 1, 8, 6, 16, "const"), ("C64_inf", 2, 4, 4, 64, "inf"),
    ("C1_W2", 3, 10, 2, 1, "ints"), ("C3_H2_inf", 2, 2, 6, 3, "inf"), ("C6_neginf", 1, 6, 6, 6, "neginf"),
    ("C4_one_partial_cta", 1, 4, 4, 4, "ints"), ("C3_one_partial_cta", 1, 2, 2, 3, "neginf"),
    ("cap_V4", 17, 256, 256, 64, "ints"), ("cap_V1", 12, 1024, 1024, 3, "ints"),
]
# (id, B, H, W, C, n, operand kind)
POOL_CASES = [
    ("n1", 2, 5, 7, 3, 1, "ints"), ("n2_odd", 2, 7, 9, 4, 2, "ints"), ("n3", 1, 10, 11, 5, 3, "ints"),
    ("n4_const", 2, 9, 6, 3, 4, "const"), ("n5_gt_map", 1, 3, 2, 6, 5, "ints"), ("n8_W2_inf", 2, 13, 2, 4, 8, "inf"),
    ("n3_neginf", 1, 7, 8, 2, 3, "neginf"), ("n2_H2_neginf", 2, 2, 5, 3, 2, "neginf"), ("n5_inf", 1, 11, 12, 3, 5, "inf"),
    ("cap_n2", 5, 1024, 1024, 8, 2, "ints"),
]
# (id, B, H, W, C, p)
MIRROR_CASES = [
    ("p0", 2, 4, 7, 5, 0), ("p1", 2, 5, 3, 3, 1), ("p2", 1, 6, 9, 7, 2), ("p3", 2, 7, 4, 3, 3),
    ("p_eq_H", 2, 3, 5, 3, 3), ("H3_W5_p2", 1, 3, 5, 3, 2), ("H1_W4_p1", 2, 1, 4, 5, 1), ("H2_W2_p2", 1, 2, 2, 3, 2),
    ("cap", 8, 256, 300, 33, 1),
]
# (id, B, a, b, G, r, Ctot, coff, ntile, order_b1)
PS_CASES = [
    ("r1", 2, 3, 4, 2, 1, 9, 1, 3, 0), ("r2_b1", 1, 3, 5, 5, 2, 12, 2, 1, 1), ("r2", 3, 2, 3, 1, 2, 6, 1, 3, 0),
    ("r4", 2, 2, 3, 5, 4, 20, 3, 3, 0), ("r4_b1", 1, 3, 2, 2, 4, 8, 1, 3, 1), ("r8", 2, 2, 2, 2, 8, 10, 2, 3, 0),
    ("r8_b1", 1, 2, 3, 5, 8, 7, 1, 1, 1), ("cap", 8, 64, 64, 9, 8, 11, 1, 1, 0),
]
# (id, B, a, b, r, order_b1, Gs, ntiles, NC)
DISC_CASES = [
    ("real_B8", 8, 32, 32, 8, 0, (2, 4, 8, 8), (3, 1, 1, 1), 5),
    ("r8_b5", 3, 2, 5, 8, 0, (2, 4, 8, 8), (3, 1, 1, 1), 5),
    ("r8_b6_NC1", 2, 3, 6, 8, 0, (2,), (3,), 1),
    ("r8_b7", 2, 1, 7, 8, 0, (3, 2), (1, 3), 6),
    ("r8_NC8", 2, 2, 4, 8, 0, (3,), (1,), 8),
    ("r8_Ctot64", 2, 2, 3, 8, 0, (8, 8, 8, 8), (4, 1, 1, 1), 7),
    ("r8_one_cta", 1, 1, 3, 8, 0, (2, 4, 8, 8), (3, 1, 1, 1), 5),
    ("B1_order", 1, 4, 3, 8, 1, (2, 4, 8, 8), (3, 1, 1, 1), 5),
    ("r4", 2, 5, 6, 4, 0, (2, 4), (3, 1), 5),
    ("lines33", 2, 2, 3, 8, 0, (9, 8, 8, 8), (1, 1, 1, 1), 2),
    ("generic_one_cta", 1, 1, 1, 4, 0, (2, 4), (3, 1), 5),
    ("generic_cap", 2, 128, 128, 4, 0, (2, 4, 8, 8), (3, 1, 1, 1), 5),
]
# (id, P, C, Ctot, coff)
LAC_CASES = [("C5", 100, 5, 9, 2), ("C1", 300, 1, 4, 1), ("C8", 1000, 8, 12, 3), ("coff0", 77, 3, 4, 0),
             ("cap", 4400000, 3, 5, 1)]
# (id, M, C, off, Cs, accumulate)
SLICE_CASES = [("off0", 100, 7, 0, 3, 0), ("off0_acc", 100, 7, 0, 3, 1), ("end", 100, 7, 4, 3, 0), ("end_acc", 100, 7, 4, 3, 1),
               ("C1", 5, 1, 0, 1, 1), ("cap_acc", 3000000, 10, 4, 6, 1), ("cap", 3000000, 10, 0, 6, 0)]
# (id, B, H1, W1, C1, H2, W2, C2, dx1, dx2)
CAT_CASES = [
    ("odd", 2, 9, 8, 3, 6, 5, 2, True, True), ("C1_1_no_dx2", 1, 5, 7, 1, 4, 4, 3, True, False),
    ("C2_1_no_dx1", 3, 6, 6, 4, 6, 6, 1, False, True), ("tiny", 1, 2, 2, 1, 1, 1, 1, True, True),
    ("odd_W", 2, 4, 7, 2, 4, 2, 5, True, True), ("cap", 4, 700, 700, 4, 695, 695, 4, True, True),
]
# (id, P, C)
ONE_HOT_CASES = [("C1", 1000, 1), ("C5", 777, 5), ("C8", 300, 8), ("C12", 5000, 12), ("cap", 4400000, 5)]
FILL_N = [1, 2, 3, 4, 5, 1027, 36000003]
# (id, P, C)
PS2_CASES = [("C1", 3000, 1), ("C2", 300, 2), ("C5", 5000, 5), ("C8", 4099, 8), ("cap", 4400000, 2)]
CE_N = [1, 1000, 100003, 70000000]     # the last is above the cap with more than 32 elements per accumulating thread


def ids(cases):
    return [c[0] for c in cases]


# ------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------
def operand(kind, shape, seed, dev=DEV):
    """the pooling operands.  ints: integers in [-2, 2]; const: one integer per (image, channel) plane; inf: +-inf, +-FLT_MAX and
    small integers; neginf: mostly -inf (many windows are all -inf); randn.  None holds -0.0."""
    g = cpu_gen(seed)
    if kind == "ints":
        v = torch.randint(-2, 3, shape, generator=g).float()
    elif kind == "const":
        v = torch.randint(-2, 3, (shape[0], 1, 1, shape[3]), generator=g).float().expand(*shape).contiguous()
    elif kind == "inf":
        v = pick(shape, [-INF, INF, -M.FLT_MAX, M.FLT_MAX, -1.0, 1.0, 2.0], g)
    elif kind == "neginf":
        v = pick(shape, [-INF] * 6 + [0.0, 1.0], g)
    elif kind == "randn":
        v = torch.randn(shape, generator=g)
    else:
        raise ValueError(kind)
    return v.to(dev)


def distinct(shape, dev=DEV, offset=1):
    """distinct positive integers (below 2^23, so sums of a few stay exact)"""
    n = 1
    for s in shape:
        n *= s
    return ((torch.arange(n, device=dev) * 7919 + offset) % (1 << 22) + 1).float().view(*shape)


def small_ints(shape, seed, lo=-8, hi=8, dev=DEV):
    return ints(shape, lo, hi, cpu_gen(seed)).to(dev)


def ps_operands(case, dev=DEV):
    tag, B, a, b, G, r, Ctot, coff, ntile, o = case
    X = distinct((B, a, b, G * r * r), dev)
    dout = small_ints((B, a * r, b * r, Ctot), 11 + B * a * b, dev=dev)
    return X, dout


def disc_operands(case, dev=DEV):
    tag, B, a, b, r, o, Gs, nts, NC = case
    srcs = [distinct((B, a, b, G * r * r), dev, offset=1 + 1000003 * s) for s, G in enumerate(Gs)]
    logits = small_ints((B, a * r, b * r, NC), 5 + B + NC, -1, 1, dev)       # many ties
    return srcs, logits


def one_hot_labels(P, C, seed, dev=DEV):
    vals = torch.tensor([-1, C, 1 << 40, -(1 << 40)] + list(range(C)), dtype=torch.int64)
    return vals[torch.randint(0, len(vals), (P,), generator=cpu_gen(seed))].to(dev)


def _launch_note(tag, launch):
    print("  %-22s grid %5d capped %d iters %d single partial CTA %d" % (tag, launch.grid, launch.capped, launch.iters,
                                                                         launch.single_partial))


# ------------------------------------------------------------------------------------------------
# a. pooling
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", MAXPOOL2_CASES, ids=ids(MAXPOOL2_CASES))
def test_maxpool2_exact(case):
    _C, rt = lib()
    tag, B, H, W, C, kind = case
    V, launch = M.maxpool2_launch(B, H, W, C)
    _launch_note("%s V=%d" % (tag, V), launch)
    x = operand(kind, (B, H, W, C), B + H + W + C)
    y = sentinel((B, H // 2, W // 2, C))
    _C.call("pnp_maxpool2_fwd", ptr(x), ptr(y), B, H, W, C, rt.stream())
    sync()
    assert_bits(tag + " fwd", y, M.pool_max_ref(x, 2))
    dy = distinct(tuple(y.shape))
    dx = sentinel((B, H, W, C))
    _C.call("pnp_maxpool2_bwd", ptr(x), ptr(dy), ptr(dx), B, H, W, C, rt.stream())
    sync()
    assert_bits(tag + " bwd", dx, M.pool_max_bwd_ref(x, dy, 2))


@pytest.mark.parametrize("case", MAXPOOL2_CASES, ids=ids(MAXPOOL2_CASES))
def test_avgpool2_exact(case):
    """integer operands: the fp32 window sum is exact and 0.25f * sum = sum / 4; the backward 0.25f * dy is exact for any dy"""
    _C, rt = lib()
    tag, B, H, W, C, _ = case
    _launch_note(tag, M.avgpool2_launch(B, H, W, C))
    x = operand("ints", (B, H, W, C), 3 + B + H)
    y = sentinel((B, H // 2, W // 2, C))
    _C.call("pnp_avgpool2", ptr(x), ptr(y), B, H, W, C, 0, rt.stream())
    sync()
    assert_bits(tag + " fwd", y, M.pool_avg_ref(x, 2)[0])
    dy = operand("randn", tuple(y.shape), 4 + C)
    dx = sentinel((B, H, W, C))
    _C.call("pnp_avgpool2", ptr(dy), ptr(dx), B, H, W, C, 1, rt.stream())
    sync()
    assert_bits(tag + " bwd", dx, M.pool_avg_bwd_ref(dy, H, W, 2))


@pytest.mark.parametrize("case", POOL_CASES, ids=ids(POOL_CASES))
def test_pool_exact(case):
    """pnp_pool_fwd / _bwd, max and average: bit for bit (average on integer operands; its backward with x = NULL)"""
    _C, rt = lib()
    tag, B, H, W, C, n, kind = case
    Ho, Wo, pt, pl = M.pool_geom(H, W, n)
    _launch_note(tag + " fwd", M.pool_launch(B, H, W, C, n, False))
    _launch_note(tag + " bwd", M.pool_launch(B, H, W, C, n, True))
    x = operand(kind, (B, H, W, C), 7 * B + H + W + n)
    y = sentinel((B, Ho, Wo, C))
    _C.call("pnp_pool_fwd", ptr(x), ptr(y), B, H, W, C, n, 0, rt.stream())
    sync()
    assert_bits(tag + " max fwd", y, M.pool_max_ref(x, n))
    dy = distinct((B, Ho, Wo, C))
    dx = sentinel((B, H, W, C))
    _C.call("pnp_pool_bwd", ptr(x), ptr(dy), ptr(dx), B, H, W, C, n, 0, rt.stream())
    sync()
    assert_bits(tag + " max bwd", dx, M.pool_max_bwd_ref(x, dy, n))
    if kind in ("ints", "const"):
        y = sentinel((B, Ho, Wo, C))
        _C.call("pnp_pool_fwd", ptr(x), ptr(y), B, H, W, C, n, 1, rt.stream())
        sync()
        assert_bits(tag + " avg fwd", y, M.pool_avg_ref(x, n)[0])
    dy = operand("randn", (B, Ho, Wo, C), 9 + n)
    dx = sentinel((B, H, W, C))
    _C.call("pnp_pool_bwd", None, ptr(dy), ptr(dx), B, H, W, C, n, 1, rt.stream())
    sync()
    assert_bits(tag + " avg bwd", dx, M.pool_avg_bwd_ref(dy, H, W, n))


def test_maxpool_signed_zero_tie():
    """windows of +0.0 and -0.0 only: the max compares equal to 0 (which zero fmaxf returns is not pinned) and the gradient goes
    to the window's first element"""
    _C, rt = lib()
    for C, n in ((4, 2), (3, 2), (2, 3)):
        B, H, W = 2, 6, 6
        x = pick((B, H, W, C), [0.0, -0.0], cpu_gen(C + n)).to(DEV)
        Ho, Wo, _, _ = M.pool_geom(H, W, n)
        dy = distinct((B, Ho, Wo, C))
        for fwd, bwd, extra in (("pnp_maxpool2_fwd", "pnp_maxpool2_bwd", ()), ("pnp_pool_fwd", "pnp_pool_bwd", (n, 0))):
            if fwd == "pnp_maxpool2_fwd" and n != 2:
                continue
            y = sentinel((B, Ho, Wo, C))
            _C.call(fwd, ptr(x), ptr(y), B, H, W, C, *extra, rt.stream())
            dx = sentinel((B, H, W, C))
            _C.call(bwd, ptr(x), ptr(dy), ptr(dx), B, H, W, C, *extra, rt.stream())
            sync()
            assert bool((y == 0).all()), "%s C%d n%d: %s" % (fwd, C, n, y.unique())
            assert_bits("%s C%d n%d" % (bwd, C, n), dx, M.pool_max_bwd_ref(x, dy, n))


@pytest.mark.parametrize("case", [("avgpool2_C4", 2, 10, 6, 4, 2), ("n3", 2, 10, 11, 5, 3), ("n5", 1, 13, 9, 3, 5)],
                         ids=lambda c: c[0])
def test_avg_pool_real(case):
    """randn: |y - y64| <= gamma_k * sum|x| / k for a window of k valid elements (k - 1 additions and one division)"""
    _C, rt = lib()
    tag, B, H, W, C, n = case
    x = operand("randn", (B, H, W, C), 21 + n)
    Ho, Wo, _, _ = M.pool_geom(H, W, n)
    y = sentinel((B, Ho, Wo, C))
    if tag.startswith("avgpool2"):
        _C.call("pnp_avgpool2", ptr(x), ptr(y), B, H, W, C, 0, rt.stream())
    else:
        _C.call("pnp_pool_fwd", ptr(x), ptr(y), B, H, W, C, n, 1, rt.stream())
    sync()
    _, y64, mag, cnt = M.pool_avg_ref(x, n)
    bound = cnt * M.U / (1 - cnt * M.U)
    ratio = M.worst_ratio(y, y64, mag * bound)
    print("  RATIO avg pool %-12s worst |got-ref| / (gamma_k sum|x|/k) %.3f  bound 1" % (tag, ratio))
    assert ratio <= 1.0


# ------------------------------------------------------------------------------------------------
# a. SYMMETRIC pad
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", MIRROR_CASES, ids=ids(MIRROR_CASES))
def test_mirror_pad_exact(case):
    _C, rt = lib()
    tag, B, H, W, C, p = case
    _launch_note(tag + " fwd", M.mirror_pad_launch(B, H, W, C, p, False))
    _launch_note(tag + " bwd", M.mirror_pad_launch(B, H, W, C, p, True))
    x = operand("randn", (B, H, W, C), 31 + H * W)
    y = sentinel((B, H + 2 * p, W + 2 * p, C))
    _C.call("pnp_mirror_pad_fwd", ptr(x), ptr(y), B, H, W, C, p, rt.stream())
    sync()
    assert_bits(tag + " fwd", y, M.mirror_pad_ref(x, p))
    dy = small_ints(tuple(y.shape), 32 + p)
    dx = sentinel((B, H, W, C))
    _C.call("pnp_mirror_pad_bwd", ptr(dy), ptr(dx), B, H, W, C, p, rt.stream())
    sync()
    assert_bits(tag + " bwd", dx, M.mirror_pad_bwd_ref(dy, H, W, p)[0])


@pytest.mark.parametrize("case", [c for c in MIRROR_CASES if c[0] != "cap"], ids=[c[0] for c in MIRROR_CASES if c[0] != "cap"])
def test_mirror_pad_bwd_real(case):
    """randn dy: |dx - dx64| <= gamma_k * sum|terms| for an element that sums k padded positions"""
    _C, rt = lib()
    tag, B, H, W, C, p = case
    dy = operand("randn", (B, H + 2 * p, W + 2 * p, C), 33 + p)
    dx = sentinel((B, H, W, C))
    _C.call("pnp_mirror_pad_bwd", ptr(dy), ptr(dx), B, H, W, C, p, rt.stream())
    sync()
    ref, mag, cnt = M.mirror_pad_bwd_ref(dy, H, W, p)
    ratio = M.worst_ratio(dx, ref, mag * (cnt * M.U / (1 - cnt * M.U)))
    print("  RATIO mirror pad bwd %-10s worst |got-ref| / (gamma_k sum|dy|) %.3f  bound 1" % (tag, ratio))
    assert ratio <= 1.0


# ------------------------------------------------------------------------------------------------
# a. phase shift, discriminator input, logits | argmax, channel slice
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", PS_CASES, ids=ids(PS_CASES))
def test_phase_shift_exact(case):
    """forward into a sentinel tensor: channels outside [coff, coff + ntile*G) keep the sentinel; backward sums the ntile copies"""
    _C, rt = lib()
    tag, B, a, b, G, r, Ctot, coff, ntile, o = case
    _launch_note(tag, M.phase_shift_launch(B, a, b, G, r))
    X, dout = ps_operands(case)
    out = sentinel((B, a * r, b * r, Ctot))
    ref = M.phase_shift_fwd_ref(X, out.clone(), r, G, coff, ntile, o)
    _C.call("pnp_phase_shift_fwd", ptr(X), ptr(out), B, a, b, G, r, Ctot, coff, ntile, o, rt.stream())
    sync()
    assert_bits(tag + " fwd", out, ref)
    dX = sentinel(tuple(X.shape))
    _C.call("pnp_phase_shift_bwd", ptr(dout), ptr(dX), B, a, b, G, r, Ctot, coff, ntile, o, rt.stream())
    sync()
    assert_bits(tag + " bwd", dX, M.phase_shift_bwd_ref(dout, r, G, coff, ntile, o))


def _disc_call(_C, rt, srcs, Gs, nts, logits, out, B, a, b, r, o):
    n = len(srcs)
    P = ctypes.c_void_p * n
    I = ctypes.c_int * n
    return _C.lib.pnp_disc_input_fwd(P(*[ptr(s) for s in srcs]), I(*[a] * n), I(*[b] * n), I(*Gs), I(*nts), n, ptr(logits),
                                     logits.shape[-1], ptr(out), B, a * r, b * r, r, o, rt.stream())


@pytest.mark.parametrize("case", DISC_CASES, ids=ids(DISC_CASES))
def test_disc_input_exact(case):
    _C, rt = lib()
    tag, B, a, b, r, o, Gs, nts, NC = case
    path, launch = M.disc_input_launch(B, a, b, r, o, Gs, nts, NC)
    _launch_note("%s %s" % (tag, path), launch)
    srcs, logits = disc_operands(case)
    Ctot = M.disc_ctot(Gs, nts, NC)
    out = sentinel((B, a * r, b * r, Ctot))
    rc = _disc_call(_C, rt, srcs, Gs, nts, logits, out, B, a, b, r, o)
    sync()
    assert rc == 0, "%s: pnp_disc_input_fwd returned %d" % (tag, rc)
    assert_bits(tag, out, M.disc_input_ref(srcs, Gs, nts, logits, r, o))


@pytest.mark.parametrize("B,o", [(2, 0), (1, 1)])
def test_disc_input_functional_fallback(B, o):
    """functional.disc_input with 4 logits channels: Ctot = 31 is not a multiple of 4, so the layer runs pnp_phase_shift_fwd per
    source and pnp_logits_argmax_concat; forward bit for bit, backward (pnp_phase_shift_bwd with ntile 3, pnp_channel_slice)
    bit for bit on integer dout"""
    lib()
    from pnp_b200 import functional as F
    a = b = 2
    r, Gs, nts, NC = 8, (2, 4, 8, 8), (3, 1, 1, 1), 4
    case = ("fallback", B, a, b, r, o, Gs, nts, NC)
    srcs, logits = disc_operands(case)
    Ctot = M.disc_ctot(Gs, nts, NC)
    assert Ctot % 4 != 0
    xs = [s.clone().requires_grad_(True) for s in srcs]
    lg = logits.clone().requires_grad_(True)
    out = F.disc_input(*xs, lg, B, r)
    sync()
    assert_bits("fallback fwd", out.detach(), M.disc_input_ref(srcs, Gs, nts, logits, r, o))
    dout = small_ints(tuple(out.shape), 41 + B)
    out.backward(dout)
    sync()
    coff = 0
    for i, (x, G, t) in enumerate(zip(xs, Gs, nts)):
        assert_bits("fallback d src %d" % i, x.grad, M.phase_shift_bwd_ref(dout, r, G, coff, t, o))
        coff += G * t
    assert_bits("fallback d logits", lg.grad, dout[..., coff:coff + NC])


@pytest.mark.parametrize("case", LAC_CASES, ids=ids(LAC_CASES))
def test_logits_argmax_concat_exact(case):
    """channels outside [coff, coff + C] keep the sentinel; argmax takes the lowest index on ties"""
    _C, rt = lib()
    tag, P, C, Ctot, coff = case
    _launch_note(tag, M.pixel_launch(P))
    logits = small_ints((P, C), P + C, -1, 1)
    out = sentinel((P, Ctot))
    ref = M.logits_argmax_concat_ref(logits, out.clone(), coff)
    _C.call("pnp_logits_argmax_concat", ptr(logits), ptr(out), P, C, Ctot, coff, rt.stream())
    sync()
    assert_bits(tag, out, ref)


@pytest.mark.parametrize("case", SLICE_CASES, ids=ids(SLICE_CASES))
def test_channel_slice_exact(case):
    _C, rt = lib()
    tag, Mr, C, off, Cs, acc = case
    _launch_note(tag, M.channel_slice_launch(Mr, Cs))
    g = operand("randn", (Mr, C), Mr + C)
    out = operand("randn", (Mr, Cs), 3 * Mr + Cs) if acc else sentinel((Mr, Cs))
    ref = M.channel_slice_ref(g, C, off, Cs, out.clone(), acc)
    _C.call("pnp_channel_slice", ptr(g), C, off, Cs, ptr(out), Mr, acc, rt.stream())
    sync()
    assert_bits(tag, out, ref)


# ------------------------------------------------------------------------------------------------
# a. crop-concat, one-hot, fill
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CAT_CASES, ids=ids(CAT_CASES))
def test_crop_concat_exact(case):
    _C, rt = lib()
    tag, B, H1, W1, C1, H2, W2, C2, w1, w2 = case
    _launch_note(tag + " fwd", M.crop_concat_launch(B, H1, W1, C1, H2, W2, C2, False))
    _launch_note(tag + " bwd", M.crop_concat_launch(B, H1, W1, C1, H2, W2, C2, True, w1, w2))
    x1 = operand("randn", (B, H1, W1, C1), H1 + W1)
    x2 = operand("randn", (B, H2, W2, C2), H2 + W2 + 1)
    out = sentinel((B, H2, W2, C1 + C2))
    _C.call("pnp_crop_concat_fwd", ptr(x1), ptr(x2), ptr(out), B, H1, W1, C1, H2, W2, C2, rt.stream())
    sync()
    assert_bits(tag + " fwd", out, M.crop_concat_fwd_ref(x1, x2))
    dout = operand("randn", tuple(out.shape), 5 + C1)
    dx1 = sentinel(tuple(x1.shape))
    dx2 = sentinel(tuple(x2.shape))
    _C.call("pnp_crop_concat_bwd", ptr(dout), ptr(dx1) if w1 else None, ptr(dx2) if w2 else None, B, H1, W1, C1, H2, W2, C2,
            rt.stream())
    sync()
    r1, r2 = M.crop_concat_bwd_ref(dout, H1, W1, C1)
    assert_bits(tag + " dx1", dx1, r1 if w1 else sentinel(tuple(x1.shape)))
    assert_bits(tag + " dx2", dx2, r2 if w2 else sentinel(tuple(x2.shape)))


@pytest.mark.parametrize("case", ONE_HOT_CASES, ids=ids(ONE_HOT_CASES))
def test_one_hot_exact(case):
    """labels -1, C, 2^40 and -2^40 give a zero row"""
    _C, rt = lib()
    tag, P, C = case
    _launch_note(tag, M.pixel_launch(P))
    labels = one_hot_labels(P, C, P + C)
    out = sentinel((P, C))
    _C.call("pnp_one_hot", ptr(labels), ptr(out), P, C, rt.stream())
    sync()
    assert_bits(tag, out, M.one_hot_ref(labels, C))


@pytest.mark.parametrize("n", FILL_N)
def test_fill_exact(n):
    """the n % 4 tail is written by CTA 0; nothing past n is touched"""
    _C, rt = lib()
    fl = M.fill_launch(n)
    print("  n %d grid %d capped %d iters %d tail %d" % (n, fl.grid, fl.capped, fl.iters, fl.tail))
    buf = sentinel(n + 5)
    ref = M.fill_ref(buf, -3.25, n)
    _C.call("pnp_fill", ptr(buf), -3.25, n, rt.stream())
    sync()
    assert_bits("fill %d" % n, buf, ref)


# ------------------------------------------------------------------------------------------------
# b. the two transcendental kernels
# ------------------------------------------------------------------------------------------------
def ps2_logits(P, C, seed, dev=DEV):
    """randn * 3 logits, with every 97th pixel at -200 + c (every expf underflows) and every 89th at 89 + c (expf overflows)"""
    l = (torch.randn((P, C), generator=cpu_gen(seed)) * 3).float()
    l[::97] = -200.0 + torch.arange(C, dtype=torch.float32)
    l[1::89] = 89.0 + torch.arange(C, dtype=torch.float32)
    return l.to(dev)


@pytest.mark.parametrize("case", PS2_CASES, ids=ids(PS2_CASES))
def test_pixel_softmax2(case):
    """|p - p64| <= ps2_bound(C) * p64 per element; the underflow and overflow pixels are -1e15f exactly"""
    _C, rt = lib()
    tag, P, C = case
    _launch_note(tag, M.pixel_launch(P))
    l = ps2_logits(P, C, P + C)
    out = sentinel((P, C))
    _C.call("pnp_pixel_softmax2", ptr(l), ptr(out), P, C, rt.stream())
    sync()
    special = M.ps2_special(l)
    assert int(special.sum()) >= 2
    assert_bits(tag + " clipped pixels", out[special], torch.full_like(out[special], M.PS2_CLIPPED))
    ref = M.pixel_softmax2_ref(l[~special])
    got = out[~special]
    bound = M.ps2_bound(C)
    ratio = M.worst_ratio(got, ref, ref)
    print("  RATIO pixel_softmax2 %-6s worst |got-ref|/p %.3e  a priori bound %.3e  (%.3f of it)" % (tag, ratio, bound,
                                                                                                     ratio / bound))
    assert ratio <= bound


def ce_operands(n, seed, dev=DEV):
    """y in [0, 1) at multiples of 1/8, p = 2^-k (k in 0..20) with a few p outside [1e-10, 1] and at its ends"""
    g = cpu_gen(seed)
    y = (torch.randint(0, 8, (n,), generator=g).float() / 8)
    p = torch.pow(2.0, -torch.randint(0, 21, (n,), generator=g).float())
    special = torch.tensor([1.0, 2.0, 1e-11, 0.0, -1.0, 1.5], dtype=torch.float32)
    k = min(n, special.numel())
    p[:k] = special[:k]
    p[1::1009] = 2.0
    p[2::1013] = 0.0
    return y.to(dev), p.to(dev)


@pytest.mark.parametrize("n", CE_N)
def test_cross_entropy_bwd(n):
    """dp bit for bit (dyadic y, power-of-two p, k = -g/n = -1/2 exact) and 0 outside [1e-10, 1]; dy = k log(clip p) within
    CE_DY_BOUND (0 exactly at p = 1)"""
    _C, rt = lib()
    _launch_note("n %d" % n, M.ce_bwd_launch(n))
    y, p = ce_operands(n, n)
    g = torch.tensor([0.5 * n], dtype=torch.float32, device=DEV)
    assert float(g) == 0.5 * n and float(torch.tensor(float(n), dtype=torch.float32)) == n     # k = -g / (float)n = -1/2
    dy, dp = sentinel(n), sentinel(n)
    _C.call("pnp_cross_entropy_bwd", ptr(y), ptr(p), ptr(g), n, ptr(dy), ptr(dp), rt.stream())
    sync()
    rdy, rdp = M.cross_entropy_bwd_ref(y, p, float(g), n)
    exact = ((p < M.CE_CLIP_LO) | (p > 1) | (torch.frexp(p).mantissa.abs() == 0.5))
    assert bool(exact.all())
    assert_bits("dp n %d" % n, dp, rdp.float())
    ratio = M.worst_ratio(dy, rdy, rdy.abs())
    print("  RATIO cross_entropy dy n %-9d worst |got-ref|/|ref| %.3e  a priori bound %.3e" % (n, ratio, M.CE_DY_BOUND))
    assert ratio <= M.CE_DY_BOUND
    assert bool((dy[p == 1] == 0).all())


def test_cross_entropy_bwd_real():
    """randn-derived y and p in (0, 1.5), an inexact k: dy within CE_DY_BOUND, dp within CE_DP_BOUND; one output NULL at a time"""
    _C, rt = lib()
    n = 100003
    g = cpu_gen(5)
    y = torch.rand((n,), generator=g).to(DEV)
    p = torch.rand((n,), generator=g) * 1.5
    p[:3] = torch.tensor([M.CE_CLIP_LO, 1.0, 1e-12])
    p = p.to(DEV)
    gout = torch.tensor([0.3], dtype=torch.float32, device=DEV)
    rdy, rdp = M.cross_entropy_bwd_ref(y, p, float(gout), n)
    dy, dp = sentinel(n), sentinel(n)
    _C.call("pnp_cross_entropy_bwd", ptr(y), ptr(p), ptr(gout), n, ptr(dy), None, rt.stream())
    _C.call("pnp_cross_entropy_bwd", ptr(y), ptr(p), ptr(gout), n, None, ptr(dp), rt.stream())
    sync()
    r1 = M.worst_ratio(dy, rdy, rdy.abs())
    r2 = M.worst_ratio(dp, rdp, rdp.abs())
    print("  RATIO cross_entropy dy %.3e (bound %.3e)  dp %.3e (bound %.3e)" % (r1, M.CE_DY_BOUND, r2, M.CE_DP_BOUND))
    assert r1 <= M.CE_DY_BOUND and r2 <= M.CE_DP_BOUND


@pytest.mark.parametrize("n", CE_N)
def test_cross_entropy_fwd(n):
    """acc (caller-zeroed) receives sum y log(clip p) within ce_acc_bound(n) * sum|y log clip p|; out = fl32(-acc / n) of the
    kernel's own acc.  A second call without re-zeroing adds the same sum again."""
    _C, rt = lib()
    launch = M.ce_acc_launch(n)
    _launch_note("n %d" % n, launch)
    y, p = ce_operands(n, n + 1)
    if n > 1:
        y = y + torch.rand((n,), generator=cpu_gen(n)).to(DEV) / 8        # inexact terms
    ref, mag = M.cross_entropy_fwd_ref(y, p)
    acc = torch.zeros(1, dtype=torch.float64, device=DEV)
    out = sentinel(1)
    bound = M.ce_acc_bound(n)
    ratios = []
    for k in (1, 2):
        _C.call("pnp_cross_entropy_fwd", ptr(y), ptr(p), n, ptr(acc), ptr(out), rt.stream())
        sync()
        ratios.append(abs(float(acc) - k * float(ref)) / (k * float(mag)) if float(mag) else abs(float(acc)))
        assert_bits("out after call %d" % k, out, torch.tensor([-float(acc) / n], dtype=torch.float64, device=DEV).float())
    print("  RATIO cross_entropy acc n %-9d worst |acc-ref|/sum|terms| %.3e  a priori bound %.3e" % (n, max(ratios), bound))
    assert max(ratios) <= bound, ratios


# ------------------------------------------------------------------------------------------------
# d. rejected calls
# ------------------------------------------------------------------------------------------------
NBUF = 4096


def _rejections():
    """(tag, builder, expected code); the builder gets a dict of sentinel-filled buffers of NBUF elements and returns
    (launcher, args without the stream).  Every shape is small enough for those buffers."""
    R = []
    f = lambda name, *a: (lambda b: (name, tuple(ptr(b[x]) if isinstance(x, str) else x for x in a)))  # noqa: E731
    N = None
    for H, W in ((3, 4), (4, 5)):
        R += [("maxpool2_fwd %dx%d" % (H, W), f("pnp_maxpool2_fwd", "x", "y", 2, H, W, 4), UNSUPPORTED),
              ("maxpool2_bwd %dx%d" % (H, W), f("pnp_maxpool2_bwd", "x", "dy", "dx", 2, H, W, 3), UNSUPPORTED),
              ("avgpool2 %dx%d" % (H, W), f("pnp_avgpool2", "x", "y", 2, H, W, 4, 0), UNSUPPORTED),
              ("avgpool2 bwd %dx%d" % (H, W), f("pnp_avgpool2", "dy", "dx", 2, H, W, 4, 1), UNSUPPORTED)]
    R += [("maxpool2_fwd B0", f("pnp_maxpool2_fwd", "x", "y", 0, 4, 4, 4), BAD_ARG),
          ("maxpool2_fwd C0", f("pnp_maxpool2_fwd", "x", "y", 2, 4, 4, 0), BAD_ARG),
          ("maxpool2_fwd no y", f("pnp_maxpool2_fwd", "x", N, 2, 4, 4, 4), BAD_ARG),
          ("maxpool2_bwd no x", f("pnp_maxpool2_bwd", N, "dy", "dx", 2, 4, 4, 4), BAD_ARG),
          ("maxpool2_bwd H0", f("pnp_maxpool2_bwd", "x", "dy", "dx", 2, 0, 4, 4), BAD_ARG),
          ("avgpool2 W0", f("pnp_avgpool2", "x", "y", 2, 4, 0, 4, 0), BAD_ARG),
          ("pool_fwd n0", f("pnp_pool_fwd", "x", "y", 2, 5, 5, 3, 0, 0), BAD_ARG),
          ("pool_fwd n-1", f("pnp_pool_fwd", "x", "y", 2, 5, 5, 3, -1, 1), BAD_ARG),
          ("pool_fwd C0", f("pnp_pool_fwd", "x", "y", 2, 5, 5, 0, 2, 0), BAD_ARG),
          ("pool_fwd no x", f("pnp_pool_fwd", N, "y", 2, 5, 5, 3, 2, 0), BAD_ARG),
          ("pool_bwd n0", f("pnp_pool_bwd", "x", "dy", "dx", 2, 5, 5, 3, 0, 0), BAD_ARG),
          ("pool_bwd max without x", f("pnp_pool_bwd", N, "dy", "dx", 2, 5, 5, 3, 2, 0), BAD_ARG),
          ("pool_bwd no dx", f("pnp_pool_bwd", "x", "dy", N, 2, 5, 5, 3, 2, 1), BAD_ARG),
          ("pool_bwd B0", f("pnp_pool_bwd", "x", "dy", "dx", 0, 5, 5, 3, 2, 1), BAD_ARG)]
    for name in ("pnp_mirror_pad_fwd", "pnp_mirror_pad_bwd"):
        s = name[4:]
        R += [("%s p>H" % s, f(name, "x", "y", 2, 3, 5, 3, 4), UNSUPPORTED),
              ("%s p>W" % s, f(name, "x", "y", 2, 5, 3, 3, 4), UNSUPPORTED),
              ("%s p<0" % s, f(name, "x", "y", 2, 5, 5, 3, -1), BAD_ARG),
              ("%s C0" % s, f(name, "x", "y", 2, 5, 5, 0, 1), BAD_ARG),
              ("%s no out" % s, f(name, "x", N, 2, 5, 5, 3, 1), BAD_ARG)]
    for name in ("pnp_phase_shift_fwd", "pnp_phase_shift_bwd"):
        s = name[4:]
        R += [("%s coff+ntile*G>Ctot" % s, f(name, "x", "y", 2, 2, 2, 2, 2, 7, 2, 3, 0), BAD_ARG),
              ("%s coff<0" % s, f(name, "x", "y", 2, 2, 2, 2, 2, 8, -1, 1, 0), BAD_ARG),
              ("%s r0" % s, f(name, "x", "y", 2, 2, 2, 2, 0, 8, 0, 1, 0), BAD_ARG),
              ("%s ntile0" % s, f(name, "x", "y", 2, 2, 2, 2, 2, 8, 0, 0, 0), BAD_ARG),
              ("%s G0" % s, f(name, "x", "y", 2, 2, 2, 0, 2, 8, 0, 1, 0), BAD_ARG),
              ("%s no src" % s, f(name, N, "y", 2, 2, 2, 2, 2, 8, 0, 1, 0), BAD_ARG)]
    R += [("logits_argmax_concat coff+C+1>Ctot", f("pnp_logits_argmax_concat", "x", "y", 64, 5, 6, 1), BAD_ARG),
          ("logits_argmax_concat coff<0", f("pnp_logits_argmax_concat", "x", "y", 64, 3, 6, -1), BAD_ARG),
          ("logits_argmax_concat P0", f("pnp_logits_argmax_concat", "x", "y", 0, 3, 6, 0), BAD_ARG),
          ("logits_argmax_concat C0", f("pnp_logits_argmax_concat", "x", "y", 64, 0, 6, 0), BAD_ARG),
          ("channel_slice off+Cs>C", f("pnp_channel_slice", "x", 8, 5, 4, "y", 64, 0), BAD_ARG),
          ("channel_slice off<0", f("pnp_channel_slice", "x", 8, -1, 4, "y", 64, 1), BAD_ARG),
          ("channel_slice Cs0", f("pnp_channel_slice", "x", 8, 0, 0, "y", 64, 0), BAD_ARG),
          ("channel_slice M0", f("pnp_channel_slice", "x", 8, 0, 4, "y", 0, 0), BAD_ARG),
          ("crop_concat_fwd H2>H1", f("pnp_crop_concat_fwd", "x", "x2", "y", 2, 4, 6, 3, 5, 4, 2), BAD_ARG),
          ("crop_concat_fwd W2>W1", f("pnp_crop_concat_fwd", "x", "x2", "y", 2, 6, 4, 3, 4, 5, 2), BAD_ARG),
          ("crop_concat_fwd C2 0", f("pnp_crop_concat_fwd", "x", "x2", "y", 2, 6, 6, 3, 4, 4, 0), BAD_ARG),
          ("crop_concat_fwd no x2", f("pnp_crop_concat_fwd", "x", N, "y", 2, 6, 6, 3, 4, 4, 2), BAD_ARG),
          ("crop_concat_bwd no outputs", f("pnp_crop_concat_bwd", "dy", N, N, 2, 6, 6, 3, 4, 4, 2), BAD_ARG),
          ("crop_concat_bwd H2>H1", f("pnp_crop_concat_bwd", "dy", "dx", "dx2", 2, 4, 6, 3, 5, 4, 2), BAD_ARG),
          ("one_hot C0", f("pnp_one_hot", "lab", "y", 64, 0), BAD_ARG),
          ("one_hot P0", f("pnp_one_hot", "lab", "y", 0, 4), BAD_ARG),
          ("fill n0", f("pnp_fill", "y", 1.0, 0), BAD_ARG),
          ("fill n-3", f("pnp_fill", "y", 1.0, -3), BAD_ARG),
          ("fill NULL", f("pnp_fill", N, 1.0, 16), BAD_ARG),
          ("pixel_softmax2 C9", f("pnp_pixel_softmax2", "x", "y", 64, 9), UNSUPPORTED),
          ("pixel_softmax2 C0", f("pnp_pixel_softmax2", "x", "y", 64, 0), BAD_ARG),
          ("pixel_softmax2 P0", f("pnp_pixel_softmax2", "x", "y", 0, 2), BAD_ARG),
          ("cross_entropy_fwd n0", f("pnp_cross_entropy_fwd", "x", "x2", 0, "acc", "y"), BAD_ARG),
          ("cross_entropy_fwd no acc", f("pnp_cross_entropy_fwd", "x", "x2", 64, N, "y"), BAD_ARG),
          ("cross_entropy_fwd no out", f("pnp_cross_entropy_fwd", "x", "x2", 64, "acc", N), BAD_ARG),
          ("cross_entropy_bwd no outputs", f("pnp_cross_entropy_bwd", "x", "x2", "g", 64, N, N), BAD_ARG),
          ("cross_entropy_bwd n-1", f("pnp_cross_entropy_bwd", "x", "x2", "g", -1, "dx", "dx2"), BAD_ARG)]
    return R


def _disc_rejections():
    """(tag, plan overrides, expected code) of pnp_disc_input_fwd around the valid plan B 2, a = b = 1, r 4, G (2, 4), ntile
    (3, 1), NC 5 (Ctot 16)"""
    return [("a*r != H", dict(H=8), BAD_ARG), ("b*r != W", dict(W=5), BAD_ARG), ("nsrc 0", dict(nsrc=0), BAD_ARG),
            ("nsrc 5", dict(nsrc=5), BAD_ARG), ("NC 0", dict(NC=0), BAD_ARG), ("NC 9", dict(NC=9), BAD_ARG),
            ("r 0", dict(r=0), BAD_ARG), ("B 0", dict(B=0), BAD_ARG), ("G 0", dict(G=(0, 4)), BAD_ARG),
            ("ntile 0", dict(nt=(0, 1)), BAD_ARG), ("NULL source", dict(null_src=1), BAD_ARG),
            ("NULL logits", dict(null_logits=True), BAD_ARG),
            ("Ctot 15", dict(NC=4), UNSUPPORTED), ("sources past 64 channels", dict(G=(8, 8), nt=(8, 1), NC=1), UNSUPPORTED),
            ("logits past 64 channels", dict(G=(8, 8), nt=(6, 2), NC=1), UNSUPPORTED),
            ("argmax past 64 channels", dict(G=(8, 8), nt=(6, 1), NC=8), UNSUPPORTED)]


REJECT = _rejections()
DISC_REJECT = _disc_rejections()


def _buffers():
    b = {k: sentinel(NBUF) for k in ("x", "x2", "y", "dy", "dx", "dx2", "g")}
    b["lab"] = torch.zeros(NBUF, dtype=torch.int64, device=DEV)
    b["acc"] = torch.full((NBUF,), 1234.5, dtype=torch.float64, device=DEV)
    return b


@pytest.mark.parametrize("i", range(len(REJECT)), ids=[r[0].replace(" ", "_") for r in REJECT])
def test_rejected_calls_leave_outputs_untouched(i):
    _C, rt = lib()
    tag, build, code = REJECT[i]
    b = _buffers()
    before = snapshot(b)
    name, args = build(b)
    sync()
    rc = getattr(_C.lib, name)(*(args + (rt.stream(),)))
    sync()
    assert rc == code, "%s: %s returned %d, expected %d" % (tag, name, rc, code)
    assert_untouched(tag, name, b, before)


@pytest.mark.parametrize("i", range(len(DISC_REJECT)), ids=[r[0].replace(" ", "_") for r in DISC_REJECT])
def test_disc_input_rejections(i):
    _C, rt = lib()
    tag, o, code = DISC_REJECT[i]
    B, r, G, nt, NC = o.get("B", 2), o.get("r", 4), o.get("G", (2, 4)), o.get("nt", (3, 1)), o.get("NC", 5)
    H, W = o.get("H", 4), o.get("W", 4)
    nsrc = o.get("nsrc", 2)
    b = _buffers()
    before = snapshot(b)
    srcs = (ctypes.c_void_p * 5)(*([ptr(b["x"]), ptr(b["x2"])] * 3)[:5])
    if "null_src" in o:
        srcs[o["null_src"]] = None
    I = ctypes.c_int * 5
    Gs, nts = I(*(list(G) + [1, 1, 1])), I(*(list(nt) + [1, 1, 1]))
    a_, b_ = I(*[1] * 5), I(*[1] * 5)
    rc = _C.lib.pnp_disc_input_fwd(srcs, a_, b_, Gs, nts, nsrc, None if o.get("null_logits") else ptr(b["g"]), NC, ptr(b["y"]),
                                   B, H, W, r, 0, rt.stream())
    sync()
    assert rc == code, "%s: pnp_disc_input_fwd returned %d, expected %d" % (tag, rc, code)
    assert_untouched(tag, "pnp_disc_input_fwd", b, before)


def test_disc_input_rejects_the_32bit_index_limit():
    """B * H * W * 64 >= 2^31 pixels-times-64 is UNSUPPORTED (the kernels index in 32 bits), with real buffers of that size"""
    _C, rt = lib()
    H = W = 5793                                  # 5793^2 * 64 >= 2^31
    assert H * W * 64 >= 1 << 31 and H * W * 4 < 1 << 31
    src = sentinel(H * W)
    logits = sentinel(H * W * 2)
    out = sentinel(H * W * 4)
    rc = _disc_call(_C, rt, [src], (1,), (1,), logits.view(1, H, W, 2), out, 1, H, W, 1, 0)
    sync()
    assert rc == UNSUPPORTED, rc
    for t in (src, logits, out):
        assert bool((t.view(torch.int32) == SENTINEL).all())


# ------------------------------------------------------------------------------------------------
# e. programmatic dependent launch
# ------------------------------------------------------------------------------------------------
PDL_SELECTION = " or ".join(["maxpool2_exact", "avgpool2_exact", "test_pool_exact", "signed_zero", "mirror_pad_exact",
                              "phase_shift_exact", "disc_input_exact", "functional_fallback", "logits_argmax_concat_exact",
                              "channel_slice_exact", "crop_concat_exact", "one_hot_exact", "fill_exact"])


@pytest.mark.timeout(600)
def test_exact_cases_under_pdl():
    passed, _ = rerun({"PNP_PDL": "1"}, __file__, PDL_SELECTION, flags=("-s",), timeout=580)
    assert passed == (2 * len(MAXPOOL2_CASES) + len(POOL_CASES) + 1 + len(MIRROR_CASES) + len(PS_CASES) + len(DISC_CASES) + 2 +
                      len(LAC_CASES) + len(SLICE_CASES) + len(CAT_CASES) + len(ONE_HOT_CASES) + len(FILL_N)), passed
