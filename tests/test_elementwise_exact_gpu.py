"""The batch-norm, activation, loss and metric kernels of elementwise.cu against fp64 references (oracle/elementwise_exact.py),
called at the C-ABI, at every launch regime of the BN reductions.

a. exact cases: operands are chosen so that every intermediate is representable (integers, dyadic scale / invstd / gamma,
   sums that are M times a dyadic value, logits equal within a pixel), so results equal the fp64 reference at every element
   (torch.equal).  Each case asserts its own precondition first.  The BN reductions run every threads-per-row count from 1 to
   256, idle channel lanes, a ragged last CTA, odd row counts, M below the row-lane count, the grid cap at the real 16-channel
   layer and the fp32 -> fp64 promotion; fused and separate backward routes are bit-equal;
b. real-valued cases (randn): |got - ref| <= TAU * magnitude per element, the invstd ulp sweep of pnp_bn_finalize;
c. the sign of subnormal activations (y against its bf16 hi plane) and the conditioning of the one-pass variance;
d. rejected calls return PNP_ERR_BAD_ARG / PNP_ERR_UNSUPPORTED and leave every output untouched;
e. the exact reduce and apply cases again under PNP_PDL=1, in their own process.

Each real-valued test prints its worst ratio |got - ref| / magnitude next to TAU."""
import ctypes

import pytest
import torch

from oracle import bf16_split as S
from oracle import elementwise_exact as E
from tests.cabi import (BAD_ARG, DEV, UNSUPPORTED, assert_planes, assert_untouched, dev_gen, drop_cfg, drop_mask, empty_planes, ints,
                        lib, pick, ptr, rerun, snapshot, sync)

pytestmark = pytest.mark.gpu

# (id, M, C) of the BN reductions; the CPU file checks that together they reach every regime of E.reduce_regimes
REDUCE_CASES = [
    ("tpr1_C4", 3001, 4), ("tpr2_C8", 3001, 8), ("tpr4_C16", 3001, 16), ("tpr8_C32", 3001, 32), ("tpr16_C64", 3001, 64),
    ("tpr32_C128", 3001, 128), ("tpr64_C256", 3001, 256), ("tpr128_C512", 3001, 512), ("tpr256_C1024", 3001, 1024),
    ("idle_C12", 777, 12), ("idle_C40", 777, 40), ("idle_C320", 777, 320), ("idle_C520", 777, 520),
    ("M1_C4", 1, 4), ("M4_C4", 4, 4), ("M4_C64", 4, 64), ("critic2x2_B8_C512", 32, 512),
    ("capped_16ch_B16", 1048576, 16),            # the 16-channel layers at B = 16 (256 x 256 maps)
    ("promoted_C1024", 70001, 1024),             # > 64 rows per thread: fp32 partials promoted to fp64 mid-row-loop
]
BIG = {"capped_16ch_B16", "promoted_C1024"}
# (id, M, C) of the streaming apply kernels: the shared-memory extremes and a grid above grid_for's 8448-CTA cap
APPLY_SHAPES = [("C4", 1001, 4), ("C1024", 37, 1024), ("C96", 1000, 96), ("grid_stride_C16", 600000, 16)]
SKIPS = {4: [(4, 0)], 1024: [(512, 256), (4, 1020)], 96: [(32, 40), (96, 0)], 16: [(8, 8)]}
BWD_SHAPES = [("C64", 3000, 64), ("C1024", 4, 1024), ("C4_M1", 1, 4), ("grid_stride_C16", 600000, 16)]
SEG_P = [524288, 100003]


def var_for_invstd(inv):
    """an fp32 variance v with fl(v + 1e-3f) == 1 / inv^2 exactly, so that pnp_bn_finalize's invstd is exactly inv"""
    target = torch.tensor(1.0 / (inv * inv), dtype=torch.float32)
    eps = torch.tensor(E.BN_EPS, dtype=torch.float32)
    v = target - eps
    for k in range(-4, 5):
        c = (v.view(torch.int32) + k).view(torch.float32)
        if bool(c + eps == target):
            return float(c)
    raise AssertionError("no fp32 variance lands on %r" % inv)


def _report(key, tag, ratio):
    tau = E.TAU[key]
    print("  RATIO %-13s %-36s worst |got-ref|/magnitude %.3e  tau %.3e" % (key, tag, ratio, tau))
    return tau


def check(key, tag, got, ref, mag):
    ratio = E.worst_ratio(got, ref, mag)
    tau = _report(key, tag, ratio)
    bad = E.violations(got, ref, mag, tau)
    assert bad == 0, "%s %s: %d elements beyond tau %.3e (worst ratio %.3e)" % (key, tag, bad, tau, ratio)


# ------------------------------------------------------------------------------------------------
# a. BN reductions, exact
# ------------------------------------------------------------------------------------------------
def reduce_operands(M, C, seed):
    """integer z in [-8, 8], integer mean, invstd in {1, .5}, dy in 5 * [-8, 8] (fl(0.2f * dy) = dy / 5), y in [-3, 3]"""
    gen = dev_gen(seed)
    z = ints((M, C), -8, 8, gen)
    mean = ints((C,), -2, 2, gen)
    invstd = pick((C,), [1.0, 0.5], gen)
    dy = ints((M, C), -8, 8, gen, 5.0)
    y = ints((M, C), -3, 3, gen)
    return z, mean, invstd, dy, y


def reduce_precondition(term_max):
    """each thread sums at most 64 rows in fp32 before promoting: those partials must stay exact integers (or halves)"""
    assert E.PROMOTE_ROWS * term_max < E.F32_EXACT / 2, term_max


@pytest.mark.parametrize("case", REDUCE_CASES, ids=[c[0] for c in REDUCE_CASES])
def test_bn_stats_exact(case):
    _C, rt = lib()
    tag, M, C = case
    gen = dev_gen(M + C)
    z = ints((M, C), -8, 8, gen)
    reduce_precondition(64)
    init = ints((C,), -3, 3, gen).double()
    s1, s2 = init.clone(), init.clone()
    _C.call("pnp_bn_stats", ptr(z), M, C, ptr(s1), ptr(s2), rt.stream())
    sync()
    r1, r2, _ = E.bn_stats_ref(z)
    print("  %s: %s" % (tag, sorted(E.reduce_regimes(M, C))))
    assert torch.equal(s1, init + r1), "%s: sum differs by up to %g" % (tag, float((s1 - init - r1).abs().max()))
    assert torch.equal(s2, init + r2), "%s: sumsq differs by up to %g" % (tag, float((s2 - init - r2).abs().max()))


@pytest.mark.parametrize("case", REDUCE_CASES, ids=[c[0] for c in REDUCE_CASES])
def test_bn_bwd_reduce_exact(case):
    """pnp_bn_bwd_reduce (g and sums, sign from y) and pnp_bn_bwd_reduce_sums (sign from y and from y_hi) against fp64 sums of
    the same g: all three sums are equal, so the sums-only route is the sums of the g-writing route"""
    _C, rt = lib()
    tag, M, C = case
    z, mean, invstd, dy, y = reduce_operands(M, C, 7 + M + C)
    yhi = y.to(torch.bfloat16)
    reduce_precondition(40 * 10)
    gen = dev_gen(3)
    for act in ((E.LRELU,) if tag in BIG else (E.NONE, E.RELU, E.LRELU)):
        g_ref, sg_ref, sgx_ref, _, _ = E.bn_bwd_reduce_ref(dy, y, z, mean, invstd, act)
        init = ints((C,), -3, 3, gen).double()
        g = torch.full((M, C), float("nan"), device=DEV)
        sg, sgx = init.clone(), init.clone()
        _C.call("pnp_bn_bwd_reduce", ptr(dy), ptr(y), ptr(z), ptr(mean), ptr(invstd), act, ptr(g), ptr(sg), ptr(sgx), M, C, rt.stream())
        sync()
        assert torch.equal(g, g_ref), "%s act %d: g = dy * act'(y) is not exact" % (tag, act)
        assert torch.equal(sg, init + sg_ref), "%s act %d: sum_g" % (tag, act)
        assert torch.equal(sgx, init + sgx_ref), "%s act %d: sum_gx" % (tag, act)
        for src in ("y", "y_hi"):
            sg2, sgx2 = init.clone(), init.clone()
            _C.call("pnp_bn_bwd_reduce_sums", ptr(dy), ptr(y) if src == "y" else None, ptr(yhi) if src == "y_hi" else None,
                    ptr(z), ptr(mean), ptr(invstd), act, ptr(sg2), ptr(sgx2), M, C, rt.stream())
            sync()
            assert torch.equal(sg2, sg) and torch.equal(sgx2, sgx), "%s act %d %s: reduce_sums != reduce" % (tag, act, src)
        del g


# ------------------------------------------------------------------------------------------------
# a. BN forward apply, exact
# ------------------------------------------------------------------------------------------------
def _skip_variants(C):
    return [(None, 0)] + SKIPS[C]


@pytest.mark.parametrize("shape", APPLY_SHAPES, ids=[s[0] for s in APPLY_SHAPES])
def test_bn_act_apply_exact(shape):
    """dyadic scale / shift and integer z, skip: fma + skip + act is exact; y only, and y with planes (planes == split(y))"""
    _C, rt = lib()
    tag, M, C = shape
    gen = dev_gen(M * 3 + C)
    z = ints((M, C), -8, 8, gen)
    scale = pick((C,), [-1.5, -1.0, -0.5, 0.5, 1.0, 2.0], gen)
    shift = ints((C,), -4, 4, gen, 0.5)
    for Cs, off in _skip_variants(C):
        skip = None if Cs is None else ints((M, Cs), -4, 4, gen)
        for act in (E.NONE, E.RELU, E.LRELU):
            y_ref, _ = E.bn_apply_ref(z, scale, shift, skip, off, act)
            for planes in (False, True):
                y = torch.full((M, C), float("nan"), device=DEV)
                hi, lo = empty_planes((M, C), 3) if planes else (None, None)
                _C.call("pnp_bn_act_apply", ptr(z), ptr(scale), ptr(shift), ptr(skip), Cs or 0, off, act, ptr(y), ptr(hi), ptr(lo),
                        M, C, rt.stream())
                sync()
                what = "%s skip=%s@%d act %d planes %d" % (tag, Cs, off, act, planes)
                assert torch.equal(y, y_ref), what
                if planes:
                    assert_planes(what, hi, lo, y_ref)


@pytest.mark.parametrize("training", [0, 1])
@pytest.mark.parametrize("shape", APPLY_SHAPES, ids=[s[0] for s in APPLY_SHAPES])
def test_bn_apply_fused_exact(shape, training):
    """pnp_bn_apply_fused with statistics that make invstd exactly 1 or 2 (training 0: moving statistics; training 1: fp64
    sums that are M times an integer mean and an exact variance): scale, shift and y are exact; mean_out / invstd_out are the
    statistics; y only, planes only and both write the same values; training 1 updates the moving statistics (within TAU)"""
    _C, rt = lib()
    tag, M, C = shape
    gen = dev_gen(M + 5 * C + training)
    z = ints((M, C), -8, 8, gen)
    inv = pick((C,), [1.0, 2.0], gen)
    var = torch.where(inv == 1.0, torch.full_like(inv, var_for_invstd(1.0)), torch.full_like(inv, var_for_invstd(2.0)))
    mu = ints((C,), -2, 2, gen)
    gamma = pick((C,), [0.5, 1.0, 1.5, 2.0], gen)
    beta = ints((C,), -4, 4, gen, 0.25)
    mm0, mv0 = ints((C,), -2, 2, gen), pick((C,), [1.0, 2.0], gen)
    if training:
        s1 = mu.double() * M
        s2 = (var.double() + mu.double() ** 2) * M
        assert torch.equal(s2 / M - (s1 / M) ** 2, var.double()), "the variance is not exact in fp64"
        mm_in, mv_in = mm0, mv0
    else:
        s1 = s2 = None
        mm_in, mv_in = mu, var
    scale = gamma * inv
    shift = beta - mu * scale
    outs = []
    for Cs, off in _skip_variants(C):
        skip = None if Cs is None else ints((M, Cs), -4, 4, gen)
        for act in (E.NONE, E.RELU, E.LRELU):
            y_ref, _ = E.bn_apply_ref(z, scale, shift, skip, off, act)
            got = {}
            for mode in ("y", "planes", "both"):
                y = torch.full((M, C), float("nan"), device=DEV) if mode != "planes" else None
                hi, lo = empty_planes((M, C), 3) if mode != "y" else (None, None)
                mm, mv = mm_in.clone(), mv_in.clone()
                mo, io = torch.full((C,), float("nan"), device=DEV), torch.full((C,), float("nan"), device=DEV)
                _C.call("pnp_bn_apply_fused", ptr(z), ptr(s1), ptr(s2), M, C, ptr(gamma), ptr(beta), ptr(mm), ptr(mv), training,
                        ptr(skip), Cs or 0, off, act, ptr(y), ptr(hi), ptr(lo), ptr(mo), ptr(io), rt.stream())
                sync()
                what = "%s train %d skip=%s@%d act %d %s" % (tag, training, Cs, off, act, mode)
                assert torch.equal(io, inv), what + ": invstd_out"
                assert torch.equal(mo, mu), what + ": mean_out"
                if y is not None:
                    assert torch.equal(y, y_ref), what
                if hi is not None:
                    assert_planes(what, hi, lo, y_ref)
                    got[mode] = (S.bits(hi), S.bits(lo))
                if not training:
                    assert torch.equal(mm, mm_in) and torch.equal(mv, mv_in), what + ": moving statistics changed"
                else:
                    outs.append((mm, mv))
            assert all(torch.equal(a, b) for a, b in zip(got["planes"], got["both"])), "planes-only launch wrote other planes"
    if training:
        ref = E.bn_finalize_ref(s1, s2, M, gamma, beta, mm0, mv0, 1)
        for mm, mv in outs:
            check("bn_finalize", "%s moving_mean" % tag, mm, *ref["moving_mean"])
            check("bn_finalize", "%s moving_var" % tag, mv, *ref["moving_var"])


# ------------------------------------------------------------------------------------------------
# a. BN backward apply, exact
# ------------------------------------------------------------------------------------------------
def bwd_operands(M, C, seed):
    gen = dev_gen(seed)
    z, mean, invstd, dy, y = reduce_operands(M, C, seed + 1)
    gamma = pick((C,), [0.5, 1.0, 1.5, 2.0], gen)
    c1 = ints((C,), -8, 8, gen, 0.25)
    c2 = ints((C,), -8, 8, gen, 0.25)
    sg, sgx = c1.double() * M, c2.double() * M            # c1 = sum_g / M and c2 = sum_gx / M are exact
    dgamma0, dbeta0 = ints((C,), -4, 4, gen, 0.5), ints((C,), -4, 4, gen, 0.5)
    return z, mean, invstd, dy, y, gamma, c1, c2, sg, sgx, dgamma0, dbeta0


@pytest.mark.parametrize("keep", [1.0, 0.5, 0.75])
@pytest.mark.parametrize("training", [0, 1])
@pytest.mark.parametrize("shape", BWD_SHAPES, ids=[s[0] for s in BWD_SHAPES])
def test_bn_bwd_apply_exact(shape, training, keep):
    """_bwd_finalize -> _bwd_apply, _bwd_apply_fused and _bwd_apply_direct (every act, sign from y and from y_hi, dz and
    planes-only) against the fp64 dz, the dropout multiplier applied as the final fp32 multiply; dgamma / dbeta accumulate"""
    _C, rt = lib()
    tag, M, C = shape
    z, mean, invstd, dy, y, gamma, c1, c2, sg, sgx, dg0, db0 = bwd_operands(M, C, 11 * M + C + training)
    yhi = y.to(torch.bfloat16)
    dcfg, _seed = drop_cfg(_C, keep) if keep < 1 else (None, None)
    dref = None if dcfg is None else ctypes.byref(dcfg)
    mask = drop_mask(dcfg, (M, C)) if dcfg is not None else None
    # finalize: coef exact, dgamma / dbeta += sums
    coef = torch.full((2 * C,), float("nan"), device=DEV)
    dg, db = dg0.clone(), db0.clone()
    _C.call("pnp_bn_bwd_finalize", ptr(sg), ptr(sgx), M, C, ptr(dg), ptr(db), ptr(coef), rt.stream())
    sync()
    assert torch.equal(coef, torch.cat([c1, c2])), tag + ": coef"
    assert torch.equal(dg, dg0 + sgx.float()) and torch.equal(db, db0 + sg.float()), tag + ": dgamma / dbeta"
    # separate apply from g = dy
    dz_ref, _ = E.bn_bwd_apply_ref(dy, z, mean, invstd, gamma, c1, c2, training, mask)
    dz = torch.full((M, C), float("nan"), device=DEV)
    hi, lo = empty_planes((M, C), 3)
    _C.call("pnp_bn_bwd_apply", ptr(dy), ptr(z), ptr(mean), ptr(invstd), ptr(gamma), ptr(coef), training, dref, ptr(dz), ptr(hi),
            ptr(lo), M, C, rt.stream())
    sync()
    what = "%s train %d keep %g" % (tag, training, keep)
    assert torch.equal(dz, dz_ref), what + ": pnp_bn_bwd_apply"
    assert_planes(what, hi, lo, dz_ref)
    # fused: the same dz, dgamma / dbeta accumulated by CTA 0
    dz = torch.full((M, C), float("nan"), device=DEV)
    dg, db = dg0.clone(), db0.clone()
    _C.call("pnp_bn_bwd_apply_fused", ptr(dy), ptr(z), ptr(mean), ptr(invstd), ptr(gamma), ptr(sg), ptr(sgx), M, C, training, dref,
            ptr(dg), ptr(db), ptr(dz), ptr(hi), ptr(lo), rt.stream())
    sync()
    assert torch.equal(dz, dz_ref), what + ": pnp_bn_bwd_apply_fused"
    assert_planes(what + " fused", hi, lo, dz_ref)
    assert torch.equal(dg, dg0 + sgx.float()) and torch.equal(db, db0 + sg.float()), what + ": fused dgamma / dbeta"
    # direct: g = dy * act'(y) recomputed, sign from y or y_hi; dz = NULL writes the same planes
    for act in (E.NONE, E.RELU, E.LRELU):
        g = dy * E.act_slope(y, act)
        dref_act, _ = E.bn_bwd_apply_ref(g, z, mean, invstd, gamma, c1, c2, training, mask)
        for src in ("y", "y_hi"):
            planes = []
            for with_dz in (True, False):
                dz = torch.full((M, C), float("nan"), device=DEV) if with_dz else None
                hi, lo = empty_planes((M, C), 3)
                dg, db = dg0.clone(), db0.clone()
                _C.call("pnp_bn_bwd_apply_direct", ptr(dy), ptr(y) if src == "y" else None, ptr(yhi) if src == "y_hi" else None, act,
                        ptr(z), ptr(mean), ptr(invstd), ptr(gamma), ptr(sg), ptr(sgx), M, C, training, dref, ptr(dg), ptr(db), ptr(dz),
                        ptr(hi), ptr(lo), rt.stream())
                sync()
                w = "%s direct act %d %s dz %d" % (what, act, src, with_dz)
                if with_dz:
                    assert torch.equal(dz, dref_act), w
                assert_planes(w, hi, lo, dref_act)
                assert torch.equal(dg, dg0 + sgx.float()), w + ": dgamma"
                planes.append((S.bits(hi), S.bits(lo)))
            assert torch.equal(planes[0][0], planes[1][0]) and torch.equal(planes[0][1], planes[1][1]), w


def test_bn_bwd_routes_are_bit_equal():
    """randn operands, training with dropout: _bwd_apply_fused == _bwd_reduce -> _bwd_finalize -> _bwd_apply, and
    _bwd_apply_direct(dy, y) == pnp_act_bwd -> _bwd_apply_fused, bit for bit (the same sums feed both routes)"""
    _C, rt = lib()
    M, C = 3000, 64
    g0 = torch.Generator().manual_seed(5)
    f = lambda *s: torch.randn(*s, generator=g0).to(DEV)  # noqa: E731
    z, dy, y = f(M, C) * 2 + 0.3, f(M, C), f(M, C)
    mean, invstd, gamma = f(C) * 0.1, torch.rand(C, generator=g0).to(DEV) + 0.5, 1 + 0.3 * f(C)
    dcfg, _seed = drop_cfg(_C, 0.75)
    for act in (E.NONE, E.RELU, E.LRELU):
        g = torch.empty(M, C, device=DEV)
        sg, sgx = torch.zeros(C, dtype=torch.float64, device=DEV), torch.zeros(C, dtype=torch.float64, device=DEV)
        _C.call("pnp_bn_bwd_reduce", ptr(dy), ptr(y), ptr(z), ptr(mean), ptr(invstd), act, ptr(g), ptr(sg), ptr(sgx), M, C, rt.stream())
        coef = torch.empty(2 * C, device=DEV)
        _C.call("pnp_bn_bwd_finalize", ptr(sg), ptr(sgx), M, C, None, None, ptr(coef), rt.stream())
        outs = []
        dz = torch.empty(M, C, device=DEV)
        _C.call("pnp_bn_bwd_apply", ptr(g), ptr(z), ptr(mean), ptr(invstd), ptr(gamma), ptr(coef), 1, ctypes.byref(dcfg), ptr(dz),
                None, None, M, C, rt.stream())
        outs.append(dz)
        dz = torch.empty(M, C, device=DEV)
        _C.call("pnp_bn_bwd_apply_fused", ptr(g), ptr(z), ptr(mean), ptr(invstd), ptr(gamma), ptr(sg), ptr(sgx), M, C, 1,
                ctypes.byref(dcfg), None, None, ptr(dz), None, None, rt.stream())
        outs.append(dz)
        g2 = torch.empty(M, C, device=DEV)
        _C.call("pnp_act_bwd", ptr(dy), ptr(y), act, ptr(g2), M * C, rt.stream())
        dz = torch.empty(M, C, device=DEV)
        _C.call("pnp_bn_bwd_apply_fused", ptr(g2), ptr(z), ptr(mean), ptr(invstd), ptr(gamma), ptr(sg), ptr(sgx), M, C, 1,
                ctypes.byref(dcfg), None, None, ptr(dz), None, None, rt.stream())
        outs.append(dz)
        dz = torch.empty(M, C, device=DEV)
        _C.call("pnp_bn_bwd_apply_direct", ptr(dy), ptr(y), None, act, ptr(z), ptr(mean), ptr(invstd), ptr(gamma), ptr(sg), ptr(sgx),
                M, C, 1, ctypes.byref(dcfg), None, None, ptr(dz), None, None, rt.stream())
        outs.append(dz)
        sync()
        assert torch.equal(g, g2), "act %d: pnp_act_bwd != the g of pnp_bn_bwd_reduce" % act
        names = ["reduce->finalize->apply", "apply_fused", "act_bwd->apply_fused", "apply_direct"]
        for n, o in zip(names[1:], outs[1:]):
            assert torch.equal(o, outs[0]), "act %d: %s differs from %s" % (act, n, names[0])


# ------------------------------------------------------------------------------------------------
# a. losses and metrics, exact
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P", SEG_P)
@pytest.mark.parametrize("C", [1, 2, 4, 8])
def test_segloss_reduce_exact_sums(C, P):
    """logits equal within each pixel: p = 1/C exactly, so sum y, sum p*y and sum p*p are exact for integer y"""
    _C, rt = lib()
    gen = dev_gen(C * P)
    logits = (torch.randn(P, 1, generator=gen, device=DEV) * 3).expand(P, C).contiguous()
    y = ints((P, C), 0, 3, gen)
    assert 32 * 3 < E.F32_EXACT
    acc = torch.zeros(4 * C, dtype=torch.float64, device=DEV)
    _C.call("pnp_segloss_reduce", ptr(logits), ptr(y), P, C, ptr(acc), rt.stream())
    sync()
    yd = y.double()
    want = torch.cat([yd.sum(0), yd.sum(0) / C, torch.full((C,), P / C / C, dtype=torch.float64, device=DEV)])
    assert torch.equal(acc[:3 * C], want), "C %d P %d: %s vs %s" % (C, P, acc[:3 * C].tolist(), want.tolist())
    ref, mag = E.segloss_reduce_ref(logits, y)
    check("seg_ce", "equal-logit CE C %d P %d" % (C, P), acc[3 * C:], ref[3 * C:], mag[3 * C:])


@pytest.mark.parametrize("P", SEG_P)
@pytest.mark.parametrize("C", [2, 5, 8])
def test_confusion_exact(C, P):
    """integer logits (many ties) and multi-hot labels (ties too): both argmaxes resolve to the first maximum"""
    _C, rt = lib()
    gen = dev_gen(C + P)
    logits = ints((P, C), -2, 2, gen)
    y = ints((P, C), 0, 1, gen)
    counts = torch.zeros(C * C, dtype=torch.int64, device=DEV)
    _C.call("pnp_confusion", ptr(logits), ptr(y), P, C, ptr(counts), rt.stream())
    sync()
    ref = E.confusion_ref(logits.cpu(), y.cpu())
    assert torch.equal(counts.cpu(), ref), (counts.tolist(), ref.tolist())


@pytest.mark.parametrize("n", [16 * 2048, 100003, 1])
def test_l2_loss_exact(n):
    _C, rt = lib()
    w = ints((n,), -8, 8, dev_gen(n))
    out = torch.full((1,), 3.0, dtype=torch.float64, device=DEV)
    _C.call("pnp_l2_loss_acc", ptr(w), n, ptr(out), rt.stream())
    sync()
    assert float(out) == 3.0 + float(E.l2_ref(w)), (float(out), float(E.l2_ref(w)))


@pytest.mark.parametrize("B,F", [(16, 2048), (3, 1001), (1, 1)])
def test_fc_exact(B, F):
    """out = x @ w; dx = dout * w; dw += x^T dout (accumulating into a non-zero dw)"""
    _C, rt = lib()
    gen = dev_gen(B * F)
    x, w, dout = ints((B, F), -8, 8, gen), ints((F,), -8, 8, gen), ints((B,), -8, 8, gen)
    assert 64 * F < E.F32_EXACT and 64 * B < E.F32_EXACT
    out = torch.full((B,), float("nan"), device=DEV)
    _C.call("pnp_fc_fwd", ptr(x), ptr(w), ptr(out), B, F, rt.stream())
    dx = torch.full((B, F), float("nan"), device=DEV)
    dw0 = ints((F,), -4, 4, gen)
    dw = dw0.clone()
    _C.call("pnp_fc_bwd", ptr(x), ptr(w), ptr(dout), ptr(dx), ptr(dw), B, F, rt.stream())
    sync()
    rdx, rdw = E.fc_bwd_ref(x, w, dout)
    assert torch.equal(out.double(), E.fc_fwd_ref(x, w))
    assert torch.equal(dx.double(), rdx)
    assert torch.equal(dw.double(), dw0.double() + rdw)


@pytest.mark.parametrize("n", [16 * 2048, 1001, 1])
@pytest.mark.parametrize("with_b", [True, False])
def test_mean_combo_exact(n, with_b):
    _C, rt = lib()
    gen = dev_gen(n)
    a, b = ints((n,), -8, 8, gen), ints((n,), -8, 8, gen)
    out = torch.full((1,), float("nan"), device=DEV)
    _C.call("pnp_mean_combo", ptr(a), 0.5, ptr(b) if with_b else None, -2.0, n, ptr(out), rt.stream())
    sync()
    ref = E.mean_combo_ref(a.cpu(), 0.5, b.cpu() if with_b else None, -2.0)
    assert float(out) == float(ref), (float(out), float(ref))


# ------------------------------------------------------------------------------------------------
# b. real-valued cases
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 4, 32, 3001, 8192])
def test_bn_training_real(M):
    """pnp_bn_finalize and pnp_bn_apply_fused (training, skip, leaky ReLU) from fp64 sums of randn z: mean, invstd, scale, shift,
    the moving averages (unbiased factor M / (M - 1), 1 at M = 1) and y within TAU; both launchers agree bit for bit"""
    _C, rt = lib()
    C = 64
    g0 = torch.Generator().manual_seed(M)
    f = lambda *s: torch.randn(*s, generator=g0).to(DEV)  # noqa: E731
    z = f(M, C) * 2 + 0.3
    gamma, beta, mm0, mv0 = 1 + 0.3 * f(C), 0.2 * f(C), 0.1 * f(C), 1 + 0.2 * torch.rand(C, generator=g0).to(DEV)
    skip = f(M, 32)
    s1, s2, sabs = E.bn_stats_ref(z)
    ref = E.bn_finalize_ref(s1, s2, M, gamma, beta, mm0, mv0, 1, s_abs=sabs)
    out = {k: torch.full((C,), float("nan"), device=DEV) for k in ("scale", "shift", "mean", "invstd")}
    mm, mv = mm0.clone(), mv0.clone()
    _C.call("pnp_bn_finalize", ptr(s1), ptr(s2), M, C, ptr(gamma), ptr(beta), ptr(mm), ptr(mv), 1, ptr(out["scale"]), ptr(out["shift"]),
            ptr(out["mean"]), ptr(out["invstd"]), rt.stream())
    y = torch.empty(M, C, device=DEV)
    mm2, mv2 = mm0.clone(), mv0.clone()
    mo, io = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    _C.call("pnp_bn_apply_fused", ptr(z), ptr(s1), ptr(s2), M, C, ptr(gamma), ptr(beta), ptr(mm2), ptr(mv2), 1, ptr(skip), 32, 16,
            E.LRELU, ptr(y), None, None, ptr(mo), ptr(io), rt.stream())
    sync()
    for k in ("scale", "shift", "mean", "invstd"):
        check("bn_finalize", "M %d %s" % (M, k), out[k], *ref[k])
    check("bn_finalize", "M %d moving_mean" % M, mm, *ref["moving_mean"])
    check("bn_finalize", "M %d moving_var" % M, mv, *ref["moving_var"])
    y_ref, y_mag = E.bn_apply_ref(z, ref["scale"][0], ref["shift"][0], skip, 16, E.LRELU, shift_mag=ref["shift"][1])
    check("bn_apply", "M %d y" % M, y, y_ref, y_mag)
    for a, b, n in ((mm2, mm, "moving_mean"), (mv2, mv, "moving_var"), (mo, out["mean"], "mean"), (io, out["invstd"], "invstd")):
        assert torch.equal(a, b), "M %d: pnp_bn_apply_fused and pnp_bn_finalize disagree on %s" % (M, n)


@pytest.mark.parametrize("P", SEG_P)
@pytest.mark.parametrize("C", [2, 5, 8])
def test_segloss_real(C, P):
    """randn logits, one-hot y: the four class sums, then _finalize from the kernel's own acc, then _bwd from the kernel's own
    coef, each within TAU of the fp64 value"""
    _C, rt = lib()
    g0 = torch.Generator().manual_seed(C * 7 + P)
    logits = (torch.randn(P, C, generator=g0) * 3).to(DEV)
    y = torch.nn.functional.one_hot(torch.randint(0, C, (P,), generator=g0), C).float().to(DEV)
    acc = torch.zeros(4 * C, dtype=torch.float64, device=DEV)
    _C.call("pnp_segloss_reduce", ptr(logits), ptr(y), P, C, ptr(acc), rt.stream())
    out, coef = torch.empty(2, device=DEV), torch.empty(3 * C, device=DEV)
    _C.call("pnp_segloss_finalize", ptr(acc), P, C, ptr(out), ptr(coef), rt.stream())
    gw, gd = torch.tensor([0.7], device=DEV), torch.tensor([-1.3], device=DEV)
    dl = torch.empty(P, C, device=DEV)
    _C.call("pnp_segloss_bwd", ptr(logits), ptr(y), ptr(coef), ptr(gw), ptr(gd), ptr(dl), P, C, rt.stream())
    sync()
    ref, mag = E.segloss_reduce_ref(logits, y)
    tag = "C %d P %d" % (C, P)
    check("seg_sums", tag + " sums", acc[:3 * C], ref[:3 * C], mag[:3 * C])
    check("seg_ce", tag + " ce", acc[3 * C:], ref[3 * C:], mag[3 * C:])
    o_ref, o_mag, c_ref = E.segloss_finalize_ref(acc, P, C)
    check("seg_finalize", tag + " out", out, o_ref, o_mag)
    check("seg_finalize", tag + " coef", coef, c_ref, c_ref.abs())
    d_ref, d_mag = E.segloss_bwd_ref(logits, y, coef, 0.7, -1.3)
    check("seg_bwd", tag + " dlogits", dl, d_ref, d_mag)


def invstd_sweep_variances(n=1 << 20, seed=0):
    """fp32 variances: 0, subnormals, the neighbourhood of eps (including the values that land on eps - var), 1e-30 .. 1e30"""
    g0 = torch.Generator().manual_seed(seed)
    parts = [torch.zeros(16)]
    sub = torch.randint(1, 1 << 23, (4096,), generator=g0, dtype=torch.int32)
    parts.append(sub.view(torch.float32))
    e = torch.tensor(E.BN_EPS, dtype=torch.float32).view(torch.int32)
    near = e + torch.arange(-(1 << 17), 1 << 17, dtype=torch.int32)
    parts.append(near.view(torch.float32))
    rest = n - sum(p.numel() for p in parts)
    parts.append(torch.pow(10.0, torch.rand(rest, generator=g0, dtype=torch.float64) * 60 - 30).float())
    return torch.cat(parts)


def test_bn_finalize_invstd_ulps():
    """invstd = rsqrtf + one Newton step against the correctly rounded 1 / sqrt(fl(var + eps)), over 2^20 variances"""
    _C, rt = lib()
    var = invstd_sweep_variances().to(DEV)
    C = var.numel()
    zero, one = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
    outs = [torch.empty(C, device=DEV) for _ in range(4)]
    mv = var.clone()
    _C.call("pnp_bn_finalize", None, None, 1, C, ptr(one), ptr(zero), ptr(zero), ptr(mv), 0, *[ptr(o) for o in outs], rt.stream())
    sync()
    got, ref = outs[3].cpu(), E.rsqrt_f32_ref(var.cpu())
    ulps = E.f32_ulp_distance(got, ref)
    hist = torch.bincount(ulps.clamp_max(8))
    print("  invstd ulps over %d variances: max %d, histogram %s (bound %d)" % (C, int(ulps.max()), hist.tolist(), E.INVSTD_ULP))
    assert int(ulps.max()) <= E.INVSTD_ULP
    assert torch.equal(outs[0].cpu(), got), "scale != gamma * invstd at gamma = 1"


# ------------------------------------------------------------------------------------------------
# c. the two suspects
# ------------------------------------------------------------------------------------------------
SIGN_VALUES = [0.0, -0.0, 2.0 ** -149, -2.0 ** -149, 2.0 ** -134, -2.0 ** -134, 2.0 ** -133, -2.0 ** -133, 2.0 ** -126, -2.0 ** -126]


def _slopes(_C, rt, y, yhi, act):
    """act'(y) per element as pnp_bn_bwd_apply_direct (dy = 1, frozen BN with gamma = invstd = 1) and pnp_bn_bwd_reduce_sums
    (one launch per row, dy = 1) read it, with the sign from y or from yhi"""
    M, C = y.shape
    ones, zc = torch.ones(M, C, device=DEV), torch.zeros(C, device=DEV)
    onec = torch.ones(C, device=DEV)
    res = {}
    for src, yy, hh in (("y", y, None), ("y_hi", None, yhi)):
        dz = torch.empty(M, C, device=DEV)
        _C.call("pnp_bn_bwd_apply_direct", ptr(ones), ptr(yy), ptr(hh), act, None, None, ptr(onec), ptr(onec), None, None, M, C, 0, None,
                None, None, ptr(dz), None, None, rt.stream())
        sums = torch.zeros(M, C, dtype=torch.float64, device=DEV)
        sgx = torch.zeros(C, dtype=torch.float64, device=DEV)
        for m in range(M):
            _C.call("pnp_bn_bwd_reduce_sums", ptr(ones[m]), ptr(yy[m]) if yy is not None else None, ptr(hh[m]) if hh is not None else None,
                    ptr(zc), ptr(zc), ptr(onec), act, ptr(sums[m]), ptr(sgx), 1, C, rt.stream())
        sync()
        res[src] = (dz, sums.float())
    return res


def test_subnormal_activation_sign():
    """rn_bf16 sends 0 < y <= 2^-134 to a bf16 +0, so a consumer reading the sign from y_hi would take the y <= 0 slope there.
    The producers (pnp_bn_act_apply, pnp_bn_apply_fused, the wgmma fused epilogue) flush positive subnormal activations to
    +0, so the y and y_hi paths agree on everything they write."""
    _C, rt = lib()
    vals = torch.tensor(SIGN_VALUES, dtype=torch.float32)
    z = vals.repeat_interleave(4).reshape(-1, 4).to(DEV)
    M, C = z.shape
    pos_tiny = (z > 0) & (z <= 2.0 ** -134)
    for act in (E.RELU, E.LRELU):
        # the consumers fed such a y directly disagree: this is why the producers flush
        s = _slopes(_C, rt, z, S.split(z.cpu())[0].to(DEV), act)
        assert bool((s["y"][0][pos_tiny] == 1).all()) and bool((s["y_hi"][0][pos_tiny] != 1).all())
        assert torch.equal(s["y"][0][~pos_tiny], s["y_hi"][0][~pos_tiny])
        # the references on the host, where no denormal is flushed; fmaf(z, 1, 0) turns -0 into +0
        want_z = E.act_fwd(z.cpu(), act)
        want_fma = E.act_fwd(z.cpu() + 0.0, act)
        assert bool((want_z[(z.cpu() > 0) & (z.cpu() < 2.0 ** -126)] == 0).all())
        # pnp_bn_act_apply and pnp_bn_apply_fused (frozen: mean 0, invstd 1, gamma 1, beta 0)
        mv = torch.full((C,), var_for_invstd(1.0), device=DEV)
        zero, one, mm = torch.zeros(C, device=DEV), torch.ones(C, device=DEV), torch.zeros(C, device=DEV)
        for name in ("pnp_bn_act_apply", "pnp_bn_apply_fused"):
            y = torch.empty(M, C, device=DEV)
            hi, lo = empty_planes((M, C), 3)
            if name == "pnp_bn_act_apply":
                want = want_z
                _C.call(name, ptr(z), None, None, None, 0, 0, act, ptr(y), ptr(hi), ptr(lo), M, C, rt.stream())
            else:
                want = want_fma
                _C.call(name, ptr(z), None, None, M, C, ptr(one), ptr(zero), ptr(mm), ptr(mv), 0, None, 0, 0, act, ptr(y), ptr(hi),
                        ptr(lo), None, None, rt.stream())
            sync()
            y = y.cpu()
            assert torch.equal(y.view(torch.int32), want.view(torch.int32)), "%s act %d: %s" % (name, act, y.cpu().tolist())
            assert_planes(name, hi, lo, want)
            s = _slopes(_C, rt, y.to(DEV), hi, act)
            for k in (0, 1):
                assert torch.equal(s["y"][k], s["y_hi"][k]), "%s act %d: the y and y_hi paths disagree" % (name, act)
        _tc_epilogue_sign(_C, rt, vals, act)


def _tc_epilogue_sign(_C, rt, vals, act):
    """the wgmma fused epilogue: zero operands, shift = the edge values per channel, so y = act(shift)"""
    lib(require_tc=True)
    B, H, W, Cin, Cout = 1, 8, 8, 64, 64
    x_hi = torch.zeros(B * H * W * Cin, dtype=torch.bfloat16, device=DEV)
    w_hi = torch.zeros(Cin * Cout, dtype=torch.bfloat16, device=DEV)
    shift = torch.ones(Cout)
    shift[:vals.numel()] = vals
    shift = shift.to(DEV)
    scale = torch.ones(Cout, device=DEV)
    y = torch.empty(B * H * W, Cout, device=DEV)
    hi = torch.empty(B * H * W, Cout, dtype=torch.bfloat16, device=DEV)
    ep = _C.TcEpilogue(ptr(scale), ptr(shift), None, 0, 0, act, ptr(hi), None)
    geom = _C.ConvGeom(B, H, W, Cin, H, W, Cout, 1, 1, 1, 1, 0, 0)
    _C.call("pnp_conv2d_tc_fwd_fused", ptr(x_hi), None, ptr(w_hi), None, ptr(y), ctypes.byref(geom), 1, None, 0, None, None,
            ctypes.byref(ep), rt.stream())
    sync()
    want = E.act_fwd(shift.cpu() + 0.0, act).expand(B * H * W, Cout).contiguous()     # fmaf(+0, 1, -0) = +0
    assert torch.equal(y.cpu().view(torch.int32), want.view(torch.int32)), "wgmma epilogue act %d: %s" % (act, y[0].tolist())
    assert S.planes_equal(hi.cpu(), S.split(want)[0]), "wgmma epilogue act %d: hi plane" % act


VAR_CASES = [(M, r) for M in (4, 32, 8192) for r in (0, 1, 10, 100)]


def test_bn_variance_conditioning():
    """pnp_bn_stats + pnp_bn_finalize on z = r + N(0, 1): |var - var_ref| <= TAU * E[z^2] (one-pass variance); prints the
    relative error of invstd, which grows as (mean / std)^2"""
    _C, rt = lib()
    C = 64
    rows = []
    for M, r in VAR_CASES:
        g0 = torch.Generator().manual_seed(M + r)
        z = (torch.randn(M, C, generator=g0) + r).to(DEV)
        s1 = torch.zeros(C, dtype=torch.float64, device=DEV)
        s2 = torch.zeros_like(s1)
        _C.call("pnp_bn_stats", ptr(z), M, C, ptr(s1), ptr(s2), rt.stream())
        one, zero = torch.ones(C, device=DEV), torch.zeros(C, device=DEV)
        mm, mv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
        outs = [torch.empty(C, device=DEV) for _ in range(4)]
        _C.call("pnp_bn_finalize", ptr(s1), ptr(s2), M, C, ptr(one), ptr(zero), ptr(mm), ptr(mv), 1,
                *[ptr(o) for o in outs], rt.stream())
        sync()
        mean_ref, var_ref, e2 = E.bn_moments(z)
        var_k = (s2 / M - (s1 / M) ** 2).clamp_min(0)
        inv_ref = 1.0 / torch.sqrt(var_ref + E.BN_EPS)
        rel_inv = float(((outs[3].double() - inv_ref).abs() / inv_ref).max())
        check("bn_var", "M %d mean/std %d" % (M, r), var_k, var_ref, e2)
        rows.append((M, r, float(((var_k - var_ref).abs() / e2).max()), float(((var_k - var_ref).abs() / var_ref).max()), rel_inv))
    print("  %6s %8s %14s %14s %14s" % ("M", "mean/std", "|dvar|/E[z^2]", "|dvar|/var", "|dinvstd|/invstd"))
    for row in rows:
        print("  %6d %8d %14.3e %14.3e %14.3e" % row)


# ------------------------------------------------------------------------------------------------
# d. rejected calls
# ------------------------------------------------------------------------------------------------
def _rejections():
    """(tag, launcher, argument builder, expected code); the builder gets a dict of sentinel-filled buffers"""
    R = []

    def stats(C):
        return lambda b: ("pnp_bn_stats", (ptr(b["z"]), 8, C, ptr(b["s1"]), ptr(b["s2"]), None))

    def reduce_(C, act=0, y=True):
        return lambda b: ("pnp_bn_bwd_reduce", (ptr(b["dy"]), ptr(b["y"]) if y else None, ptr(b["z"]), ptr(b["c"]), ptr(b["c"]), act,
                                                ptr(b["out"]), ptr(b["s1"]), ptr(b["s2"]), 8, C, None))

    def sums(C, act=0, y=True):
        return lambda b: ("pnp_bn_bwd_reduce_sums", (ptr(b["dy"]), ptr(b["y"]) if y else None, None, ptr(b["z"]), ptr(b["c"]),
                                                     ptr(b["c"]), act, ptr(b["s1"]), ptr(b["s2"]), 8, C, None))

    def act_apply(C, scale=True, shift=True, skip=None):
        Cs, off = skip if skip else (0, 0)
        return lambda b: ("pnp_bn_act_apply", (ptr(b["z"]), ptr(b["c"]) if scale else None, ptr(b["c"]) if shift else None,
                                               ptr(b["skip"]) if skip else None, Cs, off, 0, ptr(b["out"]), None, None, 8, C, None))

    def fused(C, y=True, mo=True, io=True, skip=None):
        Cs, off = skip if skip else (0, 0)
        return lambda b: ("pnp_bn_apply_fused", (ptr(b["z"]), ptr(b["s1c"]), ptr(b["s2c"]), 8, C, ptr(b["c"]), ptr(b["c"]), ptr(b["mm"]),
                                                 ptr(b["mv"]), 1, ptr(b["skip"]) if skip else None, Cs, off, 0,
                                                 ptr(b["out"]) if y else None, None, None, ptr(b["mo"]) if mo else None,
                                                 ptr(b["io"]) if io else None, None))

    def bwd_apply(C):
        return lambda b: ("pnp_bn_bwd_apply", (ptr(b["dy"]), ptr(b["z"]), ptr(b["c"]), ptr(b["c"]), ptr(b["c"]), ptr(b["c"]), 1, None,
                                               ptr(b["out"]), None, None, 8, C, None))

    def bwd_fused(C):
        return lambda b: ("pnp_bn_bwd_apply_fused", (ptr(b["dy"]), ptr(b["z"]), ptr(b["c"]), ptr(b["c"]), ptr(b["c"]), ptr(b["s1c"]),
                                                     ptr(b["s2c"]), 8, C, 1, None, ptr(b["mo"]), ptr(b["io"]), ptr(b["out"]), None, None,
                                                     None))

    def direct(C, act=0, y=True):
        return lambda b: ("pnp_bn_bwd_apply_direct", (ptr(b["dy"]), ptr(b["y"]) if y else None, None, act, ptr(b["z"]), ptr(b["c"]),
                                                      ptr(b["c"]), ptr(b["c"]), ptr(b["s1c"]), ptr(b["s2c"]), 8, C, 1, None, ptr(b["mo"]),
                                                      ptr(b["io"]), ptr(b["out"]), None, None, None))

    for C in (6, 1028):
        R += [("stats C%d" % C, stats(C), UNSUPPORTED), ("reduce C%d" % C, reduce_(C), UNSUPPORTED),
              ("reduce_sums C%d" % C, sums(C), UNSUPPORTED), ("apply_fused C%d" % C, fused(C), UNSUPPORTED),
              ("bwd_apply_fused C%d" % C, bwd_fused(C), UNSUPPORTED), ("direct C%d" % C, direct(C), UNSUPPORTED)]
    R += [("act_apply C6", act_apply(6), UNSUPPORTED), ("bwd_apply C6", bwd_apply(6), UNSUPPORTED),
          ("act_apply skip_off 2", act_apply(16, skip=(4, 2)), UNSUPPORTED), ("act_apply Cs 6", act_apply(16, skip=(6, 0)), UNSUPPORTED),
          ("act_apply skip past C", act_apply(16, skip=(8, 12)), UNSUPPORTED),
          ("apply_fused skip_off 2", fused(16, skip=(4, 2)), UNSUPPORTED), ("apply_fused Cs 6", fused(16, skip=(6, 0)), UNSUPPORTED),
          ("act_apply scale without shift", act_apply(16, shift=False), BAD_ARG),
          ("act_apply shift without scale", act_apply(16, scale=False), BAD_ARG),
          ("apply_fused mean_out without invstd_out", fused(16, io=False), BAD_ARG),
          ("apply_fused invstd_out without mean_out", fused(16, mo=False), BAD_ARG),
          ("apply_fused neither y nor y_hi", fused(16, y=False), BAD_ARG)]
    for act in (E.RELU, E.LRELU):
        R += [("reduce act %d no y" % act, reduce_(16, act, y=False), BAD_ARG), ("reduce_sums act %d no y" % act, sums(16, act, y=False), BAD_ARG),
              ("direct act %d no y" % act, direct(16, act, y=False), BAD_ARG)]
    return R


REJECT = _rejections()


@pytest.mark.parametrize("i", range(len(REJECT)), ids=[r[0].replace(" ", "_") for r in REJECT])
def test_rejected_calls_leave_outputs_untouched(i):
    _C, rt = lib()
    tag, build, code = REJECT[i]
    n = 8 * 1028
    b = {k: torch.full((n,), 1234.5, device=DEV) for k in ("z", "dy", "y", "c", "skip", "out", "mm", "mv", "mo", "io")}
    b.update({k: torch.full((n,), 1234.5, dtype=torch.float64, device=DEV) for k in ("s1", "s2", "s1c", "s2c")})
    before = snapshot(b)
    name, args = build(b)
    args = args[:-1] + (rt.stream(),)
    rc = getattr(_C.lib, name)(*args)
    sync()
    assert rc == code, "%s: %s returned %d, expected %d" % (tag, name, rc, code)
    assert_untouched(tag, name, b, before)


# ------------------------------------------------------------------------------------------------
# e. programmatic dependent launch
# ------------------------------------------------------------------------------------------------
@pytest.mark.timeout(300)
def test_exact_cases_under_pdl():
    passed, _ = rerun({"PNP_PDL": "1"}, __file__, "(bn_stats_exact or bwd_reduce_exact or act_apply_exact or apply_fused_exact or "
                      "bwd_apply_exact) and not under_pdl", flags=("-s",))
    assert passed == 2 * len(REDUCE_CASES) + 3 * len(APPLY_SHAPES) + 6 * len(BWD_SHAPES), passed
