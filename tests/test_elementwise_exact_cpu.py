"""The elementwise checks of tests/test_elementwise_exact_gpu.py without a GPU: its case tables reach every launch regime of the
restated configuration, the fp64 references are the oracle's batch norm, losses and their autograd gradients, and each
exactness check and TAU rejects the reference of each plausible kernel bug at the GPU file's shapes."""
import pytest
import torch

from oracle import elementwise_exact as E
from oracle import tf14_torch as T
from tests.cabi import ints, pick
from tests.test_elementwise_exact_gpu import (APPLY_SHAPES, BIG, BWD_SHAPES, REDUCE_CASES, SEG_P, VAR_CASES,
                                              invstd_sweep_variances, var_for_invstd)

REGIMES = {"tpr%d" % (1 << i) for i in range(9)} | {"idle_lanes", "ragged", "odd_rows", "m_lt_rstep", "capped", "promoted"}


# ------------------------------------------------------------------------------------------------
# launch configuration and case tables
# ------------------------------------------------------------------------------------------------
def test_reduce_cases_reach_every_regime():
    reached = set()
    for tag, M, C in REDUCE_CASES:
        reached |= E.reduce_regimes(M, C)
    assert REGIMES <= reached, sorted(REGIMES - reached)
    idle = {C for _, M, C in REDUCE_CASES if "idle_lanes" in E.reduce_regimes(M, C)}
    assert {12, 40, 320, 520} <= idle
    assert {M for _, M, C in REDUCE_CASES if M < E.reduce_launch_cfg(M, C).rstep} >= {1, 4}
    cap = [(M, C) for t, M, C in REDUCE_CASES if t == "capped_16ch_B16"]
    assert cap == [(16 * 256 * 256, 16)] and "capped" in E.reduce_regimes(*cap[0])
    prom = [t for t, M, C in REDUCE_CASES if "promoted" in E.reduce_regimes(M, C)]
    assert prom and set(prom) <= BIG


def test_launch_cfg_known_answers():
    """hand-derived: 8 rows per row lane; above 1056 CTAs (8 per SM on 132 SMs) the rows per CTA grow instead"""
    assert E.reduce_launch_cfg(3001, 1024) == E.ReduceCfg(256, 1, 8, 376, False, 8)
    assert E.reduce_launch_cfg(3001, 4) == E.ReduceCfg(1, 256, 2048, 2, False, 8)
    assert E.reduce_launch_cfg(777, 520) == E.ReduceCfg(256, 1, 8, 98, False, 8)        # 130 quads on 256 lanes
    assert E.reduce_launch_cfg(1048576, 16) == E.ReduceCfg(4, 64, 993, 1056, True, 16)
    assert E.reduce_launch_cfg(70001, 1024) == E.ReduceCfg(256, 1, 67, 1045, True, 67)
    assert E.reduce_launch_cfg(1, 4) == E.ReduceCfg(1, 256, 2048, 1, False, 1)
    for M, C in ((8, 6), (8, 1028), (0, 16), (8, 0)):
        assert E.reduce_launch_cfg(M, C) is None
    assert E.grid_for(1, 256) == 1 and E.grid_for(257, 256) == 2 and E.grid_for(10 ** 9, 256) == 132 * 64


def test_apply_shapes_reach_shared_memory_extremes_and_grid_stride():
    Cs = {C for _, _, C in APPLY_SHAPES}
    assert {4, 1024} <= Cs and {4, 1024} <= {C for _, _, C in BWD_SHAPES}
    strided = [(M, C) for _, M, C in APPLY_SHAPES if M * C // 4 > E.grid_for(M * C // 4, 256) * 256]
    assert strided and all(E.grid_for(M * C // 4, 256) == 132 * 64 for M, C in strided)
    assert [(M, C) for _, M, C in BWD_SHAPES if M * C // 4 > E.grid_for(M * C // 4, 256) * 256]


def test_exact_operand_preconditions():
    """the operand choices of the exact cases are exact: fl(0.2f * 5k) = k, the chosen variances give invstd 1 and 2, the
    fp32 row partials of the reductions stay integers"""
    k = torch.arange(-8, 9, dtype=torch.float32)
    assert torch.equal((5 * k) * torch.tensor(0.2, dtype=torch.float32), k)
    eps = torch.tensor(E.BN_EPS, dtype=torch.float32)
    for inv in (1.0, 2.0):
        v = torch.tensor(var_for_invstd(inv), dtype=torch.float32)
        assert float(v + eps) == 1.0 / inv ** 2
        assert float(E.rsqrt_f32_ref(v)) == inv
    assert E.PROMOTE_ROWS * 40 * 10 < E.F32_EXACT / 2


def test_invstd_sweep_covers_the_ranges():
    v = invstd_sweep_variances()
    assert v.numel() == 1 << 20 and bool((v >= 0).all()) and bool(torch.isfinite(v).all())
    assert bool((v == 0).any()) and int(((v > 0) & (v < 2.0 ** -126)).sum()) >= 4000
    assert float(v.max()) > 1e29 and int(((v - 1e-3).abs() < 1e-6).sum()) > 1000


# ------------------------------------------------------------------------------------------------
# the references against the oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", [E.NONE, E.RELU, E.LRELU])
@pytest.mark.parametrize("M", [1, 7, 300])
def test_bn_references_match_oracle_and_autograd(M, act):
    """forward (y, moving statistics) against tf14_torch.batch_norm; the backward chain act' -> reduce -> finalize -> apply
    against autograd of act(batch_norm(z)), including dgamma / dbeta"""
    C = 12
    gen = torch.Generator().manual_seed(M * 3 + act)
    z = torch.randn(M, C, generator=gen, dtype=torch.float64) * 2 + 0.3
    bn = T.BNState(C, dtype=torch.float64)
    with torch.no_grad():
        bn.gamma.copy_(1 + 0.3 * torch.randn(C, generator=gen, dtype=torch.float64))
        bn.beta.copy_(0.2 * torch.randn(C, generator=gen, dtype=torch.float64))
    mm0, mv0 = 0.1 * torch.randn(C, generator=gen, dtype=torch.float64), 1 + torch.rand(C, generator=gen, dtype=torch.float64)
    bn.moving_mean, bn.moving_var = mm0.clone(), mv0.clone()
    zz = z.clone().requires_grad_(True)
    pre = T.batch_norm(zz, bn, True)
    y_t = pre if act == E.NONE else torch.nn.functional.leaky_relu(pre, 0.2 if act == E.LRELU else 0.0)
    s1, s2, sa = E.bn_stats_ref(z)
    ref = E.bn_finalize_ref(s1, s2, M, bn.gamma.detach(), bn.beta.detach(), mm0, mv0, 1, s_abs=sa)
    assert torch.allclose(ref["moving_mean"][0], bn.moving_mean, rtol=1e-12, atol=1e-12)
    assert torch.allclose(ref["moving_var"][0], bn.moving_var, rtol=1e-12, atol=1e-12)
    pre_ref = z * ref["scale"][0] + ref["shift"][0]
    assert torch.allclose(pre_ref, pre.detach(), rtol=1e-10, atol=1e-10)
    y_e, _ = E.bn_apply_ref(z, ref["scale"][0], ref["shift"][0], act=act)
    assert torch.allclose(y_e.double(), y_t.detach(), rtol=1e-6, atol=1e-6)
    dy = torch.randn(M, C, generator=gen, dtype=torch.float64)
    y_t.backward(dy)
    # g = dy * act'(y) is fp32 in the kernels (and 0.2f the fp32 slope): compare at a few fp32 ulps of the largest gradient
    g, sg, sgx, _, _ = E.bn_bwd_reduce_ref(dy, pre.detach(), z, ref["mean"][0], ref["invstd"][0], act)
    coef = E.bn_bwd_finalize_ref(sg, sgx, M)
    dz, _ = E.bn_bwd_apply_ref(g, z, ref["mean"][0], ref["invstd"][0], bn.gamma.detach(), coef[:C], coef[C:], 1)
    for got, want in ((dz, zz.grad), (sgx, bn.gamma.grad), (sg, bn.beta.grad)):
        assert float((got.double() - want).abs().max()) <= 1e-6 * float(want.abs().max()) + 1e-9


def test_bn_bwd_apply_ref_matches_the_formula():
    gen = torch.Generator().manual_seed(4)
    M, C = 50, 8
    z, g = torch.randn(M, C, generator=gen), torch.randn(M, C, generator=gen)
    mean, inv, gamma = torch.randn(C, generator=gen), torch.rand(C, generator=gen) + 0.5, torch.randn(C, generator=gen)
    c1, c2 = torch.randn(C, generator=gen), torch.randn(C, generator=gen)
    dz, mag = E.bn_bwd_apply_ref(g, z, mean, inv, gamma, c1, c2, 1)
    d = lambda t: t.double()  # noqa: E731
    want = d(gamma) * d(inv) * (d(g) - d(c1) - (d(z) - d(mean)) * d(inv) * d(c2))
    assert torch.equal(dz, want.float()) and bool((mag >= want.abs() - 1e-12).all())
    dz0, _ = E.bn_bwd_apply_ref(g, z, mean, inv, gamma, c1, c2, 0)
    assert torch.equal(dz0, (d(gamma) * d(inv) * d(g)).float())


@pytest.mark.parametrize("C", [2, 5, 8])
def test_segloss_references_match_oracle_and_autograd(C):
    gen = torch.Generator().manual_seed(C)
    P = 2 * 9 * 7
    logits = torch.randn(2, 9, 7, C, generator=gen, dtype=torch.float64) * 3
    y = torch.nn.functional.one_hot(torch.randint(0, C, (2, 9, 7), generator=gen), C).double()
    acc, mag = E.segloss_reduce_ref(logits.reshape(P, C), y.reshape(P, C))
    out, _, coef = E.segloss_finalize_ref(acc, P, C)
    lg = logits.clone().requires_grad_(True)
    wce, dice = T.softmax_weighted_loss(lg, y), T.dice_loss(lg, y)
    assert abs(float(out[0]) - float(wce.detach())) < 1e-12 and abs(float(out[1]) - float(dice.detach())) < 1e-12
    gw, gd = 0.7, -1.3
    (gw * wce + gd * dice).backward()
    dl, dmag = E.segloss_bwd_ref(logits.reshape(P, C), y.reshape(P, C), coef, gw, gd)
    assert torch.allclose(dl, lg.grad.reshape(P, C), rtol=1e-9, atol=1e-12)
    assert bool((dmag >= dl.abs() - 1e-15).all()) and bool((mag >= acc.abs() - 1e-12).all())


def test_metric_references():
    logits = torch.tensor([[1.0, 3.0, 3.0], [2.0, 2.0, 0.0], [0.0, 0.0, 0.0]])
    y = torch.tensor([[0.0, 1.0, 1.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    assert E.confusion_ref(logits, y).tolist() == [1, 0, 0, 0, 1, 0, 1, 0, 0]     # ties: first maximum
    assert float(E.l2_ref(torch.tensor([3.0, -4.0]))) == float(T.l2_loss(torch.tensor([3.0, -4.0]).double()))
    x, w, dout = torch.randn(3, 5), torch.randn(5), torch.randn(3)
    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
    out = xr @ wr
    out.backward(dout.double())
    dx, dw = E.fc_bwd_ref(x, w, dout)
    assert torch.allclose(E.fc_fwd_ref(x, w), out.detach()) and torch.allclose(dx, xr.grad) and torch.allclose(dw, wr.grad)
    a, b = torch.arange(6.0), torch.ones(6)
    assert float(E.mean_combo_ref(a, 0.5, b, -2.0)) == 0.5 * 2.5 - 2.0 and float(E.mean_combo_ref(a, 1.0, None, 0.0)) == 2.5


def test_act_fwd_flushes_positive_subnormals():
    v = torch.tensor([2.0 ** -149, 2.0 ** -134, 2.0 ** -127, 2.0 ** -126, -2.0 ** -149, -1.0, 0.0, -0.0])
    assert E.act_fwd(v, E.RELU).tolist() == [0.0, 0.0, 0.0, 2.0 ** -126, 0.0, 0.0, 0.0, 0.0]
    lr = E.act_fwd(v, E.LRELU)
    assert lr[:4].tolist() == [0.0, 0.0, 0.0, 2.0 ** -126] and float(lr[5]) == float(torch.tensor(-1.0) * torch.tensor(0.2))
    # after the flush, the sign of every written y survives the bf16 hi plane
    from oracle import bf16_split as S
    for act in (E.RELU, E.LRELU):
        y = E.act_fwd(v, act)
        assert torch.equal(y > 0, S.split(y)[0].float() > 0)


# ------------------------------------------------------------------------------------------------
# negative controls at the GPU file's shapes
# ------------------------------------------------------------------------------------------------
def _tau(key):
    tau = E.TAU[key]
    assert tau is not None
    return tau


def _reject(key, tag, bug, ref, mag, fp32_out=True):
    """TAU[key] rejects the bug's reference; for an fp32 output, the fp32 rounding of the right answer passes"""
    tau = _tau(key)
    n = E.violations(bug, ref, mag, tau)
    print("  %-12s %-40s %6d of %7d rejected, worst ratio %.2e vs tau %.2e" % (key, tag, n, ref.numel(), E.worst_ratio(bug, ref, mag), tau))
    if fp32_out:
        assert E.violations(ref.float().double(), ref, mag, tau) == 0
    assert n > 0, "%s: tau %.2e cannot see this bug" % (tag, tau)


def _boundary_row(M, C):
    cfg = E.reduce_launch_cfg(M, C)
    return cfg.rpb if cfg.grid > 1 else M - 1          # the first row of CTA 1, or the last row of the only CTA


def _small_reduce_cases():
    return [c for c in REDUCE_CASES if c[0] not in BIG or c[0] == "capped_16ch_B16"]


@pytest.mark.parametrize("mode", ["dropped", "doubled"])
def test_exact_stats_reject_a_row_at_a_cta_boundary(mode):
    """a row left out of (or counted twice in) the BN sums at a CTA boundary changes an exact integer sum"""
    for tag, M, C in _small_reduce_cases():
        gen = torch.Generator().manual_seed(M + C)
        z = ints((M, C), -8, 8, gen).double()
        r = _boundary_row(M, C)
        s1, s2, _ = E.bn_stats_ref(z)
        row = z[r]
        sign = -1 if mode == "dropped" else 1
        assert not (torch.equal(s1 + sign * row, s1) and torch.equal(s2 + sign * row * row, s2)), tag
        # the same row in the g-sums of the backward reduce
        gen = torch.Generator().manual_seed(7 + M + C)
        dy = ints((M, C), -8, 8, gen, 5.0).double()
        g, sg, _, _, _ = E.bn_bwd_reduce_ref(dy, dy, z, torch.zeros(C), torch.ones(C), E.NONE)
        assert not torch.equal(sg + sign * g[r].double(), sg), tag


@pytest.mark.parametrize("mode", ["dropped", "doubled"])
def test_tau_var_rejects_a_row_at_a_cta_boundary(mode):
    """the same bug in the real-valued variance check at the conditioning shapes.  At M = 8192 and mean/std = 100 one row moves
    the variance by about 1e-8 E[z^2], below what the one-pass variance itself resolves: there the exact integer sums of
    test_exact_stats_reject_a_row_at_a_cta_boundary are the guard"""
    C = 64
    for M, r in VAR_CASES:
        if M == 8192 and r == 100:
            continue
        g0 = torch.Generator().manual_seed(M + r)
        z = (torch.randn(M, C, generator=g0) + r).double()
        _, var_ref, e2 = E.bn_moments(z)
        row = _boundary_row(M, C)
        w = torch.ones(M, 1, dtype=torch.float64)
        w[row] = 0.0 if mode == "dropped" else 2.0
        n = M - 1 if mode == "dropped" else M + 1
        mb = (z * w).sum(0) / n
        var_bug = (z * z * w).sum(0) / n - mb * mb
        _reject("bn_var", "M %d mean/std %d %s row %d" % (M, r, mode, row), var_bug, var_ref, e2, fp32_out=False)


def test_tau_finalize_rejects_the_biased_moving_variance():
    C = 64
    for M in (4, 32, 3001, 8192):
        g0 = torch.Generator().manual_seed(M)
        f = lambda *s: torch.randn(*s, generator=g0)  # noqa: E731
        z = f(M, C) * 2 + 0.3
        gamma, beta, mm0 = 1 + 0.3 * f(C), 0.2 * f(C), 0.1 * f(C)
        mv0 = 1 + 0.2 * torch.rand(C, generator=g0)
        s1, s2, sa = E.bn_stats_ref(z)
        ref = E.bn_finalize_ref(s1, s2, M, gamma, beta, mm0, mv0, 1, s_abs=sa)
        bug = E.bn_finalize_ref(s1, s2, M, gamma, beta, mm0, mv0, 1, s_abs=sa, unbiased=False)
        _reject("bn_finalize", "M %d biased moving_var" % M, bug["moving_var"][0], *ref["moving_var"])


@pytest.mark.parametrize("act", [E.RELU, E.LRELU])
def test_exact_reduce_rejects_slope_one_at_zero(act):
    for tag, M, C in _small_reduce_cases():
        gen = torch.Generator().manual_seed(M + C)
        z, mean = ints((M, C), -8, 8, gen).double(), ints((C,), -2, 2, gen).double()
        dy, y = ints((M, C), -8, 8, gen, 5.0).double(), ints((M, C), -3, 3, gen).double()
        if not bool(((y == 0) & (dy != 0)).any()):
            continue                                           # M = 1: the row may hold no zero y
        good = E.bn_bwd_reduce_ref(dy, y, z, mean, torch.ones(C), act)
        bug = E.bn_bwd_reduce_ref(dy, y, z, mean, torch.ones(C), act, slope_at_zero=1.0)
        assert not torch.equal(good[0], bug[0]), tag


def _bwd_operands_cpu(M, C, seed, keep=None):
    gen = torch.Generator().manual_seed(seed)
    z, mean = ints((M, C), -8, 8, gen).double(), ints((C,), -2, 2, gen).double()
    invstd = pick((C,), [1.0, 0.5], gen).double()
    invstd[0] = 0.5
    dy = ints((M, C), -8, 8, gen, 5.0).double()
    gamma = pick((C,), [0.5, 1.0, 1.5, 2.0], gen).double()
    c1, c2 = ints((C,), -8, 8, gen, 0.25).double(), ints((C,), -8, 8, gen, 0.25).double()
    c2[0] = 1.0
    mask = None if keep is None else (torch.rand(M, C, generator=gen) < keep).float() / keep
    return z, mean, invstd, dy, gamma, c1, c2, mask


def test_exact_bwd_apply_rejects_c2_without_invstd_and_a_missing_dropout():
    for tag, M, C in BWD_SHAPES:
        z, mean, invstd, dy, gamma, c1, c2, mask = _bwd_operands_cpu(M, C, M + C, keep=0.5)
        good, _ = E.bn_bwd_apply_ref(dy, z, mean, invstd, gamma, c1, c2, 1, mask)
        bug, _ = E.bn_bwd_apply_ref(dy, z, mean, invstd, gamma, c1, c2, 1, mask, c2_invstd=False)
        if bool(((z - mean)[:, 0] != 0).any()):
            assert not torch.equal(good, bug), tag + ": c2 without invstd"
        nodrop, _ = E.bn_bwd_apply_ref(dy, z, mean, invstd, gamma, c1, c2, 1, None)
        if bool((mask == 0).any() & (nodrop != 0).any()):
            assert not torch.equal(good, nodrop), tag + ": missing dropout multiply"


@pytest.mark.parametrize("P", SEG_P)
@pytest.mark.parametrize("C", [2, 5, 8])
def test_seg_sums_reject_a_dropped_pixel(C, P):
    """one pixel left out of the class sums: exact for integer y (the exact-sum cases), beyond TAU for one-hot y at the
    real-valued shapes"""
    g0 = torch.Generator().manual_seed(C * 7 + P)
    logits = torch.randn(P, C, generator=g0) * 3
    y = torch.nn.functional.one_hot(torch.randint(0, C, (P,), generator=g0), C).float()
    ref, mag = E.segloss_reduce_ref(logits, y)
    for pix in (0, 256 * 8 - 1, P - 1):                       # the first pixel, the last of CTA 0, the last
        bug, _ = E.segloss_reduce_ref(logits, y, drop_pixel=pix)
        _reject("seg_sums", "C %d P %d pixel %d" % (C, P, pix), bug[:3 * C], ref[:3 * C], mag[:3 * C], fp32_out=False)


def test_tau_values_are_calibrated():
    """every TAU is set, and below the error of a bf16 or TF32 rounding (2^-14); the fp64 sums sit below one fp32 rounding"""
    for k, v in E.TAU.items():
        assert v is not None and 2.0 ** -30 < v < 2.0 ** -14, (k, v)
    assert 0 <= E.INVSTD_ULP <= 2
