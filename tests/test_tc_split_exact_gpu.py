"""The wgmma convolutions and every bf16 operand-plane producer against the split-aware fp64 reference (oracle/bf16_split.py).

a. every producer of (hi, lo) planes writes exactly split() of the fp32 value the same launch wrote (rounding mode, the lo of
   the right value, layout, zero padding), and planes-only launches write the same planes as launches that also write fp32;
b. fwd / dgrad / wgrad, nterms 1 and 3, on shapes that reach every instantiation and path, hold |got - ref| <= TAU * sum|a||b|
   per element, where ref is the fp64 value of exactly the products the kernel issues -- plus accumulate, dropout (the
   epilogue's index map at every element), the fused inference-BN / skip / activation epilogue and the fused or split-K BN sums;
c. the same check rejects a zeroed lo plane, an off-by-one pad and a dropped accumulate (its power, on valid memory only);
d. shapes the launchers cannot tile are declined with PNP_ERR_UNSUPPORTED and leave the output untouched;
e. the tile / order / launch-mode switches (read once per process) run the same checks in their own processes.

The C-ABI is called directly (_C.call / ptr / ConvGeom / TcEpilogue) on the runtime's stream; the fp64 references run on the
device too.  Each conv test prints its worst ratio |got - ref| / sum|a||b| next to TAU."""
import ctypes
import os

import pytest
import torch

from oracle import bf16_split as S
from tests.cabi import (DEV, assert_planes, drop_cfg, drop_mask, empty_planes, expected_ksplit, last_config, lib, rerun, same_pad,
                        sm_count, split_dev, split_w_dev)

pytestmark = pytest.mark.gpu
U32 = 2.0 ** -23      # one fp32 ulp, relative

# (id, B, H, W, Cin, Cout, k, stride, dil, padding, what it reaches; flags)
#   flags: wgrad = the weight gradient runs on the tensor cores; drop / bn / ep = the forward also runs with dropout / BN sums /
#   the fused epilogue.  Whether a launch splits K depends on the SM count: the split factor each launch chose is asserted
#   against expected_ksplit() for the device at hand.  On the 132 SMs of an H100 SXM, dil2, k5s4, 32x64, 128x64_4x4, 64_12x20,
#   32x32 and the wg_* cases split both the forward and the data gradient, 32x64_s2, 16x32_k5s4 and 64_7x9_s2 the forward only, so
#   accumulate runs on both paths of both launchers.
CASES = [
    ("g10_512x2560_sym", 2, 32, 32, 512, 2560, 3, 1, 1, "SYMMETRIC", {"wgrad", "drop", "ep"}),   # 20 n-tiles, dgrad K = 23040
    ("dil2_512_B5", 5, 16, 16, 512, 512, 3, 1, 2, "SAME", {"bn", "wgrad"}),  # split-K + BN sums
    ("k5s4_512_B3", 3, 16, 16, 512, 512, 5, 4, 1, "SAME", {"bn", "wgrad"}),  # 16-phase dgrad
    ("256x512_B8", 8, 32, 32, 256, 512, 3, 1, 1, "SAME", {"bn", "drop", "ep", "wgrad"}),           # persistent CTAs, n-tile change
    ("64_s2_256wide", 1, 256, 256, 64, 64, 3, 2, 1, "SAME", {"wgrad"}),                            # 256-wide strided TMA box
    ("32x64_s2", 2, 32, 32, 32, 64, 3, 2, 1, "SAME", {"wgrad"}),                                 # 32-channel phase dgrad
    ("16x32_k5s4", 8, 32, 32, 16, 32, 5, 4, 1, "SAME", set()),                                # N16 phase dgrad
    ("64x32", 1, 128, 128, 64, 32, 3, 1, 1, "SAME", {"ep"}),                                       # <32,*,64> tile
    ("32x64", 2, 32, 32, 32, 64, 3, 1, 1, "SAME", {"wgrad"}),                                # dgrad on <32,*,64>
    ("16x16_256wide", 1, 256, 256, 16, 16, 3, 1, 1, "SAME", {"ep"}),                               # 16-channel tiles, full width
    ("128x64_4x4_B9", 9, 4, 4, 128, 64, 3, 1, 1, "SAME", {"wgrad"}),                              # several images per tile, ragged
    ("64_7x9_s2", 1, 7, 9, 64, 64, 3, 2, 1, "SAME", set()),                                # odd grid, strided
    ("64_12x20", 3, 12, 20, 64, 64, 3, 1, 1, "SAME", set()),                                       # ragged tiles
    ("wg_cin192", 2, 16, 16, 192, 128, 3, 1, 1, "SAME", {"wgrad"}),                                # wgrad pack 1, half-OOB M tile
    ("wg_cin64", 2, 32, 32, 64, 128, 3, 1, 1, "SAME", {"wgrad"}),                                # wgrad pack 2
    ("wg_cin32_3x3", 2, 32, 32, 32, 64, 3, 1, 1, "SYMMETRIC", {"wgrad"}),                          # wgrad pack 4, dummy tap rows
    ("wg_cin32_5x5", 2, 32, 32, 32, 128, 5, 1, 1, "SAME", {"wgrad"}),                              # pack 4, 25 taps
    ("32x32", 2, 32, 32, 32, 32, 3, 1, 1, "SAME", set()),                                          # <32,*,32>: fwd and dgrad
]
CASE_IDS = [c[0] for c in CASES]


def geom_of(case):
    """-> oracle Geom (SYMMETRIC: H, W of the already mirror-padded input, VALID conv)"""
    _, B, H, W, Cin, Cout, k, s, d, pad, _ = case
    if pad == "SYMMETRIC":
        p = k // 2
        Hp, Wp = H + 2 * p, W + 2 * p
        Ho, Wo = (Hp - (k - 1) * d - 1) // s + 1, (Wp - (k - 1) * d - 1) // s + 1
        return S.Geom(B, Hp, Wp, Cin, Ho, Wo, Cout, k, k, s, d, 0, 0)
    return S.Geom(B, H, W, Cin, -(-H // s), -(-W // s), Cout, k, k, s, d, same_pad(H, k, s, d), same_pad(W, k, s, d))


def operands(g, seed):
    """fp32 x [B,H,W,Cin], w HWIO, dy [B,Ho,Wo,Cout] (CPU, seeded)"""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(g.B, g.H, g.W, g.Cin, generator=gen)
    w = torch.randn(g.kh, g.kw, g.Cin, g.Cout, generator=gen) * 0.05
    dy = torch.randn(g.B, g.Ho, g.Wo, g.Cout, generator=gen)
    return x, w, dy


# ------------------------------------------------------------------------------------------------
# C-ABI plumbing
# ------------------------------------------------------------------------------------------------
def _cgeom(_C, g):
    return _C.ConvGeom(*[int(v) for v in g])


def _f64(t):
    return t.to(DEV).to(torch.float64)


def _report(tag, launcher, nterms, ratio):
    tau = S.TAU[(launcher, nterms)]
    print("  RATIO %-6s nterms %d %-34s worst |got-ref|/sum|a||b| %.3e  tau %.3e" % (launcher, nterms, tag, ratio, tau))
    return tau


def _check(tag, launcher, nterms, got, ref, cond, slack=None):
    ratio = S.worst_ratio(got, ref, cond, slack)
    tau = _report(tag, launcher, nterms, ratio)
    print("        tau * max(sum|a||b|) / max|ref| = %.2e (the same bound normalised like the fp64-oracle tests)" %
          (tau * float(cond.max()) / max(float(ref.abs().max()), 1e-300)))
    bad = S.violations(got, ref, cond, tau, slack)
    assert bad == 0, "%s %s nterms %d: %d elements beyond tau %.3e (worst ratio %.3e)" % (tag, launcher, nterms, bad, tau, ratio)


# ------------------------------------------------------------------------------------------------
# a. plane producers, bit for bit
# ------------------------------------------------------------------------------------------------
def edge_values():
    """fp32 edge values of the split (the same list the CPU test pins against a bit-level RNE)"""
    pats = [0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00008000, 0x00018000, 0x00800000,
            0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000, 0x3F808001, 0x3F817FFF, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F7F8000,
            0x7F7F7FFF, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7F800001, 0xFFC00001, 0x3F800000, 0x33800000, 0x3EAAAAAB]
    return torch.tensor([p - (1 << 32) if p >= (1 << 31) else p for p in pats], dtype=torch.int32).view(torch.float32)


@pytest.mark.parametrize("n", [1, 2, 3, 5, 7, 27, 1_000_003])
def test_split_bf16_planes_are_exact(n):
    _C, rt = lib(require_tc=True)
    gen = torch.Generator().manual_seed(n)
    x = torch.randn(n, generator=gen) * torch.exp2(torch.randint(-140, 120, (n,), generator=gen).float())
    e = edge_values()
    x[:min(n, e.numel())] = e[:min(n, e.numel())]
    x = x.to(DEV)
    for nterms in (3, 1):
        hi, lo = split_dev(_C, rt, x, nterms)
        torch.cuda.synchronize()
        assert_planes("pnp_split_bf16 n=%d nterms=%d" % (n, nterms), hi, lo, x)


def test_split_bf16_pad_planes_are_exact():
    _C, rt = lib(require_tc=True)
    for rows, C, Cpad in ((37, 32, 64), (5, 4, 16), (300, 48, 64), (9, 64, 64)):
        x = (torch.randn(rows, C) * 3).to(DEV)
        hi = torch.full((rows, Cpad), 1.0, dtype=torch.bfloat16, device=DEV)
        lo = torch.full((rows, Cpad), 1.0, dtype=torch.bfloat16, device=DEV)
        _C.call("pnp_split_bf16_pad", _C.ptr(x), _C.ptr(hi), _C.ptr(lo), rows, C, Cpad, rt.stream())
        torch.cuda.synchronize()
        assert_planes("pnp_split_bf16_pad", hi[:, :C].contiguous(), lo[:, :C].contiguous(), x)
        assert int(S.bits(hi[:, C:]).abs().sum()) == 0 and int(S.bits(lo[:, C:]).abs().sum()) == 0, "padding channels not zero"


@pytest.mark.parametrize("kh,Cin,Cout,cin_pad", [(3, 64, 128, 0), (5, 32, 64, 64), (1, 16, 16, 0), (3, 48, 40, 64), (3, 5, 33, 0)])
def test_split_weight_planes_are_exact(kh, Cin, Cout, cin_pad):
    _C, rt = lib(require_tc=True)
    w = torch.randn(kh, kh, Cin, Cout) * 0.05
    w.view(-1)[:27] = edge_values()[:27]
    w = w.to(DEV)
    hi, lo = split_w_dev(_C, rt, w, False, 3, cin_pad)
    torch.cuda.synchronize()
    cp = max(Cin, cin_pad)
    wf = torch.zeros(kh * kh, Cout, cp)
    wf[:, :, :Cin] = w.cpu().reshape(kh * kh, Cin, Cout).permute(0, 2, 1)
    assert_planes("pnp_split_weight_bf16 fwd layout", hi, lo, wf.reshape(-1))
    if cin_pad <= Cin:
        hi, lo = split_w_dev(_C, rt, w, True, 3)
        torch.cuda.synchronize()
        assert_planes("pnp_split_weight_bf16 dgrad layout", hi, lo, w.cpu().reshape(-1))


def _bn_inputs(M, C, seed):
    gen = torch.Generator().manual_seed(seed)
    z = torch.randn(M, C, generator=gen) * 2 + 0.3
    f = lambda *s: torch.randn(*s, generator=gen)  # noqa: E731
    return (z.to(DEV), (1 + 0.3 * f(C)).to(DEV), (0.2 * f(C)).to(DEV), (0.1 * f(C)).to(DEV), (1 + 0.2 * torch.rand(C, generator=gen)).to(DEV),
            f(M, C).to(DEV))


@pytest.mark.parametrize("act", [0, 1, 2])
def test_bn_act_apply_planes(act):
    _C, rt = lib(require_tc=True)
    M, C = 1000, 96
    z, scale, shift, _, _, skip_src = _bn_inputs(M, C, 5 + act)
    skip = skip_src[:, :32].contiguous()
    for sk, Cs, off in ((None, 0, 0), (skip, 32, 40)):
        y = torch.empty(M, C, device=DEV)
        hi, lo = empty_planes((M, C), 3)
        _C.call("pnp_bn_act_apply", _C.ptr(z), _C.ptr(scale), _C.ptr(shift), _C.ptr(sk), Cs, off, act, _C.ptr(y), _C.ptr(hi),
                _C.ptr(lo), M, C, rt.stream())
        torch.cuda.synchronize()
        assert_planes("pnp_bn_act_apply act=%d skip=%s" % (act, sk is not None), hi, lo, y)


@pytest.mark.parametrize("training", [1, 0])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_bn_apply_fused_planes(training, act):
    _C, rt = lib(require_tc=True)
    M, C = 2048, 128
    z, gamma, beta, mm, mv, skip_src = _bn_inputs(M, C, 17 + act)
    zs = z.double()
    s1, s2 = zs.sum(0).contiguous(), (zs * zs).sum(0).contiguous()
    skip = skip_src[:, :64].contiguous()
    outs = []
    for with_y in (True, False):
        y = torch.empty(M, C, device=DEV) if with_y else None
        hi, lo = empty_planes((M, C), 3)
        mm_, mv_ = mm.clone(), mv.clone()
        _C.call("pnp_bn_apply_fused", _C.ptr(z), _C.ptr(s1), _C.ptr(s2), M, C, _C.ptr(gamma), _C.ptr(beta), _C.ptr(mm_), _C.ptr(mv_),
                training, _C.ptr(skip), 64, 32, act, _C.ptr(y), _C.ptr(hi), _C.ptr(lo), None, None, rt.stream())
        torch.cuda.synchronize()
        if with_y:
            assert_planes("pnp_bn_apply_fused train=%d act=%d" % (training, act), hi, lo, y)
        outs.append((hi, lo))
    assert torch.equal(S.bits(outs[0][0]), S.bits(outs[1][0])) and torch.equal(S.bits(outs[0][1]), S.bits(outs[1][1])), \
        "planes-only launch wrote different planes"


@pytest.mark.parametrize("keep", [1.0, 0.75])
@pytest.mark.parametrize("training", [1, 0])
def test_bn_bwd_apply_planes(keep, training):
    _C, rt = lib(require_tc=True)
    M, C = 3000, 64
    z, gamma, _, mean, var, g = _bn_inputs(M, C, 31)
    invstd = torch.rsqrt(var + 1e-3)
    dcfg, seed_t = drop_cfg(_C, keep) if keep < 1 else (None, None)
    dref = None if dcfg is None else ctypes.byref(dcfg)
    coef = (torch.randn(2 * C) * 0.1).to(DEV)
    dz = torch.empty(M, C, device=DEV)
    hi, lo = empty_planes((M, C), 3)
    _C.call("pnp_bn_bwd_apply", _C.ptr(g), _C.ptr(z), _C.ptr(mean), _C.ptr(invstd), _C.ptr(gamma), _C.ptr(coef), training, dref,
            _C.ptr(dz), _C.ptr(hi), _C.ptr(lo), M, C, rt.stream())
    torch.cuda.synchronize()
    assert_planes("pnp_bn_bwd_apply", hi, lo, dz)
    gs = g.double()
    sg, sgx = gs.sum(0).contiguous(), (gs * ((z.double() - mean.double()) * invstd.double())).sum(0).contiguous()
    dz = torch.empty(M, C, device=DEV)
    hi, lo = empty_planes((M, C), 3)
    _C.call("pnp_bn_bwd_apply_fused", _C.ptr(g), _C.ptr(z), _C.ptr(mean), _C.ptr(invstd), _C.ptr(gamma), _C.ptr(sg), _C.ptr(sgx), M, C,
            training, dref, None, None, _C.ptr(dz), _C.ptr(hi), _C.ptr(lo), rt.stream())
    torch.cuda.synchronize()
    assert_planes("pnp_bn_bwd_apply_fused", hi, lo, dz)
    # direct: g recomputed from dy and the activation sign (from y, or from y's hi plane); planes-only == planes with fp32
    y = torch.randn(M, C).to(DEV)
    yhi, _ = split_dev(_C, rt, y, 1)
    for act in (0, 1, 2):
        for src in ("y", "y_hi"):
            outs = []
            for with_dz in (True, False):
                dz = torch.empty(M, C, device=DEV) if with_dz else None
                hi, lo = empty_planes((M, C), 3)
                _C.call("pnp_bn_bwd_apply_direct", _C.ptr(g), _C.ptr(y if src == "y" else None), _C.ptr(yhi if src == "y_hi" else None),
                        act, _C.ptr(z), _C.ptr(mean), _C.ptr(invstd), _C.ptr(gamma), _C.ptr(sg), _C.ptr(sgx), M, C, training, dref,
                        None, None, _C.ptr(dz), _C.ptr(hi), _C.ptr(lo), rt.stream())
                torch.cuda.synchronize()
                if with_dz:
                    assert_planes("pnp_bn_bwd_apply_direct act=%d %s" % (act, src), hi, lo, dz)
                outs.append((S.bits(hi), S.bits(lo)))
            assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), "planes-only dz planes differ"


# ------------------------------------------------------------------------------------------------
# b. convolutions against the split reference
# ------------------------------------------------------------------------------------------------
def _fwd(_C, rt, xh, xl, wh, wl, y, g, nterms, drop=None, acc=0, bn=None, ep=None):
    _C.call("pnp_conv2d_tc_fwd_fused", _C.ptr(xh), _C.ptr(xl), _C.ptr(wh), _C.ptr(wl), _C.ptr(y), ctypes.byref(_cgeom(_C, g)), nterms,
            None if drop is None else ctypes.byref(drop), acc, _C.ptr(bn[0]) if bn else None, _C.ptr(bn[1]) if bn else None,
            None if ep is None else ctypes.byref(ep), rt.stream())


def _dgrad(_C, rt, dh, dl, wh, wl, dx, g, nterms, acc):
    _C.call("pnp_conv2d_tc_dgrad", _C.ptr(dh), _C.ptr(dl), _C.ptr(wh), _C.ptr(wl), _C.ptr(dx), ctypes.byref(_cgeom(_C, g)), nterms, acc,
            rt.stream())


def _wgrad(_C, rt, xh, xl, dh, dl, dw, g, nterms):
    _C.call("pnp_conv2d_tc_wgrad", _C.ptr(xh), _C.ptr(xl), _C.ptr(dh), _C.ptr(dl), _C.ptr(dw), ctypes.byref(_cgeom(_C, g)), nterms, 0,
            rt.stream())


class Prepared:
    """device operands and their planes for one case and nterms, plus the fp64 split references"""

    def __init__(self, _C, rt, case, nterms, seed=101):
        self.g = g = geom_of(case)
        self.nterms = nterms
        x, w, dy = operands(g, seed)
        self.x, self.w, self.dy = x.to(DEV), w.to(DEV), dy.to(DEV)
        self.xh, self.xl = split_dev(_C, rt, self.x, nterms)
        self.wh, self.wl = split_w_dev(_C, rt, self.w, False, nterms)
        self.wdh, self.wdl = split_w_dev(_C, rt, self.w, True, nterms)
        self.dh, self.dl = split_dev(_C, rt, self.dy, nterms)
        torch.cuda.synchronize()
        lo = (lambda p: None if p is None else _f64(p))
        self.x64 = (_f64(self.xh), lo(self.xl))
        self.dy64 = (_f64(self.dh), lo(self.dl))
        self.wf64 = S.fwd_weight_planes(self.wh, self.wl, g.kh, g.kw, g.Cin, g.Cout)
        self.wd64 = S.dgrad_weight_planes(self.wdh, self.wdl, g.kh, g.kw, g.Cin, g.Cout)
        self.wf64 = tuple(None if p is None else p.to(DEV) for p in self.wf64)
        self.wd64 = tuple(None if p is None else p.to(DEV) for p in self.wd64)

    def fwd_ref(self):
        return S.fwd_ref(self.x64[0], self.x64[1], self.wf64[0], self.wf64[1], self.g, self.nterms)

    def dgrad_ref(self):
        return S.dgrad_ref(self.dy64[0], self.dy64[1], self.wd64[0], self.wd64[1], self.g, self.nterms)

    def wgrad_ref(self):
        return S.wgrad_ref(self.x64[0], self.x64[1], self.dy64[0], self.dy64[1], self.g, self.nterms)


def _yshape(g):
    return (g.B, g.Ho, g.Wo, g.Cout)


def _xshape(g):
    return (g.B, g.H, g.W, g.Cin)


@pytest.mark.parametrize("nterms", [3, 1])
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_conv_split_exact(case, nterms):
    """fwd (+accumulate, dropout, BN sums), dgrad (+accumulate), wgrad (+accumulate) per element against the split reference"""
    _C, rt = lib(require_tc=True)
    tag, flags = case[0], case[-1]
    P = Prepared(_C, rt, case, nterms)
    g = P.g
    gen = torch.Generator().manual_seed(7)

    # -- forward, plain
    ref, cond = P.fwd_ref()
    y = torch.full(_yshape(g), float("nan"), device=DEV)
    _fwd(_C, rt, P.xh, P.xl, P.wh, P.wl, y, g, nterms)
    torch.cuda.synchronize()
    ks_fwd = last_config(_C)[2]
    print("  %s: forward tile %s" % (tag, last_config(_C)))
    assert ks_fwd == expected_ksplit("fwd", g, sm_count()), "%s: forward split-K factor %d" % (tag, ks_fwd)
    _check(tag, "fwd", nterms, y, ref, cond)

    # -- forward, accumulate into a non-zero y (split-K: atomics onto it; else read-add-write)
    y0 = torch.randn(_yshape(g), generator=gen).to(DEV)
    y = y0.clone()
    _fwd(_C, rt, P.xh, P.xl, P.wh, P.wl, y, g, nterms, acc=1)
    torch.cuda.synchronize()
    assert last_config(_C)[2] == ks_fwd
    y064 = y0.double()
    _check(tag + " acc", "fwd", nterms, y, y064 + ref, cond, slack=2 * U32 * (y064.abs() + ref.abs()))

    # -- forward with dropout: mask (x) conv_split at every element, with the multiplier of pnp_dropout_apply
    if "drop" in flags:
        cfg, seed_t = drop_cfg(_C, 0.75)
        mask = drop_mask(cfg, _yshape(g)).double()
        y = torch.full(_yshape(g), float("nan"), device=DEV)
        _fwd(_C, rt, P.xh, P.xl, P.wh, P.wl, y, g, nterms, drop=cfg)
        torch.cuda.synchronize()
        assert 0.7 < float((mask != 0).double().mean()) < 0.8
        _check(tag + " dropout", "fwd", nterms, y, mask * ref, mask * cond, slack=U32 * (mask * ref).abs())

    # -- forward with BN sums (fused epilogue statistics, or pnp_bn_stats after split-K) against fp64 sums of its own output
    if "bn" in flags:
        s1 = torch.zeros(g.Cout, dtype=torch.float64, device=DEV)
        s2 = torch.zeros_like(s1)
        y = torch.full(_yshape(g), float("nan"), device=DEV)
        _fwd(_C, rt, P.xh, P.xl, P.wh, P.wl, y, g, nterms, bn=(s1, s2))
        torch.cuda.synchronize()
        _check(tag + " bn", "fwd", nterms, y, ref, cond)
        z = y.double().reshape(-1, g.Cout)
        e1 = float(((s1 - z.sum(0)).abs() / z.abs().sum(0)).max())
        e2 = float(((s2 - (z * z).sum(0)).abs() / (z * z).sum(0)).max())
        print("  BN sums %-30s split-K %d: sum err %.2e of sum|z|, sumsq err %.2e of sum z^2 (tol 2^-19 = %.2e)" %
              (tag, ks_fwd, e1, e2, 2.0 ** -19))
        assert e1 <= 2.0 ** -19 and e2 <= 2.0 ** -19

    # -- data gradient, plain and accumulating
    ref, cond = P.dgrad_ref()
    dx = torch.full(_xshape(g), float("nan"), device=DEV)
    _dgrad(_C, rt, P.dh, P.dl, P.wdh, P.wdl, dx, g, nterms, 0)
    torch.cuda.synchronize()
    ks_dg = last_config(_C)[2]
    print("  %s: dgrad tile %s" % (tag, last_config(_C)))
    assert ks_dg == expected_ksplit("dgrad", g, sm_count()), "%s: dgrad split-K factor %d" % (tag, ks_dg)
    _check(tag, "dgrad", nterms, dx, ref, cond)
    dx0 = torch.randn(_xshape(g), generator=gen).to(DEV)
    dx = dx0.clone()
    _dgrad(_C, rt, P.dh, P.dl, P.wdh, P.wdl, dx, g, nterms, 1)
    torch.cuda.synchronize()
    d064 = dx0.double()
    _check(tag + " acc", "dgrad", nterms, dx, d064 + ref, cond, slack=2 * U32 * (d064.abs() + ref.abs()))

    # -- weight gradient (always accumulates) into a non-zero dw
    if "wgrad" in flags:
        ref, cond = P.wgrad_ref()
        dw0 = (torch.randn(g.kh, g.kw, g.Cin, g.Cout, generator=gen) * 0.01).to(DEV)
        dw = dw0.clone()
        _wgrad(_C, rt, P.xh, P.xl, P.dh, P.dl, dw, g, nterms)
        torch.cuda.synchronize()
        w064 = dw0.double()
        _check(tag, "wgrad", nterms, dw, w064 + ref, cond, slack=2 * U32 * (w064.abs() + ref.abs()))


EP_CASES = [c for c in CASES if "ep" in c[-1]]


@pytest.mark.parametrize("nterms", [3, 1])
@pytest.mark.parametrize("act", [0, 1, 2], ids=["none", "relu", "lrelu"])
@pytest.mark.parametrize("case", EP_CASES, ids=[c[0] for c in EP_CASES])
def test_conv_fused_epilogue_split_exact(case, act, nterms):
    """y = act(dropout(conv) * scale + shift + skip) against the fp64 epilogue of the split reference; its bf16 planes are
    split(y) bit for bit (tc1: hi only, y_lo = NULL), and a planes-only launch (y = NULL) writes the same planes"""
    _C, rt = lib(require_tc=True)
    tag, flags = case[0], case[-1]
    P = Prepared(_C, rt, case, nterms)
    g = P.g
    gen = torch.Generator().manual_seed(100 + act)
    scale = (1 + 0.5 * torch.randn(g.Cout, generator=gen)).to(DEV)
    shift = (0.3 * torch.randn(g.Cout, generator=gen)).to(DEV)
    skip_c, skip_off = g.Cout // 2, g.Cout // 4
    skip = torch.randn(g.B, g.Ho, g.Wo, skip_c, generator=gen).to(DEV)
    cfg, seed_t = drop_cfg(_C, 0.75, stream_id=23) if "drop" in flags else (None, None)
    ref, cond = P.fwd_ref()
    mask = drop_mask(cfg, _yshape(g)).double() if cfg is not None else torch.ones(_yshape(g), dtype=torch.float64, device=DEV)
    sc, sh = scale.double(), shift.double()
    sk = torch.zeros(_yshape(g), dtype=torch.float64, device=DEV)
    sk[..., skip_off:skip_off + skip_c] = skip.double()
    zs = mask * ref * sc
    pre = zs + sh + sk
    out = pre if act == 0 else (pre.clamp_min(0) if act == 1 else torch.where(pre > 0, pre, 0.2 * pre))
    bound_cond = mask * cond * sc.abs()
    slack = 4 * U32 * (zs.abs() + sh.abs() + sk.abs())
    written = []
    for with_y in (True, False):
        y = torch.full(_yshape(g), float("nan"), device=DEV) if with_y else None
        yh, yl = empty_planes(_yshape(g), nterms)
        ep = _C.TcEpilogue(_C.ptr(scale), _C.ptr(shift), _C.ptr(skip), skip_c, skip_off, act, _C.ptr(yh), _C.ptr(yl))
        _fwd(_C, rt, P.xh, P.xl, P.wh, P.wl, y, g, nterms, drop=cfg, ep=ep)
        torch.cuda.synchronize()
        assert last_config(_C)[2] == 1
        if with_y:
            _check("%s ep act=%d" % (tag, act), "fwd", nterms, y, out, bound_cond, slack=slack)
            assert_planes("%s epilogue planes" % tag, yh, yl, y)
        written.append([S.bits(p) for p in (yh, yl) if p is not None])
    assert all(torch.equal(a, b) for a, b in zip(*written)), "planes-only epilogue wrote different planes"


# ------------------------------------------------------------------------------------------------
# c. the check has power on the device too (valid memory only: TMA zero-fills the shifted window)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [CASES[3], CASES[1]], ids=[CASES[3][0], CASES[1][0]])
def test_split_check_rejects_broken_launches(case):
    _C, rt = lib(require_tc=True)
    tag = case[0]
    P = Prepared(_C, rt, case, 3)
    g = P.g
    ref, cond = P.fwd_ref()
    tau = S.TAU[("fwd", 3)]
    # zeroed lo plane of the activation operand
    y = torch.empty(_yshape(g), device=DEV)
    _fwd(_C, rt, P.xh, torch.zeros_like(P.xl), P.wh, P.wl, y, g, 3)
    torch.cuda.synchronize()
    n1 = S.violations(y, ref, cond, tau)
    # pad_l off by one (every tap window shifted one pixel left)
    y2 = torch.empty(_yshape(g), device=DEV)
    _fwd(_C, rt, P.xh, P.xl, P.wh, P.wl, y2, g._replace(pad_l=g.pad_l + 1), 3)
    torch.cuda.synchronize()
    n2 = S.violations(y2, ref, cond, tau)
    # accumulate = 0 where 1 was meant
    y0 = torch.randn(_yshape(g)).to(DEV)
    y3 = y0.clone()
    _fwd(_C, rt, P.xh, P.xl, P.wh, P.wl, y3, g, 3, acc=0)
    torch.cuda.synchronize()
    exp = y0.double() + ref
    n3 = S.violations(y3, exp, cond, tau, slack=2 * U32 * (y0.double().abs() + ref.abs()))
    # the zeroed lo plane of the data-gradient weights
    dx = torch.empty(_xshape(g), device=DEV)
    _dgrad(_C, rt, P.dh, P.dl, P.wdh, torch.zeros_like(P.wdl), dx, g, 3, 0)
    torch.cuda.synchronize()
    dref, dcond = P.dgrad_ref()
    n4 = S.violations(dx, dref, dcond, S.TAU[("dgrad", 3)])
    print("  %s: elements rejected: zero x_lo %d, pad_l+1 %d, accumulate dropped %d, zero w_lo (dgrad) %d of %d" %
          (tag, n1, n2, n3, n4, y.numel()))
    assert n1 > 0 and n2 > 0 and n3 > 0 and n4 > 0


# ------------------------------------------------------------------------------------------------
# d. the decline contract
# ------------------------------------------------------------------------------------------------
DECLINE = [
    ("fwd", S.Geom(1, 8, 200, 64, 8, 200, 64, 3, 3, 1, 1, 1, 1)),          # W = 200 at stride 1: no 128-pixel tiling
    ("dgrad", S.Geom(1, 8, 200, 64, 8, 200, 64, 3, 3, 1, 1, 1, 1)),
    ("fwd", S.Geom(2, 16, 16, 48, 16, 16, 64, 3, 3, 1, 1, 1, 1)),          # Cin = 48
    ("dgrad", S.Geom(2, 16, 16, 64, 16, 16, 48, 3, 3, 1, 1, 1, 1)),        # Cout = 48
    ("fwd", S.Geom(2, 16, 16, 64, 16, 16, 64, 7, 7, 1, 1, 3, 3)),          # 49 taps
    ("dgrad", S.Geom(2, 16, 16, 64, 16, 16, 64, 7, 7, 1, 1, 3, 3)),
    ("wgrad", S.Geom(2, 16, 16, 64, 16, 16, 32, 3, 3, 1, 1, 1, 1)),        # wgrad Cout = 32
    ("wgrad", S.Geom(2, 16, 16, 16, 16, 16, 64, 3, 3, 1, 1, 1, 1)),        # wgrad Cin = 16
    ("fwd", S.Geom(1, 512, 512, 64, 128, 128, 64, 3, 3, 4, 1, 0, 0)),      # TMA box 128 x 4 = 512 pixels wide
]


@pytest.mark.parametrize("launcher,g", DECLINE, ids=["%s_%d" % (d[0], i) for i, d in enumerate(DECLINE)])
def test_unsupported_shapes_are_declined_untouched(launcher, g):
    _C, rt = lib(require_tc=True)
    xh = torch.zeros(g.B * g.H * g.W * g.Cin, dtype=torch.bfloat16, device=DEV)
    dh = torch.zeros(g.B * g.Ho * g.Wo * g.Cout, dtype=torch.bfloat16, device=DEV)
    wh = torch.zeros(g.kh * g.kw * g.Cin * g.Cout, dtype=torch.bfloat16, device=DEV)
    shape = {"fwd": _yshape(g), "dgrad": _xshape(g), "wgrad": (g.kh, g.kw, g.Cin, g.Cout)}[launcher]
    out = torch.full(shape, 1234.5, device=DEV)
    with pytest.raises(_C.Unsupported):
        if launcher == "fwd":
            _fwd(_C, rt, xh, xh, wh, wh, out, g, 3)
        elif launcher == "dgrad":
            _dgrad(_C, rt, dh, dh, wh, wh, out, g, 3, 0)
        else:
            _wgrad(_C, rt, xh, xh, dh, dh, out, g, 3)
    torch.cuda.synchronize()
    assert bool((out == 1234.5).all()), "a declined launch wrote its output"


def test_accumulate_with_bn_sums_is_rejected():
    """batch statistics of an accumulating forward would be of the new contribution on one path and of old + new on the
    split-K path: the launcher refuses the combination"""
    _C, rt = lib(require_tc=True)
    for case in (CASES[1], CASES[3]):            # split-K (on an H100) and single-pass forward
        g = geom_of(case)
        P = Prepared(_C, rt, case, 3)
        s1 = torch.zeros(g.Cout, dtype=torch.float64, device=DEV)
        s2 = torch.zeros_like(s1)
        y = torch.zeros(_yshape(g), device=DEV)
        with pytest.raises(RuntimeError, match="100001"):
            _fwd(_C, rt, P.xh, P.xl, P.wh, P.wl, y, g, 3, acc=1, bn=(s1, s2))
        torch.cuda.synchronize()
        assert bool((y == 0).all()) and bool((s1 == 0).all())


# ------------------------------------------------------------------------------------------------
# e. tile / order / launch-mode switches, each in its own process
# ------------------------------------------------------------------------------------------------
def test_last_config_reports_k_block():
    """PNP_TC_BK128 / PNP_TC_BK64 = 32 select the <128,*,32> / <64,*,32> instantiations for 64-multiple reductions"""
    _C, rt = lib(require_tc=True)
    want = {128: int(os.environ.get("PNP_TC_BK128", "64")) == 32 and 32 or 64,
            64: int(os.environ.get("PNP_TC_BK64", "64")) == 32 and 32 or 64}
    for case, bn in ((CASES[3], 128), (CASES[12], 64)):
        P = Prepared(_C, rt, case, 3)
        y = torch.empty(_yshape(P.g), device=DEV)
        _fwd(_C, rt, P.xh, P.xl, P.wh, P.wl, y, P.g, 3)
        torch.cuda.synchronize()
        assert last_config(_C)[:2] == (bn, want[bn]), (case[0], last_config(_C))


# each switch re-runs only the cases whose kernels it changes: the K-block switches the 128- and 64-column tiles over 64-multiple
# reductions (and the tile report); the taps-inner order and the rotation the multi-chunk reductions (rotation needs >= 16
# k-blocks); programmatic dependent launch every kernel family once (plane producers, plain, split-K and phase convolutions,
# the fused epilogue).  The last entry is the number of tests each selection runs.
def _n(cases, *names):
    return sum(1 for c in cases if any(n in c[0] for n in names))


SWITCHES = [
    ({"PNP_TC_BK128": "32", "PNP_TC_BK64": "32"},
     "last_config or (conv_split_exact and (g10 or dil2 or 256x512 or 64_s2_256wide or 64_12x20 or wg_cin64))",
     1 + 2 * _n(CASES, "g10", "dil2", "256x512", "64_s2_256wide", "64_12x20", "wg_cin64")),
    ({"PNP_TC_ORDER": "1", "PNP_TC_ROT": "0"}, "conv_split_exact and (g10 or dil2 or k5s4 or 256x512 or wg_cin192)",
     2 * _n(CASES, "g10", "dil2", "k5s4", "256x512", "wg_cin192")),
    ({"PNP_PDL": "1"}, "split_bf16 or bn_ or (conv_split_exact and (k5s4 or 256x512 or 16x32_k5s4)) or (epilogue and 64x32)",
     # split_bf16: 7 sizes + the padded split; bn_: 3 + 6 + 4 plane tests and the accumulate-with-BN-sums rejection
     8 + 14 + 2 * _n(CASES, "k5s4", "256x512") + 6 * _n(EP_CASES, "64x32")),
]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("env,kexpr,n", SWITCHES, ids=["bk32", "order1_rot0", "pdl"])
def test_switch_variants(env, kexpr, n):
    passed, lines = rerun(env, __file__, kexpr, flags=("-s",))
    print("\n".join(l for l in lines if "RATIO" in l or "BN sums" in l))
    assert passed == n, "%s: %d of %d tests passed" % (env, passed, n)
