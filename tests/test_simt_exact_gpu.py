"""The fp32 SIMT convolutions (conv_simt.cu) and the fused segmenter tail, bit for bit on integer operands and per element on
real ones, at shapes that reach every kernel instantiation.

a. integer operands in [-4, 4]: every product and partial sum is an integer below 2^24, so the fp32 result does not depend on
   summation order, pixel splits or atomic order and must equal the fp64 reference exactly (torch.equal) -- at every element,
   with accumulate, with dropout (the multiplier pnp_dropout_apply draws at the same flat index), through the weight transpose,
   and for the tail's backward also against the three-kernel route (data gradient -> mirror-pad fold -> inverse phase shift).
   Each case first asserts that precondition on the reference: max sum|a||b| < 2^24;
b. randn operands: |got - ref| <= tau * sum|a||b| per element with the calibrated TAU of oracle/simt_exact.py, and within the
   rigorous gamma_n bound.  Small integers are exact in TF32 and bf16 too, so this is what pins the kernels to fp32 arithmetic;
c. the kernels each launch ran are the ones oracle/simt_exact.simt_instance() names (torch.profiler), so the CPU test's
   coverage claim -- the case tables reach every instantiation in the library -- is about the real dispatch;
d. bad arguments and shapes the launchers cannot run are declined with PNP_ERR_BAD_ARG / PNP_ERR_UNSUPPORTED, output untouched;
e. PNP_TAIL5 (read once per process) = 0, 1, 2 re-runs the 5x5 tail cases in a process of its own each.

The C-ABI is called directly (_C.call / ptr / ConvGeom / DropCfg) on the runtime's stream; the fp64 references run on the device."""
import ctypes
import os
import time

import pytest
import torch

from oracle import bf16_split as S
from oracle import simt_exact as E
from oracle.simt_exact import TailGeom
from tests.cabi import BAD_ARG, DEV, cpu_gen, drop_cfg, drop_mask, ints, lib, rerun, same_pad

pytestmark = pytest.mark.gpu
EXACT = 2.0 ** 24


def conv(B, H, W, Cin, Cout, kh, kw=None, s=1, d=1, pad="SAME"):
    """oracle Geom: pad = 'SAME', 'VALID' or explicit (pad_t, pad_l) with the same amount at the bottom / right"""
    kw = kh if kw is None else kw
    if pad == "SAME":
        return S.Geom(B, H, W, Cin, -(-H // s), -(-W // s), Cout, kh, kw, s, d, same_pad(H, kh, s, d), same_pad(W, kw, s, d))
    pt, pl = (0, 0) if pad == "VALID" else pad
    Ho, Wo = (H + 2 * pt - (kh - 1) * d - 1) // s + 1, (W + 2 * pl - (kw - 1) * d - 1) // s + 1
    return S.Geom(B, H, W, Cin, Ho, Wo, Cout, kh, kw, s, d, pt, pl)


# (id, forward geometry, flags).  flags: drop50 / drop75 = the forward also runs with dropout at keep 0.5 / 0.75; real = the
# case also runs on randn operands.  The comment names the instantiation (restated by oracle/simt_exact.simt_instance).
FWD = [
    ("s3_o8", conv(2, 37, 29, 3, 8, 3), {"real"}),                             # gather <1024,8,8,4,8,1>, K = 27
    ("s5_o5_k5_drop75", conv(2, 33, 35, 5, 5, 5), {"drop75"}),                  # same tile, scalar store with dropout
    ("s3_o16_s2_drop75", conv(2, 64, 64, 3, 16, 3, s=2), {"drop75"}),           # <256,16,16,4,4,1>, float4 store with dropout
    ("s5_o12_d2", conv(1, 40, 36, 5, 12, 3, d=2), set()),                      # <256,16,16,4,4,1>, Cout 12 of a 16 tile
    ("s3_o32", conv(2, 48, 48, 3, 32, 3), {"real"}),                           # <128,64,16,8,4,1>
    ("s5_o40_3x5_d2", conv(1, 30, 41, 5, 40, 3, 5, d=2), set()),               # <128,64,16,8,4,1>, kh != kw
    ("c8_o8_s2", conv(2, 40, 40, 8, 8, 3, s=2), set()),                        # <1024,8,8,4,8,4> (strided: no few-output kernel)
    ("c12_o6_drop50", conv(2, 35, 30, 12, 6, 3), {"drop50"}),                  # <1024,8,8,4,8,4>, Cout % 4 != 0 with dropout
    ("c12_o5_k5", conv(1, 50, 45, 12, 5, 5), set()),                          # Cin % 8 != 0: gather, Cout 5
    ("c16_o16", conv(2, 30, 30, 16, 16, 3), {"real"}),                         # <256,16,16,4,4,4>
    ("c12_o12_s2", conv(2, 33, 31, 12, 12, 3, s=2), set()),                    # <256,16,8,4,4,4>, K = 108 (ragged BK)
    ("c32_o32_k5s4", conv(4, 32, 32, 32, 32, 5, s=4), set()),                  # <256,32,16,8,4,4>, stride 4
    ("c20_o24", conv(2, 26, 22, 20, 24, 3), {"real"}),                         # <256,32,8,8,4,4>, K = 180
    ("c48_o64_d2", conv(2, 24, 24, 48, 64, 3, d=2), set()),                    # <128,64,16,8,4,4>, dilation 2
    ("c16_o128_8tiles", conv(1, 32, 32, 16, 128, 3), set()),                   # <128,64,16,8,4,4>: Cout 128, too few 128x128 tiles
    ("c40_o40_drop50", conv(2, 32, 32, 40, 40, 3), {"drop50", "real"}),        # <128,64,8,8,4,4>
    ("c16_o128_192_drop75", conv(1, 192, 192, 16, 128, 3), {"drop75", "real"}),  # <128,128,16,8,8,4>: 288 tiles
    ("c20_o130_192_drop50", conv(1, 192, 192, 20, 130, 3), {"drop50"}),        # <128,128,8,8,8,4>, Cout % 4 != 0
    ("fo5_3x5_B3", conv(3, 45, 70, 16, 5, 3, 5, pad=(0, 2)), {"real"}),         # few-output <5>: ragged tiles, pad_t != pad_l
    ("fo8_k5", conv(2, 33, 40, 40, 8, 5), {"real"}),                           # few-output <8>
    ("fo5_valid_68", conv(2, 68, 68, 40, 5, 5, pad="VALID"), set()),           # few-output <5>: the 40 -> 5 output conv
    ("fo8_1x1", conv(1, 20, 50, 8, 8, 1), set()),                              # few-output <8>, 1x1
]

# forward geometries of the data-gradient cases; the instantiation is chosen by the forward Cout (gathered) and Cin (produced)
DGRAD = [
    ("o5_c8_k5", conv(2, 36, 30, 8, 5, 5), set()),                             # <1024,8,8,4,8,1,T>
    ("o3_c16_s2_odd", conv(2, 33, 34, 16, 3, 3, s=2), set()),                  # <256,16,16,4,4,1,T>, odd H
    ("o5_c40_valid_68", conv(2, 68, 68, 40, 5, 5, pad="VALID"), {"real"}),     # <128,64,16,8,4,1,T>: the output conv
    ("o16_c3", conv(2, 40, 40, 3, 16, 3), {"real"}),                           # <1024,8,8,4,8,4,T>
    ("o32_c16_s2_phase", conv(1, 32, 32, 16, 32, 3, s=2), set()),              # <256,16,16,4,4,4,T>, phase-major (256 rows)
    ("o12_c12_s2_odd", conv(2, 33, 30, 12, 12, 3, s=2), set()),                # <256,16,8,4,4,4,T>, odd H: plain row order
    ("o16_c32_s2_pr100", conv(1, 20, 20, 32, 16, 3, s=2), set()),              # <256,32,16,8,4,4,T>, 100 rows per phase % 256
    ("o20_c24", conv(2, 26, 22, 24, 20, 3), {"real"}),                         # <256,32,8,8,4,4,T>
    ("o32_c64_s2_phase", conv(2, 16, 16, 64, 32, 3, s=2), {"real"}),           # <128,64,16,8,4,4,T>, phase-major (128 rows)
    ("o40_c40", conv(2, 32, 32, 40, 40, 3), set()),                            # <128,64,8,8,4,4,T>
    ("o16_c128_192", conv(1, 192, 192, 128, 16, 3), {"real"}),                 # <128,128,16,8,8,4,T>
    ("o20_c128_192_d2", conv(1, 192, 192, 128, 20, 3, d=2), set()),            # <128,128,8,8,8,4,T>
    ("o32_c32_k5s4_phase", conv(4, 32, 32, 32, 32, 5, s=4), set()),            # <256,32,16,8,4,4,T>, 16 phases
    ("o16_c16_k3s4_phase", conv(4, 32, 32, 16, 16, 3, s=4), set()),            # phase-major with a phase that no tap reaches
    ("o16_c16_d2", conv(2, 30, 30, 16, 16, 3, d=2), set()),                    # dilated data gradient
]

WGRAD = [
    ("c3_o16_128splits", conv(2, 64, 64, 3, 16, 3), {"real"}),                 # <64,16,16,4,1,1>
    ("c5_o32_s2", conv(2, 40, 40, 5, 32, 3, s=2), set()),                      # <64,64,16,4,4,1>
    ("c40_o5_valid_68", conv(2, 68, 68, 40, 5, 5, pad="VALID"), {"real"}),     # <128,8,16,4,1,4>, KK = 1000
    ("c16_o12_1split", conv(1, 6, 7, 16, 12, 3), set()),                       # <64,16,16,4,1,4>, M = 42: one split
    ("c32_o32_d2", conv(2, 24, 24, 32, 32, 3, d=2), set()),                    # <64,32,16,4,2,4>
    ("c12_o40", conv(2, 30, 30, 12, 40, 3), {"real"}),                         # <64,64,16,4,4,4>, KK = 108
    ("c8_o128_kk72", conv(2, 20, 20, 8, 128, 3), set()),                       # <64,64,16,4,4,4> because KK < 128
    ("c64_o70_s2", conv(2, 32, 32, 64, 70, 3, s=2), {"real"}),                 # <128,128,16,8,8,4>, Cout % 4 != 0
]

TRANSPOSE = [(9, 37, 45), (25, 40, 5), (1, 70, 33), (9, 3, 16)]

# (id, TailGeom(B, a, b, G, r, kh, kw, Cout, order_b1), flags).  Ids of 5x5 cases start with k5_ (the PNP_TAIL5 re-runs select
# them).  r = 8 with order_b1 = 0 takes the 5x5 kernels' fast loader / store; any other r or order the generic loader.
TAIL = [
    ("k5_r8_G40_o5", TailGeom(2, 4, 5, 40, 8, 5, 5, 5, 0), {"real"}),          # 32 x 40
    ("k5_r8_G13_o8_b1", TailGeom(1, 3, 2, 13, 8, 5, 5, 8, 1), set()),          # 24 x 16: less than one tile, G % 8 != 0
    ("k5_r8_G13_o8", TailGeom(2, 5, 3, 13, 8, 5, 5, 8, 0), {"real"}),          # 40 x 24
    ("k5_r4_G40_o8", TailGeom(2, 5, 9, 40, 4, 5, 5, 8, 0), set()),             # 20 x 36
    ("k5_r3_G40_o5_B3", TailGeom(3, 7, 11, 40, 3, 5, 5, 5, 0), set()),         # 21 x 33
    ("k5_r2_a1_edge", TailGeom(2, 1, 3, 13, 2, 5, 5, 5, 0), set()),            # kh / 2 == a * r: every row is folded twice
    ("k5_r8_256", TailGeom(2, 32, 32, 40, 8, 5, 5, 5, 0), {"real"}),           # the segmenter's tail, 256 x 256
    ("k5_r8_256_o8_b1", TailGeom(1, 32, 32, 40, 8, 5, 5, 8, 1), set()),
    ("k3_r8_G40_o5", TailGeom(2, 4, 5, 40, 8, 3, 3, 5, 0), {"real"}),          # generic kernels from here on
    ("k1_r4_G13_o8", TailGeom(2, 5, 9, 13, 4, 1, 1, 8, 0), set()),
    ("k3x5_r2_G13_o5_b1", TailGeom(1, 9, 17, 13, 2, 3, 5, 5, 1), {"real"}),
    ("k3_r1_a1_edge_o8", TailGeom(2, 1, 5, 16, 1, 3, 3, 8, 0), set()),         # kh / 2 == a * r = 1
]


def _drop_keep(flags):
    return 0.5 if "drop50" in flags else (0.75 if "drop75" in flags else None)


def int_launches():
    """every (launcher, geometry, dropout, accumulate) the integer tests below launch in the default process"""
    out = []
    for _, g, flags in FWD:
        out += [("fwd", g, False, 0), ("fwd", g, False, 1)]
        if _drop_keep(flags):
            out.append(("fwd", g, True, 0))
    out += [("dgrad", g, False, a) for _, g, _ in DGRAD for a in (0, 1)]
    out += [("wgrad", g, False, 1) for _, g, _ in WGRAD]
    out += [(l, t, False, 0) for _, t, _ in TAIL for l in ("tail_fwd", "tail_bwd")]
    return out


# ------------------------------------------------------------------------------------------------
# C-ABI plumbing
# ------------------------------------------------------------------------------------------------
def _fwd(_C, rt, x, w, y, g, drop=None, acc=0):
    _C.call("pnp_conv2d_fwd", _C.ptr(x), _C.ptr(w), _C.ptr(y), ctypes.byref(_C.ConvGeom(*[int(v) for v in g])),
            None if drop is None else ctypes.byref(drop), acc, rt.stream())


def _dgrad(_C, rt, dy, wT, dx, g, acc=0):
    _C.call("pnp_conv2d_dgrad", _C.ptr(dy), _C.ptr(wT), _C.ptr(dx), ctypes.byref(_C.ConvGeom(*[int(v) for v in g])), acc, rt.stream())


def _wgrad(_C, rt, x, dy, dw, g):
    _C.call("pnp_conv2d_wgrad", _C.ptr(x), _C.ptr(dy), _C.ptr(dw), ctypes.byref(_C.ConvGeom(*[int(v) for v in g])), rt.stream())


def _transpose(_C, rt, w):
    kh, kw, cin, cout = w.shape
    wT = torch.full((kh, kw, cout, cin), float("nan"), device=DEV)
    _C.call("pnp_weight_transpose", _C.ptr(w), _C.ptr(wT), kh * kw, cin, cout, rt.stream())
    return wT


def _tail(_C, rt, name, src, w, out, t):
    _C.call(name, _C.ptr(src), _C.ptr(w), _C.ptr(out), t.B, t.a, t.b, t.G, t.r, t.kh, t.kw, t.Cout, t.order_b1, rt.stream())


def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _operands(g, seed, integer, dev=DEV):
    """fp32 x [B,H,W,Cin], w HWIO, dy [B,Ho,Wo,Cout] (on `dev`)"""
    gen = torch.Generator().manual_seed(seed)
    shapes = ((g.B, g.H, g.W, g.Cin), (g.kh, g.kw, g.Cin, g.Cout), (g.B, g.Ho, g.Wo, g.Cout))
    if integer:
        return tuple(ints(s, -4, 4, gen).to(dev) for s in shapes)
    x, w, dy = (torch.randn(s, generator=gen) for s in shapes)
    return x.to(dev), (w * 0.05).to(dev), dy.to(dev)


def _tail_operands(t, seed, integer, dev=DEV):
    """X [B, a, b, G*r*r], w HWIO [kh, kw, G, Cout], dy [B, a*r, b*r, Cout] (on `dev`)"""
    gen = torch.Generator().manual_seed(seed)
    shapes = ((t.B, t.a, t.b, t.G * t.r * t.r), (t.kh, t.kw, t.G, t.Cout), (t.B, t.a * t.r, t.b * t.r, t.Cout))
    if integer:
        return tuple(ints(s, -4, 4, gen).to(dev) for s in shapes)
    X, w, dy = (torch.randn(s, generator=gen) for s in shapes)
    return X.to(dev), (w * 0.05).to(dev), dy.to(dev)


def _d(t):
    return t.double()


def _exact(tag, got, want, cond):
    """got equals the fp64 value `want` bit for bit; cond = sum|a||b| (+|accumulated value|) proves that want is exact in fp32"""
    assert float(cond.max()) < EXACT, "%s: sum|a||b| reaches %g: integer results would not be exact in fp32" % (tag, float(cond.max()))
    exp = want.float()
    assert torch.equal(exp.double(), want), "%s: the reference is not an fp32 value" % tag
    torch.cuda.synchronize()
    if not torch.equal(got, exp):
        bad = (got != exp).nonzero()
        idx = [tuple(int(v) for v in b) for b in bad[:6]]
        raise AssertionError("%s: %d of %d elements differ, first %s: got %s want %s" % (
            tag, bad.shape[0], got.numel(), idx, [float(got[i]) for i in idx], [float(exp[i]) for i in idx]))


def _real(tag, launcher, got, ref, cond, n):
    """|got - ref| <= gamma_n * cond (rigorous) and <= TAU[launcher] * cond (calibrated) at every element"""
    torch.cuda.synchronize()
    ratio = S.worst_ratio(got, ref, cond)
    tau = E.TAU[launcher]
    print("  RATIO %-8s %-26s worst |got-ref|/sum|a||b| %.3e  tau %s  gamma_%d %.3e" % (
        launcher, tag, ratio, "%.2e" % tau if tau else "-", n, E.gamma(n)))
    assert S.violations(got, ref, cond, E.gamma(n)) == 0, "%s: beyond the rigorous bound gamma_%d (ratio %.3e)" % (tag, n, ratio)
    assert tau is not None, "TAU[%s] is not calibrated" % launcher
    bad = S.violations(got, ref, cond, tau)
    assert bad == 0, "%s %s: %d elements beyond tau %.3e (worst ratio %.3e)" % (tag, launcher, bad, tau, ratio)


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.time()
    yield
    print("\n  test_simt_exact_gpu: wall time %.1f s" % (time.time() - t0))


def _ids(cases):
    return [c[0] for c in cases]


# ------------------------------------------------------------------------------------------------
# a. integer operands, bit for bit
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", FWD, ids=_ids(FWD))
def test_fwd_exact(case):
    """plain, accumulating into a non-zero y, and (flagged cases) with dropout: mask * fp32(exact) at every element"""
    _C, rt = lib()
    tag, g, flags = case
    x, w, _ = _operands(g, 11, True)
    ref, cond = S.fwd_bilinear(_d(x), _d(w), g), S.fwd_bilinear(_d(x).abs(), _d(w).abs(), g)
    y = _nan(g.B, g.Ho, g.Wo, g.Cout)
    _fwd(_C, rt, x, w, y, g)
    _exact(tag, y, ref, cond)
    y0 = ints((g.B, g.Ho, g.Wo, g.Cout), -4, 4, cpu_gen(12)).to(DEV)
    y = y0.clone()
    _fwd(_C, rt, x, w, y, g, acc=1)
    _exact(tag + " acc", y, _d(y0) + ref, cond + _d(y0).abs())
    keep = _drop_keep(flags)
    if keep:
        cfg, seed_t = drop_cfg(_C, keep, stream_id=5)
        mask = drop_mask(cfg, y.shape)
        y = _nan(*y.shape)
        _fwd(_C, rt, x, w, y, g, drop=cfg)
        torch.cuda.synchronize()
        frac = float((mask != 0).double().mean())
        assert abs(frac - keep) < 0.05, frac
        assert set(torch.unique(mask).tolist()) <= {0.0, float(torch.tensor(1.0 / keep, dtype=torch.float32))}
        _exact(tag + " dropout", y, _d(ref.float() * mask), cond)


@pytest.mark.parametrize("case", DGRAD, ids=_ids(DGRAD))
def test_dgrad_exact(case):
    """dx = conv^T(dy, w) with w transposed by pnp_weight_transpose, plain and accumulating into a non-zero dx"""
    _C, rt = lib()
    tag, g, _ = case
    _, w, dy = _operands(g, 21, True)
    wT = _transpose(_C, rt, w)
    ref, cond = S.dgrad_bilinear(_d(dy), _d(w), g), S.dgrad_bilinear(_d(dy).abs(), _d(w).abs(), g)
    dx = _nan(g.B, g.H, g.W, g.Cin)
    _dgrad(_C, rt, dy, wT, dx, g)
    _exact(tag, dx, ref, cond)
    dx0 = ints(dx.shape, -4, 4, cpu_gen(22)).to(DEV)
    dx = dx0.clone()
    _dgrad(_C, rt, dy, wT, dx, g, acc=1)
    _exact(tag + " acc", dx, _d(dx0) + ref, cond + _d(dx0).abs())


@pytest.mark.parametrize("case", WGRAD, ids=_ids(WGRAD))
def test_wgrad_exact(case):
    """dw += x (*) dy into a non-zero dw (the launcher always accumulates)"""
    _C, rt = lib()
    tag, g, _ = case
    x, _, dy = _operands(g, 31, True)
    ref, cond = S.wgrad_bilinear(_d(x), _d(dy), g), S.wgrad_bilinear(_d(x).abs(), _d(dy).abs(), g)
    dw0 = ints((g.kh, g.kw, g.Cin, g.Cout), -4, 4, cpu_gen(32)).to(DEV)
    dw = dw0.clone()
    _wgrad(_C, rt, x, dy, dw, g)
    print("  %s: %s" % (tag, E.simt_instance("wgrad", g)))
    _exact(tag, dw, _d(dw0) + ref, cond + _d(dw0).abs())


@pytest.mark.parametrize("taps,cin,cout", TRANSPOSE)
def test_weight_transpose_exact(taps, cin, cout):
    _C, rt = lib()
    w = torch.randn(taps, 1, cin, cout, generator=torch.Generator().manual_seed(taps + cin)).to(DEV)
    wT = _transpose(_C, rt, w)
    torch.cuda.synchronize()
    assert torch.equal(wT, w.transpose(2, 3))


def _three_kernel_bwd(_C, rt, dy, w, t):
    """the tail's input gradient as three launches: SIMT data gradient over the padded map, mirror-pad fold, inverse PS"""
    p = t.kh // 2
    H, W = t.a * t.r, t.b * t.r
    g = E.tail_conv_geom(t)
    dxp = _nan(t.B, H + 2 * p, W + 2 * p, t.G)
    _dgrad(_C, rt, dy, _transpose(_C, rt, w), dxp, g)
    dflat = _nan(t.B, H, W, t.G)
    _C.call("pnp_mirror_pad_bwd", _C.ptr(dxp), _C.ptr(dflat), t.B, H, W, t.G, p, rt.stream())
    dX = _nan(t.B, t.a, t.b, t.G * t.r * t.r)
    _C.call("pnp_phase_shift_bwd", _C.ptr(dflat), _C.ptr(dX), t.B, t.a, t.b, t.G, t.r, t.G, 0, 1, t.order_b1, rt.stream())
    return dX


@pytest.mark.parametrize("case", TAIL, ids=_ids(TAIL))
def test_tail_exact(case):
    """pnp_ps_mirror_conv_fwd / _bwd against the fp64 composition conv(mirror_pad(PS(X))) and its autograd; the backward also
    equals the three-kernel route bit for bit where that route runs (square kernel, 2p <= H, W)"""
    _C, rt = lib()
    tag, t, _ = case
    X, w, dy = _tail_operands(t, 41, True)
    H, W = t.a * t.r, t.b * t.r
    print("  %s: %s / %s (PNP_TAIL5=%s)" % (tag, E.simt_instance("tail_fwd", t)[0], E.simt_instance("tail_bwd", t)[0],
                                            os.environ.get("PNP_TAIL5", "default")))
    ref, cond = E.tail_fwd_ref(_d(X), _d(w), t)
    y = _nan(t.B, H, W, t.Cout)
    _tail(_C, rt, "pnp_ps_mirror_conv_fwd", X, w, y, t)
    _exact(tag + " fwd", y, ref, cond)
    ref, cond = E.tail_bwd_ref(_d(dy), _d(w), t)
    dX = _nan(*X.shape)
    _tail(_C, rt, "pnp_ps_mirror_conv_bwd", dy, w, dX, t)
    _exact(tag + " bwd", dX, ref, cond)
    p = t.kh // 2
    if t.kh == t.kw and 2 * p <= H and 2 * p <= W:
        three = _three_kernel_bwd(_C, rt, dy, w, t)
        torch.cuda.synchronize()
        assert torch.equal(three, dX), "%s: fused backward differs from the three-kernel route" % tag


# ------------------------------------------------------------------------------------------------
# b. randn operands: the calibrated per-element bound and gamma_n
# ------------------------------------------------------------------------------------------------
def _real_cases(cases):
    return [c for c in cases if "real" in c[2]]


@pytest.mark.parametrize("case", _real_cases(FWD), ids=_ids(_real_cases(FWD)))
def test_fwd_real(case):
    _C, rt = lib()
    tag, g, _ = case
    x, w, _ = _operands(g, 51, False)
    y = _nan(g.B, g.Ho, g.Wo, g.Cout)
    _fwd(_C, rt, x, w, y, g)
    ref, cond = S.fwd_bilinear(_d(x), _d(w), g), S.fwd_bilinear(_d(x).abs(), _d(w).abs(), g)
    _real(tag, "fwd", y, ref, cond, g.kh * g.kw * g.Cin)


@pytest.mark.parametrize("case", _real_cases(DGRAD), ids=_ids(_real_cases(DGRAD)))
def test_dgrad_real(case):
    _C, rt = lib()
    tag, g, _ = case
    _, w, dy = _operands(g, 52, False)
    dx = _nan(g.B, g.H, g.W, g.Cin)
    _dgrad(_C, rt, dy, _transpose(_C, rt, w), dx, g)
    ref, cond = S.dgrad_bilinear(_d(dy), _d(w), g), S.dgrad_bilinear(_d(dy).abs(), _d(w).abs(), g)
    _real(tag, "dgrad", dx, ref, cond, g.kh * g.kw * g.Cout)


@pytest.mark.parametrize("case", _real_cases(WGRAD), ids=_ids(_real_cases(WGRAD)))
def test_wgrad_real(case):
    _C, rt = lib()
    tag, g, _ = case
    x, _, dy = _operands(g, 53, False)
    dw0 = (torch.randn(g.kh, g.kw, g.Cin, g.Cout, generator=torch.Generator().manual_seed(54)) * 0.01).to(DEV)
    dw = dw0.clone()
    _wgrad(_C, rt, x, dy, dw, g)
    ref, cond = S.wgrad_bilinear(_d(x), _d(dy), g), S.wgrad_bilinear(_d(x).abs(), _d(dy).abs(), g)
    _real(tag, "wgrad", dw, _d(dw0) + ref, cond + _d(dw0).abs(), g.B * g.Ho * g.Wo + 1)


@pytest.mark.parametrize("case", _real_cases(TAIL), ids=_ids(_real_cases(TAIL)))
def test_tail_real(case):
    _C, rt = lib()
    tag, t, _ = case
    X, w, dy = _tail_operands(t, 55, False)
    y = _nan(t.B, t.a * t.r, t.b * t.r, t.Cout)
    _tail(_C, rt, "pnp_ps_mirror_conv_fwd", X, w, y, t)
    ref, cond = E.tail_fwd_ref(_d(X), _d(w), t)
    _real(tag, "tail_fwd", y, ref, cond, t.kh * t.kw * t.G)
    dX = _nan(*X.shape)
    _tail(_C, rt, "pnp_ps_mirror_conv_bwd", dy, w, dX, t)
    ref, cond = E.tail_bwd_ref(_d(dy), _d(w), t)
    # a border pixel sums the padded position itself and up to two reflections per axis: at most 9 * kh * kw * Cout products
    _real(tag, "tail_bwd", dX, ref, cond, 9 * t.kh * t.kw * t.Cout)


# ------------------------------------------------------------------------------------------------
# c. the kernels that ran are the ones the restatement names
# ------------------------------------------------------------------------------------------------
def test_launched_kernels_match_restatement():
    """one launch per entry of int_launches() under torch.profiler; the SIMT kernel each one ran, in launch order, is
    simt_instance() of its geometry (the operands are zero: only the dispatch matters here)"""
    from torch.profiler import ProfilerActivity, profile
    _C, rt = lib()
    plan = int_launches()
    want = [E.simt_instance(l, g, drop, acc)[0] for l, g, drop, acc in plan]
    cfg, seed_t = drop_cfg(_C, 0.5, stream_id=9)
    bufs = []
    for l, g, _, _ in plan:
        if l in ("tail_fwd", "tail_bwd"):
            t = g
            bufs.append(tuple(torch.zeros(s, device=DEV) for s in ((t.B, t.a, t.b, t.G * t.r * t.r), (t.kh, t.kw, t.G, t.Cout),
                                                                   (t.B, t.a * t.r, t.b * t.r, t.Cout))))
        else:
            bufs.append(tuple(torch.zeros(s, device=DEV) for s in ((g.B, g.H, g.W, g.Cin), (g.kh, g.kw, g.Cin, g.Cout),
                                                                   (g.B, g.Ho, g.Wo, g.Cout), (g.kh, g.kw, g.Cout, g.Cin))))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for (l, g, drop, acc), b in zip(plan, bufs):
            if l == "fwd":
                _fwd(_C, rt, b[0], b[1], b[2], g, drop=cfg if drop else None, acc=acc)
            elif l == "dgrad":
                _dgrad(_C, rt, b[2], b[3], b[0], g, acc=acc)
            elif l == "wgrad":
                _wgrad(_C, rt, b[0], b[2], b[1], g)
            elif l == "tail_fwd":
                _tail(_C, rt, "pnp_ps_mirror_conv_fwd", b[0], b[1], b[2], g)
            else:
                _tail(_C, rt, "pnp_ps_mirror_conv_bwd", b[2], b[1], b[0], g)
            torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    kern.sort(key=lambda e: e.time_range.start)
    got = []
    for e in kern:
        inst = E.instances_in(e.name)
        got += sorted(inst)
    print("  %d launches, %d SIMT kernels recorded, %d distinct" % (len(plan), len(got), len(set(got))))
    assert len(got) == len(want), "recorded %d SIMT kernels for %d launches" % (len(got), len(want))
    bad = [(i, plan[i][0], w, g) for i, (w, g) in enumerate(zip(want, got)) if w != g]
    assert not bad, bad[:5]


# ------------------------------------------------------------------------------------------------
# d. the decline contract
# ------------------------------------------------------------------------------------------------
_G = conv(2, 16, 16, 8, 16, 3)
_T = TailGeom(2, 4, 4, 8, 4, 5, 5, 5, 0)

# (id, launcher, geometry, null operand index or None, expected code)
DECLINE = [
    ("fwd_stride0", "fwd", _G._replace(stride=0), None, BAD_ARG),
    ("fwd_null_x", "fwd", _G, 0, BAD_ARG),
    ("fwd_null_y", "fwd", _G, 2, BAD_ARG),
    ("dgrad_pad_neg", "dgrad", _G._replace(pad_t=-1), None, BAD_ARG),
    ("dgrad_null_w", "dgrad", _G, 1, BAD_ARG),
    ("wgrad_cout0", "wgrad", _G._replace(Cout=0), None, BAD_ARG),
    ("wgrad_null_dy", "wgrad", _G, 1, BAD_ARG),
    ("transpose_taps0", "transpose", _G._replace(kh=0), None, BAD_ARG),
    ("tail_fwd_G0", "tail_fwd", _T._replace(G=0), None, BAD_ARG),
    ("tail_bwd_null_w", "tail_bwd", _T, 1, BAD_ARG),
    ("tail_fwd_even_k", "tail_fwd", _T._replace(kh=4, kw=4), None, "unsupported"),
    ("tail_bwd_even_k", "tail_bwd", _T._replace(kw=2), None, "unsupported"),
    ("tail_fwd_k7", "tail_fwd", _T._replace(kh=7, kw=7), None, "unsupported"),
    ("tail_fwd_cout6", "tail_fwd", _T._replace(Cout=6), None, "unsupported"),
    ("tail_bwd_cout4_k3", "tail_bwd", _T._replace(Cout=4, kh=3, kw=3), None, "unsupported"),
    ("tail_fwd_pad_beyond_map", "tail_fwd", _T._replace(a=1, r=1), None, "unsupported"),     # kh / 2 = 2 > a * r = 1
    ("tail_bwd_pad_beyond_map", "tail_bwd", _T._replace(b=1, r=1, kh=3), None, "unsupported"),
]


@pytest.mark.parametrize("case", DECLINE, ids=_ids(DECLINE))
def test_declined_launches_leave_output_untouched(case):
    _C, rt = lib()
    _, launcher, g, null, code = case
    src = torch.zeros(4096, device=DEV)
    wt = torch.zeros(4096, device=DEV)
    out = torch.full((4096,), 1234.5, device=DEV)
    ops = [src, wt, out]
    if null is not None:
        ops[null] = None
    a, b, c = ops
    raises = pytest.raises(_C.Unsupported) if code == "unsupported" else pytest.raises(RuntimeError, match=r"\[%d\]" % code)
    with raises:
        if launcher == "fwd":
            _fwd(_C, rt, a, b, c, g)
        elif launcher == "dgrad":
            _dgrad(_C, rt, a, b, c, g)
        elif launcher == "wgrad":
            _wgrad(_C, rt, a, b, c, g)
        elif launcher == "transpose":
            _C.call("pnp_weight_transpose", _C.ptr(a), _C.ptr(c), g.kh * g.kw, g.Cin, g.Cout, rt.stream())
        else:
            _tail(_C, rt, "pnp_ps_mirror_conv_fwd" if launcher == "tail_fwd" else "pnp_ps_mirror_conv_bwd", a, b, c, g)
    torch.cuda.synchronize()
    assert bool((out == 1234.5).all()), "a declined launch wrote its output"


# ------------------------------------------------------------------------------------------------
# e. PNP_TAIL5 variants, each in its own process
# ------------------------------------------------------------------------------------------------
@pytest.mark.timeout(300)
@pytest.mark.parametrize("mode", ["0", "1", "2"])
def test_tail5_switch(mode):
    """PNP_TAIL5 bit 0 = register-tiled 5x5 forward, bit 1 = register-tiled 5x5 backward; every 5x5 tail case, integer and
    real, through the other kernel of each pair"""
    passed, lines = rerun({"PNP_TAIL5": mode}, __file__, "(tail_exact or tail_real) and k5_", flags=("-s",))
    print("\n".join(l for l in lines if "RATIO" in l or "PNP_TAIL5" in l))
    k5 = [c for c in TAIL if c[0].startswith("k5_")]
    assert passed == len(k5) + len(_real_cases(k5)), passed
