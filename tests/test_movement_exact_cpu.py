"""The checks of tests/test_movement_exact_gpu.py without a GPU: its case tables reach every launch regime of the restated
configuration, each reference of oracle/movement_exact.py equals an independent form (the oracle's numpy loops, np.pad, the
literal emulation of ops.py, the disc-input graph pinned to the executed reference lines, the label decomposition, torch.cat),
each plausible kernel bug changes the reference output on the GPU file's operands, and every kernel entry point of the header
is named by a C-ABI reference test."""
import glob
import os
import re

import numpy as np
import pytest
import torch

from oracle import movement_exact as M
from oracle import pnp_graphs as PG
from oracle import tf14_numpy as N
from oracle import tf14_torch as T
from tests import test_movement_exact_gpu as G
from tests.cabi import sentinel

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPU = "cpu"


def small(cases):
    """the cases whose operands are cheap on the host"""
    return [c for c in cases if "cap" not in c[0]]


def ndiff(a, b):
    """elements whose fp32 bit patterns differ"""
    a, b = a.float().contiguous(), b.float().contiguous()
    assert a.shape == b.shape
    return int((a.view(torch.int32) != b.view(torch.int32)).sum())


# ------------------------------------------------------------------------------------------------
# launch configuration and case tables
# ------------------------------------------------------------------------------------------------
def _regimes(launches):
    """(capped with >= 2 grid-stride iterations, single partial CTA) reached by a list of launches"""
    return any(l.capped and l.iters >= 2 for l in launches), any(l.single_partial for l in launches)


def test_every_launcher_reaches_the_cap_and_a_single_partial_cta():
    mp = [M.maxpool2_launch(B, H, W, C) for _, B, H, W, C, _ in G.MAXPOOL2_CASES]
    table = {
        "maxpool2 V=4": [l for V, l in mp if V == 4],
        "maxpool2 V=1": [l for V, l in mp if V == 1],
        "avgpool2": [M.avgpool2_launch(B, H, W, C) for _, B, H, W, C, _ in G.MAXPOOL2_CASES],
        "pool_fwd": [M.pool_launch(B, H, W, C, n, False) for _, B, H, W, C, n, _ in G.POOL_CASES],
        "pool_bwd": [M.pool_launch(B, H, W, C, n, True) for _, B, H, W, C, n, _ in G.POOL_CASES],
        "mirror_pad_fwd": [M.mirror_pad_launch(B, H, W, C, p, False) for _, B, H, W, C, p in G.MIRROR_CASES],
        "mirror_pad_bwd": [M.mirror_pad_launch(B, H, W, C, p, True) for _, B, H, W, C, p in G.MIRROR_CASES],
        "phase_shift": [M.phase_shift_launch(c[1], c[2], c[3], c[4], c[5]) for c in G.PS_CASES],
        "disc_input generic": [l for p, l in (M.disc_input_launch(*c[1:]) for c in G.DISC_CASES) if p == "generic"],
        "logits_argmax_concat": [M.pixel_launch(c[1]) for c in G.LAC_CASES],
        "channel_slice": [M.channel_slice_launch(c[1], c[4]) for c in G.SLICE_CASES],
        "crop_concat_fwd": [M.crop_concat_launch(*c[1:8], False) for c in G.CAT_CASES],
        "crop_concat_bwd": [M.crop_concat_launch(*c[1:8], True, c[8], c[9]) for c in G.CAT_CASES],
        "one_hot": [M.pixel_launch(c[1]) for c in G.ONE_HOT_CASES],
        "pixel_softmax2": [M.pixel_launch(c[1]) for c in G.PS2_CASES],
        "cross_entropy_bwd": [M.ce_bwd_launch(n) for n in G.CE_N],
        "cross_entropy_acc": [M.ce_acc_launch(n) for n in G.CE_N],
        "fill": [M.Launch(f.grid, f.capped, f.iters, f.grid == 1 and n // 4 < 1024) for n, f in ((n, M.fill_launch(n))
                                                                                               for n in G.FILL_N)],
    }
    missing = []
    for name, launches in table.items():
        cap, one = _regimes(launches)
        print("  %-22s cap with >= 2 iterations %d, single partial CTA %d" % (name, cap, one))
        if not (cap and one):
            missing.append(name)
    assert not missing, missing
    # the accumulating threads of the capped cross-entropy case hold more than one fp32 partial
    assert max(M.ce_acc_launch(n).iters for n in G.CE_N) > M.CE_FLUSH


def test_case_tables_reach_every_dispatch_path_and_edge():
    assert {C for *_, C, _ in G.MAXPOOL2_CASES} >= {4, 16, 64, 1, 3, 6}
    assert {M.maxpool2_launch(*c[1:5])[0] for c in G.MAXPOOL2_CASES} == {1, 4}
    assert any(c[2] == 2 for c in G.MAXPOOL2_CASES) and any(c[3] == 2 for c in G.MAXPOOL2_CASES)
    assert {c[5] for c in G.POOL_CASES} >= {1, 2, 3, 4, 5, 8}
    geoms = [M.pool_geom(c[2], c[3], c[5]) for c in G.POOL_CASES]
    assert any((Ho * c[5] - c[2]) % 2 for c, (Ho, Wo, _, _) in zip(G.POOL_CASES, geoms))       # asymmetric SAME padding
    assert any(c[5] > c[2] and c[5] > c[3] for c in G.POOL_CASES)
    assert any(c[2] % 2 and c[3] % 2 for c in G.POOL_CASES) and any(2 in (c[2], c[3]) for c in G.POOL_CASES)
    kinds = {c[-1] for c in G.POOL_CASES} | {c[-1] for c in G.MAXPOOL2_CASES}
    assert kinds >= {"ints", "const", "inf", "neginf"}
    # mirror pad: every p, p = H, and backward cases with H < 2p <= 2H
    assert {c[5] for c in G.MIRROR_CASES} >= {0, 1, 2, 3}
    assert any(c[5] == c[2] for c in G.MIRROR_CASES)
    assert {(c[2], c[3], c[5]) for c in G.MIRROR_CASES} >= {(3, 5, 2), (1, 4, 1), (2, 2, 2)}
    assert all(c[4] % 2 for c in G.MIRROR_CASES) and any(c[2] != c[3] for c in G.MIRROR_CASES)
    # phase shift
    assert {c[5] for c in G.PS_CASES} >= {1, 2, 4, 8} and {c[9] for c in G.PS_CASES} == {0, 1}
    assert {c[4] for c in G.PS_CASES} >= {1, 2, 5} and {c[8] for c in G.PS_CASES} >= {1, 3}
    assert all(c[7] > 0 and c[6] > c[7] + c[8] * c[4] for c in G.PS_CASES)
    # discriminator input: the real plan on the r8 path, every ragged width, every generic-kernel trigger, NC 1 and 8, Ctot 64
    paths = {c[0]: M.disc_input_launch(*c[1:])[0] for c in G.DISC_CASES}
    real = [c for c in G.DISC_CASES if c[1:] == (8, 32, 32, 8, 0, (2, 4, 8, 8), (3, 1, 1, 1), 5)]
    assert real and paths[real[0][0]] == "r8" and M.disc_ctot(*real[0][6:]) == 32
    assert {c[3] % 4 for c in G.DISC_CASES if paths[c[0]] == "r8"} == {0, 1, 2, 3}
    generic = [c for c in G.DISC_CASES if paths[c[0]] == "generic"]
    assert any(c[5] for c in generic) and any(c[4] != 8 for c in generic)
    assert any(c[4] == 8 and not c[5] and M.disc_lines(c[6], c[7]) == 33 for c in generic)
    assert {c[8] for c in G.DISC_CASES} >= {1, 8} and 64 in {M.disc_ctot(*c[6:]) for c in G.DISC_CASES}
    assert all(M.disc_ctot(*c[6:]) % 4 == 0 and M.disc_ctot(*c[6:]) <= 64 for c in G.DISC_CASES)
    # slice / concat / one-hot / fill / softmax
    assert {(c[3] == 0, c[3] + c[4] == c[2], c[5]) for c in G.SLICE_CASES} >= {(True, False, 0), (True, False, 1),
                                                                              (False, True, 0), (False, True, 1)}
    assert any((c[2] - c[5]) % 2 and (c[3] - c[6]) % 2 for c in G.CAT_CASES)
    assert any(c[4] == 1 for c in G.CAT_CASES) and any(c[7] == 1 for c in G.CAT_CASES)
    assert any(not c[8] for c in G.CAT_CASES) and any(not c[9] for c in G.CAT_CASES)
    assert {c[2] for c in G.ONE_HOT_CASES} >= {1, 5, 8, 12}
    assert {n % 4 for n in G.FILL_N} == {0, 1, 2, 3} and set(G.FILL_N) >= {1, 2, 3, 4, 5}
    assert any(M.fill_launch(n).capped and n % 4 == 3 for n in G.FILL_N)
    assert {c[2] for c in G.PS2_CASES} >= {1, 2, 5, 8}


def test_launch_known_answers():
    """hand-derived from the launchers: 256-thread CTAs, grid_for caps at 132 * 64"""
    assert M.maxpool2_launch(17, 256, 256, 64) == (4, M.Launch(8448, True, 3, False))      # 4456448 float4 items
    assert M.maxpool2_launch(1, 2, 2, 3) == (1, M.Launch(1, False, 1, True))
    assert M.mirror_pad_launch(1, 3, 5, 3, 2, False) == M.Launch(1, False, 1, True)        # 7 * 9 * 3 = 189 items
    assert M.disc_input_launch(8, 32, 32, 8, 0, (2, 4, 8, 8), (3, 1, 1, 1), 5) == ("r8", M.Launch(2048, False, 1, False))
    assert M.disc_input_launch(2, 2, 3, 8, 0, (9, 8, 8, 8), (1, 1, 1, 1), 2)[0] == "generic"
    assert M.disc_input_launch(2, 128, 128, 4, 0, (2, 4, 8, 8), (3, 1, 1, 1), 5) == ("generic", M.Launch(8448, True, 2, False))
    assert M.fill_launch(36000003) == M.FillLaunch(8448, True, 5, 3)
    assert M.fill_launch(3) == M.FillLaunch(1, False, 0, 3)
    assert M.ce_acc_launch(70000000) == M.Launch(8448, True, 33, False)
    assert M.pool_geom(9, 6, 4) == (3, 2, 1, 1) and M.pool_geom(13, 2, 8) == (2, 1, 1, 3)


def test_a_priori_bounds():
    """the bounds are a few fp32 roundings wide: gamma_{C+9} (C <= 8), gamma_4, gamma_3, gamma_34 + n 2^-53"""
    assert M.gamma(1) > M.U and abs(M.gamma(10) / (10 * M.U) - 1) < 1e-5
    assert M.ps2_bound(1) == M.gamma(10) and M.ps2_bound(8) == M.gamma(17) < 1.1e-6
    assert M.CE_DY_BOUND == M.gamma(4) and M.CE_DP_BOUND == M.gamma(3)
    assert M.gamma(34) < M.ce_acc_bound(70000000) < 2.1e-6


# ------------------------------------------------------------------------------------------------
# the references against independent forms
# ------------------------------------------------------------------------------------------------
def _pool_bwd_loops(x, dy, n):
    """MaxPoolGrad by loops: scan each window's valid elements in row-major order with '>' starting from -inf"""
    B, H, W, C = x.shape
    Ho, Wo, pt, pl = M.pool_geom(H, W, n)
    dx = np.zeros_like(x)
    for b in range(B):
        for oy in range(Ho):
            for ox in range(Wo):
                for c in range(C):
                    best, arg = -np.inf, None
                    for yy in range(max(oy * n - pt, 0), min(oy * n - pt + n, H)):
                        for xx in range(max(ox * n - pl, 0), min(ox * n - pl + n, W)):
                            if arg is None or x[b, yy, xx, c] > best:
                                best, arg = x[b, yy, xx, c], (yy, xx)
                    dx[b, arg[0], arg[1], c] = dy[b, oy, ox, c]
    return dx


@pytest.mark.parametrize("case", small(G.POOL_CASES) + [("maxpool2 " + c[0],) + c[1:5] + (2, c[5]) for c in small(G.MAXPOOL2_CASES)],
                         ids=lambda c: c[0])
def test_pool_references_equal_the_numpy_loops(case):
    tag, B, H, W, C, n, kind = case
    x = G.operand(kind, (B, H, W, C), 1, CPU)
    xn = x.numpy().astype(np.float64)
    assert np.array_equal(M.pool_max_ref(x, n).numpy(), N.pool_same(xn, n))
    Ho, Wo, _, _ = M.pool_geom(H, W, n)
    dy = G.distinct((B, Ho, Wo, C), CPU)
    assert np.array_equal(M.pool_max_bwd_ref(x, dy, n).numpy(), _pool_bwd_loops(xn, dy.numpy().astype(np.float64), n))
    if kind in ("ints", "const"):
        y32, y64, _, cnt = M.pool_avg_ref(x, n)
        ref = N.pool_same(xn, n, avg=True)
        assert np.allclose(y64.numpy(), ref, rtol=0, atol=1e-15)
        assert np.array_equal(y32.numpy(), (N.pool_same(xn, n, avg=True) * cnt.numpy()).astype(np.float32) / cnt.numpy().astype(
            np.float32))
    if n == 2 and H % 2 == 0 and W % 2 == 0 and kind != "neginf":
        assert np.array_equal(M.pool_max_ref(x, 2).numpy(), N.max_pool2x2(x.numpy()))
    # the average backward is the adjoint of the average (sum over windows of dy * mean = sum of x * dx)
    dya = torch.randn(B, Ho, Wo, C, dtype=torch.float64)
    xa = torch.randn(B, H, W, C, dtype=torch.float64)
    lhs = float((M.pool_avg_ref(xa, n)[1] * dya).sum())
    rhs = float((xa * M.pool_avg_bwd_ref(dya, H, W, n)).sum())
    assert abs(lhs - rhs) <= 1e-12 * (abs(lhs) + 1)


def _np_adjoint(dy, fwd_index, shape):
    """dx = J^T dy of a pure gather y = x.flat[idx]: np.add.at of dy into the gathered positions"""
    dx = np.zeros(int(np.prod(shape)), dtype=np.float64)
    np.add.at(dx, fwd_index.reshape(-1), dy.reshape(-1).astype(np.float64))
    return dx.reshape(shape)


@pytest.mark.parametrize("case", small(G.MIRROR_CASES), ids=lambda c: c[0])
def test_mirror_pad_references_equal_np_pad(case):
    tag, B, H, W, C, p = case
    x = G.operand("randn", (B, H, W, C), 2, CPU)
    pad = [(0, 0), (p, p), (p, p), (0, 0)]
    assert np.array_equal(M.mirror_pad_ref(x, p).numpy(), np.pad(x.numpy(), pad, mode="symmetric"))
    assert np.array_equal(M.mirror_pad_ref(x, p).numpy(), N.symmetric_pad(x.numpy(), p))
    idx = np.pad(np.arange(B * H * W * C).reshape(B, H, W, C), pad, mode="symmetric")
    dy = G.small_ints((B, H + 2 * p, W + 2 * p, C), 3, dev=CPU)
    assert np.array_equal(M.mirror_pad_bwd_ref(dy, H, W, p)[0].numpy(), _np_adjoint(dy.numpy(), idx, (B, H, W, C)))
    cnt = M.mirror_pad_bwd_ref(dy, H, W, p)[2]
    assert int(cnt.max()) <= 9 and float(cnt.sum()) == (H + 2 * p) * (W + 2 * p)


@pytest.mark.parametrize("case", small(G.PS_CASES), ids=lambda c: c[0])
def test_phase_shift_references_equal_ops_literal(case):
    """PS_literal executes ops.py's reshape / transpose / split / concat sequence (pinned to the executed ops.py)"""
    tag, B, a, b, G_, r, Ctot, coff, ntile, o = case
    X, dout = G.ps_operands(case, CPU)
    if o and a != b:
        # ops.py's batch_size == 1 branch ends in a transpose of the two spatial axes: it is defined for square maps only (the
        # reference's are), and the closed form the kernels implement is its restriction to them
        b = a
        X = G.distinct((B, a, b, G_ * r * r), CPU)
        dout = G.small_ints((B, a * r, b * r, Ctot), 4, dev=CPU)
    assert (B == 1) == bool(o)
    # the literal emulation squeezes the unit sub-pixel axes of r = 1, where PS is the identity
    ps_lit = (lambda A: A) if r == 1 else (lambda A: N.PS_literal(A, r, G_, 1 if o else B))
    lit = ps_lit(X.numpy())
    assert np.array_equal(M.phase_shift_ref(X, r, G_, o).numpy(), lit)
    out = M.phase_shift_fwd_ref(X, torch.full((B, a * r, b * r, Ctot), -7.0), r, G_, coff, ntile, o)
    want = np.full((B, a * r, b * r, Ctot), -7.0, np.float32)
    want[..., coff:coff + ntile * G_] = np.tile(lit, (1, 1, 1, ntile))            # tf.tile, adversarial.py:326
    assert np.array_equal(out.numpy(), want)
    idx = ps_lit(np.arange(X.numel()).reshape(X.shape))
    d = sum(dout.numpy()[..., coff + t * G_:coff + (t + 1) * G_] for t in range(ntile))
    assert np.array_equal(M.phase_shift_bwd_ref(dout, r, G_, coff, ntile, o).numpy(), _np_adjoint(d, idx, tuple(X.shape)))


@pytest.mark.parametrize("B", [2, 1])
def test_disc_input_reference_equals_the_pinned_graph(B):
    """oracle.pnp_graphs.disc_input is pinned to the executed adversarial.py:320-335"""
    case = ("pin", B, 2, 3, 8, 1 if B == 1 else 0, (2, 4, 8, 8), (3, 1, 1, 1), 5)
    srcs, logits = G.disc_operands(case, CPU)
    got = M.disc_input_ref(srcs, (2, 4, 8, 8), (3, 1, 1, 1), logits, 8, 1 if B == 1 else 0)
    assert torch.equal(got, PG.disc_input(*srcs, logits, B))


def test_logits_argmax_slice_concat_one_hot_fill_references():
    g = torch.Generator().manual_seed(0)
    l = torch.randint(-1, 2, (500, 6), generator=g).float()
    out = M.logits_argmax_concat_ref(l, torch.full((500, 10), -9.0), 2)
    assert torch.equal(out[:, 2:8], l) and np.array_equal(out[:, 8].numpy(), np.argmax(l.numpy(), 1).astype(np.float32))
    assert bool((out[:, :2] == -9).all()) and bool((out[:, 9:] == -9).all())
    gg = torch.randn(40, 7, generator=g)
    o0 = torch.randn(40, 3, generator=g)
    assert torch.equal(M.channel_slice_ref(gg, 7, 4, 3, o0, 1), o0 + gg[:, 4:])
    assert torch.equal(M.channel_slice_ref(gg, 7, 0, 3, o0, 0), gg[:, :3])
    x1, x2 = torch.randn(2, 9, 8, 3, generator=g, dtype=torch.float64), torch.randn(2, 6, 5, 2, generator=g, dtype=torch.float64)
    assert torch.equal(M.crop_concat_fwd_ref(x1, x2), T.crop_and_concat(x1, x2))
    a1, a2 = x1.clone().requires_grad_(True), x2.clone().requires_grad_(True)
    dout = torch.randn(2, 6, 5, 5, generator=g, dtype=torch.float64)
    T.crop_and_concat(a1, a2).backward(dout)
    d1, d2 = M.crop_concat_bwd_ref(dout, 9, 8, 3)
    assert torch.equal(d1, a1.grad) and torch.equal(d2, a2.grad)
    for C in (1, 5, 8, 12):
        lab = G.one_hot_labels(3000, C, C, CPU)
        assert np.array_equal(M.one_hot_ref(lab, C).numpy(), N.label_decomp(C, lab.numpy()))
        assert int((M.one_hot_ref(lab, C).sum(1) == 0).sum()) == int(((lab < 0) | (lab >= C)).sum()) > 0
    buf = torch.full((12,), 5.0)
    assert torch.equal(M.fill_ref(buf, 1.0, 7), torch.tensor([1.0] * 7 + [5.0] * 5))


def test_transcendental_references():
    l = G.ps2_logits(1000, 5, 0, CPU)
    sp = M.ps2_special(l)
    assert int(sp.sum()) == len(range(0, 1000, 97)) + len(range(1, 1000, 89))
    ref = M.pixel_softmax2_ref(l[~sp])
    assert np.allclose(ref.numpy(), N.pixel_wise_softmax_2(l[~sp].numpy().astype(np.float64)[None, None]).reshape(-1, 5),
                       rtol=1e-15, atol=0)
    assert float(torch.tensor(-1e15, dtype=torch.float32)) == M.PS2_CLIPPED
    y, p = G.ce_operands(1000, 1, CPU)
    s, mag = M.cross_entropy_fwd_ref(y, p)
    yn, pn = y.numpy().astype(np.float64), p.numpy().astype(np.float64)
    lg = np.log(np.clip(pn, np.float32(1e-10), 1.0))
    assert abs(float(s) - float((yn * lg).sum())) <= 1e-12 * float(mag)
    dy, dp = M.cross_entropy_bwd_ref(y, p, 500.0, 1000)
    assert np.allclose(dy.numpy(), -0.5 * lg, rtol=1e-15, atol=0)
    inside = (pn >= np.float32(1e-10)) & (pn <= 1)
    assert np.array_equal(dp.numpy(), np.where(inside, -0.5 * yn / np.where(inside, pn, 1), 0.0))
    assert (~inside).sum() > 2 and bool((dy[p == 1] == 0).all())


# ------------------------------------------------------------------------------------------------
# negative controls: each plausible kernel bug changes the reference output on the GPU file's operands
# ------------------------------------------------------------------------------------------------
def _pool_inputs():
    for c in small(G.MAXPOOL2_CASES):
        tag, B, H, W, C, kind = c
        yield tag, G.operand(kind, (B, H, W, C), B + H + W + C, CPU), 2
    for c in small(G.POOL_CASES):
        tag, B, H, W, C, n, kind = c
        yield tag, G.operand(kind, (B, H, W, C), 7 * B + H + W + n, CPU), n


def _margin_pool_bwd(**bug):
    d = 0
    for tag, x, n in _pool_inputs():
        B, H, W, C = x.shape
        Ho, Wo, _, _ = M.pool_geom(H, W, n)
        dy = G.distinct((B, Ho, Wo, C), CPU)
        d += ndiff(M.pool_max_bwd_ref(x, dy, n, **bug), M.pool_max_bwd_ref(x, dy, n))
    return d


def _margin_pool_geom(avg, **bug):
    d = 0
    for c in small(G.POOL_CASES):
        tag, B, H, W, C, n, kind = c
        x = G.operand(kind, (B, H, W, C), 7 * B + H + W + n, CPU)
        if avg:
            if kind in ("ints", "const"):
                d += ndiff(M.pool_avg_ref(x, n, **bug)[0], M.pool_avg_ref(x, n)[0])
        else:
            Ho, Wo, _, _ = M.pool_geom(H, W, n)
            dy = G.distinct((B, Ho, Wo, C), CPU)
            d += ndiff(M.pool_max_ref(x, n, **bug), M.pool_max_ref(x, n))
            d += ndiff(M.pool_max_bwd_ref(x, dy, n, **bug), M.pool_max_bwd_ref(x, dy, n))
    return d


def _margin_mirror(bwd, **bug):
    d = 0
    for c in small(G.MIRROR_CASES):
        tag, B, H, W, C, p = c
        if bwd:
            dy = G.small_ints((B, H + 2 * p, W + 2 * p, C), 32 + p, dev=CPU)
            d += ndiff(M.mirror_pad_bwd_ref(dy, H, W, p, **bug)[0], M.mirror_pad_bwd_ref(dy, H, W, p)[0])
        elif p < H and p < W:          # REFLECT needs p < H, W
            x = G.operand("randn", (B, H, W, C), 31 + H * W, CPU)
            d += ndiff(M.mirror_pad_ref(x, p, **bug), M.mirror_pad_ref(x, p))
    return d


def _margin_ps(bwd, **bug):
    d = 0
    for c in small(G.PS_CASES):
        tag, B, a, b, G_, r, Ctot, coff, ntile, o = c
        X, dout = G.ps_operands(c, CPU)
        if bwd:
            d += ndiff(M.phase_shift_bwd_ref(dout, r, G_, coff, ntile, o, **bug), M.phase_shift_bwd_ref(dout, r, G_, coff, ntile, o))
        else:
            base = sentinel((B, a * r, b * r, Ctot), CPU)
            d += ndiff(M.phase_shift_fwd_ref(X, base, r, G_, coff, ntile, o, **bug), M.phase_shift_fwd_ref(X, base, r, G_, coff,
                                                                                                           ntile, o))
    return d


def _margin_disc(**bug):
    d = 0
    for c in small(G.DISC_CASES):
        srcs, logits = G.disc_operands(c, CPU)
        _, B, a, b, r, o, Gs, nts, NC = c
        d += ndiff(M.disc_input_ref(srcs, Gs, nts, logits, r, o, **bug), M.disc_input_ref(srcs, Gs, nts, logits, r, o))
    return d


def _margin_lac():
    d = 0
    for tag, P, C, Ctot, coff in small(G.LAC_CASES):
        logits = G.small_ints((P, C), P + C, -1, 1, CPU)
        base = sentinel((P, Ctot), CPU)
        d += ndiff(M.logits_argmax_concat_ref(logits, base, coff, last=True), M.logits_argmax_concat_ref(logits, base, coff))
    return d + _margin_disc(last=True)


def _margin_crop():
    d = 0
    for c in small(G.CAT_CASES):
        tag, B, H1, W1, C1, H2, W2, C2, _, _ = c
        x1 = G.operand("randn", (B, H1, W1, C1), H1 + W1, CPU)
        x2 = G.operand("randn", (B, H2, W2, C2), H2 + W2 + 1, CPU)
        dout = G.operand("randn", (B, H2, W2, C1 + C2), 5 + C1, CPU)
        d += ndiff(M.crop_concat_fwd_ref(x1, x2, round_up=True), M.crop_concat_fwd_ref(x1, x2))
        d += ndiff(M.crop_concat_bwd_ref(dout, H1, W1, C1, round_up=True)[0], M.crop_concat_bwd_ref(dout, H1, W1, C1)[0])
    return d


def _margin_slice():
    d = 0
    for tag, Mr, C, off, Cs, acc in small(G.SLICE_CASES):
        g = G.operand("randn", (Mr, C), Mr + C, CPU)
        out = G.operand("randn", (Mr, Cs), 3 * Mr + Cs, CPU) if acc else sentinel((Mr, Cs), CPU)
        d += ndiff(M.channel_slice_ref(g, C, off, Cs, out, acc, ignore_acc=True), M.channel_slice_ref(g, C, off, Cs, out, acc))
    return d


def _margin_one_hot():
    return sum(ndiff(M.one_hot_ref(l, C, clamp=True), M.one_hot_ref(l, C))
               for l, C in ((G.one_hot_labels(P, C, P + C, CPU), C) for _, P, C in small(G.ONE_HOT_CASES)))


def _margin_fill():
    return sum(ndiff(M.fill_ref(sentinel(n + 5, CPU), -3.25, n, drop_tail=True), M.fill_ref(sentinel(n + 5, CPU), -3.25, n))
               for n in G.FILL_N if n < 10 ** 6)


NEGATIVE_CONTROLS = {
    "last maximum instead of the first": lambda: _margin_pool_bwd(first=False),
    "column-major window order": lambda: _margin_pool_bwd(col_major=True),
    "pad_before rounded up": lambda: _margin_pool_geom(False, round_up=True) + _margin_pool_geom(True, round_up=True),
    "average over n^2 instead of the valid count": lambda: _margin_pool_geom(True, full_count=True),
    "REFLECT instead of SYMMETRIC": lambda: _margin_mirror(False, reflect=True),
    "mirror-pad backward drops the third preimage": lambda: _margin_mirror(True, drop_third=True),
    "sub-pixel orders swapped": lambda: _margin_ps(False, swap=True) + _margin_disc(swap=True),
    "phase-shift backward drops tiles 1..ntile-1": lambda: _margin_ps(True, drop_tiles=True),
    "coff ignored": lambda: _margin_ps(False, ignore_coff=True),
    "tile order [g0 g0 g0 g1 ...]": lambda: _margin_ps(False, blocked=True) + _margin_disc(blocked=True),
    "last index on argmax ties": _margin_lac,
    "crop offset rounded up": _margin_crop,
    "accumulate ignored": _margin_slice,
    "out-of-range labels clamped": _margin_one_hot,
    "fill tail dropped": _margin_fill,
}


@pytest.mark.parametrize("bug", list(NEGATIVE_CONTROLS), ids=[k.replace(" ", "_") for k in NEGATIVE_CONTROLS])
def test_negative_control(bug):
    margin = NEGATIVE_CONTROLS[bug]()
    print("  NEGATIVE CONTROL %-46s %d differing elements" % (bug, margin))
    assert margin >= 1


# ------------------------------------------------------------------------------------------------
# coverage guard
# ------------------------------------------------------------------------------------------------
HOST_ONLY = {"pnp_error_string", "pnp_version", "pnp_tc_available", "pnp_tc_last_config"}
C_ABI_TEST_FILES = ["test_conv_bn_epilogue_gpu.py", "test_image_summary_gpu.py", "test_surface_distance_gpu.py"]


def test_every_kernel_entry_point_has_a_c_abi_reference_test():
    with open(os.path.join(ROOT, "include", "pnp_b200.h")) as f:
        header = f.read()
    declared = set(re.findall(r"^\s*(?:int|const char\*)\s+(pnp_\w+)\s*\(", header, re.M))
    assert len(declared) > 50 and HOST_ONLY <= declared
    files = sorted(glob.glob(os.path.join(ROOT, "tests", "test_*_exact_gpu.py"))) + [os.path.join(ROOT, "tests", f)
                                                                                     for f in C_ABI_TEST_FILES]
    text = ""
    for p in files:
        with open(p) as f:
            text += f.read()
    missing = sorted(n for n in declared - HOST_ONLY if not re.search(r"\b%s\b" % n, text))
    assert not missing, missing
