"""The SIMT checks of tests/test_simt_exact_gpu.py without a GPU: its case tables reach every SIMT kernel instantiation in the
built library (restated dispatch, nm), the tail reference is the oracle's composition, and the committed TAU rejects the
reference of each plausible kernel bug at the GPU file's real-valued shapes -- so a kernel that passes there cannot have one."""
import os
import shutil
import subprocess

import pytest
import torch

from oracle import bf16_split as S
from oracle import simt_exact as E
from oracle import tf14_torch as T
from oracle.simt_exact import TailGeom
from tests.test_simt_exact_gpu import DGRAD, FWD, TAIL, WGRAD, _operands, _tail_operands, conv, int_launches

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "medical-cross-modality-domain-adaptation_b200", "libpnp_b200.so")


# ------------------------------------------------------------------------------------------------
# dispatch restatement and coverage
# ------------------------------------------------------------------------------------------------
def library_instances():
    if not os.path.exists(LIB):
        pytest.fail("libpnp_b200.so is not built (run __graft_entry__.build())")
    nm = shutil.which("nm")
    assert nm, "nm (binutils) is needed to list the library's kernels"
    out = subprocess.run([nm, "-C", LIB], capture_output=True, text=True, check=True).stdout
    return E.instances_in(out)


def test_case_tables_reach_every_instantiation(monkeypatch):
    """the union of the instantiations the GPU file's launches select (default PNP_TAIL5) is exactly the set of SIMT kernel
    instantiations in the library: a new instantiation without a case fails here"""
    monkeypatch.delenv("PNP_TAIL5", raising=False)
    lib = library_instances()
    assert len(lib) >= 41, sorted(lib)
    reached = {E.simt_instance(l, g, drop, acc)[0] for l, g, drop, acc in int_launches()}
    assert not reached - lib, "restated instantiations missing from the library: %s" % sorted(reached - lib)
    assert not lib - reached, "instantiations no case reaches: %s" % sorted(lib - reached)


def test_wgrad_cases_cover_one_and_many_splits():
    splits = {tag: E.simt_instance("wgrad", g)[1] for tag, g, _ in WGRAD}
    print(splits)
    assert min(splits.values()) == 1 and max(splits.values()) > 1
    assert splits["c16_o12_1split"] == 1 and splits["c3_o16_128splits"] == 128


def test_dgrad_cases_cover_both_row_orders():
    """strided data gradients in the phase-major row order and in its fallback, for both reasons it falls back"""
    orders = {}
    for tag, g, _ in DGRAD:
        kern = E.simt_instance("dgrad", g)[0]
        orders[tag] = E.dgrad_phase_rows(g, kern)
    phased = [t for t, pr in orders.items() if pr]
    assert {"o32_c16_s2_phase", "o32_c64_s2_phase", "o32_c32_k5s4_phase", "o16_c16_k3s4_phase"} <= set(phased), orders
    odd = [t for t, g, _ in DGRAD if g.stride > 1 and (g.H % g.stride or g.W % g.stride)]
    ragged = [t for t, g, _ in DGRAD if g.stride > 1 and not orders[t] and not (g.H % g.stride or g.W % g.stride)]
    assert odd and ragged, orders


def test_fwd_cases_cover_dropout_store_paths():
    """dropout on the float4 store (Cout % 4 == 0) and on the per-element store, at keep 0.5 and 0.75"""
    drops = [(g.Cout % 4 == 0, "drop50" in f) for _, g, f in FWD if f & {"drop50", "drop75"}]
    assert {(True, True), (True, False), (False, True), (False, False)} <= set(drops)


@pytest.mark.parametrize("mode,fwd5,bwd5", [("0", False, False), ("1", True, False), ("2", False, True), ("3", True, True),
                                            (None, True, True)])
def test_tail5_mode_selects_kernels(monkeypatch, mode, fwd5, bwd5):
    if mode is None:
        monkeypatch.delenv("PNP_TAIL5", raising=False)
    else:
        monkeypatch.setenv("PNP_TAIL5", mode)
    t = TailGeom(2, 4, 4, 40, 8, 5, 5, 5, 0)
    assert E.simt_instance("tail_fwd", t)[0] == ("ps_mirror_conv5_kernel<5>" if fwd5 else "ps_mirror_conv_kernel<5>")
    assert E.simt_instance("tail_bwd", t)[0] == ("ps_mirror_conv5_bwd_kernel<5>" if bwd5 else "ps_mirror_conv_bwd_kernel<5>")
    assert E.simt_instance("tail_fwd", t._replace(kh=3, kw=3, Cout=8))[0] == "ps_mirror_conv_kernel<8>"


def test_restatement_known_answers():
    """hand-derived selections: the 128x128 tile needs 2 x 132 tiles, the few-output kernel only the plain stride-1 forward"""
    assert E.simt_instance("fwd", conv(1, 192, 192, 16, 128, 3))[0] == "conv_gather_kernel<128,128,16,8,8,4,false>"
    assert E.simt_instance("fwd", conv(1, 180, 180, 16, 128, 3))[0] == "conv_gather_kernel<128,64,16,8,4,4,false>"   # 254 tiles
    assert E.simt_instance("fwd", conv(2, 64, 64, 40, 5, 5))[0] == "conv_few_out_kernel<5>"
    assert E.simt_instance("fwd", conv(2, 64, 64, 40, 5, 5), accumulate=1)[0] == "conv_gather_kernel<1024,8,8,4,8,4,false>"
    assert E.simt_instance("fwd", conv(2, 64, 64, 40, 5, 5), drop=True)[0] == "conv_gather_kernel<1024,8,8,4,8,4,false>"
    assert E.simt_instance("dgrad", conv(2, 64, 64, 40, 5, 5))[0] == "conv_gather_kernel<128,64,16,8,4,1,true>"
    # 8 tiles of 128 KK: 99 splits wanted, 8192 / 99 -> 83 pixels, rounded up to 96 (6 reduction blocks) -> 86 splits
    assert E.simt_instance("wgrad", conv(2, 64, 64, 40, 5, 5)) == ("conv_wgrad_kernel<128,8,16,4,1,4>", 86)


# ------------------------------------------------------------------------------------------------
# the tail reference
# ------------------------------------------------------------------------------------------------
def test_ps_and_mirror_pad_match_the_oracle():
    gen = torch.Generator().manual_seed(1)
    for B, order in ((2, 0), (1, 1), (3, 0)):
        X = torch.randn(B, 3, 4, 5 * 9, generator=gen, dtype=torch.float64)
        assert torch.equal(E.ps(X, 3, order), T.PS(X, 3, 5, B))
    x = torch.randn(2, 5, 7, 3, generator=gen, dtype=torch.float64)
    for p in (1, 2, 5):
        assert torch.equal(E.mirror_pad(x, p, p), T.symmetric_pad(x, p))
    assert torch.equal(E.mirror_pad(x, 1, 2)[:, :, 1:-1], T.symmetric_pad(x, 1))


@pytest.mark.parametrize("t", [TailGeom(2, 3, 2, 5, 4, 5, 5, 5, 0), TailGeom(1, 1, 3, 3, 2, 5, 5, 8, 1),
                               TailGeom(2, 2, 3, 3, 2, 3, 5, 5, 0), TailGeom(1, 1, 2, 2, 1, 1, 1, 8, 1)])
def test_tail_reference_is_the_composition(t):
    """tail_fwd is tf14_torch's conv2d(PS(X), w, padding='SYMMETRIC'); the autograd backward equals the written-out fold"""
    gen = torch.Generator().manual_seed(2)
    X = torch.randn(t.B, t.a, t.b, t.G * t.r * t.r, generator=gen, dtype=torch.float64)
    w = torch.randn(t.kh, t.kw, t.G, t.Cout, generator=gen, dtype=torch.float64)
    y = E.tail_fwd(X, w, t)
    if t.kh == t.kw and (t.B >= 2) != bool(t.order_b1):
        assert torch.allclose(y, T.conv2d_raw(T.PS(X, t.r, t.G, t.B), w, padding="SYMMETRIC"), atol=1e-12)
    dy = torch.randn(y.shape, generator=gen, dtype=torch.float64)
    ref, cond = E.tail_bwd_ref(dy, w, t)
    assert torch.allclose(E.tail_bwd_explicit(dy, w, t), ref, atol=1e-12)
    assert bool((cond >= ref.abs() - 1e-12).all())


# ------------------------------------------------------------------------------------------------
# the power of TAU at the GPU file's real-valued shapes
# ------------------------------------------------------------------------------------------------
def _round_tf32(t):
    """round fp32 values to TF32 (10 explicit mantissa bits), to nearest even"""
    u = t.float().contiguous().view(torch.int32).to(torch.int64)
    u = (u + 0xFFF + ((u >> 13) & 1)) & ~0x1FFF
    return u.to(torch.int32).view(torch.float32)


def _round_bf16(t):
    return t.float().to(torch.bfloat16).float()


def _reject(launcher, tag, bug, ref, cond):
    tau = E.TAU[launcher]
    assert tau is not None, "TAU[%s] is not calibrated" % launcher
    ok = S.violations(ref.float().double(), ref, cond, tau)           # the fp32 rounding of the right answer passes
    n = S.violations(bug, ref, cond, tau)
    print("  %-8s %-28s %7d of %8d elements rejected, worst ratio %.2e vs tau %.2e" % (
        launcher, tag, n, ref.numel(), S.worst_ratio(bug, ref, cond), tau))
    assert ok == 0
    assert n > 0, "%s: tau %.2e cannot see this bug" % (tag, tau)


def _real(cases):
    return [c for c in cases if "real" in c[2]]


def _d(t):
    return t.double()


@pytest.mark.parametrize("rnd", [_round_tf32, _round_bf16], ids=["tf32", "bf16"])
def test_tau_rejects_reduced_precision_operands(rnd):
    """a kernel that multiplied TF32- or bf16-rounded operands (fp32 accumulation) fails TAU on every real-valued shape"""
    for tag, g, _ in _real(FWD):
        x, w, _ = _operands(g, 51, False, dev="cpu")
        ref, cond = S.fwd_bilinear(_d(x), _d(w), g), S.fwd_bilinear(_d(x).abs(), _d(w).abs(), g)
        _reject("fwd", tag, S.fwd_bilinear(_d(rnd(x)), _d(rnd(w)), g), ref, cond)
    for tag, g, _ in _real(DGRAD):
        _, w, dy = _operands(g, 52, False, dev="cpu")
        ref, cond = S.dgrad_bilinear(_d(dy), _d(w), g), S.dgrad_bilinear(_d(dy).abs(), _d(w).abs(), g)
        _reject("dgrad", tag, S.dgrad_bilinear(_d(rnd(dy)), _d(rnd(w)), g), ref, cond)
    for tag, g, _ in _real(WGRAD):
        x, _, dy = _operands(g, 53, False, dev="cpu")
        ref, cond = S.wgrad_bilinear(_d(x), _d(dy), g), S.wgrad_bilinear(_d(x).abs(), _d(dy).abs(), g)
        _reject("wgrad", tag, S.wgrad_bilinear(_d(rnd(x)), _d(rnd(dy)), g), ref, cond)
    for tag, t, _ in _real(TAIL):
        X, w, dy = _tail_operands(t, 55, False, dev="cpu")
        ref, cond = E.tail_fwd_ref(_d(X), _d(w), t)
        _reject("tail_fwd", tag, E.tail_fwd(_d(rnd(X)), _d(rnd(w)), t), ref, cond)
        ref, cond = E.tail_bwd_ref(_d(dy), _d(w), t)
        _reject("tail_bwd", tag, E.tail_bwd_explicit(_d(rnd(dy)), _d(rnd(w)), t), ref, cond)


def test_tau_rejects_a_dropped_border_tap():
    """one tap skipped on the first output row only (fwd, tail fwd), on the last dx row only (dgrad), or for the pixels of the
    first dy row only (wgrad)"""
    for tag, g, _ in _real(FWD):
        x, w, _ = _operands(g, 51, False, dev="cpu")
        x, w = _d(x), _d(w)
        ref, cond = S.fwd_bilinear(x, w, g), S.fwd_bilinear(x.abs(), w.abs(), g)
        bug = ref.clone()
        bug[:, 0] -= S.fwd_bilinear(x, w, g, taps={g.kh * g.kw - 1})[:, 0]
        _reject("fwd", tag, bug, ref, cond)
    for tag, g, _ in _real(DGRAD):
        _, w, dy = _operands(g, 52, False, dev="cpu")
        dy, w = _d(dy), _d(w)
        ref, cond = S.dgrad_bilinear(dy, w, g), S.dgrad_bilinear(dy.abs(), w.abs(), g)
        bug = ref.clone()
        part = S.dgrad_bilinear(dy, w, g, taps={0})
        row = max(i for i in range(g.H) if bool(part[:, i].abs().sum() > 0))
        bug[:, row] -= part[:, row]
        _reject("dgrad", tag, bug, ref, cond)
    for tag, g, _ in _real(WGRAD):
        x, _, dy = _operands(g, 53, False, dev="cpu")
        x, dy = _d(x), _d(dy)
        ref, cond = S.wgrad_bilinear(x, dy, g), S.wgrad_bilinear(x.abs(), dy.abs(), g)
        row0 = torch.zeros_like(dy)
        row0[:, 0] = dy[:, 0]
        _reject("wgrad", tag, ref - S.wgrad_bilinear(x, row0, g, taps={g.kh * g.kw - 1}), ref, cond)
    for tag, t, _ in _real(TAIL):
        X, w, _ = _tail_operands(t, 55, False, dev="cpu")
        X, w = _d(X), _d(w)
        ref, cond = E.tail_fwd_ref(X, w, t)
        gp = E.tail_conv_geom(t)
        padded = E.mirror_pad(E.ps(X, t.r, t.order_b1), t.kh // 2, t.kw // 2)
        bug = ref.clone()
        bug[:, 0] -= S.fwd_bilinear(padded, w, gp, taps={0})[:, 0]
        _reject("tail_fwd", tag, bug, ref, cond)


@pytest.mark.parametrize("edge", ["top", "bottom", "left", "right"])
def test_tau_rejects_a_missing_mirror_fold(edge):
    """the tail backward without the fold of the reflected rows / columns of one edge"""
    for tag, t, _ in _real(TAIL):
        if t.kh == 1 and edge in ("top", "bottom") or t.kw == 1 and edge in ("left", "right"):
            continue
        _, w, dy = _tail_operands(t, 55, False, dev="cpu")
        ref, cond = E.tail_bwd_ref(_d(dy), _d(w), t)
        _reject("tail_bwd", tag + " " + edge, E.tail_bwd_explicit(_d(dy), _d(w), t, drop_fold=edge), ref, cond)


def test_tau_values_are_calibrated():
    """every launcher has a TAU, far below the error of a TF32 product (2^-11) and above one fp32 rounding"""
    for k, v in E.TAU.items():
        assert v is not None and 2.0 ** -24 < v < 2.0 ** -14, (k, v)
