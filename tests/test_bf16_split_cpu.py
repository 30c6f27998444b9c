"""The split-aware reference (oracle/bf16_split.py) without a GPU: split() is the device's round-to-nearest-even bf16 split bit
for bit, and the committed per-element tolerance TAU rejects the reference of each plausible tensor-core bug at the shapes of
tests/test_tc_split_exact_gpu.py -- so a kernel that passes there cannot have one of them."""
import numpy as np
import pytest
import torch

from oracle import bf16_split as S
from tests.cabi import expected_ksplit
from tests.test_tc_split_exact_gpu import CASES, edge_values, geom_of, operands

U32 = 2.0 ** -23


def rne_bits(x):
    """independent statement of fp32 -> bf16 round to nearest even on the bit pattern; NaN -> None"""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    nan = ((u & 0x7F800000) == 0x7F800000) & ((u & 0x007FFFFF) != 0)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF
    return r.astype(np.int64), nan


def bits_as_float(b):
    return (b.astype(np.uint32) << 16).view(np.float32)


def _expect(x):
    hi, hi_nan = rne_bits(x)
    with np.errstate(invalid="ignore", over="ignore"):
        rem = (x - np.where(hi_nan, np.float32(0), bits_as_float(hi))).astype(np.float32)
    lo, lo_nan = rne_bits(rem)
    return hi, hi_nan, lo, lo_nan | hi_nan


def _assert_split(x):
    hi, lo = S.split(torch.from_numpy(x))
    gh, gl = S.bits(hi).numpy(), S.bits(lo).numpy()
    eh, eh_nan, el, el_nan = _expect(x)
    gh_nan, gl_nan = np.isnan(hi.float().numpy()), np.isnan(lo.float().numpy())
    assert np.array_equal(gh_nan, eh_nan) and np.array_equal(gl_nan, el_nan)
    bad = (~eh_nan & (gh != eh)) | (~el_nan & (gl != el))
    assert not bad.any(), [(hex(int(v)), hex(int(a)), hex(int(b))) for v, a, b in
                           zip(x.view(np.uint32)[bad][:5], gh[bad][:5], gl[bad][:5])]


def test_split_edge_values_bit_exact():
    """+-0, smallest / largest denormals, exact ties with even and odd hi (normal and denormal), FLT_MAX and the values that
    round up to inf, +-inf, NaN"""
    x = edge_values().numpy()
    _assert_split(x)
    hi, lo = S.split(torch.from_numpy(x))
    hb = S.bits(hi).numpy()
    pat = x.view(np.uint32)
    expect = {0x00000000: 0x0000, 0x80000000: 0x8000, 0x00000001: 0x0000, 0x007FFFFF: 0x0080, 0x00008000: 0x0000,
              0x00018000: 0x0002, 0x3F808000: 0x3F80, 0x3F818000: 0x3F82, 0x7F7FFFFF: 0x7F80, 0x7F7F8000: 0x7F80,
              0x7F7F7FFF: 0x7F7F, 0xFF7FFFFF: 0xFF80, 0x7F800000: 0x7F80, 0xFF800000: 0xFF80}
    for p, h in expect.items():
        assert int(hb[list(pat).index(p)]) == h, hex(p)
    # denormals are kept, not flushed: bf16's smallest denormal 2^-133 is its own hi, and a small normal's lo is a denormal
    assert int(S.bits(S.split(torch.tensor([2.0 ** -133]))[0])[0]) == 0x0001
    lo_den = S.split(torch.tensor([2.0 ** -120 + 2.0 ** -130]))[1]
    assert int(S.bits(lo_den)[0]) == 0x0008


def test_split_random_bit_patterns():
    rng = np.random.RandomState(0)
    x = rng.randint(0, 2 ** 32, size=1 << 20, dtype=np.uint64).astype(np.uint32).view(np.float32)
    _assert_split(x)


def test_split_recomposes_to_17_bits():
    x = torch.randn(100000, generator=torch.Generator().manual_seed(5), dtype=torch.float32) * 1e3
    x[:2] = torch.tensor([0.0, -0.0])
    hi, lo = S.split(x)
    r = hi.double() + lo.double()
    assert bool(((r - x.double()).abs() <= 2.0 ** -17 * x.double().abs()).all())


# ------------------------------------------------------------------------------------------------
# negative controls: the reference of each bug is rejected by the committed TAU
# ------------------------------------------------------------------------------------------------
CASE = {c[0]: c for c in CASES}


def _prep(name, B=None, cin=None, cout=None):
    """split fp64 operands of a GPU-file case (optionally fewer images / channels: the per-element test only depends on the
    reduction depth, which is kept)"""
    g = geom_of(CASE[name])
    x, w, dy = operands(g, 101)
    if B is not None:
        g, x, dy = g._replace(B=B), x[:B], dy[:B]
    if cin is not None:
        g, x, w = g._replace(Cin=cin), x[..., :cin], w[:, :, :cin, :]
    if cout is not None:
        g, w, dy = g._replace(Cout=cout), w[..., :cout], dy[..., :cout]
    sp = lambda t: tuple(p.double() for p in S.split(t.contiguous()))  # noqa: E731
    return g, sp(x), sp(w), sp(dy)


def _reject(launcher, nterms, got, ref, cond, slack=None):
    tau = S.TAU[(launcher, nterms)]
    n = S.violations(got, ref, cond, tau, slack)
    ratio = S.worst_ratio(got, ref, cond, slack)
    ok = S.violations(ref.float().double(), ref, cond, tau, slack)      # the fp32 rounding of the right answer passes
    print("  %-6s nterms %d: %d of %d elements rejected, worst ratio %.2e vs tau %.2e" % (launcher, nterms, n, ref.numel(), ratio, tau))
    assert ok == 0
    assert n > 0, "tau %.2e cannot see this bug (worst ratio %.2e)" % (tau, ratio)


@pytest.mark.parametrize("nterms", [3, 1])
def test_missing_kblock_in_one_tile_is_rejected(nterms):
    """one (tap, 64-channel k-block) skipped by one 128-pixel output tile"""
    g, (xh, xl), (wh, wl), _ = _prep("g10_512x2560_sym", B=1, cout=128)
    ref, cond = S.fwd_ref(xh, xl, wh, wl, g, nterms)
    m = torch.zeros(g.Cin, dtype=torch.float64)
    m[64:128] = 1
    part, _ = S.fwd_ref(xh * m, xl * m, wh, wl, g, nterms, taps={4})
    bug = ref.clone()
    bug[0, 0:4] -= part[0, 0:4]            # the tile: 4 rows of 32 pixels
    _reject("fwd", nterms, bug, ref, cond)
    # the data gradient at K = 23040: tap 4, dy channels 0..63, one 3-row tile of the 34-wide dx
    g, _, (wh, wl), (dh, dl) = _prep("g10_512x2560_sym", B=1, cin=64)
    ref, cond = S.dgrad_ref(dh, dl, wh, wl, g, nterms)
    m = torch.zeros(g.Cout, dtype=torch.float64)
    m[:64] = 1
    part, _ = S.dgrad_ref(dh * m, dl * m, wh, wl, g, nterms, taps={4})
    bug = ref.clone()
    bug[0, 3:6] -= part[0, 3:6]
    _reject("dgrad", nterms, bug, ref, cond)


def test_missing_cross_term_is_rejected():
    """nterms 3 without a_lo * b_hi, at the deepest reductions of the model"""
    g, (xh, xl), (wh, wl), _ = _prep("g10_512x2560_sym", B=1, cout=128)
    ref, cond = S.fwd_ref(xh, xl, wh, wl, g, 3)
    bug, _ = S.split_terms(lambda a, b: S.fwd_bilinear(a, b, g), xh, xl, wh, wl, 3, cross=False)
    _reject("fwd", 3, bug, ref, cond)
    g, _, (wh, wl), (dh, dl) = _prep("g10_512x2560_sym", B=1, cin=64)
    ref, cond = S.dgrad_ref(dh, dl, wh, wl, g, 3)
    bug, _ = S.split_terms(lambda a, b: S.dgrad_bilinear(a, b, g), dh, dl, wh, wl, 3, cross=False)
    _reject("dgrad", 3, bug, ref, cond)
    g, (xh, xl), _, (dh, dl) = _prep("g10_512x2560_sym", cin=64, cout=128)
    ref, cond = S.wgrad_ref(xh, xl, dh, dl, g, 3)
    bug, _ = S.split_terms(lambda a, b: S.wgrad_bilinear(a, b, g), xh, xl, dh, dl, 3, cross=False)
    _reject("wgrad", 3, bug, ref, cond)


@pytest.mark.parametrize("name", ["g10_512x2560_sym", "64_12x20", "dil2_512_B5"])
def test_tap_moved_by_one_pixel_is_rejected(name):
    g, (xh, xl), (wh, wl), _ = _prep(name, B=1, cout=64)
    for nterms in (3, 1):
        ref, cond = S.fwd_ref(xh, xl, wh, wl, g, nterms)
        bug, _ = S.fwd_ref(xh, xl, wh, wl, g, nterms, shift={g.kh * g.kw - 1: (0, 1)})
        _reject("fwd", nterms, bug, ref, cond)


@pytest.mark.parametrize("name,cin", [("k5s4_512_B3", 64), ("16x32_k5s4", None), ("32x64_s2", None), ("64_7x9_s2", None)])
def test_missing_dgrad_phase_is_rejected(name, cin):
    g, _, (wh, wl), (dh, dl) = _prep(name, B=1, cin=cin)
    s = g.stride
    for nterms in (3, 1):
        ref, cond = S.dgrad_ref(dh, dl, wh, wl, g, nterms)
        for py, px in ((s - 1, s - 1), (0, 1)):
            assert S.dgrad_phase_taps(g, py, px), "every phase has taps"
            bug = ref.clone()
            bug[:, py::s, px::s, :] = 0
            _reject("dgrad", nterms, bug, ref, cond)


@pytest.mark.parametrize("name", ["64_12x20", "dil2_512_B5"])
def test_ignored_accumulate_is_rejected(name):
    g, (xh, xl), (wh, wl), (dh, dl) = _prep(name, B=1)
    gen = torch.Generator().manual_seed(7)
    for nterms in (3, 1):
        ref, cond = S.fwd_ref(xh, xl, wh, wl, g, nterms)
        y0 = torch.randn(ref.shape, generator=gen).double()
        _reject("fwd", nterms, ref, y0 + ref, cond, slack=2 * U32 * (y0.abs() + ref.abs()))
        ref, cond = S.dgrad_ref(dh, dl, wh, wl, g, nterms)
        d0 = torch.randn(ref.shape, generator=gen).double()
        _reject("dgrad", nterms, ref, d0 + ref, cond, slack=2 * U32 * (d0.abs() + ref.abs()))


def test_reference_matches_torch_convolution():
    """the tap-loop bilinear maps are the convolution, its input gradient and its weight gradient (strided, dilated, padded)"""
    for name in ("64_7x9_s2", "dil2_512_B5", "16x32_k5s4"):
        g, _, _, _ = _prep(name, B=1)
        gen = torch.Generator().manual_seed(3)
        x = torch.randn(1, g.H, g.W, min(g.Cin, 16), generator=gen, dtype=torch.float64)
        w = torch.randn(g.kh, g.kw, x.shape[3], min(g.Cout, 8), generator=gen, dtype=torch.float64)
        g = g._replace(Cin=x.shape[3], Cout=w.shape[3])
        xn = torch.nn.functional.pad(x.permute(0, 3, 1, 2), (g.pad_l, g.W + g.W, g.pad_t, g.H + g.H)).requires_grad_(True)
        wn = w.permute(3, 2, 0, 1).contiguous().requires_grad_(True)
        yn = torch.nn.functional.conv2d(xn, wn, stride=g.stride, dilation=g.dil)[:, :, :g.Ho, :g.Wo]
        y = S.fwd_bilinear(x, w, g)
        assert torch.allclose(y, yn.permute(0, 2, 3, 1), atol=1e-10)
        dy = torch.randn(y.shape, generator=gen, dtype=torch.float64)
        yn.backward(dy.permute(0, 3, 1, 2))
        dx = xn.grad[:, :, g.pad_t:g.pad_t + g.H, g.pad_l:g.pad_l + g.W].permute(0, 2, 3, 1)
        assert torch.allclose(S.dgrad_bilinear(dy, w, g), dx, atol=1e-10)
        assert torch.allclose(S.wgrad_bilinear(x, dy, g), wn.grad.permute(2, 3, 1, 0), atol=1e-10)


# split-K factors the launchers chose on the 132 SMs of an H100 SXM (pnp_tc_last_config): (forward, data gradient)
SPLITK_H100_SXM = {
    "g10_512x2560_sym": (1, 1), "dil2_512_B5": (3, 3), "k5s4_512_B3": (32, 2), "256x512_B8": (1, 1), "64_s2_256wide": (1, 1),
    "32x64_s2": (2, 1), "16x32_k5s4": (6, 1), "64x32": (1, 1), "32x64": (2, 2), "16x16_256wide": (1, 1), "128x64_4x4_B9": (4, 2),
    "64_7x9_s2": (2, 1), "64_12x20": (2, 2), "wg_cin192": (6, 4), "wg_cin64": (2, 4), "wg_cin32_3x3": (2, 2), "wg_cin32_5x5": (6, 8),
    "32x32": (2, 2),
}


def test_expected_ksplit_matches_h100_launches(monkeypatch):
    """the split-K rule the GPU test asserts for any SM count reproduces what the launchers chose on an H100 SXM"""
    for k in ("PNP_TC_BK128", "PNP_TC_BK64"):
        monkeypatch.delenv(k, raising=False)
    for name, want in SPLITK_H100_SXM.items():
        g = geom_of(CASE[name])
        assert (expected_ksplit("fwd", g, 132), expected_ksplit("dgrad", g, 132)) == want, name
