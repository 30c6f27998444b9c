"""Residency of the wgmma forward / data-gradient convolution (conv_tc_kernel<BLOCK_N, NTERMS, BK, CTAS_PER_SM>).

The tiles of at most 64 columns run two CTAs per SM, so that one CTA's epilogue overlaps the other's MMAs; the 128-column
tiles stay at one.  Only the number of persistent CTAs walking the tile list changes: every tile is computed by the same
code in the same K order whichever CTA takes it, so a launch at two CTAs per SM must equal the same launch forced to one
(pnp_tc_set_residency_cap(1)):
  - outputs and bf16 (hi, lo) planes bit for bit;
  - fused batch-norm sums within fp64 atomic-order rounding (the per-CTA partials reach the fp64 atomics in another order);
  - split-K outputs within fp32 atomic-order rounding.
The cases reach every 2-CTA instantiation, at nterms 3 and 1.

(CPU) cuobjdump -res-usage of the built library: the 2-CTA kernels use at most 96 registers per thread (two CTAs of 9 warps
fit an SM's four 16K-register sub-partitions only up to 96) and have no local-memory spill."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from tests.cabi import DEV, ROOT, last_config, lib, sm_count, split_dev, split_w_dev

LIB = os.path.join(ROOT, "medical-cross-modality-domain-adaptation_b200", "libpnp_b200.so")
MAX_REGS_2CTA = 96

# (BLOCK_N, BK) of every 2-CTA instantiation -> (Cout, Cin) of a forward that selects it (Cout 192: three 64-column n-tiles,
# so CTAs cross n-tiles and flush their BN rows mid-list)
INST = [(64, 64), (64, 32), (32, 64), (32, 32), (32, 16), (16, 16), (16, 32)]
INST_IDS = ["n%d_k%d" % nk for nk in INST]


def _cout(n):
    return 192 if n == 64 else n


def _residency(_C):
    c, g = ctypes.c_int(0), ctypes.c_int(0)
    _C.lib.pnp_tc_last_residency(ctypes.byref(c), ctypes.byref(g))
    return c.value, g.value


def _both(_C, run):
    """run() at the default residency and at one CTA per SM -> ((result, (ctas, grid)), (result, (ctas, grid)))"""
    out = []
    for cap in (2, 1):
        prev = _C.lib.pnp_tc_set_residency_cap(cap)
        try:
            r = run()
            torch.cuda.synchronize()
            out.append((r, _residency(_C)))
        finally:
            _C.lib.pnp_tc_set_residency_cap(prev)
    return out


def _check_grids(two, one):
    (c2, g2), (c1, g1) = two, one
    assert c2 == 2 and c1 == 1, "residency %d / %d, expected 2 / 1" % (c2, c1)
    assert g1 == min(g2, sm_count()) and g2 > sm_count(), "grids %d / %d: the case does not fill two CTAs per SM" % (g2, g1)


def _bits_equal(tag, a, b):
    assert torch.equal(a.contiguous().view(torch.int32 if a.element_size() == 4 else torch.int16),
                       b.contiguous().view(torch.int32 if b.element_size() == 4 else torch.int16)), "%s differs" % tag


def _operands(g, seed, dgrad):
    gen = torch.Generator().manual_seed(seed)
    src = (g.B, g.Ho, g.Wo, g.Cout) if dgrad else (g.B, g.H, g.W, g.Cin)
    x = (torch.randn(src, generator=gen) + 0.2).to(DEV)
    w = (torch.randn(g.kh, g.kw, g.Cin, g.Cout, generator=gen) * 0.05).to(DEV)
    return x, w


@pytest.mark.gpu
@pytest.mark.parametrize("nterms", [3, 1])
@pytest.mark.parametrize("inst", INST, ids=INST_IDS)
def test_forward_bn_dropout_matches_one_cta(inst, nterms):
    _C, rt = lib(require_tc=True)
    n, k = inst
    g = _C.ConvGeom(8, 64, 64, k, 64, 64, _cout(n), 3, 3, 1, 1, 1, 1)
    x, w = _operands(g, 7 * n + k + nterms, False)
    xh, xl = split_dev(_C, rt, x, nterms)
    wh, wl = split_w_dev(_C, rt, w, False, nterms)
    seed_t = torch.tensor([0x1234_5678_9ABC], dtype=torch.int64, device=DEV)
    drop = _C.DropCfg(seed_t.data_ptr(), 5, 0.75)

    def run():
        y = torch.full((g.B, g.Ho, g.Wo, g.Cout), float("nan"), device=DEV)
        s = torch.zeros(2, g.Cout, dtype=torch.float64, device=DEV)
        _C.call("pnp_conv2d_tc_fwd", _C.ptr(xh), _C.ptr(xl), _C.ptr(wh), _C.ptr(wl), _C.ptr(y), ctypes.byref(g), nterms,
                ctypes.byref(drop), 0, _C.ptr(s[0]), _C.ptr(s[1]), rt.stream())
        assert last_config(_C) == (n, k, 1), last_config(_C)
        return y, s

    ((y2, s2), r2), ((y1, s1), r1) = _both(_C, run)
    _check_grids(r2, r1)
    assert bool(torch.isfinite(y2).all())
    _bits_equal("y", y2, y1)
    z = y1.double().reshape(-1, g.Cout)
    for name, a, b, ref in (("sum", s2[0], s1[0], z.abs().sum(0)), ("sumsq", s2[1], s1[1], (z * z).sum(0))):
        err = float(((a - b).abs() / ref).max())
        print("  %s nterms %d: BN %s differs by %.2e of its magnitude" % (INST_IDS[INST.index(inst)], nterms, name, err))
        assert err <= 2.0 ** -44, (name, err)


@pytest.mark.gpu
@pytest.mark.parametrize("nterms", [3, 1])
@pytest.mark.parametrize("inst", INST, ids=INST_IDS)
def test_fused_epilogue_planes_match_one_cta(inst, nterms):
    """inference-mode BN + channel-pad skip + leaky ReLU, fp32 y and its bf16 planes"""
    _C, rt = lib(require_tc=True)
    n, k = inst
    g = _C.ConvGeom(8, 64, 64, k, 64, 64, _cout(n), 3, 3, 1, 1, 1, 1)
    x, w = _operands(g, 11 * n + k + nterms, False)
    xh, xl = split_dev(_C, rt, x, nterms)
    wh, wl = split_w_dev(_C, rt, w, False, nterms)
    gen = torch.Generator().manual_seed(n + k)
    scale = (torch.rand(g.Cout, generator=gen) + 0.5).to(DEV)
    shift = (torch.randn(g.Cout, generator=gen) * 0.1).to(DEV)
    skip_c, skip_off = g.Cout // 2, 4
    skip = torch.randn(g.B, g.Ho, g.Wo, skip_c, generator=gen).to(DEV)

    def run():
        y = torch.full((g.B, g.Ho, g.Wo, g.Cout), float("nan"), device=DEV)
        yh = torch.zeros((g.B, g.Ho, g.Wo, g.Cout), dtype=torch.bfloat16, device=DEV)
        yl = torch.zeros_like(yh) if nterms == 3 else None
        ep = _C.TcEpilogue(scale.data_ptr(), shift.data_ptr(), skip.data_ptr(), skip_c, skip_off, 2, yh.data_ptr(), _C.ptr(yl))
        _C.call("pnp_conv2d_tc_fwd_fused", _C.ptr(xh), _C.ptr(xl), _C.ptr(wh), _C.ptr(wl), _C.ptr(y), ctypes.byref(g), nterms,
                None, 0, None, None, ctypes.byref(ep), rt.stream())
        return y, yh, yl

    ((y2, h2, l2), r2), ((y1, h1, l1), r1) = _both(_C, run)
    _check_grids(r2, r1)
    assert bool(torch.isfinite(y2).all())
    _bits_equal("y", y2, y1)
    _bits_equal("hi plane", h2, h1)
    if nterms == 3:
        _bits_equal("lo plane", l2, l1)


@pytest.mark.gpu
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("nterms", [3, 1])
@pytest.mark.parametrize("inst", INST, ids=INST_IDS)
def test_data_gradient_matches_one_cta(inst, nterms, stride):
    """dx = conv^T(dy, w): the data gradient's output channels are the forward's Cin (the tile's columns), its reduction the
    forward's Cout; stride 2 runs its four phases in one launch"""
    _C, rt = lib(require_tc=True)
    n, k = inst
    H = 64 if stride == 1 else 128
    g = _C.ConvGeom(8, H, H, _cout(n), 64, 64, k, 3, 3, stride, 1, 1 if stride == 1 else 0, 1 if stride == 1 else 0)
    dy, w = _operands(g, 13 * n + k + nterms + stride, True)
    dh, dl = split_dev(_C, rt, dy, nterms)
    wh, wl = split_w_dev(_C, rt, w, True, nterms)

    def run():
        dx = torch.full((g.B, g.H, g.W, g.Cin), float("nan"), device=DEV)
        _C.call("pnp_conv2d_tc_dgrad", _C.ptr(dh), _C.ptr(dl), _C.ptr(wh), _C.ptr(wl), _C.ptr(dx), ctypes.byref(g), nterms, 0,
                rt.stream())
        assert last_config(_C) == (n, k, 1), last_config(_C)
        return dx

    (dx2, r2), (dx1, r1) = _both(_C, run)
    _check_grids(r2, r1)
    assert bool(torch.isfinite(dx2).all())
    _bits_equal("dx", dx2, dx1)


@pytest.mark.gpu
@pytest.mark.parametrize("nterms", [3, 1])
def test_split_k_matches_one_cta(nterms):
    """few tiles, deep K: 4 tiles x 9 K blocks are split two ways and added with fp32 atomics into a zeroed output"""
    _C, rt = lib(require_tc=True)
    g = _C.ConvGeom(2, 16, 16, 64, 16, 16, 64, 3, 3, 1, 1, 1, 1)
    x, w = _operands(g, 17 + nterms, False)
    xh, xl = split_dev(_C, rt, x, nterms)
    wh, wl = split_w_dev(_C, rt, w, False, nterms)

    def run():
        y = torch.full((g.B, g.Ho, g.Wo, g.Cout), float("nan"), device=DEV)
        _C.call("pnp_conv2d_tc_fwd", _C.ptr(xh), _C.ptr(xl), _C.ptr(wh), _C.ptr(wl), _C.ptr(y), ctypes.byref(g), nterms, None, 0,
                None, None, rt.stream())
        n_, k_, ks = last_config(_C)
        assert (n_, k_) == (64, 64) and ks > 1, last_config(_C)
        return y, ks

    ((y2, ks), r2), ((y1, _), r1) = _both(_C, run)
    assert r2[0] == 2 and r1[0] == 1 and r2[1] == r1[1] <= sm_count()
    # each output is the fp32 sum of ks partials: reordering them moves it by a few roundings of the running sum
    tol = ks * 2.0 ** -22 * float(y1.abs().max())
    assert float((y2 - y1).abs().max()) <= tol, (float((y2 - y1).abs().max()), tol)


@pytest.mark.gpu
@pytest.mark.parametrize("nterms", [3, 1])
def test_128_column_tiles_stay_at_one_cta(nterms):
    _C, rt = lib(require_tc=True)
    g = _C.ConvGeom(8, 64, 64, 64, 64, 64, 128, 3, 3, 1, 1, 1, 1)
    x, w = _operands(g, 19, False)
    xh, xl = split_dev(_C, rt, x, nterms)
    wh, wl = split_w_dev(_C, rt, w, False, nterms)
    y = torch.empty(g.B, g.Ho, g.Wo, g.Cout, device=DEV)
    _C.call("pnp_conv2d_tc_fwd", _C.ptr(xh), _C.ptr(xl), _C.ptr(wh), _C.ptr(wl), _C.ptr(y), ctypes.byref(g), nterms, None, 0,
            None, None, rt.stream())
    torch.cuda.synchronize()
    assert last_config(_C)[0] == 128
    assert _residency(_C) == (1, sm_count())


def _cuobjdump():
    return shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)


@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump not installed")
def test_two_cta_kernels_fit_registers_without_spill():
    assert os.path.exists(LIB), "build the library first (__graft_entry__.build())"
    out = subprocess.run([_cuobjdump(), "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    found = {}
    for m in re.finditer(r"Function (\S*conv_tc_kernelILi(\d+)ELi(\d)ELi(\d+)ELi(\d)E\S*):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ "
                         r"LOCAL:(\d+)", out):
        n, nterms, k, ctas, reg, stack, local = (int(v) for v in m.groups()[1:])
        found[(n, nterms, k)] = (ctas, reg, stack, local)
    assert len(found) == 18, "expected 18 conv_tc_kernel instantiations, found %d" % len(found)
    for (n, nterms, k), (ctas, reg, stack, local) in sorted(found.items()):
        print("  conv_tc_kernel<%d,%d,%d,%d>: %d registers, stack %d, local %d" % (n, nterms, k, ctas, reg, stack, local))
        assert ctas == (2 if n <= 64 else 1), (n, nterms, k, ctas)
        if ctas == 2:
            assert reg <= MAX_REGS_2CTA and stack == 0 and local == 0, (n, nterms, k, reg, stack, local)
