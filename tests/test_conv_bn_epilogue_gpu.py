"""Batch-norm partial sums that the wgmma forward convolution reduces in its epilogue (pnp_conv2d_tc_fwd with bn_sum /
bn_sumsq), per column, against fp64 sums of the launch's own output.

Each consumer warp adds its fp32 16-row partials, promoted to fp64, into its own shared-memory row over every tile the CTA
walks with one n-tile; when the n-tile changes and at the end the eight rows are summed in a fixed order and each column
takes one fp64 global atomic.  The cases reach every N tile (128 / 64 / 32 / 16 columns) at nterms 1 and 3, with ragged tiles
(rows past the image), dropout, and CTAs that walk tiles of more than one n-tile (a flush in the middle of the tile list).

a. random operands: |sum - fp64 sum| <= 2^-19 sum|z| and |sumsq - fp64 sumsq| <= 2^-19 sum z^2 per column (the bound of
   test_tc_split_exact_gpu.py's fused BN sums), with dropout off and on;
b. integer operands small enough that every fp32 warp partial is exact: both sums equal the fp64 reference bit for bit;
c. (CPU) no shared-memory compare-and-swap loop is left in any conv_tc_kernel instantiation of the built library."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest
import torch

from tests.cabi import DEV, ROOT, block_n, crosses_ntile, drop_cfg, drop_mask, last_config, lib, sm_count, split_dev, split_w_dev

LIB = os.path.join(ROOT, "medical-cross-modality-domain-adaptation_b200", "libpnp_b200.so")

# (id, B, H, W, Cin, Cout): 3x3 SAME stride-1 convolutions.  Widths 40 and 56 leave 8 / 16 of each 128-row tile past the image
# row, and 40 / 56 rows are not a multiple of the tile's 3 / 2 rows: the last row of tiles is ragged too.
CASES = [
    ("n128_5ntiles", 8, 40, 40, 64, 640),     # <128,*,64>, 560 tiles: CTAs cross n-tiles
    ("n64_5ntiles", 8, 40, 40, 64, 320),      # <64,*,64>, 560 tiles: CTAs cross n-tiles
    ("n32", 8, 56, 56, 32, 32),               # <32,*,32>, 224 tiles: two tiles of one n-tile per CTA
    ("n16", 8, 56, 56, 16, 16),               # <16,*,16>
]
CASE_IDS = [c[0] for c in CASES]


def _geom(_C, case):
    _, B, H, W, Cin, Cout = case
    return _C.ConvGeom(B, H, W, Cin, H, W, Cout, 3, 3, 1, 1, 1, 1)


def _fwd_bn(_C, rt, g, x, w, nterms, keep=None):
    """-> (y, sum, sumsq) of one pnp_conv2d_tc_fwd launch with fused BN sums"""
    xh, xl = split_dev(_C, rt, x, nterms)
    wh, wl = split_w_dev(_C, rt, w, False, nterms)
    y = torch.full((g.B, g.Ho, g.Wo, g.Cout), float("nan"), device=DEV)
    s = torch.zeros(2, g.Cout, dtype=torch.float64, device=DEV)
    drop, seed_t = drop_cfg(_C, keep) if keep is not None else (None, None)
    _C.call("pnp_conv2d_tc_fwd", _C.ptr(xh), _C.ptr(xl), _C.ptr(wh), _C.ptr(wl), _C.ptr(y), ctypes.byref(g), nterms,
            None if drop is None else ctypes.byref(drop), 0, _C.ptr(s[0]), _C.ptr(s[1]), rt.stream())
    torch.cuda.synchronize()
    n, _, ks = last_config(_C)
    assert n == block_n(g.Cout) and ks == 1, "expected the fused-epilogue path, got %s" % (last_config(_C),)
    return y, s[0], s[1]


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [None, 0.75], ids=["nodrop", "drop"])
@pytest.mark.parametrize("nterms", [3, 1])
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_bn_sums_match_fp64(case, nterms, keep):
    _C, rt = lib(require_tc=True)
    g = _geom(_C, case)
    if case[-1] // block_n(case[-1]) > 1:
        assert crosses_ntile(g, sm_count()), "no CTA flushes mid-list"
    gen = torch.Generator().manual_seed(case[-1] + nterms)
    x = (torch.randn(g.B, g.H, g.W, g.Cin, generator=gen) + 0.3).to(DEV)
    w = (torch.randn(3, 3, g.Cin, g.Cout, generator=gen) * 0.05).to(DEV)
    y, s1, s2 = _fwd_bn(_C, rt, g, x, w, nterms, keep)
    assert bool(torch.isfinite(y).all())
    z = y.double().reshape(-1, g.Cout)
    e1 = float(((s1 - z.sum(0)).abs() / z.abs().sum(0)).max())
    e2 = float(((s2 - (z * z).sum(0)).abs() / (z * z).sum(0)).max())
    print("  BN sums %s nterms %d keep %s: sum err %.2e of sum|z|, sumsq err %.2e of sum z^2 (tol 2^-19 = %.2e)" %
          (case[0], nterms, keep, e1, e2, 2.0 ** -19))
    assert e1 <= 2.0 ** -19 and e2 <= 2.0 ** -19


@pytest.mark.gpu
@pytest.mark.parametrize("nterms", [3, 1])
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_bn_sums_exact_on_integers(case, nterms):
    """x, w in {-1, 0, 1} (exact in the hi plane): |z| <= 9 Cin, so a warp's 16-row fp32 sum of z^2 stays below 2^24 and is exact
    for Cin <= 64 (and for Cin <= 32 with keep = 0.5, whose multiplier is 2); every fp64 sum after it is exact as well"""
    _C, rt = lib(require_tc=True)
    g = _geom(_C, case)
    gen = torch.Generator().manual_seed(3 * case[-1] + nterms)
    x = torch.randint(-1, 2, (g.B, g.H, g.W, g.Cin), generator=gen).float().to(DEV)
    w = torch.randint(-1, 2, (3, 3, g.Cin, g.Cout), generator=gen).float().to(DEV)
    ref = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), w.double().permute(3, 2, 0, 1), padding=1).permute(0, 2, 3, 1)
    for keep in ([None, 0.5] if g.Cin <= 32 else [None]):
        assert 16 * (9 * g.Cin * (2 if keep else 1)) ** 2 < 2 ** 24
        y, s1, s2 = _fwd_bn(_C, rt, g, x, w, nterms, keep)
        want = ref
        if keep is not None:
            want = ref * drop_mask(drop_cfg(_C, keep)[0], ref.shape).double()
        assert torch.equal(y.double(), want), "%s nterms %d keep %s: output not exact" % (case[0], nterms, keep)
        z = want.reshape(-1, g.Cout)
        assert torch.equal(s1, z.sum(0)), "%s nterms %d keep %s: BN sum not exact" % (case[0], nterms, keep)
        assert torch.equal(s2, (z * z).sum(0)), "%s nterms %d keep %s: BN sumsq not exact" % (case[0], nterms, keep)


def _cuobjdump():
    return shutil.which("cuobjdump") or next((p for p in ("/usr/local/cuda/bin/cuobjdump",) if os.path.exists(p)), None)


@pytest.mark.skipif(_cuobjdump() is None, reason="cuobjdump not installed")
def test_no_shared_memory_cas_in_conv_tc_kernel():
    """the epilogue's BN partials take plain shared-memory adds: a CAS loop (how sm_90 runs an fp64 shared-memory atomicAdd)
    would serialise the consumer warps on the same columns while the tensor cores wait"""
    assert os.path.exists(LIB), "build the library first (__graft_entry__.build())"
    sass = subprocess.run([_cuobjdump(), "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    conv = [f for f in funcs if "conv_tc_kernel" in f.split("\n", 1)[0]]
    assert len(conv) == 18, "expected 18 conv_tc_kernel instantiations, found %d" % len(conv)
    bad = [f.split("\n", 1)[0].strip() for f in conv if "ATOMS.CAS" in f]
    assert not bad, "shared-memory CAS loops in: %s" % bad
