"""Every dropout producer against the independent Philox4x32-10 reference of oracle/philox.py, bit for bit, at the C-ABI.

a. pnp_dropout_apply: y == fl32(x * mult) over seeds {0, 0x5EED, 2^63 - 1, 2^64 - 1} x streams {0, 1, 2^32 - 1, 2^32 + 5, 2^64 - 1}
   x keep {0.5, 0.75, 0.3, 0.6137, 2^-16, 1 - 2^-16, 0.99999}; every scalar tail n = 1 .. 9; a grid above grid_for's 8448-CTA
   cap; in place; the disabled paths (NULL seed, keep 1) out of place and in place;
b. the SIMT forward convolution (float4 and scalar stores, with accumulate) and the wgmma forward convolution (plain and fused
   epilogue, nterms 1 and 3, every accumulator width 16 / 32 / 64 / 128, a ragged last tile, a split-K layer) on integer
   operands: y == [y0 +] fl32(mult * conv) with conv the exact fp64 convolution.  (The batch-norm backward entry points are
   pinned to the same reference through drop_mask of tests/cabi.py, which now draws from it.)
c. pnp_seed_advance against the Python LCG, runtime.manual_seed, a captured graph of [pnp_seed_advance, pnp_dropout_apply];
d. the seed-advance -> dropout and seed-advance -> convolution sequences again under PNP_PDL=1, in their own process."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import philox as PH
from tests.cabi import DEV, last_config, lib, rerun, split_dev, split_w_dev

pytestmark = pytest.mark.gpu

SEEDS = [0, 0x5EED, (1 << 63) - 1, (1 << 64) - 1]
STREAMS = [0, 1, (1 << 32) - 1, (1 << 32) + 5, (1 << 64) - 1]
KEEPS = [0.5, 0.75, 0.3, 0.6137, 2.0 ** -16, 1 - 2.0 ** -16, 0.99999]
GRID_CAP_N = 4 * 8448 * 1024 + 5
# (id, B, H, W, Cin, Cout, keep): SIMT forward; the CPU file records the store path each reaches
SIMT_CASES = [("float4_C16", 2, 19, 21, 8, 16, 0.75), ("scalar_C6", 2, 17, 23, 12, 6, 0.3), ("scalar_C5", 1, 33, 35, 5, 5, 0.6137)]
# (id, B, H, W, Cin, Cout, keep, expected BLOCK_N, split-K expected): wgmma forward, 3x3 SAME stride 1.  Every case but the
# last has more than 66 tiles, so that it does not split K on 132 SMs (a split-K partial times a non-dyadic 1/keep rounds).
TC_CASES = [
    ("n16_72wide", 2, 72, 72, 16, 16, 0.75, 16, False),         # 72 of the 128 tile rows are pixels: rows that draw unused
    ("n32", 4, 64, 64, 32, 32, 0.3, 32, False),
    ("n64_ragged", 6, 40, 40, 64, 64, 0.6137, 64, False),       # 3-row tiles over 40 rows: the last tile of an image is ragged
    ("n128", 3, 64, 64, 64, 128, 0.5, 128, False),
    ("n128_8imgs_per_tile", 537, 4, 4, 128, 128, 0.75, 128, False),   # 8 images per tile, the last tile holds one
    ("splitk", 1, 8, 8, 512, 64, 0.5, 64, True),                # 1 tile, 72 k-blocks: split along K; mult 2 keeps it exact
]


def seed_tensor(s):
    return torch.tensor([s - (1 << 64) if s >= (1 << 63) else s], dtype=torch.int64, device=DEV)


def cfg_for(_C, seed_t, stream, keep):
    return _C.DropCfg(None if seed_t is None else seed_t.data_ptr(), stream, keep)


def ref_mult(seed, stream, keep, shape):
    n = int(np.prod(shape))
    return torch.from_numpy(PH.dropout_mult(seed, stream, keep, n)).reshape(shape).to(DEV)


def apply(_C, rt, x, y, cfg):
    _C.call("pnp_dropout_apply", x.data_ptr(), y.data_ptr(), x.numel(), None if cfg is None else ctypes.byref(cfg), rt.stream())


def assert_same(tag, got, want):
    torch.cuda.synchronize()
    if not torch.equal(got, want):
        bad = (got != want).flatten().nonzero().flatten()
        i = int(bad[0])
        raise AssertionError("%s: %d of %d elements differ, first %d: got %r want %r" % (
            tag, bad.numel(), got.numel(), i, float(got.flatten()[i]), float(want.flatten()[i])))


# ------------------------------------------------------------------------------------------------
# a. pnp_dropout_apply
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keep", KEEPS)
def test_dropout_apply_matches_philox(keep):
    _C, rt = lib()
    gen = torch.Generator(device=DEV).manual_seed(7)
    n = 4099
    x = torch.randn(n, generator=gen, device=DEV)
    for seed in SEEDS:
        seed_t = seed_tensor(seed)
        for stream in STREAMS:
            y = torch.full_like(x, float("nan"))
            apply(_C, rt, x, y, cfg_for(_C, seed_t, stream, keep))
            assert_same("seed %#x stream %#x keep %r" % (seed, stream, keep), y, x * ref_mult(seed, stream, keep, (n,)))


def test_dropout_apply_tails():
    """n = 1 .. 9: every value of n & 3, the scalar tail alone and after whole quads"""
    _C, rt = lib()
    seed_t = seed_tensor(SEEDS[3])
    for n in range(1, 10):
        x = torch.randn(n, device=DEV)
        y = torch.full_like(x, float("nan"))
        apply(_C, rt, x, y, cfg_for(_C, seed_t, STREAMS[3], 0.5))
        assert_same("n %d" % n, y, x * ref_mult(SEEDS[3], STREAMS[3], 0.5, (n,)))


def test_dropout_apply_grid_stride_and_in_place():
    """n above 4 * 8448 * 1024 (grid-stride loop past the CTA cap) with a tail, in place"""
    _C, rt = lib()
    x = torch.randn(GRID_CAP_N, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)
    want = x * ref_mult(SEEDS[2], STREAMS[4], 0.3, (GRID_CAP_N,))
    seed_t = seed_tensor(SEEDS[2])
    apply(_C, rt, x, x, cfg_for(_C, seed_t, STREAMS[4], 0.3))
    assert_same("grid cap, in place", x, want)


def test_dropout_disabled_paths():
    _C, rt = lib()
    x = torch.randn(1001, device=DEV)
    seed_t = seed_tensor(5)
    for tag, cfg in (("NULL seed", cfg_for(_C, None, 3, 0.5)), ("keep 1", cfg_for(_C, seed_t, 3, 1.0)), ("no cfg", None)):
        y = torch.full_like(x, float("nan"))
        apply(_C, rt, x, y, cfg)
        assert_same(tag + " out of place", y, x)
        z = x.clone()
        apply(_C, rt, z, z, cfg)
        assert_same(tag + " in place", z, x)


# ------------------------------------------------------------------------------------------------
# b. convolutions
# ------------------------------------------------------------------------------------------------
def _geom(_C, B, H, W, Cin, Cout):
    return _C.ConvGeom(B, H, W, Cin, H, W, Cout, 3, 3, 1, 1, 1, 1)


def _int_operands(B, H, W, Cin, Cout, seed):
    gen = torch.Generator().manual_seed(seed)
    x = torch.randint(-4, 5, (B, H, W, Cin), generator=gen).float().to(DEV)
    w = torch.randint(-4, 5, (3, 3, Cin, Cout), generator=gen).float().to(DEV)
    return x, w


def conv_exact(x, w):
    """fp64 3x3 SAME convolution of integer operands, NHWC / HWIO: exact, and an fp32 value while 9 Cin 16 < 2^24"""
    assert 9 * x.shape[-1] * 16 < 2 ** 24
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double().permute(3, 2, 0, 1), padding=1).permute(0, 2, 3, 1).contiguous()
    assert torch.equal(y.float().double(), y)
    return y.float()


@pytest.mark.parametrize("case", SIMT_CASES, ids=[c[0] for c in SIMT_CASES])
def test_simt_conv_dropout(case):
    _C, rt = lib()
    tag, B, H, W, Cin, Cout, keep = case
    x, w = _int_operands(B, H, W, Cin, Cout, 31)
    ref = conv_exact(x, w)
    g = _geom(_C, B, H, W, Cin, Cout)
    for seed, stream in ((SEEDS[1], STREAMS[2]), (SEEDS[3], STREAMS[4])):
        seed_t = seed_tensor(seed)
        cfg = cfg_for(_C, seed_t, stream, keep)
        mult = ref_mult(seed, stream, keep, ref.shape)
        y = torch.full_like(ref, float("nan"))
        _C.call("pnp_conv2d_fwd", x.data_ptr(), w.data_ptr(), y.data_ptr(), ctypes.byref(g), ctypes.byref(cfg), 0, rt.stream())
        assert_same(tag, y, ref * mult)
        y0 = torch.randint(-9, 10, ref.shape, device=DEV).float()
        y = y0.clone()
        _C.call("pnp_conv2d_fwd", x.data_ptr(), w.data_ptr(), y.data_ptr(), ctypes.byref(g), ctypes.byref(cfg), 1, rt.stream())
        assert_same(tag + " accumulate", y, y0 + ref * mult)


@pytest.mark.parametrize("nterms", [1, 3])
@pytest.mark.parametrize("case", TC_CASES, ids=[c[0] for c in TC_CASES])
def test_tc_conv_dropout(case, nterms):
    _C, rt = lib(require_tc=True)
    tag, B, H, W, Cin, Cout, keep, block_n, split = case
    x, w = _int_operands(B, H, W, Cin, Cout, 37)
    ref = conv_exact(x, w)
    g = _geom(_C, B, H, W, Cin, Cout)
    xh, xl = split_dev(_C, rt, x, nterms)
    wh, wl = split_w_dev(_C, rt, w, False, nterms)
    seed, stream = SEEDS[3], STREAMS[3]
    seed_t = seed_tensor(seed)
    cfg = cfg_for(_C, seed_t, stream, keep)
    mult = ref_mult(seed, stream, keep, ref.shape)
    p = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    y = torch.full_like(ref, float("nan"))
    _C.call("pnp_conv2d_tc_fwd", p(xh), p(xl), p(wh), p(wl), y.data_ptr(), ctypes.byref(g), nterms, ctypes.byref(cfg), 0, None, None,
            rt.stream())
    bn, _, ks = last_config(_C)
    assert bn == block_n and (ks > 1) == split, "%s: BLOCK_N %d split-K %d" % (tag, bn, ks)
    assert_same("%s nterms %d" % (tag, nterms), y, ref * mult)
    y0 = torch.randint(-9, 10, ref.shape, device=DEV).float()
    y = y0.clone()
    _C.call("pnp_conv2d_tc_fwd", p(xh), p(xl), p(wh), p(wl), y.data_ptr(), ctypes.byref(g), nterms, ctypes.byref(cfg), 1, None, None,
            rt.stream())
    assert_same("%s nterms %d accumulate" % (tag, nterms), y, y0 + ref * mult)
    if split:
        return          # a fused epilogue never splits K
    # fused epilogue: relu(dropout(conv) * scale + shift), scale in {1/2, 1, 2}, integer shift: still exact
    scale = torch.tensor([0.5, 1.0, 2.0], device=DEV)[torch.arange(Cout, device=DEV) % 3].contiguous()
    shift = (torch.arange(Cout, device=DEV) % 7 - 3).float()
    ep = _C.TcEpilogue(scale.data_ptr(), shift.data_ptr(), None, 0, 0, 1, None, None)
    y = torch.full_like(ref, float("nan"))
    _C.call("pnp_conv2d_tc_fwd_fused", p(xh), p(xl), p(wh), p(wl), y.data_ptr(), ctypes.byref(g), nterms, ctypes.byref(cfg), 0, None,
            None, ctypes.byref(ep), rt.stream())
    assert last_config(_C)[0] == block_n
    assert_same("%s nterms %d fused" % (tag, nterms), y, torch.relu(ref * mult * scale + shift))


# ------------------------------------------------------------------------------------------------
# c. seed advance, manual_seed, graphs
# ------------------------------------------------------------------------------------------------
def test_seed_advance_matches_lcg():
    _C, rt = lib()
    for s in SEEDS + [0x1234_5678_9ABC]:
        t = seed_tensor(s)
        for k in range(1, 6):
            _C.call("pnp_seed_advance", t.data_ptr(), rt.stream())
            got = int(t.item()) & ((1 << 64) - 1)
            assert got == PH.seed_advance(s, k), "seed %#x after %d advances: %#x" % (s, k, got)


def test_manual_seed_masks_the_sign_bit():
    _, rt = lib()
    for s in (0, 5, (1 << 63) - 1, 1 << 63, (1 << 64) - 1, 0xDEAD_BEEF_0123_4567_89):
        rt.manual_seed(s)
        assert int(rt.rng.seed_t.item()) == s & ((1 << 63) - 1)
    rt.manual_seed(0x5EED)


def test_seed_advance_then_producers():
    """the advance and the draw back to back in stream order: the draw must see the advanced seed"""
    _C, rt = lib()
    seed = SEEDS[1]
    x, w = _int_operands(2, 16, 16, 16, 16, 41)
    ref = conv_exact(x, w)
    g = _geom(_C, 2, 16, 16, 16, 16)
    xh, xl = split_dev(_C, rt, x, 3)
    wh, wl = split_w_dev(_C, rt, w, False, 3)
    seed_t = seed_tensor(seed)
    cfg = cfg_for(_C, seed_t, 77, 0.5)       # the 4-tile wgmma layer splits K: mult 2 keeps the partial products exact
    xs = torch.randn(5003, device=DEV)
    torch.cuda.synchronize()
    for k in range(1, 4):
        _C.call("pnp_seed_advance", seed_t.data_ptr(), rt.stream())
        y = torch.empty_like(xs)
        apply(_C, rt, xs, y, cfg)
        _C.call("pnp_seed_advance", seed_t.data_ptr(), rt.stream())
        ys = torch.empty_like(ref)
        _C.call("pnp_conv2d_fwd", x.data_ptr(), w.data_ptr(), ys.data_ptr(), ctypes.byref(g), ctypes.byref(cfg), 0, rt.stream())
        _C.call("pnp_seed_advance", seed_t.data_ptr(), rt.stream())
        yt = torch.empty_like(ref)
        _C.call("pnp_conv2d_tc_fwd", xh.data_ptr(), xl.data_ptr(), wh.data_ptr(), wl.data_ptr(), yt.data_ptr(), ctypes.byref(g), 3,
                ctypes.byref(cfg), 0, None, None, rt.stream())
        s1, s2, s3 = (PH.seed_advance(seed, 3 * (k - 1) + j) for j in (1, 2, 3))
        assert_same("dropout after advance %d" % k, y, xs * ref_mult(s1, 77, 0.5, xs.shape))
        assert_same("SIMT conv after advance %d" % k, ys, ref * ref_mult(s2, 77, 0.5, ref.shape))
        assert_same("wgmma conv after advance %d" % k, yt, ref * ref_mult(s3, 77, 0.5, ref.shape))


def test_graph_replays_draw_fresh_masks():
    """[pnp_seed_advance, pnp_dropout_apply] captured once, replayed 3 times: replay k draws the mask of LCG^k(seed)"""
    _C, rt = lib()
    seed = SEEDS[3]
    seed_t = seed_tensor(seed)
    x = torch.randn(10007, device=DEV)
    y = torch.empty_like(x)
    cfg = cfg_for(_C, seed_t, STREAMS[3], 0.6137)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            cs = torch.cuda.current_stream().cuda_stream
            _C.call("pnp_seed_advance", seed_t.data_ptr(), cs)
            _C.call("pnp_dropout_apply", x.data_ptr(), y.data_ptr(), x.numel(), ctypes.byref(cfg), cs)
    torch.cuda.synchronize()
    for k in range(1, 4):
        graph.replay()
        assert_same("replay %d" % k, y, x * ref_mult(PH.seed_advance(seed, k), STREAMS[3], 0.6137, x.shape))
    del graph


# ------------------------------------------------------------------------------------------------
# d. PDL
# ------------------------------------------------------------------------------------------------
PDL_TESTS = ("seed_advance_matches_lcg", "seed_advance_then_producers", "graph_replays_draw_fresh_masks", "dropout_apply_tails")


@pytest.mark.timeout(300)
def test_exact_cases_under_pdl():
    passed, _ = rerun({"PNP_PDL": "1"}, __file__, " or ".join(PDL_TESTS))
    assert passed == len(PDL_TESTS), passed
