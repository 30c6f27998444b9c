"""GPU parity of every operator of the hot path: CUDA product (through layers.py / ops.py -> ctypes ->
C-ABI) vs the CPU oracle (oracle/tf14_torch.py, fp64) on identical seeded inputs.  fp32 kernels: tolerance
1e-4 relative to the largest reference magnitude; the 3-term bf16-split tensor-core path: 2e-4; stated per test.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests.util import check, check_grad, randn

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _prod():
    import pnp_b200
    from pnp_b200 import layers, ops, functional, runtime
    return layers, ops, functional, runtime


def _oracle():
    from oracle import tf14_torch as T
    return T


def _var(t, grad=True):
    v = t.to(DEV).contiguous()
    v.requires_grad_(grad)
    return v


# (B, H, W, Cin, Cout, k, stride, dil, padding) -- every conv flavour the graphs contain, at reduced spatial size
CONV_CASES = [
    (2, 16, 16, 3, 16, 3, 1, 1, "SAME"),       # conv1_1: Cin=3 scalar gather
    (2, 16, 16, 16, 16, 3, 1, 1, "SAME"),      # g1 res
    (2, 16, 16, 16, 32, 3, 1, 1, "SAME"),      # g2 inc
    (2, 8, 8, 64, 128, 3, 1, 1, "SAME"),       # g4
    (2, 8, 8, 128, 128, 3, 1, 2, "SAME"),      # dilated
    (2, 8, 8, 64, 320, 3, 1, 1, "SYMMETRIC"),  # g10-like (mirror pad)
    (2, 16, 16, 40, 5, 5, 1, 1, "SYMMETRIC"),  # output conv: Cin=40, Cout=5
    (2, 16, 16, 64, 64, 3, 2, 1, "SAME"),      # cls_1_3 down: stride 2, pad (0,1)
    (2, 16, 16, 32, 32, 5, 2, 1, "SAME"),      # cls_2_3: 5x5 stride 2, pad (1,2)
    (2, 16, 16, 16, 32, 5, 4, 1, "SAME"),      # m_cls_2_3: 5x5 stride 4
    (2, 4, 4, 64, 64, 3, 2, 1, "SYMMETRIC"),   # cls_6
    (2, 8, 8, 32, 64, 5, 4, 1, "SYMMETRIC"),   # m_cls_4
    (2, 3, 3, 8, 8, 5, 1, 1, "SYMMETRIC"),     # 5x5 mirror pad by 2 on a 3x3 map: a border row mirrors onto 3 padded rows
    (2, 16, 16, 5, 16, 3, 2, 1, "SAME"),       # mask_cls_1: Cin=5
    (3, 12, 20, 24, 40, 3, 1, 1, "SAME"),      # odd sizes / ragged tiles
    (1, 7, 9, 8, 12, 3, 2, 1, "SAME"),         # odd spatial, stride 2
    (1, 70, 45, 40, 5, 5, 1, 1, "SAME"),       # few-output direct kernel: ragged 32x32 tiles, zero padding
    (2, 40, 33, 8, 8, 3, 1, 1, "SAME"),        # few-output direct kernel, 8 outputs
    # strided data gradients large enough for the phase-major row order of the SIMT gather (one phase per CTA)
    (8, 32, 32, 16, 32, 5, 4, 1, "SAME"),      # m_cls_2_3 at batch 8: 16 phases x 512 rows
    (4, 32, 32, 16, 32, 3, 2, 1, "SAME"),      # stride 2, pad (0,1): 4 phases x 1024 rows
    (4, 32, 32, 64, 64, 3, 2, 1, "SAME"),      # 64-channel output tile (BM = 128)
]


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "B%d_%dx%d_%d-%d_k%d_s%d_d%d_%s" % c)
@pytest.mark.parametrize("backend", ["simt", "auto"])
def test_conv_fwd_bwd(case, backend):
    """conv2d / dilate_conv2d forward, dgrad and wgrad vs oracle autograd"""
    L, ops, F, rt = _prod()
    T = _oracle()
    rt.set_conv_backend(backend)
    B, H, W, Cin, Cout, k, s, d, pad = case
    x = randn((B, H, W, Cin), 1)
    w = randn((k, k, Cin, Cout), 2, 0.2)
    xo, wo = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yo = T.conv2d_raw(xo, wo, stride=s, dilation=d, padding=pad)
    r = randn(tuple(yo.shape), 3)
    (yo * r.double()).sum().backward()
    xg, wg = _var(x), _var(w)
    if d == 1:
        y = L.conv2d(xg, wg, 1.0, strides=[1, s, s, 1], padding=pad)
    else:
        y = L.dilate_conv2d(xg, wg, 1.0, rate=d, padding=pad)
    tol = 1e-4 if backend == "simt" else 2e-4
    check("y", y, yo, tol)
    y.backward(r.to(DEV))
    check("dx", xg.grad, xo.grad, tol)
    check("dw", wg.grad, wo.grad, tol)
    rt.set_conv_backend("auto")


TC_CASES = [
    (2, 32, 32, 64, 64, 3, 1, 1, "SAME"),
    (2, 32, 32, 128, 256, 3, 1, 1, "SAME"),
    (3, 32, 32, 512, 512, 3, 1, 2, "SAME"),     # DR block conv, B not a multiple of the image tile
    (2, 32, 32, 64, 320, 3, 1, 1, "SYMMETRIC"), # g10-like: 34x34 padded input, dgrad on a 34-wide grid
    (2, 64, 64, 64, 64, 3, 1, 1, "SAME"),
    (1, 128, 128, 64, 128, 3, 1, 1, "SAME"),
    (1, 256, 256, 64, 64, 3, 1, 1, "SAME"),     # cls_1 res b: two 128-wide tiles per row
    (5, 16, 16, 512, 512, 3, 1, 1, "SAME"),     # cls_5: 16x16 images, 8 rows per tile
    (9, 4, 4, 128, 64, 3, 1, 1, "SAME"),        # tiny images: 8 images per tile, ragged batch
    (2, 64, 64, 32, 64, 3, 1, 1, "SAME"),       # Cin = 32 (cls_1 res a): zero-padded 64-channel planes, fwd + wgrad
    (8, 32, 32, 256, 512, 3, 1, 1, "SAME"),     # 128x128 tiles over 4 n-tiles (fwd), 2 n-tiles (dgrad)
    # strided layers: forward through TMA element strides, dgrad as s*s phase convolutions, wgrad with strided x boxes
    (2, 32, 32, 64, 64, 3, 2, 1, "SAME"),       # cls_x_3 style 3x3 s2, pad (0,1)
    (2, 32, 32, 128, 128, 5, 2, 1, "SAME"),     # cls_2_3: 5x5 s2, pad (1,2)
    (3, 16, 16, 512, 512, 5, 4, 1, "SAME"),     # cls_5_3: 5x5 s4 16 -> 4
    (2, 4, 4, 64, 64, 3, 2, 1, "SYMMETRIC"),    # cls_6: mirror pad + s2 -> 2x2
    (1, 256, 256, 64, 64, 3, 2, 1, "SAME"),     # cls_1_3 at full size: 256-wide strided TMA box
    (2, 8, 8, 128, 256, 5, 4, 1, "SYMMETRIC"),  # m_cls_4
    # 32-channel layers: native 32-wide K blocks (SWIZZLE_64B operand tiles) and 32-wide N tiles
    (2, 32, 32, 32, 32, 3, 1, 1, "SAME"),       # g2 / m_cls_3 style: K block 32, N tile 32
    (1, 128, 128, 64, 32, 3, 1, 1, "SAME"),     # N tile 32 with 64-wide K; its dgrad reduces over 32 channels into 64
    (2, 32, 32, 32, 64, 3, 2, 1, "SAME"),       # strided, Cin = 32: phase dgrad with N = 32
    (1, 256, 256, 32, 64, 3, 1, 1, "SAME"),     # cls_1 res a at full width
    (3, 16, 16, 32, 128, 3, 1, 2, "SAME"),      # dilated, Cout = 128 from 32 channels
    # 16-channel layers: 16-wide K blocks (SWIZZLE_32B operand tiles), 16-wide N tiles
    (2, 32, 32, 16, 16, 3, 1, 1, "SAME"),       # g1 res
    (2, 32, 32, 16, 32, 3, 1, 1, "SAME"),       # g2 inc: forward N 32 / K 16, dgrad N 16 / K 32
    (1, 256, 256, 16, 16, 3, 1, 1, "SAME"),     # g1 at full width
    (8, 32, 32, 16, 32, 5, 4, 1, "SAME"),       # m_cls_2_3: 5x5 stride 4, phase dgrad with N = 16
    # more tiles than the 132 SMs of an H100, so every persistent CTA walks several tiles (and changes n-tile on the way)
    (16, 32, 32, 512, 512, 3, 1, 2, "SAME"),    # g8 at config 1's batch: 128 m-tiles x 4 n-tiles of 128x128, dilated
    (4, 64, 64, 128, 128, 3, 1, 1, "SAME"),     # 128x128 tiles
    (2, 128, 128, 64, 64, 3, 1, 1, "SAME"),     # 128x64 tiles
]


@pytest.mark.parametrize("case", TC_CASES, ids=lambda c: "B%d_%dx%d_%d-%d_k%d_s%d_d%d_%s" % c)
@pytest.mark.parametrize("backend,tol", [("tc3", 2e-4), ("tc1", 3e-2)])
def test_conv_tensor_core(case, backend, tol):
    """tensor-core path (3-term split = fp32-grade, 1-term = plain bf16) forward + dgrad vs oracle"""
    L, ops, F, rt = _prod()
    T = _oracle()
    if not rt.tc_available():
        pytest.fail("wgmma path unavailable on this device -- it must be the one that runs on H100")
    rt.set_conv_backend(backend)
    B, H, W, Cin, Cout, k, s, d, pad = case
    F.TC_PAD32 = True          # exercise the zero-padded 64-channel plane path for the Cin = 32 case
    x = randn((B, H, W, Cin), 11)
    w = randn((k, k, Cin, Cout), 12, 0.05)
    xo, wo = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yo = T.conv2d_raw(xo, wo, stride=s, dilation=d, padding=pad)
    r = randn(tuple(yo.shape), 13)
    (yo * r.double()).sum().backward()
    xg, wg = _var(x), _var(w)
    y = L.conv2d(xg, wg, 1.0, strides=[1, s, s, 1], padding=pad) if d == 1 else L.dilate_conv2d(xg, wg, 1.0, rate=d, padding=pad)
    check("y", y, yo, tol)
    y.backward(r.to(DEV))
    check("dx", xg.grad, xo.grad, tol)
    check("dw", wg.grad, wo.grad, tol)
    F.TC_PAD32 = False
    assert not F._tc_declined, "these shapes must run on the tensor cores: %s" % (F._tc_declined,)
    rt.set_conv_backend("auto")


def test_wide_layers_select_the_128_column_tile():
    """the 512-channel 32x32 layers of the segmenter (the step's dominant launches) run on the widest tile, 128x128 with
    64-channel K blocks, without split-K"""
    L, ops, F, rt = _prod()
    from pnp_b200 import _C
    rt.set_conv_backend("tc3")
    x, w = randn((8, 32, 32, 512), 3).to(DEV), randn((3, 3, 512, 512), 4, 0.05).to(DEV)
    with torch.no_grad():
        y = L.conv2d(x, w, 1.0)
    torch.cuda.synchronize()
    n_, k_, s_ = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int(0)
    _C.lib.pnp_tc_last_config(ctypes.byref(n_), ctypes.byref(k_), ctypes.byref(s_))
    assert (n_.value, k_.value, s_.value) == (128, 64, 1)
    ref = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).double(), w.permute(3, 2, 0, 1).double(), padding=1).permute(0, 2, 3, 1)
    assert float((y.double() - ref).abs().max() / ref.abs().max()) < 2e-5
    rt.set_conv_backend("auto")


def _bn_pair(T, C, seed):
    """oracle BNState + matching product variables with non-trivial gamma/beta/moving stats"""
    bn = T.BNState(C, torch.float64)
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        bn.gamma.copy_(1 + 0.3 * torch.randn(C, generator=g, dtype=torch.float64))
        bn.beta.copy_(0.2 * torch.randn(C, generator=g, dtype=torch.float64))
        bn.moving_mean = 0.1 * torch.randn(C, generator=g, dtype=torch.float64)
        bn.moving_var = 1 + 0.2 * torch.rand(C, generator=g, dtype=torch.float64)
    return bn


def _load_bn(rt, scope, bn):
    rt.load_state_dict({scope + "/gamma": bn.gamma.detach().numpy(), scope + "/beta": bn.beta.detach().numpy(),
                        scope + "/moving_mean": bn.moving_mean.numpy(), scope + "/moving_variance": bn.moving_var.numpy()})


@pytest.mark.parametrize("is_train", [True, False])
@pytest.mark.parametrize("leak", [True, False])
@pytest.mark.parametrize("backend", ["simt", "auto"])
def test_conv_bn_relu(is_train, leak, backend):
    """conv_bn_relu2d: conv -> BN(train|infer) -> (l)relu, forward, all gradients, moving statistics"""
    L, ops, F, rt = _prod()
    T = _oracle()
    rt.reset_default_graph()
    rt.set_conv_backend(backend)
    B, H, W, Cin, Cout = 3, 16, 16, 64, 64
    x, w = randn((B, H, W, Cin), 21), randn((3, 3, Cin, Cout), 22, 0.1)
    bn = _bn_pair(T, Cout, 23)
    xo, wo = x.double().requires_grad_(True), w.double().requires_grad_(True)
    mm0, mv0 = bn.moving_mean.clone(), bn.moving_var.clone()
    st = 1 if backend == "auto" else 2          # stride 1 rides the tensor-core path (+ fused BN statistics)
    yo = T.conv_bn_relu2d(xo, wo, 1.0, bn, strides=(1, st, st, 1), is_train=is_train, leak=leak)
    r = randn(tuple(yo.shape), 24)
    (yo * r.double()).sum().backward()
    L.bn_variables("t", Cout)
    bn0 = _bn_pair(T, Cout, 23)
    _load_bn(rt, "t", bn0)
    xg, wg = _var(x), _var(w)
    y = L.conv_bn_relu2d(xg, wg, 1.0, strides=[1, st, st, 1], is_train=is_train, scope="t", leak=leak)
    check("y", y, yo, 2e-4)
    y.backward(r.to(DEV))
    # fp32 SIMT: 3e-4; the bf16-split tensor-core path carries ~1e-5 per conv, amplified by the BN-backward cancellation
    tm, tl = (3e-4, 1e-4) if backend == "simt" else (2e-2, 2e-3)
    check_grad("dx", xg.grad, xo.grad, tm, tl)
    check_grad("dw", wg.grad, wo.grad, tm, tl)
    v = rt.graph.vars
    check_grad("dgamma", v["t/gamma"].grad, bn.gamma.grad, tm, tl)
    check_grad("dbeta", v["t/beta"].grad, bn.beta.grad, tm, tl)
    check("moving_mean", v["t/moving_mean"], bn.moving_mean, 1e-5)
    check("moving_var", v["t/moving_variance"], bn.moving_var, 1e-5)
    if not is_train:
        assert torch.equal(bn.moving_mean, mm0) and torch.equal(bn.moving_var, mv0)
    rt.set_conv_backend("auto")


@pytest.mark.parametrize("inc_dim", [False, True])
@pytest.mark.parametrize("kind", ["res", "dr"])
@pytest.mark.parametrize("is_train", [True, False])
@pytest.mark.parametrize("backend", ["simt", "auto"])
def test_residual_blocks(inc_dim, kind, is_train, backend):
    """residual_block / DR_block incl. the channel-pad skip; dgrad of the first conv merged with the skip grad"""
    L, ops, F, rt = _prod()
    T = _oracle()
    rt.reset_default_graph()
    rt.set_conv_backend(backend)
    B, H, W, Cin = 2, 16, 16, 64
    Cout = 2 * Cin if inc_dim else Cin
    x = randn((B, H, W, Cin), 31)
    w1, w2 = randn((3, 3, Cin, Cout), 32, 0.1), randn((3, 3, Cout, Cout), 33, 0.1)
    b1, b2 = _bn_pair(T, Cout, 34), _bn_pair(T, Cout, 35)
    xo = x.double().requires_grad_(True)
    w1o, w2o = w1.double().requires_grad_(True), w2.double().requires_grad_(True)
    if kind == "res":
        yo = T.residual_block(xo, w1o, w2o, 1.0, b1, b2, inc_dim=inc_dim, is_train=is_train, leak=True)
    else:
        yo = T.DR_block(xo, w1o, w2o, 2, 1.0, b1, b2, inc_dim=inc_dim, is_train=is_train, leak=True)
    r = randn(tuple(yo.shape), 36)
    (yo * r.double()).sum().backward()
    L.bn_variables("s_1", Cout)
    L.bn_variables("s_2", Cout)
    _load_bn(rt, "s_1", _bn_pair(T, Cout, 34))
    _load_bn(rt, "s_2", _bn_pair(T, Cout, 35))
    xg, w1g, w2g = _var(x), _var(w1), _var(w2)
    if kind == "res":
        y = L.residual_block(xg, w1g, w2g, 1.0, inc_dim=inc_dim, is_train=is_train, scope="s", leak=True)
    else:
        y = L.DR_block(xg, w1g, w2g, 2, 1.0, inc_dim=inc_dim, is_train=is_train, scope="s", leak=True)
    check("y", y, yo, 2e-4)
    y.backward(r.to(DEV))
    tm, tl = (5e-4, 1e-4) if backend == "simt" else (5e-2, 5e-3)
    check_grad("dx", xg.grad, xo.grad, tm, tl)
    check_grad("dw1", w1g.grad, w1o.grad, tm, tl)
    check_grad("dw2", w2g.grad, w2o.grad, tm, tl)
    v = rt.graph.vars
    check_grad("dgamma1", v["s_1/gamma"].grad, b1.gamma.grad, tm, tl)
    check_grad("dbeta2", v["s_2/beta"].grad, b2.beta.grad, tm, tl)
    check("mm2", v["s_2/moving_mean"], b2.moving_mean, 1e-5)
    check("mv1", v["s_1/moving_variance"], b1.moving_var, 1e-5)
    rt.set_conv_backend("auto")


def test_fused_bn_stats_match_separate_pass():
    """BN statistics reduced in the wgmma epilogue == the standalone pnp_bn_stats pass"""
    L, ops, F, rt = _prod()
    rt.reset_default_graph()
    rt.set_conv_backend("tc3")
    _fused_vs_separate(L, F, rt, randn((3, 32, 32, 64), 41), randn((3, 3, 64, 128), 42, 0.1))
    # enough tiles that every persistent CTA walks several 128x128 tiles and changes n-tile on the way
    _fused_vs_separate(L, F, rt, randn((8, 32, 32, 256), 43), randn((3, 3, 256, 512), 44, 0.05))
    rt.set_conv_backend("auto")


def _fused_vs_separate(L, F, rt, x, w):
    outs = []
    for fuse in (True, False):
        rt.reset_default_graph()
        F.FUSE_BN_STATS = fuse
        y = L.conv_bn_relu2d(_var(x, False), _var(w, False), 1.0, is_train=True, scope="q", leak=True)
        outs.append((y, rt.graph.vars["q/moving_mean"].clone(), rt.graph.vars["q/moving_variance"].clone()))
    F.FUSE_BN_STATS = True
    check("y", outs[0][0], outs[1][0], 1e-5)
    check("moving_mean", outs[0][1], outs[1][1], 1e-5)
    check("moving_var", outs[0][2], outs[1][2], 1e-5)


def test_maxpool():
    L, ops, F, rt = _prod()
    T = _oracle()
    for C in (16, 6):
        x = randn((2, 8, 12, C), 51)
        xo = x.double().requires_grad_(True)
        yo = T.max_pool2d(xo, 2)
        r = randn(tuple(yo.shape), 52)
        (yo * r.double()).sum().backward()
        xg = _var(x)
        y = L.max_pool2d(xg, 2)
        check("y", y, yo, 1e-7)
        y.backward(r.to(DEV))
        check("dx", xg.grad, xo.grad, 1e-7)


def test_avgpool():
    L, ops, F, rt = _prod()
    x = randn((2, 8, 12, 6), 53)
    xo = x.double().requires_grad_(True)
    yo = torch.nn.functional.avg_pool2d(xo.permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    r = randn(tuple(yo.shape), 54)
    (yo * r.double()).sum().backward()
    xg = _var(x)
    y = L.avg_pool2d(xg, 2)
    check("y", y, yo, 1e-6)
    y.backward(r.to(DEV))
    check("dx", xg.grad, xo.grad, 1e-6)


@pytest.mark.parametrize("H,W,C,n", [(5, 7, 6, 2), (9, 9, 16, 4), (4, 4, 3, 3), (6, 5, 8, 1), (3, 10, 5, 5), (8, 12, 6, 2), (256, 256, 16, 3)])
@pytest.mark.parametrize("avg", [False, True])
def test_pool_same_any_n(H, W, C, n, avg):
    """layers.max_pool2d / avg_pool2d for any n and any map size (tf.nn.*_pool ksize = strides = n, 'SAME', layers.py:102-106) vs the
    oracle (KAT-pinned SAME geometry); n = 2 on even maps is the vectorised 2x2 kernel and must agree with the general one"""
    L, ops, F, rt = _prod()
    T = _oracle()
    B = 2 if H < 256 else 1
    x = randn((B, H, W, C), 151)
    xo = x.double().requires_grad_(True)
    yo = T.pool_same(xo, n, avg)
    r = randn(tuple(yo.shape), 152)
    (yo * r.double()).sum().backward()
    xg = _var(x)
    y = (L.avg_pool2d if avg else L.max_pool2d)(xg, n)
    assert tuple(y.shape) == (B, -(-H // n), -(-W // n), C)
    check("y", y, yo, 1e-6)
    y.backward(r.to(DEV))
    check("dx", xg.grad, xo.grad, 1e-6)
    if n == 2 and H % 2 == 0 and W % 2 == 0:
        xs = _var(x)
        ys = F.pool_same(xs, 2, avg)
        ys.backward(r.to(DEV))
        assert torch.equal(ys, y) and torch.equal(xs.grad, xg.grad)


@pytest.mark.parametrize("shape1,shape2", [((2, 8, 12, 3), (2, 8, 12, 5)), ((2, 10, 13, 4), (2, 6, 8, 2)), ((1, 9, 9, 1), (1, 8, 8, 7)),
                                           ((2, 64, 64, 16), (2, 64, 64, 16))])
def test_crop_and_concat(shape1, shape2):
    """layers.crop_and_concat / simple_concat2d (layers.py:108-127): centre crop + channel concat, and its gradients (zero outside the
    crop) -- exact copies, so bit equality"""
    L, ops, F, rt = _prod()
    T = _oracle()
    x1, x2 = randn(shape1, 161), randn(shape2, 162)
    o1, o2 = x1.clone().requires_grad_(True), x2.clone().requires_grad_(True)
    yo = T.crop_and_concat(o1, o2)
    r = randn(tuple(yo.shape), 163)
    (yo * r).sum().backward()
    g1, g2 = _var(x1), _var(x2)
    y = L.crop_and_concat(g1, g2)
    assert torch.equal(y.cpu(), yo.detach())
    y.backward(r.to(DEV))
    assert torch.equal(g1.grad.cpu(), o1.grad) and torch.equal(g2.grad.cpu(), o2.grad)
    if shape1[:3] == shape2[:3]:
        assert torch.equal(L.simple_concat2d(g1.detach(), g2.detach()).cpu(), yo.detach())
    # only one side needs a gradient
    g1, g2 = _var(x1), _var(x2, False)
    L.crop_and_concat(g1, g2).backward(r.to(DEV))
    assert torch.equal(g1.grad.cpu(), o1.grad) and g2.grad is None


def test_cross_entropy():
    """layers.cross_entropy (layers.py:140-141): -mean(y * log(clip(p, 1e-10, 1))), gradients w.r.t. both arguments; probabilities
    outside [1e-10, 1] are clipped in the value and receive no gradient"""
    L, ops, F, rt = _prod()
    T = _oracle()
    p = torch.softmax(randn((2, 16, 16, 5), 171) * 3, -1)
    p[0, 0, 0] = torch.tensor([0.0, 1e-12, 1.5, 1.0, 0.5])                # below / above the clip range, on its upper bound
    y = torch.nn.functional.one_hot(torch.randint(0, 5, (2, 16, 16), generator=torch.Generator().manual_seed(3)), 5).float()
    y[0, 0, 0] = torch.tensor([0.2, 0.2, 0.2, 0.2, 0.2])
    y[1, 3, 3] = torch.tensor([0.3, 0.2, 0.5, 0.0, 0.0])                  # soft labels are legal inputs
    yo, po = y.double().requires_grad_(True), p.double().requires_grad_(True)
    ce_o = T.cross_entropy(yo, po)
    (ce_o * 1.7).backward()
    yg, pg = _var(y), _var(p)
    ce = L.cross_entropy(yg, pg)
    assert ce.dim() == 0
    check("cross_entropy", ce, ce_o, 1e-6)
    (ce * 1.7).backward()
    check("d labels", yg.grad, yo.grad, 1e-6)
    check("d probabilities", pg.grad, po.grad, 1e-5)
    assert float(pg.grad[0, 0, 0, 0]) == 0.0 and float(pg.grad[0, 0, 0, 1]) == 0.0 and float(pg.grad[0, 0, 0, 2]) == 0.0
    assert float(pg.grad[0, 0, 0, 3]) != 0.0


@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("G", [1, 5])
def test_phase_shift(B, G):
    """PS: bit-exact data movement vs the LITERAL numpy emulation of ops.py (both batch regimes)"""
    L, ops, F, rt = _prod()
    from oracle.tf14_numpy import PS_literal
    r = 4
    a, b = (4, 4) if B == 1 else (3, 5)      # the reference's B==1 branch is only defined for square maps
    x = randn((B, a, b, G * r * r), 61)
    ref = torch.from_numpy(PS_literal(x.numpy(), r, G, B))
    xg = _var(x)
    y = ops.PS(xg, r, n_channel=G, batch_size=B)
    assert torch.equal(y.cpu(), ref), "PS forward is pure data movement and must be bit-exact"
    g = randn(tuple(ref.shape), 62)
    y.backward(g.to(DEV))
    # adjoint of a permutation = inverse permutation: check <PS(x), g> == <x, PS^T(g)>
    lhs = float((ref.double() * g.double()).sum())
    rhs = float((x.double() * xg.grad.cpu().double()).sum())
    assert abs(lhs - rhs) <= 1e-6 * max(1.0, abs(lhs))
    with pytest.raises(ValueError):
        ops.PS(xg, r, n_channel=G, batch_size=B + 1)


def test_disc_input_gather():
    """adversarial.py:325-335 channel order + gradients (argmax channel carries none)"""
    L, ops, F, rt = _prod()
    T = _oracle()
    B, a = 2, 4
    c4, c6 = randn((B, a, a, 128), 71), randn((B, a, a, 256), 72)
    b7, c9 = randn((B, a, a, 512), 73), randn((B, a, a, 512), 74)
    lg = randn((B, a * 8, a * 8, 5), 75)
    ins_o = [t.double().requires_grad_(True) for t in (c4, c6, b7, c9, lg)]
    f4 = T.PS(ins_o[0], 8, 2, B).repeat(1, 1, 1, 3)
    ref = torch.cat([f4, T.PS(ins_o[1], 8, 4, B), T.PS(ins_o[2], 8, 8, B), T.PS(ins_o[3], 8, 8, B), ins_o[4],
                     ins_o[4].argmax(3).double().unsqueeze(3)], 3)
    r = randn(tuple(ref.shape), 76)
    (ref * r.double()).sum().backward()
    ins = [_var(t) for t in (c4, c6, b7, c9, lg)]
    out = F.disc_input(*ins, batch_size=B)
    assert out.shape[-1] == 32
    check("d_input", out, ref, 1e-7)
    out.backward(r.to(DEV))
    for n, a_, b_ in zip(("c4", "c6", "b7", "c9", "logits"), ins, ins_o):
        check("d" + n, a_.grad, b_.grad, 1e-6)


def test_seg_losses_and_metrics():
    """weighted CE + soft Dice (forward, gradient), pixel_wise_softmax_2, hard Dice / confusion matrix"""
    L, ops, F, rt = _prod()
    T = _oracle()
    from oracle.pnp_graphs import synthetic_labels
    from oracle.tf14_numpy import label_decomp
    B, S = 2, 64
    logits = randn((B, S, S, 5), 81, 2.0)
    lab = synthetic_labels(B, 5, size=S)
    y = torch.from_numpy(label_decomp(5, lab))
    lo = logits.double().requires_grad_(True)
    wce_o, dice_o = T.softmax_weighted_loss(lo, y.double()), T.dice_loss(lo, y.double())
    (0.7 * wce_o + 1.3 * dice_o).backward()
    lg = _var(logits)
    yg = F.one_hot(torch.from_numpy(lab).to(DEV), 5)
    assert torch.equal(yg.cpu(), y)
    wce, dice = F.seg_losses(lg, yg)
    check("wce", wce.reshape(1), wce_o.reshape(1), 1e-5)
    check("dice", dice.reshape(1), dice_o.reshape(1), 1e-5)
    torch.autograd.backward([wce, dice], [torch.tensor(0.7, device=DEV), torch.tensor(1.3, device=DEV)])
    check("dlogits", lg.grad, lo.grad, 1e-4)
    check("softmax2", L.pixel_wise_softmax_2(lg.detach()), T.pixel_wise_softmax_2(logits.double()), 1e-6)
    from pnp_b200.lib import _dice_eval
    d, arr = _dice_eval(lg.detach(), yg, 5)
    do, arro = T.dice_eval(logits.double().argmax(3), y.double(), 5)
    check("dice_eval", d.reshape(1), do.reshape(1), 1e-6)
    cm = F.confusion_counts(lg.detach(), yg).cpu().numpy()
    pred = logits.argmax(3).numpy()
    ref_cm = np.zeros((5, 5), np.int64)
    np.add.at(ref_cm, (lab.reshape(-1), pred.reshape(-1)), 1)
    assert (cm == ref_cm).all()


def test_fc_and_wgan_means():
    L, ops, F, rt = _prod()
    B, Fd = 6, 2048
    x, w = randn((B, Fd), 91), randn((Fd, 1), 92, 0.1)
    x2 = randn((B, Fd), 93)
    xo, x2o, wo = x.double().requires_grad_(True), x2.double().requires_grad_(True), w.double().requires_grad_(True)
    mr, ct = xo @ wo, x2o @ wo
    loss_o = -0.002 * (mr - ct).mean()
    loss_o.backward()
    xg, x2g, wg = _var(x), _var(x2), _var(w)
    mrg, ctg = F.fc(xg, wg), F.fc(x2g, wg)
    check("fc", mrg, mr, 1e-5)
    loss = F.mean_combo(mrg, -0.002, ctg, 0.002)
    check("dis_loss", loss.reshape(1), loss_o.reshape(1), 1e-5)
    loss.backward()
    check("dx_mr", xg.grad, xo.grad, 1e-5)
    check("dx_ct", x2g.grad, x2o.grad, 1e-5)
    check("dw", wg.grad, wo.grad, 1e-5)


def test_optimizers_match_tf_semantics():
    """fused Adam (epsilon-hat) and RMSProp (ms0 = 1, eps inside sqrt, wd, clip) vs the oracle, 3 steps"""
    L, ops, F, rt = _prod()
    T = _oracle()
    from pnp_b200 import optim
    shapes = [(3, 3, 8, 16), (16,), (5, 5, 16, 7), (2048, 1)]
    for kind in ("adam", "rms"):
        ps = [randn(s, 100 + i, 0.05) for i, s in enumerate(shapes)]
        po = [p.double().clone() for p in ps]
        pg = [_var(p) for p in ps]
        arena = optim.Arena(pg)
        wd = [1e-4, 0.0, 2e-4, 1e-4]
        if kind == "adam":
            opt = optim.Adam(arena, lr=1e-3, weight_decay=wd)
            oo = T.TFAdam(po, lr=1e-3)
        else:
            opt = optim.RMSProp(arena, lr=3e-4, weight_decay=wd, clip=[0.03, 0.0, 0.03, 0.03])
            oo = T.TFRMSProp(po, lr=3e-4)
        for step in range(3):
            gs = [randn(s, 200 + 10 * step + i, 0.1) for i, s in enumerate(shapes)]
            arena.zero_grad()
            for p, g in zip(pg, gs):
                p.grad.copy_(g.to(DEV) * 2.0)          # pretend 2 ranks summed their gradients
            opt.step(grad_scale=0.5)
            oo.step([g.double() + c * p for g, c, p in zip(gs, wd, po)])
            if kind == "rms":
                for p, c in zip(po, [0.03, 0.0, 0.03, 0.03]):
                    if c > 0:
                        p.clamp_(-c, c)
        for i, (p, q) in enumerate(zip(pg, po)):
            check("%s theta[%d]" % (kind, i), p.detach(), q, 1e-5)


def test_momentum_optimizer_matches_tf_semantics():
    """the source segmenter's `optimizer="momentum"` branch (source_segmenter.py:360-372): tf.train.MomentumOptimizer
    (accum = momentum*accum + g; theta -= lr*accum) under exponential_decay(lr, step, decay_steps, decay_rate, staircase=True),
    against a numpy statement of those two published formulas; 5 steps across a staircase boundary"""
    L, ops, F, rt = _prod()
    from pnp_b200 import optim
    shapes = [(3, 3, 8, 16), (16,), (2048, 1)]
    ps = [randn(s, 300 + i, 0.05) for i, s in enumerate(shapes)]
    po = [p.double().numpy().copy() for p in ps]
    acc = [np.zeros_like(p) for p in po]
    pg = [_var(p) for p in ps]
    arena = optim.Arena(pg)
    wd = [1e-4, 0.0, 2e-4]
    opt = optim.Momentum(arena, lr=0.2, decay_rate=0.95, momentum=0.2, decay_steps=2, weight_decay=wd)
    for step in range(5):
        gs = [randn(s, 400 + 10 * step + i, 0.1) for i, s in enumerate(shapes)]
        arena.zero_grad()
        for p, g in zip(pg, gs):
            p.grad.copy_(g.to(DEV) * 4.0)              # 4 ranks summed
        opt.step(grad_scale=0.25)
        lr = 0.2 * 0.95 ** (step // 2)
        for i, g in enumerate(gs):
            acc[i] = 0.2 * acc[i] + (g.double().numpy() + wd[i] * po[i])
            po[i] = po[i] - lr * acc[i]
    assert abs(opt.get_lr() - 0.2 * 0.95 ** 2) < 1e-12
    for i, (p, q) in enumerate(zip(pg, po)):
        check("momentum theta[%d]" % i, p.detach(), torch.from_numpy(q), 1e-5)


def test_dropout_statistics_and_backward_consistency():
    """tf.nn.dropout semantics: keep fraction ~ keep_prob, kept values scaled by 1/keep, the backward pass
    regenerates the same mask; distinct call sites / steps draw distinct masks."""
    L, ops, F, rt = _prod()
    rt.manual_seed(123)
    x = torch.ones(2, 32, 32, 64)
    w = torch.zeros(1, 1, 64, 64)
    w[0, 0] = torch.eye(64)
    xg, wg = _var(x), _var(w, False)
    rt.set_conv_backend("simt")
    y = L.conv2d(xg, wg, 0.75)
    frac = float((y != 0).float().mean())
    assert abs(frac - 0.75) < 0.01, frac
    vals = torch.unique(y.detach())
    assert set(round(float(v), 5) for v in vals) <= {0.0, round(1 / 0.75, 5)}
    y.backward(torch.ones_like(y))
    assert torch.equal((xg.grad != 0), (y.detach() != 0)), "backward must regenerate the forward mask"
    y2 = L.conv2d(xg.detach(), wg, 0.75)
    assert not torch.equal(y2 != 0, y.detach() != 0)
    rt.set_conv_backend("tc3")
    rt.manual_seed(123)
    y3 = L.conv2d(xg.detach(), wg, 0.75)        # same seed + first call site => same mask through the TC epilogue
    assert torch.equal(y3 != 0, y.detach() != 0)
    rt.set_conv_backend("auto")


# (B, H, W, Cin, Cout, stride, dil, inc_dim skip) -- one case per accumulator tile width of the wgmma kernel
FUSED_EP_CASES = [
    (8, 32, 32, 256, 512, 1, 1, True),     # N = 256 tile (8 epilogue warps x 4 chunks), channel-pad skip
    (3, 32, 32, 64, 128, 1, 2, True),      # N = 128, dilated
    (2, 64, 64, 64, 64, 1, 1, False),      # N = 64, same-width skip
    (2, 64, 64, 32, 32, 1, 1, False),      # N = 32 (4 epilogue warps)
    (2, 64, 64, 16, 16, 1, 1, False),      # N = 16 (m64n16 wgmma)
    (4, 32, 32, 64, 64, 2, 1, None),       # strided, no skip
]


@pytest.mark.parametrize("case", FUSED_EP_CASES)
@pytest.mark.parametrize("keep_prob", [1.0, 0.75])
def test_fused_epilogue_equals_separate_bn_apply(case, keep_prob):
    """inference-mode BN + skip + leaky relu folded into the wgmma epilogue (pnp_conv2d_tc_fwd_fused) == convolution followed by
    the streaming pnp_bn_apply_fused pass: same fp32 operations in the same order (y to 1e-6, its bf16 planes must re-compose y to
    2^-16); the backward pass (which no longer has z) must give the same gradients."""
    L, ops, F, rt = _prod()
    B, H, W, Cin, Cout, stride, dil, inc = case
    rt.set_conv_backend("tc3")
    x = randn((B, H, W, Cin), 61)
    w = randn((3, 3, Cin, Cout), 62, 0.1)
    skip = None
    if inc is not None:
        skip = randn((B, H, W, Cout // 2 if inc else Cout), 63)
    r = randn((B, -(-H // stride), -(-W // stride), Cout), 64)
    outs = []
    for fuse in (True, False):
        rt.reset_default_graph()
        rt.manual_seed(77)
        F.FUSE_EPILOGUE = fuse
        bn = L.bn_variables("q", Cout, trainable=False)
        g = torch.Generator().manual_seed(65)
        with torch.no_grad():
            bn.gamma.copy_((1 + 0.3 * torch.randn(Cout, generator=g)).to(DEV))
            bn.beta.copy_((0.2 * torch.randn(Cout, generator=g)).to(DEV))
            bn.moving_mean.copy_((0.1 * torch.randn(Cout, generator=g)).to(DEV))
            bn.moving_var.copy_((0.5 + torch.rand(Cout, generator=g)).to(DEV))
        xg, wg = _var(x), _var(w)
        sg = _var(skip) if skip is not None else None
        cfg = F.LayerCfg(stride=stride, dil=dil, keep_prob=keep_prob, bn=bn, bn_training=False, act=F.ACT_LRELU,
                         skip_off=(Cout // 4 if inc else 0))
        y = F.conv_layer(xg, wg, cfg, sg)
        planes = getattr(y, "_pnp_planes", None)
        y.backward(r.to(DEV))
        outs.append((y.detach().clone(), planes, xg.grad.clone(), wg.grad.clone(), sg.grad.clone() if sg is not None else None))
    F.FUSE_EPILOGUE = True
    (ya, pa, dxa, dwa, dsa), (yb, pb, dxb, dwb, dsb) = outs
    print("  fused y bit-identical to the separate pass: %s" % bool(torch.equal(ya, yb)))
    check("y fused vs separate", ya, yb, 1e-5)      # (few-tile layers: the separate pass may split K and sum through atomics)
    assert (pa is None) == (pb is None)
    if pa is not None:
        check("hi plane", pa[1].float(), pb[1].float(), 1e-2)
        check("hi+lo planes", pa[1].float() + pa[2].float(), yb, 2e-5)
    # few-tile layers: the separate pass splits K (two partial sums through atomics), so y differs by ~1e-6 and the leaky-relu
    # slope of an element with |y| < 1e-6 may flip (0.2 expected flips per case; measured: dx bit-identical in 10 of 12 cases,
    # relative L2 7e-4 / 1.8e-3 in the two cases where one element flips)
    same = bool(torch.equal(ya, yb))
    tm, tl = (1e-4, 1e-4) if same else (1.0, 5e-3)        # (dskip IS g: one flipped element changes by a factor 5 in max-norm)
    check_grad("dx", dxa, dxb, tm, tl)
    check_grad("dw", dwa, dwb, tm, tl)
    if dsa is not None:
        check_grad("dskip", dsa, dsb, tm, tl)
    # and against the fp64 oracle
    T = _oracle()
    bno = T.BNState(Cout, torch.float64)
    bno.gamma.data.copy_(rt.graph.vars["q/gamma"].double().cpu())
    bno.beta.data.copy_(rt.graph.vars["q/beta"].double().cpu())
    bno.moving_mean = rt.graph.vars["q/moving_mean"].double().cpu()
    bno.moving_var = rt.graph.vars["q/moving_variance"].double().cpu()
    if keep_prob == 1.0:
        z = T.conv2d_raw(x.double(), w.double(), stride=stride, dilation=dil, padding="SAME")
        zo = T.batch_norm(z, bno, False)
        if skip is not None:
            zo = zo + (T.channel_pad_skip(skip.double()) if inc else skip.double())
        check("y vs fp64 oracle", ya, T.act(zo, True), 2e-4)
    rt.set_conv_backend("auto")


def test_dropout_draw_is_16_bit_exact_for_three_quarters():
    """the dropout mask keeps an element when its 16-bit Philox draw is below keep*2^16: the kept fraction over 2^22 elements
    must match keep_prob to binomial accuracy, for 0.75 (exactly representable) and for an awkward value"""
    L, ops, F, rt = _prod()
    from pnp_b200._C import call, ptr, DropCfg
    import ctypes
    rt.manual_seed(123)
    n = 1 << 22
    x = torch.ones(n, device=DEV)
    for keep in (0.75, 0.6137):
        y = torch.empty_like(x)
        d = DropCfg(rt.rng.seed_ptr(), rt.rng.next_stream(), keep)
        call("pnp_dropout_apply", ptr(x), ptr(y), n, ctypes.byref(d), rt.stream())
        frac = float((y > 0).float().mean())
        vals = torch.unique(y)
        print("  keep %.4f: kept fraction %.5f, values %s" % (keep, frac, vals.tolist()))
        assert abs(frac - keep) <= 5 * math.sqrt(keep * (1 - keep) / n) + 2.0 ** -16
        assert len(vals) == 2 and abs(float(vals[1]) - 1.0 / keep) <= 1e-6


@pytest.mark.parametrize("B,a", [(1, 6), (2, 6), (3, 6), (2, 32)])
def test_tail_ps_mirror_conv_equals_three_kernels(B, a):
    """pnp_ps_mirror_conv_fwd (phase shift + SYMMETRIC pad folded into the output convolution's tile loader) == ops.PS ->
    layers.conv2d(padding='SYMMETRIC') as separate kernels == the fp64 oracle; gradient w.r.t. the feature map too.
    B == 1 exercises the reference's transposed sub-pixel order (ops.py:11-20)."""
    L, ops, F, rt = _prod()
    T = _oracle()
    b = a                        # a = 6: 48 x 48 output, two (ragged) tiles per axis, mirrored borders on all sides; a = 32: the real
                                 # 256 x 256 map with interior tiles that see no border at all
    G, r, nc = 40, 8, 5
    X = randn((B, a, b, G * r * r), 71)
    w = randn((5, 5, G, nc), 72, 0.1)
    rr = randn((B, a * r, b * r, nc), 73)
    Xo, wo = X.double().requires_grad_(True), w.double()
    yo = T.conv2d(T.PS(Xo, r, G, B), wo, 1.0, padding="SYMMETRIC")
    (yo * rr.double()).sum().backward()
    Xg, wg = _var(X), _var(w, False)
    y = F.tail_ps_conv(Xg, wg, r, G, B)
    check("fused tail vs oracle", y, yo, 1e-5)
    y.backward(rr.to(DEV))
    check("dX (one-kernel backward)", Xg.grad, Xo.grad, 1e-5)
    F.FUSE_TAIL_BWD = False
    Xg2 = _var(X)
    F.tail_ps_conv(Xg2, wg, r, G, B).backward(rr.to(DEV))
    F.FUSE_TAIL_BWD = True
    check("dX (three-kernel backward)", Xg2.grad, Xo.grad, 1e-5)
    Xs = _var(X, False)
    ys = L.conv2d(ops.PS(Xs, r, n_channel=G, batch_size=B), wg, 1.0, padding="SYMMETRIC")
    check("fused tail vs separate kernels", y, ys, 5e-6)      # fp32 both; the register-tiled kernel sums the taps column by column
