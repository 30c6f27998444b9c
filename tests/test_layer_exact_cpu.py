"""oracle/layer_exact.py against fp64 torch autograd of the same layer built from oracle/tf14_torch.py, and its bounds against
records with the four mistakes the GPU taps (tests/test_layer_taps_gpu.py) must catch.

a. Every reference (conv z on both kernel families, BN statistics and moving averages, y with skip and activation, the folded
   epilogue, g, dz, dgamma, dbeta, dskip, dW, dx through SAME / SYMMETRIC padding) equals autograd to 1e-12 of scale, over SAME,
   SYMMETRIC, strided and dilated convolutions, BN in training / inference mode / absent, every activation, a skip at a channel
   offset and a given dropout mask.  Operands of the wgmma references are bf16-representable, so their split is exact.  The
   leaky-ReLU slope is the kernels' 0.2f.
b. A record holding the fp32 rounding of the true values passes every bound; the same record with stale BN sums, a dropout mask
   of the wrong stream, the wrong activation or the skip gradient left out of dx is rejected."""
import pytest
import torch

from oracle import bf16_split as S
from oracle import elementwise_exact as E
from oracle import layer_exact as LX
from oracle import simt_exact as X
from oracle import tf14_torch as T

NONE, RELU, LRELU = LX.NONE, LX.RELU, LX.LRELU
KEEP = 0.5          # 1 / keep is exact, so tf14's x * mask / keep equals the kernels' x * fl32(1 / keep)

# (id, padding, stride, dilation, bn: "train" / "infer" / None, act, skip: None or (channels, offset), dropout mask)
CASES = [
    ("same_bntrain_lrelu_drop", "SAME", 1, 1, "train", LRELU, None, True),
    ("symmetric_bninfer_relu", "SYMMETRIC", 1, 1, "infer", RELU, None, False),
    ("strided_nobn_lrelu_drop", "SAME", 2, 1, None, LRELU, None, True),
    ("dilated_bntrain_none_skip", "SAME", 1, 2, "train", NONE, (6, 0), True),
    ("skip_offset_bntrain_lrelu", "SAME", 1, 1, "train", LRELU, (2, 3), False),
    ("symmetric_strided_nobn_none_drop", "SYMMETRIC", 2, 1, None, NONE, None, True),
    ("dilated_bninfer_relu_skip_offset", "SAME", 1, 2, "infer", RELU, (4, 1), True),
    ("nobn_relu_skip", "SAME", 1, 1, None, RELU, (6, 0), False),
]
B, H, CIN, COUT, K = 2, 9, 4, 6, 3


def _geometry(padding, stride, dil):
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F
    cfg = F.LayerCfg(stride=stride, dil=dil, padding=padding)
    p, g = F._geometry((B, H, H, CIN), (K, K, CIN, COUT), cfg)
    return p, LX.geom(g)


def _bf16(t):
    return t.to(torch.bfloat16).to(torch.float64)


def _close(tag, got, ref, tol=1e-12):
    scale = float(ref.abs().max()) or 1.0
    err = float((got - ref).abs().max())
    assert err <= tol * scale, "%s: %.3e of scale %.3e" % (tag, err / scale, scale)


def _act(v, act):
    if act == NONE:
        return v
    return torch.nn.functional.leaky_relu(v, LX.LEAK32) if act == LRELU else torch.relu(v)


def _run(case, seed=0):
    """the layer in fp64 autograd -> dict of operands, intermediate values and gradients"""
    _, padding, stride, dil, bn, act, skip, drop = case
    g0 = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g0, dtype=torch.float64)  # noqa: E731
    x = _bf16(rn(B, H, H, CIN)).requires_grad_(True)
    W = _bf16(0.3 * rn(K, K, CIN, COUT)).requires_grad_(True)
    p, g = _geometry(padding, stride, dil)
    zc = T.conv2d_raw(x, W, stride=stride, dilation=dil, padding=padding)
    assert tuple(zc.shape) == (B, g.Ho, g.Wo, COUT)
    zc.retain_grad()            # the kernels' dz is the gradient of the convolution's output, before the dropout multiplier
    mask = None
    if drop:
        mask = (torch.rand(zc.shape, generator=g0) < KEEP).to(torch.float64) / KEEP
        z = T.dropout(zc, KEEP, mask * KEEP)
    else:
        z = zc
    st = T.BNState(COUT, torch.float64)
    with torch.no_grad():
        st.gamma = (1 + 0.3 * rn(COUT)).requires_grad_(True)
        st.beta = (0.2 * rn(COUT)).requires_grad_(True)
        st.moving_mean, st.moving_var = 0.1 * rn(COUT), 0.5 + torch.rand(COUT, generator=g0, dtype=torch.float64)
    mm0, mv0 = st.moving_mean.clone(), st.moving_var.clone()
    v = T.batch_norm(z, st, bn == "train") if bn else z
    sk = None
    if skip is not None:
        cs, off = skip
        sk = rn(B, g.Ho, g.Wo, cs).requires_grad_(True)
        v = v + torch.nn.functional.pad(sk, (off, COUT - off - cs))
    y = _act(v, act)
    r = rn(*y.shape)
    (y * r).sum().backward()
    return {"x": x.detach(), "W": W.detach(), "p": p, "g": g, "mask": mask, "z": z.detach(), "dz": zc.grad, "st": st, "mm0": mm0,
            "mv0": mv0, "skip": None if sk is None else sk.detach(), "y": y.detach(), "dy": r, "dx": x.grad, "dW": W.grad,
            "dgamma": st.gamma.grad if bn else None, "dbeta": st.beta.grad if bn else None,
            "dskip": None if sk is None else sk.grad}


def _stats(case, run):
    """(mean, invstd) the layer's batch norm used"""
    st, z = run["st"], run["z"]
    if case[4] == "train":
        zf = z.reshape(-1, COUT)
        return zf.mean(0), 1.0 / torch.sqrt(zf.var(0, unbiased=False) + E.BN_EPS)
    return run["mm0"], 1.0 / torch.sqrt(run["mv0"] + E.BN_EPS)


def _refs(case, run, dz=None, mask=None, act=None, into=None):
    """every reference of layer_exact from the record's own stage inputs"""
    _, padding, stride, dil, bn, act0, skip, drop = case
    act = act0 if act is None else act
    mask = run["mask"] if mask is None else mask
    x, W, p, g, st = run["x"], run["W"], run["p"], run["g"], run["st"]
    xp = X.mirror_pad(x, p, p) if p else x
    out = {"z_simt": LX.fwd_simt(xp, W, g, mask), "z_tc": LX.fwd_tc(*S.split(xp), W, g, 3, mask)}
    mean, invstd = _stats(case, run)
    cs, off = skip if skip else (0, 0)
    if bn == "train":
        out["stats"] = LX.bn_train_stats(run["z"], st.gamma.detach(), st.beta.detach(), run["mm0"], run["mv0"])
    if bn:
        out["y"] = LX.bn_apply(run["z"], mean, invstd, st.gamma.detach(), st.beta.detach(), run["skip"], off, act)
    else:
        out["y"] = LX.act_apply(run["z"], run["skip"], off, act)
    if bn != "train":
        coef = LX.moving_coef(st.gamma.detach(), st.beta.detach(), run["mm0"], run["mv0"]) if bn else (None, None, None)
        out["y_fused"] = LX.fused_epilogue(*out["z_simt"], *coef, run["skip"], off, act)
    bwd = LX.layer_bwd(run["dy"], run["y"], act, run["z"] if bn else None, mean if bn else None, invstd if bn else None,
                       st.gamma.detach() if bn else None, bn == "train", mask)
    out.update(bwd)
    dzr = bwd["dz"][0] if dz is None else dz
    out["dW"] = LX.wgrad_simt(xp, dzr, g)
    out["dx"] = LX.dgrad_simt(dzr, W, g, p, into)
    dzb = _bf16(dzr)
    out["dW_tc"], out["dW_bf16"] = LX.wgrad_tc(*S.split(xp), dzb, None, g, 1), LX.wgrad_simt(xp, dzb, g)
    out["dx_tc"], out["dx_bf16"] = LX.dgrad_tc(dzb, torch.zeros_like(dzb), W, g, 3, p), LX.dgrad_simt(dzb, W, g, p)
    if skip:
        out["dskip"] = (bwd["g"][0][..., off:off + cs], bwd["g"][1][..., off:off + cs])
    return out


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_references_equal_autograd(case):
    run = _run(case)
    ref = _refs(case, run)
    tag = case[0]
    _close(tag + " z simt", ref["z_simt"][0], run["z"])
    _close(tag + " z tc", ref["z_tc"][0], run["z"])
    _close(tag + " y", ref["y"][0], run["y"])
    if "y_fused" in ref:
        _close(tag + " y fused epilogue", ref["y_fused"][0], run["y"])
    if "stats" in ref:
        mean, invstd = _stats(case, run)
        _close(tag + " mean", ref["stats"]["mean"][0], mean)
        _close(tag + " invstd", ref["stats"]["invstd"][0], invstd)
        _close(tag + " moving mean", ref["stats"]["moving_mean"][0], run["st"].moving_mean)
        _close(tag + " moving var", ref["stats"]["moving_var"][0], run["st"].moving_var)
    _close(tag + " dz", ref["dz"][0], run["dz"])
    _close(tag + " dW", ref["dW"][0], run["dW"])
    _close(tag + " dx", ref["dx"][0], run["dx"])
    _close(tag + " dW tc", ref["dW_tc"][0], ref["dW_bf16"][0])
    _close(tag + " dx tc", ref["dx_tc"][0], ref["dx_bf16"][0])
    if case[4]:
        _close(tag + " dgamma", ref["dgamma"][0], run["dgamma"])
        _close(tag + " dbeta", ref["dbeta"][0], run["dbeta"])
    if case[6]:
        _close(tag + " dskip", ref["dskip"][0], run["dskip"])


def test_mirror_fold_is_the_adjoint_of_the_pad():
    g0 = torch.Generator().manual_seed(3)
    x = torch.randn(2, 7, 5, 3, generator=g0, dtype=torch.float64)
    yb = torch.randn(2, 11, 9, 3, generator=g0, dtype=torch.float64)
    lhs = (X.mirror_pad(x, 2, 2) * yb).sum()
    rhs = (x * LX.mirror_fold(yb, 2)).sum()
    assert abs(float(lhs - rhs)) <= 1e-12 * float(yb.abs().sum())


def test_tail_references_hold_their_own_rounding():
    """the tail references are simt_exact's; their gamma_n bounds accept the fp32 rounding of the true values"""
    t = X.TailGeom(2, 2, 3, 4, 2, 5, 5, 3, 0)
    g0 = torch.Generator().manual_seed(4)
    Xi = torch.randn(2, 2, 3, 16, generator=g0, dtype=torch.float64)
    w = torch.randn(5, 5, 4, 3, generator=g0, dtype=torch.float64)
    y, yb = LX.tail_fwd(Xi, w, t)
    assert LX.ratio(y.float(), y, yb) <= 1
    dy = torch.randn(y.shape, generator=g0, dtype=torch.float64)
    dX, dXb = LX.tail_bwd(dy, w, t)
    _close("tail dX", dX, X.tail_bwd_explicit(dy, w, t))
    assert LX.ratio(dX.float(), dX, dXb) <= 1


# ------------------------------------------------------------------------------------------------
# b. the bounds accept the fp32 truth and reject the four mistakes
# ------------------------------------------------------------------------------------------------
NEG_CASE = CASES[0]          # SAME, BN training, leaky ReLU, dropout


def _worst(pairs):
    return max(LX.ratio(got, *ref) for got, ref in pairs)


def test_fp32_truth_passes_every_bound():
    for case in CASES:
        run = _run(case)
        ref = _refs(case, run)
        f = lambda t: t.float()  # noqa: E731
        pairs = [(f(run["z"]), ref["z_simt"]), (f(run["z"]), ref["z_tc"]), (f(run["y"]), ref["y"]), (f(run["dz"]), ref["dz"]),
                 (f(run["dW"]), ref["dW"]), (f(run["dx"]), ref["dx"])]
        if "stats" in ref:
            mean, invstd = _stats(case, run)
            pairs += [(f(mean), ref["stats"]["mean"]), (f(invstd), ref["stats"]["invstd"])]
        if case[4]:
            pairs += [(f(run["dgamma"]), ref["dgamma"]), (f(run["dbeta"]), ref["dbeta"])]
        if case[6]:
            pairs.append((f(run["dskip"]), ref["dskip"]))
        assert _worst(pairs) <= 1, case[0]


def test_stale_bn_sums_are_rejected():
    """the scratch pool not zeroed between steps: the fp64 sums carry the previous step's"""
    run = _run(NEG_CASE)
    ref = _refs(NEG_CASE, run)["stats"]
    zf = run["z"].reshape(-1, COUT)
    prev = _run(NEG_CASE, seed=1)["z"].reshape(-1, COUT)
    M = zf.shape[0]
    s1, s2 = zf.sum(0) + prev.sum(0), (zf * zf).sum(0) + (prev * prev).sum(0)
    mean = s1 / M
    invstd = 1.0 / torch.sqrt((s2 / M - mean * mean).clamp_min(0) + E.BN_EPS)
    assert LX.ratio(mean.float(), *ref["mean"]) > 1 or LX.ratio(invstd.float(), *ref["invstd"]) > 1


def test_wrong_stream_mask_is_rejected():
    """the backward pass drew its dropout mask from stream id + 1"""
    run = _run(NEG_CASE)
    other = _run(NEG_CASE, seed=1)["mask"]
    bad = _refs(NEG_CASE, run, mask=other)["dz"][0]
    assert LX.ratio(bad.float(), *_refs(NEG_CASE, run)["dz"]) > 1


def test_wrong_activation_is_rejected():
    """the backward pass ran with ReLU where the forward pass applied leaky ReLU"""
    run = _run(NEG_CASE)
    bad = _refs(NEG_CASE, run, act=RELU)["dz"][0]
    assert LX.ratio(bad.float(), *_refs(NEG_CASE, run)["dz"]) > 1


def test_dropped_skip_gradient_is_rejected():
    """dx of a residual block's first convolution computed without the skip gradient it must merge"""
    case = CASES[4]
    run = _run(case)
    into = torch.randn(run["x"].shape, generator=torch.Generator().manual_seed(9), dtype=torch.float64)
    good = _refs(case, run, into=into)["dx"]
    assert LX.ratio((good[0] - into).float(), *good) > 1
    assert LX.ratio(good[0].float(), *good) <= 1


# ------------------------------------------------------------------------------------------------
# c. the weight-gradient bounds follow the launch, and stay sharp at the benchmarked batch
# ------------------------------------------------------------------------------------------------
def _geom(B, H, C_in, C_out):
    return S.Geom(B, H, H, C_in, H, H, C_out, 3, 3, 1, 1, 1, 1)


def _smooth(shape, cell, gen, relu):
    """piecewise-constant fields over cell x cell pixels plus a little noise: ReLU'd activations, or a zero-mean gradient"""
    B, H, W, C = shape
    t = torch.randn(B, H // cell, W // cell, C, generator=gen).repeat_interleave(cell, 1).repeat_interleave(cell, 2)
    t = t + 0.1 * torch.randn(shape, generator=gen)
    return torch.relu(t) if relu else t - t.mean((0, 1, 2))


def test_wgrad_splits_cover_the_reduction():
    """the restated launch rules split B*Ho*Wo pixels into chains that cover it with no empty split, and agree with
    simt_exact's restatement of launch_wgrad"""
    for B, H, ci, co in ((16, 256, 16, 16), (16, 128, 32, 32), (2, 256, 3, 16), (16, 32, 512, 512), (32, 8, 512, 512)):
        g = _geom(B, H, ci, co)
        M = B * H * H
        mps, splits = LX.simt_wgrad_split(g)
        assert (splits - 1) * mps < M <= splits * mps, (g, mps, splits)
        inst, ref_splits = X.simt_instance("wgrad", g)
        assert splits == ref_splits, (g, splits, ref_splits)
    for B, H, ci, co, want in ((16, 64, 64, 64, 52), (16, 32, 512, 512, 1), (8, 128, 32, 64, None)):
        g = _geom(B, H, ci, co)
        chain, splits = LX.tc_wgrad_split(g)
        assert (splits - 1) * chain < B * H * H <= splits * chain, (g, chain, splits)
        assert want is None or splits == want, (g, splits)
    assert LX.tc_wgrad_split(_geom(16, 32, 512, 512))[0] == 16384      # the unsplit 512-channel layers of a B = 16 step


@pytest.mark.parametrize("kind", ["simt_B16_256x256_16to16", "tc3_B16_64x64_64to64"])
def test_wgrad_bound_rejects_a_lost_split_at_the_benchmarked_batch(kind):
    """at a B = 16 layer the right weight gradient (rounded to fp32) passes, and the gradient with nothing written, with one
    image's pixels missing or with one CTA's pixel range missing is rejected"""
    gen = torch.Generator().manual_seed(17)
    if kind.startswith("simt"):
        g = _geom(16, 256, 16, 16)
        x, dz = _smooth((16, 256, 256, 16), 16, gen, True), _smooth((16, 256, 256, 16), 16, gen, False)
        chain = LX.simt_wgrad_split(g)[0]
        ref = lambda a, b: LX.wgrad_simt(a, b, g)  # noqa: E731
    else:
        g = _geom(16, 64, 64, 64)
        x, dz = _smooth((16, 64, 64, 64), 8, gen, True), _smooth((16, 64, 64, 64), 8, gen, False)
        chain = LX.tc_wgrad_split(g)[0]
        ref = lambda a, b: LX.wgrad_tc(*S.split(a), *S.split(b), g, 3)  # noqa: E731
    good = ref(x, dz)
    assert LX.ratio(good[0].float(), *good) <= 1
    assert LX.ratio(torch.zeros_like(good[0]), *good) > 1, "nothing written"
    flat = dz.reshape(-1, dz.shape[-1])
    for tag, lost in (("image 0", slice(0, dz.shape[1] * dz.shape[2])), ("the first CTA's pixels", slice(0, chain))):
        part = torch.zeros_like(flat)
        part[lost] = flat[lost]
        bad = good[0] - S.wgrad_bilinear(x.double(), part.reshape(dz.shape).double(), g)
        r = LX.ratio(bad.float(), *good)
        print("  %s: %s missing, ratio %.2f" % (kind, tag, r))
        assert r > 1, "%s: %s missing passes (ratio %.3f)" % (kind, tag, r)
