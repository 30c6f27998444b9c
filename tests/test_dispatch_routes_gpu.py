"""The same result whichever route the layer dispatcher takes.

`functional` chooses a layer's data flow from process history (`_tc_proven` / `_tc_declined`: the first call of a geometry
writes the fp32 `dz` and the fp32 hidden activation, later calls may keep only their bf16 planes and take the activation's sign
from the hi plane) and from module flags.  Here one layer or residual block runs on the same seeded operands by two routes and
the results are held against each other: bit for bit where the routes only move work between elementwise kernels, to the
spread that two runs of ONE route show where a sum goes through atomics (measured in the test and printed), and to the
split-exact bound of test_ops_gpu.py (2e-4 of scale per convolution) where the convolution implementation changes.  The routes
that must fail do so with a Python exception before the launch that would read a missing tensor."""
import pytest
import torch

from tests import cabi
from tests.util import check, check_grad

pytestmark = pytest.mark.gpu

DEV = cabi.DEV
B, H = 4, 64                     # 128 pixel tiles per layer: no forward or data-gradient launch splits K on a 132-SM device


def _prod():
    import pnp_b200  # noqa: F401
    from pnp_b200 import layers, functional, runtime
    return layers, functional, runtime


@pytest.fixture(autouse=True)
def _clean_dispatcher():
    L, F, rt = _prod()
    flags = {k: getattr(F, k) for k in FLAGS + ("FUSE_TAIL",)}
    rt.set_conv_backend("auto")
    yield
    for k, v in flags.items():
        setattr(F, k, v)
    F.DEBUG_HOOK = None
    F._tc_proven.clear()
    F._tc_declined.clear()
    rt.set_conv_backend("auto")


ELEMENTWISE_FLAGS = ("BN_BWD_DIRECT", "PLANES_ONLY", "FUSE_SPLIT")
CONV_FLAGS = ("TC_WGRAD", "TC_K32", "TC_K16")
FLAGS = ELEMENTWISE_FLAGS + CONV_FLAGS


def _operands(kind, C, inc):
    cin = C // 2 if inc else C
    g = cabi.dev_gen(1000 + C + (7 if inc else 0))
    rn = lambda *s: torch.randn(*s, generator=g, device=DEV)
    ops = {"x": rn(B, H, H, cin), "w1": 0.1 * rn(3, 3, cin, C), "w2": 0.1 * rn(3, 3, C, C), "r": rn(B, H, H, C)}
    for s in ("s_1", "s_2"):
        ops[s] = {"gamma": 1 + 0.3 * rn(C), "beta": 0.2 * rn(C), "moving_mean": 0.1 * rn(C), "moving_variance": 0.5 + torch.rand(C, generator=g, device=DEV)}
    return ops


def _run(kind, C, inc, train, kp, ops):
    """one forward and backward pass of the layer on fresh variables -> every result, and per layer_backward call what the
    debug hook saw: (dz exists as planes only, the saved activation exists as its hi plane only, the planes of dz, fp32 dz)"""
    L, F, rt = _prod()
    rt.reset_default_graph()
    rt.manual_seed(77)
    rt.scratch.begin_step()
    for s in ("s_1", "s_2"):
        bn = L.bn_variables(s, C)
        with torch.no_grad():
            for leaf, t in zip(("gamma", "beta", "moving_mean", "moving_variance"), (bn.gamma, bn.beta, bn.moving_mean, bn.moving_var)):
                t.copy_(ops[s][leaf])
    x = ops["x"].clone().requires_grad_(True)
    w1, w2 = ops["w1"].clone().requires_grad_(True), ops["w2"].clone().requires_grad_(True)
    seen = []

    def hook(sv, dy, g, dz, dx):
        p = getattr(dz, "_pnp_planes", None)
        seen.append({"dz_planes_only": isinstance(dz, F._PlanesOnly), "y_hi": sv.get("y_hi") is not None,
                     "planes": None if p is None else tuple(None if t is None else t.clone() for t in p[1:]),
                     "dz": dz.clone() if isinstance(dz, torch.Tensor) else None})
    F.DEBUG_HOOK = hook
    try:
        if kind == "conv":
            y = L.conv_bn_relu2d(x, w1, kp, is_train=train, scope="s_1", leak=True)
        elif kind == "res":
            y = L.residual_block(x, w1, w2, kp, inc_dim=inc, is_train=train, scope="s", leak=True)
        else:
            y = L.DR_block(x, w1, w2, 2, kp, inc_dim=inc, is_train=train, scope="s", leak=True)
        y.backward(ops["r"])
    finally:
        F.DEBUG_HOOK = None
    torch.cuda.synchronize()
    v = rt.graph.vars
    out = {"y": y.detach().clone(), "dx": x.grad.clone(), "dw1": w1.grad.clone(), "dgamma1": v["s_1/gamma"].grad.clone(),
           "dbeta1": v["s_1/beta"].grad.clone(), "layers": seen}
    if kind != "conv":
        out.update(dw2=w2.grad.clone(), dgamma2=v["s_2/gamma"].grad.clone(), dbeta2=v["s_2/beta"].grad.clone())
    return out


def _planes(run):
    """the bf16 planes of every layer's dz, as one flat fp32 vector per plane"""
    out = {}
    for i, l in enumerate(run["layers"]):
        for j, t in enumerate(l["planes"] or ()):
            if t is not None:
                out["dz%d.%s" % (i, "hi" if j == 0 else "lo")] = t.float()
    return out


def _maxabs(t):
    return float(t.abs().max()) if t.numel() else 0.0


def _held(label, key, a, b, same, floor=None):
    """a (one route) against b (the other).  floor None: an output no atomics touch -- two runs of each route must be bit-equal
    with each other, and so must the routes.  Otherwise (a sum through atomics) within 4x the largest same-route difference,
    or `floor` of scale where two runs agree by chance"""
    spread = max(_maxabs(p - q) for p, q in same)
    err, scale = _maxabs(a - b), _maxabs(b)
    if err > 0 or spread > 0:
        print("  %-40s %-8s |route - route| %.3e, same-route spread %.3e, scale %.3e" % (label, key, err, spread, scale))
    if floor is None:
        assert spread == 0 and all(torch.equal(p, q) for p, q in same), \
            "%s %s: two runs of one route differ by %.3e (scale %.3e); this output is expected to be bit-reproducible" % (label, key, spread, scale)
        assert torch.equal(a, b), "%s %s: the routes differ (max %.3e, scale %.3e)" % (label, key, err, scale)
        return
    assert spread <= 1e-4 * scale, "%s %s: two runs of one route differ by %.3e of scale" % (label, key, spread / scale)
    bound = max(4 * spread, floor * scale)
    assert err <= bound, "%s %s: |route - route| %.3e > %.3e (scale %.3e)" % (label, key, err, bound, scale)


def _hold_runs(label, a, b, keys_exact, keys_atomic):
    """a, b: two runs per route"""
    for k in keys_exact:
        if k in a[0]:
            _held(label, k, a[0][k], b[0][k], [(a[0][k], a[1][k]), (b[0][k], b[1][k])])
    for k in keys_atomic:
        if k in a[0]:
            _held(label, k, a[0][k], b[0][k], [(a[0][k], a[1][k]), (b[0][k], b[1][k])], floor=1e-6)
    pa, pb = [_planes(r) for r in a], [_planes(r) for r in b]
    assert pa[0].keys() == pb[0].keys() and pa[0], (label, list(pa[0]), list(pb[0]))
    for k in pa[0]:
        _held(label, k, pa[0][k], pb[0][k], [(pa[0][k], pa[1][k]), (pb[0][k], pb[1][k])])


EXACT = ("y", "dx", "dgamma1", "dbeta1", "dgamma2", "dbeta2")
ATOMIC = ("dw1", "dw2")

BLOCKS = [("conv", False), ("res", False), ("res", True), ("dr", False), ("dr", True)]


def _tc_wgrad(cin, cout):
    return cout % 64 == 0 and (cin % 64 == 0 or cin == 32)


@pytest.mark.parametrize("kp", [1.0, 0.75])
@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("C", [16, 32, 64, 128])
@pytest.mark.parametrize("kind,inc", BLOCKS)
def test_first_call_and_warmed_call_agree(kind, inc, C, train, kp):
    """cold: no geometry has run on the tensor cores yet (fp32 dz, fp32 hidden activation); warmed: every consumer is proven"""
    L, F, rt = _prod()
    ops = _operands(kind, C, inc)
    label = "%s%s C%d %s kp%.2f" % (kind, "+inc" if inc else "", C, "train" if train else "infer", kp)

    def cold():
        F._tc_proven.clear()
        F._tc_declined.clear()
        return _run(kind, C, inc, train, kp, ops)
    c = [cold(), cold()]
    w = [_run(kind, C, inc, train, kp, ops) for _ in range(3)][1:]
    assert not F._tc_declined, "these geometries must run on the tensor cores: %s" % (F._tc_declined,)
    # the routes really differ, or the comparison is vacuous: layer_backward runs last layer first
    cins = [C] if kind == "conv" else [C, C // 2 if inc else C]
    for run, warmed in ((c[0], False), (c[1], False), (w[0], True), (w[1], True)):
        assert len(run["layers"]) == len(cins)
        for i, (l, cin) in enumerate(zip(run["layers"], cins)):
            # (a block whose two convolutions share one geometry proves it in its second layer's backward pass, which runs first)
            proven = warmed or (i == 1 and not inc)
            assert l["dz_planes_only"] == (proven and _tc_wgrad(cin, C)), (label, warmed, i, cin, l["dz_planes_only"])
            assert (l["dz"] is None) == l["dz_planes_only"]
        if kind != "conv":
            assert run["layers"][1]["y_hi"] == (warmed and C % 64 == 0), (label, warmed, run["layers"][1]["y_hi"])
            assert not run["layers"][0]["y_hi"]
    _hold_runs(label, c, w, EXACT, ATOMIC)


@pytest.mark.parametrize("train", [True, False])
@pytest.mark.parametrize("C", [16, 32, 64, 128])
@pytest.mark.parametrize("kind,inc", [("res", True), ("dr", False)])
@pytest.mark.parametrize("flag", FLAGS)
def test_both_sides_of_each_flag_agree(flag, kind, inc, C, train):
    L, F, rt = _prod()
    kp = 0.75
    ops = _operands(kind, C, inc)
    label = "%s=0 %s%s C%d %s" % (flag, kind, "+inc" if inc else "", C, "train" if train else "infer")

    def warmed(value):
        setattr(F, flag, value)
        F._tc_proven.clear()
        F._tc_declined.clear()
        return [_run(kind, C, inc, train, kp, ops) for _ in range(3)][1:]
    try:
        off = warmed(False)
        on = warmed(True)
    finally:
        setattr(F, flag, True)
    if flag in ELEMENTWISE_FLAGS:
        if C % 64 == 0:
            assert on[0]["layers"][1]["y_hi"] and not off[0]["layers"][1]["y_hi"], "%s did not change the route" % flag
        # FUSE_SPLIT off leaves dz without attached planes: compare what the convolutions consume, the split of the fp32 dz
        if flag == "FUSE_SPLIT":
            for r_off, r_on in zip(off, on):
                for l, l_on in zip(r_off["layers"], r_on["layers"]):
                    assert l["planes"] is None and l["dz"] is not None
                    if l_on["planes"] is not None:
                        l["planes"] = F.split_bf16(l["dz"], 3)
        _hold_runs(label, off, on, EXACT, ATOMIC)
        return
    # the convolution implementation changes (fp32 SIMT against the bf16-split wgmma kernels)
    touched = {"TC_WGRAD": C % 64 == 0, "TC_K32": C in (16, 32) or (inc and C == 64), "TC_K16": C == 16 or (inc and C == 32)}[flag]
    if flag == "TC_WGRAD":
        _hold_runs(label, off, on, EXACT, ())
        for k in ATOMIC:
            check("%s %s" % (label, k), off[0][k], on[0][k], 2e-4)
            if touched:
                assert not torch.equal(off[0][k], on[0][k]), "%s: the flag did not change the weight-gradient kernel" % label
        return
    if not touched:
        _hold_runs(label, off, on, EXACT, ATOMIC)
        return
    assert not torch.equal(off[0]["y"], on[0]["y"]), "%s: the flag did not change the convolution kernel" % label
    check(label + " y", off[0]["y"], on[0]["y"], 4e-4)            # two convolutions
    for k in ("dx", "dw1", "dw2", "dgamma1", "dbeta1", "dgamma2", "dbeta2"):
        check_grad("%s %s" % (label, k), off[0][k], on[0][k], 5e-2, 5e-3)       # the block bars of test_residual_blocks


def test_both_sides_of_fuse_tail_agree():
    """phase shift + mirror pad + output convolution as one kernel against three, behind the segmenter's 3x3 tail convolution"""
    L, F, rt = _prod()
    from pnp_b200.networks import SegmenterTail
    g = cabi.dev_gen(55)
    Bt, a = 2, 8
    c9 = torch.randn(Bt, a, a, 512, generator=g, device=DEV)
    r = torch.randn(Bt, a * 8, a * 8, 5, generator=g, device=DEV)
    rt.reset_default_graph()
    tail = SegmenterTail(5, False, 0.05)
    runs = {}
    try:
        for fuse in (True, True, False):
            F.FUSE_TAIL = fuse
            rt.manual_seed(3)
            x = c9.clone().requires_grad_(True)
            y = tail.run(x, 1.0, Bt)
            y.backward(r)
            runs.setdefault(fuse, []).append((y.detach().clone(), x.grad.clone()))
    finally:
        F.FUSE_TAIL = True
    (y1, d1), (y2, d2) = runs[True]
    y0, d0 = runs[False][0]
    sy, sd = _maxabs(y1 - y2), _maxabs(d1 - d2)
    print("  tail: same-route spread y %.3e dX %.3e; fused - separate y %.3e (scale %.3e) dX %.3e (scale %.3e)" % (
        sy, sd, _maxabs(y1 - y0), _maxabs(y0), _maxabs(d1 - d0), _maxabs(d0)))
    assert not torch.equal(y1, y0) or not torch.equal(d1, d0), "FUSE_TAIL did not change the route"
    assert _maxabs(y1 - y0) <= 5e-6 * _maxabs(y0) + 4 * sy          # the bar of test_tail_ps_mirror_conv_equals_three_kernels
    assert _maxabs(d1 - d0) <= 2e-5 * _maxabs(d0) + 4 * sd          # each side is within 1e-5 of the oracle there


# ------------------------------------------------------------------------------------------------
# the loud failures stay loud
# ------------------------------------------------------------------------------------------------
def test_planes_only_activation_handed_to_a_simt_kernel_raises():
    """a warmed block keeps its hidden activation as planes only; if the backward pass then runs on the SIMT backend, the weight
    gradient asks for the activation's address, which raises before the launch"""
    L, F, rt = _prod()
    C = 64
    ops = _operands("res", C, False)
    for _ in range(2):
        _run("res", C, False, True, 1.0, ops)
    rt.reset_default_graph()
    x = ops["x"].clone().requires_grad_(True)
    w1, w2 = ops["w1"].clone().requires_grad_(True), ops["w2"].clone().requires_grad_(True)
    y = L.residual_block(x, w1, w2, 1.0, is_train=True, scope="s", leak=True)
    rt.set_conv_backend("simt")
    with pytest.raises(RuntimeError, match="exists only as bf16 operand planes"):
        y.backward(ops["r"])
    torch.cuda.synchronize()


def test_planes_only_activation_meeting_a_skip_gradient_raises():
    """the g-less batch-norm backward is the only one that can take the activation's sign from the hi plane: asking a layer
    whose activation was elided for its skip gradient must raise, not read a null pointer"""
    L, F, rt = _prod()
    C = 64
    ops = _operands("res", C, False)
    rt.reset_default_graph()
    bn = L.bn_variables("s_1", C)
    cfg = F.LayerCfg(bn=bn, bn_training=True, act=F.ACT_LRELU)
    x, w = ops["x"], ops["w1"].clone().requires_grad_(True)
    y, sv = F.layer_forward(x, w, cfg, skip=x, save=True, planes_only=True)
    assert isinstance(y, F._PlanesOnly) and sv["y_hi"] is not None and sv["y"] is None
    with pytest.raises(RuntimeError, match="planes-only activation reached a backward path that needs its fp32 copy"):
        F.layer_backward(sv, ops["r"], True, None, want_dskip=True)
    torch.cuda.synchronize()
