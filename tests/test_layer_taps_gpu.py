"""Every convolution layer of real training steps, at the benchmarked batches, held to an fp64 reference of that layer alone.

Taps installed with monkeypatch wrap functional.layer_forward, layer_backward, _ResBlockFn.backward, the three raw convolution
launchers (to learn which kernel ran and its split-K) and _TailFn.  Each stage of each layer is checked inside the wrapper, as
soon as it has run, against oracle/layer_exact.py fed the kernel's own inputs to that stage (the x planes the convolution
consumed, the kernel's z, mean, invstd, dy, its dz planes, dx_into and the parameter gradients as they were before the call),
with the dropout multipliers taken from pnp_dropout_apply on a ones tensor at the layer's (seed, stream id, keep) and spot-checked
against oracle/philox.py.  The activation's slope comes from the kernel's own y, so no leaky-ReLU slope can flip and every bound
is a priori and per element.  A residual block's returned dx is also held to dgrad(conv1) + the skip gradient of conv2.

Each step runs once untapped first (so that the dispatcher has proven its tensor-core geometries and takes the planes-only
routes), then once tapped, eagerly.  Per step the test asserts that every layer_forward / layer_backward call was checked, that
their number is the reference graph's convolution count (tests/golden/reference_graph_trace.json) less the segmenter's output
convolution wherever the fused tail (_TailFn, checked by its own tap) runs it, that every dropout site drew its own stream id
and that each backward pass handed its dropout kernels (functional._drop_from, tapped) the id its forward pass drew.  It prints the
route census and each stage's worst |got - ref| / bound; the census test runs every step it needs (each step runs once per
session) and asserts that together they reach every route.  The negative controls at B = 2 break the dispatcher in four ways the model-level
tests may miss, and each must trip a tap."""
import collections
import copy
import ctypes
import time

import numpy as np
import pytest
import torch

from oracle import bf16_split as S
from oracle import layer_exact as LX
from oracle import philox
from oracle import simt_exact as X
from tests import cabi
from tests.models import prepare_step

pytestmark = pytest.mark.gpu

DEV = cabi.DEV
SEED = 4242
PHILOX_SPOT = 4096           # elements of every site's mask compared with the independent Philox reference

# every route of the dispatcher that a step of these graphs takes.  The activation-only backward (an activated convolution without
# batch norm) is not among them: neither graph has such a layer, so no step calls it.
ROUTES = ("tc_fwd", "fused_epilogue", "splitk_fwd", "splitk_dgrad", "phase_dgrad", "simt_fwd", "simt_dgrad", "simt_wgrad",
          "tc_wgrad", "tc_dgrad", "split_wgrad", "bn_direct_bwd", "bn_g_bwd", "dropout_only_bwd", "planes_only_y", "planes_only_dz", "symmetric",
          "dx_into", "bn_train_fwd", "tail_fwd", "tail_bwd")


def _prod():
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F, runtime as rt, _C
    return F, rt, _C


class Taps:
    def __init__(self, monkeypatch):
        F, rt, _C = _prod()
        self.F, self.rt, self._C = F, rt, _C
        self.census = collections.Counter()
        self.worst, self.worst_at = {}, {}
        self.fail = []
        self.n_fwd = self.n_bwd = self.n_tail_fwd = self.n_tail_bwd = 0
        self.fwd_sids, self.bwd_sids = [], []
        self.conv_log = []
        self.hook = {}
        self.block = None
        self.tag = ""
        self.mp = monkeypatch
        self._masks = {}
        self.drop_used = []
        self.sms = torch.cuda.get_device_properties(DEV).multi_processor_count

    # ---- bookkeeping ------------------------------------------------------------------------------------------------
    def stage(self, name, got, rb):
        r = LX.ratio(got, *rb)
        if r >= self.worst.get(name, 0.0):
            self.worst[name], self.worst_at[name] = r, self.tag
        if not r <= 1:
            self.fail.append("%s: %s ratio %.3e" % (self.tag, name, r))
        return r

    def exact(self, name, ok):
        self.worst.setdefault(name, 0.0)
        if not ok:
            self.worst[name] = float("inf")
            self.fail.append("%s: %s not bit-equal" % (self.tag, name))

    def mask(self, drop, shape):
        """the layer's dropout multipliers: pnp_dropout_apply on ones, its first elements against oracle/philox.py"""
        if drop is None:
            return None
        sid, keep = drop
        key = (sid, keep, tuple(shape))
        if key in self._masks:
            return self._masks[key]
        F, rt, _C = self.F, self.rt, self._C
        ones = torch.ones(shape, device=DEV)
        m = torch.empty_like(ones)
        cfg = _C.DropCfg(rt.rng.seed_ptr(), sid, keep)
        _C.call("pnp_dropout_apply", cabi.ptr(ones), cabi.ptr(m), m.numel(), ctypes.byref(cfg), rt.stream())
        n = min(PHILOX_SPOT, m.numel())
        ref = philox.dropout_mult(int(rt.rng.seed_t.item()), sid, keep, n)
        self.exact("dropout_mask_vs_philox", np.array_equal(m.reshape(-1)[:n].cpu().numpy(), ref))
        self._masks = {key: m}
        return m

    def check_y(self, name, y, rb, nt):
        F = self.F
        if isinstance(y, F._PlanesOnly):
            self.census["planes_only_y"] += 1
            ntp, hi, lo = y._pnp_planes
            v, rel = LX.planes_value(hi, lo, ntp)
            self.stage(name, v, (rb[0], rb[1] + rel * (rb[0].abs() + rb[1])))
            return
        self.stage(name, y, rb)
        p = getattr(y, "_pnp_planes", None)
        if p is not None:
            hi, lo = S.split(y)
            self.exact("y_planes", S.planes_equal(p[1], hi) and (p[0] != 3 or S.planes_equal(p[2], lo)))

    # ---- the raw convolution launchers: which kernel ran ------------------------------------------------------------------
    def _conv_wrappers(self):
        F = self.F
        real = {k: getattr(F, k) for k in ("conv_fwd_raw", "conv_dgrad_raw", "conv_wgrad_raw")}

        def launched(kind, geom):
            return (F._tc_mode() and F._tc_candidate(kind, geom) and (kind != "wgrad" or F.TC_WGRAD)), F._gkey(kind, geom)

        def after(kind, will, key):
            tc = bool(will) and key not in F._tc_declined
            return tc, (cabi.last_config(self._C)[2] if tc and kind != "wgrad" else 1)

        def fwd(xp, W, geom, drop=None, stats=None, keep_planes=False, ep=None):
            will, key = launched("fwd", geom)
            out = real["conv_fwd_raw"](xp, W, geom, drop, stats, keep_planes, ep)
            tc, ks = after("fwd", will, key)
            self.conv_log.append({"kind": "fwd", "tc": tc, "ksplit": ks, "out": out[0], "applied": out[3], "xp": xp})
            return out

        def dgrad(dz, W, geom, into=None, dz_planes=None):
            will, key = launched("dgrad", geom)
            out = real["conv_dgrad_raw"](dz, W, geom, into, dz_planes)
            tc, ks = after("dgrad", will, key)
            self.conv_log.append({"kind": "dgrad", "tc": tc, "ksplit": ks})
            return out

        def wgrad(xp, dz, W, geom, x_planes=None, dz_planes=None):
            will, key = launched("wgrad", geom)
            out = real["conv_wgrad_raw"](xp, dz, W, geom, x_planes, dz_planes)
            tc = after("wgrad", will, key)[0]
            g = LX.geom(geom)
            splits = LX.tc_wgrad_split(g, self.sms, F._cin_pad(geom))[1] if tc else LX.simt_wgrad_split(g)[1]
            self.conv_log.append({"kind": "wgrad", "tc": tc, "ksplit": splits})
            return out
        self.mp.setattr(F, "conv_fwd_raw", fwd)
        self.mp.setattr(F, "conv_dgrad_raw", dgrad)
        self.mp.setattr(F, "conv_wgrad_raw", wgrad)

    def _log(self, kind):
        recs = [r for r in self.conv_log if r["kind"] == kind]
        assert len(recs) <= 1, (self.tag, kind, len(recs))
        return recs[0] if recs else None

    # ---- layer_forward ----------------------------------------------------------------------------------------------
    def forward(self, real, x, W, cfg, skip=None, save=True, planes_only=False):
        F, rt = self.F, self.rt
        bn = cfg.bn
        pre = None
        if bn is not None and cfg.bn_training:
            pre = (bn.moving_mean.clone(), bn.moving_var.clone())
        self.conv_log = []
        c0 = rt.rng.counter
        y, sv = real(x, W, cfg, skip, save, planes_only)
        torch.cuda.synchronize()
        drop = None
        if rt.rng.counter != c0:
            assert rt.rng.counter == c0 + 1
            drop = (rt.rng.counter, float(cfg.keep_prob))
            self.fwd_sids.append(drop[0])
        self.n_fwd += 1
        self.tag = "fwd#%d %s" % (self.n_fwd, tuple(W.shape))
        self._check_forward(x, W, cfg, skip, y, sv, pre, drop)
        if sv is not None:
            sv["_tap"] = {"act": cfg.act, "drop": drop, "training": cfg.bn_training, "n": self.n_fwd}
        self.conv_log = []
        return y, sv

    def _check_forward(self, x, W, cfg, skip, y, sv, pre, drop):
        F = self.F
        nt = F._tc_mode()
        bn = cfg.bn
        p, geom = F._geometry(tuple(x.shape), tuple(W.shape), cfg)
        g = LX.geom(geom)
        rec = self._log("fwd")
        xp = rec["xp"]
        if p:
            self.census["symmetric"] += 1
            if isinstance(x, torch.Tensor):
                self.exact("mirror_pad", torch.equal(xp, X.mirror_pad(x, p, p)))
        mask = self.mask(drop, (g.B, g.Ho, g.Wo, g.Cout))
        if rec["tc"]:
            self.census["tc_fwd"] += 1
            self.census["splitk_fwd"] += rec["ksplit"] > 1
            planes = getattr(xp, "_pnp_planes", None)
            xh, xl = (planes[1], planes[2]) if planes is not None and planes[0] == nt else S.split(xp)
            conv, cname = LX.fwd_tc(xh, xl, W, g, nt, mask), "conv_fwd_tc%d" % nt
        else:
            self.census["simt_fwd"] += 1
            conv, cname = LX.fwd_simt(xp, W, g, mask), "conv_fwd_simt"
        if rec["applied"]:
            self.census["fused_epilogue"] += 1
            coef = LX.moving_coef(bn.gamma, bn.beta, bn.moving_mean, bn.moving_var) if bn is not None else (None, None, None)
            self.check_y("fused_epilogue_y", y, LX.fused_epilogue(*conv, *coef, skip, cfg.skip_off, cfg.act), nt)
            return
        z = rec["out"]
        self.stage(cname, z, conv)
        if bn is not None:
            if cfg.bn_training:
                self.census["bn_train_fwd"] += 1
                assert sv is not None, "%s: a training-mode batch norm ran without saving its statistics" % self.tag
                st = LX.bn_train_stats(z, bn.gamma, bn.beta, *pre)
                self.stage("bn_mean", sv["mean"], st["mean"])
                self.stage("bn_invstd", sv["invstd"], st["invstd"])
                self.stage("bn_moving_mean", bn.moving_mean, st["moving_mean"])
                self.stage("bn_moving_var", bn.moving_var, st["moving_var"])
                mean, invstd = sv["mean"], sv["invstd"]
            else:
                mean = bn.moving_mean
                invstd = sv["invstd"] if sv is not None else 1.0 / torch.sqrt(bn.moving_var.double() + LX.E.BN_EPS)
            self.check_y("bn_apply_y", y, LX.bn_apply(z, mean, invstd, bn.gamma, bn.beta, skip, cfg.skip_off, cfg.act), nt)
        elif cfg.act != F.ACT_NONE or skip is not None:
            self.check_y("act_apply_y", y, LX.act_apply(z, skip, cfg.skip_off, cfg.act), nt)
        else:
            assert y is z

    # ---- layer_backward ---------------------------------------------------------------------------------------------
    def backward(self, real, sv, dy, need_dx=True, dx_into=None, want_dskip=False):
        F = self.F
        cfg, W = sv["cfg"], sv["W"]
        bn = cfg.bn
        t = sv["_tap"]
        cl = lambda v: None if v.grad is None else v.grad.clone()  # noqa: E731
        before = {"W": cl(W)}
        if bn is not None:
            before.update(gamma=cl(bn.gamma), beta=cl(bn.beta))
        into0 = None if dx_into is None else dx_into.clone()
        self.conv_log = []
        self.hook = {}
        self.drop_used = []
        dx, dskip = real(sv, dy, need_dx, dx_into, want_dskip)
        torch.cuda.synchronize()
        self.n_bwd += 1
        self.tag = "bwd#%d of fwd#%d %s" % (self.n_bwd, t["n"], tuple(W.shape))
        # the stream id the backward pass handed to its dropout kernels, against the one its forward pass drew
        self.exact("backward_stream_id", self.drop_used == [None if t["drop"] is None else t["drop"][0]])
        self.bwd_sids += [sid for sid in self.drop_used if sid is not None]
        rec = self._check_backward(sv, t, dy, need_dx, into0, dx, dskip, before)
        if self.block is not None:
            self.block.append(rec)
        self.conv_log = []
        self.hook = {}
        return dx, dskip

    def _check_backward(self, sv, t, dy, need_dx, into0, dx, dskip, before):
        F = self.F
        cfg, W, geom, p = sv["cfg"], sv["W"], sv["geom"], sv["p"]
        bn = cfg.bn
        g = LX.geom(geom)
        nt = F._tc_mode()
        act = t["act"]
        mask = self.mask(t["drop"], (g.B, g.Ho, g.Wo, g.Cout))
        y_sign = sv["y"] if sv["y"] is not None else sv.get("y_hi")
        gk, dzk = self.hook["g"], self.hook["dz"]
        if bn is not None:
            ref = LX.layer_bwd(dy, y_sign, act, sv["z"], sv["mean"], sv["invstd"], bn.gamma, t["training"], mask)
            self.census["bn_direct_bwd" if gk is None else "bn_g_bwd"] += 1
        else:
            ref = LX.layer_bwd(dy, y_sign, act, mask=mask)
            self.census["act_only_bwd" if act != F.ACT_NONE else ("dropout_only_bwd" if mask is not None else "identity_bwd")] += 1
        if gk is not None and gk is not dy:
            self.stage("g", gk, ref["g"])
        if isinstance(dzk, F._PlanesOnly):
            self.census["planes_only_dz"] += 1
            ntp, hi, lo = dzk._pnp_planes
            v, rel = LX.planes_value(hi, lo, ntp)
            self.stage("dz", v, (ref["dz"][0], ref["dz"][1] + rel * (ref["dz"][0].abs() + ref["dz"][1])))
            dz_planes = (hi, lo)
        else:
            self.stage("dz", dzk, ref["dz"])
            pl = getattr(dzk, "_pnp_planes", None)
            if pl is not None:
                hi, lo = S.split(dzk)
                self.exact("dz_planes", S.planes_equal(pl[1], hi) and (pl[0] != 3 or S.planes_equal(pl[2], lo)))
                dz_planes = (pl[1], pl[2])
            else:
                dz_planes = S.split(dzk) if nt else None
        if bn is not None and "dgamma" in ref:
            for name, v in (("dgamma", bn.gamma), ("dbeta", bn.beta)):
                if v.requires_grad:
                    self.stage(name, v.grad, LX.accumulated(*ref[name], before[name[1:]]))
        out = {"dskip": None, "dx0": None}
        if dskip is not None:
            cs, C = sv["skip_c"], g.Cout
            off = cfg.skip_off if cs != C else 0
            rds = (ref["g"][0][..., off:off + cs], ref["g"][1][..., off:off + cs])
            self.stage("dskip", dskip, rds)
            out["dskip"] = rds
        xp = sv["xp"]
        if W.requires_grad:
            rec = self._log("wgrad")
            self.census["split_wgrad"] += rec["ksplit"] > 1
            if rec["tc"]:
                self.census["tc_wgrad"] += 1
                xs = sv.get("xs")
                if xs is None:
                    pl = getattr(xp, "_pnp_planes", None)
                    xs = (pl[1], pl[2]) if pl is not None and pl[0] == nt else S.split(xp)
                self.stage("wgrad_tc%d" % nt, W.grad, LX.wgrad_tc(xs[0], xs[1], dz_planes[0], dz_planes[1], g, nt, before["W"],
                                                                           self.sms, F._cin_pad(geom)))
            else:
                self.census["simt_wgrad"] += 1
                self.stage("wgrad_simt", W.grad, LX.wgrad_simt(xp, dzk, g, before["W"]))
        if need_dx:
            rec = self._log("dgrad")
            if rec["tc"]:
                self.census["tc_dgrad"] += 1
                self.census["splitk_dgrad"] += rec["ksplit"] > 1
                self.census["phase_dgrad"] += g.stride > 1
                dx0 = LX.dgrad_tc(dz_planes[0], dz_planes[1], W, g, nt, p)
                name = "dgrad_tc%d" % nt
            else:
                self.census["simt_dgrad"] += 1
                dx0 = LX.dgrad_simt(dzk, W, g, p)
                name = "dgrad_simt"
            if into0 is not None:
                self.census["dx_into"] += 1
            self.stage(name, dx, LX.accumulated(*dx0, into0))
            out["dx0"] = dx0
        return out

    # ---- _ResBlockFn.backward: dx = dgrad(conv1) + the skip gradient of conv2 ------------------------------------
    def block_backward(self, real, ctx, dy):
        self.block = []
        out = real(ctx, dy)
        recs, self.block = self.block, None
        assert len(recs) == 2, (self.tag, len(recs))
        if ctx_needs_dx(ctx):
            r2, r1 = recs
            (a, ab), (s, sb) = r1["dx0"], r2["dskip"]
            ref = a + s
            self.tag += " (block)"
            self.stage("block_dx", out[0], (ref, ab + sb + LX.U * (s.abs() + ref.abs())))
        return out

    # ---- the fused segmenter tail ------------------------------------------------------------------------------------
    def tail_forward(self, real, ctx, Xin, w, r, G, order_b1):
        y = real(ctx, Xin, w, r, G, order_b1)
        torch.cuda.synchronize()
        B, a, b, _ = Xin.shape
        t = X.TailGeom(B, a, b, G, r, w.shape[0], w.shape[1], w.shape[3], order_b1)
        self.n_tail_fwd += 1
        self.census["tail_fwd"] += 1
        self.tag = "tail fwd#%d" % self.n_tail_fwd
        self.stage("tail_fwd", y, LX.tail_fwd(Xin, w, t))
        return y

    def tail_backward(self, real, ctx, dy):
        B, a, b, G, r, o = ctx.meta
        w = ctx.w
        out = real(ctx, dy)
        torch.cuda.synchronize()
        t = X.TailGeom(B, a, b, G, r, w.shape[0], w.shape[1], w.shape[3], o)
        self.n_tail_bwd += 1
        self.census["tail_bwd"] += 1
        self.tag = "tail bwd#%d" % self.n_tail_bwd
        self.stage("tail_bwd", out[0], LX.tail_bwd(dy.contiguous(), w, t))
        return out

    def install(self):
        F = self.F
        self._conv_wrappers()
        rf, rb = F.layer_forward, F.layer_backward
        self.mp.setattr(F, "layer_forward", lambda *a, **k: self.forward(rf, *a, **k))
        self.mp.setattr(F, "layer_backward", lambda *a, **k: self.backward(rb, *a, **k))
        rblk = F._ResBlockFn.backward
        self.mp.setattr(F._ResBlockFn, "backward", staticmethod(lambda ctx, dy: self.block_backward(rblk, ctx, dy)))
        tf, tb = F._TailFn.forward, F._TailFn.backward
        self.mp.setattr(F._TailFn, "forward", staticmethod(lambda ctx, *a: self.tail_forward(tf, ctx, *a)))
        self.mp.setattr(F._TailFn, "backward", staticmethod(lambda ctx, dy: self.tail_backward(tb, ctx, dy)))
        self.mp.setattr(F, "DEBUG_HOOK", lambda sv, dy, g, dz, dx: self.hook.update(g=g, dz=dz))
        rdf = F._drop_from

        def drop_from(info):
            cfg = rdf(info)
            self.drop_used.append(None if cfg is None else int(cfg.stream))
            return cfg
        self.mp.setattr(F, "_drop_from", drop_from)


def ctx_needs_dx(ctx):
    return bool(ctx.needs_input_grad[0])


@pytest.fixture(autouse=True)
def _restore():
    F, rt, _C = _prod()
    cap = _C.lib.pnp_tc_set_residency_cap(2)
    _C.lib.pnp_tc_set_residency_cap(cap)
    hook = F.DEBUG_HOOK
    yield
    _C.lib.pnp_tc_set_residency_cap(cap)
    F.DEBUG_HOOK = hook
    F._tc_proven.clear()
    F._tc_declined.clear()
    rt.set_conv_backend("auto")


# ------------------------------------------------------------------------------------------------
# the steps
# ------------------------------------------------------------------------------------------------
def _tapped_step(monkeypatch, kind, backend, B, keep, mutate=None):
    run, expect, _ = prepare_step(monkeypatch, kind, backend, B, keep, SEED, mutate)
    taps = Taps(monkeypatch)
    taps.install()
    t0 = time.time()
    run(keep)
    torch.cuda.synchronize()
    taps.seconds = time.time() - t0
    monkeypatch.undo()
    taps.expect = expect
    return taps


def _report(label, taps):
    print("\n  %s: %d layer_forward, %d layer_backward, %d tail fwd, %d tail bwd checked in %.1f s" % (
        label, taps.n_fwd, taps.n_bwd, taps.n_tail_fwd, taps.n_tail_bwd, taps.seconds))
    print("  routes: " + ", ".join("%s %d" % (k, v) for k, v in sorted(taps.census.items()) if v))
    for k in sorted(taps.worst):
        print("  RATIO %-22s worst |got - ref| / bound %.3e  %s" % (k, taps.worst[k], taps.worst_at.get(k, "")))


STEPS = [
    # (id, step, backend, B, keep)
    ("segmenter_tc3_B16_keep0.75", "seg", "auto", 16, 0.75),      # config 2
    ("segmenter_tc3_B16_keep1", "seg", "auto", 16, 1.0),
    ("segmenter_simt_B2", "seg", "simt", 2, 0.75),
    ("segmenter_tc1_B2", "seg", "tc1", 2, 0.75),
    ("d_step_pretrain_tc3_B32", "d", "auto", 32, 0.75),           # config 3
    ("d_then_g_step_tc3_B8", "dg", "auto", 8, 0.75),              # config 4
    ("d_then_g_step_simt_B2", "dg", "simt", 2, 0.75),
    ("g_step_tc3_B16", "g", "auto", 16, 0.75),                    # the tail's backward at B = 16
    ("evaluate_tc3_B16", "eval", "auto", 16, 1.0),
]


_RESULTS = {}


def _step_result(step):
    """the tapped run of one step, once per session: the census test below needs every step, whichever tests were selected"""
    if step not in _RESULTS:
        label, kind, backend, B, keep = step
        with pytest.MonkeyPatch.context() as mp:
            taps = _tapped_step(mp, kind, backend, B, keep)
        taps._masks, taps.conv_log, taps.hook = {}, [], {}
        _report(label, taps)
        _RESULTS[step] = taps
    return _RESULTS[step]


@pytest.mark.parametrize("step", STEPS, ids=[s[0] for s in STEPS])
def test_every_layer_of_the_step_within_its_bound(step):
    label, kind, backend, B, keep = step
    taps = _step_result(step)
    got = (taps.n_fwd, taps.n_bwd, taps.n_tail_fwd, taps.n_tail_bwd)
    assert got == taps.expect, "%s: checked (layer_forward, layer_backward, tail fwd, tail bwd) %s, the graph has %s" % (
        label, got, taps.expect)
    assert not taps.fail, "%s: %d stage(s) beyond their bound:\n  %s" % (label, len(taps.fail), "\n  ".join(taps.fail[:20]))
    assert len(set(taps.fwd_sids)) == len(taps.fwd_sids), "%s: two dropout sites drew one stream id" % label
    assert set(taps.bwd_sids) <= set(taps.fwd_sids), "%s: a backward pass used a stream id no forward site drew" % label
    if keep < 1:
        assert taps.fwd_sids, "%s: no dropout site" % label


def test_steps_reach_every_route():
    union = collections.Counter()
    for step in STEPS:
        union.update(_step_result(step).census)
    missing = [r for r in ROUTES if not union[r]]
    print("\n  route census over every step: " + ", ".join("%s %d" % (r, union[r]) for r in ROUTES))
    assert not missing, "no step reached: %s" % missing


# ------------------------------------------------------------------------------------------------
# negative controls at B = 2
# ------------------------------------------------------------------------------------------------
def _stale_scratch(mp, tr):
    """(a) begin_step resets the offset but skips the fill: the fp64 BN accumulators carry the previous step's sums"""
    F, rt, _C = _prod()

    def begin_step(self):
        self.off = self.high = 0
    mp.setattr(type(rt.scratch), "begin_step", begin_step)


def _drop_plus_one(mp, tr):
    """(b) the backward pass reads its dropout mask from stream id + 1"""
    F, rt, _C = _prod()
    real = F._drop_from
    mp.setattr(F, "_drop_from", lambda info: real(None if info is None else (info[0] + 1, info[1])))


def _wrong_act(mp, tr):
    """(c) the backward pass runs with the activation code of a wrong LayerCfg copy (leaky ReLU <-> ReLU)"""
    F, rt, _C = _prod()
    real = F.layer_backward

    def bwd(sv, *a, **k):
        cfg = copy.copy(sv["cfg"])
        cfg.act = {F.ACT_LRELU: F.ACT_RELU, F.ACT_RELU: F.ACT_LRELU}.get(cfg.act, cfg.act)
        return real(dict(sv, cfg=cfg), *a, **k)
    mp.setattr(F, "layer_backward", bwd)


def _no_dx_into(mp, tr):
    """(d) _ResBlockFn.backward does not merge the skip gradient into the first convolution's dgrad"""
    F, rt, _C = _prod()

    def backward(ctx, dy):
        need_dx = ctx.needs_input_grad[0]
        dh, _ = F.layer_backward(ctx.s2, dy, True, None, need_dx)
        dx, _ = F.layer_backward(ctx.s1, dh, need_dx, None, False)
        ctx.s1 = ctx.s2 = None
        return (dx, None, None, None, None) + (None,) * (len(ctx.needs_input_grad) - 5)
    mp.setattr(F._ResBlockFn, "backward", staticmethod(backward))


# (id, mutation, stages that must each reject it)
CONTROLS = [("stale_bn_sums", _stale_scratch, ("bn_mean", "bn_invstd")),
            ("backward_stream_plus_one", _drop_plus_one, ("dz", "backward_stream_id")),
            ("wrong_activation", _wrong_act, ("dz", "g")), ("dx_into_dropped", _no_dx_into, ("block_dx",))]


@pytest.mark.parametrize("control", CONTROLS, ids=[c[0] for c in CONTROLS])
def test_negative_control_is_rejected(control, monkeypatch):
    label, mutate, stages = control
    taps = _tapped_step(monkeypatch, "seg", "auto", 2, 0.75, mutate)
    _report("control " + label, taps)
    failed = {f.split(": ")[-1].split(" ")[0] for f in taps.fail}
    assert set(stages) <= failed, "%s: stages %s did not all fail (failures: %s)" % (label, stages, taps.fail[:5])
