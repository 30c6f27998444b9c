"""Every non-convolution node and every gradient hand-off of real training steps, at the benchmarked batches, held to fp64
references fed the kernels' own inputs (oracle/node_exact.py).

The steps are those of tests/test_layer_taps_gpu.py: each runs once untapped, then once tapped, eagerly.  Taps installed with
monkeypatch wrap the autograd Functions of the step graph (apply, forward and backward), functional.layer_backward, the
confusion counts, torch.autograd.backward and the optimizers' step.  They check:
- node stages, each as soon as it has run: max-pool forward / backward, the disc-input gather and its backward (which adds c4's
  three tiles), the channel slice of the logits' gradient, the segmenter's phase shift, FC forward / dx / dw (dw against the arena
  slot as it was before the call), the WGAN mean combos, the seg-loss accumulator, losses, coef and dlogits, the confusion counts;
- the tensor ledger: every tensor a tapped node produces that needs a gradient carries a hook; the gradient autograd delivers
  must equal the fp64 sum of what the consumers' backwards returned for it (views count as their base), within gamma_{k-1}
  sum|g_i|, and no backward may return None for an activation that needs a gradient (variables take theirs in the arena);
- the seeds handed to torch.autograd.backward against the coefficients of tests/golden/reference_config.json;
- the variable ledger, just before the optimizer runs: each arena variable's gradient against the fp64 sum of the contributions
  launched for it in this step, from the zeroed arena (the convolution weight, gamma and beta gradients as the layer launches
  changed them -- tests/test_layer_taps_gpu.py holds each launch to its reference -- and each FC dw reference); every variable
  outside the optimizer's list must be left as it was;
- the optimizer hand-off: theta and the slots after the step against oracle/optim_exact.py at its TAU, with the weight decay,
  clip and learning rate built from tests/golden/reference_graph_trace.json and reference_config.json, grad_scale 1;
- the monitoring scalars (regularizer_loss, dis_reg, gen_reg, fixed_coeff_reg) against an fp64 sum of squares over the trace's
  weight lists with their multiplicities;
- the census: per step, the max-pool, FC and phase-shift nodes (a disc-input node is four phase shifts, a fused tail one) equal
  the trace's maxpool, fc and PS events.
The negative controls at B = 2 break the wiring in five ways, and each must be rejected by the check named for it."""
import collections
import json
import os
import time

import pytest
import torch

from oracle import elementwise_exact as E
from oracle import layer_exact as LX
from oracle import movement_exact as M
from oracle import node_exact as N
from oracle import optim_exact as O
from tests.models import GOLDEN, prepare_step, reference_trace, trace_counts

pytestmark = pytest.mark.gpu

SEED = 4242
SUB_ITER = (1, 1)            # build_step trains with dis_sub_iter = gen_sub_iter = 1
NODES = {"_ConvLayerFn": "conv", "_ResBlockFn": "resblock", "_TailFn": "tail", "_MaxPool2Fn": "maxpool",
         "_DiscInputFn": "disc_input", "_FCFn": "fc", "_MeanComboFn": "mean_combo", "_SegLossFn": "segloss",
         "_PhaseShiftFn": "phase_shift"}
# every stage some step reaches
STAGES = ("maxpool_fwd", "maxpool_bwd", "disc_input_fwd", "disc_input_bwd", "channel_slice", "phase_shift_fwd", "phase_shift_bwd",
          "fc_fwd", "fc_dx", "fc_dw", "mean_combo_fwd", "mean_combo_bwd", "segloss_acc", "segloss_out", "segloss_coef", "segloss_bwd",
          "confusion", "ledger", "no_none", "seed", "variable_ledger", "outside_var_list", "adam_step", "rmsprop_step",
          "monitor_regularizer_loss", "monitor_dis_reg", "monitor_gen_reg", "monitor_fixed_coeff_reg")
# every (producer, consumer) edge of the step graphs that carries a gradient; "seed" is torch.autograd.backward
EDGES = (("conv", "resblock"), ("resblock", "resblock"), ("resblock", "maxpool"), ("maxpool", "resblock"), ("resblock", "conv"),
         ("conv", "conv"), ("conv", "phase_shift"), ("phase_shift", "conv"), ("conv", "segloss"), ("segloss", "seed"),
         ("conv", "tail"), ("tail", "disc_input"), ("tail", "conv"), ("resblock", "disc_input"), ("conv", "disc_input"),
         ("disc_input", "resblock"), ("conv", "fc"), ("fc", "mean_combo"), ("mean_combo", "seed"))


def _prod():
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F, runtime as rt, optim
    return F, rt, optim


def _config():
    with open(os.path.join(GOLDEN, "reference_config.json")) as f:
        return json.load(f)


def _gan_ck(kind):
    return _config()["train_gan"]["pre-train" if kind == "d" else "train-gan"]["Full_DRN"]["cost_kwargs"]


def expected_seeds(kind):
    """the grad_tensors of every torch.autograd.backward call of one run, from the reference's configuration"""
    if kind == "eval":
        return []
    if kind == "seg":
        ck = _config()["train_segmenter"]["Full_DRN"]["cost_kwargs"]
        return [[N.f32(ck["miu_cross"] if ck["cross_flag"] else 0.0), N.f32(ck["miu_dice"] if ck["dice_flag"] else 0.0)]]
    lam = _gan_ck(kind)["lambda_mask_loss"]
    one = [1.0] + ([N.f32(lam)] if lam else [])
    return [one, one] if kind == "dg" else [one]


def expected_nodes(kind):
    """{maxpool, fc, PS}: the trace's events of one run"""
    lam = 0 if kind == "seg" else _gan_ck(kind)["lambda_mask_loss"]
    out = {}
    for op in ("maxpool", "fc", "PS"):
        n = trace_counts(op)
        if kind == "seg":
            out[op] = n["source_segmenter"]
            continue
        streams, critics = {"d": (2, 2), "g": (1, 1), "dg": (3, 3), "eval": (1, 0)}[kind]
        out[op] = streams * n["stream"] + critics * (n["classifier"] + (n["mask_critic"] if lam else 0))
    return out


class NodeTaps:
    def __init__(self, monkeypatch, kind, trainer):
        F, rt, optim = _prod()
        self.F, self.rt, self.optim = F, rt, optim
        self.mp, self.kind, self.tr = monkeypatch, kind, trainer
        self.worst, self.worst_at = {}, {}
        self.fail, self.failed = [], set()
        self.nodes = collections.Counter()
        self.edges = collections.Counter()
        self.tag = ""
        self.ctx = []                 # forward contexts of the apply calls in flight
        self.produced, self.keep = {}, []
        self.seeds = []
        self.var_sum = {}             # id(variable) -> [fp64 sum of its contributions, bound]
        self.all_vars = rt.global_variables()
        self.snap = self._grads()
        self.trace = reference_trace()

    # ---- bookkeeping ------------------------------------------------------------------------------------------------
    def stage(self, name, got, rb):
        r = LX.ratio(got.detach(), *rb)
        if r >= self.worst.get(name, 0.0):
            self.worst[name], self.worst_at[name] = r, self.tag
        if not r <= 1:
            self.fail.append("%s: %s ratio %.3e" % (self.tag, name, r))
            self.failed.add(name)
        return r

    def exact(self, name, ok, what="not bit-equal"):
        self.worst.setdefault(name, 0.0)
        if not ok:
            self.worst[name], self.worst_at[name] = float("inf"), self.tag
            self.fail.append("%s: %s %s" % (self.tag, name, what))
            self.failed.add(name)

    def _grads(self):
        return {id(v): (None if v.grad is None else v.grad.clone()) for v in self.all_vars}

    def _contribute(self, v, ref, bound):
        s = self.var_sum.get(id(v))
        if s is None:
            self.var_sum[id(v)] = [ref.reshape(v.shape).clone(), bound.reshape(v.shape).clone()]
        else:
            s[0] += ref.reshape(v.shape)
            s[1] += bound.reshape(v.shape)

    # ---- the tensor ledger ------------------------------------------------------------------------------------------
    def _entry(self, a):
        e = self.produced.get(id(a))
        if e is None and a._base is not None:
            e = self.produced.get(id(a._base))
        return e

    def _produce(self, kind, o):
        e = {"kind": kind, "shape": tuple(o.shape), "contrib": [], "from": [], "tag": self.tag}
        self.produced[id(o)] = e
        self.keep.append(o)
        o.register_hook(lambda g, e=e: self._arrived(e, g))

    def _arrived(self, e, g):
        self.tag = "ledger of %s (%s)" % (e["tag"], "+".join(e["from"]) or "no tapped consumer")
        if not e["contrib"]:
            self.exact("ledger", False, "gradient from an untapped consumer")
            return None
        ref, bound = N.ledger(e["contrib"])
        self.stage("ledger", g.reshape(ref.shape), (ref, bound))
        e["contrib"], e["done"] = [], True
        return None

    def _hand_back(self, kind, rec, ctx, res):
        for i, a in rec["inputs"]:
            if not ctx.needs_input_grad[i]:
                continue
            if i >= len(res) or res[i] is None:
                self.exact("no_none", False, "returned None for input %d, which needs a gradient" % i)
                continue
            e = self._entry(a)
            if e is None:
                self.exact("ledger", False, "input %d was produced outside the tapped nodes" % i)
                continue
            e["contrib"].append(res[i].detach().reshape(e["shape"]).clone())
            e["from"].append(kind)
            self.edges[(e["kind"], kind)] += 1
        self.worst.setdefault("no_none", 0.0)

    # ---- apply / forward / backward of the nodes ---------------------------------------------------------------------
    def _forward(self, real, ctx, *args):
        self.ctx.append(ctx)
        return real(ctx, *args)

    def _apply(self, kind, real, *args):
        F = self.F
        self.nodes[kind] += 1
        tag = "%s#%d" % (kind, self.nodes[kind])
        grabbed = []
        if kind == "segloss":                 # the kernel's own accumulator: the one _zeros_f64 slice of the forward
            rz = F._zeros_f64
            F._zeros_f64 = lambda n, dev: grabbed.append(rz(n, dev)) or grabbed[-1]
        try:
            out = real(*args)
        finally:
            if kind == "segloss":
                F._zeros_f64 = rz
        ctx = self.ctx.pop()
        torch.cuda.synchronize()
        self.tag = tag
        outs = out if isinstance(out, tuple) else (out,)
        rec = {"kind": kind, "tag": tag,
               "inputs": [(i, a) for i, a in enumerate(args) if torch.is_tensor(a) and a.grad_fn is not None]}
        if grabbed:
            rec["acc"] = grabbed[0].clone()
        with torch.no_grad():
            self._check_forward(kind, args, outs, rec)
        if any(o.requires_grad for o in outs):
            ctx._node_tap = rec
            for o in outs:
                if o.requires_grad:
                    self._produce(kind, o)
        return out

    def _check_forward(self, kind, args, outs, rec):
        if kind == "maxpool":
            self.exact("maxpool_fwd", torch.equal(outs[0], N.maxpool_fwd(args[0].contiguous())))
        elif kind == "disc_input":
            c4, c6, b7, c9, logits, r, o = args
            srcs = [t.contiguous() for t in (c4, c6, b7, c9)]
            self.exact("disc_input_fwd", torch.equal(outs[0], N.disc_input_fwd(srcs, logits.contiguous(), r, o)))
        elif kind == "phase_shift":
            X, r, G, o = args
            self.exact("phase_shift_fwd", torch.equal(outs[0], M.phase_shift_ref(X.contiguous(), r, G, o)))
        elif kind == "fc":
            self.stage("fc_fwd", outs[0], N.fc_fwd(args[0], args[1]))
        elif kind == "mean_combo":
            a, ca, b, cb = args
            self.stage("mean_combo_fwd", outs[0], N.mean_combo_fwd(a, ca, b, cb))
        elif kind == "segloss":
            logits, y = args
            C = logits.shape[-1]
            acc = rec["acc"]
            self.stage("segloss_acc", acc, N.segloss_acc(logits, y))
            (o_ref, o_b), _ = N.segloss_out(acc, logits.numel() // C, C)
            self.stage("segloss_out", torch.stack([outs[0], outs[1]]), (o_ref, o_b))

    def _backward(self, kind, real, ctx, *grads):
        rec = ctx._node_tap
        pre = None
        if kind in ("maxpool", "fc", "segloss"):
            pre = [t for t in ctx.saved_tensors]
        if kind == "fc" and ctx.w.requires_grad:
            pre.append(None if ctx.w.grad is None else ctx.w.grad.clone())
        res = real(ctx, *grads)
        res_t = res if isinstance(res, tuple) else (res,)
        torch.cuda.synchronize()
        self.tag = rec["tag"] + " bwd"
        self._check_backward(kind, ctx, rec, grads, res_t, pre)
        self._hand_back(kind, rec, ctx, res_t)
        return res

    def _check_backward(self, kind, ctx, rec, grads, res, pre):
        g = grads[0]
        if kind == "maxpool":
            self.exact("maxpool_bwd", torch.equal(res[0], N.maxpool_bwd(pre[0], g.contiguous())))
        elif kind == "phase_shift":
            B, a, b, G, r, o = ctx.meta
            self.exact("phase_shift_bwd", torch.equal(res[0], N.disc_input_bwd(g.contiguous(), r, G, 0, 1, o)))
        elif kind == "disc_input":
            B, H, W, NC, r, o, plan, ctot, off = ctx.meta
            dout = g.contiguous()
            for i, (a, b, G, coff, ntile) in enumerate(plan):
                if res[i] is not None:
                    self.exact("disc_input_bwd", torch.equal(res[i], N.disc_input_bwd(dout, r, G, coff, ntile, o)))
            if res[4] is not None:
                self.exact("channel_slice", torch.equal(res[4].reshape(-1, NC), N.channel_slice(dout, ctot, off, NC)))
        elif kind == "fc":
            x, w = pre[0], ctx.w
            if res[0] is not None:
                self.stage("fc_dx", res[0], N.fc_dx(g, w))
            if w.requires_grad:
                ref, bound = N.fc_dw(x, g, pre[1])
                self.stage("fc_dw", w.grad, (ref.reshape(w.shape), bound.reshape(w.shape)))
                self._contribute(w, *N.fc_dw(x, g))
        elif kind == "mean_combo":
            ca, cb, n, shape, has_b = ctx.meta
            if res[0] is not None:
                self.stage("mean_combo_bwd", res[0], N.mean_combo_bwd(g, ca, n, shape))
            if has_b and res[2] is not None:
                self.stage("mean_combo_bwd", res[2], N.mean_combo_bwd(g, cb, n, shape))
        elif kind == "segloss":
            logits, y, coef = pre
            C = logits.shape[-1]
            _, (c_ref, c_b) = N.segloss_out(rec["acc"], logits.numel() // C, C)
            self.stage("segloss_coef", coef, (c_ref, c_b))
            self.stage("segloss_bwd", res[0], N.segloss_bwd(logits, y, coef, float(grads[0]), float(grads[1])))

    # ---- parameter gradients of the convolution layers -----------------------------------------------------------------
    def _layer_backward(self, real, sv, dy, *a, **k):
        bn = sv["cfg"].bn
        vs = [v for v in [sv["W"]] + ([bn.gamma, bn.beta] if bn is not None else []) if v.requires_grad]
        before = [None if v.grad is None else v.grad.double() for v in vs]
        out = real(sv, dy, *a, **k)
        for v, b in zip(vs, before):
            after = v.grad.double()
            delta = after - (0.0 if b is None else b)
            # the difference of two fp32 values is exact in fp64 unless their exponents are more than 29 apart
            self._contribute(v, delta, N.U64 * (after.abs() + (0.0 if b is None else b.abs())))
        return out

    # ---- seeds, confusion counts ---------------------------------------------------------------------------------------
    def _autograd_backward(self, real, tensors, grad_tensors=None, *a, **k):
        self.seeds.append([float(g) for g in grad_tensors])
        for t, g in zip(tensors, grad_tensors):
            e = self._entry(t)
            if e is not None:
                e["contrib"].append(g.detach().reshape(e["shape"]).clone())
                e["from"].append("seed")
                self.edges[(e["kind"], "seed")] += 1
        return real(tensors, grad_tensors, *a, **k)

    def _confusion(self, real, logits, y):
        cm = real(logits, y)
        self.tag = "confusion"
        self.exact("confusion", torch.equal(cm.reshape(-1), N.confusion(logits, y)))
        return cm

    # ---- the optimizer hand-off --------------------------------------------------------------------------------------
    def _tables(self, opt):
        """(weight decay {name: wd}, clip {name: c}, lr) of this optimizer, from the reference's trace and configuration"""
        tr = self.tr
        if self.kind == "seg":
            c = _config()["train_segmenter"]
            return N.segmenter_weight_decay(self.trace, c["Full_DRN"]["cost_kwargs"]), {}, c["Trainer"]["opt_kwargs"]["learning_rate"]
        ck = _gan_ck(self.kind)
        wd_d, wd_g = N.gan_weight_decay(self.trace, ck, ck["lambda_mask_loss"], *SUB_ITER)
        d_ref, g_ref = self.trace["optimizer"]["optimizers"]
        if opt is tr.dis_optimizer:
            return wd_d, N.critic_clip(self.trace), d_ref["learning_rate"]
        assert opt is tr.gen_optimizer
        return wd_g, {}, g_ref["learning_rate"]

    def _opt_step(self, real, opt, grad_scale=1.0):
        a = opt.arena
        torch.cuda.synchronize()
        mine = {id(v) for v in a.vars}
        # the variable ledger
        for v in a.vars:
            self.tag = "variable ledger %s" % v.pnp_name
            s = self.var_sum.pop(id(v), None)
            if s is None:
                z = torch.zeros(v.shape, dtype=torch.float64, device=v.device)
                s = [z, z]
            self.stage("variable_ledger", v.grad, tuple(s))
        self.tag = "outside the var list of %s" % type(opt).__name__
        stray = [k for k in self.var_sum if k not in mine]
        self.exact("outside_var_list", not stray, "%d contribution(s) to variables outside the list" % len(stray))
        for v in self.all_vars:
            if id(v) in mine:
                continue
            was = self.snap[id(v)]
            same = (v.grad is None and was is None) or (v.grad is not None and was is not None and torch.equal(v.grad, was))
            self.exact("outside_var_list", same, "%s's gradient changed" % v.pnp_name)
        # the hand-off
        th0, g0 = a.theta.clone(), a.grad.clone()
        adam = isinstance(opt, self.optim.Adam)
        slots0 = (opt.m.clone(), opt.v.clone()) if adam else (opt.ms.clone(), opt.mom.clone())
        state0 = opt.state.tolist() if adam else None
        real(opt, grad_scale)
        torch.cuda.synchronize()
        wd, clip, lr = self._tables(opt)
        seg_wd = a.seg_table([wd.get(v.pnp_name, 0.0) for v in a.vars])
        self.tag = "%s step" % type(opt).__name__
        if adam:
            st = O.adam_advance(state0, 0.9, 0.999)
            ref = O.adam_step(th0, g0, *slots0, a.chunk_seg, seg_wd, st, 0.9, 0.999, 1e-8, 1.0)
            got = {"theta": a.theta, "m": opt.m, "v": opt.v}
        else:
            seg_clip = a.seg_table([clip.get(v.pnp_name, 0.0) for v in a.vars])
            ref = O.rmsprop_step(th0, g0, *slots0, a.chunk_seg, seg_wd, seg_clip, lr, 0.9, 0.0, 1e-10, 1.0)
            got = {"theta": a.theta, "ms": opt.ms, "mom": opt.mom}
        name = "adam_step" if adam else "rmsprop_step"
        for key, t in got.items():
            self.stage(name, t, (ref[key], O.TAU["adam" if adam else "rmsprop"] * ref["mag_" + key]))
        self.snap = self._grads()

    # ---- the monitoring scalars ----------------------------------------------------------------------------------------
    def check_regularisers(self):
        net, live = self.tr.net, self.rt.graph.vars
        rel = N.gamma(N.L2_CHAIN) + (sum(v.numel() for v in live.values()) + 16) * N.U64
        l2v = lambda n: float(E.l2_ref(live[n].detach()))  # noqa: E731
        l2b = lambda n: rel * l2v(n)  # noqa: E731
        if self.kind == "seg":
            ck = _config()["train_segmenter"]["Full_DRN"]["cost_kwargs"]
            got = {"regularizer_loss": net.regularizer_loss()}
            ref = {"regularizer_loss": N.segmenter_regulariser(self.trace, ck, l2v)}
            bnd = {"regularizer_loss": N.segmenter_regulariser(self.trace, ck, l2b)}
        else:
            ck = _gan_ck(self.kind)
            got = {"dis_reg": net.dis_reg(), "gen_reg": net.gen_reg(), "fixed_coeff_reg": net.fixed_coeff_reg()}
            ref = N.regularisers(self.trace, ck, ck["lambda_mask_loss"], l2v)
            bnd = N.regularisers(self.trace, ck, ck["lambda_mask_loss"], l2b)
        self.tag = "monitoring"
        for k in got:
            t = lambda v: torch.tensor(v, dtype=torch.float64)  # noqa: E731
            self.stage("monitor_" + k, t(got[k]), (t(ref[k]), t(bnd[k] + 8 * N.U64 * abs(ref[k]))))

    def install(self):
        F, mp = self.F, self.mp
        for cname, kind in NODES.items():
            cls = getattr(F, cname)
            rf, rb, ra = cls.forward, cls.backward, cls.apply
            mp.setattr(cls, "forward", staticmethod(lambda ctx, *a, rf=rf: self._forward(rf, ctx, *a)))
            mp.setattr(cls, "backward", staticmethod(lambda ctx, *g, rb=rb, kind=kind: self._backward(kind, rb, ctx, *g)))
            mp.setattr(cls, "apply", classmethod(lambda c, *a, ra=ra, kind=kind: self._apply(kind, ra, *a)))
        rlb = F.layer_backward
        mp.setattr(F, "layer_backward", lambda sv, dy, *a, **k: self._layer_backward(rlb, sv, dy, *a, **k))
        rcc = F.confusion_counts
        mp.setattr(F, "confusion_counts", lambda logits, y: self._confusion(rcc, logits, y))
        rab = torch.autograd.backward
        mp.setattr(torch.autograd, "backward", lambda t, g=None, *a, **k: self._autograd_backward(rab, t, g, *a, **k))
        for cls in (self.optim.Adam, self.optim.RMSProp):
            rs = cls.step
            mp.setattr(cls, "step", lambda opt, grad_scale=1.0, rs=rs: self._opt_step(rs, opt, grad_scale))

    def finish(self):
        self.tag = "after the step"
        left = [e["tag"] for e in self.produced.values() if e["contrib"]]
        self.exact("ledger", not left, "gradients returned for %s never arrived" % left[:3])
        self.exact("outside_var_list", not self.var_sum, "contributions no optimizer took")
        self.exact("seed", self.seeds == expected_seeds(self.kind), "%s, the reference's %s" % (self.seeds, expected_seeds(self.kind)))
        self.check_regularisers()
        self.produced, self.keep, self.var_sum, self.snap, self.all_vars, self.trace = {}, [], {}, None, None, None


def _tapped_step(monkeypatch, kind, backend, B, keep, mutate=None):
    run, _, tr = prepare_step(monkeypatch, kind, backend, B, keep, SEED, mutate)
    taps = NodeTaps(monkeypatch, kind, tr)
    taps.install()
    t0 = time.time()
    run(keep)
    torch.cuda.synchronize()
    taps.seconds = time.time() - t0
    taps.finish()
    monkeypatch.undo()
    taps.tr = None
    return taps


def _census(taps):
    n = taps.nodes
    return {"maxpool": n["maxpool"], "fc": n["fc"], "PS": 4 * n["disc_input"] + n["phase_shift"] + n["tail"]}


def _report(label, taps):
    print("\n  %s: nodes %s, %d ledger edges, checked in %.1f s" % (
        label, ", ".join("%s %d" % kv for kv in sorted(taps.nodes.items())), sum(taps.edges.values()), taps.seconds))
    for k in sorted(taps.worst):
        print("  RATIO %-24s worst |got - ref| / bound %.3e  %s" % (k, taps.worst[k], taps.worst_at.get(k, "")))


@pytest.fixture(autouse=True)
def _restore():
    F, rt, _ = _prod()
    yield
    F._tc_proven.clear()
    F._tc_declined.clear()
    rt.set_conv_backend("auto")


STEPS = [
    # (id, step, backend, B, keep): the steps of tests/test_layer_taps_gpu.py
    ("segmenter_tc3_B16_keep0.75", "seg", "auto", 16, 0.75),
    ("segmenter_tc3_B16_keep1", "seg", "auto", 16, 1.0),
    ("segmenter_simt_B2", "seg", "simt", 2, 0.75),
    ("segmenter_tc1_B2", "seg", "tc1", 2, 0.75),
    ("d_step_pretrain_tc3_B32", "d", "auto", 32, 0.75),
    ("d_then_g_step_tc3_B8", "dg", "auto", 8, 0.75),
    ("d_then_g_step_simt_B2", "dg", "simt", 2, 0.75),
    ("g_step_tc3_B16", "g", "auto", 16, 0.75),
    ("evaluate_tc3_B16", "eval", "auto", 16, 1.0),
]

_RESULTS = {}


def _step_result(step):
    """the tapped run of one step, once per session: the census test below needs every step, whichever tests were selected"""
    if step not in _RESULTS:
        label, kind, backend, B, keep = step
        with pytest.MonkeyPatch.context() as mp:
            taps = _tapped_step(mp, kind, backend, B, keep)
        _report(label, taps)
        _RESULTS[step] = taps
    return _RESULTS[step]


@pytest.mark.parametrize("step", STEPS, ids=[s[0] for s in STEPS])
def test_every_node_and_hand_off_of_the_step_within_its_bound(step):
    label, kind, backend, B, keep = step
    taps = _step_result(step)
    got, want = _census(taps), expected_nodes(kind)
    assert got == want, "%s: checked %s nodes, the reference graph has %s" % (label, got, want)
    assert not taps.fail, "%s: %d check(s) failed:\n  %s" % (label, len(taps.fail), "\n  ".join(taps.fail[:20]))


def test_steps_reach_every_node_stage_and_edge():
    stages, edges = set(), collections.Counter()
    for step in STEPS:
        taps = _step_result(step)
        stages |= set(taps.worst)
        edges.update(taps.edges)
    print("\n  ledger edges over every step: " + ", ".join("%s->%s %d" % (a, b, edges[(a, b)]) for a, b in sorted(edges)))
    missing = [s for s in STAGES if s not in stages]
    assert not missing, "no step reached: %s" % missing
    missing = [e for e in EDGES if not edges[e]]
    assert not missing, "no step handed a gradient along: %s" % missing
    extra = [e for e in edges if e not in EDGES]
    assert not extra, "edges outside the step graphs: %s" % extra


# ------------------------------------------------------------------------------------------------
# negative controls at B = 2
# ------------------------------------------------------------------------------------------------
def _two_tiles(mp, tr):
    """(1) _DiscInputFn.backward adds two of c4's three tiles"""
    F, _, _ = _prod()
    real = F._DiscInputFn.backward

    def backward(ctx, dout):
        meta = ctx.meta
        a, b, G, coff, _ = meta[6][0]
        ctx.meta = meta[:6] + ([(a, b, G, coff, 2)] + meta[6][1:],) + meta[7:]
        try:
            return real(ctx, dout)
        finally:
            ctx.meta = meta
    mp.setattr(F._DiscInputFn, "backward", staticmethod(backward))


def _fc_overwrites(mp, tr):
    """(2) _FCFn.backward zeroes dw before pnp_fc_bwd: the second critic call overwrites the first"""
    F, _, _ = _prod()
    real = F._FCFn.backward

    def backward(ctx, dout):
        if ctx.w.requires_grad and ctx.w.grad is not None:
            ctx.w.grad.zero_()
        return real(ctx, dout)
    mp.setattr(F._FCFn, "backward", staticmethod(backward))


def _mean_combo_drops_b(mp, tr):
    """(3) _MeanComboFn.backward returns None for b"""
    F, _, _ = _prod()
    real = F._MeanComboFn.backward

    def backward(ctx, g):
        da, _, _, _ = real(ctx, g)
        return da, None, None, None
    mp.setattr(F._MeanComboFn, "backward", staticmethod(backward))


def _lambda_seed_one(mp, tr):
    """(4) the trainer seeds the mask-critic term with 1 instead of lambda_mask_loss"""
    tr._lam.fill_(1.0)


def _single_weight_decay(mp, tr):
    """(5) the critic weights, listed twice in the reference's weight lists, decay with multiplicity 1"""
    tr.dis_optimizer.seg_wd.mul_(0.5)


# (id, mutation, checks that must each reject it)
CONTROLS = [("disc_input_two_tiles", _two_tiles, ("disc_input_bwd",)),
            ("fc_dw_overwrites", _fc_overwrites, ("fc_dw", "variable_ledger")),
            ("mean_combo_none_for_b", _mean_combo_drops_b, ("no_none",)),
            ("lambda_seed_one", _lambda_seed_one, ("seed",)),
            ("weight_decay_multiplicity_one", _single_weight_decay, ("rmsprop_step",))]

_MODEL_GRADS = {}


def _model_check_catches(mutate):
    """whether tests/test_models_gpu.py's first-step gradient check (config 4, B = 2, keep 1) rejects the mutation.  The fp32
    and fp64 oracle gradients are computed once; the product runs its D then G step with the mutation applied."""
    from pnp_b200 import runtime as rt
    from oracle.pnp_graphs import synthetic_images
    from tests.models import adv_pair, compare_adv_grads, snapshot
    B = 2
    mr, ct = synthetic_images(B, 1234), synthetic_images(B, 4321, 0.3, 0.8)
    if not _MODEL_GRADS:
        _, _, oracle = adv_pair("auto", 0.3, "train-gan", B, dis_sub_iter=3, o64=True)
        _MODEL_GRADS["oracle"] = oracle
        _MODEL_GRADS["d"] = (oracle.d_step(mr, ct, keep_prob=1.0)["grads"], oracle.o64.d_step(mr.double(), ct.double(), keep_prob=1.0)["grads"])
        _MODEL_GRADS["g"] = (oracle.g_step(ct, keep_prob=1.0)["grads"], oracle.o64.g_step(ct.double(), keep_prob=1.0)["grads"])
    oracle = _MODEL_GRADS["oracle"]
    caught = []
    with pytest.MonkeyPatch.context() as mp:
        _, trainer, _ = adv_pair("auto", 0.3, "train-gan", B, with_oracle=False, dis_sub_iter=3)
        mutate(mp, trainer)
        for which, step in (("d", lambda: trainer.d_step(mr.to("cuda"), ct.to("cuda"), keep_prob=1.0)),
                            ("g", lambda: trainer.g_step(ct.to("cuda"), keep_prob=1.0))):
            pre = snapshot(rt)
            step()
            try:
                compare_adv_grads(rt, oracle, which, *_MODEL_GRADS[which], pre, "auto")
            except AssertionError:
                caught.append(which)
    rt.set_conv_backend("auto")
    return caught


@pytest.mark.parametrize("control", CONTROLS, ids=[c[0] for c in CONTROLS])
def test_negative_control_is_rejected(control, monkeypatch):
    label, mutate, checks = control
    taps = _tapped_step(monkeypatch, "dg", "auto", 2, 0.75, mutate)
    _report("control " + label, taps)
    caught = _model_check_catches(mutate)
    print("  control %s: the model-level gradient check of test_models_gpu %s" % (
        label, ("rejects it (%s step)" % " and ".join(caught)) if caught else "does not reject it"))
    missing = [c for c in checks if c not in taps.failed]
    assert not missing, "%s: checks %s did not reject it (failures: %s)" % (label, missing, taps.fail[:5])
