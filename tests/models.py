"""The model-level builders of the parity tests: the product's segmenter / adversarial network and trainer next to the CPU
oracle on identical seeded initial variables, the loss and variable comparisons between them, and the real training steps that
the in-step taps (tests/test_layer_taps_gpu.py, tests/test_node_taps_gpu.py) run."""
import json
import os

import numpy as np
import torch

from tests.util import l2_err, rel_err

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def bn_noise(P, bns, seed):
    rng = np.random.RandomState(seed)
    for n, c in bns:   # non-trivial BN state so that inference-mode BN is really exercised
        P[n + "/gamma"] = (1 + 0.2 * rng.randn(c)).astype(np.float32)
        P[n + "/beta"] = (0.1 * rng.randn(c)).astype(np.float32)
        P[n + "/moving_mean"] = (0.05 * rng.randn(c)).astype(np.float32)
        P[n + "/moving_variance"] = (1 + 0.2 * rng.rand(c)).astype(np.float32)


def adv_pair(backend, lam, phase, B, with_oracle=True, lr=3e-4, dis_sub_iter=1, o64=False, critic_keep_prob=1.0):
    """-> (net, trainer, oracle); o64: the oracle carries an fp64 companion as oracle.o64; critic_keep_prob: both sides' critic
    dropout (the reference hard-wires 0.75)"""
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv
    from pnp_b200.train_gan import configure
    from oracle.pnp_graphs import OracleAdversarial, init_numpy_params
    rt.set_conv_backend(backend)
    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 6)
    for n, s in ws:   # keep the critic weights inside the clip range so the clip is exercised but not dominant
        if "cls" in n:
            P[n] = np.clip(P[n] * 0.5, -0.05, 0.05).astype(np.float32)
    ck, nc, tc = configure(phase)
    ck["lambda_mask_loss"] = lam
    tc["dis_sub_iter"] = dis_sub_iter
    net = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc, critic_keep_prob=critic_keep_prob)
    rt.load_state_dict(P)
    trainer = adv.Trainer(net, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": lr}, train_config=tc)
    oracle = None
    if with_oracle:
        kw = dict(lambda_mask_loss=lam, dis_sub_iter=dis_sub_iter, gen_sub_iter=1, critic_keep_prob=critic_keep_prob, lr=lr)
        oracle = OracleAdversarial(P, B, **kw)
        if o64:
            oracle.o64 = OracleAdversarial(P, B, dtype=torch.float64, **kw)
    return net, trainer, oracle


def seg_pair(backend, B, lr=1e-3, dtype=torch.float32, optimizer="adam", **net_kw):
    """-> (net, trainer, oracle, initial variables); dtype: the oracle's (which always steps with Adam and trains every variable);
    net_kw: further arguments of the product's Full_DRN (main_trainable, adapt_trainable)"""
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, source_segmenter as seg
    from oracle.pnp_graphs import OracleSegmenter, init_numpy_params
    rt.set_conv_backend(backend)
    ws, bns = OracleSegmenter.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 5)
    ck = {"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0, "regularizer": 1e-4}
    net = seg.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=dict(ck), **net_kw)
    rt.load_state_dict(P)
    trainer = seg.Trainer(net, [], [], num_cls=5, batch_size=B, optimizer=optimizer, opt_kwargs={"learning_rate": lr})
    return net, trainer, OracleSegmenter(P, B, dtype=dtype, lr=lr), P


class PhiloxMasks:
    """Stand-in for oracle.tf14_torch.dropout that applies the library's own dropout masks (oracle/philox.py), so that the oracle
    can follow a training step with dropout on.  The masks come from the stream-id contract of runtime._Rng, not from the
    product's state:
      * manual_seed(S) stores s0 = S & (2^63 - 1); every executed step advances the seed once before its forward pass, so step
        k (1-based, counting every D, G and segmenter step that runs kernels) reads seed_advance(s0, k);
      * every dropout site with keep < 1 draws the next stream id, counting from 1 after manual_seed, in execution order.
    Site n of the current step multiplies x by dropout_mult(seed, id, keep, x.numel()) laid over x's NHWC flat index, cast to x's
    dtype (so an fp64 oracle multiplies by the exact fp32 values 0 and fl32(1/keep)).  keep >= 1 is the identity and draws no id.
    Masks are cached by (seed, id, keep, n), so the fp32 and the fp64 oracle of one step see the same ones; moving to another
    step drops the other seeds' masks (a B = 2 adversarial step draws ~70 M of them).  `seen` records the (shape, keep) of every
    call."""

    def __init__(self, seed):
        self.s0 = int(seed) & 0x7FFFFFFFFFFFFFFF
        self.k = 0          # the step whose seed the next site reads
        self.sid = 0        # the last stream id drawn
        self.cache = {}
        self.seen = []

    def at(self, k, sid):
        """the next sites belong to step k and draw ids sid + 1, sid + 2, ..."""
        self.k, self.sid = k, sid
        s = self.seed()
        self.cache = {key: v for key, v in self.cache.items() if key[0] == s}
        return self

    def seed(self, k=None):
        from oracle import philox
        return philox.seed_advance(self.s0, self.k if k is None else k)

    def mult(self, seed, sid, keep, n):
        """[n] fp32: dropout_mult(seed, sid, keep, n), the kept elements cached as a bool map"""
        from oracle import philox
        key = (seed, sid, float(keep), n)
        if key not in self.cache:
            self.cache[key] = torch.from_numpy(philox.dropout_mult(seed, sid, keep, n) != 0)
        return torch.where(self.cache[key], torch.tensor(float(philox.inv_keep(keep))), torch.tensor(0.0))

    def __call__(self, x, keep_prob, mask=None):
        assert mask is None, "the stand-in draws its own mask"
        self.seen.append((tuple(x.shape), float(keep_prob)))
        if keep_prob >= 1.0:
            return x
        self.sid += 1
        m = self.mult(self.seed(), self.sid, keep_prob, x.numel())
        return x * m.reshape(x.shape).to(device=x.device, dtype=x.dtype)


def grad_report(names, ours, g32, g64, slack=4.0, floor=2e-3):
    """first-step gradients, variable by variable, in relative L2 against the fp64 oracle: the product may sit `slack` times as
    far from fp64 as the fp32 oracle does (+ floor).  Returns (ours, fp32 oracle) worst errors"""
    wp = wo = 0.0
    for n, a, b32, b64 in zip(names, ours, g32, g64):
        if float(b64.abs().max()) == 0.0:
            assert float(a.abs().max()) == 0.0, n
            continue
        ep, eo = l2_err(a, b64), l2_err(b32, b64)
        if ep > max(floor, slack * eo):
            print("  grad %-40s l2 err %.3e (fp32 oracle %.3e)" % (n, ep, eo))
        wp, wo = max(wp, ep), max(wo, eo)
    print("  worst gradient l2 err vs fp64 oracle: ours %.3e, fp32 oracle %.3e" % (wp, wo))
    assert wp <= slack * wo + floor, (wp, wo)
    return wp, wo


def snapshot(rt):
    """every variable before a step (the weight-decay fold of adv_grads reads them)"""
    return {n: rt.graph.vars[n].detach().cpu().clone() for n in rt.graph.order}


def adv_grads(rt, oracle, which, pre):
    """-> (names, the product's gradients of an adversarial step).  The optimizer's L2 term is folded into its kernel on our
    side: wd * theta (theta from `pre`, the variables before the step) is added before comparing"""
    if which == "d":
        names = oracle.cls_w + [n + "/" + l for n in oracle.cls_bn for l in ("gamma", "beta")]
        wd = {n: oracle.gan_reg * oracle.miu_dis * 2.0 / oracle.dis_sub_iter * (1.0 if n.startswith("cls_scope") else oracle.lam)
              for n in oracle.cls_w}
    else:
        names = oracle.adapt_w + [n + "/" + l for n in oracle.adapt_bn for l in ("gamma", "beta")]
        wd = {n: oracle.gan_reg * oracle.miu_gen / oracle.gen_sub_iter for n in oracle.adapt_w}
    ours = []
    for n in names:
        a = rt.graph.vars[n].grad.cpu().double()
        if n in wd:
            a = a + wd[n] * pre[n].double()
        ours.append(a)
    return names, ours


def compare_adv_grads(rt, oracle, which, g32, g64, pre, backend="simt"):
    """first-step gradients of an adversarial step against the fp64 oracle.  fp32 SIMT path: as accurate as an fp32 reference
    (slack 4); the bf16-split tensor-core path carries ~1e-5 per conv instead of ~1e-7, amplified by the same BN-backward
    cancellation: slack 10"""
    names, ours = adv_grads(rt, oracle, which, pre)
    return grad_report(names, ours, g32, g64, slack=4.0 if backend == "simt" else 10.0)


def loss_close(name, got, ref, scale_floor, tol=1e-3):
    den = max(abs(ref), scale_floor)
    e = abs(got - ref) / den
    print("  %-34s %.6e (oracle %.6e)  err/scale %.2e (tol %.0e)" % (name, got, ref, e, tol))
    assert np.isfinite(got) and e <= tol, (name, got, ref, e)
    return e


def state_close(rt, oracle, tol, only=None, norm=rel_err, label="worst variable: {name} err {err:.3e} (tol {tol:.0e})"):
    """the largest error `norm` of a product variable against the oracle's, printed with `label`"""
    ref, got = oracle.ps.to_numpy(), rt.state_dict()
    worst, wname = 0.0, None
    for n in ref:
        if only and not only(n):
            continue
        e = norm(torch.tensor(got[n]), torch.tensor(ref[n]))
        if e > worst:
            worst, wname = e, n
    print("  " + label.format(name=wname, err=worst, tol=tol))
    assert worst <= tol, (wname, worst)
    return worst


# ------------------------------------------------------------------------------------------------
# the real training steps of the in-step taps
# ------------------------------------------------------------------------------------------------
def reference_trace():
    with open(os.path.join(GOLDEN, "reference_graph_trace.json")) as f:
        return json.load(f)


def trace_counts(op="conv"):
    """events of kind `op` ("conv", "maxpool", "fc", "PS") per sub-graph of the reference's recorded graphs"""
    ref = reference_trace()
    count = lambda evs: sum(1 for e in evs if e["op"] == op)  # noqa: E731
    sec = lambda s: [e for e in ref["events"] if e["section"] == s]  # noqa: E731
    return {"source_segmenter": count(ref["source_segmenter"]["events"]),
            # one adversarial stream: half of the zip network (the MR and the CT front) + the shared second half
            "stream": count(sec("create_zip_network#1")) // 2 + count(sec("create_second_half#1")),
            "classifier": count(sec("create_classifier#1")), "mask_critic": count(sec("create_mask_critic#1"))}


def step_images(B, seed, shift=0.0, scale=1.0):
    from oracle.pnp_graphs import synthetic_images
    return synthetic_images(B, seed, shift, scale).to("cuda")


def step_onehot(B, seed):
    from oracle.pnp_graphs import synthetic_labels
    return torch.nn.functional.one_hot(torch.from_numpy(synthetic_labels(B, seed)), 5).float().to("cuda")


def build_step(kind, backend, B):
    """one training step of kind "seg" (segmenter), "d" (pre-train critic step), "g" (generator step), "dg" (critic then
    generator step) or "eval" (the folded CT evaluation) -> (run(keep_prob), expected (layer_forward, layer_backward, tail forward,
    tail backward) counts of one run, trainer)"""
    n = trace_counts()
    if kind == "seg":
        net, tr, _, _ = seg_pair(backend, B)
        x, y = step_images(B, 11), step_onehot(B, 12)
        ns = n["source_segmenter"]           # the output convolution trains: it runs through layer_forward
        return (lambda kp: tr.train_step(x, y, kp)), (ns, ns, 0, 0), tr
    from pnp_b200.train_gan import configure
    phase = "pre-train" if kind == "d" else "train-gan"
    lam = configure(phase)[0]["lambda_mask_loss"]
    net, tr, _ = adv_pair(backend, lam, phase, B, with_oracle=False, critic_keep_prob=0.75)
    mr, ct, ct2 = step_images(B, 21), step_images(B, 22, 0.3, 0.8), step_images(B, 23, 0.3, 0.8)
    seg_l = n["stream"] - 1                  # the frozen output convolution runs inside _TailFn
    critics = n["classifier"] + (n["mask_critic"] if lam else 0)
    d_counts = (2 * seg_l + 2 * critics, 2 * critics, 2, 0)
    g_counts = (seg_l + critics, seg_l + critics, 1, 1)
    if kind == "d":
        return (lambda kp: tr.d_step(mr, ct, kp)), d_counts, tr
    if kind == "g":
        return (lambda kp: tr.g_step(ct2, kp)), g_counts, tr
    if kind == "dg":
        return (lambda kp: (tr.d_step(mr, ct, kp), tr.g_step(ct2, kp))), tuple(a + b for a, b in zip(d_counts, g_counts)), tr
    labels = step_onehot(B, 24)
    return (lambda kp: tr.evaluate(ct, labels)), (seg_l, 0, 1, 0), tr


def prepare_step(monkeypatch, kind, backend, B, keep, seed, mutate=None):
    """a fresh graph and trainer for build_step's step, the RNG seeded, mutate(monkeypatch, trainer) applied (a negative control),
    and the step run once untapped, so that the dispatcher has proven its tensor-core geometries -> (run, expected counts,
    trainer)"""
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F, runtime as rt
    rt.reset_default_graph()
    F._tc_proven.clear()
    F._tc_declined.clear()
    run, expect, tr = build_step(kind, backend, B)
    rt.manual_seed(seed)
    if mutate is not None:
        mutate(monkeypatch, tr)
    run(keep)
    torch.cuda.synchronize()
    return run, expect, tr
