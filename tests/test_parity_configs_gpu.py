"""Model-level parity AT THE BENCHMARKED CONFIGURATIONS (BASELINE.json configs 2-5), CUDA path vs the CPU oracle on identical
seeded synthetic inputs and identical initial variables:

  config 4, B = 8/GPU, backend auto, through Trainer.capture_joint_step REPLAY -- the first model-level exercise of the
            dominant 128x128 wgmma tile at the benchmarked batch and of the CUDA-graph path on the wgmma backend
  config 2, B = 16: segmenter Adam steps (losses, logits)
  config 3, B = 32 per domain: pre-train D step (dis_loss, updated critic variables)
  config 5: the plain-bf16 (one MMA term) path -- its model-level deviation from the fp32 reference, stated and bounded
  CUDA graph vs eager with the critic weights perturbed between steps (a graph running on stale operands cannot pass)

Tolerance (BASELINE.json north_star): 1e-3 relative, written at each check.  Dropout off (TF's Philox stream cannot be reproduced).
"""
import numpy as np
import pytest
import torch

from tests.util import check, rel_err, l2_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _bn_noise(P, bns, seed):
    rng = np.random.RandomState(seed)
    for n, c in bns:   # non-trivial BN state so that inference-mode BN is really exercised
        P[n + "/gamma"] = (1 + 0.2 * rng.randn(c)).astype(np.float32)
        P[n + "/beta"] = (0.1 * rng.randn(c)).astype(np.float32)
        P[n + "/moving_mean"] = (0.05 * rng.randn(c)).astype(np.float32)
        P[n + "/moving_variance"] = (1 + 0.2 * rng.rand(c)).astype(np.float32)


def adv_pair(backend, lam, phase, B, with_oracle=True, lr=3e-4):
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv
    from pnp_b200.train_gan import configure
    from oracle.pnp_graphs import OracleAdversarial, init_numpy_params
    rt.set_conv_backend(backend)
    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    _bn_noise(P, bns, 6)
    for n, s in ws:   # keep the critic weights inside the clip range so the clip is exercised but not dominant
        if "cls" in n:
            P[n] = np.clip(P[n] * 0.5, -0.05, 0.05).astype(np.float32)
    ck, nc, tc = configure(phase)
    ck["lambda_mask_loss"] = lam
    tc["dis_sub_iter"] = 1
    net = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc, critic_keep_prob=1.0)
    rt.load_state_dict(P)
    trainer = adv.Trainer(net, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": lr}, train_config=tc)
    oracle = None
    if with_oracle:
        oracle = OracleAdversarial(P, B, lambda_mask_loss=lam, dis_sub_iter=1, gen_sub_iter=1, critic_keep_prob=1.0, lr=lr)
    return net, trainer, oracle


def seg_pair(backend, B, lr=1e-3):
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, source_segmenter as seg
    from oracle.pnp_graphs import OracleSegmenter, init_numpy_params
    rt.set_conv_backend(backend)
    ws, bns = OracleSegmenter.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    _bn_noise(P, bns, 5)
    ck = {"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0, "regularizer": 1e-4}
    net = seg.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=dict(ck))
    rt.load_state_dict(P)
    trainer = seg.Trainer(net, [], [], num_cls=5, batch_size=B, optimizer="adam", opt_kwargs={"learning_rate": lr})
    return net, trainer, OracleSegmenter(P, B, lr=lr), P


def loss_close(name, got, ref, scale_floor, tol=1e-3):
    den = max(abs(ref), scale_floor)
    e = abs(got - ref) / den
    print("  %-34s %.6e (oracle %.6e)  err/scale %.2e (tol %.0e)" % (name, got, ref, e, tol))
    assert np.isfinite(got) and e <= tol, (name, got, ref, e)
    return e


def state_close(rt, oracle, tol, only=None, norm=rel_err):
    ref, got = oracle.ps.to_numpy(), rt.state_dict()
    worst, wname = 0.0, None
    for n in ref:
        if only and not only(n):
            continue
        e = norm(torch.tensor(got[n]), torch.tensor(ref[n]))
        if e > worst:
            worst, wname = e, n
    print("  worst variable: %s err %.3e (tol %.0e)" % (wname, worst, tol))
    assert worst <= tol, (wname, worst)
    return worst


def test_config4_b8_tcgen05_graph_replay_matches_oracle():
    """B = 8 per domain (the benchmarked batch), backend auto, 1 warm-up step + 2 graph replays == 3 oracle joint steps"""
    from pnp_b200 import runtime as rt, functional as F
    from oracle.pnp_graphs import synthetic_images
    B = 8
    net, trainer, oracle = adv_pair("auto", 0.3, "train-gan", B)
    mr, ct, ct2 = synthetic_images(B, 1234), synthetic_images(B, 4321, 0.3, 0.8), synthetic_images(B, 8765, 0.3, 0.8)
    # the 128x128 tile must actually be selected at this batch (it is the benchmark's dominant kernel)
    F.PROFILE = []
    assert trainer.capture_joint_step(mr.to(DEV), ct.to(DEV), keep_prob=1.0, warmup=1), "CUDA-graph capture failed"
    kerns = {r[4] for r in F.PROFILE}
    F.PROFILE = None
    print("  conv kernels in the step:", sorted(kerns))
    assert any(k.startswith("conv_tc_kernel<128") for k in kerns), kerns
    ro_d, ro_g = oracle.d_step(mr, ct, 1.0), oracle.g_step(ct, 1.0)          # the warm-up step (G on the D step's CT batch)
    for k in range(2):
        d, g = trainer.joint_step(mr.to(DEV), ct.to(DEV), keep_prob=1.0, ct_batch_g=ct2.to(DEV))
        ro_d, ro_g = oracle.d_step(mr, ct, 1.0), oracle.g_step(ct2, 1.0)
        sc = 2e-3 * float(ro_d["mr_cls"].abs().max())
        loss_close("replay %d dis_loss" % k, trainer.loss_value(d), ro_d["dis_loss"], sc)
        loss_close("replay %d gen_loss" % k, trainer.loss_value(g), ro_g["gen_loss"], sc)
    state_close(rt, oracle, 1e-3)
    rt.set_conv_backend("auto")


def test_config2_b16_segmenter_train_steps():
    from pnp_b200 import runtime as rt
    from oracle.pnp_graphs import synthetic_images, synthetic_labels
    from oracle.tf14_numpy import label_decomp
    B = 16
    net, trainer, oracle, P = seg_pair("auto", B)
    x, lab = synthetic_images(B, 1234), synthetic_labels(B, 99)
    y = torch.from_numpy(label_decomp(5, lab))
    xg, yg = trainer.feed(x, torch.from_numpy(lab))
    with torch.no_grad():
        ref = oracle.forward(x, 1.0, True)
        # (a train-mode forward moves the BN moving averages on both sides alike)
        logits = net.forward(xg, keep_prob=1.0, main_bn=True, adapt_bn=True)
    check("logits B=16", logits, ref["logits"], 1e-3)
    for step in range(2):
        ro = oracle.train_step(x, y, keep_prob=1.0)
        wce, dice = trainer.train_step(xg, yg, keep_prob=1.0)
        loss_close("step %d wce" % step, float(wce), ro["wce"], 1e-6)
        loss_close("step %d dice" % step, float(dice), ro["dice"], 1e-6)
    # Adam's first updates are lr*sign(g): variables are compared in relative L2 (see test_models_gpu.py)
    state_close(rt, oracle, 2e-2, norm=l2_err)
    rt.set_conv_backend("auto")


def test_config3_b32_pretrain_discriminator_step():
    from pnp_b200 import runtime as rt
    from oracle.pnp_graphs import synthetic_images
    B = 32
    net, trainer, oracle = adv_pair("auto", 0, "pre-train", B)
    mr, ct = synthetic_images(B, 1234), synthetic_images(B, 4321, 0.3, 0.8)
    ro = oracle.d_step(mr, ct, keep_prob=1.0)
    terms = trainer.d_step(mr.to(DEV), ct.to(DEV), keep_prob=1.0)
    loss_close("dis_loss B=32", trainer.loss_value(terms), ro["dis_loss"], 2e-3 * float(ro["mr_cls"].abs().max()))
    state_close(rt, oracle, 1e-3, only=lambda n: "cls" in n)
    rt.set_conv_backend("auto")


def test_config5_plain_bf16_path_deviation_is_stated_and_bounded():
    """the one-term bf16 path (--backend tc1, BASELINE config 5) is NOT fp32-grade: state what it costs at model level.
    Measured (r2): logits 1.1e-2 of the fp32 reference's largest logit, 99.5 % argmax agreement, hard Dice within 6e-5, but the
    WGAN critic loss -- a difference of critic means -- moves by 0.15 of its scale.  Bounds: 3e-2 / 99 % / 1e-2 / 0.5 of scale.
    (The fp32-grade default path holds 1e-3 on the same quantities; config 5 is a throughput configuration, not a parity one.)"""
    from pnp_b200 import runtime as rt
    from oracle.pnp_graphs import synthetic_images, synthetic_labels
    from oracle.tf14_numpy import label_decomp
    from oracle import tf14_torch as T
    B = 2
    net, trainer, oracle, P = seg_pair("tc1", B)
    x = synthetic_images(B, 1234)
    y = torch.from_numpy(label_decomp(5, synthetic_labels(B, 99)))
    with torch.no_grad():
        ref = oracle.forward(x, 1.0, False)["logits"]
        got = net.forward(x.to(DEV), keep_prob=1.0, main_bn=False, adapt_bn=False)
    e = rel_err(got, ref)
    agree = float((got.argmax(3).cpu() == ref.argmax(3)).float().mean())
    d, _ = net.dice_eval(got, y.to(DEV))
    do, _ = T.dice_eval(ref.argmax(3), y, 5)
    print("  tc1 segmenter forward: logits rel err %.3e, argmax agreement %.6f, Dice %.6f vs %.6f" % (e, agree, float(d), float(do)))
    assert e <= 3e-2 and agree >= 0.99 and abs(float(d) - float(do)) <= 1e-2
    net, trainer, oracle = adv_pair("tc1", 0.3, "train-gan", B)
    mr, ct = synthetic_images(B, 1234), synthetic_images(B, 4321, 0.3, 0.8)
    ro = oracle.d_step(mr, ct, 1.0)
    got = trainer.loss_value(trainer.d_step(mr.to(DEV), ct.to(DEV), 1.0))
    sc = 2e-3 * float(ro["mr_cls"].abs().max())
    loss_close("tc1 dis_loss", got, ro["dis_loss"], sc, tol=0.5)
    rg = oracle.g_step(ct, 1.0)
    loss_close("tc1 gen_loss", trainer.loss_value(trainer.g_step(ct.to(DEV), 1.0)), rg["gen_loss"], sc, tol=0.5)
    rt.set_conv_backend("auto")


@pytest.mark.parametrize("backend", ["auto", "simt"])
def test_graph_replay_tracks_weights_changed_between_steps(backend):
    """A captured step must read the LIVE weights: the critic / DAM arenas are perturbed (seeded noise) after every step; a
    graph that froze operand buffers at capture time (bf16 weight planes, transposed SIMT weights) computes different losses.
    Three runs: eager, eager again (the control: fp32 atomics make two eager runs differ, and the perturbed dynamics amplify
    that), graph.  The graph run must sit as close to an eager run as the two eager runs sit to each other (x4, floor 2e-3 of
    the loss spread), while a stale-operand graph is off by the size of the perturbation's effect itself."""
    from pnp_b200 import runtime as rt
    from oracle.pnp_graphs import synthetic_images
    B = 2
    mr, ct = synthetic_images(B, 1234).to(DEV), synthetic_images(B, 4321, 0.3, 0.8).to(DEV)
    runs = []
    for use_graph in (False, False, True):
        net, trainer, _ = adv_pair(backend, 0.3, "train-gan", B, with_oracle=False, lr=3e-4)
        gen = torch.Generator(device=DEV).manual_seed(99)

        def perturb():
            for arena, amp in ((trainer.d_arena, 1e-3), (trainer.g_arena, 2e-3)):
                arena.theta.add_(torch.randn(arena.theta.shape, generator=gen, device=DEV) * amp)
                arena.bump_versions()          # whoever writes an arena owns the version bump
        losses = []
        if use_graph:
            assert trainer.capture_joint_step(mr, ct, keep_prob=1.0, warmup=1), "CUDA-graph capture failed"
        else:
            trainer.joint_step(mr, ct, keep_prob=1.0)
        perturb()
        for k in range(5):
            _junk = torch.empty(64 << 20, device=DEV)      # allocator traffic: freed warm-up buffers get reused
            d, g = trainer.joint_step(mr, ct, keep_prob=1.0)
            torch.cuda.synchronize()
            losses.append((trainer.loss_value(d), trainer.loss_value(g)))
            del _junk
            perturb()
        runs.append(losses)
    e1, e2, gr = runs
    spread = max(abs(a[0] - b[0]) for a in e1 for b in e1)
    assert spread > 1e-5, "the perturbation must move the loss, otherwise this test proves nothing (%g)" % spread
    worst_ctl = worst_gr = 0.0
    for k in range(5):
        ctl = max(abs(e1[k][0] - e2[k][0]), abs(e1[k][1] - e2[k][1])) / spread
        dev = max(abs(e1[k][0] - gr[k][0]), abs(e1[k][1] - gr[k][1])) / spread
        worst_ctl, worst_gr = max(worst_ctl, ctl), max(worst_gr, dev)
        print("  step %d  dis eager %.6e / eager %.6e / graph %.6e   |eager-eager| %.2e  |eager-graph| %.2e  (of the loss spread %.2e)"
              % (k, e1[k][0], e2[k][0], gr[k][0], ctl, dev, spread))
    assert worst_gr <= max(2e-3, 4 * worst_ctl), (worst_gr, worst_ctl)
    rt.set_conv_backend("auto")
