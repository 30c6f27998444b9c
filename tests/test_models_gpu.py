"""GPU parity of the whole hot path against the CPU oracle (oracle/pnp_graphs.py) on identical seeded
synthetic 256x256x3 inputs and identical initial variables (loaded by TF variable name):
  config 1: segmenter forward, B=2              -> logits / softmax / argmax / Dice
  config 2: segmenter Adam train step           -> losses, updated variables, BN moving statistics
  config 3: D step (pre-train, lambda=0) + clip -> dis_loss, critic logits, updated variables
  config 4: D step + G step (train-gan, lambda=0.3)
Tolerance (BASELINE.json north_star): 1e-3 relative fp32, stated per check; dropout off (keep_prob=1,
critic_keep_prob=1).  The same steps with dropout on, the oracle applying the library's own Philox masks, are
tests/test_dropout_model_gpu.py.
"""
import pytest
import torch

from tests.models import adv_pair, compare_adv_grads, grad_report, seg_pair, snapshot, state_close
from tests.util import check, rel_err, l2_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
B = 2


def _inputs():
    from oracle.pnp_graphs import synthetic_images, synthetic_labels
    from oracle.tf14_numpy import label_decomp
    x = synthetic_images(B, 1234)
    lab = synthetic_labels(B, 99)
    y = torch.from_numpy(label_decomp(5, lab))
    return x, lab, y


@pytest.mark.parametrize("backend", ["simt", "auto"])
@pytest.mark.parametrize("bn_train", [True, False])
def test_config1_segmenter_forward(backend, bn_train):
    from pnp_b200 import runtime as rt
    net, _, oracle, _ = seg_pair(backend, B)
    x, lab, y = _inputs()
    with torch.no_grad():
        ref = oracle.forward(x, 1.0, bn_train)
        logits, taps = net.forward(x.to(DEV), keep_prob=1.0, main_bn=bn_train, adapt_bn=bn_train, return_taps=True)
    for k in ("c4_2", "c6_2", "b7", "c9_2"):
        check(k, taps[k], ref[k], 1e-3)
    check("logits", logits, ref["logits"], 1e-3)
    from oracle import tf14_torch as T
    sm_ref = T.pixel_wise_softmax_2(ref["logits"])
    if bool(torch.isfinite(sm_ref).all()):      # layers.py:135 has no max subtraction: exp() overflows for large logits
        check("softmax", net.predicter(logits), sm_ref, 1e-3)
    agree = float((logits.argmax(3).cpu() == ref["logits"].argmax(3)).float().mean())
    print("  argmax agreement %.6f" % agree)
    assert agree > 0.999
    d, arr = net.dice_eval(logits, y.to(DEV))
    do, _ = T.dice_eval(ref["logits"].argmax(3), y, 5)
    assert abs(float(d) - float(do)) <= 1e-3, (float(d), float(do))
    rt.set_conv_backend("auto")


@pytest.mark.parametrize("backend", ["simt", "auto"])
def test_config2_segmenter_train_step(backend):
    from pnp_b200 import runtime as rt
    net, trainer, oracle, P = seg_pair(backend, B)
    x, lab, y = _inputs()
    xg, yg = trainer.feed(x, torch.from_numpy(lab))
    assert torch.equal(yg.cpu(), y)
    from oracle.pnp_graphs import OracleSegmenter
    g64 = OracleSegmenter(P, B, dtype=torch.float64).train_step(x.double(), y.double(), keep_prob=1.0)["grads"]
    for step in range(2):
        ro = oracle.train_step(x, y, keep_prob=1.0)
        wce, dice = trainer.train_step(xg, yg, keep_prob=1.0)
        check("step%d wce" % step, wce.reshape(1), torch.tensor([ro["wce"]]), 1e-3)
        check("step%d dice" % step, dice.reshape(1), torch.tensor([ro["dice"]]), 1e-3)
        if step == 0:
            # first-step gradients, variable by variable, against the fp64 oracle; bound calibrated by how far an fp32
            # reference implementation (the fp32 oracle) itself sits from fp64 on this ill-conditioned backward pass (grad_report)
            names = [n for n, _ in type(oracle).layout()[0]]
            bn_names = [n for n, _ in type(oracle).layout()[1]]
            all_names = names + [n + "/" + l for n in bn_names for l in ("gamma", "beta")]
            ours = []
            for n in all_names:
                v = rt.graph.vars[n]
                mult = sum(1 for w in net.conv_weights if w is v)
                ours.append(v.grad.cpu().double() + 1e-4 * mult * torch.tensor(P[n]).double())
            grad_report(all_names, ours, ro["grads"], g64, slack=4.0 if backend == "simt" else 10.0)
    # Adam's first updates are ~ lr*sign(g): elements whose gradient sits below the fp32 noise floor of this backward pass
    # (see _grad_report) may step the other way, so variables are compared in relative L2 (a few 1e-3 of the elements
    # moving by 2*lr), not max-norm; the per-step losses above are the end-to-end check at 1e-3
    state_close(rt, oracle, 2e-2, norm=l2_err, label="worst variable after 2 Adam steps: {name} l2 err {err:.3e}")
    reg = net.regularizer_loss()
    assert abs(reg - float(oracle.losses(oracle.forward(x, 1.0, False)["logits"], y)[1])) <= 1e-3 * abs(reg)
    rt.set_conv_backend("auto")


@pytest.mark.parametrize("backend", ["simt", "auto"])
def test_config3_discriminator_pretrain_step(backend):
    from pnp_b200 import runtime as rt
    from oracle.pnp_graphs import synthetic_images
    net, trainer, oracle = adv_pair(backend, 0, "pre-train", B, dis_sub_iter=3, o64=True)
    mr, ct = synthetic_images(B, 1234), synthetic_images(B, 4321, 0.3, 0.8)
    for step in range(2):
        pre = snapshot(rt)
        ro = oracle.d_step(mr, ct, keep_prob=1.0)
        terms = trainer.d_step(mr.to(DEV), ct.to(DEV), keep_prob=1.0)
        if step == 0:
            compare_adv_grads(rt, oracle, "d", ro["grads"], oracle.o64.d_step(mr.double(), ct.double(), keep_prob=1.0)["grads"], pre,
                              backend)
        got = trainer.loss_value(terms)
        print("  step %d dis_loss %.6e (oracle %.6e)" % (step, got, ro["dis_loss"]))
        assert abs(got - ro["dis_loss"]) <= 1e-3 * max(abs(ro["dis_loss"]), 2e-3 * float(ro["mr_cls"].abs().max()))
    state_close(rt, oracle, 1e-3, label="worst variable: {name} rel err {err:.3e}")
    check("dis_reg", torch.tensor([net.dis_reg()]), torch.tensor([float(oracle.dis_losses(ro["ct_cls"], ro["mr_cls"], None, None)[1])]), 1e-3)
    rt.set_conv_backend("auto")


@pytest.mark.parametrize("backend", ["simt", "auto"])
def test_config4_joint_adversarial_step(backend):
    from pnp_b200 import runtime as rt
    from oracle.pnp_graphs import synthetic_images
    net, trainer, oracle = adv_pair(backend, 0.3, "train-gan", B, dis_sub_iter=3, o64=True)
    mr, ct = synthetic_images(B, 1234), synthetic_images(B, 4321, 0.3, 0.8)
    pre = snapshot(rt)
    ro = oracle.d_step(mr, ct, keep_prob=1.0)
    terms = trainer.d_step(mr.to(DEV), ct.to(DEV), keep_prob=1.0)
    compare_adv_grads(rt, oracle, "d", ro["grads"], oracle.o64.d_step(mr.double(), ct.double(), keep_prob=1.0)["grads"], pre, backend)
    got = trainer.loss_value(terms)
    print("  dis_loss %.6e (oracle %.6e)" % (got, ro["dis_loss"]))
    assert abs(got - ro["dis_loss"]) <= 1e-3 * max(abs(ro["dis_loss"]), 2e-3 * float(ro["mr_cls"].abs().max()))
    pre = snapshot(rt)
    rg = oracle.g_step(ct, keep_prob=1.0)
    terms = trainer.g_step(ct.to(DEV), keep_prob=1.0)
    compare_adv_grads(rt, oracle, "g", rg["grads"], oracle.o64.g_step(ct.double(), keep_prob=1.0)["grads"], pre, backend)
    got = trainer.loss_value(terms)
    print("  gen_loss %.6e (oracle %.6e)" % (got, rg["gen_loss"]))
    assert abs(got - rg["gen_loss"]) <= 1e-3 * max(abs(rg["gen_loss"]), 2e-3 * float(rg["ct_cls"].abs().max()))
    state_close(rt, oracle, 1e-3, label="worst variable: {name} rel err {err:.3e}")
    rt.set_conv_backend("auto")


def test_cuda_graph_replay_equals_eager_steps():
    """Trainer.capture_joint_step: replaying the captured D+G step k times == k eager joint steps (same data, dropout off):
    the graph must carry every side effect of a step (BN moving statistics, RMSProp slots, clip, seeds) in device memory."""
    from pnp_b200 import runtime as rt
    from oracle.pnp_graphs import synthetic_images
    mr, ct = synthetic_images(B, 1234).to(DEV), synthetic_images(B, 4321, 0.3, 0.8).to(DEV)
    states = []
    for use_graph in (False, True):
        net, trainer, _ = adv_pair("simt", 0.3, "train-gan", B, dis_sub_iter=3, o64=True)
        if use_graph:
            assert trainer.capture_joint_step(mr, ct, keep_prob=1.0, warmup=1), "CUDA-graph capture failed"
            for _ in range(2):
                d, g = trainer.joint_step(mr, ct, keep_prob=1.0)
        else:
            for _ in range(3):
                d, g = trainer.joint_step(mr, ct, keep_prob=1.0)
        torch.cuda.synchronize()
        states.append((rt.state_dict(), trainer.loss_value(d), trainer.loss_value(g)))
    (sa, da, ga), (sb, db, gb) = states
    worst = max(rel_err(torch.tensor(sb[n]), torch.tensor(sa[n])) for n in sa)
    print("  graph vs eager after 3 joint steps: worst variable rel err %.3e, dis_loss %.6e / %.6e" % (worst, da, db))
    # fp32 atomics (wgrad, BN partials) make two runs differ at the 1e-5 level; the critic means are differences of O(1) logits
    assert worst <= 1e-4 and abs(da - db) <= 1e-3 * max(abs(da), 1e-3) and abs(ga - gb) <= 1e-3 * max(abs(ga), 1e-3)
    rt.set_conv_backend("auto")
