"""The training steps with dropout ON -- the configuration train_segmenter.py / train_gan.py train with (--keep-prob 0.75, critics
hard-wired to 0.75) and bench.py measures, as CUDA-graph replays -- against the CPU oracle fed the library's own Philox masks.

The oracle's dropout (oracle/tf14_torch.dropout) is replaced by tests/models.PhiloxMasks, which derives every mask from the
stream-id contract of runtime._Rng alone: step k (every D, G and segmenter step that executes kernels counts, a graph capture
does not) reads seed_advance(s0, k), and the dropout sites draw stream ids 1, 2, ... after manual_seed in execution order.  Dropout
sites (keep < 1) per sub-graph, counted against the reference's own graph in tests/test_dropout_model_cpu.py:
    segment (front 21 + back 11) 32 | feature critic 16 | mask critic 8
    D step 112 (lambda != 0) / 96 (lambda = 0) | G step 56 (lambda != 0) | segmenter step 32

So the forward / backward wiring of the masks is checked end to end: the stream id a backward pass rebuilds (functional._drop_from),
the once-per-step seed advance, every backward route that applies a mask (BN direct with and without coefficients, the g route, the
no-BN pnp_dropout_apply route of group_1's first convolution and the SYMMETRIC group_10 convolution, the folded inference-BN
epilogue, the fused tail, SIMT, cold and warmed dispatcher routes), and the seed advance inside a captured graph.  Each step also
asserts the contract values themselves: the device seed (read as uint64) and rt.rng.counter.

Bars are those of the dropout-off parity tests (test_models_gpu.py, test_parity_configs_gpu.py).  The negative controls rerun the
fp32 oracle with a wrong mask (seed not advanced, or stream ids offset by one) and require the product to sit more than 20x the bar
away from it: the compared quantities do depend on the masks.
"""
import copy
import time

import numpy as np
import pytest
import torch

from tests.models import PhiloxMasks, adv_pair, compare_adv_grads, grad_report, loss_close, seg_pair, snapshot, state_close
from tests.util import check, l2_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
B = 2
KEEP = 0.75
SEED = 0x5EED_D20F_0A75
SEG, CLS, MASK = 32, 16, 8                       # dropout sites per sub-graph
N_D = {0.0: 2 * SEG + 2 * CLS, 0.3: 2 * SEG + 2 * CLS + 2 * MASK}      # 96 / 112
N_G = SEG + CLS + MASK                                                 # 56
CONTROL = 20.0


@pytest.fixture(scope="module", autouse=True)
def _wall_time():
    t0 = time.time()
    yield
    print("\n  tests/test_dropout_model_gpu.py wall time %.1f s" % (time.time() - t0))


@pytest.fixture
def masks(monkeypatch):
    """the oracle's dropout -> the library's Philox masks; the dispatcher starts cold (no geometry proven on the tensor cores)"""
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F, runtime as rt
    from oracle import tf14_torch as T
    m = PhiloxMasks(SEED)
    monkeypatch.setattr(T, "dropout", m)
    F._tc_proven.clear()
    F._tc_declined.clear()
    yield m
    rt.set_conv_backend("auto")


def _contract(rt, masks, k, what):
    """the device seed after step k is seed_advance(s0, k); the host has drawn exactly the ids the oracle drew"""
    seed = int(rt.rng.seed_t.item()) & 0xFFFFFFFFFFFFFFFF
    print("  %-22s device seed %#018x (seed_advance(s0, %d) %#018x), stream ids drawn %d (oracle %d)"
          % (what, seed, k, masks.seed(k), rt.rng.counter, masks.sid))
    assert seed == masks.seed(k), (what, hex(seed), hex(masks.seed(k)))
    assert rt.rng.counter == masks.sid, (what, rt.rng.counter, masks.sid)


def _seg_inputs():
    from oracle.pnp_graphs import synthetic_images, synthetic_labels
    from oracle.tf14_numpy import label_decomp
    lab = synthetic_labels(B, 99)
    return synthetic_images(B, 1234), lab, torch.from_numpy(label_decomp(5, lab))


def _adv_inputs(B=B):
    from oracle.pnp_graphs import synthetic_images
    return synthetic_images(B, 1234), synthetic_images(B, 4321, 0.3, 0.8), synthetic_images(B, 8765, 0.3, 0.8)


def _seg_grads(rt, net, oracle, pre):
    """-> (names, the product's gradients of a segmenter step + the L2 term its Adam kernel folds: 1e-4 * multiplicity * theta)"""
    names = [n for n, _ in type(oracle).layout()[0]]
    names += [n + "/" + l for n, _ in type(oracle).layout()[1] for l in ("gamma", "beta")]
    ours = []
    for n in names:
        v = rt.graph.vars[n]
        mult = sum(1 for w in net.conv_weights if w is v)
        ours.append(v.grad.cpu().double() + 1e-4 * mult * torch.as_tensor(np.asarray(pre[n])).double())
    return names, ours


def _grad_control(what, ours, wrong, g64, bar):
    """the product's gradients against an fp32 oracle that used a wrong mask: the median variable (relative L2) must sit more than
    CONTROL x the gradient bar away"""
    d = [l2_err(a, w) for a, w, b in zip(ours, wrong, g64) if float(b.abs().max()) != 0.0]
    med = float(np.median(d))
    print("  control %-26s gradient l2 distance min %.3e median %.3e max %.3e over %d variables (%.0f x bar = %.3e)"
          % (what, min(d), med, max(d), len(d), CONTROL, CONTROL * bar))
    assert med > CONTROL * bar, (what, med, bar)


def _loss_scale(ro):
    return 2e-3 * float(ro["mr_cls"].abs().max())


# ---- (a) segmenter Adam steps: step 1 takes the cold dispatcher routes, step 2 the warmed ones ----------------------------------
@pytest.mark.parametrize("backend", ["simt", "auto"])
def test_segmenter_adam_steps(backend, masks):
    from pnp_b200 import runtime as rt
    from oracle.pnp_graphs import OracleSegmenter
    net, trainer, oracle, P = seg_pair(backend, B)
    x, lab, y = _seg_inputs()
    xg, yg = trainer.feed(x, torch.from_numpy(lab))
    rt.manual_seed(SEED)
    slack = 4.0 if backend == "simt" else 10.0
    for k in (1, 2):                               # step k: seed k, ids (k-1)*32 + 1 .. k*32
        if k == 1:
            masks.at(1, 0)
            g64 = OracleSegmenter(P, B, dtype=torch.float64).train_step(x.double(), y.double(), keep_prob=KEEP)["grads"]
        masks.at(k, (k - 1) * SEG)
        ro = oracle.train_step(x, y, keep_prob=KEEP)
        assert masks.sid == k * SEG
        wce, dice = trainer.train_step(xg, yg, keep_prob=KEEP)
        _contract(rt, masks, k, "segmenter step %d" % k)
        check("step %d wce" % k, wce.reshape(1), torch.tensor([ro["wce"]]), 1e-3)
        check("step %d dice" % k, dice.reshape(1), torch.tensor([ro["dice"]]), 1e-3)
        if k == 1:
            names, ours = _seg_grads(rt, net, oracle, P)
            wp, wo = grad_report(names, ours, ro["grads"], g64, slack=slack)
            if backend == "simt":
                # negative controls (fp32 oracle only): the seed not advanced (k = 0), the ids offset by one.  On the simt bar
                # (4x the fp32 oracle's distance from fp64): gradients of two different masks sit ~1.4 apart in relative L2, which
                # is less than 20x the auto bar (10x)
                for what, kk, sid in (("seed not advanced", 0, 0), ("stream ids + 1", 1, 1)):
                    masks.at(kk, sid)
                    wrong = OracleSegmenter(P, B).train_step(x, y, keep_prob=KEEP)["grads"]
                    _grad_control(what, ours, wrong, g64, slack * wo + 2e-3)
    state_close(rt, oracle, 2e-2, norm=l2_err, label="worst variable after 2 Adam steps: {name} l2 err {err:.3e} (tol {tol:.0e})")


# ---- (b) adversarial steps ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("backend", ["simt", "auto"])
def test_pretrain_discriminator_steps(backend, masks):
    """pre-train phase (lambda = 0): two D steps; step k reads seed k and ids (k-1)*96 + 1 .. k*96"""
    from pnp_b200 import runtime as rt
    net, trainer, oracle = adv_pair(backend, 0.0, "pre-train", B, dis_sub_iter=3, o64=True, critic_keep_prob=KEEP)
    mr, ct, _ = _adv_inputs()
    rt.manual_seed(SEED)
    n = N_D[0.0]
    for k in (1, 2):
        pre = snapshot(rt)
        masks.at(k, (k - 1) * n)
        ro = oracle.d_step(mr, ct, keep_prob=KEEP)
        assert masks.sid == k * n
        terms = trainer.d_step(mr.to(DEV), ct.to(DEV), keep_prob=KEEP)
        _contract(rt, masks, k, "D step %d" % k)
        if k == 1:
            masks.at(1, 0)
            g64 = oracle.o64.d_step(mr.double(), ct.double(), keep_prob=KEEP)["grads"]
            compare_adv_grads(rt, oracle, "d", ro["grads"], g64, pre, backend)
        loss_close("D step %d dis_loss" % k, trainer.loss_value(terms), ro["dis_loss"], _loss_scale(ro))
    state_close(rt, oracle, 1e-3, label="worst variable: {name} rel err {err:.3e} (tol {tol:.0e})")


@pytest.mark.parametrize("backend", ["simt", "auto"])
def test_train_gan_d_and_g_steps(backend, masks):
    """train-gan phase (lambda = 0.3): D step = step 1 (seed 1, ids 1..112), G step = step 2 (seed 2, ids 113..168)"""
    from pnp_b200 import runtime as rt
    net, trainer, oracle = adv_pair(backend, 0.3, "train-gan", B, dis_sub_iter=3, o64=True, critic_keep_prob=KEEP)
    mr, ct, _ = _adv_inputs()
    rt.manual_seed(SEED)
    nd = N_D[0.3]
    pre = snapshot(rt)
    masks.at(1, 0)
    ro = oracle.d_step(mr, ct, keep_prob=KEEP)
    assert masks.sid == nd
    terms = trainer.d_step(mr.to(DEV), ct.to(DEV), keep_prob=KEEP)
    _contract(rt, masks, 1, "D step")
    masks.at(1, 0)
    compare_adv_grads(rt, oracle, "d", ro["grads"], oracle.o64.d_step(mr.double(), ct.double(), keep_prob=KEEP)["grads"], pre, backend)
    loss_close("dis_loss", trainer.loss_value(terms), ro["dis_loss"], _loss_scale(ro))
    pre = snapshot(rt)
    masks.at(2, nd)
    rg = oracle.g_step(ct, keep_prob=KEEP)
    assert masks.sid == nd + N_G
    terms = trainer.g_step(ct.to(DEV), keep_prob=KEEP)
    _contract(rt, masks, 2, "G step")
    masks.at(2, nd)
    compare_adv_grads(rt, oracle, "g", rg["grads"], oracle.o64.g_step(ct.double(), keep_prob=KEEP)["grads"], pre, backend)
    loss_close("gen_loss", trainer.loss_value(terms), rg["gen_loss"], 2e-3 * float(rg["ct_cls"].abs().max()))
    state_close(rt, oracle, 1e-3, label="worst variable: {name} rel err {err:.3e} (tol {tol:.0e})")


# ---- (c) CUDA-graph replays, backend auto ----------------------------------------------------------------------------------------
def test_segmenter_graph_replay(masks):
    """capture_train_step(warmup=1) + 2 replays == 3 oracle steps.
    The warm-up is step 1: seed 1, ids 1..32.  The capture draws ids 33..64 and runs no kernel (its seed advance is recorded, not
    executed).  Replay r is step r + 1: seed r + 1 -- the seed advance runs inside the graph -- with the ids frozen at capture.
    No gradient check: after one Adam step (~lr * sign(g)) the fp32 and fp64 oracles already sit 0.3 apart in gradient
    (relative L2), so fp64 no longer bounds anything; the losses and the state are the check."""
    from pnp_b200 import runtime as rt
    net, trainer, oracle, P = seg_pair("auto", B)
    x, lab, y = _seg_inputs()
    xg, yg = trainer.feed(x, torch.from_numpy(lab))
    rt.manual_seed(SEED)
    assert trainer.capture_train_step(xg, yg, keep_prob=KEEP, warmup=1), "CUDA-graph capture failed"
    masks.at(1, 0)
    oracle.train_step(x, y, keep_prob=KEEP)
    masks.sid = 2 * SEG
    _contract(rt, masks, 1, "after capture")
    for r in (1, 2):
        wce, dice = trainer.train_step_replay(xg, yg, keep_prob=KEEP)
        masks.at(r + 1, SEG)
        ro = oracle.train_step(x, y, keep_prob=KEEP)
        masks.sid = 2 * SEG
        _contract(rt, masks, r + 1, "replay %d" % r)
        check("replay %d wce" % r, wce.reshape(1), torch.tensor([ro["wce"]]), 1e-3)
        check("replay %d dice" % r, dice.reshape(1), torch.tensor([ro["dice"]]), 1e-3)
    state_close(rt, oracle, 2e-2, norm=l2_err, label="worst variable after warm-up + 2 replays: {name} l2 err {err:.3e} (tol {tol:.0e})")


def _oracle_joint(o, masks, r, n, mr, ct_d, ct_g, dtype=torch.float32):
    """oracle joint step of graph step r (0 = the warm-up): D reads seed 2r + 1, G seed 2r + 2; the warm-up draws ids 1..n, every
    replay the ids the capture froze, n + 1 .. 2n"""
    nd = N_D[o.lam]
    sid = 0 if r == 0 else n
    masks.at(2 * r + 1, sid)
    ro_d = o.d_step(mr.to(dtype), ct_d.to(dtype), KEEP)
    masks.at(2 * r + 2, sid + nd)
    ro_g = o.g_step(ct_g.to(dtype), KEEP)
    assert masks.sid == sid + n
    masks.sid = 2 * n                 # what the host drew: the warm-up's ids and the capture's
    return ro_d, ro_g


@pytest.mark.parametrize("b", [2, 8])
def test_joint_graph_replay(b, masks):
    """capture_joint_step(warmup=1) + 2 replays == 3 oracle joint steps; n = N_D + N_G = 168 sites per joint step.
    Warm-up: D = step 1 (seed 1, ids 1..112), G = step 2 (seed 2, ids 113..168), G on the D step's CT batch.  The capture draws
    ids 169..336 and runs no kernel.  Replay r: D = step 2r + 1, G = step 2r + 2, with the ids frozen at capture (D 169..280,
    G 281..336), G on a fresh CT batch.
    B = 2: losses, first-replay D and G gradients against fp64, state, and the negative control on the first replay's losses.
    B = 8 (the benchmarked batch, where the 128-wide wgmma tile runs): losses and state."""
    from pnp_b200 import runtime as rt, functional as F
    net, trainer, oracle = adv_pair("auto", 0.3, "train-gan", b, dis_sub_iter=3, o64=(b == 2), critic_keep_prob=KEEP)
    o64 = oracle.__dict__.pop("o64", None)
    mr, ct, ct2 = _adv_inputs(b)
    n = N_D[0.3] + N_G
    rt.manual_seed(SEED)
    F.PROFILE = []
    assert trainer.capture_joint_step(mr.to(DEV), ct.to(DEV), keep_prob=KEEP, warmup=1), "CUDA-graph capture failed"
    kerns = {p[4] for p in F.PROFILE}
    F.PROFILE = None
    if b == 8:
        assert any(k.startswith("conv_tc_kernel<128") for k in kerns), sorted(kerns)
    _oracle_joint(oracle, masks, 0, n, mr, ct, ct)
    if o64 is not None:
        _oracle_joint(o64, masks, 0, n, mr, ct, ct, torch.float64)
    _contract(rt, masks, 2, "after capture")
    for r in (1, 2):
        pre = snapshot(rt)
        before = copy.deepcopy(oracle) if r == 1 and b == 2 else None
        d, g = trainer.joint_step(mr.to(DEV), ct.to(DEV), keep_prob=KEEP, ct_batch_g=ct2.to(DEV))
        ro_d, ro_g = _oracle_joint(oracle, masks, r, n, mr, ct, ct2)
        _contract(rt, masks, 2 * r + 2, "replay %d" % r)
        sc = _loss_scale(ro_d)
        got_d, got_g = trainer.loss_value(d), trainer.loss_value(g)
        loss_close("B=%d replay %d dis_loss" % (b, r), got_d, ro_d["dis_loss"], sc)
        loss_close("B=%d replay %d gen_loss" % (b, r), got_g, ro_g["gen_loss"], sc)
        if o64 is not None and r == 1:
            r64_d, r64_g = _oracle_joint(o64, masks, r, n, mr, ct, ct2, torch.float64)
            compare_adv_grads(rt, oracle, "d", ro_d["grads"], r64_d["grads"], pre, "auto")
            compare_adv_grads(rt, oracle, "g", ro_g["grads"], r64_g["grads"], pre, "auto")
        if before is not None:
            # negative controls (fp32 oracle only): the replay reuses the warm-up's last seed (2) for D and G, or every id is off by one
            for what, kd, kg, sid in (("seed not advanced", 2, 2, n), ("stream ids + 1", 3, 4, n + 1)):
                o = copy.deepcopy(before)
                masks.at(kd, sid)
                wd = o.d_step(mr, ct, KEEP)["dis_loss"]
                masks.at(kg, sid + N_D[0.3])
                wg = o.g_step(ct2, KEEP)["gen_loss"]
                ed, eg = abs(got_d - wd) / max(abs(wd), sc), abs(got_g - wg) / max(abs(wg), sc)
                print("  control %-26s dis_loss %.2e, gen_loss %.2e of scale from the product (%.0f x bar = %.0e)"
                      % (what, ed, eg, CONTROL, CONTROL * 1e-3))
                assert ed > CONTROL * 1e-3 and eg > CONTROL * 1e-3, (what, ed, eg)
            masks.sid = 2 * n
    state_close(rt, oracle, 1e-3, label="worst variable after warm-up + 2 replays: {name} rel err {err:.3e} (tol {tol:.0e})")
