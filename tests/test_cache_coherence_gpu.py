"""Every cached operand is the live variable after every writer.

The bf16 weight planes, the transposed SIMT weights and the folded inference-mode batch-norm coefficients are stamped with a
hand-maintained version counter (`pnp_version`), and whoever writes a variable owns the bump.  Each writer of the package gets
one test of the same shape: warm the caches, audit (tests/coherence.py), run the writer, audit again -- an entry that still
claims the current version must be bit for bit what the pinned kernel makes of the live values --, then run the inference
forward once on the caches as they stand and once on cold caches: the two agree to the spread two cold runs show (the split-K
layers sum through fp32 atomics).  Activation planes that travel as a tensor attribute are re-split at every consumer during
full eager steps.  Four negative controls do the forbidden thing and require the audit to name the variable."""
import numpy as np
import pytest
import torch

from tests import cabi
from tests.coherence import audit, bn_key, cache_fingerprint, drop_caches, watch_planes
from tests.models import adv_pair, seg_pair

pytestmark = pytest.mark.gpu

DEV = cabi.DEV
B = 2


def _prod():
    import pnp_b200  # noqa: F401
    from pnp_b200 import layers, functional, runtime
    return layers, functional, runtime


@pytest.fixture(autouse=True)
def _default_backend():
    yield
    _, F, rt = _prod()
    rt.set_conv_backend("auto")


def _need(counts, kinds, where):
    for k in kinds:
        assert counts[k] > 0, "%s: the audit saw no live %s entry (%r), so it proved nothing" % (where, k, counts)


def _agree(label, y_warm, y_cold, y_cold2):
    """the forward on the caches as the writer left them against the cold-cache control, at the spread of two cold runs"""
    scale = float(y_cold.abs().max())
    spread = float((y_cold - y_cold2).abs().max())
    err = float((y_warm - y_cold).abs().max())
    bound = max(8 * spread, 1e-6 * scale)
    print("  %-44s |warm - cold| %.3e, |cold - cold| %.3e, scale %.3e (bound %.3e)%s" % (
        label, err, spread, scale, bound, "  bit-equal" if torch.equal(y_warm, y_cold) else ""))
    assert np.isfinite(err) and err <= bound, (label, err, spread, scale)


def _round_trip(label, warm, writer, infer, kinds, changes=True, after=None):
    """warm -> audit -> writer -> audit -> forward -> audit -> cold-cache controls; -> the three audits' counts.
    kinds: cache kinds that must be live when warm; after: after the forward (default: the same)"""
    _, F, rt = _prod()
    warm()
    y0 = infer()
    c0 = audit(rt, F)
    _need(c0, kinds, label + ", warm")
    writer()
    c1 = audit(rt, F)
    y1 = infer()
    c2 = audit(rt, F)
    _need(c2, kinds if after is None else after, label + ", after the writer")
    drop_caches(rt)
    y2 = infer()
    drop_caches(rt)
    y3 = infer()
    print("  %-44s audited warm %r, after the writer %r, after the forward %r" % (label, c0, c1, c2))
    if changes:
        assert not torch.equal(y0, y1), "%s: the writer did not move the forward, so stale operands would go unseen" % label
    _agree(label, y1, y2, y3)
    return c0, c1, c2


# ------------------------------------------------------------------------------------------------
# the two small models
# ------------------------------------------------------------------------------------------------
class _Seg:
    def __init__(self, backend="auto", optimizer="adam", **net_kw):
        from oracle.pnp_graphs import synthetic_images, synthetic_labels
        _, F, rt = _prod()
        self.net, self.trainer, _, self.P = seg_pair(backend, B, optimizer=optimizer, **net_kw)
        self.x = synthetic_images(B, 1234).to(DEV)
        self.y = F.one_hot(torch.from_numpy(synthetic_labels(B, 99)).to(DEV), 5)

    def warm(self):
        """forward and backward of a training step without its update (Trainer.train_step up to its finish_backward, which has
        no switch for leaving the update out), then the inference forward"""
        _, F, rt = _prod()
        t = self.trainer
        t.arena.zero_grad()
        rt.scratch.begin_step()
        logits = self.net.forward(self.x, keep_prob=0.75, main_bn=True, adapt_bn=True)
        wce, dice = self.net.losses(logits, self.y)
        torch.autograd.backward([wce, dice], [t._g_cross, t._g_dice])
        self.infer()

    def infer(self):
        with torch.no_grad():
            return self.net.forward(self.x, keep_prob=1.0, main_bn=False, adapt_bn=False).clone()


class _Adv:
    def __init__(self, backend="auto"):
        from oracle.pnp_graphs import synthetic_images
        self.net, self.trainer, _ = adv_pair(backend, 0.3, "train-gan", B, with_oracle=False)
        self.mr = synthetic_images(B, 1234).to(DEV)
        self.ct = synthetic_images(B, 4321, 0.3, 0.8).to(DEV)

    def warm(self):
        self.trainer.d_step(self.mr, self.ct, 0.75, apply=False)
        self.trainer.g_step(self.ct, 0.75, apply=False)
        self.infer()
        self.critic()

    def infer(self):
        """what Trainer.evaluate runs: the adapted CT stream in inference mode"""
        with torch.no_grad():
            return self.net.segment(self.ct, "ct", 1.0, front_bn=False, joint_bn=False)["logits"].clone()

    def critic(self):
        with torch.no_grad():
            return self.net.classify(self.net.segment(self.mr, "mr", 1.0, front_bn=False, joint_bn=False)).clone()


def _noisy(state, seed, amp=0.02):
    """the variables of `state` moved by seeded noise (moving variances stay positive)"""
    rng = np.random.RandomState(seed)
    out = {}
    for k, v in state.items():
        v = np.asarray(v)
        if v.dtype != np.float32 or v.ndim == 0:
            out[k] = v
            continue
        n = amp * rng.randn(*v.shape).astype(np.float32)
        out[k] = v + (np.abs(n) if k.endswith("moving_variance") else n)
    return out


# ------------------------------------------------------------------------------------------------
# optimizer steps
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("optimizer", ["adam", "momentum"])
def test_segmenter_optimizer_step_invalidates_every_operand(optimizer):
    m = _Seg(optimizer=optimizer)
    _round_trip("%s step" % optimizer, m.warm, lambda: m.trainer.optimizer.step(), m.infer, ("planes", "bncoef"))


def test_adam_step_invalidates_the_transposed_simt_weights():
    m = _Seg(backend="simt")
    _round_trip("adam step, simt", m.warm, lambda: m.trainer.optimizer.step(), m.infer, ("wT",), after=())      # (only a backward pass reads them)


def test_rmsprop_steps_with_and_without_the_clip_table():
    m = _Adv()
    assert float(m.trainer.dis_optimizer.seg_clip.max()) > 0 and float(m.trainer.gen_optimizer.seg_clip.max()) == 0
    _round_trip("rmsprop step (no clip), DAM", m.warm, lambda: m.trainer.gen_optimizer.step(), m.infer, ("planes", "bncoef"))
    _round_trip("rmsprop step + clip, critics", m.warm, lambda: m.trainer.dis_optimizer.step(), m.critic, ("planes",))


# ------------------------------------------------------------------------------------------------
# loaders
# ------------------------------------------------------------------------------------------------
def test_load_state_dict_invalidates_every_operand():
    _, F, rt = _prod()
    m = _Seg()
    _round_trip("load_state_dict", m.warm, lambda: rt.load_state_dict(_noisy(m.P, 17)), m.infer, ("planes", "bncoef"))


def test_slot_loader_lr_update_and_clear_rms_change_no_variable():
    """the optimizer-slot loader, a learning-rate refresh and a clear_rms restore of the optimizer state write no variable: the
    audit sees the same entries, none is re-derived by the forward that follows"""
    _, F, rt = _prod()
    m = _Adv()
    m.warm()
    c0, f0 = audit(rt, F), cache_fingerprint(rt)
    _need(c0, ("planes", "bncoef"), "warm")
    t = m.trainer
    slots = _noisy(dict(t.dis_optimizer.slot_state(), **t.gen_optimizer.slot_state()), 23)
    assert t.dis_optimizer.load_slot_state(slots) > 0 and t.gen_optimizer.load_slot_state(slots) > 0
    slots["pnp/learning_rate"] = np.float32(1e-4)
    assert t.load_optimizer_state(slots, clear_rms=True) == 0
    t.dis_optimizer.set_lr(t.LR_refresh)
    t.gen_optimizer.set_lr(t.LR_refresh)
    assert audit(rt, F) == c0 and cache_fingerprint(rt) == f0
    m.infer()
    m.critic()
    assert audit(rt, F) == c0 and cache_fingerprint(rt) == f0, "a forward after writers that change no variable re-derived operands"


@pytest.mark.parametrize("mode", ["full", "clear_rms", "relaxed", "no_gan"])
def test_restore_invalidates_every_operand(mode, tmp_path):
    from pnp_b200.lib import _save
    m = _Adv()
    st = _noisy(m.trainer.checkpoint_state(), 31)
    if mode == "relaxed":
        del st["cls_scope/cls_out/Variable"]           # a checkpoint that lacks a variable of the graph takes the relaxed branch
    ck = _save(st, str(tmp_path / "model.cpkt"))
    kw = {"clear_rms": True} if mode == "clear_rms" else ({"no_gan": True} if mode == "no_gan" else {})

    def writer():
        m.net.restore(ck, **kw)
        m.trainer.load_optimizer_state(m.net.last_restored, clear_rms=(mode == "clear_rms"))
    _round_trip("restore (%s)" % mode, m.warm, writer, m.infer, ("planes", "bncoef"))


def test_baseline_transplant_invalidates_every_operand(tmp_path):
    """restore(no_gan) + load_batch_norm_weights + adapt_copy_weights, audited after each"""
    from pnp_b200.lib import _save
    _, F, rt = _prod()
    seg = _Seg()
    ck = _save(_noisy(rt.state_dict(), 41, amp=0.05), str(tmp_path / "baseline.cpkt"))
    m = _Adv()
    seen = []

    def writer():
        m.net.restore(ck, no_gan=True)
        seen.append(audit(rt, F))
        m.net.load_batch_norm_weights(ck)
        seen.append(audit(rt, F))
        m.net.adapt_copy_weights()
    _round_trip("baseline transplant", m.warm, writer, m.infer, ("planes", "bncoef"))
    assert all(c["stale"] > 0 for c in seen), seen


def test_checkpoint_reread_after_saving_leaves_the_operands_coherent(tmp_path):
    """Trainer.train re-reads the checkpoint it has just written"""
    import os
    m = _Adv()

    def writer():
        m.trainer.save(str(tmp_path / "model.cpkt"), str(tmp_path))
        m.net.restore(os.path.join(str(tmp_path), "latest.npz"))
        assert m.trainer.load_optimizer_state(m.net.last_restored) > 0
    _round_trip("checkpoint re-read", m.warm, writer, m.infer, ("planes", "bncoef"), changes=False)


# ------------------------------------------------------------------------------------------------
# train-mode batch norm as a writer of the moving statistics
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("route", ["layer_forward", "layers_batch_norm"])
def test_train_mode_bn_then_inference_folds_the_new_statistics(route):
    """a batch norm with frozen gamma / beta runs once in training mode: the only thing that changes the coefficient cache's key is
    the bump of its moving statistics"""
    L, F, rt = _prod()
    rt.reset_default_graph()
    rt.set_conv_backend("auto")
    C = 64
    W = L.weight_variable([3, 3, C, C], stddev=0.05, trainable=False)
    bn = L.bn_variables("t", C, trainable=False)
    g = cabi.dev_gen(5)
    with torch.no_grad():
        bn.gamma.copy_(1 + 0.3 * torch.randn(C, generator=g, device=DEV))
        bn.beta.copy_(0.2 * torch.randn(C, generator=g, device=DEV))
    x = torch.randn(4, 32, 32, C, generator=g, device=DEV)
    x2 = 3 * torch.randn(4, 32, 32, C, generator=g, device=DEV) + 1

    def infer():
        with torch.no_grad():
            return L.conv_bn_relu2d(x, W, 1.0, is_train=False, scope="t", bn_trainable=False, leak=True).clone()

    def writer():
        before = bn.moving_mean.clone()
        with torch.no_grad():
            if route == "layer_forward":
                L.conv_bn_relu2d(x2, W, 1.0, is_train=True, scope="t", bn_trainable=False, leak=True)
            else:
                L.batch_norm(x2, is_training=True, scope="t", trainable=False)
        assert not torch.equal(before, bn.moving_mean)
    c0, c1, c2 = _round_trip("train-mode BN (%s)" % route, lambda: None, writer, infer, ("planes", "bncoef"))
    assert c1["bncoef"] == 0 and c1["stale"] == 1, c1          # the old coefficients are recognisably stale, not wrong


def test_quirk_pass_outside_a_step_then_val_stats():
    """the segmenter's monitoring pass runs batch-statistics BN outside any step (the reference's quirk): the inference pass
    that follows must fold the statistics it moved"""
    m = _Seg()
    _round_trip("output_minibatch_stats", m.warm, lambda: m.trainer.output_minibatch_stats(m.x, m.y), m.infer, ("planes", "bncoef"))
    s1 = m.trainer.val_stats(m.x, m.y)
    _, F, rt = _prod()
    drop_caches(rt)
    s2 = m.trainer.val_stats(m.x, m.y)
    assert abs(s1["loss"] - s2["loss"]) <= 1e-5 * max(1.0, abs(s2["loss"])) and abs(s1["dice_eval"] - s2["dice_eval"]) <= 1e-5, (s1, s2)


# ------------------------------------------------------------------------------------------------
# graph replay
# ------------------------------------------------------------------------------------------------
def _bn_snapshot(rt):
    """{gamma name: (moving statistics, coefficient-cache key)} of every batch norm of the graph"""
    snap = {}
    for name in rt.graph.order:
        if name.endswith("/gamma"):
            scope = name[:-len("/gamma")]
            mm, mv = rt.graph.vars[scope + "/moving_mean"], rt.graph.vars[scope + "/moving_variance"]
            snap[name] = (mm.clone(), mv.clone(), bn_key(rt, name))
    return snap


def _replay_case(label, m, capture, replay, kinds):
    _, F, rt = _prod()
    m.warm()
    assert capture(), "CUDA-graph capture failed"
    before = _bn_snapshot(rt)
    for _ in range(3):
        replay()
    torch.cuda.synchronize()
    after = _bn_snapshot(rt)
    moved = [n for n in before if not (torch.equal(before[n][0], after[n][0]) and torch.equal(before[n][1], after[n][1]))]
    assert moved, "%s: three replays moved no batch-norm statistics" % label
    stuck = [n for n in moved if before[n][2] == after[n][2]]
    print("  %-44s %d of %d batch norms moved their statistics, %d kept their coefficient key" % (label, len(moved), len(before), len(stuck)))
    assert not stuck, "%s: the replays moved these statistics but not their coefficient-cache key: %s" % (label, stuck[:4])
    c1 = audit(rt, F)
    y1 = m.infer()
    c2 = audit(rt, F)
    _need(c2, kinds, label)
    drop_caches(rt)
    y2 = m.infer()
    drop_caches(rt)
    y3 = m.infer()
    print("  %-44s audited after the replays %r, after the forward %r" % (label, c1, c2))
    _agree(label, y1, y2, y3)


@pytest.mark.parametrize("frozen_back", [False, True])
def test_segmenter_graph_replay_keeps_the_operands_coherent(frozen_back):
    """frozen_back: the back half takes no gradient but its batch norms still run on batch statistics, so their gamma / beta are
    in no arena and the replay's bump of the moving statistics is all that changes their coefficient-cache key"""
    m = _Seg(main_trainable=False) if frozen_back else _Seg()
    t = m.trainer
    _replay_case("segmenter replay%s" % (", frozen back half" if frozen_back else ""), m,
                 lambda: t.capture_train_step(m.x, m.y, 0.75, warmup=1), lambda: t.train_step_replay(m.x, m.y, 0.75),
                 ("planes", "bncoef"))
    assert t._graph is not None
    # a second capture while the first one's outputs are still around, and one right after eager steps on the default stream
    t.train_step(m.x, m.y, 0.75)
    assert t.capture_train_step(m.x, m.y, 0.75, warmup=2), "CUDA-graph capture failed the second time"
    t.train_step_replay(m.x, m.y, 0.75)
    torch.cuda.synchronize()
    t._graph = None


@pytest.mark.parametrize("step", ["joint", "d", "g"])
def test_adversarial_graph_replay_keeps_the_operands_coherent(step):
    """`g`: the G step trains the critics' batch norms too, whose gamma / beta live in the D arena that a G replay does not bump"""
    m = _Adv()
    t = m.trainer
    capture = {"joint": lambda: t.capture_joint_step(m.mr, m.ct, 0.75, warmup=1),
               "d": lambda: t.capture_d_step(m.mr, m.ct, 0.75, warmup=1),
               "g": lambda: t.capture_g_step(m.ct, 0.75, warmup=1)}[step]
    replay = {"joint": lambda: t.joint_step(m.mr, m.ct, 0.75),
              "d": lambda: t.d_step_replay(m.mr, m.ct, 0.75),
              "g": lambda: t.g_step_replay(m.ct, 0.75)}[step]
    _replay_case("adversarial replay (%s)" % step, m, capture, replay, ("planes", "bncoef"))
    r1 = t.evaluate(m.ct, torch.zeros(B, 256, 256, 5, device=DEV))
    _, F, rt = _prod()
    drop_caches(rt)
    r2 = t.evaluate(m.ct, torch.zeros(B, 256, 256, 5, device=DEV))
    assert np.abs(r1["confusion_matrix"] - r2["confusion_matrix"]).sum() <= 4, (r1["confusion_matrix"], r2["confusion_matrix"])
    t.release_graphs()


# ------------------------------------------------------------------------------------------------
# activation planes during full eager steps
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keep_prob", [0.75, 1.0])
def test_attached_activation_planes_are_the_split_of_the_live_tensor(keep_prob):
    """two eager steps of each trainer (the second takes the planes-only routes the first one proved): every activation whose
    attached planes a convolution trusts is re-split there"""
    _, F, rt = _prod()
    s = _Seg()
    with watch_planes(F) as w:
        for _ in range(2):
            s.trainer.train_step(s.x, s.y, keep_prob)
        torch.cuda.synchronize()
    print("  segmenter: %d attached-plane hits" % w.hits)
    assert w.hits > 0
    a = _Adv()
    with watch_planes(F) as w:
        for _ in range(2):
            a.trainer.d_step(a.mr, a.ct, keep_prob)
            a.trainer.g_step(a.ct, keep_prob)
        torch.cuda.synchronize()
    print("  adversarial: %d attached-plane hits" % w.hits)
    assert w.hits > 0


# ------------------------------------------------------------------------------------------------
# negative controls: the audit bites
# ------------------------------------------------------------------------------------------------
def test_audit_names_a_weight_written_without_a_bump():
    _, F, rt = _prod()
    m = _Seg()
    m.warm()
    audit(rt, F)
    name = "group_5/Variable"
    with torch.no_grad():
        rt.graph.vars[name].add_(0.01)
    with pytest.raises(AssertionError, match=name + ": cached bf16 weight planes"):
        audit(rt, F)


def test_audit_names_a_moving_mean_written_without_a_bump():
    _, F, rt = _prod()
    m = _Seg()
    m.warm()
    assert audit(rt, F)["bncoef"] > 0
    with torch.no_grad():
        rt.graph.vars["BatchNorm_7/moving_mean"].add_(0.01)
    with pytest.raises(AssertionError, match="BatchNorm_7/gamma: folded batch-norm coefficients"):
        audit(rt, F)


def test_watch_names_an_activation_written_in_place_under_its_planes():
    L, F, rt = _prod()
    rt.reset_default_graph()
    rt.set_conv_backend("auto")
    g = cabi.dev_gen(9)
    x = torch.randn(2, 32, 32, 64, generator=g, device=DEV)
    w1, w2 = (0.05 * torch.randn(3, 3, 64, 64, generator=g, device=DEV) for _ in range(2))
    h = L.conv_bn_relu2d(x, w1, 1.0, is_train=True, scope="a", leak=True)
    assert getattr(h, "_pnp_planes", None) is not None, "the layer attached no planes: nothing to go stale"
    with watch_planes(F) as w:
        L.conv2d(h, w2, 1.0)
    assert w.hits == 1
    with torch.no_grad():
        h.add_(1.0)
    with pytest.raises(AssertionError, match="conv_fwd_raw 32x32.64.64"):
        with watch_planes(F):
            L.conv2d(h, w2, 1.0)


def test_audit_names_stale_transposed_weights_on_the_simt_backend():
    L, F, rt = _prod()
    rt.reset_default_graph()
    rt.set_conv_backend("simt")
    g = cabi.dev_gen(10)
    W = L.weight_variable([3, 3, 16, 24], stddev=0.05)
    x = torch.randn(2, 16, 16, 16, generator=g, device=DEV).requires_grad_(True)
    L.conv2d(x, W, 1.0).sum().backward()
    assert audit(rt, F)["wT"] == 1
    with torch.no_grad():
        W.add_(0.01)
    with pytest.raises(AssertionError, match="Variable: cached transposed weights"):
        audit(rt, F)
