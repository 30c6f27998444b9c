"""Both trainers' adapt_entropy (tent.py) end to end at B = 2: the segmenter over all 30 batch norms, the GAN trainer over the
DAM's 20.

1. the first eager step's dgamma / dbeta of every covered layer agree with fp64 autograd of the same objective through the fp64
   oracle network, within the bounds of the G-step gradient parity (tests/models.grad_report): frozen weights, trainable
   gamma / beta, batch-statistics batch norm;
2. the update is oracle/optim_exact.py's Adam applied to the gradients the step wrote;
3. nothing else moves: weights, critics, groups 7-9, the trainer's optimizer slots, learning rate and global_step, the arena
   outside the covered segments, and the arena's gradient stays zero outside them (no weight gradient ran);
4. N eager steps and 2 + (N - 2) captured steps from one state agree within the forward's run-to-run spread (split-K
   convolutions add their partial sums with fp32 atomics; DESIGN 2), and so do their history rows;
5. repeated steps on one fixed batch lower its mean entropy;
6. the statistics after the call equal recalibrate_bn on the adapted gamma / beta over the same further batches;
7. a source raising mid-run, a NaN batch and every argument error leave every snapshotted variable, flag and the GAN mode as
   they were, every cached operand is the live variable's afterwards, and a training step runs;
8. a fresh trainer restored from the written checkpoint holds the live variables bit for bit and its inference agrees;
9. adapt_entropy.py runs end to end on phantom subjects for both trainers."""
import numpy as np
import pytest
import torch

from tests import coherence
from tests import mmwhs_phantom as ph
from tests.models import adv_pair, grad_report, seg_pair, step_images, step_onehot

pytestmark = pytest.mark.gpu

B = 2
KINDS = ["seg", "gan"]
SPREAD = 1e-4


class Stream:
    """seeded synthetic slices from call `start` on, labels ignored; `fail_at`: next() raises on that call; `nan_at`: that
    call's batch holds a NaN"""

    def __init__(self, kind, seed, batch=B, start=0, fail_at=None, nan_at=None):
        from oracle.pnp_graphs import synthetic_images
        self.kw = {} if kind == "seg" else {"shift": 0.3, "scale": 0.8}         # CT-like slices for the DAM
        self.seed, self.batch, self.calls, self.fail_at, self.nan_at = seed, batch, start, fail_at, nan_at
        self._img = synthetic_images

    def next(self):
        if self.calls == self.fail_at:
            raise RuntimeError("source failed")
        x = self._img(self.batch, self.seed + self.calls, **self.kw).cuda()
        if self.calls == self.nan_at:
            x[0, 7, 9, 1] = float("nan")
        self.calls += 1
        return x, None


def _build(kind):
    """-> (net, trainer, variables).  The seeded GAN saturates its prediction (mean entropy ~1e-4), where the entropy is only
    the forward's rounding noise; its output layer is scaled so that the logits of a probe batch have a standard deviation
    of 2, as a trained network's uncertain pixels do"""
    from pnp_b200 import runtime as rt
    if kind == "seg":
        net, tr, _, P = seg_pair("auto", B)
        return net, tr, P
    net, tr, _ = adv_pair("auto", 1.0, "train-gan", B, with_oracle=False)
    w = rt.graph.vars["output/Variable"]
    with torch.no_grad():
        logits = net.segment(step_images(B, 5, 0.3, 0.8), "ct", 1.0, front_bn=False, joint_bn=False)["logits"]
        w.mul_(2.0 / float(logits.std()))
    w.pnp_version += 1
    return net, tr, rt.state_dict()


def _arena(tr, kind):
    return tr.arena if kind == "seg" else tr.g_arena


def _bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _covered(tr, kind):
    return [v for v in _arena(tr, kind).vars if v.pnp_kind in ("bn_gamma", "bn_beta")]


def _trainer_state(tr, kind):
    st = {k: np.asarray(v).copy() for k, v in tr.checkpoint_state().items()}
    lrs = [tr.optimizer.get_lr()] if kind == "seg" else [tr.dis_optimizer.get_lr(), tr.gen_optimizer.get_lr()]
    return st, lrs, tr.global_step


def _entropy64(logits):
    return -(torch.softmax(logits, -1) * torch.log_softmax(logits, -1)).sum(-1).mean()


def test_covered_channels():
    for kind, layers, channels in (("seg", 30, 8032), ("gan", 20, 2912)):
        _, tr, _ = _build(kind)
        cov = _covered(tr, kind)
        assert len(cov) == 2 * layers and sum(v.numel() for v in cov) == 2 * channels, kind


@pytest.mark.parametrize("kind", KINDS)
def test_first_step_gradients_against_the_fp64_oracle(kind):
    from oracle.pnp_graphs import OracleAdversarial, OracleSegmenter
    net, tr, P = _build(kind)
    x = step_images(B, 21) if kind == "seg" else step_images(B, 22, 0.3, 0.8)
    if kind == "seg":
        o32, o64 = OracleSegmenter(P, B), OracleSegmenter(P, B, dtype=torch.float64)
        fwd = lambda o, xx: o.forward(xx, 1.0, bn_train=True)["logits"]
    else:
        o32, o64 = OracleAdversarial(P, B), OracleAdversarial(P, B, dtype=torch.float64)
        fwd = lambda o, xx: o.segment(xx, "ct", 1.0, front_bn=True)["logits"]
    cov = _covered(tr, kind)
    names = [v.pnp_name for v in cov]
    s = tr.entropy_adaptation()
    try:
        s.step(x)
        ours = [v.grad.detach().cpu().double().clone() for v in cov]
    finally:
        s.restore()
        s.close()

    def ref(o, dtype):
        params = [getattr(o.ps.bn[n.rsplit("/", 1)[0]], n.rsplit("/", 1)[1]) for n in names]
        L = _entropy64(fwd(o, x.cpu().to(dtype)))
        return [g.detach().double() for g in torch.autograd.grad(L, params)]

    g32, g64 = ref(o32, torch.float32), ref(o64, torch.float64)
    grad_report(names, ours, g32, g64, slack=10.0)


@pytest.mark.parametrize("kind", KINDS)
def test_update_is_adam_and_nothing_else_moves(kind):
    from pnp_b200 import runtime as rt
    from oracle import optim_exact as OE
    net, tr, _ = _build(kind)
    arena = _arena(tr, kind)
    cov = _covered(tr, kind)
    st0, lrs0, gs0 = _trainer_state(tr, kind)
    theta0 = arena.theta.detach().clone()
    s = tr.entropy_adaptation(lr=1e-4)
    try:
        s.step(step_images(B, 31, **({} if kind == "seg" else {"shift": 0.3, "scale": 0.8})))
        torch.cuda.synchronize()
        inside = torch.zeros(arena.total, dtype=torch.bool, device=arena.theta.device)
        ids = {id(v) for v in cov}
        for v, (o, n) in zip(arena.vars, arena.offsets):
            if id(v) in ids:
                inside[o:o + n] = True
        grad, theta = arena.grad.detach().clone(), arena.theta.detach().clone()
        assert torch.count_nonzero(grad[~inside]) == 0, "a gradient outside the covered gamma / beta"
        assert torch.count_nonzero(grad[inside]) > 0
        assert torch.equal(theta[~inside].view(torch.int32), theta0[~inside].view(torch.int32))
        # the covered elements alone (no weight decay anywhere, fresh zero slots)
        state = OE.adam_advance([1.0, 1.0, 1e-4, 0.0], 0.9, 0.999)
        t0, g0 = theta0[inside].cpu(), grad[inside].cpu()
        zeros = torch.zeros_like(t0)
        seg = torch.zeros(-(-t0.numel() // OE.CHUNK), dtype=torch.int32)
        ref = OE.adam_step(t0, g0, zeros, zeros, seg, torch.zeros(1), state, 0.9, 0.999, 1e-8, 1.0)
        assert OE.worst_ratio(theta[inside].cpu(), ref["theta"], ref["mag_theta"]) <= 8 * OE.U32
    finally:
        s.close()
    # N steps through the public call: only the covered gamma / beta and the moving statistics move
    before = rt.state_dict()
    names, hist, slices = tr.adapt_entropy(Stream(kind, 40), 4, recalibrate_batches=2)
    assert hist.shape == (4, 6) and slices == 6 * B
    after = rt.state_dict()
    moving = {v.pnp_name for v in s.moving}
    moved = {k for k in before if not _bits(before[k], after[k])}
    assert moved <= set(names), sorted(moved - set(names))[:5]
    assert {v.pnp_name for v in cov} <= moved
    assert all(n in moving for n in moved if n not in {v.pnp_name for v in cov})
    if kind == "gan":
        assert not any(n.startswith(("group_7", "group_8", "group_9", "cls_", "m_cls")) for n in moved)
    st1, lrs1, gs1 = _trainer_state(tr, kind)
    assert lrs1 == lrs0 and gs1 == gs0
    for k in st0:
        if k not in moved:
            assert _bits(st0[k], st1[k]), k
    assert torch.count_nonzero(arena.grad[~inside]) == 0


@pytest.mark.parametrize("kind", KINDS)
def test_eager_and_captured_steps_agree(kind):
    """two eager runs of N steps from one state measure the run-to-run spread; 2 eager + (N - 2) captured steps from the same
    state stay within four times it"""
    from pnp_b200 import runtime as rt, tent
    N, lr = 5, 1e-4
    net, tr, _ = _build(kind)
    snap = rt.state_dict()
    cov = [v.pnp_name for v in _covered(tr, kind)]

    def eager():
        rt.load_state_dict(snap)
        src = Stream(kind, 50)
        s = tr.entropy_adaptation(lr)
        rows = []
        for _ in range(N):
            loss, pbar = s.step(src.next()[0])
            rows.append(torch.cat([loss.reshape(1), pbar]).cpu().numpy())
        s.close()
        return np.array(rows, np.float64), rt.state_dict()

    h1, st1 = eager()
    h2, st2 = eager()
    rt.load_state_dict(snap)
    _, hc, _ = tent.adapt(tr.entropy_adaptation, Stream(kind, 50), N, lr, 1, lambda src, n: ([], 0))
    stc = rt.state_dict()
    spread_h = np.abs(h2 - h1).max()
    assert np.all(np.abs(hc - h1) <= 4 * spread_h + 1e-6 * np.abs(h1)), (np.abs(hc - h1).max(), spread_h)
    spread = max(np.abs(st2[k].astype(np.float64) - st1[k]).max() for k in cov)
    worst = max(np.abs(stc[k].astype(np.float64) - st1[k]).max() for k in cov)
    print(kind, "history spread %.3e, gamma / beta spread %.3e, captured %.3e" % (spread_h, spread, worst))
    assert worst <= 4 * spread + 1e-7, (worst, spread)
    for k in snap:
        if k not in cov and not k.endswith(("moving_mean", "moving_variance")):
            assert _bits(st1[k], stc[k]), k


@pytest.mark.parametrize("kind", KINDS)
def test_repeated_steps_lower_the_entropy_of_one_batch(kind):
    net, tr, _ = _build(kind)
    x = Stream(kind, 60).next()[0]
    s = tr.entropy_adaptation(1e-3)
    try:
        losses = [float(s.step(x)[0]) for _ in range(8)]
    finally:
        s.restore()
        s.close()
    print(kind, losses)
    assert losses[-1] < losses[0], losses


@pytest.mark.parametrize("kind", KINDS)
def test_statistics_are_the_recalibration_of_the_adapted_network(kind):
    from pnp_b200 import runtime as rt
    net, tr, _ = _build(kind)
    names, _, _ = tr.adapt_entropy(Stream(kind, 70), 3, recalibrate_batches=2)
    adapted = rt.state_dict()
    stats = [n for n in names if n.endswith(("moving_mean", "moving_variance"))]
    assert stats
    with torch.no_grad():                       # the population does not depend on the old statistics
        for n in stats:
            rt.graph.vars[n].fill_(0.5)
    if kind == "seg":
        tr.recalibrate_bn(Stream(kind, 70, start=3), 2)
    else:
        tr.recalibrate_bn(Stream(kind, 70, start=3), 2, scope="dam")
    again = rt.state_dict()
    for n in stats:
        var = adapted[n.replace("moving_mean", "moving_variance")]
        scale = np.sqrt(np.abs(var)) + np.abs(adapted[n]) + 1e-6 if n.endswith("moving_mean") else np.abs(adapted[n]) + 1e-6
        assert np.all(np.abs(again[n].astype(np.float64) - adapted[n]) <= SPREAD * scale), n


@pytest.mark.parametrize("kind", KINDS)
def test_raises_restore_everything(kind):
    from pnp_b200 import functional as F, runtime as rt
    net, tr, _ = _build(kind)
    if kind == "gan":
        tr._set_mode("G")
    before = rt.state_dict()
    flags = [v.requires_grad for v in rt.global_variables()]

    def unchanged(tag):
        after = rt.state_dict()
        for k in before:
            assert _bits(before[k], after[k]), (tag, k)
        assert [v.requires_grad for v in rt.global_variables()] == flags, tag
        if kind == "gan":
            assert tr._mode is None, tag
        coherence.audit(rt, F)

    with pytest.raises(RuntimeError, match="source failed"):
        tr.adapt_entropy(Stream(kind, 80, fail_at=4), 6, recalibrate_batches=2)       # two eager steps and a replay ran
    unchanged("source")
    with pytest.raises(FloatingPointError):
        tr.adapt_entropy(Stream(kind, 80, nan_at=3), 5, recalibrate_batches=2)
    unchanged("nan")
    for kw in ({"steps": 0}, {"recalibrate_batches": 0}, {"lr": 0.0}, {"lr": -1e-4}, {"lr": float("inf")}, {"lr": float("nan")}):
        args = dict(steps=3, lr=1e-4, recalibrate_batches=1)
        args.update(kw)
        with pytest.raises(ValueError):
            tr.adapt_entropy(Stream(kind, 80), **args)
        unchanged(str(kw))
    with pytest.raises(ValueError):
        tr.adapt_entropy(Stream(kind, 80, batch=B + 1), 3, recalibrate_batches=1)
    unchanged("batch size")
    # a training step runs afterwards
    x = step_images(B, 91)
    if kind == "seg":
        wce, dice = tr.train_step(x, step_onehot(B, 92), 1.0)
        assert np.isfinite(float(wce)) and np.isfinite(float(dice))
    else:
        terms = tr.g_step(step_images(B, 93, 0.3, 0.8), 1.0)
        assert all(np.isfinite(float(t)) for t, _ in terms)


@pytest.mark.parametrize("kind", KINDS)
def test_a_fresh_trainer_restored_from_the_checkpoint_agrees(kind, tmp_path):
    from pnp_b200 import bnstats, functional as F, lib, runtime as rt
    net, tr, _ = _build(kind)
    tr.adapt_entropy(Stream(kind, 100), 3, recalibrate_batches=2)
    coherence.audit(rt, F)
    ck = lib._save(bnstats.recalibrated_checkpoint(tr), str(tmp_path / "tent"))
    live = rt.state_dict()
    x = step_images(B, 101) if kind == "seg" else step_images(B, 102, 0.3, 0.8)

    def logits(t):
        with torch.no_grad():
            return (t._logits(x) if kind == "seg" else t._ct_logits(x)).cpu().numpy()

    got = logits(tr)
    net2, tr2, _ = _build(kind)
    net2.restore(ck)
    restored = rt.state_dict()
    for k in live:
        assert _bits(restored[k], live[k]), k
    ref = logits(tr2)
    assert np.all(np.abs(got - ref) <= SPREAD * np.abs(ref).max())


def test_cli_end_to_end_on_phantom_subjects(tmp_path):
    from pnp_b200 import lib, native, nifti, runtime as rt, tent
    ct_pairs = ph.write_pairs(str(tmp_path), "ct", [61, 62], shape=(40, 36, 30), spacing=(0.8, 1.1, 1.7))
    pairs_file = str(tmp_path / "ct_pairs")
    with open(pairs_file, "w") as f:
        f.writelines("%s %s\n" % p for p in ct_pairs)
    for kind in ("gan", "segmenter"):
        native.build_trainer(kind, None, B)
        st = rt.state_dict()
        st["pnp/global_step"] = np.int64(41)
        ck = lib._save(st, str(tmp_path / ("%s_latest_ema" % kind)))
        out = str(tmp_path / ("%s_tent.npz" % kind))
        argv = ["--trainer", kind, "--checkpoint", ck, "--out", out, "--volumes", pairs_file, "--steps", "4",
                "--recalibrate-batches", "2", "--batch-size", str(B), "--seed", "5"]
        names, hist, slices = tent.main(argv)
        assert hist.shape == (4, 6) and slices == 6 * B
        rows = open(tent.log_path(out)).read().splitlines()
        assert len(rows) == 5 and rows[0].startswith("step,entropy,pbar_0")
        a = np.load(out)
        assert set(a.files) == set(rt.graph.order) | {"pnp/global_step"} and int(a["pnp/global_step"]) == 41
        assert any(not _bits(a[k], st[k]) for k in names)
        tr = native.build_trainer(kind, out, B)
        res = tr.test_native(ct_pairs[:1], str(tmp_path / ("native_" + kind)))
        lab = nifti.load(res[0]["path"]).get_data()
        assert lab.shape == nifti.load(ct_pairs[0][0]).get_data().shape
