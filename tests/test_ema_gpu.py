"""The weights' moving average in both trainers (Trainer(ema_decay=...), ema.EMA), at a small batch:
1. the average never feeds back: at every eager step its launches leave every graph variable (weights, batch-norm
   statistics), the optimizer slots and the dropout seed bit-identical, and they run after the losses are computed.  (Two
   separate runs of a training step need not agree bit for bit -- floating-point atomics in the convolution and batch-norm
   reductions reorder -- so the check is made inside one run, around the launches themselves);
2. the shadows equal oracle/ema_exact.py's recurrence over per-step snapshots of the live covered variables, bit for bit, eager
   and under captured-graph replay, where n counts the averaged steps and D steps leave n and the shadows alone;
3. before the first update the ema_* scalars of a validation pass equal the live Dice scalars bit for bit (read back with
   tensorboard's EventAccumulator), and the swap leaves the live variables and the existing scalars as they were;
4. checkpoints: the shadow keys are the shadows; latest_ema.npz restored into a fresh trainer makes them the live variables;
   test_native on it writes the labels of a checkpoint rewritten by hand from the shadow keys; train()'s resume continues the
   shadows, n, the live variables and the slots, and the resumed run's shadows then follow the oracle from there; with the
   average off the files and keys are those without the feature;
5. two ranks (skipped below 2 GPUs): equal arena shadows, and the saved batch-norm shadows are the rank mean."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ema_exact as E
from tests import mmwhs_phantom as ph
from tests.models import adv_pair, seg_pair, step_images, step_onehot

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B = 2
DECAY = 0.99
SUFFIX = "/ExponentialMovingAverage"


def _seg(ema=DECAY):
    net, tr, _, _ = seg_pair("simt", B)
    if ema is not None:
        from pnp_b200.ema import EMA
        from pnp_b200 import runtime as rt
        tr.ema = EMA(tr.arena, [v for v in rt.global_variables() if v.pnp_kind == "bn_moving"], ema)
    return net, tr


def _gan(ema=DECAY):
    from pnp_b200.train_gan import configure
    net, tr, _ = adv_pair("simt", configure("train-gan")[0]["lambda_mask_loss"], "train-gan", B, with_oracle=False,
                          critic_keep_prob=0.75)
    if ema is not None:
        from pnp_b200.ema import EMA
        tr.ema = EMA(tr.g_arena, [v for v in net.adapt_vars if v.pnp_kind == "bn_moving"], ema)
    return net, tr


def _build(kind, ema=DECAY):
    """the trainer as its constructor builds it with ema_decay=ema (checked against the constructor in test_constructor)"""
    return (_seg if kind == "seg" else _gan)(ema)


def _live(ema):
    """the covered live values in the shadow's layout (chunk padding of the statistics: zeros)"""
    out = torch.zeros_like(ema.shadow)
    out[:ema.arena.total] = ema.arena.theta
    for v, o in zip(ema.extra, ema.extra_offsets):
        out[o:o + v.numel()] = v.reshape(-1)
    return out.cpu().numpy()


def _covered(ema):
    m = np.zeros(ema.total, bool)
    m[:ema.arena.total] = True
    for v, o in zip(ema.extra, ema.extra_offsets):
        m[o:o + v.numel()] = True
    return m


def _oracle(ema, s, n, live):
    cov = _covered(ema)
    c, n = E.advance(n, ema.decay)
    s = s.copy()
    s[cov] = E.update(s[cov], live[cov], c)
    return s, n


def _bits(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.int32), np.asarray(b, np.float32).view(np.int32))


def _batches(kind):
    if kind == "seg":
        return [(step_images(B, 11 + k), step_onehot(B, 40 + k)) for k in range(3)]
    return [(step_images(B, 21 + k), step_images(B, 31 + k, 0.3, 0.8), step_images(B, 51 + k, 0.3, 0.8)) for k in range(3)]


def _step(kind, tr, b, keep=0.75):
    if kind == "seg":
        return [float(t) for t in tr.train_step(b[0], b[1], keep)]
    d, g = tr.d_step(b[0], b[1], keep), tr.g_step(b[2], keep)
    return [tr.loss_value(d), tr.loss_value(g)]


def _slots(kind, tr):
    if kind == "seg":
        return [tr.optimizer.m.cpu().numpy(), tr.optimizer.v.cpu().numpy()]
    return [o.cpu().numpy() for opt in (tr.dis_optimizer, tr.gen_optimizer) for o in (opt.ms, opt.mom)]


@pytest.mark.parametrize("kind", ["seg", "gan"])
def test_constructor(kind):
    from pnp_b200 import adversarial as adv, runtime as rt, source_segmenter as seg
    from pnp_b200.train_gan import configure
    if kind == "seg":
        net = seg.Full_DRN(channels=3, n_class=5, batch_size=B)
        tr = seg.Trainer(net, [], [], num_cls=5, batch_size=B, optimizer="adam", ema_decay=DECAY)
        want = {v.pnp_name for v in tr.trainables} | {n for n in rt.graph.order if rt.graph.vars[n].pnp_kind == "bn_moving"}
    else:
        ck, nc, tc = configure("train-gan")
        ck["lambda_mask_loss"] = 0.3
        net = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc)
        tr = adv.Trainer(net, num_cls=5, batch_size=B, train_config=tc, ema_decay=DECAY)
        want = {n for n in rt.graph.order if "adapt" in n and "cls" not in n}
        assert not any("cls" in v.pnp_name for v in tr.ema.variables)
    assert {v.pnp_name for v in tr.ema.variables} == want
    assert _bits(tr.ema.shadow.cpu().numpy()[_covered(tr.ema)], _live(tr.ema)[_covered(tr.ema)])
    assert int(tr.ema.num_updates.item()) == 0 and tr.ema.decay == DECAY


def _slot_state(kind, tr):
    """the stored slots (the arena padding of RMSProp's ms is not part of them)"""
    if kind == "seg":
        return tr.optimizer.slot_state()
    return dict(tr.dis_optimizer.slot_state(), **tr.gen_optimizer.slot_state())


def _everything(kind, tr):
    from pnp_b200 import runtime as rt
    torch.cuda.synchronize()
    return rt.state_dict(), _slots(kind, tr), rt.rng.seed_t.cpu().clone(), rt.rng.counter


@pytest.mark.parametrize("kind", ["seg", "gan"])
def test_average_never_feeds_back_and_follows_the_oracle(kind, monkeypatch):
    from pnp_b200 import runtime as rt
    _, tr = _build(kind, DECAY)
    ema = tr.ema
    s, n = ema.shadow.cpu().numpy(), 0
    rt.manual_seed(77)
    real_update, seen = ema.update, []

    def checked_update():
        before = _everything(kind, tr)
        real_update()
        after = _everything(kind, tr)
        for name in before[0]:
            assert _bits(after[0][name], before[0][name]), name
        assert all(_bits(a, b) for a, b in zip(after[1], before[1]))
        assert torch.equal(after[2], before[2]) and after[3] == before[3]
        seen.append(_live(ema))
    monkeypatch.setattr(ema, "update", checked_update)
    for b in _batches(kind):
        losses = _step(kind, tr, b)
        assert all(np.isfinite(losses))
    assert len(seen) == 3
    for live in seen:
        s, n = _oracle(ema, s, n, live)
    assert int(ema.num_updates.item()) == n == 3
    assert _bits(ema.shadow.cpu().numpy()[_covered(ema)], s[_covered(ema)])


@pytest.mark.parametrize("kind", ["seg", "gan"])
def test_captured_steps_advance_the_average(kind):
    from pnp_b200 import runtime as rt
    _, tr = _build(kind, DECAY)
    rt.manual_seed(5)
    batches = _batches(kind)
    if kind == "seg":
        assert tr.capture_train_step(batches[0][0], batches[0][1], 0.75, warmup=2)
        replay = lambda b: tr.train_step_replay(b[0], b[1], 0.75)  # noqa: E731
    else:
        assert tr.capture_joint_step(batches[0][0], batches[0][1], 0.75, warmup=2)
        assert tr.capture_d_step(batches[0][0], batches[0][1], 0.75, warmup=1)
        replay = lambda b: tr.joint_step(b[0], b[1], 0.75, ct_batch_g=b[2])  # noqa: E731
    torch.cuda.synchronize()
    ema = tr.ema
    n0 = int(ema.num_updates.item())
    assert n0 == 2                                  # the warm-up G / segmenter steps are real steps; D steps never count
    s, n = ema.shadow.cpu().numpy(), n0
    for k, b in enumerate(batches):
        replay(b)
        torch.cuda.synchronize()
        s, n = _oracle(ema, s, n, _live(ema))
        assert int(ema.num_updates.item()) == n == n0 + k + 1
        assert _bits(ema.shadow.cpu().numpy(), s), k
    if kind == "gan":
        before = ema.shadow.clone()
        for b in batches:
            tr.d_step_replay(b[0], b[1], 0.75)
            tr.d_step(b[0], b[1], 0.75)
        torch.cuda.synchronize()
        assert int(ema.num_updates.item()) == n and torch.equal(ema.shadow, before)


def _scalars(log_dir):
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    acc = EventAccumulator(log_dir)
    acc.Reload()
    return {t: [(e.step, e.value) for e in acc.Scalars(t)] for t in acc.Tags()["scalars"]}


@pytest.mark.parametrize("kind", ["seg", "gan"])
def test_monitoring_tags(kind, tmp_path):
    from pnp_b200 import runtime as rt
    _, tr = _build(kind, DECAY)
    log = str(tmp_path / "val_log")
    vx, vy = step_images(B, 91, *(() if kind == "seg" else (0.3, 0.8))), step_onehot(B, 92)
    mr, mry = step_images(B, 93), step_onehot(B, 94)

    def pass_(step):
        if kind == "seg":
            tr.val_stats(vx, vy, step, log, detail=True)
            return tr.ema_val_stats(vx, vy, step, log)
        tr.output_minibatch_stats(step, vx, vy, mr, mry, log, True)
        return tr.ema_stats(step, vx, vy, log)

    before = rt.state_dict()
    pass_(0)
    torch.cuda.synchronize()
    after = rt.state_dict()
    for n in before:
        if kind == "gan" and "cls" in n:         # the critics' batch-statistics BN moves in the existing pass
            continue
        assert _bits(after[n], before[n]), n
    for b in _batches(kind)[:2]:
        _step(kind, tr, b)
    pass_(5)
    torch.cuda.synchronize()
    sc = _scalars(log)
    pairs = ([("ema_dice_eval", "dice_eval")] if kind == "seg" else []) + \
        [(e, l) for e, l in zip(tr.EMA_TAGS[-4:], (tr.SCALAR_TAGS[5:9] if kind == "seg" else tr.SCALAR_TAGS[3:7]))]
    for e, l in pairs:
        assert sc[e][0] == sc[l][0], (e, sc[e], l, sc[l])      # step 0: no update yet, the shadows are the live variables
        assert [s for s, _ in sc[e]] == [0, 5]
    # the ema scalars are written after the pass's own, in the same file
    files = os.listdir(log)
    assert len([f for f in files if f.startswith("events.out.tfevents")]) == 1


def _save(tr, out):
    tr.save(os.path.join(out, "model.cpkt"), out)
    torch.cuda.synchronize()


@pytest.mark.parametrize("kind", ["seg", "gan"])
def test_checkpoints(kind, tmp_path):
    from pnp_b200 import runtime as rt
    _, tr = _build(kind, DECAY)
    rt.manual_seed(9)
    for b in _batches(kind):
        _step(kind, tr, b)
    out = str(tmp_path / "run")
    os.makedirs(out)
    _save(tr, out)
    gs = tr.global_step
    assert set(os.listdir(out)) == {"model.cpkt-%d.npz" % gs, "latest.npz", "model.cpkt-%d_ema.npz" % gs, "latest_ema.npz"}
    d = np.load(os.path.join(out, "latest.npz"))
    for v, sv in tr.ema._pairs():
        assert _bits(d[v.pnp_name + SUFFIX], sv.cpu().numpy()), v.pnp_name
    assert int(d["pnp/ema_num_updates"]) == 3 and d["pnp/ema_decay"] == np.float32(DECAY)
    shadows = {v.pnp_name: sv.cpu().numpy().copy() for v, sv in tr.ema._pairs()}
    live = rt.state_dict()
    e = np.load(os.path.join(out, "latest_ema.npz"))
    assert set(e.files) == set(rt.graph.order) | {"pnp/global_step"}

    # restored into a fresh trainer, the averaged checkpoint makes the shadows the live variables
    net2, tr2 = _build(kind, None)
    net2.restore(os.path.join(out, "latest_ema.npz"))
    got = rt.state_dict()
    for n in rt.graph.order:
        assert _bits(got[n], shadows.get(n, live[n])), n

    # test_native on it == test_native on a checkpoint rewritten by hand from the shadow keys
    pairs = ph.write_pairs(str(tmp_path), "ct", [61], perms=[ph.SIGNED_PERMUTATIONS[5]], shape=(40, 36, 30),
                           spacing=(0.8, 1.1, 1.7))
    hand = {n: (d[n + SUFFIX] if n + SUFFIX in d.files else d[n]) for n in rt.graph.order}
    np.savez(str(tmp_path / "hand.npz"), **hand)
    from pnp_b200 import nifti
    labels = []
    for ck in (os.path.join(out, "latest_ema.npz"), str(tmp_path / "hand.npz")):
        net2.restore(ck)
        res = tr2.test_native(pairs, str(tmp_path / ("native_" + os.path.basename(ck)[:-4])))
        labels.append(nifti.load(res[0]["path"]).get_data())
    assert np.array_equal(labels[0], labels[1])

    # train()'s resume continues the shadows and their count
    _, tr3 = _build(kind, DECAY)
    tr3.train(out, restore=True, restored_path=out, training_iters=0, epochs=1)
    assert int(tr3.ema.num_updates.item()) == 3
    for v, sv in tr3.ema._pairs():
        assert _bits(sv.cpu().numpy(), shadows[v.pnp_name]), v.pnp_name


@pytest.mark.parametrize("kind", ["seg", "gan"])
def test_interrupted_run_resumes_where_it_stopped(kind, tmp_path):
    from pnp_b200 import runtime as rt
    batches = _batches(kind)
    _, tr = _build(kind, DECAY)
    rt.manual_seed(3)
    out = str(tmp_path)
    _step(kind, tr, batches[0])
    _save(tr, out)
    want, want_slots = rt.state_dict(), _slot_state(kind, tr)
    want_s, want_n = tr.ema.shadow.cpu().numpy(), int(tr.ema.num_updates.item())

    _, tr2 = _build(kind, DECAY)
    tr2.train(out, restore=True, restored_path=out, training_iters=0, epochs=1)
    got = rt.state_dict()
    for n in want:
        assert _bits(got[n], want[n]), n
    got_slots = _slot_state(kind, tr2)
    assert set(got_slots) == set(want_slots) and all(_bits(got_slots[k], want_slots[k]) for k in want_slots)
    assert int(tr2.ema.num_updates.item()) == want_n == 1
    assert _bits(tr2.ema.shadow.cpu().numpy()[_covered(tr2.ema)], want_s[_covered(tr2.ema)])
    # the resumed average goes on from the saved one: the next steps follow the recurrence from the saved shadows and count
    s, n = want_s, want_n
    for b in batches[1:]:
        _step(kind, tr2, b)
        torch.cuda.synchronize()
        s, n = _oracle(tr2.ema, s, n, _live(tr2.ema))
    assert int(tr2.ema.num_updates.item()) == n == 3
    assert _bits(tr2.ema.shadow.cpu().numpy()[_covered(tr2.ema)], s[_covered(tr2.ema)])


@pytest.mark.parametrize("kind", ["seg", "gan"])
def test_off_keeps_the_files_and_keys(kind, tmp_path):
    from pnp_b200 import runtime as rt
    _, tr = _build(kind, None)
    assert tr.ema is None
    _step(kind, tr, _batches(kind)[0])
    out = str(tmp_path)
    _save(tr, out)
    assert set(os.listdir(out)) == {"model.cpkt-%d.npz" % tr.global_step, "latest.npz"}
    d = np.load(os.path.join(out, "latest.npz"))
    slots = set(tr.optimizer.slot_state()) if kind == "seg" else set(tr.dis_optimizer.slot_state()) | set(tr.gen_optimizer.slot_state())
    assert set(d.files) == set(rt.graph.order) | slots | {"pnp/learning_rate", "pnp/global_step"}


def _dp_worker(rank, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK=str(rank))
    sys.path.insert(0, ROOT)
    torch.cuda.set_device(rank)
    from pnp_b200 import parallel, runtime as rt
    parallel.init_from_env()
    _, tr = _build("gan", DECAY)
    rt.manual_seed(8)
    b = _batches("gan")[rank]                       # per-rank batches: the DAM statistics differ between the ranks
    _step("gan", tr, tuple(x.cuda() for x in b))
    torch.cuda.synchronize()
    out["arena_%d" % rank] = tr.ema.shadow[:tr.ema.arena.total].cpu().numpy()
    out["stats_%d" % rank] = tr.ema.shadow[tr.ema.arena.total:].cpu().numpy()
    torch.distributed.barrier()
    st = tr.checkpoint_state()
    if rank == 0:
        out["saved"] = {k: v for k, v in st.items() if k.endswith(SUFFIX)}
        out["layout"] = [(v.pnp_name, o, v.numel()) for v, o in zip(tr.ema.extra, tr.ema.extra_offsets)]
        out["arena_total"] = tr.ema.arena.total
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


def test_two_ranks():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    out = mp.Manager().dict()
    mp.spawn(_dp_worker, args=(29633 + os.getpid() % 1000, out), nprocs=2, join=True)
    assert _bits(out["arena_0"], out["arena_1"])
    mean = (out["stats_0"] + out["stats_1"]) * np.float32(0.5)
    base = out["arena_total"]
    for name, o, n in out["layout"]:
        assert np.array_equal(out["saved"][name + SUFFIX], mean[o - base:o - base + n]), name
