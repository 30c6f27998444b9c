"""Both trainers' recalibrate_bn (bnstats.py) end to end: the segmenter over its 30 batch norms, the GAN trainer over the DAM's
20 ('dam') and over those plus the shared groups 7-9 ('all').

1. every accumulator is the pass-ordered fp64 sum of the statistics the layers handed over, bit for bit;
2. every covered statistic is the fp64 oracle network's pooled population statistic over the same batches (training-mode BN,
   keep_prob 1), within a bound that grows with the layer's depth;
3. nothing else moves: weights, gamma / beta, uncovered statistics, critics, optimizer slots and EMA shadows;
4. the result does not depend on the old statistics: from NaN statistics the output is, bit for bit, the population of the
   statistics that run's layers handed over, and it agrees with the run from the real statistics to the run-to-run spread of
   the forward (split-K convolutions add their partial sums with fp32 atomics, so two forwards of one batch may differ in the
   last bits; DESIGN §2);
5. a raise mid-run puts the snapshot back bit for bit;
6. afterwards every cached operand is that of the live variables, a fresh trainer restored from the written checkpoint holds
   the live variables bit for bit, its inference forward agrees with the recalibrated trainer's to the run-to-run spread, and
   a step captured on each replays (the segmenter's losses within 5 %);
7. recalibrate_bn.py runs end to end on phantom subjects for both trainers and on an _ema.npz input, its output goes
   through test_native, and two runs with one seed write byte-identical uncovered arrays and covered statistics within the
   run-to-run spread."""
import os

import numpy as np
import pytest
import torch

from tests import coherence
from tests import mmwhs_phantom as ph
from tests.models import adv_pair, seg_pair

pytestmark = pytest.mark.gpu

B = 2
CASES = [("seg", None), ("gan", "dam"), ("gan", "all")]
IDS = ["segmenter", "gan-dam", "gan-all"]
N_COVERED = {("seg", None): 30, ("gan", "dam"): 20, ("gan", "all"): 30}


class Stream:
    """seeded synthetic slices, labels ignored; `fail_at`: next() raises on that call"""

    def __init__(self, seed, batch=B, fail_at=None, shift=0.0, scale=1.0):
        from oracle.pnp_graphs import synthetic_images
        self.seed, self.batch, self.fail_at, self.calls = seed, batch, fail_at, 0
        self.shift, self.scale, self._img = shift, scale, synthetic_images

    def next(self):
        if self.calls == self.fail_at:
            raise RuntimeError("source failed")
        x = self._img(self.batch, self.seed + self.calls, self.shift, self.scale).cuda()
        self.calls += 1
        return x, None


def _build(kind):
    if kind == "seg":
        net, tr, _, _ = seg_pair("auto", B)
        return net, tr, None
    net, tr, _ = adv_pair("auto", 1.0, "train-gan", B, with_oracle=False)
    return net, tr, None


def _recal(kind, scope, tr, src, batches):
    return tr.recalibrate_bn(src, batches) if kind == "seg" else tr.recalibrate_bn(src, batches, scope=scope)


def _bits(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


SPREAD = 1e-4          # relative; the forward's run-to-run differences are ~1e-6


def _close(a, b, scale=None):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    s = np.abs(b) + 1e-6 if scale is None else scale
    return a.shape == b.shape and bool(np.all(np.abs(a - b) <= SPREAD * s))


def _stat_close(name, a, b, var):
    """moving means against the channel's standard deviation, variances relative"""
    return _close(a, b, np.sqrt(np.abs(var)) + np.abs(b) + 1e-6) if name.endswith("moving_mean") else _close(a, b)


def _stream_kw(kind):
    return {} if kind == "seg" else {"shift": 0.3, "scale": 0.8}            # CT-like slices for the DAM


@pytest.mark.parametrize("kind,scope", CASES, ids=IDS)
def test_accumulators_and_population_against_the_fp64_oracle(kind, scope, monkeypatch):
    from pnp_b200 import bnstats, runtime as rt
    from oracle import tf14_torch as T
    from oracle.pnp_graphs import OracleAdversarial, OracleSegmenter
    net, tr, _ = _build(kind)
    # the fp64 oracle on the same variables
    P = rt.state_dict()
    o64 = (OracleSegmenter(P, B, dtype=torch.float64) if kind == "seg" else OracleAdversarial(P, B, dtype=torch.float64))
    names = {id(bn): s for s, bn in o64.ps.bn.items()}
    pooled = {}
    orig_bn = T.batch_norm

    def tap_bn(x, bn, is_training):
        if is_training:
            flat = x.detach().reshape(-1, x.shape[-1]).double()
            s = names[id(bn)]
            prev = pooled.get(s, [])
            prev.append(flat)
            pooled[s] = prev
        return orig_bn(x, bn, is_training)

    # tap 1: every statistic a covered layer hands over, cloned at that point of the stream
    handed = {}
    orig_add = bnstats.Collector.add

    def tap_add(self, bn, stats, M):
        handed.setdefault(bn.moving_mean.pnp_name, []).append((stats[0].clone(), stats[1].clone()))
        return orig_add(self, bn, stats, M)

    cols = []
    orig_finish = bnstats.Collector.finish

    def tap_finish(self):
        cols.append(self)
        return orig_finish(self)

    monkeypatch.setattr(bnstats.Collector, "add", tap_add)
    monkeypatch.setattr(bnstats.Collector, "finish", tap_finish)
    batches = 2
    src = Stream(77, **_stream_kw(kind))
    covered, slices = _recal(kind, scope, tr, src, batches)
    torch.cuda.synchronize()
    assert slices == batches * B and len(covered) == 2 * N_COVERED[(kind, scope)]
    col = cols[0]
    for (mm, _), acc in zip(col.moving, col.acc):
        per_pass = handed[mm.pnp_name]
        assert len(per_pass) == batches
        ref = np.zeros(acc.numel())
        C = mm.numel()
        for s1, s2 in per_pass:
            ref[:C] = ref[:C] + s1.cpu().numpy()
            ref[C:] = ref[C:] + s2.cpu().numpy()
        assert _bits(acc.cpu().numpy(), ref), "%s: accumulator is not the pass-ordered sum" % mm.pnp_name

    # 2: the fp64 oracle network run on the same batches, training-mode BN on the covered layers, keep_prob 1
    monkeypatch.setattr(T, "batch_norm", tap_bn)
    with torch.no_grad():
        for b in range(batches):
            x = Stream(77, **_stream_kw(kind))
            x.calls = b
            xb = x.next()[0].cpu().double()
            if kind == "seg":
                o64.forward(xb, 1.0, True)
            else:
                o64.segment(xb, "ct", 1.0, front_bn=True, joint_bn=(scope == "all"))
    assert len(pooled) == N_COVERED[(kind, scope)]
    # A layer's forward is fp32-grade (3-term bf16 split or fp32 SIMT), and each batch norm re-normalises what reaches it, so
    # the relative error of a layer's statistics grows with its depth d (1-based, in forward order): 2e-4 * d of the channel's
    # standard deviation for the mean, 4e-4 * d relative for the variance
    live = {v.pnp_name: v for v in rt.global_variables()}
    for d, (scope_name, vals) in enumerate(pooled.items(), start=1):
        x = torch.cat(vals, 0)
        n = x.shape[0]
        m = x.mean(0)
        v = ((x - m) ** 2).sum(0) / (n - 1)
        got_m = live[scope_name + "/moving_mean"].double().cpu()
        got_v = live[scope_name + "/moving_variance"].double().cpu()
        sd = v.sqrt() + 1e-6
        err_m = float(((got_m - m).abs() / sd).max())
        err_v = float(((got_v - v).abs() / (v + 1e-12)).max())
        assert err_m <= 2e-4 * d and err_v <= 4e-4 * d, (scope_name, d, err_m, err_v)


def _all_state(tr, kind):
    st = tr.checkpoint_state()
    return {k: np.asarray(v).copy() for k, v in st.items()}


@pytest.mark.parametrize("kind,scope", CASES, ids=IDS)
def test_nothing_else_moves_and_old_statistics_do_not_matter(kind, scope, monkeypatch):
    from pnp_b200 import bnstats, runtime as rt
    from oracle import bn_population_exact as E
    from pnp_b200.ema import EMA
    net, tr, _ = _build(kind)
    arena = tr.arena if kind == "seg" else tr.g_arena
    tr.ema = EMA(arena, [v for v in rt.global_variables() if v.pnp_kind == "bn_moving" and (kind == "seg" or "adapt" in v.pnp_name)],
                 0.99)
    tr.ema.update()                               # shadows away from the live values
    # a captured step (its warm-up step moves the variables and slots first) is released by the call
    x, ct = Stream(5).next()[0], Stream(6, shift=0.3, scale=0.8).next()[0]
    if kind == "seg":
        from tests.models import step_onehot
        assert tr.capture_train_step(x, step_onehot(B, 23).cuda(), 1.0, warmup=1)
    else:
        assert tr.capture_joint_step(x, ct, 1.0, warmup=1)
    before = _all_state(tr, kind)
    snap = rt.state_dict()
    covered, _ = _recal(kind, scope, tr, Stream(9, **_stream_kw(kind)), 3)
    assert tr._graph is None
    after = _all_state(tr, kind)
    assert set(before) == set(after)
    moved = [k for k in before if not _bits(before[k], after[k])]
    assert set(moved) <= set(covered), sorted(set(moved) - set(covered))[:5]
    assert len(moved) == len(covered)
    result = {k: after[k] for k in covered}

    # 4: the same call from NaN statistics writes the population of what its own layers handed over
    rt.load_state_dict(snap)
    with torch.no_grad():
        for k in covered:
            rt.graph.vars[k].fill_(float("nan"))
    handed, cols = {}, []
    orig_add, orig_finish = bnstats.Collector.add, bnstats.Collector.finish

    def tap_add(self, bn, stats, M):
        handed.setdefault(bn.moving_mean.pnp_name, []).append((stats[0].clone(), stats[1].clone(), M))
        return orig_add(self, bn, stats, M)

    def tap_finish(self):
        cols.append(self)
        return orig_finish(self)

    monkeypatch.setattr(bnstats.Collector, "add", tap_add)
    monkeypatch.setattr(bnstats.Collector, "finish", tap_finish)
    _recal(kind, scope, tr, Stream(9, **_stream_kw(kind)), 3)
    again = rt.state_dict()
    for mm, mv in cols[0].moving:
        passes = [(s1.cpu().numpy(), s2.cpu().numpy(), M) for s1, s2, M in handed[mm.pnp_name]]
        m, v = E.recalibrate(passes)
        assert np.all(np.isfinite(m)) and np.all(np.isfinite(v)), mm.pnp_name
        assert _bits(again[mm.pnp_name], m) and _bits(again[mv.pnp_name], v), mm.pnp_name
        var = result[mv.pnp_name]
        assert _stat_close(mm.pnp_name, again[mm.pnp_name], result[mm.pnp_name], var), mm.pnp_name
        assert _stat_close(mv.pnp_name, again[mv.pnp_name], var, var), mv.pnp_name


@pytest.mark.parametrize("kind,scope", CASES, ids=IDS)
def test_a_raise_mid_run_restores_the_statistics(kind, scope):
    from pnp_b200 import functional as F, runtime as rt
    net, tr, _ = _build(kind)
    before = rt.state_dict()
    with pytest.raises(RuntimeError, match="source failed"):
        _recal(kind, scope, tr, Stream(3, fail_at=2, **_stream_kw(kind)), 5)      # two passes moved the statistics
    after = rt.state_dict()
    for k in before:
        assert _bits(before[k], after[k]), k
    assert F.BN_COLLECTOR is None
    # the argument errors
    with pytest.raises(ValueError):
        _recal(kind, scope, tr, Stream(3), 0)
    with pytest.raises(ValueError):
        _recal(kind, scope, tr, Stream(3, batch=B + 1), 2)
    for k, v in rt.state_dict().items():
        assert _bits(before[k], v), k


def test_standalone_batch_norm_and_a_second_visit_raise():
    from pnp_b200 import bnstats, layers as L, runtime as rt
    net, tr, _ = _build("seg")
    covered = bnstats.covered_statistics([v for v in rt.global_variables() if v.pnp_kind == "bn_moving"])
    before = rt.state_dict()
    with pytest.raises(RuntimeError, match="standalone"):
        with bnstats.collecting(covered) as col, torch.no_grad():
            col.begin_pass()
            L.batch_norm(torch.randn(B, 8, 8, 16, device="cuda"), True, scope="loose")
    with pytest.raises(RuntimeError, match="twice"):
        with bnstats.collecting(covered) as col, torch.no_grad():
            x = Stream(1).next()[0]
            col.begin_pass()
            net.forward(x, 1.0, main_bn=True, adapt_bn=True)
            net.forward(x, 1.0, main_bn=True, adapt_bn=True)
    with pytest.raises(RuntimeError, match="values per channel"):
        with bnstats.collecting(covered) as col, torch.no_grad():
            for b in (B, 1):
                x = Stream(1, batch=2).next()[0][:b].contiguous()
                col.begin_pass()
                net.forward(x, 1.0, main_bn=True, adapt_bn=True)
                col.end_pass()
    after = rt.state_dict()
    for k in before:
        assert _bits(before[k], after[k]), k


@pytest.mark.parametrize("kind,scope", CASES, ids=IDS)
def test_inference_and_a_captured_step_equal_a_fresh_trainer_from_the_checkpoint(kind, scope, tmp_path):
    from pnp_b200 import bnstats, functional as F, lib, runtime as rt
    from tests.models import step_images, step_onehot
    net, tr, _ = _build(kind)
    x = step_images(B, 21).cuda()
    ct = step_images(B, 22, 0.3, 0.8).cuda()
    y = step_onehot(B, 23).cuda()
    _recal(kind, scope, tr, Stream(13, **_stream_kw(kind)), 3)
    coherence.audit(rt, F)
    ck = lib._save(bnstats.recalibrated_checkpoint(tr), str(tmp_path / "recal"))
    live = rt.state_dict()

    def run(tr):
        with torch.no_grad():
            logits = (tr._logits(x) if kind == "seg" else tr._ct_logits(ct)).cpu().numpy()
        rt.manual_seed(3)
        if kind == "seg":
            assert tr.capture_train_step(x, y, 1.0, warmup=1)
            out = tr.train_step_replay(x, y, 1.0)
        else:
            assert tr.capture_joint_step(x, ct, 1.0, warmup=1)
            out = tr.joint_step(x, ct, 1.0)
        flat = [t for t in (out if kind == "seg" else [u for terms in out for u, _ in terms])]
        return logits, [t.detach().cpu().numpy().copy() for t in flat]

    got = run(tr)
    net2, tr2, _ = _build(kind)
    net2.restore(ck)
    restored = rt.state_dict()
    for k in live:
        assert _bits(restored[k], live[k]), k
    ref = run(tr2)
    assert _close(got[0], ref[0], np.abs(ref[0]).max()), "inference logits differ"
    # the replayed losses follow one warm-up optimizer step, which amplifies the forward's run-to-run spread (Adam's first step
    # moves every weight by about +-lr whatever its gradient's size), so the segmenter's are held to 5 %.  The WGAN terms are
    # differences of near-equal critic means, with no relative scale of their own: they are only required to be finite
    for a, b in zip(got[1], ref[1]):
        a, b = float(a), float(b)
        assert np.isfinite(a) and np.isfinite(b)
        if kind == "seg":
            assert abs(a - b) <= 0.05 * max(abs(a), abs(b)) + 1e-6, ("captured step outputs differ", a, b)


def test_cli_end_to_end_on_phantom_subjects(tmp_path):
    from pnp_b200 import bnstats, lib, native, nifti, runtime as rt
    ct_pairs = ph.write_pairs(str(tmp_path), "ct", [61, 62], shape=(40, 36, 30), spacing=(0.8, 1.1, 1.7))
    pairs_file = str(tmp_path / "ct_train_pairs")
    with open(pairs_file, "w") as f:
        f.writelines("%s %s\n" % p for p in ct_pairs)
    for kind in ("gan", "segmenter"):
        tr = native.build_trainer(kind, None, B)
        st = rt.state_dict()
        st["pnp/global_step"] = np.int64(41)
        for name in ("latest", "latest_ema"):
            lib._save(st, str(tmp_path / ("%s_%s" % (kind, name))))
        outs = []
        for name, run in (("latest", "a"), ("latest", "b"), ("latest_ema", "c")):
            out = str(tmp_path / ("%s_%s_bn_%s.npz" % (kind, name, run)))
            argv = ["--trainer", kind, "--checkpoint", str(tmp_path / ("%s_%s.npz" % (kind, name))), "--out", out,
                    "--volumes", pairs_file, "--batches", "3", "--batch-size", str(B), "--seed", "5"]
            names, slices = bnstats.main(argv)
            assert slices == 3 * B and len(names) == (40 if kind == "gan" else 60)
            outs.append(out)
        a, b, c = (np.load(o) for o in outs)
        assert set(a.files) == set(rt.graph.order) | {"pnp/global_step"} and int(a["pnp/global_step"]) == 41
        covered = set(names)
        for k in a.files:
            if k in covered:
                var = a[k.replace("moving_mean", "moving_variance")]
                assert _stat_close(k, b[k], a[k], var) and _stat_close(k, c[k], a[k], var), k
            else:
                assert _bits(a[k], b[k]) and _bits(a[k], c[k]), k
        assert any(not _bits(a[k], st[k]) for k in names)
        tr = native.build_trainer(kind, outs[0], B)
        res = tr.test_native(ct_pairs[:1], str(tmp_path / ("native_" + kind)))
        lab = nifti.load(res[0]["path"]).get_data()
        assert lab.shape == nifti.load(ct_pairs[0][0]).get_data().shape
