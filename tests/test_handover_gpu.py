"""SURVEY 8(f) rows on the device:
  f1  the phase hand-over chain  train_segmenter.py -> checkpoint -> train_gan.py --phase pre-train
      (reference: train_gan.py:74-77, adversarial.py:796-801 = restore(no_gan) -> _load_batch_norm_weights -> _adapt_copy_weights,
      :503-531, :706-765) executed end to end on the GPU and compared with the oracle, whose side of the transplant is done
      independently in numpy from the reference's own name lists (tests/golden/reference_var_names.json = lists/half_zip_*_vars,
      lists/old_bn_list, lists/pred_bn_list);
  f3  the evaluation path (adversarial.py:894-922 / 993-1052: inference-mode BN -- folded into the wgmma epilogue here --,
      keep_prob 1, hard Dice + confusion matrix) against the oracle.
"""
import json
import os

import numpy as np
import pytest
import torch

from tests.util import check
from tests.models import bn_noise, loss_close, state_close

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
B = 2


def reference_transplant(ckpt, P, gold):
    """what adversarial.py:503-531 (no_gan), :743-765 and :706-741 do to a freshly initialised GAN graph, on plain dicts"""
    out = dict(P)
    for k, v in ckpt.items():                                                    # restore(no_gan=True)
        if k in out and not any(s in k for s in ("adapt", "cls", "Adam")) and ("group" in k or "output" in k):
            out[k] = np.asarray(v)
    for old, new in zip(gold["old_bn_list"], gold["pred_bn_list"]):              # _load_batch_norm_weights
        new = new.split(":")[0]
        out["group_%s/%s" % (new.split("_")[1], new)] = np.asarray(ckpt[old.split(":")[0]])
    for mr, ad in zip(gold["half_zip_mri_vars"], gold["half_zip_ct_vars"]):      # _adapt_copy_weights
        out[ad.split(":")[0]] = out[mr.split(":")[0]]
    return out


def test_segmenter_checkpoint_hands_over_to_pretrain_discriminator_step(tmp_path):
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv, source_segmenter as seg
    from pnp_b200.train_gan import configure
    from oracle.pnp_graphs import (OracleAdversarial, OracleSegmenter, init_numpy_params, synthetic_images, synthetic_labels)
    rt.set_conv_backend("auto")
    gold = json.load(open(os.path.join(HERE, "golden", "reference_var_names.json")))
    # ---- phase 0: source segmenter, two Adam steps on the GPU, checkpoint --------------------------------------------
    ws, bns = OracleSegmenter.layout()
    Pseg = init_numpy_params(ws, bns, 0, 0.05)
    net = seg.Full_DRN(channels=3, n_class=5, batch_size=B,
                       cost_kwargs={"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0, "regularizer": 1e-4})
    rt.load_state_dict(Pseg)
    tr = seg.Trainer(net, [], [], num_cls=5, batch_size=B, optimizer="adam", opt_kwargs={"learning_rate": 1e-3})
    x, lab = synthetic_images(B, 1234), synthetic_labels(B, 99)
    xg, yg = tr.feed(x, torch.from_numpy(lab))
    for _ in range(2):
        tr.train_step(xg, yg, keep_prob=1.0)
    out_dir = str(tmp_path / "seg")
    os.makedirs(out_dir)
    tr.save(os.path.join(out_dir, "model.cpkt"), out_dir)
    ck_path = os.path.join(out_dir, "latest.npz")
    ckpt = dict(np.load(ck_path))
    assert "group_3/Variable_1/Adam" in ckpt and "pnp/global_step" in ckpt and int(ckpt["pnp/global_step"]) == 2
    assert not np.array_equal(ckpt["BatchNorm_5/moving_mean"], np.zeros_like(ckpt["BatchNorm_5/moving_mean"]))
    # ---- phase 1: pre-train graph, the reference's restore chain ------------------------------------------------------
    ws, bns = OracleAdversarial.layout()
    Padv = init_numpy_params(ws, bns, 1, 0.05)            # a DIFFERENT seed: everything the chain must overwrite differs
    bn_noise(Padv, bns, 11)
    for n, s in ws:
        if "cls" in n:
            Padv[n] = np.clip(Padv[n] * 0.5, -0.05, 0.05).astype(np.float32)
    ck, nc, tc = configure("pre-train")
    anet = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc, critic_keep_prob=1.0)
    rt.load_state_dict(Padv)
    atr = adv.Trainer(anet, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": 3e-4}, train_config=tc)
    anet.restore(ck_path, no_gan=True)
    anet.load_batch_norm_weights(ck_path)
    anet.adapt_copy_weights()
    want = reference_transplant(ckpt, Padv, gold)
    got = rt.state_dict()
    moved = 0
    for n in want:
        assert np.array_equal(got[n], want[n]), "transplant mismatch at %s" % n
        moved += int(not np.array_equal(want[n], Padv[n]))
    print("  transplant: %d of %d variables overwritten from the segmenter checkpoint, all bit-identical to the reference's mapping" % (moved, len(want)))
    assert moved >= 33 + 120 + 101
    # ---- the first pre-train D step on the transplanted state vs the oracle on the same state --------------------------
    oracle = OracleAdversarial(want, B, lambda_mask_loss=0, dis_sub_iter=tc["dis_sub_iter"], gen_sub_iter=1, critic_keep_prob=1.0)
    mr, ct = synthetic_images(B, 1234), synthetic_images(B, 4321, 0.3, 0.8)
    ro = oracle.d_step(mr, ct, keep_prob=1.0)
    terms = atr.d_step(mr.to(DEV), ct.to(DEV), keep_prob=1.0)
    loss_close("dis_loss after hand-over", atr.loss_value(terms), ro["dis_loss"], 2e-3 * float(ro["mr_cls"].abs().max()))
    state_close(rt, oracle, 1e-3, only=lambda n: "cls" in n)
    # ---- and back: a GAN checkpoint restores with its RMSProp slots, learning rate and step --------------------------
    gan_dir = str(tmp_path / "gan")
    os.makedirs(gan_dir)
    atr.dis_optimizer.set_lr(1.23e-4)
    atr.save(os.path.join(gan_dir, "model.cpkt"), gan_dir)
    slots_before = atr.dis_optimizer.slot_state()              # per-variable views (the arena's padding is not part of a checkpoint)
    assert any(float(np.abs(v - 1.0).max()) > 0 for k, v in slots_before.items() if k.endswith("/RMSProp"))
    atr.dis_optimizer.ms.fill_(1.0)
    atr.dis_optimizer.set_lr(3e-4)
    anet.restore(os.path.join(gan_dir, "latest.npz"))
    n = atr.load_optimizer_state(anet.last_restored)
    slots_after = atr.dis_optimizer.slot_state()
    assert n > 0 and all(np.array_equal(slots_before[k], slots_after[k]) for k in slots_before)
    assert abs(atr.dis_optimizer.get_lr() - 1.23e-4) < 1e-10
    atr.dis_optimizer.ms.fill_(1.0)
    anet.restore(os.path.join(gan_dir, "latest.npz"), clear_rms=True)          # 'RMS' names are filtered out (:541)
    assert atr.load_optimizer_state(anet.last_restored, clear_rms=True) == 0 and float(atr.dis_optimizer.ms.min()) == 1.0


def test_evaluation_path_matches_oracle():
    """Trainer.evaluate: CT slices through the DAM + shared back half in inference mode (every BN folded into its
    convolution's epilogue on the tensor-core path), hard Dice with background (lib.py:96-110) and the confusion matrix"""
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv, functional as F
    from pnp_b200.train_gan import configure
    from oracle.pnp_graphs import OracleAdversarial, init_numpy_params, synthetic_images, synthetic_labels
    from oracle.tf14_numpy import label_decomp
    from oracle import tf14_torch as T
    rt.set_conv_backend("auto")
    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 6)
    ck, nc, tc = configure("train-gan")
    net = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc)
    rt.load_state_dict(P)
    trainer = adv.Trainer(net, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": 3e-4}, train_config=tc)
    oracle = OracleAdversarial(P, B, lambda_mask_loss=0.3, dis_sub_iter=1, gen_sub_iter=1)
    ct = synthetic_images(B, 4321, 0.3, 0.8)
    y = torch.from_numpy(label_decomp(5, synthetic_labels(B, 99)))
    F.PROFILE = []
    st = trainer.evaluate(ct.to(DEV), y.to(DEV))
    n_conv = len(F.PROFILE)
    F.PROFILE = None
    with torch.no_grad():
        ref = oracle.segment(ct, "ct", 1.0, False)["logits"]
        logits = net.segment(ct.to(DEV), "ct", 1.0, front_bn=False)["logits"]
    check("evaluation logits", logits, ref, 1e-3)
    d_ref, arr_ref = T.dice_eval(ref.argmax(3), y, 5)
    print("  dice_eval %.6f (oracle %.6f), %d convolution launches in one evaluation forward" % (st["dice_eval"], float(d_ref), n_conv))
    assert abs(st["dice_eval"] - float(d_ref)) <= 1e-3
    assert max(abs(a - float(b)) for a, b in zip(st["dice_arr"], arr_ref)) <= 1e-3
    pred, truth = ref.argmax(3).reshape(-1).numpy(), y.argmax(3).reshape(-1).numpy()
    cm_ref = np.zeros((5, 5), np.int64)
    np.add.at(cm_ref, (truth, pred), 1)
    cm = st["confusion_matrix"]
    assert cm.sum() == B * 256 * 256 and np.abs(cm - cm_ref).sum() <= 2e-3 * cm.sum(), (cm, cm_ref)
    rt.set_conv_backend("auto")


def test_per_volume_evaluation_matches_oracle():
    """Trainer.test_eval_volume (adversarial.py:993-1052 without the NIfTI reader): a synthetic [256,256,D] subject, frames fed with
    their neighbours as channels, confusion matrix over the subject -> per-class Dice / Jaccard (lib.py:121-152) == the same
    protocol run on the oracle"""
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv
    from pnp_b200.data import label_maps
    from pnp_b200.lib import _dice, _jaccard
    from pnp_b200.train_gan import configure
    from oracle.pnp_graphs import OracleAdversarial, init_numpy_params
    rt.set_conv_backend("auto")
    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 6)
    ck, nc, tc = configure("train-gan")
    net = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc)
    rt.load_state_dict(P)
    trainer = adv.Trainer(net, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": 3e-4}, train_config=tc)
    D = 7                                   # 5 usable frames -> floor(7 / 2) = 3 batches of 2, as the reference counts them
    rng = np.random.RandomState(3)
    raw = rng.randn(256, 256, D).astype(np.float32)
    raw_y = np.transpose(label_maps(D, 55), (1, 2, 0)).copy()
    dice, jac, cm, pred = trainer.test_eval_volume(raw, raw_y, flip_correction=True, shuffle_seed=9)
    # the same protocol on the oracle
    oracle = OracleAdversarial(P, B, lambda_mask_loss=0.3, dis_sub_iter=1, gen_sub_iter=1)
    r2, y2 = np.flip(np.flip(raw, 0), 1), np.flip(np.flip(raw_y, 0), 1)
    frames = list(range(1, D - 1))
    np.random.RandomState(9).shuffle(frames)
    cm_ref = np.zeros((5, 5), np.int64)
    for ii in range(D // B):
        idx = frames[ii * B:(ii + 1) * B]
        vol = np.zeros((B, 256, 256, 3), np.float32)
        sl = np.zeros((B, 256, 256), np.int64)
        for k, jj in enumerate(idx):
            vol[k] = r2[..., jj - 1:jj + 2]
            sl[k] = y2[..., jj]
        with torch.no_grad():
            p_ref = oracle.segment(torch.from_numpy(vol), "ct", 1.0, False)["logits"].argmax(3).numpy()
        np.add.at(cm_ref, (sl.reshape(-1), p_ref.reshape(-1)), 1)
    print("  per-class Dice   ours", np.round(dice, 5), "oracle", np.round(_dice(cm_ref), 5))
    print("  per-class Jaccard ours", np.round(jac, 5), "oracle", np.round(_jaccard(cm_ref), 5))
    assert cm.sum() == cm_ref.sum() == (D // B) * B * 256 * 256
    assert np.abs(cm - cm_ref).sum() <= 2e-3 * cm.sum()
    assert np.abs(dice - _dice(cm_ref)).max() <= 1e-3 and np.abs(jac - _jaccard(cm_ref)).max() <= 1e-3


def test_test_eval_on_nifti_subjects_both_trainers(tmp_path):
    """`Trainer.test_eval` of both trainers (adversarial.py:993-1052, source_segmenter.py:572-632) end to end: NIfTI subjects on disk
    -> lib.read_nii_image -> flip -> frame batches -> inference-mode forward on the GPU -> confusion matrix / Dice / Jaccard ->
    cm.csv, dense predictions as .nii.gz.  With every frame fed (D - 2 <= floor(D / B) * B) the subject's confusion matrix does not
    depend on the shuffle, so it must equal `test_eval_volume` of the same arrays; the host protocol itself is pinned to the
    executed reference on CPU (tests/test_nifti_eval_cpu.py)."""
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv, source_segmenter as seg
    from pnp_b200.data import label_maps
    from pnp_b200.lib import write_nii, read_nii_image, _dice, _jaccard
    from pnp_b200.train_gan import configure
    from oracle.pnp_graphs import OracleAdversarial, OracleSegmenter, init_numpy_params
    rt.set_conv_backend("auto")
    depths = [5, 6]
    rng = np.random.RandomState(21)
    nii, lab, vols = [], [], []
    for i, D in enumerate(depths):
        raw = rng.randn(256, 256, D).astype(np.float32)
        raw_y = np.transpose(label_maps(D, 70 + i), (1, 2, 0)).astype(np.int16)
        nii.append(write_nii(raw, "ct_%d_image.nii.gz" % i, str(tmp_path)))
        lab.append(write_nii(raw_y, "ct_%d_label.nii.gz" % i, str(tmp_path)))
        vols.append((raw, raw_y))
    # ---- adversarial trainer: the adapted CT stream -----------------------------------------------------------------
    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 6)
    ck, nc, tc = configure("train-gan")
    net = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc)
    rt.load_state_dict(P)
    trainer = adv.Trainer(net, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": 3e-4}, train_config=tc, test_label_list=lab,
                          test_nii_list=nii)
    out = str(tmp_path / "adv_out")
    os.makedirs(out)
    np.random.seed(3)
    dice_list, jac_quirk = trainer.test_eval(out, flip_correction=True, save_result=True)
    per_subject = [trainer.test_eval_volume(r, y, flip_correction=True, shuffle_seed=17) for r, y in vols]
    cm_sum = sum(s[2] for s in per_subject)
    cm_csv = np.loadtxt(os.path.join(out, "cm.csv"))
    assert cm_csv.sum() == cm_sum.sum() == sum((D // B) * B for D in depths) * 256 * 256
    assert np.abs(cm_csv - cm_sum).sum() <= 1e-4 * cm_sum.sum()
    np.testing.assert_allclose(dice_list, np.mean([s[0] for s in per_subject], 0), atol=1e-3)
    assert np.asarray(jac_quirk).shape == (1, 2)
    for (d, j), s in zip(trainer.sample_eval_list, per_subject):
        np.testing.assert_allclose(d, s[0], atol=1e-3)
        np.testing.assert_allclose(j, s[1], atol=1e-3)
    for i, D in enumerate(depths):
        p = read_nii_image(os.path.join(out, "dense_pred", "dense_pred_ct_%d_image.nii.gz" % i))
        assert p.shape == (256, 256, D) and p.min() >= 0 and p.max() <= 4 and not p[..., 0].any() and not p[..., D - 1].any()
        agree = (p[..., 1:D - 1] == per_subject[i][3][..., 1:D - 1]).mean()
        print("  subject %d: saved prediction agrees with test_eval_volume on %.5f of the voxels" % (i, agree))
        assert agree >= 1 - 1e-4
    # ---- segmenter trainer: frames in order --------------------------------------------------------------------------
    ws, bns = OracleSegmenter.layout()
    Ps = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(Ps, bns, 6)
    snet = seg.Full_DRN(channels=3, n_class=5, batch_size=B,
                        cost_kwargs={"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0})
    rt.load_state_dict(Ps)
    st = seg.Trainer(snet, None, None, num_cls=5, batch_size=B, test_nii_list=nii, test_label_list=lab, optimizer="adam",
                     opt_kwargs={"learning_rate": 1e-3})
    out2 = str(tmp_path / "seg_out")
    os.makedirs(out2)
    dice2, _ = st.test_eval(out2, flip_correction=False, save_result=True)
    ref = [st.test_eval_volume(r, y, flip_correction=False) for r, y in vols]
    np.testing.assert_allclose(dice2, np.mean([s[0] for s in ref], 0), atol=1e-12)
    oracle = OracleSegmenter(Ps, B)
    r0, y0 = vols[0]
    vol = np.stack([r0[..., 0:3], r0[..., 1:4]])                                  # frames 1 and 2: the first batch of subject 0
    with torch.no_grad():
        p_ref = oracle.forward(torch.from_numpy(vol), 1.0, False)["logits"].argmax(3).numpy()
    p = read_nii_image(os.path.join(out2, "test_pred", "dense_pred_ct_0_image.nii.gz"))
    agree = np.mean([(p[..., 1] == p_ref[0]).mean(), (p[..., 2] == p_ref[1]).mean()])
    print("  segmenter test_eval: saved prediction agrees with the oracle's argmax on %.5f of the voxels" % agree)
    assert agree >= 1 - 2e-3
    assert np.abs(ref[0][0] - _dice(ref[0][2])).max() == 0 and np.abs(ref[0][1] - _jaccard(ref[0][2])).max() == 0


def _read_events(log_dir):
    from tensorboard.backend.event_processing.event_file_loader import RawEventFileLoader
    from tensorboard.compat.proto import event_pb2
    (fn,) = [f for f in os.listdir(log_dir) if f.startswith("events.out.tfevents.")]
    evs = [event_pb2.Event.FromString(raw) for raw in RawEventFileLoader(os.path.join(log_dir, fn)).Load()]
    assert evs[0].file_version == "brain.Event:2"
    return [(ev.step, [(v.tag, v.simple_value) for v in ev.summary.value]) for ev in evs[1:]]


def test_training_loops_run_end_to_end_on_the_device(tmp_path):
    """`Trainer.train` of both trainers on the GPU for a few iterations, the way the entry scripts call them (source_segmenter.py:429-523,
    adversarial.py:767-946): optimizer steps, the monitoring passes with their TensorBoard scalar summaries (event files read back with
    the `tensorboard` package), and for the GAN loop the checkpoint -> re-read -> LR x 0.98 sequence."""
    pytest.importorskip("tensorboard")
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv, source_segmenter as seg
    from pnp_b200.train_gan import configure
    rt.set_conv_backend("auto")
    # ---- source segmenter: 6 Adam steps, monitoring at steps 0 and 5 -------------------------------------------------
    torch.manual_seed(0)
    net = seg.Full_DRN(channels=3, n_class=5, batch_size=B,
                       cost_kwargs={"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0, "regularizer": 1e-4})
    tr = seg.Trainer(net, [], [], num_cls=5, batch_size=B, optimizer="adam", opt_kwargs={"learning_rate": 1e-3})
    out = str(tmp_path / "seg")
    tr.train(out, training_iters=6, epochs=1, display_step=5, dropout=0.75)
    assert tr.global_step == 6
    for sub in ("train_log", "val_log"):
        evs = _read_events(os.path.join(out, sub))
        assert [s for s, _ in evs] == [0, 5]
        for _, vals in evs:
            d = dict(vals)
            assert tuple(t for t, _ in vals) == seg.Trainer.SCALAR_TAGS and all(np.isfinite(v) for v in d.values())
            assert abs(d["loss"] - (d["weighted_loss"] + d["dice_loss"])) <= 1e-5 * max(1.0, abs(d["loss"]))
            assert 0.0 <= d["dice_eval"] <= 1.0 and d["regularizer_loss"] > 0
        lines = [json.loads(ln) for ln in open(os.path.join(out, sub, "scalars.jsonl"))]
        assert [ln["step"] for ln in lines] == [0, 5] and abs(lines[1]["loss"] - dict(evs[1][1])["loss"]) <= 1e-6 * max(1.0, abs(lines[1]["loss"]))
    # ---- GAN loop: steps 0..4, D and G updates at 1..4, monitoring at 0/2/4, checkpoint + re-read + LR decay at step 3 -----------
    ck, nc, tc = configure("train-gan")
    tc.update(dis_sub_iter=1, gen_sub_iter=1, checkpoint_space=3, iter_upd_interval=2, dis_sub_iter_inc=1)
    anet = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc)
    atr = adv.Trainer(anet, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": 3e-4}, train_config=tc)
    out = str(tmp_path / "gan")
    atr.train(out, restore=False, training_iters=5, epochs=1, dropout=0.75, display_step=2)
    # D updates: steps 1, 2 x1, steps 3, 4 x2 (the sub-iteration count grows AFTER the updates of steps 2 and 4) = 6; G updates: 4
    assert atr.global_step == 10 and atr.dis_sub_iter == 3
    assert os.path.exists(os.path.join(out, "latest.npz")) and any(f.startswith("model.cpkt-") for f in os.listdir(out))
    assert atr.dis_optimizer.get_lr() == pytest.approx(3e-4 * 0.98) and atr.gen_optimizer.get_lr() == pytest.approx(3e-4 * 0.98)
    for sub in ("train_log", "val_log"):
        evs = _read_events(os.path.join(out, sub + tc["tag"]))
        assert [s for s, _ in evs] == [0, 2, 4]
        for _, vals in evs:
            assert tuple(t for t, _ in vals) == adv.Trainer.SCALAR_TAGS and all(np.isfinite(v) for _, v in vals)
        assert dict(evs[0][1])["learning_rate"] == pytest.approx(3e-4) and dict(evs[2][1])["learning_rate"] == pytest.approx(3e-4 * 0.98)
    ckpt = dict(np.load(os.path.join(out, "latest.npz")))
    assert any(k.endswith("/RMSProp") for k in ckpt) and "cls_scope/cls_out/Variable" in ckpt
    w = ckpt["cls_scope/cls_out/Variable"]
    assert np.abs(w).max() <= 0.03 + 1e-7                                   # the clip after every D update
