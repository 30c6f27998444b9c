"""Image summaries on the H100: pnp_image_summary_u8 bit for bit against the numpy restatement of TF-1.4's ImageSummaryOp
(tests/image_summary_oracle.py) for all three source kinds, and both trainers' `train` loops writing them into TensorBoard event
files when asked to (and never touching the kernel when not)."""
import os

import numpy as np
import pytest
import torch

from tests.image_summary_oracle import compact_panels, first_argmax, image_summary_u8

pytestmark = pytest.mark.gpu


def _variant(rng, k, H, W, C):
    """one image of a channel source: 0 random with planted NaN / +-inf, 1 all zero, 2 below the zero threshold, 3 all negative,
    4 all positive"""
    if k == 0:
        a = (rng.standard_normal((H, W, C)) * 3).astype(np.float32)
        for v in (np.nan, np.inf, -np.inf):
            a[rng.randint(H), rng.randint(W), :] = v
        return a
    if k == 1:
        return np.zeros((H, W, C), np.float32)
    if k == 2:
        return (rng.uniform(-9e-7, 9e-7, (H, W, C))).astype(np.float32)
    if k == 3:
        return -rng.uniform(0.5, 4.0, (H, W, C)).astype(np.float32)
    return rng.uniform(0.25, 7.0, (H, W, C)).astype(np.float32)


def _logits(rng, B, H, W, C):
    """random logits with planted exact ties, and pixels whose pixel_softmax2 values tie although the logits do not: exp underflow
    (0/0 -> clipped to -1e15), exp overflow (inf/inf -> -1e15) and a denormal step (exp(0) == exp(1e-30) in fp32)"""
    l = (rng.standard_normal((B, H, W, C)) * 2).astype(np.float32)
    flat = l.reshape(-1, C)
    P = flat.shape[0]
    idx = rng.permutation(P)
    q = max(1, P // 16)
    ties = idx[:q]
    flat[ties, C - 1] = flat[ties].max(axis=1)                  # exact tie between the first max and the last class
    under = idx[q:2 * q]
    flat[under] = np.float32(-200.0) + np.arange(C, dtype=np.float32)
    over = idx[2 * q:3 * q]
    flat[over] = np.float32(89.0) + np.arange(C, dtype=np.float32)
    den = idx[3 * q:4 * q]
    flat[den] = np.float32(-5.0)
    flat[den, 0] = 0.0
    flat[den, C - 1] = np.float32(1e-30)
    return flat.reshape(B, H, W, C)


@pytest.mark.parametrize("B", [1, 2, 5])
@pytest.mark.parametrize("HW", [(256, 256), (37, 53)])
@pytest.mark.parametrize("C", [3, 5, 8])
def test_kernel_is_bit_identical_to_the_oracle(B, HW, C):
    import pnp_b200  # noqa: F401
    from pnp_b200 import functional as F
    H, W = HW
    rng = np.random.RandomState(B * 1000 + H + C)
    n = min(B, 3)
    for k in range(5):                                                # every image variant at every image position
        x = np.stack([_variant(rng, (i + k) % 5, H, W, C) for i in range(B)])
        y = rng.randint(0, 3, size=(B, H, W, C)).astype(np.float32)    # small integers: many exact ties
        logits = _logits(rng, B, H, W, C)
        xd, yd, ld = (torch.from_numpy(a).cuda() for a in (x, y, logits))
        got = F.image_summary([(xd, "channel", 1), (yd, "argmax", 0), (ld, "softmax2_argmax", 0), (xd, "channel", C - 1)])
        assert got.dtype == np.uint8 and got.shape == (4, n, H, W)
        np.testing.assert_array_equal(got[0], image_summary_u8(x[..., 1:2]))
        np.testing.assert_array_equal(got[1], compact_panels(first_argmax(y)))
        cls = torch.argmax(F.pixel_softmax2(ld), 3).cpu().numpy()
        assert (cls != first_argmax(logits)).any()                     # the softmax ties really differ from the logits' argmax
        np.testing.assert_array_equal(got[2], compact_panels(cls))
        np.testing.assert_array_equal(got[3], image_summary_u8(x[..., C - 1:C]))
        if k == 0 and B > 1:
            assert (got[0][0] == 255).sum() >= 3 and (got[0][1] == 0).all()     # bad colour; all-zero image


def test_launcher_rejects_bad_arguments():
    import ctypes
    import pnp_b200  # noqa: F401
    from pnp_b200 import _C, functional as F, runtime as rt
    x = torch.zeros(2, 8, 8, 9, device="cuda")
    out = torch.zeros(16, 2, 8, 8, dtype=torch.uint8, device="cuda")

    def launch(ns, kind, C, ch, n, B=2):
        arr = lambda v: (ctypes.c_int * ns)(*([v] * ns))
        return _C.lib.pnp_image_summary_u8((ctypes.c_void_p * ns)(*([x.data_ptr()] * ns)), arr(kind), arr(C), arr(ch), ns, B, 8, 8, n,
                                           out.data_ptr(), rt.stream())
    assert launch(1, 0, 9, 1, 2) == 0
    assert launch(1, 0, 9, 9, 2) == 100001            # channel >= C
    assert launch(1, 0, 9, 1, 3) == 100001            # n > B
    assert launch(1, 1, 9, 0, 2) == 100002            # C > 8 for an argmax kind
    assert launch(7, 0, 9, 1, 1) == 100002            # more than 6 sources
    assert launch(1, 5, 9, 0, 1) == 100001            # unknown kind
    torch.cuda.synchronize()
    with pytest.raises(_C.Unsupported):
        F.image_summary([(x, "argmax", 0)])


def _events(log_dir):
    from tensorboard.backend.event_processing.event_file_loader import RawEventFileLoader
    from tensorboard.compat.proto import event_pb2
    files = [f for f in os.listdir(log_dir) if f.startswith("events.out.tfevents.")]
    assert len(files) == 1, files
    evs = [event_pb2.Event.FromString(raw) for raw in RawEventFileLoader(os.path.join(log_dir, files[0])).Load()]
    assert evs[0].file_version == "brain.Event:2"
    return evs[1:]


class _Spy(object):
    def __init__(self, real):
        self.real = real
        self.calls = []

    def __call__(self, sources, max_outputs=3):
        out = self.real(sources, max_outputs)
        self.calls.append(([(t.detach().clone(), k, c) for t, k, c in sources], out.copy()))
        return out


def _check_log(log_dir, tags, steps, calls):
    """scalar event then image event at each step; images decode to the spy's panels, which equal the oracle on the pass's tensors"""
    import cv2
    from pnp_b200.summary import image_tags
    evs = _events(log_dir)
    assert [e.step for e in evs] == [s for s in steps for _ in range(2)]
    for j, st in enumerate(steps):
        sc, im = evs[2 * j], evs[2 * j + 1]
        assert all(v.WhichOneof("value") == "simple_value" for v in sc.summary.value)
        sources, u8 = calls[j]
        n = u8.shape[1]
        assert [v.tag for v in im.summary.value] == [t for name in tags for t in image_tags(name, n)]
        vals = iter(im.summary.value)
        for s, (t, kind, c) in enumerate(sources):
            a = t.cpu().numpy()
            if kind == "channel":
                want = image_summary_u8(a[..., c:c + 1])
            elif kind == "argmax":
                want = compact_panels(first_argmax(a))
            else:
                from pnp_b200 import functional as F
                want = compact_panels(torch.argmax(F.pixel_softmax2(t), 3).cpu().numpy())
            np.testing.assert_array_equal(u8[s], want)
            for i in range(n):
                v = next(vals)
                assert (v.image.height, v.image.width, v.image.colorspace) == (256, 256, 1)
                dec = cv2.imdecode(np.frombuffer(v.image.encoded_image_string, np.uint8), cv2.IMREAD_UNCHANGED)
                assert dec.shape == (256, 256) and np.array_equal(dec, u8[s, i])


def _run_both(tmp_path, monkeypatch, image_summaries):
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv, source_segmenter as seg, functional as F
    from pnp_b200.train_gan import configure
    spy = _Spy(F.image_summary)
    monkeypatch.setattr(F, "image_summary", spy)
    rt.set_conv_backend("auto")
    B = 2
    torch.manual_seed(0)
    net = seg.Full_DRN(channels=3, n_class=5, batch_size=B,
                       cost_kwargs={"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0, "regularizer": 1e-4})
    tr = seg.Trainer(net, [], [], num_cls=5, batch_size=B, optimizer="adam", opt_kwargs={"learning_rate": 1e-3})
    seg_out = str(tmp_path / "seg")
    tr.train(seg_out, training_iters=6, epochs=1, display_step=5, dropout=0.75, image_summaries=image_summaries)
    seg_calls = list(spy.calls)
    del spy.calls[:]
    ck, nc, tc = configure("train-gan")
    tc.update(dis_sub_iter=1, gen_sub_iter=1, checkpoint_space=100)
    anet = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc)
    atr = adv.Trainer(anet, num_cls=5, batch_size=B, opt_kwargs={"learning_rate": 3e-4}, train_config=tc)
    gan_out = str(tmp_path / "gan")
    atr.train(gan_out, restore=False, training_iters=5, epochs=1, dropout=0.75, display_step=2, image_summaries=image_summaries)
    return seg, adv, seg_out, seg_calls, gan_out, tc["tag"], list(spy.calls)


def test_training_loops_write_image_summaries(tmp_path, monkeypatch):
    pytest.importorskip("tensorboard")
    pytest.importorskip("cv2")
    seg, adv, seg_out, seg_calls, gan_out, tag, gan_calls = _run_both(tmp_path, monkeypatch, True)
    # segmenter: per display step the training pass (train_log) then the validation pass (val_log)
    assert len(seg_calls) == 4
    _check_log(os.path.join(seg_out, "train_log"), seg.Trainer.TRAIN_IMAGE_TAGS, [0, 5], seg_calls[0::2])
    _check_log(os.path.join(seg_out, "val_log"), seg.Trainer.VAL_IMAGE_TAGS, [0, 5], seg_calls[1::2])
    for sources, _ in seg_calls:
        assert [k for _, k, _ in sources] == ["softmax2_argmax", "channel", "argmax"] and sources[0][0].shape[-1] == 5
    # GAN: both passes write the training list, never ct_val_*
    assert len(gan_calls) == 6
    _check_log(os.path.join(gan_out, "train_log" + tag), adv.Trainer.TRAIN_IMAGE_TAGS, [0, 2, 4], gan_calls[0::2])
    _check_log(os.path.join(gan_out, "val_log" + tag), adv.Trainer.TRAIN_IMAGE_TAGS, [0, 2, 4], gan_calls[1::2])
    for sources, _ in gan_calls:
        assert [k for _, k, _ in sources] == ["softmax2_argmax", "channel", "argmax"] * 2


def test_image_summaries_off_leaves_scalar_events_only(tmp_path, monkeypatch):
    pytest.importorskip("tensorboard")
    seg, adv, seg_out, seg_calls, gan_out, tag, gan_calls = _run_both(tmp_path, monkeypatch, False)
    assert seg_calls == [] and gan_calls == []
    for d, steps in ((os.path.join(seg_out, "train_log"), [0, 5]), (os.path.join(seg_out, "val_log"), [0, 5]),
                     (os.path.join(gan_out, "train_log" + tag), [0, 2, 4]), (os.path.join(gan_out, "val_log" + tag), [0, 2, 4])):
        evs = _events(d)
        assert [e.step for e in evs] == steps
        assert all(v.WhichOneof("value") == "simple_value" for e in evs for v in e.summary.value)
