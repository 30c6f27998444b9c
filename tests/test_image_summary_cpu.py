"""TensorBoard image summaries without a GPU: the numpy restatement of TF-1.4's ImageSummaryOp (tests/image_summary_oracle.py) on
hand-derived answers, the PNG encoder against two independent decoders (OpenCV, Pillow), the Summary.Image bytes against the
`tensorboard` package's protobuf classes, event files read back by TensorBoard's EventAccumulator, and the trainers' tags and
per-pass routing against the reference's own wiring (tests/golden/reference_image_summaries.json)."""
import json
import os

import numpy as np
import pytest

from tests.image_summary_oracle import image_summary_u8

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_image_summaries.json")


def _row(vals):
    return np.asarray(vals, np.float32).reshape(1, 1, -1, 1)


@pytest.mark.parametrize("vals,want", [
    ([0, 1, 2, 4], [0, 63, 127, 255]),
    ([1, 2, 3, 4], [63, 127, 191, 255]),
    ([-2, 0, 1, 2], [1, 128, 191, 255]),
    ([-3, 3, 1], [1, 255, 170]),
    ([-0.1, 0.3], [85, 255]),
    ([-7, 7, np.nan, np.inf], [1, 255, 255, 255]),          # non-finite pixels: excluded from the bounds, bad_color[0] = 255
    ([-7, 7, -np.inf, np.nan], [1, 255, 255, 255]),
    ([0, 0, 0], [0, 0, 0]),
    ([-5e-7, 2e-7], [128, 128]),                            # max |v| below the 1e-6 zero threshold: scale 0, offset 128
    ([5e-7, 2e-7], [0, 0]),
    ([np.nan, np.inf], [255, 255]),
])
def test_oracle_known_answers(vals, want):
    got = image_summary_u8(_row(vals))
    assert got.dtype == np.uint8 and got.shape == (1, 1, len(vals))
    assert got[0, 0].tolist() == want


def test_oracle_image_count_and_per_image_normalisation():
    for B, n in ((1, 1), (2, 2), (5, 3)):
        x = np.arange(B * 2 * 3, dtype=np.float32).reshape(B, 2, 3, 1) * np.float32(0.5)
        got = image_summary_u8(x)
        assert got.shape == (n, 2, 3)
        for i in range(n):
            assert got[i].max() == 255                       # every image reaches 255 on its own maximum
    assert image_summary_u8(np.zeros((5, 4, 4, 1), np.float32), max_outputs=1).shape == (1, 4, 4)


def test_image_tags_follow_image_summary_op():
    import pnp_b200  # noqa: F401
    from pnp_b200.summary import image_tags
    assert image_tags("image_1", 3) == ["image_1/image/0", "image_1/image/1", "image_1/image/2"]
    assert image_tags("GND", 1) == ["GND/image/0"]


@pytest.mark.parametrize("shape,kind", [((256, 256), "random"), ((256, 256), "constant"), ((1, 1), "random"), ((37, 53), "random"),
                                        ((37, 53), "constant"), ((1, 1), "constant")])
def test_png_round_trip_through_two_decoders(shape, kind):
    import pnp_b200  # noqa: F401
    from pnp_b200.summary import encode_png
    cv2 = pytest.importorskip("cv2")
    Image = pytest.importorskip("PIL.Image")
    import io
    rng = np.random.RandomState(hash((shape, kind)) & 0xFFFF)
    a = rng.randint(0, 256, size=shape).astype(np.uint8) if kind == "random" else np.full(shape, 173, np.uint8)
    png = encode_png(a)
    assert png[:8] == b"\x89PNG\r\n\x1a\n" and png.count(b"IDAT") == 1
    d1 = cv2.imdecode(np.frombuffer(png, np.uint8), cv2.IMREAD_UNCHANGED)
    assert d1.dtype == np.uint8 and d1.shape == shape and np.array_equal(d1, a)
    im = Image.open(io.BytesIO(png))
    im.load()
    assert im.mode == "L" and im.size == (shape[1], shape[0]) and np.array_equal(np.asarray(im), a)


def test_image_summary_bytes_equal_tensorboard_protobuf():
    pytest.importorskip("tensorboard")
    import pnp_b200  # noqa: F401
    from pnp_b200 import summary
    from tensorboard.compat.proto import summary_pb2
    rng = np.random.RandomState(3)
    panels = [("train_pred/image/0", rng.randint(0, 5, (37, 53)).astype(np.uint8)), ("image/image/0", rng.randint(0, 256, (1, 1)).astype(np.uint8)),
              ("GND/image/1", np.zeros((256, 256), np.uint8))]
    msg = summary_pb2.Summary()
    for tag, a in panels:
        v = msg.value.add()
        v.tag = tag
        v.image.height, v.image.width, v.image.colorspace = a.shape[0], a.shape[1], 1
        v.image.encoded_image_string = summary.encode_png(a)
    ours = summary.encode_image_summary(panels)
    assert ours == msg.SerializeToString()
    back = summary_pb2.Summary.FromString(ours)
    assert [v.tag for v in back.value] == [t for t, _ in panels]


def test_event_file_with_scalar_and_image_events_reads_back(tmp_path):
    pytest.importorskip("tensorboard")
    cv2 = pytest.importorskip("cv2")
    import pnp_b200  # noqa: F401
    from pnp_b200 import summary
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator, DEFAULT_SIZE_GUIDANCE, IMAGES
    w = summary.FileWriter(str(tmp_path / "train_log"))
    rng = np.random.RandomState(5)
    written = {}
    for step in (0, 5):
        w.add_scalars({"loss": 1.5 + step}, step)
        panels = [(t, rng.randint(0, 256, (37, 53)).astype(np.uint8)) for t in summary.image_tags("image", 2)]
        w.add_images(panels, step)
        written[step] = dict(panels)
    w.close()
    acc = EventAccumulator(w.logdir, size_guidance=dict(DEFAULT_SIZE_GUIDANCE, **{IMAGES: 0}))
    acc.Reload()
    assert sorted(acc.Tags()["images"]) == ["image/image/0", "image/image/1"] and acc.Tags()["scalars"] == ["loss"]
    for tag in ("image/image/0", "image/image/1"):
        evs = acc.Images(tag)
        assert [e.step for e in evs] == [0, 5]
        for e in evs:
            assert (e.width, e.height) == (53, 37)
            dec = cv2.imdecode(np.frombuffer(e.encoded_image_string, np.uint8), cv2.IMREAD_UNCHANGED)
            assert np.array_equal(dec, written[e.step][tag])


def _fixture():
    with open(GOLDEN) as f:
        return json.load(f)


def _routing(rec):
    """per monitoring call: (writer, step, [tags of the merged image op written after the scalars])"""
    merged = {m["op"]: m for m in rec["merged"]}
    out = []
    for call in rec["monitor_calls"]:
        w = rec["writes"][call["first_write"]:call["first_write"] + 2]
        assert [merged[x["summary"].split(":", 1)[1]]["kinds"] for x in w] == [["scalar"], ["image"]]     # scalars, then images
        assert w[0]["writer"] == w[1]["writer"] and w[0]["step"] == w[1]["step"]                          # same writer, same step
        assert [x["summary"] for x in w] == ["value_of:" + op for op in call["fetch_merged"]]
        out.append((w[1]["writer"], w[1]["step"], merged[call["fetch_merged"][1]]["tags"]))
    return out


def test_segmenter_image_tags_and_routing_match_the_reference():
    import pnp_b200  # noqa: F401
    from pnp_b200.source_segmenter import Trainer
    rec = _fixture()["source_segmenter"]
    ims = rec["image_summaries"]
    assert all(not s["max_outputs_passed"] and s["max_outputs"] == 3 for s in ims)
    by_list = {}
    for s in ims:
        by_list.setdefault(s["lists"][0], []).append(s["tag"])
    assert sorted(by_list.values()) == sorted([list(Trainer.TRAIN_IMAGE_TAGS), list(Trainer.VAL_IMAGE_TAGS)])
    assert [s["name"] for s in ims if s["tag"] == "image_1"] == ["image"]                  # the uniquified second 'image'
    # provenance: compact_pred = argmax(pixel_wise_softmax_2(logits)), x[:,:,:,1], compact_y = argmax(y)
    kinds = [("pixel_wise_softmax_2" in s["tensor"] and s["tensor"].startswith("argmax("), s["tensor"].endswith("[:,:,:,1]"),
              s["tensor"].startswith("argmax(ph:")) for s in ims]
    assert kinds == [(True, False, False), (False, True, False), (False, False, True)] * 2
    # training pass -> train_log with TRAIN_IMAGE_TAGS, validation pass -> val_log with VAL_IMAGE_TAGS, at every display step
    steps = sorted({st for _, st, _ in _routing(rec)})
    assert steps == [0, 5]
    for st in steps:
        assert [(w, t) for w, s_, t in _routing(rec) if s_ == st] == [("train_log", list(Trainer.TRAIN_IMAGE_TAGS)),
                                                                     ("val_log", list(Trainer.VAL_IMAGE_TAGS))]


def test_gan_image_tags_and_routing_match_the_reference():
    import pnp_b200  # noqa: F401
    from pnp_b200.adversarial import Trainer
    rec = _fixture()["adversarial"]
    ims = rec["image_summaries"]
    assert all(not s["max_outputs_passed"] and s["max_outputs"] == 3 for s in ims)
    train = [s["tag"] for s in ims if s["lists"] == ["merged_1"]]
    val = [s["tag"] for s in ims if s["lists"] == ["merged_2"]]
    assert tuple(train) == Trainer.TRAIN_IMAGE_TAGS and tuple(val) == Trainer.VAL_IMAGE_TAGS
    src = {s["tag"]: s["tensor"] for s in ims}
    assert "pixel_wise_softmax_2" in src["ct_pred"] and "pixel_wise_softmax_2" in src["mri_validation_pred"]
    assert src["ct_image"].endswith("[:,:,:,1]") and src["mri_image"].endswith("[:,:,:,1]")
    assert src["ct_gt"].startswith("argmax(ph:") and src["mri_gt"].startswith("argmax(ph:")
    tag = rec["loop_args"]["tag"]
    routing = _routing(rec)
    assert [(w, s) for w, s, _ in routing] == [(sub + tag, st) for st in (0, 2, 4) for sub in ("train_log", "val_log")]
    # both passes write the TRAIN list; the validation list (ct_val_*) is never fetched
    assert all(t == list(Trainer.TRAIN_IMAGE_TAGS) for _, _, t in routing)
    assert not any(c["fetch_merged"][1] == "merged_2" for c in rec["monitor_calls"])


def test_image_summaries_are_off_by_default():
    import inspect
    import pnp_b200  # noqa: F401
    from pnp_b200 import adversarial, source_segmenter
    for fn in (adversarial.Trainer.train, adversarial.Trainer.output_minibatch_stats, source_segmenter.Trainer.train,
               source_segmenter.Trainer.output_minibatch_stats, source_segmenter.Trainer.val_stats):
        assert inspect.signature(fn).parameters["image_summaries"].default is False, fn
