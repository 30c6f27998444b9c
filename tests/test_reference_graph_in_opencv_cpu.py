"""The reference's segmenter graph executed by a THIRD-PARTY TensorFlow-graph engine, against the oracle, at full size.

Chain of custody:
  reference code --(executed under a recording shim, tests/golden/make_reference_graph_trace.py)--> layer-by-layer trace of
  `Full_DRN.create_network` (source_segmenter.py:88-209): every conv's filter variable, stride, dilation, padding rule, BN scope,
  skip kind, activation; pooling; PS
  --> HERE: a frozen inference GraphDef built from THAT TRACE (not from the product's or the oracle's network code) out of the node
  types TF 1.4 emits for those calls -- Conv2D('SAME'), SpaceToBatchND -> Conv2D('VALID') -> BatchToSpaceND for atrous_conv2d,
  FusedBatchNorm(is_training=False, epsilon=1e-3), Pad (channel pad of the inc_dim skip, layers.py:160) + Add, Maximum(Mul(0.2, x), x)
  for tf.nn.leaky_relu, MaxPool('SAME') -- with the oracle's seeded weights and non-trivial BN statistics
  --> executed by OpenCV's TensorFlow importer (cv2.dnn.readNetFromTensorflow; own process)
  --> compared with `OracleSegmenter.forward(..., bn_train=False)`: the c9_2 feature map (31 convolutions -- 4 of them atrous --, 30 batch norms,
  14 residual skips of which 5 channel-padded, 3 poolings) and the logits.

The three ops OpenCV cannot run for us are bridged outside it by code that is pinned elsewhere: tf.pad(..., 'SYMMETRIC') (OpenCV's
MirrorPad ignores the mode; numpy form pinned by TF's documented example, KAT 3) around the two SYMMETRIC convolutions (executed by
OpenCV as Conv2D('VALID')), and `ops.PS` (its literal emulation, pinned bit-exactly to the EXECUTED reference ops.py:3-27).
B = 2 so that PS takes the batch >= 2 branch the training graphs use."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from tests.opencv_graphdef import const, have_cv2, node, placeholder, protos

pytest.importorskip("tensorboard")
pytestmark = pytest.mark.skipif(not have_cv2(), reason="OpenCV with the dnn module is not importable")
HERE = os.path.dirname(os.path.abspath(__file__))
REF = json.load(open(os.path.join(HERE, "golden", "reference_graph_trace.json")))
B = 2


def _run_opencv(d, name, nodes, x):
    graph_pb2 = protos()[0]
    g = graph_pb2.GraphDef()
    g.node.extend(nodes)
    open(os.path.join(d, name + ".pb"), "wb").write(g.SerializeToString())
    np.save(os.path.join(d, name + "_x.npy"), np.asarray(x, np.float32))
    json.dump([{"name": name}], open(os.path.join(d, "manifest.json"), "w"))
    p = subprocess.run([sys.executable, os.path.join(HERE, "opencv_tf_runner.py"), d], capture_output=True, text=True, timeout=1500)
    assert p.returncode == 0, p.stderr[-2000:]
    y = np.load(os.path.join(d, name + "_y.npy"))
    os.remove(os.path.join(d, name + ".pb"))
    return y


def _conv_nodes(name, src, ev, W):
    """the nodes TF 1.4 emits for conv2d / atrous_conv2d with padding 'SAME' (layers.py:18,67,86)"""
    k, rate, s = ev["wshape"][0], ev["dil"], ev["stride"]
    nodes = [const(name + "/w", W)]
    if rate == 1:
        nodes.append(node(name, "Conv2D", [src, name + "/w"], strides=[1, s, s, 1], padding=b"SAME", data_format=b"NHWC"))
        return nodes
    H, Wd = ev["in"][0], ev["in"][1]
    keff = k + (k - 1) * (rate - 1)
    p0 = (keff - 1) // 2
    p1 = keff - 1 - p0
    eh, ew = (rate - (H + p0 + p1) % rate) % rate, (rate - (Wd + p0 + p1) % rate) % rate
    nodes += [const(name + "/bs", [rate, rate], True), const(name + "/pads", [[p0, p1 + eh], [p0, p1 + ew]], True),
              const(name + "/crops", [[0, eh], [0, ew]], True),
              node(name + "/s2b", "SpaceToBatchND", [src, name + "/bs", name + "/pads"]),
              node(name + "/conv", "Conv2D", [name + "/s2b", name + "/w"], strides=[1, 1, 1, 1], padding=b"VALID", data_format=b"NHWC"),
              node(name, "BatchToSpaceND", [name + "/conv", name + "/bs", name + "/crops"])]
    return nodes


def build_body_from_trace(events, P):
    """GraphDef nodes of every traced layer up to (not including) the first SYMMETRIC convolution; returns (nodes, output name)"""
    nodes = [placeholder("x", [B, 256, 256, 3])]
    cur, prev_in = "x", None
    stats = {"conv": 0, "atrous": 0, "bn": 0, "skip": 0, "pad_skip": 0, "pool": 0}
    for i, ev in enumerate(events):
        if ev["op"] == "maxpool":
            assert ev["k"] == 2 and ev["stride"] == 2 and ev["padding"] == "SAME"
            nodes.append(node("pool%d" % i, "MaxPool", [cur], ksize=[1, 2, 2, 1], strides=[1, 2, 2, 1], padding=b"SAME", data_format=b"NHWC"))
            cur, prev_in = "pool%d" % i, None
            stats["pool"] += 1
            continue
        assert ev["op"] == "conv"
        if ev["padding"] == "SYMMETRIC":
            return nodes, cur, i, stats
        layer_in = cur
        name = "L%d" % i
        nodes += _conv_nodes(name, cur, ev, P[ev["w"]])
        stats["atrous" if ev["dil"] > 1 else "conv"] += 1
        cur = name
        if ev["bn"] is not None:                                   # tf.contrib.layers.batch_norm in inference mode (layers.py:100)
            s = ev["bn"]
            nodes += [const(name + "/gamma", P[s + "/gamma"]), const(name + "/beta", P[s + "/beta"]),
                      const(name + "/mean", P[s + "/moving_mean"]), const(name + "/var", P[s + "/moving_variance"]),
                      node(name + "/bn", "FusedBatchNorm", [cur, name + "/gamma", name + "/beta", name + "/mean", name + "/var"],
                           epsilon=1e-3, is_training=False, data_format=b"NHWC")]
            cur = name + "/bn"
            stats["bn"] += 1
        if ev["skip"] != "none":                                   # residual_block / DR_block: x_s + bn2 (layers.py:160-163,182-186)
            assert prev_in is not None
            src = prev_in
            if ev["skip"].startswith("pad"):
                n = int(ev["skip"][3:])
                nodes += [const(name + "/cpad", [[0, 0], [0, 0], [0, 0], [n, n]], True), node(name + "/xs", "Pad", [src, name + "/cpad"])]
                src = name + "/xs"
                stats["pad_skip"] += 1
            nodes.append(node(name + "/add", "Add", [src, cur]))
            cur = name + "/add"
            stats["skip"] += 1
        if ev["act"] == "lrelu0.2":                                # tf.nn.leaky_relu in TF 1.4: maximum(alpha * x, x)
            nodes += [const(name + "/alpha", np.float32(0.2)), node(name + "/ax", "Mul", [name + "/alpha", cur]),
                      node(name + "/act", "Maximum", [name + "/ax", cur])]
            cur = name + "/act"
        else:
            assert ev["act"] == "none"
        prev_in = layer_in
    raise AssertionError("the trace has no SYMMETRIC convolution")


def run_stream_in_opencv(events, P, x, d, expect_stats):
    """one segmenter stream (front + back half + tail) of a traced graph: returns (c9_2, logits) computed by OpenCV + the two bridges"""
    from oracle import tf14_numpy as N
    nodes, out, i_sym, stats = build_body_from_trace(events, P)
    assert stats == expect_stats, stats
    c9 = _run_opencv(d, "body", nodes, np.asarray(x))
    assert c9.shape == (B, 32, 32, 512)
    # group_10: conv2d(..., padding='SYMMETRIC') = tf.pad SYMMETRIC by k // 2, then 'VALID' (layers.py:68-73); dropout is off (keep 1)
    ev10 = events[i_sym]
    assert ev10["w"] == "group_10/Variable" and ev10["padding"] == "SYMMETRIC" and ev10["bn"] is None and ev10["act"] == "none"
    padded = N.symmetric_pad(c9.astype(np.float64), ev10["wshape"][0] // 2).astype(np.float32)
    conv10 = _run_opencv(d, "g10", [placeholder("x", padded.shape), const("w", P[ev10["w"]]),
                                    node("y", "Conv2D", ["x", "w"], strides=[1, 1, 1, 1], padding=b"VALID", data_format=b"NHWC")], padded)
    evps = events[i_sym + 1]
    assert evps["op"] == "PS" and evps["r"] == 8 and evps["n_channel"] == 40
    flat = N.PS_literal(conv10.astype(np.float64), 8, 40, B)                       # pinned to the executed ops.py
    evo = events[i_sym + 2]
    assert evo["w"] == "output/Variable" and evo["padding"] == "SYMMETRIC" and evo["keep"] == 1.0 and len(events) == i_sym + 3
    padded = N.symmetric_pad(flat, evo["wshape"][0] // 2).astype(np.float32)
    logits = _run_opencv(d, "out", [placeholder("x", padded.shape), const("w", P[evo["w"]]),
                                    node("y", "Conv2D", ["x", "w"], strides=[1, 1, 1, 1], padding=b"VALID", data_format=b"NHWC")], padded)
    return c9, logits


def _compare(tag, c9, logits, ref):
    ref_logits, r9 = ref["logits"].numpy(), ref["c9_2"].numpy()
    e_logits = float(np.abs(logits - ref_logits).max() / np.abs(ref_logits).max())
    e9 = float(np.abs(c9 - r9).max() / np.abs(r9).max())
    agree = float((logits.argmax(-1) == ref_logits.argmax(-1)).mean())
    print("%s: c9_2 max rel err %.3e, logits max rel err %.3e, argmax agreement %.6f" % (tag, e9, e_logits, agree))
    assert logits.shape == ref_logits.shape == (B, 256, 256, 5)
    assert e9 <= 1e-4 and e_logits <= 1e-4 and agree >= 0.9999


SEG_STATS = {"conv": 27, "atrous": 4, "bn": 30, "skip": 14, "pad_skip": 5, "pool": 3}


@pytest.mark.timeout(1800)
def test_reference_segmenter_graph_in_opencv_equals_the_oracle(tmp_path):
    from oracle.pnp_graphs import OracleSegmenter, init_numpy_params, synthetic_images
    from tests.models import bn_noise
    events = REF["source_segmenter"]["events"]
    ws, bns = OracleSegmenter.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 6)
    x = synthetic_images(B, 1234)
    t0 = time.time()
    c9, logits = run_stream_in_opencv(events, P, x.numpy(), str(tmp_path), SEG_STATS)
    t1 = time.time()
    with torch.no_grad():
        ref = OracleSegmenter(P, B, dtype=torch.float64).forward(x.double(), 1.0, False)
    print("OpenCV %.1f s, oracle (fp64) %.1f s" % (t1 - t0, time.time() - t1))
    _compare("source_segmenter.Full_DRN.create_network", c9, logits, ref)


@pytest.mark.timeout(1800)
@pytest.mark.parametrize("stream", ["mr", "ct"])
def test_reference_adversarial_segmenter_streams_in_opencv_equal_the_oracle(tmp_path, stream):
    """adversarial.py:66-92: create_zip_network builds the MR front (group_1..6, BN scopes pred_*) and the CT front (adapt_1..6, BN
    scopes adapt_*); create_second_half (group_7..output, AUTO_REUSE) is called first on the CT features, then on the MR features.
    Each stream's chain of traced layers, with the oracle's GAN-graph parameters, through OpenCV vs OracleAdversarial.segment."""
    from oracle.pnp_graphs import OracleAdversarial, init_numpy_params, synthetic_images
    from tests.models import bn_noise
    ev = REF["events"]
    zipn = [e for e in ev if e["section"] == "create_zip_network#1"]
    starts = [i for i, e in enumerate(zipn) if e.get("input_src")]
    assert len(starts) == 2 and zipn[starts[0]]["input_src"] == "ph:mr_ph" and zipn[starts[1]]["w"] == "adapt_1/Variable"
    front = {"mr": zipn[:starts[1]], "ct": zipn[starts[1]:]}[stream]
    back = [e for e in ev if e["section"] == {"ct": "create_second_half#1", "mr": "create_second_half#2"}[stream]]
    assert all(e["w"].startswith("group_" if stream == "mr" else "adapt_") for e in front if e["op"] == "conv")
    assert all((e["bn"] is None) or ("/pred_" if stream == "mr" else "/adapt_") in e["bn"] for e in front if e["op"] == "conv")
    assert back[0]["w"] == "group_7/Variable" and back[-1]["w"] == "output/Variable"
    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 6)
    x = synthetic_images(B, 1234) if stream == "mr" else synthetic_images(B, 4321, 0.3, 0.8)
    c9, logits = run_stream_in_opencv(front + back, P, x.numpy(), str(tmp_path), SEG_STATS)
    oracle = OracleAdversarial(P, B, lambda_mask_loss=0.3, dis_sub_iter=1, gen_sub_iter=1)
    with torch.no_grad():
        ref = oracle.segment(x, stream, 1.0, False)
    _compare("adversarial.Full_DRN %s stream" % stream, c9, logits, ref)


def test_committed_opencv_vectors_match_the_oracle():
    """the fixture the GPU tests compare the CUDA path with (tests/golden/opencv_reference_graph_vectors.npz) -- read back through the
    very helper the GPU tests use and held against the oracle here, so a fixture / indexing mistake cannot hide behind a GPU tolerance"""
    from oracle.pnp_graphs import OracleSegmenter, OracleAdversarial, init_numpy_params, synthetic_images
    from tests.models import bn_noise
    from tests.util import compare_with_opencv_vectors
    ws, bns = OracleSegmenter.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 6)
    with torch.no_grad():
        lg = OracleSegmenter(P, B).forward(synthetic_images(B, 1234), 1.0, False)["logits"]
    err, agree = compare_with_opencv_vectors("segmenter", lg, 2e-5, 0.99995)
    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    bn_noise(P, bns, 6)
    with torch.no_grad():
        lg = OracleAdversarial(P, B, lambda_mask_loss=0.3, dis_sub_iter=1, gen_sub_iter=1).segment(
            synthetic_images(B, 4321, 0.3, 0.8), "ct", 1.0, False)["logits"]
    compare_with_opencv_vectors("gan_ct", lg, 2e-5, 0.99995)
    # a shifted input must NOT pass: the comparison is not vacuous
    with pytest.raises(AssertionError):
        compare_with_opencv_vectors("gan_ct", torch.roll(lg, 1, dims=2), 2e-5, 0.99995)
