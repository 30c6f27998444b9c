"""The oracle's TensorFlow-kernel semantics against an INDEPENDENT implementation of TensorFlow graph semantics: OpenCV's TensorFlow
importer (`cv2.dnn.readNetFromTensorflow`, OpenCV 4.x in this image), which exists to execute frozen TF graphs and therefore encodes
TF's op definitions -- the 'SAME' padding rule of strided convolutions (the asymmetric (0,1) / (1,2) offsets of SURVEY App. B), the
SpaceToBatchND -> Conv2D(VALID) -> BatchToSpaceND graph that `tf.nn.atrous_conv2d` emits in TF 1.4 (layers.py:86,92), 'SAME' max /
average pooling for any window (padding excluded from the average), FusedBatchNorm in inference mode (epsilon inside the square
root), LeakyRelu(alpha), MatMul and Softmax.

TensorFlow itself cannot run here (DESIGN.md section 2: "TF-kernel numerics unpinned"); this closes the forward half of that gap with
code that is neither ours nor derived from ours.  The GraphDefs are built from the `tensorboard` package's TF protos with exactly the
node types / attributes the reference's calls produce, executed by OpenCV in a separate process (tests/opencv_tf_runner.py), and
compared with oracle/tf14_numpy.py (naive fp64 loops) -- the oracle the GPU parity tests hold the CUDA kernels to.
Not covered by any third-party code in this image: train-mode batch norm (moving-average update), dropout scaling, Adam / RMSProp --
those stay restated from the published TF-1.4 behaviour + known-answer tests."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.opencv_graphdef import const, have_cv2, node, placeholder, protos

pytest.importorskip("tensorboard")
HERE = os.path.dirname(os.path.abspath(__file__))
pytestmark = pytest.mark.skipif(not have_cv2(), reason="OpenCV with the dnn module is not importable")


class Batch(object):
    """collects (graph, input, expected) cases, runs them all in ONE OpenCV process"""

    def __init__(self, d):
        self.d, self.cases = str(d), []

    def add(self, name, nodes, x, expected, tol):
        graph_pb2 = protos()[0]
        g = graph_pb2.GraphDef()
        g.node.extend(nodes)
        open(os.path.join(self.d, name + ".pb"), "wb").write(g.SerializeToString())
        np.save(os.path.join(self.d, name + "_x.npy"), np.asarray(x, np.float32))
        self.cases.append((name, np.asarray(expected, np.float64), tol))

    def run(self):
        json.dump([{"name": n} for n, _, _ in self.cases], open(os.path.join(self.d, "manifest.json"), "w"))
        p = subprocess.run([sys.executable, os.path.join(HERE, "opencv_tf_runner.py"), self.d], capture_output=True, text=True, timeout=600)
        assert p.returncode == 0, p.stderr[-2000:]
        done = json.load(open(os.path.join(self.d, "done.json")))
        assert done["done"] == [n for n, _, _ in self.cases]
        worst = {}
        for name, ref, tol in self.cases:
            y = np.load(os.path.join(self.d, name + "_y.npy")).astype(np.float64)
            assert y.size == ref.size, "%s: OpenCV returned shape %s, the oracle %s" % (name, y.shape, ref.shape)
            if y.ndim == 4:
                assert y.shape == ref.shape, "%s: OpenCV returned shape %s, the oracle %s" % (name, y.shape, ref.shape)
            y = y.reshape(ref.shape)
            err = float(np.abs(y - ref).max() / max(1.0, np.abs(ref).max()))
            worst[name] = err
            assert err <= tol, "%s: OpenCV's TF importer and the oracle differ by %.3e (tol %.1e)" % (name, err, tol)
        return done["opencv"], worst


def _oracle():
    from oracle import tf14_numpy as N
    return N


# (H, W, Cin, Cout, k, stride): every strided / unstrided 'SAME' geometry class of the graphs at reduced size, with the SAME pad parity
# of the real layers -- 256 -> 128 k3 s2 pads (0,1) like 10 -> 5; 128 -> 64 k5 s2 pads (1,2) like 12 -> 6; 16 -> 4 and 128 -> 32 k5 s4
# pad (0,1) like 16 -> 4 and 8 -> 2; odd sizes for good measure
CONV_CASES = [(10, 10, 3, 4, 3, 2), (12, 12, 3, 4, 5, 2), (16, 16, 2, 3, 5, 4), (8, 8, 2, 3, 5, 4), (9, 7, 3, 4, 3, 1), (10, 11, 3, 2, 3, 2),
              (6, 6, 4, 4, 5, 1), (7, 9, 2, 2, 1, 1), (13, 13, 2, 2, 5, 4)]


def test_same_padding_of_strided_convolutions_matches_opencvs_tf_importer(tmp_path):
    N = _oracle()
    rng = np.random.RandomState(0)
    b = Batch(tmp_path)
    for i, (H, W, ci, co, k, s) in enumerate(CONV_CASES):
        x = rng.standard_normal((2, H, W, ci)).astype(np.float32)
        w = rng.standard_normal((k, k, ci, co)).astype(np.float32)
        nodes = [placeholder("x", x.shape), const("w", w),
                 node("y", "Conv2D", ["x", "w"], strides=[1, s, s, 1], padding=b"SAME", data_format=b"NHWC")]     # layers.py:18,67
        b.add("conv%d" % i, nodes, x, N.conv2d(x.astype(np.float64), w.astype(np.float64), stride=s, padding="SAME"), 2e-5)
        pt = N.same_pad(H, k, s)
        if (H, k, s) in ((10, 3, 2), (16, 5, 4), (8, 5, 4)):
            assert pt == (0, 1)                                    # the asymmetric offsets of SURVEY App. B
        if (H, k, s) == (12, 5, 2):
            assert pt == (1, 2)
    ver, worst = b.run()
    print("OpenCV %s: worst relative deviation over %d SAME convolutions %.2e" % (ver, len(worst), max(worst.values())))


def test_atrous_conv2d_graph_of_tf14_matches_the_oracles_dilated_convolution(tmp_path):
    """tf.nn.atrous_conv2d(value, filters, rate, 'SAME') in TF 1.4 is SpaceToBatchND(paddings) -> Conv2D('VALID') -> BatchToSpaceND(crops)
    with paddings = SAME padding of the effective (k + (k-1)(rate-1)) kernel plus what rounds the padded size up to a multiple of rate
    (nn_ops.atrous_conv2d / with_space_to_batch).  The oracle (and the kernels) compute it as a dilated convolution."""
    N = _oracle()
    rng = np.random.RandomState(1)
    b = Batch(tmp_path)
    for i, (H, W, rate, k) in enumerate([(8, 8, 2, 3), (9, 9, 2, 3), (32, 32, 2, 3), (7, 10, 2, 3), (12, 12, 3, 3), (16, 16, 2, 5)]):
        x = rng.standard_normal((2, H, W, 3)).astype(np.float32)
        w = rng.standard_normal((k, k, 3, 4)).astype(np.float32)
        keff = k + (k - 1) * (rate - 1)
        p0 = (keff - 1) // 2
        p1 = keff - 1 - p0
        eh, ew = (rate - (H + p0 + p1) % rate) % rate, (rate - (W + p0 + p1) % rate) % rate
        nodes = [placeholder("x", x.shape), const("w", w), const("bs", [rate, rate], True),
                 const("pads", [[p0, p1 + eh], [p0, p1 + ew]], True), const("crops", [[0, eh], [0, ew]], True),
                 node("s2b", "SpaceToBatchND", ["x", "bs", "pads"]),
                 node("conv", "Conv2D", ["s2b", "w"], strides=[1, 1, 1, 1], padding=b"VALID", data_format=b"NHWC"),
                 node("y", "BatchToSpaceND", ["conv", "bs", "crops"])]
        b.add("atrous%d" % i, nodes, x, N.conv2d(x.astype(np.float64), w.astype(np.float64), stride=1, dilation=rate, padding="SAME"), 2e-5)
    ver, worst = b.run()
    print("OpenCV %s: worst relative deviation over %d atrous convolutions %.2e" % (ver, len(worst), max(worst.values())))


def test_same_pooling_for_any_window_matches_opencvs_tf_importer(tmp_path):
    """tf.nn.max_pool / avg_pool, ksize = strides = n, 'SAME' (layers.py:102-106) -- the n = 2 pooling of the graphs and the general
    geometry behind layers.max_pool2d(x, n) / avg_pool2d(x, n) (csrc/surface.cu): window grid, padding never wins / is not averaged"""
    N = _oracle()
    rng = np.random.RandomState(2)
    b = Batch(tmp_path)
    for i, (H, W, n) in enumerate([(8, 12, 2), (5, 7, 2), (4, 4, 3), (9, 9, 4), (6, 5, 1), (3, 10, 5), (7, 7, 3)]):
        x = rng.standard_normal((2, H, W, 3)).astype(np.float32)
        for op, avg in (("MaxPool", False), ("AvgPool", True)):
            nodes = [placeholder("x", x.shape), node("y", op, ["x"], ksize=[1, n, n, 1], strides=[1, n, n, 1], padding=b"SAME", data_format=b"NHWC")]
            b.add("%s%d" % (op, i), nodes, x, N.pool_same(x.astype(np.float64), n, avg), 1e-6)
    ver, worst = b.run()
    print("OpenCV %s: worst relative deviation over %d poolings %.2e" % (ver, len(worst), max(worst.values())))


def test_inference_batch_norm_activation_matmul_softmax_match_opencvs_tf_importer(tmp_path):
    N = _oracle()
    rng = np.random.RandomState(3)
    b = Batch(tmp_path)
    x = rng.standard_normal((2, 6, 5, 4)).astype(np.float32) * 2
    gam, bet, mu = [rng.uniform(0.5, 1.5, 4).astype(np.float32) for _ in range(3)]
    var = rng.uniform(1e-4, 2.0, 4).astype(np.float32)                              # small variances: epsilon placement matters
    bn_nodes = [placeholder("x", x.shape), const("g", gam), const("b", bet), const("m", mu), const("v", var),
                node("y", "FusedBatchNorm", ["x", "g", "b", "m", "v"], epsilon=1e-3, is_training=False, data_format=b"NHWC")]
    ref_bn, _, _ = N.batch_norm(x.astype(np.float64), gam.astype(np.float64), bet.astype(np.float64), mu.astype(np.float64),
                                var.astype(np.float64), False)
    b.add("bn", bn_nodes, x, ref_bn, 1e-5)
    b.add("lrelu", [placeholder("x", x.shape), node("y", "LeakyRelu", ["x"], alpha=0.2)], x, N.leaky_relu(x.astype(np.float64)), 1e-7)
    b.add("relu", [placeholder("x", x.shape), node("y", "Relu", ["x"])], x, N.relu(x.astype(np.float64)), 1e-7)
    x2 = rng.standard_normal((3, 32)).astype(np.float32)
    w2 = rng.standard_normal((32, 1)).astype(np.float32)
    b.add("fc", [placeholder("x", x2.shape), const("w", w2), node("y", "MatMul", ["x", "w"], transpose_a=False, transpose_b=False)], x2,
          x2.astype(np.float64) @ w2.astype(np.float64), 1e-5)                      # adversarial.py:397,440
    x3 = rng.standard_normal((2, 6, 5, 5)).astype(np.float32) * 3
    b.add("softmax", [placeholder("x", x3.shape), node("y", "Softmax", ["x"])], x3, N.softmax(x3.astype(np.float64)), 1e-6)
    ver, worst = b.run()
    print("OpenCV %s: %s" % (ver, {k: "%.1e" % v for k, v in worst.items()}))
