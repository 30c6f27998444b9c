"""Generate tests/golden/opencv_reference_graph_vectors.npz: logits of the REFERENCE'S traced segmenter graphs computed by a third-party
TensorFlow-graph engine (OpenCV's TensorFlow importer), for the GPU parity tests to compare the CUDA path with directly.

Inputs of the computation, all committed / seeded: the layer-by-layer trace of the reference's graph-building code
(tests/golden/reference_graph_trace.json, produced by executing the reference), seeded parameters (`init_numpy_params(seed 0, stddev
0.05)` + `_bn_noise(seed 6)`: non-trivial BN statistics) and seeded inputs (`synthetic_images`).  The GraphDef construction and the
OpenCV execution are tests/test_reference_graph_in_opencv_cpu.py's (which also checks the same numbers against the oracle).

Stored per graph (B = 2, 256 x 256): the logits at 4096 seeded pixel positions per image and the full argmax map.

    python tests/golden/make_opencv_reference_vectors.py       # needs cv2 + tensorboard; /root/reference is NOT needed
"""
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
OUT = os.path.join(HERE, "opencv_reference_graph_vectors.npz")
N_SAMPLES = 4096


def sample_positions(B, seed=20260924):
    rng = np.random.RandomState(seed)
    return np.stack([rng.choice(256 * 256, N_SAMPLES, replace=False) for _ in range(B)]).astype(np.int32)


def main():
    from tests import test_reference_graph_in_opencv_cpu as G
    from tests.models import bn_noise as _bn_noise
    from oracle.pnp_graphs import OracleSegmenter, OracleAdversarial, init_numpy_params, synthetic_images
    REF = json.load(open(os.path.join(HERE, "reference_graph_trace.json")))
    B = G.B
    pos = sample_positions(B)
    out = {"positions": pos, "batch": np.int64(B)}

    def store(tag, logits):
        flat = logits.reshape(B, 256 * 256, 5)
        out[tag + "_logits_at_positions"] = np.stack([flat[b][pos[b]] for b in range(B)]).astype(np.float32)
        out[tag + "_argmax"] = logits.argmax(-1).astype(np.uint8)
        out[tag + "_max_abs_logit"] = np.float32(np.abs(logits).max())

    # source_segmenter.Full_DRN.create_network
    ws, bns = OracleSegmenter.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    _bn_noise(P, bns, 6)
    with tempfile.TemporaryDirectory() as d:
        _, logits = G.run_stream_in_opencv(REF["source_segmenter"]["events"], P, synthetic_images(B, 1234).numpy(), d, G.SEG_STATS)
    store("segmenter", logits)
    # adversarial.Full_DRN, CT stream (adapt_1..6 + shared back half): the adapted segmenter the evaluation path runs
    ev = REF["events"]
    zipn = [e for e in ev if e["section"] == "create_zip_network#1"]
    start_ct = [i for i, e in enumerate(zipn) if e.get("input_src")][1]
    events = zipn[start_ct:] + [e for e in ev if e["section"] == "create_second_half#1"]
    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    _bn_noise(P, bns, 6)
    with tempfile.TemporaryDirectory() as d:
        _, logits = G.run_stream_in_opencv(events, P, synthetic_images(B, 4321, 0.3, 0.8).numpy(), d, G.SEG_STATS)
    store("gan_ct", logits)
    np.savez_compressed(OUT, **out)
    print("wrote %s (%.0f KB)" % (OUT, os.path.getsize(OUT) / 1e3))


if __name__ == "__main__":
    main()
