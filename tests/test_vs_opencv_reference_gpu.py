"""CUDA path vs a THIRD-PARTY execution of the reference's graphs -- no oracle in between.

tests/golden/opencv_reference_graph_vectors.npz holds the logits of `source_segmenter.Full_DRN.create_network` and of the adapted CT
stream of `adversarial.Full_DRN` (create_zip_network + create_second_half), computed by OpenCV's TensorFlow importer from a frozen
GraphDef that was built out of the recorded trace of the reference's own graph-building code
(tests/golden/make_opencv_reference_vectors.py; tests/test_reference_graph_in_opencv_cpu.py checks the same numbers against the oracle
on the CPU).  Here the product runs the same seeded parameters and inputs on the GPU -- inference-mode batch norm folded into the
wgmma epilogues, fused tail -- and must reproduce them: logits within 1e-3 of the largest |logit| (north-star tolerance), argmax maps
equal on >= 99.9 % of the pixels."""
import numpy as np
import pytest
import torch

from tests.util import compare_with_opencv_vectors
from tests.test_parity_configs_gpu import _bn_noise

pytestmark = pytest.mark.gpu
B = 2


@pytest.mark.parametrize("backend", ["auto", "simt"])
def test_segmenter_logits_match_the_opencv_executed_reference_graph(backend):
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, source_segmenter as seg
    from oracle.pnp_graphs import OracleSegmenter, init_numpy_params, synthetic_images
    rt.set_conv_backend(backend)
    try:
        ws, bns = OracleSegmenter.layout()
        P = init_numpy_params(ws, bns, 0, 0.05)
        _bn_noise(P, bns, 6)
        net = seg.Full_DRN(channels=3, n_class=5, batch_size=B,
                           cost_kwargs={"cross_flag": True, "miu_cross": 1.0, "dice_flag": True, "miu_dice": 1.0})
        rt.load_state_dict(P)
        x = synthetic_images(B, 1234).cuda()
        with torch.no_grad():
            logits = net.forward(x, keep_prob=1.0, main_bn=False, adapt_bn=False)
        compare_with_opencv_vectors("segmenter", logits, 1e-3, 0.999)
    finally:
        rt.set_conv_backend("auto")


def test_adapted_ct_stream_logits_match_the_opencv_executed_reference_graph():
    import pnp_b200  # noqa: F401
    from pnp_b200 import runtime as rt, adversarial as adv
    from pnp_b200.train_gan import configure
    from oracle.pnp_graphs import OracleAdversarial, init_numpy_params, synthetic_images
    rt.set_conv_backend("auto")
    ws, bns = OracleAdversarial.layout()
    P = init_numpy_params(ws, bns, 0, 0.05)
    _bn_noise(P, bns, 6)
    ck, nc, tc = configure("train-gan")
    net = adv.Full_DRN(channels=3, n_class=5, batch_size=B, cost_kwargs=ck, network_config=nc)
    rt.load_state_dict(P)
    x = synthetic_images(B, 4321, 0.3, 0.8).cuda()
    with torch.no_grad():
        logits = net.segment(x, "ct", 1.0, front_bn=False, joint_bn=False)["logits"]
    compare_with_opencv_vectors("gan_ct", logits, 1e-3, 0.999)
