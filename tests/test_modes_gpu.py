"""Opt-in launch modes of the C-ABI library, each in its own process (the switches are read once per process):
PNP_PDL=1 (programmatic dependent launch on every kernel) and
PNP_TAIL5=3 / 0 (register-tiled 5x5 tail kernels in both directions -- the default, set explicitly here -- / the generic tail kernels) must give the same operator parity as the defaults, eagerly and through CUDA-graph replay.
Each re-run asserts how many tests its selection holds in the file it runs."""
import pytest

from tests.cabi import rerun

pytestmark = pytest.mark.gpu


def _run(env, file, selection, n):
    passed, lines = rerun(env, file, selection, timeout=850)
    print("\n".join(lines[-15:]))
    assert passed == n, "%d of %d tests passed" % (passed, n)


@pytest.mark.timeout(900)
def test_operator_parity_with_pdl():
    _run({"PNP_PDL": "1", "PNP_TAIL5": "3"}, "tests/test_ops_gpu.py",
         "tensor_core or wide_layers or fused_epilogue or residual or conv_bn or tail", 99)


@pytest.mark.timeout(900)
def test_graph_replay_with_pdl():
    _run({"PNP_PDL": "1"}, "tests/test_models_gpu.py", "cuda_graph_replay_equals_eager_steps", 1)


@pytest.mark.timeout(300)
def test_tail_parity_with_generic_kernels():
    _run({"PNP_TAIL5": "0"}, "tests/test_ops_gpu.py", "tail", 4)
