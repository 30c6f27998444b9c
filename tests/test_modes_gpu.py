"""Opt-in launch modes of the C-ABI library, each in its own process (the switches are read once per process):
PNP_PDL=1 (programmatic dependent launch on every kernel) and
PNP_TAIL5=3 / 0 (register-tiled 5x5 tail kernels in both directions -- the default, set explicitly here -- / the generic tail kernels) must give the same operator parity as the defaults, eagerly and through CUDA-graph replay."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(env_extra, args):
    env = dict(os.environ)
    env.update(env_extra)
    p = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider"] + args, cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=850)
    tail = "\n".join(p.stdout.splitlines()[-15:])
    assert p.returncode == 0, tail
    return tail


@pytest.mark.timeout(900)
def test_operator_parity_with_pdl():
    tail = _run({"PNP_PDL": "1", "PNP_TAIL5": "3"},
                ["tests/test_ops_gpu.py", "-k", "tensor_core or wide_layers or fused_epilogue or residual or conv_bn or tail"])
    print(tail)


@pytest.mark.timeout(900)
def test_graph_replay_with_pdl():
    tail = _run({"PNP_PDL": "1"}, ["tests/test_models_gpu.py", "-k", "cuda_graph_replay_equals_eager_steps"])
    print(tail)


@pytest.mark.timeout(300)
def test_tail_parity_with_generic_kernels():
    tail = _run({"PNP_TAIL5": "0"}, ["tests/test_ops_gpu.py", "-k", "tail"])
    print(tail)
