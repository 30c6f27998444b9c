"""H100-native (sm_90a) implementation of the PnP-AdaNet data-parallel hot path
(carrenD/Medical-Cross-Modality-Domain-Adaptation): the dilated-residual segmenter forward/backward and
the feature-map discriminator's adversarial step, behind the reference's layers.py / ops.py operator
surface and its train_segmenter.py / train_gan.py entry points.

Importable as `pnp_b200` (repo-root alias package; this directory's name is not a Python identifier).
"""
from . import _C, runtime, functional, layers, ops  # noqa: F401

__all__ = ["_C", "runtime", "functional", "layers", "ops"]
