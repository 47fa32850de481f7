"""H100-native (sm_90a) implementation of the e2-tts-pytorch flow-matching hot path.

Same public surface as the reference package (`/root/reference/e2_tts_pytorch/__init__.py:1-8` minus the
trainer): `E2TTS`, `DurationPredictor`, `Transformer`, `MelSpec`, `E2TTSReturn`, and the `Vocos` decoder E2TTS loads. Host code is Python/PyTorch
(memory, streams, autograd graph, DDP); all arithmetic on the path runs in libb200e2tts.so.
"""

from .modules import (  # noqa: E402,F401
    E2TTS, DurationPredictor, Transformer, MelSpec, E2TTSReturn, LossBreakdown, inject_randomness,
    list_str_to_tensor, lens_to_mask, mask_from_frac_lengths,
)
from .vocos import Vocos  # noqa: E402,F401
from . import lib, ops, optim  # noqa: E402,F401
from .graphed import GraphedTrainStep, BucketedTrainStep  # noqa: E402,F401
from .sampler import GraphedSampler  # noqa: E402,F401
from .optim import GradSync, FusedAdoptEMA, broadcast_module  # noqa: E402,F401

__all__ = ['E2TTS', 'DurationPredictor', 'Transformer', 'MelSpec', 'E2TTSReturn', 'LossBreakdown', 'inject_randomness', 'GraphedTrainStep', 'BucketedTrainStep', 'GraphedSampler', 'Vocos', 'GradSync', 'FusedAdoptEMA', 'broadcast_module']
