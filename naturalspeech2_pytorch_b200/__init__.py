"""H100-native (sm_90a) implementation of the NaturalSpeech2 denoiser hot path.

Public names mirror naturalspeech2_pytorch/__init__.py:8-24 for the path this package accelerates:
`Model` (the denoiser) and, once imported below, `NaturalSpeech2` (diffusion wrapper) and `EncodecRVQ`
(the residual-VQ step of the codec).  All compute goes through libns2b200.so (see include/ns2_b200.h).
"""
from . import _lib, ops  # noqa: F401
from .model import Model  # noqa: F401
from .diffusion import NaturalSpeech2  # noqa: F401
from .codec import EncodecRVQ  # noqa: F401
from .seanet import SEANetDecoder, SEANetEncoder  # noqa: F401
from . import parallel  # noqa: F401
from .aligner import maximum_path  # noqa: F401
from .encoders import (Conditioner, DurationPitchPredictor, PhonemeEncoder,  # noqa: F401
                       SpeechPromptEncoder)

__version__ = "0.1.0"
