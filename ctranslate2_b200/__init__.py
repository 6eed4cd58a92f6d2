"""ctranslate2_b200 — the H100-native (sm_90a) quantized-transformer decode path behind CTranslate2's
Generator / ops surface.  Host-side mirror of the reference interface over the C-ABI in include/ct2b200.h.
There is no CPU or PyTorch fallback: importing works anywhere, every compute call needs libct2b200.so and a
H100."""
from . import ops  # noqa: F401
from ._lib import Ct2B200Error, kernel_launch_count, lib, set_random_seed  # noqa: F401
from .encoder import Encoder, EncoderForwardOutput, encoder_summary  # noqa: F401
from .generator import GenerationResult, Generator, ScoringResult, model_summary  # noqa: F401
from .translator import TranslationResult, Translator, translator_summary  # noqa: F401
from .whisper import Whisper, WhisperAlignmentResult, WhisperGenerationResult  # noqa: F401

__version__ = "0.1.0"
