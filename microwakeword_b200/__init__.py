"""microwakeword_b200 -- H100-native (sm_90a) streaming inference for microWakeWord.

Host side mirrors the reference's Python surface (`inference.Model`,
`audio.audio_utils.generate_features_for_clip`); the arithmetic lives in libmww_b200.so
(hand-written CUDA behind the C-ABI of include/mww.h).  Importing this package does not touch CUDA.
"""

from .model_file import OKAY_NABU, Arch  # noqa: F401

__all__ = ["OKAY_NABU", "Arch"]
