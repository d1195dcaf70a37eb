"""H100-native streaming Whisper engine behind WhisperLiveKit's backend surface.

Importing the package does not load CUDA; ``whisperlivekit_b200.engine`` loads
the in-tree C-ABI library (``csrc/libwlk_b200.so``) and raises if it is missing.
"""
from .dims import DIMS, ModelDimensions, SpecialTokens, ALIGNMENT_HEADS  # noqa: F401

__version__ = "0.1.0"
