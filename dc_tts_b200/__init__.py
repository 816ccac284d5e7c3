"""dc_tts_b200 -- H100-native DC-TTS synthesis path (Text2Mel + SSRN).

Host side mirrors the reference's operator API (modules.py / networks.py /
train.Graph / synthesize.py); device side is hand-written sm_90a CUDA behind the
C-ABI declared in include/dctts.h.  There is no CPU fallback: importing the
compute modules without the built shared library raises.
"""
from .hyperparams import Hyperparams  # noqa: F401

__version__ = "0.1.0"
