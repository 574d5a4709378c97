"""audioflux_b200: H100-native (sm_90a) drop-in for audioFlux's time-frequency hot path.

Host-side mirror of the reference's operator interface (same class / method / argument
names as python/audioflux/{stft,bft,cqt,cwt,spectrogram}.py and feature/xxcc.py) over the C-ABI
library ``lib/libaudioflux_b200.so``.  No CPU fallback exists.
"""
from .types import *  # noqa: F401,F403
from .stft import STFT  # noqa: F401
from .bft import BFT  # noqa: F401
from .xxcc import XXCC  # noqa: F401
from .cqt import CQT  # noqa: F401
from .cwt import CWT  # noqa: F401
from .pwt import PWT  # noqa: F401
from .wsst import WSST, Synsq  # noqa: F401
from .reassign import Reassign  # noqa: F401
from .spectrogram import Spectrogram, MelSpectrogram, BarkSpectrogram, ErbSpectrogram  # noqa: F401
from . import lib  # noqa: F401

__version__ = "0.1.0"
