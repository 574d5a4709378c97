"""audioflux_b200: H100-native (sm_90a) drop-in for audioFlux's time-frequency hot path.

Host-side mirror of the reference's operator interface (same class / method / argument
names as python/audioflux/{stft,bft,cqt,cwt,nsgt,st,fst,cepstrogram,spectrogram}.py, feature/xxcc.py,
dsp/resample.py, dsp/xcorr.py, dsp/czt.py, mir/hpss.py, mir/onset.py, mir/harmonic_ratio.py, mir/pitch_pef.py, mir/pitch_yin.py, mir/pitch_ncf.py, mir/pitch_cep.py, dwt.py / swt.py / wpt.py and classic/nmf.py) over the C-ABI
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
from .spectral import Spectral  # noqa: F401
from .nsgt import NSGT  # noqa: F401
from .st import ST, FST  # noqa: F401
from .cepstrogram import Cepstrogram  # noqa: F401
from .resample import Resample, WindowResample  # noqa: F401
from .hpss import HPSS  # noqa: F401
from .onset import Onset, NoveltyParam  # noqa: F401
from .harmonic_ratio import HarmonicRatio  # noqa: F401
from .pitch_pef import PitchPEF  # noqa: F401
from .pitch_yin import PitchYIN  # noqa: F401
from .pitch_ncf import PitchNCF  # noqa: F401
from .pitch_cep import PitchCEP  # noqa: F401
from .wavelet import DWT, SWT, WPT  # noqa: F401
from .nmf import nmf, nmf_batch  # noqa: F401
from .xcorr import Xcorr  # noqa: F401
from .czt import CZT  # noqa: F401
from . import lib  # noqa: F401

__version__ = "0.1.0"
