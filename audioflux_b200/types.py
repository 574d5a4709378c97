"""Enum ints shared with the C ABI (reference: src/flux_base.h:14-168,
python/audioflux/type/basic.py:25-353). Same names and values."""
from enum import Enum


class WindowType(Enum):
    RECT = 0
    HANN = 1
    HAMM = 2
    BLACKMAN = 3
    KAISER = 4
    BARTLETT = 5
    TRIANG = 6
    FLATTOP = 7
    GAUSS = 8
    BLACKMAN_HARRIS = 9
    BLACKMAN_NUTTALL = 10
    BARTLETT_HANN = 11
    BOHMAN = 12
    TUKEY = 13


class SpectralDataType(Enum):
    POWER = 0
    MAG = 1


class SpectralFilterBankScaleType(Enum):
    LINEAR = 0
    LINSPACE = 1
    MEL = 2
    BARK = 3
    ERB = 4
    OCTAVE = 5
    LOG = 6


class SpectralFilterBankStyleType(Enum):
    SLANEY = 0
    ETSI = 1
    GAMMATONE = 2
    POINT = 3
    RECT = 4
    HANN = 5
    HAMM = 6
    BLACKMAN = 7
    BOHMAN = 8
    KAISER = 9
    GAUSS = 10


class SpectralFilterBankNormalType(Enum):
    NONE = 0
    AREA = 1
    BAND_WIDTH = 2


class NSGTFilterBankType(Enum):
    """src/nsgt_algorithm.h:14-18"""
    EFFICIENT = 0
    STANDARD = 1


class CepstralRectifyType(Enum):
    LOG = 0
    CUBIC_ROOT = 1


class CepstralEnergyType(Enum):
    REPLACE = 0
    APPEND = 1
    IGNORE = 2


class ChromaDataNormalType(Enum):
    NONE = 0
    MAX = 1
    MIN = 2
    P2 = 3
    P1 = 4


class SpectralNoveltyMethodType(Enum):
    SUB = 0
    ENTROY = 1      # the reference's spelling
    KL = 2
    IS = 3


class SpectralNoveltyDataType(Enum):
    VALUE = 0
    NUMBER = 1


class PaddingPositionType(Enum):
    CENTER = 0
    RIGHT = 1
    LEFT = 2


class PaddingModeType(Enum):
    CONSTANT = 0
    REFLECT = 1
    WRAP = 2


class ReassignType(Enum):
    ALL = 0
    FRE = 1
    TIME = 2
    NONE = 3


class WaveletContinueType(Enum):
    MORSE = 0
    MORLET = 1
    BUMP = 2
    PAUL = 3
    DOG = 4
    MEXICAN = 5
    HERMIT = 6
    RICKER = 7


class WaveletDiscreteType(Enum):
    HAAR = 0
    DB = 1
    SYM = 2
    COIF = 3
    FK = 4
    BIOR = 5
    DMEY = 6


class ResampleQualityType(Enum):
    """src/dsp/resample_algorithm.h"""
    BEST = 0
    MID = 1
    FAST = 2


class XcorrNormalType(Enum):
    """normalisation of a cross-correlation (include/dsp/xcorr_algorithm.h:14-18)"""
    NONE = 0
    COEFF = 1


class NoveltyType(Enum):
    """novelty function of an onset (include/mir/onset_algorithm.h:13-30)"""
    FLUX = 0
    HFC = 1
    SD = 2
    SF = 3
    MKL = 4
    PD = 5
    WPD = 6
    NWPD = 7
    CD = 8
    RCD = 9
    BROADBAND = 10


def enum_value(v):
    return int(v.value) if isinstance(v, Enum) else int(v)
