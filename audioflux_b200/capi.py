"""ctypes signatures of the audioFlux C API for the time-frequency hot path.

The same table binds ``libaudioflux_b200.so`` (this repo) and any other library
exporting the reference's symbols (e.g. the reference build used as test oracle),
because the drop-in boundary IS this C ABI:

* reference symbols  -- src/stft_algorithm.h:14-40, src/bft_algorithm.h:14-57,
  src/feature/xxcc_algorithm.h:12-39, src/cqt_algorithm.h:14-62,
  src/cwt_algorithm.h:14-45, src/spectrogram_algorithm.h:40-119 (signatures reproduced in include/*.h)
* additive ``*Batch`` / ``afb200_*`` symbols -- include/afb200_ext.h (only bound when present)
"""
from __future__ import annotations

import ctypes as C

P = C.POINTER
c_int_p = P(C.c_int)
c_float_p = P(C.c_float)
vp = C.c_void_p

# name -> (restype, argtypes)
REFERENCE_API = {
    # ---- STFT
    "stftObj_new": (C.c_int, [P(vp), C.c_int, c_int_p, c_int_p, c_int_p]),
    "stftObj_setSlideLength": (None, [vp, C.c_int]),
    "stftObj_enablePadding": (None, [vp, C.c_int]),
    "stftObj_enableContinue": (None, [vp, C.c_int]),
    "stftObj_setPadding": (None, [vp, c_int_p, c_int_p, c_float_p, c_float_p]),
    "stftObj_useWindowDataArr": (None, [vp, vp]),
    "stftObj_getWindowDataArr": (vp, [vp]),
    "stftObj_calTimeLength": (C.c_int, [vp, C.c_int]),
    "stftObj_calDataLength": (C.c_int, [vp, C.c_int]),
    "stftObj_stft": (None, [vp, vp, C.c_int, vp, vp]),
    "stftObj_istft": (None, [vp, vp, vp, C.c_int, C.c_int, vp]),
    "stftObj_free": (None, [vp]),
    # ---- BFT
    "bftObj_new": (C.c_int, [P(vp), C.c_int, C.c_int, c_int_p, c_float_p, c_float_p, c_int_p,
                             c_int_p, c_int_p, c_int_p, c_int_p, c_int_p, c_int_p, c_int_p, c_int_p]),
    "bftObj_calTimeLength": (C.c_int, [vp, C.c_int]),
    "bftObj_getFreBandArr": (vp, [vp]),
    "bftObj_getBinBandArr": (vp, [vp]),
    "bftObj_setResultType": (None, [vp, C.c_int]),
    "bftObj_setDataNormValue": (None, [vp, C.c_float]),
    "bftObj_bft": (None, [vp, vp, C.c_int, vp, vp]),
    "bftObj_getTemporalData": (None, [vp, P(c_float_p), P(c_float_p), P(c_float_p)]),
    "bftObj_free": (None, [vp]),
    # ---- XXCC
    "xxccObj_new": (C.c_int, [P(vp), C.c_int]),
    "xxccObj_setTimeLength": (None, [vp, C.c_int]),
    "xxccObj_xxcc": (None, [vp, vp, C.c_int, c_int_p, vp]),
    "xxccObj_xxccStandard": (None, [vp, vp, C.c_int, vp, c_int_p, c_int_p, c_int_p, vp, vp, vp]),
    "xxccObj_free": (None, [vp]),
    # ---- CQT
    "cqtObj_new": (C.c_int, [P(vp), C.c_int, C.c_int, C.c_float, c_int_p]),
    "cqtObj_newWith": (C.c_int, [P(vp), C.c_int, c_int_p, c_float_p, c_int_p, c_float_p, c_float_p,
                                 c_float_p, c_int_p, c_int_p, c_int_p, c_int_p, c_int_p]),
    "cqtObj_calTimeLength": (C.c_int, [vp, C.c_int]),
    "cqtObj_getFFTLength": (C.c_int, [vp]),
    "cqtObj_getFreBandArr": (vp, [vp]),
    "cqtObj_setScale": (None, [vp, C.c_int]),
    "cqtObj_cqt": (None, [vp, vp, C.c_int, vp, vp]),
    "cqtObj_chroma": (None, [vp, c_int_p, c_int_p, c_int_p, vp, vp, vp]),
    "cqtObj_cqcc": (None, [vp, vp, C.c_int, c_int_p, vp]),
    "cqtObj_cqhc": (None, [vp, vp, C.c_int, vp]),
    "cqtObj_deconv": (None, [vp, vp, vp, vp]),
    "cqtObj_free": (None, [vp]),
    # ---- CWT
    "cwtObj_new": (C.c_int, [P(vp), C.c_int, C.c_int, c_int_p, c_float_p, c_float_p, c_int_p,
                             c_int_p, c_int_p, c_float_p, c_float_p, c_int_p]),
    "cwtObj_getFreBandArr": (vp, [vp]),
    "cwtObj_getBinBandArr": (vp, [vp]),
    "cwtObj_cwt": (None, [vp, vp, vp, vp]),
    "cwtObj_enableDet": (None, [vp, C.c_int]),
    "cwtObj_cwtDet": (None, [vp, vp, vp, vp]),
    "cwtObj_free": (None, [vp]),
    # ---- PWT (src/pwt_algorithm.h:16-31)
    "pwtObj_new": (C.c_int, [P(vp), C.c_int, C.c_int, c_int_p, c_float_p, c_float_p, c_int_p, c_int_p, c_int_p,
                             c_int_p, c_int_p]),
    "pwtObj_getFreBandArr": (vp, [vp]),
    "pwtObj_getBinBandArr": (vp, [vp]),
    "pwtObj_pwt": (None, [vp, vp, vp, vp]),
    "pwtObj_enableDet": (None, [vp, C.c_int]),
    "pwtObj_pwtDet": (None, [vp, vp, vp, vp]),
    "pwtObj_free": (None, [vp]),
    # reassignment (src/reassign_algorithm.h)
    "reassignObj_new": (C.c_int, [P(vp), C.c_int, c_int_p, c_int_p, c_int_p, c_int_p, c_float_p, c_int_p, c_int_p]),
    "reassignObj_calTimeLength": (C.c_int, [vp, C.c_int]),
    "reassignObj_setResultType": (None, [vp, C.c_int]),
    "reassignObj_setOrder": (None, [vp, C.c_int]),
    "reassignObj_reassign": (None, [vp, vp, C.c_int, vp, vp, vp, vp]),
    "reassignObj_free": (None, [vp]),
    # synchrosqueezing (src/wsst_algorithm.h, src/synsq_algorithm.h)
    "wsstObj_new": (C.c_int, [P(vp), C.c_int, C.c_int, c_int_p, c_float_p, c_float_p, c_int_p, c_int_p, c_int_p,
                              c_float_p, c_float_p, c_float_p, c_int_p]),
    "wsstObj_getFreBandArr": (vp, [vp]),
    "wsstObj_getBinBandArr": (vp, [vp]),
    "wsstObj_setOrder": (None, [vp, C.c_int]),
    "wsstObj_wsst": (None, [vp, vp, vp, vp, vp, vp]),
    "wsstObj_free": (None, [vp]),
    "synsqObj_new": (C.c_int, [P(vp), C.c_int, C.c_int, c_int_p, c_int_p, c_float_p]),
    "synsqObj_synsq": (None, [vp, vp, C.c_int, vp, vp, vp, vp]),
    "synsqObj_free": (None, [vp]),
    # ---- Spectrogram (front door; src/spectrogram_algorithm.h:40-119)
    "spectrogramObj_new": (C.c_int, [P(vp), C.c_int, c_int_p, c_float_p, c_float_p, c_int_p, c_int_p, c_int_p,
                                     c_int_p, c_int_p, c_int_p, c_int_p, c_int_p, c_int_p]),
    "spectrogramObj_newLinear": (C.c_int, [P(vp), C.c_int, C.c_int, c_int_p]),
    "spectrogramObj_newMel": (C.c_int, [P(vp), C.c_int, C.c_int, C.c_int, c_int_p]),
    "spectrogramObj_newBark": (C.c_int, [P(vp), C.c_int, C.c_int, C.c_int, c_int_p]),
    "spectrogramObj_newErb": (C.c_int, [P(vp), C.c_int, C.c_int, C.c_int, c_int_p]),
    "spectrogramObj_newChroma": (C.c_int, [P(vp), C.c_int, C.c_int, c_int_p]),
    "spectrogramObj_newDeep": (C.c_int, [P(vp), C.c_int, C.c_int, C.c_int, c_int_p]),
    "spectrogramObj_newDeepChroma": (C.c_int, [P(vp), C.c_int, C.c_int, c_int_p]),
    "spectrogramObj_enableDebug": (None, [vp, C.c_int]),
    "spectrogramObj_setDataNormValue": (None, [vp, C.c_float]),
    "spectrogramObj_calTimeLength": (C.c_int, [vp, C.c_int]),
    "spectrogramObj_getFreBandArr": (vp, [vp]),
    "spectrogramObj_getBinBandArr": (vp, [vp]),
    "spectrogramObj_getBandNum": (C.c_int, [vp]),
    "spectrogramObj_getBinBandLength": (C.c_int, [vp]),
    "spectrogramObj_spectrogram": (None, [vp, vp, C.c_int, vp, vp]),
    "spectrogramObj_xxcc": (None, [vp, vp, C.c_int, c_int_p, vp]),
    "spectrogramObj_mfcc": (None, [vp, vp, C.c_int, vp]),
    "spectrogramObj_deconv": (None, [vp, vp, vp, vp]),
    "spectrogramObj_bfcc": (None, [vp, vp, C.c_int, vp]),
    "spectrogramObj_gtcc": (None, [vp, vp, C.c_int, vp]),
    "spectrogramObj_lfcc": (None, [vp, vp, C.c_int, vp]),
    "spectrogramObj_free": (None, [vp]),
}

# additive entry points of libaudioflux_b200.so (include/afb200_ext.h)
EXTENSION_API = {
    "afb200_version": (C.c_int, []),
    "afb200_deviceCount": (C.c_int, []),
    "afb200_setDevice": (C.c_int, [C.c_int]),
    "afb200_getDevice": (C.c_int, []),
    "afb200_lastError": (C.c_char_p, []),
    "afb200_kernelLaunchCount": (C.c_longlong, []),
    "afb200_deviceSynchronize": (C.c_int, []),
    "stftObj_stftBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp]),
    "stftObj_istftBatch": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp]),
    "bftObj_bftBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp]),
    "bftObj_mfccBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp]),
    "bftObj_getFilterBankArr": (C.c_int, [vp, vp]),
    "bftObj_mfccPlanMode": (C.c_int, [vp]),
    "bftObj_mfccBatchScatter": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, P(vp), vp]),
    "afb200_peerAlloc": (C.c_int, [P(vp), C.c_size_t]),
    "afb200_peerFree": (C.c_int, [vp]),
    "afb200_ipcGetHandle": (C.c_int, [vp, vp]),
    "afb200_ipcOpenHandle": (C.c_int, [vp, P(vp)]),
    "afb200_ipcCloseHandle": (C.c_int, [vp]),
    "xxccObj_xxccBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp]),
    "cqtObj_cqtBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp]),
    "cqtObj_getKernelBank": (C.c_int, [vp, vp, vp]),
    "cqtObj_octavePlan": (C.c_int, [vp, vp, vp, vp, vp, vp, vp]),
    "cqtObj_chromaBatch": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp]),
    "cqtObj_cqccBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp]),
    "cqtObj_cqhcBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, C.c_int, vp]),
    "cqtObj_deconvBatch": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_int, vp]),
    "xxccObj_xxccStandardBatch": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                            vp, vp, vp, C.c_int, vp]),
    "spectrogramObj_spectrogramBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp]),
    "spectrogramObj_mfccBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int, vp]),
    "spectrogramObj_deconvBatch": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_int, vp]),
    "cwtObj_cwtBatch": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_int, vp]),
    "cwtObj_cwtDetBatch": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_int, vp]),
    "cwtObj_getFilterBankArr": (C.c_int, [vp, vp]),
    "pwtObj_pwtBatch": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_int, vp]),
    "pwtObj_pwtDetBatch": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_int, vp]),
    "pwtObj_getFilterBankArr": (C.c_int, [vp, vp]),
    "wsstObj_wsstDevice": (C.c_int, [vp, vp, vp, vp, vp, vp, vp]),
    "reassignObj_reassignBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, C.c_int, vp]),
    "synsqObj_synsqDevice": (C.c_int, [vp, vp, C.c_int, vp, vp, vp, vp, vp]),
    "afb200_window": (C.c_int, [C.c_int, C.c_int, vp]),
    "afb200_auditoryFilterBank": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                            C.c_float, C.c_float, C.c_int, vp, vp, vp]),
    "afb200_decimatorTaps": (C.c_int, [vp, vp]),
    "afb200_mfccBankPlan2": (C.c_int, [vp, C.c_int, vp, vp, vp, vp, vp, vp, vp]),
    "afb200_mfccCarve2": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp]),
    "afb200_chromaCqtFilterBank": (C.c_int, [C.c_int, C.c_int, C.c_int, C.c_float, vp]),
}

# spectral descriptors (src/feature/spectral_algorithm.h:16-81, include/afb200_spectral.h) and the additive batched
# entry point (include/afb200_ext.h)
_SPEC1 = (None, [vp, vp, vp])                       # (obj, mDataArr, dataArr)
_SPEC_PH = (None, [vp, vp, vp, vp])                 # (obj, mSpecArr, mPhaseArr, dataArr)
SPECTRAL_API = {
    "spectralObj_new": (C.c_int, [P(vp), C.c_int, vp]),
    "spectralObj_setEdge": (None, [vp, C.c_int, C.c_int]),
    "spectralObj_setEdgeArr": (None, [vp, vp, C.c_int]),
    "spectralObj_setTimeLength": (None, [vp, C.c_int]),
    "spectralObj_flatness": _SPEC1,
    "spectralObj_flux": (None, [vp, vp, C.c_int, C.c_float, C.c_int, c_int_p, c_int_p, vp]),
    "spectralObj_rolloff": (None, [vp, vp, C.c_float, vp]),
    "spectralObj_centroid": _SPEC1,
    "spectralObj_spread": _SPEC1,
    "spectralObj_skewness": _SPEC1,
    "spectralObj_kurtosis": _SPEC1,
    "spectralObj_entropy": (None, [vp, vp, C.c_int, vp]),
    "spectralObj_crest": _SPEC1,
    "spectralObj_slope": _SPEC1,
    "spectralObj_decrease": _SPEC1,
    "spectralObj_bandWidth": (None, [vp, vp, C.c_float, vp]),
    "spectralObj_rms": _SPEC1,
    "spectralObj_energy": (None, [vp, vp, C.c_int, C.c_float, vp]),
    "spectralObj_hfc": _SPEC1,
    "spectralObj_sd": (None, [vp, vp, C.c_int, C.c_int, vp]),
    "spectralObj_sf": (None, [vp, vp, C.c_int, C.c_int, vp]),
    "spectralObj_mkl": (None, [vp, vp, C.c_int, vp]),
    "spectralObj_pd": _SPEC_PH,
    "spectralObj_wpd": _SPEC_PH,
    "spectralObj_nwpd": _SPEC_PH,
    "spectralObj_cd": _SPEC_PH,
    "spectralObj_rcd": _SPEC_PH,
    "spectralObj_broadband": (None, [vp, vp, C.c_float, vp]),
    "spectralObj_novelty": (None, [vp, vp, C.c_int, C.c_float, c_int_p, c_int_p, vp]),
    "spectralObj_eef": (None, [vp, vp, C.c_int, vp]),
    "spectralObj_eer": (None, [vp, vp, C.c_int, C.c_float, vp]),
    "spectralObj_max": _SPEC_PH,
    "spectralObj_mean": _SPEC_PH,
    "spectralObj_var": _SPEC_PH,
    "spectralObj_free": (None, [vp]),
    "spectralObj_spectralBatch": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp]),
}

# non-stationary Gabor transform (src/nsgt_algorithm.h:34-57, include/afb200_nsgt.h) and the additive batched entry point
# (include/afb200_ext.h)
NSGT_API = {
    "nsgtObj_new": (C.c_int, [P(vp), C.c_int, C.c_int, c_int_p, c_float_p, c_float_p, c_int_p, c_int_p,
                              c_int_p, c_int_p, c_int_p, c_int_p]),
    "nsgtObj_getMaxTimeLength": (C.c_int, [vp]),
    "nsgtObj_getTotalTimeLength": (C.c_int, [vp]),
    "nsgtObj_getTimeLengthArr": (vp, [vp]),
    "nsgtObj_getFreBandArr": (vp, [vp]),
    "nsgtObj_getBinBandArr": (vp, [vp]),
    "nsgtObj_setMinLength": (None, [vp, C.c_int]),
    "nsgtObj_nsgt": (None, [vp, vp, vp, vp]),
    "nsgtObj_getCellData": (None, [vp, P(vp), P(vp)]),
    "nsgtObj_free": (None, [vp]),
    "nsgtObj_nsgtBatch": (C.c_int, [vp, vp, C.c_int, vp, vp, vp, vp, C.c_int, vp]),
}

# Stockwell transforms (src/st_algorithm.h:17-24, src/fst_algorithm.h:16-20, include/afb200_st.h) and the additive
# entry points (include/afb200_ext.h)
ST_API = {
    "stObj_new": (C.c_int, [P(vp), C.c_int, C.c_int, C.c_int, c_float_p, c_float_p]),
    "stObj_useBinArr": (None, [vp, vp, C.c_int]),
    "stObj_setValue": (None, [vp, C.c_float, C.c_float]),
    "stObj_st": (None, [vp, vp, vp, vp]),
    "stObj_free": (None, [vp]),
    "fstObj_new": (C.c_int, [P(vp), C.c_int]),
    "fstObj_fst": (None, [vp, vp, C.c_int, C.c_int, vp, vp]),
    "fstObj_free": (None, [vp]),
    "stObj_stBatch": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_int, vp]),
    "stObj_getBinLength": (C.c_int, [vp]),
    "fstObj_fstBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int, vp]),
}

# cepstrogram (include/cepstrogram_algorithm.h:21-39, include/afb200_cepstrogram.h) and the additive entry points
# (include/afb200_ext.h)
CEPSTROGRAM_API = {
    "cepstrogramObj_new": (C.c_int, [P(vp), C.c_int, c_int_p, c_int_p]),
    "cepstrogramObj_calTimeLength": (C.c_int, [vp, C.c_int]),
    "cepstrogramObj_cepstrogram": (None, [vp, C.c_int, vp, C.c_int, vp, vp, vp]),
    "cepstrogramObj_cepstrogram2": (None, [vp, C.c_int, vp, vp, C.c_int, vp, vp, vp]),
    "cepstrogramObj_enableDebug": (None, [vp, C.c_int]),
    "cepstrogramObj_free": (None, [vp]),
    "cepstrogramObj_cepstrogramBatch": (C.c_int, [vp, C.c_int, vp, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp]),
    "cepstrogramObj_cepstrogram2Batch": (C.c_int, [vp, C.c_int, vp, vp, C.c_int, C.c_int, vp, vp, vp, C.c_int, vp]),
}

# resampler (src/dsp/resample_algorithm.h, include/afb200_resample.h) and the additive batched entry point
# (include/afb200_ext.h)
RESAMPLE_API = {
    "resampleObj_new": (C.c_int, [P(vp), c_int_p, c_int_p, c_int_p]),
    "resampleObj_newWithWindow": (C.c_int, [P(vp), c_int_p, c_int_p, c_int_p, c_float_p, c_float_p, c_int_p, c_int_p]),
    "resampleObj_calDataLength": (C.c_int, [vp, C.c_int]),
    "resampleObj_setSamplate": (None, [vp, C.c_int, C.c_int]),
    "resampleObj_setSamplateRatio": (None, [vp, C.c_float]),
    "resampleObj_enableContinue": (None, [vp, C.c_int]),
    "resampleObj_resample": (C.c_int, [vp, vp, C.c_int, vp]),
    "resampleObj_free": (None, [vp]),
    "resampleObj_debug": (None, [vp]),
    "resampleObj_resampleBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, C.c_int, vp]),
}

# harmonic-percussive separation (include/mir/hpss_algorithm.h, include/afb200_hpss.h) and the additive batched entry
# point (include/afb200_ext.h)
HPSS_API = {
    "hpssObj_new": (C.c_int, [P(vp), C.c_int, c_int_p, c_int_p, c_int_p, c_int_p]),
    "hpssObj_calDataLength": (C.c_int, [vp, C.c_int]),
    "hpssObj_hpss": (None, [vp, vp, C.c_int, vp, vp]),
    "hpssObj_free": (None, [vp]),
    "hpssObj_debug": (None, [vp]),
    "hpssObj_hpssBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, vp, C.c_int, vp]),
}

# onset detection (include/mir/onset_algorithm.h, include/afb200_onset.h) and the additive batched entry point
# (include/afb200_ext.h)
ONSET_API = {
    "onsetObj_new": (C.c_int, [P(vp), C.c_int, C.c_int, C.c_int, c_int_p, c_int_p, c_int_p]),
    "onsetObj_onset": (C.c_int, [vp, vp, vp, vp, vp, C.c_int, vp, vp]),
    "onsetObj_free": (None, [vp]),
    "onsetObj_debug": (None, [vp]),
    "onsetObj_onsetBatch": (C.c_int, [vp, vp, vp, C.c_int, vp, vp, C.c_int, vp, vp, vp, C.c_int, vp]),
}

# harmonic ratio (include/mir/harmonicRatio_algorithm.h, include/afb200_harmonic_ratio.h) and the additive batched entry
# point (include/afb200_ext.h)
HARMONIC_RATIO_API = {
    "harmonicRatioObj_new": (C.c_int, [P(vp), c_int_p, c_float_p, c_int_p, c_int_p, c_int_p]),
    "harmonicRatioObj_calTimeLength": (C.c_int, [vp, C.c_int]),
    "harmonicRatioObj_harmonicRatio": (None, [vp, vp, C.c_int, vp]),
    "harmonicRatioObj_free": (None, [vp]),
    "harmonicRatioObj_harmonicRatioBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, C.c_int, vp]),
}

# pitch by the pitch estimation filter (include/mir/_pitch_pef.h, include/afb200_pitch_pef.h) and the additive batched
# entry point (include/afb200_ext.h)
PITCH_PEF_API = {
    "pitchPEFObj_new": (C.c_int, [P(vp), c_int_p, c_float_p, c_float_p, c_float_p, c_int_p, c_int_p, c_int_p, c_float_p,
                                  c_float_p, c_float_p, c_int_p]),
    "pitchPEFObj_calTimeLength": (C.c_int, [vp, C.c_int]),
    "pitchPEFObj_setFilterParams": (None, [vp, C.c_float, C.c_float, C.c_float]),
    "pitchPEFObj_pitch": (None, [vp, vp, C.c_int, vp]),
    "pitchPEFObj_enableDebug": (None, [vp, C.c_int]),
    "pitchPEFObj_free": (None, [vp]),
    "pitchPEFObj_pitchBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, C.c_int, vp]),
}

# pitch by YIN (include/mir/_pitch_yin.h, include/afb200_pitch_yin.h) and the additive batched entry point
# (include/afb200_ext.h)
PITCH_YIN_API = {
    "pitchYINObj_new": (C.c_int, [P(vp), c_int_p, c_float_p, c_float_p, c_int_p, c_int_p, c_int_p, c_int_p]),
    "pitchYINObj_setThresh": (None, [vp, C.c_float]),
    "pitchYINObj_calTimeLength": (C.c_int, [vp, C.c_int]),
    "pitchYINObj_pitch": (None, [vp, vp, C.c_int, vp, vp, vp]),
    "pitchYINObj_getTroughData": (C.c_int, [vp, P(P(C.c_float)), P(P(C.c_float)), P(P(C.c_int))]),
    "pitchYINObj_enableDebug": (None, [vp, C.c_int]),
    "pitchYINObj_free": (None, [vp]),
    "pitchYINObj_pitchBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, C.c_int, vp]),
}

# pitch by the normalised correlation and by the cepstrum (include/mir/_pitch_{ncf,cep}.h,
# include/afb200_pitch_{ncf,cep}.h) and the additive batched entry points (include/afb200_ext.h)
PITCH_NCF_API = {
    "pitchNCFObj_new": (C.c_int, [P(vp), c_int_p, c_float_p, c_float_p, c_int_p, c_int_p, c_int_p, c_int_p]),
    "pitchNCFObj_calTimeLength": (C.c_int, [vp, C.c_int]),
    "pitchNCFObj_pitch": (None, [vp, vp, C.c_int, vp]),
    "pitchNCFObj_enableDebug": (None, [vp, C.c_int]),
    "pitchNCFObj_free": (None, [vp]),
    "pitchNCFObj_pitchBatch": (C.c_int, [vp, vp, C.c_int, C.c_int, vp, C.c_int, vp]),
}
PITCH_CEP_API = {k.replace("NCF", "CEP"): v for k, v in PITCH_NCF_API.items()}

# setup-time builders exported (non-static) by the reference only; used by tests to
# compare constant tables (src/dsp/flux_window.h, src/filterbank/*.h)
REFERENCE_BUILDERS = {
    "window_calFFTWindow": (vp, [C.c_int, C.c_int]),
    "auditory_filterBank": (None, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                   C.c_float, C.c_float, C.c_int, vp, vp, vp]),
    "chroma_cqtFilterBank": (None, [C.c_int, C.c_int, C.c_int, c_float_p, vp]),
    # src/filterbank/nsgt_filterBank.h (nsgt_filterBank.c:48-239)
    "nsgt_filterBank": (None, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                               C.c_float, C.c_float, C.c_int, P(vp), vp, vp, vp, vp, c_int_p, c_int_p]),
}


WAVELET_API = {
    "dwtObj_new": (C.c_int, [P(vp), C.c_int, C.c_int, c_int_p, c_int_p, c_int_p]),
    "dwtObj_dwt": (None, [vp, vp, vp, vp]),
    "dwtObj_free": (None, [vp]),
    "wptObj_new": (C.c_int, [P(vp), C.c_int, C.c_int, c_int_p, c_int_p, c_int_p]),
    "wptObj_wpt": (None, [vp, vp, vp, vp]),
    "wptObj_free": (None, [vp]),
    "swtObj_new": (C.c_int, [P(vp), C.c_int, C.c_int, c_int_p, c_int_p, c_int_p]),
    "swtObj_swt": (None, [vp, vp, vp, vp]),
    "swtObj_free": (None, [vp]),
    "dwtObj_dwtBatch": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_int, vp]),
    "wptObj_wptBatch": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_int, vp]),
    "swtObj_swtBatch": (C.c_int, [vp, vp, C.c_int, vp, vp, C.c_int, vp]),
}


# non-negative matrix factorisation (include/classic/nmf.h, include/afb200_nmf.h) and the additive batched entry point
# (include/afb200_ext.h)
NMF_API = {
    "nmf": (None, [vp, C.c_int, C.c_int, C.c_int, vp, vp, c_int_p, c_int_p, c_float_p, c_int_p]),
    "nmfBatch": (C.c_int, [vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp, c_int_p, c_int_p, c_float_p, c_int_p, vp,
                           C.c_int, vp]),
}


# cross-correlation and the chirp z-transform (include/dsp/xcorr_algorithm.h, czt_algorithm.h; include/afb200_xcorr.h,
# afb200_czt.h) and the additive batched entry points (include/afb200_ext.h)
DSP_API = {
    "xcorrObj_new": (C.c_int, [P(vp)]),
    "xcorrObj_xcorr": (C.c_int, [vp, vp, vp, C.c_int, c_int_p, vp, c_float_p]),
    "xcorrObj_free": (None, [vp]),
    "xcorrObj_xcorrBatch": (C.c_int, [vp, vp, vp, C.c_int, C.c_int, c_int_p, vp, vp, vp, C.c_int, vp]),
    "cztObj_new": (C.c_int, [P(vp), C.c_int]),
    "cztObj_czt": (None, [vp, vp, vp, C.c_float, C.c_float, vp, vp]),
    "cztObj_free": (None, [vp]),
    "cztObj_cztBatch": (C.c_int, [vp, vp, vp, C.c_int, C.c_float, C.c_float, vp, vp, C.c_int, vp]),
}


def bind(lib: C.CDLL, tables=(REFERENCE_API, EXTENSION_API, SPECTRAL_API, NSGT_API, ST_API, CEPSTROGRAM_API,
                              RESAMPLE_API, HPSS_API, ONSET_API, HARMONIC_RATIO_API, PITCH_PEF_API, PITCH_YIN_API,
                              PITCH_NCF_API, PITCH_CEP_API, WAVELET_API, NMF_API, DSP_API, REFERENCE_BUILDERS)) -> dict:
    """Apply argtypes/restype for every symbol the library actually exports.
    Returns {name: bool present}."""
    present = {}
    for table in tables:
        for name, (res, args) in table.items():
            try:
                fn = getattr(lib, name)
            except AttributeError:
                present[name] = False
                continue
            fn.restype = res
            fn.argtypes = args
            present[name] = True
    return present


def opt_int(v):
    return None if v is None else C.byref(C.c_int(int(v)))


def opt_float(v):
    return None if v is None else C.byref(C.c_float(float(v)))
