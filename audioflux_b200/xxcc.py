"""XXCC cepstral coefficients: rectify (log10 | cube root) -> DCT-II ortho -> first cc_num
(reference binding: python/audioflux/feature/xxcc.py:14-136; C: src/feature/xxcc_algorithm.c)."""
from __future__ import annotations

import numpy as np

from .base import Base, Batch, as_f32, np_ptr, per_clip, swap_last2
from .capi import opt_int
from .types import CepstralRectifyType, CepstralEnergyType, enum_value


class XXCC(Base):
    def __init__(self, num, _lib=None):
        super().__init__(_lib)
        if num < 2:
            raise ValueError("num must be >= 2")
        self.num = num
        self.time_length = 0
        self._new("xxccObj_new", "xxccObj_free", num)

    def set_time_length(self, time_length):
        self._lib.xxccObj_setTimeLength(self._obj, int(time_length))
        self.time_length = int(time_length)

    def xxcc_planes(self, m_tn, cc_num=13, rectify_type=CepstralRectifyType.LOG):
        """Raw C layout: in [T, num] -> out [T, cc_num]."""
        m = as_f32(m_tn)
        if m.shape[0] != self.time_length:
            self.set_time_length(m.shape[0])
        out = np.zeros((m.shape[0], cc_num), np.float32)
        self._lib.xxccObj_xxcc(self._obj, np_ptr(m), cc_num, opt_int(enum_value(rectify_type)), np_ptr(out))
        return out

    def xxcc(self, m_data_arr, cc_num=13, rectify_type=CepstralRectifyType.LOG):
        """m_data_arr [..., num, T] -> [..., cc_num, T] as feature/xxcc.py:90-136."""
        m = np.asarray(m_data_arr)
        if np.iscomplexobj(m):
            m = np.abs(m)
        m = as_f32(m)
        if cc_num > self.num:
            raise ValueError("cc_num must be <= num")
        out, = per_clip(lambda clip: (self.xxcc_planes(clip, cc_num, rectify_type),), swap_last2(m), clip_ndim=2)
        return swap_last2(out)

    def xxcc_batch(self, m_tn, cc_num=13, rectify_type=CepstralRectifyType.LOG):
        """Additive: m_tn [..., T, num] time-major (numpy host | torch cuda) -> [..., T, cc_num]."""
        b = Batch(m_tn)
        out = b.alloc(b.rows, cc_num)
        self._call("xxccObj_xxccBatch", b, b.x, b.rows, cc_num, enum_value(rectify_type), out)
        return b.shaped(out)

    def xxcc_standard_planes(self, m_tn, energy, cc_num=13, delta_window_length=9,
                             energy_type=CepstralEnergyType.REPLACE, rectify_type=CepstralRectifyType.LOG):
        """Raw C layout: in [T, num], energy [T] -> (coe, delta, delta2) each [T, W], W = cc_num (+1 for APPEND)
        (xxccObj_xxccStandard, src/feature/xxcc_algorithm.c:168-296)."""
        m = as_f32(m_tn)
        e = as_f32(energy)
        if m.shape[0] != self.time_length:
            self.set_time_length(m.shape[0])
        w = cc_num + (1 if enum_value(energy_type) == 1 else 0)
        outs = [np.zeros((m.shape[0], w), np.float32) for _ in range(3)]
        self._lib.xxccObj_xxccStandard(self._obj, np_ptr(m), cc_num, np_ptr(e), opt_int(delta_window_length),
                                       opt_int(enum_value(energy_type)), opt_int(enum_value(rectify_type)),
                                       np_ptr(outs[0]), np_ptr(outs[1]), np_ptr(outs[2]))
        return tuple(outs)

    def xxcc_standard(self, m_data_arr, energy_arr, cc_num=13, delta_window_length=9,
                      energy_type=CepstralEnergyType.REPLACE, rectify_type=CepstralRectifyType.LOG):
        """m_data_arr [..., num, T], energy_arr [..., T] -> three arrays [..., W, T] as feature/xxcc.py:138-240."""
        outs = per_clip(lambda m, e: self.xxcc_standard_planes(m, e, cc_num, delta_window_length, energy_type, rectify_type),
                        swap_last2(as_f32(m_data_arr)), clip_ndim=2, y=as_f32(energy_arr))
        return tuple(map(swap_last2, outs))

    def xxcc_standard_batch(self, m_tn, energy, cc_num=13, delta_window_length=9,
                            energy_type=CepstralEnergyType.REPLACE, rectify_type=CepstralRectifyType.LOG):
        """Additive: m_tn [..., T, num], energy [..., T] (numpy host | torch cuda) -> three [..., T, W]."""
        b = Batch(m_tn)
        e = b.second(energy, "energy (one value per frame)", (b.rows,))
        w = cc_num + (1 if enum_value(energy_type) == 1 else 0)
        outs = [b.alloc(b.rows, w) for _ in range(3)]
        self._call("xxccObj_xxccStandardBatch", b, b.x, e, b.rows, cc_num, int(delta_window_length),
                   enum_value(energy_type), enum_value(rectify_type), *outs)
        return tuple(map(b.shaped, outs))