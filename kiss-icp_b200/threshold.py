"""Adaptive / fixed threshold — python/kiss_icp/threshold.py:29-58 surface over kb_threshold_*."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as N
from .config import KISSConfig
from .mapping import check_value


def get_threshold_estimator(config: KISSConfig):
    if config.adaptive_threshold.fixed_threshold is not None:
        return FixedThreshold(config.adaptive_threshold.fixed_threshold)
    return AdaptiveThreshold(config)


class FixedThreshold:
    def __init__(self, fixed_threshold: float):
        self.fixed_threshold = fixed_threshold

    def get_threshold(self):
        return self.fixed_threshold

    def update_model_deviation(self, model_deviation):
        pass


class AdaptiveThreshold:
    def __init__(self, config: KISSConfig):
        self._h = N.vp()
        N.check(N.lib().kb_threshold_create(float(config.adaptive_threshold.initial_threshold),
                                            float(config.adaptive_threshold.min_motion_th),
                                            float(config.data.max_range), C.byref(self._h)))

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and N._lib is not None:
            N._lib.kb_threshold_destroy(h)
            self._h = None

    def get_threshold(self):
        s = N.dbl(0)
        N.check(N.lib().kb_threshold_compute(self._h, C.byref(s)))
        return s.value

    def update_model_deviation(self, model_deviation: np.ndarray):
        T = N.mat4_arg(model_deviation)
        N.check(N.lib().kb_threshold_update_model_deviation(self._h, N.ptr(T)))

    def get_state(self):
        """(model_sse, num_samples): AdaptiveThreshold::model_sse_ / num_samples_ (Threshold.hpp:44-46)"""
        s, n = N.dbl(0), N.i32(0)
        N.check(N.lib().kb_threshold_get_state(self._h, C.byref(s), C.byref(n)))
        return s.value, n.value

    def set_state(self, model_sse: float, num_samples: int):
        """ValueError for a non-finite or negative model_sse or num_samples < 1"""
        check_value(N.lib().kb_threshold_set_state(self._h, float(model_sse), int(num_samples)))
