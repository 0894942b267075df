"""ORACLE — test infrastructure only (see oracle/guided_fast_oracle.cpp).

Guided matching on double (undistorted) positions:

* ``GuidedFastOracle("ref")``  -> oracle/_ref/libref_guided_fast.so: descriptor distances from the reference's own
  Regions::SquaredDescriptorDistance compiled from an AliceVision source tree; the geometry is restated.
* ``GuidedFastOracle("port")`` -> oracle/libport_guided_fast.so: the restated metrics.

``reference_output()`` stores the "ref" outputs in tests/golden/reference_guided_fast.npz and replays them where the
reference is not built, like ``oracle.reference_output`` does for the other comparisons.
"""
from __future__ import annotations

import ctypes as C
import functools
import os

import numpy as np

import oracle
from oracle import _p

_HERE = os.path.dirname(os.path.abspath(__file__))
STORED = os.path.join(os.path.dirname(_HERE), "tests", "golden", "reference_guided_fast.npz")


available = functools.partial(oracle.lib_available, "guided_fast")


def _dt(a: np.ndarray, binary: bool) -> int:
    if a.dtype == np.float32:
        return oracle.DT_F32
    return oracle.DT_BIN if binary else oracle.DT_U8


class GuidedFastOracle:
    def __init__(self, kind: str = "port"):
        assert kind in ("ref", "port")
        self.kind = kind
        self.lib = oracle.load_lib("guided_fast", kind)
        self.lib.gf_guided_fast.restype = C.c_int
        self.lib.gf_guided_match.restype = C.c_int

    def guided_fast(self, desc_l, xy_l, desc_r, xy_r, F, epipole2, widthR: int, heightR: int, errorTh: float, distRatio: float,
                    binary: bool = False) -> np.ndarray:
        """guidedMatchingFundamentalFast on double positions.  Returns matches[MATCH_DTYPE] in ascending i (ratio = dist = 0)."""
        desc_l = np.ascontiguousarray(desc_l); desc_r = np.ascontiguousarray(desc_r)
        xy_l = np.ascontiguousarray(xy_l, np.float64).reshape(-1, 2); xy_r = np.ascontiguousarray(xy_r, np.float64).reshape(-1, 2)
        Fm = np.ascontiguousarray(F, np.float64).reshape(9); e = np.ascontiguousarray(epipole2, np.float64).reshape(3)
        out = np.zeros((max(desc_l.shape[0], 1), 2), np.uint32)
        n = self.lib.gf_guided_fast(C.c_int(_dt(desc_l, binary)), _p(desc_l), _p(xy_l), C.c_int(desc_l.shape[0]), _p(desc_r), _p(xy_r),
                                    C.c_int(desc_r.shape[0]), _p(Fm), _p(e), C.c_int(widthR), C.c_int(heightR), C.c_double(errorTh),
                                    C.c_double(distRatio), _p(out))
        m = np.zeros(n, oracle.MATCH_DTYPE)
        m["i"] = out[:n, 0]; m["j"] = out[:n, 1]
        return m

    def guided_match(self, desc_l, xy_l, desc_r, xy_r, F, errorTh: float, distRatio: float, binary: bool = False, model: int = 0) -> np.ndarray:
        """guidedMatching (F or homography model) on double positions; sorted and de-duplicated like the reference."""
        desc_l = np.ascontiguousarray(desc_l); desc_r = np.ascontiguousarray(desc_r)
        xy_l = np.ascontiguousarray(xy_l, np.float64).reshape(-1, 2); xy_r = np.ascontiguousarray(xy_r, np.float64).reshape(-1, 2)
        Fm = np.ascontiguousarray(F, np.float64).reshape(9)
        out = np.zeros((max(desc_l.shape[0], 1), 2), np.uint32)
        n = self.lib.gf_guided_match(C.c_int(_dt(desc_l, binary)), C.c_int(model), _p(desc_l), _p(xy_l), C.c_int(desc_l.shape[0]), _p(desc_r),
                                     _p(xy_r), C.c_int(desc_r.shape[0]), _p(Fm), C.c_double(errorTh), C.c_double(distRatio), _p(out))
        m = np.zeros(n, oracle.MATCH_DTYPE)
        m["i"] = out[:n, 0]; m["j"] = out[:n, 1]
        return m


def best(prefer_ref: bool = True) -> GuidedFastOracle:
    """The compiled reference's distances if built, else the port."""
    return GuidedFastOracle("ref" if prefer_ref and available("ref") else "port")


reference_output = functools.partial(oracle.reference_output, path=STORED)
