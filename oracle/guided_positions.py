"""ORACLE — test infrastructure only (see oracle/guided_positions_oracle.cpp).

Position-only guided matching on double positions: ``GuidedPositionsOracle().guided_match_positions`` ->
oracle/libguided_positions.so, the guidedMatching.hpp:37-70 loop and IndMatch::getDeduplicated.  It reads no descriptor, so there is one
build.  The IndMatchDecorator step that GeometricFilterMatrix_H_AC applies next is ``oracle.best().decorator_dedup`` (the compiled
reference's own when it is built).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "libguided_positions.so")


def available() -> bool:
    return os.path.exists(LIB)


def build() -> None:
    """Compile the oracle; with an AliceVision tree (oracle.reference_src()) and the CUDA library built, also the C++ test of the
    homography-filter adaptor."""
    mk = ["make", "-C", _HERE, "-f", "homography_filter.mk"]
    subprocess.run(mk + ["all"], check=True, stdout=subprocess.DEVNULL)
    src = oracle.reference_src()
    if src is not None and os.path.exists(os.path.join(os.path.dirname(_HERE), "alicevision_b200", "libb200match.so")):
        subprocess.run(mk + ["adaptor", f"REF={src}"], check=True, stdout=subprocess.DEVNULL)


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class GuidedPositionsOracle:
    def __init__(self):
        if not available():
            raise FileNotFoundError(f"{LIB} missing: run oracle.guided_positions.build()")
        self.lib = C.CDLL(LIB)
        self.lib.gf_guided_match_positions.restype = C.c_int

    def guided_match_positions(self, xy_l, xy_r, M, errorTh: float, model: int = 1) -> np.ndarray:
        """guidedMatching(model, xLeft, xRight, errorTh) on double positions (model 1 = homography, 0 = fundamental matrix), sorted and
        de-duplicated like the reference.  Returns matches[MATCH_DTYPE] (ratio = dist = 0)."""
        xy_l = np.ascontiguousarray(xy_l, np.float64).reshape(-1, 2); xy_r = np.ascontiguousarray(xy_r, np.float64).reshape(-1, 2)
        Mm = np.ascontiguousarray(M, np.float64).reshape(9)
        out = np.zeros((max(xy_l.shape[0], 1), 2), np.uint32)
        n = self.lib.gf_guided_match_positions(C.c_int(model), _p(xy_l), C.c_int(xy_l.shape[0]), _p(xy_r), C.c_int(xy_r.shape[0]), _p(Mm),
                                               C.c_double(errorTh), _p(out))
        m = np.zeros(n, oracle.MATCH_DTYPE)
        m["i"] = out[:n, 0]; m["j"] = out[:n, 1]
        return m
