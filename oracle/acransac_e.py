"""ORACLE — test infrastructure only (see oracle/acransac_e_oracle.cpp).

A-contrario RANSAC essential-matrix estimation of one pair of pinhole cameras (GeometricFilterMatrix_E_AC::geometricEstimation):

* ``AcransacEOracle("ref")``  -> oracle/_ref/libref_acransac_e.so: the reference's ACRANSAC loop, sampling and NFA tables compiled
  verbatim from an AliceVision source tree, around the restated E kernel.
* ``AcransacEOracle("port")`` -> oracle/libport_acransac_e.so: all of it restated.

``reference_output()`` stores the "ref" outputs in tests/golden/reference_acransac_e.npz and replays them where the reference is
not built, like ``oracle.acransac_s.reference_output`` does for the spherical model.
"""
from __future__ import annotations

import ctypes as C
import functools
import os

import numpy as np

import oracle
from oracle import _p

_HERE = os.path.dirname(os.path.abspath(__file__))
STORED = os.path.join(os.path.dirname(_HERE), "tests", "golden", "reference_acransac_e.npz")
TRACE_CAP = 4096
FIELDS = ("valid", "inliers", "E", "error_max", "min_nfa", "iterations", "trace", "mt_state_out")   # stored fields of estimate()


available = functools.partial(oracle.lib_available, "acransac_e")


class AcransacEOracle:
    def __init__(self, kind: str = "port"):
        assert kind in ("ref", "port")
        self.kind = kind
        self.lib = oracle.load_lib("acransac_e", kind)
        self.lib.acre_estimate.restype = C.c_long
        self.lib.acre_fit5.restype = C.c_int
        self.lib.acre_eigen.restype = C.c_int

    def mt_seed(self, seed: int) -> np.ndarray:
        st = np.zeros(625, np.uint32)
        self.lib.acre_mt_seed(C.c_uint32(seed), _p(st))
        return st

    def fit5(self, corr) -> list:
        """The 5-point solver on 5 normalised correspondences (5 x (xI, yI, xJ, yJ)): its models (0..10 matrices, x_J^T E x_I = 0)."""
        c = np.ascontiguousarray(corr, np.float64).reshape(5, 4)
        E = np.zeros(90, np.float64)
        nb = self.lib.acre_fit5(_p(c), _p(E))
        return [E[9 * m:9 * m + 9].reshape(3, 3).copy() for m in range(nb)]

    def action(self, corr) -> np.ndarray:
        """The 10 x 10 action matrix the 5-point solver builds from 5 normalised correspondences (5 x (xI, yI, xJ, yJ))."""
        c = np.ascontiguousarray(corr, np.float64).reshape(5, 4)
        A = np.zeros(100, np.float64)
        self.lib.acre_action(_p(c), _p(A))
        return A.reshape(10, 10)

    def eigen(self, A):
        """The solver's eigen-decomposition of a 10 x 10 matrix: (real parts, imaginary parts) in Schur order, or None where it gives
        no model (no convergence)."""
        a = np.ascontiguousarray(A, np.float64).reshape(10, 10)
        re = np.zeros(10); im = np.zeros(10)
        return (re, im) if self.lib.acre_eigen(_p(a), _p(re), _p(im)) else None

    def estimate(self, corr, K, wh_j, state, max_iteration: int = 50000, precision: float = np.inf) -> dict:
        """One pair: corr n x 4 pixels (xI, yI, xJ, yJ), K = (K_I, K_J) 3 x 3 each, wh_j = view J's (width, height), state = 625
        generator words (left unchanged; the state after the estimation is "mt_state_out").  precision is ACRANSAC's argument."""
        c = np.ascontiguousarray(corr, np.float64).reshape(-1, 4)
        n = c.shape[0]
        Km = np.ascontiguousarray(np.concatenate([np.asarray(k, np.float64).reshape(9) for k in K]))
        st = np.ascontiguousarray(state, np.uint32).reshape(625)
        sto = np.zeros(625, np.uint32)
        valid = C.c_int(); ninl = C.c_int(); ntr = C.c_int(); em = C.c_double(); nfa = C.c_double()
        inl = np.zeros(max(n, 1), np.uint32); E = np.zeros(9, np.float64); tr = np.zeros(TRACE_CAP, np.int32); trn = np.zeros(TRACE_CAP)
        it = self.lib.acre_estimate(C.c_int(n), _p(c), _p(Km), C.c_int(int(wh_j[0])), C.c_int(int(wh_j[1])), _p(st), C.c_long(max_iteration),
                                    C.c_double(precision), C.byref(valid), C.byref(ninl), _p(inl), _p(E), C.byref(em), C.byref(nfa), _p(tr),
                                    _p(trn), C.c_int(TRACE_CAP), C.byref(ntr), _p(sto))
        return {"valid": np.array(bool(valid.value)), "inliers": inl[:ninl.value].copy(), "E": E.reshape(3, 3),
                "error_max": np.array(em.value), "min_nfa": np.array(nfa.value), "iterations": np.array(int(it)),
                "trace": tr[:min(ntr.value, TRACE_CAP)].copy(), "n_trace": int(ntr.value), "trace_nfa": trn[:min(ntr.value, TRACE_CAP)].copy(),
                "mt_state_out": sto}


reference_output = functools.partial(oracle.reference_output, path=STORED)
