"""ORACLE — test infrastructure only (see oracle/acransac_oracle.cpp).

A-contrario RANSAC fundamental-matrix estimation of one pair (GeometricFilterMatrix_F_AC::geometricEstimation_Mat_ACRANSAC):

* ``AcransacOracle("ref")``  -> oracle/_ref/libref_acransac.so: the reference's ACRANSAC loop, sampling, NFA tables and cubic
  solver compiled verbatim from an AliceVision source tree, around the restated F kernel.
* ``AcransacOracle("port")`` -> oracle/libport_acransac.so: all of it restated.

``reference_output()`` stores the "ref" outputs in tests/golden/reference_acransac.npz and replays them where the reference is
not built, like ``oracle.guided_fast.reference_output`` does.
"""
from __future__ import annotations

import ctypes as C
import functools
import os

import numpy as np

import oracle
from oracle import _p

_HERE = os.path.dirname(os.path.abspath(__file__))
STORED = os.path.join(os.path.dirname(_HERE), "tests", "golden", "reference_acransac.npz")
TRACE_CAP = 4096
FIELDS = ("valid", "inliers", "F", "error_max", "min_nfa", "iterations", "trace")   # the stored fields of AcransacOracle.estimate


available = functools.partial(oracle.lib_available, "acransac")
current = functools.partial(oracle.lib_current, "acransac")


class AcransacOracle:
    def __init__(self, kind: str = "port"):
        assert kind in ("ref", "port")
        self.kind = kind
        self.lib = oracle.load_lib("acransac", kind)
        self.lib.acr_estimate.restype = C.c_long
        self.lib.acr_fit7.restype = C.c_int

    def mt_seed(self, seed: int) -> np.ndarray:
        st = np.zeros(625, np.uint32)
        self.lib.acr_mt_seed(C.c_uint32(seed), _p(st))
        return st

    def rand_sample(self, state: np.ndarray, rng: int, draws: int, states: bool = False):
        """`draws` consecutive randSample(g, 0, rng, 7): (draws x 7 samples in their order, draws x 625 states after each or None)."""
        st = np.ascontiguousarray(state, np.uint32)
        out = np.zeros((draws, 7), np.uint32)
        sts = np.zeros((draws, 625), np.uint32) if states else None
        self.lib.acr_rand_sample(_p(st), C.c_int(rng), C.c_int(draws), _p(out), _p(sts) if states else None)
        return out, sts

    def logc(self, n: int):
        a = np.zeros(n + 1, np.float32); b = np.zeros(n + 1, np.float32)
        self.lib.acr_logc(C.c_int(n), _p(a), _p(b))
        return a, b

    def fit7(self, corr: np.ndarray) -> np.ndarray:
        c = np.ascontiguousarray(corr, np.float64).reshape(7, 4)
        F = np.zeros((3, 9), np.float64)
        nb = self.lib.acr_fit7(_p(c), _p(F))
        return F[:nb].reshape(-1, 3, 3)

    # -- the F kernel's primitives (the tests of test_acransac_exact.py check them against mpmath)
    def solve_cubic(self, P) -> np.ndarray:
        """SolveCubicPolynomial(P, x), P in ascending powers: the roots it returns (0, 1 or 3)."""
        p = np.ascontiguousarray(P, np.float64).reshape(4)
        x = np.zeros(3, np.float64)
        f = self.lib.acr_solve_cubic
        f.restype = C.c_int
        nb = f(_p(p), _p(x))
        return x[:nb].copy()

    def nullspace7(self, A) -> np.ndarray:
        a = np.ascontiguousarray(A, np.float64).reshape(7, 9)
        N = np.zeros((2, 9), np.float64)
        self.lib.acr_nullspace7(_p(a), _p(N))
        return N

    def errors(self, F, corr) -> np.ndarray:
        """FundamentalEpipolarDistanceError of F on the correspondences as given (no normalisation)."""
        c = np.ascontiguousarray(corr, np.float64).reshape(-1, 4)
        f = np.ascontiguousarray(F, np.float64).reshape(9)
        e = np.zeros(c.shape[0])
        self.lib.acr_epipolar_error(_p(f), C.c_int(c.shape[0]), _p(c), _p(e))
        return e

    def precondition(self, w: int, h: int, x=(), y=()):
        """((s, tx, ty), x normalised, y normalised) of preconditionerFromImageSize(w, h)."""
        sxy = np.zeros(3)
        xs = np.array(x, np.float64).reshape(-1).copy(); ys = np.array(y, np.float64).reshape(-1).copy()
        assert xs.size == ys.size
        self.lib.acr_precondition(C.c_int(w), C.c_int(h), _p(sxy), C.c_int(xs.size), _p(xs), _p(ys))
        return sxy, xs, ys

    def unnormalize(self, wh, F) -> np.ndarray:
        f = np.ascontiguousarray(F, np.float64).reshape(9).copy()
        self.lib.acr_unnormalize(*(C.c_int(int(v)) for v in wh), _p(f))
        return f.reshape(3, 3)

    def logalpha0(self, wh) -> float:
        f = self.lib.acr_logalpha0
        f.restype = C.c_double
        return f(*(C.c_int(int(v)) for v in wh))

    def unnormalize_error(self, wh, v: float) -> float:
        f = self.lib.acr_unnormalize_error
        f.restype = C.c_double
        return f(*(C.c_int(int(x)) for x in wh), C.c_double(v))

    def estimate(self, corr, wh, state, max_iteration: int = 50000, precision: float = np.inf) -> dict:
        """One pair: corr n x 4 (xI, yI, xJ, yJ), wh = (wI, hI, wJ, hJ), state = 625 generator words."""
        c = np.ascontiguousarray(corr, np.float64).reshape(-1, 4)
        n = c.shape[0]
        st = np.ascontiguousarray(state, np.uint32)
        valid = C.c_int(); ninl = C.c_int(); ntr = C.c_int(); em = C.c_double(); nfa = C.c_double()
        inl = np.zeros(max(n, 1), np.uint32); F = np.zeros(9, np.float64); tr = np.zeros(TRACE_CAP, np.int32); trn = np.zeros(TRACE_CAP)
        it = self.lib.acr_estimate(C.c_int(n), _p(c), C.c_int(int(wh[0])), C.c_int(int(wh[1])), C.c_int(int(wh[2])), C.c_int(int(wh[3])),
                                   _p(st), C.c_long(max_iteration), C.c_double(precision), C.byref(valid), C.byref(ninl), _p(inl), _p(F),
                                   C.byref(em), C.byref(nfa), _p(tr), _p(trn), C.c_int(TRACE_CAP), C.byref(ntr))
        return {"valid": np.array(bool(valid.value)), "inliers": inl[:ninl.value].copy(), "F": F.reshape(3, 3),
                "error_max": np.array(em.value), "min_nfa": np.array(nfa.value), "iterations": np.array(int(it)),
                "trace": tr[:min(ntr.value, TRACE_CAP)].copy(), "n_trace": int(ntr.value), "trace_nfa": trn[:min(ntr.value, TRACE_CAP)].copy()}


def best(prefer_ref: bool = True) -> AcransacOracle:
    return AcransacOracle("ref" if prefer_ref and available("ref") else "port")


reference_output = functools.partial(oracle.reference_output, path=STORED)
