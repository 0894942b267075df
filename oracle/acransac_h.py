"""ORACLE — test infrastructure only (see oracle/acransac_h_oracle.cpp).

A-contrario RANSAC homography estimation of one pair (GeometricFilterMatrix_H_AC::geometricEstimation):

* ``AcransacHOracle("ref")``  -> oracle/_ref/libref_acransac_h.so: the reference's ACRANSAC loop, sampling and NFA tables compiled
  verbatim from an AliceVision source tree, around the restated H kernel.
* ``AcransacHOracle("port")`` -> oracle/libport_acransac_h.so: all of it restated.

``reference_output()`` stores the "ref" outputs in tests/golden/reference_acransac_h.npz and replays them where the reference is
not built, like ``oracle.acransac.reference_output`` does for the fundamental matrix.
"""
from __future__ import annotations

import ctypes as C
import functools
import os

import numpy as np

import oracle
from oracle import _p

_HERE = os.path.dirname(os.path.abspath(__file__))
STORED = os.path.join(os.path.dirname(_HERE), "tests", "golden", "reference_acransac_h.npz")
TRACE_CAP = 4096
FIELDS = ("valid", "inliers", "H", "error_max", "min_nfa", "iterations", "trace", "mt_state_out")   # stored fields of estimate()


available = functools.partial(oracle.lib_available, "acransac_h")
current = functools.partial(oracle.lib_current, "acransac_h")


class AcransacHOracle:
    def __init__(self, kind: str = "port"):
        assert kind in ("ref", "port")
        self.kind = kind
        self.lib = oracle.load_lib("acransac_h", kind)
        self.lib.acr_estimate_h.restype = C.c_long
        self.lib.acr_fit4.restype = C.c_int

    def mt_seed(self, seed: int) -> np.ndarray:
        st = np.zeros(625, np.uint32)
        self.lib.acrh_mt_seed(C.c_uint32(seed), _p(st))
        return st

    def rand_sample(self, state: np.ndarray, k: int, rng: int, draws: int, states: bool = False):
        """`draws` consecutive randSample(g, 0, rng, k): (draws x k samples in their order, draws x 625 states after each or None)."""
        st = np.ascontiguousarray(state, np.uint32)
        out = np.zeros((draws, k), np.uint32)
        sts = np.zeros((draws, 625), np.uint32) if states else None
        self.lib.acr_rand_sample_k(_p(st), C.c_int(k), C.c_int(rng), C.c_int(draws), _p(out), _p(sts) if states else None)
        return out, sts

    def logc(self, k: int, n: int):
        a = np.zeros(n + 1, np.float32); b = np.zeros(n + 1, np.float32)
        self.lib.acr_logc_k(C.c_int(k), C.c_int(n), _p(a), _p(b))
        return a, b

    def fit4(self, corr: np.ndarray) -> np.ndarray:
        c = np.ascontiguousarray(corr, np.float64).reshape(4, 4)
        H = np.zeros(9, np.float64)
        assert self.lib.acr_fit4(_p(c), _p(H)) == 1
        return H.reshape(3, 3)

    def errors(self, H, corr) -> np.ndarray:
        c = np.ascontiguousarray(corr, np.float64).reshape(-1, 4)
        h = np.ascontiguousarray(H, np.float64).reshape(9)
        e = np.zeros(c.shape[0])
        self.lib.acr_homography_error(_p(h), C.c_int(c.shape[0]), _p(c), _p(e))
        return e

    # -- the H kernel's primitives (the tests of test_acransac_exact.py check them against mpmath)
    def nullspace8(self, A) -> np.ndarray:
        a = np.ascontiguousarray(A, np.float64).reshape(8, 9)
        N = np.zeros(9, np.float64)
        self.lib.acr_nullspace8(_p(a), _p(N))
        return N

    def inverse3(self, M) -> np.ndarray:
        m = np.ascontiguousarray(M, np.float64).reshape(9)
        R = np.zeros(9, np.float64)
        self.lib.acr_inverse3(_p(m), _p(R))
        return R.reshape(3, 3)

    def unnormalize(self, wh, H) -> np.ndarray:
        h = np.ascontiguousarray(H, np.float64).reshape(9).copy()
        self.lib.acr_unnormalize_h(*(C.c_int(int(v)) for v in wh), _p(h))
        return h.reshape(3, 3)

    def logalpha0(self, wh) -> float:
        f = self.lib.acr_logalpha0_h
        f.restype = C.c_double
        return f(*(C.c_int(int(v)) for v in wh))

    def unnormalize_error(self, wh, v: float) -> float:
        f = self.lib.acr_unnormalize_error_h
        f.restype = C.c_double
        return f(*(C.c_int(int(x)) for x in wh), C.c_double(v))

    def estimate(self, corr, wh, state, max_iteration: int = 50000, precision: float = np.inf) -> dict:
        """One pair: corr n x 4 (xI, yI, xJ, yJ), wh = (wI, hI, wJ, hJ), state = 625 generator words (left unchanged; the state
        after the estimation is "mt_state_out")."""
        c = np.ascontiguousarray(corr, np.float64).reshape(-1, 4)
        n = c.shape[0]
        st = np.ascontiguousarray(state, np.uint32).reshape(625)
        sto = np.zeros(625, np.uint32)
        valid = C.c_int(); ninl = C.c_int(); ntr = C.c_int(); em = C.c_double(); nfa = C.c_double()
        inl = np.zeros(max(n, 1), np.uint32); H = np.zeros(9, np.float64); tr = np.zeros(TRACE_CAP, np.int32); trn = np.zeros(TRACE_CAP)
        it = self.lib.acr_estimate_h(C.c_int(n), _p(c), C.c_int(int(wh[0])), C.c_int(int(wh[1])), C.c_int(int(wh[2])), C.c_int(int(wh[3])),
                                     _p(st), C.c_long(max_iteration), C.c_double(precision), C.byref(valid), C.byref(ninl), _p(inl), _p(H),
                                     C.byref(em), C.byref(nfa), _p(tr), _p(trn), C.c_int(TRACE_CAP), C.byref(ntr), _p(sto))
        return {"valid": np.array(bool(valid.value)), "inliers": inl[:ninl.value].copy(), "H": H.reshape(3, 3),
                "error_max": np.array(em.value), "min_nfa": np.array(nfa.value), "iterations": np.array(int(it)),
                "trace": tr[:min(ntr.value, TRACE_CAP)].copy(), "n_trace": int(ntr.value), "trace_nfa": trn[:min(ntr.value, TRACE_CAP)].copy(),
                "mt_state_out": sto}


reference_output = functools.partial(oracle.reference_output, path=STORED)
