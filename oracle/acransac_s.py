"""ORACLE — test infrastructure only (see oracle/acransac_s_oracle.cpp).

A-contrario RANSAC fundamental-matrix estimation of one pair of equidistant cameras on lifted unit vectors
(GeometricFilterMatrix_F_AC::geometricEstimation_Spherical_Mat):

* ``AcransacSOracle("ref")``  -> oracle/_ref/libref_acransac_s.so: the reference's ACRANSAC loop, sampling, NFA tables and cubic solver
  compiled verbatim from an AliceVision source tree, around the restated spherical kernel.
* ``AcransacSOracle("port")`` -> oracle/libport_acransac_s.so: all of it restated.

``reference_output()`` stores the "ref" outputs in tests/golden/reference_acransac_s.npz and replays them where the reference is
not built, like ``oracle.acransac_h.reference_output`` does for the homography.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
STORED = os.path.join(os.path.dirname(_HERE), "tests", "golden", "reference_acransac_s.npz")
TRACE_CAP = 4096
FIELDS = ("valid", "inliers", "F", "error_max", "min_nfa", "iterations", "trace", "mt_state_out")   # stored fields of estimate()
PRIMITIVES = ("acrs_fit7s", "acrs_spherical_error", "acrs_estimate")


def _lib_path(kind: str) -> str:
    return os.path.join(_HERE, "_ref", "libref_acransac_s.so") if kind == "ref" else os.path.join(_HERE, "libport_acransac_s.so")


def available(kind: str) -> bool:
    return os.path.exists(_lib_path(kind))


def build(ref: bool | None = None) -> None:
    """Compile the port always, the "ref" build when oracle.reference_src() finds an AliceVision tree."""
    src = oracle.reference_src()
    ref = (src is not None) if ref is None else ref
    targets = {"libport_acransac_s.so": (_lib_path("port"), PRIMITIVES)}
    if ref:
        targets["_ref/libref_acransac_s.so"] = (_lib_path("ref"), PRIMITIVES)
    oracle.make_current("acransac_s.mk", targets, ["all"] + (["ref", f"REF={src}"] if ref else []))


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class AcransacSOracle:
    def __init__(self, kind: str = "port"):
        assert kind in ("ref", "port")
        self.kind = kind
        if not available(kind):
            raise FileNotFoundError(f"{_lib_path(kind)} missing: run oracle.acransac_s.build()")
        self.lib = C.CDLL(_lib_path(kind))
        self.lib.acrs_estimate.restype = C.c_long
        self.lib.acrs_fit7s.restype = C.c_int

    def mt_seed(self, seed: int) -> np.ndarray:
        st = np.zeros(625, np.uint32)
        self.lib.acrs_mt_seed(C.c_uint32(seed), _p(st))
        return st

    def fit7s(self, bearings) -> list:
        """The spherical 7-point solver on 7 bearing pairs (7 x 6): its models (0..3 matrices, x_J^T F x_I = 0)."""
        b = np.ascontiguousarray(bearings, np.float64).reshape(7, 6)
        F = np.zeros(27, np.float64)
        nb = self.lib.acrs_fit7s(_p(b), _p(F))
        return [F[9 * m:9 * m + 9].reshape(3, 3).copy() for m in range(nb)]

    def errors(self, F, bearings) -> np.ndarray:
        b = np.ascontiguousarray(bearings, np.float64).reshape(-1, 6)
        f = np.ascontiguousarray(F, np.float64).reshape(9)
        e = np.zeros(b.shape[0])
        self.lib.acrs_spherical_error(_p(f), C.c_int(b.shape[0]), _p(b), _p(e))
        return e

    def estimate(self, bearings, state, max_iteration: int = 50000, precision: float = np.inf) -> dict:
        """One pair: bearings n x 6 (xI, yI, zI, xJ, yJ, zJ), state = 625 generator words (left unchanged; the state after the
        estimation is "mt_state_out")."""
        b = np.ascontiguousarray(bearings, np.float64).reshape(-1, 6)
        n = b.shape[0]
        st = np.ascontiguousarray(state, np.uint32).reshape(625)
        sto = np.zeros(625, np.uint32)
        valid = C.c_int(); ninl = C.c_int(); ntr = C.c_int(); em = C.c_double(); nfa = C.c_double()
        inl = np.zeros(max(n, 1), np.uint32); F = np.zeros(9, np.float64); tr = np.zeros(TRACE_CAP, np.int32); trn = np.zeros(TRACE_CAP)
        it = self.lib.acrs_estimate(C.c_int(n), _p(b), _p(st), C.c_long(max_iteration), C.c_double(precision), C.byref(valid), C.byref(ninl),
                                    _p(inl), _p(F), C.byref(em), C.byref(nfa), _p(tr), _p(trn), C.c_int(TRACE_CAP), C.byref(ntr), _p(sto))
        return {"valid": np.array(bool(valid.value)), "inliers": inl[:ninl.value].copy(), "F": F.reshape(3, 3),
                "error_max": np.array(em.value), "min_nfa": np.array(nfa.value), "iterations": np.array(int(it)),
                "trace": tr[:min(ntr.value, TRACE_CAP)].copy(), "n_trace": int(ntr.value), "trace_nfa": trn[:min(ntr.value, TRACE_CAP)].copy(),
                "mt_state_out": sto}


_stored: dict | None = None


def reference_output(key: str, compute, live: bool):
    """What the "ref" build returns for test case `key`: computed and checked against the stored copy when it is built (stored with
    ORACLE_RECORD_REFERENCE=1), else the stored copy."""
    global _stored
    if _stored is None:
        _stored = {}
        if os.path.exists(STORED):
            flat = oracle._load_flat(STORED)
            tops = {k.split("/")[0].split("#")[0] for k in flat}
            _stored = {t: oracle._unflatten(t, flat) for t in tops}
    if not live:
        if key not in _stored:
            raise KeyError(f"no stored reference output for {key!r}: regenerate {STORED} with the reference built")
        return _stored[key]
    v = compute()
    if os.environ.get("ORACLE_RECORD_REFERENCE") == "1":
        _stored[key] = v
        out = {}
        for k, x in _stored.items():
            oracle._flatten(k, x, out)
        oracle._save_flat(STORED, out)
    elif key in _stored:
        assert oracle._same(v, _stored[key]), f"the compiled reference no longer gives the stored output for {key!r}"
    return v
