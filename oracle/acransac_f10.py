"""ORACLE — test infrastructure only (see oracle/acransac_f10_oracle.cpp).

A-contrario RANSAC fundamental-matrix estimation with radial distortion of one planar pair
(GeometricFilterMatrix_F_AC::geometricEstimation_Mat_ACRANSAC<Fundamental10PSolver, Fundamental10PModel>):

* ``AcransacF10Oracle("ref")``  -> oracle/_ref/libref_acransac_f10.so: the reference's ACRANSAC loop, sampling and NFA tables
  compiled verbatim from an AliceVision source tree, around the restated F10 kernel.
* ``AcransacF10Oracle("port")`` -> oracle/libport_acransac_f10.so: all of it restated.

``reference_output()`` stores the "ref" outputs in tests/golden/reference_acransac_f10.npz and replays them where the reference is
not built, like ``oracle.acransac_e.reference_output`` does for the essential matrix.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
STORED = os.path.join(os.path.dirname(_HERE), "tests", "golden", "reference_acransac_f10.npz")
TRACE_CAP = 4096
FIELDS = ("valid", "inliers", "F", "L", "error_max", "min_nfa", "iterations", "trace", "mt_state_out")   # stored fields of estimate()
PRIMITIVES = ("acrf10_fit10", "acrf10_estimate", "acrf10_mt_seed")


def _lib_path(kind: str) -> str:
    return os.path.join(_HERE, "_ref", "libref_acransac_f10.so") if kind == "ref" else os.path.join(_HERE, "libport_acransac_f10.so")


def available(kind: str) -> bool:
    return os.path.exists(_lib_path(kind))


def build(ref: bool | None = None) -> None:
    """Compile the port always, the "ref" build when oracle.reference_src() finds an AliceVision tree."""
    src = oracle.reference_src()
    ref = (src is not None) if ref is None else ref
    targets = {"libport_acransac_f10.so": (_lib_path("port"), PRIMITIVES)}
    if ref:
        targets["_ref/libref_acransac_f10.so"] = (_lib_path("ref"), PRIMITIVES)
    oracle.make_current("acransac_f10.mk", targets, ["all"] + (["ref", f"REF={src}"] if ref else []))


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class AcransacF10Oracle:
    def __init__(self, kind: str = "port"):
        assert kind in ("ref", "port")
        self.kind = kind
        if not available(kind):
            raise FileNotFoundError(f"{_lib_path(kind)} missing: run oracle.acransac_f10.build()")
        self.lib = C.CDLL(_lib_path(kind))
        self.lib.acrf10_estimate.restype = C.c_long
        self.lib.acrf10_fit10.restype = C.c_int

    def mt_seed(self, seed: int) -> np.ndarray:
        st = np.zeros(625, np.uint32)
        self.lib.acrf10_mt_seed(C.c_uint32(seed), _p(st))
        return st

    def fit10(self, corr, action: bool = False):
        """The 10-point solver on 10 correspondences (10 x (xI, yI, xJ, yJ)): its models as a list of (F 3 x 3, L = (l1, l2)),
        [x_I, y_I, 1 + l1 r_I^2] F [x_J, y_J, 1 + l2 r_J^2]^T = 0; with action=True also the 10 x 10 action matrix it built."""
        c = np.ascontiguousarray(corr, np.float64).reshape(10, 4)
        F = np.zeros(90); L = np.zeros(20); At = np.zeros(100)
        nb = self.lib.acrf10_fit10(_p(c), _p(F), _p(L), _p(At))
        models = [(F[9 * m:9 * m + 9].reshape(3, 3).copy(), L[2 * m:2 * m + 2].copy()) for m in range(nb)]
        return (models, At.reshape(10, 10)) if action else models

    def estimate(self, corr, wh, state, max_iteration: int = 50000, precision: float = np.inf) -> dict:
        """One pair: corr n x 4 pixels (xI, yI, xJ, yJ), wh = (wI, hI, wJ, hJ), state = 625 generator words (left unchanged; the
        state after the estimation is "mt_state_out").  precision is ACRANSAC's argument."""
        c = np.ascontiguousarray(corr, np.float64).reshape(-1, 4)
        n = c.shape[0]
        w = np.ascontiguousarray(wh, np.int32).reshape(4)
        st = np.ascontiguousarray(state, np.uint32).reshape(625)
        sto = np.zeros(625, np.uint32)
        valid = C.c_int(); ninl = C.c_int(); ntr = C.c_int(); em = C.c_double(); nfa = C.c_double()
        inl = np.zeros(max(n, 1), np.uint32); F = np.zeros(9); L = np.zeros(2); tr = np.zeros(TRACE_CAP, np.int32); trn = np.zeros(TRACE_CAP)
        it = self.lib.acrf10_estimate(C.c_int(n), _p(c), _p(w), _p(st), C.c_long(max_iteration), C.c_double(precision), C.byref(valid),
                                      C.byref(ninl), _p(inl), _p(F), _p(L), C.byref(em), C.byref(nfa), _p(tr), _p(trn), C.c_int(TRACE_CAP),
                                      C.byref(ntr), _p(sto))
        return {"valid": np.array(bool(valid.value)), "inliers": inl[:ninl.value].copy(), "F": F.reshape(3, 3), "L": L,
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
