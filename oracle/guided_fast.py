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
import os
import subprocess

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
STORED = os.path.join(os.path.dirname(_HERE), "tests", "golden", "reference_guided_fast.npz")


def _lib_path(kind: str) -> str:
    return os.path.join(_HERE, "_ref", "libref_guided_fast.so") if kind == "ref" else os.path.join(_HERE, "libport_guided_fast.so")


def available(kind: str) -> bool:
    return os.path.exists(_lib_path(kind))


def build(ref: bool | None = None) -> None:
    """Compile the port always, the "ref" build and the C++ adaptor test when oracle.reference_src() finds an AliceVision tree."""
    src = oracle.reference_src()
    ref = (src is not None) if ref is None else ref
    mk = ["make", "-C", _HERE, "-f", "guided_fast.mk"]
    subprocess.run(mk + ["all"] + (["ref", f"REF={src}"] if ref else []), check=True, stdout=subprocess.DEVNULL)
    if ref and os.path.exists(os.path.join(os.path.dirname(_HERE), "alicevision_b200", "libb200match.so")):
        subprocess.run(mk + ["adaptor", f"REF={src}"], check=True, stdout=subprocess.DEVNULL)


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def _dt(a: np.ndarray, binary: bool) -> int:
    if a.dtype == np.float32:
        return oracle.DT_F32
    return oracle.DT_BIN if binary else oracle.DT_U8


class GuidedFastOracle:
    def __init__(self, kind: str = "port"):
        assert kind in ("ref", "port")
        self.kind = kind
        if not available(kind):
            raise FileNotFoundError(f"{_lib_path(kind)} missing: run oracle.guided_fast.build()")
        self.lib = C.CDLL(_lib_path(kind))
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
