"""ORACLE — test infrastructure only (see oracle/hgrowing_oracle.cpp).

The single-threaded port of filterMatchesByHGrowing (the `homography_growing` filter of featureMatching) on the engine's shared
math header, ``oracle/libport_hgrowing.so``, and the stage around it (``stage``), which mirrors
``matching.robustModelEstimation_HGrowing`` with the port in place of the engine.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(_HERE, "libport_hgrowing.so")
SYMBOLS = ("hg_filter", "hg_grow_steps", "hg_refine", "hg_exp", "hg_log")

# GrowParameters / HGrowingFilteringParam defaults (GeometricFilterMatrix_HGrowing.hpp)
DEFAULT_PARAM = dict(similarityTolerance=20.0, affinityTolerance=10.0, homographyTolerance=5.0, minInliersToRefine=6,
                     nbRefiningIterations=8, maxNbHomographies=10, minNbMatchesPerH=20)


def available() -> bool:
    return os.path.exists(LIB)


def build() -> None:
    oracle.make_current("hgrowing.mk", {"libport_hgrowing.so": (LIB, SYMBOLS)}, ["all"])


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def param_arrays(param: dict | None):
    q = dict(DEFAULT_PARAM, **(param or {}))
    tols = np.array([q["similarityTolerance"], q["affinityTolerance"], q["homographyTolerance"]], np.float64)
    ints = np.array([q["minInliersToRefine"], q["nbRefiningIterations"], q["maxNbHomographies"], q["minNbMatchesPerH"]], np.int32)
    return tols, ints


class HGrowingOracle:
    def __init__(self):
        if not available():
            raise FileNotFoundError(f"{LIB} missing: run oracle.hgrowing.build()")
        self.lib = C.CDLL(LIB)
        self.lib.hg_exp.restype = C.c_double
        self.lib.hg_exp.argtypes = [C.c_double]
        self.lib.hg_log.restype = C.c_double
        self.lib.hg_log.argtypes = [C.c_double]

    def filter(self, feat, param: dict | None = None) -> dict:
        """filterMatchesByHGrowing on n putatives (n x 8 float32: xI, yI, scaleI, orientationI, xJ, yJ, scaleJ, orientationJ).
        Returns {"H": (n_h, 3, 3), "counts": (n_h,), "inliers": putative indices in outGeometricInliers order, "trace": (rounds, 3) with
        the chosen seed's position in the round's remaining list (-1: no seed grew) and the best-set size before and after the refine,
        "grown", "skipped"}."""
        f = np.ascontiguousarray(feat, np.float32).reshape(-1, 8)
        tols, ints = param_arrays(param)
        mh = int(ints[2])
        nh, rounds = np.zeros(1, np.int32), np.zeros(1, np.int32)
        H = np.zeros((max(mh, 1), 9)); counts = np.zeros(max(mh, 1), np.int32); trace = np.zeros((max(mh, 1), 3), np.int32)
        inl = np.zeros(max(len(f), 1), np.int32); stats = np.zeros(2, np.int64)
        n_out = self.lib.hg_filter(C.c_int(len(f)), _p(f), _p(tols), _p(ints), _p(nh), _p(H), _p(counts), _p(inl), _p(trace), _p(rounds), _p(stats))
        k = int(nh[0])
        return {"H": H[:k].reshape(k, 3, 3), "counts": counts[:k].copy(), "inliers": inl[:n_out].copy(), "trace": trace[:int(rounds[0])].copy(),
                "grown": int(stats[0]), "skipped": int(stats[1])}

    def grow_steps(self, feat, seed: int, param: dict | None = None):
        """Every growHomography step of one seed over the whole list: (steps x 3 x 3 transformations, inlier counts)."""
        f = np.ascontiguousarray(feat, np.float32).reshape(-1, 8)
        tols, ints = param_arrays(param)
        T = np.zeros((max(int(ints[1]), 1), 9)); cnt = np.zeros(max(int(ints[1]), 1), np.int32)
        s = self.lib.hg_grow_steps(C.c_int(len(f)), _p(f), _p(tols), _p(ints), C.c_int(seed), _p(T), _p(cnt))
        return T[:s].reshape(s, 3, 3), cnt[:s].copy()

    def refine(self, feat, H, tol: float = 5.0):
        """refineHomography of H on every match of feat: (usable, refined H normalised by H(2,2))."""
        f = np.ascontiguousarray(feat, np.float32).reshape(-1, 8)
        h = np.ascontiguousarray(H, np.float64).reshape(9).copy()
        ok = self.lib.hg_refine(C.c_int(len(f)), _p(f), C.c_double(tol), _p(h))
        return bool(ok), h.reshape(3, 3)


def putative_features(featuresI, featuresJ, matches) -> np.ndarray:
    """The n x 8 work item of one (pair, type): the PointFeatures (x, y, scale, orientation) of each putative's two features."""
    fi = np.asarray(featuresI, np.float32).reshape(-1, 4)
    fj = np.asarray(featuresJ, np.float32).reshape(-1, 4)
    return np.ascontiguousarray(np.concatenate([fi[matches["i"]], fj[matches["j"]]], axis=1), np.float32)


def stage(putatives: dict, features_per_view: dict, guidedMatching: bool = False, param: dict | None = None, desc_types=None,
          tag_types=("cctag3", "cctag4", "tag16h5")):
    """matching.robustModelEstimation_HGrowing with the port in place of the engine: the same rules, one port call per (pair, type)."""
    from alicevision_b200.matching import DESCRIBER_TYPES
    order = list(desc_types) if desc_types is not None else DESCRIBER_TYPES
    ora = HGrowingOracle()
    out, hs = {}, {}
    for (I, J), per_type in putatives.items():
        common = [t for t in order if t in features_per_view[I] and t in features_per_view[J]]
        if any(t in tag_types for t in common):
            continue
        done = {}
        for t in common:
            if t not in per_type:
                continue
            m = per_type[t]
            r = ora.filter(putative_features(features_per_view[I][t], features_per_view[J][t], m), param)
            done[t] = (r, m)
        if not done:
            continue
        hs[(I, J)] = {t: [(r["H"][k], m[r["inliers"][sum(r["counts"][:k]):sum(r["counts"][:k + 1])]]) for k in range(len(r["counts"]))]
                      for t, (r, m) in done.items()}
        out[(I, J)] = {} if guidedMatching else {t: m[r["inliers"]] for t, (r, m) in done.items()}
    return out, hs
