"""Python host-side mirror of the reference interface for the descriptor-matching path, over the C ABI.

The product is the C-ABI library (include/b200match.h) plus the C++ adaptors in alicevision_b200/adaptor/.
This module binds the same C entry points with ctypes so that the parity tests and the bench read like the
reference's own tests (same method names and argument meaning):

* ``ArrayMatcherB200``            <->  matching::ArrayMatcher<Scalar,Metric>      (matching/ArrayMatcher.hpp:19-66)
* ``ImageCollectionMatcherB200``  <->  matchingImageCollection::IImageCollectionMatcher (IImageCollectionMatcher.hpp:28-42)
* ``EMatcherType``                <->  matching::EMatcherType                      (matching/matcherType.hpp:15-22)

Nothing here computes distances: if the CUDA library is missing or no GPU is present, construction fails loudly.
"""
from __future__ import annotations

import atexit
import ctypes as C
import itertools
import os
import weakref
from enum import IntEnum

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200match.so")

F32, U8, BIN = 0, 1, 2
L2_SIMPLE, L2_VECTORIZED, HAMMING = 0, 1, 2
STAGE_DEVICE, STAGE_RAW, STAGE_FULL = 0, 1, 2
MODEL_FUNDAMENTAL, MODEL_HOMOGRAPHY = 0, 1

MATCH_DTYPE = np.dtype([("i", np.uint32), ("j", np.uint32), ("ratio", np.float32), ("dist", np.float32)])

# every symbol include/b200match.h declares (checked by tests/test_abi.py)
ABI_SYMBOLS = [
    "b200m_last_error", "b200m_version", "b200m_device_count", "b200m_ctx_create", "b200m_ctx_destroy", "b200m_ctx_set_host_threads",
    "b200m_ctx_set_force_exact", "b200m_ctx_set_tc_variant", "b200m_debug_trace", "b200m_debug_convert_f32_u8", "b200m_db_create", "b200m_db_destroy", "b200m_knn", "b200m_upload_view", "b200m_upload_views", "b200m_upload_views_async", "b200m_wait_uploads", "b200m_clear_views", "b200m_remove_view",
    "b200m_match_pairs", "b200m_result_num_pairs", "b200m_result_get", "b200m_result_free", "b200m_last_gpu_ms",
    "b200m_last_search_kernel_ms", "b200m_last_launches", "b200m_last_tc_pairs", "b200m_exactness_errors", "b200m_last_records", "b200m_last_real_tc_pairs", "b200m_last_fallback_rows", "b200m_last_u8_tc_pairs", "b200m_last_batches",
    "b200m_last_u8_norm_gemm_pairs",
    "b200m_shard_pairs", "b200m_shard_pairs_2d", "b200m_multi_create", "b200m_multi_destroy", "b200m_multi_num_devices", "b200m_multi_ctx", "b200m_multi_match",
    "b200m_multi_last_gpu_ms", "b200m_guided_match", "b200m_guided_match_model", "b200m_set_view_geometry", "b200m_guided_match_fast_pairs",
    "b200m_acransac_fundamental_pairs", "b200m_acransac_last_stats", "b200m_acransac_last_trace", "b200m_ctx_set_acransac_skip",
    "b200m_mt19937_seed", "b200m_debug_rand_sample", "b200m_acransac_homography_pairs", "b200m_debug_rand_sample_k", "b200m_guided_match_pairs",
    "b200m_guided_match_positions_pairs", "b200m_acransac_fundamental_spherical_pairs", "b200m_hgrowing_pairs", "b200m_hgrowing_last_stats",
    "b200m_ctx_set_hgrowing_window", "b200m_acransac_essential_pairs", "b200m_acransac_fundamental_distortion_pairs",
]


class EMatcherType(IntEnum):
    """matching/matcherType.hpp:15-22 plus the two values an integration adds for this engine."""
    BRUTE_FORCE_L2 = 0
    ANN_L2 = 1
    CASCADE_HASHING_L2 = 2
    FAST_CASCADE_HASHING_L2 = 3
    BRUTE_FORCE_HAMMING = 4
    BRUTE_FORCE_L2_B200 = 5
    BRUTE_FORCE_HAMMING_B200 = 6


class B200MatchError(RuntimeError):
    pass


_lib = None


def load_library() -> C.CDLL:
    """Load libb200match.so (no fallback: a missing library is an error)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200MatchError(f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    lib.b200m_last_error.restype = C.c_char_p
    lib.b200m_last_gpu_ms.restype = C.c_double
    lib.b200m_last_search_kernel_ms.restype = C.c_double
    lib.b200m_last_records.restype = C.c_int64
    lib.b200m_last_fallback_rows.restype = C.c_int64
    lib.b200m_exactness_errors.restype = C.c_uint
    lib.b200m_multi_last_gpu_ms.restype = C.c_double
    lib.b200m_multi_ctx.restype = C.c_void_p
    lib.b200m_acransac_last_stats.restype = C.c_double
    lib.b200m_hgrowing_last_stats.restype = C.c_double
    for name in ("b200m_ctx_destroy", "b200m_db_destroy", "b200m_result_free", "b200m_multi_destroy", "b200m_mt19937_seed"):
        getattr(lib, name).restype = None
    _lib = lib
    return lib


def _check(rc: int, what: str) -> None:
    if rc != 0:
        raise B200MatchError(f"{what} failed (status {rc}): {load_library().b200m_last_error().decode()}")


def _dtype_code(a: np.ndarray, binary: bool) -> int:
    if a.dtype == np.float32:
        return F32
    if a.dtype == np.uint8:
        return BIN if binary else U8
    raise TypeError(f"unsupported descriptor dtype {a.dtype} (float32 / uint8 only)")


_live_contexts: "weakref.WeakSet[Context]" = weakref.WeakSet()


@atexit.register
def _drain_uploads_at_exit() -> None:
    """Asynchronous uploads read numpy memory from an engine thread: let them finish before the interpreter frees it."""
    for ctx in list(_live_contexts):
        try:
            if ctx._h:
                ctx.lib.b200m_wait_uploads(ctx._h)
        except Exception:
            pass


class Context:
    """One engine instance bound to one GPU (``b200m_ctx``)."""

    def __init__(self, device: int = 0, stream: int | None = None):
        self.lib = load_library()
        self._h = C.c_void_p()
        _check(self.lib.b200m_ctx_create(C.c_int(device), C.c_void_p(stream or 0), C.byref(self._h)), "b200m_ctx_create")
        _live_contexts.add(self)

    def close(self) -> None:
        if self._h:
            self.lib.b200m_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_host_threads(self, n: int) -> None:
        _check(self.lib.b200m_ctx_set_host_threads(self._h, C.c_int(n)), "b200m_ctx_set_host_threads")

    def set_force_exact(self, on: bool) -> None:
        _check(self.lib.b200m_ctx_set_force_exact(self._h, C.c_int(int(on))), "b200m_ctx_set_force_exact")

    def set_tc_variant(self, variant: int) -> None:
        _check(self.lib.b200m_ctx_set_tc_variant(self._h, C.c_int(variant)), "b200m_ctx_set_tc_variant")

    def debug_trace(self, enable: bool = True, read: bool = False):
        """Enable / read the per-tile pipeline trace (roles x 512 tiles x 4 stamps) of CTA 0 of the tensor-core kernel."""
        out = np.zeros((4, 512, 4), np.int64)
        _check(self.lib.b200m_debug_trace(self._h, C.c_int(int(enable)), out.ctypes.data_as(C.c_void_p) if read else None, C.c_int(out.size)), "b200m_debug_trace")
        return out

    # instrumentation
    def last_gpu_ms(self) -> float: return self.lib.b200m_last_gpu_ms(self._h)
    def last_search_kernel_ms(self) -> float: return self.lib.b200m_last_search_kernel_ms(self._h)
    def last_launches(self) -> int: return self.lib.b200m_last_launches(self._h)
    def last_tc_pairs(self) -> int: return self.lib.b200m_last_tc_pairs(self._h)
    def exactness_errors(self) -> int: return self.lib.b200m_exactness_errors(self._h)
    def last_records(self) -> int: return self.lib.b200m_last_records(self._h)
    def last_real_tc_pairs(self) -> int: return self.lib.b200m_last_real_tc_pairs(self._h)
    def last_fallback_rows(self) -> int: return self.lib.b200m_last_fallback_rows(self._h)
    def last_u8_tc_pairs(self) -> int: return self.lib.b200m_last_u8_tc_pairs(self._h)
    def last_u8_norm_gemm_pairs(self) -> int: return self.lib.b200m_last_u8_norm_gemm_pairs(self._h)
    def last_batches(self) -> int: return self.lib.b200m_last_batches(self._h)

    def set_view_geometry(self, view_id: int, xy) -> None:
        """b200m_set_view_geometry: the n x 2 double positions guided matching uses for an uploaded view instead of its float
        upload positions (typically camera::IntrinsicBase::getUndistortedPixel of every feature); None drops them."""
        if xy is None:
            _check(self.lib.b200m_set_view_geometry(self._h, C.c_uint32(view_id), None, C.c_int(0)), "b200m_set_view_geometry")
            return
        a = np.ascontiguousarray(xy, np.float64).reshape(-1, 2)
        _check(self.lib.b200m_set_view_geometry(self._h, C.c_uint32(view_id), a.ctypes.data_as(C.c_void_p), C.c_int(a.shape[0])),
               "b200m_set_view_geometry")

    def guided_match_fast_pairs(self, pairs, F, epipole2, wh, errorTh: float, distRatio: float) -> dict:
        """b200m_guided_match_fast_pairs on resident views: guidedMatchingFundamentalFast (matching/guidedMatching.hpp:353-460) for
        every (L, R) of `pairs`, with per-pair F [n, 3, 3] (x_R^T F x_L = 0), epipole2 [n, 3] (not normalised) and wh [n, 2] =
        (widthR, heightR); errorTh / distRatio already squared.  Returns {(L, R): matches[MATCH_DTYPE]} in input order, empty lists
        included; matches in ascending i, not de-duplicated."""
        p = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
        n = p.shape[0]
        Fm = np.ascontiguousarray(F, np.float64).reshape(n, 9)
        ep = np.ascontiguousarray(epipole2, np.float64).reshape(n, 3)
        whm = np.ascontiguousarray(wh, np.int32).reshape(n, 2)
        res = C.c_void_p()
        _check(self.lib.b200m_guided_match_fast_pairs(self._h, p.ctypes.data_as(C.c_void_p), C.c_int(n), Fm.ctypes.data_as(C.c_void_p),
                                                      ep.ctypes.data_as(C.c_void_p), whm.ctypes.data_as(C.c_void_p), C.c_double(errorTh),
                                                      C.c_double(distRatio), C.byref(res)), "b200m_guided_match_fast_pairs")
        return {(int(a), int(b)): m for (a, b), m in zip(p.tolist(), self._pair_lists(res, n))}

    def guided_match_pairs(self, pairs, M, errorTh, distRatio: float, model: int = MODEL_FUNDAMENTAL) -> list:
        """b200m_guided_match_pairs on resident views: guidedMatching (matching/guidedMatching.hpp:206-268) for every (L, R) of `pairs`
        with its own model M [n, 3, 3] (MODEL_FUNDAMENTAL: x_R^T F x_L = 0; MODEL_HOMOGRAPHY: x_R ~ H x_L) and errorTh [n], already
        squared; distRatio already squared, one for the call.  Returns one matches[MATCH_DTYPE] per input pair, in input order (a pair
        may appear more than once): ascending i, ratio and distance 0."""
        p = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
        n = p.shape[0]
        Mm = np.ascontiguousarray(M, np.float64).reshape(n, 9)
        th = np.ascontiguousarray(errorTh, np.float64).reshape(n)
        res = C.c_void_p()
        _check(self.lib.b200m_guided_match_pairs(self._h, p.ctypes.data_as(C.c_void_p), C.c_int(n), C.c_int(model), Mm.ctypes.data_as(C.c_void_p),
                                                 th.ctypes.data_as(C.c_void_p), C.c_double(distRatio), C.byref(res)), "b200m_guided_match_pairs")
        return self._pair_lists(res, n)

    def guided_match_positions_pairs(self, pairs, M, errorTh, model: int = MODEL_HOMOGRAPHY, decorate: bool = True) -> list:
        """b200m_guided_match_positions_pairs on resident views: position-only guidedMatching (matching/guidedMatching.hpp:37-70) for
        every (L, R) of `pairs`, with its own model M [n, 3, 3] and errorTh [n] (already squared): per left feature the right feature of
        smallest error below errorTh, the first on ties; no descriptors.  decorate=True then applies IndMatchDecorator::getDeduplicated
        on the upload positions, as GeometricFilterMatrix_H_AC does with distanceRatio < 0.  Returns one matches[MATCH_DTYPE] per input
        pair, in input order: sorted by (i, j) without decoration, in the decorator's order with it; ratio and distance 0."""
        p = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
        n = p.shape[0]
        Mm = np.ascontiguousarray(M, np.float64).reshape(n, 9)
        th = np.ascontiguousarray(errorTh, np.float64).reshape(n)
        res = C.c_void_p()
        _check(self.lib.b200m_guided_match_positions_pairs(self._h, p.ctypes.data_as(C.c_void_p), C.c_int(n), C.c_int(model),
                                                           Mm.ctypes.data_as(C.c_void_p), th.ctypes.data_as(C.c_void_p), C.c_int(int(bool(decorate))),
                                                           C.byref(res)), "b200m_guided_match_positions_pairs")
        return self._pair_lists(res, n)

    def _pair_lists(self, res, n: int) -> list:
        owner = _ResultOwner(self.lib, res)
        off, mat = C.c_void_p(), C.c_void_p()
        _check(self.lib.b200m_result_get(res, None, C.byref(off), C.byref(mat)), "b200m_result_get")
        offsets = _alias(off.value, (n + 1) * 8, np.int64, owner) if n else np.zeros(1, np.int64)
        matches = _alias(mat.value, int(offsets[-1]) * MATCH_DTYPE.itemsize, MATCH_DTYPE, owner)
        return [matches[offsets[k]:offsets[k + 1]].copy() for k in range(n)]

    def set_acransac_skip(self, on: bool) -> None:
        """Debug: the certified skip of models that cannot beat the running minNFA (on by default); results do not depend on it."""
        _check(self.lib.b200m_ctx_set_acransac_skip(self._h, C.c_int(int(on))), "b200m_ctx_set_acransac_skip")

    def acransac_fundamental_pairs(self, corr_list, wh, mt_state, maxIteration: int = 50000, precision: float = np.inf) -> list[dict]:
        """b200m_acransac_fundamental_pairs: GeometricFilterMatrix_F_AC::geometricEstimation_Mat_ACRANSAC<Fundamental7PSolver> for
        every pair.  corr_list: per pair an n x 4 array (xI, yI, xJ, yJ); wh: per pair (widthI, heightI, widthJ, heightJ);
        mt_state: 625 words (mt19937_state), the same for every pair.  Returns per pair, in input order, {"valid", "inliers" (the
        reference's order), "F" (3 x 3, x_J^T F x_I = 0), "error_max", "min_nfa", "iterations", "trace" / "trace_nfa" (iterations at
        which a better model was found and its minNFA, the first 256), "n_trace"}."""
        return self._acransac_pairs("F", corr_list, wh, np.ascontiguousarray(mt_state, np.uint32).reshape(625), maxIteration, precision)

    def acransac_homography_pairs(self, corr_list, wh, mt_state_or_states, maxIteration: int = 50000, precision: float = np.inf) -> list[dict]:
        """b200m_acransac_homography_pairs: GeometricFilterMatrix_H_AC::geometricEstimation (ACRANSAC with Homography4PSolver and the
        point-to-point error) for every pair.  corr_list and wh as in acransac_fundamental_pairs; mt_state_or_states: one 625-word
        state for every pair, or an n_pairs x 625 array of per-pair start states.  Returns per pair the fields of
        acransac_fundamental_pairs with "H" (3 x 3, x_J ~ H x_I) in place of "F", and "mt_state_out": the generator state after the
        pair's estimation (the reference passes its generator on from pair to pair)."""
        return self._acransac_pairs("H", corr_list, wh, _mt_states(mt_state_or_states, len(corr_list)), maxIteration, precision)

    def acransac_fundamental_spherical_pairs(self, corr_list, mt_state_or_states, maxIteration: int = 50000,
                                             precision: float = np.inf) -> list[dict]:
        """b200m_acransac_fundamental_spherical_pairs: GeometricFilterMatrix_F_AC::geometricEstimation_Spherical_Mat (ACRANSAC with
        Fundamental7PSphericalSolver and EpipolarSphericalDistanceError, the branch for two equidistant cameras) for every pair.
        corr_list: per pair an n x 6 array (xI, yI, zI, xJ, yJ, zJ) of lifted unit vectors; no image sizes.  mt_state_or_states as in
        acransac_homography_pairs.  Returns per pair the fields of acransac_fundamental_pairs ("F": x_J^T F x_I = 0 on the bearings)
        and "mt_state_out": the generator state after the pair's estimation (the reference passes this generator by reference)."""
        return self._acransac_pairs("S", corr_list, None, _mt_states(mt_state_or_states, len(corr_list)), maxIteration, precision)

    def acransac_essential_pairs(self, corr_list, wh, K, mt_state_or_states, maxIteration: int = 50000, precision: float = np.inf) -> list[dict]:
        """b200m_acransac_essential_pairs: GeometricFilterMatrix_E_AC::geometricEstimation (ACRANSAC with Essential5PSolver on K^-1 x
        and the point-to-line error of K_J^-T E K_I^-1 on the pixels) for every pair.  corr_list and wh as in
        acransac_fundamental_pairs; K: per pair (K_I, K_J), two 3 x 3 camera matrices; mt_state_or_states as in
        acransac_homography_pairs.  `precision` is ACRANSAC's own argument (the filter passes it squared).  Returns per pair the fields
        of acransac_fundamental_pairs with "E" (3 x 3) in place of "F", and "mt_state_out"."""
        Km = np.ascontiguousarray(K, np.float64).reshape(len(corr_list), 18)
        return self._acransac_pairs("E", corr_list, wh, _mt_states(mt_state_or_states, len(corr_list)), maxIteration, precision, Km)

    def acransac_fundamental_distortion_pairs(self, corr_list, wh, mt_state, maxIteration: int = 50000, precision: float = np.inf) -> list[dict]:
        """b200m_acransac_fundamental_distortion_pairs: GeometricFilterMatrix_F_AC::geometricEstimation_Mat_ACRANSAC<Fundamental10PSolver,
        Fundamental10PModel> (the fundamental_with_distortion filter on a planar pair) for every pair.  Arguments as in
        acransac_fundamental_pairs (every pair starts from mt_state).  Returns per pair its fields, with "F" the reference's model
        matrix (the solver's constraint is [x_I, y_I, 1 + l1 r_I^2] F [x_J, y_J, 1 + l2 r_J^2]^T = 0 on preconditioned points; the
        score reads F as x_J^T F x_I on undistorted pixels, as the reference does), and "L" = (l1, l2), the same model's radial
        distortion in preconditioned units (0 without a model).  A pair with at most 10 correspondences returns (0, 0)."""
        return self._acransac_pairs("F10", corr_list, wh, np.ascontiguousarray(mt_state, np.uint32).reshape(625), maxIteration, precision)

    def _acransac_pairs(self, kind: str, corr_list, wh, st, maxIteration, precision, K=None) -> list[dict]:
        width = 6 if kind == "S" else 4
        cs = [np.ascontiguousarray(c, np.float64).reshape(-1, width) for c in corr_list]
        n = len(cs)
        offsets = np.zeros(n + 1, np.int64)
        offsets[1:] = np.cumsum([c.shape[0] for c in cs]) if n else []
        corr = np.ascontiguousarray(np.concatenate(cs) if n and offsets[-1] else np.zeros((1, width)), np.float64)
        whm = np.ascontiguousarray(wh, np.int32).reshape(n, 4) if kind != "S" else None
        valid = np.zeros(max(n, 1), np.uint8); ninl = np.zeros(max(n, 1), np.int32); it = np.zeros(max(n, 1), np.int32)
        inl = np.zeros(max(int(offsets[-1]), 1), np.uint32); M = np.zeros((max(n, 1), 9)); em = np.zeros(max(n, 1)); nfa = np.zeros(max(n, 1))
        ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        sto = np.zeros((max(n, 1), 625), np.uint32) if kind not in ("F", "F10") else None
        Ls = np.zeros((max(n, 1), 2)) if kind == "F10" else None
        if kind == "H":
            _check(self.lib.b200m_acransac_homography_pairs(self._h, C.c_int(n), ptr(offsets), ptr(corr), ptr(whm), ptr(st), C.c_int(int(st.ndim == 2)),
                                                            C.c_int64(maxIteration), C.c_double(precision), ptr(valid), ptr(ninl), ptr(inl), ptr(M),
                                                            ptr(em), ptr(nfa), ptr(it), ptr(sto)),
                   "b200m_acransac_homography_pairs")
        elif kind == "E":
            _check(self.lib.b200m_acransac_essential_pairs(self._h, C.c_int(n), ptr(offsets), ptr(corr), ptr(whm), ptr(K if n else np.zeros(18)),
                                                           ptr(st), C.c_int(int(st.ndim == 2)), C.c_int64(maxIteration), C.c_double(precision),
                                                           ptr(valid), ptr(ninl), ptr(inl), ptr(M), ptr(em), ptr(nfa), ptr(it), ptr(sto)),
                   "b200m_acransac_essential_pairs")
        elif kind == "S":
            _check(self.lib.b200m_acransac_fundamental_spherical_pairs(self._h, C.c_int(n), ptr(offsets), ptr(corr), ptr(st), C.c_int(int(st.ndim == 2)),
                                                                       C.c_int64(maxIteration), C.c_double(precision), ptr(valid), ptr(ninl),
                                                                       ptr(inl), ptr(M), ptr(em), ptr(nfa), ptr(it), ptr(sto)),
                   "b200m_acransac_fundamental_spherical_pairs")
        elif kind == "F10":
            _check(self.lib.b200m_acransac_fundamental_distortion_pairs(self._h, C.c_int(n), ptr(offsets), ptr(corr), ptr(whm), ptr(st),
                                                                        C.c_int64(maxIteration), C.c_double(precision), ptr(valid), ptr(ninl),
                                                                        ptr(inl), ptr(M), ptr(Ls), ptr(em), ptr(nfa), ptr(it)),
                   "b200m_acransac_fundamental_distortion_pairs")
        else:
            _check(self.lib.b200m_acransac_fundamental_pairs(self._h, C.c_int(n), ptr(offsets), ptr(corr), ptr(whm), ptr(st), C.c_int64(maxIteration),
                                                             C.c_double(precision), ptr(valid), ptr(ninl), ptr(inl), ptr(M), ptr(em), ptr(nfa), ptr(it)),
                   "b200m_acransac_fundamental_pairs")
        out = []
        tr = np.zeros(256, np.int32); trn = np.zeros(256, np.float64)
        for k in range(n):
            nt = self.lib.b200m_acransac_last_trace(self._h, C.c_int(k), ptr(tr), ptr(trn), C.c_int(tr.size))
            r = {"valid": bool(valid[k]), "inliers": inl[offsets[k]:offsets[k] + ninl[k]].copy(), kind if kind in "HE" else "F": M[k].reshape(3, 3).copy(),
                 "error_max": float(em[k]), "min_nfa": float(nfa[k]), "iterations": int(it[k]), "n_trace": int(nt),
                 "trace": tr[:min(nt, tr.size)].copy(), "trace_nfa": trn[:min(nt, trn.size)].copy()}
            if sto is not None:
                r["mt_state_out"] = sto[k].copy()
            if Ls is not None:
                r["L"] = Ls[k].copy()
            out.append(r)
        return out

    def acransac_last_stats(self) -> dict:
        """Instrumentation of the last acransac_fundamental_pairs, acransac_homography_pairs, acransac_fundamental_spherical_pairs,
        acransac_essential_pairs or acransac_fundamental_distortion_pairs call."""
        st = np.zeros(4, np.int64)
        ms = self.lib.b200m_acransac_last_stats(self._h, st.ctypes.data_as(C.c_void_p))
        return {"gpu_ms": ms, "models_evaluated": int(st[0]), "models_skipped": int(st[1]), "models_exact": int(st[2]), "launches": int(st[3])}

    def set_hgrowing_window(self, window: int) -> None:
        """Debug: seeds per item grown speculatively per window by hgrowing_pairs (default 256); 1 is the reference's loop.  Results
        do not depend on it."""
        _check(self.lib.b200m_ctx_set_hgrowing_window(self._h, C.c_int(int(window))), "b200m_ctx_set_hgrowing_window")

    def hgrowing_pairs(self, items, param: dict | None = None) -> list[dict]:
        """b200m_hgrowing_pairs: filterMatchesByHGrowing for every work item, one (pair, describer type) each: an n x 8 float32 array of
        its putatives (xI, yI, scaleI, orientationI, xJ, yJ, scaleJ, orientationJ), in the caller's order.  param: HGrowingParam fields
        (HGROWING_DEFAULTS).  Returns per item {"H": (n_h, 3, 3), "counts": (n_h,), "inliers": putative indices in outGeometricInliers
        order, "trace": (rounds, 3): per round the chosen seed's position in the remaining list (-1: none grew) and the best set's size
        before and after the refine}."""
        q = dict(HGROWING_DEFAULTS, **(param or {}))
        feats = [np.ascontiguousarray(f, np.float32).reshape(-1, 8) for f in items]
        n = len(feats)
        offsets = np.zeros(n + 1, np.int64)
        offsets[1:] = np.cumsum([len(f) for f in feats])
        feat = np.ascontiguousarray(np.concatenate(feats) if n else np.zeros((0, 8), np.float32), np.float32)
        mh = int(q["maxNbHomographies"])
        nh = np.zeros(max(n, 1), np.int32); rounds = np.zeros(max(n, 1), np.int32)
        H = np.zeros((max(n, 1), max(mh, 1), 9)); counts = np.zeros((max(n, 1), max(mh, 1)), np.int32)
        trace = np.zeros((max(n, 1), max(mh, 1), 3), np.int32); inl = np.zeros(max(int(offsets[-1]), 1), np.int32)
        ptr = lambda a: a.ctypes.data_as(C.c_void_p)
        _check(self.lib.b200m_hgrowing_pairs(self._h, C.c_int(n), ptr(offsets), ptr(feat), C.c_double(q["similarityTolerance"]),
                                             C.c_double(q["affinityTolerance"]), C.c_double(q["homographyTolerance"]),
                                             C.c_int(int(q["minInliersToRefine"])), C.c_int(int(q["nbRefiningIterations"])), C.c_int(mh),
                                             C.c_int(int(q["minNbMatchesPerH"])), ptr(nh), ptr(H), ptr(counts), ptr(inl), ptr(trace), ptr(rounds)),
               "b200m_hgrowing_pairs")
        out = []
        for k in range(n):
            h = int(nh[k])
            c = counts[k, :h].copy()
            out.append({"H": H[k, :h].reshape(h, 3, 3).copy(), "counts": c, "inliers": inl[offsets[k]:offsets[k] + int(c.sum())].copy(),
                        "trace": trace[k, :int(rounds[k])].copy()})
        return out

    def hgrowing_last_stats(self) -> dict:
        """Instrumentation of the last hgrowing_pairs call."""
        st = np.zeros(3, np.int64)
        ms = self.lib.b200m_hgrowing_last_stats(self._h, st.ctypes.data_as(C.c_void_p))
        return {"gpu_ms": ms, "seeds_grown": int(st[0]), "seeds_skipped": int(st[1]), "rounds": int(st[2])}


def _mt_states(mt_state_or_states, n: int) -> np.ndarray:
    """One 625-word generator state (shape (625,)) or n per-pair states (n x 625)."""
    st = np.ascontiguousarray(mt_state_or_states, np.uint32)
    if st.ndim == 1:
        return st.reshape(625)
    if st.shape != (n, 625):
        raise ValueError(f"mt_state_or_states: 625 words or n_pairs x 625, got {st.shape}")
    return st


def mt19937_state(seed: int) -> np.ndarray:
    """std::mt19937(seed) as the 625 words of its operator<< (b200m_mt19937_seed; host only)."""
    st = np.zeros(625, np.uint32)
    load_library().b200m_mt19937_seed(C.c_uint32(seed), st.ctypes.data_as(C.c_void_p))
    return st


def debug_rand_sample(state, rng: int, draws: int, sample_size: int = 7):
    """The engine's sampler on the CPU (b200m_debug_rand_sample_k): `draws` consecutive randSample(g, 0, rng, sample_size) from
    `state`, sample_size 7 (fundamental matrix) or 4 (homography).  Returns (draws x sample_size samples in their order, draws x 625
    generator states after each draw)."""
    st = np.ascontiguousarray(state, np.uint32).reshape(625)
    out = np.zeros((draws, sample_size), np.uint32); sts = np.zeros((draws, 625), np.uint32)
    _check(load_library().b200m_debug_rand_sample_k(st.ctypes.data_as(C.c_void_p), C.c_int(sample_size), C.c_int(rng), C.c_int(draws),
                                                    out.ctypes.data_as(C.c_void_p), sts.ctypes.data_as(C.c_void_p)), "b200m_debug_rand_sample_k")
    return out, sts


def geometricEstimation_F_AC(xI, xJ, sizeI, sizeJ, seed_or_state, maxIteration: int = 50000, precision: float = np.inf,
                             ctx: Context | None = None) -> dict:
    """GeometricFilterMatrix_F_AC::geometricEstimation_Mat_ACRANSAC<Fundamental7PSolver, Mat3Model> of one pair on the GPU.
    xI, xJ: n x 2 positions (the 2 x n matrices of fillMatricesWithUndistortFeaturesMatches, transposed); sizeI / sizeJ: (width,
    height); seed_or_state: a std::mt19937 seed or its 625-word state.  Returns the dict of Context.acransac_fundamental_pairs."""
    ctx = ctx or default_context()
    return ctx.acransac_fundamental_pairs(*_one_pair(xI, xJ, sizeI, sizeJ), _start_state(seed_or_state), maxIteration, precision)[0]


def geometricEstimation_F10_AC(xI, xJ, sizeI, sizeJ, seed_or_state, maxIteration: int = 50000, precision: float = np.inf,
                               ctx: Context | None = None) -> dict:
    """GeometricFilterMatrix_F_AC::geometricEstimation_Mat_ACRANSAC<Fundamental10PSolver, Fundamental10PModel> of one planar pair on the
    GPU (the fundamental_with_distortion filter; arguments as geometricEstimation_F_AC).  Returns the dict of
    Context.acransac_fundamental_distortion_pairs: "F" and "L"."""
    ctx = ctx or default_context()
    return ctx.acransac_fundamental_distortion_pairs(*_one_pair(xI, xJ, sizeI, sizeJ), _start_state(seed_or_state), maxIteration, precision)[0]


def geometricEstimation_H_AC(xI, xJ, sizeI, sizeJ, seed_or_state, maxIteration: int = 50000, precision: float = np.inf,
                             ctx: Context | None = None) -> dict:
    """GeometricFilterMatrix_H_AC::geometricEstimation of one pair on the GPU (arguments as geometricEstimation_F_AC).  Returns the
    dict of Context.acransac_homography_pairs: "H" and "mt_state_out", the generator advanced past this pair's draws, which the
    reference's single-threaded filter hands to the next pair."""
    ctx = ctx or default_context()
    return ctx.acransac_homography_pairs(*_one_pair(xI, xJ, sizeI, sizeJ), _start_state(seed_or_state), maxIteration, precision)[0]


def _start_state(seed_or_state) -> np.ndarray:
    """The caller's std::mt19937, given as a seed or as its 625-word state."""
    return mt19937_state(int(seed_or_state)) if np.ndim(seed_or_state) == 0 else np.ascontiguousarray(seed_or_state, np.uint32)


def _one_pair(xI, xJ, sizeI, sizeJ):
    """The correspondence list (one n x 4 array: xI, yI, xJ, yJ) and size list of a single pair's K10 call."""
    corr = np.concatenate([np.asarray(xI, np.float64).reshape(-1, 2), np.asarray(xJ, np.float64).reshape(-1, 2)], axis=1)
    return [corr], [tuple(sizeI) + tuple(sizeJ)]


# EImageDescriberType in enum order (feature/imageDescriberCommon.hpp:19-55): getCommonDescTypes returns the common types in this order
DESCRIBER_TYPES = ["sift", "sift_float", "sift_upright", "dspsift", "akaze", "akaze_liop", "akaze_mldb", "cctag3", "cctag4", "sift_ocv", "akaze_ocv",
                   "tag16h5"]
# feature::getStrongSupportCoeff (imageDescriberCommon.hpp:103-140)
STRONG_SUPPORT_COEFF = {t: 1.0 if t in ("cctag3", "cctag4", "tag16h5") else 0.14 for t in DESCRIBER_TYPES}


def copyInlierMatches(inliers, putatives_per_type: dict, desc_types) -> dict:
    """matchingImageCollection::copyInlierMatches (geometricFilterUtils.cpp:13-37): the inlier indices, sorted ascending, index the
    putative matches concatenated in `desc_types` order; each is copied (ratio and distance kept) into the list of its type.  Types
    without an inlier get no entry."""
    order = np.sort(np.asarray(inliers, np.int64))
    out, start = {}, 0
    for t in desc_types:
        m = putatives_per_type.get(t, np.zeros(0, MATCH_DTYPE))
        sel = order[(order >= start) & (order < start + len(m))] - start
        if sel.size:
            out[t] = m[sel].copy()
        start += len(m)
    return out


def hasStrongSupport(matches_per_type: dict, minimumSamples: int = 7) -> bool:
    """matching::hasStrongSupport(MatchesPerDescType, minimumSamples) (supportEstimation.cpp:48-59): the float sum over the types, in
    enum order, of getStrongSupportCoeff(type) * count must exceed minimumSamples (7 for Fundamental7PSolver)."""
    score = np.float32(0)
    for t in sorted(matches_per_type, key=DESCRIBER_TYPES.index):
        score = np.float32(score + np.float32(STRONG_SUPPORT_COEFF[t]) * np.float32(len(matches_per_type[t])))
    return bool(score > minimumSamples)


def robustModelEstimation_F_AC(putatives: dict, regions_per_view: dict, image_sizes: dict, seed_or_state, maxIteration: int = 50000,
                               precision: float = np.inf, guidedMatching: bool = False, distanceRatio: float = 0.6, geometry: dict | None = None,
                               guided_geometry: dict | None = None, desc_types=None, ctx: Context | None = None, bearings: dict | None = None,
                               chain: bool = False, estimateDistortion: bool = False):
    """matchingImageCollection::robustModelEstimation with GeometricFilterMatrix_F_AC (ACRANSAC, Fundamental7PSolver; GeometricFilter.hpp:40-88),
    the default `fundamental_matrix` filter of featureMatching, for a whole putative list: one a-contrario RANSAC call for every pair
    (b200m_acransac_fundamental_pairs), then, with guidedMatching, one guided-matching call for every kept pair and common descriptor
    type (b200m_guided_match_pairs).

    putatives        {(I, J): {describer type: matches[MATCH_DTYPE]}}
    regions_per_view {view: {describer type: Regions}}
    image_sizes      {view: (width, height)}
    seed_or_state    the caller's std::mt19937 (seed or 625-word state): every pair starts from it, as geometricEstimation_Mat_ACRANSAC
                     takes the generator by value (GeometricFilterMatrix_F_AC.hpp:271)
    geometry         optional {view: {type: n x 2 double}}: the undistorted positions of a view whose camera isValid() && hasDistortion()
                     (fillMatricesWithUndistortFeaturesMatches, geometricFilterUtils.hpp:36-66); otherwise the regions' positions
    guided_geometry  optional {view: {type: n x 2 double}}: getUndistortedPixel of every feature of a view whose camera isValid()
                     (guidedMatching.hpp:229-248), the positions guided matching uses
    desc_types       the describer types in EImageDescriberType order (default DESCRIBER_TYPES)
    bearings         optional {view: {type: n x 3 double}}: for a view whose camera is camera::Equidistant, the unit vector
                     toUnitSphere(removeDistortion(ima2cam(x))) of every feature, x its position as `geometry` gives it.  A pair whose
                     two views have bearings for every common type is spherical: it is estimated by geometricEstimation_Spherical_Mat
                     (GeometricFilterMatrix_F_AC.hpp:186-253, b200m_acransac_fundamental_spherical_pairs) on those vectors.  A view
                     with bearings for some but not all of a pair's common types is a ValueError.
    chain            the generator contract of spherical pairs, which take the std::mt19937 by reference:
                       False  every pair starts from the caller's state: one planar and one spherical K10 call for the whole list;
                       True   the single-threaded reference: a spherical pair starts where the previous spherical pair left the
                              generator and hands it on; each run of planar pairs between two of them is one planar call from the
                              current state.  Bit for bit the reference's run; meant for tests and short lists.
                     Without spherical pairs both give today's single planar call.
    estimateDistortion  GeometricFilterMatrix_F_AC's m_estimateDistortion, the `fundamental_with_distortion` filter: the planar
                     pairs are estimated by geometricEstimation_Mat_ACRANSAC<Fundamental10PSolver, Fundamental10PModel>
                     (b200m_acransac_fundamental_distortion_pairs), whose minimum sample count 10 is their hasStrongSupport threshold;
                     spherical pairs are estimated as without it (7).  Their "F" is the reference's model matrix, scored and
                     guided-matched as x_J^T F x_I while the solver fits it transposed with distortion (see
                     acransac_fundamental_distortion_pairs), and info gains "L" ((l1, l2) in preconditioned units, 0 for the
                     other pairs).  The filter itself does not use L.

    Returns (geometric matches {(I, J): {type: matches}} of the pairs with strong support, per-pair estimation
    {(I, J): {"valid", "strong_support", "F", "error_max", "spherical"}, plus "mt_state_out" for the spherical pairs estimated, and
    "L" with estimateDistortion}).
    Without guided matching the kept lists are the inlier putatives (ratio and distance kept); with it, the guided lists of every
    common type (empty ones included) replace them, or nothing when error_max is infinite (GeometricFilterMatrix_F_AC.hpp:363).  A
    spherical pair's guided matching uses its F and error_max on the guided positions, as the reference does."""
    ctx = ctx or default_context()
    common, est, corrs, whs = _estimation_inputs(putatives, regions_per_view, image_sizes, geometry, desc_types)
    sph = _spherical_inputs(putatives, regions_per_view, bearings or {}, common, est)
    planar = ctx.acransac_fundamental_distortion_pairs if estimateDistortion else ctx.acransac_fundamental_pairs
    calls = [(lambda ks, st: planar([corrs[k] for k in ks], [whs[k] for k in ks], st, maxIteration, precision), False),
             (lambda ks, st: ctx.acransac_fundamental_spherical_pairs([sph[est[k]] for k in ks], st, maxIteration, precision), True)]
    out, info = _acransac_stage(ctx, putatives, regions_per_view, guided_geometry, common, est, [int(p in sph) for p in est], calls, "F",
                                [10, 7] if estimateDistortion else 7, seed_or_state, chain, guidedMatching, distanceRatio,
                                lambda vp, items, Fs, th, ratio: ctx.guided_match_pairs(vp, Fs, th, ratio))
    for p, d in info.items():
        d["spherical"] = p in sph
        if estimateDistortion:
            d.setdefault("L", np.zeros(2))
    return out, info


def _estimation_inputs(putatives: dict, regions_per_view: dict, image_sizes: dict, geometry: dict | None, desc_types):
    """Each pair's common describer types (EImageDescriberType order), the pairs that have one, and for those the correspondences of
    fillMatricesWithUndistortFeaturesMatches (n x 4: xI, yI, xJ, yJ, types concatenated in order) and image sizes."""
    order = list(desc_types) if desc_types is not None else DESCRIBER_TYPES
    geometry = geometry or {}
    common = {p: [t for t in order if t in regions_per_view[p[0]] and t in regions_per_view[p[1]]] for p in putatives}

    def positions(v, t):
        g = geometry.get(v, {}).get(t)
        return np.asarray(g, np.float64).reshape(-1, 2) if g is not None else regions_per_view[v][t].positions.astype(np.float64)

    est = [p for p in putatives if common[p]]                 # no common type: EstimationStatus(false, false)
    corrs, whs = [], []
    for I, J in est:
        parts = [np.zeros((0, 4))]
        for t in common[(I, J)]:
            m = putatives[(I, J)].get(t)
            if m is not None and len(m):
                parts.append(np.concatenate([positions(I, t)[m["i"]], positions(J, t)[m["j"]]], axis=1))
        corrs.append(np.concatenate(parts))
        whs.append(tuple(image_sizes[I]) + tuple(image_sizes[J]))
    return common, est, corrs, whs


def _spherical_inputs(putatives: dict, regions_per_view: dict, bearings: dict, common: dict, est) -> dict:
    """{pair: n x 6 bearing pairs (xI, yI, zI, xJ, yJ, zJ), types concatenated in order} for the estimated pairs whose two views
    have bearings for every common type (the rows of _estimation_inputs' correspondences, lifted)."""
    out = {}
    for I, J in est:
        types = common[(I, J)]
        have = [[t in bearings.get(v, {}) for t in types] for v in (I, J)]
        for v, h in zip((I, J), have):
            if any(h) and not all(h):
                raise ValueError(f"bearings of view {v}: some but not all of the common types {types} of pair {(I, J)}")
        if not all(have[0]) or not all(have[1]):
            continue
        parts = [np.zeros((0, 6))]
        for t in types:
            bI, bJ = (np.asarray(bearings[v][t], np.float64).reshape(-1, 3) for v in (I, J))
            for v, b in ((I, bI), (J, bJ)):
                if b.shape[0] != regions_per_view[v][t].RegionCount():
                    raise ValueError(f"bearings of view {v}, type {t}: {b.shape[0]} vectors for {regions_per_view[v][t].RegionCount()} features")
            m = putatives[(I, J)].get(t)
            if m is not None and len(m):
                parts.append(np.concatenate([bI[m["i"]], bJ[m["j"]]], axis=1))
        out[(I, J)] = np.concatenate(parts)
    return out


def _guided_stage(ctx: Context, out: dict, info: dict, common: dict, regions_per_view: dict, guided_geometry: dict | None, run) -> None:
    """The guided-matching step of a geometric filter stage: every kept pair's lists are replaced by one entry per common type (empty
    ones included) when its error_max is finite, else by nothing.  The views of those pairs are uploaded once per (view, type), with
    their guided positions, and run(view_pairs, items) makes the one batched call over items = [(pair, type)]."""
    guided = [p for p in out if np.isfinite(info[p]["error_max"])]
    for p in out:
        out[p] = {}
    ids, up = {}, []
    try:
        for I, J in guided:
            for t in common[(I, J)]:
                for v in (I, J):
                    if (v, t) not in ids:
                        ids[(v, t)] = _new_view_id()
                        xy = (guided_geometry or {}).get(v, {}).get(t)
                        _upload_pair(ctx, [ids[(v, t)]], [regions_per_view[v][t]], [xy], up)
        items = [(p, t) for p in guided for t in common[p]]
        lists = run([(ids[(p[0], t)], ids[(p[1], t)]) for p, t in items], items) if items else []
        for (p, t), m in zip(items, lists):
            out[p][t] = m
    finally:
        for vid in up:
            ctx.lib.b200m_remove_view(ctx._h, C.c_uint32(vid))


def _acransac_stage(ctx: Context, putatives: dict, regions_per_view: dict, guided_geometry: dict | None, common: dict, est: list, groups: list,
                    calls: list, key: str, min_samples: int, seed_or_state, chain: bool, guidedMatching: bool, distanceRatio: float, guided):
    """The stage rules the a-contrario filters share (robustModelEstimation around GeometricFilterMatrix_F_AC, _H_AC and _E_AC), over
    the estimated pairs `est` in putative-list order.
      groups, calls  pair k goes through calls[groups[k]] = (run(ks, state) -> the results of pairs ks, by_reference), by_reference
                     the generator contract of its geometricEstimation.  chain=False: one call per group from the caller's state, in
                     `calls` order.  chain=True: in list order, a by-reference pair alone, handing its mt_state_out to the next call,
                     and each run of by-value pairs of one group in one call from the current state.
      key            the model's name in the results and in info; min_samples: the solver's getMinimumNbRequiredSamples, one for
                     every group or a list with one per group (the hasStrongSupport threshold of the group's pairs)
      guided         guided(view_pairs, items, models, errorTh, distRatio): the batched guided call over items = [(pair, type)],
                     with errorTh = error_max^2 and distRatio = distanceRatio^2
    ACRANSAC's validity comes before support.  Returns (out, info) as robustModelEstimation_H_AC describes them, "mt_state_out"
    on the pairs whose call returned one."""
    st = _start_state(seed_or_state)
    if chain:
        segments = [list(ks) for _, ks in itertools.groupby(range(len(est)), lambda k: (groups[k], k if calls[groups[k]][1] else -1))]
    else:
        segments = [ks for g in range(len(calls)) if (ks := [k for k, h in enumerate(groups) if h == g])]
    res = [None] * len(est)
    for ks in segments:
        run, by_reference = calls[groups[ks[0]]]
        for k, r in zip(ks, run(ks, st)):
            res[k] = r
        if chain and by_reference:
            st = res[ks[0]]["mt_state_out"]
    info = {p: {"valid": False, "strong_support": False, key: np.zeros((3, 3)), "error_max": np.inf} for p in putatives}
    out = {}
    for p, g, r in zip(est, groups, res):
        info[p].update({"valid": r["valid"], key: r[key], "error_max": r["error_max"]})
        for extra in ("mt_state_out", "L"):
            if extra in r:
                info[p][extra] = r[extra]
        if not r["valid"]:
            continue
        inl = copyInlierMatches(r["inliers"], putatives[p], common[p])
        info[p]["strong_support"] = hasStrongSupport(inl, min_samples[g] if isinstance(min_samples, (list, tuple)) else min_samples)
        if info[p]["strong_support"]:
            out[p] = inl
    if guidedMatching and out:
        _guided_stage(ctx, out, info, common, regions_per_view, guided_geometry,
                      lambda vp, items: guided(vp, items, [info[p][key] for p, _ in items],
                                               [info[p]["error_max"] * info[p]["error_max"] for p, _ in items], distanceRatio * distanceRatio))
    return out, info


def robustModelEstimation_H_AC(putatives: dict, regions_per_view: dict, image_sizes: dict, seed_or_state, maxIteration: int = 50000,
                               precision: float = np.inf, guidedMatching: bool = False, distanceRatio: float = -1.0, geometry: dict | None = None,
                               guided_geometry: dict | None = None, desc_types=None, chain: bool = False, ctx: Context | None = None):
    """matchingImageCollection::robustModelEstimation with GeometricFilterMatrix_H_AC (ACRANSAC, Homography4PSolver, point-to-point
    error; GeometricFilterMatrix_H_AC.hpp:43-103), the `homography_matrix` filter of featureMatching, for a whole putative list: a-contrario
    RANSAC for every pair (b200m_acransac_homography_pairs), copyInlierMatches and hasStrongSupport(.., 4); then, with guidedMatching,
    one guided-matching call for every kept pair with a finite error_max and every common type, errorTh = error_max^2:
      distanceRatio < 0   position-only guidedMatching + IndMatchDecorator (b200m_guided_match_positions_pairs), what featureMatching
                          runs (it passes distanceRatio = -1 with --guidedMatching)
      distanceRatio >= 0  guidedMatching with descriptors and distRatio = distanceRatio^2 (b200m_guided_match_pairs, homography model)

    Arguments as robustModelEstimation_F_AC, except the generator contract.  geometricEstimation takes the std::mt19937 by reference, so
    the reference's filter hands one generator from pair to pair; under featureMatching's OpenMP loop every thread draws from it without
    synchronisation, and no run is reproducible.
      chain=False  every pair starts from the caller's state (as the F stage does): deterministic, one K10 call for the whole list.
      chain=True   the single-threaded reference: K10 runs one pair per call in putative-list order, each starting from the state the
                   previous pair left (pairs without a common type draw nothing).  Bit for bit the reference's run; meant for tests and
                   short lists.

    Returns (geometric matches {(I, J): {type: matches}} of the pairs with strong support, per-pair estimation
    {(I, J): {"valid", "strong_support", "H", "error_max"}, plus "mt_state_out" for the estimated pairs}).  The kept lists are as in
    robustModelEstimation_F_AC; the position-only guided lists are in the decorator's order (ratio and distance 0)."""
    ctx = ctx or default_context()
    common, est, corrs, whs = _estimation_inputs(putatives, regions_per_view, image_sizes, geometry, desc_types)

    def guided(vp, items, Hs, th, ratio):
        if distanceRatio < 0:
            return ctx.guided_match_positions_pairs(vp, Hs, th, MODEL_HOMOGRAPHY, decorate=True)
        return ctx.guided_match_pairs(vp, Hs, th, ratio, MODEL_HOMOGRAPHY)
    calls = [(lambda ks, st: ctx.acransac_homography_pairs([corrs[k] for k in ks], [whs[k] for k in ks], st, maxIteration, precision), True)]
    return _acransac_stage(ctx, putatives, regions_per_view, guided_geometry, common, est, [0] * len(est), calls, "H", 4, seed_or_state,
                           chain, guidedMatching, distanceRatio, guided)


def geometricEstimation_E_AC(xI, xJ, sizeI, sizeJ, KI, KJ, seed_or_state, maxIteration: int = 50000, precision: float = np.inf,
                             ctx: Context | None = None) -> dict:
    """GeometricFilterMatrix_E_AC::geometricEstimation's ACRANSAC of one pair on the GPU: arguments as geometricEstimation_F_AC plus
    the two pinhole matrices K (3 x 3); `precision` is what the filter passes to ACRANSAC, Square(m_dPrecision).  Returns the dict of
    Context.acransac_essential_pairs ("E", "mt_state_out")."""
    ctx = ctx or default_context()
    K = np.concatenate([np.asarray(KI, np.float64).reshape(9), np.asarray(KJ, np.float64).reshape(9)])
    return ctx.acransac_essential_pairs(*_one_pair(xI, xJ, sizeI, sizeJ), [K], _start_state(seed_or_state), maxIteration, precision)[0]


def _inverse3(M) -> np.ndarray:
    """The engine's 3 x 3 inverse (acr::inverse3): cofactors over the determinant expanded along the first column."""
    M = np.asarray(M, np.float64).reshape(3, 3)
    C_ = np.empty((3, 3))
    for i in range(3):
        for j in range(3):
            i1, i2, j1, j2 = (i + 1) % 3, (i + 2) % 3, (j + 1) % 3, (j + 2) % 3
            C_[i, j] = M[i1, j1] * M[i2, j2] - M[i1, j2] * M[i2, j1]
    inv = 1.0 / ((C_[0, 0] * M[0, 0] + C_[1, 0] * M[1, 0]) + C_[2, 0] * M[2, 0])
    return C_.T * inv


def fundamentalFromEssential(E, KI, KJ) -> np.ndarray:
    """multiview::fundamentalFromEssential: F = K_J^-T E K_I^-1, formed as (K_J^-T E) K_I^-1 with the engine's inverses, each entry
    summed in index order (the C++ adaptor's and acr::fundamental_from_essential's arithmetic)."""
    E, iI, iJ = np.asarray(E, np.float64).reshape(3, 3), _inverse3(KI), _inverse3(KJ)
    T = (iJ[0][:, None] * E[0] + iJ[1][:, None] * E[1]) + iJ[2][:, None] * E[2]      # T[r, c] = sum_k iJ[k, r] E[k, c], k in order
    return (T[:, 0:1] * iI[0] + T[:, 1:2] * iI[1]) + T[:, 2:3] * iI[2]


def robustModelEstimation_E_AC(putatives: dict, regions_per_view: dict, image_sizes: dict, intrinsics: dict, seed_or_state,
                               maxIteration: int = 50000, precision: float = np.inf, guidedMatching: bool = False, distanceRatio: float = 0.6,
                               geometry: dict | None = None, guided_geometry: dict | None = None, desc_types=None, chain: bool = False,
                               ctx: Context | None = None):
    """matchingImageCollection::robustModelEstimation with GeometricFilterMatrix_E_AC (ACRANSAC, Essential5PSolver;
    GeometricFilterMatrix_E_AC.hpp), the `essential_matrix` filter of featureMatching, for a whole putative list: a-contrario RANSAC
    for every estimated pair (b200m_acransac_essential_pairs), copyInlierMatches and hasStrongSupport(.., 5); then, with guidedMatching,
    one guided-matching call (b200m_guided_match_pairs) for every kept pair with a finite error_max and every common type, with
    F = K_J^-T E K_I^-1, errorTh = error_max^2 and distRatio = distanceRatio^2.  featureMatching then applies
    removePoorlyOverlappingImagePairs to the result.

    intrinsics  {view: 3 x 3 K of its camera::Pinhole (equidistant cameras included), or None for a missing or non-pinhole intrinsic}.
                A pair is not estimated (EstimationStatus(false, false)) without a common describer type, or when either view has no
                pinhole K.
    precision   the filter's m_dPrecision (geometricErrorMax; +inf = none): the filter passes Square(precision) to ACRANSAC, which
                squares it again, so the residual threshold is precision^4, as in the reference.
    Other arguments as robustModelEstimation_H_AC, the generator contract (chain) included.

    Returns (geometric matches {(I, J): {type: matches}} of the pairs with strong support, per-pair estimation
    {(I, J): {"valid", "strong_support", "E", "error_max"}, plus "mt_state_out" for the estimated pairs})."""
    ctx = ctx or default_context()
    common, est, corrs, whs = _estimation_inputs(putatives, regions_per_view, image_sizes, geometry, desc_types)
    Ks = {p: [intrinsics.get(v) for v in p] for p in est}
    keep = [k for k, p in enumerate(est) if all(K is not None for K in Ks[p])]
    est, corrs, whs = [est[k] for k in keep], [corrs[k] for k in keep], [whs[k] for k in keep]
    Kp = [np.concatenate([np.asarray(K, np.float64).reshape(9) for K in Ks[p]]) for p in est]
    upper = precision * precision   # upperBoundPrecision = Square(m_dPrecision)
    calls = [(lambda ks, st: ctx.acransac_essential_pairs([corrs[k] for k in ks], [whs[k] for k in ks], [Kp[k] for k in ks], st, maxIteration,
                                                          upper), True)]
    return _acransac_stage(ctx, putatives, regions_per_view, guided_geometry, common, est, [0] * len(est), calls, "E", 5, seed_or_state,
                           chain, guidedMatching, distanceRatio,
                           lambda vp, items, Es, th, ratio: ctx.guided_match_pairs(
                               vp, [fundamentalFromEssential(E, *Ks[p]) for (p, _), E in zip(items, Es)], th, ratio))


def removePoorlyOverlappingImagePairs(geometric: dict, putatives: dict, minimumRatio: float = 0.3, minimumGeometricCount: int = 50) -> dict:
    """matchingImageCollection::removePoorlyOverlappingImagePairs (GeometricFilter.cpp:12-34): a pair of `geometric` is removed when
    its match count (all types) is below minimumGeometricCount, or when that count over its putative count, divided in float, is below
    minimumRatio (a float).  Returns the kept pairs."""
    out = {}
    for p, m in geometric.items():
        g = sum(len(v) for v in m.values())
        n = sum(len(v) for v in putatives[p].values())
        if g < minimumGeometricCount or np.float32(g) / np.float32(n) < np.float32(minimumRatio):
            continue
        out[p] = m
    return out


# GrowParameters / HGrowingFilteringParam defaults (GeometricFilterMatrix_HGrowing.hpp:23-106); featureMatching never changes them
HGROWING_DEFAULTS = dict(similarityTolerance=20.0, affinityTolerance=10.0, homographyTolerance=5.0, minInliersToRefine=6,
                         nbRefiningIterations=8, maxNbHomographies=10, minNbMatchesPerH=20)
# describer types whose presence among a pair's common types drops the pair (GeometricFilterMatrix_HGrowing.hpp, CCTag / AprilTag builds)
HGROWING_TAG_TYPES = ("cctag3", "cctag4", "tag16h5")


def _hgrowing_item(featuresI, featuresJ, matches) -> np.ndarray:
    fi = np.asarray(featuresI, np.float32).reshape(-1, 4)
    fj = np.asarray(featuresJ, np.float32).reshape(-1, 4)
    return np.ascontiguousarray(np.concatenate([fi[matches["i"]], fj[matches["j"]]], axis=1), np.float32)


def _hgrowing_split(r: dict, matches: np.ndarray):
    bounds = np.concatenate([[0], np.cumsum(r["counts"])]).astype(np.int64)
    return [(r["H"][k], matches[r["inliers"][bounds[k]:bounds[k + 1]]]) for k in range(len(r["counts"]))], matches[r["inliers"]]


def filterMatchesByHGrowing(featuresI, featuresJ, putatives, param: dict | None = None, ctx: Context | None = None):
    """filterMatchesByHGrowing (GeometricFilterMatrix_HGrowing.cpp:108-194) of one putative list on the GPU.  featuresI / featuresJ:
    n x 4 float32 PointFeatures (x, y, scale, orientation); putatives: matches[MATCH_DTYPE] (or any array with "i" and "j" fields) in
    the order the filter walks them.  Returns (homographiesAndMatches: [(H 3 x 3, matches)], outGeometricInliers)."""
    ctx = ctx or default_context()
    r = ctx.hgrowing_pairs([_hgrowing_item(featuresI, featuresJ, putatives)], param)[0]
    return _hgrowing_split(r, putatives)


def robustModelEstimation_HGrowing(putatives: dict, features_per_view: dict, guidedMatching: bool = False, param: dict | None = None,
                                   desc_types=None, ctx: Context | None = None):
    """matchingImageCollection::robustModelEstimation with GeometricFilterMatrix_HGrowing (the `homography_growing` filter of
    featureMatching) for a whole putative list, with one engine call for every (pair, describer type):
      putatives          {(I, J): {describer type: matches[MATCH_DTYPE]}}, used in the caller's order (featureMatching sorts each list
                         by Lowe ratio first: matches_filtering.sortMatches_byDistanceRatio)
      features_per_view  {view: {describer type: n x 4 float32 (x, y, scale, orientation)}}, as regions_io.loadFeatsFromFile returns them
    The stage rules of geometricEstimation (GeometricFilterMatrix_HGrowing.hpp:176-266): every common type with a putative entry is
    filtered and gets an entry, even an empty one, and such a pair is kept; a pair with a CCTag or AprilTag type among its common types
    is dropped; with guidedMatching the kept pair's lists become an empty map (Geometry_guided_matching is an empty stub).
    Returns (geometric matches {(I, J): {type: matches}}, {(I, J): {type: [(H, matches)]}} like the reference's _HsAndMatchesPerDesc)."""
    ctx = ctx or default_context()
    order = list(desc_types) if desc_types is not None else DESCRIBER_TYPES
    work, items = [], []
    for (I, J), per_type in putatives.items():
        common = [t for t in order if t in features_per_view[I] and t in features_per_view[J]]
        if any(t in HGROWING_TAG_TYPES for t in common):
            continue
        for t in common:
            if t in per_type:
                work.append(((I, J), t))
                items.append(_hgrowing_item(features_per_view[I][t], features_per_view[J][t], per_type[t]))
    res = ctx.hgrowing_pairs(items, param) if items else []
    out, hs = {}, {}
    for (p, t), r in zip(work, res):
        m = putatives[p][t]
        h_list, inl = _hgrowing_split(r, m)
        hs.setdefault(p, {})[t] = h_list
        out.setdefault(p, {})
        if not guidedMatching:
            out[p][t] = inl
    return out, hs


_default_ctx: dict[int, Context] = {}


def default_context(device: int = 0) -> Context:
    if device not in _default_ctx:
        _default_ctx[device] = Context(device)
    return _default_ctx[device]


class _ResultOwner:
    """Owns one b200m_result; freed when the last numpy view onto it is garbage collected."""

    def __init__(self, lib, handle):
        self.lib, self.handle = lib, handle

    def __del__(self):
        try:
            if self.handle:
                self.lib.b200m_result_free(self.handle)
                self.handle = None
        except Exception:
            pass


def _alias(addr, nbytes: int, dtype, owner) -> np.ndarray:
    """Zero-copy numpy view of engine-owned memory (keeps `owner` alive through the buffer object)."""
    if not addr or nbytes <= 0:
        return np.zeros(0, dtype)
    buf = (C.c_uint8 * nbytes).from_address(addr)
    buf._owner = owner
    return np.frombuffer(buf, dtype=dtype)


class ArrayMatcherB200:
    """Mirror of matching::ArrayMatcher (Build / SearchNeighbour / SearchNeighbours), bool returns, no exceptions
    on the matcher surface (ArrayMatcher_bruteForce.hpp:42-51,63-85,98-142)."""

    def __init__(self, metric: int = L2_SIMPLE, ctx: Context | None = None, binary: bool = False):
        self.ctx = ctx or default_context()
        self.metric = HAMMING if binary else metric
        self.binary = binary
        self._db = C.c_void_p()
        self._dim = 0
        self._dtype = None

    def Build(self, dataset: np.ndarray, nbRows: int | None = None, dimension: int | None = None) -> bool:
        self._release()
        a = np.ascontiguousarray(dataset)
        rows = a.shape[0] if nbRows is None else nbRows
        dim = (a.shape[1] if a.ndim == 2 else 0) if dimension is None else dimension
        if rows < 1:
            return False
        rc = self.ctx.lib.b200m_db_create(self.ctx._h, a.ctypes.data_as(C.c_void_p), C.c_int(rows), C.c_int(dim),
                                          C.c_int(_dtype_code(a, self.binary)), C.c_int(self.metric), C.byref(self._db))
        self._dim, self._dtype = dim, a.dtype
        return rc == 0

    def SearchNeighbours(self, query: np.ndarray, nbQuery: int | None = None, NN: int = 2):
        """Returns (ok, indices[nq,NN] int32 database rows, distances[nq,NN] float32|uint32)."""
        q = np.ascontiguousarray(query, dtype=self._dtype) if self._dtype is not None else np.ascontiguousarray(query)
        nq = (q.shape[0] if q.ndim == 2 else (1 if q.size else 0)) if nbQuery is None else nbQuery
        idx = np.zeros((max(nq, 1), NN), np.int32)
        dist = np.zeros((max(nq, 1), NN), np.uint32 if self.metric == HAMMING else np.float32)
        if not self._db:
            return False, idx[:0], dist[:0]
        rc = self.ctx.lib.b200m_knn(self.ctx._h, self._db, q.ctypes.data_as(C.c_void_p), C.c_int(nq), C.c_int(NN),
                                    idx.ctypes.data_as(C.c_void_p), dist.ctypes.data_as(C.c_void_p))
        if rc != 0:
            return False, idx[:0], dist[:0]
        return True, idx[:nq], dist[:nq]

    def SearchNeighbour(self, query: np.ndarray):
        """Single nearest neighbour: returns (ok, index, distance)."""
        ok, idx, dist = self.SearchNeighbours(np.ascontiguousarray(query).reshape(1, -1), 1, 1)
        if not ok:
            return False, -1, -1.0
        return True, int(idx[0, 0]), dist[0, 0]

    def _release(self):
        if self._db:
            self.ctx.lib.b200m_db_destroy(self._db)
            self._db = C.c_void_p()

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass


def shard_pairs(pairs, n_shards: int) -> np.ndarray:
    """b200m_shard_pairs: shard index of every pair (database images dealt round-robin, alternating direction). Host only."""
    p = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
    out = np.zeros(max(p.shape[0], 1), np.int32)
    _check(load_library().b200m_shard_pairs(p.ctypes.data_as(C.c_void_p), C.c_int(p.shape[0]), C.c_int(n_shards), out.ctypes.data_as(C.c_void_p)),
           "b200m_shard_pairs")
    return out[: p.shape[0]]


def shard_pairs_2d(pairs, n_shards: int) -> np.ndarray:
    """b200m_shard_pairs_2d: shard index of every pair with 2-D block sharding (a shard needs only part of the views). Host only."""
    p = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
    out = np.zeros(max(p.shape[0], 1), np.int32)
    _check(load_library().b200m_shard_pairs_2d(p.ctypes.data_as(C.c_void_p), C.c_int(p.shape[0]), C.c_int(n_shards), out.ctypes.data_as(C.c_void_p)),
           "b200m_shard_pairs_2d")
    return out[: p.shape[0]]


class MultiContext:
    """``b200m_multi``: one engine context per device, driven by one host thread each (single-process multi-GPU)."""

    def __init__(self, devices):
        self.lib = load_library()
        self.devices = [int(d) for d in devices]
        self._h = C.c_void_p()
        arr = (C.c_int * len(self.devices))(*self.devices)
        _check(self.lib.b200m_multi_create(arr, C.c_int(len(self.devices)), C.byref(self._h)), "b200m_multi_create")

    def close(self) -> None:
        if self._h:
            self.lib.b200m_multi_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def last_gpu_ms(self) -> float: return self.lib.b200m_multi_last_gpu_ms(self._h)

    def exactness_errors(self) -> int:
        return sum(self.lib.b200m_exactness_errors(C.c_void_p(self.lib.b200m_multi_ctx(self._h, C.c_int(k)))) for k in range(len(self.devices)))


class ImageCollectionMatcherB200:
    """Mirror of IImageCollectionMatcher / ImageCollectionMatcher_generic (distRatio, crossMatching, matcherType).
    ``devices``: several CUDA ordinals -> the pair list is sharded over one context per device inside this process."""

    def __init__(self, distRatio: float = 0.8, crossMatching: bool = False, matcherType: EMatcherType = EMatcherType.BRUTE_FORCE_L2_B200,
                 ctx: Context | None = None, devices=None):
        if matcherType not in (EMatcherType.BRUTE_FORCE_L2_B200, EMatcherType.BRUTE_FORCE_HAMMING_B200, EMatcherType.BRUTE_FORCE_L2,
                               EMatcherType.BRUTE_FORCE_HAMMING):
            raise IndexError("Invalid matcherType enum")    # matchingCommon.cpp:41-42 throws std::out_of_range
        self.multi = MultiContext(devices) if devices is not None and len(devices) > 1 else None
        self.ctx = ctx or (default_context(devices[0] if devices else 0) if self.multi is None else None)
        self.distRatio, self.crossMatching, self.matcherType = float(distRatio), bool(crossMatching), matcherType
        self.hamming = matcherType in (EMatcherType.BRUTE_FORCE_HAMMING_B200, EMatcherType.BRUTE_FORCE_HAMMING)
        self._keepalive = []      # descriptor arrays of asynchronous uploads still in flight

    def upload(self, regionsPerView: dict) -> None:
        """regionsPerView: {viewId: (descriptors[n,dim], positions[n,2] or None)} for ONE descriptor type.
        Asynchronous (b200m_upload_views_async): the copies overlap the first batches of the next match call; the
        descriptor arrays are kept alive here until that call (or clear / wait_uploads) returns."""
        lib = self.ctx.lib
        groups = {}                                   # one bulk call per (dim, element type)
        for vid, (desc, xy) in regionsPerView.items():
            d = np.ascontiguousarray(desc)
            dim = d.shape[1] if d.ndim == 2 else 0
            binary = d.dtype == np.uint8 and self.hamming
            xya = None if xy is None else np.ascontiguousarray(xy, np.float32)
            groups.setdefault((max(dim, 1), _dtype_code(d, binary)), []).append((vid, d, xya))
        for (dim, code), items in groups.items():
            n = len(items)
            ids = np.array([v for v, _, _ in items], np.uint32)
            counts = np.array([d.shape[0] for _, d, _ in items], np.int32)
            dptr = (C.c_void_p * n)(*[d.ctypes.data if d.shape[0] else None for _, d, _ in items])
            have_xy = any(x is not None for _, _, x in items)
            xptr = (C.c_void_p * n)(*[(x.ctypes.data if x is not None and x.size else None) for _, _, x in items]) if have_xy else None
            self._keepalive.append(items)
            _check(lib.b200m_upload_views_async(self.ctx._h, C.c_int(n), ids.ctypes.data_as(C.c_void_p), dptr, counts.ctypes.data_as(C.c_void_p),
                                                C.c_int(dim), C.c_int(code), xptr), "b200m_upload_views_async")

    def wait_uploads(self) -> None:
        try:
            _check(self.ctx.lib.b200m_wait_uploads(self.ctx._h), "b200m_wait_uploads")
        finally:
            self._keepalive.clear()

    def clear(self) -> None:
        try:
            _check(self.ctx.lib.b200m_clear_views(self.ctx._h), "b200m_clear_views")
        finally:
            self._keepalive.clear()

    def match_uploaded(self, pairs, stage: int = STAGE_FULL):
        """Runs b200m_match_pairs on already-uploaded views. Returns (pair_ids[n,2], offsets[n+1], matches[MATCH_DTYPE])."""
        lib = self.ctx.lib
        p = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
        res = C.c_void_p()
        try:
            _check(lib.b200m_match_pairs(self.ctx._h, p.ctypes.data_as(C.c_void_p), C.c_int(p.shape[0]), C.c_float(self.distRatio),
                                         C.c_int(int(self.crossMatching)), C.c_int(stage), C.byref(res)), "b200m_match_pairs")
        finally:
            self._keepalive.clear()      # b200m_match_pairs returns after every pending upload has left caller memory
        return self._wrap_result(lib, res)

    def _wrap_result(self, lib, res):
        owner = _ResultOwner(lib, res)      # the numpy arrays below alias the result's memory; it is freed when they die
        n = lib.b200m_result_num_pairs(res)
        pid, off, mat = C.c_void_p(), C.c_void_p(), C.c_void_p()
        _check(lib.b200m_result_get(res, C.byref(pid), C.byref(off), C.byref(mat)), "b200m_result_get")
        offsets = _alias(off.value, (n + 1) * 8, np.int64, owner)
        pair_ids = _alias(pid.value, n * 8, np.uint32, owner).reshape(-1, 2)
        matches = _alias(mat.value, int(offsets[-1]) * MATCH_DTYPE.itemsize, MATCH_DTYPE, owner)
        return pair_ids, offsets, matches

    def _match_multi(self, regionsPerView: dict, pairs):
        """b200m_multi_match: all views of ONE element type, pair list sharded over the devices."""
        lib = self.multi.lib
        items = []
        for vid, (desc, xy) in regionsPerView.items():
            d = np.ascontiguousarray(desc)
            items.append((vid, d, None if xy is None else np.ascontiguousarray(xy, np.float32)))
        codes = {(_dtype_code(d, d.dtype == np.uint8 and self.hamming), d.shape[1] if d.ndim == 2 else 0) for _, d, _ in items}
        if len(codes) == 0:      # nothing referenced (empty pair list): the empty result
            return np.zeros((0, 2), np.uint32), np.zeros(1, np.int64), np.zeros(0, MATCH_DTYPE)
        if len(codes) != 1:
            raise B200MatchError("the multi-device path takes views of one descriptor type per call")
        (code, dim), = codes
        n = len(items)
        ids = np.array([v for v, _, _ in items], np.uint32)
        counts = np.array([d.shape[0] for _, d, _ in items], np.int32)
        dptr = (C.c_void_p * n)(*[d.ctypes.data if d.shape[0] else None for _, d, _ in items])
        xptr = (C.c_void_p * n)(*[(x.ctypes.data if x is not None and x.size else None) for _, _, x in items])
        p = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
        res = C.c_void_p()
        _check(lib.b200m_multi_match(self.multi._h, C.c_int(n), ids.ctypes.data_as(C.c_void_p), dptr, counts.ctypes.data_as(C.c_void_p), C.c_int(max(dim, 1)),
                                     C.c_int(code), xptr, p.ctypes.data_as(C.c_void_p), C.c_int(p.shape[0]), C.c_float(self.distRatio),
                                     C.c_int(int(self.crossMatching)), C.byref(res)), "b200m_multi_match")
        return self._wrap_result(lib, res)

    def Match(self, regionsPerView: dict, pairs, map_PutativesMatches: dict | None = None) -> dict:
        """IImageCollectionMatcher::Match: appends {(I, J): matches} for every pair with a non-empty result
        (ImageCollectionMatcher_generic.cpp:116-119: empty lists are not inserted; the output map is appended to).
        Only the regions the pair list references are touched (the reference calls getRegions for those only, :55,:72).
        Without an output map the result is a ``PairwiseMatches`` mapping (a dict view onto the engine's result arrays)."""
        p = np.ascontiguousarray(pairs, np.uint32).reshape(-1, 2)
        used = set(np.unique(p).tolist())
        needed = {v: r for v, r in regionsPerView.items() if v in used} if len(used) < len(regionsPerView) else regionsPerView
        if self.multi is not None:
            pair_ids, offsets, matches = self._match_multi(needed, p)
        else:
            self.upload(needed)
            pair_ids, offsets, matches = self.match_uploaded(p, STAGE_FULL)
        res = PairwiseMatches(pair_ids, offsets, matches)
        if map_PutativesMatches is None:
            return res
        map_PutativesMatches.update(res)
        return map_PutativesMatches


class PairwiseMatches(dict):
    """{(I, J): matches[MATCH_DTYPE]} of one Match call for the pairs with a non-empty result, in PairSet order
    (matching::PairwiseMatches, matching/IndMatch.hpp:148).  A dict whose entries are views into the engine's result arena;
    the entries are materialised on first access, so a caller that only forwards the arrays (``pair_ids``, ``offsets``,
    ``matches``: all pairs, CSR layout) pays nothing for the map."""

    def __init__(self, pair_ids, offsets, matches):
        super().__init__()
        self.pair_ids, self.offsets, self.matches = pair_ids, offsets, matches
        self._filled = False

    def _fill(self):
        if not self._filled:
            self._filled = True
            offs = self.offsets.tolist()
            m = self.matches
            for (i, j), a, b in zip(self.pair_ids.tolist(), offs[:-1], offs[1:]):
                if b > a:
                    dict.__setitem__(self, (i, j), m[a:b])
        return self

    def num_matches(self) -> int:
        return int(self.offsets[-1]) if len(self.offsets) else 0


def _lazy(name):
    def f(self, *a, **k):
        return getattr(dict, name)(self._fill(), *a, **k)
    f.__name__ = name
    return f


for _n in ("__getitem__", "__contains__", "__iter__", "__len__", "__eq__", "__ne__", "__repr__", "keys", "values", "items", "get", "copy", "__bool__",
           "pop", "__setitem__", "__delitem__", "setdefault", "update", "__reversed__", "__or__", "__ror__"):
    if hasattr(dict, _n):
        setattr(PairwiseMatches, _n, _lazy(_n))
PairwiseMatches.__bool__ = lambda self: len(self) > 0
PairwiseMatches.__hash__ = None


def _upload_pair(ctx: Context, ids, regions, geometry, up: list) -> None:
    """Uploads two Regions (and their geometry positions, when given) under `ids`; appends each uploaded id to `up`."""
    lib = ctx.lib
    for vid, r, xy in zip(ids, regions, geometry):
        n = r.RegionCount()
        code = _dtype_code(r.descriptors, r.binary)
        _check(lib.b200m_upload_view(ctx._h, C.c_uint32(vid), r.descriptors.ctypes.data_as(C.c_void_p) if n else None, C.c_int(n),
                                     C.c_int(max(r.DescriptorLength(), 1)), C.c_int(code), r.positions.ctypes.data_as(C.c_void_p) if n else None), "b200m_upload_view")
        up.append(vid)
        if xy is not None:
            ctx.set_view_geometry(vid, xy)


def guidedMatching(F, regions_left: "Regions", regions_right: "Regions", errorTh: float, distRatio: float, ctx: Context | None = None,
                   model: int = MODEL_FUNDAMENTAL, xy_left=None, xy_right=None) -> np.ndarray:
    """matching::guidedMatching<Mat3Model, FundamentalEpipolarDistanceError> (matching/guidedMatching.hpp:206-268): F = 3x3
    fundamental matrix (x_right^T F x_left = 0), errorTh / distRatio already squared as at the call site
    (GeometricFilterMatrix_F_AC.hpp:387-388).  model = MODEL_HOMOGRAPHY: F is a homography and the error is
    HomographyAsymmetricError (GeometricFilterMatrix_H_AC.hpp:217-225).  xy_left / xy_right: optional n x 2 double positions used
    instead of the regions' positions - the undistorted pixels the reference matches on when the camera is valid (:229-248).
    Returns matches[MATCH_DTYPE] with i = left, j = right feature."""
    ctx = ctx or default_context()
    lib = ctx.lib
    ids = (_new_view_id(), _new_view_id())
    Fm = np.ascontiguousarray(F, np.float64).reshape(9)
    up = []
    try:
        _upload_pair(ctx, ids, (regions_left, regions_right), (xy_left, xy_right), up)
        res = C.c_void_p()
        _check(lib.b200m_guided_match_model(ctx._h, C.c_uint32(ids[0]), C.c_uint32(ids[1]), C.c_int(model), Fm.ctypes.data_as(C.c_void_p), C.c_double(errorTh),
                                            C.c_double(distRatio), C.byref(res)), "b200m_guided_match_model")
        owner = _ResultOwner(lib, res)
        off, mat = C.c_void_p(), C.c_void_p()
        _check(lib.b200m_result_get(res, None, C.byref(off), C.byref(mat)), "b200m_result_get")
        n = int(_alias(off.value, 16, np.int64, owner)[1])
        return _alias(mat.value, n * MATCH_DTYPE.itemsize, MATCH_DTYPE, owner).copy()
    finally:
        for vid in up:
            lib.b200m_remove_view(ctx._h, C.c_uint32(vid))


def guidedMatchingFundamentalFast(F, epipole2, regions_left: "Regions", regions_right: "Regions", widthR: int, heightR: int, errorTh: float,
                                  distRatio: float, xy_left=None, xy_right=None, ctx: Context | None = None) -> np.ndarray:
    """matching::guidedMatchingFundamentalFast<FundamentalEpipolarDistanceError> (matching/guidedMatching.hpp:353-460) for one pair:
    F (x_right^T F x_left = 0), epipole2 = the left camera centre in the right image, not normalised (epipole_from_P), the right
    image's size, errorTh / distRatio already squared (StructureEstimationFromKnownPoses.cpp:138-150).  xy_left / xy_right: optional
    n x 2 double (undistorted) positions used instead of the regions' positions.  Returns matches[MATCH_DTYPE] in ascending i, not
    de-duplicated.  For lists of pairs over resident views use Context.guided_match_fast_pairs."""
    ctx = ctx or default_context()
    ids = (_new_view_id(), _new_view_id())
    up = []
    try:
        _upload_pair(ctx, ids, (regions_left, regions_right), (xy_left, xy_right), up)
        return ctx.guided_match_fast_pairs([ids], [F], [epipole2], [(widthR, heightR)], errorTh, distRatio)[ids]
    finally:
        for vid in up:
            ctx.lib.b200m_remove_view(ctx._h, C.c_uint32(vid))


def createImageCollectionMatcher(matcherType: EMatcherType, distRatio: float, crossMatching: bool, ctx: Context | None = None):
    """matchingImageCollection/matchingCommon.cpp:19-47 restricted to the matcher types this engine implements."""
    return ImageCollectionMatcherB200(distRatio, crossMatching, matcherType, ctx)


# ---- Surface 1b: IRegionsMatcher / RegionsDatabaseMatcher / DistanceRatioMatch ----------------------------------------
_next_view_id = [0x40000000]


def _new_view_id() -> int:
    _next_view_id[0] += 1
    return _next_view_id[0]


class Regions:
    """The slice of feature::Regions the matchers read (feature/Regions.hpp:46-118): descriptors[n, L], positions[n, 2],
    IsBinary().  ``binary`` distinguishes AKAZE_BinaryRegions (uchar[64] bit strings) from SIFT_Regions (uchar[128])."""

    def __init__(self, descriptors: np.ndarray, positions: np.ndarray | None = None, binary: bool = False):
        self.descriptors = np.ascontiguousarray(descriptors)
        if self.descriptors.ndim != 2:
            raise ValueError("descriptors must be [n, L]")
        n = self.descriptors.shape[0]
        self.positions = np.zeros((n, 2), np.float32) if positions is None else np.ascontiguousarray(positions, np.float32).reshape(n, 2)
        self.binary = bool(binary)

    def RegionCount(self) -> int: return int(self.descriptors.shape[0])
    def DescriptorLength(self) -> int: return int(self.descriptors.shape[1])
    def IsBinary(self) -> bool: return self.binary
    def IsScalar(self) -> bool: return not self.binary
    def Type_id(self) -> str: return "f" if self.descriptors.dtype == np.float32 else "h"


class RegionsMatcherB200:
    """IRegionsMatcher (matching/RegionsMatcher.hpp:49-78) on the engine: the database Regions are uploaded once by the
    constructor, Match(f_dist_ratio, query_regions) runs RegionsMatcher::Match (:126-176) for that pair on the GPU and
    returns (ok, matches[MATCH_DTYPE]); ok == "the list is not empty" as in the reference (:175)."""

    def __init__(self, regions: Regions, ctx: Context | None = None):
        self.ctx = ctx or default_context()
        self.regions_ = regions
        self._code = _dtype_code(regions.descriptors, regions.binary)
        self._id = None
        if regions.RegionCount() > 0:
            self._id = _new_view_id()
            self._upload(self._id, regions)

    def _upload(self, vid: int, r: Regions) -> None:
        n = r.RegionCount()
        _check(self.ctx.lib.b200m_upload_view(self.ctx._h, C.c_uint32(vid), r.descriptors.ctypes.data_as(C.c_void_p) if n else None, C.c_int(n),
                                              C.c_int(max(r.DescriptorLength(), 1)), C.c_int(self._code),
                                              r.positions.ctypes.data_as(C.c_void_p) if n else None), "b200m_upload_view")

    def getDatabaseRegions(self) -> Regions:
        return self.regions_

    def Match(self, f_dist_ratio: float, query_regions: Regions):
        empty = np.zeros(0, MATCH_DTYPE)
        if query_regions.RegionCount() == 0 or self._id is None:
            return False, empty
        if (query_regions.descriptors.dtype != self.regions_.descriptors.dtype or query_regions.binary != self.regions_.binary
                or query_regions.DescriptorLength() != self.regions_.DescriptorLength()):
            return False, empty
        lib = self.ctx.lib
        qid = _new_view_id()
        self._upload(qid, query_regions)
        try:
            pair = np.array([[self._id, qid]], np.uint32)
            res = C.c_void_p()
            _check(lib.b200m_match_pairs(self.ctx._h, pair.ctypes.data_as(C.c_void_p), C.c_int(1), C.c_float(f_dist_ratio), C.c_int(0),
                                         C.c_int(STAGE_FULL), C.byref(res)), "b200m_match_pairs")
            owner = _ResultOwner(lib, res)
            off, mat = C.c_void_p(), C.c_void_p()
            _check(lib.b200m_result_get(res, None, C.byref(off), C.byref(mat)), "b200m_result_get")
            n = int(_alias(off.value, 16, np.int64, owner)[1])
            matches = _alias(mat.value, n * MATCH_DTYPE.itemsize, MATCH_DTYPE, owner).copy()
        finally:
            lib.b200m_remove_view(self.ctx._h, C.c_uint32(qid))
        return len(matches) > 0, matches

    def close(self) -> None:
        if self._id is not None and self.ctx._h:
            self.ctx.lib.b200m_remove_view(self.ctx._h, C.c_uint32(self._id))
        self._id = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def createRegionsMatcher(regions: Regions, matcherType: EMatcherType, ctx: Context | None = None):
    """matching/RegionsMatcher.cpp:54-176 for the matcher types this engine implements.  Invalid requests return None
    like the reference's null unique_ptr (:61-64): scalar regions + Hamming matcher, binary regions + L2 matcher."""
    hamming = matcherType in (EMatcherType.BRUTE_FORCE_HAMMING, EMatcherType.BRUTE_FORCE_HAMMING_B200)
    if matcherType not in (EMatcherType.BRUTE_FORCE_L2, EMatcherType.BRUTE_FORCE_L2_B200) and not hamming:
        return None
    if regions.IsScalar() and hamming:
        return None
    if regions.IsBinary() and not hamming:
        return None
    if regions.descriptors.dtype not in (np.float32, np.uint8):
        return None
    return RegionsMatcherB200(regions, ctx)


class RegionsDatabaseMatcherB200:
    """matching::RegionsDatabaseMatcher (RegionsMatcher.hpp:183-220, RegionsMatcher.cpp:30-52)."""

    def __init__(self, matcherType: EMatcherType = EMatcherType.BRUTE_FORCE_L2_B200, database_regions: Regions | None = None, ctx: Context | None = None):
        self._matcherType = matcherType
        self._regionsMatcher = None if database_regions is None else createRegionsMatcher(database_regions, matcherType, ctx)

    def Match(self, distRatio: float, queryRegions: Regions):
        if queryRegions.RegionCount() == 0 or self._regionsMatcher is None:      # RegionsMatcher.cpp:32-38
            return False, np.zeros(0, MATCH_DTYPE)
        return self._regionsMatcher.Match(distRatio, queryRegions)

    def getDatabaseRegions(self) -> Regions:
        return self._regionsMatcher.getDatabaseRegions()


def DistanceRatioMatch(f_dist_ratio: float, eMatcherType: EMatcherType, regions_I: Regions, regions_J: Regions, ctx: Context | None = None) -> np.ndarray:
    """matching::DistanceRatioMatch (RegionsMatcher.cpp:19-28): regions_I = database, regions_J = query."""
    matcher = RegionsDatabaseMatcherB200(eMatcherType, regions_I, ctx)
    _, matches = matcher.Match(f_dist_ratio, regions_J)
    return matches
