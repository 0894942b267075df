"""alicevision_b200 — H100 (sm_90a) engine for AliceVision's descriptor-matching hot path.

Only what the path needs lives here: ``csrc/`` (CUDA kernels + the C ABI of include/b200match.h),
``adaptor/`` (C++ classes deriving from the reference's ArrayMatcher / IRegionsMatcher / IImageCollectionMatcher),
``matching`` (the same surface bound from Python for tests and bench), ``synth`` (deterministic inputs).
"""
from .matching import (ArrayMatcherB200, B200MatchError, Context, DistanceRatioMatch, EMatcherType, ImageCollectionMatcherB200,  # noqa: F401
                       Regions, RegionsDatabaseMatcherB200, RegionsMatcherB200, createImageCollectionMatcher, createRegionsMatcher,
                       default_context, load_library)

__all__ = ["ArrayMatcherB200", "ImageCollectionMatcherB200", "EMatcherType", "Context", "B200MatchError",
           "createImageCollectionMatcher", "default_context", "load_library", "Regions", "RegionsMatcherB200", "RegionsDatabaseMatcherB200",
           "DistanceRatioMatch", "createRegionsMatcher"]
