"""The reference-side binding (integration/patches/aliceVision_b200.patch, INTEGRATION.md): applied to a scratch copy of the
reference files it touches, the patched enum file compiles with the reference's -Werror=switch and the patched factory passes
a syntax check against the reference's own headers (through oracle/shim) with the adaptors in place.  Needs the AliceVision
source tree (oracle.reference_src()); nothing is written there."""
import os
import shutil
import subprocess

import pytest

import oracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = oracle.reference_src()
REF = os.path.join(SRC, "aliceVision") if SRC else None
PATCH = os.path.join(ROOT, "integration", "patches", "aliceVision_b200.patch")
FILES = ["matching/matcherType.hpp", "matching/matcherType.cpp", "matching/RegionsMatcher.cpp", "matching/CMakeLists.txt",
         "matchingImageCollection/matchingCommon.cpp", "matchingImageCollection/matchingCommon.hpp",
         "matchingImageCollection/GeometricFilterMatrix_F_AC.hpp", "matchingImageCollection/CMakeLists.txt"]


@pytest.mark.skipif(SRC is None, reason="no AliceVision source tree (ALICEVISION_SRC)")
def test_patch_applies_and_compiles(tmp_path):
    for f in FILES:
        dst = tmp_path / "src" / "aliceVision" / f
        dst.parent.mkdir(parents=True, exist_ok=True)
        shutil.copy(os.path.join(REF, f), dst)
    r = subprocess.run(["patch", "-p1", "-s", "-i", PATCH], cwd=tmp_path, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    mt = tmp_path / "src" / "aliceVision" / "matching" / "matcherType.cpp"
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror=switch", "-c", str(mt), "-o", str(tmp_path / "mt.o")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    text = mt.read_text()
    assert '"BRUTE_FORCE_L2_B200"' in text and '"BRUTE_FORCE_HAMMING_B200"' in text
    # the adaptors at the places INTEGRATION.md puts them
    inc = tmp_path / "inc" / "aliceVision"
    (inc / "matching").mkdir(parents=True); (inc / "matchingImageCollection").mkdir(parents=True)
    shutil.copy(tmp_path / "src" / "aliceVision" / "matching" / "matcherType.hpp", inc / "matching" / "matcherType.hpp")
    ad = os.path.join(ROOT, "alicevision_b200", "adaptor")
    for h in ("ArrayMatcher_b200.hpp", "RegionsMatcher_b200.hpp", "guidedMatching_b200.hpp"):
        shutil.copy(os.path.join(ad, h), inc / "matching" / h)
    shutil.copy(os.path.join(ad, "ImageCollectionMatcher_b200.hpp"), inc / "matchingImageCollection" / "ImageCollectionMatcher_b200.hpp")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", str(tmp_path / "inc"), "-I", os.path.join(ROOT, "oracle", "shim"),
                        "-I", SRC, "-I", os.path.join(ROOT, "include"),
                        str(tmp_path / "src" / "aliceVision" / "matchingImageCollection" / "matchingCommon.cpp")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[:2000]
