"""Guided matching from known poses: b200m_guided_match_fast_pairs / matching.guidedMatchingFundamentalFast against
matching::guidedMatchingFundamentalFast (matching/guidedMatching.hpp:353-460, guidedMatching.cpp:13-70), and guided matching on
per-view geometry (undistorted) positions (b200m_set_view_geometry).

The oracle (oracle/guided_fast_oracle.cpp) takes double positions.  Its "ref" build computes descriptor distances with the
reference's own Regions::SquaredDescriptorDistance; the geometry (3x3 products, cross products, lineToEndPoints, pixToBucket) is
restated in both builds - Eigen and guidedMatching.cpp cannot be compiled here, so that part is not pinned by compiled reference
code.  Without the compiled reference its stored outputs (tests/golden/reference_guided_fast.npz) stand in for it.

Scenes: a synthetic 3D point cloud seen by pinhole cameras with known K, R, t; shared points are re-observed with descriptor noise
and sub-pixel position noise, among fresh features and decoys (copies of re-observed descriptors far from their epipolar line);
F and the epipole come from the two projection matrices; optionally a radial distortion moves the observed (uploaded) positions
and the undistorted ones are passed as geometry positions."""
import os

import numpy as np
import pytest

import oracle
from oracle import guided_fast as gfo
from alicevision_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------- scene generator
def rot(ax, ay, az):
    cx, sx, cy, sy, cz, sz = np.cos(ax), np.sin(ax), np.cos(ay), np.sin(ay), np.cos(az), np.sin(az)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]); Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


class Camera:
    def __init__(self, W, H, R, C, k1=0.0):
        f = 0.9 * W
        self.W, self.H, self.k1 = int(W), int(H), k1
        self.K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], np.float64)
        self.R, self.C = np.asarray(R, np.float64), np.asarray(C, np.float64)
        self.P = self.K @ np.concatenate([self.R, -(self.R @ self.C)[:, None]], 1)

    def project(self, X):
        h = np.concatenate([X, np.ones((len(X), 1))], 1) @ self.P.T
        return h[:, :2] / h[:, 2:], h[:, 2]

    def distort(self, x):
        """Radial distortion around the principal point (normalised by f): what a real camera would observe."""
        c = self.K[:2, 2]; f = self.K[0, 0]
        d = (x - c) / f
        r2 = (d * d).sum(1, keepdims=True)
        return c + d * (1 + self.k1 * r2) * f


def fundamental(camL: Camera, camR: Camera):
    """F (x_R^T F x_L = 0) and epipole2 = P_R C_L (homogeneous, not normalised) as F_from_P (numeric/projection.cpp:115-143: the
    determinants of stacked row pairs, which fix the sign of F relative to the epipole) and epipole_from_P give them."""
    def rows(P):
        return [P[[1, 2]], P[[2, 0]], P[[0, 1]]]
    X, Y = rows(camL.P), rows(camR.P)
    F = np.array([[np.linalg.det(np.concatenate([X[c], Y[r]])) for c in range(3)] for r in range(3)])
    return F, camR.P @ np.append(camL.C, 1.0)


def observe(cam, X, base, kind, rng, n_fresh, decoy_src):
    """Features of one view: the visible points (descriptor noise, <= 0.7 px position noise) + fresh features, some of them decoys.
    Returns (descriptors, uploaded float32 positions, undistorted double positions, point id per feature (-1: fresh))."""
    x, z = cam.project(X)
    vis = np.where((z > 0) & (x[:, 0] >= 0) & (x[:, 0] < cam.W - 1) & (x[:, 1] >= 0) & (x[:, 1] < cam.H - 1))[0]
    und = x[vis] + rng.uniform(-0.7, 0.7, (len(vis), 2))
    if kind == "bin":
        flip = rng.random((len(vis), 64, 8)) < 0.05
        d = base[vis] ^ np.packbits(flip, axis=2, bitorder="little")[:, :, 0]
        fresh = synth.mldb_images(1, n_fresh, seed=int(rng.integers(1 << 30)))[0][0]
    else:
        d = np.clip(base[vis].astype(np.int32) + rng.integers(-5, 6, (len(vis), 128)), 0, 255).astype(np.uint8)
        fresh = synth.sift_images(1, n_fresh, np.uint8, seed=int(rng.integers(1 << 30)), pool_factor=1.0)[0][0]
    nd = min(n_fresh // 2, len(decoy_src))
    fresh[:nd] = base[rng.choice(decoy_src, nd, replace=False)]
    fu = np.stack([rng.uniform(0, cam.W - 1, n_fresh), rng.uniform(0, cam.H - 1, n_fresh)], 1)
    desc = np.concatenate([d, fresh]); und = np.concatenate([und, fu]); pid = np.concatenate([vis, -np.ones(n_fresh, np.int64)])
    perm = rng.permutation(len(desc))
    desc, und, pid = desc[perm], und[perm], pid[perm]
    obs = cam.distort(und) if cam.k1 else und
    return desc, obs.astype(np.float32), und, pid


def world(n, rng, kind):
    X = np.stack([rng.uniform(-4, 4, n), rng.uniform(-3, 3, n), rng.uniform(7, 12, n)], 1)
    base = synth.mldb_images(1, n, seed=int(rng.integers(1 << 30)))[0][0] if kind == "bin" else \
        synth.sift_images(1, n, np.uint8, seed=int(rng.integers(1 << 30)), pool_factor=1.0)[0][0]
    return X, base


# two-view geometries: (name, right camera centre and rotation relative to the left one at the origin)
GEOMS = {
    "outside": (np.array([1.6, 0.15, 0.2]), (0.01, -0.12, 0.02)),      # lateral motion: epipole far outside, ep2(2) > 0
    "outside_neg": (np.array([1.4, -0.2, -0.3]), (-0.02, -0.1, 0.0)),  # lateral motion backwards: ep2(2) < 0
    "inside": (np.array([0.15, 0.1, -1.5]), (0.01, 0.02, 0.03)),       # camera behind the left one: epipole inside the right image
    "inside_fwd": (np.array([-0.1, 0.05, 1.2]), (0.0, 0.03, -0.02)),   # forward motion: epipole inside, ep2(2) < 0
}


def two_view(kind, geom="outside", n=1500, W=4000, H=3000, seed=3, k1=0.0, WL=None, HL=None):
    """Left / right views of one scene.  Returns dict(dl, xl, ul, dr, xr, ur, F, ep2, W, H, truth) - x*: uploaded float32, u*: double
    undistorted positions, truth {left i: right j}."""
    rng = np.random.default_rng(seed)
    X, base = world(int(n * 1.6), rng, kind)
    C2, ang = GEOMS[geom]
    camL = Camera(WL or W, HL or H, np.eye(3), np.zeros(3), k1)
    camR = Camera(W, H, rot(*ang), C2, k1)
    shared = np.arange(len(X))
    dl, xl, ul, pl = observe(camL, X[: int(n * 0.75)], base, kind, rng, n // 4, shared[: int(n * 0.75)])
    dr, xr, ur, pr = observe(camR, X, base, kind, rng, n // 3, shared)
    dl, xl, ul, pl = dl[:n], xl[:n], ul[:n], pl[:n]
    dr, xr, ur, pr = dr[:n], xr[:n], ur[:n], pr[:n]
    if kind in ("f32", "real", "mixed"):
        dl, dr = dl.astype(np.float32), dr.astype(np.float32)
    if kind == "real":
        dl, dr = synth.real_valued([dl, dr])
    if kind == "mixed":                      # integer-valued left (stored as uchar by the engine), real-valued right
        dr = synth.real_valued([dr])[0]
    F, ep2 = fundamental(camL, camR)
    rmap = {int(p): j for j, p in enumerate(pr) if p >= 0}
    truth = {i: rmap[int(p)] for i, p in enumerate(pl) if p >= 0 and int(p) in rmap}
    return dict(dl=dl, xl=xl, ul=ul, dr=dr, xr=xr, ur=ur, F=F, ep2=ep2, W=W, H=H, truth=truth)


def ij(m):
    return np.stack([m["i"], m["j"]], 1) if len(m) else np.zeros((0, 2), np.uint32)


def same(got, want):
    return len(got) == len(want) and np.array_equal(got["i"], want["i"]) and np.array_equal(got["j"], want["j"])


# the CPU grid: geometry x (W, H) x sign of (F, ep2)
GRID = [("outside", 4000, 3000, 1), ("outside", 4000, 3000, -1), ("outside_neg", 1920, 1080, 1), ("inside", 4000, 3000, 1),
        ("inside_fwd", 640, 480, 1), ("inside_fwd", 640, 480, -1)]
THRESHOLDS = (1.0, 25.0, 400.0)


def reference():
    R = gfo.GuidedFastOracle("ref") if gfo.available("ref") else None
    return R, lambda key, f: gfo.reference_output("guided_fast." + key, f, R is not None)


# ---------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("kind", ["u8", "f32", "real", "bin"])
def test_port_equals_reference(kind):
    (R, ref), P = reference(), gfo.GuidedFastOracle("port")
    for geom, W, H, sign in GRID:
        s = two_view(kind, geom, 600, W, H, seed=5)
        F, ep2 = sign * s["F"], sign * s["ep2"]
        for th in THRESHOLDS:
            args = (s["dl"], s["ul"], s["dr"], s["ur"], F, ep2, W, H, th, 0.64)
            a = ref(f"{kind}.{geom}.{W}x{H}.{sign}.{th}", lambda: R.guided_fast(*args, binary=kind == "bin"))
            b = P.guided_fast(*args, binary=kind == "bin")
            assert same(a, b), (geom, W, H, sign, th)
            assert np.all(np.diff(a["i"].astype(np.int64)) > 0)
        if sign == 1 and geom.startswith("outside"):
            a = P.guided_fast(s["dl"], s["ul"], s["dr"], s["ur"], F, ep2, W, H, 25.0, 0.64, binary=kind == "bin")
            good = sum(1 for m in a if s["truth"].get(int(m["i"])) == int(m["j"]))
            assert len(a) > 50 and good > 0.9 * len(a)


def test_sign_of_epipole_does_not_matter():
    """(F, ep2) and (-F, -ep2) are the same geometry: the normalisation of :378-384 makes the results identical."""
    P = gfo.GuidedFastOracle("port")
    for geom in GEOMS:
        s = two_view("u8", geom, 500, seed=9)
        a = P.guided_fast(s["dl"], s["ul"], s["dr"], s["ur"], s["F"], s["ep2"], 4000, 3000, 25.0, 0.64)
        b = P.guided_fast(s["dl"], s["ul"], s["dr"], s["ur"], -s["F"], -s["ep2"], 4000, 3000, 25.0, 0.64)
        assert same(a, b) and len(a) > 0


def test_port_guided_match_on_double_positions_equals_reference():
    """The guidedMatching loop on double positions: the "ref" build (reference distances) equals the port."""
    (R, ref), P = reference(), gfo.GuidedFastOracle("port")
    for kind in ("u8", "real", "bin"):
        s = two_view(kind, "outside", 500, seed=13, k1=-0.08)
        for th in (4.0, 25.0):
            args = (s["dl"], s["ul"], s["dr"], s["ur"], s["F"], th, 0.64)
            a = ref(f"match.{kind}.{th}", lambda: R.guided_match(*args, binary=kind == "bin"))
            assert same(a, P.guided_match(*args, binary=kind == "bin"))


def test_guided_match_float_positions_equal_existing_oracle():
    """On float positions widened to double, the new loop is the existing oracle's guidedMatching."""
    P, O = gfo.GuidedFastOracle("port"), oracle.Oracle("port")
    s = two_view("u8", "outside", 500, seed=21)
    for th in (4.0, 25.0):
        a = P.guided_match(s["dl"], s["xl"].astype(np.float64), s["dr"], s["xr"].astype(np.float64), s["F"], th, 0.64)
        b = O.guided_match(s["dl"], s["xl"], s["dr"], s["xr"], s["F"], th, 0.64)
        assert np.array_equal(ij(a), ij(b))


def test_known_poses_patch_applies(tmp_path):
    src = oracle.reference_src()
    if src is None:
        pytest.skip("no AliceVision source tree (ALICEVISION_SRC)")
    import shutil
    import subprocess
    files = ["sfm/pipeline/structureFromKnownPoses/StructureEstimationFromKnownPoses.cpp", "matching/CMakeLists.txt"]
    for f in files:
        dst = tmp_path / "src" / "aliceVision" / f
        dst.parent.mkdir(parents=True, exist_ok=True)
        shutil.copy(os.path.join(src, "aliceVision", f), dst)
    patch = os.path.join(ROOT, "integration", "patches", "aliceVision_b200_knownPoses.patch")
    r = subprocess.run(["patch", "-p1", "-s", "-i", patch], cwd=tmp_path, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    text = (tmp_path / "src" / "aliceVision" / files[0]).read_text()
    assert "guidedMatchingFast_b200.hpp" in text and "GuidedMatchingFastBatch_b200" in text


def test_fast_adaptor_header_compiles():
    src = oracle.reference_src()
    if src is None:
        pytest.skip("no AliceVision source tree (ALICEVISION_SRC)")
    import subprocess
    hdr = os.path.join(ROOT, "alicevision_b200", "adaptor", "guidedMatchingFast_b200.hpp")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-x", "c++", "-I", os.path.join(ROOT, "oracle", "shim"), "-I", src,
                        "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "alicevision_b200", "adaptor"), hdr],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[:2000]


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["u8", "f32", "real", "bin", "mixed"])
def test_gpu_fast_single_pair_equals_oracle(kind):
    from alicevision_b200 import Regions, matching
    O = gfo.best()
    for geom, W, H, sign in GRID:
        s = two_view(kind, geom, 1500, W, H, seed=7, k1=-0.05)
        F, ep2 = sign * s["F"], sign * s["ep2"]
        L, Rr = Regions(s["dl"], s["xl"], binary=kind == "bin"), Regions(s["dr"], s["xr"], binary=kind == "bin")
        for th in THRESHOLDS:
            want = O.guided_fast(s["dl"], s["ul"], s["dr"], s["ur"], F, ep2, W, H, th, 0.64, binary=kind == "bin")
            got = matching.guidedMatchingFundamentalFast(F, ep2, L, Rr, W, H, th, 0.64, xy_left=s["ul"], xy_right=s["ur"])
            assert same(got, want), (kind, geom, W, H, sign, th, len(got), len(want))
            assert not got["ratio"].any() and not got["dist"].any()
        # without geometry positions: the uploaded (distorted) float positions, widened
        want = O.guided_fast(s["dl"], s["xl"], s["dr"], s["xr"], F, ep2, W, H, 25.0, 0.64, binary=kind == "bin")
        assert same(matching.guidedMatchingFundamentalFast(F, ep2, L, Rr, W, H, 25.0, 0.64), want)


def multi_view(n_views=12, n=1000, seed=31, kind="u8"):
    """n_views cameras around one point cloud, image sizes mixed.  Returns (cams, views) with views[v] = (desc, xy, und)."""
    rng = np.random.default_rng(seed)
    X, base = world(4000, rng, kind)
    sizes = [(4000, 3000), (1920, 1080), (3000, 2000), (640, 480)]
    cams, views = [], []
    for v in range(n_views):
        W, H = sizes[v % len(sizes)]
        C = np.array([rng.uniform(-2.5, 2.5), rng.uniform(-1, 1), rng.uniform(-1.5, 1.5)])
        cam = Camera(W, H, rot(rng.uniform(-0.05, 0.05), rng.uniform(-0.2, 0.2), rng.uniform(-0.05, 0.05)), C, k1=-0.04 * (v % 2))
        d, xy, und, _ = observe(cam, X, base, kind, rng, n // 4, np.arange(len(X)))
        cams.append(cam); views.append((d[:n], xy[:n], und[:n]))
    return cams, views


@pytest.mark.gpu
def test_gpu_fast_batch_equals_oracle_and_single_calls(monkeypatch):
    from alicevision_b200 import ImageCollectionMatcherB200, matching
    monkeypatch.setenv("B200M_GUIDED_FAST_LEFT_CAP", "6000")      # about six pairs per internal batch: the list spans several
    ctx = matching.Context(0)
    try:
        O = gfo.best()
        cams, views = multi_view(12, 1000)
        geo = {v for v in range(12) if v % 3 != 2}                  # some views with geometry positions, some without
        up = ImageCollectionMatcherB200(0.8, False, ctx=ctx)
        up.upload({v: (views[v][0], views[v][1]) for v in range(12)})      # asynchronous
        for v in sorted(geo):
            ctx.set_view_geometry(v, views[v][2])
        rng = np.random.default_rng(2)
        pairs = [(a, b) for a in range(12) for b in range(12) if a != b]
        pairs = [pairs[k] for k in rng.permutation(len(pairs))[:60]]
        Fs, eps, whs = [], [], []
        for a, b in pairs:
            F, e = fundamental(cams[a], cams[b])
            Fs.append(F); eps.append(e); whs.append((cams[b].W, cams[b].H))
        errs = ctx.exactness_errors()
        got = ctx.guided_match_fast_pairs(pairs, Fs, eps, whs, 16.0, 0.64)
        assert list(got) == pairs
        assert ctx.last_launches() >= 2 * 11 and ctx.exactness_errors() == errs
        total = 0
        pos = lambda v: views[v][2] if v in geo else views[v][1].astype(np.float64)
        for k, (a, b) in enumerate(pairs):
            want = O.guided_fast(views[a][0], pos(a), views[b][0], pos(b), Fs[k], eps[k], whs[k][0], whs[k][1], 16.0, 0.64)
            assert same(got[(a, b)], want), (a, b)
            one = ctx.guided_match_fast_pairs([(a, b)], [Fs[k]], [eps[k]], [whs[k]], 16.0, 0.64)[(a, b)]
            assert same(one, got[(a, b)])
            total += len(want)
        assert total > 1000
    finally:
        ctx.close()


@pytest.mark.gpu
def test_gpu_fast_edge_cases():
    from alicevision_b200 import ImageCollectionMatcherB200, Regions, matching
    O = gfo.best()
    s = two_view("u8", "outside", 400, seed=41)
    L, Rr = Regions(s["dl"], s["xl"]), Regions(s["dr"], s["xr"])
    F, ep2, W, H = s["F"], s["ep2"], s["W"], s["H"]
    fast = lambda F_, e_, l=L, r=Rr, th=25.0: matching.guidedMatchingFundamentalFast(F_, e_, l, r, W, H, th, 0.64)
    # lines with a == 0 / b == 0: no end points, no buckets
    Fa = np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0]], np.float64)          # line (0, -1, y): a == 0
    Fb = np.array([[0, 0, -1], [0, 0, 0], [1, 0, 0]], np.float64)          # line (-1, 0, x): b == 0
    for Fx in (Fa, Fb):
        want = O.guided_fast(s["dl"], s["xl"], s["dr"], s["xr"], Fx, ep2, W, H, 25.0, 0.64)
        assert len(want) == 0 and len(fast(Fx, ep2)) == 0
    # right features on the epipole's row / column (right lines with a zero coefficient) and an epipole inside (ranges that wrap
    # across bucket 0 have no candidates): compared with the oracle
    t = two_view("u8", "inside", 1200, seed=43)
    e = t["ep2"] / t["ep2"][2]
    xr = t["xr"].copy(); xr[:40, 1] = np.float32(e[1]); xr[40:80, 0] = np.float32(e[0])
    want = O.guided_fast(t["dl"], t["xl"], t["dr"], xr, t["F"], t["ep2"], 4000, 3000, 400.0, 0.64)
    got = matching.guidedMatchingFundamentalFast(t["F"], t["ep2"], Regions(t["dl"], t["xl"]), Regions(t["dr"], xr), 4000, 3000, 400.0, 0.64)
    assert same(got, want) and len(got) > 0
    # empty views, a single candidate, differing descriptor types
    empty = Regions(s["dl"][:0], s["xl"][:0])
    assert len(fast(F, ep2, l=empty)) == 0 and len(fast(F, ep2, r=empty)) == 0
    one = Regions(s["dr"][:1], s["xr"][:1])
    assert len(fast(F, ep2, r=one, th=1e12)) == 0                           # no second distance (:115-117)
    assert len(fast(F, ep2, r=Regions(s["dr"].astype(np.float32) + 0.5, s["xr"]))) == 0       # u8 vs f32: no common type
    bl = synth.mldb_images(1, 400, seed=3)[0][0]
    assert len(fast(F, ep2, r=Regions(bl, s["xr"], binary=True))) == 0     # u8 vs binary
    # a batch with such pairs: one (possibly empty) list per input pair, in input order
    ctx = matching.default_context()
    up = ImageCollectionMatcherB200(0.8, False, ctx=ctx)
    up.upload({900001: (s["dl"], s["xl"]), 900002: (s["dr"], s["xr"]), 900003: (s["dl"][:0], s["xl"][:0])})
    pairs = [(900001, 900003), (900001, 900002), (900003, 900002), (900001, 900002)]
    got = ctx.guided_match_fast_pairs(pairs, [F] * 4, [ep2] * 4, [(W, H)] * 4, 25.0, 0.64)
    want = O.guided_fast(s["dl"], s["xl"], s["dr"], s["xr"], F, ep2, W, H, 25.0, 0.64)
    assert len(got[(900001, 900003)]) == 0 and len(got[(900003, 900002)]) == 0 and same(got[(900001, 900002)], want)
    # W or H < 2, geometry of the wrong length
    for w, h in ((1, 3000), (4000, 1), (0, 0)):
        with pytest.raises(matching.B200MatchError):
            ctx.guided_match_fast_pairs([(900001, 900002)], [F], [ep2], [(w, h)], 25.0, 0.64)
    with pytest.raises(matching.B200MatchError):
        ctx.set_view_geometry(900001, s["ul"][:-1])
    with pytest.raises(matching.B200MatchError):
        ctx.set_view_geometry(123456789, s["ul"])
    up.clear()


@pytest.mark.gpu
def test_gpu_fast_undefined_inputs_do_not_fault():
    """Where the reference is undefined (NaN cast to int): an epipole at infinity gives an empty list, a right feature exactly at the
    epipole gets no candidates.  Not compared with the oracle."""
    from alicevision_b200 import Regions, matching
    ctx = matching.default_context()
    errs = ctx.exactness_errors()
    s = two_view("u8", "outside", 800, seed=51)
    L, Rr = Regions(s["dl"], s["xl"]), Regions(s["dr"], s["xr"])
    ep_inf = s["ep2"].copy(); ep_inf[2] = 0.0
    assert len(matching.guidedMatchingFundamentalFast(s["F"], ep_inf, L, Rr, 4000, 3000, 25.0, 0.64)) == 0
    t = two_view("u8", "inside", 800, seed=53)
    e = t["ep2"] / t["ep2"][2]
    ur = t["ur"].copy(); ur[5] = e[:2]                                      # exactly at the epipole (double geometry position)
    got = matching.guidedMatchingFundamentalFast(t["F"], t["ep2"], Regions(t["dl"], t["xl"]), Regions(t["dr"], t["xr"]), 4000, 3000, 25.0, 0.64,
                                                 xy_left=t["ul"], xy_right=ur)
    assert 5 not in set(got["j"].tolist()) and len(got) > 0
    assert ctx.exactness_errors() == errs


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["u8", "real", "bin"])
def test_gpu_guided_match_with_geometry_equals_oracle(kind):
    """b200m_guided_match_model on geometry positions = the guidedMatching loop on those double positions."""
    from alicevision_b200 import Regions, matching
    O = gfo.best()
    s = two_view(kind, "outside", 1500, seed=61, k1=-0.08)
    L, Rr = Regions(s["dl"], s["xl"], binary=kind == "bin"), Regions(s["dr"], s["xr"], binary=kind == "bin")
    for th in (4.0, 25.0):
        want = O.guided_match(s["dl"], s["ul"], s["dr"], s["ur"], s["F"], th, 0.64, binary=kind == "bin")
        got = matching.guidedMatching(s["F"], L, Rr, th, 0.64, xy_left=s["ul"], xy_right=s["ur"])
        assert same(got, want) and len(got) > 100
        # only one side with geometry: the other side keeps its float positions
        want = O.guided_match(s["dl"], s["ul"], s["dr"], s["xr"].astype(np.float64), s["F"], th, 0.64, binary=kind == "bin")
        assert same(matching.guidedMatching(s["F"], L, Rr, th, 0.64, xy_left=s["ul"]), want)


@pytest.mark.gpu
def test_gpu_fast_full_size():
    """8192 x 8192 features at 4000 x 3000: the complete lists equal the oracle on two pairs, and > 90 % of the kept matches are
    true correspondences."""
    from alicevision_b200 import Regions, matching
    O = gfo.best()
    for geom in ("outside", "inside"):
        s = two_view("u8", geom, 8192, seed=71, k1=-0.05)
        want = O.guided_fast(s["dl"], s["ul"], s["dr"], s["ur"], s["F"], s["ep2"], 4000, 3000, 16.0, 0.64)
        got = matching.guidedMatchingFundamentalFast(s["F"], s["ep2"], Regions(s["dl"], s["xl"]), Regions(s["dr"], s["xr"]), 4000, 3000, 16.0, 0.64,
                                                     xy_left=s["ul"], xy_right=s["ur"])
        assert same(got, want)
        good = sum(1 for m in got if s["truth"].get(int(m["i"])) == int(m["j"]))
        assert len(got) > 1000 and good > 0.9 * len(got), (geom, len(got), good)


@pytest.mark.gpu
def test_gpu_fast_cpp_adaptor():
    """The C++ batch adaptor (alicevision_b200/adaptor/guidedMatchingFast_b200.hpp) against the "ref" oracle in one executable."""
    exe = os.path.join(ROOT, "oracle", "_ref", "guided_fast_adaptor_test")
    if not os.path.exists(exe):
        pytest.skip("the C++ adaptor test is built where the AliceVision source tree is readable")
    import subprocess
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "guided_fast adaptor ok" in r.stdout
