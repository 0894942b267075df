"""Deterministic synthetic regions for tests and bench (SURVEY.md §8(d) "Synthetic inputs").

SIFT-like descriptors follow the reference extractor's quantisation (feature/sift/SIFT.hpp:80-110:
RootSIFT ``floor(512*sqrt(x/sum x))``), so they are small non-negative integers and every squared
L2 distance is an exact integer < 2^24 — the property that makes bit-exact index parity possible.
MLDB-like descriptors are 486 random bits packed LSB-first into 64 bytes
(feature/akaze/ImageDescriber_AKAZE.cpp:138-150).  numpy only; no product or oracle code here.
"""
from __future__ import annotations

import numpy as np

SEED_DATA = 20260922
SEED_PAIRS = 7


def _rootsift(raw: np.ndarray) -> np.ndarray:
    x = raw / np.linalg.norm(raw, axis=1, keepdims=True)
    x = np.minimum(x, 0.2)
    x = x / np.linalg.norm(x, axis=1, keepdims=True)
    return np.floor(512.0 * np.sqrt(x / x.sum(axis=1, keepdims=True)))


def sift_pool(n: int, rng: np.random.Generator) -> np.ndarray:
    return _rootsift(rng.gamma(0.6, 1.0, size=(n, 128)) + 1e-6).astype(np.int16)


def positions(m: int, rng: np.random.Generator, generic: bool = True) -> np.ndarray:
    """(m,2) float32 feature positions. generic=True: all x distinct and all y distinct (Appendix B)."""
    if generic:
        x = rng.permutation(m).astype(np.float32) + np.float32(0.25)
        y = rng.permutation(m).astype(np.float32) + np.float32(0.5)
    else:  # adversarial: duplicated (x,y), equal-x and equal-y collisions
        x = rng.integers(0, max(m // 4, 2), m).astype(np.float32)
        y = rng.integers(0, max(m // 4, 2), m).astype(np.float32)
    return np.stack([x, y], axis=1)


def sift_images(n_images: int, m: int, dtype=np.uint8, seed: int = SEED_DATA, shared: float = 0.4, noise: int = 4,
                generic_positions: bool = True, pool_factor: float = 2.0):
    """Returns (descs, xys): lists of (m,128) ``dtype`` arrays and (m,2) float32 positions.

    Each image takes a seeded ~``shared`` fraction of a world pool (planted correspondences, +-noise per
    component) and fills up to ``m`` with fresh descriptors.
    """
    rng = np.random.Generator(np.random.PCG64(seed))
    pool = sift_pool(max(int(m * pool_factor), 8), rng)
    descs, xys = [], []
    for _ in range(n_images):
        k = min(int(m * (shared + rng.uniform(-0.1, 0.1))), m, pool.shape[0])
        sel = rng.choice(pool.shape[0], size=k, replace=False)
        a = pool[sel].astype(np.int16) + rng.integers(-noise, noise + 1, size=(k, 128), dtype=np.int16)
        a = np.clip(a, 0, 255)
        b = sift_pool(m - k, rng) if m > k else np.zeros((0, 128), np.int16)
        d = np.concatenate([a, np.clip(b, 0, 255)], axis=0)
        d = d[rng.permutation(m)]
        descs.append(np.ascontiguousarray(d.astype(dtype)))
        xys.append(positions(m, rng, generic_positions))
    return descs, xys


def real_valued(descs, seed: int = 1, sigma: float = 0.37):
    """Non-integer fp32 variant (exercises the exact, non-tensor-core path)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    return [np.ascontiguousarray((d.astype(np.float32) + rng.normal(0, sigma, d.shape).astype(np.float32))) for d in descs]


def mldb_images(n_images: int, m: int, seed: int = SEED_DATA, shared: float = 0.4, flip: float = 0.08, generic_positions: bool = True):
    """Returns (descs, xys): (m,64) uint8 binary descriptors (486 used bits) + positions."""
    rng = np.random.Generator(np.random.PCG64(seed ^ 0xB17))
    def rnd(n):
        bits = rng.integers(0, 2, size=(n, 512), dtype=np.uint8)
        bits[:, 486:] = 0
        return bits
    pool = rnd(max(2 * m, 8))
    descs, xys = [], []
    for _ in range(n_images):
        k = min(int(m * (shared + rng.uniform(-0.1, 0.1))), m)
        sel = rng.choice(pool.shape[0], size=k, replace=False)
        a = pool[sel] ^ (rng.random((k, 512)) < flip).astype(np.uint8)
        a[:, 486:] = 0
        bits = np.concatenate([a, rnd(m - k)], axis=0)[rng.permutation(m)]
        descs.append(np.ascontiguousarray(np.packbits(bits, axis=1, bitorder="little")))
        xys.append(positions(m, rng, generic_positions))
    return descs, xys


class IndexedImages:
    """Image k of a synthetic collection generated on its own (seeded by (seed, k)): a rank of a multi-GPU run builds only the
    views its shard references, and every rank sees the same image k.  Same recipe as sift_images / mldb_images: a shared world
    pool (planted correspondences, +-noise) plus fresh descriptors, general-position feature positions."""

    def __init__(self, m: int, kind: str = "f32", seed: int = SEED_DATA, shared: float = 0.4, noise: int = 4, flip: float = 0.08, real: bool = False):
        assert kind in ("f32", "u8", "bin")
        self.m, self.kind, self.seed, self.shared, self.noise, self.flip, self.real = m, kind, seed, shared, noise, flip, real
        rng = np.random.Generator(np.random.PCG64(seed))
        if kind == "bin":
            self.pool = rng.integers(0, 2, size=(max(2 * m, 8), 512), dtype=np.uint8)
            self.pool[:, 486:] = 0
        else:
            self.pool = sift_pool(max(m, 8), rng)

    def __call__(self, k: int):
        rng = np.random.Generator(np.random.PCG64([self.seed, 0x5EED, int(k)]))
        m = self.m
        n_shared = min(int(m * (self.shared + rng.uniform(-0.1, 0.1))), m, self.pool.shape[0])
        sel = rng.choice(self.pool.shape[0], size=n_shared, replace=False)
        if self.kind == "bin":
            a = self.pool[sel] ^ (rng.random((n_shared, 512)) < self.flip).astype(np.uint8)
            a[:, 486:] = 0
            b = rng.integers(0, 2, size=(m - n_shared, 512), dtype=np.uint8)
            b[:, 486:] = 0
            bits = np.concatenate([a, b], axis=0)[rng.permutation(m)]
            return np.ascontiguousarray(np.packbits(bits, axis=1, bitorder="little")), positions(m, rng)
        a = np.clip(self.pool[sel].astype(np.int16) + rng.integers(-self.noise, self.noise + 1, size=(n_shared, 128), dtype=np.int16), 0, 255)
        b = sift_pool(m - n_shared, rng) if m > n_shared else np.zeros((0, 128), np.int16)
        d = np.concatenate([a, np.clip(b, 0, 255)], axis=0)[rng.permutation(m)]
        d = np.ascontiguousarray(d.astype(np.float32 if self.kind == "f32" else np.uint8))
        if self.real and self.kind == "f32":
            d = np.ascontiguousarray(d + rng.normal(0, 0.37, d.shape).astype(np.float32))
        return d, positions(m, rng)


def exhaustive_pairs(n: int) -> np.ndarray:
    """Upper-triangular pair list (matchingImageCollection/pairBuilder.cpp:22-46 with ids 0..n-1)."""
    i, j = np.triu_indices(n, 1)
    return np.stack([i, j], axis=1).astype(np.uint32)


def voctree_like_pairs(n: int, k: int = 50, seed: int = SEED_PAIRS) -> np.ndarray:
    """Synthetic stand-in for a vocabulary-tree pair list (imageMatching/ImageMatching.cpp:233-284 +
    convertAllMatchesToPairList): k seeded neighbours per image, normalised to I<J, de-duplicated."""
    rng = np.random.Generator(np.random.PCG64(seed))
    s = set()
    for i in range(n):
        for j in rng.choice(n, size=min(k, n - 1), replace=False):
            if int(j) != i:
                s.add((min(i, int(j)), max(i, int(j))))
    return np.array(sorted(s), np.uint32).reshape(-1, 2)


def vocabulary_tree(k: int = 8, levels: int = 3, seed: int = 4, pool: np.ndarray | None = None, invalid_tail: int = 0):
    """A synthetic vocabulary tree in the reference's layout (voctree/VocabularyTree.hpp:139-146): node centers level by level,
    children of node i at (i+1)*k.., float centers.  Centers are SIFT-like descriptors (from `pool` or freshly drawn) with
    real-valued jitter, children scattered around their parent so that the descent is meaningful.  `invalid_tail` marks the
    last children of some nodes invalid (fewer than k children, :182-183)."""
    rng = np.random.default_rng(seed)
    n_nodes = sum(k ** (l + 1) for l in range(levels))
    base = sift_pool(max(k, 64), rng).astype(np.float32) if pool is None else np.asarray(pool, np.float32)
    centers = np.zeros((n_nodes, 128), np.float32)
    valid = np.ones(n_nodes, np.uint8)
    first = 0
    parents = None
    for l in range(levels):
        cnt = k ** (l + 1)
        if parents is None:
            c = base[rng.choice(len(base), cnt, replace=len(base) < cnt)] + rng.normal(0, 0.37, (cnt, 128)).astype(np.float32)
        else:
            spread = 24.0 / (l + 1)
            c = np.repeat(parents, k, axis=0) + rng.normal(0, spread, (cnt, 128)).astype(np.float32)
        centers[first:first + cnt] = np.maximum(c, 0)
        parents = centers[first:first + cnt]
        first += cnt
    if invalid_tail:
        start = 0
        for l in range(levels):
            cnt = k ** (l + 1)
            groups = cnt // k
            for g in rng.choice(groups, max(1, groups // 5), replace=False):
                valid[start + g * k + k - invalid_tail:start + (g + 1) * k] = 0
            start += cnt
    return centers, valid


def planar_views(n_views: int, n_points: int, planes: int = 2, dtype=np.uint8, seed: int = SEED_DATA, visible: float = 1.0,
                 fresh: float = 0.3, noise: int = 4, ring: bool = False):
    """A multi-plane scene seen by n_views cameras, for the homography-growing filter.  Returns (descs, feats): per view an (m,128)
    ``dtype`` array and an (m,4) float32 array of PointFeatures (x, y, scale, orientation).  Each world point lies on one of `planes`
    planes; view v maps plane p by its own homography, so every pair of views relates each plane by a homography, and each feature's
    scale and orientation follow that homography's local affinity.  A view sees a seeded `visible` fraction of the points (descriptor
    +-noise per component) and adds a `fresh` fraction of unrelated features.  ring=True: the points and the views lie on a circle and
    a view sees the points within a `visible` fraction of the circle around it, so only nearby views share points."""
    rng = np.random.Generator(np.random.PCG64(seed))
    pool = sift_pool(n_points, rng)
    plane = rng.integers(0, planes, n_points)
    base = np.c_[rng.uniform(0, 2000, (n_points, 2)), rng.uniform(1.5, 8, n_points), rng.uniform(-np.pi, np.pi, n_points)]
    angle = rng.uniform(0, 1, n_points)
    descs, feats = [], []
    for v in range(n_views):
        Hs = []
        for _ in range(planes):
            th, s = rng.uniform(-0.2, 0.2), rng.uniform(0.85, 1.15)
            Hs.append(np.array([[s * np.cos(th), -s * np.sin(th), rng.uniform(-150, 150)], [s * np.sin(th), s * np.cos(th), rng.uniform(-150, 150)],
                                [rng.uniform(-5e-5, 5e-5), rng.uniform(-5e-5, 5e-5), 1.0]]))
        if ring:
            d_ang = np.abs((angle - v / n_views + 0.5) % 1.0 - 0.5)
            sel = np.flatnonzero(d_ang < visible / 2)
        else:
            sel = np.flatnonzero(rng.uniform(0, 1, n_points) < visible)
        f = np.zeros((len(sel), 4))
        for r, i in enumerate(sel):
            H = Hs[plane[i]]
            x = np.array([base[i, 0], base[i, 1], 1.0])
            X = H @ x
            A = (H[:2, :2] * X[2] - np.outer(X[:2], H[2, :2])) / X[2] ** 2
            F = A @ (base[i, 2] * np.array([[np.cos(base[i, 3]), -np.sin(base[i, 3])], [np.sin(base[i, 3]), np.cos(base[i, 3])]]))
            f[r] = [X[0] / X[2], X[1] / X[2], np.sqrt(abs(np.linalg.det(F))), np.arctan2(F[1, 0] - F[0, 1], F[0, 0] + F[1, 1])]
        d = np.clip(pool[sel].astype(np.int16) + rng.integers(-noise, noise + 1, size=(len(sel), 128), dtype=np.int16), 0, 255)
        k = int(len(sel) * fresh)
        d = np.concatenate([d, np.clip(sift_pool(k, rng), 0, 255)])
        f = np.concatenate([f, np.c_[rng.uniform(0, 2000, (k, 2)), rng.uniform(1.5, 8, k), rng.uniform(-np.pi, np.pi, k)]])
        order = rng.permutation(len(d))
        descs.append(np.ascontiguousarray(d[order].astype(dtype)))
        feats.append(np.ascontiguousarray(f[order].astype(np.float32)))
    return descs, feats
