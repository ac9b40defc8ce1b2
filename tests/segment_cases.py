"""Clouds for the RANSAC plane segmentation tests (PointCloud.segment_plane).  Deterministic in (size, seed).

    single_plane   points on z = 0.3x - 0.2y + 0.5 (rounded to f32) plus uniform outliers: every sample of three
                   plane points gives the same inlier set, so the best fitness is known and the early stop can be
                   placed (wave_boundary_probability)
    multi_plane    three planes of different sizes and uniform outliers
    noisy          a plane with Gaussian noise of about the threshold, and outliers
    collinear      every point on one line: every hypothesis is degenerate
    scene          tests/synth.py's height field, a floor plane and uniform outliers
"""
import math

import numpy as np

from tests.synth import _surface

THRESHOLD = 0.01


def _outliers(rng, m):
    return rng.uniform(-1.0, 1.0, (m, 3))


def _shuffle(rng, parts):
    p = np.concatenate(parts).astype(np.float32)
    return p[rng.permutation(p.shape[0])]


def single_plane(n, seed, on_plane=0.6):
    rng = np.random.default_rng(seed)
    k = int(round(n * on_plane))
    x, y = rng.uniform(-1, 1, k), rng.uniform(-1, 1, k)
    plane = np.stack([x, y, 0.3 * x - 0.2 * y + 0.5], 1)
    # outliers at least 0.1 off the plane, far outside the threshold
    o = _outliers(rng, n - k)
    o[:, 2] = 0.3 * o[:, 0] - 0.2 * o[:, 1] + 0.5 + np.where(rng.random(n - k) < 0.5, -1, 1) * rng.uniform(0.1, 1, n - k)
    return _shuffle(rng, [plane, o])


def multi_plane(n, seed):
    rng = np.random.default_rng(seed)
    a, b, c = int(0.4 * n), int(0.3 * n), int(0.2 * n)
    u = rng.uniform(-1, 1, (a + b + c, 2))
    p1 = np.stack([u[:a, 0], u[:a, 1], np.full(a, -0.5)], 1)
    p2 = np.stack([np.full(b, 0.7), u[a:a + b, 0], u[a:a + b, 1]], 1)
    w = u[a + b:]
    p3 = np.stack([w[:, 0], 0.5 * w[:, 0] + 0.1, w[:, 1]], 1)
    return _shuffle(rng, [p1, p2, p3, _outliers(rng, n - a - b - c)])


def noisy(n, seed):
    rng = np.random.default_rng(seed)
    k = int(0.7 * n)
    x, y = rng.uniform(-1, 1, k), rng.uniform(-1, 1, k)
    z = -0.1 * x + 0.4 * y - 0.2 + rng.normal(0, THRESHOLD, k)
    return _shuffle(rng, [np.stack([x, y, z], 1), _outliers(rng, n - k)])


def collinear(n, seed):
    rng = np.random.default_rng(seed)
    t = rng.integers(-1000, 1000, n).astype(np.float64)
    return np.stack([t, 2 * t, -t], 1).astype(np.float32)   # exact in f32: every cross product is exactly zero


def scene(n, seed):
    rng = np.random.default_rng(seed)
    h, f = int(0.5 * n), int(0.4 * n)
    x, y = rng.uniform(-2, 2, h), rng.uniform(-2, 2, h)
    z, _ = _surface(x, y)
    floor = np.stack([rng.uniform(-2, 2, f), rng.uniform(-2, 2, f), rng.normal(-0.6, 0.002, f)], 1)
    return _shuffle(rng, [np.stack([x, y, z], 1), floor, 2 * _outliers(rng, n - h - f)])


def wave_boundary_probability(n, on_plane=0.6, ransac_n=3, brk=127):
    """A probability for which single_plane(n, ., on_plane)'s best fitness k/n gives break = brk, with the quotient
    half-way between brk and brk + 1."""
    f = int(round(n * on_plane)) / n
    return -math.expm1((brk + 0.5) * math.log1p(-f ** ransac_n))
