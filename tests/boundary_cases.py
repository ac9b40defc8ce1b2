"""Point clouds with normals for the boundary-detection tests (PointCloud.compute_boundary_points), each with the
search radius and max_nn it is meant for.

    normals_<name>  every cloud of tests/normals_cases.py, with the oracle's estimated normals
    special_normals a jittered plane whose normals include exactly (0, 0, +-1), zero normals, NaN components and
                    normals within 1e-6 of the x = y = z diagonal (the frame's second branch)
    lattice4        an exact xz-plane lattice with normal (0, 1, 0) and a radius that catches only the 4 axis
                    neighbours: u = (0, -0, 1), v = (-1, 0, 0), so every gap of an interior point is f32(pi/2), which
                    is above pi/2, and every interior point is a boundary point at 90 degrees
    duplicates2     every point of a jittered plane twice: the higher index's list starts with its lower twin, so the
                    point itself is among the kept neighbours with d = 0 and an angle of +-0 or +-pi
    single          isolated pairs of points: one kept neighbour each
    scan_200k       make_icp_pair(200_000, spacing=0.005)'s target with its analytic normals, at radius 0.02
"""
import math

import numpy as np

from tests import normals_cases as nc
from tests.synth import make_icp_pair


def _estimated(pts, radius, max_nn):
    from oracle import normals as on
    nrm, _, _ = on.estimate_normals(pts, radius, max_nn)
    return nrm


def special_normals(n=3000, seed=21):
    pts, nrm = nc.tilted_plane(n, seed)
    nrm = nrm.astype(np.float32)
    nrm[0::11] = (0.0, 0.0, 1.0)
    nrm[1::11] = (0.0, 0.0, -1.0)
    nrm[2::11] = 0.0
    nrm[3::11, 1] = np.nan
    d = np.float32(1 / math.sqrt(3))
    nrm[4::11] = (d, d, d)
    nrm[5::11] = (d, np.nextafter(d, np.float32(1)), d)
    nrm[6::11] = (-d, -d, -d)
    return pts, nrm


def lattice4(side=24, spacing=1 / 16):
    g = np.arange(side, dtype=np.float64) * spacing
    a, b = np.meshgrid(g, g)
    pts = np.stack([a.ravel(), np.full(a.size, 0.25), b.ravel()], 1).astype(np.float32)
    nrm = np.tile(np.float32([0.0, 1.0, 0.0]), (len(pts), 1))
    return pts, nrm, 1.2 * spacing


def duplicates2(n=1500, seed=22):
    pts, nrm = nc.tilted_plane(n, seed)
    return np.repeat(pts, 2, axis=0), np.repeat(nrm, 2, axis=0).astype(np.float32)


def single(pairs=100, seed=23):
    rng = np.random.default_rng(seed)
    base = np.stack([np.arange(pairs) * 1.0, np.zeros(pairs), np.zeros(pairs)], 1)
    pts = np.concatenate([base, base + rng.uniform(-0.01, 0.01, (pairs, 3))]).astype(np.float32)
    nrm = rng.normal(size=(len(pts), 3))
    return pts, (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(np.float32)


def scan_200k():
    _, tgt, nrm, _ = make_icp_pair(200_000, seed=2, spacing=0.005)
    return tgt, nrm


# name -> (points, normals, radius, max_nn)
def cases():
    out = {}
    for name, (pts, radius, max_nn) in nc.cases().items():
        out[f"normals_{name}"] = (pts, _estimated(pts, radius, max_nn), radius, max_nn)
    out["special_normals"] = (*special_normals(), 0.05, 30)
    pts, nrm, r = lattice4()
    out["lattice4"] = (pts, nrm, r, 30)
    out["duplicates2"] = (*duplicates2(), 0.06, 30)
    out["single"] = (*single(), 0.05, 30)
    return out


def random_normals(n=10000, seed=24):
    """unit normals, with every 10th one within float rounding of an axis or of the x = y = z diagonal"""
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(n, 3))
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    v = v.astype(np.float32)
    d = np.float32(1 / math.sqrt(3))
    k = np.arange(0, n, 10)
    v[k] = np.array([[d, d, d], [0, 0, 1], [0, 1, 0], [1, 0, 0], [-d, -d, -d]], np.float32)[np.arange(len(k)) % 5]
    v[k] += rng.integers(-2, 3, (len(k), 3)).astype(np.float32) * np.float32(2 ** -24)
    return v
