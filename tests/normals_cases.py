"""Point clouds for the normal-estimation tests (PointCloud.estimate_normals), each with the search radius and
max_nn it is meant for and, where the surface is known, the analytic normal of the points it holds for.

    scan        make_icp_pair's noisy source cloud (a smooth height field, 0.5 mm noise)
    axis_planes three exact 5x5 dyadic grids, one normal to each axis: every point sees its whole grid, whose
                off-diagonal cumulants are exactly zero, so the eigen solve takes its diagonal branch and returns
                (1,0,0), (0,1,0) and (0,0,1) in turn
    tilted      a jittered square of the plane with normal (1, 2, 3) / |.|
    sphere      200 patches of a sphere of radius 0.8; each patch is a 5x5 square stencil mapped onto the sphere
                around its centre, so that the centre's neighbourhood is symmetric and its normal is radial
    line        points along one direction: a rank-1 covariance
    duplicates  groups of coincident points: a zero covariance (max_coeff == 0)
    sparse      isolated points, pairs, triples and quadruples: 1, 2, 3 and 4 neighbours
"""
import math

import numpy as np

from tests.synth import make_icp_pair


def _dyadic_grid(axis, offset):
    g = np.arange(-2, 3, dtype=np.float64) / 16.0   # exact in f32 and f64, and so is every sum over the grid
    a, b = np.meshgrid(g, g)
    p = np.zeros((25, 3))
    others = [k for k in range(3) if k != axis]
    p[:, others[0]] = a.ravel()
    p[:, others[1]] = b.ravel()
    return p + np.asarray(offset, np.float64)


def axis_planes():
    parts, nrm = [], []
    for axis, off in ((0, (0.0, 0.0, 0.0)), (1, (4.0, 0.0, 0.0)), (2, (0.0, 4.0, 0.0))):
        parts.append(_dyadic_grid(axis, off))
        nrm.append(np.tile(np.eye(3)[axis], (25, 1)))
    return np.concatenate(parts).astype(np.float32), np.concatenate(nrm)


def tilted_plane(n=4000, seed=3):
    rng = np.random.default_rng(seed)
    nz = np.array([1.0, 2.0, 3.0]) / math.sqrt(14.0)
    e1 = np.cross(nz, [1.0, 0.0, 0.0])
    e1 /= np.linalg.norm(e1)
    e2 = np.cross(nz, e1)
    st = rng.uniform(-0.5, 0.5, (n, 2))
    p = np.array([0.3, -0.2, 0.5]) + st[:, :1] * e1 + st[:, 1:] * e2
    return p.astype(np.float32), np.tile(nz, (n, 1))


def sphere(patches=200, R=0.8, step=0.02):
    """-> (points, analytic normals, index of every patch centre)"""
    k = np.arange(patches) + 0.5
    phi = np.arccos(1 - 2 * k / patches)
    th = math.pi * (1 + 5 ** 0.5) * k
    dirs = np.stack([np.cos(th) * np.sin(phi), np.sin(th) * np.sin(phi), np.cos(phi)], 1)
    g = np.arange(-2, 3) * step
    s, t = (a.ravel() for a in np.meshgrid(g, g))
    c = np.array([0.1, -0.3, 0.2])
    pts, centres = [], []
    for u in dirs:
        e1 = np.cross(u, [0.0, 0.0, 1.0] if abs(u[2]) < 0.9 else [1.0, 0.0, 0.0])
        e1 /= np.linalg.norm(e1)
        e2 = np.cross(u, e1)
        q = u + (s[:, None] * e1 + t[:, None] * e2) / R
        centres.append(len(pts) * 25 + 12)
        pts.append(c + R * q / np.linalg.norm(q, axis=1, keepdims=True))
    p = np.concatenate(pts).astype(np.float32)
    an = p.astype(np.float64) - c
    return p, an / np.linalg.norm(an, axis=1, keepdims=True), np.array(centres)


def line(n=500, seed=4):
    rng = np.random.default_rng(seed)
    d = np.array([0.6, -0.48, 0.64])
    return (np.array([0.2, 0.1, -0.3]) + rng.uniform(-1, 1, (n, 1)) * d).astype(np.float32)


def duplicates(groups=40, copies=(1, 2, 3, 5, 12), seed=5):
    rng = np.random.default_rng(seed)
    out = []
    for g in range(groups):
        out.append(np.tile(rng.uniform(-1, 1, 3) + [3.0 * g, 0.0, 0.0], (copies[g % len(copies)], 1)))
    return np.concatenate(out).astype(np.float32)


def sparse(seed=6):
    """clusters of 1..4 points, 0.01 apart inside a cluster and 1 apart between clusters"""
    rng = np.random.default_rng(seed)
    out = []
    for g in range(80):
        size = 1 + g % 4
        base = np.array([g * 1.0, 0.5, -0.5])
        out.append(base + rng.uniform(-0.01, 0.01, (size, 3)))
    return np.concatenate(out).astype(np.float32)


def scan(n=20000, seed=7):
    src, _, _, _ = make_icp_pair(n, seed=seed)
    return src


# name -> (points, radius, max_nn)
def cases():
    sph, _, _ = sphere()
    return {
        "scan": (scan(), 0.08, 30),
        "scan_knn8": (scan(), 0.05, 8),
        "axis_planes": (axis_planes()[0], 0.5, 30),
        "tilted": (tilted_plane()[0], 0.05, 32),
        "sphere": (sph, 0.06, 30),
        "line": (line(), 0.05, 30),
        "duplicates": (duplicates(), 0.1, 8),
        "sparse": (sparse(), 0.05, 3),
        "sparse_knn32": (sparse(), 0.05, 32),
    }
