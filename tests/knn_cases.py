"""Point clouds for the k-nearest-neighbour tests (NearestNeighborSearch.knn_search, remove_statistical_outliers,
compute_metrics).  Each case is (dataset, queries); the queries are the dataset itself unless stated.

    scan       make_icp_pair's noisy source cloud, 20 k points (a smooth height field)
    uniform    20 k points uniform in the unit cube
    lattice    the 10 x 10 x 10 integer lattice: every shell of neighbours is a set of exactly equal distances, so
               the k-th neighbour is decided by the lower-index rule whenever k cuts a shell
    duplicates normals_cases.duplicates: groups of coincident points
    sparse     normals_cases.sparse: clusters of 1..4 points one unit apart
    clusters   two dense 1-unit clusters 100 units apart, plus 1 % uniform outliers in a box 50 times the clusters'
               size: density ratios of about 10^6
    line       normals_cases.line: points along one direction
    offset     a 5 k scan moved by 1e4 along every axis
    external   the scan searched from queries about 1e3 outside its bounding box
"""
import numpy as np

from tests import normals_cases as nc


def uniform(n=20000, seed=11):
    return np.random.default_rng(seed).uniform(0, 1, (n, 3)).astype(np.float32)


def lattice(side=10):
    g = np.arange(side, dtype=np.float32)
    z, y, x = np.meshgrid(g, g, g, indexing="ij")
    return np.stack([x.ravel(), y.ravel(), z.ravel()], 1).astype(np.float32)


def clusters(n=20000, seed=12):
    rng = np.random.default_rng(seed)
    a = rng.uniform(0, 1, (n // 2, 3))
    b = rng.uniform(0, 1, (n // 2, 3)) + [100.0, 0.0, 0.0]
    out = rng.uniform([-25.0, -25.0, -25.0], [125.0, 25.0, 25.0], (n // 100, 3))
    p = np.concatenate([a, b, out])
    return p[rng.permutation(len(p))].astype(np.float32)


def external(seed=13):
    data = nc.scan(5000, seed=7)
    rng = np.random.default_rng(seed)
    lo, hi = data.min(0), data.max(0)
    dirs = rng.normal(size=(500, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    q = (lo + hi) / 2 + dirs * (1e3 + np.linalg.norm(hi - lo))
    return data, q.astype(np.float32)


def cases():
    scan = nc.scan()
    return {
        "scan": (scan, scan),
        "uniform": (uniform(), uniform()),
        "lattice": (lattice(), lattice()),
        "duplicates": (nc.duplicates(), nc.duplicates()),
        "sparse": (nc.sparse(), nc.sparse()),
        "clusters": (clusters(), clusters()),
        "line": (nc.line(), nc.line()),
        "offset": (nc.scan(5000, seed=8) + np.float32(1e4), nc.scan(5000, seed=8) + np.float32(1e4)),
        "external": external(),
    }
