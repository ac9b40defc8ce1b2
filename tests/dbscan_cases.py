"""Point clouds and parameters for the DBSCAN tests (PointCloud.cluster_dbscan).

fixtures()      the clouds of knn_cases (scan, uniform, lattice, duplicates, sparse, clusters, line, offset)
eps_grid(p)     (eps, min_points) pairs for a cloud, from its typical nearest-neighbour spacing d: eps = d / 2, where
                most points have no neighbour but themselves and are noise; 1.5 d and 4 d; and an eps above the
                cloud's diagonal, where every point is every point's neighbour and one cluster spans the cloud
constructed()   the boundary cases: a power-of-two lattice at eps equal to its spacing (no neighbours: d2 == eps^2)
                and at the next double above it; a border point between two clusters in both index orders;
                min_points 0, 1 and above n; many coincident points
"""
import numpy as np

from tests import knn_cases as kc

FIXTURES = ("scan", "uniform", "lattice", "duplicates", "sparse", "clusters", "line", "offset")


def fixtures():
    cases = kc.cases()
    return {name: np.ascontiguousarray(cases[name][0], np.float32) for name in FIXTURES}


def spacing(p):
    """The median distance from a point to its nearest other point (coincident points skipped), in f64."""
    from oracle import knn as ok
    _, d2 = ok.knn(p, p, 8)
    d = np.sqrt(d2.astype(np.float64))
    d = np.where(d > 0, d, np.inf).min(1)
    d = d[np.isfinite(d)]
    return float(np.median(d)) if d.size else 1.0


def eps_grid(p):
    d = spacing(p)
    diag = float(np.linalg.norm(p.max(0).astype(np.float64) - p.min(0).astype(np.float64)))
    grid = [(e * d, m) for e in (0.5, 1.5, 4.0) for m in (1, 4, 12)]
    grid.append((diag * 1.01 + d, 4))
    return grid


def pow2_lattice(side=8, step=0.25):
    g = np.arange(side, dtype=np.float32) * np.float32(step)
    z, y, x = np.meshgrid(g, g, g, indexing="ij")
    return np.stack([x.ravel(), y.ravel(), z.ravel()], 1).astype(np.float32)


def two_clusters_and_a_border(border_first=True, a_first=False):
    """1-D runs A = 0.00..0.30 and C = 0.50..0.80 (step 0.05) and b = 0.40.  At eps 0.12 and min_points 4 every point
    of A and C is core, and b (neighbours 0.30, 0.50 and itself) is not, so b takes the lower of the two cluster ids.
    -> (points, expected labels)."""
    a = np.round(np.arange(7) * 0.05, 2)
    c = np.round(0.5 + np.arange(7) * 0.05, 2)
    runs = [a, c] if a_first else [c, a]
    xs = np.concatenate(([0.40], *runs) if border_first else (*runs, [0.40]))
    p = np.zeros((len(xs), 3), np.float32)
    p[:, 0] = xs
    off = 1 if border_first else 0
    want = np.zeros(len(xs), np.int32)   # the border point and the first run: cluster 0
    want[off + 7:off + 14] = 1
    return p, want


def coincident(seed=21):
    """2 000 copies of one point, 300 copies of another 0.05 away, and 200 scattered points around them."""
    rng = np.random.default_rng(seed)
    p = np.concatenate([np.tile([[0.3, 0.3, 0.3]], (2000, 1)), np.tile([[0.35, 0.3, 0.3]], (300, 1)),
                        rng.uniform(0, 1, (200, 3))])
    return p[rng.permutation(len(p))].astype(np.float32)


def constructed():
    """-> {name: (points, eps, min_points, expected labels or None)}"""
    lat = pow2_lattice()
    n = len(lat)
    out = {
        "lattice at eps = spacing": (lat, 0.25, 2, np.full(n, -1, np.int32)),
        "lattice above spacing": (lat, float(np.nextafter(0.25, 1.0)), 2, np.zeros(n, np.int32)),
        "lattice min_points 0": (lat, 0.25, 0, np.arange(n, dtype=np.int32)),
        "lattice min_points 1": (lat, 0.25, 1, np.arange(n, dtype=np.int32)),
        "lattice min_points above n": (lat, 100.0, n + 1, np.full(n, -1, np.int32)),
        "lattice min_points n": (lat, 100.0, n, np.zeros(n, np.int32)),
        "coincident": (coincident(), 0.02, 50, None),
        "coincident joined": (coincident(), 0.06, 50, None),
    }
    for border_first in (True, False):
        for a_first in (True, False):
            p, want = two_clusters_and_a_border(border_first, a_first)
            out[f"border {'first' if border_first else 'last'} {'A' if a_first else 'C'} first"] = (p, 0.12, 4, want)
    return out
