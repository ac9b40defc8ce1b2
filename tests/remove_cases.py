"""Point clouds for the clean-up filter tests (PointCloud.remove_radius_outliers, remove_duplicated_points and
remove_non_finite_points).

radius_cases()  name -> (points, [(nb_points, radius), ...]):
    scan        normals_cases.scan, 20 k points of a smooth height field at a spacing of about 0.02
    clusters    knn_cases.clusters: two dense clusters and 1 % isolated outliers
    offset      a 5 k scan moved by 1e4 along every axis, where an f32 ulp is about 1e-3
    lattice     exact_lattice(): the spacing equals the radius and every square is exact in f32
    ulp_pairs   ulp_pairs(): pairs whose distance lies within an ulp of the threshold
    coincident  groups of coincident points, each of which counts separately
scan_2m()       make_icp_pair(2 M points)'s target, for radius 0.02 and 0.05
exact_lattice() a 12^3 lattice of spacing 0.5 searched at radius 0.5: an axis neighbour's dist is exactly 0.25, the
                threshold, so it counts under upstream's <= (an interior point counts 7) and not under a strict <
ulp_pairs()     isolated pairs (p, q) of f32 points whose contracted and uncontracted dist fall on different sides of
                the threshold, for both orders of the outcome
duplicate_cases() name -> points: groups of 2..1000 copies at random indices, +-0.0, NaNs with equal and unequal
                payloads, a cloud that is one point repeated, a cloud without duplicates
non_finite_cloud() NaN, +inf and -inf in each coordinate, among finite points
"""
import numpy as np

from tests import knn_cases as kc
from tests import normals_cases as nc
from tests.synth import make_icp_pair


def exact_lattice(side=12, spacing=0.5):
    g = np.arange(side, dtype=np.float32) * np.float32(spacing)
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    return np.stack([x.ravel(), y.ravel(), z.ravel()], 1).astype(np.float32), spacing


def ulp_pairs(radius=0.7, want=64, seed=5):
    """Pairs on a 40^3 grid of spacing 3 around the origin, each p at the radius from its q up to a few ulps: both
    outcomes of the contraction, `want` pairs each at most.  The coordinates stay within 90 radii of the origin, so
    the f32 rounding of p spreads the pairs' dist over about a hundred ulps of the threshold, and some land within
    one."""
    from oracle import remove as orm
    rng = np.random.default_rng(seed)
    g = (np.arange(40, dtype=np.float64) - 20) * 3
    base = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    m = len(base)
    q = (base + rng.uniform(0, 0.3, (m, 3))).astype(np.float32)
    d = rng.normal(size=(m, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    p = (q.astype(np.float64) + d * radius * (1 + rng.uniform(-1e-7, 1e-7, (m, 1)))).astype(np.float32)
    pts = np.empty((2 * m, 3), np.float32)
    pts[0::2], pts[1::2] = q, p
    cuda = orm.radius_counts(pts, radius, "cuda")[0::2] == 2
    plain = orm.radius_counts(pts, radius, "plain")[0::2] == 2
    keep = np.concatenate([np.flatnonzero(cuda & ~plain)[:want], np.flatnonzero(plain & ~cuda)[:want]])
    keep.sort()
    out = np.empty((2 * len(keep), 3), np.float32)
    out[0::2], out[1::2] = q[keep], p[keep]
    return out, radius


def coincident(seed=3):
    rng = np.random.default_rng(seed)
    centres = rng.uniform(0, 1, (200, 3)).astype(np.float32)
    reps = rng.integers(1, 9, 200)
    pts = np.repeat(centres, reps, axis=0)
    return pts[rng.permutation(len(pts))]


def radius_cases():
    scan = nc.scan()
    offset = nc.scan(5000, seed=8) + np.float32(1e4)
    lat, s = exact_lattice()
    ulp, r = ulp_pairs()
    return {
        "scan": (scan, [(1, 0.02), (2, 0.02), (6, 0.02), (16, 0.05), (64, 0.05), (len(scan) + 1, 0.05)]),
        "clusters": (kc.clusters(), [(2, 0.05), (8, 0.05), (30, 0.2)]),
        "offset": (offset, [(4, 0.05), (16, 0.08)]),
        "lattice": (lat, [(7, s), (8, s), (1, s)]),
        "ulp_pairs": (ulp, [(2, r)]),
        "coincident": (coincident(), [(1, 1e-3), (3, 1e-3), (8, 1e-3)]),
    }


def scan_2m():
    _, tgt, _, _ = make_icp_pair(2_000_000, seed=3)
    return tgt


def _groups(n=20000, seed=9):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    src = rng.choice(n, 40, replace=False)
    sizes = np.concatenate([[2, 3, 1000], rng.integers(2, 50, 37)])
    for s, k in zip(src, sizes):
        pts[rng.choice(n, k - 1, replace=False)] = pts[s]
    return pts


def _signed_zeros():
    v = np.float32([0.0, -0.0])
    g = np.stack(np.meshgrid(v, v, v, indexing="ij"), -1).reshape(-1, 3)
    return np.concatenate([g, g[::-1], g]).astype(np.float32)


def _nans():
    bits = np.array([0x7FC00000, 0x7FC00001, 0xFFC00000, 0x7F800001, 0x7FC00000, 0x7FC00001], np.uint32)
    nan = bits.view(np.float32)
    pts = np.zeros((len(nan) * 2, 3), np.float32)
    pts[: len(nan), 0] = nan
    pts[len(nan):, 1] = nan
    pts[len(nan):, 0] = 1.0
    return np.concatenate([pts, pts[::-1]])


def duplicate_cases():
    rng = np.random.default_rng(4)
    return {
        "groups": _groups(),
        "signed_zeros": _signed_zeros(),
        "nans": _nans(),
        "one_point": np.tile(np.float32([0.25, -1.5, 3.0]), (5000, 1)),
        "distinct": rng.uniform(0, 1, (30000, 3)).astype(np.float32),
        "single": np.float32([[1.0, 2.0, 3.0]]),
    }


def duplicated_2m(frac=0.1, seed=6):
    """scan_2m() with 10 % of its points overwritten by copies of others."""
    pts = scan_2m().copy()
    rng = np.random.default_rng(seed)
    n = len(pts)
    k = int(n * frac)
    pts[rng.choice(n, k, replace=False)] = pts[rng.integers(0, n, k)]
    return pts


def non_finite_cloud():
    vals = np.float32([np.nan, np.inf, -np.inf])
    rows = []
    for a in range(3):
        for v in vals:
            r = np.float32([0.5, -0.25, 2.0])
            r[a] = v
            rows.append(r)
    rows.append(np.float32([np.nan, np.inf, 1.0]))
    rows.append(np.float32([-np.inf, 0.0, np.nan]))
    pts = np.concatenate([np.stack(rows), np.random.default_rng(2).uniform(-1, 1, (50, 3)).astype(np.float32)])
    return pts[np.random.default_rng(3).permutation(len(pts))]
