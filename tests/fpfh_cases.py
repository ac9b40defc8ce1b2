"""Point clouds with normals for the FPFH tests (registration.compute_fpfh_feature), each with the radius and max_nn it
is meant for (radius None: KNN only).

    scan        nc.scan's cloud with the oracle's estimated normals
    sphere      nc.sphere's patches with estimated normals
    clusters    tight clusters plus isolated points: a list with fewer than 2 entries gives a zero row
    duplicates  every point of a jittered plane twice: d2 == 0 entries are skipped, and a list's dropped first entry
                may be the point's lower twin rather than the point itself
    zero_normal a jittered plane with every third normal zero, which gives a zero pair feature
    lattice     an exact cubic lattice with axis normals: pair features land on bin edges
    offset      the scan moved by 1e4
"""
import numpy as np

from tests import normals_cases as nc
from tests.synth import make_icp_pair


def _points(r):
    return np.ascontiguousarray(r[0] if isinstance(r, tuple) else r, np.float32)


def _estimated(pts, radius, max_nn):
    from oracle import normals as on
    nrm, _, _ = on.estimate_normals(pts, radius, max_nn)
    return np.ascontiguousarray(nrm, np.float32)


def scan(n=6000, seed=31):
    pts = _points(nc.scan(n, seed))
    return pts, _estimated(pts, 0.05, 30)


def sphere():
    pts = _points(nc.sphere(patches=40))
    return pts, _estimated(pts, 0.06, 30)


def clusters(seed=32):
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-5, 5, (40, 3))
    pts = np.concatenate([c + rng.normal(scale=0.01, size=(60, 3)) for c in centres] +
                         [rng.uniform(-5, 5, (80, 3)) + 20.0]).astype(np.float32)
    nrm = rng.normal(size=pts.shape)
    return pts, (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(np.float32)


def duplicates(n=1500, seed=33):
    pts, nrm = nc.tilted_plane(n, seed)
    return np.repeat(pts, 2, axis=0).astype(np.float32), np.repeat(nrm, 2, axis=0).astype(np.float32)


def zero_normal(n=3000, seed=34):
    pts, nrm = nc.tilted_plane(n, seed)
    nrm = nrm.astype(np.float32)
    nrm[::3] = 0.0
    return pts.astype(np.float32), nrm


def lattice(side=14, spacing=0.125):
    g = np.arange(side, dtype=np.float64) * spacing
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    pts = np.stack([x.ravel(), y.ravel(), z.ravel()], 1).astype(np.float32)
    axes = np.eye(3, dtype=np.float32)
    return pts, axes[np.arange(len(pts)) % 3]


def offset():
    pts, nrm = scan(4000, 35)
    return (pts.astype(np.float64) + 1e4).astype(np.float32), nrm


def scan_2m():
    _, tgt, nrm, _ = make_icp_pair(2_000_000, seed=3)
    return tgt, nrm


# name -> (points, normals, radius, max_nn)
def cases():
    out = {}
    p, n = scan()
    out["scan_hybrid"] = (p, n, 0.05, 100)
    out["scan_knn30"] = (p, n, None, 30)
    out["scan_knn128"] = (p, n, None, 128)
    out["scan_hybrid4"] = (p, n, 0.05, 4)
    p, n = sphere()
    out["sphere"] = (p, n, 0.06, 100)
    p, n = clusters()
    out["clusters"] = (p, n, 0.03, 30)
    p, n = duplicates()
    out["duplicates"] = (p, n, 0.05, 30)
    p, n = zero_normal()
    out["zero_normal"] = (p, n, 0.05, 30)
    p, n = lattice()
    out["lattice"] = (p, n, 0.2, 100)
    p, n = offset()
    out["offset"] = (p, n, 0.08, 60)
    return out
