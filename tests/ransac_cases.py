"""Inputs for the RANSAC registration tests (registration_ransac_based_on_correspondence).  Deterministic in seed.

    pair(n, ratio)   a source cloud, a target that is the source moved by a known rigid motion with a little noise,
                     and n correspondences of which a fraction `ratio` are true (i, i) pairs and the rest random
    ties             a target with every point duplicated, so that every match ties between two indices
    scene            a height field with six bumps (tests/synth.py's surface), for the global registration pipeline
    overlap_pair     two 80 % parts of a scene overlapping by 60 %, the second turned 100 degrees about an oblique
                     axis, shifted and given noise
    radius_probes    an estimate that is exactly the identity, with probe points at the distance, one ulp inside and
                     one ulp outside it
"""
import numpy as np

from tests.synth import axis_angle


def motion(deg=35.0, axis=(1.0, 2.0, 0.5), shift=(0.3, -0.2, 0.1)):
    T = np.eye(4)
    T[:3, :3] = axis_angle(axis, deg)
    T[:3, 3] = shift
    return T


def cloud(n, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(-1.0, 1.0, (n, 3)).astype(np.float32)


def normals(n, seed):
    rng = np.random.default_rng(seed + 1000)
    v = rng.normal(size=(n, 3))
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def pair(n, k, ratio, seed, noise=0.002):
    """(source, target, corres [k, 2] int64, true T): target = T source + noise, the first round(k ratio) pairs true."""
    rng = np.random.default_rng(seed)
    src = cloud(n, seed)
    T = motion()
    tgt = (src.astype(np.float64) @ T[:3, :3].T + T[:3, 3] + rng.normal(0, noise, (n, 3))).astype(np.float32)
    good = int(round(k * ratio))
    a = rng.choice(n, k, replace=k > n)
    b = a.copy()
    b[good:] = rng.integers(0, n, k - good)
    c = np.stack([a, b], 1).astype(np.int64)
    return src, tgt, c[rng.permutation(k)], T


def ties(n, seed):
    src, tgt, c, T = pair(n, n // 2, 0.5, seed)
    tgt2 = np.concatenate([tgt, tgt]).astype(np.float32)
    return src, tgt2, c, T


def scene(n_side, spacing, seed):
    from tests.synth import _jittered_lattice, _surface
    rng = np.random.default_rng(seed)
    x, y = _jittered_lattice(n_side, spacing, rng)
    z, _ = _surface(x, y)
    for cx, cy, h, w in ((1.0, 0.6, 0.15, 0.05), (0.4, 1.9, -0.1, 0.08), (2.2, 2.3, 0.2, 0.03), (1.6, 1.4, 0.12, 0.02),
                         (0.7, 0.3, -0.08, 0.04), (2.5, 0.8, 0.1, 0.06)):
        z = z + h * np.exp(-((x - cx) ** 2 + (y - cy) ** 2) / w)
    return np.stack([x, y, z], 1)


def overlap_pair(pts, seed, noise=0.002):
    """(source, target, true T) with target = T (part of pts) + noise."""
    L = pts[:, 0].max()
    T = motion(100.0, (1.0, -0.6, 0.8), (0.5, -0.3, 1.2))
    rng = np.random.default_rng(seed)
    src = pts[pts[:, 0] < 0.8 * L]
    tp = pts[pts[:, 0] > 0.2 * L]
    return src, tp @ T[:3, :3].T + T[:3, 3] + rng.normal(0, noise, tp.shape), T


RADIUS = 0.25


def radius_probes(r=RADIUS):
    """(source, target, corres, expected [n] correspondence set) for ransac_n 4 on the four anchor pairs, whose
    estimate is exactly the identity: anchors (+-2, 0, 0), (0, +-1, 0) give means 0 and a diagonal cross-covariance
    (2, 0.5, 0) of powers of two, so the Kabsch rotation is exactly I and t exactly 0.  Each probe is a source point
    with one target point moved from it along one axis by exactly r (no match: the test is strict), by r less one f32
    ulp of the coordinate (a match) and by r plus one ulp (no match), at coordinates 5, 1000 and -30000 so that the
    query's rounding to f32 and the widened search box matter.  Any sample of the four anchor indices in any order
    gives the same estimate only when it is a permutation of them."""
    anchors = np.array([[2, 0, 0], [-2, 0, 0], [0, 1, 0], [0, -1, 0]], np.float32)
    src, tgt = [anchors], [anchors]
    expect = list(range(4))
    k = 4
    for ci, c in enumerate((5.0, 1000.0, -30000.0)):
        for axis in range(3):
            for kind in ("at", "inside", "outside"):
                p = np.full(3, c, np.float32)
                p[(axis + 1) % 3] += np.float32(20 * (3 * axis + ("at", "inside", "outside").index(kind)))
                q = p.copy()
                edge = np.float32(p[axis] + np.float32(r))   # exact: r and every c are dyadic
                assert float(edge) - float(p[axis]) == r
                if kind == "inside":
                    edge = np.nextafter(edge, p[axis])
                elif kind == "outside":
                    edge = np.nextafter(edge, np.float32(np.inf) if edge > p[axis] else np.float32(-np.inf))
                q[axis] = edge
                src.append(p[None])
                tgt.append(q[None])
                d = (p.astype(np.float64) - q.astype(np.float64))
                d2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
                assert (d2 < r * r) == (kind == "inside"), (c, axis, kind, d2)
                expect.append(k if kind == "inside" else -1)
                k += 1
    corres = np.stack([np.arange(4), np.arange(4)], 1).astype(np.int64)
    return np.concatenate(src), np.concatenate(tgt), corres, np.array(expect, np.int64)
