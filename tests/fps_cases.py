"""Clouds and reference loops for the farthest-point down-sampling tests (PointCloud.farthest_point_down_sample).

    numpy_fps   upstream's tensor loop (t/geometry/PointCloud.cpp:633-645) restated in numpy f32 with its op order, the
                argmax taken over the points not yet selected, ties to the lowest index
    legacy_fps  the legacy geometry::PointCloud::FarthestPointDownSample (geometry/PointCloud.cpp:543-554) in f64: a
                strict > scan, so ties go to the lowest index
    integer_cloud  distinct integer points with |coordinate| < 2^10: every squared distance is below 2^24, exact in f32
                   and f64 alike, so the two loops above select the same points
    coincident  a few distinct positions, each repeated many times: fewer distinct positions than samples
    overflow    coordinates near 1e19, whose squared distances overflow f32 to +inf
"""
import numpy as np

from tests import knn_cases as kc


def numpy_fps(points, num_samples, start_index=0):
    p = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    d = np.full(p.shape[0], np.inf, np.float32)
    taken = np.zeros(p.shape[0], bool)
    f = int(start_index)
    out = []
    for r in range(num_samples):
        out.append(f)
        taken[f] = True
        if r + 1 == num_samples:
            break
        diff = p - p[f]
        sq = diff * diff
        e = (sq[:, 0] + sq[:, 1]) + sq[:, 2]
        d = np.minimum(d, e)
        f = int(np.argmax(np.where(taken, np.float32(-1), d)))
    return np.asarray(out, np.int32)


def legacy_fps(points, num_samples, start_index=0):
    p = np.asarray(points, np.float64).reshape(-1, 3)
    d = np.full(p.shape[0], np.inf)
    f = int(start_index)
    out = []
    for _ in range(num_samples):
        out.append(f)
        diff = p - p[f]
        d = np.minimum(d, (diff * diff).sum(1))
        if d.max() > 0:
            f = int(np.argmax(d))
    return np.asarray(out, np.int32)


def integer_cloud(n, seed):
    rng = np.random.default_rng(seed)
    p = np.unique(rng.integers(-1023, 1024, (n, 3)), axis=0)
    return p[rng.permutation(len(p))].astype(np.float32)


def coincident(distinct=12, copies=40, seed=21):
    rng = np.random.default_rng(seed)
    pos = rng.uniform(0, 1, (distinct, 3))
    p = np.repeat(pos, copies, axis=0)
    return p[rng.permutation(len(p))].astype(np.float32)


def overflow(n=4000, seed=22):
    rng = np.random.default_rng(seed)
    p = rng.uniform(-1.0, 1.0, (n, 3))
    far = rng.random(n) < 0.3
    p[far] *= 3e19
    return p.astype(np.float32)


def external():
    data, queries = kc.external()
    return np.concatenate([data, queries]).astype(np.float32)


def fixtures():
    """The k-NN fixtures as single clouds: the dataset, and for "external" the dataset with its far queries."""
    return {name: (external() if name == "external" else data) for name, (data, _) in kc.cases().items()}
