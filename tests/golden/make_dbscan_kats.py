"""Writes tests/golden/dbscan_kats.json: the labels the reference's own geometry::PointCloud::ClusterDBSCAN
(oracle/_ref/libo3dref_dbscan.so, built by oracle/ref_shim_dbscan from the reference sources) gives on small seeded
clouds, so that the GPU tests need no reference tree.

Upstream's own known answer (cpp/tests/t/geometry/PointCloud.cpp:1534-1555: fragment.ply, 196 133 points, 11 labels
summing to 398 580) needs a dataset download and is not used.

    python tests/golden/make_dbscan_kats.py
"""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests import dbscan_cases as dc  # noqa: E402


def blobs(seed=31):
    """Three Gaussian blobs of different spreads and 10 % uniform noise."""
    rng = np.random.default_rng(seed)
    p = np.concatenate([rng.normal([0, 0, 0], 0.05, (300, 3)), rng.normal([1, 0, 0], 0.1, (300, 3)),
                        rng.normal([0, 1, 0.5], 0.02, (150, 3)), rng.uniform(-0.5, 1.5, (75, 3))])
    return p[rng.permutation(len(p))].astype(np.float32)


def rings(seed=32):
    """Two interleaved noisy rings in a plane."""
    rng = np.random.default_rng(seed)
    t = rng.uniform(0, 2 * np.pi, 400)
    a = np.stack([np.cos(t[:200]), np.sin(t[:200]), np.zeros(200)], 1)
    b = np.stack([1 + np.cos(t[200:]), np.zeros(200), np.sin(t[200:])], 1)
    p = np.concatenate([a, b]) + rng.normal(0, 0.01, (400, 3))
    return p.astype(np.float32)


def main():
    L = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libo3dref_dbscan.so"))
    L.ref_cluster_dbscan_f32.argtypes = [C.c_void_p, C.c_int64, C.c_double, C.c_int64, C.c_void_p]
    cases = []
    for name, p, eps, min_points in (("blobs", blobs(), 0.05, 10), ("blobs wide", blobs(), 0.12, 5),
                                     ("rings", rings(), 0.1, 4), ("rings sparse", rings(), 0.03, 3),
                                     ("border", dc.two_clusters_and_a_border()[0], 0.12, 4),
                                     ("pow2 lattice at spacing", dc.pow2_lattice(4), 0.25, 2)):
        p = np.ascontiguousarray(p, np.float32)
        labels = np.empty(len(p), np.int32)
        assert L.ref_cluster_dbscan_f32(p.ctypes.data, len(p), eps, min_points, labels.ctypes.data) == 0
        cases.append({"name": name, "eps": eps, "min_points": min_points, "points": p.tolist(),
                      "labels": labels.tolist()})
        print(name, len(p), "clusters", int(labels.max()) + 1, "noise", int((labels < 0).sum()))
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dbscan_kats.json")
    with open(out, "w") as f:
        json.dump({"source": "geometry::PointCloud::ClusterDBSCAN (geometry/PointCloudCluster.cpp:21-97), compiled "
                             "from the reference sources with a brute-force radius search", "cases": cases}, f)
        f.write("\n")


if __name__ == "__main__":
    main()
