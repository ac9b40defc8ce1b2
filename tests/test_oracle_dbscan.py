"""The DBSCAN oracle (oracle/dbscan) against the reference's own geometry::PointCloud::ClusterDBSCAN, compiled
unmodified into oracle/_ref/libo3dref_dbscan.so (oracle/ref_shim_dbscan) with a brute-force radius search, label for
label.  Also: the oracle's grid and brute-force neighbour passes agree, the oracle reproduces the reference's labels in
tests/golden/dbscan_kats.json, and o3db_cluster_dbscan checks its arguments before any CUDA call.  CPU only."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import dbscan as od
from tests import dbscan_cases as dc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libo3dref_dbscan.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "dbscan_kats.json")
ROWS = 1500   # points of each fixture: the reference's search is the O(n^2) brute force


@pytest.fixture(scope="module")
def ref():
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref/libo3dref_dbscan.so not built (needs the reference sources)")
    L = C.CDLL(REF)
    L.ref_cluster_dbscan_f32.restype = C.c_int
    L.ref_cluster_dbscan_f32.argtypes = [C.c_void_p, C.c_int64, C.c_double, C.c_int64, C.c_void_p]

    def run(p, eps, min_points):
        p = np.ascontiguousarray(p, np.float32)
        out = np.empty(len(p), np.int32)
        assert L.ref_cluster_dbscan_f32(p.ctypes.data, len(p), float(eps), int(min_points), out.ctypes.data) == 0
        return out
    return run


@pytest.mark.parametrize("name", dc.FIXTURES)
def test_oracle_matches_reference(ref, name):
    p = np.ascontiguousarray(dc.fixtures()[name][:ROWS])
    for eps, min_points in dc.eps_grid(p):
        want = ref(p, eps, min_points)
        np.testing.assert_array_equal(od.cluster_dbscan(p, eps, min_points), want, err_msg=f"{name} {eps} {min_points}")
        np.testing.assert_array_equal(od.cluster_dbscan(p, eps, min_points, bruteforce=True), want)


@pytest.mark.parametrize("name", list(dc.constructed()))
def test_constructed_cases_match_reference(ref, name):
    p, eps, min_points, want = dc.constructed()[name]
    got = ref(p, eps, min_points)
    np.testing.assert_array_equal(od.cluster_dbscan(p, eps, min_points), got, err_msg=name)
    if want is not None:
        np.testing.assert_array_equal(got, want, err_msg=name)


@pytest.mark.parametrize("name", dc.FIXTURES)
def test_grid_and_bruteforce_core_flags_agree(name):
    p = np.ascontiguousarray(dc.fixtures()[name][:5000])
    for eps, min_points in dc.eps_grid(p):
        grid = od.core_points(p, eps, min_points)
        np.testing.assert_array_equal(grid, od.core_points(p, eps, min_points, bruteforce=True))
        labels, core = od.cluster_dbscan(p, eps, min_points, return_core=True)
        np.testing.assert_array_equal(core, grid)
        assert (labels[core] >= 0).all()


def test_constructed_expectations_without_reference():
    for name, (p, eps, min_points, want) in dc.constructed().items():
        if want is not None:
            np.testing.assert_array_equal(od.cluster_dbscan(p, eps, min_points), want, err_msg=name)


def test_oracle_reproduces_kats():
    kats = json.load(open(GOLDEN))
    assert kats["cases"]
    for case in kats["cases"]:
        got = od.cluster_dbscan(np.asarray(case["points"], np.float32), case["eps"], case["min_points"])
        np.testing.assert_array_equal(got, np.asarray(case["labels"], np.int32), err_msg=case["name"])


def test_cabi_argument_checks():
    from open3d_b200 import _lib as L
    fake = 16   # never dereferenced: every call below fails its checks first
    for args, msg in (((None, 10, 0.1, 5, fake), "null"), ((fake, 10, 0.1, 5, None), "null"),
                      ((fake, -1, 0.1, 5, fake), "bad point count"), ((fake, 2**31 - 1, 0.1, 5, fake), "bad point count"),
                      ((fake, 10, 0.0, 5, fake), "eps"), ((fake, 10, -0.5, 5, fake), "eps"),
                      ((fake, 10, float("nan"), 5, fake), "eps"), ((fake, 10, float("inf"), 5, fake), "eps"),
                      ((fake, 10, 0.1, -1, fake), "min_points")):
        rc = L.lib.o3db_cluster_dbscan(*args, None)
        assert rc == L.ERR_INVALID and msg in L.last_error(), (args, rc, L.last_error())
    assert L.lib.o3db_cluster_dbscan(fake, 0, 0.1, 5, fake, None) == L.OK
