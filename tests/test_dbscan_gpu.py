"""DBSCAN clustering on the GPU (PointCloud.cluster_dbscan) against the CPU oracle (oracle/dbscan), label for label.

The oracle restates upstream's ClusterDBSCAN and matches the reference's own function on these clouds
(tests/test_oracle_dbscan.py); tests/golden/dbscan_kats.json holds labels the reference computed."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import dbscan as od
from tests import dbscan_cases as dc
from tests import knn_cases as kc
from tests.synth import make_icp_pair

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dbscan_kats.json")


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


def _lib():
    from open3d_b200 import _lib
    return _lib


def _stream():
    return int(torch.cuda.current_stream().cuda_stream)


def _labels(o3d, p, eps, min_points):
    return o3d.t.geometry.PointCloud(np.ascontiguousarray(p, np.float32)).cluster_dbscan(eps, min_points).cpu().numpy()


@pytest.mark.parametrize("name", dc.FIXTURES)
def test_labels_match_oracle(o3d, name):
    p = dc.fixtures()[name]
    for eps, min_points in dc.eps_grid(p):
        want = od.cluster_dbscan(p, eps, min_points)
        got = _labels(o3d, p, eps, min_points)
        np.testing.assert_array_equal(got, want, err_msg=f"{name} eps={eps!r} min_points={min_points}")


@pytest.mark.parametrize("name", list(dc.constructed()))
def test_constructed_cases(o3d, name):
    p, eps, min_points, want = dc.constructed()[name]
    got = _labels(o3d, p, eps, min_points)
    np.testing.assert_array_equal(got, od.cluster_dbscan(p, eps, min_points), err_msg=name)
    if want is not None:
        np.testing.assert_array_equal(got, want, err_msg=name)


def test_full_size_cloud(o3d):
    """The 2 M-point cloud of profiles/dbscan_time.py, whole."""
    p = make_icp_pair(2_000_000, seed=1)[1]
    got = _labels(o3d, p, 0.05, 10)
    want = od.cluster_dbscan(p, 0.05, 10)
    np.testing.assert_array_equal(got, want)
    assert want.max() >= 0


def test_kats(o3d):
    kats = json.load(open(GOLDEN))
    assert kats["cases"]
    for case in kats["cases"]:
        got = _labels(o3d, np.asarray(case["points"], np.float32), case["eps"], case["min_points"])
        np.testing.assert_array_equal(got, np.asarray(case["labels"], np.int32), err_msg=case["name"])


def test_repeated_calls_are_bit_identical(o3d):
    for p, eps in ((kc.clusters(), 0.05), (dc.coincident(), 0.06), (make_icp_pair(200_000, seed=3)[1], 0.05)):
        pc = o3d.t.geometry.PointCloud(p)
        a = pc.cluster_dbscan(eps, 10)
        b = pc.cluster_dbscan(eps, 10)
        assert torch.equal(a, b)


def test_result_and_errors(o3d):
    geo = o3d.t.geometry
    p = kc.uniform(2000)
    pc = geo.PointCloud(p)
    out = pc.cluster_dbscan(0.05, 5, print_progress=True)
    assert out.dtype == torch.int32 and out.shape == (2000,) and out.device == pc.point["positions"].device
    empty = geo.PointCloud(np.zeros((0, 3), np.float32)).cluster_dbscan(0.05, 5)
    assert empty.dtype == torch.int32 and empty.shape == (0,) and empty.is_cuda
    for eps in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(RuntimeError, match="eps must be positive and finite"):
            pc.cluster_dbscan(eps, 5)
    with pytest.raises(RuntimeError, match="min_points must be non-negative"):
        pc.cluster_dbscan(0.05, -1)
    for bad in (float("nan"), float("inf")):
        q = p.copy()
        q[7, 1] = bad
        with pytest.raises(RuntimeError, match="non-finite"):
            geo.PointCloud(q).cluster_dbscan(0.05, 5)
    f64 = geo.PointCloud()
    f64.point["positions"] = torch.from_numpy(p.astype(np.float64)).cuda()
    with pytest.raises(RuntimeError, match="Float32"):
        f64.cluster_dbscan(0.05, 5)


def test_launch_count_is_fixed_per_call(o3d):
    L = _lib()
    counts = []
    for n in (2000, 50000, 200000):
        pc = o3d.t.geometry.PointCloud(kc.uniform(n, seed=n))
        for eps in (0.01, 0.05, 0.3):
            before = L.launch_count()
            pc.cluster_dbscan(eps, 10)
            torch.cuda.synchronize()
            counts.append(L.launch_count() - before)
    assert counts[0] >= 6 and len(set(counts)) == 1, counts


def test_memory_balances_on_success_and_failure():
    if torch.cuda.get_allocator_backend() == "cudaMallocAsync":
        pytest.skip("torch shares the default memory pool")
    from tests.test_host_ownership_gpu import _Pool
    L = _lib()
    pool = _Pool()
    data = torch.from_numpy(kc.clusters()).cuda()
    n = int(data.shape[0])
    bad = data.clone()
    bad[3, 0] = float("nan")
    labels = torch.empty(n, dtype=torch.int32, device="cuda")
    cases = []

    def balanced(name, call, expect=0):
        u0 = pool.used()
        rc = call()
        assert rc == expect, (name, rc, L.last_error())
        cases.append((name, u0, pool.used()))

    for _ in range(2):
        for eps in (0.02, 0.2):
            balanced(f"eps {eps}", lambda: L.lib.o3db_cluster_dbscan(data.data_ptr(), n, eps, 10, labels.data_ptr(),
                                                                     _stream()))
        balanced("a NaN", lambda: L.lib.o3db_cluster_dbscan(bad.data_ptr(), n, 0.05, 10, labels.data_ptr(), _stream()),
                 L.ERR_INVALID)
    torch.cuda.synchronize()
    for name, u0, u1 in cases:
        assert u1 == u0, (name, u0, u1)
