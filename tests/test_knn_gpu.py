"""The exact k-nearest-neighbour search (o3db_knn_*, NearestNeighborSearch.knn_search) and its two consumers,
PointCloud.remove_statistical_outliers and PointCloud.compute_metrics, on the GPU against the brute-force CPU oracle
(oracle/knn): indices and distances, per-point mean distances, masks and metric values are bit-identical."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import knn as ok
from tests import knn_cases as kc
from tests.synth import make_icp_pair

pytestmark = pytest.mark.gpu

KS = (1, 2, 8, 20, 30, 32)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "knn_kats.json")


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


@pytest.fixture(scope="module")
def cases():
    """name -> (data, queries, oracle idx at k = 32, oracle dist2 at k = 32); the k-list is a prefix of the 32-list"""
    out = {}
    for name, (data, queries) in kc.cases().items():
        idx, d2 = ok.knn(data, queries, 32)
        out[name] = (data, queries, idx, d2)
    return out


def _lib():
    from open3d_b200 import _lib
    return _lib


def _stream():
    return int(torch.cuda.current_stream().cuda_stream)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _search(o3d, data, queries, k, dtype=torch.int64):
    nns = o3d.core.nns.NearestNeighborSearch(_dev(data), dtype)
    assert nns.knn_index() is True
    idx, d2 = nns.knn_search(_dev(queries), k)
    return idx.cpu().numpy(), d2.cpu().numpy()


@pytest.mark.parametrize("name", list(kc.cases()))
def test_search_matches_oracle(o3d, cases, name):
    data, queries, oidx, od2 = cases[name]
    for k in KS:
        kp = min(k, len(data))
        idx, d2 = _search(o3d, data, queries, k)
        assert idx.shape == (len(queries), kp) and idx.dtype == np.int64
        np.testing.assert_array_equal(idx, oidx[:, :kp], err_msg=f"{name} k={k}")
        np.testing.assert_array_equal(_bits(d2), _bits(od2[:, :kp]), err_msg=f"{name} k={k}")


def test_search_edge_cases(o3d):
    data = kc.uniform(500)
    q = kc.uniform(300, seed=3)
    q[5] = [np.nan, 0.0, 0.0]
    q[9] = [0.0, np.inf, 0.0]
    want_i, want_d = ok.knn(data, q, 20)
    for dtype in (torch.int32, torch.int64):
        idx, d2 = _search(o3d, data, q, 20, dtype)
        assert idx.dtype == (np.int32 if dtype == torch.int32 else np.int64)
        np.testing.assert_array_equal(idx, want_i)
        np.testing.assert_array_equal(_bits(d2), _bits(want_d))
        assert (idx[5] == -1).all() and (d2[5] == 0).all() and (idx[9] == -1).all()
    # k > M returns M columns; M = 1
    idx, d2 = _search(o3d, data[:7], q, 32)
    assert idx.shape == (300, 7)
    np.testing.assert_array_equal(idx[:5], ok.knn(data[:7], q[:5], 32)[0])
    idx, d2 = _search(o3d, data[:1], q[:4], 5)
    assert idx.shape == (4, 1) and (idx == 0).all()
    # Q = 0
    idx, d2 = _search(o3d, data, np.zeros((0, 3), np.float32), 8)
    assert idx.shape == (0, 8) and d2.shape == (0, 8)
    # two calls are bit-identical
    a = _search(o3d, kc.clusters(), kc.clusters()[:3000], 30)
    b = _search(o3d, kc.clusters(), kc.clusters()[:3000], 30)
    assert np.array_equal(a[0], b[0]) and np.array_equal(_bits(a[1]), _bits(b[1]))


def test_search_errors(o3d):
    nns = o3d.core.nns.NearestNeighborSearch(_dev(kc.uniform(100)))
    with pytest.raises(RuntimeError, match="Index is not set."):
        nns.knn_search(_dev(kc.uniform(10)), 3)
    with pytest.raises(RuntimeError, match="Index is not set."):
        nns.hybrid_search(_dev(kc.uniform(10)), 0.1, 3)
    nns.knn_index()
    with pytest.raises(RuntimeError, match="knn should be larger than 0."):
        nns.knn_search(_dev(kc.uniform(10)), 0)
    with pytest.raises(RuntimeError, match="32"):
        nns.knn_search(_dev(kc.uniform(10)), 33)
    with pytest.raises(RuntimeError, match="DESIGN.md"):
        nns.fixed_radius_index(0.1)
    with pytest.raises(RuntimeError, match="DESIGN.md"):
        nns.multi_radius_search(_dev(kc.uniform(10)), [0.1])
    with pytest.raises(RuntimeError, match="Float32"):
        o3d.core.nns.NearestNeighborSearch(torch.zeros((5, 3), dtype=torch.float64))
    L = _lib()
    h = C.c_void_p()
    assert L.lib.o3db_knn_create(None, 0, None, C.byref(h)) == L.ERR_INVALID and "empty" in L.last_error()
    bad = kc.uniform(100)
    bad[17, 2] = np.nan
    with pytest.raises(RuntimeError, match="non-finite"):
        o3d.core.nns.NearestNeighborSearch(_dev(bad)).knn_index()
    bad[17, 2] = np.inf
    with pytest.raises(RuntimeError, match="non-finite"):
        o3d.core.nns.NearestNeighborSearch(_dev(bad)).knn_index()


def test_hybrid_wrapper(o3d):
    data = kc.uniform(3000)
    nns = o3d.core.nns.NearestNeighborSearch(_dev(data))
    assert nns.hybrid_index(0.1) is True
    idx, d2, cnt = nns.hybrid_search(_dev(data[:500]), 0.1, 16)
    import oracle
    hi, hd, hc = oracle.hybrid_search(data, data[:500], 0.1, 16)
    np.testing.assert_array_equal(idx.cpu().numpy(), hi)
    np.testing.assert_array_equal(cnt.cpu().numpy(), hc)
    assert idx.dtype == torch.int64


def test_kat(o3d):
    kat = json.load(open(GOLDEN))
    s = kat["knn_search"]
    idx, d2 = _search(o3d, s["dataset_points"], s["query_points"], s["knn"])
    np.testing.assert_array_equal(idx, s["indices"])
    np.testing.assert_allclose(d2, s["distances"], rtol=s["rtol"], atol=0)
    m = kat["metrics"]
    geo = o3d.t.geometry
    p1 = np.asarray(m["box_vertices"], np.float32)
    got = geo.PointCloud(p1).compute_metrics(
        geo.PointCloud(p1 * np.float32(m["scale"])),
        (geo.Metric.ChamferDistance, geo.Metric.HausdorffDistance, geo.Metric.FScore),
        geo.MetricParameters(fscore_radius=m["fscore_radius"]))
    assert got.device.type == "cpu" and got.dtype == torch.float32
    np.testing.assert_allclose(got.numpy(), m["values"], rtol=m["rtol"])


def test_large_cloud_against_bruteforce(o3d):
    src, tgt, _, _ = make_icp_pair(2_000_000, seed=1)
    rng = np.random.default_rng(5)
    q = tgt[rng.choice(len(tgt), 2000, replace=False)]
    nns = o3d.core.nns.NearestNeighborSearch(_dev(tgt))
    nns.knn_index()
    idx, d2 = nns.knn_search(_dev(q), 30)
    wi, wd = ok.knn(tgt, q, 30)
    np.testing.assert_array_equal(idx.cpu().numpy(), wi)
    np.testing.assert_array_equal(_bits(d2.cpu().numpy()), _bits(wd))
    qs = src[rng.choice(len(src), 2000, replace=False)]
    idx, d2 = nns.knn_search(_dev(qs), 1)
    wi, wd = ok.knn(tgt, qs, 1)
    np.testing.assert_array_equal(idx.cpu().numpy(), wi)
    np.testing.assert_array_equal(_bits(d2.cpu().numpy()), _bits(wd))


def test_launch_count_is_fixed_per_call(o3d):
    L = _lib()
    steps = []
    for n in (2000, 50000, 200000):
        data = kc.uniform(n, seed=n)
        before = L.launch_count()
        _search(o3d, data, data[:1000], 20)
        torch.cuda.synchronize()
        steps.append(L.launch_count() - before)
    assert steps[0] >= 2 and len(set(steps)) == 1, steps


@pytest.mark.parametrize("name", list(kc.cases()))
def test_statistical_outliers_match_oracle(o3d, cases, name):
    L = _lib()
    data, _, _, od2 = cases[name]
    n = len(data)
    p = _dev(data)
    for nb, ratio in ((20, 2.0), (6, 0.5)):
        mask = torch.empty((n,), dtype=torch.bool, device="cuda")
        avg = torch.full((n,), float("nan"), device="cuda")
        L.check(L.lib.o3db_remove_statistical_outliers(p.data_ptr(), n, nb, ratio, mask.data_ptr(), avg.data_ptr(),
                                                        _stream()))
        kp = min(nb, n)
        wavg, wmask, _ = ok.statistical_outliers_from_dist2(od2[:, :kp] if name != "external" else ok.knn(data, data, nb)[1],
                                                            ratio)
        np.testing.assert_array_equal(_bits(avg.cpu().numpy()), _bits(wavg), err_msg=f"{name} nb={nb}")
        np.testing.assert_array_equal(mask.cpu().numpy(), wmask, err_msg=f"{name} nb={nb}")


def test_statistical_outliers_api(o3d):
    geo = o3d.t.geometry
    data = kc.clusters()
    pc = geo.PointCloud(data)
    pc.set_point_colors(np.abs(data) / 200)
    pc.point["labels"] = torch.arange(len(data), device="cuda")
    out, mask = pc.remove_statistical_outliers(20, 2.0)
    assert mask.dtype == torch.bool and mask.is_cuda and mask.shape == (len(data),)
    _, wmask, _ = ok.remove_statistical_outliers(data, 20, 2.0)
    np.testing.assert_array_equal(mask.cpu().numpy(), wmask)
    m = mask.cpu().numpy()
    np.testing.assert_array_equal(out.point["positions"].cpu().numpy(), data[m])
    np.testing.assert_array_equal(out.point["colors"].cpu().numpy(), (np.abs(data) / 200).astype(np.float32)[m])
    np.testing.assert_array_equal(out.point["labels"].cpu().numpy(), np.nonzero(m)[0])
    # repeated calls are bit-identical
    assert torch.equal(pc.remove_statistical_outliers(20, 2.0)[1], mask)
    # n = 0, n = 1, nb_neighbors > n
    e, em = geo.PointCloud(np.zeros((0, 3), np.float32)).remove_statistical_outliers(5, 1.0)
    assert em.shape == (0,) and em.dtype == torch.bool and not e.has_point_positions()
    one, om = geo.PointCloud(np.ones((1, 3), np.float32)).remove_statistical_outliers(5, 1.0)
    assert om.shape == (1,) and not om.any()
    few = kc.uniform(12)
    _, fm = geo.PointCloud(few).remove_statistical_outliers(30, 1.0)
    np.testing.assert_array_equal(fm.cpu().numpy(), ok.remove_statistical_outliers(few, 30, 1.0)[1])
    msg = "Illegal input parameters, the number of neighbors and standard deviation ratio must be positive."
    for nb, ratio in ((0, 1.0), (5, 0.0), (5, -1.0)):
        with pytest.raises(RuntimeError, match=msg):
            pc.remove_statistical_outliers(nb, ratio)
    with pytest.raises(RuntimeError, match="32"):
        pc.remove_statistical_outliers(33, 1.0)
    f64 = geo.PointCloud()
    f64.point["positions"] = torch.from_numpy(data.astype(np.float64)).cuda()
    with pytest.raises(RuntimeError, match="Float32"):
        f64.remove_statistical_outliers(5, 1.0)


@pytest.mark.parametrize("pair", [("scan", "uniform"), ("clusters", "sparse"), ("offset", "offset"),
                                  ("lattice", "line")])
def test_metrics_match_oracle(o3d, cases, pair):
    geo = o3d.t.geometry
    a = cases[pair[0]][0]
    b = cases[pair[1]][0]
    if pair[0] == pair[1]:
        b = b[::2] + np.float32(0.002)
    radius = (0.001, 0.01, 0.05, 0.5)
    metrics = (geo.Metric.FScore, geo.Metric.ChamferDistance, geo.Metric.HausdorffDistance)
    got = geo.PointCloud(a).compute_metrics(geo.PointCloud(b), metrics, geo.MetricParameters(radius))
    want = ok.compute_metrics(a, b, [ok.FSCORE, ok.CHAMFER, ok.HAUSDORFF], radius)
    np.testing.assert_array_equal(_bits(got.numpy()), _bits(want))
    one = geo.PointCloud(a).compute_metrics(geo.PointCloud(b), [geo.Metric.HausdorffDistance])
    assert one.shape == (1,) and one[0] == got[-1]


def test_metrics_errors(o3d):
    geo = o3d.t.geometry
    pc = geo.PointCloud(kc.uniform(10))
    for x, y in ((geo.PointCloud(), pc), (pc, geo.PointCloud(np.zeros((0, 3), np.float32)))):
        with pytest.raises(RuntimeError, match="One or both input point clouds are empty!"):
            x.compute_metrics(y, [geo.Metric.ChamferDistance])
    f64 = geo.PointCloud()
    f64.point["positions"] = torch.zeros((4, 3), dtype=torch.float64, device="cuda")
    with pytest.raises(RuntimeError, match="Float32"):
        f64.compute_metrics(pc, [geo.Metric.ChamferDistance])


def test_memory_balances_on_success_and_failure():
    if torch.cuda.get_allocator_backend() == "cudaMallocAsync":
        pytest.skip("torch shares the default memory pool")
    from tests.test_host_ownership_gpu import _Pool
    L = _lib()
    pool = _Pool()
    data = _dev(kc.clusters())
    n = int(data.shape[0])
    bad = data.clone()
    bad[3, 0] = float("nan")
    idx = torch.empty((n, 30), dtype=torch.int64, device="cuda")
    d2 = torch.empty((n, 30), dtype=torch.float32, device="cuda")
    mask = torch.empty((n,), dtype=torch.bool, device="cuda")
    out = np.zeros(4, np.float32)
    ms = np.array([0, 1, 2], np.int32)
    rad = np.array([0.01, 0.1], np.float32)
    cases = []

    def balanced(name, call, expect=0):
        u0 = pool.used()
        rc = call()
        assert rc == expect, (name, rc, L.last_error())
        cases.append((name, u0, pool.used()))

    def create_search_destroy():
        h = C.c_void_p()
        L.check(L.lib.o3db_knn_create(data.data_ptr(), n, _stream(), C.byref(h)))
        rc = L.lib.o3db_knn_search(h, data.data_ptr(), n, 30, L.INDEX_INT64, idx.data_ptr(), d2.data_ptr(), _stream())
        L.lib.o3db_knn_destroy(h)
        return rc

    def create_failing():
        h = C.c_void_p()
        return L.lib.o3db_knn_create(bad.data_ptr(), n, _stream(), C.byref(h))

    for _ in range(2):
        balanced("knn", create_search_destroy)
        balanced("knn_create with a NaN", create_failing, L.ERR_INVALID)
        balanced("outliers", lambda: L.lib.o3db_remove_statistical_outliers(data.data_ptr(), n, 20, 2.0, mask.data_ptr(),
                                                                           None, _stream()))
        balanced("outliers with a NaN", lambda: L.lib.o3db_remove_statistical_outliers(
            bad.data_ptr(), n, 20, 2.0, mask.data_ptr(), None, _stream()), L.ERR_INVALID)
        balanced("metrics", lambda: L.lib.o3db_compute_metrics(data.data_ptr(), n, data.data_ptr(), n // 2, ms.ctypes.data,
                                                               3, rad.ctypes.data, 2, out.ctypes.data, 4, _stream()))
        balanced("metrics with a NaN", lambda: L.lib.o3db_compute_metrics(
            data.data_ptr(), n, bad.data_ptr(), n, ms.ctypes.data, 3, rad.ctypes.data, 2, out.ctypes.data, 4, _stream()),
            L.ERR_INVALID)
    for name, u0, u1 in cases:
        assert u1 == u0, (name, u0, u1)
