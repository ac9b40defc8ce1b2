"""Farthest-point down-sampling on the GPU (o3db_farthest_point_down_sample, PointCloud.farthest_point_down_sample)
against the CPU oracle (oracle/fps), index for index in selection order.

The oracle reproduces upstream's unit-test fixture and equals a numpy restatement of upstream's loop
(tests/test_oracle_fps.py)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import fps as of
from tests import fps_cases as fc
from tests import knn_cases as kc
from tests.synth import make_icp_pair

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fps_kats.json")


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


def _select(p, num_samples, start_index=0):
    """The C ABI's indices in selection order."""
    L = _lib()
    d = torch.from_numpy(np.ascontiguousarray(p, np.float32)).cuda()
    out = torch.empty(num_samples, dtype=torch.int32, device="cuda")
    rc = L.lib.o3db_farthest_point_down_sample(d.data_ptr(), d.shape[0], num_samples, start_index, out.data_ptr(),
                                               _stream())
    assert rc == 0, L.last_error()
    return out.cpu().numpy()


def _check(p, num_samples, start_index, what):
    got = _select(p, num_samples, start_index)
    want = of.farthest_point_down_sample(p, num_samples, start_index)
    np.testing.assert_array_equal(got, want, err_msg=f"{what} num_samples={num_samples} start_index={start_index}")
    return got


@pytest.mark.parametrize("name", ["uniform", "clusters", "lattice", "external"])
def test_sequence_matches_oracle(o3d, name):
    p = fc.fixtures()[name]
    n = len(p)
    for m, s in ((1, 0), (1, n - 1), (2, 0), (257, 0), (1000, n - 1), (3000, n // 2), (n, 0), (n, n - 1)):
        if m <= n:
            sel = _check(p, m, s, name)
            assert len(np.unique(sel)) == m


def test_coincident_points_give_distinct_indices(o3d):
    p = fc.coincident()
    distinct = len(np.unique(p, axis=0))
    for m, s in ((100, 5), (len(p), 0)):
        sel = _check(p, m, s, "coincident")
        assert len(np.unique(sel)) == m
        first = set(sel[:distinct].tolist())
        rest = [j for j in range(len(p)) if j not in first][:m - distinct]
        np.testing.assert_array_equal(sel[distinct:], rest)


def test_overflowing_distances(o3d):
    p = fc.overflow()
    _check(p, 500, 0, "overflow")
    _check(p, 200, len(p) - 1, "overflow")


def test_profile_cloud(o3d):
    """The 2 M-point cloud of profiles/fps_time.py at 4096 samples: every point on chip."""
    p = make_icp_pair(2_000_000, seed=1)[1]
    _check(p, 4096, 0, "profile cloud")


def test_cloud_above_on_chip_capacity(o3d):
    """4 M points: each CTA holds 18432 points on chip and reads and writes the rest of its slice every round."""
    p = kc.uniform(4_000_000, seed=5)
    _check(p, 1024, 123, "4 M uniform")
    # one more point than a whole number of rows, and distances that tie in the part read from global memory
    q = fc.integer_cloud(4_000_000, seed=6)[:2_600_001]
    _check(q, 700, 0, "2.6 M integer")


def test_python_result_gathers_every_attribute(o3d):
    geo = o3d.t.geometry
    p = kc.clusters()
    n = len(p)
    rng = np.random.default_rng(3)
    nrm = rng.normal(size=(n, 3)).astype(np.float32)
    col = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    label = torch.arange(n, dtype=torch.int64, device="cuda") * 7
    pc = geo.PointCloud(p).set_point_normals(nrm).set_point_colors(col)
    pc.point["label"] = label
    for m, s in ((500, 0), (37, n - 1)):
        out = pc.farthest_point_down_sample(m, s)
        idx = np.sort(of.farthest_point_down_sample(p, m, s))
        assert sorted(out.point) == sorted(pc.point)
        np.testing.assert_array_equal(out.point["positions"].cpu().numpy(), p[idx])
        np.testing.assert_array_equal(out.point["normals"].cpu().numpy(), nrm[idx])
        np.testing.assert_array_equal(out.point["colors"].cpu().numpy(), col[idx])
        assert out.point["label"].dtype == torch.int64
        np.testing.assert_array_equal(out.point["label"].cpu().numpy(), idx.astype(np.int64) * 7)
        for v in out.point.values():
            assert v.is_cuda and v.shape[0] == m
        assert out.point["positions"].dtype == torch.float32


def test_golden_fixture(o3d):
    kats = json.load(open(GOLDEN))
    p = np.asarray(kats["points"], np.float32)
    pc = o3d.t.geometry.PointCloud(p)
    for case in kats["cases"]:
        np.testing.assert_array_equal(_select(p, case["num_samples"], case["start_index"]), case["selection_order"])
        out = pc.farthest_point_down_sample(case["num_samples"], case["start_index"])
        np.testing.assert_array_equal(out.point["positions"].cpu().numpy(), np.asarray(case["expected"], np.float32))


def test_repeated_calls_are_bit_identical(o3d):
    for p, m in ((kc.clusters(), 2000), (fc.coincident(), 300), (make_icp_pair(200_000, seed=3)[1], 1000)):
        a = _select(p, m, 1)
        b = _select(p, m, 1)
        np.testing.assert_array_equal(a, b)
        pc = o3d.t.geometry.PointCloud(p)
        assert torch.equal(pc.farthest_point_down_sample(m, 1).point["positions"],
                           pc.farthest_point_down_sample(m, 1).point["positions"])


def test_arguments_and_errors(o3d):
    geo = o3d.t.geometry
    L = _lib()
    p = kc.uniform(2000)
    pc = geo.PointCloud(p)
    before = L.launch_count()
    empty = pc.farthest_point_down_sample(0)
    assert isinstance(empty, geo.PointCloud) and not empty.point
    whole = pc.farthest_point_down_sample(2000, 5000)      # a clone, before start_index is looked at
    assert torch.equal(whole.point["positions"], pc.point["positions"])
    assert whole.point["positions"].data_ptr() != pc.point["positions"].data_ptr()
    torch.cuda.synchronize()
    assert L.launch_count() == before
    with pytest.raises(RuntimeError, match="Illegal number of samples: 2001, must <= point size: 2000"):
        pc.farthest_point_down_sample(2001)
    for s in (2000, 10**6):
        with pytest.raises(RuntimeError, match="Illegal start index"):
            pc.farthest_point_down_sample(10, s)
    for m, s in ((-1, 0), (10, -1)):
        with pytest.raises(RuntimeError, match="non-negative"):
            pc.farthest_point_down_sample(m, s)
    for bad in (float("nan"), float("inf"), float("-inf")):
        for row in (7, 1999):
            q = p.copy()
            q[row, 1] = bad
            with pytest.raises(RuntimeError, match="non-finite"):
                geo.PointCloud(q).farthest_point_down_sample(10)
    big = kc.uniform(3_000_000, seed=9)
    big[2_999_000, 2] = float("nan")                       # in the part of a slice read from global memory
    with pytest.raises(RuntimeError, match="non-finite"):
        geo.PointCloud(big).farthest_point_down_sample(10)
    f64 = geo.PointCloud()
    f64.point["positions"] = torch.from_numpy(p.astype(np.float64)).cuda()
    with pytest.raises(RuntimeError, match="Float32"):
        f64.farthest_point_down_sample(10)
    # the C ABI's own checks
    d = pc.point["positions"]
    out = torch.empty(10, dtype=torch.int32, device="cuda")
    for args in ((0, 2000, 10, 0, out.data_ptr()), (d.data_ptr(), 2000, 10, 0, 0), (d.data_ptr(), -1, 10, 0,
                 out.data_ptr()), (d.data_ptr(), 2**31 - 1, 10, 0, out.data_ptr()), (d.data_ptr(), 2000, 0, 0,
                 out.data_ptr()), (d.data_ptr(), 2000, 2001, 0, out.data_ptr()), (d.data_ptr(), 2000, 10, -1,
                 out.data_ptr()), (d.data_ptr(), 2000, 10, 2000, out.data_ptr())):
        assert L.lib.o3db_farthest_point_down_sample(*args, _stream()) == L.ERR_INVALID, args


def test_launch_count_is_fixed_per_call(o3d):
    L = _lib()
    counts = []
    for n in (2000, 200_000, 4_000_000):
        p = kc.uniform(n, seed=n)
        for m in (1, 10, 1000):
            before = L.launch_count()
            _select(p, m, 0)
            torch.cuda.synchronize()
            counts.append(L.launch_count() - before)
    assert counts[0] >= 1 and len(set(counts)) == 1, counts


def test_memory_balances_on_success_and_failure():
    if torch.cuda.get_allocator_backend() == "cudaMallocAsync":
        pytest.skip("torch shares the default memory pool")
    from tests.test_host_ownership_gpu import _Pool
    L = _lib()
    pool = _Pool()
    small = torch.from_numpy(kc.clusters()).cuda()
    big = torch.from_numpy(kc.uniform(3_000_000, seed=4)).cuda()     # past the on-chip capacity: a remainder buffer
    bad = small.clone()
    bad[3, 0] = float("nan")
    out = torch.empty(500, dtype=torch.int32, device="cuda")
    cases = []

    def balanced(name, data, expect=0):
        u0 = pool.used()
        rc = L.lib.o3db_farthest_point_down_sample(data.data_ptr(), data.shape[0], 500, 0, out.data_ptr(), _stream())
        assert rc == expect, (name, rc, L.last_error())
        cases.append((name, u0, pool.used()))

    for _ in range(2):
        balanced("on chip", small)
        balanced("with remainder", big)
        balanced("a NaN", bad, L.ERR_INVALID)
    torch.cuda.synchronize()
    for name, u0, u1 in cases:
        assert u1 == u0, (name, u0, u1)
