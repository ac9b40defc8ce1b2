"""The clean-up filters on the GPU (PointCloud.remove_radius_outliers, remove_duplicated_points,
remove_non_finite_points) against the CPU oracle (oracle/remove) and numpy, mask for mask.

The radius count uses upstream's CUDA distance test as nvcc contracts it (the oracle's "cuda" mode); the ulp_pairs
cloud shows it differs from the uncontracted test on pairs within an ulp of the threshold, and the exact lattice that
a distance equal to the radius counts."""
import numpy as np
import pytest
import torch

from oracle import remove as orm
from tests import remove_cases as rc

pytestmark = pytest.mark.gpu


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


def _pc(o3d, pts):
    return o3d.t.geometry.PointCloud(torch.from_numpy(np.ascontiguousarray(pts, np.float32)).cuda())


def _radius_mask(o3d, pts, nb, r):
    _, m = _pc(o3d, pts).remove_radius_outliers(nb, r)
    assert m.dtype == torch.bool and m.device.type == "cuda" and m.shape == (len(pts),)
    return m.cpu().numpy()


@pytest.fixture(scope="module")
def radius_cases():
    return rc.radius_cases()


@pytest.mark.parametrize("name", ["scan", "clusters", "offset", "lattice", "ulp_pairs", "coincident"])
def test_radius_masks_equal_oracle(o3d, radius_cases, name):
    pts, params = radius_cases[name]
    for nb, r in params:
        want = orm.remove_radius_outliers(pts, nb, r, "cuda")
        got = _radius_mask(o3d, pts, nb, r)
        assert np.array_equal(got, want), (name, nb, r, int((got != want).sum()))


def test_exact_boundary_and_ulp_cases(o3d):
    p, s = rc.exact_lattice()
    g = np.round(p / np.float32(s)).astype(int)
    inside = np.all((g > 0) & (g < g.max()), axis=1)
    assert np.array_equal(_radius_mask(o3d, p, 7, s), inside)       # self + 6 neighbours at dist == thr
    assert not _radius_mask(o3d, p, 8, s).any()
    u, r = rc.ulp_pairs()
    got = _radius_mask(o3d, u, 2, r)
    assert np.array_equal(got, orm.remove_radius_outliers(u, 2, r, "cuda"))
    assert not np.array_equal(got, orm.remove_radius_outliers(u, 2, r, "plain"))


@pytest.fixture(scope="module")
def scan2m():
    return rc.scan_2m()


@pytest.mark.parametrize("r", [0.02, 0.05])
def test_radius_2m_equal_oracle(o3d, scan2m, r):
    pc = _pc(o3d, scan2m)
    for nb in (1, 2, 16, 64, len(scan2m) + 1):
        want = orm.remove_radius_outliers(scan2m, nb, r, "cuda")
        got = pc.remove_radius_outliers(nb, r)[1].cpu().numpy()
        assert np.array_equal(got, want), (r, nb, int((got != want).sum()))


def _first_occurrence(p):
    _, first = np.unique(p.view(np.int32).reshape(-1, 3), axis=0, return_index=True)
    want = np.zeros(len(p), bool)
    want[first] = True
    return want


@pytest.mark.parametrize("name", sorted(rc.duplicate_cases()))
def test_duplicates_first_occurrence(o3d, name):
    p = rc.duplicate_cases()[name]
    _, m = _pc(o3d, p).remove_duplicated_points()
    m = m.cpu().numpy()
    assert np.array_equal(m, _first_occurrence(p))
    assert np.array_equal(m, orm.remove_duplicated_points(p))
    if name == "one_point":
        assert m[0] and m.sum() == 1


def test_duplicates_2m(o3d):
    p = rc.duplicated_2m()
    got = _pc(o3d, p).remove_duplicated_points()[1].cpu().numpy()
    assert np.array_equal(got, orm.remove_duplicated_points(p))
    assert got.sum() < 0.92 * len(p)


def test_non_finite_flags(o3d):
    p = rc.non_finite_cloud()
    pc = _pc(o3d, p)
    for rn in (False, True):
        for ri in (False, True):
            out, m = pc.remove_non_finite_points(rn, ri)
            want = orm.remove_non_finite_points(p, rn, ri)
            assert np.array_equal(m.cpu().numpy(), want), (rn, ri)
            assert np.array_equal(out.positions.cpu().numpy().view(np.int32), p[want].view(np.int32))
    assert np.array_equal(pc.remove_non_finite_points()[1].cpu().numpy(), np.isfinite(p).all(1))


def test_attributes_are_carried(o3d):
    p = rc.coincident()
    n = len(p)
    pc = _pc(o3d, p)
    pc.set_point_normals(torch.arange(3 * n, dtype=torch.float32, device="cuda").reshape(n, 3))
    pc.set_point_colors(torch.rand(n, 3, device="cuda"))
    for out, m in (pc.remove_radius_outliers(3, 1e-3), pc.remove_duplicated_points(), pc.remove_non_finite_points()):
        assert set(out.point) == set(pc.point)
        for k, v in pc.point.items():
            assert torch.equal(out.point[k], v[m])


def test_errors_and_empty(o3d):
    pc = _pc(o3d, rc.nc.scan(1000, seed=1))
    for nb, r in ((0, 0.1), (3, 0.0), (3, -0.1)):
        with pytest.raises(RuntimeError, match="number of points and radius must be positive"):
            pc.remove_radius_outliers(nb, r)
    for r in (float("nan"), float("inf")):
        with pytest.raises(RuntimeError, match="finite"):
            pc.remove_radius_outliers(3, r)
    bad = rc.nc.scan(1000, seed=1)
    bad[17, 1] = np.nan
    with pytest.raises(RuntimeError, match="remove_non_finite_points"):
        _pc(o3d, bad).remove_radius_outliers(3, 0.05)
    f64 = o3d.t.geometry.PointCloud()
    f64.point["positions"] = torch.zeros(4, 3, dtype=torch.float64, device="cuda")
    for call in (lambda: f64.remove_radius_outliers(2, 0.1), f64.remove_duplicated_points,
                 f64.remove_non_finite_points):
        with pytest.raises(RuntimeError, match="only Float32"):
            call()
    empty = _pc(o3d, np.zeros((0, 3), np.float32))
    for out, m in (empty.remove_radius_outliers(2, 0.1), empty.remove_duplicated_points(),
                   empty.remove_non_finite_points()):
        assert m.shape == (0,) and m.dtype == torch.bool and out.positions.shape == (0, 3)


def test_non_finite_then_dbscan(o3d):
    p = rc.nc.scan(5000, seed=4)
    p[::97, 2] = np.inf
    p[5::101, 0] = np.nan
    pc = _pc(o3d, p)
    with pytest.raises(RuntimeError):
        pc.cluster_dbscan(0.05, 5)
    clean, m = pc.remove_non_finite_points()
    assert np.array_equal(m.cpu().numpy(), np.isfinite(p).all(1))
    labels = clean.cluster_dbscan(0.05, 5)
    assert labels.shape[0] == int(m.sum())
    clean.remove_radius_outliers(5, 0.05)


def test_repeated_calls_are_identical(o3d):
    p = rc.duplicated_2m()[:300000]
    pc = _pc(o3d, p)
    for call in (lambda: pc.remove_radius_outliers(16, 0.05), pc.remove_duplicated_points,
                 pc.remove_non_finite_points):
        a = call()[1]
        for _ in range(3):
            assert torch.equal(call()[1], a)


def test_launch_count_is_fixed_per_call(o3d, radius_cases):
    L = _lib()
    calls = {
        "radius": lambda pc: pc.remove_radius_outliers(4, 0.05),
        "duplicates": lambda pc: pc.remove_duplicated_points(),
        "non_finite": lambda pc: pc.remove_non_finite_points(),
    }
    for what, call in calls.items():
        steps = []
        for name in ("scan", "clusters", "lattice", "coincident"):
            pc = _pc(o3d, radius_cases[name][0])
            torch.cuda.synchronize()
            before = L.launch_count()
            call(pc)
            torch.cuda.synchronize()
            steps.append(L.launch_count() - before)
        assert steps[0] >= 1 and len(set(steps)) == 1, (what, steps)


def test_memory_balances_on_success_and_failure(o3d):
    if torch.cuda.get_allocator_backend() == "cudaMallocAsync":
        pytest.skip("torch shares the default memory pool")
    from tests.test_host_ownership_gpu import _Pool
    L = _lib()
    pool = _Pool()
    pts = rc.nc.scan(50000, seed=6)
    p = torch.from_numpy(pts).cuda()
    bad = p.clone()
    bad[7, 2] = float("inf")
    mask = torch.empty(len(pts), dtype=torch.uint8, device="cuda")
    rows = []
    for _ in range(2):
        for name, fn, expect in (
                ("radius ok", lambda: L.lib.o3db_remove_radius_outliers(p.data_ptr(), len(pts), 8, 0.05,
                                                                        mask.data_ptr(), _stream()), 0),
                ("radius non-finite", lambda: L.lib.o3db_remove_radius_outliers(bad.data_ptr(), len(pts), 8, 0.05,
                                                                                mask.data_ptr(), _stream()),
                 L.ERR_INVALID),
                ("radius nan radius", lambda: L.lib.o3db_remove_radius_outliers(p.data_ptr(), len(pts), 8,
                                                                                float("nan"), mask.data_ptr(),
                                                                                _stream()), L.ERR_INVALID),
                ("duplicates ok", lambda: L.lib.o3db_remove_duplicated_points(p.data_ptr(), len(pts), mask.data_ptr(),
                                                                              _stream()), 0),
                ("non-finite ok", lambda: L.lib.o3db_remove_non_finite_points(p.data_ptr(), len(pts), 1, 1,
                                                                              mask.data_ptr(), _stream()), 0)):
            u0 = pool.used()
            rc_ = fn()
            assert rc_ == expect, (name, rc_, L.last_error())
            rows.append((name, u0, pool.used()))
    torch.cuda.synchronize()
    for name, u0, u1 in rows:
        assert u1 == u0, (name, u0, u1)
