"""Boundary detection on the GPU (o3db_compute_boundary_points, PointCloud.compute_boundary_points) against the CPU
oracle (oracle/boundary) on the oracle's own hybrid search.

In the oracle's f64 mode, which evaluates atan2 as the device does, every mask bit and every max_gap bit is equal.  In
its libm mode, which equals the reference's own code bit for bit (tests/test_oracle_vs_ref_boundary.py), the masks
differ only where the largest gap lies within a few f32 ulps of the threshold, since libm's atan2f is not correctly
rounded."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import boundary as ob
from oracle import normals as on
from tests import boundary_cases as bc
from tests import normals_cases as nc
from tests.synth import make_icp_pair

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


@pytest.fixture(scope="module")
def cases():
    return bc.cases()


def _lib():
    from open3d_b200 import _lib
    return _lib


def _stream():
    return int(torch.cuda.current_stream().cuda_stream)


def _gpu(pts, nrm, radius, max_nn, thr=90.0):
    """-> (mask bool [n], max_gap f32 [n]) from the C ABI"""
    L = _lib()
    p = torch.from_numpy(np.ascontiguousarray(pts, np.float32)).cuda()
    q = torch.from_numpy(np.ascontiguousarray(nrm, np.float32)).cuda()
    n = p.shape[0]
    mask = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
    gap = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    L.check(L.lib.o3db_compute_boundary_points(p.data_ptr(), q.data_ptr(), n, float(radius), int(max_nn), float(thr),
                                               mask.data_ptr(), gap.data_ptr(), _stream()))
    m = mask.cpu().numpy()
    assert set(np.unique(m)) <= {0, 1}
    return m.astype(bool), gap.cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _assert_f64_parity(pts, nrm, radius, max_nn, thr=90.0):
    got, gap = _gpu(pts, nrm, radius, max_nn, thr)
    want, wgap = ob.compute_boundary_points(pts, nrm, radius, max_nn, thr, mode="f64")
    assert np.array_equal(got, want), int(np.count_nonzero(got != want))
    assert np.array_equal(_bits(gap), _bits(wgap)), int(np.count_nonzero(_bits(gap) != _bits(wgap)))
    return got, gap


def _ulps_from(x, t):
    """distance in f32 ulps between the f32 values x and t"""
    def key(v):
        b = np.asarray(v, np.float32).view(np.int32).astype(np.int64)
        return np.where(b < 0, -(b & 0x7FFFFFFF), b)
    return np.abs(key(x) - key(np.float32(t)))


@pytest.mark.parametrize("name", sorted(bc.cases()))
def test_cases_vs_f64_oracle(cases, name):
    pts, nrm, radius, max_nn = cases[name]
    for thr in (90.0, 45.0, -1.0):
        _assert_f64_parity(pts, nrm, radius, max_nn, thr)


@pytest.mark.parametrize("max_nn", [1, 2, 8, 30, 32])
def test_max_nn_vs_f64_oracle(max_nn):
    pts = nc.scan(20000, seed=8)
    nrm, _, _ = on.estimate_normals(pts, 0.08, 30)
    mask, _ = _assert_f64_parity(pts, nrm, 0.05, max_nn)
    if max_nn == 1:
        assert not mask.any()   # the one neighbour is dropped as the point itself
    elif max_nn == 2:
        assert mask.all()   # one kept neighbour: the wrap gap is about 2 pi


def test_target_2m_vs_f64_oracle():
    _, tgt, nrm, _ = make_icp_pair(2_000_000, seed=1)
    mask, _ = _assert_f64_parity(tgt, nrm, 0.08, 30)
    assert 0 < mask.sum() < len(tgt) // 20


@pytest.mark.parametrize("name", sorted(bc.cases()) + ["scan_200k"])
def test_libm_differences_lie_at_the_threshold(cases, name):
    if name == "scan_200k":
        pts, nrm = bc.scan_200k()
        radius, max_nn = 0.02, 30
    else:
        pts, nrm, radius, max_nn = cases[name]
    thr = 90.0
    got, _ = _gpu(pts, nrm, radius, max_nn, thr)
    want, wgap = ob.compute_boundary_points(pts, nrm, radius, max_nn, thr, mode="libm")
    diff = np.flatnonzero(got != want)
    near = _ulps_from(wgap[diff], thr * math.pi / 180.0)
    print(f"{name}: {len(diff)} of {len(pts)} points differ from the libm-mode oracle, each within "
          f"{int(near.max()) if len(diff) else 0} ulps of the threshold")
    assert (near <= 4).all(), (name, diff[:10], near[:10])
    if name == "lattice4":
        assert len(diff) == 0


def _tilted_frame():
    nz = np.array([1.0, 2.0, 3.0]) / math.sqrt(14.0)
    e1 = np.cross(nz, [1.0, 0.0, 0.0])
    e1 /= np.linalg.norm(e1)
    return nz, e1, np.cross(nz, e1)


def _plane_lattice(keep, side=81, h=0.01):
    """points of a square lattice in the tilted plane where keep(s, t) holds -> (points, normals, s, t)"""
    nz, e1, e2 = _tilted_frame()
    g = (np.arange(side) - side // 2) * h
    s, t = (a.ravel() for a in np.meshgrid(g, g))
    k = keep(s, t)
    s, t = s[k], t[k]
    p = np.array([0.2, -0.1, 0.4]) + s[:, None] * e1 + t[:, None] * e2
    return p.astype(np.float32), np.tile(nz, (len(p), 1)).astype(np.float32), s, t


def _disc(h, R):
    """concentric rings h apart, each with points about h apart along it, in the tilted plane -> (points, normals, r)"""
    nz, e1, e2 = _tilted_frame()
    s, t, r = [0.0], [0.0], [0.0]
    for k in range(1, int(round(R / h)) + 1):
        m = int(round(2 * math.pi * k))
        a = 2 * math.pi * (np.arange(m) + 0.5 * (k % 2)) / m
        s.extend(k * h * np.cos(a))
        t.extend(k * h * np.sin(a))
        r.extend([k * h] * m)
    s, t = np.array(s), np.array(t)
    p = np.array([0.2, -0.1, 0.4]) + s[:, None] * e1 + t[:, None] * e2
    return p.astype(np.float32), np.tile(nz, (len(p), 1)).astype(np.float32), np.array(r)


def test_disc_rim_is_boundary_and_interior_is_not(o3d):
    h, R = 0.01, 0.3
    pts, nrm, r = _disc(h, R)
    pc = o3d.t.geometry.PointCloud(torch.from_numpy(pts).cuda()).set_point_normals(torch.from_numpy(nrm).cuda())
    out, mask = pc.compute_boundary_points(3 * h, 30)
    m = mask.cpu().numpy()
    rim = r > R - h / 2
    assert rim.sum() == round(2 * math.pi * R / h) and m[rim].all()
    assert not m[r < R - 3.5 * h].any()
    assert np.array_equal(out.point["positions"].cpu().numpy(), pts[m])


def test_hole_is_found(o3d):
    h, hole = 0.01, 0.1
    pts, nrm, s, t = _plane_lattice(lambda s, t: np.hypot(s - 0.05, t + 0.02) > hole, h=h)
    rh = np.hypot(s - 0.05, t + 0.02)
    edge = np.maximum(np.abs(s), np.abs(t)) > 0.4 - 3.5 * h   # the square's own edge
    pc = o3d.t.geometry.PointCloud(torch.from_numpy(pts).cuda()).set_point_normals(torch.from_numpy(nrm).cuda())
    _, mask = pc.compute_boundary_points(3 * h, 30)
    m = mask.cpu().numpy()
    assert m[rh < hole + h].all()
    assert not m[(rh > hole + 3.5 * h) & ~edge].any()


def test_z_facing_plane_has_no_boundary(o3d):
    g = np.arange(40) * 0.01
    a, b = np.meshgrid(g, g)
    pts = np.stack([a.ravel(), b.ravel(), np.full(a.size, 0.5)], 1).astype(np.float32)
    for z in (1.0, -1.0):
        nrm = np.tile(np.float32([0.0, 0.0, z]), (len(pts), 1))
        pc = o3d.t.geometry.PointCloud(torch.from_numpy(pts).cuda()).set_point_normals(torch.from_numpy(nrm).cuda())
        out, mask = pc.compute_boundary_points(0.03)
        assert not mask.any() and out.point["positions"].shape == (0, 3)


def test_point_cloud_api_carries_attributes(o3d, cases):
    pts, nrm, radius, max_nn = cases["normals_tilted"]
    rng = np.random.default_rng(3)
    col = rng.uniform(0, 1, (len(pts), 3)).astype(np.float32)
    pc = o3d.t.geometry.PointCloud(torch.from_numpy(pts).cuda()).set_point_normals(torch.from_numpy(nrm).cuda())
    pc.set_point_colors(torch.from_numpy(col).cuda())
    out, mask = pc.compute_boundary_points(radius, max_nn, 70.0)
    assert mask.dtype == torch.bool and mask.device.type == "cuda" and mask.shape == (len(pts),)
    want, _ = ob.compute_boundary_points(pts, nrm, radius, max_nn, 70.0, mode="f64")
    m = mask.cpu().numpy()
    assert np.array_equal(m, want) and m.sum() > 0
    assert set(out.point) == {"positions", "normals", "colors"}
    for key, arr in (("positions", pts), ("normals", nrm), ("colors", col)):
        assert np.array_equal(out.point[key].cpu().numpy(), arr[m])
    # defaults: max_nn 30, 90 degrees
    _, m90 = pc.compute_boundary_points(radius)
    assert np.array_equal(m90.cpu().numpy(), ob.compute_boundary_points(pts, nrm, radius, 30, 90.0)[0])


def test_argument_errors_and_empty_clouds(o3d):
    pts = nc.scan(2000, seed=4)
    pc = o3d.t.geometry.PointCloud(pts)
    with pytest.raises(RuntimeError, match=r"PointCloud must have normals attribute to compute boundary points\."):
        pc.compute_boundary_points(0.05)
    pc.set_point_normals(np.tile(np.float32([0.0, 0.6, 0.8]), (len(pts), 1)))
    for bad in (0, 33):
        with pytest.raises(RuntimeError, match=r"max_nn must be in 1\.\.32"):
            pc.compute_boundary_points(0.05, bad)
    for bad in (0.0, -1.0, float("nan")):
        with pytest.raises(RuntimeError, match="radius must be positive"):
            pc.compute_boundary_points(bad)
    f64 = o3d.t.geometry.PointCloud()
    f64.point["positions"] = torch.from_numpy(pts.astype(np.float64)).cuda()
    f64.point["normals"] = torch.zeros((len(pts), 3), dtype=torch.float64, device="cuda")
    with pytest.raises(RuntimeError, match="Float32"):
        f64.compute_boundary_points(0.05)
    empty = o3d.t.geometry.PointCloud(np.zeros((0, 3), np.float32)).set_point_normals(np.zeros((0, 3), np.float32))
    out, mask = empty.compute_boundary_points(0.05)
    assert mask.shape == (0,) and mask.dtype == torch.bool and out.point["positions"].shape == (0, 3)
    out, mask = o3d.t.geometry.PointCloud(np.zeros((0, 3), np.float32)).compute_boundary_points(0.05)
    assert mask.shape == (0,) and out.point["positions"].shape == (0, 3)
    L = _lib()
    assert L.lib.o3db_compute_boundary_points(None, None, 0, 0.05, 30, 90.0, None, None, _stream()) == 0


def test_non_finite_input_is_rejected(o3d):
    pts = nc.scan(3000, seed=5)
    nrm = np.tile(np.float32([0.0, 0.6, 0.8]), (len(pts), 1))
    for where, value in (("positions", np.nan), ("positions", np.inf), ("positions", -np.inf), ("normals", np.inf),
                         ("normals", -np.inf)):
        p, q = pts.copy(), nrm.copy()
        (p if where == "positions" else q)[1234, 1] = value
        pc = o3d.t.geometry.PointCloud(p).set_point_normals(q)
        with pytest.raises(RuntimeError, match="non-finite positions or infinite normal components"):
            pc.compute_boundary_points(0.05)
    q = nrm.copy()
    q[1234, 0] = np.nan   # a NaN normal is upstream's NaN frame: accepted, and never a boundary point
    _, mask = o3d.t.geometry.PointCloud(pts).set_point_normals(q).compute_boundary_points(0.05)
    assert not mask[1234].item()


def test_launch_count_is_fixed_per_call(o3d, cases):
    L = _lib()
    steps = []
    for name in ("normals_scan", "lattice4", "special_normals", "single"):
        pts, nrm, radius, max_nn = cases[name]
        pc = o3d.t.geometry.PointCloud(pts).set_point_normals(nrm)
        before = L.launch_count()
        pc.compute_boundary_points(radius, max_nn)
        torch.cuda.synchronize()
        steps.append(L.launch_count() - before)
    assert steps[0] >= 3 and len(set(steps)) == 1, steps


def test_memory_balances_on_success_and_failure(o3d):
    if torch.cuda.get_allocator_backend() == "cudaMallocAsync":
        pytest.skip("torch shares the default memory pool")
    from tests.test_host_ownership_gpu import _Pool
    L = _lib()
    pool = _Pool()
    pts = nc.scan(50000, seed=6)
    p = torch.from_numpy(pts).cuda()
    q = torch.from_numpy(np.tile(np.float32([0.0, 0.6, 0.8]), (len(pts), 1))).cuda()
    bad = q.clone()
    bad[7, 2] = float("inf")
    mask = torch.empty(len(pts), dtype=torch.uint8, device="cuda")
    rows = []

    def balanced(name, nrm, max_nn, expect=0):
        u0 = pool.used()
        rc = L.lib.o3db_compute_boundary_points(p.data_ptr(), nrm.data_ptr(), len(pts), 0.05, max_nn, 90.0,
                                                mask.data_ptr(), None, _stream())
        assert rc == expect, (name, rc, L.last_error())
        rows.append((name, u0, pool.used()))

    for _ in range(2):
        balanced("ok", q, 30)
        balanced("infinite normal", bad, 30, L.ERR_INVALID)
        balanced("max_nn 33", q, 33, L.ERR_INVALID)
    torch.cuda.synchronize()
    for name, u0, u1 in rows:
        assert u1 == u0, (name, u0, u1)
