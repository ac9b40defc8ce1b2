"""PointCloud.estimate_normals and the two orient_normals calls on the GPU against the CPU oracle (oracle/normals),
which is itself bit-exact against the reference's own code (tests/test_oracle_vs_ref_normals.py).

Neighbour counts and covariances must be bit-identical.  Normals cannot all be: the reference's eigen solve calls
libm's acosf / cosf, which are not correctly rounded, and the GPU evaluates acos / cos in f64 and rounds.  So at least
95 % of the rows must be bit-identical, the fallback rows exactly so, and every other row must be a unit eigenvector
of the same covariance (see _check_normals)."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from oracle import normals as on
from tests import normals_cases as nc
from tests.synth import make_colors, make_icp_pair

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


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def _gpu_normals(pts, radius, max_nn, prior=None):
    """o3db_estimate_normals with the covariance output, and the hybrid search's neighbour counts."""
    L = _lib()
    p = _dev(pts)
    n = p.shape[0]
    nrm = _dev(prior) if prior is not None else torch.full((n, 3), float("nan"), device="cuda")
    cov = torch.full((n, 9), float("nan"), device="cuda")
    L.check(L.lib.o3db_estimate_normals(p.data_ptr(), n, float(radius), int(max_nn), int(prior is not None),
                                        nrm.data_ptr(), cov.data_ptr(), _stream()))
    h = C.c_void_p()
    L.check(L.lib.o3db_nns_create(p.data_ptr(), n, float(radius), _stream(), C.byref(h)))
    cnt = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    L.check(L.lib.o3db_nns_hybrid_search(h, p.data_ptr(), n, float(radius), int(max_nn), None, None, cnt.data_ptr(),
                                         _stream()))
    torch.cuda.synchronize()
    L.lib.o3db_nns_destroy(h)
    return nrm.cpu().numpy(), cov.cpu().numpy(), cnt.cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _fallback_rows(cov):
    """rows the eigen solve does not reach: a zero covariance, or exactly zero off-diagonals (f32, as the kernel)"""
    mx = cov.max(axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        A = cov / mx[:, None]
        norm = A[:, 1] * A[:, 1] + A[:, 2] * A[:, 2] + A[:, 5] * A[:, 5]
    return (mx == 0) | ~(norm > 0)


def _check_normals(got, want, cov, prior=None):
    """-> the fraction of bit-identical rows, after checking every row against the oracle's"""
    same = (_bits(got) == _bits(want)).all(axis=1)
    assert same.mean() >= 0.95, same.mean()
    fb = _fallback_rows(cov)
    assert same[fb].all()                                       # (0,0,1), the axis vectors, zero under a prior
    zero = ~want.any(axis=1)
    if prior is None:
        assert not zero.any()
    norm = np.linalg.norm(got.astype(np.float64), axis=1)
    assert (np.abs(norm[~zero] - 1.0) <= 1e-5).all(), np.abs(norm[~zero] - 1.0).max()
    differ = np.flatnonzero(~same)
    if len(differ):
        C3 = cov[differ].reshape(-1, 3, 3).astype(np.float64)
        lam = np.linalg.eigvalsh(C3)
        g, w = got[differ].astype(np.float64), want[differ].astype(np.float64)
        gap = (lam[:, 1] - lam[:, 0]) >= 1e-3 * lam[:, 2]
        assert (np.abs((g[gap] * w[gap]).sum(1)) >= 1 - 1e-5).all()
        rq = np.einsum("ni,nij,nj->n", g[~gap], C3[~gap], g[~gap])
        assert (rq <= lam[~gap, 1] + 1e-5 * lam[~gap, 2]).all()
    if prior is not None:
        pw = (prior.astype(np.float64) * want).sum(1)
        pg = (prior.astype(np.float64) * got).sum(1)
        decided = np.abs(pw) > 1e-3
        assert (np.sign(pg[decided]) == np.sign(pw[decided])).all()
    return float(same.mean())


def _prior(normals, seed):
    rng = np.random.default_rng(seed)
    prior = normals * rng.choice([-1.0, 1.0], (len(normals), 1))
    prior[::7] = 0.0
    return np.ascontiguousarray(prior, np.float32)


@pytest.mark.parametrize("name", sorted(nc.cases()))
def test_cases_vs_oracle(name):
    pts, radius, max_nn = nc.cases()[name]
    want, want_cov, want_cnt = on.estimate_normals(pts, radius, max_nn)
    got, cov, cnt = _gpu_normals(pts, radius, max_nn)
    assert np.array_equal(cnt, want_cnt)
    assert np.array_equal(_bits(cov), _bits(want_cov))
    _check_normals(got, want, want_cov)
    prior = _prior(want, 5)
    want_p, _, _ = on.estimate_normals(pts, radius, max_nn, prior_normals=prior)
    got_p, _, _ = _gpu_normals(pts, radius, max_nn, prior)
    _check_normals(got_p, want_p, want_cov, prior)


@pytest.mark.parametrize("n,radius,max_nn", [(20000, 0.08, 30), (20000, 0.03, 16), (2000000, 0.08, 30),
                                             (2000000, 0.04, 30)])
def test_icp_target_vs_oracle(n, radius, max_nn):
    _, tgt, _, _ = make_icp_pair(n, seed=2)
    want, want_cov, want_cnt = on.estimate_normals(tgt, radius, max_nn)
    got, cov, cnt = _gpu_normals(tgt, radius, max_nn)
    assert np.array_equal(cnt, want_cnt)
    assert np.array_equal(_bits(cov), _bits(want_cov))
    frac = _check_normals(got, want, want_cov)
    print(f"\n{n} points, radius {radius}, max_nn {max_nn}: {frac:.6f} of the normals bit-identical")


def test_point_cloud_api(o3d):
    """estimate_normals sets "normals" in place and orients against existing ones; the orient calls match the
    oracle bit for bit, zero-norm fallbacks included."""
    pts, radius, max_nn = nc.cases()["scan"]
    pc = o3d.t.geometry.PointCloud(pts)
    assert pc.estimate_normals(max_nn, radius) is pc
    got = pc.point["normals"].cpu().numpy()
    want, cov, _ = on.estimate_normals(pts, radius, max_nn)
    _check_normals(got, want, cov)
    prior = _prior(want, 9)
    pc.set_point_normals(prior)
    buf = pc.point["normals"]
    pc.estimate_normals(max_nn, radius)
    assert pc.point["normals"].data_ptr() == buf.data_ptr()       # in place, like upstream
    want_p, _, _ = on.estimate_normals(pts, radius, max_nn, prior_normals=prior)
    _check_normals(pc.point["normals"].cpu().numpy(), want_p, cov, prior)

    rng = np.random.default_rng(3)
    nrm = rng.normal(size=pts.shape).astype(np.float32)
    nrm[::9] = 0.0
    for d in ((0.0, 0.0, 1.0), (0.3, -0.7, 0.2), (0.0, 0.0, 0.0)):
        pc.set_point_normals(nrm)
        pc.orient_normals_to_align_with_direction(d)
        assert np.array_equal(_bits(pc.point["normals"].cpu().numpy()),
                              _bits(on.orient_normals_to_align_with_direction(nrm, d)))
    pts2 = pts.copy()
    pts2[::18] = [0.25, -0.5, 0.75]
    pc2 = o3d.t.geometry.PointCloud(pts2)
    for cam in ((0.25, -0.5, 0.75), (0.0, 0.0, 0.0), (10.0, 3.0, -2.0)):
        pc2.set_point_normals(nrm)
        pc2.orient_normals_towards_camera_location(cam)
        got = pc2.point["normals"].cpu().numpy()
        assert np.array_equal(_bits(got), _bits(on.orient_normals_towards_camera_location(pts2, nrm, cam)))
    pc2.set_point_normals(nrm)
    pc2.orient_normals_towards_camera_location(torch.tensor([0.25, -0.5, 0.75], dtype=torch.float64))
    assert (pc2.point["normals"].cpu().numpy()[::18] == [0, 0, 1]).all()


def test_icp_with_estimated_normals_recovers_the_motion(o3d):
    """Point-to-plane ICP and ColoredICP on a target whose normals (and colour gradients) the GPU estimated."""
    reg = o3d.t.pipelines.registration
    src, tgt, _, T_gt = make_icp_pair(40000, seed=31)
    s = o3d.t.geometry.PointCloud(src)
    t = o3d.t.geometry.PointCloud(tgt).estimate_normals(30, 0.08)
    res = reg.icp(s, t, 0.05, np.eye(4), reg.TransformationEstimationPointToPlane(),
                  reg.ICPConvergenceCriteria(0, 0, 30))
    np.testing.assert_allclose(res.transformation, T_gt, atol=2e-3)

    sc, tc = make_colors(oracle.transform_points(T_gt, src), 1), make_colors(tgt, 1)
    s = o3d.t.geometry.PointCloud(src).set_point_colors(sc)
    t = o3d.t.geometry.PointCloud(tgt).set_point_colors(tc).estimate_normals(30, 0.08)
    t.estimate_color_gradients(30, 0.08)
    res = reg.icp(s, t, 0.05, np.eye(4), reg.TransformationEstimationForColoredICP(),
                  reg.ICPConvergenceCriteria(0, 0, 30))
    np.testing.assert_allclose(res.transformation, T_gt, atol=2e-3)


def test_argument_errors(o3d):
    pts = nc.scan(2000, seed=4)
    pc = o3d.t.geometry.PointCloud(pts)
    with pytest.raises(RuntimeError, match="hybrid-search"):
        pc.estimate_normals(30)
    for bad in (0, 33):
        with pytest.raises(RuntimeError, match="max_nn"):
            pc.estimate_normals(bad, 0.05)
    with pytest.raises(RuntimeError, match="radius"):
        pc.estimate_normals(30, -1.0)
    assert "normals" not in pc.point
    f64 = o3d.t.geometry.PointCloud()
    f64.point["positions"] = torch.from_numpy(pts.astype(np.float64)).cuda()
    with pytest.raises(RuntimeError, match="Float32"):
        f64.estimate_normals(30, 0.05)
    msg = "No normals in the PointCloud. Call EstimateNormals\\(\\) first."
    with pytest.raises(RuntimeError, match=msg):
        pc.orient_normals_to_align_with_direction()
    with pytest.raises(RuntimeError, match=msg):
        pc.orient_normals_towards_camera_location()
    with pytest.raises(RuntimeError, match="shape"):
        pc.set_point_normals(pts).orient_normals_to_align_with_direction((0.0, 1.0))
    empty = o3d.t.geometry.PointCloud(np.zeros((0, 3), np.float32))
    assert empty.estimate_normals(30, 0.05).point["normals"].shape == (0, 3)


def test_launch_count_is_fixed_per_call(o3d):
    L = _lib()
    steps = []
    for n, radius, max_nn in ((2000, 0.05, 30), (50000, 0.08, 8), (50000, 0.02, 30)):
        pc = o3d.t.geometry.PointCloud(nc.scan(n, seed=6))
        before = L.launch_count()
        pc.estimate_normals(max_nn, radius)
        torch.cuda.synchronize()
        steps.append(L.launch_count() - before)
    assert steps[0] >= 2 and len(set(steps)) == 1, steps
