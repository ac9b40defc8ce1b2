"""RANSAC registration on the GPU (o3db_registration_ransac, registration.registration_ransac_based_on_*) against the
CPU oracle (oracle/ransac) on the library's own draws: every bit of the result, the counts and the engine's state
after the call; then the global registration pipeline end to end."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import ransac as orc
from tests import ransac_cases as rc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


def _L():
    from open3d_b200 import _lib
    return _lib


def _draws(seed, K, count):
    L = _L()
    L.check(L.lib.o3db_random_seed(seed))
    out = np.zeros(count, np.int32)
    L.check(L.lib.o3db_random_uniform_ints(0, max(K - 1, 0), count, out.ctypes.data))
    return out


def _next_draw(K):
    L = _L()
    out = np.zeros(1, np.int32)
    L.check(L.lib.o3db_random_uniform_ints(0, max(K - 1, 0), 1, out.ctypes.data))
    return int(out[0])


def _ransac(src, tgt, c, dist, rn, max_it, conf, ck=None, sn=None, tn=None):
    """The C ABI call on device copies -> (T [4,4], corres [n], stats)."""
    L = _L()
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    s, t, dsn, dtn = dev(src), dev(tgt), dev(sn), dev(tn)
    dc = torch.from_numpy(np.ascontiguousarray(c, np.int64).reshape(-1, 2)).cuda()
    n = src.shape[0]
    out = torch.empty(max(n, 1), dtype=torch.int64, device="cuda")
    T = np.zeros(16)
    st = L.RansacStats()
    ckc = None if ck is None else C.byref(L.RansacCheckers(*[getattr(ck, f) for f, _ in ck._fields_]))
    L.check(L.lib.o3db_registration_ransac(s.data_ptr(), None if dsn is None else dsn.data_ptr(), n, t.data_ptr(),
                                           None if dtn is None else dtn.data_ptr(), tgt.shape[0], dc.data_ptr(),
                                           dc.shape[0], float(dist), rn, max_it, float(conf), ckc, T.ctypes.data,
                                           out.data_ptr(), C.byref(st), int(torch.cuda.current_stream().cuda_stream)))
    return T.reshape(4, 4), out[:n].cpu().numpy(), st


def _check(src, tgt, c, dist, rn, max_it, conf, ck=None, sn=None, tn=None, seed=7):
    K = len(c)
    draws = _draws(seed, K, max_it * rn + 1) if K >= 1 and max_it > 0 else np.zeros(1, np.int32)
    _L().check(_L().lib.o3db_random_seed(seed))
    T, corr, st = _ransac(src, tgt, c, dist, rn, max_it, conf, ck, sn, tn)
    want = orc.ransac(src, tgt, c, draws, dist, rn, max_it, conf, ck, sn, tn)
    got = (st.drawn, st.validated, st.best_index)
    assert got == (want.drawn, want.validated, want.best_index), (got, want[2:])
    assert st.fitness == want.fitness and st.inlier_rmse == want.rmse, (st.fitness, want.fitness, st.inlier_rmse,
                                                                        want.rmse)
    np.testing.assert_array_equal(T, want.transformation)
    np.testing.assert_array_equal(corr, want.correspondence_set)
    if K >= 1 and max_it > 0 and not (rn < 3 or K < rn or dist <= 0):
        assert _next_draw(K) == draws[want.drawn * rn], "the engine is not where one thread leaves it"
    return want


@pytest.mark.parametrize("ratio", [0.05, 0.3, 1.0])
@pytest.mark.parametrize("rn", [3, 4, 10, 64])
def test_ratios_and_sample_sizes(o3d, ratio, rn):
    src, tgt, c, _ = rc.pair(3000, 1500, ratio, seed=rn)
    _check(src, tgt, c, 0.02, rn, 300, 0.999)


@pytest.mark.parametrize("conf", [0.0, 0.5, 0.999, 1.0, float("nan")])
def test_confidence(o3d, conf):
    src, tgt, c, _ = rc.pair(2000, 1000, 0.3, seed=2)
    _check(src, tgt, c, 0.02, 3, 400, conf)


@pytest.mark.parametrize("which", ["edge", "distance", "normal", "normal_without_normals", "all"])
def test_checkers(o3d, which):
    src, tgt, c, T = rc.pair(2000, 1000, 0.3, seed=4)
    sn = rc.normals(len(src), 4)
    tn = (sn.astype(np.float64) @ T[:3, :3].T).astype(np.float32)
    kw = {"edge": dict(edge=0.9), "distance": dict(distance=0.03), "normal": dict(normal_angle=0.3),
          "normal_without_normals": dict(normal_angle=0.3), "all": dict(edge=0.9, distance=0.03, normal_angle=0.3)}
    with_normals = which != "normal_without_normals"
    w = _check(src, tgt, c, 0.02, 3, 2000, 0.999, orc.checkers(**kw[which]), sn if with_normals else None,
               tn if with_normals else None)
    if which != "normal_without_normals":
        assert w.validated < w.drawn


def test_early_stop_across_waves_and_batches(o3d):
    """Without checkers and with confidence 1 every hypothesis is validated: the loop runs through many waves and past
    a batch boundary (8192) without stopping.  With the edge checker few pass, and at 0.999 it stops early."""
    src, tgt, c, _ = rc.pair(600, 400, 0.05, seed=9)
    w = _check(src, tgt, c, 0.02, 3, 9000, 1.0)
    assert w.drawn == 9000 and w.validated == 9000
    src, tgt, c, _ = rc.pair(1500, 800, 0.3, seed=9)
    w = _check(src, tgt, c, 0.02, 3, 20000, 0.999, orc.checkers(edge=0.9))
    assert w.drawn < 20000


@pytest.mark.parametrize("case", ["max_iteration_0", "max_iteration_1", "k_below_n", "distance_0", "ransac_n_2"])
def test_early_outs(o3d, case):
    src, tgt, c, _ = rc.pair(500, 200, 0.5, seed=1)
    args = {"max_iteration_0": (c, 0.02, 3, 0), "max_iteration_1": (c, 0.02, 3, 1), "k_below_n": (c[:2], 0.02, 3, 10),
            "distance_0": (c, 0.0, 3, 10), "ransac_n_2": (c, 0.02, 2, 10)}[case]
    cc, d, rn, it = args
    _L().check(_L().lib.o3db_random_seed(3))
    before = _next_draw(len(cc))
    _L().check(_L().lib.o3db_random_seed(3))
    T, corr, st = _ransac(src, tgt, cc, d, rn, it, 0.999)
    if case == "max_iteration_1":
        _check(src, tgt, cc, d, rn, it, 0.999, seed=3)
        return
    assert _next_draw(len(cc)) == before, "an early out consumed draws"
    np.testing.assert_array_equal(T, np.eye(4))
    assert (corr == -1).all() and st.drawn == 0 and st.best_index == -1


def test_repeated_indices_in_a_sample(o3d):
    src, tgt, c, _ = rc.pair(1000, 6, 1.0, seed=5)
    _check(src, tgt, c, 0.02, 4, 200, 1.0)


def test_ties(o3d):
    src, tgt, c, _ = rc.ties(1500, seed=6)
    w = _check(src, tgt, c, 0.02, 3, 200, 0.999)
    assert (w.correspondence_set[w.correspondence_set >= 0] < 1500).all()   # ties go to the lower copy


def _permutation_seed(K, rn):
    """A seed whose first rn draws of uniform_int_distribution<int>(0, K-1) are all different."""
    for seed in range(1000):
        d = _draws(seed, K, rn)
        if len(set(d.tolist())) == rn:
            return seed
    raise AssertionError("no seed found")


def test_radius_probes(o3d):
    """Points exactly at the distance, one f32 ulp inside and one outside, along each axis and at |q| of 5, 1000 and
    30000, under an estimate that is exactly the identity: the strict d^2 < r^2 and the widened search box."""
    src, tgt, c, expect = rc.radius_probes()
    seed = _permutation_seed(4, 4)
    w = _check(src, tgt, c, rc.RADIUS, 4, 1, 1.0, seed=seed)
    np.testing.assert_array_equal(w.transformation, np.eye(4))
    np.testing.assert_array_equal(w.correspondence_set, expect)


def _pinned_stop(i, seed=3, n=300, K=20000):
    """Correspondences on which, with the draws of `seed`, the first hypothesis with a match is exactly hypothesis i:
    every pair is a wrong match except the three that hypothesis i draws, which are true (the target is the source
    moved without noise), and the distance is 1e-5, so that no other hypothesis matches a point.  With confidence 0 the
    first hypothesis with a match sets est_k = 0, so the run stops at i + 1."""
    rng = np.random.default_rng(i)
    src = rc.cloud(n, i)
    T = rc.motion()
    tgt = (src.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    d = _draws(seed, K, 3 * (i + 1)).reshape(-1, 3)
    pick = d[i]
    assert len(set(pick.tolist())) == 3
    assert not any(set(row.tolist()) <= set(pick.tolist()) for row in d[:i])
    a = rng.integers(0, n, K)
    c = np.stack([a, (a + rng.integers(1, n, K)) % n], 1).astype(np.int64)
    for k, p in enumerate(pick):
        c[p] = (k * 97 + 5, k * 97 + 5)
    return src, tgt, c


@pytest.mark.parametrize("i", [40, 63, 64, 8191, 9000])
def test_early_stop_pinned(o3d, i):
    """The stop falls mid-wave (40), at the end of the first wave of 64 (63) and at the start of the next (64), at the
    end of the first batch of 8192 (8191) and inside the second batch (9000), where the engine is restored and the
    batch's prefix replayed."""
    src, tgt, c = _pinned_stop(i)
    w = _check(src, tgt, c, 1e-5, 3, 10000, 0.0, seed=3)
    assert w.drawn == i + 1 and w.validated == i + 1 and w.best_index == i and w.fitness > 0


def test_normal_checker_warns_without_normals(o3d, capsys):
    reg = o3d.t.pipelines.registration
    src, tgt, c, _ = rc.pair(500, 200, 0.5, seed=1)
    P = o3d.t.geometry.PointCloud
    reg.registration_ransac_based_on_correspondence(
        P(torch.from_numpy(src).cuda()), P(torch.from_numpy(tgt).cuda()), c, 0.02,
        checkers=[reg.CorrespondenceCheckerBasedOnNormal(0.3)], criteria=reg.RANSACConvergenceCriteria(10, 0.999))
    assert "[CorrespondenceCheckerBasedOnNormal::Check] Pointcloud has no normals." in capsys.readouterr().out


def test_argument_errors(o3d):
    reg = o3d.t.pipelines.registration
    src, tgt, c, _ = rc.pair(500, 200, 0.5, seed=1)
    P = o3d.t.geometry.PointCloud
    s, t = P(torch.from_numpy(src).cuda()), P(torch.from_numpy(tgt).cuda())
    with pytest.raises(RuntimeError, match="Float32"):
        reg.registration_ransac_based_on_correspondence(P(torch.from_numpy(src).double().cuda()), t, c, 0.02)
    bad = src.copy()
    bad[3, 1] = np.nan
    with pytest.raises(RuntimeError, match="remove_non_finite_points"):
        reg.registration_ransac_based_on_correspondence(P(torch.from_numpy(bad).cuda()), t, c, 0.02)
    with pytest.raises(RuntimeError, match="remove_non_finite_points"):
        reg.registration_ransac_based_on_correspondence(s, P(torch.from_numpy(bad).cuda()), c, 0.02)
    for cc in (np.array([[0, 500], [1, 1], [2, 2]]), np.array([[-1, 0], [1, 1], [2, 2]])):
        with pytest.raises(RuntimeError, match="outside"):
            reg.registration_ransac_based_on_correspondence(s, t, cc, 0.02)
    with pytest.raises(RuntimeError, match="supported"):
        reg.registration_ransac_based_on_correspondence(s, t, c, 0.02, checkers=[object()])
    with pytest.raises(RuntimeError, match="PointToPoint"):
        reg.registration_ransac_based_on_correspondence(s, t, c, 0.02, reg.TransformationEstimationPointToPlane())
    with pytest.raises(RuntimeError, match="finite"):
        reg.registration_ransac_based_on_correspondence(s, t, c, float("inf"))
    with pytest.raises(RuntimeError, match="rows"):
        reg.registration_ransac_based_on_feature_matching(s, t, torch.zeros(3, 33), torch.zeros(500, 33), False, 0.02)


def test_criteria_clamp():
    from open3d_b200.t.pipelines.registration import RANSACConvergenceCriteria as R
    assert R().max_iteration == 100000 and R().confidence == 0.999
    assert R(10, 2.0).confidence == 1.0 and R(10, -1.0).confidence == 0.0 and math.isnan(R(10, math.nan).confidence)


def test_python_call_matches_c_abi(o3d):
    reg = o3d.t.pipelines.registration
    src, tgt, c, _ = rc.pair(2000, 1000, 0.3, seed=8)
    P = o3d.t.geometry.PointCloud
    s, t = P(torch.from_numpy(src).cuda()), P(torch.from_numpy(tgt).cuda())
    o3d.utility.random.seed(11)
    res = reg.registration_ransac_based_on_correspondence(
        s, t, torch.from_numpy(c.astype(np.int32)), 0.02, reg.TransformationEstimationPointToPoint(), 3,
        [reg.CorrespondenceCheckerBasedOnEdgeLength(0.9), reg.CorrespondenceCheckerBasedOnDistance(0.03)],
        reg.RANSACConvergenceCriteria(1000, 0.999))
    _L().check(_L().lib.o3db_random_seed(11))
    T, corr, st = _ransac(src, tgt, c, 0.02, 3, 1000, 0.999, orc.checkers(edge=0.9, distance=0.03))
    np.testing.assert_array_equal(res.transformation, T)
    np.testing.assert_array_equal(res.correspondence_set.cpu().numpy(), corr)
    assert res.fitness == st.fitness and res.inlier_rmse == st.inlier_rmse
    assert not res.converged and res.num_iterations == 0


def _sorted_cloud(P, pc):
    """The cloud's points in lexicographic order: the down-sampled order varies from run to run, and the pairs the
    draws pick with it."""
    p = pc.point["positions"].cpu().numpy()
    return P(torch.from_numpy(np.ascontiguousarray(p[np.lexsort((p[:, 2], p[:, 1], p[:, 0]))])).cuda())


def test_global_registration_pipeline(o3d):
    """voxel_down_sample -> estimate_normals -> compute_fpfh_feature -> RANSAC on the feature matches, then
    point-to-plane ICP from its pose (at two voxels, then at one lattice spacing), on a partially overlapping, noisy
    copy turned 100 degrees about an oblique axis.  The down-sampled clouds are sorted, so the run is reproducible."""
    reg = o3d.t.pipelines.registration
    P = o3d.t.geometry.PointCloud
    pts = rc.scene(150, 0.02, 1)   # 22 500 points, 3 m x 3 m
    src, tgt, T = rc.overlap_pair(pts, 2)
    voxel = 0.05
    clouds = []
    for p in (src, tgt):
        pc = _sorted_cloud(P, P(torch.from_numpy(p.astype(np.float32)).cuda()).voxel_down_sample(voxel))
        pc.estimate_normals(30, 2 * voxel)
        clouds.append((pc, reg.compute_fpfh_feature(pc, 100, 5 * voxel)))
    (s, fs), (t, ft) = clouds
    o3d.utility.random.seed(0)
    res = reg.registration_ransac_based_on_feature_matching(
        s, t, fs, ft, False, 1.5 * voxel, reg.TransformationEstimationPointToPoint(), 3,
        [reg.CorrespondenceCheckerBasedOnEdgeLength(0.9), reg.CorrespondenceCheckerBasedOnDistance(1.5 * voxel)],
        reg.RANSACConvergenceCriteria(100000, 0.999))
    G = res.transformation
    ang = math.degrees(math.acos(max(-1.0, min(1.0, (np.trace(G[:3, :3].T @ T[:3, :3]) - 1) / 2))))
    shift = float(np.linalg.norm(G[:3, 3] - T[:3, 3]))
    print(f"ransac: fitness {res.fitness:.4f} rmse {res.inlier_rmse:.5f} angle {ang:.3f} deg shift {shift:.4f}")
    assert ang < 3.0 and shift < 2 * voxel, (ang, shift)
    sf = P(torch.from_numpy(src.astype(np.float32)).cuda())
    tf = P(torch.from_numpy(tgt.astype(np.float32)).cuda())
    tf.estimate_normals(30, 0.06)
    crit = reg.ICPConvergenceCriteria(1e-9, 1e-9, 50)
    est = reg.TransformationEstimationPointToPlane()
    coarse = reg.icp(sf, tf, 2 * voxel, G, est, crit)
    fine = reg.icp(sf, tf, 0.02, coarse.transformation, est, crit)
    err = np.abs(fine.transformation - T).max()
    blind = reg.icp(sf, tf, 2 * voxel, np.eye(4), est, crit)
    err_blind = np.abs(reg.icp(sf, tf, 0.02, blind.transformation, est, crit).transformation - T).max()
    print(f"icp from ransac: max |T - truth| {err:.2e}; from the identity {err_blind:.2e}")
    assert err < 1e-3 and err_blind > 1e-1, (err, err_blind)
