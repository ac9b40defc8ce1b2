"""Doppler ICP on the GPU (TransformationEstimationForDopplerICP): the reduction seam against the CPU oracle
(oracle/doppler) for every robust pair, the fused loop against the oracle loop (through iterations where chunks replay
their cached sums), the three switch iterations, a 3-scale pyramid, determinism, misuse, and the corridor whose free
axis only the Doppler term constrains."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import doppler as dop
from tests.doppler_cases import CALIB, make_corridor, make_doppler_pair

pytestmark = pytest.mark.gpu

KERNELS = [(0, 1.0, 1.0), (5, 0.4, 1.0)]


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


def _clouds(o3d, src, d, dirs, tgt, nrm):
    S = o3d.t.geometry.PointCloud(src)
    S.point["dopplers"] = torch.from_numpy(np.ascontiguousarray(d, np.float32)).cuda()
    S.point["directions"] = torch.from_numpy(np.ascontiguousarray(dirs, np.float32)).cuda()
    return S, o3d.t.geometry.PointCloud(tgt).set_point_normals(nrm)


def _est(o3d, **kw):
    reg = o3d.t.pipelines.registration
    for k in ("geometric_kernel", "doppler_kernel"):
        if isinstance(kw.get(k), tuple):
            m, s, sh = kw[k]
            kw[k] = reg.RobustKernel(reg.RobustKernelMethod(m), s, sh)
    return reg.TransformationEstimationForDopplerICP(**kw)


@pytest.mark.parametrize("kg", KERNELS)
@pytest.mark.parametrize("kd", KERNELS)
def test_seam_sums_vs_oracle(o3d, kg, kd):
    src, d, dirs, tgt, nrm, _, _ = make_doppler_pair(200000, seed=kg[0] + 2 * kd[0], dynamic=0.1)
    rng = np.random.default_rng(5)
    corr = rng.integers(0, len(tgt), len(src)).astype(np.int64)
    corr[rng.random(len(src)) < 0.1] = -1
    T = np.eye(4)
    T[:3, 3] = [0.12, -0.05, 0.02]
    est = _est(o3d, lambda_doppler=0.2, reject_dynamic_outliers=True, geometric_kernel=kg, doppler_kernel=kd,
               geometric_robust_loss_min_iteration=1, doppler_robust_loss_min_iteration=3,
               transform_vehicle_to_sensor=CALIB)
    p = dop.from_estimator(est)
    S, Tc = _clouds(o3d, src, d, dirs, tgt, nrm)
    for it in range(5):   # both sides of every switch (geometric 1, rejection 2, Doppler 3)
        pose, residual, count, sums = est.compute_pose(S, Tc, torch.from_numpy(corr), T, it)
        ref = dop.sums(src, d, dirs, tgt, nrm, corr, p, T, it, accumulate_f64=True)
        assert count == int(ref[28]) == int((corr >= 0).sum())
        np.testing.assert_allclose(sums.cpu().numpy(), ref, rtol=2e-5, atol=1e-6 * np.abs(ref).max())
        got = est.compute_transformation(S, Tc, torch.from_numpy(corr), T, it)
        want = dop.compute_transformation(src, d, dirs, tgt, nrm, corr, p, T, it, accumulate_f64=True)
        np.testing.assert_allclose(got, want, atol=2e-6)


def _icp(o3d, S, Tc, r, est, iters, cb=None, init=None):
    reg = o3d.t.pipelines.registration
    return reg.icp(S, Tc, r, np.eye(4) if init is None else init, est, reg.ICPConvergenceCriteria(0, 0, iters), -1.0,
                   cb)


@pytest.mark.parametrize("n,iters,kw", [
    (30000, 1, {}),
    (30000, 30, {}),   # aligned early: the later iterations replay chunks once the velocity repeats
    (60000, 6, dict(reject_dynamic_outliers=True, doppler_kernel=(5, 0.5, 1.0), geometric_kernel=(5, 0.02, 1.0),
                    geometric_robust_loss_min_iteration=2, doppler_robust_loss_min_iteration=4,
                    outlier_rejection_min_iteration=3)),
    (250000, 10, dict(lambda_doppler=0.3, reject_dynamic_outliers=True)),
    (2000000, 4, {}),
])
def test_fused_loop_vs_oracle(o3d, n, iters, kw):
    src, d, dirs, tgt, nrm, T_gt, _ = make_doppler_pair(n, seed=1, dynamic=0.05)
    est = _est(o3d, transform_vehicle_to_sensor=CALIB, **kw)
    S, Tc = _clouds(o3d, src, d, dirs, tgt, nrm)
    log = []
    res = _icp(o3d, S, Tc, 0.05, est, iters, log.append)
    ref = dop.icp(src, d, dirs, tgt, nrm, 0.05, dop.from_estimator(est), max_iteration=iters, relative_fitness=0,
                  relative_rmse=0)
    assert ref.status == 0 and res.num_iterations == ref.num_iterations == iters
    per = np.array([[c["fitness"], c["inlier_rmse"]] for c in log])
    assert per[0, 0] == ref.per_iteration[0, 0]
    np.testing.assert_allclose(per[:, 0], ref.per_iteration[:, 0], atol=2e-4)
    np.testing.assert_allclose(per[:, 1], ref.per_iteration[:, 1], atol=2e-6)
    np.testing.assert_allclose(res.transformation, ref.transformation, atol=2e-5)
    assert abs(res.fitness - ref.fitness) < 2e-4 and abs(res.inlier_rmse - ref.inlier_rmse) < 2e-6
    corr = res.correspondence_set.cpu().numpy()
    assert (corr == ref.correspondences).mean() > 0.999


def test_replay_gives_the_bits_of_recomputation(o3d):
    """iterate(k); finish; iterate(rest) recomputes every chunk after the evaluation pass where one run replays the
    chunks whose points and velocity repeat: both end on the same bits."""
    from open3d_b200 import _lib as L
    src, d, dirs, tgt, nrm, _, _ = make_doppler_pair(120000, seed=4, dynamic=0.05)
    est = _est(o3d, transform_vehicle_to_sensor=CALIB, reject_dynamic_outliers=True)
    keep = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (src, d, dirs, tgt, nrm)]
    opt = L.IcpOptions()
    opt.max_correspondence_distance, opt.max_iteration, opt.relative_fitness, opt.relative_rmse = 0.05, 24, 0.0, 0.0
    p = est._params()
    stream = torch.cuda.current_stream().cuda_stream
    outs = []
    for split in (None, 12):
        h = C.c_void_p()
        L.check(L.lib.o3db_icp_create_doppler(keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), len(src),
                                              keep[3].data_ptr(), keep[4].data_ptr(), len(tgt), L.dptr(np.eye(4)),
                                              C.byref(opt), C.byref(p), None, stream, C.byref(h)))
        res = L.IcpResult()
        corr = torch.empty(len(src), dtype=torch.int64, device="cuda")
        try:
            if split:
                L.check(L.lib.o3db_icp_iterate(h, split, stream))
                L.check(L.lib.o3db_icp_finish(h, C.byref(res), corr.data_ptr(), None, stream))
                L.check(L.lib.o3db_icp_iterate(h, 24 - split, stream))
            else:
                L.check(L.lib.o3db_icp_iterate(h, 24, stream))
            L.check(L.lib.o3db_icp_finish(h, C.byref(res), corr.data_ptr(), None, stream))
        finally:
            L.lib.o3db_icp_destroy(h)
        outs.append((bytes(res.transformation), res.fitness, res.inlier_rmse, corr.cpu().numpy().tobytes()))
    assert outs[0] == outs[1]


def test_switch_thresholds_cross_inside_the_loop(o3d):
    """Each switch at a different iteration, on a run of 7: the loop matches the oracle loop, and a later switch
    changes the result, so each one acts."""
    src, d, dirs, tgt, nrm, _, _ = make_doppler_pair(40000, seed=8, dynamic=0.1)
    S, Tc = _clouds(o3d, src, d, dirs, tgt, nrm)
    kw = dict(transform_vehicle_to_sensor=CALIB, reject_dynamic_outliers=True, lambda_doppler=0.2,
              geometric_kernel=(5, 0.02, 1.0), doppler_kernel=(5, 0.5, 1.0))
    Ts = []
    for mins in ((2, 3, 4), (6, 3, 4), (2, 6, 4), (2, 3, 6)):
        est = _est(o3d, outlier_rejection_min_iteration=mins[0], geometric_robust_loss_min_iteration=mins[1],
                   doppler_robust_loss_min_iteration=mins[2], **kw)
        res = _icp(o3d, S, Tc, 0.05, est, 7)
        ref = dop.icp(src, d, dirs, tgt, nrm, 0.05, dop.from_estimator(est), max_iteration=7, relative_fitness=0,
                      relative_rmse=0)
        np.testing.assert_allclose(res.transformation, ref.transformation, atol=2e-5)
        Ts.append(res.transformation)
    for T in Ts[1:]:
        assert not np.array_equal(T, Ts[0])


def test_multi_scale_with_voxel_pyramid_vs_oracle(o3d):
    reg = o3d.t.pipelines.registration
    src, d, dirs, tgt, nrm, _, _ = make_doppler_pair(90000, seed=16)
    voxels, radii, iters = [0.08, 0.04, 0.02], [0.16, 0.08, 0.05], [5, 6, 8]
    est = _est(o3d, transform_vehicle_to_sensor=CALIB)
    S, Tc = _clouds(o3d, src, d, dirs, tgt, nrm)
    res = reg.multi_scale_icp(S, Tc, voxels, [reg.ICPConvergenceCriteria(0, 0, k) for k in iters], radii, np.eye(4),
                              est)
    # the oracle's pyramid: the same device down-sampling, checked against the averages it must equal
    from open3d_b200.t.pipelines.registration import _doppler_voxel_down_sample
    levels, cur_s, cur_t = [], S, Tc
    for v in reversed(voxels):
        cur_s, cur_t = _doppler_voxel_down_sample(cur_s, v), cur_t.voxel_down_sample(v)
        levels.insert(0, (cur_s, cur_t))
    import oracle
    fine = levels[-1][0]
    want = oracle.voxel_down_sample(src, voxels[-1], dirs)
    assert fine.point["positions"].shape[0] == want["positions"].shape[0]
    T = np.eye(4)
    p = dop.from_estimator(est)
    for (ss, tt), r, k in zip(levels, radii, iters):
        ref = dop.icp(ss.point["positions"].cpu().numpy(), ss.point["dopplers"].cpu().numpy(),
                      ss.point["directions"].cpu().numpy(), tt.point["positions"].cpu().numpy(),
                      tt.point["normals"].cpu().numpy(), r, p, init=T, max_iteration=k, relative_fitness=0,
                      relative_rmse=0)
        T = ref.transformation
    assert res.num_iterations == sum(iters)
    np.testing.assert_allclose(res.transformation, T, atol=5e-5)


def test_entry_points_agree_and_runs_are_bit_identical(o3d):
    from open3d_b200 import _lib as L
    src, d, dirs, tgt, nrm, _, _ = make_doppler_pair(100000, seed=7, dynamic=0.05)
    est = _est(o3d, transform_vehicle_to_sensor=CALIB, reject_dynamic_outliers=True)
    S, Tc = _clouds(o3d, src, d, dirs, tgt, nrm)
    runs = []
    for _ in range(2):
        log = []
        r = _icp(o3d, S, Tc, 0.05, est, 12, log.append)
        runs.append((r.transformation.tobytes(), r.fitness, r.inlier_rmse, r.correspondence_set.cpu().numpy().tobytes(),
                     [(c["fitness"], c["inlier_rmse"]) for c in log]))
    assert runs[0] == runs[1]
    keep = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (src, d, dirs, tgt, nrm)]
    opt = L.IcpOptions()
    opt.max_correspondence_distance, opt.max_iteration, opt.relative_fitness, opt.relative_rmse = 0.05, 12, 0.0, 0.0
    p, res = est._params(), L.IcpResult()
    corr = torch.empty(len(src), dtype=torch.int64, device="cuda")
    L.check(L.lib.o3db_icp_doppler(keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), len(src),
                                   keep[3].data_ptr(), keep[4].data_ptr(), len(tgt), L.dptr(np.eye(4)), C.byref(opt),
                                   C.byref(p), C.byref(res), corr.data_ptr(), None,
                                   torch.cuda.current_stream().cuda_stream))
    assert bytes(res.transformation) == runs[0][0] and res.fitness == runs[0][1]
    assert corr.cpu().numpy().tobytes() == runs[0][3]


def test_misuse_raises(o3d):
    reg = o3d.t.pipelines.registration
    src, d, dirs, tgt, nrm, _, _ = make_doppler_pair(5000, seed=2)
    est = _est(o3d)
    S, Tc = _clouds(o3d, src, d, dirs, tgt, nrm)
    bare = o3d.t.geometry.PointCloud(src)
    with pytest.raises(RuntimeError, match="DopplerICP requires target pointcloud to have normals."):
        reg.icp(S, o3d.t.geometry.PointCloud(tgt), 0.05, np.eye(4), est)
    bare.point["directions"] = S.point["directions"]
    with pytest.raises(RuntimeError, match="DopplerICP requires source pointcloud to have Doppler velocities."):
        reg.icp(bare, Tc, 0.05, np.eye(4), est)
    bare = o3d.t.geometry.PointCloud(src)
    bare.point["dopplers"] = S.point["dopplers"]
    with pytest.raises(RuntimeError, match="DopplerICP requires source pointcloud to have pre-computed direction"):
        reg.icp(bare, Tc, 0.05, np.eye(4), est)
    with pytest.raises(RuntimeError, match="Source pointcloud missing directions attribute."):
        est.compute_transformation(bare, Tc, torch.arange(len(src)))
    f64 = o3d.t.geometry.PointCloud(src)
    f64.point["dopplers"] = S.point["dopplers"].double()
    f64.point["directions"] = S.point["directions"]
    with pytest.raises(RuntimeError, match="Float64"):
        reg.icp(f64, Tc, 0.05, np.eye(4), est)
    wrong = o3d.t.geometry.PointCloud(src)
    wrong.point["dopplers"] = S.point["dopplers"].reshape(-1, 1).repeat(1, 2)
    wrong.point["directions"] = S.point["directions"]
    with pytest.raises(RuntimeError, match="dopplers must have shape"):
        reg.icp(wrong, Tc, 0.05, np.eye(4), est)
    col = o3d.t.geometry.PointCloud(src)   # [N, 1] is accepted
    col.point["dopplers"] = S.point["dopplers"].reshape(-1, 1)
    col.point["directions"] = S.point["directions"]
    a = reg.icp(col, Tc, 0.05, np.eye(4), est, reg.ICPConvergenceCriteria(0, 0, 3))
    b = reg.icp(S, Tc, 0.05, np.eye(4), est, reg.ICPConvergenceCriteria(0, 0, 3))
    assert a.transformation.tobytes() == b.transformation.tobytes()
    with pytest.raises(RuntimeError, match="TransformationEstimationForDopplerICP does not run multi-GPU"):
        reg.icp(S, Tc, 0.05, np.eye(4), est, comm=object())
    with pytest.raises(RuntimeError, match="Time period too small."):
        _est(o3d, period=1e-4)
    est.period = 1e-4   # a field set after construction is checked where the C ABI receives it
    with pytest.raises(RuntimeError, match="Time period too small."):
        reg.icp(S, Tc, 0.05, np.eye(4), est)
    with pytest.raises(RuntimeError, match="Unsupported method."):
        reg.icp(S, Tc, 0.05, np.eye(4), _est(o3d, doppler_kernel=(2, 0.5, 1.0)))


def test_corridor_translation_only_doppler_sees(o3d):
    """Point-to-plane ICP cannot see the motion along the corridor: no normal has an x component, so its 6x6 system is
    singular and it raises, as upstream does.  Doppler ICP recovers the motion, and with dynamic-outlier rejection it
    stays closer still despite 15 % dynamic points."""
    reg = o3d.t.pipelines.registration
    src, d, dirs, tgt, nrm, T_gt, _ = make_corridor(200000, seed=3, dynamic=0.15)
    S, Tc = _clouds(o3d, src, d, dirs, tgt, nrm)
    crit = reg.ICPConvergenceCriteria(0, 0, 20)
    with pytest.raises(RuntimeError, match="Singular 6x6 linear system"):
        reg.icp(S, Tc, 0.5, np.eye(4), reg.TransformationEstimationPointToPlane(), crit)
    errs = []
    for reject in (False, True):
        est = _est(o3d, transform_vehicle_to_sensor=CALIB, reject_dynamic_outliers=reject)
        res = reg.icp(S, Tc, 0.5, np.eye(4), est, crit)
        errs.append(np.abs(res.transformation[:3, 3] - T_gt[:3, 3]).max())
    assert errs[0] < 3e-3 and errs[1] < 2e-4 and errs[1] < errs[0], errs
