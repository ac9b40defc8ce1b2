"""Point-to-point ICP on the GPU (TransformationEstimationPointToPoint, the reference's default estimator): the
stand-alone Kabsch reduction against f64 numpy, the fused loop against the CPU oracle loop (oracle/p2p), and the
public surface on clouds without normals."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle
from oracle import p2p
from tests.synth import make_icp_pair

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


def numpy_kabsch(src, tgt, corr):
    """ComputeRtPointToPointCPU (RegistrationCPU.cpp:619-653) with numpy.linalg.svd, all in f64 -> R, t."""
    v = corr != -1
    s, t = np.asarray(src, np.float64)[v], np.asarray(tgt, np.float64)[corr[v]]
    ms, mt = s.mean(0), t.mean(0)
    H = (t - mt).T @ (s - ms) / len(s)
    U, _, Vt = np.linalg.svd(H)
    R = U @ np.diag([1.0, 1.0, np.sign(np.linalg.det(U) * np.linalg.det(Vt))]) @ Vt
    return R, mt - R @ ms


def _rt(o3d, src, tgt, corr):
    reg = o3d.t.pipelines.registration
    return reg.TransformationEstimationPointToPoint().compute_rt(
        o3d.t.geometry.PointCloud(np.asarray(src, np.float32)), o3d.t.geometry.PointCloud(np.asarray(tgt, np.float32)), corr)


def _rotation(rng, reflect=False):
    R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    if (np.linalg.det(R) < 0) != reflect:
        R[:, 0] = -R[:, 0]
    return R


def _eighths(a):
    """Coordinates on the lattice of eighths within +-8: differences and their pairwise products are exact in f32, and
    so are sums of 32 of them, so the device's f64 totals are the exact moments and only the Kabsch step is tested."""
    return (np.clip(np.round(np.asarray(a) * 8.0), -64, 64) / 8.0).astype(np.float32)


def test_reference_kat_through_the_public_classes(kats, o3d):
    """cpp/tests/t/pipelines/registration/TransformationEstimation.cpp:103, 130."""
    k = kats["transformation_estimation"]
    reg = o3d.t.pipelines.registration
    src = o3d.t.geometry.PointCloud(np.array(k["source_points"], np.float32))
    tgt = o3d.t.geometry.PointCloud(np.array(k["target_points"], np.float32))   # no normals
    corr = np.array(k["correspondences"], np.int64)
    est = reg.TransformationEstimationPointToPoint()
    e = k["expected"]["p2p_rmse"]
    assert abs(est.compute_rmse(src, tgt, corr) - e["value"]) < e["tol"]
    T = est.compute_transformation(src, tgt, corr)
    assert T.shape == (4, 4) and T.dtype == np.float64
    e = k["expected"]["p2p_rmse_after"]
    assert abs(est.compute_rmse(src.clone().transform(T), tgt, corr) - e["value"]) < e["tol"]
    np.testing.assert_allclose(T, p2p.compute_transformation(k["source_points"], k["target_points"], corr, np.float64),
                               atol=1e-6)


@pytest.mark.parametrize("case", ["holes", "planar", "reflection"])
def test_compute_rt_equals_numpy_kabsch_on_exact_moments(o3d, case):
    rng = np.random.default_rng({"holes": 1, "planar": 2, "reflection": 3}[case])
    n, m = 4000, 3000
    tgt = rng.uniform(-5, 5, size=(m, 3))
    if case == "planar":
        tgt[:, 2] = 1.5                                   # Sxy has an exactly zero row: rank 2
    tgt = _eighths(tgt)
    corr = rng.integers(0, m, n).astype(np.int64)
    R0 = _rotation(rng, reflect=case == "reflection")     # reflection: det(Sxy) < 0, the unconstrained optimum is R0
    src = _eighths((tgt[corr].astype(np.float64) - [0.5, -0.25, 0.125]) @ R0 + 0.2 * rng.normal(size=(n, 3)))
    if case == "holes":
        corr[rng.random(n) < 0.4] = -1
    R, t, count = _rt(o3d, src, tgt, corr)
    Rn, tn = numpy_kabsch(src, tgt, corr)
    if case == "reflection":
        v = corr != -1
        H = (tgt[corr[v]] - tgt[corr[v]].mean(0)).astype(np.float64).T @ (src[v] - src[v].mean(0)).astype(np.float64)
        assert np.linalg.det(H) < 0
    assert count == (corr != -1).sum()
    assert abs(np.linalg.det(R) - 1.0) < 1e-13
    np.testing.assert_allclose(R @ R.T, np.eye(3), atol=1e-14)
    np.testing.assert_allclose(R, Rn, atol=1e-12)
    np.testing.assert_allclose(t, tn, atol=1e-11)


def test_compute_rt_far_from_the_origin(o3d):
    """A 1 m cloud 1 km away: raw f32 products would carry ~0.06 of rounding each; about the pivot they are of the
    cloud's own size."""
    rng = np.random.default_rng(4)
    n = 20000
    centre = np.array([1000.0, -500.0, 250.0])
    tgt = (centre + rng.uniform(-0.5, 0.5, size=(n, 3))).astype(np.float32)
    a = np.deg2rad(2.0)
    R0 = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1.0]])
    src = ((tgt.astype(np.float64) - centre) @ R0 + centre + [0.01, 0.02, -0.01] + 1e-3 * rng.normal(size=(n, 3))).astype(np.float32)
    corr = np.arange(n, dtype=np.int64)
    R, t, count = _rt(o3d, src, tgt, corr)
    Rn, tn = numpy_kabsch(src, tgt, corr)
    assert count == n
    np.testing.assert_allclose(R, Rn, atol=1e-6)
    s64 = src.astype(np.float64)
    np.testing.assert_allclose(s64 @ R.T + t, s64 @ Rn.T + tn, atol=2e-6)


def test_compute_rt_degenerate_inputs(o3d):
    rng = np.random.default_rng(5)
    src, tgt = rng.normal(size=(100, 3)).astype(np.float32), rng.normal(size=(50, 3)).astype(np.float32)
    with pytest.raises(RuntimeError, match="No valid correspondence present."):
        _rt(o3d, src, tgt, np.full(100, -1, np.int64))
    # all matches on one line: no unique rotation, but a proper, finite one
    line = (np.linspace(-1, 1, 100)[:, None] * np.array([[1.0, 2.0, -1.0]])).astype(np.float32)
    for s, t in ((line, line[::-1].copy()), (line, np.repeat(line[:1], 100, 0))):
        R, tr, _ = _rt(o3d, s, t, np.arange(100, dtype=np.int64))
        assert np.isfinite(R).all() and np.isfinite(tr).all() and abs(np.linalg.det(R) - 1.0) < 1e-12
        np.testing.assert_allclose(R @ R.T, np.eye(3), atol=1e-13)


def _icp(o3d, src, tgt, r, init=None, crit=None, cb=None, est="default"):
    reg = o3d.t.pipelines.registration
    s, t = o3d.t.geometry.PointCloud(src), o3d.t.geometry.PointCloud(tgt)     # positions only
    return reg.icp(s, t, r, np.eye(4) if init is None else init, None if est == "default" else est,
                   crit or reg.ICPConvergenceCriteria(), -1.0, cb)


@pytest.mark.parametrize("n,iters", [(30000, 1), (30000, 30), (250000, 10)])
def test_fused_loop_vs_oracle(o3d, n, iters):
    reg = o3d.t.pipelines.registration
    src, tgt, _, _ = make_icp_pair(n, seed=1)
    log = []
    res = _icp(o3d, src, tgt, 0.05, crit=reg.ICPConvergenceCriteria(0, 0, iters), cb=log.append)
    ref = p2p.icp(src, tgt, 0.05, max_iteration=iters, relative_fitness=0, relative_rmse=0)
    assert ref.status == 0 and res.num_iterations == ref.num_iterations == iters and res.converged == ref.converged
    per = np.array([[c["fitness"], c["inlier_rmse"]] for c in log])
    assert per.shape == (iters, 2)
    # iteration 0 sees bit-identical inputs: the same matches, so the same fitness; rmse to summation order
    assert per[0, 0] == ref.per_iteration[0, 0]
    assert abs(per[0, 1] - ref.per_iteration[0, 1]) < 3e-7 * ref.per_iteration[0, 1]
    # later iterations see a working source that differs by the rounding of the update
    np.testing.assert_allclose(per[:, 0], ref.per_iteration[:, 0], atol=2e-4)
    np.testing.assert_allclose(per[:, 1], ref.per_iteration[:, 1], atol=2e-6)
    np.testing.assert_allclose(res.transformation, ref.transformation, atol=2e-5)
    assert abs(res.fitness - ref.fitness) < 2e-4 and abs(res.inlier_rmse - ref.inlier_rmse) < 2e-6
    corr = res.correspondence_set.cpu().numpy()
    assert corr.shape == (len(src),) and corr.dtype == np.int64
    assert (corr == ref.correspondences).mean() > 0.999


def test_one_iteration_update_is_tight_and_final_correspondences_are_exact(o3d):
    """One update from bit-identical inputs agrees to summation accuracy; the final evaluation's correspondences are
    those of a brute-force search on the source moved by the returned transformation's f32 image."""
    reg = o3d.t.pipelines.registration
    src, tgt, _, _ = make_icp_pair(20000, seed=9)
    res = _icp(o3d, src, tgt, 0.05, crit=reg.ICPConvergenceCriteria(0, 0, 1))
    ref = p2p.icp(src, tgt, 0.05, max_iteration=1, relative_fitness=0, relative_rmse=0)
    np.testing.assert_allclose(res.transformation, ref.transformation, atol=1e-7)
    ev = reg.evaluate_registration(o3d.t.geometry.PointCloud(src), o3d.t.geometry.PointCloud(tgt), 0.05, np.eye(4))
    idx, _, cnt = oracle.hybrid_search(tgt, src, 0.05, 1, bruteforce=True)
    want = np.where(cnt.reshape(-1) > 0, idx.reshape(-1), -1)
    assert np.array_equal(ev.correspondence_set.cpu().numpy(), want)
    assert ev.fitness == (want >= 0).mean()


def test_init_convergence_and_no_correspondences(o3d):
    reg = o3d.t.pipelines.registration
    src, tgt, _, T_gt = make_icp_pair(40000, seed=10)
    init = T_gt.copy()
    init[:3, 3] += [0.004, -0.003, 0.002]
    crit = reg.ICPConvergenceCriteria(1e-5, 1e-5, 60)
    res = _icp(o3d, src, tgt, 0.05, init=init, crit=crit, est=reg.TransformationEstimationPointToPoint())
    ref = p2p.icp(src, tgt, 0.05, init=init, max_iteration=60, relative_fitness=1e-5, relative_rmse=1e-5)
    assert res.converged and ref.converged and 0 < ref.num_iterations < 59
    assert abs(res.num_iterations - ref.num_iterations) <= 1     # (a change of rmse right at the threshold)
    np.testing.assert_allclose(res.transformation, ref.transformation, atol=5e-5 if res.num_iterations == ref.num_iterations else 3e-4)
    np.testing.assert_allclose(res.transformation, T_gt, atol=2e-3)
    far = _icp(o3d, src + 100.0, tgt, 0.05)
    assert far.fitness == 0.0 and far.inlier_rmse == 0.0 and not far.converged and far.num_iterations == 0
    assert np.array_equal(far.transformation, np.eye(4))
    assert (far.correspondence_set.cpu().numpy() == -1).all()


def test_default_estimator_on_clouds_without_normals_recovers_the_motion(o3d):
    reg = o3d.t.pipelines.registration
    src, tgt, _, T_gt = make_icp_pair(60000, seed=3)
    # (point-to-point slides along the surfaces more slowly than point-to-plane)
    res = _icp(o3d, src, tgt, 0.05, crit=reg.ICPConvergenceCriteria(0, 0, 80))
    assert res.fitness > 0.99
    np.testing.assert_allclose(res.transformation, T_gt, atol=3e-3)
    with pytest.raises(RuntimeError, match="require pre-computed normal vectors"):
        _icp(o3d, src, tgt, 0.05, est=reg.TransformationEstimationPointToPlane())


def test_multi_scale_with_voxel_pyramid_vs_oracle(o3d):
    reg = o3d.t.pipelines.registration
    src, tgt, _, _ = make_icp_pair(90000, seed=16)
    voxels, radii, iters = [0.08, 0.04, 0.02], [0.16, 0.08, 0.05], [5, 6, 8]
    res = reg.multi_scale_icp(o3d.t.geometry.PointCloud(src), o3d.t.geometry.PointCloud(tgt), voxels,
                              [reg.ICPConvergenceCriteria(0, 0, k) for k in iters], radii)
    levels = [(oracle.voxel_down_sample(src, voxels[2]), oracle.voxel_down_sample(tgt, voxels[2]))]
    for v in (voxels[1], voxels[0]):   # coarser levels from the finer ones
        levels.insert(0, tuple(oracle.voxel_down_sample(c["positions"], v) for c in levels[0]))
    T = np.eye(4)
    for (ss, tt), r, k in zip(levels, radii, iters):
        ref = p2p.icp(ss["positions"], tt["positions"], r, init=T, max_iteration=k, relative_fitness=0, relative_rmse=0)
        T = ref.transformation
    assert res.num_iterations == sum(iters)
    np.testing.assert_allclose(res.transformation, T, atol=5e-5)
    assert abs(res.fitness - ref.fitness) < 1e-3 and abs(res.inlier_rmse - ref.inlier_rmse) < 1e-5


def test_two_runs_are_bit_identical(o3d):
    reg = o3d.t.pipelines.registration
    src, tgt, _, _ = make_icp_pair(100000, seed=7)
    runs = []
    for _ in range(2):
        log = []
        r = _icp(o3d, src, tgt, 0.05, crit=reg.ICPConvergenceCriteria(0, 0, 12), cb=log.append)
        runs.append((r.transformation.tobytes(), r.fitness, r.inlier_rmse, r.correspondence_set.cpu().numpy().tobytes(),
                     [(c["fitness"], c["inlier_rmse"]) for c in log]))
    assert runs[0] == runs[1]


def test_evaluate_registration_without_normals_equals_the_point_to_plane_handle(o3d):
    reg = o3d.t.pipelines.registration
    src, tgt, nrm, T_gt = make_icp_pair(50000, seed=11)
    T = T_gt.copy()
    T[:3, 3] += 0.01
    s = o3d.t.geometry.PointCloud(src)
    ev = reg.evaluate_registration(s, o3d.t.geometry.PointCloud(tgt), 0.015, T)
    plane = reg.icp(s, o3d.t.geometry.PointCloud(tgt).set_point_normals(nrm), 0.015, T,
                    reg.TransformationEstimationPointToPlane(), reg.ICPConvergenceCriteria(0, 0, 0))
    assert 0 < ev.fitness < 1
    assert ev.fitness == plane.fitness and ev.inlier_rmse == plane.inlier_rmse
    assert torch.equal(ev.correspondence_set, plane.correspondence_set)
    assert np.array_equal(ev.transformation, T) and ev.num_iterations == 0


def test_one_shot_and_handle_entry_points_agree(o3d):
    """o3db_icp_point_to_point == create_point_to_point + iterate + finish, and reset restores the start."""
    import ctypes as C
    from open3d_b200 import _lib as L
    src, tgt, _, _ = make_icp_pair(20000, seed=2)
    d = [torch.from_numpy(a).cuda() for a in (src, tgt)]
    stream = int(torch.cuda.current_stream().cuda_stream)
    opt = L.IcpOptions()
    opt.max_correspondence_distance, opt.max_iteration = 0.05, 6
    opt.relative_fitness = opt.relative_rmse = 0.0
    opt.kernel = L.RobustKernel(5, 0.01, 1.0)    # ignored: the estimator has no robust kernel
    T0 = np.eye(4)
    one = L.IcpResult()
    L.check(L.lib.o3db_icp_point_to_point(d[0].data_ptr(), len(src), d[1].data_ptr(), len(tgt), L.dptr(T0), C.byref(opt),
                                          C.byref(one), None, None, stream))
    h = C.c_void_p()
    L.check(L.lib.o3db_icp_create_point_to_point(d[0].data_ptr(), len(src), d[1].data_ptr(), len(tgt), L.dptr(T0),
                                                 C.byref(opt), None, stream, C.byref(h)))
    got = []
    for _ in range(2):
        L.check(L.lib.o3db_icp_iterate(h, 6, stream))
        r = L.IcpResult()
        L.check(L.lib.o3db_icp_finish(h, C.byref(r), None, None, stream))
        got.append((list(r.transformation), r.fitness, r.inlier_rmse, r.num_iterations))
        L.check(L.lib.o3db_icp_reset(h, stream))
    L.lib.o3db_icp_destroy(h)
    assert got[0] == got[1] == (list(one.transformation), one.fitness, one.inlier_rmse, 6)
    ref = p2p.icp(src, tgt, 0.05, max_iteration=6, relative_fitness=0, relative_rmse=0)
    np.testing.assert_allclose(np.array(one.transformation).reshape(4, 4), ref.transformation, atol=2e-5)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_sharded_point_to_point_equals_single_gpu_on_2_gpus():
    """tests/multigpu_p2p_check.py under torchrun, 2 ranks, both transports of the 30-double exchange."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tests", "multigpu_p2p_check.py")]
    for no_peer in (False, True):
        env = dict(os.environ)
        if no_peer:
            env["O3DB_COMM_NO_PEER"] = "1"
        out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900, env=env)
        assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
        assert "multigpu_p2p_check ok" in out.stdout
