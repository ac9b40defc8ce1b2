"""Symmetric ICP on the GPU (TransformationEstimationSymmetric): the reference's known answers through the public
classes, the stand-alone reduction against the CPU oracle (oracle/symmetric), the fused loop and a 3-scale pyramid
against the oracle loop, and the public surface."""
import numpy as np
import pytest
import torch

from oracle import symmetric as sym
from tests.synth import make_icp_pair
from tests.test_oracle_symmetric import _kat_clouds, expected_motion, load_symmetric_kats, transform_f32, unit

pytestmark = pytest.mark.gpu

ROBUST = [(0, 1.0, 1.0), (1, 1.0, 1.0), (2, 0.02, 1.0), (3, 0.02, 1.0), (4, 0.02, 1.0), (5, 0.05, 1.0),
          (6, 0.02, 0.5)]


@pytest.fixture(scope="module")
def skats():
    return load_symmetric_kats()


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


def _cloud(o3d, p, n):
    return o3d.t.geometry.PointCloud(np.asarray(p, np.float32)).set_point_normals(np.asarray(n, np.float32))


def _est(o3d, kernel=None):
    reg = o3d.t.pipelines.registration
    if kernel is None:
        return reg.TransformationEstimationSymmetric()
    return reg.TransformationEstimationSymmetric(reg.RobustKernel(reg.RobustKernelMethod(kernel[0]), kernel[1], kernel[2]))


def test_reference_kats_through_the_public_classes(skats, o3d):
    """cpp/tests/t/pipelines/registration/TransformationEstimation.cpp:180-412."""
    est = _est(o3d)
    k = skats["rmse"]
    s, ns = [k["source_point"]], [k["source_normal"]]
    t, nt = [k["target_point"]], [k["target_normal"]]
    c = torch.zeros(1, dtype=torch.int64)
    got = [est.compute_rmse(_cloud(o3d, s, ns), _cloud(o3d, t, nt), c),
           est.compute_rmse(_cloud(o3d, s, ns), _cloud(o3d, t, -np.array(nt)), c),
           est.compute_rmse(_cloud(o3d, s, ns), _cloud(o3d, [[0, 0, 0]], ns), c),
           est.compute_rmse(_cloud(o3d, s, ns), _cloud(o3d, [[0, 0, 0]], -np.array(ns)), c)]
    np.testing.assert_allclose(got, k["expected"], atol=k["tol_f32"])

    k = skats["transformation"]
    src, sn, tgt, tn, T = _kat_clouds(k)
    corr = torch.arange(len(src))
    S, Tc = _cloud(o3d, src, sn), _cloud(o3d, tgt, tn)
    np.testing.assert_allclose(est.compute_transformation(S, Tc, corr), T, atol=k["tol_f32"])
    alt = _cloud(o3d, tgt, tn * np.array(k["alternating_signs"], np.float32)[:, None])
    np.testing.assert_allclose(est.compute_transformation(S, alt, corr), T, atol=k["tol_f32"])
    assert np.array_equal(est.compute_transformation(S, Tc, torch.full((len(src),), -1)), np.eye(4))
    for bad in (-2, len(tgt)):
        c = corr.clone()
        c[0] = bad
        for fn in (est.compute_rmse, est.compute_transformation):
            with pytest.raises(RuntimeError, match="SymmetricICP correspondences must be -1 or a target point index"):
                fn(S, Tc, c)
    bad_shape = o3d.t.geometry.PointCloud(src)
    bad_shape.point["normals"] = torch.zeros((len(src), 1), device="cuda")
    with pytest.raises(RuntimeError, match="Source normals shape"):
        est.compute_transformation(bad_shape, Tc, corr)
    with pytest.raises(RuntimeError, match="requires both source and target to have normals"):
        est.compute_rmse(o3d.t.geometry.PointCloud(src), Tc, corr)

    rs = np.array(k["robust_source_points"], np.float32)
    rn = unit(k["robust_source_normals"])
    M = expected_motion(k)
    rt = (transform_f32(M, rs) + np.array(k["robust_noise"], np.float32)).astype(np.float32)
    rk = k["robust_kernel"]
    cauchy = _est(o3d, (sym.ROBUST[rk["method"]], rk["scaling_parameter"], rk["shape_parameter"]))
    got = cauchy.compute_transformation(_cloud(o3d, rs, rn), _cloud(o3d, rt, transform_f32(M, rn, normals=True)),
                                        torch.arange(len(rs)))
    np.testing.assert_allclose(got, np.array(k["robust_expected"]), atol=k["tol_f32"])


def _moved_pair(n, seed, offset=0.0, holes=0.15, noise=0.002):
    rng = np.random.default_rng(seed)
    src = rng.uniform(-1, 1, (n, 3)) + offset
    sn = unit(rng.normal(size=(n, 3)))
    M = np.eye(4)
    M[:3, :3] = expected_motion({"angle": 0.05, "axis": [1, 2, -1], "translation": [0, 0, 0]})[:3, :3]
    M[:3, 3] = [0.02, -0.01, 0.015]
    c = src.mean(0)
    tgt = (src - c) @ M[:3, :3].T + c + M[:3, 3] + rng.normal(0, noise, (n, 3))
    tn = unit(sn @ M[:3, :3].T)
    flip = rng.random(n) < 0.5
    tn[flip] = -tn[flip]
    perm = rng.permutation(n)
    corr = np.argsort(perm).astype(np.int64)
    corr[rng.random(n) < holes] = -1
    return src.astype(np.float32), sn, tgt[perm].astype(np.float32), tn[perm], corr


@pytest.mark.parametrize("kernel", ROBUST)
def test_reduction_vs_oracle(o3d, kernel):
    src, sn, tgt, tn, corr = _moved_pair(200000, seed=kernel[0])
    est = _est(o3d, kernel)
    S, Tc = _cloud(o3d, src, sn), _cloud(o3d, tgt, tn)
    got = est.compute_transformation(S, Tc, torch.from_numpy(corr))
    want = sym.compute_transformation(src, tgt, sn, tn, corr, kernel, accumulate_f64=True)
    np.testing.assert_allclose(got, want, atol=2e-6)
    ms, mt, _ = sym.means(src, tgt, corr)
    pose, residual, count, sums = est.compute_pose(S, Tc, torch.from_numpy(corr), ms, mt)
    ref = sym.sums(src, tgt, sn, tn, corr, ms, mt, kernel, accumulate_f64=True)
    assert count == int(ref[28]) == int((corr >= 0).sum())
    np.testing.assert_allclose(sums.cpu().numpy(), ref, rtol=2e-5, atol=1e-6 * np.abs(ref).max())


def test_reduction_far_from_the_origin_and_without_correspondences(o3d):
    """1 km from the origin the coordinates keep 6e-5 m of f32 resolution; the means reach the kernel in f32 as they do
    upstream, so device and oracle share them and differ by summation order only."""
    src, sn, tgt, tn, corr = _moved_pair(100000, seed=11, offset=1000.0)
    est = _est(o3d)
    S, Tc = _cloud(o3d, src, sn), _cloud(o3d, tgt, tn)
    got = est.compute_transformation(S, Tc, torch.from_numpy(corr))
    want = sym.compute_transformation(src, tgt, sn, tn, corr, accumulate_f64=True)
    np.testing.assert_allclose(got[:3, :3], want[:3, :3], atol=1e-6)
    np.testing.assert_allclose(got[:3, 3], want[:3, 3], atol=2e-3)   # 1e-6 of rotation x 1 km
    assert np.array_equal(est.compute_transformation(S, Tc, torch.full((len(src),), -1)), np.eye(4))


def _pair_with_normals(o3d, n, seed):
    """make_icp_pair, with the source's normals estimated on the device (hybrid search, radius 0.06, 30 neighbours)."""
    src, tgt, tn, T_gt = make_icp_pair(n, seed=seed)
    S = o3d.t.geometry.PointCloud(src)
    S.estimate_normals(30, 0.06)
    sn = S.point["normals"].cpu().numpy()
    return src, sn, tgt, tn, T_gt


def _icp(o3d, src, sn, tgt, tn, r, init=None, crit=None, cb=None, est=None):
    reg = o3d.t.pipelines.registration
    return reg.icp(_cloud(o3d, src, sn), _cloud(o3d, tgt, tn), r, np.eye(4) if init is None else init,
                   est or _est(o3d), crit or reg.ICPConvergenceCriteria(), -1.0, cb)


@pytest.mark.parametrize("n,iters", [(30000, 1), (30000, 30), (250000, 10)])
def test_fused_loop_vs_oracle(o3d, n, iters):
    """30 iterations on 30k points: the first iterations search, the aligned later ones replay cached sums."""
    reg = o3d.t.pipelines.registration
    src, sn, tgt, tn, T_gt = _pair_with_normals(o3d, n, seed=1)
    log = []
    res = _icp(o3d, src, sn, tgt, tn, 0.05, crit=reg.ICPConvergenceCriteria(0, 0, iters), cb=log.append)
    ref = sym.icp(src, sn, tgt, tn, 0.05, max_iteration=iters, relative_fitness=0, relative_rmse=0)
    assert ref.status == 0 and res.num_iterations == ref.num_iterations == iters
    per = np.array([[c["fitness"], c["inlier_rmse"]] for c in log])
    assert per[0, 0] == ref.per_iteration[0, 0]
    assert abs(per[0, 1] - ref.per_iteration[0, 1]) < 3e-7 * ref.per_iteration[0, 1]
    np.testing.assert_allclose(per[:, 0], ref.per_iteration[:, 0], atol=2e-4)
    np.testing.assert_allclose(per[:, 1], ref.per_iteration[:, 1], atol=2e-6)
    np.testing.assert_allclose(res.transformation, ref.transformation, atol=2e-5)
    assert abs(res.fitness - ref.fitness) < 2e-4 and abs(res.inlier_rmse - ref.inlier_rmse) < 2e-6
    corr = res.correspondence_set.cpu().numpy()
    assert (corr == ref.correspondences).mean() > 0.999
    if iters == 30:
        np.testing.assert_allclose(res.transformation, T_gt, atol=2e-3)


def test_robust_fused_loop_vs_oracle(o3d):
    reg = o3d.t.pipelines.registration
    src, sn, tgt, tn, _ = _pair_with_normals(o3d, 40000, seed=5)
    kernel = (3, 0.01, 1.0)
    res = _icp(o3d, src, sn, tgt, tn, 0.05, crit=reg.ICPConvergenceCriteria(0, 0, 8), est=_est(o3d, kernel))
    ref = sym.icp(src, sn, tgt, tn, 0.05, max_iteration=8, relative_fitness=0, relative_rmse=0, kernel=kernel)
    np.testing.assert_allclose(res.transformation, ref.transformation, atol=2e-5)


def test_multi_scale_with_voxel_pyramid_vs_oracle(o3d):
    import oracle
    reg = o3d.t.pipelines.registration
    src, sn, tgt, tn, _ = _pair_with_normals(o3d, 90000, seed=16)
    voxels, radii, iters = [0.08, 0.04, 0.02], [0.16, 0.08, 0.05], [5, 6, 8]
    res = reg.multi_scale_icp(_cloud(o3d, src, sn), _cloud(o3d, tgt, tn), voxels,
                              [reg.ICPConvergenceCriteria(0, 0, k) for k in iters], radii, np.eye(4), _est(o3d))
    levels = [(oracle.voxel_down_sample(src, voxels[2], sn), oracle.voxel_down_sample(tgt, voxels[2], tn))]
    for v in (voxels[1], voxels[0]):
        levels.insert(0, tuple(oracle.voxel_down_sample(c["positions"], v, c["normals"]) for c in levels[0]))
    T = np.eye(4)
    for (ss, tt), r, k in zip(levels, radii, iters):
        ref = sym.icp(ss["positions"], ss["normals"], tt["positions"], tt["normals"], r, init=T, max_iteration=k,
                      relative_fitness=0, relative_rmse=0)
        T = ref.transformation
    assert res.num_iterations == sum(iters)
    np.testing.assert_allclose(res.transformation, T, atol=5e-5)
    assert abs(res.fitness - ref.fitness) < 1e-3 and abs(res.inlier_rmse - ref.inlier_rmse) < 1e-5


def test_entry_points_agree_and_runs_are_bit_identical(o3d):
    reg = o3d.t.pipelines.registration
    src, sn, tgt, tn, _ = _pair_with_normals(o3d, 100000, seed=7)
    crit = reg.ICPConvergenceCriteria(0, 0, 12)
    runs = []
    for _ in range(2):
        log = []
        r = _icp(o3d, src, sn, tgt, tn, 0.05, crit=crit, cb=log.append)
        runs.append((r.transformation.tobytes(), r.fitness, r.inlier_rmse, r.correspondence_set.cpu().numpy().tobytes(),
                     [(c["fitness"], c["inlier_rmse"]) for c in log]))
    assert runs[0] == runs[1]
    r2 = reg.registration_symmetric_icp(_cloud(o3d, src, sn), _cloud(o3d, tgt, tn), 0.05, np.eye(4), criteria=crit)
    assert r2.transformation.tobytes() == runs[0][0] and r2.fitness == runs[0][1]


def test_misuse_raises(o3d):
    reg = o3d.t.pipelines.registration
    src, sn, tgt, tn, _ = _pair_with_normals(o3d, 5000, seed=2)
    with pytest.raises(RuntimeError, match="requires both source and target to have normals"):
        reg.icp(o3d.t.geometry.PointCloud(src), _cloud(o3d, tgt, tn), 0.05, np.eye(4), _est(o3d))
    with pytest.raises(RuntimeError, match="multi-GPU"):
        reg.icp(_cloud(o3d, src, sn), _cloud(o3d, tgt, tn), 0.05, np.eye(4), _est(o3d), comm=object())
