"""The point-to-point CPU oracle (oracle/p2p) against the reference's own known answers and against numpy.

The fixture and the two expected values are the reference's (cpp/tests/t/pipelines/registration/
TransformationEstimation.cpp, parsed into tests/golden/reference_kats.json).  Runs without a GPU."""
import numpy as np
import pytest

from oracle import p2p


def _fixture(kats, dtype):
    k = kats["transformation_estimation"]
    return (np.array(k["source_points"], dtype), np.array(k["target_points"], dtype),
            np.array(k["correspondences"], np.int64), k["expected"])


def numpy_kabsch(src, tgt, corr):
    """ComputeRtPointToPointCPU with numpy.linalg.svd, all in f64 -> 4x4."""
    v = corr != -1
    s, t = np.asarray(src, np.float64)[v], np.asarray(tgt, np.float64)[corr[v]]
    ms, mt = s.mean(0), t.mean(0)
    H = (t - mt).T @ (s - ms) / len(s)
    U, _, Vt = np.linalg.svd(H)
    S = np.diag([1.0, 1.0, np.sign(np.linalg.det(U) * np.linalg.det(Vt))])
    T = np.eye(4)
    T[:3, :3] = U @ S @ Vt
    T[:3, 3] = mt - T[:3, :3] @ ms
    return T


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_p2p_rmse_kat(kats, dtype):
    src, tgt, corr, exp = _fixture(kats, dtype)
    e = exp["p2p_rmse"]
    assert abs(p2p.rmse(src, tgt, corr, dtype) - e["value"]) < e["tol"]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_p2p_compute_transformation_kat(kats, dtype):
    src, tgt, corr, exp = _fixture(kats, dtype)
    T = p2p.compute_transformation(src, tgt, corr, dtype)
    moved = (src.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(dtype)
    e = exp["p2p_rmse_after"]
    assert abs(p2p.rmse(moved, tgt, corr, dtype) - e["value"]) < e["tol"]
    np.testing.assert_allclose(T, numpy_kabsch(src, tgt, corr), atol=1e-5 if dtype == np.float32 else 1e-12)


def test_sxy_layout_and_holes_against_numpy():
    rng = np.random.default_rng(3)
    src, tgt = rng.normal(size=(500, 3)), rng.normal(size=(300, 3))
    corr = rng.integers(0, 300, 500)
    corr[rng.random(500) < 0.3] = -1
    S, mt, ms, count = p2p.sxy(src, tgt, corr, np.float64)
    v = corr != -1
    s, t = src[v], tgt[corr[v]]
    assert count == v.sum()
    np.testing.assert_allclose(ms, s.mean(0), atol=1e-13)
    np.testing.assert_allclose(mt, t.mean(0), atol=1e-13)
    np.testing.assert_allclose(S, (t - t.mean(0)).T @ (s - s.mean(0)) / count, atol=1e-13)   # target rows
    assert p2p.sxy(src, tgt, np.full(500, -1), np.float64)[3] == 0
    with pytest.raises(RuntimeError, match="No valid correspondence"):
        p2p.compute_transformation(src, tgt, np.full(500, -1))


def test_kabsch_against_numpy_on_planar_and_reflected_sets():
    rng = np.random.default_rng(4)
    for case in ("full", "planar", "reflected"):
        src = rng.normal(size=(200, 3))
        if case == "planar":
            src[:, 2] = 0.0
        R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        if (np.linalg.det(R) < 0) != (case == "reflected"):
            R[:, 0] = -R[:, 0]
        tgt = src @ R.T + [0.3, -0.2, 0.1] + (1e-3 * rng.normal(size=src.shape) if case != "planar" else 0.0)
        corr = np.arange(200)
        T = p2p.compute_transformation(src, tgt, corr, np.float64)
        np.testing.assert_allclose(T, numpy_kabsch(src, tgt, corr), atol=1e-10, err_msg=case)
        assert abs(np.linalg.det(T[:3, :3]) - 1.0) < 1e-12


def test_icp_loop_recovers_the_synthetic_motion():
    from tests.synth import make_icp_pair
    src, tgt, _, T_gt = make_icp_pair(20000, seed=1)
    # (point-to-point slides along the surfaces more slowly than point-to-plane: 60 iterations, not 30)
    res = p2p.icp(src, tgt, 0.05, max_iteration=60, relative_fitness=0, relative_rmse=0)
    assert res.status == 0 and res.num_iterations == 60 and len(res.per_iteration) == 60
    assert res.per_iteration[-1, 1] < res.per_iteration[0, 1]
    np.testing.assert_allclose(res.transformation, T_gt, atol=2e-3)
    res32 = p2p.icp(src, tgt, 0.05, max_iteration=60, relative_fitness=0, relative_rmse=0, accumulate_f64=False)
    np.testing.assert_allclose(res32.transformation, res.transformation, atol=1e-4)
    conv = p2p.icp(src, tgt, 0.05, max_iteration=50, relative_fitness=1e-3, relative_rmse=1e-3)
    assert conv.converged and conv.num_iterations < 49
    none = p2p.icp(src + 100.0, tgt, 0.05, max_iteration=5)
    assert none.fitness == 0.0 and not none.converged and np.array_equal(none.transformation, np.eye(4))
