"""Every search path of the fused ICP iteration returns the exhaustive-search winner: the certificate, the seeded box,
the seeded path's pass-1 box for a seed farther than r1, the slow path's two-pass box scan, its 9-slab scan and its
pruned row-by-row search.  The seeded paths also establish a clearance (a lower bound on the distance to every other
target point), which lets a query keep its winner by the certificate in the next iteration; a wrong clearance would show
up as a wrong winner.

The clouds have more than three chunk rows and a partial last row (see test_icp_sweep_gpu.py), and send queries down
the less common paths: a dense cluster (long slabs), a volumetric cube (pruned search), sources partly outside the
target's bounding box (no candidate), and grid cells finer than r / 2 (boxes of many rows).
"""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from tests.synth import make_colors, make_icp_pair

pytestmark = pytest.mark.gpu

THREADS = 768   # kIcpThreads: one block per SM
R = 0.05
SAMPLE = 4096   # queries checked against the brute-force search (all of them are checked against the grid oracle)
ANGLE = 0.35    # degrees: about 1.5 x make_icp_pair's default on these clouds, so the first update moves points by cm


def _cloud_points():
    row = torch.cuda.get_device_properties(0).multi_processor_count * THREADS
    return 3 * row + row // 3


def _cloud(kind, angle_deg=None):
    """(source, target, target normals) of one of the test clouds."""
    n = _cloud_points()
    if kind == "cube":
        rng = np.random.default_rng(31)
        tgt = rng.uniform(0, 1, (n, 3)).astype(np.float32)
        src = (rng.uniform(0, 1, (n, 3)) + [0.004, -0.003, 0.002]).astype(np.float32)
        nrm = rng.normal(size=(n, 3))
        nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(np.float32)
        return src, tgt, nrm
    src, tgt, nrm, _ = make_icp_pair(n, seed=7, angle_deg=angle_deg)
    if kind == "cluster":
        # 20 000 target points within ~1 cm of one surface point: slabs far longer than the flat scans take
        rng = np.random.default_rng(8)
        c = len(tgt) // 2 + 300
        blob = tgt[c] + rng.normal(0, 0.01, (20000, 3)).astype(np.float32)
        tgt = np.concatenate([tgt, blob]).astype(np.float32)
        nrm = np.concatenate([nrm, np.repeat(nrm[c:c + 1], len(blob), axis=0)]).astype(np.float32)
    elif kind == "outside":
        # the target keeps its lower half along x: about half of the source lies beyond its bounding box
        keep = tgt[:, 0] < np.median(tgt[:, 0])
        tgt, nrm = np.ascontiguousarray(tgt[keep]), np.ascontiguousarray(nrm[keep])
    return src, tgt, nrm


CLOUDS = [("standard", 0.0), ("cluster", 0.0), ("cube", 0.0), ("outside", 0.0), ("standard", 0.2), ("standard", 0.3)]


@pytest.fixture(scope="module")
def L():
    import open3d_b200  # noqa: F401
    from open3d_b200 import _lib
    assert torch.cuda.is_available()
    return _lib


def _options(L, iters, cell_scale=0.0, tukey=False):
    opt = L.IcpOptions()
    opt.max_correspondence_distance, opt.max_iteration = R, max(iters, 1)
    opt.relative_fitness = opt.relative_rmse = 0.0
    opt.kernel = L.RobustKernel(5, 0.05, 1.0) if tukey else L.RobustKernel(0, 1.0, 1.0)
    opt.cell_scale = cell_scale
    return opt


def _colors(src, tgt):
    rng = np.random.default_rng(3)
    return make_colors(src, 1), make_colors(tgt, 1), rng.normal(0, 0.05, tgt.shape).astype(np.float32)


def _run(L, src, tgt, nrm, batches, cell_scale=0.0, tukey=False, colored=False):
    """Create a handle (identity init), run o3db_icp_iterate once per entry of `batches`, then o3db_icp_finish.
    -> (T, fitness, rmse, iterations, correspondences, per-iteration log)"""
    stream = int(torch.cuda.current_stream().cuda_stream)
    iters = sum(batches)
    n = len(src)
    keep = [torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in (src, tgt, nrm)]
    opt = _options(L, iters, cell_scale, tukey)
    h = C.c_void_p()
    if colored:
        sc, tc, grad = [torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in _colors(src, tgt)]
        keep += [sc, tc, grad]
        L.check(L.lib.o3db_icp_create_colored(keep[0].data_ptr(), sc.data_ptr(), n, keep[1].data_ptr(),
                                              keep[2].data_ptr(), tc.data_ptr(), grad.data_ptr(), len(tgt),
                                              L.dptr(np.eye(4)), C.byref(opt), 0.968, None, stream, C.byref(h)))
    else:
        L.check(L.lib.o3db_icp_create(keep[0].data_ptr(), n, keep[1].data_ptr(), keep[2].data_ptr(), len(tgt),
                                      L.dptr(np.eye(4)), C.byref(opt), None, stream, C.byref(h)))
    try:
        L.check(L.lib.o3db_icp_reset(h, stream))
        for k in batches:
            L.check(L.lib.o3db_icp_iterate(h, k, stream))
        res = L.IcpResult()
        corr = torch.full((n,), -7, dtype=torch.int64, device="cuda")
        per = np.zeros((max(iters, 1), 2))
        L.check(L.lib.o3db_icp_finish(h, C.byref(res), corr.data_ptr(), L.dptr(per), stream))
        torch.cuda.synchronize()
    finally:
        L.lib.o3db_icp_destroy(h)
    return (np.array(res.transformation).reshape(4, 4), res.fitness, res.inlier_rmse, res.num_iterations, corr.cpu().numpy(),
            per)


@pytest.mark.parametrize("kind,cell_scale", CLOUDS)
def test_unsearched_queries_get_the_exhaustive_winner(L, kind, cell_scale):
    """With no iteration run, every query of the evaluation pass is unseeded and takes the slow path: its
    correspondence is the exact nearest target point within r, ties to the lower index."""
    src, tgt, nrm = _cloud(kind)
    row = torch.cuda.get_device_properties(0).multi_processor_count * THREADS
    assert len(src) > 3 * row and len(src) % row != 0
    corr = _run(L, src, tgt, nrm, [], cell_scale)[4]
    want = oracle.hybrid_search(tgt, src, R)[0][:, 0].astype(np.int64)
    assert np.array_equal(corr, want), np.flatnonzero(corr != want)[:10]
    pick = np.random.default_rng(0).choice(len(src), SAMPLE, replace=False)
    brute = oracle.hybrid_search(tgt, src[pick], R, bruteforce=True)[0][:, 0].astype(np.int64)
    assert np.array_equal(corr[pick], brute)
    if kind == "outside":
        assert (corr == -1).mean() > 0.3 and (corr >= 0).mean() > 0.3


def _oracle_loop(src, tgt, nrm, iters, tukey=False, colored=False):
    robust = ("TukeyLoss", 0.05, 1.0) if tukey else ("L2Loss", 1.0, 1.0)
    if colored:
        sc, tc, grad = _colors(src, tgt)
        return oracle.icp_colored(src, sc, tgt, nrm, tc, grad, R, max_iteration=iters, relative_fitness=0,
                                  relative_rmse=0, lambda_geometric=0.968, robust=robust)
    return oracle.icp_p2plane(src, tgt, nrm, R, max_iteration=iters, relative_fitness=0, relative_rmse=0,
                              robust=robust)


TRAJECTORIES = [("standard", 0.0, "l2"), ("standard", 0.0, "tukey"), ("standard", 0.0, "colored"),
                ("cluster", 0.0, "l2"), ("outside", 0.0, "l2"), ("standard", 0.3, "l2")]


@pytest.mark.parametrize("iters", [1, 3, 6])
@pytest.mark.parametrize("kind,cell_scale,est", TRAJECTORIES)
def test_trajectory_vs_oracle_with_far_seeds(L, kind, cell_scale, est, iters):
    """The bars of test_icp_loop_vs_oracle over the first iterations, from a larger misalignment than the default: the
    first update is large, so the seeds of iterations 2 and 3 are farther than r1 from the queries, which then scan the
    pass-1 box instead of the seed's, and the clearances that box gives decide which path they take next."""
    src, tgt, nrm = _cloud(kind, angle_deg=ANGLE)
    tukey, colored = est == "tukey", est == "colored"
    got = _run(L, src, tgt, nrm, [iters], cell_scale, tukey, colored)
    ref = _oracle_loop(src, tgt, nrm, iters, tukey, colored)
    assert got[3] == ref.num_iterations == iters
    per = got[5]
    assert per[0, 0] == ref.per_iteration[0, 0]
    assert abs(per[0, 1] - ref.per_iteration[0, 1]) < 3e-7 * ref.per_iteration[0, 1]
    np.testing.assert_allclose(per[:, 0], ref.per_iteration[:, 0], atol=2e-4)
    np.testing.assert_allclose(per[:, 1], ref.per_iteration[:, 1], atol=2e-6)
    np.testing.assert_allclose(got[0], ref.transformation, atol=2e-5)
    assert abs(got[1] - ref.fitness) < 2e-4 and abs(got[2] - ref.inlier_rmse) < 2e-6
    assert (got[4] == ref.correspondences).mean() > 0.999


@pytest.mark.parametrize("iters", [5, 8])
def test_cluster_cloud_gives_identical_bits(L, iters):
    """On the cluster cloud, whose chunks mix every search path: two registrations, and one launch per
    o3db_icp_iterate call against all launches in one call, give the same bits."""
    src, tgt, nrm = _cloud("cluster", angle_deg=ANGLE)
    runs = [_run(L, src, tgt, nrm, b) for b in ([iters], [iters], [1] * iters, [2, iters - 2])]
    assert runs[0][3] == iters and runs[0][1] > 0.5
    for other in runs[1:]:
        assert runs[0][0].tobytes() == other[0].tobytes()
        assert runs[0][1] == other[1] and runs[0][2] == other[2] and runs[0][3] == other[3]
        assert np.array_equal(runs[0][4], other[4])
        assert runs[0][5].tobytes() == other[5].tobytes()
