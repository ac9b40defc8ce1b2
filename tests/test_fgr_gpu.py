"""Fast Global Registration on the GPU (o3db_registration_fgr, registration.registration_fgr_based_on_*) against the
CPU oracle (oracle/fgr) on the library's own draws: every bit of the result, the counts and the engine's state after
the call; then the global registration pipeline end to end."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import fgr as orc
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
    out = np.zeros(max(count, 1), np.int32)
    if K >= 1 and count > 0:
        L.check(L.lib.o3db_random_uniform_ints(0, K - 1, count, out.ctypes.data))
    return out


def _next_draw(K):
    L = _L()
    out = np.zeros(1, np.int32)
    L.check(L.lib.o3db_random_uniform_ints(0, max(K - 1, 0), 1, out.ctypes.data))
    return int(out[0])


def _copt(opt):
    return _L().FgrOption(*[getattr(opt, f) for f, _ in opt._fields_])


def _fgr(src, tgt, opt, c=None, fs=None, ft=None):
    """The C ABI call on device copies -> (T [4,4], corres [n], stats)."""
    L = _L()
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    s, t = dev(src).reshape(-1, 3), dev(tgt).reshape(-1, 3)
    n, m = s.shape[0], t.shape[0]
    dc = None if c is None else torch.from_numpy(np.ascontiguousarray(c, np.int64).reshape(-1, 2)).cuda()
    dfs, dft = (None, None) if fs is None else (dev(fs), dev(ft))
    out = torch.empty(max(n, 1), dtype=torch.int64, device="cuda")
    T = np.zeros(16)
    st = L.FgrStats()
    L.check(L.lib.o3db_registration_fgr(s.data_ptr(), n, t.data_ptr(), m, None if dc is None else dc.data_ptr(),
                                        0 if dc is None else dc.shape[0], None if dfs is None else dfs.data_ptr(),
                                        None if dft is None else dft.data_ptr(), 0 if fs is None else fs.shape[1],
                                        C.byref(_copt(opt)), T.ctypes.data, out.data_ptr(), C.byref(st),
                                        int(torch.cuda.current_stream().cuda_stream)))
    return T.reshape(4, 4), out[:n].cpu().numpy(), st


def _same(T, corr, st, want):
    assert (st.tuples, st.trials, st.pairs) == (want.tuples, want.trials, len(want.pairs)), \
        ((st.tuples, st.trials, st.pairs), (want.tuples, want.trials, len(want.pairs)))
    assert st.fitness == want.fitness and st.inlier_rmse == want.rmse, (st.fitness, want.fitness, st.inlier_rmse,
                                                                        want.rmse)
    np.testing.assert_array_equal(T, want.transformation)
    np.testing.assert_array_equal(corr, want.correspondence_set)


def _check(src, tgt, c, opt, seed=7):
    """The correspondence call against the oracle on the same draws, and the engine's next draw."""
    K = len(c)
    tuple_draws = opt.tuple_test and K > 2
    draws = _draws(seed, K, 300 * K + 1 if tuple_draws else 0)
    _L().check(_L().lib.o3db_random_seed(seed))
    T, corr, st = _fgr(src, tgt, opt, c=c)
    want = orc.fgr(src, tgt, c, draws, opt)
    assert st.cross == K
    _same(T, corr, st, want)
    if tuple_draws:
        assert _next_draw(K) == draws[3 * want.trials], "the engine is not where one thread leaves it"
    return want


def _check_features(src, tgt, fs, ft, opt, seed=7):
    swapped = bool(opt.tuple_test) and len(src) < len(tgt)
    K = len(orc.mutual_pairs(fs, ft, not swapped))
    tuple_draws = opt.tuple_test and K > 2
    draws = _draws(seed, K, 300 * K + 1 if tuple_draws else 0)
    _L().check(_L().lib.o3db_random_seed(seed))
    T, corr, st = _fgr(src, tgt, opt, fs=fs, ft=ft)
    want, k = orc.fgr_features(src, tgt, fs, ft, draws, opt)
    assert st.cross == k
    _same(T, corr, st, want)
    if tuple_draws:
        assert _next_draw(K) == draws[3 * want.trials], "the engine is not where one thread leaves it"
    return want


def _features(n, seed, dim=33):
    """Integer-valued features: exact squared distances in f32 and f64, so any search finds the same rows."""
    return np.random.default_rng(seed).integers(0, 8, (n, dim)).astype(np.float32)


@pytest.mark.parametrize("ratio", [0.05, 0.3, 1.0])
@pytest.mark.parametrize("kw", [{}, dict(tuple_test=False), dict(use_absolute_scale=True), dict(decrease_mu=True),
                                dict(iteration_number=0), dict(iteration_number=1),
                                dict(maximum_tuple_count=0), dict(maximum_tuple_count=1)],
                         ids=["default", "no_tuple_test", "absolute_scale", "decrease_mu", "iter0", "iter1",
                              "max_tuples0", "max_tuples1"])
def test_correspondence_call(o3d, ratio, kw):
    src, tgt, c, _ = rc.pair(3000, 1500, ratio, seed=5)
    _check(src, tgt, c, orc.option(**dict(dict(maximum_correspondence_distance=0.02), **kw)))


def test_true_pairs_recover_the_motion(o3d):
    src, tgt, c, T = rc.pair(3000, 1500, 0.5, seed=1)
    w = _check(src, tgt, c, orc.option(maximum_correspondence_distance=0.02))
    assert np.abs(w.transformation - T).max() < 5e-3 and w.fitness > 0.9


@pytest.mark.parametrize("case", ["ncorr2", "few_pairs", "duplicates", "all_trials"])
def test_edge_cases(o3d, case):
    src, tgt, c, _ = rc.pair(1000, 400, 0.05, seed=2)
    opt = orc.option(maximum_correspondence_distance=0.02)
    if case == "ncorr2":   # at most 2 pairs: upstream's warning, no draws, no pairs, the centroid translation
        w = _check(src, tgt, c[:2], opt)
        assert w.warned and w.trials == 0 and len(w.pairs) == 0
    elif case == "few_pairs":   # fewer than 10 surviving pairs: the identity before de-normalisation
        w = _check(src, tgt, c[:20], orc.option(maximum_correspondence_distance=0.02, maximum_tuple_count=2))
        assert len(w.pairs) < 10
    elif case == "duplicates":
        _check(src, tgt, np.concatenate([c[:50]] * 4), opt)
    else:   # few pass: every one of the 100 K trials runs
        w = _check(src, tgt, c[:60], opt)
        assert w.trials == 6000 and w.tuples < 1000


def _pass_flags(src, tgt, c, draws, ntrial, scale=0.95):
    """AdvancedMatching's test of each trial, in numpy (the same f64 ops)."""
    d = draws[:3 * ntrial].reshape(-1, 3).astype(np.int64)
    a, b = src.astype(np.float64)[c[d, 0]], tgt.astype(np.float64)[c[d, 1]]

    def lengths(p):
        out = []
        for e in range(3):
            v = p[:, e] - p[:, (e + 1) % 3]
            out.append(np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2]))
        return out
    ok = np.ones(ntrial, bool)
    for li, lj in zip(lengths(a), lengths(b)):
        ok &= (li * scale < lj) & (lj < li / scale)
    return ok


@pytest.mark.parametrize("where", ["mid_batch", "batch_end", "next_batch_start", "later_batch"])
def test_tuple_stop_in_batches(o3d, where):
    """With true pairs almost every trial passes, so maximum_tuple_count pins the stop at a chosen trial: inside the
    first batch, at its last trial, at the first trial of the second and inside the third."""
    src, tgt, c, _ = rc.pair(2000, 500, 1.0, seed=3, noise=0.0005)
    seed = 11
    draws = _draws(seed, len(c), 300 * len(c) + 1)
    ok = _pass_flags(src, tgt, c, draws, 100 * len(c))
    target = {"mid_batch": 5000, "batch_end": orc.BATCH - 1, "next_batch_start": orc.BATCH,
              "later_batch": 2 * orc.BATCH + 777}[where]
    passing = np.nonzero(ok)[0]
    stop = int(passing[passing <= target][-1] if where == "batch_end" else passing[passing >= target][0])
    assert abs(stop - target) < 20
    w = _check(src, tgt, c, orc.option(maximum_correspondence_distance=0.02,
                                       maximum_tuple_count=int(ok[:stop + 1].sum())), seed=seed)
    assert w.trials == stop + 1


@pytest.mark.parametrize("sizes", [(600, 900), (900, 600), (700, 700)], ids=["swapped", "source_larger", "equal"])
@pytest.mark.parametrize("tuple_test", [True, False])
def test_feature_call(o3d, sizes, tuple_test):
    n, m = sizes
    rng = np.random.default_rng(n + m)
    src = rc.cloud(n, 1)
    T = rc.motion()
    tgt_all = (src.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    fs = _features(n, 2, dim=6)
    k = min(n, m)
    tgt = np.concatenate([tgt_all[:k], rc.cloud(m - k, 9)]) if m > k else tgt_all[:m]
    ft = np.concatenate([fs[:k], _features(m - k, 3, dim=6)]) if m > k else fs[:m].copy()
    perm = rng.permutation(m)
    w = _check_features(src, tgt[perm], fs, ft[perm],
                        orc.option(maximum_correspondence_distance=0.02, tuple_test=tuple_test))
    assert len(w.pairs) > 0


def test_pairs_beyond_shared_memory(o3d):
    """tuple_test=False on 20 000 mutual pairs: the optimisation reads its pairs from global memory."""
    n = 20000
    src = rc.cloud(n, 4)
    T = rc.motion()
    tgt = (src.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
    fs = _features(n, 5, dim=8)
    perm = np.random.default_rng(6).permutation(n)
    w = _check_features(src, tgt[perm], fs, fs[perm], orc.option(maximum_correspondence_distance=0.02,
                                                                  tuple_test=False, iteration_number=8))
    assert len(w.pairs) >= 20000 * 0.99


def test_python_equals_c_abi(o3d):
    reg = o3d.t.pipelines.registration
    P = o3d.t.geometry.PointCloud
    src, tgt, c, _ = rc.pair(2000, 1000, 0.3, seed=8)
    opt = reg.FastGlobalRegistrationOption(maximum_correspondence_distance=0.02, decrease_mu=True)
    o3d.utility.random.seed(5)
    r = reg.registration_fgr_based_on_correspondence(P(torch.from_numpy(src).cuda()), P(torch.from_numpy(tgt).cuda()),
                                                     torch.from_numpy(c.astype(np.int32)), opt)
    _L().check(_L().lib.o3db_random_seed(5))
    T, corr, st = _fgr(src, tgt, orc.option(maximum_correspondence_distance=0.02, decrease_mu=True), c=c)
    np.testing.assert_array_equal(r.transformation, T)
    np.testing.assert_array_equal(r.correspondence_set.cpu().numpy(), corr)
    assert (r.fitness, r.inlier_rmse) == (st.fitness, st.inlier_rmse)
    fs, ft = _features(len(src), 1, 5), _features(len(tgt), 1, 5)
    o3d.utility.random.seed(6)
    r = reg.registration_fgr_based_on_feature_matching(P(torch.from_numpy(src).cuda()),
                                                       P(torch.from_numpy(tgt).cuda()), torch.from_numpy(fs),
                                                       torch.from_numpy(ft))
    _L().check(_L().lib.o3db_random_seed(6))
    T, corr, st = _fgr(src, tgt, orc.option(decrease_mu=True), fs=fs, ft=ft)   # no option: upstream's C++ defaults
    np.testing.assert_array_equal(r.transformation, T)
    np.testing.assert_array_equal(r.correspondence_set.cpu().numpy(), corr)


def test_omitted_option_is_the_cpp_default(o3d):
    """Upstream binds option=FastGlobalRegistrationOption() built in C++, where decrease_mu is true; the Python class's
    own default is pybind's False.  A call without option follows the C++ object."""
    reg = o3d.t.pipelines.registration
    P = o3d.t.geometry.PointCloud
    assert reg.FastGlobalRegistrationOption().decrease_mu is False
    src, tgt, c, _ = rc.pair(2000, 1000, 0.3, seed=8)
    s, t = P(torch.from_numpy(src).cuda()), P(torch.from_numpy(tgt).cuda())

    def run(*opt):
        o3d.utility.random.seed(3)
        return reg.registration_fgr_based_on_correspondence(s, t, c, *opt).transformation
    omitted = run()
    np.testing.assert_array_equal(omitted, run(reg.FastGlobalRegistrationOption(decrease_mu=True)))
    assert not np.array_equal(omitted, run(reg.FastGlobalRegistrationOption()))


def test_argument_errors(o3d):
    reg = o3d.t.pipelines.registration
    P = o3d.t.geometry.PointCloud
    src, tgt, c, _ = rc.pair(200, 100, 0.5, seed=1)
    s, t = P(torch.from_numpy(src).cuda()), P(torch.from_numpy(tgt).cuda())
    with pytest.raises(RuntimeError, match="outside"):
        reg.registration_fgr_based_on_correspondence(s, t, torch.tensor([[0, 0], [1, 200]]))
    with pytest.raises(RuntimeError, match="Int32 or Int64"):
        reg.registration_fgr_based_on_correspondence(s, t, torch.zeros((3, 2)))
    bad = src.copy()
    bad[7, 1] = np.nan
    with pytest.raises(RuntimeError, match="non-finite"):
        reg.registration_fgr_based_on_correspondence(P(torch.from_numpy(bad).cuda()), t, c)
    with pytest.raises(RuntimeError, match="rows"):
        reg.registration_fgr_based_on_feature_matching(s, t, torch.zeros((199, 33)), torch.zeros((200, 33)))
    with pytest.raises(RuntimeError, match="dimensions"):
        reg.registration_fgr_based_on_feature_matching(s, t, torch.zeros((200, 33)), torch.zeros((200, 32)))
    with pytest.raises(RuntimeError, match="finite"):
        reg.registration_fgr_based_on_correspondence(
            s, t, c, reg.FastGlobalRegistrationOption(maximum_correspondence_distance=math.inf))
    one = P(torch.zeros((1, 3)).cuda())
    with pytest.raises(RuntimeError, match="Invalid scale_global"):
        reg.registration_fgr_based_on_correspondence(one, one, torch.zeros((1, 2), dtype=torch.int64))
    with pytest.raises(RuntimeError):
        reg.registration_fgr_based_on_correspondence(P(torch.from_numpy(src).double().cuda()), t, c)


def _sorted_cloud(P, pc):
    p = pc.point["positions"].cpu().numpy()
    order = np.lexsort((p[:, 2], p[:, 1], p[:, 0]))
    return P(torch.from_numpy(np.ascontiguousarray(p[order])).cuda())


def test_global_registration_pipeline(o3d):
    """voxel_down_sample -> estimate_normals -> compute_fpfh_feature -> FGR on the feature matches at half a voxel,
    as upstream's tutorial runs it, equal to the oracle; then point-to-plane ICP from its pose, on a partially
    overlapping, noisy copy turned 100 degrees about an oblique axis."""
    reg = o3d.t.pipelines.registration
    P = o3d.t.geometry.PointCloud
    pts = rc.scene(150, 0.02, 1)
    src, tgt, T = rc.overlap_pair(pts, 2)
    voxel = 0.05
    clouds = []
    for p in (src, tgt):
        pc = _sorted_cloud(P, P(torch.from_numpy(p.astype(np.float32)).cuda()).voxel_down_sample(voxel))
        pc.estimate_normals(30, 2 * voxel)
        clouds.append((pc, reg.compute_fpfh_feature(pc, 100, 5 * voxel)))
    (s, fs), (t, ft) = clouds
    opt = reg.FastGlobalRegistrationOption(maximum_correspondence_distance=0.5 * voxel)
    o3d.utility.random.seed(0)
    res = reg.registration_fgr_based_on_feature_matching(s, t, fs, ft, opt)
    sp, tp = s.point["positions"].cpu().numpy(), t.point["positions"].cpu().numpy()
    fsn, ftn = fs.cpu().numpy(), ft.cpu().numpy()
    swapped = len(sp) < len(tp)
    K = len(orc.mutual_pairs(fsn, ftn, not swapped))
    want, _ = orc.fgr_features(sp, tp, fsn, ftn, _draws(0, K, 300 * K), orc.option(
        maximum_correspondence_distance=0.5 * voxel))
    np.testing.assert_array_equal(res.transformation, want.transformation)
    assert (res.fitness, res.inlier_rmse) == (want.fitness, want.rmse)
    G = res.transformation
    ang = math.degrees(math.acos(max(-1.0, min(1.0, (np.trace(G[:3, :3].T @ T[:3, :3]) - 1) / 2))))
    shift = float(np.linalg.norm(G[:3, 3] - T[:3, 3]))
    print(f"fgr: {K} mutual pairs, {want.tuples} tuples, fitness {res.fitness:.4f} rmse {res.inlier_rmse:.5f} "
          f"angle {ang:.3f} deg shift {shift:.4f}")
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
    print(f"icp from fgr: max |T - truth| {err:.2e}; from the identity {err_blind:.2e}")
    assert err < 1e-3 and err_blind > 1e-1, (err, err_blind)
