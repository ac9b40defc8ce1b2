"""The CPU oracle of RANSAC registration (oracle/ransac) against numpy, and the library's integer draws against
std::uniform_int_distribution<int>; no GPU needed."""
import numpy as np
import pytest

from oracle import ransac as orc
from tests import ransac_cases as rc


def _kabsch(s, t):
    ms, mt = s.mean(0), t.mean(0)
    H = (t - mt).T @ (s - ms) / len(s)
    U, _, Vt = np.linalg.svd(H)
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U) * np.linalg.det(Vt))])
    R = U @ D @ Vt
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, mt - R @ ms
    return T


@pytest.mark.parametrize("rn", [3, 4, 10, 64])
def test_estimate_matches_numpy_kabsch(rn):
    src, tgt, c, _ = rc.pair(500, 400, 0.5, seed=rn)
    rng = np.random.default_rng(rn)
    for _ in range(50):
        pairs = c[rng.choice(len(c), rn, replace=False)]
        s, t = src[pairs[:, 0]].astype(np.float64), tgt[pairs[:, 1]].astype(np.float64)
        if np.linalg.svd((t - t.mean(0)).T @ (s - s.mean(0)), compute_uv=False)[1] < 1e-3:
            continue   # degenerate: the rotation is not unique
        np.testing.assert_allclose(orc.estimate(src, tgt, pairs), _kabsch(s, t), rtol=0, atol=1e-12)


def test_true_pairs_give_the_motion():
    src, tgt, c, T = rc.pair(2000, 1000, 1.0, seed=3)
    draws = np.random.default_rng(0).integers(0, len(c), 3 * 100).astype(np.int32)
    r = orc.ransac(src, tgt, c, draws, 0.02, 3, 100, 0.999)
    np.testing.assert_allclose(r.transformation, T, atol=2e-2)
    # every pair is an inlier: ratio 1 gives est_k = 0, so the first validated hypothesis stops the loop
    assert r.drawn == 1 and r.validated == 1 and r.best_index == 0 and r.fitness > 0.99


@pytest.mark.parametrize("conf", [0.0, 0.5, 0.999, 1.0, float("nan")])
def test_stop_rule(conf):
    src, tgt, c, _ = rc.pair(800, 600, 0.3, seed=11)
    H = 300
    draws = np.random.default_rng(1).integers(0, len(c), 3 * H).astype(np.int32)
    r = orc.ransac(src, tgt, c, draws, 0.02, 3, H, conf)
    if conf == 0.0:
        # log(1 - 0) = 0: the first hypothesis with inliers sets est_k = 0 and stops the loop
        assert r.best_index >= 0 and r.drawn == r.validated == r.best_index + 1
    if conf == 1.0 or np.isnan(conf):
        assert r.drawn == H and r.validated == H


def test_tile_changes_only_rmse_rounding():
    src, tgt, c, _ = rc.pair(3000, 2000, 0.3, seed=5)
    draws = np.random.default_rng(2).integers(0, len(c), 3 * 200).astype(np.int32)
    a = orc.ransac(src, tgt, c, draws, 0.02, 3, 200, 0.999, tile=None)
    b = orc.ransac(src, tgt, c, draws, 0.02, 3, 200, 0.999)
    assert (a.drawn, a.validated, a.best_index, a.fitness) == (b.drawn, b.validated, b.best_index, b.fitness)
    np.testing.assert_array_equal(a.transformation, b.transformation)
    np.testing.assert_array_equal(a.correspondence_set, b.correspondence_set)
    assert abs(a.rmse - b.rmse) <= 1e-12


def test_match_is_strict_at_the_radius():
    """An exact identity estimate and probes at r, one ulp inside and one outside: only the inside ones match."""
    src, tgt, c, expect = rc.radius_probes()
    for draws in ([0, 1, 2, 3], [3, 1, 0, 2]):
        r = orc.ransac(src, tgt, c, np.array(draws, np.int32), rc.RADIUS, 4, 1, 1.0)
        np.testing.assert_array_equal(r.transformation, np.eye(4))
        np.testing.assert_array_equal(r.correspondence_set, expect)


needs_ref = pytest.mark.skipif(orc.ref() is None, reason="oracle/_ref/libo3dref_ransac.so was not built here")


@needs_ref
def test_uniform_ints_equal_the_reference_generator():
    """o3db_random_uniform_ints against the reference's UniformIntGenerator<int> on its own engine, draw for draw,
    including across calls."""
    from open3d_b200 import _lib as L
    for seed, lo, hi in ((0, 0, 9), (1, 0, 2), (42, 0, 999), (7, 0, 2 ** 31 - 2), (3, 5, 5), (11, 3, 17)):
        L.check(L.lib.o3db_random_seed(seed))
        orc.ref_seed(seed)
        for count in (1000, 1, 777):
            out = np.zeros(count, np.int32)
            L.check(L.lib.o3db_random_uniform_ints(lo, hi, count, out.ctypes.data))
            np.testing.assert_array_equal(out, orc.ref_uniform_ints(lo, hi, count))


def test_uniform_ints_errors():
    import ctypes as C
    from open3d_b200 import _lib as L
    with pytest.raises(RuntimeError, match="low must be > 0"):
        L.check(L.lib.o3db_random_uniform_ints(-1, 3, 1, C.c_void_p(0)))
    with pytest.raises(RuntimeError, match="low must be <= high"):
        L.check(L.lib.o3db_random_uniform_ints(4, 3, 1, C.c_void_p(0)))


def _cases():
    """(name, source, target, corres, kwargs) for the reference comparison; small enough for two brute-force runs."""
    out = []
    for ratio in (0.05, 0.3, 1.0):
        for rn in (3, 4, 10):
            src, tgt, c, _ = rc.pair(300, 200, ratio, seed=rn)
            out.append((f"ratio{ratio}_n{rn}", src, tgt, c, dict(max_dist=0.02, ransac_n=rn, max_iteration=150)))
    src, tgt, c, T = rc.pair(300, 200, 0.3, seed=2)
    for conf in (0.0, 0.5, 0.999, 1.0, float("nan")):
        out.append((f"conf{conf}", src, tgt, c, dict(max_dist=0.02, max_iteration=150, confidence=conf)))
    sn = rc.normals(len(src), 2)
    tn = (sn.astype(np.float64) @ T[:3, :3].T).astype(np.float32)
    for name, kw in (("edge", dict(edge=0.9)), ("distance", dict(distance=0.03)), ("normal", dict(normal_angle=0.3)),
                     ("all", dict(edge=0.9, distance=0.03, normal_angle=0.3))):
        out.append((name, src, tgt, c, dict(max_dist=0.02, max_iteration=400, src_normals=sn, tgt_normals=tn, **kw)))
    out.append(("normal_without_normals", src, tgt, c, dict(max_dist=0.02, max_iteration=50, normal_angle=0.3)))
    for name, kw in (("max_iteration_0", dict(max_iteration=0)), ("max_iteration_1", dict(max_iteration=1)),
                     ("distance_0", dict(max_dist=0.0)), ("ransac_n_2", dict(ransac_n=2))):
        out.append((name, src, tgt, c, dict(dict(max_dist=0.02, max_iteration=20), **kw)))
    out.append(("k_below_n", src, tgt, c[:2], dict(max_dist=0.02, max_iteration=20)))
    s6, t6, c6, _ = rc.pair(300, 6, 1.0, seed=5)
    out.append(("repeated_indices", s6, t6, c6, dict(max_dist=0.02, ransac_n=4, max_iteration=100, confidence=1.0)))
    st, tt, ct, _ = rc.ties(300, seed=6)
    out.append(("ties", st, tt, ct, dict(max_dist=0.02, max_iteration=100)))
    sp, tp, cp, _ = rc.radius_probes()
    out.append(("radius_probes", sp, tp, cp, dict(max_dist=rc.RADIUS, ransac_n=4, max_iteration=3, confidence=1.0)))
    return out


CASES = _cases()


@needs_ref
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_reference(case):
    """With one tile for the whole cloud the oracle, on the draws the reference's engine makes, equals the reference's
    compiled RegistrationRANSACBasedOnCorrespondence in every bit: the draws consumed (the engine's next draw after the
    call), the validations, fitness, rmse, T and the correspondence pairs."""
    name, src, tgt, c, kw = case
    kw = dict(kw)
    rn, it, dist = kw.pop("ransac_n", 3), kw.pop("max_iteration"), kw.pop("max_dist")
    conf = kw.pop("confidence", 0.999)
    sn, tn = kw.pop("src_normals", None), kw.pop("tgt_normals", None)
    K = len(c)
    seed = 17
    orc.ref_seed(seed)
    draws = orc.ref_uniform_ints(0, max(K - 1, 0), max(it, 0) * rn + 1)
    orc.ref_seed(seed)
    ref = orc.ref_ransac(src, tgt, c, dist, rn, it, conf, src_normals=sn, tgt_normals=tn, **kw)
    nxt = int(orc.ref_uniform_ints(0, max(K - 1, 0), 1)[0])
    ck = orc.checkers(**kw)
    want = orc.ransac(src, tgt, c, draws, dist, rn, it, conf, ck, sn, tn, tile=None)
    early = rn < 3 or K < rn or dist <= 0
    assert nxt == (draws[0] if early else draws[want.drawn * rn]), "draws consumed differ"
    assert ref.validations == (-1 if early else want.validated)
    assert ref.fitness == want.fitness and ref.rmse == want.rmse, (ref.fitness, want.fitness, ref.rmse, want.rmse)
    np.testing.assert_array_equal(ref.transformation, want.transformation)
    np.testing.assert_array_equal(ref.correspondence_set, want.correspondence_set)
    if name == "normal_without_normals":
        assert ref.warnings > 0
    if name == "radius_probes":
        np.testing.assert_array_equal(want.correspondence_set, rc.radius_probes()[3])
