"""The CPU oracle of Fast Global Registration (oracle/fgr) against the reference's own functions compiled with the
stated Eigen orders (oracle/ref_shim_fgr), and its linear algebra against numpy and scipy; no GPU needed."""
import numpy as np
import pytest

from oracle import fgr as orc
from tests import ransac_cases as rc

needs_ref = pytest.mark.skipif(orc.ref() is None, reason="oracle/_ref/libo3dref_fgr.so was not built here")


def test_ldlt_solve_matches_numpy():
    rng = np.random.default_rng(0)
    for _ in range(200):
        B = rng.normal(size=(6, 6))
        A = B @ B.T + 0.5 * np.eye(6)
        b = rng.normal(size=6)
        x = orc.ldlt_solve(A, b)
        np.testing.assert_allclose(x, np.linalg.solve(A, b), rtol=0, atol=1e-12 * max(1.0, np.abs(x).max()))
        x = orc.ldlt_solve(-A, b)   # FGR solves with -JTJ: negative definite, pivoted on |diagonal|
        np.testing.assert_allclose(x, np.linalg.solve(-A, b), rtol=0, atol=1e-12 * max(1.0, np.abs(x).max()))


def test_ldlt_zero_pivots_give_zero():
    A = np.zeros((6, 6))
    np.testing.assert_array_equal(orc.ldlt_solve(A, np.arange(6.0)), np.zeros(6))
    A = np.diag([2.0, 0.0, 4.0, 0.0, 1.0, 8.0])
    np.testing.assert_array_equal(orc.ldlt_solve(A, np.ones(6)), [0.5, 0.0, 0.25, 0.0, 1.0, 0.125])


def test_vec6_to_mat4_matches_scipy():
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(1)
    for scale in (1e-6, 1e-2, 0.5, 3.0):
        for _ in range(100):
            x = rng.normal(size=6) * scale
            M = orc.vec6_to_mat4(x)
            R = Rotation.from_euler("ZYX", [x[2], x[1], x[0]]).as_matrix()
            np.testing.assert_allclose(M[:3, :3], R, rtol=0, atol=1e-15)
            np.testing.assert_array_equal(M[:3, 3], x[3:])
            np.testing.assert_array_equal(M[3], [0, 0, 0, 1])


def test_inverse_matches_numpy():
    rng = np.random.default_rng(2)
    for _ in range(100):
        M = np.eye(4)
        M[:3, :3] = rc.motion(rng.uniform(0, 180), rng.normal(size=3))[:3, :3]
        M[:3, 3] = rng.normal(size=3) * 10
        np.testing.assert_allclose(orc.inverse4(M), np.linalg.inv(M), rtol=0, atol=1e-13)


def _draws(K, count, seed):
    return np.random.default_rng(seed).integers(0, max(K, 1), max(count, 1)).astype(np.int32)


def test_tile_changes_only_rmse_rounding():
    src, tgt, c, _ = rc.pair(3000, 1500, 0.3, seed=5)
    d = _draws(len(c), 300 * len(c), 3)
    opt = orc.option(maximum_correspondence_distance=0.05)
    a, b = orc.fgr(src, tgt, c, d, opt, tile=None), orc.fgr(src, tgt, c, d, opt)
    assert (a.tuples, a.trials, a.fitness) == (b.tuples, b.trials, b.fitness)
    np.testing.assert_array_equal(a.transformation, b.transformation)
    np.testing.assert_array_equal(a.correspondence_set, b.correspondence_set)
    assert abs(a.rmse - b.rmse) <= 1e-12


def _features(n, seed, dim=33):
    """Integer-valued features: exact squared distances in f32 and f64, so any search finds the same rows."""
    return np.random.default_rng(seed).integers(0, 8, (n, dim)).astype(np.float32)


def _cases():
    """(name, source, target, corres or (fs, ft), option) for the reference comparison."""
    out = []
    base = dict(maximum_correspondence_distance=0.02)
    for ratio in (0.05, 0.3, 1.0):
        src, tgt, c, _ = rc.pair(400, 300, ratio, seed=int(ratio * 100))
        out.append((f"ratio{ratio}", src, tgt, c, orc.option(**base)))
    src, tgt, c, _ = rc.pair(400, 300, 0.3, seed=2)
    for name, kw in (("no_tuple_test", dict(tuple_test=False)), ("absolute_scale", dict(use_absolute_scale=True)),
                     ("decrease_mu", dict(decrease_mu=True)), ("decrease_mu_absolute",
                                                              dict(decrease_mu=True, use_absolute_scale=True)),
                     ("iter0", dict(iteration_number=0)), ("iter1", dict(iteration_number=1)),
                     ("iter64", dict(iteration_number=64)), ("max_tuples_neg", dict(maximum_tuple_count=-3)),
                     ("max_tuples0", dict(maximum_tuple_count=0)), ("max_tuples1", dict(maximum_tuple_count=1)),
                     ("max_tuples_default", {}), ("distance0", dict(maximum_correspondence_distance=0.0))):
        out.append((name, src, tgt, c, orc.option(**dict(base, **kw))))
    out.append(("ncorr2", src, tgt, c[:2], orc.option(**base)))
    out.append(("ncorr0", src, tgt, c[:0], orc.option(**base)))
    out.append(("few_pairs", src, tgt, c[:20], orc.option(**dict(base, maximum_tuple_count=2))))
    out.append(("duplicates", src, tgt, np.concatenate([c[:40]] * 3), orc.option(**base)))
    s5, t5, c5, _ = rc.pair(400, 300, 0.05, seed=9)
    out.append(("all_trials", s5, t5, c5[:40], orc.option(**base)))
    T = rc.motion()
    for name, n, m in (("feature_swapped", 300, 450), ("feature_source_larger", 450, 300), ("feature_equal", 350, 350)):
        for tt in (True, False):
            s = rc.cloud(n, 1)
            t_all = (s.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
            fs = _features(n, 2, 6)
            k = min(n, m)
            t = np.concatenate([t_all[:k], rc.cloud(m - k, 9)]) if m > k else t_all[:m]
            ft = np.concatenate([fs[:k], _features(m - k, 3, 6)]) if m > k else fs[:m].copy()
            perm = np.random.default_rng(n + m).permutation(m)
            out.append((f"{name}_{'tuples' if tt else 'no_tuples'}", s, t[perm], (fs, ft[perm]),
                        orc.option(**dict(base, tuple_test=tt))))
    return out


CASES = _cases()


@needs_ref
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_equals_reference(case):
    """With one tile for the whole cloud the oracle, on the draws the reference's engine makes, equals the reference's
    compiled function in every bit: T, fitness, rmse and the correspondence pairs; the initial pairs, the tuples and
    the trials consumed (the engine's next draw after the call)."""
    name, src, tgt, c, opt = case
    seed = 17
    features = isinstance(c, tuple)
    if features:
        fs, ft = c
        swapped = bool(opt.tuple_test) and len(src) < len(tgt)
        pairs = orc.mutual_pairs(fs, ft, not swapped)
    else:
        pairs, swapped = c, False
    K = len(pairs)
    draws_made = bool(opt.tuple_test) and K > 2
    orc.ref_seed(seed)
    draws = orc.ref_uniform_ints(0, max(K - 1, 0), 300 * K + 1)
    orc.ref_seed(seed)
    ref = orc.ref_fgr(src, tgt, opt, corres=None if features else c, source_feature=fs if features else None,
                      target_feature=ft if features else None)
    nxt = int(orc.ref_uniform_ints(0, max(K - 1, 0), 1)[0])
    want = orc.fgr(src, tgt, pairs, draws, opt, swapped, tile=None)
    assert nxt == draws[3 * want.trials if draws_made else 0], "draws consumed differ"
    if features:
        assert ref.cross == K
    if draws_made:
        assert (ref.tuples, ref.trials) == (want.tuples, want.trials)
    assert ref.warnings == int(want.warned)
    assert ref.fitness == want.fitness and ref.rmse == want.rmse, (ref.fitness, want.fitness, ref.rmse, want.rmse)
    np.testing.assert_array_equal(ref.transformation, want.transformation)
    np.testing.assert_array_equal(ref.correspondence_set, want.correspondence_set)
    if name == "all_trials":
        assert want.trials == 100 * K and want.tuples < 1000
    if name in ("max_tuples_neg", "max_tuples0"):
        assert want.trials == 1
    if name in ("ncorr2", "few_pairs"):
        assert len(want.pairs) < 10   # the identity before de-normalisation: the centroid translation


@needs_ref
def test_reference_raises_on_zero_scale():
    one = np.zeros((1, 3), np.float32)
    with pytest.raises(RuntimeError, match="Invalid scale_global"):
        orc.ref_fgr(one, one, orc.option(), corres=np.zeros((1, 2), np.int64))
    with pytest.raises(RuntimeError, match="Invalid scale_global"):
        orc.fgr(one, one, np.zeros((1, 2), np.int64), np.zeros(1, np.int32))


def _pivot_matrices():
    """6x6 systems for the LDLT: symmetric positive and negative definite ones whose largest diagonal entry moves, so
    that the factorisation swaps rows and columns; ties on the diagonal; zero and all-zero diagonals."""
    rng = np.random.default_rng(7)
    out = []
    for k in range(300):
        B = rng.normal(size=(6, 6))
        A = B @ B.T + rng.uniform(0.01, 1.0) * np.eye(6)
        A *= np.exp(rng.normal(size=6))[:, None] * np.exp(rng.normal(size=6))[None, :] if k % 3 == 0 else 1.0
        A = (A + A.T) / 2
        out.append(-A if k % 2 else A)
    tie = np.eye(6) * 3.0
    tie[5, 0] = tie[0, 5] = 1.1
    tie[3, 2] = tie[2, 3] = -0.7
    out += [tie, np.zeros((6, 6)), np.diag([0.0, 5.0, 0.0, 2.0, 5.0, 1e-320]), np.diag([1e-300, 1, 2, 4, 8, 16])]
    return out


@needs_ref
def test_stub_ldlt_equals_oracle_bit_for_bit():
    """The shim's Eigen stub states the LDLT on its own; on systems that pivot, tie and hit zero pivots its solution
    equals the oracle's (and so the kernel's) in every bit."""
    rng = np.random.default_rng(8)
    swaps = 0
    for A in _pivot_matrices():
        b = rng.normal(size=6)
        got, want = orc.ref_ldlt_solve(A, b), orc.ldlt_solve(A, b)
        np.testing.assert_array_equal(got.view(np.int64), want.view(np.int64))
        swaps += int(np.argmax(np.abs(np.diag(A))) != 0)
    assert swaps > 100


def test_ldlt_pinned_pivot_order():
    """A system that needs a pivot swap at every step: A = P^T L D L^T P with dyadic L (+-1/4 on the first
    subdiagonal, +-1/16 on the second) and
    D = 4 x 16^5 .. 4, so that A's diagonal, in construction order, strictly decreases, and P scatters it.  Eigen pivots
    on the largest |diagonal| of the trailing corner as it stands (the trailing rows' diagonal is updated only when
    their turn comes), so the stated order eliminates in construction order; every intermediate value is then exact
    and the solve returns x exactly."""
    L = np.eye(6) + np.diag([0.25, -0.25, 0.25, 0.25, -0.25], -1) + np.diag([0.0625, -0.0625, 0.0625, 0.0625], -2)
    D = np.diag(4.0 * 16.0 ** np.arange(5, -1, -1))
    perm = np.array([3, 0, 5, 1, 4, 2])
    P = np.eye(6)[perm]
    M = L @ D @ L.T
    assert np.all(np.diff(np.diag(M)) < 0)
    A = P.T @ M @ P
    x = np.array([1.0, -2.0, 3.0, -4.0, 5.0, -6.0])
    b = A @ x
    for sign in (1.0, -1.0):   # FGR solves with -JTJ
        np.testing.assert_array_equal(orc.ldlt_solve(sign * A, sign * b), x)
        if orc.ref() is not None:
            np.testing.assert_array_equal(orc.ref_ldlt_solve(sign * A, sign * b), x)
    # the construction's order really swaps: the largest diagonal entry is not first
    assert int(np.argmax(np.diag(A))) != 0


@needs_ref
def test_stub_inverse_and_rotation_equal_oracle_bit_for_bit():
    rng = np.random.default_rng(9)
    for _ in range(300):
        M = np.eye(4)
        M[:3, :3] = rc.motion(rng.uniform(0, 180), rng.normal(size=3))[:3, :3]
        M[:3, 3] = rng.normal(size=3) * 10
        np.testing.assert_array_equal(orc.ref_inverse4(M), orc.inverse4(M))
        G = rng.normal(size=(4, 4))
        np.testing.assert_array_equal(orc.ref_inverse4(G), orc.inverse4(G))
        x = rng.normal(size=6) * rng.choice([1e-4, 0.1, 1.0, 3.0])
        np.testing.assert_array_equal(orc.ref_vec6_to_mat4(x), orc.vec6_to_mat4(x))


def test_stated_sine_cosine_against_libm():
    """The stated sine and cosine differ from glibc's by at most 1 ulp.  How often they differ depends on the
    argument: about 12 % (sine) and 17 % (cosine) of arguments in [-3.2, 3.2], 0.02 % and 0.1 % in [-0.1, 0.1],
    where FGR's half-angles lie after the first iterations, and none in [-1e-3, 1e-3]."""
    rng = np.random.default_rng(10)
    for lo, hi, limit in ((-3.2, 3.2, (0.2, 0.25)), (-0.1, 0.1, (0.002, 0.005)), (-1e-3, 1e-3, (0.0, 0.0))):
        xs = rng.uniform(lo, hi, 20000)
        for want_cos, f, most in ((0, np.sin, limit[0]), (1, np.cos, limit[1])):
            got = np.array([orc.sincos(x, want_cos) for x in xs])
            ref = f(xs)
            ulps = np.abs(got - ref) / np.spacing(np.abs(ref))
            assert ulps.max() <= 1.0, (lo, hi, want_cos, ulps.max())
            assert (ulps > 0).mean() <= most, (lo, hi, want_cos, (ulps > 0).mean())


@needs_ref
def test_stub_sine_cosine_equal_oracle_bit_for_bit():
    rng = np.random.default_rng(11)
    xs = np.concatenate([rng.uniform(-7, 7, 5000), rng.normal(0, 1e-3, 2000), [0.0, -0.0, np.pi / 4, -np.pi / 2]])
    for x in xs:
        for w in (0, 1):
            a, b = orc.ref_sincos(x, w), orc.sincos(x, w)
            assert np.float64(a).view(np.int64) == np.float64(b).view(np.int64), (x, w, a, b)


def test_pair_buffer_is_bounded_by_the_trials():
    """A huge maximum_tuple_count sizes the oracle's pair list by the 100 K trials, not by the count."""
    src, tgt, c, _ = rc.pair(200, 30, 1.0, seed=4)
    d = _draws(len(c), 300 * len(c), 5)
    r = orc.fgr(src, tgt, c, d, orc.option(maximum_tuple_count=2 ** 31 - 1, iteration_number=1))
    assert r.trials == 100 * len(c) and len(r.pairs) == 3 * r.tuples
