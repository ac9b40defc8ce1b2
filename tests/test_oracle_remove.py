"""The CPU oracle of the clean-up filters (oracle/remove) against numpy, brute force and upstream's own unit-test
fixtures (tests/golden/remove_kats.json); no GPU needed.  The GPU tests compare the library with this oracle."""
import json
import os

import numpy as np
import pytest

from oracle import remove as orm
from tests import remove_cases as rc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "remove_kats.json")


def _f32(rows):
    return np.array([[float(v) for v in r] for r in rows], np.float32)


@pytest.fixture(scope="module")
def kats():
    with open(GOLDEN) as f:
        return json.load(f)


def test_kats(kats):
    for k in kats["remove_radius_outliers"]:
        p = _f32(k["positions"])
        for mode in orm.MODES:
            m = orm.remove_radius_outliers(p, k["nb_points"], k["search_radius"], mode)
            assert m.tolist() == k["mask"]
            np.testing.assert_allclose(p[m], _f32(k["expected_positions"]), rtol=1e-5)
    for k in kats["remove_duplicated_points"]:
        p = _f32(k["positions"])
        m = orm.remove_duplicated_points(p)
        assert m.tolist() == k["mask"]
        np.testing.assert_array_equal(p[m], _f32(k["expected_positions"]))
    for k in kats["remove_non_finite_points"]:
        p = _f32(k["positions"])
        for c in k["cases"]:
            m = orm.remove_non_finite_points(p, c["remove_nan"], c["remove_inf"])
            assert m.tolist() == c["mask"], c
            if "expected_positions" in c:
                np.testing.assert_array_equal(p[m], _f32(c["expected_positions"]))


@pytest.mark.parametrize("mode", sorted(orm.MODES))
def test_grid_counts_equal_brute_force(mode):
    rng = np.random.default_rng(1)
    clouds = [rc.nc.scan(4000, seed=2), rc.exact_lattice(8)[0], rc.coincident(), rc.ulp_pairs()[0],
              rng.uniform(-1, 1, (3000, 3)).astype(np.float32) + np.float32(1e4)]
    for p in clouds:
        for r in (1e-3, 0.02, 0.05, 0.5, 0.7, 3.0):
            for cap in (0, 1, 5):
                np.testing.assert_array_equal(orm.radius_counts(p, r, mode, cap),
                                              orm.radius_counts(p, r, mode, cap, brute=True))


def test_exact_lattice_counts_seven_inside():
    p, s = rc.exact_lattice()
    cnt = orm.radius_counts(p, s)
    g = np.round(p / np.float32(s)).astype(int)
    inside = np.all((g > 0) & (g < g.max()), axis=1)
    assert np.all(cnt[inside] == 7) and np.all(cnt[~inside] < 7)
    assert np.all(orm.radius_counts(p, np.nextafter(np.float32(s), np.float32(0))) == 1)


def test_ulp_pairs_tell_the_two_predicates_apart():
    p, r = rc.ulp_pairs()
    cuda = orm.radius_counts(p, r, "cuda")[0::2]
    plain = orm.radius_counts(p, r, "plain")[0::2]
    assert ((cuda == 2) & (plain == 1)).sum() >= 16 and ((cuda == 1) & (plain == 2)).sum() >= 16


def test_coincident_points_count_separately():
    p = rc.coincident()
    _, inv, counts = np.unique(p.view(np.int32).reshape(-1, 3), axis=0, return_inverse=True, return_counts=True)
    np.testing.assert_array_equal(orm.radius_counts(p, 1e-4), counts[inv.ravel()])


def test_nb_points_above_n_keeps_nothing():
    p = rc.nc.scan(2000, seed=3)
    assert not orm.remove_radius_outliers(p, len(p) + 1, 1e3).any()
    assert orm.remove_radius_outliers(p, len(p), 1e3).all()


@pytest.mark.parametrize("name", sorted(rc.duplicate_cases()))
def test_duplicates_are_first_occurrences(name):
    p = rc.duplicate_cases()[name]
    _, first = np.unique(p.view(np.int32).reshape(-1, 3), axis=0, return_index=True)
    want = np.zeros(len(p), bool)
    want[first] = True
    np.testing.assert_array_equal(orm.remove_duplicated_points(p), want)


def test_non_finite_flags_follow_numpy():
    p = rc.non_finite_cloud()
    nan, inf = np.isnan(p).any(1), np.isinf(p).any(1)
    for rn in (False, True):
        for ri in (False, True):
            want = ~((rn & nan) | (ri & inf))
            np.testing.assert_array_equal(orm.remove_non_finite_points(p, rn, ri), want)
    np.testing.assert_array_equal(orm.remove_non_finite_points(p), np.isfinite(p).all(1))
