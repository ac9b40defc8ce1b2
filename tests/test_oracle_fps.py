"""The CPU oracle of farthest-point down-sampling (oracle/fps) against upstream's unit-test fixture, a numpy f32
restatement of upstream's tensor loop, and, on integer clouds where every distance is exact, an f64 loop with the legacy
tie rule.  No GPU needed."""
import json
import os

import numpy as np
import pytest

from oracle import fps as of
from tests import fps_cases as fc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fps_kats.json")


def test_oracle_reproduces_upstream_fixture():
    kats = json.load(open(GOLDEN))
    p = np.asarray(kats["points"], np.float32)
    assert len(kats["cases"]) == 2
    for case in kats["cases"]:
        sel = of.farthest_point_down_sample(p, case["num_samples"], case["start_index"])
        np.testing.assert_array_equal(sel, case["selection_order"])
        np.testing.assert_array_equal(p[np.sort(sel)], np.asarray(case["expected"], np.float32))


@pytest.mark.parametrize("name", list(fc.fixtures()))
def test_oracle_equals_numpy_restatement(name):
    p = fc.fixtures()[name]
    n = len(p)
    for m, s in ((1, 0), (min(n, 300), 0), (min(n, 300), n - 1), (min(n, 97), n // 3)):
        np.testing.assert_array_equal(of.farthest_point_down_sample(p, m, s), fc.numpy_fps(p, m, s),
                                      err_msg=f"{name} num_samples={m} start_index={s}")


def test_oracle_on_the_lattice_selects_every_point():
    """The 10 x 10 x 10 lattice is full of equal distances: every round after the first few is decided by ties."""
    p = fc.fixtures()["lattice"]
    sel = of.farthest_point_down_sample(p, len(p), 0)
    np.testing.assert_array_equal(sel, fc.numpy_fps(p, len(p), 0))
    assert len(set(sel.tolist())) == len(p)


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_oracle_equals_f64_legacy_loop_on_integer_clouds(seed):
    p = fc.integer_cloud(3000, seed)
    assert np.abs(p).max() < 1024
    for m, s in ((500, 0), (len(p), len(p) - 1), (64, seed * 7)):
        np.testing.assert_array_equal(of.farthest_point_down_sample(p, m, s), fc.legacy_fps(p, m, s),
                                      err_msg=f"seed={seed} num_samples={m} start_index={s}")


def test_oracle_on_coincident_points_selects_distinct_indices():
    p = fc.coincident()
    distinct = len(np.unique(p, axis=0))
    sel = of.farthest_point_down_sample(p, 100, 5)
    np.testing.assert_array_equal(sel, fc.numpy_fps(p, 100, 5))
    assert len(set(sel.tolist())) == 100
    # once every position is taken, every d is 0: the lowest unselected index comes next
    first = set(sel[:distinct].tolist())
    rest = [j for j in range(len(p)) if j not in first][:100 - distinct]
    np.testing.assert_array_equal(sel[distinct:], rest)


def test_oracle_on_overflowing_distances():
    p = fc.overflow()
    with np.errstate(over="ignore"):
        want = fc.numpy_fps(p, 200, 0)
    np.testing.assert_array_equal(of.farthest_point_down_sample(p, 200, 0), want)


def test_oracle_rejects_bad_arguments():
    p = fc.coincident()
    for m, s in ((0, 0), (len(p) + 1, 0), (3, len(p)), (3, -1)):
        with pytest.raises(ValueError):
            of.farthest_point_down_sample(p, m, s)
