"""The CPU oracle of the k-nearest-neighbour search and of its consumers (oracle/knn), checked without a GPU:
against the reference's known answers, against the hybrid-search oracle's brute force, against scipy's KD-tree (an
independent implementation), and its outlier and metrics arithmetic against an f64 numpy restatement."""
import json
import os

import numpy as np
import pytest

import oracle
from oracle import knn as ok
from tests import knn_cases as kc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "knn_kats.json")


def _kats():
    with open(GOLDEN) as f:
        return json.load(f)


def test_knn_search_kat():
    kat = _kats()["knn_search"]
    idx, d2 = ok.knn(kat["dataset_points"], kat["query_points"], kat["knn"])
    np.testing.assert_array_equal(idx, kat["indices"])
    np.testing.assert_allclose(d2, kat["distances"], rtol=kat["rtol"], atol=0)


def test_metrics_kat():
    kat = _kats()["metrics"]
    p1 = np.asarray(kat["box_vertices"], np.float32)
    p2 = p1 * np.float32(kat["scale"])
    got = ok.compute_metrics(p1, p2, [ok.CHAMFER, ok.HAUSDORFF, ok.FSCORE], kat["fscore_radius"])
    np.testing.assert_allclose(got, kat["values"], rtol=kat["rtol"])


@pytest.mark.parametrize("name", ["scan", "lattice", "duplicates", "sparse", "clusters", "line", "external"])
@pytest.mark.parametrize("k", [1, 8, 32])
def test_knn_equals_the_hybrid_bruteforce_at_a_covering_radius(name, k):
    data, queries = kc.cases()[name]
    data, queries = data[:4000], queries[:1500]
    span = np.concatenate([data, queries]).astype(np.float64)
    radius = 2 * float(np.linalg.norm(span.max(0) - span.min(0))) + 1.0
    idx, d2 = ok.knn(data, queries, k)
    hidx, hd2, cnt = oracle.hybrid_search(data, queries, radius, k, bruteforce=True)
    kp = min(k, len(data))
    assert (cnt == kp).all()
    np.testing.assert_array_equal(idx, hidx[:, :kp])
    np.testing.assert_array_equal(d2.view(np.uint32), hd2[:, :kp].view(np.uint32))


@pytest.mark.parametrize("name", ["scan", "uniform", "clusters"])
def test_knn_agrees_with_scipy(name):
    spatial = pytest.importorskip("scipy.spatial")
    data, queries = kc.cases()[name]
    queries = queries[:3000]
    idx, d2 = ok.knn(data, queries, 20)
    dd, ii = spatial.cKDTree(data.astype(np.float64)).query(queries.astype(np.float64), k=20)
    # tie-free random clouds: the same index sets, distances within f32 rounding
    assert (np.sort(idx, 1) == np.sort(ii, 1)).mean() > 0.999
    np.testing.assert_allclose(d2, dd ** 2, rtol=2e-5, atol=1e-6 * float(np.abs(data).max()) ** 2 * 1e-6)


def test_fixed_order_sum_is_the_sum():
    v = np.random.default_rng(1).uniform(0, 1, 300001)
    assert abs(ok.fixed_order_sum(v) - v.sum()) < 1e-9
    assert ok.fixed_order_sum(np.arange(1000, dtype=np.float64)) == 499500.0


@pytest.mark.parametrize("name", ["scan", "uniform", "clusters", "sparse"])
def test_outlier_arithmetic_agrees_with_f64(name):
    data, _ = kc.cases()[name]
    nb, ratio = 20, 2.0
    avg, mask, (mean, std, thr) = ok.remove_statistical_outliers(data, nb, ratio)
    _, d2 = ok.knn(data, data, nb)
    a64 = np.sqrt(d2.astype(np.float64)).mean(1)
    np.testing.assert_allclose(avg, a64, rtol=1e-5)
    m64 = a64.mean()
    s64 = np.sqrt(((a64 - m64) ** 2).sum() / (len(a64) - 1))
    assert abs(mean - m64) <= 1e-6 * m64 and abs(std - s64) <= 1e-5 * s64
    t64 = m64 + ratio * s64
    away = np.abs(a64 - t64) > 1e-4 * t64
    np.testing.assert_array_equal(mask[away], (a64 <= t64)[away])
    assert 0 < (~mask).sum() < len(mask)


def test_outlier_single_point_keeps_nothing():
    avg, mask, (mean, std, thr) = ok.remove_statistical_outliers(np.zeros((1, 3), np.float32), 5, 1.0)
    assert avg[0] == 0 and np.isnan(std) and not mask.any()


@pytest.mark.parametrize("radius", [(0.005,), (0.001, 0.01, 0.05)])
def test_metrics_arithmetic_agrees_with_f64(radius):
    data = kc.cases()["scan"][0]
    other = data[::3] + np.float32(0.003)
    got = ok.compute_metrics(data, other, [ok.FSCORE, ok.CHAMFER, ok.HAUSDORFF], radius)
    _, d12 = ok.knn(other, data, 1)
    _, d21 = ok.knn(data, other, 1)
    s12, s21 = np.sqrt(d12[:, 0].astype(np.float64)), np.sqrt(d21[:, 0].astype(np.float64))
    want = []
    for r in radius:
        p, q = 100 * (s12 < r).mean(), 100 * (s21 < r).mean()
        want.append(0.0 if p + q == 0 else 2 * p * q / (p + q))
    want += [s12.mean() + s21.mean(), max(s12.max(), s21.max())]
    np.testing.assert_allclose(got, want, rtol=2e-5)
