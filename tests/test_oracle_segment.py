"""The CPU oracle of RANSAC plane segmentation (oracle/segment) and the library's host sampler against the reference's
own SegmentPlane and RandomSampler, compiled unmodified into oracle/_ref/libo3dref_segment.so
(oracle/ref_shim_segment).  No GPU needed.

With the whole cloud as one tile the oracle sums in upstream's order and must equal the reference bit for bit; with
the library's tile it must give the same inliers and a plane within 1e-12."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from oracle import segment as sg
from tests import segment_cases as sc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "segment_plane_kats.json")


@pytest.fixture(scope="module")
def ref():
    if sg.ref() is None:
        pytest.skip("oracle/_ref/libo3dref_segment.so not built (needs the reference sources)")
    return sg


def _library_samples(n, ransac_n, num_iterations):
    from open3d_b200 import _lib as L
    out = np.zeros((num_iterations, ransac_n), np.int64)
    L.check(L.lib.o3db_random_sample_indices(n, ransac_n, num_iterations, out.ctypes.data))
    return out


@pytest.mark.parametrize("seed,n,ransac_n", [(0, 3, 3), (1, 5, 4), (42, 1000, 3), (-7, 10, 10), (2**31 - 1, 2_000_000, 3),
                                             (123, 70_000, 17)])
def test_library_sampler_matches_reference(ref, seed, n, ransac_n):
    import open3d_b200 as o3d
    o3d.utility.random.seed(seed)
    ref.ref_seed(seed)
    for num_iterations in (1, 100, 37):   # consecutive calls continue the same stream
        np.testing.assert_array_equal(_library_samples(n, ransac_n, num_iterations),
                                      ref.ref_samples(n, ransac_n, num_iterations))


CLOUDS = {
    "single": lambda: sc.single_plane(3000, 1),
    "multi": lambda: sc.multi_plane(4000, 2),
    "noisy": lambda: sc.noisy(2500, 3),
    "collinear": lambda: sc.collinear(600, 4),
    "tiles": lambda: sc.noisy(5000, 6),   # several of the library's tiles
}
RUNS = [(3, 100, 0.999), (3, 1000, 1.0), (4, 300, 0.999), (10, 200, 0.999), (3, 1, 0.999), (5, 130, 1.0)]


def _away_from_threshold(points, plane, thr):
    if not np.any(plane):
        return
    p = points.astype(np.float64)
    d = np.abs((plane[0] * p[:, 0] + plane[2] * p[:, 2]) + (plane[1] * p[:, 1] + plane[3]))
    assert np.min(np.abs(d - thr)) > 1e-9 * thr


@pytest.mark.parametrize("cloud", sorted(CLOUDS))
@pytest.mark.parametrize("ransac_n,num_iterations,probability", RUNS)
def test_oracle_matches_reference(ref, cloud, ransac_n, num_iterations, probability):
    pts = CLOUDS[cloud]()
    ref.ref_seed(11)
    r = ref.ref_segment_plane(pts, sc.THRESHOLD, ransac_n, num_iterations, probability)
    ref.ref_seed(11)
    s = ref.ref_samples(len(pts), ransac_n, num_iterations)
    o = sg.segment_plane(pts, s, sc.THRESHOLD, probability, tile=None)
    assert (o.evaluated, o.fitness, o.rmse) == (r.evaluated, r.fitness, r.rmse)
    np.testing.assert_array_equal(o.inliers, r.inliers)
    np.testing.assert_array_equal(o.plane, r.plane)
    t = sg.segment_plane(pts, s, sc.THRESHOLD, probability)
    assert (t.best_index, t.evaluated) == (o.best_index, o.evaluated)
    np.testing.assert_array_equal(t.inliers, o.inliers)
    np.testing.assert_allclose(t.plane, o.plane, rtol=1e-12, atol=1e-12)
    _away_from_threshold(pts, t.plane, sc.THRESHOLD)


def test_early_stop_mid_wave_and_at_a_wave_boundary(ref):
    pts = sc.single_plane(3000, 5)
    ref.ref_seed(3)
    samples = ref.ref_samples(3000, 3, 300)
    mid = sg.segment_plane(pts, samples, sc.THRESHOLD, 0.999, tile=None)
    assert 0 < mid.evaluated < 128
    p = sc.wave_boundary_probability(3000)
    edge = sg.segment_plane(pts, samples, sc.THRESHOLD, p, tile=None)
    assert edge.evaluated == 128
    for prob, want in ((0.999, mid), (p, edge)):
        ref.ref_seed(3)
        r = ref.ref_segment_plane(pts, sc.THRESHOLD, 3, 300, prob)
        assert (r.evaluated, r.fitness, r.rmse) == (want.evaluated, want.fitness, want.rmse)
        np.testing.assert_array_equal(r.inliers, want.inliers)


def test_fitness_one_stops_after_one_hypothesis(ref):
    g = json.load(open(GOLDEN))
    pts = np.array(g["points"], np.float32)
    ref.ref_seed(0)
    s = ref.ref_samples(5, 3, 10)
    o = sg.segment_plane(pts, s, 0.01, 0.999, tile=None)
    assert (o.best_index, o.evaluated, o.fitness) == (0, 1, 1.0)


@pytest.mark.parametrize("thr,num_iterations", [(0.0, 50), (-1.0, 50), (0.01, 0)])
def test_degenerate_results_are_zero(ref, thr, num_iterations):
    pts = sc.single_plane(500, 9)
    ref.ref_seed(1)
    r = ref.ref_segment_plane(pts, thr, 3, num_iterations, 0.999)
    ref.ref_seed(1)
    o = sg.segment_plane(pts, ref.ref_samples(500, 3, num_iterations), thr, 0.999, tile=None)
    for x in (r, o):
        assert not np.any(x.plane) and x.inliers.size == 0
    assert o.best_index == -1 and o.evaluated == r.evaluated


def test_negative_iteration_count(ref):
    """Upstream's reserve(size_t(num_iterations)) throws for a negative count; the library treats it as 0
    (DESIGN.md section 7)."""
    pts = sc.single_plane(500, 9)
    with pytest.raises(RuntimeError, match="reserve"):
        ref.ref_segment_plane(pts, 0.01, 3, -3, 0.999)


def test_golden_fixtures():
    g = json.load(open(GOLDEN))
    pts = np.array(g["points"], np.float32)
    for case in g["cases"]:
        for seed in range(5):
            rng = np.random.default_rng(seed)
            s = np.stack([rng.choice(5, case["ransac_n"], replace=False) for _ in range(case["num_iterations"])])
            o = sg.segment_plane(pts, s, case["distance_threshold"], case["probability"])
            np.testing.assert_array_equal(o.inliers, case["inliers"])


def test_golden_fixtures_on_reference(ref):
    g = json.load(open(GOLDEN))
    pts = np.array(g["points"], np.float32)
    for case in g["cases"]:
        r = ref.ref_segment_plane(pts, case["distance_threshold"], case["ransac_n"], case["num_iterations"],
                                  case["probability"])
        np.testing.assert_array_equal(r.inliers, case["inliers"])
    for case in g["errors"]:
        with pytest.raises(RuntimeError, match=case["message"].replace(".", r"\.")):
            ref.ref_segment_plane(pts, case["distance_threshold"], case["ransac_n"], case["num_iterations"],
                                  case["probability"])
    with pytest.raises(RuntimeError, match="ransac_n should be set to higher than or equal to 3."):
        ref.ref_segment_plane(pts, 0.01, 2, 10, 0.999)
    with pytest.raises(RuntimeError, match="There must be at least 'ransac_n' points."):
        ref.ref_segment_plane(pts, 0.01, 6, 10, 0.999)


def test_library_errors_without_a_device():
    """Argument errors come before any CUDA call, with upstream's messages."""
    from open3d_b200 import _lib as L
    k = C.c_int64()
    plane = np.zeros(4)
    for args, msg in (((0.01, 3, 10, 0.0), "Probability must be > 0 and <= 1.0"),
                      ((0.01, 3, 10, 1.5), "Probability must be > 0 and <= 1.0"),
                      ((0.01, 2, 10, 0.5), "ransac_n should be set to higher than or equal to 3."),
                      ((0.01, 6, 10, 0.5), "There must be at least 'ransac_n' points.")):
        rc = L.lib.o3db_segment_plane(None, 5, *args, plane.ctypes.data, None, C.byref(k), None, None)
        assert rc == L.ERR_INVALID and L.last_error() == msg, (rc, L.last_error())
