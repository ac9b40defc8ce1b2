"""RANSAC plane segmentation on the GPU (o3db_segment_plane, PointCloud.segment_plane) against the CPU oracle
(oracle/segment) on the same samples: best hypothesis, evaluated count, fitness and rmse bits, inliers and plane bits.

The oracle equals the reference's own SegmentPlane bit for bit when it sums in upstream's order, and the library's
sampler draws the reference's samples (tests/test_oracle_segment.py)."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import segment as sg
from tests import segment_cases as sc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "segment_plane_kats.json")


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


def _lib():
    from open3d_b200 import _lib
    return _lib


def _stream():
    return int(torch.cuda.current_stream().cuda_stream)


def _samples(n, ransac_n, num_iterations):
    L = _lib()
    out = np.zeros((max(num_iterations, 0), ransac_n), np.int64)
    L.check(L.lib.o3db_random_sample_indices(n, ransac_n, max(num_iterations, 0), out.ctypes.data))
    return out


def _segment(pts_dev, thr, ransac_n, num_iterations, probability):
    """The C ABI call -> (plane, inliers, stats)."""
    L = _lib()
    n = pts_dev.shape[0]
    plane = torch.empty(4, dtype=torch.float64, device="cuda")
    inl = torch.empty(max(n, 1), dtype=torch.int64, device="cuda")
    k = C.c_int64()
    st = L.SegmentStats()
    L.check(L.lib.o3db_segment_plane(pts_dev.data_ptr(), n, thr, ransac_n, num_iterations, probability,
                                     plane.data_ptr(), inl.data_ptr(), C.byref(k), C.byref(st), _stream()))
    return plane.cpu().numpy(), inl[:k.value].cpu().numpy(), st


def _check(o3d, pts, ransac_n, num_iterations, probability=0.999, thr=sc.THRESHOLD, seed=5):
    o3d.utility.random.seed(seed)
    s = _samples(len(pts), ransac_n, num_iterations)
    want = sg.segment_plane(pts, s, thr, probability)
    o3d.utility.random.seed(seed)
    plane, inl, st = _segment(torch.from_numpy(pts).cuda(), thr, ransac_n, num_iterations, probability)
    assert (st.best_index, st.evaluated) == (want.best_index, want.evaluated)
    assert np.float64(st.fitness).tobytes() == np.float64(want.fitness).tobytes()
    assert np.float64(st.inlier_rmse).tobytes() == np.float64(want.rmse).tobytes()
    np.testing.assert_array_equal(inl, want.inliers)
    assert plane.tobytes() == want.plane.tobytes(), (plane, want.plane)
    return want


CLOUDS = {
    "single": lambda: sc.single_plane(30_000, 1),
    "multi": lambda: sc.multi_plane(20_000, 2),
    "noisy": lambda: sc.noisy(50_000, 3),
    "small": lambda: sc.noisy(700, 4),
}


@pytest.mark.parametrize("cloud", sorted(CLOUDS))
@pytest.mark.parametrize("ransac_n,num_iterations,probability",
                         [(3, 1, 0.999), (3, 100, 0.999), (3, 1000, 1.0), (4, 300, 0.999), (10, 200, 0.999),
                          (3, 333, 1.0)])
def test_matches_oracle(o3d, cloud, ransac_n, num_iterations, probability):
    _check(o3d, CLOUDS[cloud](), ransac_n, num_iterations, probability)


def test_early_stop_mid_wave_and_at_a_wave_boundary(o3d):
    pts = sc.single_plane(3000, 5)
    assert 0 < _check(o3d, pts, 3, 300, 0.999, seed=3).evaluated < 128
    assert _check(o3d, pts, 3, 300, sc.wave_boundary_probability(3000), seed=3).evaluated == 128


def test_scene_2m(o3d):
    pts = sc.scene(2_000_000, 7)
    want = _check(o3d, pts, 3, 100)
    assert want.inliers.size > 500_000   # the floor


def test_nan_and_collinear_and_degenerate(o3d):
    pts = sc.noisy(5000, 8)
    pts[::37] = np.nan
    pts[5, 1] = np.nan
    _check(o3d, pts, 3, 200)
    _check(o3d, pts, 4, 200)
    w = _check(o3d, sc.collinear(4000, 9), 3, 150)
    assert w.best_index == -1 and not np.any(w.plane)
    for thr, it in ((0.0, 50), (-1.0, 50), (0.01, 0), (0.01, -4)):
        w = _check(o3d, sc.single_plane(2000, 10), 3, it, thr=thr)
        assert w.best_index == -1 and w.inliers.size == 0


def test_python_call_and_seed(o3d):
    pts = sc.multi_plane(40_000, 11)
    pc = o3d.t.geometry.PointCloud(torch.from_numpy(pts).cuda())
    o3d.utility.random.seed(99)
    plane, inl = pc.segment_plane(0.01, 3, 500)
    o3d.utility.random.seed(99)
    plane2, inl2 = pc.segment_plane(0.01, 3, 500)
    assert plane.dtype == torch.float64 and plane.shape == (4,) and plane.is_cuda
    assert inl.dtype == torch.int64 and inl.is_cuda
    assert torch.equal(plane, plane2) and torch.equal(inl, inl2)
    o3d.utility.random.seed(99)
    want = sg.segment_plane(pts, _samples(len(pts), 3, 500), 0.01, 0.999)
    np.testing.assert_array_equal(inl.cpu().numpy(), want.inliers)
    assert plane.cpu().numpy().tobytes() == want.plane.tobytes()


def test_golden_fixtures(o3d):
    g = json.load(open(GOLDEN))
    pc = o3d.t.geometry.PointCloud(torch.tensor(g["points"], dtype=torch.float32, device="cuda"))
    for case in g["cases"]:
        for seed in range(5):
            o3d.utility.random.seed(seed)
            _, inl = pc.segment_plane(case["distance_threshold"], case["ransac_n"], case["num_iterations"],
                                      case["probability"])
            assert inl.cpu().tolist() == case["inliers"]
    for case in g["errors"]:
        with pytest.raises(RuntimeError, match=case["message"].replace(".", r"\.")):
            pc.segment_plane(case["distance_threshold"], case["ransac_n"], case["num_iterations"],
                             case["probability"])


def test_errors_and_sizes(o3d):
    pc = o3d.t.geometry.PointCloud(torch.from_numpy(sc.single_plane(10, 1)).cuda())
    with pytest.raises(RuntimeError, match=r"ransac_n should be set to higher than or equal to 3\."):
        pc.segment_plane(0.01, 2)
    with pytest.raises(RuntimeError, match=r"There must be at least 'ransac_n' points\."):
        pc.segment_plane(0.01, 11)
    empty = o3d.t.geometry.PointCloud(torch.zeros((0, 3), dtype=torch.float32, device="cuda"))
    with pytest.raises(RuntimeError, match=r"There must be at least 'ransac_n' points\."):
        empty.segment_plane()
    three = o3d.t.geometry.PointCloud(torch.tensor([[0, 0, 0], [1, 0, 0], [0, 1, 0]], dtype=torch.float32,
                                                   device="cuda"))
    plane, inl = three.segment_plane(0.01, 3, 10)
    assert inl.cpu().tolist() == [0, 1, 2] and abs(abs(plane[2].item()) - 1) < 1e-15
    with pytest.raises(RuntimeError, match="Float32"):
        o3d.t.geometry.PointCloud(torch.zeros((10, 3), dtype=torch.float64, device="cuda")).segment_plane()


def test_launch_count_does_not_depend_on_data(o3d):
    L = _lib()
    counts = []
    for pts in (sc.single_plane(20_000, 1), sc.noisy(20_000, 2), sc.collinear(20_000, 3)):
        d = torch.from_numpy(pts).cuda()
        c0 = L.launch_count()
        _segment(d, 0.01, 3, 700, 0.999)
        counts.append(L.launch_count() - c0)
    assert len(set(counts)) == 1, counts


def test_memory_balances_on_success_and_failure(o3d):
    if torch.cuda.get_allocator_backend() == "cudaMallocAsync":
        pytest.skip("torch shares the default memory pool")
    from tests.test_host_ownership_gpu import _Pool
    L = _lib()
    pool = _Pool()
    small = torch.from_numpy(sc.noisy(5000, 1)).cuda()
    big = torch.from_numpy(sc.noisy(300_000, 2)).cuda()
    plane = torch.empty(4, dtype=torch.float64, device="cuda")
    inl = torch.empty(300_000, dtype=torch.int64, device="cuda")
    k = C.c_int64()
    cases = []

    def balanced(name, data, prob, expect=0):
        u0 = pool.used()
        rc = L.lib.o3db_segment_plane(data.data_ptr(), data.shape[0], 0.01, 3, 300, prob, plane.data_ptr(),
                                      inl.data_ptr(), C.byref(k), None, _stream())
        assert rc == expect, (name, rc, L.last_error())
        cases.append((name, u0, pool.used()))

    for _ in range(2):
        balanced("small", small, 0.999)
        balanced("big", big, 1.0)
        balanced("bad probability", small, 2.0, L.ERR_INVALID)
    torch.cuda.synchronize()
    for name, u0, u1 in cases:
        assert u1 == u0, (name, u0, u1)
