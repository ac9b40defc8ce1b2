"""VoxelBlockGrid.extract_point_cloud / slam.Model.extract_pointcloud on the GPU against the CPU oracle
(oracle.extract.extract_point_cloud, itself pinned to the reference's ExtractPointCloudCPU by
tests/test_oracle_vs_ref_extract.py) run on the GPU volume's own read-back buffers: every row bit for bit, in the
same order."""
import numpy as np
import pytest
import torch

import oracle
import oracle.extract as extract_oracle
from tests.extract_cases import KINDS, THRESHOLD, edge_volume
from tests.synth import PRIMESENSE_K, camera_pose, render_depth

pytestmark = pytest.mark.gpu

VOXEL, TRUNC_MULT, SCALE, DMAX = 0.008, 8.0, 1000.0, 3.0


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


def _fuse(model_or_grid, frames, color=True):
    """Integrates frames of the synthetic room through the fused path (slam.Model.integrate or
    VoxelBlockGrid.integrate_frame) without synchronising."""
    from open3d_b200.t.pipelines import slam
    for n, fid in enumerate(frames):
        T = camera_pose(fid)
        depth, col = (t.cuda() for t in render_depth(T, with_color=True))
        if isinstance(model_or_grid, slam.Model):
            frame = slam.Frame(480, 640, PRIMESENSE_K)
            frame.set_data("depth", depth)
            if color:
                frame.set_data("color", col)
            model_or_grid.update_frame_pose(n, T)
            model_or_grid.integrate(frame, SCALE, DMAX, TRUNC_MULT)
        else:
            model_or_grid.integrate_frame(depth, col if color else None, PRIMESENSE_K, oracle.inverse_transformation(T),
                                          SCALE, DMAX, TRUNC_MULT)


def _oracle_of(vbg, threshold):
    """The oracle's extraction on the grid's buffers, slots 0..size-1 in the grid's own slot order."""
    n = vbg.hashmap().size()
    keys = vbg.hashmap().key_tensor()[:n].cpu().numpy()
    tsdf = vbg.attribute("tsdf")[:n].reshape(n, -1).cpu().numpy()
    wt = vbg.attribute("weight")[:n].reshape(n, -1).cpu().numpy()
    col = vbg.attribute("color")[:n].reshape(n, -1, 3).cpu().numpy() if vbg._with_color else None
    return extract_oracle.extract_point_cloud(keys, n, tsdf, wt, col, vbg.block_resolution, vbg.voxel_size, threshold)


def _assert_rows_equal(pcd, want):
    assert set(pcd.point) == set(want), (sorted(pcd.point), sorted(want))
    for name, w in want.items():
        g = pcd.point[name]
        assert g.dtype == torch.float32 and g.is_cuda and tuple(g.shape) == w.shape, (name, tuple(g.shape), w.shape)
        assert np.array_equal(g.cpu().numpy().view(np.uint32), w.view(np.uint32)), name


@pytest.fixture(scope="module")
def colour_model(o3d):
    model = o3d.t.pipelines.slam.Model(VOXEL, 16, 6000)
    _fuse(model, range(0, 90, 3))                       # 30 frames
    first = model.voxel_grid.extract_point_cloud(3.0)    # right after the last integrate, no synchronise
    return model, first


def test_colour_model_right_after_integrate(colour_model):
    model, first = colour_model
    want = _oracle_of(model.voxel_grid, 3.0)
    assert len(want["positions"]) > 100000
    _assert_rows_equal(first, want)


@pytest.mark.parametrize("threshold", [-1.0, 0.0, 3.0, 1e9])
def test_colour_model_thresholds(colour_model, threshold):
    model, _ = colour_model
    got = model.voxel_grid.extract_point_cloud(threshold)
    want = _oracle_of(model.voxel_grid, threshold)
    _assert_rows_equal(got, want)
    assert (len(want["positions"]) == 0) == (threshold > 1e8)


def test_two_calls_are_bit_identical_and_model_forwards(colour_model):
    model, _ = colour_model
    a = model.voxel_grid.extract_point_cloud()
    b = model.voxel_grid.extract_point_cloud()
    c = model.extract_pointcloud()
    for name in ("positions", "normals", "colors"):
        assert torch.equal(a.point[name].view(torch.int32), b.point[name].view(torch.int32))
        assert torch.equal(a.point[name].view(torch.int32), c.point[name].view(torch.int32))
    d = model.extract_pointcloud(0.0, 1000)
    assert torch.equal(d.point["normals"], model.voxel_grid.extract_point_cloud(0.0, 1000).point["normals"])


def test_estimated_point_number_keeps_the_head(colour_model):
    model, _ = colour_model
    full = model.voxel_grid.extract_point_cloud(3.0)
    total = int(full.point["positions"].shape[0])
    for cap in (0, 100, total, total + 1000):
        got = model.voxel_grid.extract_point_cloud(3.0, cap)
        k = min(cap, total)
        for name in ("positions", "normals", "colors"):
            assert tuple(got.point[name].shape) == (k, 3)
            assert torch.equal(got.point[name], full.point[name][:k])


def test_depth_only_grid(o3d):
    vbg = o3d.t.geometry.VoxelBlockGrid(("tsdf", "weight"), (torch.float32, torch.uint16), ((1,), (1,)), VOXEL, 16,
                                        6000)
    _fuse(vbg, (300, 304, 308, 312), color=False)
    got = vbg.extract_point_cloud(3.0)
    want = _oracle_of(vbg, 3.0)
    assert "colors" not in got.point and len(want["positions"]) > 20000
    _assert_rows_equal(got, want)


@pytest.mark.parametrize("threshold", [0.0, 3.0])
def test_resolution_8(o3d, threshold):
    model = o3d.t.pipelines.slam.Model(VOXEL, 8, 20000)
    _fuse(model, (500, 504, 508, 512))
    got = model.extract_pointcloud(threshold)
    want = _oracle_of(model.voxel_grid, threshold)
    assert len(want["positions"]) > 20000
    _assert_rows_equal(got, want)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("R", [8, 1])
@pytest.mark.parametrize("with_color", [True, False])
def test_edge_volumes(o3d, kind, R, with_color):
    """The hand-built volumes of tests/extract_cases.py written through attribute views."""
    case = edge_volume(kind, R, with_color)
    names = ("tsdf", "weight", "color") if with_color else ("tsdf", "weight")
    vbg = o3d.t.geometry.VoxelBlockGrid(names, (torch.float32, torch.uint16, torch.uint16)[: len(names)],
                                        ((1,), (1,), (3,))[: len(names)], VOXEL, R, 8)
    buf, _ = vbg.hashmap().activate(torch.from_numpy(case["keys"]).cuda())
    idx = buf.long()
    n = len(case["keys"])
    vbg.attribute("tsdf")[idx] = torch.from_numpy(case["tsdf"]).cuda().reshape(n, R, R, R, 1)
    vbg.attribute("weight").view(torch.int16)[idx] = \
        torch.from_numpy(case["weight"].view(np.int16)).cuda().reshape(n, R, R, R, 1)
    if with_color:
        vbg.attribute("color").view(torch.int16)[idx] = \
            torch.from_numpy(case["color"].view(np.int16)).cuda().reshape(n, R, R, R, 3)
    got = vbg.extract_point_cloud(THRESHOLD)
    want = _oracle_of(vbg, THRESHOLD)
    if R == 8:
        assert len(want["positions"]) > 0
    _assert_rows_equal(got, want)


def test_empty_grid(o3d):
    vbg = o3d.t.geometry.VoxelBlockGrid(voxel_size=VOXEL, block_resolution=16, block_count=100)
    got = vbg.extract_point_cloud()
    for name in ("positions", "normals", "colors"):
        assert tuple(got.point[name].shape) == (0, 3)


def test_launch_count_does_not_depend_on_the_volume(o3d):
    from open3d_b200 import _lib
    counts = []
    for frames in (range(5), range(0, 120, 2)):
        model = o3d.t.pipelines.slam.Model(VOXEL, 16, 8000)
        _fuse(model, frames)
        torch.cuda.synchronize()
        per_call = []
        for _ in range(2):
            before = _lib.launch_count()
            model.extract_pointcloud()
            per_call.append(_lib.launch_count() - before)
        counts.append(per_call)
    assert counts[0] == counts[1] and max(counts[0]) <= 7, counts
