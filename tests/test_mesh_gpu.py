"""VoxelBlockGrid.extract_triangle_mesh / slam.Model.extract_trianglemesh on the GPU against the CPU oracle
(oracle.mesh.extract_triangle_mesh, itself pinned to the reference's ExtractTriangleMeshCPU and tri_table by
tests/test_oracle_vs_ref_mesh.py) run on the GPU volume's own read-back buffers: all four arrays bit for bit, in the
same order."""
import numpy as np
import pytest
import torch

import oracle.mesh as mesh_oracle
from tests.mesh_cases import KINDS, THRESHOLD, case_histogram, mesh_volume
from tests.test_extract_gpu import VOXEL, _fuse

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


def _oracle_of(vbg, threshold):
    n = vbg.hashmap().size()
    keys = vbg.hashmap().key_tensor()[:n].cpu().numpy()
    tsdf = vbg.attribute("tsdf")[:n].reshape(n, -1).cpu().numpy()
    wt = vbg.attribute("weight")[:n].reshape(n, -1).cpu().numpy()
    col = vbg.attribute("color")[:n].reshape(n, -1, 3).cpu().numpy() if vbg._with_color else None
    return mesh_oracle.extract_triangle_mesh(keys, n, tsdf, wt, col, vbg.block_resolution, vbg.voxel_size, threshold)


def _assert_mesh_equal(mesh, want):
    got = dict(mesh.vertex, indices=mesh.triangle["indices"])
    assert set(got) == set(want), (sorted(got), sorted(want))
    for name, w in want.items():
        g = got[name]
        assert g.is_cuda and tuple(g.shape) == w.shape, (name, tuple(g.shape), w.shape)
        assert g.dtype == (torch.int32 if name == "indices" else torch.float32)
        assert np.array_equal(g.cpu().numpy().view(np.uint32), w.view(np.uint32)), name


def _same(a, b):
    return all(torch.equal(a.vertex[k].view(torch.int32), b.vertex[k].view(torch.int32)) for k in a.vertex) and \
        set(a.vertex) == set(b.vertex) and torch.equal(a.triangle["indices"], b.triangle["indices"])


def _grid_of(o3d, case, R, with_color):
    names = ("tsdf", "weight", "color") if with_color else ("tsdf", "weight")
    vbg = o3d.t.geometry.VoxelBlockGrid(names, (torch.float32, torch.uint16, torch.uint16)[: len(names)],
                                        ((1,), (1,), (3,))[: len(names)], VOXEL, R, 32)
    buf, _ = vbg.hashmap().activate(torch.from_numpy(case["keys"]).cuda())
    idx = buf.long()
    n = len(case["keys"])
    vbg.attribute("tsdf")[idx] = torch.from_numpy(case["tsdf"]).cuda().reshape(n, R, R, R, 1)
    vbg.attribute("weight").view(torch.int16)[idx] = \
        torch.from_numpy(case["weight"].view(np.int16)).cuda().reshape(n, R, R, R, 1)
    if with_color:
        vbg.attribute("color").view(torch.int16)[idx] = \
            torch.from_numpy(case["color"].view(np.int16)).cuda().reshape(n, R, R, R, 3)
    return vbg


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("R", [8, 1])
@pytest.mark.parametrize("with_color", [True, False])
def test_hand_built_volumes(o3d, kind, R, with_color):
    case = mesh_volume(kind, R, with_color)
    vbg = _grid_of(o3d, case, R, with_color)
    got = vbg.extract_triangle_mesh(THRESHOLD)
    want = _oracle_of(vbg, THRESHOLD)
    if kind == "random_signs" and R == 8:
        assert (case_histogram(case, R) > 0).all()   # every case, so the product table is pinned row by row
    _assert_mesh_equal(got, want)


@pytest.fixture(scope="module")
def colour_model(o3d):
    model = o3d.t.pipelines.slam.Model(VOXEL, 16, 6000)
    _fuse(model, range(0, 90, 3))
    first = model.voxel_grid.extract_triangle_mesh(3.0)   # right after the last integrate, no synchronise
    return model, first


def test_colour_model_right_after_integrate(colour_model):
    model, first = colour_model
    want = _oracle_of(model.voxel_grid, 3.0)
    assert len(want["indices"]) > 100000
    _assert_mesh_equal(first, want)


@pytest.mark.parametrize("threshold", [0.0, 3.0, 1e9])
def test_colour_model_thresholds(colour_model, threshold):
    model, _ = colour_model
    got = model.voxel_grid.extract_triangle_mesh(threshold)
    _assert_mesh_equal(got, _oracle_of(model.voxel_grid, threshold))
    assert (got.triangle["indices"].shape[0] == 0) == (threshold > 1e8)


def test_handle_behaviour(colour_model):
    model, _ = colour_model
    vbg = model.voxel_grid
    a = vbg.extract_triangle_mesh()
    b = vbg.extract_triangle_mesh()
    assert _same(a, b) and _same(a, model.extract_trianglemesh())
    nv = int(a.vertex["positions"].shape[0])
    for est in (1, nv - 1, nv, nv + 1, 4 * nv):
        assert _same(a, vbg.extract_triangle_mesh(3.0, est))
        assert _same(a, model.extract_trianglemesh(3.0, est))
    # the point cloud and the mesh keep separate buffers: interleaved calls leave both intact
    pcd = vbg.extract_point_cloud()
    m = vbg.extract_triangle_mesh(0.0)
    pcd2 = vbg.extract_point_cloud(0.0)
    assert torch.equal(pcd.point["positions"], vbg.extract_point_cloud().point["positions"])
    assert _same(m, vbg.extract_triangle_mesh(0.0))
    assert pcd2.point["positions"].shape[0] >= pcd.point["positions"].shape[0]


def test_output_buffers_grow_across_calls(o3d):
    model = o3d.t.pipelines.slam.Model(VOXEL, 16, 8000)
    _fuse(model, range(0, 6, 3))
    small = model.extract_trianglemesh(0.0)   # two frames: every fused voxel has weight 2
    _fuse(model, range(6, 60, 3))
    big = model.extract_trianglemesh(0.0)
    assert big.triangle["indices"].shape[0] > small.triangle["indices"].shape[0] > 0
    _assert_mesh_equal(big, _oracle_of(model.voxel_grid, 0.0))


def test_depth_only_grid(o3d):
    vbg = o3d.t.geometry.VoxelBlockGrid(("tsdf", "weight"), (torch.float32, torch.uint16), ((1,), (1,)), VOXEL, 16,
                                        6000)
    _fuse(vbg, (300, 304, 308, 312), color=False)
    got = vbg.extract_triangle_mesh(3.0)
    assert "colors" not in got.vertex
    _assert_mesh_equal(got, _oracle_of(vbg, 3.0))


def test_resolution_8(o3d):
    model = o3d.t.pipelines.slam.Model(VOXEL, 8, 20000)
    _fuse(model, (500, 504, 508, 512))
    _assert_mesh_equal(model.extract_trianglemesh(0.0), _oracle_of(model.voxel_grid, 0.0))


def test_empty_grid(o3d):
    vbg = o3d.t.geometry.VoxelBlockGrid(voxel_size=VOXEL, block_resolution=16, block_count=100)
    got = vbg.extract_triangle_mesh()
    for name in ("positions", "normals", "colors"):
        assert tuple(got.vertex[name].shape) == (0, 3)
    assert tuple(got.triangle["indices"].shape) == (0, 3) and got.triangle["indices"].dtype == torch.int32


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
            model.extract_trianglemesh()
            per_call.append(_lib.launch_count() - before)
        counts.append(per_call)
    assert counts[0] == counts[1] and max(counts[0]) <= 12, counts


def test_bench_volume(o3d):
    """bench.py's 1000-frame colour volume (profiles/mesh_time.py's workload)."""
    import profiles.extract_time as et
    model = et.build_volume()
    got = model.extract_trianglemesh(3.0)
    want = _oracle_of(model.voxel_grid, 3.0)
    assert len(want["indices"]) > 500000
    _assert_mesh_equal(got, want)
