"""PointCloud.create_from_depth_image / create_from_rgbd_image and project_to_depth_image / project_to_rgbd_image on
the GPU against the CPU oracle (oracle.projection, itself pinned to the reference's UnprojectCPU / ProjectCPU by
tests/test_oracle_vs_ref_projection.py): unprojected rows in the same order and projected images, ties included, bit
for bit.  Also a round trip, an RGB-D -> down-sample -> normals -> ICP chain, determinism, the fixed launch count, empty
inputs and the argument errors."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle
from oracle import projection
from tests import camera_cases as cc
from tests import projection_cases as pc
from tests.synth import PRIMESENSE_K, camera_pose, make_icp_pair, render_depth

pytestmark = pytest.mark.gpu

UNPROJECT = pc.unproject_cases()
PROJECT = pc.project_cases()


@pytest.fixture(scope="module")
def o3d():
    import open3d_b200
    assert torch.cuda.is_available()
    return open3d_b200


def _bits(a):
    if isinstance(a, torch.Tensor):
        a = a.cpu().numpy()
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _unproject(o3d, f: pc.Frame):
    """Depth-only frames go in as an Image of a device tensor, RGB-D frames as an RGBDImage of numpy arrays."""
    G = o3d.t.geometry
    if f.color is None:
        depth = torch.from_numpy(np.ascontiguousarray(f.depth)).cuda()
        return G.PointCloud.create_from_depth_image(G.Image(depth), f.K, f.E, f.scale, f.depth_max, f.stride)
    depth, color = f.depth, f.color
    return G.PointCloud.create_from_rgbd_image(G.RGBDImage(color, depth), f.K, f.E, f.scale, f.depth_max, f.stride)


@pytest.mark.parametrize("name", sorted(UNPROJECT))
def test_unproject_matches_oracle(o3d, name):
    f = UNPROJECT[name]
    want_p, want_c = pc.oracle_unproject(f)
    pcd = _unproject(o3d, f)
    p = pcd.point["positions"]
    assert p.is_cuda and p.dtype == torch.float32 and tuple(p.shape) == want_p.shape
    assert np.array_equal(_bits(p), _bits(want_p))
    if want_c is None:
        assert "colors" not in pcd.point
    else:
        assert np.array_equal(_bits(pcd.point["colors"]), _bits(want_c))


def test_unproject_4096_square_f32(o3d):
    """16.7 M strided pixels: 65 536 tiles, so the tile scan spans many scan blocks."""
    K = cc.intrinsic(2048.0, 2048.0, 2047.5, 2047.5)
    T = camera_pose(100)
    d = render_depth(T, K=K, width=4096, height=4096, device="cuda").cpu().numpy().astype(np.float32)
    E = oracle.inverse_transformation(T)
    pcd = o3d.t.geometry.PointCloud.create_from_depth_image(torch.from_numpy(d).cuda(), K, E)
    want = projection.unproject(d, K, E)
    assert len(want) > 10_000_000
    assert np.array_equal(_bits(pcd.point["positions"]), _bits(want))


def _project(o3d, cl: pc.Cloud, colors=True):
    pcd = o3d.t.geometry.PointCloud(torch.from_numpy(cl.points).cuda())
    if colors:
        pcd.set_point_colors(torch.from_numpy(cl.colors).cuda())
        rgbd = pcd.project_to_rgbd_image(cl.width, cl.height, cl.K, cl.E, cl.scale, cl.depth_max)
        return rgbd.depth.as_tensor(), rgbd.color.as_tensor()
    return pcd.project_to_depth_image(cl.width, cl.height, cl.K, cl.E, cl.scale, cl.depth_max).as_tensor(), None


@pytest.mark.parametrize("colors", [True, False], ids=["rgbd", "depth"])
@pytest.mark.parametrize("name", sorted(PROJECT))
def test_project_matches_oracle(o3d, name, colors):
    cl = PROJECT[name]
    d, c = _project(o3d, cl, colors)
    assert d.is_cuda and d.dtype == torch.float32 and tuple(d.shape) == (cl.height, cl.width, 1)
    if colors:
        want_d, want_c = projection.project(cl.points, cl.K, cl.E, cl.width, cl.height, cl.scale, cl.depth_max,
                                            cl.colors)
        assert tuple(c.shape) == (cl.height, cl.width, 3)
        assert np.array_equal(_bits(c), _bits(want_c))
    else:
        want_d = projection.project(cl.points, cl.K, cl.E, cl.width, cl.height, cl.scale, cl.depth_max)
    assert np.count_nonzero(want_d) > 0
    assert np.array_equal(_bits(d), _bits(want_d))


@pytest.fixture(scope="module")
def cloud_2m():
    _, tgt, _, _ = make_icp_pair(2_000_000, seed=3)
    return pc.Cloud(tgt, pc.indexed_colors(tgt), PRIMESENSE_K, pc._above(tgt, 6.0), depth_max=10.0)


def test_project_2m_points(o3d, cloud_2m):
    cl = cloud_2m
    d, c = _project(o3d, cl)
    want_d, want_c = projection.project(cl.points, cl.K, cl.E, cl.width, cl.height, cl.scale, cl.depth_max, cl.colors)
    assert np.count_nonzero(want_d) > 0.25 * cl.width * cl.height
    assert np.array_equal(_bits(d), _bits(want_d)) and np.array_equal(_bits(c), _bits(want_c))


def test_round_trip(o3d):
    """Unproject at stride 1 under a general pose, project back with the same camera: the same pixels, and each depth
    within 1e-5 relative (the f32 rotation there and back moves it by about 1e-6 at 3 m)."""
    T = camera_pose(130)
    depth, color = render_depth(T, with_color=True)
    E = oracle.inverse_transformation(T)
    G = o3d.t.geometry
    pcd = G.PointCloud.create_from_rgbd_image(G.RGBDImage(color, depth), PRIMESENSE_K, E)
    rgbd = pcd.project_to_rgbd_image(640, 480, PRIMESENSE_K, E)
    d_in = depth.numpy().astype(np.float64)
    valid = (d_in > 0) & (d_in < 3000)
    d_out = rgbd.depth.as_tensor().cpu().numpy()[..., 0].astype(np.float64)
    assert valid.sum() > 200_000
    assert np.array_equal(d_out > 0, valid)
    np.testing.assert_allclose(d_out[valid], d_in[valid], rtol=1e-5, atol=0)
    # every point is the only one at its pixel, so each pixel gets its own colour back (u8 -> 0..255 f32)
    c_out = rgbd.color.as_tensor().cpu().numpy()
    assert np.array_equal(c_out[valid], color.numpy()[valid].astype(np.float32))


def test_rgbd_downsample_normals_icp_chain(o3d):
    """Frames 100 and 110 of the synthetic room (3.6 deg of yaw, 6.3 cm apart), each unprojected in its own camera
    frame.  The same chain run on the CPU oracles (unproject, voxel_down_sample, estimate_normals, icp_p2plane) lands
    within 0.0031 deg and 0.22 mm of the true motion; the residual comes from the 1 mm depth quantisation.  The GPU's
    normals may differ from the oracle's in the last bits on about 2 % of rows (tests/test_normals_gpu.py), so the
    bound is 16x that: 0.05 deg and 2 mm, while the initial error is 3.6 deg and 63 mm."""
    G, reg = o3d.t.geometry, o3d.t.pipelines.registration

    def cloud(i):
        depth, color = (t.cuda() for t in render_depth(camera_pose(i), with_color=True))
        return G.PointCloud.create_from_rgbd_image(G.RGBDImage(color, depth), PRIMESENSE_K)

    src = cloud(110).voxel_down_sample(0.02)
    tgt = cloud(100).voxel_down_sample(0.02).estimate_normals(30, 0.08)
    res = reg.icp(src, tgt, 0.1, np.eye(4), reg.TransformationEstimationPointToPlane(),
                  reg.ICPConvergenceCriteria(0, 0, 50))
    T_true = np.linalg.inv(camera_pose(100)) @ camera_pose(110)
    D = np.linalg.inv(T_true) @ np.asarray(res.transformation)
    angle = np.degrees(np.arccos(np.clip((np.trace(D[:3, :3]) - 1) / 2, -1, 1)))
    assert angle < 0.05 and np.linalg.norm(D[:3, 3]) < 2e-3, (angle, np.linalg.norm(D[:3, 3]))
    assert res.fitness > 0.95


def test_two_calls_give_identical_bits(o3d, cloud_2m):
    f = UNPROJECT["hd_stride1"]
    a, b = _unproject(o3d, f), _unproject(o3d, f)
    for k in ("positions", "colors"):
        assert np.array_equal(_bits(a.point[k]), _bits(b.point[k]))
    d1, c1 = _project(o3d, cloud_2m)
    d2, c2 = _project(o3d, cloud_2m)
    assert torch.equal(d1.view(torch.int32), d2.view(torch.int32)) and torch.equal(c1.view(torch.int32),
                                                                                    c2.view(torch.int32))


def test_launch_count_is_fixed(o3d, cloud_2m):
    from open3d_b200 import _lib
    G = o3d.t.geometry
    counts = set()
    for w, h in ((640, 480), (333, 251), (1280, 720)):
        depth, color = (t.cuda() for t in render_depth(camera_pose(100), K=cc.scaled_k(PRIMESENSE_K, w / 640), width=w,
                                                        height=h, with_color=True))
        for stride in (1, 2, 7, 1000):
            for d in (depth, torch.zeros((h, w), dtype=torch.uint16, device="cuda")):   # a frame, an all-invalid one
                n0 = _lib.launch_count()
                G.PointCloud.create_from_rgbd_image(G.RGBDImage(color, d), PRIMESENSE_K, stride=stride)
                counts.add(("unproject", _lib.launch_count() - n0))
    assert counts == {("unproject", 5)}, counts
    counts = set()
    pts = torch.from_numpy(cloud_2m.points).cuda()
    cols = torch.from_numpy(cloud_2m.colors).cuda()
    K, E = np.ascontiguousarray(cloud_2m.K, np.float64), np.ascontiguousarray(cloud_2m.E, np.float64)
    for n in (0, 1000, len(pts)):
        for w, h in ((640, 480), (1280, 720), (0, 0)):
            depth = torch.empty((max(h, 1), max(w, 1)), dtype=torch.float32, device="cuda")
            color = torch.empty((max(h, 1), max(w, 1), 3), dtype=torch.float32, device="cuda")
            n0 = _lib.launch_count()
            _lib.check(_lib.lib.o3db_project(pts.data_ptr(), cols.data_ptr(), n, _lib.dptr(K), _lib.dptr(E), 1000.0,
                                             10.0, h, w, depth.data_ptr(), color.data_ptr(), None))
            counts.add(("project", _lib.launch_count() - n0))
    torch.cuda.synchronize()
    assert counts == {("project", 2)}, counts


def test_empty_inputs(o3d):
    G = o3d.t.geometry
    zeros = torch.zeros((480, 640), dtype=torch.uint16, device="cuda")
    pcd = G.PointCloud.create_from_depth_image(zeros, PRIMESENSE_K)
    assert tuple(pcd.point["positions"].shape) == (0, 3) and "colors" not in pcd.point
    col = torch.zeros((480, 640, 3), dtype=torch.uint8, device="cuda")
    pcd = G.PointCloud.create_from_rgbd_image(G.RGBDImage(col, zeros), PRIMESENSE_K)
    assert tuple(pcd.point["positions"].shape) == (0, 3) and tuple(pcd.point["colors"].shape) == (0, 3)
    # a stride larger than the image: an empty strided grid
    pcd = G.PointCloud.create_from_depth_image(np.full((480, 640), 1000, np.uint16), PRIMESENSE_K, stride=641)
    assert tuple(pcd.point["positions"].shape) == (0, 3)
    empty = G.PointCloud(torch.zeros((0, 3), dtype=torch.float32, device="cuda"))
    img = empty.project_to_depth_image(640, 480, PRIMESENSE_K)
    assert img.rows == 0 and img.columns == 0
    rgbd = empty.project_to_rgbd_image(640, 480, PRIMESENSE_K)
    assert rgbd.depth.rows == 0 and rgbd.color.rows == 0
    # points that all miss the image: zeros everywhere
    far = G.PointCloud(torch.tensor([[0.0, 0.0, -1.0], [100.0, 0.0, 1.0]], device="cuda")).set_point_colors(
        torch.ones((2, 3), device="cuda"))
    rgbd = far.project_to_rgbd_image(64, 48, PRIMESENSE_K)
    assert not rgbd.depth.as_tensor().any() and not rgbd.color.as_tensor().any()


def test_argument_errors(o3d):
    from open3d_b200 import _lib
    G = o3d.t.geometry
    depth, color = (t.cuda() for t in render_depth(camera_pose(0), with_color=True))
    with pytest.raises(RuntimeError, match="estimate_normals"):
        G.PointCloud.create_from_depth_image(depth, PRIMESENSE_K, with_normals=True)
    with pytest.raises(RuntimeError, match="estimate_normals"):
        G.PointCloud.create_from_rgbd_image(G.RGBDImage(color, depth), PRIMESENSE_K, with_normals=True)
    with pytest.raises(RuntimeError, match="Depth and color images have different sizes."):
        G.PointCloud.create_from_rgbd_image(G.RGBDImage(color[:-1], depth), PRIMESENSE_K)
    with pytest.raises(RuntimeError, match="stride"):
        G.PointCloud.create_from_depth_image(depth, PRIMESENSE_K, stride=0)
    for scale in (0.0, -1000.0, float("nan"), float("inf")):
        with pytest.raises(RuntimeError, match="depth_scale"):
            G.PointCloud.create_from_depth_image(depth, PRIMESENSE_K, depth_scale=scale)
    pts = G.PointCloud(torch.rand((100, 3), device="cuda"))
    with pytest.raises(RuntimeError, match="Unable to project to RGBD without the Color attribute"):
        pts.project_to_rgbd_image(64, 48, PRIMESENSE_K)
    for scale in (0.0, float("nan")):
        with pytest.raises(RuntimeError, match="depth_scale"):
            pts.project_to_depth_image(64, 48, PRIMESENSE_K, depth_scale=scale)

    # the C ABI's own checks
    K, E = np.ascontiguousarray(PRIMESENSE_K, np.float64), np.eye(4)
    out = torch.empty((480 * 640, 3), dtype=torch.float32, device="cuda")
    n = C.c_int64(0)

    def unproject(**kw):
        a = dict(depth=depth.data_ptr(), dt=_lib.DEPTH_U16, rows=480, cols=640, color=color.data_ptr(),
                 ct=_lib.COLOR_U8, scale=1000.0, stride=1, points=out.data_ptr(), colors=out.data_ptr())
        a.update(kw)
        return _lib.lib.o3db_unproject(a["depth"], a["dt"], a["rows"], a["cols"], a["color"], a["ct"], _lib.dptr(K),
                                       _lib.dptr(E), a["scale"], 3.0, a["stride"], a["points"], a["colors"],
                                       C.byref(n), None)

    assert unproject() == _lib.OK and n.value > 0
    for kw in (dict(depth=None), dict(points=None), dict(colors=None), dict(rows=-1), dict(cols=-5), dict(stride=0),
               dict(stride=-3), dict(scale=0.0), dict(scale=float("inf")), dict(ct=_lib.COLOR_NONE), dict(ct=7),
               dict(dt=2), dict(rows=46341, cols=46341)):
        assert unproject(**kw) == _lib.ERR_INVALID, kw
    assert _lib.lib.o3db_unproject(depth.data_ptr(), 0, 480, 640, None, 0, None, _lib.dptr(E), 1000.0, 3.0, 1,
                                   out.data_ptr(), None, C.byref(n), None) == _lib.ERR_INVALID
    assert _lib.lib.o3db_unproject(depth.data_ptr(), 0, 480, 640, None, 0, _lib.dptr(K), _lib.dptr(E), 1000.0, 3.0, 1,
                                   out.data_ptr(), None, None, None) == _lib.ERR_INVALID

    img = torch.empty((48, 64, 3), dtype=torch.float32, device="cuda")
    p = pts.point["positions"]

    def project(**kw):
        a = dict(points=p.data_ptr(), colors=out.data_ptr(), n=100, scale=1000.0, rows=48, cols=64,
                 depth=img.data_ptr(), color=img.data_ptr())
        a.update(kw)
        return _lib.lib.o3db_project(a["points"], a["colors"], a["n"], _lib.dptr(K), _lib.dptr(E), a["scale"], 3.0,
                                     a["rows"], a["cols"], a["depth"], a["color"], None)

    assert project() == _lib.OK
    for kw in (dict(points=None), dict(depth=None), dict(color=None), dict(colors=None), dict(n=-1), dict(n=1 << 31),
               dict(rows=-1), dict(cols=-1), dict(scale=-1.0), dict(scale=float("inf"))):
        assert project(**kw) == _lib.ERR_INVALID, kw
    torch.cuda.synchronize()
