"""The oracle's point-cloud extraction against the reference's OWN ExtractPointCloudCPU<float, uint16_t, uint16_t>
(t/geometry/kernel/VoxelBlockGridImpl.h:1122-1381, compiled unmodified into oracle/_ref/libo3dref_extract.so by
oracle/ref_shim_extract), and the oracle's extraction of a fused room against the room's analytic geometry.
CPU only."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle
import oracle.extract as extract_oracle
from tests.extract_cases import KINDS, THRESHOLD, edge_volume
from tests.synth import PRIMESENSE_K, ROOM_MAX, ROOM_MIN, SPHERE_C, SPHERE_R, camera_pose, render_depth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libo3dref_extract.so")
needs_ref = pytest.mark.skipif(not os.path.exists(REF), reason="oracle/_ref not built (needs the reference sources)")

VOXEL, TRUNC, SCALE, DMAX = 0.008, 8.0, 1000.0, 3.0
vp = C.c_void_p


@pytest.fixture(scope="module")
def ref():
    L = C.CDLL(REF)
    L.ref_extract_point_cloud.restype = C.c_int64
    L.ref_extract_point_cloud.argtypes = [vp, C.c_int64, vp, vp, vp, C.c_int, C.c_float, C.c_float, C.c_int64, vp, vp, vp]
    return L


def fuse_room(frames, R, with_color, cap=6000):
    """The synthetic room fused by the oracle's IntegrateCPU restatement -> (keys, size, tsdf, weight, colour)."""
    keys = np.zeros((cap, 3), np.int32)
    tsdf = np.zeros((cap, R ** 3), np.float32)
    wt = np.zeros((cap, R ** 3), np.uint16)
    col = np.zeros((cap, R ** 3, 3), np.uint16) if with_color else None
    size = 0
    for fid in frames:
        T = camera_pose(fid)
        E = oracle.inverse_transformation(T)
        depth, color = render_depth(T, with_color=True)
        depth, color = depth.numpy(), color.numpy()
        want = oracle.depth_touch(depth, PRIMESENSE_K, E, R, VOXEL, VOXEL * TRUNC, SCALE, DMAX, 4)
        bi, _, size, rc = oracle.hashmap_activate(keys, size, want)
        assert rc == 0
        oracle.tsdf_integrate(depth, color if with_color else None, bi, keys, tsdf, wt, col, PRIMESENSE_K,
                              PRIMESENSE_K, E, R, VOXEL, VOXEL * TRUNC, SCALE, DMAX)
    return keys[:size].copy(), size, tsdf[:size].copy(), wt[:size].copy(), None if col is None else col[:size].copy()


def reference_extract(ref, keys, size, tsdf, weight, color, R, threshold):
    keys, tsdf, weight = (np.ascontiguousarray(a) for a in (keys, tsdf, weight))
    color = None if color is None else np.ascontiguousarray(color)
    args = (keys.ctypes.data, size, tsdf.ctypes.data, weight.ctypes.data, None if color is None else color.ctypes.data,
            R, VOXEL, threshold)
    n = ref.ref_extract_point_cloud(*args, 0, None, None, None)
    out = {"positions": np.zeros((n, 3), np.float32), "normals": np.zeros((n, 3), np.float32)}
    if color is not None:
        out["colors"] = np.zeros((n, 3), np.float32)
    ref.ref_extract_point_cloud(*args, n, out["positions"].ctypes.data, out["normals"].ctypes.data,
                                out["colors"].ctypes.data if color is not None else None)
    return out


def rows(pcd):
    """All columns as one bit-pattern matrix, rows sorted lexicographically (the reference's order is an atomic
    counter's)."""
    cols = [pcd["positions"], pcd["normals"]] + ([pcd["colors"]] if "colors" in pcd else [])
    m = np.concatenate(cols, axis=1).view(np.uint32)
    return m[np.lexsort(m.T[::-1])]


def assert_same_rows(got, want):
    assert set(got) == set(want)
    a, b = rows(got), rows(want)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.array_equal(a, b)


@pytest.fixture(scope="module")
def rooms():
    return {(R, c): fuse_room((200, 203, 206, 209), R, c) for R in (16, 8) for c in (True, False)}


@needs_ref
@pytest.mark.parametrize("R", [16, 8])
@pytest.mark.parametrize("with_color", [True, False])
@pytest.mark.parametrize("threshold", [0.0, 3.0, 1e9])
def test_room_extraction_is_the_reference_extraction(ref, rooms, R, with_color, threshold):
    keys, size, tsdf, wt, col = rooms[(R, with_color)]
    got = extract_oracle.extract_point_cloud(keys, size, tsdf, wt, col, R, VOXEL, threshold)
    want = reference_extract(ref, keys, size, tsdf, wt, col, R, threshold)
    assert_same_rows(got, want)
    n = len(got["positions"])
    assert (n == 0) if threshold > 1e8 else (n > 20000)


@needs_ref
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("R", [8, 4, 1])
@pytest.mark.parametrize("with_color", [True, False])
def test_edge_volume_extraction_is_the_reference_extraction(ref, kind, R, with_color):
    v = edge_volume(kind, R, with_color)
    size = len(v["keys"])
    got = extract_oracle.extract_point_cloud(v["keys"], size, v["tsdf"], v["weight"], v["color"], R, VOXEL, THRESHOLD)
    want = reference_extract(ref, v["keys"], size, v["tsdf"], v["weight"], v["color"], R, THRESHOLD)
    assert_same_rows(got, want)
    if R == 8:
        assert len(got["positions"]) > 0


def test_edge_volumes_exercise_their_edges():
    """Each hand-built case does what its name says, on the oracle alone."""
    R = 8
    face = edge_volume("plane_face", R)
    alone = edge_volume("plane_no_neighbour", R)
    pf = extract_oracle.extract_point_cloud(face["keys"], 3, face["tsdf"], face["weight"], None, R, VOXEL, THRESHOLD)
    pa = extract_oracle.extract_point_cloud(alone["keys"], 2, alone["tsdf"], alone["weight"], None, R, VOXEL, THRESHOLD)
    x_face = R * VOXEL
    # the crossings across the block face exist only with the neighbour block
    assert (np.abs(pf["positions"][:, 0] - x_face) < VOXEL).sum() > 0
    assert (pa["positions"][:, 0] > (R - 1) * VOXEL).sum() == 0
    # with the +x block missing, the x gradient at voxel R-1 is missing, so normals there lose their x component
    edge = pa["positions"][:, 0] > (R - 2) * VOXEL
    assert edge.any() and (pa["normals"][edge, 0] == 0).any()
    # subnormal tsdf_o: the points exist and carry subnormal interpolation ratios
    sub = edge_volume("subnormal", R)
    ps = extract_oracle.extract_point_cloud(sub["keys"], 3, sub["tsdf"], sub["weight"], None, R, VOXEL, THRESHOLD)
    assert len(ps["positions"]) >= 6
    frac = ps["positions"] / VOXEL - np.floor(ps["positions"] / VOXEL + 0.5)
    assert (np.abs(frac) < 1e-30).all()   # a ratio this small leaves a point on its voxel
    # weight == threshold voxels produce nothing, weight == threshold + 1 voxels do
    w = edge_volume("weight_at_threshold", R)
    pw = extract_oracle.extract_point_cloud(w["keys"], 3, w["tsdf"], w["weight"], None, R, VOXEL, THRESHOLD)
    pw0 = extract_oracle.extract_point_cloud(w["keys"], 3, w["tsdf"], w["weight"], None, R, VOXEL, THRESHOLD - 1)
    assert 0 < len(pw["positions"]) < len(pw0["positions"])
    z = edge_volume("zero_tsdf", R)
    pz = extract_oracle.extract_point_cloud(z["keys"], 3, z["tsdf"], z["weight"], None, R, VOXEL, THRESHOLD)
    zf = edge_volume("weight_at_threshold", R)   # the same planes without the zeros
    pzf = extract_oracle.extract_point_cloud(zf["keys"], 3, zf["tsdf"], np.full_like(zf["weight"], 5), None, R, VOXEL, THRESHOLD)
    assert 0 < len(pz["positions"]) < len(pzf["positions"])


def test_oracle_extraction_order_and_cap():
    """A cap keeps the head of the full, deterministic row order and still returns the total."""
    keys, size, tsdf, wt, col = fuse_room((200, 206), 8, True, cap=3000)
    full = extract_oracle.extract_point_cloud(keys, size, tsdf, wt, col, 8, VOXEL, 0.0)
    n = len(full["positions"])
    assert n > 1000
    for cap in (0, 100, n, n + 1000):
        p, q, c = (np.zeros((max(cap, 1), 3), np.float32) for _ in range(3))
        total = extract_oracle.lib().orc_extract_point_cloud(keys.ctypes.data_as(C.POINTER(C.c_int32)), size,
                                                     tsdf.ctypes.data_as(C.POINTER(C.c_float)),
                                                     wt.ctypes.data_as(C.POINTER(C.c_uint16)), col.ctypes.data, 8,
                                                     VOXEL, 0.0, cap, p.ctypes.data, q.ctypes.data, c.ctypes.data)
        k = min(cap, n)
        assert total == n
        assert np.array_equal(p[:k], full["positions"][:k]) and np.array_equal(q[:k], full["normals"][:k])
        assert np.array_equal(c[:k], full["colors"][:k])


@pytest.fixture(scope="module")
def room100():
    keys, size, tsdf, wt, col = fuse_room(range(100), 16, True, cap=8000)
    return extract_oracle.extract_point_cloud(keys, size, tsdf, wt, col, 16, VOXEL, 3.0)


def _room_distances(p):
    lo, hi = np.asarray(ROOM_MIN), np.asarray(ROOM_MAX)
    d_wall = np.minimum(np.abs(p - lo), np.abs(p - hi))   # [n,3]: distance to the two planes of each axis
    d_sphere = np.abs(np.linalg.norm(p - np.asarray(SPHERE_C), axis=1) - SPHERE_R)
    return d_wall, d_sphere


def test_room_geometry(room100):
    """Points of a 100-frame fused room lie on the analytic surfaces and their normals point into the free space.
    The bounds are the values observed on this volume (in the comments) with a margin."""
    p, nrm = room100["positions"].astype(np.float64), room100["normals"].astype(np.float64)
    assert len(p) > 120000                                   # observed 143377 from 1319 blocks
    d_wall, d_sphere = _room_distances(p)
    on_sphere = d_sphere < 0.02                              # the same 22769 points at 0.01, 0.02 and 0.05
    wall_axis = d_wall.argmin(axis=1)
    on_wall = ~on_sphere
    assert on_sphere.sum() > 20000
    assert d_sphere[on_sphere].max() < 0.008                 # observed 0.0055
    assert d_wall[on_wall, wall_axis[on_wall]].max() < 0.006   # observed 0.0032
    # unit length up to the + 1e-5 guard of the normalisation
    assert np.abs(np.linalg.norm(nrm, axis=1) - 1).max() < 2e-4   # observed 8.5e-5
    # away from the sphere centre; towards the room's centre along the nearest wall's axis.  The minima come from
    # the sphere's silhouette and the room's corners, where the gradient mixes two surfaces.
    out = (p[on_sphere] - SPHERE_C) / np.linalg.norm(p[on_sphere] - SPHERE_C, axis=1, keepdims=True)
    dot_s = np.einsum("ij,ij->i", nrm[on_sphere], out)
    assert dot_s.min() > 0.3 and np.percentile(dot_s, 1) > 0.6          # observed 0.458 and 0.763
    centre = (np.asarray(ROOM_MIN) + np.asarray(ROOM_MAX)) / 2
    iw = np.nonzero(on_wall)[0]
    ax = wall_axis[iw]
    dot_w = nrm[iw, ax] * np.sign(centre[ax] - p[iw, ax])
    assert dot_w.min() > 0.25 and np.percentile(dot_w, 1) > 0.95        # observed 0.412 and 0.991
