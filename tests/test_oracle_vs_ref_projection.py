"""The projection oracle (oracle/projection) against the reference's own UnprojectCPU and ProjectCPU, compiled from
its sources into oracle/_ref/libo3dref_projection.so (oracle/ref_shim_projection).  Unprojected rows are compared as
sorted row sets (the reference orders them by an atomic counter), bit for bit.  Projected depth images are compared
bit for bit; colours at every pixel where the two agree on the winning point, and where they do not, the pixel must
be an exact depth tie that the oracle gives to the smaller point index (the CUDA kernel's rule; the reference's CPU
kernel keeps the last writer).  CPU only."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import projection
from tests import projection_cases as pc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libo3dref_projection.so")

_vp = C.c_void_p
UNPROJECT = pc.unproject_cases()
PROJECT = pc.project_cases()


@pytest.fixture(scope="module")
def ref():
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref/libo3dref_projection.so not built (needs the reference sources)")
    L = C.CDLL(REF)
    L.ref_unproject.restype = C.c_int64
    L.ref_unproject.argtypes = [_vp, C.c_int, C.c_int, C.c_int, _vp, _vp, _vp, C.c_float, C.c_float, C.c_int, _vp,
                                _vp]
    L.ref_project.restype = None
    L.ref_project.argtypes = [_vp, _vp, C.c_int64, _vp, _vp, C.c_float, C.c_float, C.c_int, C.c_int, _vp, _vp]
    return L


def _f64(a):
    return np.ascontiguousarray(np.asarray(a, np.float64))


def ref_unproject(L, f: pc.Frame):
    d = np.ascontiguousarray(f.depth)
    rows, cols = d.shape[:2]
    # upstream converts the colour image to Float32 without scaling before the kernel (PointCloud.cpp:1456)
    c = None if f.color is None else np.ascontiguousarray(f.color.astype(np.float32))
    cap = max((rows // f.stride) * (cols // f.stride), 1)
    pts, col = np.zeros((cap, 3), np.float32), np.zeros((cap, 3), np.float32)
    K, E = _f64(f.K), _f64(f.E)
    n = L.ref_unproject(d.ctypes.data, int(d.dtype == np.float32), rows, cols, None if c is None else c.ctypes.data,
                        K.ctypes.data, E.ctypes.data, f.scale, f.depth_max, f.stride, pts.ctypes.data,
                        col.ctypes.data)
    return pts[:n], (col[:n] if c is not None else None)


def ref_project(L, cl: pc.Cloud, with_colors=True):
    p = np.ascontiguousarray(cl.points, np.float32)
    c = np.ascontiguousarray(cl.colors, np.float32)
    depth = np.zeros((cl.height, cl.width, 1), np.float32)
    color = np.zeros((cl.height, cl.width, 3), np.float32)
    K, E = _f64(cl.K), _f64(cl.E)
    L.ref_project(p.ctypes.data, c.ctypes.data if with_colors else None, len(p), K.ctypes.data, E.ctypes.data,
                  cl.scale, cl.depth_max, cl.height, cl.width, depth.ctypes.data,
                  color.ctypes.data if with_colors else None)
    return depth, color


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _sorted_rows(*arrays):
    rows = np.concatenate([_bits(a).reshape(len(a), -1) for a in arrays if a is not None], 1)
    return rows[np.lexsort(rows.T[::-1])]


@pytest.mark.parametrize("name", sorted(UNPROJECT))
def test_unproject_matches_reference(ref, name):
    f = UNPROJECT[name]
    want_p, want_c = ref_unproject(ref, f)
    got_p, got_c = pc.oracle_unproject(f)
    assert got_p.shape == want_p.shape and (got_c is None) == (want_c is None)
    assert np.array_equal(_sorted_rows(got_p, got_c), _sorted_rows(want_p, want_c))
    # the oracle's own order: row-major over the strided grid
    d = np.asarray(f.depth).reshape(f.depth.shape[0], f.depth.shape[1])
    rs, cs = d.shape[0] // f.stride, d.shape[1] // f.stride
    g = d[: rs * f.stride: f.stride, : cs * f.stride: f.stride].astype(np.float32) / np.float32(f.scale)
    valid = (g > 0) & (g < np.float32(f.depth_max))
    assert len(got_p) == int(valid.sum())
    if got_c is not None:
        rows_, cols_ = np.nonzero(valid)
        want = f.color[rows_ * f.stride, cols_ * f.stride].astype(np.float32)
        assert np.array_equal(_bits(got_c), _bits(want))


def test_inline_fixture_values():
    """The reference unit test's expected rows (cpp/tests/t/geometry/PointCloud.cpp:1009-1039), in row-major order."""
    pts, col = pc.oracle_unproject(pc.inline_fixture())
    np.testing.assert_array_equal(pts, np.array([[-0.1, -0.1, 1.0], [-0.1, 0.0, 1.0], [0.0, 0.0, 1.0]], np.float32))
    np.testing.assert_array_equal(col, np.array([[0.0] * 3, [0.1] * 3, [0.3] * 3], np.float32))


def test_depth_max_is_excluded_on_unproject():
    f = UNPROJECT["at_depth_max_u16"]
    pts, _ = pc.oracle_unproject(pc.Frame(f.depth, None, f.K, np.eye(4), f.scale, f.depth_max))
    z = pts[:, 2]
    assert not np.any(z == np.float32(2.0)) and np.any(z == np.float32(1.999)) and z.max() < 2.0


@pytest.mark.parametrize("colors", [True, False], ids=["rgbd", "depth"])
@pytest.mark.parametrize("name", sorted(PROJECT))
def test_project_matches_reference(ref, name, colors):
    cl = PROJECT[name]
    want_d, want_c = ref_project(ref, cl, colors)
    if colors:
        got_d, got_c = projection.project(cl.points, cl.K, cl.E, cl.width, cl.height, cl.scale, cl.depth_max,
                                          cl.colors)
    else:
        got_d = projection.project(cl.points, cl.K, cl.E, cl.width, cl.height, cl.scale, cl.depth_max)
    assert np.array_equal(_bits(got_d), _bits(want_d))
    assert np.count_nonzero(got_d) > 0
    if not colors:
        return
    hit = got_d[..., 0] > 0
    same = got_c[..., 0] == want_c[..., 0]   # channel 0 is the winning point's index
    assert np.array_equal(_bits(got_c[same]), _bits(want_c[same]))
    # elsewhere: the reference kept a later point of the same depth at the same pixel
    gi, wi = got_c[~same][:, 0].astype(np.int64), want_c[~same][:, 0].astype(np.int64)
    assert np.all(hit[~same]) and np.all(gi < wi)


def test_project_rules_on_pixel_edges():
    cl = PROJECT["pixel_edges"]
    d, c = projection.project(cl.points, cl.K, cl.E, cl.width, cl.height, cl.scale, cl.depth_max, cl.colors)
    d = d[..., 0]
    # -0.5 rounds to -1 (rejected), -0.49 to -0 (column / row 0); 0.5 -> 1, 8.5 -> 9, 5.5 -> 6 (outside 6 rows)
    cols_hit = sorted(set(np.nonzero(d[4])[0].tolist()))
    assert cols_hit == [0, 1, 2, 3, 8, 9], cols_hit
    rows_hit = sorted(set(np.nonzero(d[:, 1])[0].tolist()))
    assert rows_hit == [0, 1, 4, 5], rows_hit
    # zc == depth_max is kept, the next float is not
    assert d[2, 5] == np.float32(3.0) * np.float32(1000.0) and d[2, 6] == 0
    # x = 8.5 and x = 9.0 land on the same pixel at the same depth: the smaller index wins
    xs = cl.points[:, 0]
    tie = np.nonzero(((xs == np.float32(8.5)) | (xs == np.float32(9.0))) & (cl.points[:, 1] == np.float32(0.5)))[0]
    assert len(tie) == 2 and c[1, 9, 0] == tie.min()


def test_duplicates_take_the_smallest_index():
    cl = PROJECT["duplicates"]
    d, c = projection.project(cl.points, cl.K, cl.E, cl.width, cl.height, cl.scale, cl.depth_max, cl.colors)
    winners = c[..., 0][d[..., 0] > 0].astype(np.int64)
    # every copy of a winning point is a later index with the same coordinates
    for w in winners[:200]:
        copies = np.nonzero(np.all(cl.points == cl.points[w], axis=1))[0]
        assert len(copies) == 4 and copies.min() == w


def test_nan_inf_and_behind_are_rejected():
    cl = PROJECT["behind_nan_inf"]
    d = projection.project(cl.points, cl.K, cl.E, cl.width, cl.height, cl.scale, cl.depth_max)
    assert np.all(np.isfinite(d)) and np.all(d >= 0) and np.all(d <= cl.depth_max * cl.scale)
    ok = np.isfinite(cl.points).all(1) & (cl.points[:, 2] > 0) & (cl.points[:, 2] <= cl.depth_max)
    assert 0 < np.count_nonzero(d) <= ok.sum()
