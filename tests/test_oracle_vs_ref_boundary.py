"""The boundary-detection oracle (oracle/boundary) in its libm mode against the reference's own code, compiled from its
headers into oracle/_ref/libo3dref_boundary.so (oracle/ref_shim_boundary): the plane frame of each normal, the gap test
and ComputeBoundaryPointsCPU whole.  Every comparison is bit for bit.  CPU only."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import oracle
from oracle import boundary as ob
from tests import boundary_cases as bc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref", "libo3dref_boundary.so")

_vp = C.c_void_p
THRESHOLDS = (0.0, 45.0, 90.0, 135.0, 180.0, 360.0, -1.0, float("nan"))


@pytest.fixture(scope="module")
def ref():
    if not os.path.exists(REF):
        pytest.skip("oracle/_ref/libo3dref_boundary.so not built (needs the reference sources)")
    L = C.CDLL(REF)
    L.ref_coordinate_system_on_plane_f32.restype = None
    L.ref_coordinate_system_on_plane_f32.argtypes = [_vp, _vp, _vp]
    L.ref_is_boundary_points_f32.restype = C.c_int
    L.ref_is_boundary_points_f32.argtypes = [_vp, C.c_int, C.c_double]
    L.ref_compute_boundary_points_f32.restype = None
    L.ref_compute_boundary_points_f32.argtypes = [_vp, _vp, C.c_int64, _vp, C.c_int64, _vp, _vp, C.c_double]
    return L


@pytest.fixture(scope="module")
def cases():
    return bc.cases()


def _ref_mask(ref, pts, nrm, idx, cnt, thr):
    pts = np.ascontiguousarray(pts, np.float32)
    nrm = np.ascontiguousarray(nrm, np.float32)
    mask = np.zeros(len(pts), np.uint8)
    ref.ref_compute_boundary_points_f32(pts.ctypes.data, nrm.ctypes.data, len(pts), idx.ctypes.data, idx.shape[1],
                                        cnt.ctypes.data, mask.ctypes.data, float(thr))
    return mask.astype(bool)


def _ref_frame(ref, normal):
    nrm = np.ascontiguousarray(normal, np.float32)
    u = np.zeros(3, np.float32)
    v = np.zeros(3, np.float32)
    ref.ref_coordinate_system_on_plane_f32(nrm.ctypes.data, u.ctypes.data, v.ctypes.data)
    return u, v


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", sorted(bc.cases()))
def test_mask_bit_exact(ref, cases, name):
    pts, nrm, radius, max_nn = cases[name]
    idx, _, cnt = oracle.hybrid_search(pts, pts, radius, max_nn)
    for thr in THRESHOLDS:
        got, _ = ob.compute_boundary_points_lists(pts, nrm, idx, cnt, thr, mode="libm")
        want = _ref_mask(ref, pts, nrm, idx, cnt, thr)
        assert np.array_equal(got, want), (name, thr, int(np.count_nonzero(got != want)))


@pytest.mark.parametrize("name", ["special_normals", "normals_scan", "duplicates2"])
def test_frames_bit_exact(ref, cases, name):
    _, nrm, _, _ = cases[name]
    for k in range(0, len(nrm), 7):
        u, v = ob.frame(nrm[k])
        ru, rv = _ref_frame(ref, nrm[k])
        assert np.array_equal(_bits(u), _bits(ru)) and np.array_equal(_bits(v), _bits(rv)), (k, nrm[k])


def test_random_frames_bit_exact(ref):
    for nrm in bc.random_normals():
        u, v = ob.frame(nrm)
        ru, rv = _ref_frame(ref, nrm)
        assert np.array_equal(_bits(u), _bits(ru)) and np.array_equal(_bits(v), _bits(rv)), nrm


def test_gap_test_bit_exact(ref):
    rng = np.random.default_rng(31)
    for trial in range(2000):
        m = 1 + trial % 31
        a = np.sort(rng.uniform(-math.pi, math.pi, m).astype(np.float32))
        if trial % 5 == 0:
            a[:] = np.nan
        for thr in THRESHOLDS:
            got, _ = ob.is_boundary(a, thr)
            want = ref.ref_is_boundary_points_f32(a.ctypes.data, m, float(thr))
            assert got == bool(want), (trial, thr)


def test_nan_frames_and_z_plane(ref, cases):
    """(0, 0, +-1), zero and NaN normals give a NaN frame and a largest gap of 0: never a boundary point at a threshold
    of 0 or more, and, as upstream, always one below 0 when the point has a neighbour."""
    pts, nrm, radius, max_nn = cases["special_normals"]
    idx, _, cnt = oracle.hybrid_search(pts, pts, radius, max_nn)
    bad = np.isnan(nrm).any(1) | (nrm[:, 2] == 1) | (nrm[:, 2] == -1) | ~nrm.any(1)
    assert bad.sum() > 0
    for k in np.flatnonzero(bad)[:20]:
        u, v = ob.frame(nrm[k])
        assert np.isnan(u).any() and np.isnan(v).any()
    for thr in (0.0, 90.0, -1.0):
        mask, gap = ob.compute_boundary_points_lists(pts, nrm, idx, cnt, thr, mode="libm")
        assert (gap[bad] == 0).all()
        assert not mask[bad].any() if thr >= 0 else mask[bad & (cnt > 1)].all()
        assert np.array_equal(mask, _ref_mask(ref, pts, nrm, idx, cnt, thr))


def test_lattice_interior_is_boundary_at_90(ref, cases):
    """On the 4-neighbour lattice every gap is f32(pi/2) > pi/2, in both atan2 modes and in the reference."""
    pts, nrm, radius, max_nn = cases["lattice4"]
    idx, _, cnt = oracle.hybrid_search(pts, pts, radius, max_nn)
    interior = cnt == 5
    assert interior.sum() == 22 * 22
    want = _ref_mask(ref, pts, nrm, idx, cnt, 90.0)
    assert want[interior].all()
    for mode in ("libm", "f64"):
        mask, gap = ob.compute_boundary_points_lists(pts, nrm, idx, cnt, 90.0, mode=mode)
        assert np.array_equal(mask, want)
        assert (gap[interior] == np.float32(math.pi / 2)).all()


def test_coincident_duplicates_keep_the_point_itself(ref, cases):
    pts, nrm, radius, max_nn = cases["duplicates2"]
    idx, _, cnt = oracle.hybrid_search(pts, pts, radius, max_nn)
    odd = np.arange(1, len(pts), 2)
    assert (idx[odd, 0] == odd - 1).all() and (idx[odd, 1:][:, :1] == odd[:, None]).all()
    for thr in (45.0, 90.0):
        got, _ = ob.compute_boundary_points_lists(pts, nrm, idx, cnt, thr, mode="libm")
        assert np.array_equal(got, _ref_mask(ref, pts, nrm, idx, cnt, thr))


def test_single_neighbour_points(ref, cases):
    pts, nrm, radius, max_nn = cases["single"]
    idx, _, cnt = oracle.hybrid_search(pts, pts, radius, max_nn)
    assert (cnt == 2).all()
    for thr in THRESHOLDS:
        got, gap = ob.compute_boundary_points_lists(pts, nrm, idx, cnt, thr, mode="libm")
        assert np.array_equal(got, _ref_mask(ref, pts, nrm, idx, cnt, thr))
        assert (np.abs(gap - 2 * math.pi) < 1e-6).all()
